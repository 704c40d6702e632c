"""Shared helpers for the test-suite (oracle side).  Tests are the only importers of oracle/."""
import json
import os

import numpy as np
import torch

from oracle import stylesinger_oracle as O
from stylesinger_b200 import synth
from stylesinger_b200.hparams import DEFAULT_VOCODER_CONFIG, resolve

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
_CACHE = {}


def golden(name):
    g = np.load(os.path.join(GOLDEN, name + ".npz"))
    return g, json.loads(str(g["meta"]))


def hp_for(T, f0_T=None):
    return resolve(timesteps=T, K_step=T, f0_timesteps=T if f0_T is None else f0_T)


def acoustic_sd():
    if "sd" not in _CACHE:
        _CACHE["sd"] = synth.acoustic_state_dict(hp_for(4), seed=0)
    return _CACHE["sd"]


def vocoder_sd():
    if "vsd" not in _CACHE:
        _CACHE["vsd"] = synth.vocoder_state_dict(DEFAULT_VOCODER_CONFIG, seed=0)
    return _CACHE["vsd"]


def utt_from_meta(meta):
    return synth.make_utterance(meta["frames"] / 187.5, utt_idx=meta["utt_idx"], ref_frames=meta["ref_frames"],
                                frames=meta["frames"], phones=meta["phones"])


def utt_from_fixture(g):
    """The inputs a fixture stores as in_* arrays (padded inputs that synth.make_utterance cannot rebuild)."""
    return {k[3:]: torch.from_numpy(np.array(g[k])) for k in g.files if k.startswith("in_")}


def oracle_forward(u, hp, seed, use_mel2ph=True, **kw):
    ns = O.NoiseSource(seed)
    with torch.no_grad():
        r = O.stylesinger_forward(acoustic_sd(), hp, u["txt_tokens"][None], u["note"][None], u["note_dur"][None],
                                  u["note_type"][None], u["spk_embed"][None], u["emo_embed"][None],
                                  u["ref_mels"][None], u["ref_f0"], ns,
                                  mel2ph=u["mel2ph"][None] if use_mel2ph else None, **kw)
    return r, ns


# ---- CUDA-side helpers -----------------------------------------------------------------------------
def engine_noise_from_stream(seed, T_f0, T_mel, F, device):
    """Re-draw the A.10 noise sequence of one B=1 forward from NoiseSource(seed) and lay it out the way
    the C ABI takes injected noise (include/stylesinger_b200.h: ssb_acoustic_inputs)."""
    ns = O.NoiseSource(seed)
    f0g, f0u = [], []
    for _net in range(2):
        ns.rand((1, 1, F))  # UV init draw: consumed, result unused (gaussian_multinomial_diffusion.py:924-926)
        g = [ns.randn((1, 1, F)).reshape(F)]
        u = []
        for _ in range(T_f0):
            g.append(ns.randn((1, 1, F)).reshape(F))
            u.append(ns.rand((1, 2, F))[0].t().contiguous())  # [F,2]
        f0g.append(torch.stack(g).contiguous().to(device))
        f0u.append(torch.stack(u).contiguous().to(device))
    mel = [ns.randn((1, 1, 80, F))[0, 0].t().contiguous()]
    for _ in range(T_mel):
        mel.append(ns.randn((1, 1, 80, F))[0, 0].t().contiguous())
    return {"f0_gauss": f0g, "f0_unif": f0u, "mel": torch.stack(mel).contiguous().to(device)}, ns


def batch_noise(per_utt):
    """Concatenate per-utterance injected noise along the frame axis (tight batch layout)."""
    out = {"f0_gauss": [], "f0_unif": []}
    for i in range(2):
        out["f0_gauss"].append(torch.cat([n["f0_gauss"][i] for n in per_utt], dim=1).contiguous())
        out["f0_unif"].append(torch.cat([n["f0_unif"][i] for n in per_utt], dim=1).contiguous())
    out["mel"] = torch.cat([n["mel"] for n in per_utt], dim=1).contiguous()
    return out


_ENG = {}


def acoustic_engine(T, f0_T=None):
    from stylesinger_b200.engine import AcousticModel
    if "ac" not in _ENG:
        _ENG["ac"] = AcousticModel(acoustic_sd(), hp_for(T, f0_T))
    m = _ENG["ac"]
    m.set_timesteps(T, T if f0_T is None else f0_T)
    return m


def vocoder_engine():
    from stylesinger_b200.engine import Vocoder
    if "voc" not in _ENG:
        _ENG["voc"] = Vocoder(vocoder_sd(), DEFAULT_VOCODER_CONFIG)
    return _ENG["voc"]
