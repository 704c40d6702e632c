"""Shared helpers for the test-suite (oracle side).  Tests are the only importers of oracle/."""
import json
import os

import numpy as np
import torch

from oracle import stylesinger_oracle as O
from stylesinger_b200 import synth
from stylesinger_b200.hparams import DEFAULT_VOCODER_CONFIG, HIFIGAN_V2, HIFIGAN_V3, resolve

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


def acoustic_sd64():
    """acoustic_sd() cast to float64: the oracle functions then run in double precision (the positional table stays fp32,
    as the reference's is)."""
    if "sd64" not in _CACHE:
        _CACHE["sd64"] = {k: (v.double() if v.is_floating_point() else v) for k, v in acoustic_sd().items()}
    return _CACHE["sd64"]


# ---- the model options' fixtures: hparams and synthetic checkpoints (seed 0, cached) --------------------------------
# Each keeps the resolve() arguments tools/make_golden.py generated its fixture with: the checkpoint draws follow them.
def switch_hp(cfg):
    """tests/golden/ref_switches.npz: cfg = {"T": ..., "overrides": {...}} (switches and decoder / f0_gen)."""
    return resolve(timesteps=cfg["T"], K_step=cfg["T"], f0_timesteps=cfg["T"], **cfg["overrides"])


def fft_spkid_hp(cfg):
    """tests/golden/ref_fft_spkid.npz: switch_hp with the opt-in decoder 'fft' and use_spk_id need (extended_models)."""
    return resolve(timesteps=cfg["T"], K_step=cfg["T"], f0_timesteps=cfg["T"], extended_models=True, **cfg["overrides"])


def conv_hp(meta):
    """tests/golden/ref_convf0.npz (meta, or meta['prodiff']): f0_gen 'conv' plus the fixture's overrides."""
    return resolve(timesteps=meta["T"], K_step=meta["T"], **meta["overrides"])


def prodiff_hp(T=None):
    """tests/golden/ref_prodiff_T8.npz (decoder 'prodiff', schedule 'vpsde') at T steps (default the fixture's 8)."""
    _, meta = golden("ref_prodiff_T8")
    T = meta["T"] if T is None else T
    return resolve(timesteps=T, K_step=T, f0_timesteps=meta["f0_T"], **meta["overrides"])


def kstep_hp(T, K):
    """tests/golden/ref_kstep.npz: the T-step schedule with K_step K (acoustic_sd() is its checkpoint)."""
    return resolve(timesteps=T, K_step=K, f0_timesteps=T)


def _synth_sd(hp_of, cfg):
    key = (hp_of, cfg["T"], tuple(sorted(cfg["overrides"].items())))
    if key not in _CACHE:
        _CACHE[key] = synth.acoustic_state_dict(hp_of(cfg), seed=0)
    return _CACHE[key]


def switch_sd(cfg):
    return _synth_sd(switch_hp, cfg)


def fft_spkid_sd(cfg):
    return _synth_sd(fft_spkid_hp, cfg)


def conv_sd(meta):
    return _synth_sd(conv_hp, meta)


def prodiff_sd():
    if "prodiff_sd" not in _CACHE:
        _CACHE["prodiff_sd"] = synth.acoustic_state_dict(prodiff_hp(), seed=0)
    return _CACHE["prodiff_sd"]


def predictor_inputs(meta):
    """The seeded inputs of ref_convf0's predictor-only case: [2, pred_frames, 256] (one per predictor), channel 0
    exactly 0 in the rows meta['pred_zero_rows']."""
    g = torch.Generator().manual_seed(meta["pred_seed"])
    xs = torch.randn(2, 1, meta["pred_frames"], 256, generator=g)
    xs[:, :, meta["pred_zero_rows"], 0] = 0
    return xs[:, 0]


def registry_inputs(seed=131):
    """Inputs of the per-registry drop-in fixture ref_registry (tools/make_golden.py registry), rebuilt from the seed.

    enc_tokens [3, 12]: true lengths 12, 7, 9, then trailing padding tokens (0); utterance 0 also has an interior 0 token
    (position 3), which the encoder masks like padding.  dec_x [3, 24, 256]: true lengths 24, 13, 19, then all-zero rows;
    utterance 0 has an interior all-zero row (11) and a row whose column 0 alone is 0 (5), utterance 2 another such row
    (5).  The interior cases sit in the longest utterance because only an utterance without trailing padding is the same
    in the reference's padded batch and in its own B = 1 call (a padding row after a LayerNorm holds the LN bias, and the
    FFN conv reads it); the library computes B = 1 semantics for every utterance.  style_dec_<i> /
    style_ref_<i> / style_f0_<i>: two B = 1 get_style inputs (decoder_inp [1, F, 256], ref_mels [1, R, 80], ref_f0 [R]);
    reference mel 1 has an interior all-zero row (9)."""
    g = torch.Generator().manual_seed(seed)
    enc_lens, dec_lens = (12, 7, 9), (24, 13, 19)
    tok = torch.zeros(3, max(enc_lens), dtype=torch.long)
    for b, n in enumerate(enc_lens):
        tok[b, :n] = torch.randint(3, synth.N_TOKENS, (n,), generator=g)
    tok[0, 3] = 0
    x = torch.zeros(3, max(dec_lens), 256)
    for b, n in enumerate(dec_lens):
        x[b, :n] = torch.randn(n, 256, generator=g)
    x[0, 11] = 0
    x[0, 5, 0] = 0
    x[2, 5, 0] = 0
    d = {"enc_tokens": tok, "dec_x": x}
    for i, (F_, R, idx) in enumerate(((21, 17, 110), (30, 26, 111))):
        u = synth.make_utterance(F_ / 187.5, utt_idx=idx, ref_frames=R, frames=F_, phones=6)
        ref = u["ref_mels"].clone()
        if i == 1:
            ref[9] = 0
        d[f"style_dec_{i}"] = torch.randn(1, F_, 256, generator=g)
        d[f"style_ref_{i}"] = ref[None]
        d[f"style_f0_{i}"] = u["ref_f0"]
    return d


# the layouts of tools/make_golden.py vocoder_layouts (tests/golden/ref_vocoder_layouts.npz): V3 without NSF is the
# generator the `HifiGAN` registry class builds from a config without the harmonic source
VOCODER_LAYOUTS = {"v2": HIFIGAN_V2, "v3": HIFIGAN_V3, "v3_nonsf": dict(HIFIGAN_V3, use_pitch_embed=False)}


def vocoder_sd(layout=None):
    """The synthetic checkpoint (seed 0, cached) of DEFAULT_VOCODER_CONFIG (V1), or of VOCODER_LAYOUTS[layout]."""
    key = ("vsd", layout)
    if key not in _CACHE:
        _CACHE[key] = synth.vocoder_state_dict(DEFAULT_VOCODER_CONFIG if layout is None else VOCODER_LAYOUTS[layout],
                                               seed=0)
    return _CACHE[key]


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
