"""Model switches (hparams emo / style / umln / use_txt_cond), CPU side: the test oracle and the synthetic checkpoints
against the unmodified reference (tests/golden/ref_switches.npz), the hparams rules, the C ABI's argument checks (no GPU
needed) and the host-side batch packing."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import stylesinger_oracle as O
from stylesinger_b200 import synth
from stylesinger_b200.engine import pack_batch
from stylesinger_b200.hparams import SWITCHES, resolve
from tests.common import golden, switch_hp, switch_sd, utt_from_meta

TOL = 2e-5  # fp32 CPU, same op order up to BLAS blocking (as tests/test_oracle_golden.py)
CONFIGS = ("no_emo", "no_style", "no_umln", "no_txt_cond", "all_off", "prodiff_no_emo_style", "conv_no_style")


def _maxabs(a, b):
    return float(np.abs(np.asarray(a, np.float64) - np.asarray(b, np.float64)).max())


def _cfg(meta, c):
    return {"T": meta["T"], "overrides": meta["configs"][c]["overrides"]}


def _forward(meta, c, seed, use_mel2ph=True):
    cfg = _cfg(meta, c)
    u = utt_from_meta(meta)
    ns = O.NoiseSource(seed)
    with torch.no_grad():
        r = O.stylesinger_forward(switch_sd(cfg), switch_hp(cfg), u["txt_tokens"][None], u["note"][None],
                                  u["note_dur"][None], u["note_type"][None], u["spk_embed"][None],
                                  u["emo_embed"][None], u["ref_mels"][None], u["ref_f0"], ns,
                                  mel2ph=u["mel2ph"][None] if use_mel2ph else None)
    return r, ns


def test_fixture_covers_every_configuration():
    g, meta = golden("ref_switches")
    assert tuple(meta["configs"]) == CONFIGS
    for c in CONFIGS:
        hp = switch_hp(_cfg(meta, c))
        assert (f"{c}/style" in g.files) == hp["style"] and (f"{c}/rq_codes" in g.files) == hp["style"]
        assert (f"{c}/emo_embed" in g.files) == hp["emo"]
        assert (f"{c}/coarse_mel" in g.files) == (hp["decoder"] == "diffsinger")


@pytest.mark.parametrize("c", CONFIGS)
def test_oracle_forward_matches_reference(c):
    g, meta = golden("ref_switches")
    r, ns = _forward(meta, c, meta["seed"])
    assert [[k, list(sh)] for k, sh in ns.log] == meta["configs"][c]["noise_log"]  # same draws in the same order
    errs = {}
    for k in ("mel_out", "pitch_pred", "decoder_inp", "spk_embed", "emo_embed", "style", "coarse_mel"):
        if f"{c}/{k}" in g.files:
            errs[k] = _maxabs(r[k][0].numpy(), g[f"{c}/{k}"])
    errs["f0_denorm(Hz)"] = _maxabs(r["f0_denorm"][0].numpy(), g[f"{c}/f0_denorm"])
    print(c, errs)
    assert all(v < TOL for k, v in errs.items() if k != "f0_denorm(Hz)"), errs
    assert errs["f0_denorm(Hz)"] < 1e-3
    if f"{c}/rq_codes" in g.files:
        assert np.array_equal(r["rq_codes"][0].numpy(), g[f"{c}/rq_codes"])  # RVQ indices: bit-exact
    else:
        assert "rq_codes" not in r and "style" not in r


def test_oracle_duration_path_matches_reference():
    g, meta = golden("ref_switches")
    c = meta["dur_config"]
    r, ns = _forward(meta, c, meta["seed"] + 1, use_mel2ph=False)
    assert [[k, list(sh)] for k, sh in ns.log] == meta["configs"][c]["dur_noise_log"]
    assert np.array_equal(r["mel2ph"][0].numpy(), g[f"{c}/dur_mel2ph"])  # integer path: bit-exact
    e = {"logdur": _maxabs(r["dur"][0].numpy(), g[f"{c}/dur_logdur"]),
         "mel_out": _maxabs(r["mel_out"][0].numpy(), g[f"{c}/dur_mel_out"])}
    print(c, e)
    assert max(e.values()) < TOL
    assert _maxabs(r["f0_denorm"][0].numpy(), g[f"{c}/dur_f0_denorm"]) < 1e-3


@pytest.mark.parametrize("c", CONFIGS)
def test_synth_keys_and_shapes_are_the_references(c):
    _, meta = golden("ref_switches")
    hp = switch_hp(_cfg(meta, c))
    ref = [[k, list(s)] for k, s in meta["configs"][c]["state_dict"]]
    assert [[k, list(s)] for k, s in synth.acoustic_param_shapes(hp)] == ref
    sd = switch_sd(_cfg(meta, c))
    assert [[k, list(v.shape)] for k, v in sd.items()] == ref


def test_default_synthetic_checkpoint_is_unchanged():
    """The default configuration keeps the parent's state dict (same keys, same generator draws)."""
    _, meta = golden("ref_convf0")  # a fixture whose key list was dumped before the switches existed
    hp = resolve(f0_gen="conv", timesteps=meta["T"], K_step=meta["T"])
    assert [[k, list(s)] for k, s in synth.acoustic_param_shapes(hp)] == meta["state_dict"]
    sd = synth.acoustic_state_dict(resolve(timesteps=4, K_step=4, f0_timesteps=4), seed=0)
    assert sd["ln_proj.weight"].shape == (256, 1104) and "emo_embed_proj.weight" in sd and "norm.affine_layer.linear_layer.weight" in sd


def test_resolve_accepts_booleans_only():
    for k in SWITCHES:
        for v in (True, False):
            assert resolve(**{k: v})[k] is v
        for bad in (None, 0, 1, "false", "yes"):
            with pytest.raises(NotImplementedError, match=k):
                resolve(**{k: bad})
    hp = resolve(emo=False, style=False, umln=False, use_txt_cond=False, decoder="prodiff", schedule_type="vpsde",
                 f0_gen="conv")
    assert not any(hp[k] for k in SWITCHES)
    for kw in ({"decoder": "fft"}, {"use_spk_id": True}):
        with pytest.raises(NotImplementedError):
            resolve(emo=False, **kw)


def _create_ex3(sw, tensors=(), mel_decoder=0, f0_gen=0):
    from stylesinger_b200._lib import HParams, ModelSwitches, TensorDesc, lib
    keep = []
    arr = (TensorDesc * max(len(tensors), 1))()
    for i, (name, t) in enumerate(tensors):
        t = np.ascontiguousarray(t, np.float32)
        keep.append((name.encode(), t))
        arr[i].name = keep[-1][0]
        arr[i].data = t.ctypes.data
        arr[i].ndim = t.ndim
        for d, s in enumerate(t.shape):
            arr[i].shape[d] = s
    h = C.c_void_p()
    hp = HParams(hidden_size=256)
    rc = lib.ssb_model_create_ex3(C.byref(h), arr if tensors else None, len(tensors), C.byref(hp), mel_decoder, f0_gen,
                                  C.byref(ModelSwitches(*sw)) if sw is not None else None)
    return rc, h.value, lib.ssb_last_error().decode()


@pytest.mark.parametrize("sw, cause", [((2, 1, 1, 1), "switch emo must be 0 or 1, got 2"),
                                        ((1, -1, 1, 1), "switch style must be 0 or 1, got -1"),
                                        ((1, 1, 7, 1), "switch umln must be 0 or 1, got 7"),
                                        ((1, 1, 1, 3), "switch use_txt_cond must be 0 or 1, got 3"),
                                        (None, "null switches")])
def test_model_create_ex3_rejects_bad_switches_without_a_gpu(sw, cause):
    rc, h, err = _create_ex3(sw)
    print(sw, "rc", rc, "message:", err)
    assert rc != 0 and not h and cause in err


@pytest.mark.parametrize("sw, width", [((1, 1, 1, 1), 848), ((0, 1, 1, 1), 1104), ((0, 0, 1, 0), 592),
                                        ((0, 0, 0, 0), 1104)])
def test_model_create_ex3_rejects_a_mismatched_ln_proj_without_a_gpu(sw, width):
    want = 80 + 256 * (1 + sw[3] + sw[0] + sw[1])
    rc, h, err = _create_ex3(sw, [("ln_proj.weight", np.zeros((256, width), np.float32))])
    print(sw, width, "rc", rc, "message:", err)
    assert rc != 0 and not h
    assert f"ln_proj.weight must be [256, {want}]" in err and f"got [256, {width}]" in err


def test_model_create_ex3_unknown_modes_keep_their_messages():
    rc, h, err = _create_ex3((1, 1, 1, 1), mel_decoder=5)
    assert rc != 0 and not h and "unknown mel_decoder 5" in err
    rc, h, err = _create_ex3((1, 1, 1, 1), f0_gen=9)
    assert rc != 0 and not h and "unknown f0_gen 9" in err


def test_pack_batch_leaves_out_the_fields_a_model_does_not_read():
    us = [synth.make_utterance(0.2, utt_idx=i, ref_frames=16 + i, frames=30 + i, phones=5) for i in range(3)]
    full = pack_batch(us)
    assert {"emo_embed", "ref_mels", "ref_f0"} <= set(full.t) and full.ref_offsets is not None
    for emo, style in ((False, True), (True, False), (False, False)):
        stripped = [{k: v for k, v in u.items() if (emo or k != "emo_embed") and (style or k not in ("ref_mels", "ref_f0"))}
                    for u in us]
        pb = pack_batch(stripped, emo=emo, style=style)
        assert ("emo_embed" in pb.t) == emo
        assert ("ref_mels" in pb.t) == style and ("ref_f0" in pb.t) == style
        assert (pb.ref_offsets is not None) == style
        for k in ("txt_tokens", "note", "note_type", "note_dur", "spk_embed", "mel2ph"):
            assert torch.equal(pb.t[k], full.t[k]), k
        assert np.array_equal(pb.frame_offsets, full.frame_offsets) and np.array_equal(pb.ph_offsets, full.ph_offsets)
        assert pb.h2d_bytes() < full.h2d_bytes()


def test_facade_without_emo_and_style_needs_neither():
    """modules.StyleSinger on an emo / style-off model: emo_embed, ref_mels and ref_f0 may be None, and the batch the
    engine receives carries none of them; ret has no 'emo_embed' / 'style' (the reference sets neither)."""
    import stylesinger_b200.modules as M

    class FakeEngine:
        device = torch.device("cpu")

        def __init__(self):
            self.calls = []

        def forward(self, pb, noise=None, seed=0, skip_mel_diffusion=False, dur=None, want=(), **kw):
            self.calls.append({"t": set(pb.t), "ref": pb.ref_offsets, "want": set(want)})
            Fs, B = int(pb.frame_offsets[-1]), pb.B
            shapes = {"mel_out": (Fs, 80), "coarse_mel": (Fs, 80), "f0_denorm": (Fs,), "decoder_inp": (Fs, 256),
                      "pitch_pred": (Fs, 2), "spk_proj": (B, 256)}
            out = {k: torch.zeros(shapes[k]) for k in want if k in shapes}
            out["mel2ph"] = pb.t["mel2ph"]
            return out

    us = [synth.make_utterance(0.2, utt_idx=i, ref_frames=16, frames=30, phones=5) for i in range(2)]
    eng = FakeEngine()
    m = M.StyleSinger(hparams=dict(emo=False, style=False), engine=eng)
    ret = m(torch.stack([u["txt_tokens"] for u in us]), mel2ph=torch.stack([u["mel2ph"] for u in us]),
            spk_embed=torch.stack([u["spk_embed"] for u in us]), global_steps=320000, infer=True,
            note=torch.stack([u["note"] for u in us]), note_dur=torch.stack([u["note_dur"] for u in us]),
            note_type=torch.stack([u["note_type"] for u in us]))
    call = eng.calls[-1]
    assert not {"emo_embed", "ref_mels", "ref_f0"} & call["t"] and call["ref"] is None
    assert not {"emo_proj", "style", "rq_codes"} & call["want"]
    assert "emo_embed" not in ret and "style" not in ret and ret["mel_out"].shape == (2, 30, 80)
    m2 = M.StyleSinger(hparams=dict(emo=False), engine=FakeEngine())
    with pytest.raises(ValueError, match="ref_mels, ref_f0 required"):
        m2(torch.stack([u["txt_tokens"] for u in us]), spk_embed=torch.stack([u["spk_embed"] for u in us]),
           global_steps=320000, infer=True, note=torch.stack([u["note"] for u in us]),
           note_dur=torch.stack([u["note_dur"] for u in us]), note_type=torch.stack([u["note_type"] for u in us]))
