"""Convolutional F0 generator (f0_gen 'conv') on the GPU, through the C ABI: ssb_model_create_ex2(..., SSB_F0_GEN_CONV),
ssb_pitch_predictor and ssb_acoustic_forward on a conv model, against the unmodified reference's fixture
(tests/golden/ref_convf0.npz) and the test oracle's pitch predictors in float64.  Bars, fixed before measuring and the
same as the existing tests': pitch_pred / decoder_inp < 1e-4, f0_denorm < 5e-2 Hz, mel_out < 1e-3 (DiffSinger T=4, as
tests/test_gpu_parity.py), ProDiff mel < 1e-4 max(1, |mel|) on fp32 and < 1e-3 max(1, |mel|) on tensor cores (as
tests/test_gpu_prodiff.py), each predictor alone < 1e-4; coarse bins and uv exact against the fixture."""
import numpy as np
import pytest
import torch

from oracle import stylesinger_oracle as O
from stylesinger_b200 import _lib
from stylesinger_b200._lib import SsbError
from tests.common import acoustic_engine, conv_hp, conv_sd, golden, predictor_inputs, utt_from_meta

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
BAR = {False: 1e-4, True: 1e-3}  # tensor cores off / on (relative to max(1, |x|))

_C = {}


def _maxabs(a, b):
    a = a.detach().cpu().numpy() if isinstance(a, torch.Tensor) else np.asarray(a)
    b = b.detach().cpu().numpy() if isinstance(b, torch.Tensor) else np.asarray(b)
    return float(np.abs(a.astype(np.float64) - b.astype(np.float64)).max())


def _fixture():
    if "g" not in _C:
        _C["g"], _C["meta"] = golden("ref_convf0")
    return _C["g"], _C["meta"]


def conv_engine(prodiff=False):
    """AcousticModel of the fixture's DiffSinger (or ProDiff) configuration with f0_gen 'conv'."""
    from stylesinger_b200.engine import AcousticModel
    _, meta = _fixture()
    m_meta = meta["prodiff"] if prodiff else meta
    key = "pd" if prodiff else "ds"
    if key not in _C:
        _C[key] = AcousticModel(conv_sd(m_meta), conv_hp(m_meta))
    m = _C[key]
    m.set_tensor_cores(True)
    m.set_persistent(True)
    return m


def _mel_noise(seed, T, Fr):
    """The forward's draws from NoiseSource(seed) - with f0_gen 'conv' only the mel sampler's: x_T / q_sample, then one
    per step - in the C ABI's [(T+1), F, 80] layout."""
    ns = O.NoiseSource(seed)
    return torch.stack([ns.randn((1, 1, 80, Fr))[0, 0].t() for _ in range(T + 1)]).contiguous().to(DEV)


def _coarse(f0_denorm):
    return O.f0_to_coarse(torch.as_tensor(np.asarray(f0_denorm.cpu() if isinstance(f0_denorm, torch.Tensor)
                                                     else f0_denorm))).numpy()


def _forward(m, u, seed, T, use_mel2ph=True, tc=False):
    from stylesinger_b200.engine import pack_batch
    pb = pack_batch([u], use_mel2ph=use_mel2ph).to(DEV)
    dur = None
    if not use_mel2ph:
        dur, _ = m.predict_durations(pb)
        pb.frame_offsets = np.array([0, int(dur.sum())], np.int32)
    Fr = int(pb.frame_offsets[-1])
    try:
        m.set_tensor_cores(tc)
        out = m.forward(pb, noise={"mel": _mel_noise(seed, T, Fr)}, dur=dur,
                        want=("mel_out", "f0_denorm", "decoder_inp", "pitch_pred", "mel2ph"))
        torch.cuda.synchronize()
    finally:
        m.set_tensor_cores(True)
    return out


def _check_forward(out, g, prefix, mel_bar, tag):
    e_pp = _maxabs(out["pitch_pred"], g[prefix + "pitch_pred"])
    e_dec = _maxabs(out["decoder_inp"], g[prefix + "decoder_inp"])
    e_f0 = _maxabs(out["f0_denorm"], g[prefix + "f0_denorm"])
    e_mel = _maxabs(out["mel_out"], g[prefix + "mel_out"])
    uv_ok = np.array_equal(out["pitch_pred"][:, 1].cpu().numpy() > 0, g[prefix + "pitch_pred"][:, 1] > 0)
    bins_ok = np.array_equal(_coarse(out["f0_denorm"]), _coarse(g[prefix + "f0_denorm"]))
    print(f"{tag}: pitch_pred {e_pp:.3e}, decoder_inp {e_dec:.3e}, f0_denorm {e_f0:.3e} Hz, mel_out {e_mel:.3e} "
          f"(bar {mel_bar:.1e}), uv exact {uv_ok}, coarse bins exact {bins_ok}")
    assert e_pp < 1e-4 and e_dec < 1e-4 and e_f0 < 5e-2
    assert e_mel < mel_bar
    assert uv_ok and bins_ok


# ---- fixture parity ---------------------------------------------------------------------------------------------------
def test_conv_forward_matches_reference_golden():
    g, meta = _fixture()
    out = _forward(conv_engine(), utt_from_meta(meta), meta["seed"], meta["T"])
    _check_forward(out, g, "", 1e-3, "f0_gen conv, mel2ph given, fp32")


def test_conv_duration_path_matches_reference_golden():
    g, meta = _fixture()
    out = _forward(conv_engine(), utt_from_meta(meta), meta["seed"] + 1, meta["T"], use_mel2ph=False)
    assert np.array_equal(out["mel2ph"].cpu().numpy(), g["dur_mel2ph"])
    _check_forward(out, g, "dur_", 1e-3, "f0_gen conv, durations predicted, fp32")


@pytest.mark.parametrize("tc", [False, True])
def test_prodiff_with_conv_f0_matches_reference_golden(tc):
    g, meta = _fixture()
    pm = meta["prodiff"]
    out = _forward(conv_engine(prodiff=True), utt_from_meta(pm), pm["seed"], pm["T"], tc=tc)
    sc = max(1.0, float(np.abs(g["pd_mel_out"]).max()))
    _check_forward(out, g, "pd_", BAR[tc] * sc, f"ProDiff + f0_gen conv, tc={tc}")


@pytest.mark.parametrize("tc", [False, True])
def test_each_predictor_matches_reference_golden(tc):
    """B=1 at 300 frames takes the fp32 path whatever the switch says (3 row tiles < 8)."""
    g, meta = _fixture()
    m = conv_engine()
    xs = predictor_inputs(meta)
    offs = np.array([0, xs.shape[1]], np.int32)
    try:
        m.set_tensor_cores(tc)
        for which, key in ((0, "pred_out_agnostic"), (1, "pred_out_specific")):
            out = m.pitch_predictor(which, xs[which].to(DEV).contiguous(), offs)
            torch.cuda.synchronize()
            err = _maxabs(out, g[key])
            print(f"tc={tc} {key}: L-inf {err:.3e}")
            assert err < 1e-4
    finally:
        m.set_tensor_cores(True)


# ---- a bench-sized ragged batch ---------------------------------------------------------------------------------------
def _ragged_lengths(total=20000, seed=3):
    rng = np.random.default_rng(seed)
    lens = [1, 2, 3, 5]
    while sum(lens) < total:
        lens.append(int(rng.integers(60, 1800)))
    rng.shuffle(lens)
    return lens


def _reference_f64(x, offs, sd, which):
    """float64 PitchPredictor per utterance (B=1 each), on the GPU for speed (test-side reference only)."""
    sd64 = {k: v.to(DEV) for k, v in sd.items() if k.startswith(O.PITCH_PREDICTORS[which])}
    out = []
    with torch.no_grad():
        for b in range(len(offs) - 1):
            a, e = int(offs[b]), int(offs[b + 1])
            out.append(O.pitch_predictor(x[None, a:e].to(DEV), sd64, which, dtype=torch.float64)[0])
    return torch.cat(out)


def _near_edge_flips(ref_pp, our_pp, bar):
    """uv and coarse-bin disagreements between the float64 reference and the kernel, and how many of them sit at frames
    whose reference value is within `bar` of 0 (uv) or of a bin edge (f0): only those are allowed."""
    ref_uv, our_uv = ref_pp[:, 1] > 0, our_pp[:, 1] > 0
    uv_flip = ref_uv != our_uv
    uv_near = np.abs(ref_pp[:, 1]) <= bar * np.maximum(1.0, np.abs(ref_pp[:, 1]))
    f0_ref, f0_our = torch.from_numpy(2.0 ** ref_pp[:, 0]), torch.from_numpy(2.0 ** our_pp[:, 0].astype(np.float64))
    b_ref, b_our = O.f0_to_coarse(f0_ref).numpy(), O.f0_to_coarse(f0_our).numpy()
    b_flip = b_ref != b_our
    lo = O.f0_to_coarse(torch.from_numpy(2.0 ** (ref_pp[:, 0] - bar * np.maximum(1.0, np.abs(ref_pp[:, 0]))))).numpy()
    hi = O.f0_to_coarse(torch.from_numpy(2.0 ** (ref_pp[:, 0] + bar * np.maximum(1.0, np.abs(ref_pp[:, 0]))))).numpy()
    b_near = lo != hi
    return int(uv_flip.sum()), int((uv_flip & ~uv_near).sum()), int(b_flip.sum()), int((b_flip & ~b_near).sum())


@pytest.mark.parametrize("tc", [False, True])
def test_ragged_batch_vs_float64_and_b1(tc):
    g, meta = _fixture()
    m = conv_engine()
    sd = conv_sd(meta)
    lens = _ragged_lengths()
    offs = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
    tiles = sum((n + 127) // 128 for n in lens)
    assert tiles >= 8 and offs[-1] >= 20000
    gen = torch.Generator().manual_seed(11)
    xs = torch.randn(2, int(offs[-1]), 256, generator=gen, dtype=torch.float64)
    for b in range(len(lens)):  # a few rows with channel 0 exactly 0 in the longer utterances (the position skip)
        if lens[b] > 10:
            xs[:, int(offs[b]) + 3, 0] = 0
    pred = {}
    before = _lib.variant_launches()
    try:
        m.set_tensor_cores(tc)
        for which in (0, 1):
            x = xs[which].float().to(DEV).contiguous()
            pred[which] = m.pitch_predictor(which, x, offs)
            torch.cuda.synchronize()
            ref = _reference_f64(xs[which], offs, sd, which)
            sc = torch.clamp(ref.abs(), min=1.0)
            rel = float(((pred[which].double() - ref).abs() / sc).max())
            print(f"tc={tc} which={which}: {len(lens)} utterances, {int(offs[-1])} frames, {tiles} row tiles: "
                  f"max |err| / max(1, |ref|) {rel:.3e} (bar {BAR[tc]:.0e})")
            assert rel < BAR[tc]
            pred[which, "ref"] = ref
            # each utterance against its own B=1 call (which takes the tensor-core path only from 8 row tiles on)
            worst = 0.0
            for b in range(len(lens)):
                a, e = int(offs[b]), int(offs[b + 1])
                one = m.pitch_predictor(which, x[a:e].contiguous(), np.array([0, e - a], np.int32))
                worst = max(worst, _maxabs(one, pred[which][a:e]))
            print(f"tc={tc} which={which}: batch vs per-utterance B=1 L-inf {worst:.3e}")
            assert worst < BAR[tc]
    finally:
        m.set_tensor_cores(True)
    after = _lib.variant_launches()
    tc_launches = sum(after.get(k, 0) - before.get(k, 0) for k in after if "GENERIC" in k)
    print(f"tc={tc}: tensor-core GENERIC launches {tc_launches}")
    assert (tc_launches > 0) == tc
    # the averaged pitch_pred -> uv and coarse bins: flips only where the reference lies within the bar of an edge
    ref_pp = (pred[1, "ref"] / 2 + pred[0, "ref"] / 2).cpu().numpy()
    our_pp = (pred[1] / 2 + pred[0] / 2).cpu().numpy()
    uv_f, uv_bad, b_f, b_bad = _near_edge_flips(ref_pp, our_pp, BAR[tc])
    print(f"tc={tc}: uv flips {uv_f} ({uv_bad} not near 0), coarse-bin flips {b_f} ({b_bad} not near a bin edge)")
    assert uv_bad == 0 and b_bad == 0


def test_ragged_acoustic_batch_matches_b1_forwards():
    """The whole conv pitch block on a ragged batch (tensor-core predictors, >= 8 row tiles) against each utterance's own
    B=1 forward; skip_mel_diffusion keeps it to the part this feature adds."""
    from stylesinger_b200 import synth
    from stylesinger_b200.engine import pack_batch
    m = conv_engine()
    utts = [synth.make_utterance(s, utt_idx=300 + i, ref_frames=64) for i, s in enumerate([0.6, 3.1, 1.7, 4.4, 0.2])]
    pb = pack_batch(utts).to(DEV)
    assert sum((int(pb.frame_offsets[b + 1] - pb.frame_offsets[b]) + 127) // 128 for b in range(pb.B)) >= 8
    out = m.forward(pb, skip_mel_diffusion=True, want=("f0_denorm", "pitch_pred"))
    torch.cuda.synchronize()
    worst_pp, worst_f0, flips, uv_flips = 0.0, 0.0, 0, 0
    for b, u in enumerate(utts):
        a, e = int(pb.frame_offsets[b]), int(pb.frame_offsets[b + 1])
        one = m.forward(pack_batch([u]).to(DEV), skip_mel_diffusion=True, want=("f0_denorm", "pitch_pred"))
        pp1, ppb = one["pitch_pred"].cpu().numpy(), out["pitch_pred"][a:e].cpu().numpy()
        worst_pp = max(worst_pp, _maxabs(pp1, ppb))
        same_uv = (pp1[:, 1] > 0) == (ppb[:, 1] > 0)
        assert np.all(same_uv | (np.abs(pp1[:, 1]) < 1e-3))  # a uv flip only next to 0
        uv_flips += int((~same_uv).sum())
        f1, fb = one["f0_denorm"].cpu().numpy()[same_uv], out["f0_denorm"][a:e].cpu().numpy()[same_uv]
        worst_f0 = max(worst_f0, _maxabs(f1, fb))
        flips += int((_coarse(f1) != _coarse(fb)).sum())
    print(f"batch of {pb.B} ({pb.total_frames} frames) vs B=1: pitch_pred {worst_pp:.3e}, f0_denorm {worst_f0:.3e} Hz, "
          f"uv flips {uv_flips}, coarse-bin flips {flips}")
    assert worst_pp < 1e-3 and worst_f0 < 5e-1


# ---- mode mismatches --------------------------------------------------------------------------------------------------
def test_conv_model_refuses_the_f0_diffusion_entries():
    g, meta = _fixture()
    m = conv_engine()
    Fr = 16
    offs = np.array([0, Fr], np.int32)
    cond = torch.zeros(Fr, 256, device=DEV)
    band = torch.zeros(Fr, device=DEV)
    with pytest.raises(SsbError, match="conv F0 generator"):
        m.set_timesteps(f0_T=4)
    with pytest.raises(SsbError, match="conv F0 generator"):
        m.f0_diffusion(0, cond, band, band, offs)
    for which in (1, 2):
        with pytest.raises(SsbError, match="conv F0 generator"):
            m.denoiser_eval(which, band, torch.zeros(Fr, dtype=torch.int32, device=DEV), 0, cond, offs)
    from stylesinger_b200.engine import pack_batch
    u = utt_from_meta(meta)
    F = meta["frames"]
    noise = {"f0_gauss": [torch.zeros(5, F, device=DEV)] * 2, "f0_unif": [torch.zeros(4, F, 2, device=DEV)] * 2,
             "mel": _mel_noise(0, meta["T"], F)}
    with pytest.raises(SsbError, match="draws no F0 noise"):
        m.forward(pack_batch([u]).to(DEV), noise=noise)


def test_gmdiff_model_refuses_the_pitch_predictor():
    m = acoustic_engine(4)
    with pytest.raises(SsbError, match="SSB_F0_GEN_CONV"):
        m.pitch_predictor(0, torch.zeros(8, 256, device=DEV), np.array([0, 8], np.int32))
