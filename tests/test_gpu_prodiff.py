"""ProDiff teacher mel decoder on the GPU: the CUDA path (ssb_model_create_ex(..., SSB_MEL_DECODER_PRODIFF),
ssb_mel_prodiff_sample, ssb_acoustic_forward on a ProDiff model) against the unmodified reference's fixture
(tests/golden/ref_prodiff_T8.npz) and the test oracle.  Bars, fixed before measuring and the
same as the PLMS sampler's: mel L-inf < 1e-4 max(1, |mel|) on the fp32 FFMA path, < 1e-3 max(1, |mel|) on tensor cores."""
import numpy as np
import pytest
import torch

from oracle import stylesinger_oracle as O
from stylesinger_b200._lib import SsbError
from tests.common import acoustic_engine, engine_noise_from_stream, golden, prodiff_hp, prodiff_sd, utt_from_meta

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
BAR = {False: 1e-4, True: 1e-3}  # tensor cores off / on


def _maxabs(a, b):
    a = a.detach().cpu().numpy() if isinstance(a, torch.Tensor) else np.asarray(a)
    b = b.detach().cpu().numpy() if isinstance(b, torch.Tensor) else np.asarray(b)
    return float(np.abs(a.astype(np.float64) - b.astype(np.float64)).max())


_C = {}


def _meta():
    if "g" not in _C:
        _C["g"], _C["meta"] = golden("ref_prodiff_T8")
    return _C["g"], _C["meta"]


def prodiff_engine():
    from stylesinger_b200.engine import AcousticModel
    if "m" not in _C:
        _C["m"] = AcousticModel(prodiff_sd(), prodiff_hp())
    m = _C["m"]
    m.set_tensor_cores(True)
    m.set_persistent(True)
    m.set_persistent_groups(False)
    return m


class ListNoise:
    """Hands the oracle a fixed list of draws in order (the injected noise, re-shaped to the reference's layout)."""

    def __init__(self, draws):
        self.draws = list(draws)

    def randn(self, shape):
        t = self.draws.pop(0)
        assert tuple(t.shape) == tuple(shape), (t.shape, shape)
        return t


def _prodiff_noise(seed, T, Fr):
    """ProDiffusion.forward's draws from NoiseSource(seed) in the C ABI's [(T+1), F, 80] layout."""
    ns = O.NoiseSource(seed)
    return torch.stack([ns.randn((1, 1, 80, Fr))[0, 0].t() for _ in range(T + 1)]).contiguous()


# ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("tc", [True, False])
@pytest.mark.parametrize("persistent", [True, False])
def test_prodiff_forward_matches_reference_golden(tc, persistent):
    from stylesinger_b200.engine import pack_batch
    g, meta = _meta()
    m = prodiff_engine()
    u = utt_from_meta(meta)
    Fr = meta["frames"]
    pb = pack_batch([u]).to(DEV)
    noise, _ = engine_noise_from_stream(meta["seed"], meta["f0_T"], meta["T"], Fr, DEV)
    try:
        m.set_tensor_cores(tc)
        m.set_persistent(persistent)
        out = m.forward(pb, noise=noise, want=("mel_out", "f0_denorm", "decoder_inp"))
        torch.cuda.synchronize()
    finally:
        m.set_tensor_cores(True)
        m.set_persistent(True)
    sc = max(1.0, float(np.abs(g["mel_out"]).max()))
    e_mel = _maxabs(out["mel_out"], g["mel_out"])
    e_dec = _maxabs(out["decoder_inp"], g["decoder_inp"])
    e_f0 = _maxabs(out["f0_denorm"], g["f0_denorm"])
    print(f"tc={tc} persistent={persistent}: mel_out L-inf {e_mel:.3e} (bar {BAR[tc] * sc:.1e}), decoder_inp {e_dec:.3e}, "
          f"f0_denorm {e_f0:.3e} Hz")
    assert e_dec < 1e-4
    assert e_mel < BAR[tc] * sc


@pytest.mark.parametrize("tc", [True, False])
def test_prodiff_sampler_matches_reference_golden(tc):
    g, meta = _meta()
    m = prodiff_engine()
    cond = torch.from_numpy(g["sampler_cond"]).to(DEV)
    Fr = cond.shape[0]
    noise = _prodiff_noise(meta["sampler_seed"], meta["T"], Fr).to(DEV)
    offs = np.array([0, Fr], np.int32)
    try:
        m.set_tensor_cores(tc)
        mel = m.mel_prodiff(cond, offs, noise)
        torch.cuda.synchronize()
    finally:
        m.set_tensor_cores(True)
    sc = max(1.0, float(np.abs(g["sampler_mel"]).max()))
    err = _maxabs(mel, g["sampler_mel"])
    print(f"tc={tc}: ProDiff sampler L-inf {err:.3e} (bar {BAR[tc] * sc:.1e})")
    assert err < BAR[tc] * sc


def test_prodiff_ragged_batch_vs_b1_oracle():
    m = prodiff_engine()
    hp = prodiff_hp()
    T = hp["timesteps"]
    gen = torch.Generator().manual_seed(5)
    lens = [37, 130, 64]
    offs = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
    cond = torch.randn(int(offs[-1]), 256, generator=gen)
    noise = torch.randn(T + 1, int(offs[-1]), 80, generator=gen)
    mel = m.mel_prodiff(cond.to(DEV), offs, noise.to(DEV)).cpu()
    for b in range(3):
        a, e = int(offs[b]), int(offs[b + 1])
        with torch.no_grad():
            ref = O.mel_prodiff_sample(cond[None, a:e], prodiff_sd(), hp,
                                       ListNoise([noise[k, a:e].t().contiguous()[None, None] for k in range(T + 1)]))
        sc = max(1.0, float(ref.abs().max()))
        err = _maxabs(mel[a:e], ref[0])
        print(f"utterance {b} ({lens[b]} frames): L-inf vs B=1 oracle {err:.3e} (bar {1e-3 * sc:.1e})")
        assert err < 1e-3 * sc


def test_prodiff_large_batch_pair_path_and_persistent_groups():
    """27 k frames (> 48 row tiles): the per-launch tensor-core path and the persistent groups (ssb_model_set_persistent_groups)
    against the same engine's fp32 FFMA path.  The groups run in Philox mode with one seed per group, so the fp32 reference
    runs the same groups as sub-batches with those seeds."""
    m = prodiff_engine()
    T = m.T
    gen = torch.Generator().manual_seed(6)
    lens = [1000 + 37 * i for i in range(20)]
    offs = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
    N = int(offs[-1])
    cond = torch.randn(N, 256, generator=gen).to(DEV)
    noise = torch.randn(T + 1, N, 80, generator=gen).to(DEV)
    try:
        tc_mel = m.mel_prodiff(cond, offs, noise)  # injected noise: one batch, tensor-core per-launch path
        m.set_tensor_cores(False)
        ref = m.mel_prodiff(cond, offs, noise)
        torch.cuda.synchronize()
        sc = max(1.0, float(ref.abs().max()))
        err = _maxabs(tc_mel, ref)
        print(f"{N} frames, per-launch tensor cores vs fp32 FFMA: L-inf {err:.3e} (bar {1e-3 * sc:.1e})")
        assert err < 1e-3 * sc
        # persistent groups (Philox): groups of consecutive utterances of <= 48 row tiles, seed + golden-ratio step * group
        seed = 77
        m.set_tensor_cores(True)
        m.set_persistent_groups(True)
        grp = m.mel_prodiff(cond, offs, None, seed=seed)
        m.set_persistent_groups(False)
        m.set_tensor_cores(False)
        tiles = [(n + 127) // 128 for n in lens]
        b0, gi, worst = 0, 0, 0.0
        while b0 < len(lens):
            b1, nt = b0, 0
            while b1 < len(lens) and (b1 == b0 or nt + tiles[b1] <= 48):
                nt += tiles[b1]
                b1 += 1
            a, e = int(offs[b0]), int(offs[b1])
            sub = (offs[b0:b1 + 1] - offs[b0]).astype(np.int32)
            s = (seed + 0x9E3779B97F4A7C15 * gi) % (1 << 64)
            r = m.mel_prodiff(cond[a:e].contiguous(), sub, None, seed=s)
            worst = max(worst, _maxabs(grp[a:e], r) / max(1.0, float(r.abs().max())))
            b0, gi = b1, gi + 1
        print(f"persistent groups ({gi} groups) vs fp32 FFMA per group: relative L-inf {worst:.3e} (bar 1e-3)")
        assert gi > 1 and np.isfinite(grp.cpu().numpy()).all()
        assert worst < 1e-3
    finally:
        m.set_tensor_cores(True)
        m.set_persistent_groups(False)


def test_prodiff_philox_forward_is_finite_and_differs_from_diffsinger():
    from stylesinger_b200.engine import pack_batch
    _, meta = _meta()
    u = utt_from_meta(meta)
    pb = pack_batch([u]).to(DEV)
    pd = prodiff_engine().forward(pb, seed=3)["mel_out"]
    ds = acoustic_engine(meta["T"], meta["f0_T"]).forward(pb, seed=3)["mel_out"]
    d = _maxabs(pd, ds)
    print(f"Philox: ProDiff |mel| max {float(pd.abs().max()):.3f}, max |ProDiff - DiffSinger| {d:.3f}")
    assert torch.isfinite(pd).all()
    assert d > 1e-2


def test_prodiff_mode_mismatches_are_errors():
    from stylesinger_b200.engine import pack_batch
    _, meta = _meta()
    m = prodiff_engine()
    offs = np.array([0, 40], np.int32)
    cond = torch.zeros(40, 256, device=DEV)
    coarse = torch.zeros(40, 80, device=DEV)
    msgs = []
    with pytest.raises(SsbError) as e:
        m.mel_diffusion(cond, coarse, offs)
    msgs.append(str(e.value))
    with pytest.raises(SsbError) as e:
        m.mel_diffusion_plms(cond, coarse, offs, 2)
    msgs.append(str(e.value))
    pb = pack_batch([utt_from_meta(meta)]).to(DEV)
    with pytest.raises(SsbError) as e:
        m.forward(pb, want=("mel_out", "coarse_mel"))
    msgs.append(str(e.value))
    with pytest.raises(SsbError) as e:
        m.forward(pb, want=("mel_out", "diff_cond"))
    msgs.append(str(e.value))
    with pytest.raises(SsbError) as e:
        acoustic_engine(meta["T"], meta["f0_T"]).mel_prodiff(cond, offs)
    msgs.append(str(e.value))
    for s in msgs:
        print(s)
    assert "DiffSinger model" in msgs[0] and "PLMS" in msgs[1]
    assert "coarse_mel" in msgs[2] and "coarse_mel" in msgs[3] and "PRODIFF" in msgs[4]


def test_facade_returns_prodiff_mel_below_diff_start():
    from stylesinger_b200.engine import pack_batch
    from stylesinger_b200.modules import StyleSinger
    _, meta = _meta()
    m = prodiff_engine()
    hp = prodiff_hp()
    u = utt_from_meta(meta)
    model = StyleSinger(hparams=hp, engine=m)
    steps = hp["forcing"] + 1
    assert steps < hp["diff_start"]
    ret = model(u["txt_tokens"][None], mel2ph=u["mel2ph"][None], spk_embed=u["spk_embed"][None], emo_embed=u["emo_embed"][None],
                ref_mels=u["ref_mels"][None], ref_f0=u["ref_f0"], global_steps=steps, infer=True, note=u["note"][None],
                note_dur=u["note_dur"][None], note_type=u["note_type"][None], seed=4)
    direct = m.forward(pack_batch([u]).to(DEV), seed=4)["mel_out"]
    err = _maxabs(ret["mel_out"][0], direct)
    print(f"facade mel_out {tuple(ret['mel_out'].shape)}, L-inf vs engine.forward {err:.3e}")
    assert ret["mel_out"].shape == (1, meta["frames"], 80)
    assert err == 0.0
