"""Shallow diffusion on the GPU: hparams['K_step'] < timesteps (ssb_model_set_mel_k_step) through ssb_acoustic_forward,
ssb_mel_diffusion_sample (persistent single-launch, per-launch tensor-core and fp32 FFMA paths, persistent groups) and
ssb_mel_diffusion_sample_plms, against the unmodified reference's fixture (tests/golden/ref_kstep.npz) and the test
oracle.  Bars, fixed before measuring: mel L-inf < 1e-3 for the DDPM sampler (the bar of the T=25
forward test), 1e-4 max(1, |mel|) on FFMA and 1e-3 max(1, |mel|) on tensor cores for PLMS (as the PLMS / ProDiff tests);
style, pitch and decoder_inp as tests/test_gpu_parity.py."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import stylesinger_oracle as O
from stylesinger_b200._lib import SsbError, lib
from tests.common import acoustic_sd, engine_noise_from_stream, golden, hp_for, utt_from_meta

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
PLMS_BAR = {False: 1e-4, True: 1e-3}  # tensor cores off / on
PATHS = [(True, True), (True, False), (False, True), (False, False)]  # (tensor cores, persistent)
PATH_IDS = ["tc-persistent", "tc-per-launch", "ffma-persistent-on", "ffma"]


def _maxabs(a, b):
    a = a.detach().cpu().numpy() if isinstance(a, torch.Tensor) else np.asarray(a)
    b = b.detach().cpu().numpy() if isinstance(b, torch.Tensor) else np.asarray(b)
    return float(np.abs(a.astype(np.float64) - b.astype(np.float64)).max())


_C = {}


def engine(T, K, f0_T=None):
    """One DiffSinger model for this file, at schedule T and K_step K, tensor cores + persistent sampler on."""
    from stylesinger_b200.engine import AcousticModel
    if "m" not in _C:
        _C["m"] = AcousticModel(acoustic_sd(), hp_for(T, f0_T))
    m = _C["m"]
    m.set_timesteps(T, T if f0_T is None else f0_T)
    m.set_mel_k_step(K)
    m.set_tensor_cores(True)
    m.set_persistent(True)
    m.set_persistent_groups(False)
    return m


def _reset(m):
    m.set_tensor_cores(True)
    m.set_persistent(True)
    m.set_persistent_groups(False)
    m.set_mel_k_step(0)


def _sampler_noise(seed, K, Fr):
    """DiffusionDecoder.forward's K + 1 draws from NoiseSource(seed) in the C ABI's [(K+1), F, 80] layout."""
    ns = O.NoiseSource(seed)
    return torch.stack([ns.randn((1, 1, 80, Fr))[0, 0].t() for _ in range(K + 1)]).contiguous()


def _offs(lens):
    return np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)


# ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("tc,persistent", PATHS, ids=PATH_IDS)
def test_full_forward_matches_reference_golden(tc, persistent):
    """(a): timesteps 25, K_step 11, mel2ph given; K + 1 = 12 mel draws after the F0 samplers' draws."""
    from stylesinger_b200.engine import pack_batch
    g, meta = golden("ref_kstep")
    T, K = meta["T_fwd"], meta["K_fwd"]
    m = engine(T, K)
    pb = pack_batch([utt_from_meta(meta)]).to(DEV)
    noise, _ = engine_noise_from_stream(meta["seed"], T, K, meta["frames"], DEV)
    assert noise["mel"].shape[0] == K + 1
    try:
        m.set_tensor_cores(tc)
        m.set_persistent(persistent)
        out = m.forward(pb, noise=noise, want=("mel_out", "style", "rq_codes", "pitch_pred", "decoder_inp", "coarse_mel"))
        torch.cuda.synchronize()
    finally:
        _reset(m)
    e = {k: _maxabs(out[k], g["fwd_" + k]) for k in ("mel_out", "style", "pitch_pred", "decoder_inp", "coarse_mel")}
    print(f"tc={tc} persistent={persistent}, T={T} K_step={K}: " + ", ".join(f"{k} L-inf {v:.3e}" for k, v in e.items()))
    assert np.array_equal(out["rq_codes"].cpu().numpy().astype(np.int64), g["fwd_rq_codes"])
    for k in ("style", "pitch_pred", "decoder_inp", "coarse_mel"):
        assert e[k] < 1e-4, k
    assert e["mel_out"] < 1e-3


@pytest.mark.parametrize("tc,persistent", PATHS, ids=PATH_IDS)
@pytest.mark.parametrize("key", ["smp", "smp1"])
def test_sampler_matches_reference_golden(key, tc, persistent):
    """(b) DiffusionDecoder.forward alone at timesteps 100, K_step 51; (d) the same at K_step 1 (one step at t = 0, its
    noise multiplied by 0).  The persistent arm is asserted to have taken the single-launch kernel."""
    g, meta = golden("ref_kstep")
    T = meta["T"]
    K = meta["K"] if key == "smp" else 1
    m = engine(T, K)
    cond = torch.from_numpy(g["smp_cond"]).to(DEV)
    coarse = torch.from_numpy(g["smp_coarse"]).to(DEV)
    Fr = cond.shape[0]
    noise = _sampler_noise(meta["seed"] + 2, K, Fr).to(DEV)
    try:
        m.set_tensor_cores(tc)
        m.set_persistent(persistent)
        torch.cuda.synchronize()
        l0 = lib.ssb_launch_count()
        mel = m.mel_diffusion(cond, coarse, np.array([0, Fr], np.int32), noise)
        torch.cuda.synchronize()
        launches = lib.ssb_launch_count() - l0
    finally:
        _reset(m)
    err = _maxabs(mel, g[key + "_mel"])
    print(f"tc={tc} persistent={persistent}, T={T} K_step={K}: {launches} launches, L-inf vs reference {err:.3e}")
    if tc and persistent:
        assert launches < 16  # the K steps in one launch (plus packing, conditioner hoist, q_sample, denorm)
    else:
        assert launches > 2 * K * 20  # one launch per GEMM: 2 per residual layer and step at least
    assert err < 1e-3


@pytest.mark.parametrize("tc", [True, False], ids=["tc", "ffma"])
@pytest.mark.parametrize("interval", [10, 7])
def test_plms_matches_reference_golden(interval, tc):
    """(c) the pndm_speedup loop from t = K_step 51 of the 100-step schedule: t0 = 50 at interval 10, 49 at interval 7."""
    g, meta = golden("ref_kstep")
    m = engine(meta["T"], meta["K"])
    Fr = g["smp_cond"].shape[0]
    q = O.NoiseSource(meta["seed"] + 3).randn((1, 1, 80, Fr))[0, 0].t().contiguous().to(DEV)
    try:
        m.set_tensor_cores(tc)
        mel = m.mel_diffusion_plms(torch.from_numpy(g["smp_cond"]).to(DEV), torch.from_numpy(g["smp_coarse"]).to(DEV),
                                   np.array([0, Fr], np.int32), interval, q)
        torch.cuda.synchronize()
    finally:
        _reset(m)
    ref = g[f"plms_i{interval}_mel"]
    err, sc = _maxabs(mel, ref), max(1.0, float(np.abs(ref).max()))
    print(f"tc={tc} PLMS interval {interval} (t0 {meta[f'plms_i{interval}_t0']}), K_step {meta['K']}: L-inf {err:.3e} "
          f"(bar {PLMS_BAR[tc] * sc:.1e})")
    assert err < PLMS_BAR[tc] * sc


# ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("tc,persistent", PATHS, ids=PATH_IDS)
def test_k_step_equal_to_t_or_zero_changes_nothing(tc, persistent):
    """set_mel_k_step(T) and set_mel_k_step(0) give the bits of a model that never called it: the DDPM sampler with
    Philox and with injected noise on a ragged batch, PLMS, and the acoustic forward."""
    from stylesinger_b200 import synth
    from stylesinger_b200.engine import AcousticModel, pack_batch
    T = 20
    if "fresh" not in _C:
        _C["fresh"] = AcousticModel(acoustic_sd(), hp_for(T))
    fresh = _C["fresh"]
    assert fresh.K is None
    lens = [37, 130, 5]
    offs = _offs(lens)
    n = int(offs[-1])
    gen = torch.Generator().manual_seed(11)
    cond = torch.randn(n, 256, generator=gen).to(DEV)
    coarse = (-3 + 0.8 * torch.randn(n, 80, generator=gen)).clamp(-6, 0.5).to(DEV)
    noise = torch.randn(T + 1, n, 80, generator=gen).to(DEV)
    pb = pack_batch([synth.make_utterance(0.3, utt_idx=9, ref_frames=40, frames=56, phones=7)]).to(DEV)

    def run(model):
        model.set_tensor_cores(tc)
        model.set_persistent(persistent)
        r = [model.mel_diffusion(cond, coarse, offs, None, seed=5).clone(),
             model.mel_diffusion(cond, coarse, offs, noise).clone(),
             model.mel_diffusion_plms(cond, coarse, offs, 5, noise[0].contiguous()).clone(),
             model.forward(pb, seed=6)["mel_out"].clone()]
        torch.cuda.synchronize()
        return r

    m = engine(T, 0)
    try:
        ref = run(fresh)
        for K in (T, 0):
            m.set_mel_k_step(K)
            got = run(m)
            for name, a, b in zip(("Philox", "injected", "PLMS", "forward"), got, ref):
                assert torch.isfinite(a).all() and torch.equal(a, b), (K, name)
    finally:
        _reset(m)
        _reset(fresh)
    print(f"tc={tc} persistent={persistent}: K_step {T} and 0 bit-identical to a model that never set K_step")


def test_bench_sized_ragged_batch_persistent_groups_and_per_launch():
    """The batch64 utterance lengths plus utterances of 1, 2, 3 and 5 frames, K_step 37 of 100, Philox.  The persistent
    groups (ssb_model_set_persistent_groups) are compared group by group with a direct call on that group's utterances and
    seed (persistent single launch: bit-identical, same layout, same streams), and that call with the per-launch
    tensor-core path (same streams, different kernels: 1e-3)."""
    from bench import make_workload
    T, K, seed = 100, 37, 91
    utts, _ = make_workload("batch64", 0, 1)
    lens = [1, 2] + [len(u["mel2ph"]) for u in utts] + [3, 5]
    offs = _offs(lens)
    n = int(offs[-1])
    gen = torch.Generator().manual_seed(12)
    cond = torch.randn(n, 256, generator=gen).to(DEV)
    coarse = (-3 + 0.8 * torch.randn(n, 80, generator=gen)).clamp(-6, 0.5).to(DEV)
    m = engine(T, K)
    try:
        m.set_persistent_groups(True)
        grp = m.mel_diffusion(cond, coarse, offs, None, seed=seed)
        m.set_persistent_groups(False)
        tiles = [(x + 127) // 128 for x in lens]
        b0, gi, worst_pl, ident = 0, 0, 0.0, 0
        while b0 < len(lens):
            b1, nt = b0, 0
            while b1 < len(lens) and (b1 == b0 or nt + tiles[b1] <= 48):
                nt += tiles[b1]
                b1 += 1
            a, e = int(offs[b0]), int(offs[b1])
            sub = (offs[b0:b1 + 1] - offs[b0]).astype(np.int32)
            s = (seed + 0x9E3779B97F4A7C15 * gi) % (1 << 64)
            m.set_persistent(True)
            l0 = lib.ssb_launch_count()
            r_p = m.mel_diffusion(cond[a:e].contiguous(), coarse[a:e].contiguous(), sub, None, seed=s)
            torch.cuda.synchronize()
            assert lib.ssb_launch_count() - l0 < 16, gi  # the direct call took the persistent kernel
            m.set_persistent(False)
            r_l = m.mel_diffusion(cond[a:e].contiguous(), coarse[a:e].contiguous(), sub, None, seed=s)
            assert torch.isfinite(r_p).all() and torch.isfinite(r_l).all()
            ident += int(torch.equal(grp[a:e], r_p))
            assert torch.equal(grp[a:e], r_p), (gi, _maxabs(grp[a:e], r_p))
            worst_pl = max(worst_pl, _maxabs(r_p, r_l))
            b0, gi = b1, gi + 1
        whole = m.mel_diffusion(cond, coarse, offs, None, seed=seed)  # the default large-batch path: per-launch, one call
        torch.cuda.synchronize()
    finally:
        _reset(m)
    print(f"{len(lens)} utterances, {n} frames, K_step {K}: {gi} persistent groups, {ident} bit-identical to direct calls; "
          f"persistent vs per-launch tensor cores L-inf {worst_pl:.3e} (bar 1e-3)")
    assert gi > 1 and torch.isfinite(whole).all()
    assert worst_pl < 1e-3


# ---------------------------------------------------------------------------------------------------
def _raw_sample(m, cond, coarse, offs, ws, nbytes):
    p = lambda t: C.c_void_p(t.data_ptr())
    mel = torch.empty(int(offs[-1]), 80, device=DEV)
    rc = lib.ssb_mel_diffusion_sample(m._h, p(cond), p(coarse), offs.ctypes.data, len(offs) - 1, None, 3, p(mel), p(ws),
                                      nbytes, C.c_void_p(torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    return rc


def _raw_plms(m, cond, coarse, offs, interval, ws, nbytes):
    p = lambda t: C.c_void_p(t.data_ptr())
    mel = torch.empty(int(offs[-1]), 80, device=DEV)
    rc = lib.ssb_mel_diffusion_sample_plms(m._h, p(cond), p(coarse), offs.ctypes.data, len(offs) - 1, None, 3, interval,
                                           p(mel), p(ws), nbytes, C.c_void_p(torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    return rc


@pytest.mark.parametrize("tc,persistent", PATHS, ids=PATH_IDS)
def test_workspace_bytes_are_exact_at_k_step(tc, persistent):
    """ssb_mel_diffusion_workspace_bytes / ssb_mel_diffusion_plms_workspace_bytes at K_step 37 of 100: the call succeeds
    with the queried size and with its high-water mark (the query adds 4096 bytes of slack to it), and fails one byte
    below that mark - so the dry-run plan is sized by K (the persistent kernel's K (2L + 3) phase table) and not by T."""
    T, K = 100, 37
    m = engine(T, K)
    lens = [300, 1, 77]
    offs = _offs(lens)
    n = int(offs[-1])
    gen = torch.Generator().manual_seed(13)
    cond = torch.randn(n, 256, generator=gen).to(DEV)
    coarse = (-3 + 0.8 * torch.randn(n, 80, generator=gen)).clamp(-6, 0.5).to(DEV)
    try:
        m.set_tensor_cores(tc)
        m.set_persistent(persistent)
        sizes = {}
        for name, query, call in (
                ("ddpm", lib.ssb_mel_diffusion_workspace_bytes, lambda ws, nb: _raw_sample(m, cond, coarse, offs, ws, nb)),
                ("plms", lib.ssb_mel_diffusion_plms_workspace_bytes,
                 lambda ws, nb: _raw_plms(m, cond, coarse, offs, 6, ws, nb))):
            nb = int(query(m._h, offs.ctypes.data, len(lens)))
            assert nb > 4096, name
            ws = torch.empty(nb, dtype=torch.uint8, device=DEV)
            high = nb - 4096
            assert call(ws, nb) == 0 and call(ws, high) == 0, (name, lib.ssb_last_error())
            assert call(ws, high - 1) != 0, name
            assert "workspace too small" in lib.ssb_last_error().decode(), name
            sizes[name] = nb
        m.set_mel_k_step(0)
        full = int(lib.ssb_mel_diffusion_workspace_bytes(m._h, offs.ctypes.data, len(lens)))
    finally:
        _reset(m)
    print(f"tc={tc} persistent={persistent}: workspace bytes at K_step {K}: {sizes}; DDPM at K = T: {full}")
    assert sizes["ddpm"] < full if tc and persistent else sizes["ddpm"] == full  # only the phase table scales with K


def test_k_step_errors():
    """K > T fails at the sampler call (and its workspace query); K < 0 and any K on a ProDiff model fail when set; a PLMS
    interval >= K fails."""
    from stylesinger_b200.engine import pack_batch
    from tests.test_gpu_prodiff import prodiff_engine
    T = 100
    m = engine(T, T + 1)
    offs = np.array([0, 40], np.int32)
    cond = torch.zeros(40, 256, device=DEV)
    coarse = torch.zeros(40, 80, device=DEV)
    msgs = []
    try:
        assert lib.ssb_mel_diffusion_workspace_bytes(m._h, offs.ctypes.data, 1) == 0
        with pytest.raises(SsbError) as e:
            m.mel_diffusion(cond, coarse, offs)
        msgs.append(str(e.value))
        with pytest.raises(SsbError) as e:
            m.mel_diffusion_plms(cond, coarse, offs, 10)
        msgs.append(str(e.value))
        _, meta = golden("ref_kstep")
        with pytest.raises(SsbError) as e:
            m.forward(pack_batch([utt_from_meta(meta)]).to(DEV), seed=1)
        msgs.append(str(e.value))
        m.set_mel_k_step(51)
        m.mel_diffusion_plms(cond, coarse, offs, 50)
        with pytest.raises(SsbError) as e:
            m.mel_diffusion_plms(cond, coarse, offs, 51)
        msgs.append(str(e.value))
        with pytest.raises(SsbError) as e:
            m.set_mel_k_step(-1)
        msgs.append(str(e.value))
        assert m.K == 51  # a refused call changes nothing
        m.set_timesteps(40)  # a later, shorter schedule: K 51 > T 40 fails at the next sampler call
        with pytest.raises(SsbError) as e:
            m.mel_diffusion(cond, coarse, offs)
        msgs.append(str(e.value))
    finally:
        m.set_timesteps(T)
        _reset(m)
    pd = prodiff_engine()
    for K in (0, 8):
        with pytest.raises(SsbError) as e:
            pd.set_mel_k_step(K)
        msgs.append(str(e.value))
    for s in msgs:
        print(s)
    assert all("exceeds the schedule's T" in s for s in (msgs[0], msgs[1], msgs[2], msgs[5]))
    assert "[1, K_step)" in msgs[3] and ">= 0" in msgs[4]
    assert "ProDiff" in msgs[6] and "ProDiff" in msgs[7]


# ---------------------------------------------------------------------------------------------------
def test_inference_driver_reads_k_step_from_hparams():
    """StyleSingerInfer with hparams K_step 51 (timesteps 100) against the oracle on the same injected draws."""
    from stylesinger_b200 import synth
    from stylesinger_b200.engine import pack_batch
    from stylesinger_b200.hparams import DEFAULT_VOCODER_CONFIG, resolve
    from stylesinger_b200.infer import StyleSingerInfer
    from tests.common import vocoder_sd
    T, K, f0_T, seed = 100, 51, 4, 17
    hp = resolve(timesteps=T, K_step=K, f0_timesteps=f0_T)
    u = synth.make_utterance(0.3, utt_idx=12, ref_frames=40, frames=60, phones=7)
    Fr = u["mel2ph"].shape[0]
    ns = O.NoiseSource(seed)
    with torch.no_grad():
        r = O.stylesinger_forward(acoustic_sd(), hp, u["txt_tokens"][None], u["note"][None], u["note_dur"][None],
                                  u["note_type"][None], u["spk_embed"][None], u["emo_embed"][None], u["ref_mels"][None],
                                  u["ref_f0"], ns, mel2ph=u["mel2ph"][None])
    noise, ns2 = engine_noise_from_stream(seed, f0_T, K, Fr, DEV)
    assert ns2.log == ns.log  # the oracle consumed exactly the draws handed to the engine
    drv = StyleSingerInfer(hp, DEV, acoustic_sd(), vocoder_sd(), DEFAULT_VOCODER_CONFIG)
    assert drv.model.K == K and drv.model.T == T
    mel, _, wav, _ = drv.run_device(pack_batch([u]).to(DEV), seed=seed, noise=noise)
    torch.cuda.synchronize()
    err = _maxabs(mel, r["mel_out"][0])
    print(f"StyleSingerInfer, timesteps {T}, K_step {K}: mel_out L-inf vs oracle {err:.3e}; wav {tuple(wav.shape)}")
    assert err < 1e-3 and torch.isfinite(wav).all()
