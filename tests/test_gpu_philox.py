"""The in-kernel Philox noise (seed given, noise pointers NULL) against the NumPy restatement in tests/philox_ref.py.

Direct probes: a hand-made schedule turns a sampler into a noise reader.  Every step gets post_coef1 = 0,
post_coef2 = 1 and sigma = 0 (x_{t-1} = x_t exactly), except the probed step t*, which gets post_coef2 = 0 and
sigma = 1 (x_{t*-1} = that step's noise).  To read x_T instead, row T-1 gets (sqrt_ac, sqrt_1m_ac) = (0, 1).  The
sampler output is then one block of noise: mel_out itself on a ProDiff model, denorm(noise) on a DiffSinger model, z
of the F0 sampler.  Bar: |kernel - restated| <= 4e-6 max(1, |z|) (logf / cospif against float64 Box-Muller).

Equivalence: where a draw cannot be read out (the uniforms, the NSF source) a Philox run must equal a run with the
restated noise injected, and a deliberately wrong layout must miss by at least 100 times the bar."""
import ctypes as C

import numpy as np
import pytest
import torch

from stylesinger_b200 import synth
from stylesinger_b200._lib import check, lib
from stylesinger_b200.engine import step_embedding
from stylesinger_b200.hparams import DEFAULT_VOCODER_CONFIG, resolve
from stylesinger_b200.schedules import multinomial_table, prodiff_table, sampler_table
from tests import philox_ref as P
from tests.common import acoustic_sd, golden, hp_for, vocoder_sd

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
TOL = 4e-6
NEAR1 = 1.0 - 2.0 ** -16
# mel x_T block of test_near_one_uniform_gives_a_positive_radius holds a draw with Philox word 0 >= 0xFFFFFF00
NEAR1_SEED = 24
_M = {}


# ---- models -----------------------------------------------------------------------------------------------------------
def _prodiff_hp(T=8, f0_T=4):
    _, meta = golden("ref_prodiff_T8")
    return resolve(timesteps=T, K_step=T, f0_timesteps=f0_T, **meta["overrides"])


def _model(decoder):
    """A model of this module's own: the probes overwrite its schedule tables."""
    from stylesinger_b200.engine import AcousticModel
    if decoder not in _M:
        if decoder == "prodiff":
            if "prodiff_sd" not in _M:
                _M["prodiff_sd"] = synth.acoustic_state_dict(_prodiff_hp(), seed=0)
            _M[decoder] = AcousticModel(_M["prodiff_sd"], _prodiff_hp())
        else:
            _M[decoder] = AcousticModel(acoustic_sd(), hp_for(8, 8))
    m = _M[decoder]
    m.set_tensor_cores(True)
    m.set_persistent(True)
    m.set_persistent_groups(False)
    return m


def _real_schedule(m, T, f0_T):
    m.T = m.f0_T = None  # a probe table is loaded: make set_timesteps upload the real one
    m.set_timesteps(T, f0_T)


def _probe_schedule(m, which, T, t_star):
    """Load the noise-reading table: t_star = None reads x_T, else step t_star's noise."""
    hp = m.hp
    if which == 0:
        C_ = hp["residual_channels"]
        g = prodiff_table(T, hp["schedule_type"]) if m.mel_decoder == "prodiff" else sampler_table(T, hp["max_beta"])
        mt = None
    else:
        C_ = hp["f0_residual_channels"]
        g = sampler_table(T, hp["f0_max_beta"])
        mt = np.ascontiguousarray(multinomial_table(T, hp["f0_max_beta"]))
    g = np.array(g, np.float32)
    g[:, 2], g[:, 3], g[:, 4] = 0.0, 1.0, 0.0
    if t_star is None:
        g[T - 1, 5], g[T - 1, 6] = 0.0, 1.0
    else:
        g[t_star, 3], g[t_star, 4] = 0.0, 1.0
    g = np.ascontiguousarray(g)
    emb = step_embedding(T, C_)
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    check(lib.ssb_model_set_schedule(m._h, which, T, C.c_void_p(emb.data_ptr()), g.ctypes.data_as(C.c_void_p),
                                     None if mt is None else mt.ctypes.data_as(C.c_void_p), stream), "probe schedule")
    if which == 0:
        m.T = None
    else:
        m.f0_T = None


def _offs(lens):
    return np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)


def _cond(n, seed, cols=256):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(n, cols, generator=g).to(DEV)


def _coarse(n, seed):
    g = torch.Generator().manual_seed(seed)
    return (-3 + 0.8 * torch.randn(n, 80, generator=g)).clamp(-6, 0.5).to(DEV)


# ---- comparison -------------------------------------------------------------------------------------------------------
def _compare_normals(got, want, u1, what, z=None, scale=None, extra=None):
    """Element-wise |got - want| <= TOL max(1, |z|) with z = want, or on a de-normalised output the restated noise z,
    the bar then times `scale` per element plus `extra`.  Reports the largest error overall and on the draws with
    u1 >= 1 - 2^-16."""
    got = np.asarray(got, np.float64)
    want64 = np.asarray(want, np.float64)
    bar = TOL * np.maximum(1.0, np.abs(want64 if z is None else np.asarray(z, np.float64)))
    if scale is not None:
        bar = bar * scale
    if extra is not None:
        bar = bar + extra
    err = np.abs(got - want64)
    near = np.asarray(u1) >= NEAR1
    worst = float((err / bar).max())
    e_near = float(err[near].max()) if near.any() else float("nan")
    print(f"{what}: {err.size} draws, max |d| {float(err.max()):.3e} (max |d|/bar {worst:.3f}); "
          f"{int(near.sum())} draws with u1 >= 1-2^-16, max |d| there {e_near:.3e}")
    assert np.isfinite(got).all()
    assert worst <= 1.0, f"{what}: max |d|/bar = {worst:.3f}"
    return int(near.sum())


def _mel_ctr(offs):
    ti = np.arange(int(offs[-1]), dtype=np.uint64)
    return ti[:, None] * np.uint64(80) + np.arange(80, dtype=np.uint64)[None, :]


def _mel_probe(m, lens, seed, T, blocks, *, grouped=False, stats=False):
    """Read the mel blocks (None = x_T, else the step number) through the mel sampler of `m`; compare each with the
    restatement.  Returns the count of near-1 draws seen."""
    offs = _offs(lens)
    n = int(offs[-1])
    cond = _cond(n, 1)
    coarse = _coarse(n, 2) if m.mel_decoder == "diffsinger" else None
    ctr = _mel_ctr(offs)
    near, step_draws = 0, []
    for t_star in blocks:
        _probe_schedule(m, 0, T, t_star)
        if m.mel_decoder == "prodiff":
            got = m.mel_prodiff(cond, offs, None, seed=seed).cpu().numpy()
        else:
            got = m.mel_diffusion(cond, coarse, offs, None, seed=seed).cpu().numpy()
        st = P.stream_mel_xt() if t_star is None else P.stream_mel_step(t_star)
        if grouped:
            want, u1 = [], []
            for g, (b0, b1) in enumerate(P.persistent_groups(lens)):
                gs = (seed + P.GROUP_SEED_STEP * g) % (1 << 64)
                c = _mel_ctr(_offs(lens[b0:b1]))
                want.append(P.normal(gs, st, c))
                u1.append(P.normal_u1(gs, st, c))
            want, u1 = np.concatenate(want), np.concatenate(u1)
        else:
            want, u1 = P.normal(seed, st, ctr), P.normal_u1(seed, st, ctr)
        what = f"{m.mel_decoder} mel {'x_T' if t_star is None else f't*={t_star}'} ({n} frames)"
        if m.mel_decoder == "prodiff":
            near += _compare_normals(got, want, u1, what)
        else:  # mel_out = (x + 1) / 2 * (max - min) + min in fp32
            smin = acoustic_sd()["postdiff.spec_min"].reshape(-1)[:80].numpy().astype(np.float32)
            smax = acoustic_sd()["postdiff.spec_max"].reshape(-1)[:80].numpy().astype(np.float32)
            d = smax - smin
            want_mel = (want + np.float32(1.0)) / np.float32(2.0) * d + smin
            ulp = np.finfo(np.float32).eps * (np.abs(want_mel) + np.abs(smin) + np.abs(d))
            near += _compare_normals(got, want_mel, u1, what, z=want, scale=np.abs(d) / 2, extra=4 * ulp)
            got = ((got.astype(np.float64) - smin) / d) * 2 - 1  # back to the noise for the statistics
        if stats and t_star is not None:
            step_draws.append((t_star, got))
        elif stats:
            print(f"  x_T statistics: {P.check_stats(got.reshape(1, -1), 'normal')}")
    if step_draws:  # rows in stream order: lag-1 across adjacent step streams
        step_draws.sort(key=lambda p: P.stream_mel_step(p[0]))
        print(f"  step statistics: {P.check_stats(np.stack([x.reshape(-1) for _, x in step_draws]), 'normal')}")
    return near


# ---- direct probes ----------------------------------------------------------------------------------------------------
SMALL = [37, 1500, 2900, 1200]  # 46 row tiles: the persistent kernel's range
LARGE = [2900, 3100, 2700]      # 70 row tiles: per-launch kernels, or two persistent groups


@pytest.mark.parametrize("path", ["persistent", "per_launch_tc", "ffma"])
def test_mel_probe_prodiff(path):
    m = _model("prodiff")
    T = 4
    try:
        m.set_tensor_cores(path != "ffma")
        m.set_persistent(path == "persistent")
        near = _mel_probe(m, SMALL, 1234, T, [None, T - 1, 2, 1, 0], stats=(path == "persistent"))
    finally:
        m.set_tensor_cores(True)
        m.set_persistent(True)
        _real_schedule(m, 8, 4)
    assert near > 0


@pytest.mark.parametrize("grouped", [False, True])
def test_mel_probe_prodiff_beyond_48_tiles(grouped):
    """70 row tiles: the per-launch kernels, or (grouped) the persistent kernel once per group with a group seed."""
    m = _model("prodiff")
    T = 4
    assert len(P.persistent_groups(LARGE)) >= 2
    try:
        m.set_persistent_groups(grouped)
        near = _mel_probe(m, LARGE, 99, T, [None, T - 1, 0], grouped=grouped)
    finally:
        m.set_persistent_groups(False)
        _real_schedule(m, 8, 4)
    assert near > 0


@pytest.mark.parametrize("path", ["persistent", "per_launch_tc"])
def test_mel_probe_diffsinger(path):
    """The q_sample branch of k_mel_q_sample with a coarse mel (x_T = sqrt_ac norm(coarse) + sqrt_1m_ac noise), read
    through denorm_spec; the step blocks of the DDPM sampler with its clip."""
    m = _model("diffsinger")
    T = 4
    try:
        m.set_persistent(path == "persistent")
        _mel_probe(m, SMALL[:3], 4321, T, [None, T - 1, 0])
    finally:
        m.set_persistent(True)
        _real_schedule(m, 8, 8)


def _f0_inputs(n, seed):
    cond = _cond(n, seed)
    lo = torch.full((n,), -0.9, device=DEV)
    hi = torch.full((n,), 0.9, device=DEV)
    return cond, lo, hi


@pytest.mark.parametrize("net", [0, 1])
def test_f0_probe_per_launch(net):
    m = _model("diffsinger")
    T = 4
    lens = [3000, 7001, 10000]
    offs = _offs(lens)
    n = int(offs[-1])
    ti = np.arange(n, dtype=np.uint64)
    cond, lo, hi = _f0_inputs(n, 3)
    seed = 2024 + net
    rows = []
    try:
        for t_star in (None, T - 1, 1, 0):
            _probe_schedule(m, 1, T, t_star)
            z, _ = m.f0_diffusion(net, cond, lo, hi, offs, seed=seed)
            st = P.stream_f0_xt(net) if t_star is None else P.stream_f0_gauss(net, t_star)
            z = z.cpu().numpy()
            _compare_normals(z, P.normal(seed, st, ti), P.normal_u1(seed, st, ti),
                             f"f0 net {net} {'x_T' if t_star is None else f't*={t_star}'}")
            rows.append(z)
    finally:
        _real_schedule(m, 8, 8)
    print("  statistics:", P.check_stats(np.stack(rows), "normal"))


def test_f0_probe_pair_persistent_through_forward():
    """Both F0 nets in the persistent pair kernel (forward, mel diffusion skipped): pitch_pred[:, 0] =
    f0_agnostic / 2 + f0_specific / 2 with f0 = (z + 1) / 2 * 4 + 6, i.e. it reads the two nets' draws summed."""
    from stylesinger_b200.engine import pack_batch
    m = _model("diffsinger")
    T = 4
    specs = [(600, 30, 40, 11), (1500, 60, 40, 12), (900, 40, 40, 13)]
    utts = [synth.make_utterance(f / 187.5, utt_idx=i, ref_frames=r, frames=f, phones=p) for f, p, r, i in specs]
    pb = pack_batch(utts).to(DEV)
    ti = np.arange(pb.total_frames, dtype=np.uint64)
    seed = 31337
    try:
        for t_star in (None, T - 1, 0):
            _probe_schedule(m, 1, T, t_star)
            pp = m.forward(pb, seed=seed, skip_mel_diffusion=True, want=("pitch_pred",))["pitch_pred"][:, 0].cpu().numpy()
            zs = []
            for net in range(2):
                st = P.stream_f0_xt(net) if t_star is None else P.stream_f0_gauss(net, t_star)
                zs.append(P.normal(seed, st, ti))
            f = [(z + np.float32(1)) / np.float32(2) * np.float32(4) + np.float32(6) for z in zs]
            want = (f[1] / np.float32(2) + f[0] / np.float32(2)).astype(np.float64)
            err = np.abs(pp - want)
            bar = TOL * (np.maximum(1, np.abs(zs[0])) + np.maximum(1, np.abs(zs[1]))) + 4e-6
            print(f"pair-persistent F0 {'x_T' if t_star is None else f't*={t_star}'}: max |d| {float(err.max()):.3e}, "
                  f"max |d|/bar {float((err / bar).max()):.3f}")
            assert (err <= bar).all()
    finally:
        _real_schedule(m, 8, 8)


def test_normal_at_the_top_of_the_grid():
    """A normal whose Philox word 0 is >= 0xFFFFFF00 (one in 2^24) has u1 = 1 on the (0, 1] grid of the Box-Muller
    inputs, i.e. radius 0: the kernel must return that finite draw.  NEAR1_SEED puts such a draw in this x_T block."""
    m = _model("prodiff")
    lens = [1000, 2500, 2500]
    offs = _offs(lens)
    seed = NEAR1_SEED
    ctr = _mel_ctr(offs)
    w = P.philox4x32_10(ctr, P.stream_mel_xt(), seed)
    hit = np.nonzero(w[0] >= np.uint32(0xFFFFFF00))
    assert hit[0].size > 0, "NEAR1_SEED no longer selects the top of the grid: the stream plan changed"
    try:
        _probe_schedule(m, 0, 1, None)
        got = m.mel_prodiff(_cond(int(offs[-1]), 5), offs, None, seed=seed).cpu().numpy()
    finally:
        _real_schedule(m, 8, 4)
    want = P.normal_from_words(w[0], w[1])
    for f, c in zip(*hit):
        print(f"frame {f} bin {c}: word0 {int(w[0][f, c]):#010x}, kernel z = {float(got[f, c])!r}, "
              f"restated z = {float(want[f, c])!r}")
    assert np.isfinite(got[hit]).all()
    assert np.abs(got[hit] - want[hit]).max() <= TOL


# F0 net 0, step 0: with seed UNIF1_SEED, the uniform at counter 2 * UNIF1_FRAME + 1 has Philox word 0 >= 0xFFFFFF00
UNIF1_SEED, UNIF1_FRAME, UNIF1_FRAMES = 173, 68127, 100000


def test_top_uniform_stays_below_one_in_the_gumbel_step():
    """The uniform draws promise (0, 1).  The F0 UV step reads them through g = -log(-log(u + 1e-30) + 1e-30): u = 1
    gives g = 69, any u < 1 at most 16.6.  A hand-made multinomial table (one step, slots 0-1 = (0, -30 + ln 2)) makes the
    class-1 log-probability 30 lower than class 0's, so the Gumbel draw of class 1 picks class 1 only if it is ~69, i.e.
    only if the kernel's top uniform were 1.  The control injects 1.0 there and must flip that frame."""
    m = _model("diffsinger")
    offs = _offs([UNIF1_FRAMES // 4] * 4)
    n, f, seed = int(offs[-1]), UNIF1_FRAME, UNIF1_SEED
    w = P.philox4x32_10(2 * f + 1, P.stream_f0_unif(0, 0), seed)[0]
    assert int(w) >= 0xFFFFFF00, "UNIF1_SEED no longer selects the top uniform: the stream plan changed"
    hp = m.hp
    g = np.ascontiguousarray(sampler_table(1, hp["f0_max_beta"]))
    mt = np.zeros((1, 8), np.float32)
    mt[0, 1] = np.float32(-30.0 + np.log(2.0))
    emb = step_embedding(1, hp["f0_residual_channels"])
    cond, lo, hi = _f0_inputs(n, 14)
    try:
        check(lib.ssb_model_set_schedule(m._h, 1, 1, C.c_void_p(emb.data_ptr()), g.ctypes.data_as(C.c_void_p),
                                         mt.ctypes.data_as(C.c_void_p), C.c_void_p(torch.cuda.current_stream().cuda_stream)),
              "uniform probe schedule")
        m.f0_T = None
        gauss = P.f0_gauss_noise(seed, 0, 1, offs)
        unif = P.f0_unif_noise(seed, 0, 1, offs)
        _, uv_philox = m.f0_diffusion(0, cond, lo, hi, offs, seed=seed)
        _, uv_inj = m.f0_diffusion(0, cond, lo, hi, offs, _dev(gauss), _dev(unif))
        one = unif.copy()
        one[0, f, 1] = 1.0
        _, uv_one = m.f0_diffusion(0, cond, lo, hi, offs, _dev(gauss), _dev(one))
    finally:
        _real_schedule(m, 8, 8)
    uv_philox, uv_inj, uv_one = (x.cpu().numpy() for x in (uv_philox, uv_inj, uv_one))
    print(f"frame {f}: restated u = {float(unif[0, f, 1])!r}; uv Philox {uv_philox[f]}, injected {uv_inj[f]}, "
          f"injected with u = 1: {uv_one[f]}; class-1 frames overall: Philox {int(uv_philox.sum())}, u = 1 control "
          f"{int(uv_one.sum())}")
    assert float(unif[0, f, 1]) == 1.0 - 2.0 ** -24
    assert uv_one[f] == 1, "control: a uniform of exactly 1 must force class 1 under this table"
    assert np.array_equal(uv_philox, uv_inj)
    assert uv_philox[f] == 0


def test_mel_steps_never_reuse_the_f0_draws():
    """T_mel = 1000 and the F0 nets share the seed: the first reverse mel step (t = 999) must not draw what F0 net 0
    draws for its x_T.  Both are read from the kernels and checked against the restatement."""
    m = _model("prodiff")
    lens = [160]
    offs = _offs(lens)
    seed = 4242
    cond, lo, hi = _f0_inputs(160, 6)
    try:
        _probe_schedule(m, 0, 1000, 999)
        mel = m.mel_prodiff(cond, offs, None, seed=seed).cpu().numpy()
        _probe_schedule(m, 1, 4, None)
        z, _ = m.f0_diffusion(0, cond, lo, hi, offs, seed=seed)
        z = z.cpu().numpy()
    finally:
        _real_schedule(m, 8, 4)
    ctr = _mel_ctr(offs)
    st = P.stream_mel_step(999)
    _compare_normals(mel, P.normal(seed, st, ctr), P.normal_u1(seed, st, ctr), "mel t*=999 of T=1000")
    ti = np.arange(160, dtype=np.uint64)
    _compare_normals(z, P.normal(seed, P.stream_f0_xt(0), ti), P.normal_u1(seed, P.stream_f0_xt(0), ti), "f0 net 0 x_T")
    same = int((mel.reshape(-1)[:160] == z).sum())
    print(f"mel step 999 (frames 0-1) vs f0 x_T (frames 0-159): {same} of 160 draws equal")
    assert same == 0


# ---- equivalence with injected noise ----------------------------------------------------------------------------------
def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def _shift_steps(a):
    """Wrong layout: the step blocks 1..end shifted by one (x_T block kept)."""
    b = a.copy()
    b[1:] = np.roll(a[1:], 1, axis=0)
    return b


def _miss(got, want, bar_fn):
    got = np.asarray(got, np.float64)
    want = np.asarray(want, np.float64)
    return float((np.abs(got - want) / bar_fn(want)).max())


def _mel_bar(x):
    return 1e-4 * np.maximum(1.0, np.abs(x))


@pytest.mark.parametrize("path", ["per_launch", "pair_persistent"])
def test_f0_sampler_philox_equals_injected(path):
    """F0 samplers (real schedule, T = 8): uv identical and z within 1e-4 between Philox and the restated injection."""
    from stylesinger_b200.engine import pack_batch
    m = _model("diffsinger")
    T = 8
    _real_schedule(m, 8, T)
    seed = 77
    if path == "per_launch":
        lens = [37, 150, 97]
        offs = _offs(lens)
        cond, lo, hi = _f0_inputs(int(offs[-1]), 8)
        for net in range(2):
            g = P.f0_gauss_noise(seed, net, T, offs)
            u = P.f0_unif_noise(seed, net, T, offs)
            za, uva = m.f0_diffusion(net, cond, lo, hi, offs, seed=seed)
            zb, uvb = m.f0_diffusion(net, cond, lo, hi, offs, _dev(g), _dev(u))
            zc, _ = m.f0_diffusion(net, cond, lo, hi, offs, _dev(_shift_steps(g)), _dev(np.roll(u, 1, axis=0)))
            e = _maxabs(za, zb)
            miss = _maxabs(zc, zb) / 1e-4
            flips = int((uva != uvb).sum())
            print(f"per-launch F0 net {net}: z max |d| {e:.3e} (bar 1e-4), uv flips {flips}; wrong layout misses by {miss:.0f}x")
            assert flips == 0 and e < 1e-4 and miss >= 100
        return
    specs = [(150, 11, 40, 21), (97, 9, 33, 22), (40, 6, 50, 23)]
    utts = [synth.make_utterance(f / 187.5, utt_idx=i, ref_frames=r, frames=f, phones=p) for f, p, r, i in specs]
    pb = pack_batch(utts).to(DEV)
    offs = pb.frame_offsets
    noise = P.acoustic_noise(seed, 8, T, offs)
    inj = {k: [_dev(x) for x in noise[k]] for k in ("f0_gauss", "f0_unif")}
    bad = {"f0_gauss": [_dev(_shift_steps(x)) for x in noise["f0_gauss"]],
           "f0_unif": [_dev(np.roll(x, 1, axis=0)) for x in noise["f0_unif"]]}
    run = lambda nz, s=0: m.forward(pb, noise=nz, seed=s, skip_mel_diffusion=True, want=("pitch_pred",))["pitch_pred"].clone()
    a, b, c = run(None, seed), run(inj), run(bad)
    e = _maxabs(a[:, 0], b[:, 0])
    flips = int((a[:, 1] != b[:, 1]).sum())
    miss = _maxabs(c[:, 0], b[:, 0]) / 1e-4
    print(f"pair-persistent F0: pitch max |d| {e:.3e} (bar 1e-4), uv flips {flips}; wrong layout misses by {miss:.0f}x")
    assert flips == 0 and e < 1e-4 and miss >= 100


def test_full_forward_philox_equals_injected():
    """ssb_acoustic_forward, T = 8 and f0_T = 8, ragged batch of 3: mel within 1e-4 max(1, |mel|), f0_denorm within
    5e-2 Hz."""
    from stylesinger_b200.engine import pack_batch
    m = _model("diffsinger")
    _real_schedule(m, 8, 8)
    specs = [(150, 11, 40, 31), (97, 9, 33, 32), (40, 6, 50, 33)]
    utts = [synth.make_utterance(f / 187.5, utt_idx=i, ref_frames=r, frames=f, phones=p) for f, p, r, i in specs]
    pb = pack_batch(utts).to(DEV)
    seed = 555
    noise = P.acoustic_noise(seed, 8, 8, pb.frame_offsets)
    inj = {"f0_gauss": [_dev(x) for x in noise["f0_gauss"]], "f0_unif": [_dev(x) for x in noise["f0_unif"]],
           "mel": _dev(noise["mel"])}
    bad = {"f0_gauss": [_dev(_shift_steps(x)) for x in noise["f0_gauss"]], "f0_unif": inj["f0_unif"],
           "mel": _dev(_shift_steps(noise["mel"]))}
    out = lambda nz, s=0: {k: v.cpu().numpy() for k, v in m.forward(pb, noise=nz, seed=s).items()}
    a, b, c = out(None, seed), out(inj), out(bad)
    e_mel = _miss(a["mel_out"], b["mel_out"], _mel_bar)
    e_f0 = float(np.abs(a["f0_denorm"].astype(np.float64) - b["f0_denorm"]).max())
    m_mel = _miss(c["mel_out"], b["mel_out"], _mel_bar)
    m_f0 = float(np.abs(c["f0_denorm"].astype(np.float64) - b["f0_denorm"]).max()) / 5e-2
    print(f"forward: mel max |d|/bar {e_mel:.3e}, f0_denorm max |d| {e_f0:.3e} Hz; wrong layout misses by "
          f"{m_mel:.0f}x (mel), {m_f0:.0f}x (f0)")
    assert e_mel <= 1.0 and e_f0 < 5e-2
    assert m_mel >= 100 and m_f0 >= 100


def test_plms_and_prodiff_philox_equal_injected():
    lens = [150, 97, 40]
    offs = _offs(lens)
    n = int(offs[-1])
    seed = 808
    m = _model("diffsinger")
    _real_schedule(m, 8, 8)
    cond, coarse = _cond(n, 9), _coarse(n, 10)
    q = P.mel_noise(seed, 8, offs, steps=[])[0]
    a = m.mel_diffusion_plms(cond, coarse, offs, 2, None, seed=seed).cpu().numpy()
    b = m.mel_diffusion_plms(cond, coarse, offs, 2, _dev(q)).cpu().numpy()
    c = m.mel_diffusion_plms(cond, coarse, offs, 2, _dev(np.roll(q, 1, axis=0))).cpu().numpy()
    e, miss = _miss(a, b, _mel_bar), _miss(c, b, _mel_bar)
    print(f"PLMS: mel max |d|/bar {e:.3e}; wrong layout misses by {miss:.0f}x")
    assert e <= 1.0 and miss >= 100
    m = _model("prodiff")
    _real_schedule(m, 8, 4)
    noise = P.mel_noise(seed, 8, offs)
    a = m.mel_prodiff(cond, offs, None, seed=seed).cpu().numpy()
    b = m.mel_prodiff(cond, offs, _dev(noise)).cpu().numpy()
    c = m.mel_prodiff(cond, offs, _dev(_shift_steps(noise))).cpu().numpy()
    e, miss = _miss(a, b, _mel_bar), _miss(c, b, _mel_bar)
    print(f"ProDiff: mel max |d|/bar {e:.3e}; wrong layout misses by {miss:.0f}x")
    assert e <= 1.0 and miss >= 100


@pytest.mark.parametrize("tc", [True, False])
def test_vocoder_philox_equals_injected(tc):
    """NSF source: the random initial phases (rand_ini) and the additive source noise, tensor-core and FFMA paths."""
    from stylesinger_b200.engine import Vocoder
    if "voc" not in _M:
        _M["voc"] = Vocoder(vocoder_sd(), DEFAULT_VOCODER_CONFIG)
    v = _M["voc"]
    v.set_tensor_cores(tc)
    lens = [17, 40, 25]
    offs = _offs(lens)
    n = int(offs[-1])
    gen = torch.Generator().manual_seed(12)
    mel = (-3.0 + 0.8 * torch.randn(n, 80, generator=gen)).clamp(-6, 1.5).to(DEV)
    f0 = 150 + 350 * torch.rand(n, generator=gen)
    f0[2:5] = 0
    f0[30:36] = 0
    f0 = f0.to(DEV)
    seed = 4711
    ini = P.vocoder_rand_ini(seed, len(lens))
    src = P.vocoder_src_noise(seed, offs, v.hop)
    try:
        a = v.generate(mel, f0, offs, seed=seed).cpu().numpy()
        b = v.generate(mel, f0, offs, rand_ini=_dev(ini), src_noise=_dev(src)).cpu().numpy()
        c = v.generate(mel, f0, offs, rand_ini=_dev(ini[[1, 0, 2]]), src_noise=_dev(np.roll(src, 1, axis=0))).cpu().numpy()
    finally:
        v.set_tensor_cores(True)
    e = float(np.abs(a.astype(np.float64) - b).max())
    miss = float(np.abs(c.astype(np.float64) - b).max()) / 1e-5
    print(f"vocoder tc={tc}: wav max |d| {e:.3e} (bar 1e-5); wrong layout misses by {miss:.0f}x")
    assert e < 1e-5 and miss >= 100


def _maxabs(a, b):
    a = a.detach().cpu().numpy() if isinstance(a, torch.Tensor) else np.asarray(a)
    b = b.detach().cpu().numpy() if isinstance(b, torch.Tensor) else np.asarray(b)
    return float(np.abs(a.astype(np.float64) - b.astype(np.float64)).max())
