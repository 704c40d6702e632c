"""The ProDiff and PLMS mel samplers against their float64 restatement (tests/sampler_oracle.py), on every kernel path,
at bench size and at tile edges.  The batches are tests/test_gpu_denoisers.py's: one row tile (127 frames), ragged
(lengths 1, 2, 3, 8, 9, 16, 17, 127, 128, 129, 700: 17 row tiles), tiles48 (48 utterances of one row tile each), mid
(71 row tiles) and the bench's 64 utterances (890 row tiles).  The DiffSinger model's forward gives diff_cond and
coarse_mel, the ProDiff model's forward decoder_inp.

(a) ProDiff (ssb_mel_prodiff_sample), T = 8 and T = 4 (set_timesteps re-tables the vpsde schedule), injected noise: the
persistent single launch (<= 48 row tiles), per-launch tensor cores and FFMA.  The float64 chain starts from
x_T = noise with no coarse mel, takes the net's output as x0 with no clip, and does not denormalise.
(b) ProDiff in Philox mode: the persistent single launch against philox_ref.mel_noise, and the persistent groups
(set_persistent_groups, bench lengths: 21 groups) against philox_ref.mel_noise_grouped, comparing the first and last
utterance of every fourth group and the shortest and longest.
(c) PLMS (ssb_mel_diffusion_sample_plms) at (K_step, interval) in {(100, 10), (100, 7), (37, 5), (6, 1), (4, 3),
(2, 1)} of T = 100, injected q_sample draw, per-launch tensor cores (with the persistent switch on: PLMS has no
persistent kernel) and FFMA; in Philox mode at (37, 5), whose draw is block 0 of philox_ref.mel_noise.  The
configurations reach every history order (0: the second-order start, then 1 to 3), wrap the 3-slot history ring, read
alphas_cumprod from a K-step slice of the T-step table, clamp a_prev at t = 0, and include intervals that do not
divide K (t0 = 98, 35, 3).
(d) Through ssb_acoustic_forward: DiffSinger with pndm_speedup = 10 and an injected q_sample draw, and ProDiff with the
persistent groups and a seed.  mel_out must be bit-identical to the sampler entry called on the forward's own
diff_cond / coarse_mel (decoder_inp) with the same noise or seed, and match the float64 chain.

Every sampler call asserts the tensor-core GEMM variants and the number of kernels it launched.  Errors on the 8 rows at
each utterance end are reported apart from the interior; an edge error above 4x the interior error fails whatever the
bar.  Small and mid utterances also run as their own B = 1 calls: FFMA must be bit-identical, tensor cores within a
bar.  The float64 chains run on the CPU, equal-length utterances as one batch; at bench size a named subset is compared
(shortest, longest, first, last, every sixteenth), and in mid the three utterances of 1500 frames and more are left out.

Errors are max |a - b| / max(1, |b|).  Each bar is at most 4x the largest error measured on an H100 SXM (80 GB,
700 W), with the measured value beside it; each test prints what it measured."""
import hashlib
import time

import numpy as np
import pytest
import torch

from tests import philox_ref as P
from tests import sampler_oracle as SO
from tests import test_gpu_denoisers as D
from tests.common import acoustic_engine, acoustic_sd, hp_for, prodiff_hp, prodiff_sd
from tests.gpu_checks import (Err, check_variants, cond_gemm, count, frame_offsets, launched, net_dims, ntiles, rel,
                              split, step_gemms)

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
T = 100  # the DiffSinger schedule the PLMS configurations slice
SEED = 5  # the ProDiff forward's seed (decoder_inp of every ProDiff batch, and the Philox tests' sampler seed)

# measured on an H100 80GB HBM3 (SXM, 700 W power limit); the largest error over sizes is beside each bar.  0 means
# bit-identical.  The PLMS error grows with the steps taken at large t, where get_x_pred's eps coefficient is largest
# (1 / sqrt(alphas_cumprod) reaches 3.4 at t = 99): per-evaluation tensor-core error of a few 1e-6 (as
# tests/test_gpu_denoisers.py measures) ends near 5e-5 after the 10 - 15 steps of K = 100, but near 1e-6 for K <= 6.
# The Philox draws of philox_ref.normal differ from the kernel's by a few ulp; that is not measurable here (Philox and
# injected noise give the same errors to within 10 %).
BARS = {
    "prodiff": {"ffma": 5e-6,                    # 1.5e-6
                "tc": 2e-5,                      # 5.5e-6
                "persistent": 2e-5},             # 5.6e-6
    "prodiff_philox": {"persistent": 2e-5},      # 5.6e-6 (the groups at bench size)
    "plms": {(100, 10): {"ffma": 2e-5,           # 5.2e-6
                         "tc": 1e-4},            # 4.6e-5
             (100, 7): {"ffma": 2.4e-5,          # 6.0e-6
                        "tc": 1e-4},             # 6.1e-5
             (37, 5): {"ffma": 8e-6,             # 2.1e-6
                       "tc": 4e-5},              # 1.0e-5
             (6, 1): {"ffma": 6.5e-6,            # 1.6e-6
                      "tc": 9e-6},               # 2.3e-6
             (4, 3): {"ffma": 5.3e-6,            # 1.3e-6
                      "tc": 6.5e-6},             # 1.6e-6
             (2, 1): {"ffma": 5e-6,              # 1.3e-6
                      "tc": 5.5e-6}},            # 1.4e-6
    "plms_philox": {"tc": 3.4e-5},               # 8.6e-6 (37, 5)
    "solo": {"ffma": 0.0,
             "tc": 5.5e-5},                      # 1.4e-5 (PLMS K = 100, interval 7, mid: CTA-pair kernels vs B = 1)
    "forward": {"prodiff": 2e-5,                 # 4.9e-6
                "plms": 1e-4},                   # 5.2e-5 (interval 10)
}
SIZES = ["one_tile", "ragged", "tiles48", "mid"]
PLMS = [(100, 10), (100, 7), (37, 5), (6, 1), (4, 3), (2, 1)]
SOLO = ("ragged", "mid")  # sizes whose utterances also run as B = 1 calls


def _compared(name, lens):
    """Utterances compared against float64 (the float64 chains run on the CPU): all, except in mid, whose three
    utterances of 1500 frames and more are left out, and at bench size, where the shortest, the longest, the first, the
    last and every sixteenth are compared."""
    if name == "mid":
        return [i for i, n in enumerate(lens) if n < 1500]
    if name == "bench":
        return sorted({int(np.argmin(lens)), int(np.argmax(lens)), 0, len(lens) - 1} | set(range(0, len(lens), 16)))
    return list(range(len(lens)))


# ---------------------------------------------------------------------------------------------------------------------
# inputs
def ds_batch(name):
    return D._one_tile() if name == "one_tile" else D.batch(name)


_E, _PB = {}, {}


def prodiff_engine(T_=8):
    from stylesinger_b200.engine import AcousticModel
    if "m" not in _E:
        _E["m"] = AcousticModel(prodiff_sd(), prodiff_hp())
    m = _E["m"]
    m.set_timesteps(T_)
    m.set_tensor_cores(True)
    m.set_persistent(True)
    m.set_persistent_groups(False)
    return m


def pd_batch(name):
    """{lens, offs, pb, cond = decoder_inp of the ProDiff forward with seed SEED}, memoised; ds_batch's utterances."""
    if name not in _PB:
        from stylesinger_b200.engine import pack_batch
        if name == "one_tile":
            utts = [u for u in D.batch("small")["utts"] if len(u["mel2ph"]) == 127]
        else:
            utts = D.batch(name)["utts"]
        lens = [len(u["mel2ph"]) for u in utts]
        pb = pack_batch(utts).to(DEV)
        out = prodiff_engine().forward(pb, seed=SEED, skip_mel_diffusion=True, want=("decoder_inp",))
        _PB[name] = dict(lens=lens, offs=frame_offsets(lens), pb=pb, cond=out["decoder_inp"].clone())
    return _PB[name]


# ---------------------------------------------------------------------------------------------------------------------
# float64 chains, memoised on their inputs; utterances of one length run as one float64 batch
_CH = {}
_T64 = [0.0]


def _key(*ts):
    return tuple(hashlib.sha1(t.contiguous().numpy().tobytes()).hexdigest() for t in ts)


def _many(tag, chain, dims, items):
    """chain(*stacked) -> {"mel": [B,F,80]} for items = one tuple of per-utterance tensors each; stacked along dims."""
    keys = [tag + _key(*it) for it in items]
    todo = {}
    for k, it in zip(keys, items):
        if k not in _CH:
            todo.setdefault(it[0].shape[0], {})[k] = it
    t0 = time.time()
    for group in todo.values():
        its = list(group.values())
        mel = chain(*[torch.stack([it[j] for it in its], dim=d) for j, d in enumerate(dims)])["mel"]
        for b, k in enumerate(group):
            _CH[k] = mel[b]
    _T64[0] += time.time() - t0
    return [_CH[k] for k in keys]


def prodiff64(hp, items):
    """items: (decoder_inp [F,256], noise [T+1,F,80]) per utterance."""
    return _many(("prodiff", hp["timesteps"]), lambda c, n: SO.prodiff_chain64(c, hp, n), (0, 1), items)


def plms64(K, interval, items):
    """items: (diff_cond [F,256], coarse_mel [F,80], q [F,80]) per utterance."""
    hp = dict(hp_for(T), K_step=K)
    return _many(("plms", K, interval), lambda c, co, q: SO.plms_chain64(c, co, hp, K, interval, q), (0, 0, 0), items)


def _f64_clock():
    t = _T64[0]
    _T64[0] = 0.0
    return t


def _check_launches(tag, path, got, launches, want):
    check_variants(tag, got, want)
    print(f"{tag}: {launches} launches")
    if path == "persistent":
        assert launches < 16, (tag, launches)


def _solo(tag, path, lens, offs, ys, run):
    """Each utterance as its own B = 1 call, run(i, a, e) -> [n, 80]: FFMA bit-identical, tensor cores within a bar."""
    worst = 0.0
    for i in range(len(lens)):
        a, e = int(offs[i]), int(offs[i + 1])
        y1 = run(i, a, e).cpu()
        worst = max(worst, float(rel(y1, ys[i]).max()))
        if path == "ffma":
            assert torch.equal(y1, ys[i]), (tag, i)
    bar = BARS["solo"]["ffma" if path == "ffma" else "tc"]
    print(f"{tag}: solo B=1 calls {worst:.3e} (bar {bar:.1e})")
    assert worst <= bar, (tag, worst)


# ---------------------------------------------------------------------------------------------------------------------
# (a) ProDiff, injected noise
@pytest.mark.parametrize("T_,size", [(8, s) for s in SIZES + ["bench"]] + [(4, s) for s in SIZES])
def test_prodiff_sampler_matches_float64(T_, size):
    b = pd_batch(size)
    m = prodiff_engine(T_)
    hp = prodiff_hp(T_)
    lens, offs = b["lens"], b["offs"]
    nt, n = ntiles(lens), int(offs[-1])
    noise = torch.randn(T_ + 1, n, 80, generator=torch.Generator().manual_seed(100 + T_))
    nd = noise.to(DEV)
    cs = split(b["cond"], offs)
    try:
        for path in (["persistent"] if nt <= 48 else []) + ["tc", "ffma"]:
            tag = f"prodiff T={T_} {size} {path} ({len(lens)} utterances, {nt} row tiles)"
            m.set_tensor_cores(path != "ffma")
            m.set_persistent(path == "persistent")
            mel, got, launches = launched(lambda: m.mel_prodiff(b["cond"], offs, nd).clone())
            want = {"persistent": count(cond_gemm(0), nt), "tc": count(cond_gemm(0) + step_gemms(0) * T_, nt),
                    "ffma": {}}[path]
            _check_launches(tag, path, got, launches, want)
            ys = split(mel, offs)
            err = Err()
            pick = _compared(size, lens)
            refs = prodiff64(hp, [(cs[i], noise[:, int(offs[i]):int(offs[i + 1])]) for i in pick])
            for i, r in zip(pick, refs):
                err.add(i, ys[i], r)
            if size in SOLO and path != "persistent":
                _solo(tag, path, lens, offs, ys, lambda i, a, e: m.mel_prodiff(
                    b["cond"][a:e].contiguous(), frame_offsets([e - a]), nd[:, a:e].contiguous()))
            err.report(tag, BARS["prodiff"][path])
    finally:
        prodiff_engine(8)
    print(f"prodiff T={T_} {size}: float64 reference took {_f64_clock():.1f} s")


# ---------------------------------------------------------------------------------------------------------------------
# (b) ProDiff, Philox
@pytest.mark.parametrize("size", ["ragged", "bench"])
def test_prodiff_philox_matches_float64(size):
    """ragged: one persistent launch keyed by the call's seed; bench: one persistent launch per group of <= 48 row
    tiles, group g keyed seed + 0x9E3779B97F4A7C15 g with rows counted inside the group."""
    b = pd_batch(size)
    m = prodiff_engine()
    hp = prodiff_hp()
    lens, offs = b["lens"], b["offs"]
    grouped = size == "bench"
    groups = P.persistent_groups(lens) if grouped else [(0, len(lens))]
    if grouped:
        noise, ng = P.mel_noise_grouped(SEED, 8, lens)
        assert ng == len(groups) > 1
        pick = sorted({int(np.argmin(lens)), int(np.argmax(lens))} | {i for g in groups[::4] for i in (g[0], g[1] - 1)})
    else:
        noise, pick = P.mel_noise(SEED, 8, offs), range(len(lens))
    noise = torch.from_numpy(noise)
    tag = f"prodiff Philox {size} {'persistent groups' if grouped else 'persistent'} ({len(lens)} utterances, " \
          f"{ntiles(lens)} row tiles, {len(groups)} launches of the persistent kernel)"
    try:
        m.set_persistent_groups(grouped)
        mel, got, launches = launched(lambda: m.mel_prodiff(b["cond"], offs, None, seed=SEED).clone())
    finally:
        m.set_persistent_groups(False)
    want = {}
    for b0, b1 in groups:
        for k, v in count(cond_gemm(0), ntiles(lens[b0:b1])).items():
            want[k] = want.get(k, 0) + v
    _check_launches(tag, "groups", got, launches, want)
    assert launches < 16 * len(groups), (tag, launches)
    ys, cs = split(mel, offs), split(b["cond"], offs)
    err = Err()
    for i, r in zip(pick, prodiff64(hp, [(cs[i], noise[:, int(offs[i]):int(offs[i + 1])]) for i in pick])):
        err.add(i, ys[i], r)
    print(f"{tag}: compared utterances {list(pick)}")
    err.report(tag, BARS["prodiff_philox"]["persistent"])
    print(f"prodiff Philox {size}: float64 reference took {_f64_clock():.1f} s")


# ---------------------------------------------------------------------------------------------------------------------
# (c) PLMS
def _plms_cases():
    return [(K, k, s) for K, k in PLMS for s in SIZES] + [(100, 10, "bench"), (37, 5, "bench")]


@pytest.mark.parametrize("K,interval,size", _plms_cases())
def test_plms_sampler_matches_float64(K, interval, size):
    b = ds_batch(size)
    m = acoustic_engine(T, D.F0_T)
    lens, offs = b["lens"], b["offs"]
    nt, n = ntiles(lens), int(offs[-1])
    q = torch.randn(n, 80, generator=torch.Generator().manual_seed(1000 + 7 * K + interval))
    qd = q.to(DEV)
    cs, co = split(b["cond"], offs), split(b["coarse"], offs)
    evals = SO.plms_evals(K, interval)
    m.set_mel_k_step(K)
    try:
        for path in ("tc", "ffma"):
            tag = f"plms K={K} interval={interval} {size} {path} ({len(lens)} utterances, {nt} row tiles, " \
                  f"{evals} evals)"
            m.set_tensor_cores(path == "tc")
            m.set_persistent(True)
            mel, got, launches = launched(
                lambda: m.mel_diffusion_plms(b["cond"], b["coarse"], offs, interval, qd).clone())
            _check_launches(tag, path, got, launches,
                            count(cond_gemm(0) + step_gemms(0) * evals, nt) if path == "tc" else {})
            ys = split(mel, offs)
            err = Err()
            pick = _compared(size, lens)
            refs = plms64(K, interval, [(cs[i], co[i], q[int(offs[i]):int(offs[i + 1])]) for i in pick])
            for i, r in zip(pick, refs):
                err.add(i, ys[i], r)
            if size in SOLO:
                _solo(tag, path, lens, offs, ys, lambda i, a, e: m.mel_diffusion_plms(
                    b["cond"][a:e].contiguous(), b["coarse"][a:e].contiguous(), frame_offsets([e - a]), interval,
                    qd[a:e].contiguous()))
            err.report(tag, BARS["plms"][(K, interval)][path])
    finally:
        m.set_tensor_cores(True)
        m.set_mel_k_step(0)
    print(f"plms K={K} interval={interval} {size}: float64 reference took {_f64_clock():.1f} s")


def test_plms_philox_matches_float64():
    """(37, 5) on tensor cores: the q_sample draw is block 0 of philox_ref.mel_noise (stream mel x_T, counter row = the
    frame's tight row in the call)."""
    K, interval = 37, 5
    b = ds_batch("ragged")
    m = acoustic_engine(T, D.F0_T)
    lens, offs = b["lens"], b["offs"]
    q = torch.from_numpy(P.mel_noise(SEED, K, offs, steps=[])[0])
    cs, co = split(b["cond"], offs), split(b["coarse"], offs)
    tag = f"plms Philox K={K} interval={interval} ragged tc ({len(lens)} utterances, {ntiles(lens)} row tiles)"
    m.set_mel_k_step(K)
    try:
        mel, got, launches = launched(lambda: m.mel_diffusion_plms(b["cond"], b["coarse"], offs, interval, None,
                                                                   seed=SEED).clone())
    finally:
        m.set_mel_k_step(0)
    _check_launches(tag, "tc", got, launches,
                    count(cond_gemm(0) + step_gemms(0) * SO.plms_evals(K, interval), ntiles(lens)))
    err = Err()
    refs = plms64(K, interval, [(cs[i], co[i], q[int(offs[i]):int(offs[i + 1])]) for i in range(len(lens))])
    for i, (y, r) in enumerate(zip(split(mel, offs), refs)):
        err.add(i, y, r)
    err.report(tag, BARS["plms_philox"]["tc"])
    print(f"plms Philox: float64 reference took {_f64_clock():.1f} s")


# ---------------------------------------------------------------------------------------------------------------------
# (d) through ssb_acoustic_forward
def _few(lens):
    return sorted({0, int(np.argmin(lens)), int(np.argmax(lens))})


_PLMS_E = {}


@pytest.mark.parametrize("size", ["ragged", "bench"])
def test_forward_plms_matches_sampler_and_float64(size):
    """hparams['pndm_speedup'] = 10 at T = K_step = 100; the injected mel noise supplies only the q_sample draw."""
    from stylesinger_b200.engine import AcousticModel
    interval = 10
    if "m" not in _PLMS_E:
        _PLMS_E["m"] = AcousticModel(acoustic_sd(), dict(hp_for(T, D.F0_T), pndm_speedup=interval))
    m = _PLMS_E["m"]
    b = ds_batch(size)
    lens, offs, n = b["lens"], b["offs"], int(b["offs"][-1])
    q = torch.randn(n, 80, generator=torch.Generator().manual_seed(77))
    qd = q[None].to(DEV).contiguous()
    out, got, launches = launched(lambda: m.forward(b["pb"], noise={"mel": qd}, seed=1,
                                                    want=("mel_out", "diff_cond", "coarse_mel")))
    evals = SO.plms_evals(T, interval)
    tag = f"forward plms interval={interval} {size} ({len(lens)} utterances, {ntiles(lens)} row tiles)"
    want = count(cond_gemm(0) + step_gemms(0) * evals, ntiles(lens))
    print(f"{tag}: tensor-core GEMM variants launched {got}, {launches} launches")
    for k, v in want.items():  # the forward's other GEMMs may use the same variants; the denoiser's are all there
        assert got.get(k, 0) >= v, (tag, k, got, want)
    direct = m.mel_diffusion_plms(out["diff_cond"], out["coarse_mel"], offs, interval, qd[0])
    assert torch.equal(out["mel_out"], direct), tag
    cs, co, ys = split(out["diff_cond"], offs), split(out["coarse_mel"], offs), split(out["mel_out"], offs)
    err = Err()
    pick = _few(lens)
    for i, r in zip(pick, plms64(T, interval, [(cs[i], co[i], q[int(offs[i]):int(offs[i + 1])]) for i in pick])):
        err.add(i, ys[i], r)
    print(f"{tag}: mel_out bit-identical to ssb_mel_diffusion_sample_plms; float64 on utterances {_few(lens)}")
    err.report(tag, BARS["forward"]["plms"])
    print(f"forward plms {size}: float64 reference took {_f64_clock():.1f} s")


@pytest.mark.parametrize("size", ["ragged", "bench"])
def test_forward_prodiff_matches_sampler_and_float64(size):
    """ProDiff forward with a seed and the persistent groups switched on (bench: 21 groups; ragged: one launch)."""
    b = pd_batch(size)
    m = prodiff_engine()
    hp = prodiff_hp()
    lens, offs = b["lens"], b["offs"]
    try:
        m.set_persistent_groups(True)
        out, got, launches = launched(lambda: m.forward(b["pb"], seed=SEED, want=("mel_out", "decoder_inp")))
        direct = m.mel_prodiff(out["decoder_inp"], offs, None, seed=SEED)
    finally:
        m.set_persistent_groups(False)
    tag = f"forward prodiff {size} ({len(lens)} utterances, {ntiles(lens)} row tiles)"
    print(f"{tag}: tensor-core GEMM variants launched {got}, {launches} launches")
    groups = P.persistent_groups(lens) if ntiles(lens) > 48 else [(0, len(lens))]
    for b0, b1 in groups:  # each group's hoisted conditioner; the forward's other GEMMs may add to these variants
        for k, v in count(cond_gemm(0), ntiles(lens[b0:b1])).items():
            assert got.get(k, 0) >= v, (tag, k, got)
    # the mel denoiser's layers ran inside the persistent kernel: the only residual GEMMs are the F0 samplers' (per
    # launch above 48 row tiles, both nets' f0_timesteps steps)
    f0_res = 2 * D.F0_T * net_dims(1)[1] if ntiles(lens) > 48 else 0
    assert sum(v for k, v in got.items() if "RES_SKIP" in k) == f0_res, (tag, got)
    assert torch.equal(out["mel_out"], direct), tag
    assert torch.equal(out["decoder_inp"], b["cond"]), tag  # same seed: the same F0 draws and decoder_inp
    if size == "bench":
        noise, _ = P.mel_noise_grouped(SEED, 8, lens)
    else:
        noise = P.mel_noise(SEED, 8, offs)
    noise = torch.from_numpy(noise)
    cs, ys = split(out["decoder_inp"], offs), split(out["mel_out"], offs)
    err = Err()
    pick = _few(lens)
    for i, r in zip(pick, prodiff64(hp, [(cs[i], noise[:, int(offs[i]):int(offs[i + 1])]) for i in pick])):
        err.add(i, ys[i], r)
    print(f"{tag}: mel_out bit-identical to ssb_mel_prodiff_sample; float64 on utterances {_few(lens)}")
    err.report(tag, BARS["forward"]["prodiff"])
    print(f"forward prodiff {size}: float64 reference took {_f64_clock():.1f} s")
