"""Pin the float64 ProDiff and PLMS samplers (tests/sampler_oracle.py) on the CPU: step by step against the fp32 oracles
on the same draws (every denoiser input of the fp32 run is recorded), and the final mel against the unmodified
reference's fixtures.  The PLMS configurations are the GPU file's: K_step 100, 37, 6, 4 and 2 of T = 100, with intervals
that do and do not divide K."""
import contextlib

import numpy as np
import pytest
import torch

from oracle import stylesinger_oracle as O
from tests import sampler_oracle as SO
from tests.common import acoustic_sd, golden, hp_for, prodiff_hp, prodiff_sd

TOL = 2e-5  # the fp32 oracle's bar against the reference (tests/test_oracle_golden.py)
PLMS_CONFIGS = [(100, 10), (100, 7), (37, 5), (6, 1), (4, 3), (2, 1)]  # (K_step, interval) on T = 100


def _maxabs(a, b):
    return float(np.abs(np.asarray(a, np.float64) - np.asarray(b, np.float64)).max())


def _rel(a, b):
    b = np.asarray(b, np.float64)
    return _maxabs(a, b) / max(1.0, float(np.abs(b).max()))


@contextlib.contextmanager
def _recording_diffnet():
    """Records (t, spec [F,80]) of every O.diffnet call (B = 1)."""
    calls, full = [], O.diffnet

    def rec(spec, t, *a, **kw):
        calls.append((int(t[0]), spec[0, 0].t().clone()))
        return full(spec, t, *a, **kw)

    O.diffnet = rec
    try:
        yield calls
    finally:
        O.diffnet = full


class ListNoise:
    """Hands the oracle a fixed list of draws in order."""

    def __init__(self, draws):
        self.draws = list(draws)

    def randn(self, shape):
        t = self.draws.pop(0)
        assert tuple(t.shape) == tuple(shape), (t.shape, shape)
        return t


def _cond(Fr, seed):
    g = torch.Generator().manual_seed(seed)
    cond = 0.5 * torch.randn(Fr, 256, generator=g)
    coarse = (-3 + 1.5 * torch.randn(Fr, 80, generator=g)).clamp(-6, 1.0)
    return cond, coarse


def _fp32_calls_vs_f64(calls32, calls64):
    assert [t for t, _ in calls32] == [t for t, _ in calls64], ([t for t, _ in calls32], [t for t, _ in calls64])
    return [_maxabs(a, b) for (_, a), (_, b) in zip(calls32, calls64)]


# ---------------------------------------------------------------------------------------------------------------------
# ProDiff
@pytest.mark.parametrize("T", [8, 4])
def test_prodiff_chain64_matches_fp32_oracle(T):
    hp = prodiff_hp(T)
    Fr = 70
    cond, _ = _cond(Fr, 10 + T)
    noise = torch.randn(T + 1, Fr, 80, generator=torch.Generator().manual_seed(20 + T))
    with _recording_diffnet() as calls32, torch.no_grad():
        mel32 = O.mel_prodiff_sample(cond[None], prodiff_sd(), hp,
                                     ListNoise([noise[k].t().contiguous()[None, None] for k in range(T + 1)]))[0]
    r = SO.prodiff_chain64(cond, hp, noise)
    # the k-th denoiser input is x_{T-k}
    e = _fp32_calls_vs_f64(calls32, [(T - 1 - k, x) for k, x in enumerate(r["x"][:T])])
    e_mel = _maxabs(mel32, r["mel"])
    print(f"ProDiff T={T}: x_t err per step {[f'{v:.1e}' for v in e]}, mel {e_mel:.1e}")
    assert max(e) < TOL and e_mel < TOL
    assert len(r["x0"]) == T and torch.equal(r["x"][0], noise[0].double())


def test_prodiff_chain64_matches_reference_fixture():
    """sampler_mel: ProDiffusion.forward on sampler_cond with NoiseSource(sampler_seed); mel_out: the whole forward,
    whose mel sampler draws last: its decoder_inp and the last T + 1 draws of NoiseSource(seed)."""
    g, meta = golden("ref_prodiff_T8")
    T = meta["T"]
    hp = prodiff_hp()
    ns = O.NoiseSource(meta["sampler_seed"])
    Fr = g["sampler_cond"].shape[0]
    noise = torch.stack([ns.randn((1, 1, 80, Fr))[0, 0].t() for _ in range(T + 1)])
    e_smp = _rel(SO.prodiff_chain64(torch.from_numpy(g["sampler_cond"]), hp, noise)["mel"], g["sampler_mel"])
    ns = O.NoiseSource(meta["seed"])
    Fr = meta["frames"]
    draws = [(ns.randn(sh) if k == "randn" else ns.rand(sh)) for k, sh in meta["noise_log"]][-(T + 1):]
    assert all(tuple(d.shape) == (1, 1, 80, Fr) for d in draws)
    noise = torch.stack([d[0, 0].t() for d in draws])
    e_fwd = _rel(SO.prodiff_chain64(torch.from_numpy(g["decoder_inp"]), hp, noise)["mel"], g["mel_out"])
    print(f"ProDiff float64 vs reference fixture: sampler_mel {e_smp:.2e}, mel_out {e_fwd:.2e} (relative)")
    assert e_smp < TOL and e_fwd < TOL


# ---------------------------------------------------------------------------------------------------------------------
# PLMS
def _plms32(cond, coarse, K, interval, q):
    hp = dict(hp_for(100), K_step=K)
    with _recording_diffnet() as calls32, torch.no_grad():
        mel32 = O.mel_diffusion_sample_plms(cond[None], coarse[None], acoustic_sd(), hp,
                                            ListNoise([q.t().contiguous()[None, None]]), interval)[0]
    return mel32, calls32


@pytest.mark.parametrize("K,interval", PLMS_CONFIGS)
def test_plms_chain64_matches_fp32_oracle(K, interval):
    Fr = 60
    cond, coarse = _cond(Fr, K + interval)
    q = torch.randn(Fr, 80, generator=torch.Generator().manual_seed(3 * K + interval))
    mel32, calls32 = _plms32(cond, coarse, K, interval, q)
    r = SO.plms_chain64(cond, coarse, dict(hp_for(100), K_step=K), K, interval, q)
    e = _fp32_calls_vs_f64(calls32, r["calls"])
    e_mel = _rel(mel32, r["mel"])
    steps = SO.plms_steps(K, interval)
    print(f"PLMS K={K} interval={interval}: steps {steps[0]}..{steps[-1]}, orders {r['order']}, denoiser-input err per "
          f"call {[f'{v:.1e}' for v in e]}, mel {e_mel:.1e} (relative)")
    assert len(calls32) == SO.plms_evals(K, interval) == len(r["calls"])
    assert steps[0] == (K - 1) // interval * interval and steps[-1] == 0
    assert max(e) < TOL and e_mel < TOL
    assert r["order"] == [min(k, 3) for k in range(len(steps))]


def test_plms_chain64_reaches_every_history_order_and_wraps_the_ring():
    """K = 6, interval = 1: six steps with orders 0, 1, 2, 3, 3, 3.  The library keeps 3 history slots, so the fourth
    eps overwrites the first one's slot, and the fifth and sixth steps read that reused slot; their orders and weights
    must be the third-order ones."""
    r = SO.plms_chain64(*_cond(20, 1), dict(hp_for(100), K_step=6), 6, 1,
                        torch.randn(20, 80, generator=torch.Generator().manual_seed(2)))
    assert r["order"] == [0, 1, 2, 3, 3, 3]
    assert [t for t, _ in r["calls"]] == [5, 4, 4, 3, 2, 1, 0]  # the second-order start evaluates t = 5, then 4
    assert sorted(set(r["order"])) == [0, 1, 2, 3] and r["order"].count(3) >= 3


def test_plms_chain64_matches_reference_fixtures():
    """ref_plms_T100_i10 (T = K = 100, interval 10) and the PLMS entries of ref_kstep (K_step 51 of T = 100, intervals
    10 and 7: t0 = 50 and 49)."""
    g, meta = golden("ref_plms_T100_i10")
    Fr = g["cond"].shape[0]
    q = O.NoiseSource(meta["seed"] + 1).randn((1, 1, 80, Fr))[0, 0].t()
    T, k = meta["T"], meta["interval"]
    r = SO.plms_chain64(torch.from_numpy(g["cond"]), torch.from_numpy(g["coarse"]), hp_for(T), T, k, q)
    errs = {"T100_i10": _rel(r["mel"], g["mel"])}
    g, meta = golden("ref_kstep")
    Fr = g["smp_cond"].shape[0]
    q = O.NoiseSource(meta["seed"] + 3).randn((1, 1, 80, Fr))[0, 0].t()
    K = meta["K"]
    for k in meta["intervals"]:
        assert SO.plms_steps(K, k)[0] == meta[f"plms_i{k}_t0"]
        r = SO.plms_chain64(torch.from_numpy(g["smp_cond"]), torch.from_numpy(g["smp_coarse"]),
                            dict(hp_for(meta["T"]), K_step=K), K, k, q)
        errs[f"kstep_K{K}_i{k}"] = _rel(r["mel"], g[f"plms_i{k}_mel"])
    print("PLMS float64 vs reference fixtures (relative):", {k: f"{v:.2e}" for k, v in errs.items()})
    assert max(errs.values()) < TOL, errs
