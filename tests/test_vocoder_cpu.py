"""The vocoder oracle at utterance-length edges (tools/make_golden.py vocoder_edges: 1, 2, 3, 5 and 17 frames) and its
float64 arbiter mode, which tests/test_gpu_vocoder.py measures the CUDA vocoder against."""
import numpy as np
import pytest
import torch

from oracle import stylesinger_oracle as O
from stylesinger_b200.hparams import DEFAULT_VOCODER_CONFIG
from tests.common import golden, vocoder_sd

TOL = 2e-6  # the bar of the other reference fixtures (tests/test_oracle_golden.py)
F64_BAR = 1e-5  # fp32 oracle vs float64 oracle: fp32 rounding through ~20 conv layers on a tanh-bounded waveform


def _maxabs(a, b):
    return float(np.abs(np.asarray(a, np.float64) - np.asarray(b, np.float64)).max())


def _spec2wav(mel, f0, seed, dtype=torch.float32):
    ns = O.NoiseSource(seed)
    with torch.no_grad():
        w = O.spec2wav(mel, f0, vocoder_sd(), DEFAULT_VOCODER_CONFIG, ns, dtype)
    return w, ns


@pytest.fixture(scope="module")
def edges():
    return golden("ref_vocoder_edges")


def test_edge_fixture_covers_the_edges(edges):
    g, meta = edges
    assert meta["lengths"] == [1, 2, 3, 5, 17]
    for L in meta["lengths"]:
        mel, f0 = g[f"mel_{L}"], g[f"f0_{L}"]
        assert mel.min() == -6.0 and mel.max() == 1.5
        assert (f0[1::2] == 0).all()
    assert (g["f0_3"] == 0).all()
    assert abs(float(g["f0_5"][2]) - 1100.0) < 1.0 and abs(float(g["f0_17"][2]) - 1100.0) < 1.0


@pytest.mark.parametrize("L", [1, 2, 3, 5, 17])
def test_oracle_matches_reference_at_edge_lengths(edges, L):
    g, meta = edges
    w, ns = _spec2wav(g[f"mel_{L}"], g[f"f0_{L}"], meta["seed"] + L)
    # the same draw sequence as the reference (the oracle draws the unused noise branch too)
    assert [tuple(x[1]) for x in meta["noise_log"][str(L)]] == [x[1] for x in ns.log]
    w2, _ = _spec2wav(g[f"mel_{L}"], None, 0)
    e, e2 = _maxabs(w, g[f"wav_{L}"]), _maxabs(w2, g[f"wav_nof0_{L}"])
    print(f"L={L}: oracle vs reference wav max |d| {e:.2e}, no f0 {e2:.2e} (bar {TOL:.0e})")
    assert w.shape == (256 * L,) and e < TOL and e2 < TOL


def _f64_cases():
    g, meta = golden("ref_vocoder_f24")
    yield "f24", g["mel"], g["f0"], meta["seed"] + 5
    g, meta = golden("ref_vocoder_edges")
    for L in meta["lengths"]:
        yield f"edge{L}", g[f"mel_{L}"], g[f"f0_{L}"], meta["seed"] + L


def test_float64_oracle_agrees_with_fp32_oracle():
    """The float64 arbiter computes the same function: it differs from the fp32 oracle (itself pinned to the reference
    at 2e-6) only by fp32 rounding, with and without f0 (the NSF source is fp32 in both)."""
    worst = 0.0
    for name, mel, f0, seed in _f64_cases():
        for f in (f0, None):
            a, _ = _spec2wav(mel, f, seed)
            b, _ = _spec2wav(mel, f, seed, torch.float64)
            assert b.dtype == np.float64
            e = _maxabs(a, b)
            print(f"{name} {'f0' if f is not None else 'no-f0'}: fp32 vs float64 oracle max |d| {e:.2e} (bar {F64_BAR:.0e})")
            worst = max(worst, e)
    assert worst < F64_BAR
