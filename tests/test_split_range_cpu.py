"""The float64 emulation facts tests/test_gpu_split_range.py relies on: the tensor-core GEMMs' hi / lo split of the weights
with the packer's power-of-two scale (tests/conv_gemm_ref.py split_scaled) against the split without it.

Emulated GEMM: activations and weights split as the kernels split them, the three products hi*hi + hi*lo + lo*hi summed in
float64 (the tensor core's own fp32 accumulation error is not included).  Metric: max |error| / sum |a||w| of one
768-deep dot product per output, weights randn / sqrt(768) 2^e, activations randn."""
import numpy as np
import pytest
import torch

from tests import conv_gemm_ref as R
from tests import fp16_emulation as E

K = 768


def _ops(ew, seed=0, n=64, rows=256):
    g = torch.Generator().manual_seed(seed)
    a = torch.randn(rows, K, generator=g)
    w = torch.ldexp(torch.randn(n, K, generator=g) / K ** 0.5, torch.tensor(float(ew)))
    return a, w


def _split_gemm(a, w, scaled):
    """float64 (hi_a + lo_a) (hi_w + lo_w) minus the lo_a lo_w term, over the weights' split with or without the scale."""
    ah, al = (t.double() for t in R.split(a))
    if scaled:
        wh, wl, s = R.split_scaled(w)
    else:
        (wh, wl), s = R.split(w), 0
    wh, wl = wh.double(), wl.double()
    acc = ah @ wh.t() + ah @ wl.t() + al @ wh.t()
    return torch.ldexp(acc, torch.tensor(float(-s), dtype=torch.float64))


def _rel_err(a, w, scaled):
    ref = a.double() @ w.double().t()
    d = a.double().abs() @ w.double().abs().t()
    return float(((_split_gemm(a, w, scaled) - ref).abs() / d).max())


@pytest.mark.parametrize("e", [-30, -24, -16, -12, -8, -4, -1, 1, 4, 8, 16, 20])
def test_scaled_split_is_exactly_equivariant(e):
    """out(w 2^e) == 2^e out(w) bit for bit: the scaled split of w 2^e is the split of w, exponent shifted."""
    a, w = _ops(0, seed=3)
    we = torch.ldexp(w, torch.tensor(float(e)))
    assert torch.equal(torch.ldexp(w, torch.tensor(float(e))) * 2.0 ** -e, w)  # the scaling itself is exact in fp32
    h0, l0, s0 = R.split_scaled(w)
    h1, l1, s1 = R.split_scaled(we)
    assert s1 == s0 - e and torch.equal(h0.view(torch.int16), h1.view(torch.int16)) and torch.equal(
        l0.view(torch.int16), l1.view(torch.int16))
    o0, o1 = _split_gemm(a, w, True), _split_gemm(a, we, True)
    assert torch.equal(o1, torch.ldexp(o0, torch.tensor(float(e), dtype=torch.float64)))


def test_unscaled_split_error_grows_with_small_weights():
    """Without the scale the lo planes of small weights are subnormal: the error of the split grows > 10x from weights
    randn / sqrt(768) to the same 2^-8 smaller; with the scale it stays the same."""
    a, w0 = _ops(0)
    w8 = torch.ldexp(w0, torch.tensor(-8.0))
    plain = (_rel_err(a, w0, False), _rel_err(a, w8, False))
    scaled = (_rel_err(a, w0, True), _rel_err(a, w8, True))
    print(f"emulated split error / sum |a||w|: unscaled e=0 {plain[0]:.2e}, e=-8 {plain[1]:.2e}; "
          f"scaled e=0 {scaled[0]:.2e}, e=-8 {scaled[1]:.2e}")
    assert plain[1] > 10 * plain[0]
    assert scaled[1] == scaled[0]
    assert scaled[0] < 1e-7


def test_plane_exponent():
    """s = 14 - ceil(log2 max|w|): max|w 2^s| in (2^13, 2^14]; 0 for a zero tensor."""
    for mx, s in [(1.0, 14), (0.75, 14), (0.5, 15), (2.0 ** -20, 34), (3.0, 12), (65504.0, -2), (2.0 ** -140, 126)]:
        w = torch.tensor([0.0, -mx, mx / 3])
        assert R.plane_exponent(w) == s, (mx, R.plane_exponent(w), s)
    assert R.plane_exponent(torch.zeros(5)) == 0
    rng = np.random.default_rng(1)
    for _ in range(200):
        w = torch.from_numpy(rng.standard_normal(17).astype(np.float32) * np.float32(2.0 ** rng.integers(-40, 40)))
        s = R.plane_exponent(w)
        m = float(torch.ldexp(w, torch.tensor(float(s))).abs().max())
        assert 2.0 ** 13 < m <= 2.0 ** 14


def test_packer_rounding_equals_fp16_for_normal_weights():
    """fp16(w 2^s) 2^-s == fp16(w) wherever w is a normal fp16 number (2^-14 <= |w| <= 65504), for tensors whose largest
    element is at most 2^14 (s >= 0); below 2^-14 the packer keeps more bits than a subnormal fp16.  (A larger tensor has
    s < 0: its weights below 2^(-14 - s), 2^-28 of its largest or less, are rounded as subnormals of the scaled planes.)"""
    rng = np.random.default_rng(2)
    for top in range(-14, 15):
        w = rng.standard_normal(4096).astype(np.float32) * np.float32(2.0 ** rng.uniform(-30, top, 4096))
        top_v = np.float32(2.0 ** top * 0.99)
        w = np.clip(w, -top_v, top_v)
        w[0] = top_v  # the largest element just below 2^top
        w = torch.from_numpy(w)
        normal = (w.abs() >= 2.0 ** -14) & (w.abs() <= 65504)
        got, plain = E.r16w(w), E.r16(w)
        assert torch.equal(got[normal], plain[normal]), top
        sub = ~normal & (w != 0)
        if sub.any():  # never worse than the plain rounding, and relative 2^-11 as long as w 2^s is normal
            assert bool(((got - w).abs() <= (plain - w).abs())[sub].all()), top
