"""Pin the float64 restatement of the GEMM epilogues (tests/conv_gemm_ref.py) on the CPU: composed as production composes
them, they must give the oracle's modules - one DiffNet residual layer with its skip head (GENERIC conditioner, GATE with
the addend in packed order, RES_SKIP reading its residual from planes minus the step bias, GENERIC heads), and the FFT
block's FFN (GENERIC with alpha = k^-1/2 and GELU, then GENERIC)."""
import math

import torch

from oracle import stylesinger_oracle as O
from tests import conv_gemm_ref as R

TOL = 1e-12  # float64 on both sides
LENS = [37, 1, 20]


def _rows(lens, C, gen, scale=1.0):
    rs, rows = R.layout(lens)
    x = torch.zeros(rows, C, dtype=torch.float64)
    for r, n in zip(rs, lens):
        x[r:r + n] = scale * torch.randn(n, C, generator=gen, dtype=torch.float64)
    return x, rs, rows


def _masked(v, lens, rs):
    """Rows outside the utterances are never written by the kernels: they stay zero."""
    return v * R.valid_rows(lens, rs, v.shape[0])[:, None]


def test_gate_and_res_skip_compose_to_the_oracle_residual_layer():
    gen = torch.Generator().manual_seed(0)
    C, E, M = 16, 24, 8
    p = "net."
    q = p + "residual_layers.0."
    w = lambda *s: torch.randn(*s, generator=gen, dtype=torch.float64) / math.sqrt(s[1] * (s[2] if len(s) > 2 else 1))
    sd = {q + "diffusion_projection.weight": w(C, C), q + "diffusion_projection.bias": torch.randn(C, generator=gen, dtype=torch.float64),
          q + "conditioner_projection.weight": w(2 * C, E, 1), q + "conditioner_projection.bias": torch.randn(2 * C, generator=gen, dtype=torch.float64),
          q + "dilated_conv.weight": w(2 * C, C, 3), q + "dilated_conv.bias": torch.randn(2 * C, generator=gen, dtype=torch.float64),
          q + "output_projection.weight": w(2 * C, C, 1), q + "output_projection.bias": torch.randn(2 * C, generator=gen, dtype=torch.float64),
          p + "skip_projection.weight": w(C, C, 1), p + "skip_projection.bias": torch.randn(C, generator=gen, dtype=torch.float64),
          p + "output_projection.weight": w(M, C, 1), p + "output_projection.bias": torch.randn(M, generator=gen, dtype=torch.float64)}
    x, rs, rows = _rows(LENS, C, gen)
    cond, _, _ = _rows(LENS, E, gen)
    dstep = torch.randn(len(LENS), C, generator=gen, dtype=torch.float64)
    # the step bias of each utterance, broadcast over its rows (one utterance per row block)
    dvec = dstep @ sd[q + "diffusion_projection.weight"].t() + sd[q + "diffusion_projection.bias"]
    drows = torch.zeros(rows, C, dtype=torch.float64)
    for b, (r, n) in enumerate(zip(rs, LENS)):
        drows[r:r + n] = dvec[b]
    y = _masked(x + drows, LENS, rs)  # the planes of y = x + step bias: the gate GEMM's A operand

    cvec, _ = R.generic(R.accumulator(cond, sd[q + "conditioner_projection.weight"], 1, LENS, rs),
                        sd[q + "conditioner_projection.bias"])
    z = R.gate(R.accumulator(y, sd[q + "dilated_conv.weight"], 1, LENS, rs), sd[q + "dilated_conv.bias"],
               add_packed=R.packed(cvec))
    z = _masked(z, LENS, rs)
    xres = R.planes_value(y, torch.zeros_like(y), drows)  # x = hi + lo - vec1
    _, _, skip = R.res_skip(R.accumulator(z, sd[q + "output_projection.weight"], 1, LENS, rs), C,
                            sd[q + "output_projection.bias"], x=xres, beta=2 ** -0.5, skip_init=True)
    skip = _masked(skip, LENS, rs)
    h, _ = R.generic(R.accumulator(skip, sd[p + "skip_projection.weight"], 1, LENS, rs), sd[p + "skip_projection.bias"],
                     a=R.RELU)
    h = _masked(h, LENS, rs)
    out, _ = R.generic(R.accumulator(h, sd[p + "output_projection.weight"], 1, LENS, rs), sd[p + "output_projection.bias"])

    err = 0.0
    for b, (r, n) in enumerate(zip(rs, LENS)):
        ref = O.residual_stack(x[r:r + n].t()[None], cond[r:r + n].t()[None], dstep[b:b + 1], sd, p, 1, 4)[0].t()
        err = max(err, float((out[r:r + n] - ref).abs().max()))
    print(f"residual layer (L = 1) restated from the epilogues vs the oracle: {err:.1e}")
    assert err < TOL


def test_generic_gelu_then_generic_is_the_oracle_ffn():
    gen = torch.Generator().manual_seed(1)
    C, H, k = 32, 64, 9
    sd = {"f.ffn_1.weight": torch.randn(H, C, k, generator=gen, dtype=torch.float64) / math.sqrt(C),
          "f.ffn_1.bias": torch.randn(H, generator=gen, dtype=torch.float64),
          "f.ffn_2.weight": torch.randn(C, H, generator=gen, dtype=torch.float64) / math.sqrt(H),
          "f.ffn_2.bias": torch.randn(C, generator=gen, dtype=torch.float64)}
    x, rs, _ = _rows(LENS, C, gen, 2.0)
    h, _ = R.generic(R.accumulator(x, sd["f.ffn_1.weight"], 1, LENS, rs), sd["f.ffn_1.bias"], alpha=k ** -0.5, a=R.GELU)
    h = _masked(h, LENS, rs)
    y, _ = R.generic(R.accumulator(h, sd["f.ffn_2.weight"][:, :, None], 1, LENS, rs), sd["f.ffn_2.bias"])
    err = 0.0
    for r, n in zip(rs, LENS):
        ref = O.ffn_layer(x[r:r + n][:, None], sd, "f.", k)[:, 0]
        err = max(err, float((y[r:r + n] - ref).abs().max()))
    print(f"FFN restated from the epilogues vs the oracle: {err:.1e}")
    assert err < TOL


def test_skip_tiling_round_trips():
    lens = [1, 130, 33]
    rs, rows = R.layout(lens)
    tl = R.tiles(lens, rs)
    x = torch.randn(rows, 64, dtype=torch.float64)
    back, unused = R.skip_tiled_to_rows(R.rows_to_skip_tiled(x, tl, 64), tl, 64, rows)
    valid = R.valid_rows(lens, rs, rows)
    assert torch.equal(back[valid], x[valid]) and not back[~valid].any()
    assert int((~unused).sum()) == sum(lens) * 64
