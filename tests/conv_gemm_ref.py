"""Float64 restatement of the two dense GEMM kernels (csrc/conv_gemm.cuh, csrc/conv_gemm_tc.cuh) and their epilogues.

The accumulator of one (x, W, dilation) is computed once, per utterance with zero "same" padding, and every epilogue is a
function of it, so one reference serves every option on that input.  Matrices here are [rows, cols] over the guard-banded
layout the kernels use (csrc/common.cuh): utterance b at rows [rs_b, rs_b + L_b), rs_0 = 16, rs_{b+1} = rs_b + L_b + 16, and
256 rows of tail slack.  Column order is torch's unless a function says "packed": the gate GEMM's packed order interleaves
the two halves (column 2j = sigmoid argument j, 2j + 1 = tanh argument j)."""
import math

import torch
import torch.nn.functional as F

GUARD, TAIL_SLACK, TILE_M = 16, 256, 128
NONE, RELU, GELU, LRELU, TANH, MISH = range(6)
GENERIC, GATE, RES_SKIP = range(3)


def layout(lens):
    """(row starts, total rows) of the guard-banded layout of utterances of lengths lens."""
    rs, r = [], GUARD
    for n in lens:
        rs.append(r)
        r += int(n) + GUARD
    return rs, r + TAIL_SLACK


def tiles(lens, rs):
    """The kernels' tile table: (first row, valid rows) of every 128-row tile, utterance by utterance."""
    return [(r + t0, min(TILE_M, int(n) - t0)) for r, n in zip(rs, lens) for t0 in range(0, int(n), TILE_M)]


def valid_rows(lens, rs, rows):
    m = torch.zeros(rows, dtype=torch.bool)
    for r, n in zip(rs, lens):
        m[r:r + int(n)] = True
    return m


def accumulator(x, w, dil, lens, rs, utts=None):
    """sum_j sum_c x[r + (j - (k-1)/2) dil, c] w[n, c, j] in float64 over the rows of utterances `utts` (all by default),
    zero elsewhere.  x [rows, Cin], w [N, Cin, k] (torch conv layout)."""
    x, w = x.double(), w.double()
    k = w.shape[2]
    acc = torch.zeros(x.shape[0], w.shape[0], dtype=torch.float64)
    for b in range(len(lens)) if utts is None else utts:
        r, n = rs[b], int(lens[b])
        acc[r:r + n] = F.conv1d(x[r:r + n].t()[None], w, padding=dil * (k - 1) // 2, dilation=dil)[0].t()
    return acc


def act(v, a, slope=0.1):
    if a == RELU:
        return v.clamp(min=0)
    if a == GELU:
        return F.gelu(v)
    if a == LRELU:
        return torch.where(v > 0, v, v * slope)
    if a == TANH:
        return torch.tanh(v)
    if a == MISH:
        return v * torch.tanh(F.softplus(v))
    return v


def d(t):
    return None if t is None else t.double()


def generic(acc, bias=None, add=None, alpha=1.0, a=NONE, slope=0.1, res=None, beta=1.0, rowmask=None, out=None, accum=False,
            gamma=1.0, vec2=None, plane_act=NONE, plane_slope=0.1):
    """EPI_GENERIC: v = act((acc + bias [+ add]) * alpha); v = (v + res) * beta; v *= rowmask[row];
    out = accum ? (out + v) * gamma : v.  Returns (out, the value of the fp16 planes: plane_act(out + vec2)).
    The tensor-core kernel has no add and no beta."""
    v = acc + (0 if bias is None else d(bias))
    if add is not None:
        v = v + d(add)
    v = act(v * alpha, a, slope)
    if res is not None:
        v = (v + d(res)) * beta
    if rowmask is not None:
        v = v * d(rowmask)[:, None]
    if accum:
        v = (d(out) + v) * gamma
    return v, act(v + (0 if vec2 is None else d(vec2)), plane_act, plane_slope)


def gate(acc, bias=None, add_packed=None):
    """EPI_GATE: z[:, j] = sigmoid(g_j) * tanh(f_j), g = columns [0, C), f = [C, 2C) of acc + bias, plus the addend given in
    packed order."""
    v = acc + (0 if bias is None else d(bias))
    C = v.shape[1] // 2
    g, f = v[:, :C], v[:, C:]
    if add_packed is not None:
        g, f = g + d(add_packed[:, 0::2]), f + d(add_packed[:, 1::2])
    return torch.sigmoid(g) * torch.tanh(f)


def packed(t):
    """Torch gate order [sigmoid C | tanh C] -> the kernels' packed order (interleaved)."""
    C = t.shape[-1] // 2
    return torch.stack([t[..., :C], t[..., C:]], -1).reshape(t.shape)


def planes_value(hi, lo, vec1=None):
    """The residual the tensor-core RES_SKIP epilogue reads from planes: x = hi + lo - vec1."""
    x = hi.double() + lo.double()
    return x if vec1 is None else x - d(vec1)


def res_skip(acc, C, bias=None, x=None, beta=1.0, vec2=None, skip=None, skip_init=True, rowmask=None):
    """EPI_RES_SKIP: columns [0, C): x_new = (acc + bias + x) * beta (* rowmask, FFMA only), planes of x_new + vec2;
    columns [C, 2C): skip = (skip_init ? 0 : skip) + acc + bias.  Returns (x_new, plane value, skip)."""
    v = acc + (0 if bias is None else d(bias))
    xn = (v[:, :C] + d(x)) * beta
    if rowmask is not None:
        xn = xn * d(rowmask)[:, None]
    s = v[:, C:] + (0 if skip_init else d(skip))
    return xn, xn + (0 if vec2 is None else d(vec2)), s


def split(x):
    """fp32 -> fp16 hi / lo planes as k_split_planes and the epilogues make them: hi = fp16_rn(x), lo = fp16_rn(x - hi)."""
    x = x.float()
    hi = x.half()
    return hi, (x - hi.float()).half()


def plane_exponent(w):
    """The power of two pack_conv_tc (csrc/pack.cu) scales a weight tensor by before it splits it: s = 14 - ceil(log2
    max|w|) over the fp32 tensor, so that max|w 2^s| <= 2^14; 0 for an all-zero or non-finite tensor; within [-126, 126]."""
    mx = float(w.float().abs().max()) if w.numel() else 0.0
    if not mx > 0.0 or mx == float("inf"):
        return 0
    m, e = math.frexp(mx)
    return max(-126, min(126, 14 - (e - 1 if m == 0.5 else e)))


def split_scaled(w):
    """The packer's weight planes: (hi, lo, s) with hi / lo = split(w 2^s), s = plane_exponent(w).  The kernels multiply
    the accumulator by 2^-s, so w is carried as (hi + lo) 2^-s."""
    s = plane_exponent(w)
    hi, lo = split(torch.ldexp(w.float(), torch.tensor(float(s))))
    return hi, lo, s


def weight_value(w, single_pass=False):
    """The weight value the tensor-core GEMM multiplies, in float64: (hi + lo) 2^-s, or hi 2^-s in the single-pass form."""
    hi, lo, s = split_scaled(w)
    v = hi.double() if single_pass else hi.double() + lo.double()
    return torch.ldexp(v, torch.tensor(float(-s), dtype=torch.float64))


def skip_tiled_to_rows(buf, tl, C, rows):
    """The chunk-tiled skip accumulator [tile][32-row quarter][32-col chunk][32][32] as [rows, C] (valid rows only; the rest
    zero) and the mask of its slots that belong to no valid row."""
    t = buf.reshape(len(tl), 4, C // 32, 32, 32)
    out = torch.zeros(rows, C, dtype=buf.dtype)
    unused = torch.ones(t.shape, dtype=torch.bool)
    for i, (r0, n) in enumerate(tl):
        blk = t[i].permute(0, 2, 1, 3).reshape(128, C)  # [quarter, row, chunk, col] -> [128 rows, C]
        out[r0:r0 + n] = blk[:n]
        for q in range(4):
            m = max(0, min(32, n - 32 * q))
            unused[i, q, :, :m] = False
    return out, unused


def rows_to_skip_tiled(x, tl, C):
    """Inverse of skip_tiled_to_rows (rows past a tile's valid ones are taken from x as they are)."""
    out = torch.empty(len(tl), 4, C // 32, 32, 32, dtype=x.dtype)
    for i, (r0, _) in enumerate(tl):
        out[i] = x[r0:r0 + 128].reshape(4, 32, C // 32, 32).permute(0, 2, 1, 3)
    return out.reshape(-1)

