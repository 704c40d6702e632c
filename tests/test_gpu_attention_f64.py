"""Both attention kernels, one call at a time (ssb_op_attention_ex), against the float64 restatement tests/attention_ref.py:
the fp32 kernel (attention_kernel, csrc/attention.cu) and the wgmma kernel (attention_tc_kernel, csrc/attention_tc.cu), in
the three layouts production hands them:

- op:    separate Q, K and V [rows, 256], fp32 output;
- self:  the FFT blocks' fused QKV [rows, 768] (K at column 256, V at 512); the wgmma kernel writes fp16 hi / lo planes
         [rows, 256] as the out-projection's A operand, the fp32 kernel fp32 rows at ld 768;
- cross: the style aligner's Q [rows_f, 256] with K | V [rows_r, 512], two layouts of different lengths (the wgmma kernel
         writes fp32 rows and planes at once).

Query lengths end the wgmma kernel's 8-row fragments, 64-row consumer warpgroups and 128-row CTAs; key lengths run from 0
to 2812 (44 key tiles, so the 4-slot ring wraps in both passes).  Key utterances start at every residue mod 8 (the wgmma
kernel's key grid shift kshift = row_start & 7), crossed with key lengths that end kshift + klen just before, on and just
after a 64-key tile boundary.  Score regimes: typical (randn x 1.5), peaked (randn x 6: one weight dominates), flat (q = 0:
the mean of V), exact ties (duplicated keys), and one key carrying a weight of about 2^-20 against a V row of 4096.

Every call checks: the valid rows against float64 (errors max |a - b| / max(1, |b|), the 8 rows at each utterance end
reported apart from the interior); NaN rows for an utterance without a valid key; that every element outside the
utterances' output rows is bit for bit the sentinel it held; that plane outputs are valid splits (hi == fp16(hi + lo));
that the inputs are unchanged; that a repeated call is bit-identical; and through ssb_attention_launch_count that exactly
one attention kernel (the one asked for) and, on the wgmma path, one transpose_planes launched.  Bars are 4x the largest
error measured on an H100 SXM (132 SMs, 700 W)."""
import math
import time

import numpy as np
import pytest
import torch

from stylesinger_b200._lib import SsbError
from tests import attention_ref as A
from tests import conv_gemm_ref as R
from tests.gpu_checks import Err, frame_offsets

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
H = 256
SCALE = 128 ** -0.5
SENT32, SENT16 = 0x7FC0DEAD, 0x7E5A  # NaN payloads (fp32 / fp16) no kernel produces
KERNEL = ("fp32", "wgmma")
REGIMES = ("typical", "peaked", "flat", "ties", "tiny")
# Bars: at most 4x the largest error measured on an H100 SXM (132 SMs, 700 W) over every call of the regime (all layouts,
# masks and the bench sizes), the measured value beside it; the two typical bars are also the ceilings the op-level tests
# have always had.  Peaked scores (std ~36 at randn x 6, ~7.5 at scale 0.3) move each weight by about |s| 2^-24 relative
# when s is rounded to fp32, whichever kernel computes it, hence bars 8 to 20x the typical ones; flat, tied and tiny-weight
# scores are close to 0, so those errors are the fp32 rounding of the sum over V alone.
BAR = {
    ("fp32", "typical"): 2e-5,      # 7.2e-6 (self layout; 5.5e-6 at 2812 keys, 5.4e-6 on the bench decoder)
    ("fp32", "peaked"): 4e-4,       # 1.1e-4
    ("fp32", "flat"): 7e-7,         # 1.8e-7 (mean of up to 2812 values)
    ("fp32", "ties"): 5.8e-6,       # 1.5e-6
    ("fp32", "tiny"): 1.1e-6,       # 3.0e-7
    ("fp32", "scale 0.3"): 6.4e-5,  # 1.6e-5
    ("wgmma", "typical"): 5e-5,     # 2.3e-5 (the bench decoder and 2812 keys; 1.2e-5 at 1125 keys)
    ("wgmma", "peaked"): 3.9e-4,    # 9.8e-5
    ("wgmma", "flat"): 1.3e-6,      # 3.3e-7
    ("wgmma", "ties"): 9.4e-6,      # 2.4e-6
    ("wgmma", "tiny"): 3.3e-6,      # 8.4e-7
    ("wgmma", "scale 0.3"): 9.5e-5,  # 2.4e-5
}

QL = [1, 7, 8, 9, 63, 64, 65, 127, 128, 129, 255, 256, 257]
KL = [0, 1, 2, 57, 63, 64, 65, 121, 128, 129, 320, 1125, 2812]
# (query length, key length): every length above once, short queries with short keys, and a query-less utterance between
# two normal ones
MAIN = [(1, 1), (7, 0), (8, 2), (9, 57), (63, 63), (64, 64), (0, 100), (65, 65), (127, 121), (128, 128), (129, 129),
        (255, 320), (256, 1125), (257, 2812)]
SELF = [1, 7, 0, 8, 9, 2, 57, 63, 64, 65, 121, 127, 128, 129, 255, 256, 257, 320, 1125, 2812]
# (key length, kshift): kshift + klen = 64 m - 1, 64 m, 64 m + 1 (m = 1 or 2), and 320 (5 tiles) for every kshift
GRID = [(64 * (1 + s % 2) - s + d, s) for s in range(8) for d in (-1, 0, 1)] + [(320 - s, s) for s in range(8)]


def with_shifts(base, self_layout):
    """base pairs, then the GRID utterances, each preceded where needed by a prefix utterance (query-less, or in the self
    layout as long as its keys) that puts its first key row at the residue mod 8 it asks for.  Utterance b's first row is
    16 + sum of the earlier lengths + 16 b, so its residue is that of the earlier key lengths' sum."""
    pairs = list(base)
    for i, (kl, s) in enumerate(GRID):
        r = sum(k for _, k in pairs) % 8
        if r != s:
            n = (s - r) % 8
            pairs.append((n if self_layout else 0, n))
        pairs.append((kl if self_layout else QL[i % len(QL)], kl))
    return pairs


def kshifts(klens):
    rs, _ = R.layout(klens)
    return [r & 7 for r in rs]


def check_grid(klens):
    """kshift takes all eight values, each crossed with key lengths ending a 64-key tile at -1, 0 and +1."""
    ks = kshifts(klens)
    ends = {}
    for s, kl in zip(ks, klens):
        if kl:
            ends.setdefault(s, set()).add((s + kl) % 64)
    print(f"kshift values {sorted(ends)}")
    assert sorted(ends) == list(range(8)), ends
    for s in range(8):
        assert {63, 0, 1} <= ends[s], (s, ends[s])


# ---------------------------------------------------------------------------------------------------------------------
# inputs
def _utt(regime, ql, kl, gen, scale):
    q = torch.randn(ql, H, generator=gen)
    k = torch.randn(kl, H, generator=gen)
    v = torch.randn(kl, H, generator=gen)
    if regime == "typical":
        q, k = q * 1.5, k * 1.5
    elif regime == "peaked":
        q, k = q * 6.0, k * 6.0
    elif regime == "flat":
        q, k = q * 0.0, k * 1.5
    elif regime == "ties":
        q, k = q * 1.5, (k * 1.5)[torch.arange(kl) % 5]
    elif regime == "tiny":  # key kl // 2 scores -20 ln 2 against ~0 for the others (per head, through column 128 h)
        q, k = q * 0.5, k * 0.5
        for c in (0, 128):
            q[:, c] = 1.0
            k[:, c] = 0.0
            if kl:
                k[kl // 2, c] = -20 * math.log(2) / scale
        if kl:
            v[kl // 2] = 4096.0
    return q, k, v


def _place(rows, rs, lens, parts):
    x = torch.zeros(rows, parts[0].shape[1] if parts else H)
    for r, n, t in zip(rs, lens, parts):
        x[r:r + n] = t
    return x


def _sent(shape, half=False):
    if half:
        return torch.full(shape, SENT16, dtype=torch.int16).view(torch.float16)
    return torch.full(shape, SENT32, dtype=torch.int32).view(torch.float32)


def _bits(t):
    return t.view(torch.int16) if t.dtype == torch.float16 else t.view(torch.int32)


def _half_ulp(hi):
    _, e = torch.frexp(hi.float().abs())
    return torch.clamp(torch.ldexp(torch.ones_like(hi.float()), e - 12), min=2.0 ** -25)


def _valid_split(hi, lo):
    """hi == fp16_rn(hi + lo) (or lo is exactly the half-ulp tie that rounds to even)."""
    same = (hi.float() + lo.float()).half().float() == hi.float()
    return bool((same | (lo.float().abs() == _half_ulp(hi))).all())


def build(path, layout, pairs, regime, seed, scale=SCALE, masks=None, utts=None, qkv=None):
    """Buffers (CPU), pointer map, integer arguments and float64 expectations of one call.  utts: the utterances compared
    with float64 (all by default).  qkv: per-utterance (q, k, v) instead of the regime's."""
    gen = torch.Generator().manual_seed(seed)
    qlens, klens = [p[0] for p in pairs], [p[1] for p in pairs]
    rsq, rows_q = R.layout(qlens)
    rsk, rows_k = R.layout(klens)
    parts = qkv if qkv is not None else [_utt(regime, ql, kl, gen, scale) for ql, kl in pairs]
    if layout == "self":
        assert qlens == klens
    Q = _place(rows_q, rsq, qlens, [p[0] for p in parts])
    K = _place(rows_k, rsk, klens, [p[1] for p in parts])
    V = _place(rows_k, rsk, klens, [p[2] for p in parts])
    km = None
    if masks is not None:
        km = torch.zeros(rows_k)
        for r, n, m in zip(rsk, klens, masks):
            km[r:r + n] = m
    bufs, ptrs, ints = {}, {}, {}
    if layout == "op":
        mats, where = {"q": Q, "k": K, "v": V}, {"q": ("q", 0), "k": ("k", 0), "v": ("v", 0)}
        ints.update(ldq=H, ldk=H, ldv=H)
    elif layout == "self":
        mats, where = {"qkv": torch.cat([Q, K, V], 1)}, {"q": ("qkv", 0), "k": ("qkv", H), "v": ("qkv", 2 * H)}
        ints.update(ldq=3 * H, ldk=3 * H, ldv=3 * H)
    else:
        mats, where = {"q": Q, "kv": torch.cat([K, V], 1)}, {"q": ("q", 0), "k": ("kv", 0), "v": ("kv", H)}
        ints.update(ldq=H, ldk=2 * H, ldv=2 * H)
    for name, m in mats.items():
        if path == 0:
            bufs[name] = m
        else:
            bufs[name + "_hi"], bufs[name + "_lo"] = R.split(m)
    for op, (name, col) in where.items():
        if path == 0:
            ptrs[op] = (name, col)
        else:
            ptrs[op + "_hi"], ptrs[op + "_lo"] = (name + "_hi", 0), (name + "_lo", 0)
            ints[op + "col0"] = col
    kinds = {k: "in" for k in bufs}
    if km is not None:
        bufs["keymask"], kinds["keymask"] = km, "in"
        ptrs["keymask"] = ("keymask", 0)
    if path == 0 and layout == "self":
        bufs["out"] = _sent((rows_q, 3 * H))
        ints["ldo"] = 3 * H
    elif layout != "self":
        bufs["out"] = _sent((rows_q, H))
        ints["ldo"] = H
    if path == 1 and layout != "op":
        bufs["oh"], bufs["ol"] = _sent((rows_q, H), True), _sent((rows_q, H), True)
        ints["ldh"] = H
    for k in ("out", "oh", "ol"):
        if k in bufs:
            kinds[k] = "out"
            ptrs[k] = (k, 0)
    t0 = time.perf_counter()
    idx = range(len(pairs)) if utts is None else utts
    exp = {b: A.attention(*parts[b], scale, None if masks is None else masks[b]) for b in idx if qlens[b]}
    ref_s = time.perf_counter() - t0
    return dict(path=path, layout=layout, regime=regime, qlens=qlens, klens=klens, rsq=rsq, rsk=rsk, rows_q=rows_q,
                rows_k=rows_k, scale=scale, bufs=bufs, kinds=kinds, ptrs=ptrs, ints=ints, exp=exp, ref_s=ref_s)


def counts():
    from stylesinger_b200._lib import lib
    torch.cuda.synchronize()
    return (lib.ssb_launch_count(), lib.ssb_attention_launch_count(0), lib.ssb_attention_launch_count(1))


def delta(c0, c1):
    return tuple(b - a for a, b in zip(c0, c1))


def call(st):
    """One ssb_op_attention_ex call on fresh device copies of the buffers: (device buffers, launch deltas)."""
    from stylesinger_b200.engine import op_attention_ex
    dev = {k: v.to(DEV) for k, v in st["bufs"].items()}
    args = {a: (dev[b].view(-1)[off:] if off else dev[b]) for a, (b, off) in st["ptrs"].items()}
    c0 = counts()
    op_attention_ex(st["path"], frame_offsets(st["qlens"]), frame_offsets(st["klens"]), st["rows_q"], st["rows_k"],
                    st["scale"], **args, **st["ints"])
    return dev, delta(c0, counts())


def _written(st, shape):
    m = torch.zeros(shape, dtype=torch.bool)
    for r, n in zip(st["rsq"], st["qlens"]):
        m[r:r + n, :H] = True
    return m


def run(st, bar, tag=None):
    """One call with every check; returns (CPU outputs, largest error)."""
    path = st["path"]
    tag = tag or f"{KERNEL[path]} {st['layout']} {st['regime']}"
    dev, d = call(st)
    want = (1, 1, 0) if path == 0 else (2, 0, 1)  # (all kernels, fp32 attention, wgmma attention)
    assert d == want, (tag, "launches (all, fp32 attention, wgmma attention)", d, want)
    out = {k: v.cpu() for k, v in dev.items()}
    nchk = 0
    for k, v in out.items():
        if st["kinds"][k] == "in":
            assert torch.equal(_bits(v), _bits(st["bufs"][k])), (tag, k, "an input changed")
            continue
        m = _written(st, v.shape)
        assert torch.equal(_bits(v)[~m], _bits(st["bufs"][k])[~m]), (tag, k, "an element outside the utterances changed")
        nchk += int((~m).sum())
    vals = {}
    if "out" in out:
        vals["out"] = out["out"][:, :H].double()
    if "oh" in out:
        vals["planes"] = out["oh"].double() + out["ol"].double()
    worst = 0.0
    nan_utts = []
    for name, val in vals.items():
        err = Err()
        for b, ref in st["exp"].items():
            r, n = st["rsq"][b], st["qlens"][b]
            if torch.isnan(ref).all():
                assert torch.isnan(val[r:r + n]).all(), (tag, name, b, "an utterance without a valid key is not NaN")
                nan_utts.append(b)
                continue
            assert torch.isfinite(val[r:r + n]).all(), (tag, name, b)
            if name == "planes":
                assert _valid_split(out["oh"][r:r + n], out["ol"][r:r + n]), (tag, b, "hi != fp16_rn(hi + lo)")
            err.add(b, val[r:r + n], ref)
        err.report(f"{tag} [{name}]", bar)
        worst = max(worst, err.max())
    print(f"{tag}: {len(st['exp'])} utterances against float64 ({st['ref_s']:.1f} s on the CPU), NaN rows for "
          f"{sorted(set(nan_utts))}, {nchk} elements outside the utterances unchanged")
    dev2, d2 = call(st)
    assert d2 == want
    for k in dev:
        assert torch.equal(_bits(dev2[k].cpu()), _bits(out[k])), (tag, k, "a second identical call differs")
    return out, worst


# ---------------------------------------------------------------------------------------------------------------------
# the matrix: kernel x layout x score regime
@pytest.mark.parametrize("regime", REGIMES)
@pytest.mark.parametrize("layout", ["op", "self", "cross"])
@pytest.mark.parametrize("path", [0, 1], ids=KERNEL)
def test_kernel_layout_regime(path, layout, regime):
    pairs = with_shifts([(n, n) for n in SELF] if layout == "self" else MAIN, layout == "self")
    check_grid([p[1] for p in pairs])
    st = build(path, layout, pairs, regime, seed=7 + 10 * path + REGIMES.index(regime))
    run(st, BAR[(KERNEL[path], regime)])


@pytest.mark.parametrize("path", [0, 1], ids=KERNEL)
def test_other_scale(path):
    """scale 0.3 instead of 128^-0.5: the fp32 kernel scales q on load, the wgmma kernel folds it into exp2's argument."""
    st = build(path, "op", with_shifts(MAIN, False), "typical", seed=71 + path, scale=0.3)
    run(st, BAR[(KERNEL[path], "scale 0.3")], tag=f"{KERNEL[path]} op typical scale 0.3")


# ---------------------------------------------------------------------------------------------------------------------
# key masks
def _mask(n, masked=(), valid=None):
    x = torch.ones(n)
    if valid is not None:
        x.zero_()
        x[list(valid)] = 1
    for a in masked:
        x[a] = 0
    return x


def masked_cases():
    """(query length, key length, mask): the patterns of test_gpu_padding, a fully masked utterance and a key-less one."""
    return [
        (70, 37, _mask(37, [0])),
        (1, 300, _mask(300, [63, 64, 127, 128])),
        (200, 261, _mask(261, [slice(0, 70), slice(120, 200)])),
        (129, 100, _mask(100, valid=[99])),
        (77, 48, torch.zeros(48)),
        (64, 151, _mask(151, valid=range(0, 151, 2))),
        (9, 0, torch.zeros(0)),
        (300, 90, _mask(90)),
        (5, 203, _mask(203, [slice(57, 71), slice(130, 203)])),
    ]


@pytest.mark.parametrize("layout", ["op", "self", "cross"])
@pytest.mark.parametrize("path", [0, 1], ids=KERNEL)
def test_key_masks(path, layout):
    cases = masked_cases()
    if layout == "self":
        cases = [(kl, kl, m) for _, kl, m in cases]
    pairs = [(c[0], c[1]) for c in cases]
    st = build(path, layout, pairs, "typical", seed=31 + path, masks=[c[2] for c in cases])
    nan = [b for b, (ql, kl, m) in enumerate(cases) if ql and not bool((m != 0).any())]
    assert nan == ([4] if layout == "self" else [4, 6])  # in the self layout the key-less utterance has no queries either
    assert sorted(b for b, ref in st["exp"].items() if torch.isnan(ref).all()) == nan
    run(st, BAR[(KERNEL[path], "typical")], tag=f"{KERNEL[path]} {layout} masked")


@pytest.mark.parametrize("path", [0, 1], ids=KERNEL)
def test_nan_utterances_leave_their_neighbours_bit_identical(path):
    """A fully masked utterance and a key-less one between normal ones give NaN rows; the others are bit-identical to a
    batch without them.  The removed key lengths sum to a multiple of 8, so the wgmma kernel's key grid stays put."""
    full = [(150, 203, _mask(203)), (77, 48, torch.zeros(48)), (12, 0, torch.zeros(0)),
            (140, 333, _mask(333, [10])), (3, 64, _mask(64))]
    keep = [0, 3, 4]
    gen = torch.Generator().manual_seed(41)
    parts = [_utt("typical", ql, kl, gen, SCALE) for ql, kl, _ in full]
    outs = []
    for sel in (range(len(full)), keep):
        st = build(path, "cross", [full[i][:2] for i in sel], "typical", 0, masks=[full[i][2] for i in sel],
                   qkv=[parts[i] for i in sel])
        out, _ = run(st, BAR[(KERNEL[path], "typical")], tag=f"{KERNEL[path]} NaN neighbours, {len(sel)} utterances")
        rows = {i: (r, n) for i, r, n in zip(sel, st["rsq"], st["qlens"])}
        outs.append({k: {i: v[r:r + n] for i, (r, n) in rows.items()} for k, v in out.items() if k in ("out", "oh", "ol")})
    for k in outs[1]:
        for i in keep:
            assert torch.equal(_bits(outs[0][k][i]), _bits(outs[1][k][i])), (k, i)
        for i in (1, 2):
            assert torch.isnan(outs[0][k][i].float()).all(), (k, i)


# ---------------------------------------------------------------------------------------------------------------------
# one utterance alone against its place in the batch
def test_fp32_kernel_utterance_alone_is_bit_identical_to_the_batch():
    pairs = with_shifts(MAIN, False)
    gen = torch.Generator().manual_seed(51)
    parts = [_utt("typical", ql, kl, gen, SCALE) for ql, kl in pairs]
    st = build(0, "op", pairs, "typical", 0, qkv=parts)
    out, _ = run(st, BAR[("fp32", "typical")], tag="fp32 op batch")
    picks = [0, 3, 7, 12, 13, len(pairs) - 1]
    for b in picks:
        s1 = build(0, "op", [pairs[b]], "typical", 0, qkv=[parts[b]])
        o1, _ = run(s1, BAR[("fp32", "typical")], tag=f"fp32 op alone {pairs[b]}")
        r, n = st["rsq"][b], pairs[b][0]
        r1 = s1["rsq"][0]
        assert torch.equal(_bits(o1["out"][r1:r1 + n]), _bits(out["out"][r:r + n])), b
    print(f"fp32 kernel: utterances {[pairs[b] for b in picks]} alone are bit-identical to the batch")


def test_wgmma_kernel_at_every_kshift_stays_within_the_bar():
    """DESIGN section 4: the wgmma kernel's key tiles sit on the 8-row grid of the key layout, so an utterance's output
    depends on where its keys start.  The same utterance after a key-only prefix of 0 .. 7 rows: every placement within
    the bar, and the spread between placements printed."""
    gen = torch.Generator().manual_seed(61)
    q, k, v = _utt("typical", 129, 321, gen, SCALE)
    ref = A.attention(q, k, v, SCALE)
    outs = {}
    for p in range(8):
        pairs = ([(0, p)] if p else []) + [(129, 321)]
        pre = [_utt("typical", 0, p, gen, SCALE)] if p else []
        st = build(1, "op", pairs, "typical", 0, qkv=pre + [(q, k, v)])
        assert kshifts(st["klens"])[-1] == p
        out, _ = run(st, BAR[("wgmma", "typical")], tag=f"wgmma op kshift {p}")
        r = st["rsq"][-1]
        outs[p] = out["out"][r:r + 129].double()
    spread = max(float((outs[p] - outs[0]).abs().max()) for p in range(8))
    worst = max(float(((outs[p] - ref).abs() / ref.abs().clamp(min=1)).max()) for p in range(8))
    print(f"wgmma kernel, one utterance at kshift 0 .. 7: largest error {worst:.3e}, spread between placements {spread:.3e}")


# ---------------------------------------------------------------------------------------------------------------------
# bench size: the batch64 decoder self-attention and the aligner's cross-attention with 1125-frame references
_BENCH = {}


def bench_lens():
    """Frame lengths of make_workload("batch64") at one GPU (seed 1234): the utterances of test_gpu_fft_style.bench_batch."""
    if not _BENCH:
        from stylesinger_b200 import synth
        secs = synth.batch_seconds(64, seed=1234)
        _BENCH["lens"] = [len(synth.make_utterance(float(s), utt_idx=i)["mel2ph"]) for i, s in enumerate(secs)]
        assert sum(_BENCH["lens"]) == 110119
    return _BENCH["lens"]


@pytest.mark.parametrize("which", ["decoder", "aligner"])
@pytest.mark.parametrize("path", [0, 1], ids=KERNEL)
def test_bench_size(path, which):
    lens = bench_lens()
    utts = sorted(set(range(0, len(lens), 8)) | {int(np.argmax(lens))})
    if which == "decoder":
        st = build(path, "self", [(n, n) for n in lens], "typical", seed=81 + path, utts=utts)
    else:
        st = build(path, "cross", [(n, 1125) for n in lens], "typical", seed=91 + path, utts=utts)
    run(st, BAR[(KERNEL[path], "typical")], tag=f"{KERNEL[path]} bench {which} ({len(lens)} utterances)")


# ---------------------------------------------------------------------------------------------------------------------
# which kernel the stage drivers launch: the wgmma kernel from 8 row tiles up (long_batch_tc), unless switched off
SMALL = [1, 2, 63, 64, 65, 127, 128]  # 7 row tiles


def _style_refs(lens):
    from stylesinger_b200 import synth
    us = [synth.make_utterance(1.0, utt_idx=300 + i, ref_frames=n, frames=8, phones=4) for i, n in enumerate(lens)]
    return [u["ref_mels"] for u in us], [u["ref_f0"] for u in us]


@pytest.mark.parametrize("extra", [[], [5]], ids=["7 tiles", "8 tiles"])
def test_stage_drivers_launch_the_expected_attention_kernel(extra):
    from stylesinger_b200._lib import lib
    from tests.common import acoustic_engine, hp_for
    hp = hp_for(4)
    m = acoustic_engine(4)
    flens = SMALL + extra
    rlens = [64, 1, 65, 300, 1, 64, 65] + [100] * len(extra)
    fo, ro = frame_offsets(flens), frame_offsets(rlens)
    g = torch.Generator().manual_seed(5)
    x = torch.randn(int(fo[-1]), H, generator=g).to(DEV)
    mels, f0s = _style_refs(rlens)
    mel, f0 = torch.cat(mels).to(DEV).contiguous(), torch.cat(f0s).to(DEV).contiguous()
    tok = torch.randint(3, 60, (int(fo[-1]),), generator=g, dtype=torch.int32).to(DEV)
    tc = len(extra) > 0
    L = hp["dec_layers"]

    def attn(fn):
        c0 = counts()
        fn()
        d = delta(c0, counts())
        return d[1], d[2]

    runs = {}
    try:
        for on in (1, 0):
            lib.ssb_set_attention_tensor_cores(on)
            runs[on] = (attn(lambda: m.fft_decoder(x, fo)), attn(lambda: m.get_style(x, fo, mel, f0, ro)),
                        attn(lambda: m.fft_encoder(tok, fo)))
    finally:
        lib.ssb_set_attention_tensor_cores(1)
    for on, (dec, sty, enc) in runs.items():
        print(f"{sum((n + 127) // 128 for n in flens)} row tiles, switch {on}: (fp32, wgmma) attention launches: decoder "
              f"{dec}, get_style {sty}, encoder {enc}")
        wg = tc and on
        assert dec == ((0, L) if wg else (L, 0)), (on, dec)
        assert sty == ((0, 2) if wg else (2, 0)), (on, sty)
        assert enc == (hp["enc_layers"], 0), (on, enc)


# ---------------------------------------------------------------------------------------------------------------------
# refusals: every one before any launch
REFUSALS = ["path-2", "no-output-fp32", "no-output-wgmma", "planes-on-fp32", "ld-not-4-fp32", "misaligned-fp32",
            "narrow-ld-fp32", "ld-not-8-wgmma", "ldo-not-8-wgmma", "qcol0-not-8-wgmma", "q-window-wgmma",
            "k-window-wgmma", "v-window-wgmma", "misaligned-wgmma", "heads-3-fp32", "heads-0-wgmma", "rows_q-fp32",
            "rows_k-wgmma", "B-65536"]


@pytest.mark.parametrize("case", REFUSALS)
def test_refused_before_any_launch(case):
    from stylesinger_b200.engine import op_attention_ex
    qlens, klens = [40, 7], [33, 9]
    _, rows_q = R.layout(qlens)
    _, rows_k = R.layout(klens)
    path = 1 if case.endswith("wgmma") else 0
    if path == 0:
        f = {n: torch.zeros(r, H, device=DEV) for n, r in (("q", rows_q), ("k", rows_k), ("v", rows_k))}
        args = dict(f, ldq=H, ldk=H, ldv=H, out=torch.zeros(rows_q, H, device=DEV), ldo=H)
    else:
        pq = torch.zeros(rows_q, 3 * H, dtype=torch.float16, device=DEV)
        pk = torch.zeros(rows_k, 3 * H, dtype=torch.float16, device=DEV)
        args = dict(q_hi=pq, q_lo=pq, k_hi=pk, k_lo=pk, v_hi=pk, v_lo=pk, ldq=3 * H, ldk=3 * H, ldv=3 * H, kcol0=H,
                    vcol0=2 * H, out=torch.zeros(rows_q, H, device=DEV), ldo=H)
    kw = dict(rows_q=rows_q, rows_k=rows_k, heads=2)
    qo, ko = frame_offsets(qlens), frame_offsets(klens)
    if case == "path-2":
        path = 2
    elif case.startswith("no-output"):
        args["out"] = None
    elif case == "planes-on-fp32":
        args["oh"] = args["ol"] = torch.zeros(rows_q, H, dtype=torch.float16, device=DEV)
    elif case == "ld-not-4-fp32":
        args["ldq"] = H + 2
    elif case == "misaligned-fp32":
        args["q"] = args["q"].view(-1)[1:]
    elif case == "narrow-ld-fp32":
        args["ldk"] = 128
    elif case == "ld-not-8-wgmma":
        args["ldk"] = 3 * H - 4
    elif case == "ldo-not-8-wgmma":
        args["ldo"] = H + 4
    elif case == "qcol0-not-8-wgmma":
        args["qcol0"] = 4
    elif case == "q-window-wgmma":
        args["qcol0"] = 2 * H + 8
    elif case == "k-window-wgmma":
        args["kcol0"] = 2 * H + 8
    elif case == "v-window-wgmma":
        args["vcol0"] = 2 * H + 8
    elif case == "misaligned-wgmma":
        args["k_hi"] = args["k_hi"].view(-1)[4:]
    elif case.startswith("heads"):
        kw["heads"] = int(case.split("-")[1])
    elif case.startswith("rows_q"):
        kw["rows_q"] += 8
    elif case.startswith("rows_k"):
        kw["rows_k"] -= 8
    elif case == "B-65536":
        qo = ko = np.zeros(65537, np.int32)
    c0 = counts()
    with pytest.raises(SsbError) as ei:
        op_attention_ex(path, qo, ko, kw["rows_q"], kw["rows_k"], SCALE, heads=kw["heads"], **args)
    assert counts() == c0
    print(f"{case}: refused: {ei.value}")


# ---------------------------------------------------------------------------------------------------------------------
# the tight-row wrapper engine.op_attention (both kernels) at the shapes the op-level tests have always covered
def wrapper_case(tc, ql, kl):
    from stylesinger_b200.engine import op_attention
    g = torch.Generator().manual_seed(3 + len(ql) + ql[0])
    qo, ko = frame_offsets(ql), frame_offsets(kl)
    q = torch.randn(int(qo[-1]), H, generator=g) * 1.5
    k = torch.randn(int(ko[-1]), H, generator=g) * 1.5
    v = torch.randn(int(ko[-1]), H, generator=g)
    c0 = counts()
    out = op_attention(q.to(DEV), k.to(DEV), v.to(DEV), qo, ko, SCALE, tc=tc).cpu()
    d = delta(c0, counts())
    assert d[1:] == ((0, 1) if tc else (1, 0)), d
    err = Err()
    for i in range(len(ql)):
        err.add(i, out[qo[i]:qo[i + 1]], A.attention(q[qo[i]:qo[i + 1]], k[ko[i]:ko[i + 1]], v[ko[i]:ko[i + 1]], SCALE))
    err.report(f"op_attention{' tc' if tc else ''} {ql} x {kl}", BAR[(KERNEL[int(tc)], "typical")])


def test_op_attention_matches_float64():
    """op_attention (the fp32 kernel) on ragged utterances with single-tile keys and a 1-row query."""
    wrapper_case(False, [70, 1, 200], [33, 150, 64])


@pytest.mark.parametrize("tc,ql,kl", [(True, [70, 1, 200], [33, 150, 64]),         # ragged, single-tile keys, 1-row query
                                      (False, [2812, 300, 129], [2812, 300, 129]),
                                      (True, [2812, 300, 129], [2812, 300, 129]),  # self-attention, longest bench utterance
                                      (False, [1500, 2200], [1125, 1125]),
                                      (True, [1500, 2200], [1125, 1125])])         # the style aligner's cross-attention
def test_op_attention_wrapper_shapes(tc, ql, kl):
    wrapper_case(tc, ql, kl)
