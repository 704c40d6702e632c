"""The two dense GEMM kernels, one call at a time (ssb_op_gemm), against a float64 reference of the same operation
(tests/conv_gemm_ref.py): the fp32 FFMA kernel (conv_gemm_kernel<64> / <128>) and every tensor-core instantiation the
dispatch reaches (tc<64,·>, tc2<32|64,·>, tc2r<32|64,GENERIC|GATE>), each epilogue option alone and in the combinations
production uses, at utterance lengths that end a tile 1, 31, 32 or 33 rows into an epilogue warp's 32-row quarter.

Every call checks: the valid rows against float64 (errors max|a - b| / max(1, |b|), the 8 rows at each utterance end
reported apart from the interior and held to 4x it); fp16 plane outputs as hi + lo, and that hi / lo is a valid split;
that rows outside the utterances are bit for bit what they were (a NaN-payload sentinel in write-only buffers, zeros in
buffers that are also an A operand); and on the tensor cores that a second identical call is bit-identical.  Bars are 4x
the largest error measured on an H100 SXM (132 SMs)."""
import time

import numpy as np
import pytest
import torch

from stylesinger_b200._lib import SsbError
from tests import conv_gemm_ref as R
from tests.gpu_checks import Err, frame_offsets, launched, ntiles, variant

pytestmark = pytest.mark.gpu
DEV = "cuda:0"

EDGE_LENS = [1, 2, 3, 31, 32, 33, 63, 64, 65, 95, 96, 97, 127, 128, 129, 255, 256, 257]
SENT32, SENT16 = 0x7FC0DEAD, 0x7E5A  # NaN payloads (fp32 / fp16) no kernel produces
# Bars: at most 4x the largest error measured on an H100 SXM (132 SMs, 700 W) over the cases each one guards, the measured
# value beside it.  The error grows with the depth of the sum (taps x Cin), hence a bar per shape where shapes differ.
BAR = {
    "generic-tc": 5e-5,     # 1.7e-5 (GELU tail, x ~ N(0, 16)); the other options 2.3e-6 .. 7.6e-6
    "generic-ffma": 2.5e-5,  # 7.6e-6 (GELU tail); the other options 1.0e-6 .. 3.8e-6
    "gate-tc": 2e-5,        # 5.8e-6
    "gate-ffma": 8e-6,      # 2.2e-6
    "res_skip-tc": 8e-6,    # 2.2e-6
    "batch-tc": 3e-5,       # 8.1e-6 against float64; a short utterance alone vs in the batch: measured below
    "batch-ffma": 1.5e-5,   # 3.8e-6
    "reuse": 5e-5,          # 1.4e-5
    "reuse-vs-plain": 3e-5,  # 8.2e-6
    "op_conv1d": 2.5e-5,    # 7.7e-6 (Cin 256, k 9)
    "op_conv1d_tc": 6e-5,   # 1.7e-5 (Cin 192, k 5)
}
_CPU = {"ref_s": 0.0}


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def ffma_variant(N):
    return "conv_gemm_kernel<64>" if N <= 64 else "conv_gemm_kernel<128>"


def pair_lens(N, seed):
    """EDGE_LENS, bench-like utterances, and a last utterance of length 1 (its tile over-reads into the tail slack): the
    fewest row tiles that take the CTA-pair kernel at this N on this device, made odd so the peer CTA of the last pair
    idles."""
    hb = 64 if N % 128 == 0 else 32
    per = N // (2 * hb)
    need = 2 * (-(-_sms() // per)) - 1
    lens = list(EDGE_LENS)
    rng = np.random.default_rng(seed)
    while ntiles(lens) + 1 < need:
        lens.append(int(rng.integers(100, min(3000, max(101, 128 * (need - ntiles(lens) - 1))) + 1)))
    if (ntiles(lens) + 1) % 2 == 0:
        lens.append(5)
    return lens + [1]


def subset(lens):
    """Utterances compared with float64 at pair sizes: every edge length, the longest, the last, every 7th."""
    n = len(lens)
    return sorted(set(range(min(n, len(EDGE_LENS)))) | {int(np.argmax(lens)), n - 2, n - 1} | set(range(0, n, 7)))


# ---------------------------------------------------------------------------------------------------------------------
# buffers
def _sent(shape, half=False):
    if half:
        return torch.full(shape, SENT16, dtype=torch.int16).view(torch.float16)
    return torch.full(shape, SENT32, dtype=torch.int32).view(torch.float32)


def _rows(valid, cols, gen, scale=1.0, fill=None):
    """[rows, cols] fp32: N(0, scale^2) in the utterance rows, zero (or the sentinel) elsewhere."""
    rows = valid.shape[0]
    x = torch.zeros(rows, cols) if fill is None else _sent((rows, cols))
    x[valid] = scale * torch.randn(int(valid.sum()), cols, generator=gen)
    return x


def _bits(t):
    return t.view(torch.int16) if t.dtype == torch.float16 else t.view(torch.int32)


def _half_ulp(hi):
    m, e = torch.frexp(hi.float().abs())
    return torch.clamp(torch.ldexp(torch.ones_like(m), e - 12), min=2.0 ** -25)


def _valid_split(hi, lo):
    """hi == fp16_rn(hi + lo) (or lo is exactly the half-ulp tie that rounds to even): hi / lo is a split of one value."""
    hi, lo = hi.cpu(), lo.cpu()
    same = (hi.float() + lo.float()).half().float() == hi.float()  # as values: -0 + 0 is +0
    return bool((same | (lo.float().abs() == _half_ulp(hi))).all())


class Case:
    """One GEMM: path 0 (FFMA) / 1 (tensor cores), lengths, shape, epilogue mode and options (see _build)."""

    def __init__(self, tag, path, lens, Cin, N, k=1, dil=1, mode=R.GENERIC, seed=0, xscale=1.0, bias=True, want=None, **o):
        self.tag, self.path, self.lens, self.Cin, self.N, self.k, self.dil, self.mode = tag, path, lens, Cin, N, k, dil, mode
        self.seed, self.xscale, self.bias, self.want, self.o = seed, xscale, bias, want, o


def _build(c):
    """Inputs, initial buffers (CPU), scalar arguments and float64 expectations of a case.
    expectations: name -> (float64 [rows, cols] value, kind, columns checked); kind 'f32' | 'planes' (name is the hi plane,
    name + '_lo' its lo) | 'nb' (column-block-major, o['out_nb'] columns per block) | 'tiled' (chunk-tiled skip)."""
    o, gen = c.o, torch.Generator().manual_seed(c.seed)
    rs, rows = R.layout(c.lens)
    valid = R.valid_rows(c.lens, rs, rows)
    tl = R.tiles(c.lens, rs)
    N, C = c.N, c.N // 2
    x = _rows(valid, c.Cin, gen, c.xscale)
    w = torch.randn(N, c.Cin, c.k, generator=gen) / (c.Cin * c.k) ** 0.5
    b = torch.randn(N, generator=gen) if c.bias else None
    bufs, kinds, sc = {}, {}, {}
    if c.path == 0:
        bufs["a"], kinds["a"] = x, "in"
        sc["lda"] = c.Cin
        for f in ("a_act", "a_slope", "a_scale"):
            if f in o:
                sc[f] = o[f]
        a64 = R.act(x.double() * o.get("a_scale", 1.0), o.get("a_act", R.NONE), o.get("a_slope", 0.1))
    else:
        bufs["a_hi"], bufs["a_lo"] = R.split(x)
        kinds["a_hi"] = kinds["a_lo"] = "in"
        a64 = x.double()
    t0 = time.perf_counter()
    utts = o.get("utts")
    acc = R.accumulator(a64, w, c.dil, c.lens, rs, utts)
    exp = {}

    def vec(n, scale=1.0):
        return scale * torch.randn(n, generator=gen)

    def rowmask():
        v = torch.rand(rows, generator=gen)
        pick = torch.randint(0, 3, (rows,), generator=gen)
        return torch.where(pick == 0, torch.zeros(rows), torch.where(pick == 1, torch.ones(rows), v)) * valid

    if c.mode == R.GENERIC:
        nv = o.get("n_valid", 0)
        cols = nv if nv else N
        for f in ("alpha", "act", "act_slope", "beta", "gamma", "plane_act", "plane_slope"):
            if f in o:
                sc[f] = o[f]
        ep = dict(alpha=o.get("alpha", 1.0), a=o.get("act", R.NONE), slope=o.get("act_slope", 0.1), beta=o.get("beta", 1.0),
                  gamma=o.get("gamma", 1.0), plane_act=o.get("plane_act", R.NONE), plane_slope=o.get("plane_slope", 0.1))
        if o.get("add"):
            bufs["add"], kinds["add"] = _rows(valid, N, gen), "in"
            sc["ld_add"] = N
            ep["add"] = bufs["add"]
        if o.get("res"):
            bufs["res"], kinds["res"] = _rows(valid, N, gen), "in"
            sc["ld_res"] = N
            ep["res"] = bufs["res"]
        if o.get("rowmask"):
            bufs["rowmask"], kinds["rowmask"] = rowmask(), "in"
            ep["rowmask"] = bufs["rowmask"]
        if o.get("vec2"):
            bufs["vec2"], kinds["vec2"] = vec(N), "in"
            ep["vec2"] = bufs["vec2"]
        out0 = None
        if o.get("accum"):
            out0 = _rows(valid, N, gen, fill=True)
            sc["accum"] = 1
            ep.update(out=out0, accum=True)
        v, pv = R.generic(acc, b, **ep)
        if o.get("out", True):
            nb = o.get("out_nb", 0)
            if nb:
                bufs["out"] = _sent((N // nb, rows, nb)).reshape(-1)
                sc.update(out_nb=nb, out_bs=rows * nb, ldo=N)
                exp["out"] = (v, "nb", cols)
            else:
                bufs["out"] = out0 if out0 is not None else _sent((rows, N))
                sc["ldo"] = N
                exp["out"] = (v, "f32", cols)
            kinds["out"] = "out"
            if o.get("res_is_out"):  # production's FFN / out-projection: x = (x + f(x)) * keep, in place
                bufs["out"] = bufs["res"]
                kinds["out"] = "io"
                del bufs["res"]
                sc["res_alias"] = "out"
        if o.get("out2"):
            bufs["out2"], kinds["out2"] = _sent((rows, N)), "out"
            sc["ldo2"] = N
            exp["out2"] = (v + (0 if o.get("vec2") is None else bufs["vec2"].double()), "f32", cols)
        if o.get("planes"):
            bufs["oh"], bufs["ol"] = _sent((rows, N), True), _sent((rows, N), True)
            kinds["oh"] = kinds["ol"] = "out"
            sc["ldh"] = N
            exp["oh"] = (pv, "planes", cols)
        if nv:
            sc["n_valid"] = nv
    elif c.mode == R.GATE:
        add = None
        if o.get("add"):
            bufs["add"], kinds["add"] = _rows(valid, N, gen, o.get("add_scale", 1.0)), "in"
            sc["ld_add"] = N
            add = bufs["add"]
        z = R.gate(acc, b, add)
        if c.path == 0:
            if o.get("rowmask"):
                bufs["rowmask"], kinds["rowmask"] = rowmask(), "in"
                z = z * bufs["rowmask"].double()[:, None]
            bufs["out"], kinds["out"] = _sent((rows, C)), "out"
            sc["ldo"] = C
            exp["out"] = (z, "f32", C)
        else:
            bufs["oh"], bufs["ol"] = _sent((rows, C), True), _sent((rows, C), True)
            kinds["oh"] = kinds["ol"] = "out"
            sc["ldh"] = C
            exp["oh"] = (z, "planes", C)
    else:
        sc["C"] = C
        if "beta" in o:
            sc["beta"] = o["beta"]
        src = o.get("src", "res" if c.path == 0 else "planes")
        if src == "res":
            bufs["res"], kinds["res"] = _rows(valid, C, gen), "in"
            sc["ld_res"] = C
            xr = bufs["res"].double()
        else:
            bufs["vec1"], kinds["vec1"] = vec(C), "in"
            y = _rows(valid, C, gen) + bufs["vec1"] * valid[:, None]
            bufs["rh"], bufs["rl"] = R.split(y)
            kinds["rh"] = kinds["rl"] = "in"
            sc["ld_rh"] = C
            xr = R.planes_value(bufs["rh"], bufs["rl"], None) - bufs["vec1"].double() * valid[:, None]
            if not o.get("vec1", True):  # no step bias: x = hi + lo
                xr = R.planes_value(bufs["rh"], bufs["rl"])
                del bufs["vec1"]
        rm = None
        if o.get("rowmask"):  # FFMA only
            bufs["rowmask"], kinds["rowmask"] = rowmask(), "in"
            rm = bufs["rowmask"]
        if o.get("vec2"):
            bufs["vec2"], kinds["vec2"] = vec(C), "in"
        init = o.get("skip_init", 1)
        sc["skip_init"] = init
        tiled = o.get("skip_tiled", 0)
        skip0 = _rows(valid, C, gen, fill=True)
        xn, pv, s = R.res_skip(acc, C, b, xr, o.get("beta", 1.0), bufs.get("vec2"), skip0, bool(init), rm)
        if tiled:
            sc["skip_tiled"] = 1
            bufs["skip"] = R.rows_to_skip_tiled(skip0 if not init else _sent((rows, C)), tl, C)
            exp["skip"] = (s, "tiled", C)
        else:
            sc["ld_skip"] = C
            bufs["skip"] = skip0 if not init else _sent((rows, C))
            exp["skip"] = (s, "f32", C)
        kinds["skip"] = "io" if not init else "out"
        if o.get("out", c.path == 0):
            bufs["out"], kinds["out"] = _sent((rows, C)), "out"
            sc["ldo"] = C
            exp["out"] = (xn, "f32", C)
        if o.get("out2"):  # FFMA: out2 = x_new + vec2
            bufs["out2"], kinds["out2"] = _sent((rows, C)), "out"
            sc["ldo2"] = C
            exp["out2"] = (pv, "f32", C)
        if o.get("planes"):
            if o.get("inplace"):  # the next layer's y planes over this layer's: guard rows stay zero (an A operand)
                sc["planes_alias"] = True
                kinds["rh"] = kinds["rl"] = "aop"
            else:
                bufs["oh"], bufs["ol"] = _sent((rows, C), True), _sent((rows, C), True)
                kinds["oh"] = kinds["ol"] = "out"
            sc["ldh"] = C
            exp["oh" if not o.get("inplace") else "rh"] = (pv, "planes", C)
        if o.get("sh"):
            bufs["sh"], bufs["sl"] = _sent((rows, C), True), _sent((rows, C), True)
            kinds["sh"] = kinds["sl"] = "out"
            exp["sh"] = (s, "planes", C)
    _CPU["ref_s"] += time.perf_counter() - t0
    return dict(rs=rs, rows=rows, valid=valid, tl=tl, w=w, b=b, bufs=bufs, kinds=kinds, sc=sc, exp=exp)


def _call(c, st):
    """One ssb_op_gemm call on fresh device copies of the case's buffers: (device buffers, variants, launches)."""
    from stylesinger_b200.engine import op_gemm
    dev = {k: v.to(DEV) for k, v in st["bufs"].items()}
    sc = dict(st["sc"])
    args = dict(dev)
    if sc.pop("res_alias", None):
        args["res"] = dev["out"]
    if sc.pop("planes_alias", None):
        args["oh"], args["ol"] = dev["rh"], dev["rl"]
    offs = frame_offsets(c.lens)
    _, got, nl = launched(lambda: op_gemm(c.path, offs, st["rows"], st["w"], st["b"],
                                          dilation=c.dil, gate=c.mode == R.GATE, mode=c.mode, **args, **sc))
    return dev, got, nl


def _written(kind, st, shape, cols, N, nb=0):
    """Mask (buffer layout) of the elements the kernel writes."""
    valid = st["valid"]
    if kind == "tiled":
        _, unused = R.skip_tiled_to_rows(torch.zeros(shape), st["tl"], cols, st["rows"])
        return ~unused.reshape(-1)
    if kind == "nb":
        m = torch.zeros(N // nb, st["rows"], nb, dtype=torch.bool)
        m[:, valid] = True
        colmask = (torch.arange(N) < cols).reshape(N // nb, 1, nb)
        return (m & colmask).reshape(-1)
    m = torch.zeros(shape, dtype=torch.bool)
    m[valid, :cols] = True
    return m


def _as_rows(kind, t, st, cols, N, nb=0):
    if kind == "tiled":
        return R.skip_tiled_to_rows(t, st["tl"], cols, st["rows"])[0]
    if kind == "nb":
        return t.reshape(N // nb, st["rows"], nb).permute(1, 0, 2).reshape(st["rows"], N)
    return t


def run(c):
    """Run a case and apply every check; returns the device outputs (CPU) and the largest error."""
    st = _build(c)
    dev, got, nl = _call(c, st)
    torch.cuda.synchronize()
    name = variant(ntiles(c.lens), c.N, ("GENERIC", "GATE", "RES_SKIP")[c.mode], c.k, c.dil) if c.path else ffma_variant(c.N)
    if c.path:
        assert got == {name: 1} and nl == 1, (c.tag, got, name, nl)
    else:
        assert got == {} and nl == 1, (c.tag, got, nl)
    if c.want:
        assert name == c.want, (c.tag, name, c.want)
    out = {k: v.cpu() for k, v in dev.items()}
    N, utts = c.N, c.o.get("utts") or range(len(c.lens))
    bar = c.o["bar"]
    worst = 0.0
    # rows outside the utterances: bit for bit as before
    nchk = 0
    for k, v in out.items():
        kind = st["kinds"][k]
        if kind == "in":
            assert torch.equal(_bits(v), _bits(st["bufs"][k])), (c.tag, k, "an input buffer changed")
            continue
        e = st["exp"].get(k) or st["exp"].get({"ol": "oh", "sl": "sh", "rl": "rh"}.get(k, k))
        kind_e, cols = e[1], e[2]
        lay = "f32" if kind_e == "planes" else kind_e
        m = _written(lay, st, v.shape, cols, N if lay != "tiled" else N // 2, c.o.get("out_nb", 0))
        assert torch.equal(_bits(v)[~m], _bits(st["bufs"][k])[~m]), (c.tag, k, "an element outside the utterances changed")
        assert torch.isfinite(v[m].float()).all(), (c.tag, k, "a valid element was not written")
        nchk += int((~m).sum())
    # valid rows against float64
    for k, (ref, kind, cols) in st["exp"].items():
        lo = {"oh": "ol", "sh": "sl", "rh": "rl"}.get(k)
        if kind == "planes":
            assert _valid_split(out[k][st["valid"], :cols], out[lo][st["valid"], :cols]), (c.tag, k, "hi != fp16_rn(hi + lo)")
            val = out[k].double() + out[lo].double()
        else:
            val = _as_rows(kind, out[k], st, cols, N, c.o.get("out_nb", 0)).double()
        err = Err()
        for i in utts:
            r, n = st["rs"][i], c.lens[i]
            err.add(i, val[r:r + n, :cols], ref[r:r + n, :cols])
        err.report(f"{c.tag} [{name}] {k}", bar)
        worst = max(worst, err.max())
    print(f"{c.tag} [{name}]: {nchk} elements outside the utterances unchanged")
    if c.path:  # a race in the mbarrier ring or the epilogue transpose buffers shows up as a difference between two runs
        dev2, _, _ = _call(c, st)
        for k in dev:
            assert torch.equal(_bits(dev2[k]), _bits(dev[k])), (c.tag, k, "second identical call differs")
        print(f"{c.tag} [{name}]: second identical call bit-identical")
    return out, st, worst


# ---------------------------------------------------------------------------------------------------------------------
# every kernel instantiation the dispatch reaches, by name
_TC = [  # name, Cin, N, k, dil, mode, options (bar: measured)
    ("tc<64,GENERIC>", 128, 256, 9, 2, R.GENERIC, dict(res=True, bar=6e-5)),  # 2.0e-5
    ("tc<64,GATE>", 64, 128, 3, 16, R.GATE, dict(add=True, bar=1e-5)),  # 3.0e-6
    ("tc<64,RES_SKIP>", 64, 128, 1, 1, R.RES_SKIP, dict(planes=True, vec2=True, skip_init=0, bar=8e-6)),  # 2.0e-6
    ("tc2<64,GENERIC>", 256, 512, 1, 1, R.GENERIC, dict(act=R.RELU, bar=2e-5)),  # 5.6e-6
    ("tc2<64,GATE>", 256, 512, 3, 9, R.GATE, dict(add=True, bar=4e-5)),  # 1.1e-5
    ("tc2<64,RES_SKIP>", 256, 512, 1, 1, R.RES_SKIP,
     dict(planes=True, inplace=True, vec2=True, skip_tiled=1, skip_init=0, bar=2e-5)),  # 6.1e-6
    ("tc2<32,GENERIC>", 192, 192, 5, 1, R.GENERIC, dict(planes=True, bar=6e-5)),  # 1.8e-5
    ("tc2<32,GATE>", 64, 64, 5, 2, R.GATE, dict(add=True, bar=1.5e-5)),  # 4.3e-6
    ("tc2<32,RES_SKIP>", 64, 1088, 1, 1, R.RES_SKIP, dict(out=True, planes=True, vec2=True, skip_tiled=1, bar=8e-6)),  # 2.5e-6
    ("tc2r<32,GENERIC>", 64, 192, 3, 8, R.GENERIC, dict(bar=1.5e-5)),  # 4.6e-6
    ("tc2r<32,GATE>", 1088, 1088, 3, 1, R.GATE, dict(add=True, bar=1.5e-4)),  # 4.4e-5 (3264-deep sums)
    ("tc2r<64,GENERIC>", 256, 256, 3, 1, R.GENERIC, dict(act=R.LRELU, act_slope=0.1, bar=4e-5)),  # 1.2e-5
    ("tc2r<64,GATE>", 256, 512, 3, 8, R.GATE, dict(add=True, add_scale=30.0, bar=4e-5)),  # 1.0e-5
]


@pytest.mark.parametrize("name,Cin,N,k,dil,mode,opts", _TC, ids=[t[0] for t in _TC])
def test_tensor_core_variant(name, Cin, N, k, dil, mode, opts):
    pair = name.startswith("tc2")
    lens = pair_lens(N, Cin + N) if pair else EDGE_LENS
    o = dict(opts)
    if pair:
        o["utts"] = subset(lens)
    t0 = time.perf_counter()
    run(Case(f"{name} Cin {Cin} N {N} k {k} dil {dil}", 1, lens, Cin, N, k, dil, mode, seed=Cin * 7 + N + k, want=name, **o))
    print(f"{name}: {ntiles(lens)} row tiles, {time.perf_counter() - t0:.1f} s (CPU float64 so far {_CPU['ref_s']:.1f} s)")


@pytest.mark.parametrize("Cin,N,k,dil,mode,opts", [
    (80, 64, 7, 1, R.GENERIC, dict(act=R.TANH, bar=1.2e-5)),  # 3.6e-6
    (192, 320, 11, 1, R.GENERIC, dict(act=R.MISH, bar=2.5e-5)),  # 7.8e-6
    (64, 128, 3, 16, R.GATE, dict(add=True, add_scale=30.0, rowmask=True, bar=4e-6)),  # 1.1e-6
    (128, 128, 1, 1, R.RES_SKIP, dict(out2=True, vec2=True, rowmask=True, skip_init=0, beta=0.7071067811865476,
                                      bar=6e-6)),  # 1.9e-6
], ids=["kernel64-tanh", "kernel128-mish", "gate-k3-d16", "res_skip"])
def test_ffma_variant(Cin, N, k, dil, mode, opts):
    run(Case(f"FFMA Cin {Cin} N {N} k {k} dil {dil}", 0, EDGE_LENS, Cin, N, k, dil, mode, seed=N + k, want=ffma_variant(N),
             **opts))


# ---------------------------------------------------------------------------------------------------------------------
# every epilogue option alone, on one variant per mode and path
_GENERIC_OPTS = {
    "bias-free": dict(bias=False),
    "act-relu": dict(act=R.RELU),
    "act-lrelu": dict(act=R.LRELU, act_slope=0.2),
    "act-gelu-tail": dict(act=R.GELU, xscale=4.0),
    "alpha": dict(alpha=0.37),
    "res": dict(res=True),
    "rowmask": dict(rowmask=True),
    "accum-gamma": dict(accum=True, gamma=0.25),
    "planes": dict(planes=True),
    "planes-lrelu-vec2": dict(planes=True, plane_act=R.LRELU, plane_slope=0.1, vec2=True),
    "planes-only": dict(planes=True, out=False),
    "out_nb": dict(out_nb=64),
    "n_valid": dict(n_valid=96),
}
_FFMA_ONLY = {"add": dict(add=True), "beta": dict(res=True, beta=0.6), "out2-vec2": dict(out2=True, vec2=True),
              "a-lrelu-scale": dict(a_act=R.LRELU, a_slope=0.1, a_scale=1.7), "act-tanh": dict(act=R.TANH),
              "act-mish": dict(act=R.MISH)}
_TC_ONLY = ("out_nb", "n_valid", "planes-only")


@pytest.mark.parametrize("path,opt", [(1, k) for k in _GENERIC_OPTS] +
                         [(0, k) for k in _GENERIC_OPTS if k not in _TC_ONLY] + [(0, k) for k in _FFMA_ONLY])
def test_generic_option(path, opt):
    o = dict(_GENERIC_OPTS.get(opt) or _FFMA_ONLY[opt])
    bias, xs = o.pop("bias", True), o.pop("xscale", 1.0)
    run(Case(f"GENERIC {opt} path {path}", path, EDGE_LENS, 128, 256, 3, 2, R.GENERIC, seed=11, xscale=xs, bias=bias,
             want="tc<64,GENERIC>" if path else None, bar=BAR["generic-tc" if path else "generic-ffma"], **o))


@pytest.mark.parametrize("path,opt", [(1, "plain"), (1, "add-saturating"), (0, "plain"), (0, "add-saturating"),
                                      (0, "rowmask")])
def test_gate_option(path, opt):
    o = {"plain": {}, "add-saturating": dict(add=True, add_scale=40.0), "rowmask": dict(rowmask=True)}[opt]
    run(Case(f"GATE {opt} path {path}", path, EDGE_LENS, 128, 256, 3, 4, R.GATE, seed=12, want="tc<64,GATE>" if path else None,
             bar=BAR["gate-tc" if path else "gate-ffma"], **o))


_RES_OPTS = {
    "res-fp32": dict(src="res", out=True),
    "planes-src": dict(src="planes", out=True),
    "planes-src-no-vec1": dict(src="planes", vec1=False, out=True),
    "planes-out": dict(planes=True),
    "planes-out-vec2": dict(planes=True, vec2=True),
    "inplace": dict(planes=True, inplace=True),
    "skip-accumulate": dict(skip_init=0),
    "skip-tiled": dict(skip_tiled=1),
    "skip-tiled-accumulate": dict(skip_tiled=1, skip_init=0),
    "sh-sl": dict(sh=True, skip_init=0),
    "beta": dict(beta=0.7071067811865476, planes=True),
}


@pytest.mark.parametrize("opt", list(_RES_OPTS))
def test_res_skip_option(opt):
    run(Case(f"RES_SKIP {opt}", 1, EDGE_LENS, 64, 256, 1, 1, R.RES_SKIP, seed=13, want="tc<64,RES_SKIP>",
             bar=BAR["res_skip-tc"], **_RES_OPTS[opt]))


# ---------------------------------------------------------------------------------------------------------------------
# the combinations production uses, on the variants production uses them on
_PROD = {
    # the hoisted conditioner of all L layers, one [rows, 2C] matrix per layer (stages.cu hoist_cond_tc)
    "cond-out_nb": (1, "pair", 256, 4 * 512, 1, 1, R.GENERIC, dict(out_nb=512, bias=False, bar=1.9e-5)),  # 4.9e-6
    # a DiffNet layer's gate GEMM with the hoisted conditioner as addend (stages.cu denoiser_stack)
    "gate-addend": (1, "pair", 256, 512, 3, 8, R.GATE, dict(add=True, add_scale=20.0, bar=5e-5)),  # 1.3e-5
    # its residual + skip GEMM: residual from the y planes minus this layer's step bias, next layer's planes + its step
    # bias written in place, skip accumulated chunk-tiled
    "res_skip-layer": (1, "pair", 256, 512, 1, 1, R.RES_SKIP,
                       dict(planes=True, inplace=True, vec2=True, skip_tiled=1, skip_init=0, beta=0.7071067811865476,
                            bar=2e-5)),  # 5.7e-6
    "res_skip-first-layer": (1, "pair", 256, 512, 1, 1, R.RES_SKIP,
                             dict(planes=True, inplace=True, vec2=True, skip_tiled=1, skip_init=1, beta=0.7071067811865476,
                                  bar=2e-5)),  # 5.6e-6
    # the last layer: no next planes, the finished skip sum also as planes
    "res_skip-last-layer": (1, "pair", 256, 512, 1, 1, R.RES_SKIP,
                            dict(skip_tiled=1, skip_init=0, sh=True, beta=0.7071067811865476, bar=2e-5)),  # 6.0e-6
    # denoiser heads: skip_projection + ReLU -> planes (n_valid = C), output_projection with a padded N (stages.cu)
    "head-skip": (1, "single", 256, 256, 1, 1, R.GENERIC, dict(act=R.RELU, planes=True, out=False, n_valid=256, bar=2e-5)),  # 5.3e-6
    "head-out": (1, "single", 256, 256, 1, 1, R.GENERIC, dict(n_valid=96, bar=2e-5)),  # 5.3e-6
    # mel input projection: ReLU, planes of y = relu(.) + step bias
    "mel-in": (1, "single", 128, 256, 1, 1, R.GENERIC, dict(act=R.RELU, planes=True, out=False, vec2=True, bar=1.2e-5)),  # 3.5e-6
    # vocoder MRF: residual, accumulation over the kernels with gamma = 1 / nk on the last, LReLU planes of the sum
    "mrf-accum-tc": (1, "pair", 128, 128, 3, 5, R.GENERIC,
                     dict(res=True, accum=True, gamma=1 / 3, planes=True, plane_act=R.LRELU, plane_slope=0.1, bar=1e-5)),  # 2.9e-6
    "mrf-accum-ffma": (0, "edge", 64, 64, 7, 1, R.GENERIC,
                       dict(a_act=R.LRELU, a_slope=0.1, res=True, accum=True, gamma=1 / 3, planes=True, plane_act=R.LRELU,
                            bar=4e-6)),  # 1.0e-6
    "conv_pre-ffma": (0, "edge", 80, 256, 7, 1, R.GENERIC, dict(planes=True, plane_act=R.LRELU, plane_slope=0.1, bar=1.2e-5)),  # 3.3e-6
    # FFT block FFN: conv k * k^-1/2 -> GELU, then linear with the residual and the keep mask, in place
    "ffn1-tc": (1, "single", 256, 1024, 9, 1, R.GENERIC, dict(alpha=1 / 3, act=R.GELU, xscale=3.0, bar=1.2e-4)),  # 3.4e-5
    "ffn2-tc": (1, "single", 1024, 256, 1, 1, R.GENERIC, dict(res=True, rowmask=True, res_is_out=True, bar=5e-5)),  # 1.5e-5
    "ffn1-ffma": (0, "edge", 256, 1024, 9, 1, R.GENERIC, dict(alpha=1 / 3, act=R.GELU, xscale=3.0, bar=2.5e-5)),  # 6.9e-6
    "ffn2-ffma": (0, "edge", 1024, 256, 1, 1, R.GENERIC, dict(res=True, rowmask=True, res_is_out=True, bar=1.5e-5)),  # 4.7e-6
    # vocoder output denoiser: irfft's 1 / n_fft as alpha
    "wav-denoise-inv": (1, "pair", 1088, 256, 1, 1, R.GENERIC, dict(alpha=1 / 1024, bias=False, bar=1e-7)),  # 2.6e-8
}


@pytest.mark.parametrize("name", list(_PROD))
def test_production_combination(name):
    path, size, Cin, N, k, dil, mode, opts = _PROD[name]
    o = dict(opts)
    bias, xs = o.pop("bias", True), o.pop("xscale", 1.0)
    lens = pair_lens(N, 3) if size == "pair" else EDGE_LENS
    if size == "pair":
        o["utts"] = subset(lens)
    run(Case(f"production {name}", path, lens, Cin, N, k, dil, mode, seed=21, xscale=xs, bias=bias, **o))
    if size == "pair":
        assert variant(ntiles(lens), N, ("GENERIC", "GATE", "RES_SKIP")[mode], k, dil).startswith("tc2")


# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("path", [0, 1])
def test_short_utterances_alone_match_the_batch(path):
    """Each short utterance as a B = 1 call: bit-identical on FFMA (one thread per output, same loads), within the bar on
    the tensor cores."""
    N = 256
    lens = EDGE_LENS
    opts = dict(res=True, planes=True, vec2=True, plane_act=R.LRELU, bar=BAR["batch-tc" if path else "batch-ffma"])
    out, st, _ = run(Case(f"batch path {path}", path, lens, 128, N, 3, 2, R.GENERIC, seed=5, **opts))
    x_all, res_all = st["bufs"]["a" if path == 0 else "a_hi"], st["bufs"]["res"]
    from stylesinger_b200.engine import op_gemm
    worst = 0.0
    for i, L in enumerate(lens):
        if L > 129:
            continue
        rs1, rows1 = R.layout([L])
        r, r1 = st["rs"][i], rs1[0]
        args = {}
        if path == 0:
            a = torch.zeros(rows1, 128)
            a[r1:r1 + L] = x_all[r:r + L]
            args.update(a=a.to(DEV), lda=128)
        else:
            for k in ("a_hi", "a_lo"):
                a = torch.zeros(rows1, 128, dtype=torch.float16)
                a[r1:r1 + L] = st["bufs"][k][r:r + L]
                args[k] = a.to(DEV)
        res = torch.zeros(rows1, N)
        res[r1:r1 + L] = res_all[r:r + L]
        o1 = torch.zeros(rows1, N, device=DEV)
        oh, ol = (torch.zeros(rows1, N, dtype=torch.float16, device=DEV) for _ in range(2))
        op_gemm(path, frame_offsets([L]), rows1, st["w"], st["b"], dilation=2, res=res.to(DEV), ld_res=N, out=o1, ldo=N,
                oh=oh, ol=ol, ldh=N, vec2=st["bufs"]["vec2"].to(DEV), plane_act=R.LRELU, **args)
        o1, oh = o1.cpu()[r1:r1 + L], oh.cpu()[r1:r1 + L]
        ob, ohb = out["out"][r:r + L], out["oh"][r:r + L]
        if path == 0:
            assert torch.equal(_bits(o1), _bits(ob)) and torch.equal(_bits(oh), _bits(ohb)), (i, L)
        else:
            worst = max(worst, float(((o1.double() - ob.double()).abs() / ob.double().abs().clamp(min=1)).max()))
    print(f"path {path}: utterances <= 129 rows alone vs in the batch: "
          + ("bit-identical" if path == 0 else f"max error {worst:.3e} (bar {BAR['batch-tc']:.1e})"))
    assert worst <= BAR["batch-tc"]


def test_tap_reuse_matches_plain_kernel():
    """The same 3-tap conv on the tap-reuse pair kernel and, as a 5-tap conv with zero outer taps, on the plain pair kernel."""
    lens = pair_lens(256, 8)
    utts = subset(lens)
    c3 = Case("reuse k3 d8", 1, lens, 256, 256, 3, 8, R.GENERIC, seed=8, utts=utts, want="tc2r<64,GENERIC>", bar=BAR["reuse"])
    o3, st3, _ = run(c3)
    c5 = Case("plain k5 d8", 1, lens, 256, 256, 5, 8, R.GENERIC, seed=8, utts=utts, want="tc2<64,GENERIC>", bar=BAR["reuse"])
    st5 = _build(c5)
    w5 = torch.zeros(256, 256, 5)
    w5[:, :, 1:4] = st3["w"]
    st5["w"], st5["b"], st5["bufs"] = w5, st3["b"], st3["bufs"]
    dev5, got, _ = _call(c5, st5)
    assert got == {"tc2<64,GENERIC>": 1}, got
    o5 = dev5["out"].cpu()
    err = Err()
    for i in utts:
        r, n = st3["rs"][i], lens[i]
        err.add(i, o5[r:r + n], o3["out"][r:r + n].double())
    err.report("tap reuse vs plain", BAR["reuse-vs-plain"])


@pytest.mark.parametrize("case", ["reach17-ffma", "reach17-tc", "cin96-tc", "n96-tc", "tanh-tc", "mish-tc", "no-output-tc",
                                  "no-output-ffma", "rows-mismatch"])
def test_refused_before_any_launch(case):
    from stylesinger_b200._lib import lib
    from stylesinger_b200.engine import op_gemm
    lens = [40, 7]
    rs, rows = R.layout(lens)
    Cin, N, k, dil, path = 128, 128, 3, 1, 1
    kw = {}
    if case.startswith("reach17"):
        k, dil, path = 3, 17, (0 if case.endswith("ffma") else 1)
    elif case == "cin96-tc":
        Cin = 96
    elif case == "n96-tc":
        N = 96
    elif case in ("tanh-tc", "mish-tc"):
        kw["act"] = R.TANH if case == "tanh-tc" else R.MISH
    elif case == "no-output-ffma":
        path = 0
    w = torch.randn(N, Cin, k)
    a = torch.zeros(rows, Cin, device=DEV)
    planes = torch.zeros(rows, Cin, dtype=torch.float16, device=DEV)
    out = None if case.startswith("no-output") else torch.zeros(rows, N, device=DEV)
    args = dict(a=a, lda=Cin) if path == 0 else dict(a_hi=planes, a_lo=planes)
    torch.cuda.synchronize()
    n0 = lib.ssb_launch_count()
    with pytest.raises(SsbError) as ei:
        op_gemm(path, frame_offsets(lens), rows + (1 if case == "rows-mismatch" else 0), w, None, dilation=dil, out=out,
                ldo=N, **args, **kw)
    torch.cuda.synchronize()
    assert lib.ssb_launch_count() == n0
    print(f"{case}: refused: {ei.value}")


# ---------------------------------------------------------------------------------------------------------------------
# the tight-row wrappers engine.op_conv1d / op_conv1d_tc at the shapes the op-level tests have always covered
def _tight_ref(x, offs, w, b, dil, act, idx):
    out = {}
    for i in idx:
        xi = x[offs[i]:offs[i + 1]]
        out[i] = R.generic(R.accumulator(xi, w, dil, [len(xi)], [0]), b, a=act)[0]
    return out


@pytest.mark.parametrize("cin,n,k,dil,act", [(80, 256, 1, 1, 0), (256, 512, 3, 8, 1), (256, 1024, 9, 1, 2),
                                             (80, 160, 5, 1, 2), (192, 3, 1, 1, 0), (32, 32, 11, 1, 3), (32, 64, 3, 5, 3),
                                             (1104, 256, 1, 1, 0), (64, 80, 7, 1, 4)])
def test_op_conv1d_shapes(cin, n, k, dil, act):
    from stylesinger_b200.engine import op_conv1d
    g = torch.Generator().manual_seed(cin * 7 + n)
    lens = [5, 131, 64, 300, 1, 33]
    offs = frame_offsets(lens)
    x = torch.randn(int(offs[-1]), cin, generator=g)
    w = torch.randn(n, cin, k, generator=g) / (cin * k) ** 0.5
    b = torch.randn(n, generator=g)
    (y,), got, nl = launched(lambda: (op_conv1d(x.to(DEV), offs, w, b, dilation=dil, act=act).cpu(),))
    assert got == {} and nl >= 1
    ref = _tight_ref(x, offs, w, b, dil, act, range(len(lens)))
    err = Err()
    for i in ref:
        err.add(i, y[offs[i]:offs[i + 1]], ref[i])
    err.report(f"op_conv1d {cin}->{n} k{k} d{dil} act {act}", BAR["op_conv1d"])


_TC_SHAPES = (  # (cin, n, k, dil, lens)
    [(cin, n, k, dil, "mixed") for cin, n, k, dil in [(64, 128, 1, 1), (256, 512, 1, 1), (256, 512, 3, 8), (192, 384, 3, 2),
                                                      (192, 384, 1, 1), (256, 256, 3, 1)]]
    + [(cin, n, k, dil, f"pairs{reps}+{extra}") for cin, n, k, dil, reps, extra in
       [(256, 512, 3, 4, 1, 0), (256, 384, 3, 4, 1, 0), (256, 512, 3, 2, 1, 100), (192, 384, 1, 1, 1, 77),
        (128, 128, 7, 1, 1, 0), (64, 64, 11, 1, 2, 5), (64, 2048, 3, 1, 1, 0)]]
    + [(cin, n, k, dil, f"pairs{reps}+77") for cin, n, k, dil, reps in
       [(256, 512, 3, 4, 1), (256, 384, 3, 2, 1), (256, 512, 3, 8, 1), (256, 512, 3, 1, 1), (256, 512, 1, 1, 1),
        (192, 384, 5, 1, 1), (128, 128, 7, 1, 2), (64, 64, 11, 1, 2), (128, 128, 3, 1, 1)]])


@pytest.mark.parametrize("cin,n,k,dil,lens_kind", _TC_SHAPES)
def test_op_conv1d_tc_shapes(cin, n, k, dil, lens_kind):
    from stylesinger_b200.engine import op_conv1d_tc
    g = torch.Generator().manual_seed(11 + n + k + cin)
    if lens_kind == "mixed":
        lens = [5, 131, 64, 300, 128]
    else:
        reps, extra = lens_kind[5:].split("+")
        lens = [2800, 1500, 2999, 700, 2100, 1900, 2500, 3000, 1234, 2222] * int(reps) + ([int(extra)] if int(extra) else [])
    offs = frame_offsets(lens)
    x = torch.randn(int(offs[-1]), cin, generator=g)
    w = torch.randn(n, cin, k, generator=g) / (cin * k) ** 0.5
    b = torch.randn(n, generator=g)
    (y,), got, _ = launched(lambda: (op_conv1d_tc(x.to(DEV), offs, w, b, dilation=dil).cpu(),))
    want = variant(ntiles(lens), n, "GENERIC", k, dil)
    assert got == {want: 1}, (got, want)
    idx = sorted({0, 3 % len(lens), len(lens) // 2, len(lens) - 1})
    ref = _tight_ref(x, offs, w, b, dil, 0, idx)
    err = Err()
    for i in idx:
        err.add(i, y[offs[i]:offs[i + 1]], ref[i])
    err.report(f"op_conv1d_tc {cin}->{n} k{k} d{dil} on {int(offs[-1])} rows [{want}]", BAR["op_conv1d_tc"])
