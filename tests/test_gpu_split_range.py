"""The tensor-core GEMMs across operand exponents, one ssb_op_gemm call at a time, and the denoisers' zero-initialised
output projection through ssb_denoiser_eval.

Every tensor-core GEMM carries an fp32 operand as fp16 planes hi = fp16(x), lo = fp16(x - hi).  lo is a normal fp16 number
only while |x| >= 2^-3, and hi overflows above 65504, so the split's accuracy depends on the operands' exponents.  The
packer splits w 2^s with one power of two per weight tensor (csrc/pack.cu pack_conv_tc) and the epilogue multiplies the
accumulator by 2^-s; the activations keep an absolute floor of 2^-25 per element below 2^-3 (DESIGN.md, "Precision
decision").  On every variant the dispatch reaches (the shapes of tests/test_gpu_conv_gemm_f64.py, each call asserting
its variant), in the 3-pass and the single-pass (',fp16') form, with the FFMA kernel as the control:

(a) weight-scale equivariance: out(w 2^e, b 2^e, res 2^e) == 2^e out(w, b, res) bit for bit, e in -30 .. 20, GENERIC with
    act none, ReLU and LReLU (single-pass form included: that is (e)'s sweep);
(b) float64 accuracy per output element against err <= C_gemm D + C_epi S, D = sum_{k,tap} |a||w|, S = |ref| + the
    epilogue's addends (+ 1 on GATE, the gate activation's absolute error), with constants calibrated at e = 0 and held at
    every weight exponent, on GENERIC, GATE and RES_SKIP;
(c) activations scaled by 2^f, f in -24 .. 10: FFMA bitwise equivariant, tensor cores within (b)'s bar plus the activation
    floor 2^-25 sum |w|;
(d) an all-zero weight tensor (the reference's untrained output_projection): the output is exactly the bias;
(e) the single-pass form against its float64 emulation (operands rounded as the kernel rounds them, the weights as the
    packer does: tests/fp16_emulation.py r16w), at every weight exponent;
(f) ssb_denoiser_eval of the mel DiffNet and both F0 DDiffNets with the final output_projection weight and bias scaled by
    2^e: eps is exactly 2^e eps, on the tensor cores, on FFMA and (mel) in the single-pass mode."""
import gc

import pytest
import torch

from tests import conv_gemm_ref as R
from tests import fp16_emulation as E
from tests.gpu_checks import frame_offsets, launched
from tests.test_gpu_conv_gemm_f64 import _TC, EDGE_LENS, pair_lens, subset

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
E_W = [-30, -24, -16, -12, -8, -4, -1, 1, 4, 8, 16, 20]
E_ACC = [0, -4, -8, -12, -16, -24, 4, 8]          # weight exponents of the float64 checks
F_ACT = list(range(-24, 11, 2))                    # activation exponents
MODES = ("GENERIC", "GATE", "RES_SKIP")
# Bars: C_gemm at most 4x the largest err / D measured at e = 0 over every variant and mode of its form on an H100 SXM
# (80 GB HBM3, 700 W), the measured value beside it; C_epi a few fp32 roundings of the epilogue's terms.
C_GEMM = {"split": 1e-6,     # 1.04e-6 (tc2r<64,GENERIC>)
          "fp16": 1.15e-3,   # 2.96e-4 (tc<64,RES_SKIP>)
          "ffma": 4e-7}      # 3.57e-7
C_EMU = 1e-6   # 4.3e-7: the single-pass form against its emulation, i.e. the tensor core's fp32 accumulation alone
C_EPI = 2.0 ** -21
FLOOR = 2.0 ** -25  # activation floor: half an ulp of a subnormal fp16 lo (or hi) per element

TC_CASES = [(n, Cin, N, k, dil, mode) for n, Cin, N, k, dil, mode, _ in _TC]
TC_GENERIC = [c for c in TC_CASES if c[5] == R.GENERIC]
FFMA_CASES = [("conv_gemm_kernel<128>", 128, 256, 3, 2, R.GENERIC), ("conv_gemm_kernel<128>", 64, 128, 3, 16, R.GATE),
              ("conv_gemm_kernel<128>", 128, 256, 1, 1, R.RES_SKIP)]
ACTS = [(R.NONE, 0.1), (R.RELU, 0.1), (R.LRELU, 0.2)]


def _id(c):
    return f"{c[0]}-Cin{c[1]}-N{c[2]}-k{c[3]}"


def _want(name, form):
    return name[:-1] + ",fp16>" if form == "fp16" else name


def _scale(t, e):
    return None if t is None else torch.ldexp(t, torch.tensor(float(e)))


_CASES = {}


def case(c):
    """Inputs of one shape, memoised: lens, layout, the utterances compared with float64, x, w, bias, addends."""
    if c not in _CASES:
        name, Cin, N, k, dil, mode = c
        pair = name.startswith("tc2")
        lens = pair_lens(N, Cin + N) if pair else EDGE_LENS
        rs, rows = R.layout(lens)
        valid = R.valid_rows(lens, rs, rows)
        g = torch.Generator().manual_seed(Cin * 7 + N + k)
        nv = int(valid.sum())

        def rand_rows(cols, scale=1.0):
            t = torch.zeros(rows, cols)
            t[valid] = scale * torch.randn(nv, cols, generator=g)
            return t

        C = N // 2
        _CASES[c] = dict(lens=lens, rs=rs, rows=rows, valid=valid, utts=subset(lens) if pair else list(range(len(lens))),
                         x=rand_rows(Cin), w=torch.randn(N, Cin, k, generator=g) / (Cin * k) ** 0.5,
                         b=torch.randn(N, generator=g), res=rand_rows(N if mode == R.GENERIC else C),
                         add=rand_rows(N, 4.0), skip=rand_rows(C))
    return _CASES[c]


def gemm(c, form, w, b, x, res=None, add=None, skip=None, act=R.NONE, slope=0.1, check=True):
    """One ssb_op_gemm call of shape c in `form` ('split' | 'fp16' | 'ffma'): {output name: CPU tensor}; GATE planes come
    back as their value hi + lo (float64)."""
    from stylesinger_b200.engine import op_gemm
    name, Cin, N, k, dil, mode = c
    st = case(c)
    rows, C = st["rows"], N // 2
    path = 0 if form == "ffma" else 1
    a = dict(a=x.to(DEV), lda=Cin) if path == 0 else dict(zip(("a_hi", "a_lo"), (t.to(DEV) for t in R.split(x))))
    o = {}
    if mode == R.GENERIC:
        o["out"] = torch.zeros(rows, N, device=DEV)
        a.update(out=o["out"], ldo=N, act=act, act_slope=slope)
        if res is not None:
            a.update(res=res.to(DEV), ld_res=N)
    elif mode == R.GATE:
        a.update(add=add.to(DEV), ld_add=N)
        if path == 0:
            o["out"] = torch.zeros(rows, C, device=DEV)
            a.update(out=o["out"], ldo=C)
        else:
            o["oh"], o["ol"] = (torch.zeros(rows, C, dtype=torch.float16, device=DEV) for _ in range(2))
            a.update(oh=o["oh"], ol=o["ol"], ldh=C)
    else:
        o["out"], o["skip"] = torch.zeros(rows, C, device=DEV), skip.clone().to(DEV)
        a.update(res=res.to(DEV), ld_res=C, out=o["out"], ldo=C, skip=o["skip"], ld_skip=C, C=C, skip_init=0)
    _, got, nl = launched(lambda: op_gemm(path, frame_offsets(st["lens"]), rows, w, b, dilation=dil, gate=mode == R.GATE,
                                          mode=mode, single_pass=form == "fp16", **a))
    if check:
        assert nl == 1 and got == ({} if path == 0 else {_want(name, form): 1}), (name, form, got, nl)
    out = {k_: v.cpu() for k_, v in o.items()}
    if "oh" in out:
        out = {"out": out["oh"].double() + out["ol"].double()}
    return out


_ACC = {}


def reference(c, e, f, b, res, add, skip, emu=False):
    """float64 {output: (ref, D, S)} of the case's weights scaled by 2^e and activations by 2^f, over every row (rows outside
    the compared utterances are zero).  emu: the single-pass form's operands, fp16(x) and the packer's rounding of w.  The
    accumulator and D are computed once per case: a power-of-two scale of an operand scales them exactly."""
    name, Cin, N, k, dil, mode = c
    st = case(c)
    if (c, emu) not in _ACC:
        xv, wv = st["x"].double(), st["w"].double()
        if emu:
            xv, wv = E.r16(xv), E.r16w(wv)
        lens, rs, utts = st["lens"], st["rs"], st["utts"]
        _ACC[(c, emu)] = (R.accumulator(xv, wv, dil, lens, rs, utts), R.accumulator(xv.abs(), wv.abs(), dil, lens, rs, utts))
    acc, D = (torch.ldexp(t, torch.tensor(float(e + f), dtype=torch.float64)) for t in _ACC[(c, emu)])
    bd = b.double()
    if mode == R.GENERIC:
        ref = acc + bd + res.double()
        return {"out": (ref, D, ref.abs() + bd.abs() + res.double().abs())}
    C = N // 2
    if mode == R.GATE:
        z = R.gate(acc, b, add)
        ap = add.double().abs()
        S = z.abs() + 1 + bd[:C].abs() + bd[C:].abs() + ap[:, 0::2] + ap[:, 1::2]
        return {"out": (z, D[:, :C] + D[:, C:], S)}
    xn, _, s = R.res_skip(acc, C, b, res, 1.0, None, skip, False)
    return {"out": (xn, D[:, :C], xn.abs() + bd[:C].abs() + res.double().abs()),
            "skip": (s, D[:, C:], s.abs() + bd[C:].abs() + skip.double().abs())}


def compare(tag, c, got, ref, cg, floor=None):
    """max over the compared rows of err / bar (<= 1 passes), and max err / D for the calibration."""
    st = case(c)
    rows = torch.zeros(st["rows"], dtype=torch.bool)
    for i in st["utts"]:
        rows[st["rs"][i]:st["rs"][i] + st["lens"][i]] = True
    worst, per_d = 0.0, 0.0
    for k_, (r, D, S) in ref.items():
        err = (got[k_].double() - r).abs()[rows]
        bar = cg * D[rows] + C_EPI * S[rows] + (0 if floor is None else floor)
        assert torch.isfinite(got[k_][rows]).all(), (tag, k_, "non-finite output")
        worst = max(worst, float((err / bar).max()))
        per_d = max(per_d, float((err / D[rows].clamp(min=1e-300)).max()))
    print(f"{tag}: err / bar {worst:.3f}, max err / D {per_d:.3e}")
    return worst, per_d


def _forms(c):
    return ["ffma"] if c[0].startswith("conv_gemm") else ["split", "fp16"]


# ---------------------------------------------------------------------------------------------------------------------
# (a) + (e, sweep): weight-scale equivariance, bit for bit
@pytest.mark.parametrize("form", ["split", "fp16", "ffma"])
@pytest.mark.parametrize("c", TC_GENERIC + FFMA_CASES[:1], ids=_id)
def test_weight_scale_equivariance_bitwise(c, form):
    if form not in _forms(c):
        pytest.skip("the FFMA kernel has one form")
    st = case(c)
    bad = []
    for act, slope in ACTS:
        base = gemm(c, form, st["w"], st["b"], st["x"], res=st["res"], act=act, slope=slope)["out"]
        for e in E_W:
            o = gemm(c, form, _scale(st["w"], e), _scale(st["b"], e), st["x"], res=_scale(st["res"], e), act=act,
                     slope=slope)["out"]
            want = _scale(base, e)
            same = torch.equal(o.view(torch.int32), want.view(torch.int32))
            if not same:
                nfin = int((~torch.isfinite(o[st["valid"]])).sum())
                bad.append((act, e, int((o.view(torch.int32) != want.view(torch.int32)).sum()), nfin))
    print(f"{c[0]} {form}: {len(ACTS) * len(E_W)} scaled calls, not equivariant (act, e, elements differing, non-finite): "
          f"{bad}")
    assert not bad


# ---------------------------------------------------------------------------------------------------------------------
# (b) float64 accuracy at every weight exponent, constants held
@pytest.mark.parametrize("form", ["split", "fp16", "ffma"])
@pytest.mark.parametrize("c", TC_CASES + FFMA_CASES, ids=_id)
def test_weight_exponent_accuracy(c, form):
    if form not in _forms(c):
        pytest.skip("the FFMA kernel has one form")
    st = case(c)
    mode = c[5]
    scaled = mode != R.GATE  # GATE: bias and addend stay O(1) (the gate of tiny arguments is the epilogue's, not the GEMM's)
    worst = {}
    for e in E_ACC:
        w = _scale(st["w"], e)
        b, res, skip, add = (st["b"], st["res"], st["skip"], st["add"]) if not scaled else (
            _scale(st["b"], e), _scale(st["res"], e), _scale(st["skip"], e), st["add"])
        got = gemm(c, form, w, b, st["x"], res=res, add=add, skip=skip)
        ref = reference(c, e, 0, b, res, add, skip)
        worst[e] = compare(f"{c[0]} {MODES[mode]} {form} e={e}", c, got, ref, C_GEMM[form])
    print(f"{c[0]} {form}: calibration at e = 0: max err / D {worst[0][1]:.3e} (C_gemm {C_GEMM[form]:.1e})")
    assert all(v[0] <= 1.0 for v in worst.values()), {e: v[0] for e, v in worst.items() if v[0] > 1.0}


# ---------------------------------------------------------------------------------------------------------------------
# (c) activation exponent sweep
@pytest.mark.parametrize("form", ["split", "fp16", "ffma"])
@pytest.mark.parametrize("c", TC_GENERIC + FFMA_CASES[:1], ids=_id)
def test_activation_exponent_sweep(c, form):
    if form not in _forms(c):
        pytest.skip("the FFMA kernel has one form")
    st = case(c)
    sumw = st["w"].double().abs().sum(dim=(1, 2))  # sum over Cin and taps of |w|, per output column
    base = gemm(c, form, st["w"], st["b"], st["x"], res=st["res"])["out"] if form == "ffma" else None
    worst = 0.0
    for f in F_ACT:
        x, b, res = _scale(st["x"], f), _scale(st["b"], f), _scale(st["res"], f)
        assert float(x.abs().max()) < 65504
        got = gemm(c, form, st["w"], b, x, res=res)
        if form == "ffma":
            assert torch.equal(got["out"].view(torch.int32), _scale(base, f).view(torch.int32)), f
            continue
        ref = reference(c, 0, f, b, res, None, None)
        worst = max(worst, compare(f"{c[0]} {form} f={f}", c, got, ref, C_GEMM[form], FLOOR * sumw[None, :])[0])
    if form == "ffma":
        print(f"{c[0]} ffma: activations 2^{F_ACT[0]} .. 2^{F_ACT[-1]}: bit for bit equivariant")
    assert worst <= 1.0


# ---------------------------------------------------------------------------------------------------------------------
# (d) all-zero weights
@pytest.mark.parametrize("c", TC_GENERIC + FFMA_CASES[:1], ids=_id)
def test_zero_weights_give_the_bias(c):
    st = case(c)
    w0 = torch.zeros_like(st["w"])
    want = torch.zeros(st["rows"], c[2])
    want[st["valid"]] = st["b"]
    for form in _forms(c):
        o = gemm(c, form, w0, st["b"], st["x"])["out"]
        assert torch.equal(o[st["valid"]].view(torch.int32), want[st["valid"]].view(torch.int32)), form
    print(f"{c[0]}: zero weights -> exactly the bias on {_forms(c)}")


# ---------------------------------------------------------------------------------------------------------------------
# (e) single-pass form against its float64 emulation at every weight exponent
@pytest.mark.parametrize("c", TC_CASES, ids=_id)
def test_single_pass_matches_emulation(c):
    st = case(c)
    mode = c[5]
    worst = 0.0
    w16 = E.r16w(st["w"].double())
    for e in [0] + E_W:
        w = _scale(st["w"], e)
        lin = mode != R.GATE
        b, res, skip = (_scale(st["b"], e), _scale(st["res"], e), _scale(st["skip"], e)) if lin else (
            st["b"], st["res"], st["skip"])
        assert torch.equal(E.r16w(w.double()), _scale(w16, e))  # the packer's rounding commutes with the scale
        got = gemm(c, "fp16", w, b, st["x"], res=res, add=st["add"], skip=skip)
        ref = reference(c, e, 0, b, res, st["add"], skip, emu=True)
        worst = max(worst, compare(f"{c[0]} {MODES[mode]} fp16 vs emulation e={e}", c, got, ref, C_EMU)[0])
    assert worst <= 1.0


# ---------------------------------------------------------------------------------------------------------------------
# (f) the denoisers' output projection, scaled, through ssb_denoiser_eval
PREFIX = ("postdiff.denoise_fn.", "gm_diffnet.", "gm_diffnet_inpainte.")


def _free_device_memory():
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


@pytest.fixture(scope="module", autouse=True)
def _release_caches():
    """Free the module's cached inputs and references when it ends, so that the modules after it in the same process get
    the memory back."""
    yield
    _CASES.clear()
    _ACC.clear()
    _free_device_memory()
    print(f"after test_gpu_split_range: {torch.cuda.memory_allocated() / 2**30:.2f} GiB allocated by torch, "
          f"{torch.cuda.mem_get_info()[0] / 2**30:.1f} GiB free on the device")


def _scaled_model(e):
    """An acoustic model whose three denoisers have output_projection weight and bias scaled by 2^e.  Not cached: at bench
    size a model's denoiser workspace is several GB, so one model lives at a time."""
    from stylesinger_b200.engine import AcousticModel
    from tests.common import acoustic_sd, hp_for
    from tests.test_gpu_denoisers import T
    sd = dict(acoustic_sd())
    for p in PREFIX:
        for n in ("weight", "bias"):
            sd[p + "output_projection." + n] = _scale(sd[p + "output_projection." + n], e)
    return AcousticModel(sd, hp_for(T))


@pytest.mark.parametrize("size", ["small", "mid", "bench"])
@pytest.mark.parametrize("which", [0, 1, 2], ids=["mel", "f0_agnostic", "f0_specific"])
def test_denoiser_output_projection_scale_bitwise(which, size):
    from tests.test_gpu_denoisers import batch, eval_inputs, expected_eval
    b = batch(size)
    t = 50
    x, uv = eval_inputs(which, t, b)
    paths = [("tc", "split"), ("ffma", "split")] + ([("tc", "fp16")] if which == 0 else [])
    want = expected_eval(which, b["lens"])
    outs = {p: {} for p in paths}
    for e in (0, -12, -6, 6):
        m = _scaled_model(e)
        try:
            for path, prec in paths:
                m.set_tensor_cores(path == "tc")
                m.set_mel_precision(prec)
                outs[(path, prec)][e], got, _ = launched(
                    lambda: m.denoiser_eval(which, x, uv, t, b["cond"], b["offs"]).cpu())
                if path == "tc":
                    assert {k.replace(",fp16", ""): v for k, v in got.items()} == want, (path, prec, got, want)
                    assert all(k.endswith(",fp16>") == (prec == "fp16") for k in got), got
                else:
                    assert got == {}, got
        finally:
            del m
            _free_device_memory()
    for (path, prec), o in outs.items():
        for e in (-12, -6, 6):
            diff = int((o[e].view(torch.int32) != _scale(o[0], e).view(torch.int32)).sum())
            print(f"net {which} {size} {path} {prec}: output_projection x 2^{e}: {diff} of {o[0].numel()} outputs "
                  f"differ from 2^{e} eps")
            assert diff == 0, (which, size, path, prec, e)
