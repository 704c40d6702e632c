"""The single-pass fp16 tensor-core mode (SSB_TC_FP16, hparams['tc_precision'] = 'fp16') on the GPU, against the float64
emulation of tests/fp16_emulation.py (operands of each tensor-core contraction rounded to fp16, sums in float64) and
against the fp32-faithful float64 oracles, whose distance is reported.

1. ssb_op_gemm with single_pass = 1 on every tensor-core variant (tc<64,·>, tc2<32|64,·>, tc2r<32|64,GATE|GENERIC>) and
   the GATE, RES_SKIP and GENERIC epilogues, at tile-edge lengths, with a_lo not passed (the kernel must not read it).
   Bar: 1e-5 of max(1, |x|) (fp32 accumulation of exact fp16 products); GATE 2e-5 (its ex2.approx epilogue, as the split
   kernel's bar in tests/test_gpu_conv_gemm_f64.py).
2. The mel sampler with injected noise: T = 4 on the persistent kernel and on the per-launch kernels, T = 100 on both at
   bench lengths, PLMS and ProDiff once each.  The GPU is compared with the emulation and with the float64 chain; its
   distance to the float64 chain must be within 2x the emulation's own.
3. The vocoder, V1 / V2 / V3, against the emulation, with the distance to the float64 generator reported.
4. A full forward at the bench's batch64 lengths: every output before the mel stage is bit-identical to split mode.
5. Switching a model or vocoder to fp16 and back gives output bit-identical to one never switched; with per-utterance
   seeds each utterance of an fp16 mel batch is bit-identical to its own B = 1 call (same GEMM variants: these utterances
   stay below the CTA-pair sizes).  The vocoder's B = 1 calls take other variants than its batches, so they are not
   compared bit for bit."""
import numpy as np
import pytest
import torch

from tests import conv_gemm_ref as R
from tests import denoiser_oracle as DO
from tests import fp16_emulation as E
from tests import test_gpu_denoisers as D
from tests.common import acoustic_engine, hp_for
from tests.gpu_checks import frame_offsets, launched, ntiles, split

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
EDGE_LENS = [1, 2, 3, 31, 32, 33, 63, 64, 65, 127, 128, 129, 255, 256, 257]


def _linf(a, b):
    a = a.detach().cpu().double() if isinstance(a, torch.Tensor) else torch.as_tensor(np.asarray(a, np.float64))
    b = b.detach().cpu().double() if isinstance(b, torch.Tensor) else torch.as_tensor(np.asarray(b, np.float64))
    return float((a - b).abs().max())


# ---------------------------------------------------------------------------------------------------------------------
# 1. op level
def _pair_lens(N):
    """EDGE_LENS padded with bench-like lengths to the fewest row tiles that take the CTA-pair kernel at N."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    hb = 64 if N % 128 == 0 else 32
    need = 2 * (-(-sms // (N // (2 * hb))))
    lens = list(EDGE_LENS)
    rng = np.random.default_rng(N)
    while ntiles(lens) < need:
        lens.append(int(rng.integers(100, 1500)))
    return lens


OP_CASES = [  # (tag, Cin, N, taps, dil, mode, pair, expected variant)
    ("generic-1cta", 128, 128, 1, 1, R.GENERIC, False, "tc<64,GENERIC,fp16>"),
    ("gate-1cta", 128, 256, 3, 2, R.GATE, False, "tc<64,GATE,fp16>"),
    ("res_skip-1cta", 128, 256, 1, 1, R.RES_SKIP, False, "tc<64,RES_SKIP,fp16>"),
    ("generic-pair64", 256, 256, 1, 1, R.GENERIC, True, "tc2<64,GENERIC,fp16>"),
    ("generic-pair32", 128, 192, 5, 1, R.GENERIC, True, "tc2<32,GENERIC,fp16>"),
    ("res_skip-pair64", 256, 512, 1, 1, R.RES_SKIP, True, "tc2<64,RES_SKIP,fp16>"),
    ("gate-reuse64", 256, 512, 3, 4, R.GATE, True, "tc2r<64,GATE,fp16>"),
    ("generic-reuse32", 64, 192, 3, 8, R.GENERIC, True, "tc2r<32,GENERIC,fp16>"),
    ("gate-reuse32", 64, 192, 3, 1, R.GATE, True, "tc2r<32,GATE,fp16>"),
]
BAR_OP = {R.GENERIC: 1e-5, R.RES_SKIP: 1e-5, R.GATE: 2e-5}


@pytest.mark.parametrize("case", OP_CASES, ids=[c[0] for c in OP_CASES])
def test_op_gemm_single_pass_matches_fp16_emulation(case):
    from stylesinger_b200.engine import op_gemm
    tag, Cin, N, k, dil, mode, pair, want = case
    lens = _pair_lens(N) if pair else EDGE_LENS
    rs, rows = R.layout(lens)
    valid = R.valid_rows(lens, rs, rows)
    g = torch.Generator().manual_seed(Cin + N + k)
    x = torch.zeros(rows, Cin)
    x[valid] = torch.randn(int(valid.sum()), Cin, generator=g)
    w = torch.randn(N, Cin, k, generator=g) / (Cin * k) ** 0.5
    b = torch.randn(N, generator=g)
    hi, _ = R.split(x)
    acc = R.accumulator(E.r16(x.double()), E.r16w(w.double()), dil, lens, rs)
    offs = frame_offsets(lens)
    args = dict(a_hi=hi.to(DEV))
    C = N // 2
    if mode == R.GENERIC:
        res = torch.zeros(rows, N)
        res[valid] = torch.randn(int(valid.sum()), N, generator=g)
        out = torch.zeros(rows, N, device=DEV)
        args.update(out=out, ldo=N, res=res.to(DEV), ld_res=N, act=R.LRELU, act_slope=0.1)
        ref, _ = R.generic(acc, b, a=R.LRELU, slope=0.1, res=res)
        cols = N
    elif mode == R.GATE:
        add = torch.zeros(rows, N)
        add[valid] = torch.randn(int(valid.sum()), N, generator=g)
        oh = torch.zeros(rows, C, dtype=torch.float16, device=DEV)
        ol = torch.zeros_like(oh)
        args.update(add=add.to(DEV), ld_add=N, oh=oh, ol=ol, ldh=C)
        ref = R.gate(acc, b, add)
        cols = C
    else:
        y = torch.zeros(rows, C)
        y[valid] = torch.randn(int(valid.sum()), C, generator=g)
        vec1 = torch.randn(C, generator=g)
        y = y + vec1 * valid[:, None]
        rh, rl = R.split(y)
        xr = R.planes_value(rh, rl) - vec1.double() * valid[:, None]
        skip = torch.zeros(rows, C, device=DEV)
        out = torch.zeros(rows, C, device=DEV)
        args.update(rh=rh.to(DEV), rl=rl.to(DEV), ld_rh=C, vec1=vec1.to(DEV), C=C, skip=skip, ld_skip=C, skip_init=1,
                    out=out, ldo=C, beta=0.70710678)
        xn, _, s = R.res_skip(acc, C, b, xr, 0.70710678, None, None, True, None)
        ref = torch.cat([xn, s], 1)
        cols = 2 * C
    _, variants, _ = launched(lambda: op_gemm(1, offs, rows, w, b, dilation=dil, gate=mode == R.GATE, mode=mode,
                                              single_pass=True, **args))
    torch.cuda.synchronize()
    if mode == R.GENERIC:
        got = out.cpu()
    elif mode == R.GATE:
        got = R.planes_value(oh.cpu(), ol.cpu())
    elif mode == R.RES_SKIP:
        got = torch.cat([out.cpu(), skip.cpu()], 1)
    err = float(((got.double() - ref)[valid, :cols].abs() / ref[valid, :cols].abs().clamp(min=1.0)).max())
    full = R.accumulator(x.double(), w.double(), dil, lens, rs)
    gap = float((acc - full)[valid].abs().max())
    print(f"op {tag}: {variants} err vs fp16 emulation {err:.2e} (bar {BAR_OP[mode]:.0e}); fp16 rounding moves the "
          f"accumulator by up to {gap:.2e}")
    assert all(",fp16>" in v for v in variants), variants
    if want:
        assert want in variants, variants
    assert err < BAR_OP[mode]
    assert gap > 10 * BAR_OP[mode]  # the bar separates fp16 from the split kernel's result


# ---------------------------------------------------------------------------------------------------------------------
# 2. mel samplers
def _mel_case(name, K, T):
    b = D.batch(name) if name != "one_tile" else D._one_tile()
    offs = b["offs"]
    noise = D._mel_noise(K, int(offs[-1]), 70 + K)
    coarse = D._chain_coarse(name, int(offs[-1]))
    hp = dict(hp_for(T), K_step=K)
    cs, co = split(b["cond"], offs), split(coarse, offs)
    lens = b["lens"]
    # T = 100 in float64 on the CPU: the shortest utterance only (and its own tile edges); T = 4: every utterance
    pick = list(range(len(cs))) if T < 100 else [int(np.argmin(lens))]
    ref, emu = {}, {}
    for i in pick:
        nz = noise[:, int(offs[i]):int(offs[i + 1])]
        ref[i] = DO.mel_chain64(cs[i], co[i], hp, K, nz)["mel"]
        with E.fp16_convs():
            emu[i] = DO.mel_chain64(cs[i], co[i], hp, K, nz)["mel"]
    return b, noise, coarse, ref, emu


@pytest.mark.parametrize("name,K,T", [("ragged", 4, 4), ("bench6", 4, 4), ("one_tile", 100, 100), ("bench6", 100, 100)])
def test_mel_sampler_fp16_matches_emulation(name, K, T):
    b, noise, coarse, ref, emu = _mel_case(name, K, T)
    m = acoustic_engine(T, 4)  # after _mel_case: the batch helpers re-table the shared engine
    m.set_mel_k_step(K if K != T else 0)
    offs = b["offs"]
    paths = (["persistent"] if ntiles(b["lens"]) <= 48 else []) + ["tc"]
    try:
        m.set_mel_precision("fp16")
        for path in paths:
            m.set_persistent(path == "persistent")
            mel, variants, _ = launched(lambda: m.mel_diffusion(b["cond"], coarse, offs, noise.to(DEV)).clone())
            assert all(",fp16>" in v for v in variants), variants
            ys = split(mel, offs)
            e_emu = max(_linf(ys[i], emu[i]) for i in emu)
            e_gpu = max(_linf(ys[i], ref[i]) for i in ref)
            e_ref = max(_linf(emu[i], ref[i]) for i in ref)
            print(f"mel {name} K={K} {path} fp16: L-inf vs emulation {e_emu:.2e}, vs float64 {e_gpu:.2e} "
                  f"(emulation vs float64 {e_ref:.2e})")
            assert np.isfinite(mel.cpu().numpy()).all()
            assert e_gpu <= 2 * e_ref
            assert e_emu <= e_ref  # the GPU sits at least as close to the emulation as the emulation to fp32
    finally:
        m.set_mel_precision("split")
        m.set_persistent(True)
        m.set_mel_k_step(0)


def test_plms_and_prodiff_fp16_match_emulation():
    from tests import sampler_oracle as SO
    from tests.common import prodiff_hp, prodiff_sd
    from stylesinger_b200.engine import AcousticModel
    b = D.batch("ragged")
    offs = b["offs"]
    cs = split(b["cond"], offs)
    lens = b["lens"]
    pick = [lens.index(1), lens.index(129), lens.index(700)]
    # PLMS, K = 100, interval 10, injected q_sample draw
    m = acoustic_engine(100, 4)
    q = D._mel_noise(0, int(offs[-1]), 91)[0]
    coarse = D._chain_coarse("ragged", int(offs[-1]))
    co, qs = split(coarse, offs), split(q, offs)
    hp = hp_for(100)
    try:
        m.set_mel_precision("fp16")
        mel, variants, _ = launched(lambda: m.mel_diffusion_plms(b["cond"], coarse, offs, 10, q.to(DEV)).clone())
    finally:
        m.set_mel_precision("split")
    ys = split(mel, offs)
    for i in pick:
        ref = SO.plms_chain64(cs[i], co[i], hp, 100, 10, qs[i])["mel"]
        with E.fp16_convs():
            emu = SO.plms_chain64(cs[i], co[i], hp, 100, 10, qs[i])["mel"]
        e_emu, e_gpu, e_ref = _linf(ys[i], emu), _linf(ys[i], ref), _linf(emu, ref)
        print(f"plms utt {i} fp16: L-inf vs emulation {e_emu:.2e}, vs float64 {e_gpu:.2e} (emulation {e_ref:.2e})")
        assert e_gpu <= 2 * e_ref and e_emu <= e_ref
    # ProDiff, T = 4, injected noise, persistent kernel
    hpp = prodiff_hp(4)
    pm = AcousticModel(prodiff_sd(), hpp)
    pm.set_mel_precision("fp16")
    noise = D._mel_noise(4, int(offs[-1]), 93)
    mel = pm.mel_prodiff(b["cond"], offs, noise.to(DEV)).clone()
    ys = split(mel, offs)
    for i in pick:
        nz = noise[:, int(offs[i]):int(offs[i + 1])]
        ref = SO.prodiff_chain64(cs[i], hpp, nz)["mel"]
        with E.fp16_convs():
            emu = SO.prodiff_chain64(cs[i], hpp, nz)["mel"]
        e_emu, e_gpu, e_ref = _linf(ys[i], emu), _linf(ys[i], ref), _linf(emu, ref)
        print(f"prodiff utt {i} fp16: L-inf vs emulation {e_emu:.2e}, vs float64 {e_gpu:.2e} (emulation {e_ref:.2e})")
        assert e_gpu <= 2 * e_ref and e_emu <= e_ref


# ---------------------------------------------------------------------------------------------------------------------
# 3. vocoder
@pytest.mark.parametrize("name", ["v1", "v2", "v3"])
def test_vocoder_fp16_matches_emulation(name):
    from oracle import stylesinger_oracle as O
    from stylesinger_b200.engine import Vocoder
    from stylesinger_b200.hparams import DEFAULT_VOCODER_CONFIG
    from tests import test_gpu_vocoder_layouts as VL
    from tests.common import VOCODER_LAYOUTS, vocoder_sd
    h = DEFAULT_VOCODER_CONFIG if name == "v1" else VOCODER_LAYOUTS[name]
    sd = vocoder_sd(None if name == "v1" else name)
    v = Vocoder(sd, h, tc_precision="fp16")
    utts = [VL.Utt(*VL._synth_utt(L, 40 + L), 40 + L) for L in (1, 37, 128, 400)]
    wav, variants, _ = launched(lambda: VL._generate(v, utts))
    assert variants and all(",fp16>" in k for k in variants), variants
    for u, w in zip(utts, VL._split(wav, utts)):
        ref = O.spec2wav(u.mel, u.f0, sd, h, O.NoiseSource(u.seed), torch.float64)
        with E.fp16_convs(E.vocoder_tc_conv):
            emu = O.spec2wav(u.mel, u.f0, sd, h, O.NoiseSource(u.seed), torch.float64)
        e_emu, e_gpu, e_ref = _linf(w, emu), _linf(w, ref), _linf(emu, ref)
        print(f"vocoder {name} L={u.L} fp16: wav L-inf vs emulation {e_emu:.2e}, vs float64 {e_gpu:.2e} "
              f"(emulation {e_ref:.2e})")
        assert np.isfinite(w).all()
        assert e_gpu <= 2 * e_ref + 1e-6 and e_emu <= max(e_ref, 1e-6)


# ---------------------------------------------------------------------------------------------------------------------
# 4 / 5. whole model
def _bench_pb():
    from stylesinger_b200 import synth
    from stylesinger_b200.engine import pack_batch
    utts = [synth.make_utterance(float(s), utt_idx=i) for i, s in enumerate(synth.batch_seconds(64, seed=1234))]
    return pack_batch(utts).to(DEV)


def test_forward_fp16_leaves_pre_mel_outputs_bit_identical():
    m = acoustic_engine(4, 4)
    pb = _bench_pb()
    keys = ("mel2ph", "style", "rq_codes", "pitch_pred", "f0_denorm", "mel_out")
    a = {k: v.clone() for k, v in m.forward(pb, seed=3, want=keys).items()}
    try:
        m.set_mel_precision("fp16")
        b = {k: v.clone() for k, v in m.forward(pb, seed=3, want=keys).items()}
    finally:
        m.set_mel_precision("split")
    for k in keys[:-1]:
        assert torch.equal(a[k], b[k]), k
    d = _linf(a["mel_out"], b["mel_out"])
    print(f"forward batch64 T=4: mel_out fp16 vs split L-inf {d:.2e}")
    assert torch.isfinite(b["mel_out"]).all() and 0 < d < 0.1


def test_switching_back_is_bit_identical_and_keyed_seeds_hold():
    from stylesinger_b200 import synth
    from stylesinger_b200.engine import AcousticModel, Vocoder, pack_batch
    from tests.common import acoustic_sd, vocoder_sd
    from stylesinger_b200.hparams import DEFAULT_VOCODER_CONFIG
    utts = [synth.make_utterance(s, utt_idx=50 + i) for i, s in enumerate((0.6, 2.5, 1.1))]
    pb = pack_batch(utts).to(DEV)
    fresh = AcousticModel(acoustic_sd(), hp_for(4))
    sw = AcousticModel(acoustic_sd(), hp_for(4))
    sw.set_mel_precision("fp16")
    f16 = sw.forward(pb, seeds=[7, 8, 9])["mel_out"].clone()
    sw.set_mel_precision("split")
    assert torch.equal(fresh.forward(pb, seed=2)["mel_out"], sw.forward(pb, seed=2)["mel_out"])
    sw.set_mel_precision("fp16")
    offs = pb.frame_offsets
    for i, u in enumerate(utts):
        one = sw.forward(pack_batch([u]).to(DEV), seeds=[7 + i])["mel_out"]
        assert torch.equal(one, f16[int(offs[i]):int(offs[i + 1])]), i
    with pytest.raises(ValueError):
        sw.set_mel_precision("bf16")
    assert sw.mel_precision == "fp16"
    v0 = Vocoder(vocoder_sd(), DEFAULT_VOCODER_CONFIG)
    v1 = Vocoder(vocoder_sd(), DEFAULT_VOCODER_CONFIG, tc_precision="fp16")
    mel = f16
    v1.generate(mel, None, offs, seed=4)
    v1.set_precision("split")
    assert torch.equal(v0.generate(mel, None, offs, seed=4), v1.generate(mel, None, offs, seed=4))
