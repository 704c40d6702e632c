"""The single-pass fp16 tensor-core mode without a GPU: hparams['tc_precision'] validation, the defaults (split
everywhere), the C ABI's refusals, and the float64 emulation oracle of tests/fp16_emulation.py for one op, the mel
sampler and the vocoder."""
import ctypes

import numpy as np
import pytest
import torch

from stylesinger_b200.hparams import DEFAULT_HPARAMS, TC_PRECISIONS, resolve
from tests import conv_gemm_ref as R
from tests import fp16_emulation as E


def test_tc_precision_validated():
    assert resolve()["tc_precision"] == "split"
    assert resolve(tc_precision="fp16")["tc_precision"] == "fp16"
    for bad in ("bf16", "FP16", None, 1, "", "tf32"):
        with pytest.raises(ValueError, match="tc_precision"):
            resolve(tc_precision=bad)


def test_defaults_unchanged():
    """split is the default of the hparams, of the C constants and of every Python entry point."""
    import inspect

    from stylesinger_b200 import engine
    assert DEFAULT_HPARAMS["tc_precision"] == "split" and TC_PRECISIONS == {"split": 0, "fp16": 1}
    assert inspect.signature(engine.Vocoder.__init__).parameters["tc_precision"].default == "split"
    assert inspect.signature(engine.op_gemm).parameters["single_pass"].default is False
    assert engine._lib.OpGemmArgs().single_pass == 0
    assert engine._lib.OpGemmArgs._fields_[-1] == ("single_pass", ctypes.c_int32)  # appended: earlier fields keep offsets
    hdr = open(__file__.replace("tests/test_fp16_mode_cpu.py", "include/stylesinger_b200.h")).read()
    assert "#define SSB_TC_SPLIT 0" in hdr and "#define SSB_TC_FP16 1" in hdr


def test_abi_refuses_without_a_gpu():
    """Unknown modes, null handles and single_pass on the FFMA path fail before any CUDA call, with a message."""
    from stylesinger_b200 import _lib
    lib = _lib.lib
    assert lib.ssb_model_set_mel_precision(None, 0) != 0
    assert lib.ssb_vocoder_set_precision(None, 1) != 0
    offs = np.array([0, 4], np.int32)
    w = np.zeros((64, 64, 1), np.float32)
    for path, sp in ((0, 1), (1, 2), (1, -1)):
        a = _lib.OpGemmArgs(path=path, single_pass=sp, frame_offsets=offs.ctypes.data, B=1, rows=4 + 32 + 256, Cin=64,
                            N=64, k=1, dilation=1, w_host=w.ctypes.data)
        assert lib.ssb_op_gemm(ctypes.byref(a), None) != 0
        assert b"single_pass" in lib.ssb_last_error(), lib.ssb_last_error()


def test_op_emulation_rounds_both_operands():
    """fp16_convs on one conv equals the float64 GEMM of tests/conv_gemm_ref.py on fp16-rounded operands, and differs from
    the unrounded one by about the fp16 rounding."""
    g = torch.Generator().manual_seed(3)
    lens = [5, 40, 129]
    rs, rows = R.layout(lens)
    valid = R.valid_rows(lens, rs, rows)
    x = torch.zeros(rows, 64, dtype=torch.float64)
    x[valid] = torch.randn(int(valid.sum()), 64, generator=g, dtype=torch.float64)
    w = torch.randn(128, 64, 3, generator=g, dtype=torch.float64) / 14
    want = R.accumulator(E.r16(x), E.r16w(w), 2, lens, rs)
    with E.fp16_convs() as n:
        got = torch.nn.functional.conv1d(x.t()[None], w, None, padding=2, dilation=2)[0].t()
    assert n["rounded"] == 1
    for b, (a, L) in enumerate(zip(rs, lens)):  # one utterance alone: conv1d's zero padding is the guard band
        with E.fp16_convs():
            one = torch.nn.functional.conv1d(x[a:a + L].t()[None], w, None, padding=2, dilation=2)[0].t()
        assert torch.allclose(one, want[a:a + L], rtol=0, atol=1e-12)
    full = R.accumulator(x, w, 2, lens, rs)
    d = (want - full)[valid].abs().max().item()
    assert 1e-5 < d < 1e-2, d
    assert got.shape[1] == 128


def test_vocoder_selection():
    """The vocoder's tensor-core convs: ups with 64-multiple channels, square ResBlock convs; not conv_pre / conv_post /
    the noise convs."""
    s = E.vocoder_tc_conv
    assert s("conv_transpose1d", None, torch.zeros(512, 256, 16), 8)
    assert not s("conv_transpose1d", None, torch.zeros(32, 16, 4), 2)
    assert s("conv1d", None, torch.zeros(32, 32, 3), 1) and s("conv1d", None, torch.zeros(256, 256, 11), 1)
    assert not s("conv1d", None, torch.zeros(512, 80, 7), 1)   # conv_pre
    assert not s("conv1d", None, torch.zeros(1, 32, 7), 1)     # conv_post
    assert not s("conv1d", None, torch.zeros(64, 1, 16), 8)    # noise conv


def test_mel_sampler_emulation_is_near_the_fp32_chain():
    """The DiffSinger mel chain (T = 4) under the emulation: every DiffNet conv rounded, a result that differs from the
    float64 chain by the size fp16 operands give (SURVEY.md measured 2.6e-3 at T = 4 in fp32), and is reproducible."""
    from stylesinger_b200 import synth
    from tests import denoiser_oracle as DO
    from tests.common import hp_for
    hp = dict(hp_for(4), K_step=4)
    g = torch.Generator().manual_seed(11)
    F_ = 40
    cond = torch.randn(F_, 256, generator=g)
    coarse = (-3 + 1.5 * torch.randn(F_, 80, generator=g)).clamp(-6, 1)
    noise = torch.randn(5, F_, 80, generator=g)
    ref = DO.mel_chain64(cond, coarse, hp, 4, noise)["mel"]
    with E.fp16_convs() as n:
        emu = DO.mel_chain64(cond, coarse, hp, 4, noise)["mel"]
    L = hp["residual_layers"]
    assert n["rounded"] == 4 * (3 + 3 * L) and n["kept"] == 0  # per step: in, L x (cond, dilated, out), skip, out
    d = (emu - ref).abs().max().item()
    print(f"mel T=4 emulation vs float64: L-inf {d:.2e}")
    assert 1e-5 < d < 5e-2
    with E.fp16_convs():
        again = DO.mel_chain64(cond, coarse, hp, 4, noise)["mel"]
    assert torch.equal(emu, again)
    del synth


def test_vocoder_emulation_is_near_the_fp32_generator():
    """HiFi-GAN V3 (the smallest layout) under the emulation: the ups and ResBlock convs rounded, conv_pre / conv_post /
    noise convs not; the waveform stays within the size of the fp16 rounding of the float64 generator's."""
    from oracle import stylesinger_oracle as O
    from tests.common import VOCODER_LAYOUTS, vocoder_sd
    g = torch.Generator().manual_seed(5)
    F_ = 12
    mel = (-3.0 + torch.randn(F_, 80, generator=g)).clamp(-6, 1.5).numpy()
    f0 = (150 + 350 * torch.rand(F_, generator=g)).numpy()
    sd, h = vocoder_sd("v3"), VOCODER_LAYOUTS["v3"]
    ref = O.spec2wav(mel, f0, sd, h, O.NoiseSource(3), torch.float64)
    with E.fp16_convs(E.vocoder_tc_conv) as n:
        emu = O.spec2wav(mel, f0, sd, h, O.NoiseSource(3), torch.float64)
    assert n["rounded"] == 3 + 3 * 3 * 2 and n["kept"] == 2 + 3  # ups + ResBlock2 convs; conv_pre, conv_post, noise convs
    d = float(np.abs(emu - ref).max())
    print(f"vocoder v3 emulation vs float64: L-inf {d:.2e}")
    assert 1e-6 < d < 0.1
