"""Float64 emulation of the single-pass fp16 tensor-core mode (SSB_TC_FP16, hparams['tc_precision'] = 'fp16').

In that mode every tensor-core contraction multiplies operands rounded once to fp16 and sums the products in fp32.  The
emulation runs the existing float64 oracles (tests/denoiser_oracle.py, tests/sampler_oracle.py, the float64 mode of
oracle/stylesinger_oracle.py's hifigan_generator, tests/conv_gemm_ref.py) with the activation and the weight of each
such contraction rounded to fp16 and everything else, the sums included, in float64.  fp16_convs() patches
torch.nn.functional's conv1d / conv_transpose1d for the duration of a block; `select(kind, x, w, stride)` says which
calls are tensor-core GEMMs on the CUDA path.  A weight is rounded as the tensor-core packer rounds it, fp16(w 2^s) 2^-s
with one power of two s per tensor (tests/conv_gemm_ref.py plane_exponent): that is fp16(w) for every weight that is a
normal fp16 number.  Biases are not rounded: the kernels add them in fp32 in the epilogue."""
import contextlib

import torch
import torch.nn.functional as F

from tests.conv_gemm_ref import plane_exponent


def r16(t):
    """t rounded to fp16 (round to nearest even), returned in t's dtype."""
    return t.half().to(t.dtype)


def r16w(w):
    """A weight tensor rounded as the tensor-core packer rounds it: fp16(w 2^s) 2^-s, s = plane_exponent(w)."""
    s = plane_exponent(w)
    return torch.ldexp(torch.ldexp(w, torch.tensor(float(s))).half().to(w.dtype), torch.tensor(float(-s)))


def every_conv(kind, x, w, stride):
    """The mel DiffNet: every conv of the net is a tensor-core GEMM (its step MLP is an F.linear, not patched)."""
    return True


def vocoder_tc_conv(kind, x, w, stride):
    """The HiFi-GAN generator's tensor-core GEMMs (csrc/stages.cu run_vocoder, csrc/pack.cu build_vocoder): the ups
    (transposed) convs whose input channels and u * output channels are multiples of 64, and every ResBlock conv (square,
    C >= 8: C % 64 == 0, or the time-grouped 32-, 16- and 8-channel packing).  conv_pre (80 input channels), conv_post
    (one output channel) and the NSF noise convs (one input channel) run on the FFMA kernel."""
    if kind == "conv_transpose1d":
        cin, cout = w.shape[0], w.shape[1]
        return cin % 64 == 0 and (stride * cout) % 64 == 0
    return w.shape[0] == w.shape[1] and w.shape[1] >= 8


@contextlib.contextmanager
def fp16_convs(select=every_conv):
    """Within the block, conv1d / conv_transpose1d calls that `select` picks see fp16-rounded input and weight."""
    conv1d, convt = F.conv1d, F.conv_transpose1d
    n = {"rounded": 0, "kept": 0}

    def c1(x, w, b=None, stride=1, *a, **k):
        if select("conv1d", x, w, stride):
            n["rounded"] += 1
            return conv1d(r16(x), r16w(w), b, stride, *a, **k)
        n["kept"] += 1
        return conv1d(x, w, b, stride, *a, **k)

    def ct(x, w, b=None, stride=1, *a, **k):
        if select("conv_transpose1d", x, w, stride):
            n["rounded"] += 1
            return convt(r16(x), r16w(w), b, stride, *a, **k)
        n["kept"] += 1
        return convt(x, w, b, stride, *a, **k)

    F.conv1d, F.conv_transpose1d = c1, ct
    try:
        yield n
    finally:
        F.conv1d, F.conv_transpose1d = conv1d, convt
