"""Checks shared by the GPU files that compare the diffusion denoisers and samplers with a float64 reference
(tests/test_gpu_denoisers.py, tests/test_gpu_samplers_f64.py): which tensor-core GEMM variants a call must launch, and
errors reported separately for the rows at each utterance end and for the interior."""
import numpy as np
import torch

from tests.common import hp_for

EDGE_ROWS = 8


def frame_offsets(lens):
    return np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)


def ntiles(lens):
    return sum((int(n) + 127) // 128 for n in lens)


def rel(a, b):
    a = a.detach().cpu().double() if isinstance(a, torch.Tensor) else torch.as_tensor(np.asarray(a, np.float64))
    b = b.detach().cpu().double() if isinstance(b, torch.Tensor) else torch.as_tensor(np.asarray(b, np.float64))
    return ((a - b).abs() / b.abs().clamp(min=1.0)).reshape(a.shape[0], -1)


def split(x, offs):
    x = x.detach().cpu()
    return [x[int(offs[i]):int(offs[i + 1])] for i in range(len(offs) - 1)]


# ---------------------------------------------------------------------------------------------------------------------
# which tensor-core GEMM variants a call must launch: conv_gemm_tc's dispatch.  CTA pairs when ceil(ntiles / 2) * N / (2 hb)
# >= #SMs, hb = 64 if N % 128 == 0 else 32, on the tap-reuse kernel for 3-tap GATE / GENERIC convs of dilation <= 8;
# else single CTAs with 64-wide N tiles
def variant(nt, N, mode, taps, dil=1):
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    hb = 64 if N % 128 == 0 else 32
    if ((nt + 1) // 2) * (N // (2 * hb)) >= sms:
        return f"tc2{'r' if taps == 3 and dil <= 8 and mode != 'RES_SKIP' else ''}<{hb},{mode}>"
    return f"tc<64,{mode}>"


def count(gemms, nt):
    out = {}
    for N, mode, taps in gemms:
        k = variant(nt, N, mode, taps)
        out[k] = out.get(k, 0) + 1
    return out


def net_dims(which):
    """(channels, layers, padded output N) of the mel DiffNet (0) or an F0 DDiffNet (1, 2)."""
    hp = hp_for(100)
    if which == 0:
        return hp["residual_channels"], hp["residual_layers"], 256
    return hp["f0_residual_channels"], hp["f0_residual_layers"], 128


def cond_gemm(which):
    """The hoisted conditioner projection of all layers, once per call."""
    C, L, _ = net_dims(which)
    return [(L * 2 * C, "GENERIC", 1)]


def step_gemms(which):
    """One evaluation after the conditioner: (mel) the input projection, L x (gate, residual + skip), skip_projection,
    output_projection (N padded to 256 / 128)."""
    C, L, n_out = net_dims(which)
    g = [(C, "GENERIC", 1)] if which == 0 else []
    return g + [(2 * C, "GATE", 3), (2 * C, "RES_SKIP", 1)] * L + [(256, "GENERIC", 1), (n_out, "GENERIC", 1)]


def launched(fn):
    """fn() and the tensor-core GEMM variants and the number of kernels it launched."""
    from stylesinger_b200._lib import lib, variant_launches
    torch.cuda.synchronize()
    before, l0 = variant_launches(), lib.ssb_launch_count()
    r = fn()
    torch.cuda.synchronize()
    after, l1 = variant_launches(), lib.ssb_launch_count()
    return r, {k: after[k] - before.get(k, 0) for k in after if after[k] > before.get(k, 0)}, l1 - l0


def check_variants(tag, got, want):
    print(f"{tag}: tensor-core GEMM variants launched {got}")
    assert got == want, (tag, got, want)


# ---------------------------------------------------------------------------------------------------------------------
# edge / interior errors
class Err:
    """Largest error on the interior rows and on the EDGE_ROWS rows at each utterance end, with where it is."""

    def __init__(self):
        self.v = {"interior": (0.0, None), "edge": (0.0, None)}
        self.interior_rows = 0

    def add(self, i, a, b):
        e = rel(a, b)
        n = e.shape[0]
        edge = torch.zeros(n, dtype=torch.bool)
        edge[:EDGE_ROWS] = True
        edge[-EDGE_ROWS:] = True
        self.interior_rows += int((~edge).sum())
        for k, rows in (("edge", edge), ("interior", ~edge)):
            if rows.any():
                sub = torch.where(rows[:, None], e, torch.zeros_like(e))
                j = int(sub.argmax())
                v = float(sub.reshape(-1)[j])
                if v > self.v[k][0]:
                    self.v[k] = (v, (i, j // e.shape[1], j % e.shape[1]))

    def max(self):
        return max(self.v["interior"][0], self.v["edge"][0])

    def report(self, tag, bar):
        (vi, wi), (ve, we) = self.v["interior"], self.v["edge"]
        print(f"{tag}: interior {vi:.3e} at (utterance, row, column) {wi}, edge {ve:.3e} at {we} (bar {bar:.1e})")
        assert self.max() <= bar, (tag, self.v, bar)
        if self.interior_rows:  # utterances of at most 2 x EDGE_ROWS rows have no interior to compare with
            assert ve <= 4 * vi, (tag, "edge rows err more than 4x the interior", self.v)
