"""Timing probe for the tensor-core conv GEMM kernels: one DiffNet-layer-shaped GEMM (K = 3 x 256, N = 512) on ~110k rows,
single-CTA vs CTA-pair kernel, with parts of the kernel disabled (SSB_TC_DEBUG bits) to see which of TMA / MMA /
epilogue bounds the tile loop.  Run under `ncu --metrics gpu__time_duration.sum -k regex:conv_gemm_wg` for per-kernel
times; the CUDA-event times printed here include the plane split / unpack kernels of the op wrapper."""
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from stylesinger_b200.engine import op_conv1d_tc  # noqa: E402


def main():
    cin, n, k, dil = (int(a) for a in (sys.argv[1:5] if len(sys.argv) >= 5 else (256, 512, 3, 2)))
    g = torch.Generator().manual_seed(0)
    lens = [int(v) for v in torch.randint(400, 2800, (64,), generator=g)]
    offs = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
    x = torch.randn(int(offs[-1]), cin, generator=g).cuda()
    w = torch.randn(n, cin, k, generator=g) / (cin * k) ** 0.5
    b = torch.randn(n, generator=g)
    res = {"rows": int(offs[-1]), "shape": [cin, n, k, dil]}
    for pair in (1, 0):
        if pair:
            os.environ.pop("SSB_TC_NO_PAIR", None)
        else:
            os.environ["SSB_TC_NO_PAIR"] = "1"
        for dbg in (0, 1, 2, 4, 6, 7):
            os.environ["SSB_TC_DEBUG"] = str(dbg)
            for _ in range(2):
                op_conv1d_tc(x, offs, w, b, dilation=dil)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            e0.record()
            for _ in range(3):
                op_conv1d_tc(x, offs, w, b, dilation=dil)
            e1.record()
            torch.cuda.synchronize()
            res[f"pair{pair}.dbg{dbg}"] = round(e0.elapsed_time(e1) / 3, 3)
    os.environ.pop("SSB_TC_DEBUG", None)
    os.environ.pop("SSB_TC_NO_PAIR", None)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
