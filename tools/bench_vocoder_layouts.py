"""HiFi-GAN layout timing: V1 (DEFAULT_VOCODER_CONFIG), V2 (HIFIGAN_V2) and V3 (HIFIGAN_V3), all with NSF.

    python tools/bench_vocoder_layouts.py [--reps 5] [--out FILE]

Synthetic weights (synth.vocoder_state_dict), Philox noise, on the utt10s (one 1,875-frame utterance) and batch64
(bench.make_workload: 64 utterances, 110,119 frames) lengths.  For each workload every layout runs on tensor cores and
on FFMA, the six arms alternated over --reps repetitions after a warm-up; prints one JSON line per workload with
CUDA-event medians and the card's name, power limit and max SM clock (read in the same call).  Writes nothing except
--out.
"""
import argparse
import json
import os
import sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, "tools"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from bench import make_workload  # noqa: E402
from bench_f0gen import card, timed  # noqa: E402
from stylesinger_b200 import synth  # noqa: E402
from stylesinger_b200.engine import Vocoder, pack_batch  # noqa: E402
from stylesinger_b200.hparams import DEFAULT_VOCODER_CONFIG, HIFIGAN_V2, HIFIGAN_V3  # noqa: E402

LAYOUTS = {"V1": DEFAULT_VOCODER_CONFIG, "V2": HIFIGAN_V2, "V3": HIFIGAN_V3}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_vocoder_layouts needs a CUDA device")
    dev = torch.device("cuda:0")
    info = card()
    vocs = {k: Vocoder(synth.vocoder_state_dict(h, seed=0), h, dev) for k, h in LAYOUTS.items()}
    params = {k: sum(int(np.prod(s)) for n, s in synth.vocoder_param_shapes(h) if not n.endswith("weight_g"))
              for k, h in LAYOUTS.items()}
    lines = []
    for wl in ("utt10s", "batch64"):
        utts, desc = make_workload(wl, 0, 1)
        pb = pack_batch(utts).to(dev)
        fo, Fs = pb.frame_offsets, pb.total_frames
        g = torch.Generator(device=dev).manual_seed(1)
        mel = (torch.randn(Fs, 80, generator=g, device=dev) * 0.5 - 3.0).contiguous()
        f0 = (200.0 + 100.0 * torch.rand(Fs, generator=g, device=dev)).contiguous()

        def arm(name, tc):
            def run():
                vocs[name].set_tensor_cores(tc)
                return vocs[name].generate(mel, f0, fo, seed=2)
            return run

        arms = {f"{k}_{'tc' if tc else 'ffma'}": arm(k, tc) for k in LAYOUTS for tc in (True, False)}
        for fn in arms.values():  # warm-up of every shape
            fn()
        ms = {k: [] for k in arms}
        for _ in range(args.reps):
            for k, fn in arms.items():  # alternated
                ms[k].append(timed(fn)[0])
        med = {k: round(float(np.median(v)), 3) for k, v in ms.items()}
        line = json.dumps({"what": "vocoder layouts", "workload": wl, "desc": desc, "frames": Fs, "card": info,
                           "reps": args.reps, "params_after_weight_norm_removal": params, "ms": med,
                           "ms_all": {k: [round(x, 3) for x in v] for k, v in ms.items()}})
        print(line, flush=True)
        lines.append(line)
    for v in vocs.values():
        v.set_tensor_cores(True)
    if args.out:
        with open(args.out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
