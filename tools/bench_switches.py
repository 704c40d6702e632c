"""Model-switch timing: the acoustic forward (StyleSinger.forward, T = 100 mel + 2 x 100 F0 steps) of the default
configuration, style off, emo off and all four switches off.

    python tools/bench_switches.py [--reps 5] [--out FILE]

Synthetic weights (synth.acoustic_state_dict of each configuration), Philox noise, on the utt10s (one 1,875-frame
utterance, 1,125-frame reference) and batch64 (bench.make_workload: 64 utterances) lengths.  The four arms run alternated
over --reps repetitions after a warm-up; prints one JSON line per workload with CUDA-event medians and the card's name,
power limit and max SM clock (read in the same call).  Writes nothing except --out.
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
from stylesinger_b200.engine import AcousticModel  # noqa: E402
from stylesinger_b200.hparams import resolve  # noqa: E402

ARMS = {"default": {}, "style_off": {"style": False}, "emo_off": {"emo": False},
        "all_off": {"emo": False, "style": False, "umln": False, "use_txt_cond": False}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_switches needs a CUDA device")
    dev = torch.device("cuda:0")
    info = card()
    models = {}
    for k, ov in ARMS.items():
        hp = resolve(**ov)
        models[k] = AcousticModel(synth.acoustic_state_dict(hp, seed=0), hp, dev)
    lines = []
    for wl in ("utt10s", "batch64"):
        utts, desc = make_workload(wl, 0, 1)
        pbs = {k: m.pack_batch(utts).to(dev) for k, m in models.items()}

        def arm(k):
            return lambda: models[k].forward(pbs[k], seed=3, want=("mel_out", "f0_denorm"))

        arms = {k: arm(k) for k in models}
        for fn in arms.values():  # warm-up of every shape
            fn()
        ms = {k: [] for k in arms}
        for _ in range(args.reps):
            for k, fn in arms.items():  # alternated
                ms[k].append(timed(fn)[0])
        med = {k: round(float(np.median(v)), 3) for k, v in ms.items()}
        line = json.dumps({"what": "acoustic forward per model-switch configuration", "workload": wl, "desc": desc,
                           "frames": pbs["default"].total_frames, "card": info, "reps": args.reps, "ms": med,
                           "ms_all": {k: [round(x, 3) for x in v] for k, v in ms.items()}})
        print(line, flush=True)
        lines.append(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
