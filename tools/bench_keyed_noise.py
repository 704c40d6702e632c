"""Timing of the per-utterance Philox seeds against the per-call seed: the acoustic forward plus the vocoder, legacy
(`seed`) and keyed (`seeds`, one per utterance) alternated in one process, at T = 100.

    python tools/bench_keyed_noise.py [--workloads utt10s,batch64] [--reps 5] [--out FILE]

Both modes draw the same number of values from the same streams; only the key and counter of each draw differ, read
from a per-utterance table.  Per workload it prints one JSON line: the median (CUDA events, after a warm-up of both arms)
of the acoustic forward (ssb_acoustic_forward[_keyed]), of the vocoder (ssb_hifigan_generate[_keyed]) and of their sum,
every run, keyed / legacy, and the card's name, power limit and maximum SM clock, read in the same run.  Synthetic
weights (synth.py): the timings depend on shapes only.  Writes nothing except --out.
"""
import argparse
import json
import os
import subprocess
import sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from bench import make_workload  # noqa: E402
from stylesinger_b200 import synth  # noqa: E402
from stylesinger_b200.engine import AcousticModel, Vocoder, pack_batch  # noqa: E402
from stylesinger_b200.hparams import DEFAULT_VOCODER_CONFIG, resolve  # noqa: E402

T = 100


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = "nvidia-smi unavailable"
    return {"name": name, "power_limit,clocks.max.sm": q}


def timed(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    r = fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b), r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="utt10s,batch64")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_keyed_noise needs a CUDA device")
    dev = torch.device("cuda:0")
    hp = resolve(timesteps=T, K_step=T, f0_timesteps=T)
    m = AcousticModel(synth.acoustic_state_dict(hp, seed=0), hp, dev)
    v = Vocoder(synth.vocoder_state_dict(DEFAULT_VOCODER_CONFIG, seed=0), DEFAULT_VOCODER_CONFIG, dev)
    info = card()
    lines = []
    for wl in args.workloads.split(","):
        utts, desc = make_workload(wl, 0, 1)
        pb = pack_batch(utts, pin=True).to(dev)
        fo, B = pb.frame_offsets, pb.B
        seeds = [1000 + b for b in range(B)]
        kw = {"legacy": {"seed": 7}, "keyed": {"seeds": seeds}}
        mel = {}

        def acoustic(mode):
            def run():
                o = m.forward(pb, **kw[mode])
                mel[mode] = o
                return o["mel_out"]
            return run

        def vocoder(mode):
            def run():
                o = mel[mode]
                return v.generate(o["mel_out"].clamp(-6, 1.5), o["f0_denorm"], fo, **kw[mode])
            return run

        for mode in kw:  # warm-up of every shape
            acoustic(mode)()
            vocoder(mode)()
        ms = {f"{stage}_{mode}": [] for stage in ("acoustic", "vocoder") for mode in kw}
        finite = {}
        for _ in range(args.reps):
            for mode in kw:  # alternated
                t, out = timed(acoustic(mode))
                ms[f"acoustic_{mode}"].append(t)
                t, wav = timed(vocoder(mode))
                ms[f"vocoder_{mode}"].append(t)
                finite[mode] = bool(torch.isfinite(out).all()) and bool(torch.isfinite(wav).all())
        med = {k: float(np.median(x)) for k, x in ms.items()}
        for mode in kw:
            med[f"total_{mode}"] = float(np.median([a + b for a, b in zip(ms[f"acoustic_{mode}"], ms[f"vocoder_{mode}"])]))
        res = {"workload": wl, "desc": desc, "frames": int(fo[-1]), "T": T, "card": info,
               "median_ms": {k: round(x, 2) for k, x in med.items()},
               "all_ms": {k: [round(x, 2) for x in xs] for k, xs in ms.items()},
               "keyed_vs_legacy": {s: round(med[f"{s}_keyed"] / med[f"{s}_legacy"], 4)
                                   for s in ("acoustic", "vocoder", "total")},
               "outputs_finite": finite}
        line = json.dumps(res)
        print(line, flush=True)
        lines.append(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
