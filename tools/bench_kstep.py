"""Mel-stage and acoustic-model timing of shallow diffusion: the DiffSinger mel sampler at K_step in {100, 75, 50, 25} of
the T = 100 schedule (ssb_model_set_mel_k_step), plus PLMS (pndm_speedup 10) at K_step 50, on the same utterances, every
arm alternated with the others in one process.

    python tools/bench_kstep.py [--workloads utt10s,batch64] [--reps 3] [--out FILE]

Per workload it prints one JSON line: the mel-stage time (ssb_mel_diffusion_sample / ssb_mel_diffusion_sample_plms, CUDA
events, median over --reps alternated runs after a warm-up of every arm), mel frames/s, denoiser evaluations, the acoustic
forward without the vocoder (both 100-step F0 samplers included; DDPM arms only), every arm relative to K_step 100, and
the card's name, power limit and maximum SM clock, read in the same run.  utt10s takes the persistent single-launch
sampler, batch64 the per-launch tensor-core path (the library defaults).  Synthetic weights (synth.py): the timings
depend on shapes only.  Writes nothing except --out.
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
from stylesinger_b200.engine import AcousticModel, pack_batch  # noqa: E402
from stylesinger_b200.hparams import resolve  # noqa: E402

T = 100
KS = (100, 75, 50, 25)
PLMS_K, PLMS_INTERVAL = 50, 10


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
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_kstep needs a CUDA device")
    dev = torch.device("cuda:0")
    hp = resolve(timesteps=T, K_step=T, f0_timesteps=T)
    m = AcousticModel(synth.acoustic_state_dict(hp, seed=0), hp, dev)
    info = card()
    lines = []
    for wl in args.workloads.split(","):
        utts, desc = make_workload(wl, 0, 1)
        pb = pack_batch(utts, pin=True).to(dev)
        fo, Fs = pb.frame_offsets, pb.total_frames
        o = m.forward(pb, seed=1, skip_mel_diffusion=True, want=("coarse_mel", "diff_cond"))
        cond, coarse = o["diff_cond"], o["coarse_mel"]

        def at(K, fn):
            def run():
                m.set_mel_k_step(K)
                return fn()
            return run

        mel_arms = {f"K{K}": at(K, lambda: m.mel_diffusion(cond, coarse, fo, seed=2)) for K in KS}
        mel_arms[f"K{PLMS_K}_plms{PLMS_INTERVAL}"] = at(PLMS_K, lambda: m.mel_diffusion_plms(cond, coarse, fo, PLMS_INTERVAL,
                                                                                               seed=2))
        fwd_arms = {f"K{K}": at(K, lambda: m.forward(pb, seed=3)["mel_out"]) for K in KS}
        evals = {f"K{K}": K for K in KS}
        evals[f"K{PLMS_K}_plms{PLMS_INTERVAL}"] = len(range(0, PLMS_K, PLMS_INTERVAL)) + 1
        for fn in list(mel_arms.values()) + list(fwd_arms.values()):  # warm-up of every shape
            fn()
        mel_ms = {k: [] for k in mel_arms}
        fwd_ms = {k: [] for k in fwd_arms}
        finite = {}
        for _ in range(args.reps):
            for k, fn in mel_arms.items():  # alternated
                ms, mel = timed(fn)
                mel_ms[k].append(ms)
                finite[k] = bool(torch.isfinite(mel).all())
            for k, fn in fwd_arms.items():
                fwd_ms[k].append(timed(fn)[0])
        m.set_mel_k_step(0)
        med = {k: float(np.median(v)) for k, v in mel_ms.items()}
        fmed = {k: float(np.median(v)) for k, v in fwd_ms.items()}
        res = {"workload": wl, "desc": desc, "frames": Fs, "T": T, "card": info,
               "mel_stage_ms": {k: round(v, 2) for k, v in med.items()},
               "mel_stage_ms_all": {k: [round(x, 2) for x in v] for k, v in mel_ms.items()},
               "mel_stage_vs_K100": {k: round(v / med["K100"], 3) for k, v in med.items()},
               "mel_frames_per_s": {k: round(Fs / (v / 1e3)) for k, v in med.items()},
               "denoiser_evals": evals,
               "acoustic_forward_ms": {k: round(v, 2) for k, v in fmed.items()},
               "acoustic_forward_ms_all": {k: [round(x, 2) for x in v] for k, v in fwd_ms.items()},
               "acoustic_forward_vs_K100": {k: round(v / fmed["K100"], 3) for k, v in fmed.items()},
               "outputs_finite": finite}
        line = json.dumps(res)
        print(line, flush=True)
        lines.append(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
