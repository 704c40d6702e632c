"""Mel-stage and acoustic-model timing: ProDiff teacher (decoder 'prodiff', T = 8, vpsde) against DiffSinger
(decoder 'diffsinger', T = 100 DDPM steps) on the same utterances, the two alternated in one process.

    python tools/bench_prodiff.py [--workloads utt10s,batch64] [--reps 3] [--out FILE]

Per workload it prints one JSON line: the mel-stage time (ssb_mel_prodiff_sample vs ssb_mel_diffusion_sample, CUDA events,
median over --reps alternated runs after a warm-up), mel frames/s, denoiser evaluations, the acoustic forward without the
vocoder (both 100-step F0 samplers included), and the card's name and power limit.  Synthetic weights (synth.py): the
timings depend on shapes only.  Writes nothing except --out.
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

T_DS, T_PD, T_F0 = 100, 8, 100


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
        raise SystemExit("bench_prodiff needs a CUDA device")
    dev = torch.device("cuda:0")
    hp_ds = resolve(timesteps=T_DS, K_step=T_DS, f0_timesteps=T_F0)
    hp_pd = resolve(timesteps=T_PD, f0_timesteps=T_F0, decoder="prodiff", schedule_type="vpsde", timescale=1)
    ds = AcousticModel(synth.acoustic_state_dict(hp_ds, seed=0), hp_ds, dev)
    pd = AcousticModel(synth.acoustic_state_dict(hp_pd, seed=0), hp_pd, dev)
    info = card()
    lines = []
    for wl in args.workloads.split(","):
        utts, desc = make_workload(wl, 0, 1)
        pb = pack_batch(utts, pin=True).to(dev)
        fo, Fs = pb.frame_offsets, pb.total_frames
        o_ds = ds.forward(pb, seed=1, skip_mel_diffusion=True, want=("coarse_mel", "diff_cond"))
        o_pd = pd.forward(pb, seed=1, skip_mel_diffusion=True, want=("decoder_inp",))
        cond_ds, coarse, cond_pd = o_ds["diff_cond"], o_ds["coarse_mel"], o_pd["decoder_inp"]
        arms = {
            "diffsinger_T100": lambda: ds.mel_diffusion(cond_ds, coarse, fo, seed=2),
            "prodiff_T8": lambda: pd.mel_prodiff(cond_pd, fo, seed=2),
        }
        e2e = {"diffsinger_T100": lambda: ds.forward(pb, seed=3)["mel_out"],
               "prodiff_T8": lambda: pd.forward(pb, seed=3)["mel_out"]}
        mel_ms = {k: [] for k in arms}
        fwd_ms = {k: [] for k in arms}
        for k in arms:  # warm-up of every shape
            arms[k]()
            e2e[k]()
        finite = {}
        for _ in range(args.reps):
            for k in arms:  # alternated
                ms, mel = timed(arms[k])
                mel_ms[k].append(ms)
                finite[k] = bool(torch.isfinite(mel).all())
            for k in e2e:
                fwd_ms[k].append(timed(e2e[k])[0])
        med = {k: float(np.median(v)) for k, v in mel_ms.items()}
        fmed = {k: float(np.median(v)) for k, v in fwd_ms.items()}
        res = {"workload": wl, "desc": desc, "frames": Fs, "card": info,
               "mel_stage_ms": {k: round(v, 2) for k, v in med.items()},
               "mel_stage_ms_all": {k: [round(x, 2) for x in v] for k, v in mel_ms.items()},
               "mel_frames_per_s": {k: round(Fs / (v / 1e3)) for k, v in med.items()},
               "denoiser_evals": {"diffsinger_T100": T_DS, "prodiff_T8": T_PD},
               "mel_stage_speedup": round(med["diffsinger_T100"] / med["prodiff_T8"], 2),
               "acoustic_forward_ms": {k: round(v, 2) for k, v in fmed.items()},
               "acoustic_forward_speedup": round(fmed["diffsinger_T100"] / fmed["prodiff_T8"], 3),
               "outputs_finite": finite}
        line = json.dumps(res)
        print(line, flush=True)
        lines.append(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
