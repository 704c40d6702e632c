"""F0-generator timing: the two 100-step F0 diffusion samplers (f0_gen 'gmdiff') against the two PitchPredictors
(f0_gen 'conv') on the same utterances, the acoustic forward without the vocoder for {diffsinger, prodiff, fft} x
{gmdiff, conv}, and the HiFi-GAN vocoder on the fft + conv model's mel, all arms alternated in one process.

    python tools/bench_f0gen.py [--workloads utt10s,batch64] [--reps 3] [--out FILE]

Per workload it prints one JSON line with CUDA-event medians over --reps alternated repetitions after a warm-up, and the
card's name, power limit and max SM clock.
- pitch stage: ssb_f0_diffusion_sample x 2 (agnostic, specific; one after the other) against ssb_pitch_predictor x 2, both
  on the same two conditions (decoder_inp of the workload stands in for both; the timings depend on shapes only), the
  samplers with the widest clip band.  Inside the acoustic forward the two samplers overlap on two streams, so the
  forward's own F0 cost is somewhat lower than the pitch-stage number.
- acoustic forward: ssb_acoustic_forward without the vocoder, Philox noise, DiffSinger T = 100 / ProDiff T = 8, F0 T = 100;
  the FFT decoder (decoder 'fft') has no mel sampler.
- vocoder: Vocoder.generate (HiFi-GAN V1 layout with NSF, Philox) on the mel and f0 of the fft + conv forward, so that
  fft + conv's whole ph -> wav cost is the forward plus this arm.
Synthetic weights (synth.py).  Writes nothing except --out.
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


def hparams(decoder, f0_gen):
    kw = dict(f0_timesteps=T_F0, f0_gen=f0_gen)
    if decoder == "prodiff":
        return resolve(timesteps=T_PD, decoder="prodiff", schedule_type="vpsde", timescale=1, **kw)
    if decoder == "fft":
        return resolve(decoder="fft", extended_models=True, **kw)
    return resolve(timesteps=T_DS, K_step=T_DS, **kw)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="utt10s,batch64")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_f0gen needs a CUDA device")
    dev = torch.device("cuda:0")
    models = {}
    decoders = ("diffsinger", "prodiff", "fft")
    for dec in decoders:
        for f0g in ("gmdiff", "conv"):
            hp = hparams(dec, f0g)
            models[f"{dec}+{f0g}"] = AcousticModel(synth.acoustic_state_dict(hp, seed=0), hp, dev)
    gm, cv = models["diffsinger+gmdiff"], models["diffsinger+conv"]
    voc = Vocoder(synth.vocoder_state_dict(DEFAULT_VOCODER_CONFIG, seed=0), DEFAULT_VOCODER_CONFIG, dev)
    info = card()
    lines = []
    for wl in args.workloads.split(","):
        utts, desc = make_workload(wl, 0, 1)
        pb = pack_batch(utts, pin=True).to(dev)
        fo, Fs = pb.frame_offsets, pb.total_frames
        cond = gm.forward(pb, seed=1, skip_mel_diffusion=True, want=("decoder_inp",))["decoder_inp"]
        lo = torch.full((Fs,), -1.0, device=dev)
        hi = torch.full((Fs,), 1.0, device=dev)
        pitch = {"gmdiff_2x100_steps": lambda: [gm.f0_diffusion(w, cond, lo, hi, fo, seed=2) for w in (0, 1)],
                 "conv_2_predictors": lambda: [cv.pitch_predictor(w, cond, fo) for w in (0, 1)]}
        fwd = {k: (lambda m=m: m.forward(pb, seed=3)["mel_out"]) for k, m in models.items()}
        o = models["fft+conv"].forward(pb, seed=3, want=("mel_out", "f0_denorm"))
        mel, f0 = o["mel_out"], o["f0_denorm"]
        vocoder = {"vocoder_on_fft+conv_mel": lambda: voc.generate(mel, f0, fo, seed=4)}
        arms = dict(pitch, **fwd, **vocoder)
        ms = {k: [] for k in arms}
        for k in arms:  # warm-up of every shape
            arms[k]()
        finite = {}
        for _ in range(args.reps):
            for k in arms:  # alternated
                t, r = timed(arms[k])
                ms[k].append(t)
                if k in fwd or k in vocoder:
                    finite[k] = bool(torch.isfinite(r).all())
        med = {k: float(np.median(v)) for k, v in ms.items()}
        res = {"workload": wl, "desc": desc, "frames": Fs, "card": info, "reps": args.reps,
               "pitch_stage_ms": {k: round(med[k], 3) for k in pitch},
               "pitch_stage_speedup": round(med["gmdiff_2x100_steps"] / med["conv_2_predictors"], 1),
               "acoustic_forward_ms": {k: round(med[k], 2) for k in fwd},
               "acoustic_forward_speedup_conv_vs_gmdiff": {
                   d: round(med[f"{d}+gmdiff"] / med[f"{d}+conv"], 2) for d in decoders},
               "vocoder_ms": {k: round(med[k], 2) for k in vocoder},
               "ms_all": {k: [round(x, 3) for x in v] for k, v in ms.items()},
               "outputs_finite": finite}
        line = json.dumps(res)
        print(line, flush=True)
        lines.append(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
