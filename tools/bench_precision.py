"""Split (3-pass fp16 hi/lo) against single-pass fp16 tensor-core GEMMs (hparams['tc_precision']), timed in the same
process, alternated call by call, with CUDA events; medians over the repeats.  Times the mel stage (one 10 s utterance on
the persistent sampler, the bench's batch64 on the per-launch kernels), the vocoder (V1 at batch64 and at one 10 s
utterance) and the whole acoustic forward at batch64, all at T = 100.  Also reports the mel / wav L-inf between the two
modes on the same seed.  Prints one JSON line (with the card name and power limit); writes nothing except --out.

    python tools/bench_precision.py [--reps 5] [--out FILE]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return {"device": torch.cuda.get_device_name(0), "nvidia_smi": q[0] if q else "unavailable"}


def timed(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    r = fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / 1e3, r


def compare(name, set_mode, fn, reps):
    """fn under 'split' and 'fp16', warmed up, then alternated reps times; medians and the output L-inf."""
    outs, ts = {}, {"split": [], "fp16": []}
    for mode in ("split", "fp16"):
        set_mode(mode)
        outs[mode] = fn().clone()  # warm-up (module load, workspace, descriptor cache)
    for _ in range(reps):
        for mode in ("split", "fp16"):
            set_mode(mode)
            t, _ = timed(fn)
            ts[mode].append(t)
    set_mode("split")
    s, f = float(np.median(ts["split"])), float(np.median(ts["fp16"]))
    r = {"split_s": s, "fp16_s": f, "speedup": s / f, "split_all": ts["split"], "fp16_all": ts["fp16"],
         "linf_fp16_vs_split": float((outs["fp16"] - outs["split"]).abs().max())}
    print(f"{name}: split {s:.4f} s, fp16 {f:.4f} s, x{s / f:.2f}; output L-inf {r['linf_fp16_vs_split']:.2e}", flush=True)
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--T", type=int, default=100)
    ap.add_argument("--out", default=None, help="also write the full result, every repetition included, as JSON here")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_precision needs a GPU"
    from stylesinger_b200 import synth
    from stylesinger_b200.engine import AcousticModel, Vocoder, pack_batch
    from stylesinger_b200.hparams import DEFAULT_VOCODER_CONFIG, resolve
    hp = resolve(timesteps=args.T, K_step=args.T, f0_timesteps=args.T)
    m = AcousticModel(synth.acoustic_state_dict(hp, seed=0), hp)
    v = Vocoder(synth.vocoder_state_dict(DEFAULT_VOCODER_CONFIG, seed=0), DEFAULT_VOCODER_CONFIG)
    res = {"card": card(), "T": args.T, "reps": args.reps}
    batches = {
        "batch64": [synth.make_utterance(float(s), utt_idx=i) for i, s in enumerate(synth.batch_seconds(64, seed=1234))],
        "utt10s": [synth.make_utterance(10.0, utt_idx=3)],
    }
    for name, utts in batches.items():
        pb = pack_batch(utts).to("cuda:0")
        offs = pb.frame_offsets
        pre = m.forward(pb, seed=1, want=("diff_cond", "coarse_mel", "f0_denorm"), skip_mel_diffusion=True)
        cond, coarse, f0 = pre["diff_cond"].clone(), pre["coarse_mel"].clone(), pre["f0_denorm"].clone()
        path = "persistent" if name == "utt10s" else "per-launch"
        res[f"mel_{name}"] = dict(path=path, frames=int(offs[-1]), **compare(
            f"mel stage {name} ({path})", m.set_mel_precision, lambda: m.mel_diffusion(cond, coarse, offs, seed=2), args.reps))
        mel = m.mel_diffusion(cond, coarse, offs, seed=2).clone()
        res[f"vocoder_v1_{name}"] = compare(f"vocoder V1 {name}", v.set_precision,
                                            lambda: v.generate(mel, f0, offs, seed=3), args.reps)
        if name == "batch64":
            res["forward_batch64"] = compare("acoustic forward batch64", m.set_mel_precision,
                                             lambda: m.forward(pb, seed=1)["mel_out"], args.reps)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)
    print(json.dumps({k: (v if not isinstance(v, dict) else {a: b for a, b in v.items() if not a.endswith("_all")})
                      for k, v in res.items()}))


if __name__ == "__main__":
    main()
