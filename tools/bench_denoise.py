"""Vocoder output denoiser timing (hparams['vocoder_denoise_c'] > 0, tasks/tts/vocoder_infer/hifigan_nsf.py:14-22,73-74).

    python tools/bench_denoise.py [--reps 5] [--out FILE]

Prints one JSON line per measurement with CUDA-event medians over --reps alternated repetitions after a warm-up, and the
card's name, power limit and max SM clock:
- vocoder stage at utt10s and batch64 (bench.make_workload; synthetic weights, Philox noise): the HiFi-GAN generator alone
  against the generator followed by the denoiser (v = 0.1), and the denoiser's share of the second;
- the denoiser alone, fp32 FFMA GEMMs against tensor-core GEMMs (both forced), on the batch64 waveform lengths (above the
  8-row-tile rule that selects tensor cores) and on one 3 s utterance (below it: the automatic path takes FFMA there).
Writes nothing except --out.
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
from stylesinger_b200.engine import Vocoder, WavDenoiser, pack_batch  # noqa: E402
from stylesinger_b200.hparams import DEFAULT_VOCODER_CONFIG  # noqa: E402

V = 0.1
HOP = 256


def measure(arms, reps):
    for fn in arms.values():  # warm-up of every shape
        fn()
    ms = {k: [] for k in arms}
    for _ in range(reps):
        for k, fn in arms.items():  # alternated
            ms[k].append(timed(fn)[0])
    return {k: float(np.median(v)) for k, v in ms.items()}, ms


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_denoise needs a CUDA device")
    dev = torch.device("cuda:0")
    info = card()
    voc = Vocoder(synth.vocoder_state_dict(DEFAULT_VOCODER_CONFIG, seed=0), DEFAULT_VOCODER_CONFIG, dev)
    den = WavDenoiser(None, dev)
    lines = []

    def emit(res):
        line = json.dumps(res)
        print(line, flush=True)
        lines.append(line)

    batch64_offs = None
    for wl in ("utt10s", "batch64"):
        utts, desc = make_workload(wl, 0, 1)
        pb = pack_batch(utts).to(dev)
        fo, Fs = pb.frame_offsets, pb.total_frames
        g = torch.Generator(device=dev).manual_seed(1)
        mel = (torch.randn(Fs, 80, generator=g, device=dev) * 0.5 - 3.0).contiguous()
        f0 = (200.0 + 100.0 * torch.rand(Fs, generator=g, device=dev)).contiguous()
        if wl == "batch64":
            batch64_offs = (fo * HOP).astype(np.int32)
        arms = {"vocoder": lambda: voc.generate(mel, f0, fo, seed=2),
                "vocoder+denoiser": lambda: voc.generate(mel, f0, fo, seed=2, denoise_c=V)}
        med, ms = measure(arms, args.reps)
        emit({"what": "vocoder stage", "workload": wl, "desc": desc, "frames": Fs, "samples": Fs * HOP, "v": V,
              "card": info, "reps": args.reps, "ms": {k: round(x, 3) for k, x in med.items()},
              "denoiser_share_of_stage": round((med["vocoder+denoiser"] - med["vocoder"]) / med["vocoder+denoiser"], 4),
              "ms_all": {k: [round(x, 3) for x in v] for k, v in ms.items()}})

    rng = np.random.default_rng(3)
    for name, offs in (("batch64 lengths", batch64_offs), ("one 3 s utterance", np.array([0, 3 * 48000 // HOP * HOP], np.int32))):
        n = int(offs[-1])
        x = torch.from_numpy(np.clip(0.3 * rng.standard_normal(n), -1, 1).astype(np.float32)).to(dev)
        out = torch.empty_like(x)
        frames = np.diff(offs) // HOP + 1
        row_tiles = int(sum((f + 127) // 128 for f in frames))

        def run(tc):  # forced: 0 = FFMA, 2 = tensor cores at every size
            den.set_tensor_cores(2 if tc else 0)
            return den(x, offs, V, out=out)

        arms = {"ffma": lambda: run(False), "tensor_cores": lambda: run(True)}
        med, ms = measure(arms, args.reps)
        ref = run(False).clone()
        diff = float((run(True) - ref).abs().max())
        den.set_tensor_cores(1)
        emit({"what": "denoiser alone", "workload": name, "utterances": len(offs) - 1, "samples": n, "row_tiles": row_tiles,
              "automatic_path": "tensor_cores" if row_tiles >= 8 else "ffma", "v": V, "card": info, "reps": args.reps,
              "ms": {k: round(x, 3) for k, x in med.items()}, "ms_all": {k: [round(x, 3) for x in v] for k, v in ms.items()},
              "max_abs_diff_tc_vs_ffma": diff,
              "gemm_tflop_executed": round(2.0 * float(frames.sum()) * 2 * (2 * 544) * 1024 / 1e12, 4)})
    if args.out:
        with open(args.out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
