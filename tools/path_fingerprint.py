"""Fingerprint of what the library computes and launches, for comparing two builds of it bit for bit.

    python tools/path_fingerprint.py --out fp.json [--T 4] [--workloads short,utt10s,batch64]

For each workload (short: two 1.5 s utterances, fp32 FFMA path; utt10s and batch64: bench.py's, tensor-core path) it runs, on
seeded inputs and with the in-kernel Philox noise: the acoustic forward of a gmdiff and of an f0_gen 'conv' model at T
diffusion steps, the FFT decoder, get_style and pitch-predictor entry points, and the vocoder.  The JSON holds the SHA-256 of
every output tensor, whether a second identical call reproduced it bit for bit, every ssb_*_workspace_bytes, and the launch
count and per-variant tensor-core launch counts of each call.  A refactor that launches the same kernels in the same order
with the same arguments gives the same file as its parent; run it from each tree and diff the two.  Needs a GPU.
"""
import argparse
import ctypes as C
import hashlib
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from bench import make_workload
from stylesinger_b200 import synth
from stylesinger_b200._lib import lib, variant_launches
from stylesinger_b200.engine import AcousticModel, Vocoder, pack_batch
from stylesinger_b200.hparams import DEFAULT_VOCODER_CONFIG, resolve

ALL_OUT = ("mel_out", "f0_denorm", "encoder_out", "style", "rq_codes", "pitch_pred", "decoder_inp", "coarse_mel", "diff_cond",
           "mel2ph", "spk_proj", "emo_proj")


def sha(t):
    return hashlib.sha256(t.detach().cpu().contiguous().numpy().tobytes()).hexdigest()


def call(fn):
    """Run fn twice: hashes of its tensors, launches of one call, variant launches of one call, bit-reproducibility."""
    torch.cuda.synchronize()
    l0, v0 = lib.ssb_launch_count(), variant_launches()
    r = fn()
    torch.cuda.synchronize()
    l1, v1 = lib.ssb_launch_count(), variant_launches()
    r = r if isinstance(r, dict) else dict(enumerate(r)) if isinstance(r, tuple) else {"out": r}
    h = {str(k): sha(v) for k, v in sorted(r.items(), key=lambda kv: str(kv[0]))}
    r2 = fn()
    torch.cuda.synchronize()
    r2 = r2 if isinstance(r2, dict) else dict(enumerate(r2)) if isinstance(r2, tuple) else {"out": r2}
    same = all(sha(v) == h[str(k)] for k, v in r2.items())
    return {"sha256": h, "launches": int(l1 - l0), "repeat_identical": same,
            "variants": {k: v1[k] - v0.get(k, 0) for k in sorted(v1) if v1[k] != v0.get(k, 0)}}


def workload(name):
    if name == "short":
        return [synth.make_utterance(1.5, utt_idx=i, ref_frames=96) for i in range(2)]
    return make_workload(name, 0, 1)[0]


def fingerprint(name, T, dev):
    utts = workload(name)
    pb = pack_batch(utts).to(dev)
    fo, ro, B = pb.frame_offsets, pb.ref_offsets, pb.B
    Fs = int(fo[-1])
    g = torch.Generator().manual_seed(11)
    x = torch.randn(Fs, 256, generator=g)
    x[::97] = 0  # some padding frames: the decoder and the aligner take their masks from the data
    x = x.to(dev)
    res = {"frames": Fs, "B": B}
    ws = {}
    for f0_gen in ("gmdiff", "conv"):
        hp = resolve(timesteps=T, K_step=T, f0_timesteps=T, f0_gen=f0_gen)
        m = AcousticModel(synth.acoustic_state_dict(hp, seed=0), hp, dev)
        a = m._inputs(pb, seed=1)
        ws[f0_gen + ".acoustic"] = int(lib.ssb_acoustic_workspace_bytes(m._h, C.byref(a)))
        ws[f0_gen + ".durations"] = int(lib.ssb_durations_workspace_bytes(m._h, C.byref(a)))
        res[f0_gen + ".forward"] = call(lambda: m.forward(pb, seed=1, want=ALL_OUT))
        if f0_gen == "conv":
            ws["pitch_predictor"] = int(lib.ssb_pitch_predictor_workspace_bytes(m._h, fo.ctypes.data, B))
            for which in (0, 1):
                res[f"pitch_predictor{which}"] = call(lambda: m.pitch_predictor(which, x, fo))
            continue
        ws["mel_diffusion"] = int(lib.ssb_mel_diffusion_workspace_bytes(m._h, fo.ctypes.data, B))
        ws["mel_diffusion_plms"] = int(lib.ssb_mel_diffusion_plms_workspace_bytes(m._h, fo.ctypes.data, B))
        ws["fft_encoder"] = int(lib.ssb_fft_workspace_bytes(m._h, 0, pb.ph_offsets.ctypes.data, B))
        ws["fft_decoder"] = int(lib.ssb_fft_workspace_bytes(m._h, 1, fo.ctypes.data, B))
        ws["get_style"] = int(lib.ssb_get_style_workspace_bytes(m._h, fo.ctypes.data, ro.ctypes.data, B))
        res["fft_encoder"] = call(lambda: m.fft_encoder(pb.t["txt_tokens"], pb.ph_offsets))
        res["fft_decoder"] = call(lambda: m.fft_decoder(x, fo))
        res["get_style"] = call(lambda: m.get_style(x, fo, pb.t["ref_mels"], pb.t["ref_f0"], ro))
        m.set_persistent(False)  # one launch per GEMM: the denoiser's per-step drivers
        res["gmdiff.forward.per_step_launches"] = call(lambda: m.forward(pb, seed=1, want=("mel_out", "f0_denorm")))
    voc = Vocoder(synth.vocoder_state_dict(DEFAULT_VOCODER_CONFIG, seed=0), DEFAULT_VOCODER_CONFIG, dev)
    mel = (torch.randn(Fs, 80, generator=g) * 0.8 - 2.5).clamp(-6, 1.5).to(dev)
    f0 = (220.0 + 80.0 * torch.rand(Fs, generator=g)) * (torch.rand(Fs, generator=g) > 0.2)
    f0 = f0.to(dev)
    n = B if Fs <= voc.max_frames_per_call else 1  # a larger batch is generated in groups: the first utterance's then
    ws["vocoder"] = int(lib.ssb_vocoder_workspace_bytes(voc._h, np.ascontiguousarray(fo[:n + 1]).ctypes.data, n))
    res["vocoder"] = call(lambda: voc.generate(mel, f0, fo, seed=3))
    res["vocoder.no_f0"] = call(lambda: voc.generate(mel, None, fo, seed=3))
    res["workspace_bytes"] = ws
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--T", type=int, default=4)
    ap.add_argument("--workloads", default="short,utt10s,batch64")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("path_fingerprint: no CUDA device (the fingerprint is of what runs on the GPU)")
    dev = torch.device("cuda:0")
    out = {"T": a.T}
    for name in a.workloads.split(","):
        out[name] = fingerprint(name, a.T, dev)
        torch.cuda.empty_cache()
    with open(a.out, "w") as f:
        f.write(json.dumps(out, indent=1, sort_keys=True) + "\n")
    print(json.dumps({k: {c: v[c]["launches"] for c in v if isinstance(v[c], dict) and "launches" in v[c]}
                      for k, v in out.items() if isinstance(v, dict)}))


if __name__ == "__main__":
    main()
