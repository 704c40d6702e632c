"""Build libstylesinger_b200.so in-tree with nvcc for sm_90a (H100, and only sm_90a).

    python -m stylesinger_b200.build [--force]

The .so and the object files under build/ are git-ignored build products.
"""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libstylesinger_b200.so")
SOURCES = ["conv_gemm.cu", "conv_gemm_tc.cu", "sampler_tc.cu", "ops.cu", "attention.cu", "attention_tc.cu", "pack.cu", "stages.cu", "frontend.cu", "wav_denoise.cu", "lstm.cu", "api.cu"]
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
              "-Xcompiler", "-fPIC", "--use_fast_math=false"]


def _nvcc():
    for c in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if c and (os.path.isabs(c) and os.path.exists(c) or not os.path.isabs(c)):
            return c
    return "nvcc"


def _stale(target, deps):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=True):
    hdrs = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))]
    hdrs.append(os.path.join(os.path.dirname(HERE), "include", "stylesinger_b200.h"))
    objdir = os.path.join(HERE, "build")
    os.makedirs(objdir, exist_ok=True)
    objs = []
    procs = []
    flags = [f for f in NVCC_FLAGS if not f.startswith("--use_fast_math")]
    for s in SOURCES:
        src = os.path.join(CSRC, s)
        obj = os.path.join(objdir, s.replace(".cu", ".o"))
        objs.append(obj)
        if force or _stale(obj, [src] + hdrs):
            cmd = [_nvcc()] + flags + ["-c", src, "-o", obj]
            if verbose:
                print(" ".join(cmd), flush=True)
            procs.append((s, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    failed = False
    for s, p in procs:
        out, _ = p.communicate()
        if out.strip() and verbose:
            print(out)
        if p.returncode != 0:
            print(f"nvcc failed for {s}:\n{out}", file=sys.stderr)
            failed = True
    if failed:
        raise RuntimeError("nvcc compilation failed")
    if force or procs or _stale(LIB, objs):
        tmp = LIB + ".tmp"  # link beside the target, then rename: a snapshot of the tree never sees a half-written .so
        cmd = [_nvcc()] + flags + ["-shared", "-o", tmp] + objs + ["-lcudart"]
        if verbose:
            print(" ".join(cmd), flush=True)
        subprocess.check_call(cmd)
        os.replace(tmp, LIB)
    return LIB


if __name__ == "__main__":
    build(force="--force" in sys.argv)
    print("built", LIB)
