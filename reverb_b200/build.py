"""Build the sm_90a (H100) shared library `reverb_b200/librvb_b200.so` in-tree with nvcc.

    python -m reverb_b200.build            # or: from reverb_b200.build import build; build()

nvcc cross-compiles without a GPU.  The .so and the objects under csrc/build/ are build products (git-ignored).
"""
from __future__ import annotations

import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "librvb_b200.so")
SOURCES = ["gemm.cu", "elementwise.cu", "attention.cu", "attention_tc.cu", "attention_f32.cu", "fbank.cu", "resample.cu", "ctc.cu",
           "context.cu", "align.cu", "engine.cu", "diar_seg.cu", "diar_wavlm.cu", "diar_emb.cu",
           "diar_cluster.cu", "flac.cu", "wav_codec.cu"]
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
              "-Xcompiler", "-fPIC", "-Xcompiler", "-fvisibility=hidden", "--expt-relaxed-constexpr"]


def _nvcc() -> str:
    for c in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if c and (os.path.isabs(c) and os.path.exists(c) or not os.path.isabs(c)):
            return c
    return "nvcc"


def _stale(target: str, deps) -> bool:
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps)


def build(force: bool = False, verbose: bool = False) -> str:
    objdir = os.path.join(CSRC, "build")
    os.makedirs(objdir, exist_ok=True)
    headers = [os.path.join(CSRC, h) for h in ("common.cuh", "kernels.h", "host_mem.h")] + \
              [os.path.join(HERE, "..", "include", h) for h in ("rvb_b200.h", "rvb_diar.h")]
    nvcc = _nvcc()

    def compile_one(src):
        obj = os.path.join(objdir, src.replace(".cu", ".o"))
        srcp = os.path.join(CSRC, src)
        if force or _stale(obj, [srcp] + headers):
            cmd = [nvcc] + NVCC_FLAGS + ["-c", srcp, "-o", obj]
            if verbose:
                print(" ".join(cmd), flush=True)
            r = subprocess.run(cmd, capture_output=True, text=True)
            if r.returncode != 0:
                raise RuntimeError(f"nvcc failed on {src}:\n{r.stdout}\n{r.stderr}")
        return obj

    with ThreadPoolExecutor(max_workers=min(6, os.cpu_count() or 2)) as ex:
        objs = list(ex.map(compile_one, SOURCES))
    if force or _stale(LIB, objs):
        cmd = [nvcc, "-shared", "-o", LIB] + objs + ["-gencode", "arch=compute_90a,code=sm_90a", "-lcudart"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
