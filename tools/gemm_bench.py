"""Per-shape timing of the wgmma GEMM kernel through the C ABI (CUDA events, warm, L2-cold-ish: operands >> L2)."""
import ctypes as C
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from reverb_b200 import _lib

lib = _lib.load()


def p(t):
    return C.c_void_p(t.data_ptr())


def bench(M, N, K, act, out_mode, iters=10):
    A = (torch.randn(M, K, device="cuda") * 0.5).bfloat16()
    W = (torch.randn(N, K, device="cuda") * 0.05).bfloat16()
    bias = torch.randn(N, device="cuda")
    ldo = (N + 3) & ~3
    out = torch.zeros(M, ldo, device="cuda", dtype=torch.float32 if out_mode else torch.bfloat16)
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    for _ in range(3):
        assert lib.rvb_gemm_bf16(p(A), p(W), p(bias), M, N, K, act, out_mode, 1.0, p(out), ldo, st) == 0
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(iters):
        lib.rvb_gemm_bf16(p(A), p(W), p(bias), M, N, K, act, out_mode, 1.0, p(out), ldo, st)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / iters
    tf = 2.0 * M * N * K / (ms * 1e-3) / 1e12
    # cuBLAS reference for the same shape (context only)
    C_ = torch.empty(M, N, device="cuda", dtype=torch.bfloat16)
    for _ in range(3):
        torch.matmul(A, W.t(), out=C_)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(iters):
        torch.matmul(A, W.t(), out=C_)
    e1.record()
    torch.cuda.synchronize()
    ms_cb = e0.elapsed_time(e1) / iters
    return {"M": M, "N": N, "K": K, "act": act, "out": out_mode, "ms": round(ms, 4), "tflops": round(tf, 1),
            "cublas_ms": round(ms_cb, 4), "cublas_tflops": round(2.0 * M * N * K / (ms_cb * 1e-3) / 1e12, 1)}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i",
                        str(torch.cuda.current_device())], capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name()


if __name__ == "__main__":
    if len(sys.argv) > 1 and sys.argv[1] == "one":       # single shape, for ncu captures
        print(json.dumps(bench(47872, 4096, 1024, 2, 0, iters=3)))
        sys.exit(0)
    print(json.dumps({"card": card(), "lib": os.environ.get("RVB_LIB_PATH") or "in-tree",
                      "skip_epi": os.environ.get("RVB_GEMM_SKIP_EPI", "0")}), flush=True)
    M = 47872
    shapes = [(M, 4096, 1024, 2, 0), (M, 1024, 4096, 0, 2), (M, 3072, 1024, 0, 0), (M, 1024, 1024, 0, 2),
              (M, 2048, 1024, 0, 0), (M, 10001, 1024, 0, 1), (M * 19, 1024, 1024, 1, 0), (M, 1024, 19456, 0, 1),
              (8192, 8192, 8192, 0, 0)]
    for s in shapes:
        print(json.dumps(bench(*s)), flush=True)
