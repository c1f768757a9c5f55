"""128 x 256 against 128 x 128 GEMM tiles in one process (csrc/gemm.cu `gemm_wide_kernel` / `gemm_wg_kernel`).

For each shape the two tile widths alternate (RVB_GEMM_WIDE is read per call), `--rounds` times, each round timed
with CUDA events over `--iters` launches; prints one JSON line per (shape, round, tiles) with ms and TFLOP/s, one per
shape with the mean SM clock nvidia-smi sampled over all its rounds, then the card's name, power limit and max SM
clock.  Run it with RVB_GEMM_SKIP_EPI=1 for the main loops alone (the FFN2 shape, a residual GEMM the wide tiles do not
serve, is then timed with a bf16 output: only the main loop runs).

    python tools/gemm_wide_bench.py [--rounds 3] [--iters 100]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import threading

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from reverb_b200 import _lib

M = 47872   # 64 x 30 s chunks x 748 frames
SHAPES = {   # name -> (M, N, K, act)
    "FFN1": (M, 4096, 1024, 2),
    "conv2-shaped (K = 9 x 1024, 1/8 of the rows)": (64 * 748 * 19 // 8, 1024, 9216, 1),
    "FFN2 main loop": (M, 1024, 4096, 0),
}


def _p(t):
    return C.c_void_p(t.data_ptr())


class SmClock:
    def __init__(self):
        self.proc = subprocess.Popen(["nvidia-smi", "--query-gpu=clocks.sm", "--format=csv,noheader,nounits", "-lms",
                                      "100", "-i", str(torch.cuda.current_device())], stdout=subprocess.PIPE, text=True)
        self.vals = []
        self.t = threading.Thread(target=lambda: [self.vals.append(ln.strip()) for ln in self.proc.stdout], daemon=True)
        self.t.start()

    def stop(self):
        self.proc.terminate()
        self.proc.wait()
        v = [int(x) for x in self.vals if x.isdigit()]
        return round(sum(v) / len(v)) if v else None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--iters", type=int, default=100)
    args = ap.parse_args()
    lib = _lib.load()
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    skip = os.environ.get("RVB_GEMM_SKIP_EPI", "0")
    for name, (m, n, k, act) in SHAPES.items():
        A = (torch.randn(m, k, device="cuda") * 0.5).bfloat16()
        W = (torch.randn(n, k, device="cuda") * 0.05).bfloat16()
        bias = torch.randn(n, device="cuda")
        out = torch.empty(m, n, device="cuda", dtype=torch.bfloat16)

        def launch():
            assert lib.rvb_gemm_bf16(_p(A), _p(W), _p(bias), m, n, k, act, 0, 1.0, _p(out), n, st) == 0, _lib.last_error()

        for wide in (True, False):   # warm both kernels
            os.environ["RVB_GEMM_WIDE"] = "1" if wide else "0"
            for _ in range(3):
                launch()
        torch.cuda.synchronize()
        clk = SmClock()
        for r in range(args.rounds):
            for wide in (True, False):
                os.environ["RVB_GEMM_WIDE"] = "1" if wide else "0"
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(args.iters):
                    launch()
                e1.record()
                torch.cuda.synchronize()
                ms = e0.elapsed_time(e1) / args.iters
                print(json.dumps({"shape": name, "M": m, "N": n, "K": k, "act": act, "skip_epi": skip, "round": r,
                                  "tiles": "128x256" if wide else "128x128", "ms": round(ms, 4),
                                  "tflops": round(2.0 * m * n * k / (ms * 1e-3) / 1e12, 1)}), flush=True)
        print(json.dumps({"shape": name, "skip_epi": skip, "sm_mhz_mean": clk.stop()}), flush=True)
        os.environ.pop("RVB_GEMM_WIDE", None)
        del A, W, out
        torch.cuda.empty_cache()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i",
                        str(torch.cuda.current_device())], capture_output=True, text=True)
    print(json.dumps({"card": q.stdout.strip()}), flush=True)


if __name__ == "__main__":
    main()
