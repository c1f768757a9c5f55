"""Per-kernel split of the benchmarked step: a few bench-shaped steps (64 x 30 s chunks, `decode_stream`,
attention_rescoring, the bench's synthetic model and audio) under `torch.profiler` with CUDA activities.  Writes the
per-kernel totals (launches, total ms, ms per step, share of the step) as JSON to OUT_DIR/step_profile.json and prints
a summary with the card's name and power limit.  The step time that the shares refer to is taken first, from CUDA
events with the profiler off; the profiled steps run separately.

`gemm_wg_kernel<BN, EPI, PAIR>` and `gemm_wide_kernel<EPI>` instantiations are labelled by the layer their epilogue
serves (csrc/gemm.cu `Epi`).

    python tools/step_profile.py OUT_DIR [--steps 3] [--warmup 3] [--chunks 64]
"""
import argparse
import json
import os
import re
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

GEMM_LAYERS = {0: "bf16 (embed / decoder)", 1: "conv2 (implicit GEMM, ReLU)", 2: "FFN1 (SiLU)",
               3: "fp32 out", 4: "residual (FFN2, attn out, pointwise conv2)", 5: "generic",
               6: "pointwise conv1 (GLU)", 7: "CTC / decoder head (log-sum-exp)", 8: "QKV + rel-pos keys"}
_GEMM_RE = re.compile(r"gemm_wg_kernel<(\d+),\s*(\d+),\s*(true|false)>")
_WIDE_RE = re.compile(r"gemm_wide_kernel<(\d+)>")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i",
                        str(torch.cuda.current_device())], capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name()


def label(name):
    w = _WIDE_RE.search(name)
    if w:
        return f"gemm_wide_kernel<{w.group(1)}> {GEMM_LAYERS.get(int(w.group(1)), '?')}"
    m = _GEMM_RE.search(name)
    if not m:
        return name
    bn, epi, pair = int(m.group(1)), int(m.group(2)), m.group(3) == "true"
    return f"gemm_wg_kernel<{bn},{epi}{',pair' if pair else ''}> {GEMM_LAYERS.get(epi, '?')}"


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("out_dir")
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--chunks", type=int, default=64)
    args = ap.parse_args()
    os.makedirs(args.out_dir, exist_ok=True)

    import bench
    import reverb_b200
    from reverb_b200 import synth
    mdir = bench.model_dir_for("bench")
    pcm = torch.from_numpy(bench.make_pcm(args.chunks, seed=1234))
    print(f"model {mdir}, shape {synth.BENCH_SHAPE}, {args.chunks} x 30 s chunks", file=sys.stderr)
    if not torch.cuda.is_available():
        raise SystemExit("step_profile needs a GPU")

    asr = reverb_b200.ReverbASR(os.path.join(mdir, "config.yaml"), os.path.join(mdir, "synth.pt"), gpu=0)
    eng, model = asr.engine, asr.model
    pcm_dev = pcm.cuda()
    lens = torch.full((args.chunks,), bench.CHUNK_FRAMES, dtype=torch.int32)
    dkw = dict(ctc_weight=0.1, reverse_weight=0.0, blank_id=asr.blank_id, cat_embs=torch.tensor([1.0, 0.0]))

    def run_steps(n):
        for _ in model.decode_stream(((eng.fbank_batch(pcm_dev), lens) for _ in range(n)), ["attention_rescoring"],
                                     10, **dkw):
            pass

    run_steps(args.warmup)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    run_steps(args.steps)
    e1.record()
    torch.cuda.synchronize()
    step_ms = e0.elapsed_time(e1) / args.steps

    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        run_steps(args.steps)
        torch.cuda.synchronize()
    per = {}
    for ev in prof.events():
        if ev.device_type != torch.autograd.DeviceType.CUDA:
            continue
        d = per.setdefault(label(ev.name), {"count": 0, "total_ms": 0.0})
        d["count"] += 1
        d["total_ms"] += ev.device_time_total / 1e3 if hasattr(ev, "device_time_total") else ev.cuda_time_total / 1e3
    kernels = []
    for name, d in per.items():
        ms = d["total_ms"] / args.steps
        kernels.append({"kernel": name, "count": d["count"], "total_ms": round(d["total_ms"], 3),
                        "ms_per_step": round(ms, 3), "share_of_step": round(ms / step_ms, 4)})
    kernels.sort(key=lambda k: -k["total_ms"])
    gemm_ms = sum(k["ms_per_step"] for k in kernels if k["kernel"].startswith(("gemm_wg_kernel", "gemm_wide_kernel")))
    out = {"card": card(), "lib": os.environ.get("RVB_LIB_PATH") or "in-tree", "chunks": args.chunks,
           "profiled_steps": args.steps, "step_ms_unprofiled": round(step_ms, 3),
           "gemm_ms_per_step": round(gemm_ms, 3),
           "all_kernels_ms_per_step": round(sum(k["ms_per_step"] for k in kernels), 3), "kernels": kernels}
    path = os.path.join(args.out_dir, "step_profile.json")
    with open(path, "w") as f:
        json.dump(out, f, indent=1)
    print(f"{out['card']}: step {step_ms:.2f} ms (profiler off), GEMM kernels {gemm_ms:.2f} ms/step -> {path}")
    for k in kernels[:25]:
        print(f"  {k['ms_per_step']:9.3f} ms/step {100 * k['share_of_step']:5.1f} %  x{k['count']:<5d} {k['kernel'][:110]}")


if __name__ == "__main__":
    main()
