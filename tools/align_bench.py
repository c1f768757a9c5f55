"""CTC forced alignment on one GPU (csrc/align.cu): CUDA-event times (host-clock times where a side stream is involved) of
  * the batched form on 64 chunks of 30 s (748 encoder frames each) with ~100 labels per chunk;
  * the resumable form on one 3600 s recording (120 chunks, 89 760 frames) against 12 000 labels, pushed 8 chunks at a
    time: alone, and with every push enqueued between two encoder + CTC-head passes of the benchmarked shape, where the
    trellis runs on the search side stream (the question: does it hide under the encoder?).
Also the bytes each trellis step reads and writes, computed from the shapes.  Log-probs are random (the time of the
kernels does not depend on the values); the model has synthetic weights.  Prints one JSON line with the card's name and
power limit.

    python tools/align_bench.py [--labels 12000] [--seconds 3600] > align_bench.json
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import reverb_b200  # noqa: E402
from reverb_b200 import synth  # noqa: E402
from reverb_b200.engine import Aligner  # noqa: E402


def timed(fn, iters, warmup=1):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i",
                        str(torch.cuda.current_device())], capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name()


def labels(rng, n, V):
    y = rng.integers(1, V - 1, n)
    y[1:][y[1:] == y[:-1]] -= 1
    y[y < 1] = 2
    return [int(t) for t in y]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--labels", type=int, default=12000)
    ap.add_argument("--seconds", type=float, default=3600.0)
    ap.add_argument("--push_chunks", type=int, default=8)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("align_bench needs a GPU")
    rng = np.random.default_rng(0)
    with tempfile.TemporaryDirectory() as d:
        synth.write_model_dir(d, shape=synth.BENCH_SHAPE, seed=0, causal=True, cnn_module_norm="layer_norm")
        m = reverb_b200.load_model(d)
    eng, V, Tp = m.engine, m.engine.vocab, 748
    out = {"card": card(), "vocab": V}

    # ---- batched: 64 x 30 s
    logp = torch.log_softmax(torch.randn(64, Tp, V, device="cuda") * 3, dim=-1)
    ys = [labels(rng, int(rng.integers(80, 120)), V) for _ in range(64)]
    for ll in (False, True):
        ms = timed(lambda: eng.force_align(logp, [Tp] * 64, ys, 0, ll), iters=40, warmup=3)
        out["batched_64x30s_ms" + ("_with_loglik" if ll else "")] = ms
    slots = 128                                                    # 101..120 label slots round up to one warp x 4
    out["batched_bytes_per_step_per_utt"] = {"emissions_read": (slots + 4) * 4, "backpointers_written": slots}
    del logp

    # ---- resumable: one long recording
    n_chunks = int(np.ceil(args.seconds / 29.98))
    U, total, pc = args.labels, n_chunks * Tp, args.push_chunks
    y = labels(rng, U, V)
    rows = torch.log_softmax(torch.randn(pc * Tp, V, device="cuda") * 3, dim=-1)
    out["resumable"] = {"seconds": args.seconds, "frames": total, "labels": U,
                        "workspace_bytes": Aligner.workspace_bytes(U, total)}
    P = (U + 1 + 767) // 768 * 768 if U + 1 > 4096 else (U + 1 + 127) // 128 * 128
    out["resumable"]["bytes_per_step"] = {"emissions_read": (P + 4) * 4, "backpointers_written": P}

    def pushes(al, between=None):
        done = 0
        while done < total:
            n = min(pc * Tp, total - done)
            if between is not None:
                between()
            al.push(rows[:n])
            done += n

    def alone(side):
        al = eng.aligner(y, total, 0, False, side_stream=side)
        pushes(al)
        return al

    alone(False).finish()                                          # warm-up
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    al = eng.aligner(y, total, 0, False, side_stream=False)
    torch.cuda.synchronize()
    a.record()
    pushes(al)
    b.record()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    al.finish()                                                    # synchronises
    fin_ms = (time.perf_counter() - t0) * 1e3
    out["resumable"]["caller_stream"] = {"gather_and_trellis_ms": a.elapsed_time(b),
                                         "us_per_frame": a.elapsed_time(b) * 1e3 / total,
                                         "backtrace_reduce_copy_ms": fin_ms}

    def wall(fn):                                                  # host clock around work that ends in a synchronise
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) * 1e3

    # the trellis on the search side stream: only finish() joins it, so these are host-clock times including finish
    out["resumable"]["side_stream_total_ms"] = wall(lambda: alone(True).finish())

    # ---- overlapped with the encoder + CTC head of the benchmarked shape, 8 chunks per pass
    feats = torch.randn(pc, 2998, 80, device="cuda") * 3
    lens = torch.full((pc,), 2998, dtype=torch.int32)
    cat = torch.tensor([1.0, 0.0])

    def encoder():
        enc, _ = m.model._forward_encoder(feats, lens, cat)
        return m.model.ctc_logprobs(enc)

    enc_ms = timed(encoder, iters=10, warmup=2)
    n_push = (total + pc * Tp - 1) // (pc * Tp)

    def encoder_only():
        for _ in range(n_push):
            encoder()

    parts = {}

    def encoder_and_alignment():
        t0 = time.perf_counter()
        al = eng.aligner(y, total, 0, False, side_stream=True)     # allocates the workspace
        t1 = time.perf_counter()
        pushes(al, between=encoder)
        torch.cuda.current_stream().synchronize()                  # the encoder passes and the gathers are done
        t2 = time.perf_counter()
        al.finish()                                                # what is left of the trellis, then the back-trace
        parts.update(begin_ms=(t1 - t0) * 1e3, passes_ms=(t2 - t1) * 1e3, finish_ms=(time.perf_counter() - t2) * 1e3)

    out["overlap"] = {"encoder_ctc_pass_ms": enc_ms, "passes": n_push, "encoder_only_ms": wall(encoder_only),
                      "encoder_plus_alignment_ms": wall(encoder_and_alignment), "of_which": parts}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
