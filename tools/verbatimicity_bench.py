"""Per-utterance verbatimicity cost: attention_rescoring steps of 64 x 30 s chunks at the benchmarked model shape, with
G = 1, 2, 8 and 64 distinct verbatimicity values per batch (G = 1 is the one-vector path bench.py times).

    python tools/verbatimicity_bench.py [--reps 5]

Prints the card name, power limit and max SM clock, then per G, over `reps` alternated rounds (G = 1, 2, 8, 64, 1, ...):
  step_ms      ASRModel.decode(["attention_rescoring"]) on the whole batch, a device synchronise inside the timing (the
               decoder's work depends on the transcripts, which change with the values);
  encoder_ms   the encoder pass alone (same work for every G), timed the same way;
  lsl_gemm_ms  the encoder's language-specific linear at this batch's shape (M = 64 T' rows, d x d, fp32 output) as
               the engine launches it — one plain launch for G = 1, one grouped launch over G stacked folds otherwise —
               timed by the GEMM profiler (rvb_gemm_profile_*, CUDA events around each launch), mean of 20 launches.
The rows of the G-value batches cycle through the values, so every 128-row tile of the encoder holds one or two groups.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from reverb_b200 import synth  # noqa: E402

B, CHUNK, GROUPS = 64, 2998, [1, 2, 8, 64]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else f"nvidia-smi failed: {q.stderr.strip()}"


def values(G):
    """B per-row verbatimicity values with G distinct ones, each a run of B / G consecutive rows."""
    v = [1.0] if G == 1 else [g / (G - 1) for g in range(G)]
    return [v[b * G // B] for b in range(B)]


def cat_rows(vals):
    return torch.tensor([[v, 1.0 - v] for v in vals])


def lsl_gemm_ms(lib, M, d, G, launches=20):
    """Mean time of the encoder's LSL GEMM launch at G groups (fp32 output, bf16 operands)."""
    gen = torch.Generator(device="cuda").manual_seed(G)
    A = torch.randn(M, d, device="cuda", generator=gen).bfloat16()
    W = (torch.randn(G * d, d, device="cuda", generator=gen) / d ** 0.5).bfloat16()
    bias = torch.randn(G * d, device="cuda", generator=gen)
    out = torch.empty(M, d, device="cuda")
    Tp = M // B
    grp = torch.tensor([b * G // B for b in range(B)], dtype=torch.int32, device="cuda")
    p = lambda t: C.c_void_p(t.data_ptr())                                # noqa: E731
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)

    def launch():
        rc = (lib.rvb_gemm_bf16(p(A), p(W), p(bias), M, d, d, 0, 1, 1.0, p(out), d, st) if G == 1 else
              lib.rvb_gemm_grouped(p(A), p(W), p(bias), M, G * d, d, 1, p(out), d, p(grp), Tp, d, 0, st))
        assert rc == 0
    for _ in range(3):
        launch()
    torch.cuda.synchronize()
    lib.rvb_gemm_profile_begin()
    for _ in range(launches):
        launch()
    ms, fl, n = C.c_double(), C.c_double(), C.c_longlong()
    lib.rvb_gemm_profile_end(C.byref(ms), C.byref(fl), C.byref(n))
    assert n.value == launches
    return ms.value / launches


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5, help="alternated rounds over G")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("verbatimicity_bench needs a CUDA device")
    import reverb_b200
    from reverb_b200 import _lib
    print(f"card: {card()}", flush=True)
    with tempfile.TemporaryDirectory(prefix="rvb_verb_") as tmp:
        synth.write_model_dir(tmp, shape=synth.BENCH_SHAPE, seed=0, causal=True, cnn_module_norm="layer_norm")
        m = reverb_b200.load_model(tmp)
        rows = []
        for s in range(8):
            wav = synth.write_wav(os.path.join(tmp, f"a{s}.wav"), synth.synth_audio(30.0, seed=100 + s))
            rows.append(m.compute_feats(wav, num_mel_bins=80, frame_length=25, frame_shift=10)[0][:CHUNK])
        x = torch.stack([rows[b % 8] for b in range(B)]).contiguous()
        lens = torch.full((B,), CHUNK, dtype=torch.int32)
        kw = dict(ctc_weight=0.1, blank_id=m.blank_id, infos={"tasks": ["transcribe"], "langs": ["en"]})
        cats = {G: cat_rows(values(G)) for G in GROUPS}
        for G in GROUPS:                                   # warm every shape and fold set
            m.model.decode(["attention_rescoring"], x, lens, 10, cat_embs=cats[G], **kw)
        steps = {G: [] for G in GROUPS}
        encs = {G: [] for G in GROUPS}
        xd = x.cuda()
        for _ in range(args.reps):
            for G in GROUPS:
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                m.model.decode(["attention_rescoring"], x, lens, 10, cat_embs=cats[G], **kw)
                torch.cuda.synchronize()
                steps[G].append((time.perf_counter() - t0) * 1e3)
            for G in GROUPS:
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                m.model._forward_encoder(xd, lens, cats[G])
                torch.cuda.synchronize()
                encs[G].append((time.perf_counter() - t0) * 1e3)
        lib = _lib.load()
        Tp = m.engine.encoder_out_frames(CHUNK)
        d = m.engine.d_model
        for G in GROUPS:
            gemm = [lsl_gemm_ms(lib, B * Tp, d, G) for _ in range(args.reps)]
            print(json.dumps({"G": G, "step_ms_median": round(float(np.median(steps[G])), 2),
                              "step_ms": [round(t, 2) for t in steps[G]],
                              "encoder_ms_median": round(float(np.median(encs[G])), 2),
                              "lsl_gemm_ms_median": round(float(np.median(gemm)), 4),
                              "lsl_gemm_M": B * Tp, "d": d}), flush=True)


if __name__ == "__main__":
    main()
