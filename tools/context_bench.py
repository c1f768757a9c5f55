"""Context biasing on one GPU, at the benchmarked shape (synthetic reverb_asr_v1-shaped model, 64 x 30 s chunks per step,
beam 10, attention rescoring without the right-to-left decoder, one software-pipelined stream like bench.py), with seeded phrase lists of 100, 1 000 and
10 000 phrases (reverb_b200.synth.context_phrases):
  * step time without a graph and with each graph, the configurations alternated in one run (host clock around steps
    that end in a synchronise);
  * prefix beam search kernel time, biased against unbiased, on the same top-k (torch.profiler CUDA activity, kernel
    names ctc_prefix_beam_kernel<false> / <true>);
  * one utterance through the host search `search.ctc_prefix_beam_search_biased`, for contrast.
Prints one JSON line with the card's name, power limit and max SM clock.

    python tools/context_bench.py [--steps 6] [--warmup 2] [--rounds 2] > context_bench.json
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
from reverb_b200.context_graph import ContextGraph  # noqa: E402
from reverb_b200.search import ctc_prefix_beam_search_biased  # noqa: E402

SIZES = (100, 1000, 10000)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i",
                        str(torch.cuda.current_device())], capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--chunks", type=int, default=64)
    ap.add_argument("--steps", type=int, default=6, help="timed steps per configuration and round")
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--rounds", type=int, default=2, help="times the configurations are alternated")
    ap.add_argument("--score", type=float, default=6.0)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("context_bench needs a GPU")
    with tempfile.TemporaryDirectory() as d:
        synth.write_model_dir(d, shape=synth.BENCH_SHAPE, seed=0, causal=True, cnn_module_norm="layer_norm",
                              reverse_weight=0.3)
        asr = reverb_b200.ReverbASR(os.path.join(d, "config.yaml"), os.path.join(d, "synth.pt"))
    eng, model, V = asr.engine, asr.model, asr.engine.vocab
    out = {"card": card(), "vocab": V, "chunks": args.chunks, "beam": 10, "mode": "attention_rescoring"}
    base = [synth.synth_audio(30.0, seed=1234 + i) for i in range(5)]
    pcm = torch.from_numpy(np.stack([(base[i % 5].astype(np.float32) * (1.0 - 0.03 * (i // 5 % 8))).astype(np.int16)
                                     for i in range(args.chunks)])).cuda()
    lens = torch.full((args.chunks,), 2998, dtype=torch.int32)
    cat = torch.tensor([1.0, 0.0])
    graphs = {n: ContextGraph(token_lists=synth.context_phrases(n, V, seed=n), context_score=args.score) for n in SIZES}
    out["graph_states"] = {str(n): g.num_nodes + 1 for n, g in graphs.items()}
    for g in graphs.values():
        eng.device_context_graph(g, asr.blank_id)                  # uploaded once, outside the timed steps

    def steps(n, graph):
        def batches():
            for _ in range(n):
                yield eng.fbank_batch(pcm), lens
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        ntok = 0
        for res in model.decode_stream(batches(), ["attention_rescoring"], 10, ctc_weight=0.1, reverse_weight=0.0,
                                       blank_id=asr.blank_id, cat_embs=cat, context_graph=graph):
            ntok += sum(len(r.tokens) for r in res["attention_rescoring"])
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) * 1e3 / n, ntok // n

    configs = [("none", None)] + [(str(n), graphs[n]) for n in SIZES]
    step_ms = {name: [] for name, _ in configs}
    tokens = {}
    for name, g in configs:
        steps(args.warmup, g)
    for _ in range(args.rounds):
        for name, g in configs:
            ms, tokens[name] = steps(args.steps, g)
            step_ms[name].append(ms)
    out["step_ms"] = step_ms
    out["best_hypothesis_tokens_per_step"] = tokens       # a larger graph boosts more tokens: longer hypotheses
    out["step_vs_none"] = {name: min(v) / min(step_ms["none"]) - 1.0 for name, v in step_ms.items()}

    # ---- search kernel alone, on the top-k of one real step
    feats = eng.fbank_batch(pcm)
    enc, enc_lens = model._forward_encoder(feats, lens, cat)
    val, idx, _ = eng.ctc_topk(enc, 10)
    del enc, feats
    from torch.profiler import ProfilerActivity, profile
    reps = 5
    for g in (None,) + tuple(graphs.values()):
        eng.prefix_beam_search_raw(val, idx, enc_lens, 10, asr.blank_id, context=g)
    kernel = {}
    for name, g in configs:
        with profile(activities=[ProfilerActivity.CUDA], acc_events=True) as prof:
            for _ in range(reps):
                eng.prefix_beam_search_raw(val, idx, enc_lens, 10, asr.blank_id, context=g)
            torch.cuda.synchronize()
        ts = [e.time_range.elapsed_us() for e in prof.events()
              if "ctc_prefix_beam_kernel" in e.name and e.device_type.name == "CUDA"]
        kernel[name] = {"ms_mean": float(np.mean(ts)) / 1e3, "ms_min": float(np.min(ts)) / 1e3, "launches": len(ts)}
    out["search_kernel"] = kernel

    # ---- the host search for one utterance, for contrast
    v1, i1 = val[:1].cpu().numpy(), idx[:1].cpu().numpy()
    t0 = time.perf_counter()
    ctc_prefix_beam_search_biased(v1, i1, enc_lens[:1], 10, graphs[1000], asr.blank_id)
    out["host_search_one_utterance_1000_phrases_ms"] = (time.perf_counter() - t0) * 1e3
    print(json.dumps(out))


if __name__ == "__main__":
    main()
