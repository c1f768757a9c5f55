"""Diarization leg on one GPU (SURVEY.md §8f rank 1, BASELINE configs[4]-shaped: one long recording): CUDA-event times of
the segmentation and embedding networks on batches of 10 s windows, and the wall time of the whole pipeline
(windows -> segmentation -> count -> embeddings -> clustering -> RTTM turns) on a synthetic recording.

    python tools/diar_bench.py [--seconds 2700] [--batch 64] > diar_bench.json
Synthetic weights (no checkpoint offline) — the numbers are throughput only.
"""
import argparse
import json
import sys
import time

import numpy as np
import torch

sys.path.insert(0, __import__("os").path.dirname(__import__("os").path.dirname(__import__("os").path.abspath(__file__))))

from reverb_b200.diarization import synth  # noqa: E402
from reverb_b200.diarization.embedding import EmbeddingModel  # noqa: E402
from reverb_b200.diarization.pipeline import SpeakerDiarization  # noqa: E402
from reverb_b200.diarization.segmentation import SegmentationModel  # noqa: E402


def timed(fn, iters=5, warmup=2):
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=2700.0)
    ap.add_argument("--batch", type=int, default=64)
    args = ap.parse_args()
    seg = SegmentationModel(synth.segmentation_state_dict(0))
    emb = EmbeddingModel(synth.embedding_state_dict(0))
    B = args.batch
    win = torch.from_numpy(np.stack([synth.synthetic_speech(10.0, seed=i, turns=2) for i in range(8)])).cuda()
    win = win.repeat((B + 7) // 8, 1)[:B].contiguous()
    masks = (torch.rand(B, 3, 589, device="cuda") > 0.5).float()
    seg_ms = timed(lambda: seg(win))
    emb_ms = timed(lambda: emb(win, masks))
    out = {"batch_windows": B, "segmentation_ms": seg_ms, "embedding_ms": emb_ms,
           "segmentation_windows_per_s": B / seg_ms * 1e3, "embedding_windows_per_s": B / emb_ms * 1e3,
           # 1.3 GMAC (segmentation) / 23.5 GMAC (ResNet34 trunk) per 10 s window
           "segmentation_tflops": B * 1.3e9 * 2 / seg_ms / 1e9, "embedding_tflops": B * 23.5e9 * 2 / emb_ms / 1e9}
    audio = synth.synthetic_speech(args.seconds, seed=11, turns=3)
    pipe = SpeakerDiarization(seg, emb, batch_size=B)
    pipe(audio[: 16000 * 60])                                     # warm-up (allocations)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    turns = pipe(audio)
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    out.update({"recording_seconds": args.seconds, "pipeline_seconds": dt, "pipeline_rtfx": args.seconds / dt,
                "pipeline_stages_seconds": {k: round(v, 4) for k, v in pipe.last["timing"].items()},
                "windows": int(pipe.last["binarized"].shape[0]), "turns": len(turns),
                "speakers": len({t.label for t in turns}), "data": "synthetic audio, synthetic weights"})
    print(json.dumps(out))


if __name__ == "__main__":
    main()
