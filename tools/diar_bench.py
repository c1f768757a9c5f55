"""Diarization leg on one GPU (SURVEY.md §8f rank 1, BASELINE configs[4]-shaped: one long recording): CUDA-event times of
the segmentation and embedding networks on batches of 10 s windows, and the wall time of the whole pipeline
(windows -> segmentation -> count -> embeddings -> clustering -> RTTM turns) on a synthetic recording.

    python tools/diar_bench.py [--seconds 2700] [--batch 64] [--segmentation v1|v2] > diar_bench.json
Synthetic weights (no checkpoint offline) — the numbers are throughput only.  The card's name and power limit are read
in the same run.  --segmentation v2 runs the WavLM network (reverb-diarization-v2): its FLOPs per window come from
wavlm_flops() below, and one profiled forward splits its kernel time by stage (wavlm_stage_split()).
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
from reverb_b200.diarization.segmentation import SegmentationModel, WavLMSegmentationModel  # noqa: E402


def wavlm_flops(num_samples: int = 160000) -> dict:
    """FLOPs of one WavLM segmentation window by stage (multiply-add = 2), from the layer shapes."""
    T = [num_samples]
    for k, s in synth.WAVLM_CONV:
        T.append((T[-1] - k) // s + 1)
    C, D, F, L, K, G = 512, 768, 3072, 12, 128, 16
    conv = 2 * T[1] * C * 10 + sum(2 * T[i + 1] * C * C * k for i, (k, _) in enumerate(synth.WAVLM_CONV) if i > 0)
    t = T[-1]
    proj = 2 * t * C * D
    pos = 2 * t * D * (D // G) * K
    gemm = L * (2 * t * D * 3 * D + 2 * t * D * D + 2 * 2 * t * D * F)
    attn = L * 2 * 2 * t * t * D
    head = 2 * t * 8 * 128 * D + 3 * 2 * t * 8 * 128 * 256 + 4 * 2 * t * 8 * 128 * 128 + 2 * t * 128 * 256
    return {"conv": conv, "proj": proj, "pos_conv": pos, "layer_gemm": gemm, "attention": attn, "head": head,
            "total": conv + proj + pos + gemm + attn + head}


def card() -> dict:
    """name, power limit and maximum SM clock of device 0, read with nvidia-smi (read-only query)"""
    import subprocess
    r = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    if r.returncode != 0:
        return {"name": torch.cuda.get_device_name(0), "power_limit": "unknown"}
    name, power, clock = [x.strip() for x in r.stdout.strip().splitlines()[0].split(",")]
    return {"name": name, "power_limit": power, "sm_clock_max": clock}


def wavlm_stage_split(seg, win) -> dict:
    """Kernel time of one WavLM forward by stage, from torch.profiler's kernel list in launch order: conv extractor
    (through the feature projection) up to the first positional-conv im2col, positional conv up to the relative-bias
    table, the 12 layers up to the last layer sum, then the head.  Within the layers, attention and GEMM time."""
    from torch.profiler import ProfilerActivity, profile
    seg(win)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        seg(win)
        torch.cuda.synchronize()
    ks = sorted((e for e in prof.events() if e.device_type.name == "CUDA" and e.device_time_total > 0),
                key=lambda e: e.time_range.start)
    names = [e.name for e in ks]
    first = lambda key: next(i for i, n in enumerate(names) if key in n)
    last = lambda key: max(i for i, n in enumerate(names) if key in n)
    cuts = [0, first("im2col_pos_kernel"), first("rel_bias_kernel"), last("layer_sum_kernel") + 1, len(ks)]
    us = lambda a, b, f=lambda n: True: sum(e.device_time_total for e in ks[a:b] if f(e.name))
    out = {stage: us(cuts[i], cuts[i + 1]) / 1e3 for i, stage in enumerate(["conv_extractor", "pos_conv", "layers", "head"])}
    out["extractor_im2col"] = us(cuts[0], cuts[1], lambda n: "im2col_rows_kernel" in n) / 1e3
    out["layers_attention"] = us(cuts[2], cuts[3], lambda n: "attention_tc_kernel" in n) / 1e3
    out["layers_gemm"] = us(cuts[2], cuts[3], lambda n: "gemm_wg_kernel" in n) / 1e3
    return {k: round(v, 3) for k, v in out.items()}


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
    ap.add_argument("--segmentation", choices=["v1", "v2"], default="v1")
    args = ap.parse_args()
    v2 = args.segmentation == "v2"
    seg = (WavLMSegmentationModel(synth.wavlm_segmentation_state_dict(0)) if v2
           else SegmentationModel(synth.segmentation_state_dict(0)))
    emb = EmbeddingModel(synth.embedding_state_dict(0))
    B = args.batch
    win = torch.from_numpy(np.stack([synth.synthetic_speech(10.0, seed=i, turns=2) for i in range(8)])).cuda()
    win = win.repeat((B + 7) // 8, 1)[:B].contiguous()
    masks = (torch.rand(B, 3, seg.num_frames(160000), device="cuda") > 0.5).float()
    seg_ms = timed(lambda: seg(win))
    info = card()
    emb_ms = timed(lambda: emb(win, masks))
    # 1.3 GMAC (PyanNet) / 23.5 GMAC (ResNet34 trunk) per 10 s window
    seg_flops = wavlm_flops()["total"] if v2 else 1.3e9 * 2
    out = {"segmentation": args.segmentation, "batch_windows": B, "segmentation_ms": seg_ms, "embedding_ms": emb_ms,
           "segmentation_ms_per_window": seg_ms / B,
           "segmentation_windows_per_s": B / seg_ms * 1e3, "embedding_windows_per_s": B / emb_ms * 1e3,
           "segmentation_gflop_per_window": seg_flops / 1e9,
           "segmentation_tflops": B * seg_flops / seg_ms / 1e9, "embedding_tflops": B * 23.5e9 * 2 / emb_ms / 1e9,
           "card": info}
    if v2:
        # the pipeline hands the segmentation max(batch, 264) windows per call
        big = win.repeat((264 + B - 1) // B, 1)[:264].contiguous()
        big_ms = timed(lambda: seg(big), iters=3, warmup=1)
        split = wavlm_stage_split(seg, win)
        f = wavlm_flops()
        out.update({"segmentation_ms_per_window_264": big_ms / 264, "stage_ms_per_batch": split,
                    "layer_gemm_tflops": B * f["layer_gemm"] / split["layers_gemm"] / 1e9,
                    "attention_tflops": B * f["attention"] / split["layers_attention"] / 1e9,
                    "conv_extractor_tflops": B * (f["conv"] + f["proj"]) / split["conv_extractor"] / 1e9,
                    "pos_conv_tflops": B * f["pos_conv"] / split["pos_conv"] / 1e9})
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
