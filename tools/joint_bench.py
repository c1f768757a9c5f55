"""Joint ASR + diarization on one GPU (BASELINE.json config 5 without the 8-GPU sharding): a 45-minute synthetic
multi-speaker call, the benchmark-shaped synthetic ASR model, attention_rescoring on 30 s chunks in batches of 64, and
the synthetic diarization pipeline.  Prints one JSON line with

  * the wall time of each stage: ASR (CTM), segmentation, embedding, clustering, reconstruction, STM assembly, and of
    the one call transcribe(format="stm", diarization=...) that runs them all;
  * the centroid linkage of the same embeddings both ways, on the GPU (csrc/diar_cluster.cu) and scipy on the host,
    with Z asserted equal (or, where merge heights tie, the first difference asserted to be a tie and the clusters
    asserted equal), and n;
  * the card's name and power limit, and the SM clock sampled during the run.

    python tools/joint_bench.py [--seconds 2700] [--batch 64] > joint_bench.json
Synthetic weights and audio: the numbers are throughput only.  Everything it writes goes to a temporary directory.
"""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time
import wave

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bench import CHUNK_FRAMES, ClockSampler  # noqa: E402
from reverb_b200 import load_model, synth  # noqa: E402
from reverb_b200.diarization import synth as dsynth  # noqa: E402
from reverb_b200.diarization.infer import load_pipeline, read_audio  # noqa: E402
from reverb_b200.diarization.pipeline import centroid_linkage  # noqa: E402
from reverb_b200.diarization.words2speakers import rttm_text, stm_text  # noqa: E402


def write_wav(path, audio):
    with wave.open(path, "wb") as w:
        w.setnchannels(1)
        w.setsampwidth(2)
        w.setframerate(16000)
        w.writeframes((np.clip(audio, -1, 1) * 32767).astype(np.int16).tobytes())
    return path


def wall(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return out, time.perf_counter() - t0


def clustering_input(pipe):
    """the unit-normalised embeddings agglomerative_clustering links for the last call of `pipe`"""
    emb, binarized = pipe.last["embeddings"], pipe.last["binarized"]
    active = binarized.sum(axis=1) > 0.2 * binarized.shape[1]
    valid = ~np.any(np.isnan(emb), axis=2)
    train = emb[np.where(active & valid)].astype(np.float64)
    return train / np.linalg.norm(train, axis=-1, keepdims=True)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    name, limit = (x.strip() for x in q.stdout.strip().split(",")[:2]) if q.returncode == 0 else (None, None)
    return {"name": name or torch.cuda.get_device_name(0), "power_limit": limit}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=2700.0)
    ap.add_argument("--batch", type=int, default=64)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "joint_bench measures the GPU path; no CUDA device found"
    tmp = tempfile.mkdtemp(prefix="rvb_joint_")
    model_dir = synth.write_model_dir(os.path.join(tmp, "model"), shape=synth.BENCH_SHAPE, seed=0, causal=True,
                                      cnn_module_norm="layer_norm", reverse_weight=0.3)
    asr = load_model(model_dir)
    pipe = load_pipeline(synthetic=True, batch_size=args.batch)
    wav = write_wav(os.path.join(tmp, "call.wav"), dsynth.synthetic_speech(args.seconds, seed=11, turns=3))
    warm = write_wav(os.path.join(tmp, "warm.wav"), dsynth.synthetic_speech(90.0, seed=12, turns=3))
    kw = dict(mode="attention_rescoring", chunk_size=CHUNK_FRAMES, batch_size=args.batch)
    asr.transcribe(warm, format="stm", diarization=pipe, **kw)           # modules, allocations, algorithm choices
    centroid_linkage(clustering_input(pipe), "cuda")

    clocks = ClockSampler(0)
    clocks.start()
    ctm, t_asr = wall(lambda: asr.transcribe(wav, format="ctm", **kw))
    audio = read_audio(wav)
    turns, t_diar = wall(lambda: pipe(audio))
    stage = pipe.last["timing"]
    t0 = time.perf_counter()
    rttm = rttm_text("call", turns)
    stm = stm_text("call", rttm, ctm)
    t_stm = time.perf_counter() - t0
    one_call, t_joint = wall(lambda: asr.transcribe(wav, format="stm", diarization=pipe, **kw))
    assert one_call == stm
    x = clustering_input(pipe)
    gpu_times = []
    for _ in range(3):
        Z_gpu, t = wall(lambda: centroid_linkage(x, "cuda"))
        gpu_times.append(t)
    clk = clocks.stop()
    if clocks.proc is not None:
        clocks.proc.wait()
    from scipy.cluster.hierarchy import linkage
    t0 = time.perf_counter()
    Z_cpu = linkage(x, method="centroid", metric="euclidean")
    t_scipy = time.perf_counter() - t0
    z_equal = bool(np.array_equal(Z_gpu, Z_cpu))
    # Z is scipy's bit for bit unless two candidate merge heights tie, where scipy's heap may pick another pair; then
    # the first differing row must be a tie and the cut at the pipeline's threshold must be the same partition
    ties = {"duplicate_embeddings": int(x.shape[0] - np.unique(x, axis=0).shape[0])}
    if not z_equal:
        from scipy.cluster.hierarchy import fcluster
        r = int(np.argmax(np.any(Z_gpu != Z_cpu, axis=1)))
        ties.update(first_differing_row=r, heights=[float(Z_gpu[r, 2]), float(Z_cpu[r, 2])])
        assert Z_gpu[r, 2] == Z_cpu[r, 2], "GPU linkage differs from scipy at a merge that is not a tie"
        cut = [fcluster(Z, pipe.threshold, criterion="distance") for Z in (Z_gpu, Z_cpu)]
        same = {frozenset(np.nonzero(cut[0] == k)[0].tolist()) for k in np.unique(cut[0])} == \
            {frozenset(np.nonzero(cut[1] == k)[0].tolist()) for k in np.unique(cut[1])}
        assert same, "tie broken differently and the clusters differ"
    out = {
        "recording_seconds": args.seconds, "mode": "attention_rescoring", "chunk_frames": CHUNK_FRAMES,
        "batch": args.batch,
        "stages_seconds": {"asr": round(t_asr, 4), "segmentation": round(stage["segmentation"], 4),
                           "embedding": round(stage["embedding"], 4), "clustering": round(stage["clustering"], 4),
                           "reconstruction": round(stage["reconstruction"], 4), "stm_assembly": round(t_stm, 4)},
        "diarization_seconds": round(t_diar, 4), "joint_call_seconds": round(t_joint, 4),
        "joint_rtfx": round(args.seconds / t_joint, 1),
        "linkage": {"n": int(x.shape[0]), "gpu_seconds": [round(t, 4) for t in gpu_times],
                    "scipy_host_seconds": round(t_scipy, 4), "z_equal": z_equal, **ties},
        "turns": len(turns), "speakers": len({t.label for t in turns}), "stm_lines": stm.count("\n"),
        "gpu": card(), "clocks": clk, "host_cpu": os.cpu_count(),
        "data": "synthetic audio, synthetic weights",
    }
    shutil.rmtree(tmp, ignore_errors=True)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
