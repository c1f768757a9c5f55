"""Corpus throughput: a per-file loop with padded tails (one recording per call: decode_stream over feats_batcher,
what `transcribe_modes` did before corpus batching) against `transcribe_files` (chunks of many recordings per batch,
trimmed tails), on seeded synthetic corpora at the benchmarked model shape, chunk_size 2998, batch_size 64,
attention_rescoring.

    python tools/corpus_bench.py [--reps 2] [--scale 1.0] [--corpora short long mixed]

Corpora (synth.synth_audio, 16 kHz int16 WAV in a temporary directory):
    short: 1 024 clips of 2-20 s, log-uniform;   long: 32 recordings of 1-20 min;   mixed: half of each, shuffled.
Prints card name, power limit and max SM clock, then per corpus: audio seconds per wall second of both paths
(alternated, a device synchronise inside every timing), encoder rows computed per valid encoder row (from shapes),
and asserts that every file's output is identical.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import tempfile
import time
from itertools import chain
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from reverb_b200 import corpus, synth  # noqa: E402

CHUNK, BATCH, MODES = 2998, 64, ["attention_rescoring"]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else f"nvidia-smi failed: {q.stderr.strip()}"


def make_corpora(root: Path, scale: float):
    rng = np.random.default_rng(0)
    n_short, n_long = max(1, int(1024 * scale)), max(1, int(32 * scale))
    short_s = np.exp(rng.uniform(np.log(2.0), np.log(20.0), n_short))
    long_s = rng.uniform(60.0, 1200.0, n_long)

    def write(name, secs, seed0):
        d = root / name
        d.mkdir()
        return [synth.write_wav(str(d / f"{name}_{i:04d}.wav"), synth.synth_audio(float(s), seed=seed0 + i))
                for i, s in enumerate(secs)]

    short = write("short", short_s, 1000)
    long = write("long", long_s, 5000)
    mixed = short[: n_short // 2] + long[: max(1, n_long // 2)]
    mixed = [mixed[i] for i in np.random.default_rng(1).permutation(len(mixed))]
    return {"short": short, "long": long, "mixed": mixed}


def per_file(m, files):
    """The padded one-recording-per-call path."""
    from reverb_b200.reverb import get_output
    cat = torch.tensor([1.0, 0.0])
    kw = dict(ctc_weight=0.1, blank_id=m.blank_id, infos={"tasks": ["transcribe"], "langs": ["en"]}, cat_embs=cat)
    out = {}
    for f in files:
        feats = m.compute_feats(f, num_mel_bins=80, frame_length=25, frame_shift=10)
        res = list(m.model.decode_stream(m.feats_batcher(feats, CHUNK, BATCH), MODES, 10, **kw))
        out[f] = [get_output("ctm", m.tokenizer, Path(f).name, list(chain(*(r[mode] for r in res))), 230, CHUNK,
                             m.input_frame_length, m.output_frame_length) for mode in MODES]
    return out


def batched(m, files):
    return dict(m.transcribe_files(files, MODES, format="ctm", chunk_size=CHUNK, batch_size=BATCH))


def rows(frames, right):
    """(rows computed per-file, rows computed by transcribe_files, valid rows), encoder rows from shapes."""
    t_ref = corpus.encoder_out_frames(CHUNK)
    old = new = valid = 0
    packer, windows = corpus.WindowPacker(corpus.window_frames(BATCH, CHUNK)), []
    for n in frames:
        lens = corpus.chunk_lengths(n, CHUNK)
        valid += sum(corpus.encoder_out_len(fl, CHUNK) for fl in lens)
        for i in range(0, len(lens), BATCH):
            old += len(lens[i:i + BATCH]) * t_ref
        w = packer.add(n, n)
        if w:
            windows.append(w)
    windows.append(packer.flush())
    for w in windows:
        for b in corpus.plan_window(w, CHUNK, BATCH, right):
            new += len(b.slots) * corpus.encoder_out_frames(b.T)
    return old, new, valid


def timed(fn, *a):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    r = fn(*a)
    torch.cuda.synchronize()
    return time.perf_counter() - t0, r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=2, help="alternated timings of each path per corpus")
    ap.add_argument("--scale", type=float, default=1.0, help="corpus size factor (1.0 = the sizes above)")
    ap.add_argument("--corpora", nargs="+", default=["short", "long", "mixed"])
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("corpus_bench needs a CUDA device")
    import reverb_b200
    print(f"card: {card()}", flush=True)
    with tempfile.TemporaryDirectory(prefix="rvb_corpus_") as tmp:
        root = Path(tmp)
        mdir = root / "model"
        synth.write_model_dir(str(mdir), shape=synth.BENCH_SHAPE, seed=0, causal=True, cnn_module_norm="layer_norm",
                              reverse_weight=0.3)
        m = reverb_b200.load_model(str(mdir))
        t0 = time.perf_counter()
        corpora = make_corpora(root, args.scale)
        print(f"corpora written in {time.perf_counter() - t0:.1f} s", flush=True)
        right = corpus.right_context(m.configs["encoder_conf"])
        warm = corpora["short"][:8] + corpora["long"][:1]
        per_file(m, warm)
        batched(m, warm)
        results = {}
        for name in args.corpora:
            files = corpora[name]
            # 16-bit mono WAV with a 44-byte header
            frames = [int(m.engine.lib.rvb_fbank_num_frames((os.path.getsize(f) - 44) // 2)) for f in files]
            audio_s = sum((os.path.getsize(f) - 44) / 2 / 16000 for f in files)
            t_old, t_new = [], []
            out_old = out_new = None
            for _ in range(args.reps):
                dt, out_old = timed(per_file, m, files)
                t_old.append(dt)
                dt, out_new = timed(batched, m, files)
                t_new.append(dt)
            assert out_old == out_new, f"{name}: transcribe_files output differs from the per-file path"
            old_rows, new_rows, valid = rows(frames, right)
            r = {"files": len(files), "audio_s": round(audio_s, 1),
                 "per_file_xrt": [round(audio_s / t, 1) for t in t_old],
                 "transcribe_files_xrt": [round(audio_s / t, 1) for t in t_new],
                 "per_file_rows_per_valid_row": round(old_rows / valid, 3),
                 "transcribe_files_rows_per_valid_row": round(new_rows / valid, 3),
                 "outputs_identical": True}
            results[name] = r
            print(json.dumps({name: r}), flush=True)
        print(json.dumps({"card": card(), "chunk_size": CHUNK, "batch_size": BATCH, "modes": MODES,
                          "results": results}))


if __name__ == "__main__":
    main()
