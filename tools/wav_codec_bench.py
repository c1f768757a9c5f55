"""G.711 and ADPCM WAV decoding on the GPU (csrc/wav_codec.cu): decode throughput, whole `load_audio` calls against
the PCM WAV of the same samples, and what codec input costs `transcribe_files` against PCM input.

    python tools/wav_codec_bench.py [--reps N] [--seconds S] [--out DIR]

Recordings: 1 h of 8 kHz mono synthetic speech (reverb_b200.synth) in each codec (µ-law, A-law, IMA ADPCM and MS
ADPCM at 256-byte blocks), and 1 h of 16 kHz stereo IMA ADPCM at 2048-byte blocks, encoded by oracle/wav_codec_ref.py.
Each PCM twin holds the codec's decoded samples, so both inputs must transcribe identically.  Decode times are CUDA
events around rvb_wav_decode on a data chunk already in device memory, after a warm-up decode.  `transcribe_files`
runs the benchmarked model shape (synthetic weights) over the codec corpus and its PCM twin, alternated in one
process.  The card's name and power limit are read in the same run.
"""
import argparse
import ctypes
import json
import os
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import wav_codec_ref as W  # noqa: E402
from reverb_b200 import _lib, synth  # noqa: E402
from reverb_b200.audio_io import load_audio  # noqa: E402
from tools.flac_bench import card  # noqa: E402

RECORDINGS = [  # name, codec, channels, rate, block_align
    ("ulaw8k", W.MULAW, 1, 8000, 1), ("alaw8k", W.ALAW, 1, 8000, 1), ("ima8k", W.IMA_ADPCM, 1, 8000, 256),
    ("ms8k", W.MS_ADPCM, 1, 8000, 256), ("ima16k_stereo", W.IMA_ADPCM, 2, 16000, 2048)]


def decode_on_device(lib, payload: bytes, tag: int, nch: int, ba: int, frames: int, reps: int):
    """ms per rvb_wav_decode (the data chunk already uploaded), median and min over `reps` after one warm-up"""
    spb = 1 if tag in (W.MULAW, W.ALAW) else (W.ima_spb(nch, ba) if tag == W.IMA_ADPCM else W.ms_spb(nch, ba))
    info = _lib.WavCodec(tag, nch, ba, spb, len(W.MS_COEFS) if tag == W.MS_ADPCM else 0)
    if tag == W.MS_ADPCM:
        for i, (c1, c2) in enumerate(W.MS_COEFS):
            info.coef[2 * i], info.coef[2 * i + 1] = c1, c2
    stream = torch.cuda.Stream()
    with torch.cuda.stream(stream):
        d = torch.frombuffer(bytearray(payload), dtype=torch.uint8).cuda()
        out = torch.empty((nch, frames), dtype=torch.int16, device="cuda")
        bad, st = ctypes.c_int(), ctypes.c_int()
        times = []
        for r in range(reps + 1):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            _lib.check(lib.rvb_wav_decode(d.data_ptr(), len(payload), ctypes.byref(info), frames, out.data_ptr(),
                                          ctypes.byref(bad), ctypes.byref(st), stream.cuda_stream), "rvb_wav_decode")
            e1.record(stream)
            e1.synchronize()
            assert bad.value == -1
            if r:
                times.append(e0.elapsed_time(e1))
    return float(np.median(times)), float(np.min(times))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--seconds", type=float, default=3600.0)
    ap.add_argument("--out", default=None, help="directory for wav_codec_bench.json (default: a temporary directory)")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "wav_codec_bench.py needs a CUDA device"
    args.out = args.out or tempfile.mkdtemp(prefix="wav_codec_bench_")
    os.makedirs(args.out, exist_ok=True)
    res = {"card": card()}
    print(json.dumps(res["card"]), flush=True)
    lib = _lib.load()
    tmp = tempfile.mkdtemp(prefix="wav_codec_bench_")
    t = time.time()
    audio = {(nch, rate): np.stack([synth.synth_audio(args.seconds, seed=10 + c, sample_rate=rate)
                                    for c in range(nch)]).astype(np.int64)
             for nch, rate in {(r[2], r[3]) for r in RECORDINGS}}
    recs = {}
    for name, tag, nch, rate, ba in RECORDINGS:
        x = audio[(nch, rate)]
        wav, payload = W.codec_wav(x, rate, tag, ba)
        dec = W.decode(payload, tag, nch, ba, x.shape[1])
        cp, pp = os.path.join(tmp, "codec", name + ".wav"), os.path.join(tmp, "pcm", name + ".wav")
        os.makedirs(os.path.dirname(cp), exist_ok=True)
        os.makedirs(os.path.dirname(pp), exist_ok=True)
        with open(cp, "wb") as f:
            f.write(wav)
        with open(pp, "wb") as f:
            f.write(W.write_wav(np.ascontiguousarray(dec.T).astype("<i2").tobytes(), 1, nch, rate, 2 * nch, 16))
        recs[name] = (cp, pp, payload, tag, nch, ba, dec)
    print(f"encoded in {time.time() - t:.1f} s", flush=True)
    for name, (cp, pp, payload, tag, nch, ba, dec) in recs.items():
        med, mn = decode_on_device(lib, payload, tag, nch, ba, dec.shape[1], args.reps)
        pcm, _ = load_audio(cp)
        assert np.array_equal(pcm, dec), name
        walls = {"codec": [], "pcm": []}
        for rep in range(3):
            for kind, p in (("codec", cp), ("pcm", pp)) if rep % 2 == 0 else (("pcm", pp), ("codec", cp)):
                t0 = time.perf_counter()
                load_audio(p)
                walls[kind].append(time.perf_counter() - t0)
        res[name] = {"bytes": len(payload), "frames": dec.shape[1], "decode_ms_median": round(med, 3),
                     "decode_ms_min": round(mn, 3), "audio_s_per_s": round(args.seconds / (med / 1000.0)),
                     "load_audio_codec_ms": round(1000 * float(np.median(walls["codec"])), 1),
                     "load_audio_pcm_ms": round(1000 * float(np.median(walls["pcm"])), 1)}
        print(name, json.dumps(res[name]), flush=True)
    # transcribe_files over the codec corpus and its PCM twin, alternated
    d = os.path.join(tmp, "model")
    synth.write_model_dir(d, shape=synth.BENCH_SHAPE, seed=0, causal=True, cnn_module_norm="layer_norm",
                          reverse_weight=0.3)
    import reverb_b200
    m = reverb_b200.load_model(d)
    kw = dict(format="txt", chunk_size=2998, batch_size=64)
    codecs, pcms = [r[0] for r in recs.values()], [r[1] for r in recs.values()]
    outs, walls = {}, {"codec": [], "pcm": []}
    for rep in range(3):
        for kind, files in (("codec", codecs), ("pcm", pcms)) if rep % 2 == 0 else (("pcm", pcms), ("codec", codecs)):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            got = [o for _, o in m.transcribe_files(files, ["attention_rescoring"], **kw)]
            torch.cuda.synchronize()
            if rep:                                                   # rep 0 warms both
                walls[kind].append(time.perf_counter() - t0)
            outs.setdefault(kind, got)
    assert outs["codec"] == outs["pcm"], "codec and PCM inputs transcribe differently"
    res["transcribe_files_s"] = {k: [round(v, 3) for v in vs] for k, vs in walls.items()}
    print("transcribe_files", json.dumps(res["transcribe_files_s"]), flush=True)
    with open(os.path.join(args.out, "wav_codec_bench.json"), "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
