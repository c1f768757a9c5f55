"""FLAC decoding on the GPU (csrc/flac.cu): decode throughput, the per-pass split, and what FLAC input costs
`transcribe_files` against WAV input.

    python tools/flac_bench.py [--reps N] [--out DIR]

Recordings: 1 h of 16 kHz mono 16-bit and 1 h of 44.1 kHz stereo 16-bit synthetic speech (reverb_b200.synth), encoded
by the oracle's libFLAC-layout encoder (oracle/flac_ref.py).  Decode times are CUDA events around rvb_flac_index +
rvb_flac_decode on a file already in device memory, after a warm-up decode.  The per-pass split comes from a separate
torch.profiler run.  `transcribe_files` runs the benchmarked model shape (synthetic weights) over the same recordings as
WAV and as FLAC, alternated in one process.  The card's name and power limit are read in the same run.
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

from oracle import flac_ref  # noqa: E402
from reverb_b200 import _lib, synth  # noqa: E402
from reverb_b200.audio_io import load_audio, parse_flac_metadata  # noqa: E402


def card() -> dict:
    """name, power limit and maximum SM clock of device 0, read with nvidia-smi (read-only query)"""
    import subprocess
    r = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    if r.returncode != 0:
        return {"name": torch.cuda.get_device_name(0), "power_limit": "unknown"}
    name, power, clock = [x.strip() for x in r.stdout.strip().splitlines()[0].split(",")]
    return {"name": name, "power_limit": power, "sm_clock_max": clock}


def decode_on_device(lib, data: bytes, reps: int):
    """ms per decode (index + decode, the file already uploaded), median and min over `reps` after one warm-up"""
    si = parse_flac_metadata(data)
    info = _lib.FlacInfo(si.sample_rate, si.channels, si.bits_per_sample, si.max_block_size)
    stream = torch.cuda.Stream()
    with torch.cuda.stream(stream):
        d = torch.frombuffer(bytearray(data), dtype=torch.uint8).cuda()
        ws = torch.empty(lib.rvb_flac_index_workspace_bytes(len(data)), dtype=torch.uint8, device="cuda")
        nf, total = ctypes.c_int(), ctypes.c_longlong()
        bad, off, st = ctypes.c_int(), ctypes.c_longlong(), ctypes.c_int()
        out = dws = None
        times = []
        for r in range(reps + 1):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            _lib.check(lib.rvb_flac_index(d.data_ptr(), len(data), si.audio_offset, ctypes.byref(info), ws.data_ptr(),
                                          ws.numel(), ctypes.byref(nf), ctypes.byref(total), stream.cuda_stream),
                       "rvb_flac_index")
            if out is None:
                dws = torch.empty(lib.rvb_flac_decode_workspace_bytes(nf.value, total.value, ctypes.byref(info)),
                                  dtype=torch.uint8, device="cuda")
                out = torch.empty((si.channels, total.value), dtype=torch.int16, device="cuda")
            _lib.check(lib.rvb_flac_decode(d.data_ptr(), len(data), ctypes.byref(info), ws.data_ptr(), nf.value,
                                           total.value, dws.data_ptr(), dws.numel(), out.data_ptr(), ctypes.byref(bad),
                                           ctypes.byref(off), ctypes.byref(st), stream.cuda_stream), "rvb_flac_decode")
            e1.record(stream)
            e1.synchronize()
            assert bad.value == -1
            if r:
                times.append(e0.elapsed_time(e1))
    return float(np.median(times)), float(np.min(times)), nf.value, total.value


def pass_split(lib, data: bytes):
    from torch.profiler import ProfilerActivity, profile
    decode_on_device(lib, data, 1)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        decode_on_device(lib, data, 2)
    rows = {}
    for ev in prof.key_averages():
        if "flac" in ev.key:
            name = ev.key.split("(")[0].split("<")[0].split("::")[-1]
            t = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0)
            rows[name] = rows.get(name, 0.0) + t / 1000.0 / 3          # ms per decode (warm-up + 2 timed)
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--seconds", type=float, default=3600.0)
    ap.add_argument("--out", default=None, help="directory for flac_bench.json (default: a temporary directory)")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "flac_bench.py needs a CUDA device"
    args.out = args.out or tempfile.mkdtemp(prefix="flac_bench_")
    os.makedirs(args.out, exist_ok=True)
    res = {"card": card()}
    print(json.dumps(res["card"]), flush=True)
    lib = _lib.load()
    tmp = tempfile.mkdtemp(prefix="flac_bench_")
    recs = {}
    t = time.time()
    mono = synth.synth_audio(args.seconds, seed=1).astype(np.int64)[None]
    st = np.stack([synth.synth_audio(args.seconds, seed=2, sample_rate=44100),
                   synth.synth_audio(args.seconds, seed=3, sample_rate=44100)]).astype(np.int64)
    for name, x, rate in (("mono16k", mono, 16000), ("stereo44k", st, 44100)):
        data = flac_ref.encode_libflac(x, rate, 16)
        fp, wp = os.path.join(tmp, name + ".flac"), os.path.join(tmp, name + ".wav")
        with open(fp, "wb") as f:
            f.write(data)
        import wave
        with wave.open(wp, "wb") as w:
            w.setnchannels(x.shape[0]), w.setsampwidth(2), w.setframerate(rate)
            w.writeframes(np.ascontiguousarray(x.T).astype("<i2").tobytes())
        recs[name] = (wp, fp, data, x)
    print(f"encoded in {time.time() - t:.1f} s", flush=True)
    for name, (wp, fp, data, x) in recs.items():
        med, mn, nf, total = decode_on_device(lib, data, args.reps)
        pcm, _ = load_audio(fp)
        assert np.array_equal(pcm, x.astype(np.int16))
        t0 = time.perf_counter()
        load_audio(fp)
        t_flac = time.perf_counter() - t0
        t0 = time.perf_counter()
        load_audio(wp)
        t_wav = time.perf_counter() - t0
        res[name] = {"bytes": len(data), "frames": nf, "samples": total, "decode_ms_median": round(med, 3),
                     "decode_ms_min": round(mn, 3), "audio_s_per_s": round(args.seconds / (med / 1000.0)),
                     "load_audio_flac_ms": round(t_flac * 1000, 1), "load_audio_wav_ms": round(t_wav * 1000, 1),
                     "passes_ms": {k: round(v, 3) for k, v in pass_split(lib, data).items()}}
        print(name, json.dumps(res[name]), flush=True)
    # transcribe_files over the same recordings as WAV and as FLAC, alternated
    d = os.path.join(tmp, "model")
    synth.write_model_dir(d, shape=synth.BENCH_SHAPE, seed=0, causal=True, cnn_module_norm="layer_norm",
                          reverse_weight=0.3)
    import reverb_b200
    m = reverb_b200.load_model(d)
    kw = dict(format="txt", chunk_size=2998, batch_size=64)
    wavs, flacs = [r[0] for r in recs.values()], [r[1] for r in recs.values()]
    outs, walls = {}, {"wav": [], "flac": []}
    for rep in range(4):
        for kind, files in (("wav", wavs), ("flac", flacs)) if rep % 2 == 0 else (("flac", flacs), ("wav", wavs)):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            got = [o for _, o in m.transcribe_files(files, ["attention_rescoring"], **kw)]
            torch.cuda.synchronize()
            if rep:                                                   # rep 0 warms both
                walls[kind].append(time.perf_counter() - t0)
            outs.setdefault(kind, got)
    assert outs["wav"] == outs["flac"], "FLAC and WAV inputs transcribe differently"
    res["transcribe_files_s"] = {k: [round(v, 3) for v in vs] for k, vs in walls.items()}
    print("transcribe_files", json.dumps(res["transcribe_files_s"]), flush=True)
    with open(os.path.join(args.out, "flac_bench.json"), "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
