"""Audio file reading with the contract of the reference's `torchaudio.load(audio_file, normalize=False)`
(asr/wenet/cli/reverb.py:122): a (channels, frames) array + the sample rate, where INTEGER PCM keeps its integer
sample values (the fbank front end works on int16-VALUED samples, cli/reverb.py:124, dataset/processor.py:361) and
everything else comes back as float32 in [-1, 1].

RIFF/WAVE is parsed here (PCM 8 / 16 / 24 / 32 bit, IEEE float 32 / 64, WAVE_FORMAT_EXTENSIBLE, any channel count) —
the stdlib `wave` module only does plain PCM.  Value conventions follow torchaudio: uint8 stays unsigned 0..255,
24-bit samples are left-justified in int32 (x << 8), 32-bit stay int32, float64 is narrowed to float32.

FLAC (detected by its `fLaC` magic, optionally behind an ID3v2 tag, whatever the file is called) is decoded natively:
the metadata blocks are parsed here on the host and the frames are decoded on the GPU (csrc/flac.cu, DESIGN.md §4k).
Samples come back as integers, left-justified like the WAV path's: int16 (x << (16 - bps)) for up to 16 bits per
sample, int32 (x << (32 - bps)) for 17 to 32.  This is a deliberate choice of contract: it is what torchaudio 2.2, the
version the reference pins, returns with normalize=False through its default FFmpeg backend, and it is the scale the
model's front end expects.  Backends that return float in [-1, 1] for FLAC (TorchCodec, sox, soundfile) would shift
every log-mel bin by about 2 ln 32768.  A corrupt frame is an error that names the frame and its byte offset; nothing
is concealed or skipped.

Any other container (mp3, ogg, ...) is handed to torchaudio itself when it has a working decoder backend
(torchcodec / ffmpeg), which is exactly what the reference relies on; without one a clear error is raised.
"""
from __future__ import annotations

import ctypes
import struct
from dataclasses import dataclass, field
from typing import List, Tuple

import numpy as np

WAVE_FORMAT_PCM, WAVE_FORMAT_IEEE_FLOAT, WAVE_FORMAT_EXTENSIBLE = 0x0001, 0x0003, 0xFFFE


def _parse_riff_wave(data: bytes, path: str) -> Tuple[np.ndarray, int]:
    if len(data) < 12 or data[:4] != b"RIFF" or data[8:12] != b"WAVE":
        raise ValueError(f"{path}: not a RIFF/WAVE file")
    pos, fmt, pcm = 12, None, None
    while pos + 8 <= len(data):
        cid, size = data[pos:pos + 4], struct.unpack_from("<I", data, pos + 4)[0]
        body = data[pos + 8:pos + 8 + size]
        if cid == b"fmt ":
            if len(body) < 16:
                raise ValueError(f"{path}: truncated fmt chunk")
            tag, nch, rate, _brate, block, bits = struct.unpack_from("<HHIIHH", body, 0)
            if tag == WAVE_FORMAT_EXTENSIBLE and len(body) >= 40:
                tag = struct.unpack_from("<H", body, 24)[0]          # first two bytes of the SubFormat GUID
            fmt = (tag, nch, rate, block, bits)
        elif cid == b"data":
            pcm = body                                               # a streamed file may state size 0xFFFFFFFF: slice clips
        pos += 8 + size + (size & 1)                                 # chunks are word aligned
    if fmt is None or pcm is None:
        raise ValueError(f"{path}: missing fmt or data chunk")
    tag, nch, rate, block, bits = fmt
    if nch < 1:
        raise ValueError(f"{path}: bad channel count {nch}")
    if tag not in (WAVE_FORMAT_PCM, WAVE_FORMAT_IEEE_FLOAT):
        raise ValueError(f"{path}: unsupported WAVE format tag 0x{tag:04x} (only PCM and IEEE float)")
    if bits % 8 != 0 or bits == 0:
        raise ValueError(f"{path}: unsupported sample width {bits}")
    width = bits // 8
    nfr = len(pcm) // (width * nch)
    raw = pcm[:nfr * width * nch]
    if tag == WAVE_FORMAT_PCM:
        if bits == 8:
            x = np.frombuffer(raw, dtype=np.uint8)
        elif bits == 16:
            x = np.frombuffer(raw, dtype="<i2")
        elif bits == 24:
            b = np.frombuffer(raw, dtype=np.uint8).reshape(-1, 3).astype(np.int32)
            x = (b[:, 0] << 8) | (b[:, 1] << 16) | (b[:, 2] << 24)   # left-justified in int32, like torchaudio / libsndfile
            x = x.astype(np.int32)
        elif bits == 32:
            x = np.frombuffer(raw, dtype="<i4")
        else:
            raise ValueError(f"{path}: unsupported PCM width {bits}")
    else:
        if bits == 32:
            x = np.frombuffer(raw, dtype="<f4")
        elif bits == 64:
            x = np.frombuffer(raw, dtype="<f8").astype(np.float32)
        else:
            raise ValueError(f"{path}: unsupported float width {bits}")
    return np.ascontiguousarray(x.reshape(nfr, nch).T), int(rate)


FLAC_BLOCK_TYPES = {0: "STREAMINFO", 1: "PADDING", 2: "APPLICATION", 3: "SEEKTABLE", 4: "VORBIS_COMMENT", 5: "CUESHEET",
                    6: "PICTURE"}
# rvb_flac_decode's status codes (include/rvb_b200.h)
_FLAC_STATUS = {1: "invalid frame header (syntax or CRC-8)", 2: "frame header disagrees with STREAMINFO",
                3: "invalid subframe", 4: "invalid residual coding", 5: "frame data truncated", 6: "CRC-16 mismatch",
                7: "no valid frame header where the frame ends"}


@dataclass
class FlacStreamInfo:
    """STREAMINFO of a FLAC file, where its frames begin, and the types of its metadata blocks in file order."""
    sample_rate: int
    channels: int
    bits_per_sample: int
    min_block_size: int
    max_block_size: int
    total_samples: int                     # per channel; 0 = unknown
    md5: bytes
    audio_offset: int                      # first byte of the first frame
    blocks: List[str] = field(default_factory=list)


def _id3v2_size(head: bytes) -> int:
    """Bytes an ID3v2 tag at the start of the file takes (0 when there is none)."""
    if len(head) < 10 or head[:3] != b"ID3" or any(b & 0x80 for b in head[6:10]):
        return 0
    size = (head[6] << 21) | (head[7] << 14) | (head[8] << 7) | head[9]          # syncsafe
    return 10 + size + (10 if head[5] & 0x10 else 0)                             # footer flag


def parse_flac_metadata(data: bytes, path: str = "<bytes>") -> FlacStreamInfo:
    """Parses the `fLaC` marker (after an optional ID3v2 tag) and the metadata blocks (RFC 9639 §8).  STREAMINFO must
    come first; PADDING, APPLICATION, SEEKTABLE, VORBIS_COMMENT, CUESHEET, PICTURE and reserved types are skipped."""
    def bad(msg):
        return ValueError(f"{path}: malformed FLAC: {msg} (only RIFF/WAVE and FLAC are decoded natively)")
    pos = _id3v2_size(data[:10])
    if data[pos:pos + 4] != b"fLaC":
        raise bad("no fLaC marker")
    pos += 4
    info, blocks, last = None, [], False
    while not last:
        if pos + 4 > len(data):
            raise bad(f"metadata block header at byte {pos} runs past the end of the file")
        hdr = data[pos]
        last, btype, size = bool(hdr & 0x80), hdr & 0x7F, int.from_bytes(data[pos + 1:pos + 4], "big")
        body = data[pos + 4:pos + 4 + size]
        if len(body) < size:
            raise bad(f"{FLAC_BLOCK_TYPES.get(btype, 'metadata')} block at byte {pos} runs past the end of the file")
        if btype == 127:
            raise bad(f"invalid metadata block type 127 at byte {pos}")
        if (btype == 0) != (info is None):
            raise bad(f"STREAMINFO must be the first metadata block and appear once (block at byte {pos})")
        if btype == 0:
            if size != 34:
                raise bad(f"STREAMINFO block is {size} bytes, expected 34")
            min_bs, max_bs = struct.unpack_from(">HH", body, 0)
            packed = int.from_bytes(body[10:18], "big")
            rate, nch, bps = packed >> 44, ((packed >> 41) & 7) + 1, ((packed >> 36) & 31) + 1
            total = packed & ((1 << 36) - 1)
            if rate == 0:
                raise bad("STREAMINFO sample rate is 0")
            if bps < 4:
                raise bad(f"STREAMINFO states {bps} bits per sample (4 to 32 are valid)")
            info = FlacStreamInfo(rate, nch, bps, min_bs, max_bs, total, bytes(body[18:34]), 0)
        blocks.append(FLAC_BLOCK_TYPES.get(btype, f"reserved {btype}"))
        pos += 4 + size
    info.audio_offset = pos
    info.blocks = blocks
    return info


def _decode_flac(data: bytes, path: str, device) -> Tuple[np.ndarray, int]:
    import torch

    from . import _lib
    si = parse_flac_metadata(data, path)
    if not torch.cuda.is_available():
        raise RuntimeError(f"{path}: FLAC frames are decoded on the GPU and no CUDA device is available "
                           "(reverb_b200 has no CPU fallback)")
    dev = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
    lib = _lib.load()
    info = _lib.FlacInfo(si.sample_rate, si.channels, si.bits_per_sample, si.max_block_size)
    n = len(data)
    n_frames, total = ctypes.c_int(0), ctypes.c_longlong(0)
    # a stream of its own (torch's pool streams are non-blocking): the reader thread decodes while the caller's
    # stream runs the model, and nothing here may serialise with the legacy default stream
    stream = torch.cuda.Stream(device=dev)
    with torch.cuda.device(dev), torch.cuda.stream(stream):
        d_bytes = torch.frombuffer(bytearray(data), dtype=torch.uint8).to(dev)
        ws = torch.empty(lib.rvb_flac_index_workspace_bytes(n), dtype=torch.uint8, device=dev)
        _lib.check(lib.rvb_flac_index(d_bytes.data_ptr(), n, si.audio_offset, ctypes.byref(info), ws.data_ptr(),
                                      ws.numel(), ctypes.byref(n_frames), ctypes.byref(total), stream.cuda_stream),
                   "rvb_flac_index")
        nf, total = n_frames.value, total.value
        if nf < 0:
            raise ValueError(f"{path}: not a FLAC stream: more frame sync patterns than its size allows")
        if nf == 0:
            raise ValueError(f"{path}: frame 0 at byte {si.audio_offset}: no valid frame header after the metadata")
        if si.total_samples and total != si.total_samples:
            if total < si.total_samples:
                raise ValueError(f"{path}: frame {nf} at byte {n}: missing: the stream ends after {nf} frames holding "
                                 f"{total} samples, STREAMINFO states {si.total_samples}")
            raise ValueError(f"{path}: its {nf} frames hold {total} samples, STREAMINFO states {si.total_samples}")
        dws = torch.empty(lib.rvb_flac_decode_workspace_bytes(nf, total, ctypes.byref(info)), dtype=torch.uint8,
                          device=dev)
        out = torch.empty((si.channels, total), dtype=torch.int16 if si.bits_per_sample <= 16 else torch.int32,
                          device=dev)
        bad_frame, bad_off, bad_status = ctypes.c_int(-1), ctypes.c_longlong(-1), ctypes.c_int(0)
        _lib.check(lib.rvb_flac_decode(d_bytes.data_ptr(), n, ctypes.byref(info), ws.data_ptr(), nf, total,
                                       dws.data_ptr(), dws.numel(), out.data_ptr(), ctypes.byref(bad_frame),
                                       ctypes.byref(bad_off), ctypes.byref(bad_status), stream.cuda_stream),
                   "rvb_flac_decode")
        if bad_frame.value >= 0:
            raise ValueError(f"{path}: frame {bad_frame.value} at byte {bad_off.value}: "
                             f"{_FLAC_STATUS.get(bad_status.value, f'status {bad_status.value}')}")
        pcm = out.cpu().numpy()
    return pcm, si.sample_rate


def load_audio(path: str, device=None) -> Tuple[np.ndarray, int]:
    """(channels, frames) samples + sample rate, `torchaudio.load(path, normalize=False)` semantics.
    device: the CUDA device FLAC frames are decoded on (default: the current device); WAV never touches the GPU."""
    with open(path, "rb") as f:
        head = f.read(12)
        if head[:4] == b"RIFF" and head[8:12] == b"WAVE":
            return _parse_riff_wave(head + f.read(), str(path))
        skip = _id3v2_size(head[:10])
        if skip:
            f.seek(skip)
        if (f.read(4) if skip else head[:4]) == b"fLaC":
            f.seek(0)
            return _decode_flac(f.read(), str(path), device)
    try:                                       # any other container: the reference's own route, if a backend exists here
        import torchaudio
        wav, rate = torchaudio.load(str(path), normalize=False)
        return np.ascontiguousarray(wav.numpy()), int(rate)
    except Exception as e:
        raise ValueError(f"{path}: only RIFF/WAVE and FLAC are decoded natively and torchaudio has no working decoder "
                         f"backend here for this file ({type(e).__name__}: {e}); convert it to WAV "
                         "(e.g. `ffmpeg -i in out.wav`)") from e
