"""Audio file reading with the contract of the reference's `torchaudio.load(audio_file, normalize=False)`
(asr/wenet/cli/reverb.py:122): a (channels, frames) array + the sample rate, where INTEGER PCM keeps its integer
sample values (the fbank front end works on int16-VALUED samples, cli/reverb.py:124, dataset/processor.py:361) and
everything else comes back as float32 in [-1, 1].

RIFF/WAVE is parsed here (PCM 8 / 16 / 24 / 32 bit, IEEE float 32 / 64, WAVE_FORMAT_EXTENSIBLE, any channel count) —
the stdlib `wave` module only does plain PCM.  Value conventions follow torchaudio: uint8 stays unsigned 0..255,
24-bit samples are left-justified in int32 (x << 8), 32-bit stay int32, float64 is narrowed to float32.

G.711 µ-law / A-law and IMA / Microsoft ADPCM WAV (format tags 0x0007, 0x0006, 0x0011, 0x0002; G.711 also inside
WAVE_FORMAT_EXTENSIBLE) are validated here and decoded on the GPU (csrc/wav_codec.cu, DESIGN.md §4l) to int16, what
torchaudio 2.2's FFmpeg backend returns for them with normalize=False.

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
WAVE_FORMAT_ADPCM, WAVE_FORMAT_ALAW, WAVE_FORMAT_MULAW, WAVE_FORMAT_IMA_ADPCM = 0x0002, 0x0006, 0x0007, 0x0011
# WAVE format tags decoded on the GPU (csrc/wav_codec.cu, DESIGN.md §4l) -> codec name used in error messages
WAV_CODECS = {WAVE_FORMAT_MULAW: "G.711 mu-law", WAVE_FORMAT_ALAW: "G.711 A-law", WAVE_FORMAT_IMA_ADPCM: "IMA ADPCM",
              WAVE_FORMAT_ADPCM: "MS ADPCM"}
# the seven coefficient pairs every MS ADPCM file starts its table with
MS_ADPCM_COEFS = ((256, 0), (512, -256), (0, 0), (192, 64), (240, 0), (460, -208), (392, -232))
# rvb_wav_decode's status codes (include/rvb_b200.h)
_WAV_CODEC_STATUS = {1: "IMA ADPCM step index above 88", 2: "MS ADPCM predictor index beyond the coefficient table"}


def _parse_riff_wave(data: bytes, path: str, device=None) -> Tuple[np.ndarray, int]:
    if len(data) < 12 or data[:4] != b"RIFF" or data[8:12] != b"WAVE":
        raise ValueError(f"{path}: not a RIFF/WAVE file")
    pos, fmt, pcm = 12, None, None
    fmt_body, data_off, fact = b"", 0, None
    while pos + 8 <= len(data):
        cid, size = data[pos:pos + 4], struct.unpack_from("<I", data, pos + 4)[0]
        body = data[pos + 8:pos + 8 + size]
        if cid == b"fmt ":
            if len(body) < 16:
                raise ValueError(f"{path}: truncated fmt chunk")
            tag, nch, rate, _brate, block, bits = struct.unpack_from("<HHIIHH", body, 0)
            if tag == WAVE_FORMAT_EXTENSIBLE and len(body) >= 40:
                tag = struct.unpack_from("<H", body, 24)[0]          # first two bytes of the SubFormat GUID
                if tag in (WAVE_FORMAT_ADPCM, WAVE_FORMAT_IMA_ADPCM):  # its extension is not the ADPCM one
                    raise ValueError(f"{path}: unsupported WAVE format tag 0x{tag:04x} inside WAVE_FORMAT_EXTENSIBLE")
            fmt = (tag, nch, rate, block, bits)
            fmt_body = body
        elif cid == b"data":
            pcm = body                                               # a streamed file may state size 0xFFFFFFFF: slice clips
            data_off = pos + 8
        elif cid == b"fact" and len(body) >= 4:
            fact = struct.unpack_from("<I", body, 0)[0]              # dwSampleLength: frames per channel
        pos += 8 + size + (size & 1)                                 # chunks are word aligned
    if fmt is None or pcm is None:
        raise ValueError(f"{path}: missing fmt or data chunk")
    tag, nch, rate, block, bits = fmt
    if nch < 1:
        raise ValueError(f"{path}: bad channel count {nch}")
    if tag in WAV_CODECS:
        return _decode_wav_codec(pcm, fmt, fmt_body, fact, data_off, path, device), int(rate)
    if tag not in (WAVE_FORMAT_PCM, WAVE_FORMAT_IEEE_FLOAT):
        raise ValueError(f"{path}: unsupported WAVE format tag 0x{tag:04x} (PCM, IEEE float, G.711 mu-law / A-law, "
                         "IMA ADPCM and MS ADPCM are decoded)")
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


@dataclass
class WavCodecInfo:
    """A validated compressed-WAV fmt chunk and the frame count its data chunk decodes to."""
    format_tag: int
    channels: int
    block_align: int
    samples_per_block: int                 # per channel, ADPCM; 1 for G.711
    coefs: List[Tuple[int, int]]           # MS ADPCM coefficient pairs
    frames: int                            # per channel


def parse_wav_codec(pcm: bytes, fmt, fmt_body: bytes, fact, data_off: int, path: str = "<bytes>") -> WavCodecInfo:
    """Validates the fmt chunk of a G.711 or ADPCM WAV and counts its frames: G.711 has one byte per sample; an ADPCM
    data chunk is full blocks then an optional partial block, and a `fact` chunk, when present, states the length.
    Every error is a ValueError naming the file, the format tag and the codec; nothing here touches the GPU."""
    tag, nch, _rate, block, bits = fmt
    codec = WAV_CODECS[tag]

    def bad(msg):
        return ValueError(f"{path}: format tag 0x{tag:04x} ({codec}): {msg}")
    cb = struct.unpack_from("<H", fmt_body, 16)[0] if len(fmt_body) >= 18 else 0
    if tag in (WAVE_FORMAT_MULAW, WAVE_FORMAT_ALAW):
        if bits != 8:
            raise bad(f"{bits} bits per sample (G.711 has 8)")
        if block != nch:
            raise bad(f"block_align {block} for {nch} channels (must equal the channel count)")
        return WavCodecInfo(tag, nch, block, 1, [], len(pcm) // nch)
    if bits != 4:
        raise bad(f"{bits} bits per sample (only 4-bit ADPCM is decoded)")
    if tag == WAVE_FORMAT_IMA_ADPCM:
        if cb < 2:
            raise bad(f"fmt extension of {cb} bytes (cbSize must be at least 2, for wSamplesPerBlock)")
        spb = struct.unpack_from("<H", fmt_body, 18)[0]
        if spb < 1 or (spb - 1) % 8:
            raise bad(f"{spb} samples per block (must be 1 + a multiple of 8)")
        if block != 4 * nch * (1 + (spb - 1) // 8):
            raise bad(f"block_align {block} does not hold {spb} samples of {nch} channels "
                      f"(expected {4 * nch * (1 + (spb - 1) // 8)})")
        hdr, coefs = 4 * nch, []
    else:
        if nch not in (1, 2):
            raise bad(f"{nch} channels (MS ADPCM has 1 or 2)")
        if cb < 32 or len(fmt_body) < 22:
            raise bad(f"fmt extension of {cb} bytes (cbSize must be at least 32, for the coefficient table)")
        spb, n_coef = struct.unpack_from("<HH", fmt_body, 18)
        if not 7 <= n_coef <= 256:
            raise bad(f"{n_coef} coefficient pairs (7 to 256 are valid)")
        if len(fmt_body) < 22 + 4 * n_coef or cb < 4 + 4 * n_coef:
            raise bad(f"fmt chunk too short for its {n_coef} coefficient pairs")
        coefs = [struct.unpack_from("<hh", fmt_body, 22 + 4 * i) for i in range(n_coef)]
        if tuple(coefs[:7]) != MS_ADPCM_COEFS:
            raise bad(f"the first seven coefficient pairs {coefs[:7]} are not the standard table")
        if block < 7 * nch or spb != 2 + (block - 7 * nch) * 2 // nch:
            raise bad(f"{spb} samples per block do not fit block_align {block} for {nch} channels")
        hdr = 7 * nch
    full, rem = divmod(len(pcm), block)
    part = 0
    if rem:
        if rem < hdr:
            raise bad(f"block {full} at byte {data_off + full * block}: truncated: {rem} bytes, its header needs {hdr}")
        part = 1 + 8 * ((rem - hdr) // hdr) if tag == WAVE_FORMAT_IMA_ADPCM else 2 + (rem - hdr) * 2 // nch
    frames = full * spb + part
    if fact is not None:
        if fact > frames:
            k = frames // spb
            raise bad(f"block {k} at byte {data_off + k * block}: missing: the data chunk holds {frames} samples per "
                      f"channel in {full + (1 if rem else 0)} blocks, the fact chunk states {fact}")
        frames = fact
    return WavCodecInfo(tag, nch, block, spb, coefs, frames)


def _decode_wav_codec(pcm: bytes, fmt, fmt_body: bytes, fact, data_off: int, path: str, device) -> np.ndarray:
    import torch

    from . import _lib
    wi = parse_wav_codec(pcm, fmt, fmt_body, fact, data_off, path)
    if wi.frames == 0:
        return np.zeros((wi.channels, 0), np.int16)
    if not torch.cuda.is_available():
        raise RuntimeError(f"{path}: {WAV_CODECS[wi.format_tag]} WAV is decoded on the GPU and no CUDA device is "
                           "available (reverb_b200 has no CPU fallback)")
    dev = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
    lib = _lib.load()
    info = _lib.WavCodec(wi.format_tag, wi.channels, wi.block_align, wi.samples_per_block, len(wi.coefs))
    for i, (c1, c2) in enumerate(wi.coefs):
        info.coef[2 * i], info.coef[2 * i + 1] = c1, c2
    bad_block, bad_status = ctypes.c_int(-1), ctypes.c_int(0)
    # a stream of its own, as for FLAC: the reader thread decodes while the caller's stream runs the model
    stream = torch.cuda.Stream(device=dev)
    with torch.cuda.device(dev), torch.cuda.stream(stream):
        d_bytes = torch.frombuffer(bytearray(pcm), dtype=torch.uint8).to(dev)
        out = torch.empty((wi.channels, wi.frames), dtype=torch.int16, device=dev)
        _lib.check(lib.rvb_wav_decode(d_bytes.data_ptr(), len(pcm), ctypes.byref(info), wi.frames, out.data_ptr(),
                                      ctypes.byref(bad_block), ctypes.byref(bad_status), stream.cuda_stream),
                   "rvb_wav_decode")
        if bad_block.value >= 0:
            k = bad_block.value
            raise ValueError(f"{path}: format tag 0x{wi.format_tag:04x} ({WAV_CODECS[wi.format_tag]}): block {k} at "
                             f"byte {data_off + k * wi.block_align}: "
                             f"{_WAV_CODEC_STATUS.get(bad_status.value, f'status {bad_status.value}')}")
        return out.cpu().numpy()


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
    device: the CUDA device FLAC frames and G.711 / ADPCM WAV data are decoded on (default: the current device); PCM
    and float WAV never touch the GPU."""
    with open(path, "rb") as f:
        head = f.read(12)
        if head[:4] == b"RIFF" and head[8:12] == b"WAVE":
            return _parse_riff_wave(head + f.read(), str(path), device)
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
