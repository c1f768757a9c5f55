"""FLAC on the host: the metadata parser (reverb_b200/audio_io.py) on the oracle encoder's output, its errors, and a
few frames assembled field by field from RFC 9639's tables with a bit writer of this file's own (the GPU decode of
these frames is checked in test_gpu_flac.py).  Nothing here needs a GPU."""
import ctypes
import struct

import numpy as np
import pytest

from oracle import flac_ref as F
from reverb_b200.audio_io import load_audio, parse_flac_metadata


# ------------------------------------------------------------------------------------------------ hand-built frames
class Bits:
    """MSB-first bit writer, independent of the oracle encoder."""

    def __init__(self):
        self.bits = []

    def put(self, value, n):
        self.bits += [(value >> (n - 1 - i)) & 1 for i in range(n)]

    def put_signed(self, value, n):
        self.put(value & ((1 << n) - 1), n)

    def put_rice(self, value, k):
        u = 2 * value if value >= 0 else -2 * value - 1
        self.put(0, u >> k)
        self.put(1, 1)
        self.put(u & ((1 << k) - 1), k)

    def align(self):
        self.put(0, -len(self.bits) % 8)

    def bytes(self):
        assert len(self.bits) % 8 == 0
        return bytes(int("".join(map(str, self.bits[i:i + 8])), 2) for i in range(0, len(self.bits), 8))


def _crc(data, poly, width):
    c, top, mask = 0, 1 << (width - 1), (1 << width) - 1
    for b in data:
        c ^= b << (width - 8)
        for _ in range(8):
            c = ((c << 1) ^ poly) & mask if c & top else (c << 1) & mask
    return c


def _frame(number, bs, chan_code, subframes):
    """Header (RFC 9639 §9.1): sync 0b11111111111110, reserved 0, fixed blocking; block size code 6 (8-bit value
    bs - 1 after the number); sample rate code 5 (16 kHz); bit depth code 4 (16 bits); frame number < 128 (one byte);
    CRC-8.  Then the subframes, zero padding to a byte, CRC-16."""
    h = Bits()
    h.put(0b11111111111110, 14), h.put(0, 1), h.put(0, 1)
    h.put(6, 4), h.put(5, 4), h.put(chan_code, 4), h.put(4, 3), h.put(0, 1)
    h.put(number, 8), h.put(bs - 1, 8)
    hb = h.bytes()
    body = Bits()
    body.bits = [int(c) for c in "".join(f"{b:08b}" for b in hb + bytes([_crc(hb, 0x07, 8)]))]
    for sf in subframes:
        sf(body)
    body.align()
    fb = body.bytes()
    return fb + _crc(fb, 0x8005, 16).to_bytes(2, "big")


def _sub_header(b, type_bits, wasted=0):
    b.put(0, 1), b.put(type_bits, 6)
    if wasted:
        b.put(1, 1), b.put(0, wasted - 1), b.put(1, 1)
    else:
        b.put(0, 1)


def _constant(v, bits=16):
    return lambda b: (_sub_header(b, 0b000000), b.put_signed(v, bits))


def _verbatim(xs, bits=16, wasted=0):
    def w(b):
        _sub_header(b, 0b000001, wasted)
        for x in xs:
            b.put_signed(x >> wasted, bits - wasted)           # the decoder shifts them back
    return w


def _rice_residual(b, k, res):
    b.put(0b00, 2), b.put(0, 4), b.put(k, 4)          # 4-bit parameters, partition order 0, parameter k
    for r in res:
        b.put_rice(r, k)


def _fixed2():
    def w(b):
        _sub_header(b, 0b001010)                         # FIXED, order 2
        b.put_signed(10, 16), b.put_signed(12, 16)
        _rice_residual(b, 0, [1, -1])
    return w


def _lpc1():
    def w(b):
        _sub_header(b, 0b100000)                         # LPC, order 1
        b.put_signed(100, 16)
        b.put(2, 4), b.put_signed(1, 5), b.put_signed(2, 3)   # precision 3, shift 1, coefficient 2
        _rice_residual(b, 2, [5, -3, 0])
    return w


def _streaminfo(nch, total, bs=4, bps=16, rate=16000):
    packed = (rate << 44) | ((nch - 1) << 41) | ((bps - 1) << 36) | total
    body = struct.pack(">HH", bs, bs) + bytes(6) + packed.to_bytes(8, "big") + bytes(16)
    return b"fLaC" + bytes([0x80]) + len(body).to_bytes(3, "big") + body


def hand_streams():
    """[(file bytes, expected (channels, n) samples as decoded values)]"""
    mono = [
        (_constant(-7), [-7, -7, -7, -7]),
        (_verbatim([1, -2, 300, -32768]), [1, -2, 300, -32768]),
        (_fixed2(), [10, 12, 15, 17]),                   # 2*12 - 10 + 1, 2*15 - 12 - 1
        (_lpc1(), [100, 105, 102, 102]),                 # (2 * prev) >> 1 + residual
        (_verbatim([4, -8, 12, 0], wasted=2), [4, -8, 12, 0]),
    ]
    a = _streaminfo(1, 20) + b"".join(_frame(i, 4, 0, [sf]) for i, (sf, _) in enumerate(mono))
    # mid/side (channel code 10): L = [10, -5], R = [3, -6] -> mid = (L + R) >> 1 = [6, -6], side = L - R = [7, 1]
    b = _streaminfo(2, 2, bs=2) + _frame(0, 2, 10, [_verbatim([6, -6]), _verbatim([7, 1], bits=17)])
    return [(a, np.array([sum((x for _, x in mono), [])])), (b, np.array([[10, -5], [3, -6]]))]


# ------------------------------------------------------------------------------------------------ tests
def _signal(nch, n, bps, seed=0):
    rng = np.random.default_rng(seed)
    x = np.cumsum(rng.normal(0, 2.0 ** (bps - 6), (nch, n)), 1)
    lim = 2 ** (bps - 1)
    return np.clip(np.round(x), -lim, lim - 1).astype(np.int64)


def test_streaminfo_fields_and_md5():
    x = _signal(3, 5000, 20)
    data = F.encode(x, 44100, 20, block_size=1152)
    si = parse_flac_metadata(data)
    assert (si.sample_rate, si.channels, si.bits_per_sample, si.total_samples) == (44100, 3, 20, 5000)
    assert (si.min_block_size, si.max_block_size) == (1152, 1152)
    assert si.md5 == F.md5_of(x, 20) and si.blocks == ["STREAMINFO"]
    assert data[si.audio_offset:si.audio_offset + 2] == b"\xff\xf8"


def test_every_metadata_block_type_is_skipped_and_id3v2_is_skipped():
    x = _signal(1, 3000, 16)
    blocks = [("PADDING", bytes(100)), ("APPLICATION", b"abcd" + bytes(7)), ("SEEKTABLE", F.seektable([(0, 0, 4096)])),
              ("VORBIS_COMMENT", F.vorbis_comment()), ("CUESHEET", bytes(396)), ("PICTURE", bytes(41)), (9, b"xy")]
    data = F.encode(x, 16000, 16, blocks=blocks, id3=F.id3v2())
    si = parse_flac_metadata(data)
    assert si.blocks == ["STREAMINFO", "PADDING", "APPLICATION", "SEEKTABLE", "VORBIS_COMMENT", "CUESHEET", "PICTURE",
                         "reserved 9"]
    assert data[:3] == b"ID3" and data[si.audio_offset:si.audio_offset + 2] == b"\xff\xf8"
    assert si.total_samples == 3000


def test_unknown_total_samples_and_libflac_layout():
    x = _signal(2, 9000, 16)
    si = parse_flac_metadata(F.encode(x, 16000, 16, total_samples=0))
    assert si.total_samples == 0
    si = parse_flac_metadata(F.encode_libflac(x, 16000, 16))
    assert si.blocks == ["STREAMINFO", "SEEKTABLE", "VORBIS_COMMENT", "PADDING"] and si.max_block_size == 4096


def test_hand_built_frames_parse_and_carry_their_own_crcs():
    (a, want_a), (b, want_b) = hand_streams()
    si = parse_flac_metadata(a)
    assert (si.channels, si.total_samples, si.audio_offset) == (1, 20, 42)
    # the oracle's table CRCs agree with this file's bitwise ones
    frame0 = _frame(0, 4, 0, [_constant(-7)])
    assert F.crc16(frame0[:-2]) == int.from_bytes(frame0[-2:], "big") and F.crc8(frame0[:6]) == frame0[6]
    assert want_a.shape == (1, 20) and want_b.shape == (2, 2)


def test_errors_name_the_file_and_mention_wav(tmp_path):
    p = tmp_path / "zero.flac"
    p.write_bytes(b"fLaC" + b"\x00" * 64)                      # a 0-byte STREAMINFO
    with pytest.raises(ValueError, match=r"zero\.flac.*STREAMINFO block is 0 bytes.*WAV"):
        load_audio(str(p))
    good = F.encode(_signal(1, 100, 16), 16000, 16)
    for name, data, msg in [("cut.flac", good[:30], "runs past the end"),
                            ("order.flac", good[:4] + bytes([0x01]) + good[5:], "STREAMINFO must be the first"),
                            ("b127.flac", good[:4] + bytes([0x7F]) + good[5:], "type 127")]:
        (tmp_path / name).write_bytes(data)
        with pytest.raises(ValueError, match=name.replace(".", r"\.") + ".*" + msg):
            load_audio(str(tmp_path / name))


def test_a_flac_file_without_a_gpu_is_a_runtime_error(tmp_path):
    import torch
    if torch.cuda.is_available():
        pytest.skip("a CUDA device is present")
    p = tmp_path / "ok.bin"                                      # detected by magic, not by extension
    p.write_bytes(F.encode(_signal(1, 100, 16), 16000, 16))
    with pytest.raises(RuntimeError, match="no CUDA device"):
        load_audio(str(p))


def test_ctypes_flac_info_mirrors_the_header(tmp_path):
    import subprocess
    from reverb_b200._lib import FlacInfo
    src = tmp_path / "s.c"
    src.write_text('#include "rvb_b200.h"\n#include <stdio.h>\n#include <stddef.h>\n'
                   'int main(void){printf("%zu %zu\\n", sizeof(rvb_flac_info), offsetof(rvb_flac_info, max_block_size));'
                   'return 0;}\n')
    import os
    inc = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include")
    exe = tmp_path / "s"
    r = subprocess.run(["cc", "-I", inc, str(src), "-o", str(exe)], capture_output=True, text=True)
    if r.returncode != 0:
        pytest.skip(f"no C compiler: {r.stderr[:200]}")
    size, off = map(int, subprocess.run([str(exe)], capture_output=True, text=True).stdout.split())
    assert size == ctypes.sizeof(FlacInfo) and off == FlacInfo.max_block_size.offset
