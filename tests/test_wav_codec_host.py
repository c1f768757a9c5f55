"""Compressed WAV on the host: fmt validation and frame counting (reverb_b200/audio_io.py) with every rejection raised
before any CUDA call; the oracle's G.711 tables and IMA decoder against CPython's `audioop`; the oracle's MS ADPCM
decoder against hand-worked blocks (the GPU decode of these blocks is checked in test_gpu_wav_codec.py).  Nothing here
needs a GPU."""
import struct
import warnings

import numpy as np
import pytest

from oracle import wav_codec_ref as W
from reverb_b200 import _lib
from reverb_b200.audio_io import load_audio

with warnings.catch_warnings():
    warnings.simplefilter("ignore", DeprecationWarning)      # audioop is deprecated in 3.12 and gone in 3.13
    audioop = pytest.importorskip("audioop")


@pytest.fixture
def no_cuda(monkeypatch):
    """fails the test if the decode reaches the native library"""
    def refuse(*a, **k):
        raise AssertionError("a rejected file reached the CUDA library")
    monkeypatch.setattr(_lib, "load", refuse)


def _rejects(tmp_path, name, data, tag, codec, match):
    p = tmp_path / name
    p.write_bytes(data)
    with pytest.raises(ValueError, match=rf"{name}: format tag 0x{tag:04x} \({codec}\): .*{match}"):
        load_audio(str(p))


def _ima(nch=1, ba=256, n=1000, **kw):
    x = np.zeros((nch, n), np.int64)
    return W.ima_encode(x, ba, **kw)


def _ms(nch=1, ba=256, n=1000, **kw):
    x = np.zeros((nch, n), np.int64)
    return W.ms_encode(x, ba, **kw)


def _ms_ext(spb, coefs, n_coef=None):
    return struct.pack("<HH", spb, len(coefs) if n_coef is None else n_coef) + \
        b"".join(struct.pack("<hh", *c) for c in coefs)


REJECTIONS = {
    # name: (data, tag, codec, message fragment)
    "ulaw16": (W.write_wav(b"\0" * 64, W.MULAW, 1, 8000, 2, 16), W.MULAW, "G.711 mu-law", "16 bits per sample"),
    "alaw_block": (W.write_wav(b"\0" * 64, W.ALAW, 2, 8000, 1, 8), W.ALAW, "G.711 A-law", "block_align 1 for 2 channels"),
    "ima3bit": (W.write_wav(_ima(), W.IMA_ADPCM, 1, 8000, 256, 3, W.fmt_ext(W.IMA_ADPCM, 1, 256)), W.IMA_ADPCM,
                "IMA ADPCM", "3 bits per sample"),
    "ima_cbsize": (W.write_wav(_ima(), W.IMA_ADPCM, 1, 8000, 256, 4, b""), W.IMA_ADPCM, "IMA ADPCM", "cbSize"),
    "ima_spb": (W.write_wav(_ima(), W.IMA_ADPCM, 1, 8000, 256, 4, struct.pack("<H", 504)), W.IMA_ADPCM, "IMA ADPCM",
                "504 samples per block"),
    "ima_block": (W.write_wav(_ima(), W.IMA_ADPCM, 1, 8000, 260, 4, struct.pack("<H", 505)), W.IMA_ADPCM,
                  "IMA ADPCM", "block_align 260 does not hold 505 samples"),
    "ms3bit": (W.write_wav(_ms(), W.MS_ADPCM, 1, 8000, 256, 3, W.fmt_ext(W.MS_ADPCM, 1, 256)), W.MS_ADPCM, "MS ADPCM",
               "3 bits per sample"),
    "ms3ch": (W.write_wav(b"\0" * 768, W.MS_ADPCM, 3, 8000, 256, 4, W.fmt_ext(W.MS_ADPCM, 3, 256)), W.MS_ADPCM,
              "MS ADPCM", "3 channels"),
    "ms_cbsize": (W.write_wav(_ms(), W.MS_ADPCM, 1, 8000, 256, 4, _ms_ext(500, W.MS_COEFS)[:30]), W.MS_ADPCM,
                  "MS ADPCM", "cbSize must be at least 32"),
    "ms_ncoef6": (W.write_wav(_ms(), W.MS_ADPCM, 1, 8000, 256, 4, _ms_ext(500, W.MS_COEFS, 6)), W.MS_ADPCM, "MS ADPCM",
                  "6 coefficient pairs"),
    "ms_ncoef257": (W.write_wav(_ms(), W.MS_ADPCM, 1, 8000, 256, 4, _ms_ext(500, W.MS_COEFS, 257)), W.MS_ADPCM,
                    "MS ADPCM", "257 coefficient pairs"),
    "ms_short_table": (W.write_wav(_ms(), W.MS_ADPCM, 1, 8000, 256, 4, _ms_ext(500, W.MS_COEFS, 9)), W.MS_ADPCM,
                       "MS ADPCM", "too short for its 9 coefficient pairs"),
    "ms_table": (W.write_wav(_ms(), W.MS_ADPCM, 1, 8000, 256, 4, _ms_ext(500, [(256, 0), (512, -255)] +
                                                                         list(W.MS_COEFS[2:]))),
                 W.MS_ADPCM, "MS ADPCM", "not the standard table"),
    "ms_spb": (W.write_wav(_ms(), W.MS_ADPCM, 1, 8000, 256, 4, _ms_ext(499, W.MS_COEFS)), W.MS_ADPCM, "MS ADPCM",
               "499 samples per block do not fit block_align 256"),
    # a trailing block shorter than its header: 2 full blocks + 3 bytes (IMA mono header: 4), + 13 bytes (MS stereo: 14)
    "ima_cut_header": (W.write_wav(_ima(n=1020)[:512 + 3], W.IMA_ADPCM, 1, 8000, 256, 4,
                                   W.fmt_ext(W.IMA_ADPCM, 1, 256)),
                       W.IMA_ADPCM, "IMA ADPCM", r"block 2 at byte \d+: truncated: 3 bytes, its header needs 4"),
    "ms_cut_header": (W.write_wav(_ms(2, 512, 1010)[:1024 + 13], W.MS_ADPCM, 2, 8000, 512, 4,
                                  W.fmt_ext(W.MS_ADPCM, 2, 512)),
                      W.MS_ADPCM, "MS ADPCM", r"block 2 at byte \d+: truncated: 13 bytes, its header needs 14"),
    # fact states more samples than the blocks hold: 2 full blocks of 505 + a partial one of 1 + 8 * 3
    "ima_fact_long": (W.write_wav(_ima(n=1035), W.IMA_ADPCM, 1, 8000, 256, 4, W.fmt_ext(W.IMA_ADPCM, 1, 256),
                                  fact=1100),
                      W.IMA_ADPCM, "IMA ADPCM", r"block 2 at byte \d+: missing: .* holds 1035 samples .* 3 blocks, "
                                                r"the fact chunk states 1100"),
    "ms_fact_long": (W.write_wav(_ms(n=1000), W.MS_ADPCM, 1, 8000, 256, 4, W.fmt_ext(W.MS_ADPCM, 1, 256), fact=1500),
                     W.MS_ADPCM, "MS ADPCM", "block 2 at byte .* the fact chunk states 1500"),
}


@pytest.mark.parametrize("name", sorted(REJECTIONS))
def test_each_fmt_rejection_is_raised_before_any_cuda_call(tmp_path, no_cuda, name):
    data, tag, codec, match = REJECTIONS[name]
    _rejects(tmp_path, f"{name}.wav", data, tag, codec, match)


def test_missing_block_is_named_with_its_byte_offset(tmp_path, no_cuda):
    data = W.write_wav(_ima(n=2000), W.IMA_ADPCM, 1, 8000, 256, 4, W.fmt_ext(W.IMA_ADPCM, 1, 256), fact=4000)
    data_off = data.index(b"data") + 8
    # 2000 samples: 3 full blocks of 505 + 1 + 8 * 61; fact 4000 -> the first missing sample lies in block 3
    _rejects(tmp_path, "long.wav", data, W.IMA_ADPCM, "IMA ADPCM", rf"block 3 at byte {data_off + 3 * 256}: missing")


def test_adpcm_inside_extensible_is_rejected(tmp_path, no_cuda):
    ext = struct.pack("<HI", 505, 4) + struct.pack("<H", W.IMA_ADPCM) + bytes(14)   # SubFormat GUID at byte 24
    p = tmp_path / "ext.wav"
    p.write_bytes(W.write_wav(_ima(), 0xFFFE, 1, 8000, 256, 4, ext))
    with pytest.raises(ValueError, match="format tag 0x0011 inside WAVE_FORMAT_EXTENSIBLE"):
        load_audio(str(p))


def test_empty_data_chunk_decodes_to_no_frames(tmp_path, no_cuda):
    p = tmp_path / "empty.wav"
    p.write_bytes(W.write_wav(b"", W.IMA_ADPCM, 2, 8000, 512, 4, W.fmt_ext(W.IMA_ADPCM, 2, 512)))
    pcm, rate = load_audio(str(p))
    assert rate == 8000 and pcm.dtype == np.int16 and pcm.shape == (2, 0)


@pytest.mark.parametrize("tag,nch,ba,n,last,fact,want", [
    (W.MULAW, 2, 2, 1001, None, None, 1001),
    (W.IMA_ADPCM, 1, 256, 1035, "short", False, 1035),        # 2 x 505 + (1 + 8 * 3)
    (W.IMA_ADPCM, 2, 512, 1020, "short", False, 1027),        # 2 x 505 + (1 + 8 * 2): the last group is padded
    (W.IMA_ADPCM, 2, 512, 1020, "short", True, 1020),         # ... and fact trims it
    (W.IMA_ADPCM, 6, 1536, 600, "full", True, 600),
    (W.MS_ADPCM, 1, 256, 1001, "short", False, 1002),         # 2 x 500 + 2 header samples; no odd nibble count
    (W.MS_ADPCM, 2, 512, 1001, "full", False, 1500),
    (W.MS_ADPCM, 2, 512, 1001, "full", True, 1001),
])
def test_frame_count(tag, nch, ba, n, last, fact, want):
    from reverb_b200.audio_io import parse_wav_codec
    x = np.zeros((nch, n), np.int64)
    kw = {} if tag == W.MULAW else {"last": last}
    data, payload = W.codec_wav(x, 8000, tag, ba, fact=fact, **kw)
    fmt_off = data.index(b"fmt ") + 8
    fmt_body = data[fmt_off:fmt_off + struct.unpack_from("<I", data, fmt_off - 4)[0]]
    tag_, nch_, _rate, _br, block, bits = struct.unpack_from("<HHIIHH", fmt_body)
    info = parse_wav_codec(payload, (tag_, nch_, 8000, block, bits), fmt_body, n if fact else None, 0)
    assert info.frames == want
    if not fact:
        assert W.frames_in(len(payload), tag, nch, ba) == want


# ------------------------------------------------------------------------------------------------ oracle vs audioop
def test_g711_tables_equal_audioop():
    codes = bytes(range(256))
    assert np.array_equal(W.ulaw_table(), np.frombuffer(audioop.ulaw2lin(codes, 2), "<i2"))
    assert np.array_equal(W.alaw_table(), np.frombuffer(audioop.alaw2lin(codes, 2), "<i2"))
    assert W.ulaw_table().min() == -32124 and W.ulaw_table().max() == 32124
    assert W.alaw_table().min() == -32256 and W.alaw_table().max() == 32256


@pytest.mark.parametrize("ba", [256, 1024])
def test_ima_decoder_equals_audioop_block_by_block(ba):
    """audioop.adpcm2lin decodes high nibble first and takes (predictor, step index) as its state"""
    rng = np.random.default_rng(ba)
    spb = W.ima_spb(1, ba)
    nblk = 300
    x = np.clip(np.cumsum(rng.normal(0, 900, (1, spb * nblk)), 1), -32768, 32767).astype(np.int64)
    x[0, :spb * 40] = np.where(np.arange(spb * 40) // 37 % 2, 32767, -32768)      # full-scale square: clamping
    data = W.ima_encode(x, ba, step_index=np.arange(nblk) % 89)
    got = W.ima_decode(data, 1, ba, spb * nblk)
    for k in range(nblk):
        blk = data[k * ba:(k + 1) * ba]
        pred, idx = struct.unpack_from("<hB", blk)
        swapped = bytes(((b & 15) << 4) | (b >> 4) for b in blk[4:])
        ref = np.frombuffer(audioop.adpcm2lin(swapped, 2, (pred, idx))[0], "<i2")
        assert np.array_equal(got[0, k * spb:(k + 1) * spb], np.concatenate([[pred], ref])), k


# ------------------------------------------------------------------------------------------------ hand-worked MS ADPCM
def _ms_block(pred, delta, s1, s2, data):
    """one MS ADPCM block: per-channel bPredictor, then iDelta, iSamp1, iSamp2 (int16 each), then the nibbles"""
    nch = len(pred)
    return bytes(pred) + struct.pack(f"<{3 * nch}h", *delta, *s1, *s2) + bytes(data)


def hand_ms_blocks():
    """(WAV file bytes, expected (channels, frames) int16) for blocks worked out by hand from the MS ADPCM step"""
    cases = [
        # predictor 1 = (512, -256): pred = (2 s1 - s2); nibbles 3, F (-1) at delta 16
        ([_ms_block([1], [16], [100], [50], [0x3F])], [[50, 100, 198, 280]]),
        # predictor 3 = (192, 64): (-1 * 192 + 0) / 256 truncates to 0 (an arithmetic >> 8 would give -1)
        ([_ms_block([3], [16], [-1], [0], [0x00])], [[0, -1, 0, 0]]),
        # predictor 0 = (256, 0), delta 20 -> 17 -> the floor of 16; nibble 7 adds 112 and adapts to 614 * 16 >> 8 = 38
        ([_ms_block([0], [20], [1000], [0], [0x00, 0x71])], [[0, 1000, 1000, 1000, 1112, 1150]]),
        # int16 clamping upward and downward
        ([_ms_block([1], [2000], [32000], [31000], [0x77])], [[31000, 32000, 32767, 32767]]),
        ([_ms_block([1], [2000], [-32000], [-31000], [0x88])], [[-31000, -32000, -32768, -32768]]),
        # stereo: high nibble channel 0, low nibble channel 1
        ([_ms_block([1, 0], [16, 16], [100, 7], [50, 9], [0x31, 0xF2])], [[50, 100, 198, 280], [9, 7, 23, 55]]),
    ]
    out = []
    for blocks, want in cases:
        nch, ba = len(want), len(blocks[0])
        payload = b"".join(blocks)
        wav = W.write_wav(payload, W.MS_ADPCM, nch, 8000, ba, 4, W.fmt_ext(W.MS_ADPCM, nch, ba), spb=W.ms_spb(nch, ba))
        out.append((wav, payload, np.array(want, np.int16)))
    return out


def test_hand_worked_ms_adpcm_blocks():
    for _wav, payload, want in hand_ms_blocks():
        nch = want.shape[0]
        assert W.ms_spb(nch, len(payload)) == want.shape[1]
        assert np.array_equal(W.ms_decode(payload, nch, len(payload), W.MS_COEFS, want.shape[1]), want)


def test_ctypes_mirror_matches_the_c_header(tmp_path):
    import ctypes
    import os
    import shutil
    import subprocess
    gcc = shutil.which("gcc")
    if gcc is None:
        pytest.skip("no gcc")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    src = tmp_path / "size.c"
    src.write_text('#include <stdio.h>\n#include "rvb_b200.h"\n'
                   'int main(void) { printf("%zu\\n", sizeof(rvb_wav_codec)); return 0; }\n')
    exe = tmp_path / "size"
    subprocess.run([gcc, "-std=c99", "-Wall", "-Werror", "-I", os.path.join(root, "include"), str(src), "-o", str(exe)],
                   check=True)
    assert int(subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout) == \
        ctypes.sizeof(_lib.WavCodec)
