"""numpy G.711 and ADPCM WAV codecs: test and benchmark infrastructure for the GPU decoder
(reverb_b200/csrc/wav_codec.cu).

- G.711 µ-law / A-law: the 256-entry decode tables from the G.711 formulas, and a nearest-value encoder.
- IMA ADPCM and Microsoft ADPCM encoders that write real block layouts.  Every header field can be forced per block
  (IMA step index, MS predictor index and initial delta), MS ADPCM takes any coefficient table that starts with the
  seven standard pairs, and the last block is written short (only the groups / bytes its samples need) or padded to a
  full block (the `fact` chunk then trims it).  The encoders track the decoder's state, so full-scale input drives the
  int16 clamps exactly as a decoder meets them.
- Host decoders that restate the device algorithms, vectorised across blocks (each block's recurrence runs sample by
  sample over all blocks at once).
- A WAV writer with the fmt extension (cbSize and what follows) and an optional `fact` chunk.

Samples are int16 values, (channels, n).
"""
from __future__ import annotations

import struct
from typing import Optional, Sequence, Tuple

import numpy as np

MULAW, ALAW, IMA_ADPCM, MS_ADPCM = 0x0007, 0x0006, 0x0011, 0x0002

IMA_STEPS = np.array([
    7, 8, 9, 10, 11, 12, 13, 14, 16, 17, 19, 21, 23, 25, 28, 31, 34, 37, 41, 45, 50, 55, 60, 66, 73, 80, 88, 97, 107,
    118, 130, 143, 157, 173, 190, 209, 230, 253, 279, 307, 337, 371, 408, 449, 494, 544, 598, 658, 724, 796, 876, 963,
    1060, 1166, 1282, 1411, 1552, 1707, 1878, 2066, 2272, 2499, 2749, 3024, 3327, 3660, 4026, 4428, 4871, 5358, 5894,
    6484, 7132, 7845, 8630, 9493, 10442, 11487, 12635, 13899, 15289, 16818, 18500, 20350, 22385, 24623, 27086, 29794,
    32767], dtype=np.int64)
IMA_INDEX = np.array([-1, -1, -1, -1, 2, 4, 6, 8] * 2, dtype=np.int64)
MS_ADAPT = np.array([230, 230, 230, 230, 307, 409, 512, 614, 768, 614, 512, 409, 307, 230, 230, 230], dtype=np.int64)
MS_COEFS = ((256, 0), (512, -256), (0, 0), (192, 64), (240, 0), (460, -208), (392, -232))
MS_DELTA_CAP = (2 ** 31 - 1) // 768


# ------------------------------------------------------------------------------------------------ G.711
def ulaw_table() -> np.ndarray:
    x = ~np.arange(256, dtype=np.int64) & 0xFF
    mag = ((((x & 15) << 3) + 0x84) << ((x >> 4) & 7)) - 0x84
    return np.where(x & 0x80, -mag, mag).astype(np.int16)


def alaw_table() -> np.ndarray:
    x = np.arange(256, dtype=np.int64) ^ 0x55
    m, e = x & 15, (x >> 4) & 7
    mag = np.where(e == 0, (m << 4) + 8, ((m << 4) + 0x108) << np.maximum(e - 1, 0))
    return np.where(x & 0x80, mag, -mag).astype(np.int16)


def _table(tag: int) -> np.ndarray:
    return ulaw_table() if tag == MULAW else alaw_table()


def g711_encode(x: np.ndarray, tag: int) -> bytes:
    """Interleaved codes of the table values nearest to x (channels, n)."""
    t = _table(tag).astype(np.int64)
    order = np.argsort(t, kind="stable")
    vals = t[order]
    v = np.ascontiguousarray(np.asarray(x, np.int64).T).reshape(-1)
    i = np.clip(np.searchsorted(vals, v), 1, 255)
    pick = np.where(np.abs(vals[i - 1] - v) <= np.abs(vals[i] - v), i - 1, i)
    return order[pick].astype(np.uint8).tobytes()


def g711_decode(data: bytes, nch: int, tag: int) -> np.ndarray:
    codes = np.frombuffer(data, np.uint8)[:len(data) // nch * nch]
    return np.ascontiguousarray(_table(tag)[codes].reshape(-1, nch).T)


# ------------------------------------------------------------------------------------------------ block helpers
def _blocks(x: np.ndarray, spb: int, n_last: int) -> Tuple[np.ndarray, int]:
    """x (nch, n) as (nblk, nch, spb) int64; the last block holds n_last samples, the rest repeat its last sample."""
    x = np.asarray(x, np.int64)
    nch, n = x.shape
    nblk = -(-n // spb)
    pad = nblk * spb - n
    xp = np.concatenate([x, np.repeat(x[:, -1:], pad, 1)], 1) if pad else x
    return xp.reshape(nch, nblk, spb).transpose(1, 0, 2).copy(), nblk


def _per_block(v, nblk: int, nch: int) -> Optional[np.ndarray]:
    """None, a scalar, (nblk,) or (nblk, nch) -> (nblk, nch) int64"""
    if v is None:
        return None
    a = np.asarray(v, np.int64)
    if a.ndim == 1:
        a = a[:, None]
    return np.broadcast_to(a, (nblk, nch)).copy()


def _nibbles_to_bytes_low_first(nib: np.ndarray) -> np.ndarray:
    return (nib[..., 0::2] | (nib[..., 1::2] << 4)).astype(np.uint8)


# ------------------------------------------------------------------------------------------------ IMA ADPCM
def ima_block_align(nch: int, spb: int) -> int:
    return 4 * nch * (1 + (spb - 1) // 8)


def ima_spb(nch: int, block_align: int) -> int:
    return 1 + 8 * (block_align // (4 * nch) - 1)


def ima_step(pred, idx, nib):
    """the IMA reference shift-add step, elementwise over arrays"""
    step = IMA_STEPS[idx]
    diff = (step >> 3) + np.where(nib & 4, step, 0) + np.where(nib & 2, step >> 1, 0) + np.where(nib & 1, step >> 2, 0)
    pred = np.clip(np.where(nib & 8, pred - diff, pred + diff), -32768, 32767)
    return pred, np.clip(idx + IMA_INDEX[nib], 0, 88)


def ima_encode(x: np.ndarray, block_align: int, step_index=None, last: str = "short") -> bytes:
    """IMA ADPCM blocks of x (nch, n).  step_index: the header's step index, a scalar, per block (nblk,) or per block
    and channel (nblk, nch); by default one that suits the block's first differences.  last: "short" writes only the
    4-byte groups the last block's samples need, "full" pads it to block_align (a `fact` chunk then gives the length)."""
    nch, n = np.shape(x)
    spb = ima_spb(nch, block_align)
    rem = n - (-(-n // spb) - 1) * spb
    xb, nblk = _blocks(x, spb, rem)
    idx = _per_block(step_index, nblk, nch)
    if idx is None:
        d = np.abs(np.diff(xb[:, :, :9], axis=2)).mean(axis=2)
        idx = np.clip(np.searchsorted(IMA_STEPS, d) - 8, 0, 88)
    pred = xb[:, :, 0].copy()
    hdr = np.zeros((nblk, nch, 4), np.uint8)
    hdr[:, :, 0], hdr[:, :, 1], hdr[:, :, 2] = pred & 0xFF, (pred >> 8) & 0xFF, idx
    nibs = np.zeros((nblk, nch, spb - 1), np.int64)
    for s in range(1, spb):
        delta = xb[:, :, s] - pred
        d, step = np.abs(delta), IMA_STEPS[idx]
        nib = np.where(delta < 0, 8, 0)
        b4 = d >= step
        nib |= np.where(b4, 4, 0)
        d = np.where(b4, d - step, d)
        b2 = d >= (step >> 1)
        nib |= np.where(b2, 2, 0)
        d = np.where(b2, d - (step >> 1), d)
        nib |= np.where(d >= (step >> 2), 1, 0)
        nibs[:, :, s - 1] = nib
        pred, idx = ima_step(pred, idx, nib)
    groups = _nibbles_to_bytes_low_first(nibs.reshape(nblk, nch, -1, 8))          # (nblk, nch, G, 4)
    data = groups.transpose(0, 2, 1, 3).reshape(nblk, -1)                           # group by group, channel by channel
    blocks = np.concatenate([hdr.reshape(nblk, -1), data], 1)
    out = blocks.tobytes()
    if last == "short":
        out = out[:len(out) - block_align + 4 * nch * (1 + -(-(rem - 1) // 8))]
    return out


def ima_decode(data: bytes, nch: int, block_align: int, frames: int) -> np.ndarray:
    """(nch, frames) int16; a step index above 88 raises ValueError naming the block"""
    spb = ima_spb(nch, block_align)
    nblk = -(-len(data) // block_align)
    b = np.frombuffer(data + bytes(nblk * block_align - len(data)), np.uint8).reshape(nblk, block_align)
    h = b[:, :4 * nch].reshape(nblk, nch, 4).astype(np.int64)
    pred = ((h[:, :, 0] | (h[:, :, 1] << 8)) ^ 0x8000) - 0x8000
    idx = h[:, :, 2]
    if (idx > 88).any():
        k = int(np.argmax((idx > 88).any(1)))
        raise ValueError(f"block {k}: IMA ADPCM step index above 88")
    g = b[:, 4 * nch:].reshape(nblk, -1, nch, 4).astype(np.int64)                  # (nblk, G, nch, 4)
    nib = np.stack([g & 15, g >> 4], -1).reshape(nblk, -1, nch, 8).transpose(0, 2, 1, 3).reshape(nblk, nch, -1)
    out = np.zeros((nblk, nch, spb), np.int64)
    out[:, :, 0] = pred
    for s in range(1, spb):
        pred, idx = ima_step(pred, idx, nib[:, :, s - 1])
        out[:, :, s] = pred
    return np.ascontiguousarray(out.transpose(1, 0, 2).reshape(nch, -1)[:, :frames]).astype(np.int16)


# ------------------------------------------------------------------------------------------------ MS ADPCM
def ms_spb(nch: int, block_align: int) -> int:
    return 2 + (block_align - 7 * nch) * 2 // nch


def ms_pred(s1, s2, c1, c2):
    """(s1·c1 + s2·c2) / 256 with C's truncation toward zero"""
    a = s1 * c1 + s2 * c2
    return np.sign(a) * (np.abs(a) // 256)


def ms_step(s1, s2, delta, nib, c1, c2):
    v = np.clip(ms_pred(s1, s2, c1, c2) + (((nib ^ 8) - 8) * delta), -32768, 32767)
    delta = np.minimum(np.maximum(16, (MS_ADAPT[nib] * delta) >> 8), MS_DELTA_CAP)
    return v, s1, delta


def ms_encode(x: np.ndarray, block_align: int, coefs: Sequence[Tuple[int, int]] = MS_COEFS, predictor=None,
              delta=None, last: str = "short") -> bytes:
    """MS ADPCM blocks of x (nch = 1 or 2, n).  predictor: the header's coefficient index (scalar, (nblk,) or
    (nblk, nch); default 0); delta: the header's initial delta (default: a quarter of the block's mean first difference,
    at least 16).  last: "short" writes only the bytes the last block's samples need, "full" pads it to block_align."""
    nch, n = np.shape(x)
    spb = ms_spb(nch, block_align)
    rem = n - (-(-n // spb) - 1) * spb
    xb, nblk = _blocks(x, spb, rem)
    pi = _per_block(0 if predictor is None else predictor, nblk, nch)
    dl = _per_block(delta, nblk, nch)
    if dl is None:
        dl = np.maximum(16, np.abs(np.diff(xb[:, :, :10], axis=2)).mean(axis=2).astype(np.int64) // 4)
    cf = np.array(coefs, np.int64)
    c1, c2 = cf[np.minimum(pi, len(cf) - 1), 0], cf[np.minimum(pi, len(cf) - 1), 1]
    s2, s1 = xb[:, :, 0].copy(), xb[:, :, 1].copy()
    hdr = [pi.astype(np.uint8)] + [np.stack([v & 0xFF, (v >> 8) & 0xFF], -1).astype(np.uint8).reshape(nblk, -1)
                                   for v in (dl, s1, s2)]
    d = dl.copy()
    nibs = np.zeros((nblk, spb - 2, nch), np.int64)
    for s in range(2, spb):
        err = xb[:, :, s] - ms_pred(s1, s2, c1, c2)
        dd = np.maximum(d, 1)
        q = np.clip(np.sign(err) * ((np.abs(err) + dd // 2) // dd), -8, 7)
        nib = q & 15
        nibs[:, s - 2] = nib
        v, s2, d = ms_step(s1, s2, d, nib, c1, c2)
        s1 = v
    flat = nibs.reshape(nblk, -1)                                                   # frame by frame, channel by channel
    data = ((flat[:, 0::2] << 4) | flat[:, 1::2]).astype(np.uint8)
    out = np.concatenate(hdr + [data], 1).tobytes()
    if last == "short":
        out = out[:len(out) - block_align + 7 * nch + -(-max(rem - 2, 0) * nch // 2)]
    return out


def ms_decode(data: bytes, nch: int, block_align: int, coefs: Sequence[Tuple[int, int]], frames: int) -> np.ndarray:
    """(nch, frames) int16; a predictor index beyond the table raises ValueError naming the block"""
    spb = ms_spb(nch, block_align)
    nblk = -(-len(data) // block_align)
    b = np.frombuffer(data + bytes(nblk * block_align - len(data)), np.uint8).reshape(nblk, block_align).astype(np.int64)

    def i16(off):
        v = b[:, off:off + 2 * nch:2] | (b[:, off + 1:off + 2 * nch:2] << 8)
        return (v ^ 0x8000) - 0x8000
    pi = b[:, :nch]
    if (pi >= len(coefs)).any():
        k = int(np.argmax((pi >= len(coefs)).any(1)))
        raise ValueError(f"block {k}: MS ADPCM predictor index beyond the coefficient table")
    cf = np.array(coefs, np.int64)
    c1, c2 = cf[pi, 0], cf[pi, 1]
    delta, s1, s2 = i16(nch), i16(3 * nch), i16(5 * nch)
    d = b[:, 7 * nch:]
    nib = np.stack([d >> 4, d & 15], -1).reshape(nblk, -1)[:, :(spb - 2) * nch].reshape(nblk, spb - 2, nch)
    out = np.zeros((nblk, nch, spb), np.int64)
    out[:, :, 0], out[:, :, 1] = s2, s1
    for s in range(2, spb):
        v, s2, delta = ms_step(s1, s2, delta, nib[:, s - 2], c1, c2)
        s1 = v
        out[:, :, s] = v
    return np.ascontiguousarray(out.transpose(1, 0, 2).reshape(nch, -1)[:, :frames]).astype(np.int16)


# ------------------------------------------------------------------------------------------------ frames and WAV
def frames_in(data_len: int, tag: int, nch: int, block_align: int) -> int:
    """frames per channel the data chunk holds (the `fact`-less length)"""
    if tag in (MULAW, ALAW):
        return data_len // nch
    spb = ima_spb(nch, block_align) if tag == IMA_ADPCM else ms_spb(nch, block_align)
    full, rem = divmod(data_len, block_align)
    hdr = 4 * nch if tag == IMA_ADPCM else 7 * nch
    part = 0
    if rem >= hdr:
        part = 1 + 8 * ((rem - hdr) // hdr) if tag == IMA_ADPCM else 2 + (rem - hdr) * 2 // nch
    return full * spb + part


def decode(data: bytes, tag: int, nch: int, block_align: int, frames: int,
           coefs: Sequence[Tuple[int, int]] = MS_COEFS) -> np.ndarray:
    if tag in (MULAW, ALAW):
        return g711_decode(data, nch, tag)[:, :frames]
    if tag == IMA_ADPCM:
        return ima_decode(data, nch, block_align, frames)
    return ms_decode(data, nch, block_align, coefs, frames)


def fmt_ext(tag: int, nch: int, block_align: int, coefs: Sequence[Tuple[int, int]] = MS_COEFS) -> Optional[bytes]:
    """the fmt extension after cbSize: wSamplesPerBlock (IMA), + wNumCoef and the pairs (MS); None for G.711"""
    if tag == IMA_ADPCM:
        return struct.pack("<H", ima_spb(nch, block_align))
    if tag == MS_ADPCM:
        return struct.pack("<HH", ms_spb(nch, block_align), len(coefs)) + b"".join(struct.pack("<hh", *c) for c in coefs)
    return None


def write_wav(payload: bytes, tag: int, nch: int, rate: int, block_align: int, bits: int, ext: Optional[bytes] = None,
              fact: Optional[int] = None, spb: int = 1) -> bytes:
    """RIFF/WAVE with a fmt chunk (plus cbSize and `ext` when ext is not None), an optional fact chunk and the data."""
    fmt = struct.pack("<HHIIHH", tag, nch, rate, rate * block_align // spb, block_align, bits)
    if ext is not None:
        fmt += struct.pack("<H", len(ext)) + ext
    chunks = b"fmt " + struct.pack("<I", len(fmt)) + fmt + b"\0" * (len(fmt) & 1)
    if fact is not None:
        chunks += b"fact" + struct.pack("<II", 4, fact)
    chunks += b"data" + struct.pack("<I", len(payload)) + payload + b"\0" * (len(payload) & 1)
    return b"RIFF" + struct.pack("<I", 4 + len(chunks)) + b"WAVE" + chunks


def codec_wav(x: np.ndarray, rate: int, tag: int, block_align: int = 0, fact: Optional[bool] = None,
              coefs: Sequence[Tuple[int, int]] = MS_COEFS, **enc) -> Tuple[bytes, bytes]:
    """(WAV file, data chunk) of x (nch, n) in one codec; fact=True writes a fact chunk with n (the default for ADPCM)"""
    nch, n = np.shape(x)
    if tag in (MULAW, ALAW):
        payload = g711_encode(x, tag)
        return write_wav(payload, tag, nch, rate, nch, 8, fact=n if fact else None), payload
    if tag == IMA_ADPCM:
        payload, spb = ima_encode(x, block_align, **enc), ima_spb(nch, block_align)
    else:
        payload, spb = ms_encode(x, block_align, coefs=coefs, **enc), ms_spb(nch, block_align)
    return write_wav(payload, tag, nch, rate, block_align, 4, fmt_ext(tag, nch, block_align, coefs),
                     n if fact is None or fact else None, spb), payload
