"""A numpy FLAC encoder (RFC 9639): test and benchmark infrastructure for the GPU decoder (reverb_b200/csrc/flac.cu).

`encode` gives explicit control, frame by frame (FrameSpec) and subframe by subframe (SubSpec), over everything the
decoder must handle: subframe type and order, LPC precision and shift, stereo mode, Rice partition order, parameter
width and escaped partitions, wasted bits, bits per sample, fixed or variable blocking, the uncommon block-size and
sample-rate codes, metadata blocks, an ID3v2 prefix and `total_samples = 0`.  STREAMINFO carries the MD5 of the input.

`encode_libflac` mirrors what libFLAC writes by default: 4096-sample blocks, LPC up to order 8 with automatic
precision, adaptive mid/side, partition orders up to 6, and SEEKTABLE + VORBIS_COMMENT + PADDING.  Its analysis, the
Rice coding and the bit packing are vectorised over frames, so a one-hour recording encodes in seconds.

Input samples are the codec's integers: (channels, n) int values in [-2^(bps-1), 2^(bps-1)).
"""
from __future__ import annotations

import hashlib
import struct
from dataclasses import dataclass, field
from typing import List, Optional, Sequence, Tuple

import numpy as np

BLOCK_TYPES = {"STREAMINFO": 0, "PADDING": 1, "APPLICATION": 2, "SEEKTABLE": 3, "VORBIS_COMMENT": 4, "CUESHEET": 5,
               "PICTURE": 6}
STEREO = {"independent": None, "left_side": 8, "side_right": 9, "mid_side": 10}
_RATE_CODES = {88200: 1, 176400: 2, 192000: 3, 8000: 4, 16000: 5, 22050: 6, 24000: 7, 32000: 8, 44100: 9, 48000: 10,
               96000: 11}
_BPS_CODES = {8: 1, 12: 2, 16: 4, 20: 5, 24: 6, 32: 7}


def _crc_table(poly: int, width: int) -> np.ndarray:
    top, mask = 1 << (width - 1), (1 << width) - 1
    t = []
    for i in range(256):
        c = i << (width - 8)
        for _ in range(8):
            c = ((c << 1) ^ poly) & mask if c & top else (c << 1) & mask
        t.append(c)
    return np.array(t, dtype=np.uint32)


CRC8_TABLE, CRC16_TABLE = _crc_table(0x07, 8), _crc_table(0x8005, 16)


def crc8(data: bytes) -> int:
    c = 0
    for b in data:
        c = int(CRC8_TABLE[c ^ b])
    return c


def crc16(data: bytes) -> int:
    c = 0
    for b in data:
        c = ((c << 8) & 0xFFFF) ^ int(CRC16_TABLE[(c >> 8) ^ b])
    return c


def _crc16_rows(frames: List[np.ndarray]) -> np.ndarray:
    """CRC-16 of many byte strings at once: right-aligned in one matrix (leading zero bytes leave a CRC with initial
    value 0 unchanged), one table step per column."""
    L = max(len(f) for f in frames)
    m = np.zeros((len(frames), L), dtype=np.uint32)
    for i, f in enumerate(frames):
        m[i, L - len(f):] = f
    c = np.zeros(len(frames), dtype=np.uint32)
    for j in range(L):
        c = ((c << 8) & 0xFFFF) ^ CRC16_TABLE[((c >> 8) ^ m[:, j]) & 0xFF]
    return c


def coded_number(v: int) -> bytes:
    """The UTF-8-like coded frame / sample number of a frame header (up to 36 bits)."""
    if v < 0x80:
        return bytes([v])
    for n in range(2, 8):
        if v < (1 << (5 * n + 1)):
            out = [0x80 | ((v >> (6 * i)) & 0x3F) for i in range(n - 1)][::-1]
            lead = (0xFF00 >> n) & 0xFF
            return bytes([lead | (v >> (6 * (n - 1)))] + out)
    raise ValueError(f"coded number {v} exceeds 36 bits")


@dataclass
class SubSpec:
    """How one subframe is written."""
    type: str = "lpc"                     # constant | verbatim | fixed | lpc
    order: int = 8                        # FIXED 0-4, LPC 1-32
    precision: int = 12                   # LPC coefficient bits, 1-15
    shift: Optional[int] = None           # LPC shift 0-15; None: the largest that fits the precision
    coefs: Optional[Sequence[int]] = None  # explicit quantised LPC coefficients (else from the signal)
    wasted: Optional[int] = None          # None: every trailing zero bit the block shares
    partition_order: Optional[int] = None  # None: the cheapest of 0..max_partition_order
    max_partition_order: int = 6
    rice_width: Optional[int] = None      # 4- or 5-bit Rice parameters; None: 5 above 16 bits per sample
    rice_params: Optional[Sequence[int]] = None  # explicit per-partition parameters
    escape: Sequence[int] = ()            # partitions written escaped (unencoded)


@dataclass
class FrameSpec:
    bs: int
    stereo: str = "independent"           # independent | left_side | side_right | mid_side
    sub: object = field(default_factory=SubSpec)  # one SubSpec for every channel, or a list
    bs_code: Optional[int] = None         # 6 / 7: force the uncommon 8- / 16-bit block size
    rate_code: Optional[int] = None       # 0: "from STREAMINFO", 12 / 13 / 14: the uncommon kHz / Hz / 10 Hz codes
    bps_code: Optional[int] = None        # 0: "from STREAMINFO"


# ------------------------------------------------------------------------------------------------ field helpers
# A bitstream is built as parallel arrays of fields (value, bit count), packed at the end.

def _fields(vals, nbits) -> Tuple[np.ndarray, np.ndarray]:
    v = np.asarray(vals, dtype=np.int64)
    n = np.broadcast_to(np.asarray(nbits, dtype=np.int64), v.shape)
    return (v & ((np.int64(1) << n) - 1)).astype(np.uint64) if v.size else v.astype(np.uint64), n.astype(np.int64)


def _cat(parts) -> Tuple[np.ndarray, np.ndarray]:
    return (np.concatenate([p[0] for p in parts]).astype(np.uint64), np.concatenate([p[1] for p in parts]))


def _pack(vals: np.ndarray, nbits: np.ndarray) -> np.ndarray:
    """Packs MSB-first fields (whose bit counts sum to a multiple of 8) into bytes.  A field's set bits are its low
    <= 57 bits, so a long Rice unary run is only a shift of its start."""
    total = int(nbits.sum())
    assert total % 8 == 0
    offs = np.cumsum(nbits) - nbits
    keep = vals != 0
    v, n, o = vals[keep], nbits[keep], offs[keep]
    w = np.minimum(n, 57)
    start = o + n - w
    byte0 = start >> 3
    word = v << (64 - (start & 7) - w).astype(np.uint64)
    acc = np.zeros(total // 8 + 8, dtype=np.float64)
    for j in range(8):
        b = (word >> np.uint64(56 - 8 * j)) & np.uint64(0xFF)
        nz = b != 0
        if nz.any():
            acc += np.bincount(byte0[nz] + j, weights=b[nz].astype(np.float64), minlength=acc.size)[:acc.size]
    return acc[:total // 8].astype(np.uint8)


def _signed_bits(x: np.ndarray) -> int:
    """Bits of a two's complement field that holds every value of x."""
    if x.size == 0:
        return 0
    hi, lo = int(x.max()), int(x.min())
    return max(hi.bit_length(), (-lo - 1).bit_length()) + 1 if (hi or lo) else 0


# ------------------------------------------------------------------------------------------------ analysis
def lpc_coefs(x: np.ndarray, order: int) -> np.ndarray:
    """Rows of x (R, bs) -> (R, order) float LPC coefficients: Tukey(0.5) window, autocorrelation, Levinson-Durbin."""
    x = np.asarray(x, np.float64)
    R, n = x.shape
    t = np.ones(n)
    m = int(0.25 * n)
    if m > 0:
        ramp = 0.5 * (1 - np.cos(np.pi * np.arange(m) / m))
        t[:m], t[n - m:] = ramp, ramp[::-1]
    xw = x * t
    ac = np.stack([(xw[:, l:] * xw[:, :n - l]).sum(1) for l in range(order + 1)], 1)
    ac[:, 0] *= 1.0 + 1e-9
    ac[:, 0] += 1e-9
    a = np.zeros((R, order))
    err = ac[:, 0].copy()
    for i in range(order):
        k = (ac[:, i + 1] - (a[:, :i] * ac[:, i:0:-1]).sum(1)) / err
        a_new = a.copy()
        a_new[:, i] = k
        a_new[:, :i] = a[:, :i] - k[:, None] * a[:, i - 1::-1][:, :i] if i else a_new[:, :i]
        a = a_new
        err = err * (1 - k * k)
    return a


def quantize_coefs(c: np.ndarray, precision, shift=None) -> Tuple[np.ndarray, np.ndarray]:
    """(R, order) float -> (int coefficients, shift per row), libFLAC's rule: the largest shift <= 15 whose largest
    coefficient fits `precision` signed bits."""
    R = c.shape[0]
    prec = np.broadcast_to(np.asarray(precision, np.int64), (R,))
    if shift is None:
        cmax = np.abs(c).max(1)
        _, e = np.frexp(np.where(cmax > 0, cmax, 1.0))
        shift = np.clip(prec - 1 - e, 0, 15)
    shift = np.broadcast_to(np.asarray(shift, np.int64), (R,))
    lim = (np.int64(1) << (prec - 1))[:, None]
    q = np.clip(np.round(c * np.exp2(shift)[:, None]), -lim, lim - 1).astype(np.int64)
    return q, shift.copy()


def lpc_residual(x: np.ndarray, q: np.ndarray, shift: np.ndarray) -> np.ndarray:
    """Rows of x (R, bs) int64 -> (R, bs - order) residual of the integer predictor (RFC 9639 §9.2.6)."""
    R, n = x.shape
    order = q.shape[1]
    acc = np.zeros((R, n - order), np.int64)
    for j in range(order):
        acc += q[:, j:j + 1] * x[:, order - 1 - j:n - 1 - j]
    return x[:, order:] - (acc >> shift[:, None])


def rice_plan(u: np.ndarray, order, po_max: int, kmax: int, width: int):
    """Cheapest Rice partitioning of zigzagged residual rows u (R, bs) whose first `order` entries are warm-up
    positions (ignored): -> (partition order, params (R, 2^po_max) of which the first 2^po are used, bits) per row."""
    R, bs = u.shape
    order = np.broadcast_to(np.asarray(order, np.int64), (R,))
    pf = po_max
    while pf > 0 and (bs % (1 << pf) or (bs >> pf) < order.max()):
        pf -= 1
    uz = u.copy()
    uz[np.arange(bs)[None, :] < order[:, None]] = 0
    parts = 1 << pf
    S = np.stack([(uz >> np.uint64(k)).reshape(R, parts, -1).sum(2).astype(np.int64) for k in range(kmax + 1)], 1)
    cnt = np.full((R, parts), bs >> pf, np.int64)
    cnt[:, 0] -= order
    best_po = np.zeros(R, np.int64)
    best_bits = np.full(R, np.iinfo(np.int64).max)
    best_params = np.zeros((R, 1 << po_max), np.int64)
    for po in range(pf + 1):
        g = 1 << (pf - po)
        Sp = S.reshape(R, kmax + 1, 1 << po, g).sum(3)
        cp = cnt.reshape(R, 1 << po, g).sum(2)
        cost = Sp + cp[:, None, :] * (np.arange(kmax + 1)[None, :, None] + 1)
        k = cost.argmin(1)
        bits = np.take_along_axis(cost, k[:, None, :], 1)[:, 0].sum(1) + (1 << po) * width
        better = bits < best_bits
        best_bits = np.where(better, bits, best_bits)
        best_po = np.where(better, po, best_po)
        best_params[better, :1 << po] = k[better]
    return best_po, best_params, best_bits


def zigzag(e: np.ndarray) -> np.ndarray:
    e = np.asarray(e, np.int64)
    return ((e << 1) ^ (e >> 63)).astype(np.uint64)


def residual_fields(e: np.ndarray, bs: int, order: int, po: int, params, width: int, escape=()):
    """Fields of a RESIDUAL section: method, partition order, then every partition's parameter (or escape code and
    bit count) and samples."""
    esc_code = 15 if width == 4 else 31
    parts, psize = 1 << po, bs >> po
    assert bs % parts == 0 and psize >= order, (bs, po, order)
    e = np.asarray(e, np.int64)
    u = zigzag(e)
    counts = np.full(parts, psize)
    counts[0] -= order
    starts = np.concatenate([[0], np.cumsum(counts)[:-1]])
    k = np.repeat(np.asarray(params[:parts], np.int64), counts)
    esc_s = np.zeros(len(e), bool)
    hdr_v, hdr_n = [], []
    for p in range(parts):
        if p in escape:
            seg = e[starts[p]:starts[p] + counts[p]]
            nb = _signed_bits(seg)
            assert nb <= 31
            esc_s[starts[p]:starts[p] + counts[p]] = True
            k[starts[p]:starts[p] + counts[p]] = nb
            hdr_v.append((esc_code << 5) | nb)
            hdr_n.append(width + 5)
        else:
            assert 0 <= params[p] < esc_code
            hdr_v.append(int(params[p]))
            hdr_n.append(width)
    ku = k.astype(np.uint64)
    rv = (np.uint64(1) << ku) | (u & ((np.uint64(1) << ku) - np.uint64(1)))
    rn = (u >> ku).astype(np.int64) + 1 + k
    vals = np.where(esc_s, (e & ((np.int64(1) << k) - 1)).astype(np.uint64), rv)
    nbits = np.where(esc_s, k, rn)
    vals = np.insert(vals, starts, np.asarray(hdr_v, np.uint64))
    nbits = np.insert(nbits, starts, np.asarray(hdr_n, np.int64))
    head = _fields([(0 if width == 4 else 1) << 4 | po], 6)
    return _cat([head, (vals.astype(np.uint64), nbits.astype(np.int64))])


def _subframe_header(type_code: int, wasted: int):
    f = [_fields([(type_code << 1) | (1 if wasted else 0)], 8)]
    if wasted:
        f.append(_fields([1], wasted))           # wasted - 1 zero bits, then a 1
    return f


def subframe_fields(x: np.ndarray, sbps: int, spec: SubSpec):
    """Fields of one subframe of the int64 block x (sbps bits, including a side channel's extra bit)."""
    x = np.asarray(x, np.int64)
    bs = len(x)
    if spec.wasted is None:
        nz = x[x != 0]
        w = 0
        if nz.size:
            while w < sbps - 1 and not (nz & ((1 << (w + 1)) - 1)).any():
                w += 1
    else:
        w = spec.wasted
        assert not (x & ((1 << w) - 1)).any() and w < sbps
    x = x >> w
    b = sbps - w
    if spec.type == "constant":
        assert (x == x[0]).all()
        return _cat(_subframe_header(0, w) + [_fields([x[0]], b)])
    if spec.type == "verbatim":
        return _cat(_subframe_header(1, w) + [_fields(x, b)])
    o = spec.order
    if spec.type == "fixed":
        assert 0 <= o <= 4
        e = np.diff(x, n=o) if o else x
        head = _subframe_header(8 + o, w) + [_fields(x[:o], b)]
    else:
        assert spec.type == "lpc" and 1 <= o <= 32 and 1 <= spec.precision <= 15
        if spec.coefs is not None:
            q = np.asarray(spec.coefs, np.int64)[None]
            shift = np.asarray([spec.shift or 0])
        else:
            q, shift = quantize_coefs(lpc_coefs(x[None], o), spec.precision, spec.shift)
        e = lpc_residual(x[None], q, shift)[0]
        head = _subframe_header(31 + o, w) + [_fields(x[:o], b), _fields([spec.precision - 1], 4),
                                              _fields(shift, 5), _fields(q[0], spec.precision)]
    assert e.size == 0 or (e.min() >= -(1 << 31) and e.max() < (1 << 31)), "residual exceeds 32 bits"
    width = spec.rice_width or (5 if b > 16 else 4)
    kmax = 14 if width == 4 else 30
    u = zigzag(np.concatenate([np.zeros(o, np.int64), e]))[None]
    if spec.partition_order is None:
        po, params, _ = rice_plan(u, o, spec.max_partition_order, kmax, width)
        po, params = int(po[0]), params[0]
    else:
        po = spec.partition_order
        parts = 1 << po
        uz = u[0].copy()
        uz[:o] = 0
        S = np.stack([(uz >> np.uint64(k)).reshape(parts, -1).sum(1) for k in range(kmax + 1)])
        cnt = np.full(parts, bs >> po)
        cnt[0] -= o
        params = (S + cnt[None] * (np.arange(kmax + 1)[:, None] + 1)).argmin(0)
    if spec.rice_params is not None:
        params = np.asarray(spec.rice_params, np.int64)
    return _cat(head + [residual_fields(e, bs, o, po, params, width, tuple(spec.escape))])


# ------------------------------------------------------------------------------------------------ frames and stream
def frame_header(num: int, bs: int, rate: int, chan_code: int, bps: int, variable: bool, spec: FrameSpec) -> bytes:
    if spec.bs_code is not None:
        bc = spec.bs_code
    elif bs == 192:
        bc = 1
    elif bs in (576, 1152, 2304, 4608):
        bc = {576: 2, 1152: 3, 2304: 4, 4608: 5}[bs]
    elif bs >= 256 and bs <= 32768 and bs & (bs - 1) == 0:
        bc = bs.bit_length() - 1
    else:
        bc = 6 if bs <= 256 else 7
    if spec.rate_code is not None:
        rc = spec.rate_code
    elif rate in _RATE_CODES:
        rc = _RATE_CODES[rate]
    elif rate % 1000 == 0 and rate // 1000 < 256:
        rc = 12
    elif rate < 65536:
        rc = 13
    elif rate % 10 == 0 and rate // 10 < 65536:
        rc = 14
    else:
        rc = 0
    pc = spec.bps_code if spec.bps_code is not None else _BPS_CODES.get(bps, 0)
    h = bytearray([0xFF, 0xF8 | int(variable), (bc << 4) | rc, (chan_code << 4) | (pc << 1)]) + coded_number(num)
    if bc == 6:
        h.append(bs - 1)
    elif bc == 7:
        h += (bs - 1).to_bytes(2, "big")
    if rc == 12:
        h.append(rate // 1000)
    elif rc == 13:
        h += rate.to_bytes(2, "big")
    elif rc == 14:
        h += (rate // 10).to_bytes(2, "big")
    h.append(crc8(bytes(h)))
    return bytes(h)


def stereo_channels(x: np.ndarray, mode: str) -> Tuple[List[np.ndarray], List[int]]:
    """The two coded channels of a stereo block and which of them is the side channel (one extra bit)."""
    L, R = x[0].astype(np.int64), x[1].astype(np.int64)
    if mode == "left_side":
        return [L, L - R], [0, 1]
    if mode == "side_right":
        return [L - R, R], [1, 0]
    if mode == "mid_side":
        return [(L + R) >> 1, L - R], [0, 1]
    raise ValueError(mode)


def _frame_fields(header: bytes, subs) -> Tuple[np.ndarray, np.ndarray]:
    v, n = _cat([_fields(np.frombuffer(header, np.uint8), 8)] + list(subs))
    pad = (-int(n.sum())) % 8
    return _cat([(v, n), _fields([0], pad), _fields([0], 16)])   # alignment, CRC-16 (filled in after packing)


def _assemble(frame_fields: List[Tuple[np.ndarray, np.ndarray]], chunk: int = 256) -> bytes:
    out = []
    for s in range(0, len(frame_fields), chunk):
        part = frame_fields[s:s + chunk]
        data = _pack(*_cat(part))
        sizes = np.array([int(n.sum()) // 8 for _, n in part])
        ends = np.cumsum(sizes)
        frames = [data[e - z:e - 2] for e, z in zip(ends, sizes)]
        crcs = _crc16_rows(frames)
        data[ends - 2] = (crcs >> 8).astype(np.uint8)
        data[ends - 1] = (crcs & 0xFF).astype(np.uint8)
        out.append(data.tobytes())
    return b"".join(out)


def md5_of(x: np.ndarray, bps: int) -> bytes:
    """STREAMINFO's MD5: the samples interleaved, little-endian, (bps + 7) // 8 bytes each."""
    w = (bps + 7) // 8
    h = hashlib.md5()
    xt = np.ascontiguousarray(np.asarray(x, np.int64).T)
    step = 1 << 20
    for s in range(0, xt.shape[0], step):
        h.update(xt[s:s + step].astype("<i8").view(np.uint8).reshape(-1, 8)[:, :w].tobytes())
    return h.digest()


def metadata_block(btype, payload: bytes, last: bool) -> bytes:
    t = BLOCK_TYPES[btype] if isinstance(btype, str) else int(btype)
    return bytes([(0x80 if last else 0) | t]) + len(payload).to_bytes(3, "big") + payload


def streaminfo(min_bs, max_bs, min_fr, max_fr, rate, nch, bps, total, md5) -> bytes:
    packed = (rate << 44) | ((nch - 1) << 41) | ((bps - 1) << 36) | total
    min_fr, max_fr = (min_fr, max_fr) if max_fr < (1 << 24) else (0, 0)          # 0: unknown
    return struct.pack(">HH", min_bs, max_bs) + min_fr.to_bytes(3, "big") + max_fr.to_bytes(3, "big") + \
        packed.to_bytes(8, "big") + md5


def id3v2(payload: bytes = b"TIT2\x00\x00\x00\x05\x00\x00\x03abcd") -> bytes:
    n = len(payload)
    return b"ID3\x04\x00\x00" + bytes([(n >> 21) & 0x7F, (n >> 14) & 0x7F, (n >> 7) & 0x7F, n & 0x7F]) + payload


def vorbis_comment(vendor: str = "reverb_b200 oracle", comments=("TITLE=test",)) -> bytes:
    b = struct.pack("<I", len(vendor)) + vendor.encode() + struct.pack("<I", len(comments))
    for c in comments:
        b += struct.pack("<I", len(c)) + c.encode()
    return b


def seektable(points) -> bytes:
    return b"".join(struct.pack(">QQH", s, o, n) for s, o, n in points)


def _stream(x, rate, bps, frame_fields, bss, blocks, id3, total_samples, md5, seek_every=None) -> bytes:
    audio = _assemble(frame_fields)
    sizes = [int(n.sum()) // 8 for _, n in frame_fields]
    blocks = list(blocks)
    if seek_every:
        pts, pos, smp = [], 0, 0
        for z, b in zip(sizes, bss):
            if not pts or smp - pts[-1][0] >= seek_every:
                pts.append((smp, pos, b))
            pos, smp = pos + z, smp + b
        blocks = [("SEEKTABLE", seektable(pts))] + blocks
    n = x.shape[1]
    full = bss[:-1] if len(bss) > 1 else bss
    si = streaminfo(min(full), max(bss), min(sizes), max(sizes), rate, x.shape[0], bps,
                    n if total_samples is None else total_samples, md5_of(x, bps) if md5 is None else md5)
    meta = [("STREAMINFO", si)] + blocks
    head = b"fLaC" + b"".join(metadata_block(t, p, i == len(meta) - 1) for i, (t, p) in enumerate(meta))
    return id3 + head + audio


def encode(x: np.ndarray, sample_rate: int, bps: int, frames: Optional[List[FrameSpec]] = None,
           block_size: int = 4096, variable: bool = False, blocks=(), id3: bytes = b"",
           total_samples: Optional[int] = None, md5: Optional[bytes] = None) -> bytes:
    """FLAC bytes of x (channels, n) with every frame written as its FrameSpec says (default: `block_size` blocks,
    order-8 LPC, independent channels)."""
    x = np.asarray(x, np.int64)
    nch, n = x.shape
    if frames is None:
        frames = [FrameSpec(min(block_size, n - s)) for s in range(0, n, block_size)]
    assert sum(f.bs for f in frames) == n
    ff, s = [], 0
    for i, f in enumerate(frames):
        blk = x[:, s:s + f.bs]
        subs = f.sub if isinstance(f.sub, list) else [f.sub] * nch
        if f.stereo == "independent":
            chans, side, code = list(blk), [0] * nch, nch - 1
        else:
            assert nch == 2
            chans, side = stereo_channels(blk, f.stereo)
            code = STEREO[f.stereo]
        hdr = frame_header(s if variable else i, f.bs, sample_rate, code, bps, variable, f)
        ff.append(_frame_fields(hdr, [subframe_fields(c, bps + sd, sp) for c, sd, sp in zip(chans, side, subs)]))
        s += f.bs
    return _stream(x, sample_rate, bps, ff, [f.bs for f in frames], blocks, id3, total_samples, md5)


def _libflac_precision(bps: int, bs: int) -> int:
    if bps < 16:
        return max(5, 2 + bps // 2)
    if bps == 16:
        for lim, p in ((192, 7), (384, 8), (576, 9), (1152, 10), (2304, 11), (4608, 12)):
            if bs <= lim:
                return p
        return 13
    return 15 if bs > 384 else 14


def encode_libflac(x: np.ndarray, sample_rate: int, bps: int, block_size: int = 4096) -> bytes:
    """libFLAC's default layout, with the analysis vectorised over the full-size frames."""
    x = np.asarray(x, np.int64)
    nch, n = x.shape
    nfull = n // block_size
    spec = FrameSpec(block_size)
    prec = _libflac_precision(bps, block_size)
    modes = ["independent"] * nfull
    rows, sides = [], []
    if nfull:
        X = x[:, :nfull * block_size].reshape(nch, nfull, block_size)
        if nch == 2:
            L, R = X[0], X[1]
            cand = {"L": L, "R": R, "M": (L + R) >> 1, "S": L - R}
            est = {k: np.abs(np.diff(v, n=2, axis=1)).sum(1) for k, v in cand.items()}
            costs = np.stack([est["L"] + est["R"], est["L"] + est["S"], est["S"] + est["R"], est["M"] + est["S"]])
            pick = costs.argmin(0)
            names = ["independent", "left_side", "side_right", "mid_side"]
            pairs = [("L", "R"), ("L", "S"), ("S", "R"), ("M", "S")]
            modes = [names[p] for p in pick]
            c0 = np.select([pick[:, None] == i for i in range(4)], [cand[a] for a, _ in pairs])
            c1 = np.select([pick[:, None] == i for i in range(4)], [cand[b] for _, b in pairs])
            rows = [c0, c1]
            sides = [np.isin(pick, [2]).astype(int), np.isin(pick, [1, 3]).astype(int)]
        else:
            rows = [X[c] for c in range(nch)]
            sides = [np.zeros(nfull, int)] * nch
    ff = []
    if nfull:
        order = 8
        per_ch = []
        for c in range(nch):
            Xc = rows[c]
            q, shift = quantize_coefs(lpc_coefs(Xc, order), prec)
            E = lpc_residual(Xc, q, shift)
            u = zigzag(np.concatenate([np.zeros((nfull, order), np.int64), E], 1))
            po, params, _ = rice_plan(u, order, 6, 14, 4)
            per_ch.append((Xc, q, shift, E, po, params))
        for i in range(nfull):
            subs = []
            for c in range(nch):
                Xc, q, shift, E, po, params = per_ch[c]
                sbps = bps + int(sides[c][i])
                xi = Xc[i]
                if (xi == xi[0]).all():
                    subs.append(subframe_fields(xi, sbps, SubSpec("constant", wasted=0)))
                    continue
                e = E[i]
                if e.min() < -(1 << 31) or e.max() >= (1 << 31):
                    subs.append(subframe_fields(xi, sbps, SubSpec("verbatim", wasted=0)))
                    continue
                head = _subframe_header(31 + order, 0) + [_fields(xi[:order], sbps), _fields([prec - 1], 4),
                                                          _fields([shift[i]], 5), _fields(q[i], prec)]
                subs.append(_cat(head + [residual_fields(e, block_size, order, int(po[i]), params[i], 4)]))
            code = nch - 1 if modes[i] == "independent" else STEREO[modes[i]]
            ff.append(_frame_fields(frame_header(i, block_size, sample_rate, code, bps, False, spec), subs))
    if n > nfull * block_size:
        tail = x[:, nfull * block_size:]
        bs = tail.shape[1]
        o = min(8, bs // 2)
        sub = SubSpec("lpc", order=o, precision=prec, wasted=0, max_partition_order=0) if o >= 1 else \
            SubSpec("verbatim", wasted=0)
        chans, side, code = list(tail), [0] * nch, nch - 1
        ff.append(_frame_fields(frame_header(nfull, bs, sample_rate, code, bps, False, FrameSpec(bs)),
                                [subframe_fields(c, bps + sd, sub) for c, sd in zip(chans, side)]))
    bss = [block_size] * nfull + ([n - nfull * block_size] if n > nfull * block_size else [])
    blocks = [("VORBIS_COMMENT", vorbis_comment()), ("PADDING", bytes(8192))]
    return _stream(x, sample_rate, bps, ff, bss, blocks, b"", None, None, seek_every=10 * sample_rate)
