"""Batch planning for many recordings in one call (`ReverbASR.transcribe_files`).

Every recording is cut into chunks exactly as `ReverbASR.feats_batcher` cuts it: `chunk_size` feature frames each, the
last one shorter.  Chunks are independent units, so a batch may hold chunks of several recordings, and the tail
chunks need not be padded to `chunk_size`: a batch of tails runs at its own length `T_b` (`batch_frames`), chosen so
that every value a valid encoder row reads is still computed, by the same kernels from the same inputs (DESIGN.md §4f).

Recordings are taken in input order into windows (the recordings whose features are on the device at once) of at most
`window_frames()` feature frames; a longer recording is a window of its own.  Within a window, `plan_window` makes
    * the full-length chunks, in (recording, chunk) order, `batch_size` at a time, at `T = chunk_size`;
    * the tail chunks, longest first, `batch_size` at a time, each batch at its own `T_b`;
and puts the batch with the largest B * T first, so that the engine's workspaces grow once per window.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import List, Sequence, Tuple

WINDOW_BATCHES = 16          # a window holds up to this many full batches of features


def window_frames(batch_size: int, chunk_size: int) -> int:
    """Frame budget of one window.  Results do not depend on it; it bounds the features held on the device."""
    return WINDOW_BATCHES * batch_size * chunk_size


def encoder_out_frames(T: int) -> int:
    """Encoder frames of a T-frame batch (Conv2dSubsampling4; engine.cu rvb_encoder_out_frames)."""
    if T < 3:
        return 0
    t1 = (T - 1) // 2
    return 0 if t1 < 1 else (t1 - 1) // 2


def encoder_out_len(feat_len: int, T: int) -> int:
    """Valid encoder frames of a chunk of `feat_len` frames in a T-frame batch (engine.cu rvb_encoder_out_len)."""
    feat_len = min(feat_len, T)
    e = (feat_len - 3) // 4 if feat_len >= 7 else 0
    return min(e, encoder_out_frames(T))


def right_context(encoder_conf: dict) -> int:
    """Frames to the right that one conformer convolution module reads: (K - 1) / 2, or 0 when it is causal."""
    return 0 if encoder_conf.get("causal", False) else (int(encoder_conf.get("cnn_module_kernel", 15)) - 1) // 2


def chunk_lengths(n_frames: int, chunk_size: int) -> List[int]:
    """Feature frames of each chunk of an n-frame recording, as feats_batcher cuts it."""
    full, rest = divmod(n_frames, chunk_size)
    return [chunk_size] * full + ([rest] if rest else [])


def batch_frames(lens: Sequence[int], chunk_size: int, right: int, trim: bool = True) -> int:
    """The length T_b to run a batch of chunks with `lens` feature frames at.

    The smallest T_b with T_b >= max(lens) (and >= 7, the shortest input of the subsampling) whose encoder frame count
    covers min(T'_ref, max e + right), where T'_ref is the encoder frame count of `chunk_size` and e a chunk's valid
    encoder frames: valid rows read nothing beyond that (DESIGN.md §4f).  `trim=False` gives `chunk_size`."""
    if not trim:
        return chunk_size
    t_ref = encoder_out_frames(chunk_size)
    need = min(t_ref, max(encoder_out_len(n, chunk_size) for n in lens) + right)
    # encoder_out_frames(T) >= need  <=>  T >= 4 * need + 3
    return min(chunk_size, max(max(lens), 7, 4 * need + 3))


@dataclass
class Batch:
    T: int                              # frames per row of the batch tensor
    slots: List[Tuple[int, int]]        # (recording index within the window, chunk index) of each row
    lens: List[int]                     # feature frames of each row's chunk


def plan_window(rec_frames: Sequence[int], chunk_size: int, batch_size: int, right: int,
                trim: bool = True) -> List[Batch]:
    """Batches of one window of recordings with `rec_frames` feature frames each; every chunk is in exactly one."""
    full, tails = [], []
    for r, n in enumerate(rec_frames):
        for c, fl in enumerate(chunk_lengths(n, chunk_size)):
            (full if fl == chunk_size else tails).append((r, c, fl))
    tails.sort(key=lambda s: -s[2])           # stable: equal lengths stay in (recording, chunk) order
    batches = []
    for group, is_tail in ((full, False), (tails, True)):
        for i in range(0, len(group), batch_size):
            part = group[i:i + batch_size]
            lens = [fl for _, _, fl in part]
            T = batch_frames(lens, chunk_size, right, trim) if is_tail else chunk_size
            batches.append(Batch(T, [(r, c) for r, c, _ in part], lens))
    if batches:
        big = max(range(len(batches)), key=lambda i: len(batches[i].slots) * batches[i].T)
        batches.insert(0, batches.pop(big))
    return batches


class WindowPacker:
    """Groups recordings, in input order, into windows of at most `budget` feature frames."""

    def __init__(self, budget: int):
        self.budget = budget
        self.items: list = []
        self.frames = 0

    def add(self, frames: int, item):
        """Adds a recording; returns the window it closes (a list of items), or None."""
        done = None
        if self.items and self.frames + frames > self.budget:
            done = self.flush()
        self.items.append(item)
        self.frames += frames
        return done

    def flush(self) -> list:
        done, self.items, self.frames = self.items, [], 0
        return done
