"""CTM + RTTM -> STM: which speaker said each word.  Host-side restatement of the reference's
diarization/assign_words2speakers.py (speaker_for_segment :24-61, main :64-87).

The reference keeps the speaker turns in an `intervaltree.IntervalTree` (third-party, intervaltree==3.1.0 pinned in
diarization/requirements.txt:2, absent here); the three operations it uses are restated on sorted numpy arrays:

  * `tree[a:b]`            -> turns with `begin < b and end > a` (half-open overlap; empty when `a >= b`, i.e. for a
                              zero-duration word — intervaltree's `overlap()` returns set() then)
  * `Interval.distance_to` -> 0 when the two intervals overlap, else the gap between them
  * `IntervalTree(...)`    -> rejects null intervals (`begin >= end` raises ValueError) and stores DISTINCT
                              (begin, end, data) triples (it is a set)

Tie-breaking: the reference iterates Python sets of `Interval` namedtuples, whose order depends on the per-process
string-hash seed, so on exact ties (equal distance to two turns, equal overlap with two speakers) its answer is not
reproducible.  Here ties go to the EARLIEST turn (smallest (begin, end, label)) — one of the answers the reference can
give.  Everything else is deterministic and identical.
"""
from __future__ import annotations

import csv
import io
from typing import Iterable, Iterator, List, Sequence, TextIO, Tuple

import numpy as np

from .rttm import Turn, load_rttm, write_rttm


def read_ctm(ctm_path: str) -> Iterator[List[str]]:
    """assign_words2speakers.py:17-21: space-delimited rows `<file> <channel> <start> <dur> <token> <conf>`."""
    with open(ctm_path, "r") as f:
        for row in csv.reader(f, delimiter=" "):
            yield row


class SpeakerIndex:
    """The `IntervalTree(Interval(start, end, label) ...)` of assign_words2speakers.py:80-81."""

    def __init__(self, turns: Iterable[Sequence]):
        uniq = sorted({(float(b), float(e), str(lab)) for b, e, lab in turns})
        for b, e, _ in uniq:
            if not b < e:      # intervaltree: "IntervalTree: Null Interval objects not allowed in IntervalTree"
                raise ValueError(f"IntervalTree: Null Interval objects not allowed in IntervalTree: Interval({b}, {e})")
        self.begin = np.array([t[0] for t in uniq], dtype=np.float64)
        self.end = np.array([t[1] for t in uniq], dtype=np.float64)
        self.label = [t[2] for t in uniq]

    def __len__(self) -> int:
        return len(self.label)

    def overlap(self, a: float, b: float) -> np.ndarray:
        """indices of the turns `tree[a:b]` returns"""
        if a >= b:
            return np.zeros(0, dtype=np.int64)
        return np.nonzero((self.begin < b) & (self.end > a))[0]


def speaker_for_segment(start: float, dur: float, tree: SpeakerIndex) -> str:
    """assign_words2speakers.py:24-61.  One overlapping turn -> its speaker; none -> the nearest turn's speaker
    ("" when there are no turns at all); several -> the speaker with the largest total overlap."""
    a, b = start, start + dur
    hit = tree.overlap(a, b)
    if len(hit) == 1:
        return tree.label[int(hit[0])]
    if len(hit) == 0:
        if len(tree) == 0:
            return ""
        # Interval(a, b).distance_to(turn): 0 if they overlap (begin < b and end > a), else the gap
        ov = (tree.begin < b) & (tree.end > a)
        gap = np.where(a < tree.begin, tree.begin - b, a - tree.end)
        dist = np.where(ov, 0.0, gap)
        return tree.label[int(np.argmin(dist))]            # first minimum = earliest turn
    sizes = {}
    for i in hit:                                           # ascending (begin, end, label): insertion order of ties
        i0, i1 = max(a, tree.begin[i]), min(b, tree.end[i])
        sizes[tree.label[int(i)]] = sizes.get(tree.label[int(i)], 0) + (i1 - i0)
    return max(sizes, key=sizes.get)


def assign_words_to_speakers(ctm_rows: Iterable[Sequence[str]], turns: Iterable[Turn], uri: str) -> List[str]:
    """assign_words2speakers.py:83-87: one STM line per CTM row,
    `<uri> 1 <speaker> <start:.3f> <end:.3f> <token>` (the CTM's own file / channel / confidence are dropped)."""
    tree = SpeakerIndex((t.start, t.end, t.label) for t in turns)
    out = []
    for _, _channel, start, dur, token, _ in ctm_rows:
        start, dur = float(start), float(dur)
        spk = speaker_for_segment(start, dur, tree)
        out.append(f"{uri} 1 {spk} {start:.3f} {(start + dur):.3f} {token}")
    return out


def write_stm(diarization_rttm: str, ctm_transcription: str, output_stm_transcription: str) -> None:
    """The reference script end to end (assign_words2speakers.py:64-87); the RTTM must hold exactly one uri."""
    rttm = load_rttm(diarization_rttm)
    keys = list(rttm.keys())
    assert len(keys) == 1, keys
    lines = assign_words_to_speakers(read_ctm(ctm_transcription), rttm[keys[0]], keys[0])
    with open(output_stm_transcription, "w") as f:
        for ln in lines:
            f.write(ln + "\n")


def rttm_text(uri: str, turns: Iterable[Turn]) -> str:
    """What `diarization.infer` writes to `<uri>.rttm` for these turns."""
    f = io.StringIO()
    write_rttm(f, uri, turns)
    return f.getvalue()


def stm_text(uri: str, rttm: str, ctm: str) -> str:
    """`write_stm` on an RTTM of `uri` and a CTM held in memory -> the text it writes.  Both go through the same readers
    as the files (the RTTM through load_rttm, the CTM through the csv reader with universal newlines), so the STM is
    byte-identical to the one the file chain writes.  An RTTM without turns (where write_stm finds no uri) gives every
    word the speaker ""."""
    parsed = load_rttm(io.StringIO(rttm))
    assert list(parsed.keys()) in ([], [uri]), list(parsed.keys())
    turns = parsed.get(uri, [])
    rows = csv.reader(io.StringIO(ctm, newline=None), delimiter=" ")
    return "".join(ln + "\n" for ln in assign_words_to_speakers(rows, turns, uri))


def main(argv=None) -> None:
    import argparse
    parser = argparse.ArgumentParser("Assign words to speakers based on a diarization rttm file and ctm transcription")
    parser.add_argument("diarization_rttm", help="diarization rttm file")
    parser.add_argument("ctm_transcription", help="ctm transcription file")
    parser.add_argument("output_stm_transcription", help="output file in .stm format")
    args = parser.parse_args(argv)
    write_stm(args.diarization_rttm, args.ctm_transcription, args.output_stm_transcription)


if __name__ == "__main__":
    main()
