"""RTTM reading / writing — the exchange format between the diarization pipeline and the word assignment.

Reference: diarization/infer_pyannote3.0.py:40-42 (`annotation.write_rttm(f)`, pyannote.core.Annotation) and
diarization/assign_words2speakers.py:75-81 (`pyannote.database.util.load_rttm` + `itertracks(yield_label=True)`).
pyannote is a third-party dependency not vendored in the reference repository (diarization/requirements.txt:1 pins
pyannote.audio==3.3.1); its published RTTM conventions are restated here:

    SPEAKER <uri> 1 <start:.3f> <duration:.3f> <NA> <NA> <label> <NA> <NA>

one line per speaker turn, turns iterated in (start, end) order.
"""
from __future__ import annotations

from collections import OrderedDict
from typing import Dict, Iterable, List, NamedTuple, TextIO, Union


class Turn(NamedTuple):
    start: float
    end: float
    label: str


def load_rttm(path_or_file: Union[str, TextIO]) -> "OrderedDict[str, List[Turn]]":
    """uri -> speaker turns sorted by (start, end) (what `load_rttm(...)[uri].itertracks(yield_label=True)` yields).
    Only `SPEAKER` records are kept, like pyannote's loader (it reads the columns by position: type, uri, channel,
    start, duration, NA, NA, speaker, NA, NA)."""
    close = False
    f = path_or_file
    if isinstance(path_or_file, (str, bytes)) or hasattr(path_or_file, "__fspath__"):
        f, close = open(path_or_file, "r"), True
    out: "OrderedDict[str, List[Turn]]" = OrderedDict()
    try:
        for ln in f:
            p = ln.split()
            if len(p) < 8 or p[0] != "SPEAKER":
                continue
            start, dur = float(p[3]), float(p[4])
            out.setdefault(p[1], []).append(Turn(start, start + dur, p[7]))
    finally:
        if close:
            f.close()
    for turns in out.values():
        turns.sort(key=lambda t: (t.start, t.end))
    return out


def write_rttm(f: TextIO, uri: str, turns: Iterable[Turn]) -> None:
    """pyannote.core.Annotation.write_rttm: one SPEAKER line per turn, (start, end) order, 3 decimals."""
    for t in sorted(turns, key=lambda t: (t.start, t.end)):
        f.write(f"SPEAKER {uri} 1 {t.start:.3f} {t.end - t.start:.3f} <NA> <NA> {t.label} <NA> <NA>\n")
