"""Token -> word assembly with CTC peak timestamps, and CTM / TXT rendering (host, pure Python).

Behavioural mirror of asr/wenet/bin/ctc_align.py (`ctc_align` :24-113,
`adjust_model_time_offset` :116-138) and asr/wenet/cli/utils.py (`hyps_to_ctm`, `hyps_to_txt`);
SURVEY.md Appendix A.5 states the rules.  Written from the behaviour, checked against the
reference's CTM strings in tests/golden/*.json.
"""
from __future__ import annotations

from typing import Any, Dict, Iterator, List, Optional

SPACE = "▁"
GAP_MS = 100


def _is_special(piece: str) -> bool:
    lo, hi = piece.find("<"), piece.find(">")
    return lo != -1 and hi != -1 and lo < hi


def _starts_word(piece: str) -> bool:
    return SPACE in piece


def ctc_align(tokens, times, confidences: Optional[List[float]], tokenizer, frame_shift_ms: int,
              time_shift_ms: int) -> List[Dict[str, Any]]:
    """Words with start/end (ms) from per-token peak frames.  A word ends when the NEXT piece starts a
    word (contains '▁'), is a <special> piece, or the hypothesis ends; a <special> piece is its own word."""
    if len(tokens) != len(times):           # the reference asserts (ctc_align.py:28); greedy has times=None
        raise AssertionError("ctc_align needs one timestamp per token")
    n = len(tokens)
    pieces = [tokenizer.detokenize([t])[1][0] for t in tokens]
    words: List[Dict[str, Any]] = []
    text, ids, start, first = "", [], -1, -1

    def end_time(i: int) -> int:
        end = times[i] * frame_shift_ms
        if i < n - 1 and (times[i + 1] - times[i]) * frame_shift_ms < GAP_MS:
            end = (times[i + 1] + times[i]) // 2 * frame_shift_ms
        return end

    def conf(lo: int, hi: int):
        return max(confidences[lo:hi + 1]) if confidences else 0

    for i in range(n):
        piece = pieces[i]
        nxt = pieces[i + 1] if i + 1 < n else SPACE
        text += piece[len(SPACE):] if piece.find(SPACE) != -1 else piece
        ids.append(tokens[i])
        if start == -1:
            start = max(times[i] * frame_shift_ms - GAP_MS, 0)
            if i > 0 and (times[i] - times[i - 1]) * frame_shift_ms < GAP_MS:
                start = (times[i - 1] + times[i]) // 2 * frame_shift_ms
            first = i
        if text not in ("", SPACE) and _is_special(text):
            end = end_time(i)
            assert start < end
            assert len(ids) == 1
            words.append({"word": text, "unit_id": ids[0], "start_time_ms": start + time_shift_ms,
                          "end_time_ms": end + time_shift_ms, "confidence": conf(first, i), "unit_ids": ids})
            text, ids, start, first = "", [], -1, 0
        if _starts_word(nxt) or _is_special(nxt):
            end = end_time(i)
            if text not in ("", SPACE):
                assert len(ids) > 0
                assert start <= end
                assert not _is_special(text)
                words.append({"word": text, "unit_id": -1, "start_time_ms": start + time_shift_ms,
                              "end_time_ms": end + time_shift_ms, "confidence": conf(first, i), "unit_ids": ids})
            text, ids, start, first = "", [], -1, 0
    return words


def frames_to_ms(frames, chunk_frames, chunk_ms: int, frame_shift_ms: int) -> List[int]:
    """Frames counted over the VALID encoder frames of consecutive chunks -> milliseconds in the recording.
    chunk_frames[c] = valid frames of chunk c.  Frame j of chunk c sits at c * chunk_ms + j * frame_shift_ms: chunks
    are cut in input frames, and a chunk's encoder frames do not fill it (748 x 40 ms in a 29.98 s chunk), so one
    global multiplication by frame_shift_ms would drift."""
    starts, total = [], 0
    for n in chunk_frames:
        starts.append(total)
        total += int(n)
    out, c = [], 0
    for f in frames:
        f = int(f)
        assert 0 <= f < total
        if f < starts[c]:
            c = 0
        while c + 1 < len(starts) and f >= starts[c + 1]:
            c += 1
        out.append(c * chunk_ms + (f - starts[c]) * frame_shift_ms)
    return out


def ctc_align_ms(tokens, times_ms, confidences: Optional[List[float]], tokenizer, frame_shift_ms: int) -> List[Dict[str, Any]]:
    """ctc_align() for ONE token sequence whose peaks are given in milliseconds of the whole recording (forced alignment
    of a transcript across chunks): a word whose pieces fall on both sides of a chunk boundary stays one word.  Same
    word rules; with all peaks in one chunk it returns what ctc_align(..., time_shift_ms = the chunk's start) does, except
    that a word's 100 ms lead-in is clamped at the start of the recording only, not at the start of every chunk."""
    if len(tokens) != len(times_ms):
        raise AssertionError("ctc_align_ms needs one timestamp per token")
    n = len(tokens)
    pieces = [tokenizer.detokenize([t])[1][0] for t in tokens]
    words: List[Dict[str, Any]] = []
    text, ids, start, first = "", [], -1, -1

    def midpoint(a: int, b: int) -> int:      # (t_a + t_b) // 2 * frame_shift_ms, written on milliseconds
        return a + (b - a) // (2 * frame_shift_ms) * frame_shift_ms

    def end_time(i: int) -> int:
        if i < n - 1 and times_ms[i + 1] - times_ms[i] < GAP_MS:
            return midpoint(times_ms[i], times_ms[i + 1])
        return times_ms[i]

    def conf(lo: int, hi: int):
        return max(confidences[lo:hi + 1]) if confidences else 0

    for i in range(n):
        piece = pieces[i]
        nxt = pieces[i + 1] if i + 1 < n else SPACE
        text += piece[len(SPACE):] if piece.find(SPACE) != -1 else piece
        ids.append(tokens[i])
        if start == -1:
            start = max(times_ms[i] - GAP_MS, 0)
            if i > 0 and times_ms[i] - times_ms[i - 1] < GAP_MS:
                start = midpoint(times_ms[i - 1], times_ms[i])
            first = i
        special = text not in ("", SPACE) and _is_special(text)
        if special or _starts_word(nxt) or _is_special(nxt):
            if text not in ("", SPACE):
                words.append({"word": text, "unit_id": ids[0] if special else -1, "start_time_ms": start,
                              "end_time_ms": end_time(i), "confidence": conf(first, i), "unit_ids": ids})
            text, ids, start, first = "", [], -1, 0
    return words


def adjust_model_time_offset(words: List[Dict[str, Any]], adjustment):
    """Move every word earlier by min(adjustment, gap to the previous word's end).  Like the reference
    (ctc_align.py:117-118) an adjustment of 0 returns None."""
    if adjustment == 0:
        return None
    out = []
    for i, w in enumerate(words):
        assert 0 <= w["start_time_ms"] <= w["end_time_ms"]
        if i == 0:
            shift = min(adjustment, w["start_time_ms"])
        else:
            prev = words[i - 1]
            assert w["start_time_ms"] >= prev["end_time_ms"], f"ERROR! {w} >= {prev}"
            shift = min(adjustment, w["start_time_ms"] - prev["end_time_ms"])
        assert shift >= 0
        w["start_time_ms"] -= shift
        w["end_time_ms"] -= shift
        out.append(w)
    return out


def hyps_to_ctm(audio_name: str, words: List[Dict[str, Any]]) -> Iterator[str]:
    for w in words:
        start = w["start_time_ms"] / 1000
        dur = w["end_time_ms"] / 1000 - start
        yield f"{audio_name} 0 {start:.2f} {dur:.2f} {w['word']} {w['confidence']:.2f}"


def hyps_to_txt(words: List[Dict[str, Any]]) -> Iterator[str]:
    for w in words:
        yield w["word"]
