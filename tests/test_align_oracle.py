"""CTC forced alignment without a GPU: the CPU oracle (oracle/align_ref.py) against the reference's recorded output
(tests/golden/align.*, written by oracle/make_golden_align.py from the live reference), and the host logic around the
kernels — feasibility, frame -> millisecond conversion across chunks, word assembly, CTM text, the command line."""
import json
import os
import types

import numpy as np
import pytest
import torch

from conftest import GOLDEN, load_golden


def align_cases():
    """(case dict, logp (T, V) float32, reference frame alignment) for every pinned case."""
    meta, frames = load_golden("align")
    src = {n: dict(np.load(os.path.join(GOLDEN, n + ".npz"))) for n in ("causal_ln", "sym_bn")}
    out = []
    for i, c in enumerate(meta["cases"]):
        probs, lens = src[c["fixture"]]["ctc_probs_0"], src[c["fixture"]]["enc_lens_0"]
        if c["source"] == "concat":
            logp = np.concatenate([probs[b, :int(lens[b])] for b in range(probs.shape[0])])
        else:
            logp = np.ascontiguousarray(probs[c["source"], :int(lens[c["source"]])])
        out.append((c, logp, frames[f"frames_{i}"]))
    return out


@pytest.fixture(scope="module")
def tokenizer(tmp_path_factory):
    from reverb_b200 import synth
    from reverb_b200.text import PieceTokenizer
    p = tmp_path_factory.mktemp("units") / "tk.units.txt"
    p.write_text("\n".join(synth.make_units(101)) + "\n", encoding="utf8")
    return PieceTokenizer(str(p))


def test_golden_covers_the_required_label_kinds():
    kinds = {c["kind"] for c, _, _ in align_cases()}
    assert {"best", "nbest1", "random", "repeats", "single", "limit", "long"} <= kinds
    for c, logp, _ in align_cases():
        y = c["labels"]
        need = len(y) + sum(a == b for a, b in zip(y[:-1], y[1:]))
        if c["kind"] == "limit":
            assert need == logp.shape[0]
        if c["kind"] == "long":
            assert len(y) + 1 > 128          # more label slots than one warp of the trellis kernel holds (4 per thread)
        if c["kind"] == "single":
            assert len(y) == 1


def test_oracle_equals_the_reference_frame_alignments():
    from oracle import align_ref
    for c, logp, want in align_cases():
        got = align_ref.force_align(logp, c["labels"], 0)
        assert got.dtype == np.int32 and np.array_equal(got, want), (c["fixture"], c["source"], c["kind"])


def test_oracle_path_collapses_to_the_labels_and_spans_are_consistent():
    from oracle import align_ref
    for c, logp, _ in align_cases():
        y = c["labels"]
        r = align_ref.align(logp, y, 0)
        collapsed = [int(t) for i, t in enumerate(r["frames"]) if t != 0 and (i == 0 or r["frames"][i - 1] != t)]
        if not any(a == b for a, b in zip(y[:-1], y[1:])):
            assert collapsed == y
        assert np.all(r["first"] <= r["peak"]) and np.all(r["peak"] <= r["last"])
        assert np.all(r["first"][1:] > r["last"][:-1])
        for u in range(len(y)):
            assert r["peak_logp"][u] == logp[r["peak"][u], y[u]]
            assert np.all(r["frames"][r["first"][u]:r["last"][u] + 1] == y[u])
        # the Viterbi score is the fp32 sum along the path, added in frame order
        states, score = align_ref.viterbi(logp, y, 0)
        z = align_ref.states_of(y, 0)
        acc = np.float32(0)
        for t, s in enumerate(states):
            acc = np.float32(acc + logp[t, z[s]])
        assert acc == score == r["score"]


def test_span_and_peak_reduction_on_hand_cases():
    from oracle import align_ref
    lp = np.full((6, 4), -5.0, dtype=np.float32)
    states = np.array([0, 1, 1, 1, 2, 3], dtype=np.int32)      # blank, y0 x3, blank, y1
    lp[1:4, 2] = [-1.0, -0.5, -0.5]                             # tie between frames 2 and 3: the first one wins
    lp[5, 3] = -0.25
    first, last, peak, plp = align_ref.token_spans(lp, states, [2, 3])
    assert first.tolist() == [1, 5] and last.tolist() == [3, 5] and peak.tolist() == [2, 5]
    assert plp.tolist() == [-0.5, -0.25]


def test_tie_rules_first_maximum_wins():
    from oracle import align_ref
    # uniform log-probs: every path ties, so the choices are exactly the tie rules — the end state is S-1 and the
    # back-trace stays there as long as it can, then takes s-1 before s-2
    lp = np.full((5, 3), -1.0, dtype=np.float32)
    states, score = align_ref.viterbi(lp, [1, 2], 0)
    assert states.tolist() == [1, 3, 4, 4, 4] and score == np.float32(-5.0)
    assert align_ref.force_align(lp, [1], 0).tolist() == [1, 0, 0, 0, 0]
    assert align_ref.viterbi(lp[:, :2], [1, 1], 0)[0].tolist() == [1, 2, 3, 4, 4]      # a repeat has no s-2 arc


def test_loglik_equals_torch_ctc_loss_in_float64():
    from oracle import align_ref
    for c, logp, _ in align_cases():
        if c["kind"] not in ("best", "random", "repeats", "single", "limit", "long"):
            continue
        y = c["labels"]
        want = -torch.nn.functional.ctc_loss(torch.from_numpy(logp).double().unsqueeze(1), torch.tensor([y]),
                                             torch.tensor([logp.shape[0]]), torch.tensor([len(y)]), blank=0,
                                             reduction="sum").item()
        got = align_ref.forward_loglik(logp, y, 0)
        assert abs(got - want) <= 1e-9 * abs(want), (c["kind"], got, want)
        assert align_ref.viterbi(logp, y, 0)[1] <= got + 1e-4


def test_feasibility_rule():
    from oracle import align_ref
    from reverb_b200.engine import check_alignable
    assert align_ref.feasible([5], 1) and not align_ref.feasible([], 10)
    assert align_ref.feasible([5, 6, 7], 3) and not align_ref.feasible([5, 6, 7], 2)
    assert align_ref.feasible([5, 5, 6], 4) and not align_ref.feasible([5, 5, 6], 3)     # a repeat costs a blank frame
    check_alignable([5, 5, 6], 4)
    with pytest.raises(ValueError, match="infeasible"):
        check_alignable([5, 5, 6], 3)
    with pytest.raises(ValueError, match="empty"):
        check_alignable([], 100)
    with pytest.raises(ValueError):
        align_ref.viterbi(np.zeros((3, 4), np.float32), [], 0)


def test_frames_to_ms_respects_chunk_boundaries():
    from reverb_b200.ctc_align import frames_to_ms
    # chunk_size 2998 input frames of 10 ms -> 748 encoder frames of 40 ms: 29.92 s of frames per 29.98 s chunk
    cf = [748, 748, 100]
    assert frames_to_ms([0, 747, 748, 749, 1495, 1496, 1595], cf, 29980, 40) == \
        [0, 29880, 29980, 30020, 29980 + 29880, 59960, 59960 + 99 * 40]
    assert frames_to_ms([748], cf, 29980, 40)[0] != 748 * 40                 # a single global x 40 drifts
    assert frames_to_ms([5, 3], [4, 4], 1000, 40) == [1040, 120]             # any order
    with pytest.raises(AssertionError):
        frames_to_ms([8], [4, 4], 1000, 40)
    assert frames_to_ms([0, 1], [0, 2], 1000, 40) == [1000, 1040]            # a chunk without valid frames


def test_ctc_align_ms_equals_ctc_align_inside_one_chunk(tokenizer):
    from reverb_b200.ctc_align import ctc_align, ctc_align_ms
    rng = np.random.default_rng(3)
    for _ in range(20):
        n = int(rng.integers(1, 25))
        toks = [int(t) for t in rng.integers(2, 100, n)]
        times = (2 + np.cumsum(rng.integers(1, 6, n))).tolist()     # >= 3: ctc_align clamps a lead-in at its chunk's start
        conf = [float(x) for x in rng.random(n)]
        shift = 7 * 20510
        want = ctc_align(toks, times, conf, tokenizer, 40, shift)
        got = ctc_align_ms(toks, [shift + 40 * t for t in times], conf, tokenizer, 40)
        assert got == want


def test_word_straddling_a_chunk_boundary_stays_one_word(tokenizer):
    from reverb_b200.ctc_align import ctc_align_ms, frames_to_ms, hyps_to_ctm
    toks = [3, 4, 7, 6, 8]                      # "▁w3" "p4" "p7" | "▁w6" "p8": two words, the first of three pieces
    pieces = tokenizer.ids2tokens(toks)
    assert pieces[0].startswith("▁") and pieces[3].startswith("▁") and "▁" not in pieces[1] + pieces[2] + pieces[4]
    ms = frames_to_ms([98, 99, 101, 110, 112], [100, 100], 4100, 40)       # pieces 0, 1 in chunk 0, piece 2 in chunk 1
    assert ms == [3920, 3960, 4140, 4500, 4580]
    words = ctc_align_ms(toks, ms, [0.5, 0.9, 0.7, 0.4, 0.3], tokenizer, 40)
    assert [w["word"] for w in words] == ["w3p4p7", "w6p8"]
    assert words[0]["unit_ids"] == [3, 4, 7] and words[0]["confidence"] == 0.9
    assert words[0]["start_time_ms"] == 3820 and words[0]["end_time_ms"] == 4140
    assert words[1]["start_time_ms"] == 4400 and words[1]["end_time_ms"] == 4580
    assert list(hyps_to_ctm("a.wav", words)) == ["a.wav 0 3.82 0.32 w3p4p7 0.90", "a.wav 0 4.40 0.18 w6p8 0.40"]


def test_transcript_string_goes_through_the_sentencepiece_pieces(tokenizer):
    """The synthetic model directories carry an empty tk.model, so the text front-end is exercised with a stand-in for
    the sentencepiece processor whose pieces are looked up in tk.units.txt; unknown pieces stay, as <unk>."""
    from reverb_b200.reverb import ReverbASR

    class Pieces:
        def encode(self, line, out_type=str):
            return [p for w in line.split() for p in ("▁" + w[:2], w[2:]) if p]

    tokenizer._sp = Pieces()
    me = types.SimpleNamespace(tokenizer=tokenizer, blank_id=0)
    assert ReverbASR.transcript_ids(me, "w3p4 w6 zzzz") == [3, 4, 6, 1, 1]
    assert ReverbASR.transcript_ids(me, [3, 4, 6]) == [3, 4, 6]
    with pytest.raises(ValueError, match="empty"):
        ReverbASR.transcript_ids(me, "   ")
    with pytest.raises(ValueError, match="empty"):
        ReverbASR.transcript_ids(me, [])
    with pytest.raises(ValueError, match="non-blank"):
        ReverbASR.transcript_ids(me, [3, 0, 4])
    with pytest.raises(ValueError, match="non-blank"):
        ReverbASR.transcript_ids(me, [3, 101])


def test_cli_arguments(tmp_path):
    from reverb_b200 import align_wav
    base = ["--model", "m", "--audio_file", "a.wav", "--result_dir", str(tmp_path)]
    for bad in (base, base + ["--text_file", "t", "--token_file", "i"], base[2:] + ["--text_file", "t"],
                base + ["--text_file", "t", "--format", "json"]):
        with pytest.raises(SystemExit):
            align_wav.get_args(bad)
    args = align_wav.get_args(base + ["--token_file", "ids.txt", "--chunk_size", "2998", "--batch_size", "4"])
    assert (args.chunk_size, args.batch_size, args.format, args.timings_adjustment) == (2998, 4, "ctm", 230)
    ids = tmp_path / "ids.txt"
    ids.write_text("3 4\n6\n")
    assert align_wav.read_transcript(align_wav.get_args(base + ["--token_file", str(ids)])) == [3, 4, 6]
    ids.write_text("3 four")
    with pytest.raises(ValueError, match="integers"):
        align_wav.read_transcript(align_wav.get_args(base + ["--token_file", str(ids)]))
    txt = tmp_path / "t.txt"
    txt.write_text("hello\n  world \n")
    assert align_wav.read_transcript(align_wav.get_args(base + ["--text_file", str(txt)])) == "hello world"
    txt.write_text(" \n")
    with pytest.raises(ValueError, match="empty"):
        align_wav.main(base + ["--text_file", str(txt)])


def test_alignment_entry_points_are_bound():
    from reverb_b200 import _lib
    lib = _lib.load()
    for name in ("rvb_ctc_force_align", "rvb_aligner_workspace_bytes", "rvb_aligner_begin", "rvb_aligner_push",
                 "rvb_aligner_finish", "rvb_aligner_abort"):
        assert getattr(lib, name).argtypes == _lib.SIGNATURES[name][1]
    from reverb_b200.engine import Aligner
    # about 5 bytes per frame and label slot: one hour (90 000 frames) against 12 000 tokens
    need = Aligner.workspace_bytes(12000, 90000)
    assert 5.3e9 < need < 5.7e9
    assert Aligner.workspace_bytes(12000, 90000, True) > need
    assert Aligner.workspace_bytes(0, 100) == -1 and Aligner.workspace_bytes(12288, 100000) == -1
    assert json.dumps(need)
