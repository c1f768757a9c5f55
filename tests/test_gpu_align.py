"""CTC forced alignment on the GPU (csrc/align.cu behind rvb_ctc_force_align / rvb_aligner_*): the kernels against the
reference's recorded alignments (tests/golden/align.*) and against the CPU oracle on GPU-produced log-probs.

Bars: frame alignment, spans and peaks identical, Viterbi score bit-equal fp32 (the trellis is fp32 max + one add per
cell, so nothing depends on evaluation order); log-likelihood within 1e-9 relative (CUDA fp64 exp / log vs glibc).
"""
import os

import numpy as np
import pytest
import torch

from test_align_oracle import align_cases

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def asr(model_dirs):
    import reverb_b200
    return {n: reverb_b200.load_model(d) for n, (d, _) in model_dirs.items()}


@pytest.fixture(scope="module")
def bench_asr(tmp_path_factory):
    """The benchmarked shape (reverb_asr_v1-like: d=1024, 18 blocks, V=10001), the weights bench.py times."""
    import reverb_b200
    from reverb_b200 import synth
    d = str(tmp_path_factory.mktemp("bench_shape_align"))
    synth.write_model_dir(d, shape=synth.BENCH_SHAPE, seed=0, causal=True, cnn_module_norm="layer_norm", reverse_weight=0.3)
    return reverb_b200.load_model(d), d


def same_as_oracle(got, logp, labels, loglik=False):
    """got: engine.Alignment; logp (T, V) float32 numpy."""
    from oracle import align_ref
    want = align_ref.align(logp, labels, 0)
    assert np.array_equal(got.frames, want["frames"])
    for k in ("first", "last", "peak"):
        assert np.array_equal(getattr(got, k), want[k]), k
    assert got.peak_logp.tobytes() == want["peak_logp"].tobytes()
    assert np.float32(got.score).tobytes() == np.float32(want["score"]).tobytes()
    if loglik:
        ll = align_ref.forward_loglik(logp, labels, 0)
        assert abs(got.loglik - ll) <= 1e-9 * abs(ll)


def random_labels(rng, n, V, repeats=False):
    """Ids in [1, V - 2] that are not <special> pieces (synth.make_units: id % 17 == 5); adjacent repeats only on demand."""
    y = [int(x) for x in rng.integers(1, V - 1, n)]
    for i in range(n):
        if y[i] % 17 == 5:
            y[i] += 1
        if i and repeats and i % 5 == 0:
            y[i] = y[i - 1]
        elif i and y[i] == y[i - 1]:
            y[i] = y[i] - 2 if y[i] > 2 and (y[i] - 2) % 17 != 5 else y[i] + 2
    return y


def test_kernel_equals_the_reference_alignments(asr):
    eng = asr["causal_ln"].engine
    for c, logp, want in align_cases():
        got = eng.force_align(torch.from_numpy(logp).cuda().unsqueeze(0), [logp.shape[0]], [c["labels"]], 0, True)[0]
        assert np.array_equal(got.frames, want), (c["fixture"], c["source"], c["kind"])
        same_as_oracle(got, logp, c["labels"], loglik=True)


def test_batched_form_with_padding_and_mixed_lengths(asr):
    """Utterances of different length and label count in one call: every CTA sees only its own rows and labels."""
    eng = asr["sym_bn"].engine
    cases = [x for x in align_cases() if x[0]["fixture"] == "sym_bn" and x[0]["kind"] in ("best", "repeats", "single", "limit")]
    Tp = max(lp.shape[0] for _, lp, _ in cases) + 3
    batch = np.full((len(cases), Tp, cases[0][1].shape[1]), -1.0, dtype=np.float32)
    for b, (_, lp, _) in enumerate(cases):
        batch[b, :lp.shape[0]] = lp
    got = eng.force_align(torch.from_numpy(batch).cuda(), [lp.shape[0] for _, lp, _ in cases],
                          [c["labels"] for c, _, _ in cases], 0, True)
    for (c, lp, want), g in zip(cases, got):
        assert np.array_equal(g.frames, want)
        same_as_oracle(g, lp, c["labels"], loglik=True)


def test_resumable_form_equals_one_shot_and_handles_do_not_interfere(asr):
    eng = asr["causal_ln"].engine
    rng = np.random.default_rng(2)
    T, V = 700, eng.vocab
    logp = torch.log_softmax(torch.from_numpy(rng.standard_normal((2, T, V)).astype(np.float32)) * 3, dim=-1).cuda()
    ya, yb = random_labels(rng, 300, V, repeats=True), random_labels(rng, 40, V)
    one_a, one_b = eng.force_align(logp, [T, T], [ya, yb], 0, True)
    for side in (True, False):
        a = eng.aligner(ya, T, 0, True, side_stream=side)
        b = eng.aligner(yb, T, 0, True, side_stream=side)
        a.push(logp[0, :1])
        b.push(logp[1, :333])
        a.push(logp[0, 1:301])
        b.push(logp[1, 333:])
        a.push(logp[0, 301:])
        ra, rb = a.finish(), b.finish()
        for r, one in ((ra, one_a), (rb, one_b)):
            assert np.array_equal(r.frames, one.frames) and np.array_equal(r.peak, one.peak)
            assert np.array_equal(r.first, one.first) and np.array_equal(r.last, one.last)
            assert r.peak_logp.tobytes() == one.peak_logp.tobytes()
            assert np.float32(r.score).tobytes() == np.float32(one.score).tobytes()
            assert r.loglik == one.loglik
    same_as_oracle(one_a, logp[0].cpu().numpy(), ya, loglik=True)
    same_as_oracle(one_b, logp[1].cpu().numpy(), yb, loglik=True)


def test_long_label_sequences_use_the_wide_kernel(asr):
    """More than 4095 labels: 24 label slots per thread instead of 4."""
    eng = asr["causal_ln"].engine
    rng = np.random.default_rng(4)
    T, V, U = 5400, eng.vocab, 4300
    logp = torch.log_softmax(torch.from_numpy(rng.standard_normal((T, V)).astype(np.float32)) * 2, dim=-1).cuda()
    y = random_labels(rng, U, V, repeats=True)
    al = eng.aligner(y, T, 0, True)
    for lo, hi in ((0, 1), (1, 1200), (1200, T)):
        al.push(logp[lo:hi])
    same_as_oracle(al.finish(), logp.cpu().numpy(), y, loglik=True)


@pytest.mark.parametrize("precision", ["bf16", "fp32"])
def test_model_align_equals_the_oracle_on_gpu_logprobs(model_dirs, golden_cases, precision):
    import reverb_b200
    from reverb_b200.ctc_align import ctc_align
    from reverb_b200.reverb import get_output
    meta, arr = golden_cases["causal_ln"]
    m = reverb_b200.load_model(model_dirs["causal_ln"][0], precision=precision)
    cat = torch.tensor([meta["verbatimicity"], 1.0 - meta["verbatimicity"]])
    feats = torch.from_numpy(arr["feats"]).unsqueeze(0).cuda()
    rng = np.random.default_rng(6)
    fb, fl = next(iter(m.feats_batcher(feats, meta["chunk_size"], meta["batch_size"])))
    enc, enc_lens = m.model._forward_encoder(fb, fl, cat)
    logp = m.model.ctc_logprobs(enc).cpu().numpy()
    labels = [random_labels(rng, 20 + 7 * b, m.engine.vocab, repeats=True) for b in range(fb.shape[0])]
    tok = np.zeros((fb.shape[0], max(map(len, labels))), dtype=np.int64)
    for b, y in enumerate(labels):
        tok[b, :len(y)] = y
    res = m.model.align(fb, fl, torch.from_numpy(tok), torch.tensor([len(y) for y in labels]), 0, cat, want_loglik=True)
    from oracle import align_ref
    for b, r in enumerate(res):
        T = int(enc_lens[b])
        want = align_ref.align(logp[b, :T], labels[b], 0)
        assert np.array_equal(r.alignment, want["frames"]) and r.times == want["peak"].tolist()
        assert r.tokens == labels[b] and np.float32(r.score).tobytes() == np.float32(want["score"]).tobytes()
        np.testing.assert_allclose(r.tokens_confidence, np.exp(want["peak_logp"].astype(np.float64)), rtol=1e-12)
        assert abs(r.confidence - np.exp(float(want["score"]) / T)) < 1e-12
        ll = align_ref.forward_loglik(logp[b, :T], labels[b], 0)
        assert abs(r.loglik - ll) <= 1e-9 * abs(ll)
    # times and confidences are filled, so the result renders through get_output like a search result
    text = get_output("ctm", m.tokenizer, "a.wav", res, 230, meta["chunk_size"], 10, 40)
    assert len(text.split("\n")) == sum(len(ctc_align(r.tokens, r.times, r.tokens_confidence, m.tokenizer, 40, 0)) for r in res)


def test_aligning_the_prefix_search_best_hypothesis_is_self_consistent(asr, golden_cases):
    from oracle.search_ref import remove_duplicates_and_blank
    for case in ("causal_ln", "sym_bn"):
        meta, arr = golden_cases[case]
        m = asr[case]
        cat = torch.tensor([meta["verbatimicity"], 1.0 - meta["verbatimicity"]])
        feats = torch.from_numpy(arr["feats"]).unsqueeze(0).cuda()
        for fb, fl in m.feats_batcher(feats, meta["chunk_size"], meta["batch_size"]):
            enc, enc_lens = m.model._forward_encoder(fb, fl, cat)
            val, idx, logp = m.engine.ctc_topk(enc, 10, want_logp=True)
            pb = m.engine.prefix_beam_search(val, idx, enc_lens, 10, 0)
            keep = [b for b in range(fb.shape[0]) if len(pb[b][0][0])]
            if not keep:
                continue
            got = m.engine.force_align(logp[keep], enc_lens[keep], [list(pb[b][0][0]) for b in keep], 0, True)
            for b, g in zip(keep, got):
                assert remove_duplicates_and_blank(g.frames.tolist(), 0) == list(pb[b][0][0])
                # one path <= all paths of y; the prefix score sums the paths of y that stayed in the beam (and only the
                # top-10 tokens of a frame), so it is a lower bound of log p(y | x) as well
                assert g.score <= g.loglik + 1e-4
                assert pb[b][1][0] <= g.loglik + 1e-9 * abs(g.loglik)


def _multi_chunk_wav(m, d, seconds, seed):
    from reverb_b200 import synth
    return synth.write_wav(os.path.join(d, f"long_{seed}.wav"), synth.synth_audio(seconds, seed=seed))


def _valid_logp(m, wav, chunk_size, batch_size, verbatimicity=1.0):
    """The concatenated valid log-prob rows of every chunk, and the valid frames per chunk."""
    feats = m.compute_feats(wav, num_mel_bins=80, frame_length=25, frame_shift=10)
    cat = torch.tensor([verbatimicity, 1.0 - verbatimicity])
    rows, frames = [], []
    for fb, fl in m.feats_batcher(feats, chunk_size, batch_size):
        enc, enc_lens = m.model._forward_encoder(fb, fl, cat)
        logp = m.model.ctc_logprobs(enc, 0.0, m.blank_id)
        for b in range(fb.shape[0]):
            rows.append(logp[b, :int(enc_lens[b])].cpu().numpy())
            frames.append(int(enc_lens[b]))
    return np.concatenate(rows), frames


def test_reverb_align_across_chunks(asr, model_dirs):
    from oracle import align_ref
    from reverb_b200.ctc_align import adjust_model_time_offset, ctc_align_ms, frames_to_ms, hyps_to_ctm
    m = asr["causal_ln"]
    wav = _multi_chunk_wav(m, model_dirs["causal_ln"][0], 21.7, 77)        # 5 chunks of 4.1 s + a tail chunk
    chunk = 410
    logp, frames = _valid_logp(m, wav, chunk, 1)
    assert len(frames) == 6 and frames[-1] < frames[0]
    bounds = np.cumsum(frames)[:-1]
    for seed in range(20):
        rng = np.random.default_rng(seed)
        # word-initial pieces are the ids divisible by 3 (synth.make_units): words of 2-4 pieces, one <special> piece
        ids = []
        while len(ids) < 150:
            ids += [int(3 * rng.integers(1, 30))] + [int(3 * rng.integers(1, 30) + 1) for _ in range(rng.integers(1, 4))]
        ids[40] = 22                                                       # "<sp22>"
        want = align_ref.align(logp, ids, 0)
        chunk_of = np.searchsorted(bounds, want["peak"], side="right")
        pos, straddles = 0, 0
        for w in ctc_align_ms(ids, want["peak"].tolist(), None, m.tokenizer, 40):
            straddles += chunk_of[pos] != chunk_of[pos + len(w["unit_ids"]) - 1]
            pos += len(w["unit_ids"])
        if straddles:
            break
    assert straddles, "no label set put a multi-piece word across a chunk boundary"
    ms = frames_to_ms(want["peak"], frames, chunk * 10, 40)
    words = adjust_model_time_offset(ctc_align_ms(ids, ms, np.exp(want["peak_logp"].astype(np.float64)).tolist(),
                                                  m.tokenizer, 40), 230)
    ctm = {bs: m.align(wav, ids, chunk_size=chunk, batch_size=bs) for bs in (1, 4)}
    assert ctm[1] == ctm[4]
    assert ctm[1] == "\n".join(hyps_to_ctm(os.path.basename(wav), words))
    starts = [float(line.split()[2]) for line in ctm[1].split("\n")]
    assert starts == sorted(starts) and len(starts) == len(words)
    # no word is split where its pieces straddle a chunk boundary: the words are those of the token sequence
    assert m.align(wav, ids, format="txt", chunk_size=chunk) == " ".join(w["word"] for w in words)
    res, times_ms = m.align_tokens(wav, ids, chunk_size=chunk, batch_size=4, want_loglik=True)
    assert times_ms == ms and np.array_equal(res.alignment, want["frames"])
    ll = align_ref.forward_loglik(logp, ids, 0)
    assert abs(res.loglik - ll) <= 1e-9 * abs(ll)


def test_align_wav_command_line(asr, model_dirs, tmp_path):
    from reverb_b200 import align_wav
    d, wav = model_dirs["sym_bn"]
    ids = [3, 4, 7, 6, 8, 9, 10, 22, 12, 13]
    tok = tmp_path / "ids.txt"
    tok.write_text(" ".join(map(str, ids)))
    out = align_wav.main(["--model", d, "--audio_file", wav, "--token_file", str(tok), "--result_dir", str(tmp_path),
                          "--chunk_size", "400", "--batch_size", "2"])
    assert out == str(tmp_path / "alignment" / "golden.ctm")
    words = [line.split()[4] for line in open(out).read().split("\n")]
    assert words == ["w3p4p7", "w6p8", "w9p10", "<sp22>", "w12p13"]


def test_errors_are_raised_before_any_launch(asr):
    from reverb_b200.engine import Aligner, launch_count
    m = asr["causal_ln"]
    eng = m.engine
    logp = torch.log_softmax(torch.randn(1, 20, eng.vocab, device="cuda"), dim=-1)
    torch.cuda.synchronize()
    before = launch_count()
    with pytest.raises(ValueError, match="infeasible"):
        eng.force_align(logp, [20], [[5] * 11], 0)            # 11 labels + 10 repeats need 21 frames
    with pytest.raises(ValueError, match="empty"):
        eng.force_align(logp, [20], [[]], 0)
    with pytest.raises(ValueError, match="infeasible"):
        eng.aligner(list(range(1, 31)), 20)
    with pytest.raises(ValueError, match="empty"):
        eng.aligner([], 20)
    need = Aligner.workspace_bytes(10, 20)
    with pytest.raises(RuntimeError, match="budget"):
        eng.aligner(list(range(1, 11)), 20, budget_bytes=need - 1)
    with pytest.raises(RuntimeError, match="label"):
        eng.force_align(logp, [20], [[5, eng.vocab]], 0)      # the native check names what the Python one lets through
    assert launch_count() == before
    eng.aligner(list(range(1, 11)), 20, budget_bytes=need).abort()
    al = eng.aligner(list(range(1, 11)), 20)
    al.push(logp[0, :5])
    with pytest.raises(RuntimeError, match="5 of the 20"):
        al.finish()                                           # frees the handle
    got = eng.force_align(logp, [20], [[5, 6, 7]], 0)[0]      # and the engine still works
    same_as_oracle(got, logp[0].cpu().numpy(), [5, 6, 7])


def test_alignment_at_the_benchmarked_shape(bench_asr, tmp_path):
    """64 chunks of 30 s with ~100 labels each through ASRModel.align, and one 10-minute recording against ~2000 labels
    through ReverbASR.align_tokens; a sample of the utterances / the whole recording against the oracle."""
    from oracle import align_ref
    from reverb_b200.ctc_align import frames_to_ms
    m, d = bench_asr
    rng = np.random.default_rng(9)
    V = m.engine.vocab
    feats = torch.randn(64, 2998, 80, device="cuda") * 3
    lens = torch.full((64,), 2998, dtype=torch.int32)
    lens[5], lens[63] = 1500, 2000
    cat = torch.tensor([1.0, 0.0])
    labels = [random_labels(rng, int(rng.integers(80, 120)), V, repeats=(b % 2 == 0)) for b in range(64)]
    tok = np.zeros((64, max(map(len, labels))), dtype=np.int64)
    for b, y in enumerate(labels):
        tok[b, :len(y)] = y
    res = m.model.align(feats, lens, torch.from_numpy(tok), torch.tensor([len(y) for y in labels]), 0, cat)
    enc, enc_lens = m.model._forward_encoder(feats, lens, cat)
    logp = m.model.ctc_logprobs(enc)
    for b in (0, 5, 31, 63):
        T = int(enc_lens[b])
        want = align_ref.align(logp[b, :T].cpu().numpy(), labels[b], 0)
        assert np.array_equal(res[b].alignment, want["frames"]) and res[b].times == want["peak"].tolist()
        assert np.float32(res[b].score).tobytes() == np.float32(want["score"]).tobytes()
    del feats, enc, logp
    wav = _multi_chunk_wav(m, str(tmp_path), 600.0, 5)
    ids = random_labels(rng, 2000, V, repeats=True)
    got, times_ms = m.align_tokens(wav, ids, chunk_size=2998, batch_size=8)
    rows, frames = _valid_logp(m, wav, 2998, 8)
    want = align_ref.align(rows, ids, 0)
    assert np.array_equal(got.alignment, want["frames"]) and got.times == want["peak"].tolist()
    assert np.float32(got.score).tobytes() == np.float32(want["score"]).tobytes()
    assert times_ms == frames_to_ms(want["peak"], frames, 29980, 40) and times_ms == sorted(times_ms)
