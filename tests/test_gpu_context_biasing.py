"""Context biasing on the GPU: the biased instantiation of the prefix beam search kernel (csrc/ctc.cu) with the graph in
device memory (csrc/context.cu), against the live reference's results (tests/golden/context.json) and against the host
restatement `search.ctc_prefix_beam_search_biased` at the sizes users run; then decode / decode_stream /
transcribe_modes / the CLI with a graph."""
import json
import os

import numpy as np
import pytest
import torch

from reverb_b200 import synth
from reverb_b200.context_graph import ContextGraph
from reverb_b200.search import ctc_prefix_beam_search_biased, rescoring_pick

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
V = 5000          # vocabulary of the synthetic top-k arrays
T = 748           # encoder frames of a 30 s chunk
B = 8


@pytest.fixture(scope="module")
def asr(model_dirs):
    import reverb_b200
    return {n: reverb_b200.load_model(d) for n, (d, _) in model_dirs.items()}


def _assert_same(gpu, host):
    """n-best token lists and times identical, scores to the bar of the unbiased GPU search (CUDA fp64 exp / log)."""
    for (nbest, scores, times), w in zip(gpu, host):
        assert [list(h) for h in nbest] == [list(h) for h in w.nbest]
        assert times == [list(t) for t in w.nbest_times]
        np.testing.assert_allclose(scores, w.nbest_scores, rtol=1e-9, atol=0)


@pytest.mark.parametrize("case", ["causal_ln", "sym_bn"])
def test_biased_search_equals_the_reference_on_recorded_ctc_probs(asr, case):
    from reverb_b200.engine import DeviceContextGraph
    with open(os.path.join(GOLDEN, "context.json")) as f:
        g = json.load(f)["cases"][case]
    arr = np.load(os.path.join(GOLDEN, case + ".npz"))
    probs = torch.from_numpy(arr["ctc_probs_0"]).cuda()
    lens = arr["enc_lens_0"]
    beam = g["beam_size"]
    eng = asr[case].engine
    val, idx = eng.logp_topk(probs, beam)
    for run in g["runs"]:
        graph = ContextGraph(token_lists=g["phrases"], context_score=run["context_score"])
        dg = DeviceContextGraph(graph, probs.shape[2], 0)
        got = eng.prefix_beam_search(val, idx, lens, beam, 0, context=dg)
        for (nbest, scores, times), want in zip(got, run["results"]):
            assert [list(h) for h in nbest] == want["nbest"]
            assert times == want["nbest_times"]
            np.testing.assert_allclose(scores, want["nbest_scores"], rtol=1e-9, atol=0)


def _graphs():
    """Graphs that exercise every branch of the automaton."""
    tricky = [[11, 12, 13], [12, 13], [13], [11, 12],           # nested / overlapping; [11, 12] ends on an existing node
              [12, 13, 14, 15], [15], [14, 15, 11], [16, 17], [17, 16, 17, 16]]
    # deep fail chains: x, xx, ..., x^9 and phrases that leave them late
    deep = [[21] * n for n in range(1, 10)] + [[21] * 6 + [22], [22, 21, 21, 21, 23], [21, 23, 21, 23, 21, 23]]
    rng = np.random.default_rng(5)
    wide = [[int(t)] + ([int(rng.integers(1, V))] if rng.random() < 0.5 else [])
            for t in rng.permutation(np.arange(1, V))[:3000]]    # a root with 3000 children
    return {"tricky": tricky, "deep_fail": deep, "wide_root": wide, "10k": synth.context_phrases(10000, V, seed=7)}


GRAPHS = _graphs()


@pytest.mark.parametrize("beam", [4, 10, 16])
@pytest.mark.parametrize("name", list(GRAPHS))
def test_biased_search_equals_the_host_search(asr, name, beam):
    """T' = 748, B = 8: beams 4 and 10 keep the search trie in shared memory, beam 16 (227 KB) in global memory."""
    from reverb_b200.engine import DeviceContextGraph
    phrases = GRAPHS[name]
    graph = ContextGraph(token_lists=phrases, context_score=3.0 if name != "10k" else 2.0)
    val, idx = synth.context_topk(B, T, beam, V, phrases, seed=100 + beam)
    lens = np.asarray([T, T - 1, T - 37, 1, T, 500, T - 3, 2], dtype=np.int32)
    eng = asr["causal_ln"].engine
    dval, didx = torch.from_numpy(val).cuda(), torch.from_numpy(idx).cuda()
    got = eng.prefix_beam_search(dval, didx, lens, beam, 0, context=DeviceContextGraph(graph, V, 0))
    want = ctc_prefix_beam_search_biased(val, idx, lens, beam, graph, 0)
    _assert_same(got, want)
    plain = eng.prefix_beam_search(dval, didx, lens, beam, 0)
    assert any(g[0] != p[0] for g, p in zip(got, plain)), "biasing changed no n-best"
    # the plain search is unaffected by a biased one having run before it
    assert eng.prefix_beam_search(dval, didx, lens, beam, 0) == plain


def test_graph_outlives_its_python_handle_until_the_search_is_done(asr):
    """destroy waits for searches enqueued with the graph: dropping the handle right after an asynchronous submit must
    not change the result."""
    import gc
    from reverb_b200.engine import DeviceContextGraph
    phrases = GRAPHS["tricky"]
    graph = ContextGraph(token_lists=phrases, context_score=3.0)
    val, idx = synth.context_topk(B, T, 10, V, phrases, seed=3)
    lens = np.full(B, T, dtype=np.int32)
    eng = asr["causal_ln"].engine
    dval, didx = torch.from_numpy(val).cuda(), torch.from_numpy(idx).cuda()
    want = eng.prefix_beam_search(dval, didx, lens, 10, 0, context=DeviceContextGraph(graph, V, 0))
    enc = torch.zeros((B, T, eng.d_model), device="cuda")
    t = eng.search_submit(dval, didx, enc, lens, 10, 0, context=DeviceContextGraph(graph, V, 0))
    gc.collect()                        # the ticket still holds the graph
    eng.rescoring_submit(t, None, 0.0, run_decoder=False)
    toks, tims, olen, scores, nhyp, _, _ = eng.rescoring_collect(t)
    for b in range(B):
        assert [tuple(toks[b, r, :olen[b, r, 0]].tolist()) for r in range(int(nhyp[b]))] == want[b][0]
        np.testing.assert_array_equal(scores[b, :int(nhyp[b])], want[b][1])


def _first_batch(m, meta, arr):
    cat = torch.tensor([meta["verbatimicity"], 1.0 - meta["verbatimicity"]])
    feats = torch.from_numpy(arr["feats"]).unsqueeze(0).cuda()
    return cat, feats


def _phrases_from(results, n=6):
    """Token snippets of the lower-ranked hypotheses: phrases the bias can promote."""
    out = []
    for r in results:
        for h in r.nbest[1:]:
            if len(h) >= 3 and len(out) < n:
                out.append(list(h[-3:]))
    return out or [[5, 6]]


@pytest.mark.parametrize("case", ["causal_ln", "sym_bn"])
def test_decode_equals_host_search_plus_rescoring_pick(asr, golden_cases, case):
    meta, arr = golden_cases[case]
    m = asr[case]
    cat, feats = _first_batch(m, meta, arr)
    fb, fl = next(iter(m.feats_batcher(feats, meta["chunk_size"], meta["batch_size"])))
    beam, rw, cw = meta["beam_size"], meta["reverse_weight"], 0.5
    modes = ["ctc_prefix_beam_search", "attention_rescoring"]
    plain = m.model.decode(modes, fb, fl, beam, ctc_weight=cw, reverse_weight=rw, cat_embs=cat)
    graph = ContextGraph(token_lists=_phrases_from(plain["ctc_prefix_beam_search"]), context_score=3.0)
    got = m.model.decode(modes, fb, fl, beam, ctc_weight=cw, reverse_weight=rw, cat_embs=cat, context_graph=graph)
    enc, enc_lens = m.model._forward_encoder(fb, fl, cat)
    val, idx, _ = m.engine.ctc_topk(enc, beam)
    host = ctc_prefix_beam_search_biased(val.cpu().numpy(), idx.cpu().numpy(), enc_lens, beam, graph, 0)
    _assert_same([(r.nbest, r.nbest_scores, r.nbest_times) for r in got["ctc_prefix_beam_search"]], host)
    l2r, r2l = m.engine.rescoring_scores(enc, enc_lens, [h.nbest for h in host], cat, rw)
    for b, (g, h) in enumerate(zip(got["attention_rescoring"], host)):
        w = rescoring_pick(h.nbest, h.nbest_scores, h.nbest_times, l2r[b], None if r2l is None else r2l[b], cw, rw)
        assert list(g.tokens) == list(w.tokens) and list(g.times) == list(w.times)
        # the decoder scores come from the prefix-tree decoder on one side and the flat one on the other (ctc.cu):
        # equal to float32 rounding
        np.testing.assert_allclose(g.score, w.score, rtol=1e-5)
        np.testing.assert_allclose(np.log(g.tokens_confidence), np.log(w.tokens_confidence), rtol=0, atol=2e-3)


def test_decode_stream_equals_batch_by_batch_decode(asr, golden_cases):
    meta, arr = golden_cases["causal_ln"]
    m = asr["causal_ln"]
    cat, feats = _first_batch(m, meta, arr)
    batches = list(m.feats_batcher(feats, 200, 2))
    assert len(batches) >= 3
    modes = ["ctc_prefix_beam_search", "attention_rescoring"]
    graph = ContextGraph(token_lists=GRAPHS["tricky"] + [[5, 6], [7, 8, 9], [10]], context_score=3.0)
    kw = dict(ctc_weight=0.3, reverse_weight=0.3, cat_embs=cat, context_graph=graph)
    streamed = list(m.model.decode_stream(batches, modes, 10, **kw))
    for (fb, fl), s in zip(batches, streamed):
        one = m.model.decode(modes, fb, fl, 10, **kw)
        for mode in modes:
            for a, b in zip(s[mode], one[mode]):
                assert list(a.tokens) == list(b.tokens) and a.times == b.times and a.score == b.score


def _phrase_file(m, wav, tmp_path):
    """A phrase file from words of the unbiased transcript, and a small sentencepiece model to tokenize it with (the
    synthetic model directory's tk.model is an empty placeholder)."""
    import sentencepiece as spm
    words = m.transcribe(wav, mode="ctc_prefix_beam_search", format="txt", chunk_size=200, batch_size=2).split(" ")
    corpus = tmp_path / "corpus.txt"
    corpus.write_text("\n".join(" ".join(words[i:i + 6]) for i in range(0, len(words), 6)).upper() + "\n")
    spm.SentencePieceTrainer.train(input=str(corpus), model_prefix=str(tmp_path / "tiny"), vocab_size=40,
                                   model_type="bpe", hard_vocab_limit=False, minloglevel=2)
    p = tmp_path / "phrases.txt"
    p.write_text("\n".join(w for w in words[::3][:8] if w) + "\n")
    return p, str(tmp_path / "tiny.model")


def test_transcribe_with_context_graph_batch_size_and_cli(asr, model_dirs, tmp_path):
    import reverb_b200
    from reverb_b200 import recognize_wav
    d, wav = model_dirs["causal_ln"]
    p, bpe = _phrase_file(asr["causal_ln"], wav, tmp_path)
    m = reverb_b200.ReverbASR(os.path.join(d, "config.yaml"), os.path.join(d, "synth.pt"), bpe_path=bpe)
    graph = m.context_graph(str(p), 4.0)
    assert graph.num_nodes > 0
    assert m.context_graph(p.read_text().splitlines(), 4.0).context_list == graph.context_list
    modes = ["ctc_prefix_beam_search", "attention_rescoring"]
    out1 = m.transcribe_modes(wav, modes, format="ctm", chunk_size=200, batch_size=1, context_graph=graph)
    out4 = m.transcribe_modes(wav, modes, format="ctm", chunk_size=200, batch_size=4, context_graph=graph)
    assert out1 == out4
    plain = m.transcribe_modes(wav, modes, format="ctm", chunk_size=200, batch_size=4)
    assert m.transcribe_modes(wav, modes, format="ctm", chunk_size=200, batch_size=4, context_graph=None) == plain
    recognize_wav.main(["--config", os.path.join(d, "config.yaml"), "--checkpoint", os.path.join(d, "synth.pt"),
                        "--bpe-path", bpe, "--audio_file", wav, "--result_dir", str(tmp_path / "out"), "--modes"] +
                       modes + ["--chunk_size", "200", "--batch_size", "2", "--context_list_path", str(p),
                                "--context_graph_score", "4.0"])
    for mode, text in zip(modes, out1):
        assert (tmp_path / "out" / mode / "golden.ctm").read_text() == text
