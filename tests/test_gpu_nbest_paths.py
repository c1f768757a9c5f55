"""The three ways an n-best reaches the device share one layout and one search launch (csrc/engine.cu NBest): the
synchronous search (rvb_ctc_prefix_beam_search*), the ticket search (rvb_search_submit*) and the flat rescoring API
(rvb_attention_rescoring).  These tests hold the paths to each other, bit for bit, at the benchmarked model shape:

  * the synchronous search and a ticket search with run_decoder = 0 return the same n-best, plain and biased;
  * the flat rescoring API, given a ticket's n-best at the ticket's row length, returns the ticket's flat rescoring
    scores (RVB_RESCORE=flat) byte for byte, both directions;
  * a synchronous search issued on the host thread whose ticket search is still running (B = 64, T' = 748, beam 10)
    returns what it returns alone, and so does the ticket: each search has its own workspace.
"""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import rescoring_ref
from reverb_b200 import synth
from reverb_b200.context_graph import ContextGraph
from reverb_b200.engine import nbest_lists
from test_rescoring_nbest_shapes import BEAM, ENC_LENS, FAMILIES, SEED, TP, V

pytestmark = pytest.mark.gpu

CAT = [0.7, 0.3]
RW = 0.3
PHRASES = synth.context_phrases(200, V, seed=3)


@pytest.fixture(scope="module")
def eng(bench_model_dir):
    import reverb_b200
    return reverb_b200.load_model(bench_model_dir, precision="bf16").engine


def _ticket_search(eng, val, idx, enc, lens, beam, context=None):
    """the n-best of a ticket without the decoder: (toks, tims, olen, scores, nhyp)"""
    t = eng.search_submit(val, idx, enc, lens, beam, 0, context)
    eng.rescoring_submit(t, None, 0.0, run_decoder=False)
    return eng.rescoring_collect(t)[:5]


def _assert_same_nbest(a, b):
    assert np.array_equal(a[4], b[4]), "hypothesis counts differ"
    la, lb = nbest_lists(*a), nbest_lists(*b)
    for u, (x, y) in enumerate(zip(la, lb)):
        assert x[0] == y[0], f"utterance {u}: tokens differ"
        assert x[1] == y[1], f"utterance {u}: scores differ"
        assert x[2] == y[2], f"utterance {u}: times differ"
    for u, n in enumerate(a[4]):
        assert np.array_equal(a[2][u, :n], b[2][u, :n]), f"utterance {u}: lengths differ"


def _topk(B, T, seed):
    val, idx = synth.context_topk(B, T, BEAM, V, PHRASES, seed=seed)
    return torch.from_numpy(val).cuda(), torch.from_numpy(idx).cuda()


@pytest.mark.parametrize("biased", [False, True])
def test_synchronous_and_ticket_search_agree(eng, biased):
    B, T = 8, TP
    val, idx = _topk(B, T, seed=21)
    lens = np.asarray([T, T - 1, T - 37, 1, T, 500, T - 3, 2], dtype=np.int32)
    enc = torch.empty((B, T, eng.d_model), device="cuda")
    graph = ContextGraph(token_lists=PHRASES, context_score=3.0) if biased else None
    sync = eng.prefix_beam_search_raw(val, idx, lens, BEAM, 0, context=graph)
    _assert_same_nbest(sync, _ticket_search(eng, val, idx, enc, lens, BEAM, context=graph))


def test_flat_api_on_a_ticket_nbest_is_the_ticket_flat_rescoring(eng, monkeypatch):
    val, idx = rescoring_ref.synthetic_topk(FAMILIES, ENC_LENS, TP, V, BEAM, SEED)
    val, idx = torch.from_numpy(val).cuda(), torch.from_numpy(idx).cuda()
    g = torch.Generator().manual_seed(5)
    enc = torch.randn(len(FAMILIES), TP, eng.d_model, generator=g).cuda()
    lens = np.asarray(ENC_LENS, np.int32)
    monkeypatch.setenv("RVB_RESCORE", "flat")
    toks, _, olen, _, nhyp, l2r, r2l = eng.beam_search_rescoring(val, idx, enc, lens, BEAM, 0, CAT, RW)
    assert r2l is not None
    B, N, L = toks.shape
    hlen = np.where(np.arange(N)[None, :] < nhyp[:, None], olen[:, :, 0], -1).astype(np.int32)
    toks = np.ascontiguousarray(toks, dtype=np.int32)
    cat = np.asarray(CAT, np.float32)
    got_l, got_r = np.zeros_like(l2r), np.zeros_like(r2l)
    p = lambda a: a.ctypes.data_as(C.c_void_p)  # noqa: E731
    rc = eng.lib.rvb_attention_rescoring(eng._h, C.c_void_p(enc.data_ptr()), p(lens), B, TP, p(toks), p(hlen), N, L,
                                         p(cat), len(CAT), RW, p(got_l), p(got_r), eng._stream())
    assert rc == 0
    assert np.array_equal(got_l.view(np.uint32), np.ascontiguousarray(l2r).view(np.uint32))
    assert np.array_equal(got_r.view(np.uint32), np.ascontiguousarray(r2l).view(np.uint32))


def test_synchronous_search_while_a_ticket_search_runs(eng):
    B, T = 64, TP
    rng = np.random.default_rng(9)
    lens = rng.integers(T - 160, T + 1, size=B).astype(np.int32)
    val1, idx1 = _topk(B, T, seed=31)
    val2, idx2 = _topk(B, T, seed=32)
    enc = torch.empty((B, T, eng.d_model), device="cuda")
    ticket_alone = _ticket_search(eng, val1, idx1, enc, lens, BEAM)
    sync_alone = eng.prefix_beam_search_raw(val2, idx2, lens, BEAM)
    t = eng.search_submit(val1, idx1, enc, lens, BEAM)          # searches on the model's side stream
    sync_during = eng.prefix_beam_search_raw(val2, idx2, lens, BEAM)
    eng.rescoring_submit(t, None, 0.0, run_decoder=False)
    ticket_during = eng.rescoring_collect(t)[:5]
    _assert_same_nbest(sync_alone, sync_during)
    _assert_same_nbest(ticket_alone, ticket_during)
