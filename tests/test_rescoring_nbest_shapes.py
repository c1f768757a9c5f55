"""The synthetic CTC top-k inputs of tests/test_gpu_rescoring_decoder.py reach the edges of the tree-structured
rescoring decoder (ctc.cu trie_build_kernel / trie_inputs_kernel, engine.cu decoder_pass_trie).

The n-best comes from the CPU prefix beam search (oracle/search_ref.py) on the same top-k; the trees are rebuilt in
Python with the kernel's insertion rule.  The GPU test asserts the same coverage on the n-best the device returns."""
import numpy as np
import pytest

from oracle import rescoring_ref, search_ref

# the batch of tests/test_gpu_rescoring_decoder.py: bench T' = 748, vocabulary 10 001, beam = k = 10
FAMILIES = ("deep", "deep", "bushy", "bushy", "blank", "short", "short", "prefix")
ENC_LENS = (748, 600, 600, 420, 300, 1, 3, 420)
TP, V, BEAM, SEED = 748, 10001, 10, 1234


def nbest_coverage(nbest, beam):
    """Structural facts of a batch of n-best lists (one list of token tuples per utterance) that the tree decoder
    must handle; see test_crafted_nbest_reaches_every_tree_edge for the bounds."""
    trees = [[rescoring_ref.prefix_tree(h, reverse=r) for h in nbest] for r in (False, True)]
    nodes = [[len(t["par"]) for t in tr] for tr in trees]
    P = [rescoring_ref.padded_slots(n) for n in nodes]
    hy = [h for hs in nbest for h in hs]
    return {
        "max_nodes": max(max(n) for n in nodes),
        "P": P,
        # deepest point at which a hypothesis leaves the tree of the earlier ones (warp-strided LCP loop)
        "max_divergence": max(l for tr in trees[0] for l, h in zip(tr["lcp"], tr["node_of"]) if len(h) - 1 > l),
        # longest shared suffix of two different hypotheses (= shared prefix in the reversed tree)
        "max_shared_suffix": max(l for tr in trees[1] for l in tr["lcp"]),
        "empty": sum(len(h) == 0 for h in hy),
        "proper_prefix": sum(any(len(a) < len(b) and b[:len(a)] == a for b in hs) for hs in nbest for a in hs),
        "proper_suffix": sum(any(0 < len(a) < len(b) and b[len(b) - len(a):] == a for b in hs) for hs in nbest
                             for a in hs),
        "longest": max(len(h) for h in hy),
        "short_nhyp": [len(hs) for hs in nbest],
        "full_beam": all(len(hs) == beam for hs in nbest),
    }


def check_coverage(cov):
    assert cov["max_nodes"] >= 512, cov                       # several hundred node slots (bushy tree)
    assert any(p % 64 != 0 and p > 64 for p in cov["P"]), cov  # mask rows end inside a 64-slot word, past the first
    assert cov["max_divergence"] > 64, cov                    # past two warp strides of the LCP loop
    assert cov["max_shared_suffix"] > 64, cov                 # the reversed tree shares long suffixes
    assert cov["empty"] >= 1 and cov["proper_prefix"] >= 1 and cov["proper_suffix"] >= 1, cov
    assert cov["longest"] >= 200, cov


@pytest.fixture(scope="module")
def cpu_nbest():
    val, idx = rescoring_ref.synthetic_topk(FAMILIES, ENC_LENS, TP, V, BEAM, SEED)
    out = []
    for b, L in enumerate(ENC_LENS):
        lp = rescoring_ref.full_logp(val, idx, V, b, L)
        r = search_ref.ctc_prefix_beam_search(lp, np.array([L]), BEAM, 0)[0]
        out.append([tuple(h) for h in r.nbest])
    return val, idx, out


def test_crafted_nbest_reaches_every_tree_edge(cpu_nbest):
    _, _, nbest = cpu_nbest
    cov = nbest_coverage(nbest, BEAM)
    print(cov)
    check_coverage(cov)
    # k >= beam (the device search refuses less) and every utterance has a frame: the search always returns a full
    # beam, so hypothesis slots past n_hyp are reached only through rvb_attention_rescoring's absent rows
    assert cov["full_beam"]


def test_synthetic_topk_rows_are_sorted_distinct_and_valid(cpu_nbest):
    val, idx, _ = cpu_nbest
    assert (np.diff(val, axis=2) <= 0).all()
    s = np.sort(idx, axis=2)
    assert (np.diff(s, axis=2) != 0).all()
    assert idx.min() >= 0 and idx.max() < V - 1               # never sos / eos


def test_prefix_tree_matches_the_kernel_insertion_rule():
    """Hand-checked trees: shared prefixes, a proper prefix (no new node), an empty hypothesis, ties between two
    earlier hypotheses resolved to the first; ancestor bit rows with unused slots seeing only themselves."""
    hyps = [(5, 6, 7), (5, 6), (), (5, 8), (9,), (5, 6, 7, 1)]
    t = rescoring_ref.prefix_tree(hyps)
    assert t["par"] == [-1, 0, 1, 2, 1, 0, 3]
    assert t["tok"][1:] == [5, 6, 7, 8, 9, 1]
    assert t["node_of"] == [[0, 1, 2, 3], [0, 1, 2], [0], [0, 1, 4], [0, 5], [0, 1, 2, 3, 6]]
    assert t["lcp"] == [0, 2, 0, 1, 0, 3]
    r = rescoring_ref.prefix_tree(hyps, reverse=True)
    assert r["node_of"][1] == [0, 4, 5] and r["tok"][4:6] == [6, 5]   # (6, 5) reversed shares nothing with (7, 6, 5)
    P = rescoring_ref.padded_slots([len(t["par"])])
    assert P == 8
    bits = rescoring_ref.ancestor_bits(t["par"], 72).view(np.uint32)
    assert bits.shape == (72, 4)
    assert bits[6, 0] == (1 << 0) | (1 << 1) | (1 << 2) | (1 << 3) | (1 << 6)
    assert bits[7, 0] == 1 << 7 and bits[71, 2] == 1 << 7 and bits[71, [0, 1, 3]].sum() == 0
