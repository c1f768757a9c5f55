"""Attention rescoring at the benchmarked shape (d = 1024, 16 heads, 3 + 3 decoder blocks, V = 10 001) against float64
references: the prefix-tree decoder (default) and the flat one, both decoder directions, both precisions.

The n-best lists come from the device prefix beam search on synthetic CTC top-k (oracle/rescoring_ref.synthetic_topk):
hypotheses of 200-250 tokens that diverge past token 64, bushy trees of 1 000-2 000 node slots, an empty hypothesis,
one- to three-frame utterances, hypotheses that are proper prefixes or suffixes of others.  Encoder frames past each
utterance's length hold +-1e3, so a cross-attention key read past `enc_len` is a large error.  With k >= beam and at
least one frame the search always fills the beam, so absent hypothesis slots are exercised through the flat host
API's -1 rows.

Stated bounds, about 2x the errors measured on one H100 80GB HBM3 (700 W, max SM clock 1980 MHz); `pytest -s` prints
the measured values:
  * precision="fp32" (bf16x3 GEMMs, fp32 attention): every (hypothesis, position) log-prob within max 4e-5 / RMS 1e-5
    of float64 (measured 1.6e-5 / 4.2e-6), tree and flat layouts, left-to-right and right-to-left; the rescoring pick
    equals the pick on float64 scores.
  * bf16: max 0.012 / RMS 0.003 (measured 5.6e-3 / 1.3e-3) for either layout and direction.  The wgmma ancestor-mask
    self-attention (default) against the fp32 ancestor-list one (RVB_TRIE_ATTN=list): max 1.5e-3 / RMS 2.5e-4
    (measured 6.9e-4 / 1.2e-4).
  * the ancestor-mask attention kernel alone (rvb_attention_tc_bits) against a float64 masked softmax whose value rows
    are +-100: within 2^-6 (|ref| + 100 ||p||_2) per element (measured at most 0.98 x 2^-7 (...)), where p is the row's
    attention weights.  A key leaking into a row of depth d moves it by ~100 / d.
  * rvb_attention_rescoring (flat host API) with lengths 0-255, absent rows and a one-frame utterance: max 4e-5 (fp32,
    measured 1.9e-5) and 0.01 (bf16, measured 5.0e-3) of float64.
"""
import ctypes as C
import math
import os

import numpy as np
import pytest
import torch

from oracle import rescoring_ref, search_ref
from test_rescoring_nbest_shapes import BEAM, ENC_LENS, FAMILIES, SEED, TP, V, check_coverage, nbest_coverage

pytestmark = pytest.mark.gpu

CAT = [0.7, 0.3]
RW, CW = 0.3, 0.1
# (precision, layout) -> (max abs, RMS) bound of the per-position log-probs against float64, both directions
BOUNDS = {("fp32", "tree"): (4e-5, 1e-5), ("fp32", "flat"): (4e-5, 1e-5),
          ("bf16", "tree"): (0.012, 0.003), ("bf16", "flat"): (0.012, 0.003)}
LIST_VS_BITS = (1.5e-3, 2.5e-4)
FLAT_API = {"fp32": 4e-5, "bf16": 0.01}


def poisoned(B, T, d, lens, seed):
    """(B, T, d) float32 encoder output, N(0, 1) on valid frames and +-1e3 (a per-frame sign pattern) behind them"""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, T, d, generator=g)
    sign = torch.where((torch.arange(T)[:, None] * 7 + torch.arange(d)[None, :] * 3) % 5 < 2, 1.0, -1.0)
    for b, L in enumerate(lens):
        x[b, L:] = 1e3 * sign[L:]
    return x


@pytest.fixture(scope="module")
def ref_model(bench_model_dir):
    from oracle import pipeline_ref
    orc = pipeline_ref.OracleASR(bench_model_dir)
    torch.set_num_threads(min(32, os.cpu_count() or 8))
    return {"sd64": rescoring_ref.to_float64(orc.sd), "cfg": orc.cfg, "sos": orc.sos, "eos": orc.eos,
            "cat64": torch.tensor(CAT, dtype=torch.float64)}


@pytest.fixture(scope="module")
def engines(bench_model_dir):
    import reverb_b200
    return {p: reverb_b200.load_model(bench_model_dir, precision=p).engine for p in ("fp32", "bf16")}


def _run(eng, val, idx, enc, layout, trie_attn=None):
    env = {"RVB_RESCORE": "flat" if layout == "flat" else None, "RVB_TRIE_ATTN": trie_attn}
    old = {k: os.environ.pop(k, None) for k in env}
    try:
        for k, v in env.items():
            if v is not None:
                os.environ[k] = v
        return eng.beam_search_rescoring(val, idx, enc, np.asarray(ENC_LENS, np.int32), BEAM, 0, CAT, RW)
    finally:
        for k, v in old.items():
            os.environ.pop(k, None)
            if v is not None:
                os.environ[k] = v


@pytest.fixture(scope="module")
def crafted(engines, ref_model):
    """device results of every (precision, layout), the device n-best and its float64 scores"""
    val, idx = rescoring_ref.synthetic_topk(FAMILIES, ENC_LENS, TP, V, BEAM, SEED)
    enc = poisoned(len(FAMILIES), TP, 1024, ENC_LENS, seed=11)
    dval, didx, denc = torch.from_numpy(val).cuda(), torch.from_numpy(idx).cuda(), enc.cuda()
    out = {(p, lay): _run(engines[p], dval, didx, denc, lay) for p in ("fp32", "bf16") for lay in ("tree", "flat")}
    out[("bf16", "list")] = _run(engines["bf16"], dval, didx, denc, "tree", trie_attn="list")
    toks, _, olen, _, nhyp = out[("fp32", "tree")][:5]
    nbest = [[tuple(toks[b, i, :olen[b, i, 0]].tolist()) for i in range(int(nhyp[b]))] for b in range(len(FAMILIES))]
    r = ref_model
    ref = {side: [rescoring_ref.decoder_scores(enc[b, :L], nbest[b], r["sd64"], r["cfg"], r["cat64"], r["sos"],
                                               r["eos"], side) for b, L in enumerate(ENC_LENS)]
           for side in ("left_decoder", "right_decoder")}
    return {"val": val, "idx": idx, "out": out, "nbest": nbest, "ref": ref}


def _errors(res, nbest, ref_l, ref_r):
    """concatenated (got - float64) over every (utterance, hypothesis < nhyp, position <= U), per direction"""
    err = {"l2r": [], "r2l": []}
    for b, hs in enumerate(nbest):
        for i, h in enumerate(hs):
            U = len(h)
            err["l2r"].append(res[5][b, i, :U + 1].astype(np.float64) - ref_l[b][i])
            err["r2l"].append(res[6][b, i, :U + 1].astype(np.float64) - ref_r[b][i])
    return {k: np.concatenate(v) for k, v in err.items()}


def _stats(e):
    return float(np.abs(e).max()), float(np.sqrt((e ** 2).mean()))


def test_device_nbest_is_the_oracle_nbest_and_reaches_every_tree_edge(crafted):
    val, idx, nbest = crafted["val"], crafted["idx"], crafted["nbest"]
    for b, L in enumerate(ENC_LENS):
        want = search_ref.ctc_prefix_beam_search(rescoring_ref.full_logp(val, idx, V, b, L), np.array([L]), BEAM, 0)[0]
        assert nbest[b] == [tuple(h) for h in want.nbest], b
    check_coverage(nbest_coverage(nbest, BEAM))


def test_layouts_agree_on_the_search_results(crafted):
    """tokens, times, lengths, CTC scores and counts do not depend on the decoder layout"""
    out = crafted["out"]
    base = out[("fp32", "tree")]
    for key, res in out.items():
        for i in range(5):
            assert np.array_equal(res[i], base[i]), (key, i)


@pytest.mark.parametrize("precision,layout", sorted(BOUNDS))
def test_rescoring_scores_vs_float64(crafted, precision, layout):
    """every (utterance, hypothesis, position) log-prob of both decoders against float64; bounds in BOUNDS"""
    res = crafted["out"][(precision, layout)]
    err = _errors(res, crafted["nbest"], crafted["ref"]["left_decoder"], crafted["ref"]["right_decoder"])
    mx, rms = BOUNDS[(precision, layout)]
    for d, e in err.items():
        m, r = _stats(e)
        print(f"RESCORING {precision} {layout} {d}: max {m:.3e} rms {r:.3e} over {e.size} positions")
    for d, e in err.items():
        m, r = _stats(e)
        assert m < mx and r < rms, (precision, layout, d, m, r)


def test_accurate_mode_pick_is_the_float64_pick(crafted):
    from reverb_b200.search import rescoring_pick_batch
    res = crafted["out"][("fp32", "tree")]
    ref_l, ref_r = (np.zeros_like(res[5]), np.zeros_like(res[6]))
    for b, hs in enumerate(crafted["nbest"]):
        for i, h in enumerate(hs):
            ref_l[b, i, :len(h) + 1] = crafted["ref"]["left_decoder"][b][i]
            ref_r[b, i, :len(h) + 1] = crafted["ref"]["right_decoder"][b][i]
    got = rescoring_pick_batch(*res[:5], res[5], res[6], CW, RW)
    want = rescoring_pick_batch(*res[:5], ref_l, ref_r, CW, RW)
    assert [tuple(x.tokens) for x in got] == [tuple(x.tokens) for x in want]
    for g, w in zip(got, want):
        assert abs(g.score - w.score) < 2e-3


def test_ancestor_mask_attention_in_situ(crafted):
    """bf16 tree decoder: the wgmma self-attention with the ancestor bit mask against the fp32 ancestor-list kernel
    (same bf16 Q / K / V, only the self-attention kernel differs)"""
    a, b = crafted["out"][("bf16", "tree")], crafted["out"][("bf16", "list")]
    for k in (5, 6):
        e = []
        for bb, hs in enumerate(crafted["nbest"]):
            for i, h in enumerate(hs):
                e.append(a[k][bb, i, :len(h) + 1].astype(np.float64) - b[k][bb, i, :len(h) + 1])
        m, r = _stats(np.concatenate(e))
        print(f"RESCORING bf16 bits-vs-list {'l2r' if k == 5 else 'r2l'}: max {m:.3e} rms {r:.3e}")
        assert m < LIST_VS_BITS[0] and r < LIST_VS_BITS[1], (k, m, r)


# ------------------------------------------------------------------------------------------------------------------
# the ancestor-mask attention kernel alone
def _random_tree(rng, n_used):
    par = [-1]
    for i in range(1, n_used):
        par.append(int(rng.integers(max(0, i - 6), i)) if rng.random() < 0.8 else int(rng.integers(0, i)))
    return par


def _bits_case(trees, P, seed):
    """q / k / v (G, P, 3 * 1024) bf16, bits (G, P, bits_ld), visibility (G, P, P)"""
    H, dk = 16, 64
    G, d = len(trees), H * dk
    g = torch.Generator(device="cuda").manual_seed(seed)
    qkv = torch.empty(G, P, 3 * d, device="cuda")
    qkv[..., :2 * d] = torch.randn(G, P, 2 * d, generator=g, device="cuda") * 0.7
    # every key has its own +-100 value row: a key that leaks into a row moves it by O(100 / depth)
    qkv[..., 2 * d:] = torch.where(torch.rand(G, P, d, generator=g, device="cuda") < 0.5, 100.0, -100.0)
    qkv = qkv.bfloat16()
    bits = np.stack([rescoring_ref.ancestor_bits(par, P) for par in trees])
    vis = (bits.view(np.uint32)[..., None] >> np.arange(32, dtype=np.uint32)) & 1
    vis = vis.reshape(G, P, -1)[:, :, :P].astype(bool)
    return qkv, torch.from_numpy(bits).cuda(), bits.shape[-1], torch.from_numpy(vis).cuda()


def _bits_attention(qkv, bits, bits_ld, P):
    from reverb_b200 import _lib
    lib = _lib.load()
    G, d = qkv.shape[0], qkv.shape[2] // 3
    out = torch.full((G, P, d), 7.0, device="cuda", dtype=torch.bfloat16)
    base = qkv.data_ptr()
    rc = lib.rvb_attention_tc_bits(C.c_void_p(base), C.c_void_p(base + 2 * d), C.c_void_p(base + 4 * d),
                                   C.c_void_p(out.data_ptr()), 3 * d, 3 * d, 3 * d, d, G, P, P, 16, 64, None, None, 1,
                                   C.c_void_p(bits.data_ptr()), bits_ld, 1.0 / 8.0,
                                   C.c_void_p(torch.cuda.current_stream().cuda_stream))
    assert rc == 0, _lib.last_error()
    return out


def _check_bits_attention(trees, P, seed):
    qkv, bits, bits_ld, vis = _bits_case(trees, P, seed)
    out = _bits_attention(qkv, bits, bits_ld, P).double()
    G, d = qkv.shape[0], qkv.shape[2] // 3
    worst = 0.0
    for gi in range(G):
        x = qkv[gi].double().view(P, 3, 16, 64)
        q, k, v = (x[:, j].transpose(0, 1) for j in range(3))                       # (16, P, 64)
        s = (q @ k.transpose(1, 2)) / 8.0
        s = s.masked_fill(~vis[gi][None], -math.inf)
        p = torch.softmax(s, -1)
        ref = (p @ v).transpose(0, 1).reshape(P, d)
        tol = 2.0 ** -6 * (ref.abs() + 100.0 * p.norm(dim=-1).transpose(0, 1).repeat_interleave(64, 1))
        worst = max(worst, float(((out[gi] - ref).abs() / tol).max()))
    print(f"ATTN_BITS P={P} groups={G}: max |err| / tol = {worst:.3f}")
    assert worst <= 1.0, (P, G, worst)


@pytest.mark.parametrize("P", [8, 64, 72, 128, 136])
@pytest.mark.parametrize("groups", [1, 8])
def test_ancestor_mask_attention_kernel_random_trees(P, groups):
    rng = np.random.default_rng(P * 10 + groups)
    # trees of up to P nodes; the slots behind each tree are unused and see only themselves
    trees = [_random_tree(rng, P - int(rng.integers(0, min(6, P - 1) + 1))) for _ in range(groups)]
    _check_bits_attention(trees, P, seed=P + groups)


def test_ancestor_mask_attention_kernel_nbest_trees(crafted):
    """the trees of the crafted n-best (both directions): the whole batch (8 groups) and its largest tree alone"""
    for reverse in (False, True):
        trees = [rescoring_ref.prefix_tree(hs, reverse)["par"] for hs in crafted["nbest"]]
        P = rescoring_ref.padded_slots([len(t) for t in trees])
        _check_bits_attention(trees, P, seed=P)
        big = max(trees, key=len)
        _check_bits_attention([big], rescoring_ref.padded_slots([len(big)]), seed=len(big))


# ------------------------------------------------------------------------------------------------------------------
# the flat host API (rvb_attention_rescoring) at the edges of its row tiles
LENGTHS = (0, 1, 63, 64, 65, 127, 128, 129, 255)


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("N", [1, 16])
def test_flat_api_lengths_absent_rows_and_one_frame(engines, ref_model, precision, N):
    """hypothesis lengths across the 64-row tiles, absent (-1) rows, a one-frame utterance next to a full one"""
    rng = np.random.default_rng(N)
    lens = [1, TP]
    enc = poisoned(2, TP, 1024, lens, seed=N)
    hlen = np.full((2, N), -1, np.int32)
    if N == 1:
        hlen[:, 0] = [255, 64]
    else:
        hlen[0, :len(LENGTHS)] = LENGTHS
        hlen[1, 2:2 + len(LENGTHS)] = LENGTHS[::-1]   # absent rows before and after
    toks = rng.integers(1, V - 1, size=(2, N, 255)).astype(np.int32)
    l2r, r2l = engines[precision].rescoring_scores_raw(enc.cuda(), np.asarray(lens, np.int32), toks, hlen, CAT, RW)
    r = ref_model
    worst = {"l2r": 0.0, "r2l": 0.0}
    for b in range(2):
        present = [i for i in range(N) if hlen[b, i] >= 0]
        hyps = [tuple(toks[b, i, :hlen[b, i]].tolist()) for i in present]
        for side, got, key in (("left_decoder", l2r, "l2r"), ("right_decoder", r2l, "r2l")):
            want = rescoring_ref.decoder_scores(enc[b, :lens[b]], hyps, r["sd64"], r["cfg"], r["cat64"], r["sos"],
                                                r["eos"], side)
            for i, w in zip(present, want):
                worst[key] = max(worst[key], float(np.abs(got[b, i, :len(w)] - w).max()))
        assert np.isfinite(l2r[b]).all() and np.isfinite(r2l[b]).all()
    print(f"FLAT_API {precision} N={N}: max l2r {worst['l2r']:.3e} r2l {worst['r2l']:.3e}")
    assert max(worst.values()) < FLAT_API[precision], worst
