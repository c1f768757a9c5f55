"""The CTC head kernels of csrc/ctc.cu against plain references, at the production vocabulary and at the sizes and
edges where each kernel has its own code:

  logsoftmax_topk    both selection paths (the lane-group filter and the block arg-max fallback), ties, -inf, the
                     softmax / blank-penalty / padded-stride path of `Engine.ctc_topk` on exactly known logits;
  ctc_greedy         32-frame warp steps, the id carried across them, `lens` of 0 and beyond T, index strides;
  ctc_prefix_beam    the plain search with its trie in shared and in global memory, against oracle/search_ref.py.

The top-k order reference is a stable sort (value descending, ties to the lower index); torch.topk does not specify
its order on ties, so it is only used where the inputs have none.
"""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from oracle import search_ref
from reverb_b200 import synth

pytestmark = pytest.mark.gpu

TOPK_CAP = 64                 # candidates the filter path ranks (csrc/ctc.cu)
SMEM_TRIE_BYTES = 150 * 1024  # largest prefix-search trie kept in shared memory (csrc/ctc.cu, launch_prefix_beam)
MAX_TOPK_V = 51200            # largest row the top-k launcher stages in shared memory (200 KB of float32)


@pytest.fixture(scope="module")
def eng(tmp_path_factory):
    """An engine for the entry points that take their inputs directly (no model weights involved)."""
    import reverb_b200
    d = synth.write_model_dir(str(tmp_path_factory.mktemp("ctc_head")), seed=11)
    return reverb_b200.load_model(d).engine


def stable_topk(x: np.ndarray, k: int) -> np.ndarray:
    """Indices of the first k entries of every row of a stable sort by value, descending.  Only the entries not below
    the row's k-th largest value can rank before k, so only those are sorted."""
    x = np.asarray(x, dtype=np.float32)
    kth = -np.partition(-x, k - 1, axis=1)[:, k - 1]
    out = np.empty((x.shape[0], k), dtype=np.int64)
    for r in range(x.shape[0]):
        col = np.nonzero(x[r] >= kth[r])[0]
        out[r] = col[np.lexsort((col, -x[r, col]))][:k]
    return out


# ---------------------------------------------------------------------------------------------------------------------
# 1. logsoftmax_topk without the softmax: recorded log-probs through Engine.logp_topk

ROWS = 293
VOCABS = [1, 2, 16, 31, 32, 33, 255, 256, 257, 5000, 10001, MAX_TOPK_V]
KS = [1, 2, 4, 10, 16]
FAMILIES = ["gauss", "peaky", "overflow", "ties", "neginf"]


def _last_stride(V):
    """Columns of the last 256-wide stride of the kernel's row loop (partial unless 256 divides V)."""
    return np.arange((V - 1) // 256 * 256, V)


def _rows_gauss(rng, V, k, n):
    return rng.standard_normal((n, V)).astype(np.float32)


def _rows_peaky(rng, V, k, n):
    """CTC-like rows: blank near 0, a few tokens 1-3 nats below it, the rest far below; a third of the rows have
    their maximum in the last (partial) stride, a third at column V - 1."""
    x = rng.normal(-25.0, 3.0, (n, V))
    x[:, 0] = rng.uniform(-0.5, 0.0, n)
    for r in range(n):
        toks = rng.choice(V, size=min(V, 5), replace=False)
        x[r, toks[toks != 0]] = rng.uniform(-3.0, -1.0, int((toks != 0).sum()))
        if r % 3 == 1:
            x[r, rng.choice(_last_stride(V))] = 0.5
        elif r % 3 == 2:
            x[r, V - 1] = 0.5
    return x.astype(np.float32)


def _rows_overflow(rng, V, k, n):
    """Rows whose candidate list (the elements not worse than the k-th best lane-group maximum) has exactly
    63, 64, 65 or 97 entries: k - 1 mid values, each alone in its lane group, and the rest of the candidates high
    values in ONE residue class mod 32, either all tied or distinct.  63 and 64 stay on the filter path, 65 and 97
    take the fallback.  Rows that cannot be built at this (V, k) are plain Gaussian rows."""
    x = rng.uniform(-10.0, -9.0, (n, V)).astype(np.float32)
    for r in range(n):
        ncand = (63, 64, 65, 97)[r % 4]
        res = int(rng.integers(32))
        cls = np.arange(res, V, 32)
        n_high = ncand - (k - 1)
        if k < 2 or n_high > cls.size:
            x[r] = rng.standard_normal(V)
            continue
        high = rng.choice(cls, size=n_high, replace=False)
        x[r, high] = 5.0 if (r // 4) % 2 == 0 else 5.0 + 0.01 * rng.permutation(n_high)
        groups = rng.choice(np.setdiff1d(np.arange(32), [res]), size=k - 1, replace=False)
        for i, g in enumerate(groups):
            x[r, g + 32 * int(rng.integers((V - 1 - g) // 32 + 1))] = -1.0 - 0.5 * i
    return x


def _rows_ties(rng, V, k, n):
    """Exact ties at the k-th position: the whole row equal, or a block of equal values straddling rank k below
    0..k-1 distinct higher values."""
    x = rng.uniform(-10.0, -9.0, (n, V)).astype(np.float32)
    for r in range(n):
        if r % 3 == 0:
            x[r] = np.float32(rng.normal())
            continue
        n_above = int(rng.integers(0, k)) if V > 1 else 0
        block = min(V - n_above, k - n_above + int(rng.integers(1, 6)))
        cols = rng.choice(V, size=n_above + block, replace=False)
        x[r, cols[:n_above]] = 3.0 + rng.permutation(n_above).astype(np.float32)
        x[r, cols[n_above:]] = 1.5
    return x


def _rows_neginf(rng, V, k, n):
    """-inf entries: fewer than k finite entries (the rest -inf); k or more finite entries all in one lane group
    (fallback with finite values); or finite entries spread over many lane groups among -inf (filter path)."""
    x = np.full((n, V), -np.inf, dtype=np.float32)
    for r in range(n):
        kind = r % 3
        if kind == 0:
            nf = int(rng.integers(0, k))
            cols = rng.choice(V, size=nf, replace=False)
        elif kind == 1:
            cls = np.arange(int(rng.integers(min(V, 32))), V, 32)
            cols = rng.choice(cls, size=min(cls.size, k + int(rng.integers(0, 4))), replace=False)
        else:
            cols = rng.choice(V, size=min(V, k + 40), replace=False)
        x[r, cols] = rng.standard_normal(cols.size)
    return x


ROW_MAKERS = {"gauss": _rows_gauss, "peaky": _rows_peaky, "overflow": _rows_overflow, "ties": _rows_ties,
              "neginf": _rows_neginf}


def _topk_cases():
    return [(V, k, f) for V in VOCABS for k in KS if k <= V for f in FAMILIES]


@pytest.mark.parametrize("V,k,family", _topk_cases())
def test_logp_topk_is_the_stable_order(eng, V, k, family):
    """Indices equal a stable sort, position by position; values are x[row, idx] bit for bit (no softmax)."""
    rng = np.random.default_rng([V, k, FAMILIES.index(family)])
    x = ROW_MAKERS[family](rng, V, k, ROWS)
    want = stable_topk(x, k)
    val, idx = eng.logp_topk(torch.from_numpy(x).cuda().view(1, ROWS, V), k)
    idx = idx.view(ROWS, k).cpu().numpy()
    val = val.view(ROWS, k).cpu().numpy()
    bad = np.nonzero((idx != want).any(axis=1))[0]
    assert bad.size == 0, (f"{bad.size} rows differ, first row {bad[0]}: got {idx[bad[0]].tolist()} "
                           f"want {want[bad[0]].tolist()}")
    np.testing.assert_array_equal(val.view(np.int32), np.take_along_axis(x, want, axis=1).view(np.int32))


def test_topk_row_builders_reach_the_paths_they_name():
    """The overflow rows have the candidate counts they claim, and the -inf rows have a -inf k-th lane-group maximum
    where they should (restating the kernel's filter on the host)."""
    def ncand(row, k):
        order = stable_topk(row[None], row.size)[0]
        rank = np.empty(row.size, np.int64)
        rank[order] = np.arange(row.size)
        groups = [np.arange(g, row.size, 32) for g in range(min(32, row.size))]
        gmax = sorted(int(g[np.argmin(rank[g])]) for g in groups)
        th = sorted(gmax, key=lambda i: rank[i])[k - 1] if len(gmax) >= k else None
        return None if th is None or row[th] == -np.inf else int((rank <= rank[th]).sum())
    rng = np.random.default_rng(0)
    for V in (5000, 10001):
        x = _rows_overflow(rng, V, 4, 8)
        assert [ncand(x[r], 4) for r in range(8)] == [63, 64, 65, 97] * 2
    x = _rows_neginf(rng, 10001, 10, 6)
    assert [ncand(x[r], 10) is None for r in range(6)] == [True, True, False] * 2


@pytest.mark.parametrize("V,k", [(10001, 0), (10001, 17), (10, 11), (MAX_TOPK_V + 1, 10)])
def test_logp_topk_rejects_before_any_launch(eng, V, k):
    from reverb_b200 import _lib, engine
    x = torch.zeros((1, 3, V), dtype=torch.float32, device="cuda")
    before = engine.launch_count()
    with pytest.raises(RuntimeError, match="logsoftmax_topk"):
        eng.logp_topk(x, k)
    assert engine.launch_count() == before
    assert "logsoftmax_topk" in _lib.last_error()


# ---------------------------------------------------------------------------------------------------------------------
# 2. logsoftmax_topk with the softmax, through Engine.ctc_topk on exactly known logits

CTC_VOCABS = [33, 257, 4999, 10001]
D_MODEL = synth.TEST_SHAPE["d"]
B_LEVELS = np.array([0.0, 0.3183099, -0.7182818], dtype=np.float32)   # bias = B_LEVELS[n % 3]: fp32, not bf16


def _bf16(a):
    return torch.from_numpy(np.asarray(a, np.float32)).to(torch.bfloat16).float().numpy()


def _ctc_head(V):
    """ctc_lo weight (V, d), bf16-representable, and bias (V,) float32.  With a one-hot encoder row at column j the
    logits are float32(W[:, j] + b) exactly, in both precisions.  Column patterns:
      j % 4 == 0   spread: uniform over 6 nats, real probability mass in every column including the tail
      j % 4 == 1   spread, maximum in the last (partial) 256-column stride or at column V - 1
      j % 4 == 2   coarse levels: groups of exactly equal logits; the top group (10-12 columns) and the next one
                   straddle rank k
      j % 4 == 3   blank-led: blank 6.0, token 4.0 (ties with the blank at penalty 2.0), a few tokens just below"""
    rng = np.random.default_rng(V)
    W = np.empty((V, D_MODEL), np.float32)
    for j in range(D_MODEL):
        kind = j % 4
        if kind in (0, 1):
            W[:, j] = rng.uniform(-3.0, 3.0, V)
            if kind == 1:
                W[V - 1 if j % 8 == 1 else rng.choice(_last_stride(V)), j] = 4.0
        elif kind == 2:
            W[:, j] = rng.integers(0, 6, V) * 0.5
            same_bias = np.arange(1, V, 3)
            W[rng.choice(same_bias, size=min(same_bias.size, 12), replace=False), j] = 3.0
        else:
            W[:, j] = rng.uniform(-3.0, 1.0, V)
            W[0, j] = 6.0
            W[3 * int(rng.integers(1, max(2, V // 3))), j] = 4.0            # b = 0 there: logit 4.0 exactly
            few = rng.choice(np.arange(1, V), size=min(V - 1, 6), replace=False)
            W[few[few % 3 != 0], j] = 3.5
    W = _bf16(W)
    b = B_LEVELS[np.arange(V) % 3].copy()
    return W, b


@pytest.fixture(scope="module")
def ctc_models(tmp_path_factory):
    """(V, precision) -> (ReverbASR, W, b), loaded on first use."""
    import reverb_b200
    dirs, models = {}, {}

    def get(V, precision):
        if V not in dirs:
            d = synth.write_model_dir(str(tmp_path_factory.mktemp(f"ctc_v{V}")), shape=dict(synth.TEST_SHAPE, vocab=V))
            W, b = _ctc_head(V)
            p = os.path.join(d, "synth.pt")
            sd = torch.load(p)
            assert tuple(sd["ctc.ctc_lo.weight"].shape) == W.shape
            sd["ctc.ctc_lo.weight"] = torch.from_numpy(W)
            sd["ctc.ctc_lo.bias"] = torch.from_numpy(b)
            torch.save(sd, p)
            dirs[V] = (d, W, b)
        if (V, precision) not in models:
            d, W, b = dirs[V]
            models[(V, precision)] = (reverb_b200.load_model(d, precision=precision), W, b)
        return models[(V, precision)]
    return get


def _one_hot_enc(cols, B, Tp):
    e = np.zeros((B * Tp, D_MODEL), np.float32)
    e[np.arange(B * Tp), cols] = 1.0
    return torch.from_numpy(e).view(B, Tp, D_MODEL).cuda()


def _logsoftmax64(x):
    x = np.asarray(x, np.float64)
    m = x.max(axis=1, keepdims=True)
    return (x - m) - np.log(np.exp(x - m).sum(axis=1, keepdims=True))


@pytest.mark.parametrize("precision", ["bf16", "fp32"])
@pytest.mark.parametrize("V", CTC_VOCABS)
def test_ctc_topk_on_exact_logits(ctc_models, V, precision):
    """Indices: the stable order of the float32 logits after the blank penalty.  Values and the full logp rows:
    float64 log_softmax to 1e-5.  A larger batch runs first, so the smaller one reads a logits buffer that already
    holds values; V is never a multiple of 4, so every logits row has padding columns."""
    m, W, b = ctc_models(V, precision)
    eng = m.engine
    rng = np.random.default_rng(V + 7)
    Tp = 43
    for B in (6, 2):
        cols = rng.permutation(np.resize(np.arange(D_MODEL), B * Tp))
        logits = W[:, cols].T + b                                          # float32 arithmetic: exact GEMM output
        for k, pen in ((10, 0.0), (16, 2.0), (4, 1.25), (16, 40.0), (1, 0.0)):
            x = logits.copy()
            if pen > 0:
                x[:, 0] = x[:, 0] - np.float32(pen)
            val, idx, logp = eng.ctc_topk(_one_hot_enc(cols, B, Tp), k, pen, 0, want_logp=True)
            idx = idx.view(B * Tp, k).cpu().numpy()
            val = val.view(B * Tp, k).cpu().numpy()
            logp = logp.view(B * Tp, V).cpu().numpy()
            want = stable_topk(x, k)
            bad = np.nonzero((idx != want).any(axis=1))[0]
            assert bad.size == 0, (B, k, pen, bad[0], idx[bad[0]].tolist(), want[bad[0]].tolist())
            ref = _logsoftmax64(x)
            np.testing.assert_allclose(logp, ref, rtol=0, atol=1e-5, err_msg=f"logp B={B} k={k} pen={pen}")
            np.testing.assert_allclose(val, np.take_along_axis(ref, want, 1), rtol=0, atol=1e-5)
            np.testing.assert_array_equal(val.view(np.int32), np.take_along_axis(logp, idx, 1).view(np.int32))
            blank_led = cols % 4 == 3
            if pen == 2.0:                          # penalised blank 4.0 ties with a token at 4.0: blank first
                assert (idx[blank_led, 0] == 0).all() and (idx[blank_led, 1] % 3 == 0).all()
                assert (x[blank_led, idx[blank_led, 1]] == x[blank_led, 0]).all()
            if pen == 40.0:
                assert not (idx == 0).any()         # the blank left the top-k
            if pen == 0.0 and k == 10:
                # the coarse-level rows tie across the top-k: they are the ones that pin the index order on ties
                tied = cols % 4 == 2
                assert (x[tied, want[tied, k - 1]] == x[tied, want[tied, 0]]).all()


# ---------------------------------------------------------------------------------------------------------------------
# 3. ctc_greedy through Engine.greedy_search

def _collapse(ids, blank=0):
    out, prev = [], None
    for i in ids:
        if i != prev and i != blank:
            out.append(int(i))
        prev = i
    return out


def _greedy_sequences(rng, T, V=1000):
    """Id sequences aimed at the 32-frame steps of the kernel."""
    seqs = []
    a = rng.integers(0, 6, T)                                  # general: short runs of few ids, blanks included
    for s, e, tok in ((30, 34, 7), (62, 66, 9)):               # repeats across 31|32 and 63|64
        a[s:e] = tok
    seqs.append(a)
    for blanks in ((31, 63), (32, 64)):                        # a repeat split by one blank at the end / the start
        a = rng.integers(1, V, T)                              # of a step
        for p, tok in zip(blanks, (5, 6)):
            if p + 1 < T:
                a[p - 1], a[p], a[p + 1] = tok, 0, tok
        seqs.append(a)
    seqs.append(np.zeros(T, np.int64))                         # all blank
    seqs.append(1 + np.arange(T) % 2)                          # alternating: output length = input length
    a = np.zeros(T, np.int64)                                  # a run filling a whole step, then the same id again
    a[32:64] = 8
    a[64:66] = 8
    a[:32] = 3
    a[96:128] = 4
    seqs.append(a)
    seqs.append(np.where(rng.random(T) < 0.6, 0, rng.integers(1, V, T)))
    return [np.asarray(s, np.int64) for s in seqs]


@pytest.mark.parametrize("k", [1, 10, 16])
@pytest.mark.parametrize("T", [1, 31, 32, 33, 64, 65, 748, 3001])
def test_greedy_collapse(eng, T, k):
    """Token lists equal the collapse of idx[b, :min(len, T), 0]; later index columns hold decoys; lens beyond T are
    clamped to T."""
    rng = np.random.default_rng([T, k])
    seqs = _greedy_sequences(rng, T)
    lens_per_seq = sorted({0, 1, max(T - 1, 0), T, T + 5, int(rng.integers(0, T + 1))})
    ids = np.stack([s for s in seqs for _ in lens_per_seq])
    lens = np.array([n for _ in seqs for n in lens_per_seq], np.int32)
    B = ids.shape[0]
    top = rng.integers(0, 1000, (B, T, k)).astype(np.int32)   # decoys
    top[:, :, 0] = ids
    got = eng.greedy_search(torch.from_numpy(top).cuda(), lens, 0)
    for b in range(B):
        assert got[b] == _collapse(ids[b, :min(int(lens[b]), T)]), (b, int(lens[b]))
    clamp = lens == T + 5
    assert [got[b] for b in np.nonzero(clamp)[0]] == [got[b] for b in np.nonzero(lens == T)[0]]


def test_greedy_on_kernel_topk_equals_the_oracle(eng):
    """Kernel top-k of random peaky log-probs at V = 10001, then greedy: equal to search_ref.ctc_greedy_search."""
    rng = np.random.default_rng(3)
    B, T, V = 4, 300, 10001
    logp = np.concatenate([_peaky_logp(rng, T, V, 1)[None] for _ in range(B)])
    lens = np.array([T, T - 1, 37, 1], np.int32)
    _, idx = eng.logp_topk(torch.from_numpy(logp).cuda(), 1)
    got = eng.greedy_search(idx, lens, 0)
    want = search_ref.ctc_greedy_search(torch.from_numpy(logp), torch.from_numpy(lens), 0)
    assert got == [w.tokens for w in want]
    assert sum(len(g) for g in got) > 50


# ---------------------------------------------------------------------------------------------------------------------
# 4. The plain prefix beam search on both trie layouts, against oracle/search_ref.py

def trie_in_smem(T, beam):
    """The launcher's choice (csrc/ctc.cu pb_layout / launch_prefix_beam): node pool of beam * T + 2 entries (parent
    and token) plus a power-of-two hash table of at least twice the pool, in shared memory up to 150 KB."""
    pool = beam * T + 2
    h = 64
    while h < 2 * pool:
        h <<= 1
    return (2 * pool + h) * 4 <= SMEM_TRIE_BYTES


def _peaky_logp(rng, T, V, beam):
    """(T, V) float32 CTC-like log-probs (float64 log_softmax): blank-dominated, with token bursts, repeats,
    repeats split by one blank and near-ties between 2-3 tokens.  Frames are redrawn until the top beam + 1 values of
    every frame are distinct, so the top-k of the GPU and torch.topk in the oracle agree without a tie rule."""
    x = rng.standard_normal((T, V))
    x[:, 0] += 7.0                                              # blank is always a strong candidate
    rows = np.arange(T)[:, None]
    x[rows, rng.integers(1, V, (T, 3))] += rng.uniform(4.0, 8.0, (T, 3))   # competitors a few nats down
    t = 0
    while t < T:
        r = rng.random()
        if r < 0.4:                                             # blank run
            n = int(rng.integers(1, 6))
            x[t:t + n, 0] += rng.uniform(3.0, 6.0)
        elif r < 0.65:                                          # a token held 1-3 frames
            n = int(rng.integers(1, 4))
            x[t:t + n, int(rng.integers(1, V))] += rng.uniform(8.0, 11.0)
        elif r < 0.8:                                           # token, one blank frame, the same token
            n = 3
            tok = int(rng.integers(1, V))
            x[t:t + 3:2, tok] += 10.0
            x[t + 1:t + 2, 0] += 6.0
        else:                                                   # near-tie of 2-3 tokens
            n = 1
            toks = rng.choice(np.arange(1, V), size=int(rng.integers(2, 4)), replace=False)
            x[t, toks] += 9.0 + rng.uniform(0.0, 0.2, toks.size)
        t += n
    while True:
        m = x.max(axis=1, keepdims=True)
        lp = ((x - m) - np.log(np.exp(x - m).sum(axis=1, keepdims=True))).astype(np.float32)
        top = np.sort(-np.partition(-lp, beam, axis=1)[:, :beam + 1], axis=1)
        tied = np.nonzero((np.diff(top, axis=1) == 0).any(axis=1))[0]
        if tied.size == 0:
            return lp
        x[tied] += 1e-3 * rng.standard_normal((tied.size, V))


PB_CASES = [(1, 748), (4, 748), (10, 748), (16, 748), (10, 1500), (16, 3000)]
PB_SMEM = {(1, 748): True, (4, 748): True, (10, 748): True, (16, 748): False, (10, 1500): False, (16, 3000): False}
PB_V = 10001


def test_prefix_search_cases_cover_both_trie_layouts():
    assert {c: trie_in_smem(c[1], c[0]) for c in PB_CASES} == PB_SMEM
    assert set(PB_SMEM.values()) == {True, False}


@pytest.fixture(scope="module")
def pb_inputs():
    """(beam, T) -> (logp (B, T, V) float32 numpy, lens, host search results).  The cases that more than one test
    uses are kept: the host search is the slow part."""
    cache = {}

    def get(beam, T):
        if (beam, T) in cache:
            return cache[(beam, T)]
        rng = np.random.default_rng([beam, T])
        lens = np.array([T, T - 1, 1, 2, T // 2 + 7], np.int32)
        logp = np.stack([_peaky_logp(rng, T, PB_V, beam) for _ in lens])
        want = search_ref.ctc_prefix_beam_search(torch.from_numpy(logp), torch.from_numpy(lens), beam, 0)
        if T == 748 and beam >= 10:
            cache[(beam, T)] = (logp, lens, want)
        return logp, lens, want
    return get


def _assert_equals_oracle(got, want):
    for b, ((nbest, scores, times), w) in enumerate(zip(got, want)):
        assert len(nbest) == len(w.nbest), b
        assert [list(h) for h in nbest] == [list(h) for h in w.nbest], b
        assert times == [list(t) for t in w.nbest_times], b
        np.testing.assert_allclose(scores, w.nbest_scores, rtol=1e-9, atol=0)


@pytest.mark.parametrize("beam,T", PB_CASES)
def test_prefix_search_equals_the_oracle(eng, pb_inputs, beam, T):
    """Kernel top-k + plain prefix beam search == search_ref.ctc_prefix_beam_search on the same float32 log-probs:
    n-best tokens and times identical, scores to 1e-9; two launches give the same bytes."""
    logp, lens, want = pb_inputs(beam, T)
    val, idx = eng.logp_topk(torch.from_numpy(logp).cuda(), beam)
    got = eng.prefix_beam_search(val, idx, lens, beam, 0)
    _assert_equals_oracle(got, want)
    assert max(len(h) for g in got for h in g[0]) > 10
    one = eng.prefix_beam_search_raw(val, idx, lens, beam, 0)
    two = eng.prefix_beam_search_raw(val, idx, lens, beam, 0)
    for a, b in zip(one, two):
        assert a.tobytes() == b.tobytes()


@pytest.mark.parametrize("beam,T", [(10, 748), (16, 748)])
def test_plain_search_after_a_biased_one_equals_the_oracle(eng, pb_inputs, beam, T):
    """The biased and the plain search share the workspace and, for the global layout, the trie in it."""
    from reverb_b200.context_graph import ContextGraph
    from reverb_b200.engine import DeviceContextGraph
    logp, lens, want = pb_inputs(beam, T)
    val, idx = eng.logp_topk(torch.from_numpy(logp).cuda(), beam)
    phrases = [list(h[-3:]) for w in want for h in w.nbest[1:] if len(h) >= 3][:20]   # promotes lower-ranked ones
    biased = eng.prefix_beam_search(val, idx, lens, beam, 0,
                                    context=DeviceContextGraph(ContextGraph(token_lists=phrases, context_score=3.0),
                                                               PB_V, 0))
    assert any(g[0] != list(w.nbest) for g, w in zip(biased, want))
    _assert_equals_oracle(eng.prefix_beam_search(val, idx, lens, beam, 0), want)


def _raw_prefix_search(eng, val, idx, lens, beam, max_len):
    B, T, k = idx.shape
    toks = np.full((B, beam, max_len), -7, np.int32)
    tims = np.full((B, beam, max_len), -7, np.int32)
    olen = np.full((B, beam, 2), -7, np.int32)
    scores = np.full((B, beam), -7.0)
    nhyp = np.full(B, -7, np.int32)
    p = lambda a: a.ctypes.data_as(C.c_void_p)                          # noqa: E731
    with torch.cuda.device(eng.device):
        rc = eng.lib.rvb_ctc_prefix_beam_search(C.c_void_p(val.data_ptr()), C.c_void_p(idx.data_ptr()), k, p(lens),
                                                B, T, beam, 0, max_len, p(toks), p(tims), p(olen), p(scores), p(nhyp),
                                                eng._stream())
    return rc, (toks, tims, olen, scores, nhyp)


def test_prefix_search_reports_max_len_overflow_and_k_below_beam(eng, pb_inputs):
    from reverb_b200 import _lib
    logp, lens, want = pb_inputs(10, 748)
    val, idx = eng.logp_topk(torch.from_numpy(logp).cuda(), 10)
    longest = max(len(h) for w in want for h in w.nbest)
    rc, _ = _raw_prefix_search(eng, val, idx, lens, 10, longest)
    assert rc == 0
    rc, _ = _raw_prefix_search(eng, val, idx, lens, 10, longest - 1)
    assert rc != 0 and "exceeds max_len" in _lib.last_error()
    val4, idx4 = val[..., :4].contiguous(), idx[..., :4].contiguous()
    rc, outs = _raw_prefix_search(eng, val4, idx4, lens, 10, longest)
    assert rc != 0 and "k >= beam" in _lib.last_error()
    for a in outs:
        assert (a == -7).all()
