"""Float64 reference of attention rescoring and the prefix trees the tree-structured decoder builds.

* `synthetic_topk`: CTC top-k tensors whose prefix beam search gives n-best lists of a known structure (long shared
  prefixes, bushy trees, blank-only and very short utterances, hypotheses that are prefixes / suffixes of others).
* `prefix_tree`: the prefix tree of one utterance's n-best with the insertion rule of ctc.cu trie_build_kernel, and
  `ancestor_bits`: the self-attention mask rows trie_inputs_kernel writes for it.
* `decoder_scores`: the teacher-forced log-probability of every (hypothesis, position) of attention_rescoring, from
  `model_ref.decoder_forward` run in float64.
"""
from __future__ import annotations

import math
from typing import Dict, List, Sequence

import numpy as np
import torch

from . import model_ref


def _frame(rng, k: int, V: int, cands, floor=(-9.0, -6.0)):
    """One top-k row: the given (token, log-prob) candidates plus low fillers, distinct tokens, sorted descending."""
    used = {t for t, _ in cands}
    out = list(cands)
    while len(out) < k:
        t = int(rng.integers(1, V - 1))
        if t not in used:
            used.add(t)
            out.append((t, float(rng.uniform(*floor))))
    out.sort(key=lambda x: -x[1])
    return out[:k]


def _tokens(rng, n: int, V: int) -> List[int]:
    """n tokens (not blank, not sos/eos), no two neighbours equal"""
    out = []
    while len(out) < n:
        t = int(rng.integers(1, V - 1))
        if not out or out[-1] != t:
            out.append(t)
    return out


def synthetic_topk(families: Sequence[str], enc_lens: Sequence[int], Tp: int, V: int, k: int, seed: int = 0):
    """-> (val (B, Tp, k) float32 sorted descending, idx (B, Tp, k) int32).  Frames at or past enc_len hold fillers.

    deep:   one dominant token every 3rd frame, blank in between; near-tied pairs at the 41st and 81st emission, so the
            n-best shares long prefixes and diverges late (U ~ enc_len / 3).
    bushy:  one emission every 4th frame; the first 12 emissions are near-tied pairs, so the n-best diverges early and
            the tree has ~ beam x U nodes.
    blank:  every frame blank-dominant: the n-best holds the empty hypothesis and one- or two-token hypotheses.
    short:  flat rows (meant for enc_len 1-3): the cross-attention sees one to three keys.
    prefix: like deep, but the first emission ties two tokens and blank (the reversed trees share long prefixes, one
            reversed hypothesis is a proper prefix of others) and the last emission ties with blank (one hypothesis is
            a proper prefix of another)."""
    rng = np.random.default_rng(seed)
    B = len(families)
    val = np.zeros((B, Tp, k), np.float32)
    idx = np.zeros((B, Tp, k), np.int32)
    j = lambda: float(rng.uniform(-0.02, 0.02))  # noqa: E731  (jitter: no exact score ties between paths)
    for b, (fam, L) in enumerate(zip(families, enc_lens)):
        rows = []
        if fam in ("deep", "prefix", "bushy"):
            step = 4 if fam == "bushy" else 3
            n_emit = (L + step - 1) // step
            seq = _tokens(rng, n_emit, V)
            alt = _tokens(rng, n_emit, V)
            for t in range(L):
                e, ph = divmod(t, step)
                if ph == 0:
                    tie = (fam == "deep" and e in (40, 80)) or (fam == "bushy" and e < 12)
                    a = alt[e] if alt[e] != seq[e] else (seq[e] % (V - 2)) + 1
                    if tie:
                        c = [(seq[e], math.log(0.48) + j()), (a, math.log(0.46) + j()), (0, -3.0 + j())]
                    elif fam == "prefix" and e == 0:
                        c = [(seq[e], math.log(0.36) + j()), (a, math.log(0.32) + j()), (0, math.log(0.28) + j())]
                    elif fam == "prefix" and e == n_emit - 1:
                        c = [(seq[e], math.log(0.49) + j()), (0, math.log(0.47) + j())]
                    else:
                        c = [(seq[e], math.log(0.9) + j()), (0, -2.8 + j()), (a, -4.0 + j())]
                else:
                    c = [(0, math.log(0.92) + j()), (seq[e], -3.2 + j())]
                rows.append(_frame(rng, k, V, c))
        elif fam == "blank":
            for t in range(L):
                rows.append(_frame(rng, k, V, [(0, math.log(0.95) + j()), (int(rng.integers(1, V - 1)), -3.5 + j())]))
        elif fam == "short":
            for t in range(L):
                c = [(0, -1.0 + j())] + [(tt, -1.4 - 0.25 * i + j()) for i, tt in enumerate(_tokens(rng, 6, V))]
                rows.append(_frame(rng, k, V, c))
        else:
            raise ValueError(fam)
        for t in range(Tp):
            r = rows[t] if t < L else _frame(rng, k, V, [])
            idx[b, t] = [x[0] for x in r]
            val[b, t] = [x[1] for x in r]
    return val, idx


def full_logp(val: np.ndarray, idx: np.ndarray, V: int, b: int, length: int) -> torch.Tensor:
    """(1, length, V) float32 rows holding the top-k entries and -1e30 elsewhere: the top-k of a row is the given one,
    so search_ref.ctc_prefix_beam_search sees what the device search sees."""
    x = torch.full((1, length, V), -1e30, dtype=torch.float32)
    x[0].scatter_(1, torch.from_numpy(idx[b, :length].astype(np.int64)), torch.from_numpy(val[b, :length]))
    return x


def prefix_tree(hyps: Sequence[Sequence[int]], reverse: bool = False) -> Dict[str, list]:
    """The prefix tree of one utterance's n-best, built as trie_build_kernel builds it: hypotheses in n-best order,
    each sharing the nodes of the FIRST earlier hypothesis with the longest common prefix.  node 0 = empty prefix.
    -> {"par", "tok", "dep": per node; "node_of": per hypothesis the node of each prefix length 0..U; "lcp": per
    hypothesis the shared prefix length (0 for the first)}."""
    seqs = [tuple(h)[::-1] if reverse else tuple(h) for h in hyps]
    par, tok, dep, node_of, lcp = [-1], [None], [0], [], []
    for i, s in enumerate(seqs):
        best, bl = -1, 0
        for ip in range(i):
            o = seqs[ip]
            n = 0
            while n < min(len(s), len(o)) and s[n] == o[n]:
                n += 1
            if n > bl:
                best, bl = ip, n
        mine = [0] + (node_of[best][1:bl + 1] if best >= 0 else [])
        for jj in range(bl, len(s)):
            par.append(mine[-1])
            tok.append(s[jj])
            dep.append(jj + 1)
            mine.append(len(par) - 1)
        node_of.append(mine)
        lcp.append(bl)
    return {"par": par, "tok": tok, "dep": dep, "node_of": node_of, "lcp": lcp}


def padded_slots(node_counts: Sequence[int]) -> int:
    """P: node slots per utterance of a batch (engine.cu rescoring_submit), the largest tree rounded up to 8"""
    return (max([1] + list(node_counts)) + 7) & ~7


def ancestor_bits(par: Sequence[int], P: int) -> np.ndarray:
    """(P, 2 * ceil(P / 64)) int32 mask rows as trie_inputs_kernel writes them: bit j of row i set iff node slot j is
    node i or one of its ancestors; unused slots (>= len(par)) see only themselves."""
    ld = 2 * ((P + 63) // 64)
    vis = np.zeros((P, ld * 32), bool)
    for i in range(P):
        if i < len(par):
            c = i
            while c >= 0:
                vis[i, c] = True
                c = par[c]
        else:
            vis[i, i] = True
    words = (vis.reshape(P, ld, 32).astype(np.uint64) << np.arange(32, dtype=np.uint64)).sum(-1)
    return words.astype(np.uint32).view(np.int32)


def decoder_scores(memory: torch.Tensor, hyps: Sequence[Sequence[int]], sd64, cfg, cat64, sos: int, eos: int,
                   side: str) -> List[np.ndarray]:
    """Float64 attention-rescoring scores of one utterance: memory (T, d) = its valid encoder frames.  -> per
    hypothesis a (U + 1,) array whose entry j is log p(w_j) (j < U) and entry U is log p(<eos>), both decoders in
    hypothesis order (search.py:413-430): the right-to-left decoder reads [sos, w_U .. w_1] and its position U-1-j
    scores w_j."""
    from .search_ref import rescoring_inputs
    hyps = [tuple(h) for h in hyps]
    ys, ylens = rescoring_inputs(hyps, sos, eos)
    if side == "right_decoder":
        ys = model_ref.reverse_hyps(ys, ylens, eos) if ys.shape[1] > 1 else ys
    mem = memory.to(torch.float64).unsqueeze(0).expand(len(hyps), -1, -1)
    with torch.no_grad():
        lp = torch.log_softmax(model_ref.decoder_forward(mem, ys, ylens, sd64, cfg, side, cat64), -1)
    out = []
    for i, h in enumerate(hyps):
        U = len(h)
        pos = range(U) if side == "left_decoder" else range(U - 1, -1, -1)
        s = [float(lp[i, p, w]) for p, w in zip(pos, h)] + [float(lp[i, U, eos])]
        out.append(np.asarray(s, np.float64))
    return out


def to_float64(sd) -> dict:
    return {k: (v.double() if v.is_floating_point() else v) for k, v in sd.items()}
