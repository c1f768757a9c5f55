"""Host side of the decoding methods: result container and the (tiny) score arithmetic that
stays on the CPU.  The searches themselves run on the GPU (csrc/ctc.cu) through Engine.

Mirrors asr/wenet/transformer/search.py of the reference: `DecodeResult` (:29-58), the
output contract of `ctc_greedy_search` (:106-121), `ctc_prefix_beam_search` (:124-248)
and the score combination of `attention_rescoring` (:413-447).
"""
from __future__ import annotations

import math
from typing import List, Optional, Sequence

import numpy as np


class DecodeResult:
    """Same fields, defaults and meaning as the reference's DecodeResult (search.py:29-58)."""

    def __init__(self, tokens, score: float = 0.0, confidence: float = 0.0,
                 tokens_confidence: Optional[List[float]] = None, times: Optional[List[int]] = None,
                 nbest=None, nbest_scores: Optional[List[float]] = None, nbest_times=None):
        self.tokens = tokens
        self.score = score
        self.confidence = confidence
        self.tokens_confidence = tokens_confidence
        self.times = times
        self.nbest = nbest
        self.nbest_scores = nbest_scores
        self.nbest_times = nbest_times

    def __repr__(self):
        return f"DecodeResult(tokens={list(self.tokens)}, score={self.score}, confidence={self.confidence})"


def greedy_results(token_lists: Sequence[Sequence[int]]) -> List[DecodeResult]:
    # the reference's greedy search returns tokens only (times / confidence stay None, search.py:119)
    return [DecodeResult(list(t)) for t in token_lists]


def prefix_beam_results(per_utt) -> List[DecodeResult]:
    """per_utt: Engine.prefix_beam_search output.  Best hypothesis = first of the n-best (search.py:235-247)."""
    out = []
    for nbest, scores, times in per_utt:
        out.append(DecodeResult(tokens=nbest[0], score=scores[0], times=times[0], nbest=nbest,
                                nbest_scores=scores, nbest_times=times))
    return out


def _log_add2(a: float, b: float) -> float:
    """utils/common.py log_add([a, b]): max + log(sum(exp(x - max))) in double precision, -inf when both are."""
    if a == -math.inf and b == -math.inf:
        return -math.inf
    m = a if a > b else b
    return m + math.log(math.exp(a - m) + math.exp(b - m))


class _Prefix:
    """PrefixScore of the reference (search.py:60-104)."""
    __slots__ = ("s", "ns", "v_s", "v_ns", "cur_token_prob", "times_s", "times_ns", "context_state", "context_score",
                 "has_context")

    def __init__(self, s=-math.inf, ns=-math.inf, v_s=-math.inf, v_ns=-math.inf, context_state=None, context_score=0.0):
        self.s, self.ns, self.v_s, self.v_ns = s, ns, v_s, v_ns
        self.cur_token_prob = -math.inf
        self.times_s: List[int] = []
        self.times_ns: List[int] = []
        self.context_state = context_state
        self.context_score = context_score
        self.has_context = False

    def score(self) -> float:
        return _log_add2(self.s, self.ns)

    def viterbi(self) -> float:
        return self.v_s if self.v_s > self.v_ns else self.v_ns

    def times(self) -> List[int]:
        return self.times_s if self.v_s > self.v_ns else self.times_ns

    def total(self) -> float:
        return self.score() + self.context_score


def ctc_prefix_beam_search_biased(topk_val: np.ndarray, topk_idx: np.ndarray, lens: Sequence[int], beam_size: int,
                                  context_graph, blank_id: int = 0) -> List[DecodeResult]:
    """CTC prefix beam search WITH a context graph (search.py:124-248, the `context_graph is not None` branches), on the
    host over the per-frame top-`beam_size` log-probabilities the GPU CTC head produced.  `ASRModel.decode` runs the
    biased GPU search (csrc/ctc.cu, csrc/context.cu) instead; this restatement is what the tests compare it against.
    topk_val / topk_idx: (B, T', beam) in `torch.topk` order.  Reference behaviours kept: ranking by score + context score; the `u == last` repeat branch never updates
    `v_ns` (the `vs_ns` typo, :177); after the last frame `finalize` REPLACES each hypothesis' context score by minus the
    bonus of its unfinished match (:228-233) and the list is not re-sorted."""
    out: List[DecodeResult] = []
    for b in range(topk_val.shape[0]):
        cur = [((), _Prefix(s=0.0, ns=-math.inf, v_s=0.0, v_ns=0.0, context_state=context_graph.root, context_score=0.0))]
        for t in range(int(lens[b])):
            nxt: dict = {}

            def slot(key):
                ps = nxt.get(key)
                if ps is None:
                    ps = nxt[key] = _Prefix()
                return ps

            for j in range(beam_size):
                u = int(topk_idx[b, t, j])
                prob = float(topk_val[b, t, j])
                for prefix, ps in cur:
                    last = prefix[-1] if prefix else None
                    if u == blank_id:
                        n = slot(prefix)
                        n.s = _log_add2(n.s, ps.score() + prob)
                        n.v_s = ps.viterbi() + prob
                        n.times_s = list(ps.times())
                        if not n.has_context:
                            n.context_score, n.context_state, n.has_context = ps.context_score, ps.context_state, True
                    elif u == last:
                        n1 = slot(prefix)
                        n1.ns = _log_add2(n1.ns, ps.ns + prob)
                        if n1.v_ns < ps.v_ns + prob:
                            # the reference assigns to a misspelt attribute here: v_ns itself stays as it was
                            if n1.cur_token_prob < prob:
                                n1.cur_token_prob = prob
                                n1.times_ns = list(ps.times_ns)
                                n1.times_ns[-1] = t
                        if not n1.has_context:
                            n1.context_score, n1.context_state, n1.has_context = ps.context_score, ps.context_state, True
                        n2 = slot(prefix + (u,))
                        n2.ns = _log_add2(n2.ns, ps.s + prob)
                        if n2.v_ns < ps.v_s + prob:
                            n2.v_ns = ps.v_s + prob
                            n2.cur_token_prob = prob
                            n2.times_ns = list(ps.times_s)
                            n2.times_ns.append(t)
                        if not n2.has_context:
                            sc, st = context_graph.forward_one_step(ps.context_state, u)
                            n2.context_score, n2.context_state, n2.has_context = ps.context_score + sc, st, True
                    else:
                        n = slot(prefix + (u,))
                        n.ns = _log_add2(n.ns, ps.score() + prob)
                        if n.v_ns < ps.viterbi() + prob:
                            n.v_ns = ps.viterbi() + prob
                            n.cur_token_prob = prob
                            n.times_ns = list(ps.times())
                            n.times_ns.append(t)
                        if not n.has_context:
                            sc, st = context_graph.forward_one_step(ps.context_state, u)
                            n.context_score, n.context_state, n.has_context = ps.context_score + sc, st, True
            # sorted() is stable: equal totals keep dict insertion order, like the reference
            cur = sorted(nxt.items(), key=lambda kv: kv[1].total(), reverse=True)[:beam_size]
        for _, ps in cur:
            ps.context_score, ps.context_state = context_graph.finalize(ps.context_state)
        nbest = [k for k, _ in cur]
        scores = [ps.total() for _, ps in cur]
        times = [ps.times() for _, ps in cur]
        out.append(DecodeResult(tokens=nbest[0], score=scores[0], times=times[0], nbest=nbest, nbest_scores=scores,
                                nbest_times=times))
    return out


def rescoring_pick(hyps: Sequence[tuple], ctc_scores: Sequence[float], nbest_times, l2r: np.ndarray,
                   r2l: Optional[np.ndarray], ctc_weight: float, reverse_weight: float) -> DecodeResult:
    """Combine decoder and CTC scores and keep the first strict maximum (search.py:413-447).

    l2r[i, j] = log p(w_j | w_<j) for j < U_i, l2r[i, U_i] = log p(eos), zeros behind; r2l likewise for the
    right-to-left decoder (already re-indexed to hypothesis order).  Float semantics follow the reference: the
    decoder scores are summed sequentially in float32 (0-d float32 tensors there) — `np.add.accumulate` is the same
    left-to-right float32 recurrence, and the trailing zeros are exact no-ops — while confidences and the CTC term
    go through double precision Python floats.
    """
    n = len(hyps)
    lens = np.fromiter((len(h) for h in hyps), dtype=np.int64, count=n)
    score = np.add.accumulate(np.ascontiguousarray(l2r[:n], dtype=np.float32), axis=1, dtype=np.float32)[:, -1]
    use_r = reverse_weight > 0 and r2l is not None
    if use_r:
        r_score = np.add.accumulate(np.ascontiguousarray(r2l[:n], dtype=np.float32), axis=1, dtype=np.float32)[:, -1]
        score = (score * np.float32(1 - reverse_weight) + r_score * np.float32(reverse_weight)).astype(np.float32)
    norm = (score / (lens + 1).astype(np.float32)).astype(np.float32)
    ctc_term = np.asarray([c * ctc_weight for c in ctc_scores[:n]], dtype=np.float64).astype(np.float32)
    total = (score + ctc_term).astype(np.float32)
    best = int(np.argmax(total)) if n and not np.isnan(total).any() else 0     # first maximum == strict `>` scan
    if n and np.isnan(total).any():                                            # keep the reference's scan semantics
        best, best_score = 0, -float("inf")
        for i in range(n):
            if float(total[i]) > best_score:
                best, best_score = i, float(total[i])
    U = int(lens[best])
    tc = [math.exp(float(l2r[best, j])) for j in range(U)]
    if use_r:
        tc = [(tc[j] + math.exp(float(r2l[best, j]))) / 2 for j in range(U)]
    return DecodeResult(hyps[best], float(total[best]), confidence=math.exp(float(norm[best])),
                        times=nbest_times[best], tokens_confidence=tc)


def rescoring_pick_batch(toks: np.ndarray, tims: np.ndarray, olen: np.ndarray, ctc_scores: np.ndarray,
                         nhyp: np.ndarray, l2r: np.ndarray, r2l: Optional[np.ndarray], ctc_weight: float,
                         reverse_weight: float) -> List[DecodeResult]:
    """`rescoring_pick` for a whole batch straight from the prefix-beam arrays (no per-hypothesis Python objects):
    toks/tims (B, N, L), olen (B, N, 2), ctc_scores (B, N) float64, nhyp (B,), l2r/r2l (B, N, Lmax+1) float32.
    Same float semantics as `rescoring_pick` (sequential float32 sums, see there)."""
    B, N = ctc_scores.shape
    lens = olen[:, :, 0].astype(np.int64)
    score = np.add.accumulate(l2r, axis=2, dtype=np.float32)[:, :, -1]
    use_r = reverse_weight > 0 and r2l is not None
    if use_r:
        r_score = np.add.accumulate(r2l, axis=2, dtype=np.float32)[:, :, -1]
        score = (score * np.float32(1 - reverse_weight) + r_score * np.float32(reverse_weight)).astype(np.float32)
    norm = (score / (lens + 1).astype(np.float32)).astype(np.float32)
    total = (score + (ctc_scores * ctc_weight).astype(np.float32)).astype(np.float32)
    valid = np.arange(N)[None, :] < nhyp[:, None]
    total = np.where(valid, total, -np.inf).astype(np.float32)
    best = np.argmax(total, axis=1)                      # first maximum == the reference's strict `>` scan
    out = []
    for b in range(B):
        i = int(best[b])
        U = int(lens[b, i])
        # exp in float64 of the float32 log-probs (numpy's vectorised exp; the reference's math.exp may differ by 1 ulp)
        tc = np.exp(l2r[b, i, :U].astype(np.float64))
        if use_r:
            tc = (tc + np.exp(r2l[b, i, :U].astype(np.float64))) / 2
        nt = int(olen[b, i, 1])
        out.append(DecodeResult(tuple(toks[b, i, :U].tolist()), float(total[b, i]),
                                confidence=math.exp(float(norm[b, i])), times=tims[b, i, :nt].tolist(),
                                tokens_confidence=tc.tolist()))
    return out


def attention_beam_search(step_topk, batch_size: int, maxlen: int, beam_size: int, sos: int, eos: int,
                          length_penalty: float = 0.0) -> List[DecodeResult]:
    """Host bookkeeping of the `attention` decode mode (transformer/search.py:251-360, non-whisper branch), numpy
    float32 like the reference's tensors.  step_topk(hyps (B*N, i) int64, parents (B*N,) or None) -> (logp (B*N, N),
    index (B*N, N)) is the decoder step: `parents[s]` = row (of the previous call's hyps) that row s extends — what the
    reference uses to re-index its decoder cache (:341-346) and what the KV-cached native step needs
    (Engine.decoder_cache_step); a step function that recomputes the prefix (Engine.decoder_step_topk) ignores it.  Finished beams keep one zero-cost <eos> branch (utils/mask.py:257-303);
    the best beam per utterance is chosen after the length penalty; returns DecodeResult(tokens) only (no times /
    confidences: `transcribe(mode="attention")` fails in the reference for that reason, SURVEY.md §8a quirk 1)."""
    B, N = batch_size, beam_size
    running = B * N
    neg_inf = np.float32(-np.inf)
    hyps = np.full((running, 1), sos, dtype=np.int64)
    scores = np.tile(np.array([0.0] + [-np.inf] * (N - 1), dtype=np.float32), B).reshape(-1, 1)
    end_flag = np.zeros((running, 1), dtype=bool)
    zeros = np.zeros((running, 1), dtype=bool)
    parents = None
    for _ in range(1, maxlen + 1):
        if int(end_flag.sum()) == running:
            break
        logp, index = step_topk(hyps, parents)
        logp = np.array(logp, dtype=np.float32, copy=True).reshape(running, N)
        index = np.array(index, dtype=np.int64, copy=True).reshape(running, N)
        if N > 1:
            unfinished = np.concatenate([zeros, np.repeat(end_flag, N - 1, axis=1)], axis=1)
            finished = np.concatenate([end_flag, np.repeat(zeros, N - 1, axis=1)], axis=1)
        else:
            unfinished, finished = zeros, end_flag
        logp[unfinished] = neg_inf
        logp[finished] = 0.0
        index[np.repeat(end_flag, N, axis=1)] = eos
        cand = (scores + logp).astype(np.float32).reshape(B, N * N)
        order = np.argsort(-cand, axis=1, kind="stable")[:, :N]            # topk, sorted, ties -> lowest index
        scores = np.take_along_axis(cand, order, axis=1).reshape(-1, 1)
        best_k_index = (np.arange(B)[:, None] * N * N + order).reshape(-1)
        best_k_pred = index.reshape(-1)[best_k_index]
        parents = best_k_index // N
        hyps = np.concatenate([hyps[parents], best_k_pred[:, None]], axis=1)
        end_flag = hyps[:, -1:] == eos
    final = scores.reshape(B, N)
    lengths = (hyps != eos).sum(axis=1).reshape(B, N).astype(np.float32)
    with np.errstate(divide="ignore", invalid="ignore"):
        final = (final / np.power(lengths, np.float32(length_penalty))).astype(np.float32)
    best = np.argmax(final, axis=1)
    out = []
    for b in range(B):
        hyp = hyps[b * N + int(best[b]), 1:]
        out.append(DecodeResult(hyp[hyp != eos].tolist()))
    return out


# ---------------------------------------------------------------------------------------------------------------------
# joint_decoding: time-synchronous one-pass CTC / attention beam search
_NEG_INF = float("-inf")


def _lse(values) -> float:
    """Stable log-sum-exp over python floats, -inf when all are -inf (espnet/beam_search_timesync.py:29-37)."""
    top = max(values)
    if top == _NEG_INF:
        return _NEG_INF
    return top + math.log(sum(math.exp(v - top) for v in values))


def time_sync_joint_search(cand_val: np.ndarray, cand_idx: np.ndarray, blank_logp: np.ndarray, decoder_rows,
                           beam_size: int, ctc_weight: float, length_bonus: float, sos: int, blank: int = 0,
                           blank_threshold: float = 1.0):
    """One utterance of the reference's `joint_decoding` (transformer/search.py:450-496): the time-synchronous joint
    CTC / attention beam search `BeamSearchTimeSync.__call__` (espnet/beam_search_timesync.py:433-508, time_step
    :262-431, joint_score :221-260, cached_score :171-219), host bookkeeping in double precision like the reference's
    Python floats.  Hypotheses are tuples starting with `sos`.

    cand_val / cand_idx (T, P): the P = int(pre_beam_ratio * beam) best CTC log-probs of every frame and their token
        ids (the reference thresholds the frame at its P-th largest value and keeps `p >= threshold`, :288-290 — the
        same set unless the P-th value is tied);  blank_logp (T,): log p(blank) per frame.
    decoder_rows(list of prefixes, all of one length) -> (n, V) float32: log_softmax of the left decoder at the last
        position of each prefix (decoder.forward_one_step_with_attn; the engine recomputes the prefix, the reference
        carries a per-layer cache — same values).
    Returns (hyps, scores, start_times, end_times, confs) of the final beam, best first; confs = per token
    max(ctc log-prob, attention log-prob) (`confs_type = "max"`, :498-500).
    """
    dec_w = 1.0 - ctc_weight
    root0 = (sos,)
    cache = {root0: (decoder_rows([root0])[0], 0.0)}         # prefix -> (log_softmax row after it, log p_att(prefix))
    hyps = [root0]
    scores = {}
    times = {root0: ([0], [0])}
    confs = {root0: [(_NEG_INF, _NEG_INF)]}
    dp = {root0: (_NEG_INF, 0.0)}                             # (log p_nonblank, log p_blank)
    log_thr = math.log(blank_threshold)

    def ensure_cached(roots):
        missing = []
        for r in roots:
            if r not in cache and r not in missing:
                missing.append(r)
        by_len = {}
        for r in missing:
            by_len.setdefault(len(r), []).append(r)
        for _, group in sorted(by_len.items()):
            rows = decoder_rows(group)
            for r, row in zip(group, rows):
                parent_row, parent_sum = cache[r[:-1]]
                cache[r] = (row, parent_sum + float(parent_row[r[-1]]))

    for t in range(cand_val.shape[0]):
        # :284-286 — `argmax(p_ctc[0])` of a 0-d value is 0, so the frame is skipped only when token 0 is the blank and
        # its log-prob reaches log(blank_threshold) (= 0, i.e. never in practice)
        if blank == 0 and float(blank_logp[t]) >= log_thr:
            continue
        order = np.argsort(cand_idx[t], kind="stable")         # `.nonzero()` lists the candidates by ascending id
        cands = [(int(cand_idx[t, i]), float(cand_val[t, i])) for i in order]
        p_blank = float(blank_logp[t])
        in_beam = set(hyps)
        new_hyps, seen_new, nxt = [], set(), {}

        def push(h):
            if h not in seen_new:
                seen_new.add(h)
                new_hyps.append(h)

        for hyp in hyps:
            p_prev = _lse(dp[hyp])
            for c, lp in cands:
                if c == blank:
                    nb, b = nxt.get(hyp, (_NEG_INF, _NEG_INF))
                    nxt[hyp] = (nb, _lse([b, lp + p_prev]))
                    push(hyp)
                    continue
                ext = hyp + (c,)
                nb, b = nxt.get(ext, (_NEG_INF, _NEG_INF))
                if ext not in times:                           # first sighting: start and end frame
                    times[ext] = (times[hyp][0] + [t], times[hyp][1] + [t + 1])
                else:
                    times[ext][1][-1] = t + 1
                if ext not in confs:
                    confs[ext] = confs[hyp] + [(_NEG_INF, _NEG_INF)]
                confs[ext][-1] = (max(confs[ext][-1][0], lp), confs[ext][-1][1])
                if c == hyp[-1]:
                    # repeated token: the extension needs a blank in between; the hypothesis itself absorbs the repeat
                    nb_prev, b_prev = dp[hyp]
                    nb = _lse([nb, lp + b_prev])
                    nb_h, b_h = nxt.get(hyp, (_NEG_INF, _NEG_INF))
                    nxt[hyp] = (_lse([nb_h, lp + nb_prev]), b_h)
                    times[hyp][1][-1] = t + 1
                    confs[hyp][-1] = (max(confs[hyp][-1][0], lp), confs[hyp][-1][1])
                else:
                    nb = _lse([nb, lp + p_prev])
                if ext not in in_beam and ext in dp:
                    # proposed in the previous frame but pruned from the beam: fold its mass back in
                    b = _lse([b, p_blank + _lse(dp[ext])])
                    nb = _lse([nb, lp + dp[ext][0]])
                nxt[ext] = (nb, b)
                push(ext)

        # joint score of every proposal (no lexicon constraint: `words` is empty in joint_decoding)
        if dec_w > 0:
            ensure_cached([h[:-1] for h in new_hyps if len(h) > 1])
        scores = {}
        for h in new_hyps:
            sc = ctc_weight * _lse(nxt[h])
            if len(h) > 1 and dec_w > 0:
                row, log_sum = cache[h[:-1]]
                att = float(row[h[-1]])
                sc += (log_sum + att) * dec_w
                confs[h][-1] = (confs[h][-1][0], att)
            sc += length_bonus * (len(h) - 1)
            scores[h] = sc
        # the reference sorts through a {score: hypothesis} dict: equal scores collapse onto the LAST such hypothesis
        by_score = {}
        for h, sc in scores.items():
            by_score[sc] = h
        hyps = [by_score[sc] for sc in sorted(by_score, reverse=True)[:beam_size]]
        dp = dict(nxt)

    out_conf = [[max(c0, c1) for c0, c1 in confs[h]] for h in hyps]
    return hyps, [scores[h] for h in hyps], [times[h][0] for h in hyps], [times[h][1] for h in hyps], out_conf


def joint_decoding_results(per_utt) -> List[DecodeResult]:
    """search.py:484-494: the best hypothesis of every utterance without its <sos>; times = start frames."""
    out = []
    for hyps, scores, starts, _ends, confs in per_utt:
        # the reference passes score / confidences through float32 tensors before `.item()` (search.py:489-493)
        out.append(DecodeResult(list(hyps[0][1:]), float(np.float32(scores[0])), times=list(starts[0][1:]),
                                tokens_confidence=[math.exp(float(np.float32(c))) for c in confs[0][1:]]))
    return out
