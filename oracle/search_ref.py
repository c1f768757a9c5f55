"""ORACLE (test infrastructure, never shipped): pure-Python restatement of the reference's
CTC searches and attention rescoring (asr/wenet/transformer/search.py), operating on
numpy/torch fp32 log-prob arrays.  Float semantics follow the reference: prefix scores are
Python floats (C doubles) built from fp32 log-probs (`.item()`), rescoring scores are
accumulated in fp32 (0-d torch tensors).

Pinned against the LIVE reference (fixtures recorded by oracle/make_golden.py, checked by
tests/test_oracle_vs_reference.py); the reference itself holds no tests (SURVEY.md §4).
"""
from __future__ import annotations

import math
from typing import List, Optional

import numpy as np
import torch

NEG_INF = -float("inf")


class DecodeResult:
    """transformer/search.py:29-58."""

    def __init__(self, tokens, score=0.0, confidence=0.0, tokens_confidence=None, times=None,
                 nbest=None, nbest_scores=None, nbest_times=None):
        self.tokens = tokens
        self.score = score
        self.confidence = confidence
        self.tokens_confidence = tokens_confidence
        self.times = times
        self.nbest = nbest
        self.nbest_scores = nbest_scores
        self.nbest_times = nbest_times


def log_add(args) -> float:
    """utils/common.py:355-363."""
    if all(a == NEG_INF for a in args):
        return NEG_INF
    a_max = max(args)
    return a_max + math.log(sum(math.exp(a - a_max) for a in args))


class PrefixScore:
    """transformer/search.py:61-103 (context-graph fields omitted: ReverbASR always passes
    context_graph=None, cli/reverb.py:227)."""
    __slots__ = ("s", "ns", "v_s", "v_ns", "cur_token_prob", "times_s", "times_ns")

    def __init__(self, s=NEG_INF, ns=NEG_INF, v_s=NEG_INF, v_ns=NEG_INF):
        self.s, self.ns, self.v_s, self.v_ns = s, ns, v_s, v_ns
        self.cur_token_prob = NEG_INF
        self.times_s: List[int] = []
        self.times_ns: List[int] = []

    def score(self):
        return log_add([self.s, self.ns])

    def viterbi_score(self):
        return self.v_s if self.v_s > self.v_ns else self.v_ns

    def times(self):
        return self.times_s if self.v_s > self.v_ns else self.times_ns


def remove_duplicates_and_blank(hyp: List[int], blank_id: int = 0) -> List[int]:
    """utils/ctc_utils.py:22-32."""
    out, cur = [], 0
    while cur < len(hyp):
        if hyp[cur] != blank_id:
            out.append(hyp[cur])
        prev = cur
        while cur < len(hyp) and hyp[cur] == hyp[prev]:
            cur += 1
    return out


def ctc_greedy_search(ctc_probs: torch.Tensor, ctc_lens: torch.Tensor, blank_id: int = 0) -> List[DecodeResult]:
    """transformer/search.py:106-121."""
    B, T, _ = ctc_probs.shape
    idx = ctc_probs.topk(1, dim=2)[1].view(B, T)
    pad = torch.arange(T)[None, :] >= ctc_lens[:, None].long()
    idx = idx.masked_fill(pad, blank_id)
    return [DecodeResult(remove_duplicates_and_blank(h.tolist(), blank_id)) for h in idx]


def ctc_prefix_beam_search(ctc_probs: torch.Tensor, ctc_lens: torch.Tensor, beam_size: int,
                           blank_id: int = 0) -> List[DecodeResult]:
    """transformer/search.py:124-248, literal update rules including the `vs_ns` typo at :178
    (the repeated-token branch never updates v_ns)."""
    results = []
    for i in range(ctc_probs.shape[0]):
        ctc_prob = ctc_probs[i]
        num_t = int(ctc_lens[i])
        cur_hyps = [(tuple(), PrefixScore(s=0.0, ns=NEG_INF, v_s=0.0, v_ns=0.0))]
        for t in range(num_t):
            logp = ctc_prob[t]
            next_hyps = {}

            def get(prefix):
                ps = next_hyps.get(prefix)
                if ps is None:
                    ps = next_hyps[prefix] = PrefixScore()
                return ps

            _, top_k_index = logp.topk(beam_size)
            for u in top_k_index.tolist():
                prob = logp[u].item()
                for prefix, ps in cur_hyps:
                    last = prefix[-1] if len(prefix) > 0 else None
                    if u == blank_id:
                        n = get(prefix)
                        n.s = log_add([n.s, ps.score() + prob])
                        n.v_s = ps.viterbi_score() + prob
                        n.times_s = ps.times().copy()
                    elif u == last:
                        n1 = get(prefix)
                        n1.ns = log_add([n1.ns, ps.ns + prob])
                        if n1.v_ns < ps.v_ns + prob:
                            # reference assigns the misspelt attribute `vs_ns`: v_ns stays put
                            if n1.cur_token_prob < prob:
                                n1.cur_token_prob = prob
                                n1.times_ns = ps.times_ns.copy()
                                n1.times_ns[-1] = t
                        n2 = get(prefix + (u,))
                        n2.ns = log_add([n2.ns, ps.s + prob])
                        if n2.v_ns < ps.v_s + prob:
                            n2.v_ns = ps.v_s + prob
                            n2.cur_token_prob = prob
                            n2.times_ns = ps.times_s.copy()
                            n2.times_ns.append(t)
                    else:
                        n = get(prefix + (u,))
                        n.ns = log_add([n.ns, ps.score() + prob])
                        if n.v_ns < ps.viterbi_score() + prob:
                            n.v_ns = ps.viterbi_score() + prob
                            n.cur_token_prob = prob
                            n.times_ns = ps.times().copy()
                            n.times_ns.append(t)
            ordered = sorted(next_hyps.items(), key=lambda x: x[1].score(), reverse=True)
            cur_hyps = ordered[:beam_size]
        nbest = [y[0] for y in cur_hyps]
        nbest_scores = [y[1].score() for y in cur_hyps]
        nbest_times = [y[1].times() for y in cur_hyps]
        results.append(DecodeResult(tokens=nbest[0], score=nbest_scores[0], times=nbest_times[0],
                                    nbest=nbest, nbest_scores=nbest_scores, nbest_times=nbest_times))
    return results


def rescoring_inputs(hyps: List[tuple], sos: int, eos: int):
    """Padded decoder inputs of attention_rescoring (transformer/search.py:384-409) /
    add_sos_eos (utils/common.py:112-155): rows [sos, w_1..w_U, eos...], lens U+1."""
    umax = max(len(h) for h in hyps)
    ys = torch.full((len(hyps), umax + 1), eos, dtype=torch.long)
    ys[:, 0] = sos
    for i, h in enumerate(hyps):
        if len(h):
            ys[i, 1:1 + len(h)] = torch.tensor(h, dtype=torch.long)
    lens = torch.tensor([len(h) + 1 for h in hyps], dtype=torch.long)
    return ys, lens


def rescoring_combine(hyps: List[tuple], ctc_scores: List[float], nbest_times, decoder_out: torch.Tensor,
                      r_decoder_out: Optional[torch.Tensor], ctc_weight: float, reverse_weight: float,
                      eos: int) -> DecodeResult:
    """Score combination loop of attention_rescoring (transformer/search.py:413-447);
    decoder_out / r_decoder_out are log-softmaxed (N, L, V) fp32. prefix_len == 1."""
    best_score = -float("inf")
    best_index = 0
    confidences, tokens_confidences = [], []
    for i, hyp in enumerate(hyps):
        score = 0.0
        tc = []
        for j, w in enumerate(hyp):
            s = decoder_out[i][j][w]
            score += s
            tc.append(math.exp(s))
        score += decoder_out[i][len(hyp)][eos]
        if reverse_weight > 0 and r_decoder_out is not None and r_decoder_out.dim() > 0:
            r_score = 0.0
            for j, w in enumerate(hyp):
                s = r_decoder_out[i][len(hyp) - j - 1][w]
                r_score += s
                tc[j] = (tc[j] + math.exp(s)) / 2
            r_score += r_decoder_out[i][len(hyp)][eos]
            score = score * (1 - reverse_weight) + r_score * reverse_weight
        confidences.append(math.exp(score / (len(hyp) + 1)))
        score += ctc_scores[i] * ctc_weight
        if score > best_score:
            best_score = score
            best_index = i
        tokens_confidences.append(tc)
    return DecodeResult(hyps[best_index], best_score, confidence=confidences[best_index],
                        times=nbest_times[best_index], tokens_confidence=tokens_confidences[best_index])


def attention_beam_search(step_topk, batch_size: int, maxlen: int, beam_size: int, sos: int, eos: int,
                          length_penalty: float = 0.0) -> List[DecodeResult]:
    """transformer/search.py:251-360 (non-whisper branch: hyps start as [sos], prefix_len = 1).
    step_topk(hyps (B*N, i) int64) -> (top_k_logp (B*N, N) fp32, top_k_index (B*N, N) int64): the decoder step
    (decoder.forward_one_step + logp.topk(beam_size), :302-306) is the caller's, everything else — finished-beam
    masking (utils/mask.py:257-303), the two-stage prune, hypothesis bookkeeping, length penalty — is restated."""
    B, N = batch_size, beam_size
    running = B * N
    hyps = torch.full((running, 1), sos, dtype=torch.long)
    prefix_len = 1
    scores = torch.tensor([0.0] + [-float("inf")] * (N - 1), dtype=torch.float).repeat([B]).unsqueeze(1)
    end_flag = torch.zeros_like(scores, dtype=torch.bool)
    for i in range(prefix_len, maxlen + 1):
        if end_flag.sum() == running:
            break
        top_k_logp, top_k_index = step_topk(hyps)
        top_k_logp = top_k_logp.clone().float()
        top_k_index = top_k_index.clone().long()
        # mask_finished_scores / mask_finished_preds
        if N > 1:
            unfinished = torch.cat((torch.zeros_like(end_flag), end_flag.repeat([1, N - 1])), dim=1)
            finished = torch.cat((end_flag, torch.zeros_like(end_flag).repeat([1, N - 1])), dim=1)
        else:
            unfinished, finished = torch.zeros_like(end_flag), end_flag
        top_k_logp.masked_fill_(unfinished, -float("inf"))
        top_k_logp.masked_fill_(finished, 0)
        top_k_index.masked_fill_(end_flag.repeat([1, N]), eos)
        scores = scores + top_k_logp
        scores = scores.view(B, N * N)
        scores, offset_k_index = scores.topk(k=N)
        scores = scores.view(-1, 1)
        base_k_index = torch.arange(B).view(-1, 1).repeat([1, N]) * N * N
        best_k_index = base_k_index.view(-1) + offset_k_index.view(-1)
        best_k_pred = torch.index_select(top_k_index.view(-1), dim=-1, index=best_k_index)
        best_hyps_index = best_k_index // N
        last_best_k_hyps = torch.index_select(hyps, dim=0, index=best_hyps_index)
        hyps = torch.cat((last_best_k_hyps, best_k_pred.view(-1, 1)), dim=1)
        end_flag = torch.eq(hyps[:, -1], eos).view(-1, 1)
    scores = scores.view(B, N)
    lengths = hyps.ne(eos).sum(dim=1).view(B, N).float()
    scores = scores / lengths.pow(length_penalty)
    best_scores, best_index = scores.max(dim=-1)
    best_hyps_index = best_index + torch.arange(B, dtype=torch.long) * N
    best_hyps = torch.index_select(hyps, dim=0, index=best_hyps_index)[:, prefix_len:]
    results = []
    for b in range(B):
        hyp = best_hyps[b]
        results.append(DecodeResult(hyp[hyp != eos].tolist()))
    return results


# ---------------------------------------------------------------------------------------------------------------------
def _log_add_list(args) -> float:
    """espnet/beam_search_timesync.py:29-37."""
    if all(a == -float("inf") for a in args):
        return -float("inf")
    a_max = max(args)
    return a_max + math.log(sum(math.exp(a - a_max) for a in args))


def joint_decoding(decoder_row, ctc_probs: torch.Tensor, enc_lens: torch.Tensor, ctc_weight: float = 0.5,
                   beam_size: int = 4, pre_beam_ratio: float = 1.5, length_bonus: float = 0.5,
                   sos: int = 10000, blank: int = 0) -> List[DecodeResult]:
    """transformer/search.py:450-496 + espnet/beam_search_timesync.py:87-508 (BeamSearchTimeSync without lexicon / LM).
    decoder_row(b, prefix list) -> (V,) fp32 log_softmax of the LEFT decoder after `prefix` on utterance b's valid
    encoder frames (forward_one_step_with_attn, decoder.py:236-281) is the caller's; the search — CTC prefix scores
    (p_nb, p_b) per hypothesis, the pre-beam candidate set of each frame, re-entry of pruned hypotheses, start / end
    times, (ctc, attention) confidences, the joint score with length bonus and the score-keyed prune — is restated on
    the FULL log-prob rows, python floats like the reference."""
    inf = float("inf")
    pre_beam = int(pre_beam_ratio * beam_size)
    dec_w = 1.0 - ctc_weight
    results = []
    for bi in range(ctc_probs.shape[0]):
        lpz = ctc_probs[bi, :int(enc_lens[bi])]
        first = (sos,)
        att = {first: (decoder_row(bi, [sos]), 0.0)}
        hyps = [first]
        scores = {}
        times = {first: ([0], [0])}
        confs = {first: [(-inf, -inf)]}
        dp = {first: (-inf, 0.0)}
        for t in range(lpz.shape[0]):
            p = lpz[t]
            best_cand = int(torch.argmax(p[0]))                 # :284 — argmax of a 0-d tensor: always 0
            if best_cand == blank and float(p[best_cand]) >= math.log(1.0):
                continue
            thr = torch.sort(p)[0][-pre_beam]
            cands = [z[0] for z in (p >= thr).nonzero().tolist()]
            new_hyps, nxt = [], {}
            for h in hyps:
                prev = _log_add_list(list(dp[h]))
                for c in cands:
                    pc = float(p[c])
                    if c == blank:
                        nb, b = nxt.get(h, (-inf, -inf))
                        nxt[h] = (nb, _log_add_list([b, pc + prev]))
                        if h not in new_hyps:
                            new_hyps.append(h)
                        continue
                    lp_ = h + (int(c),)
                    nb, b = nxt.get(lp_, (-inf, -inf))
                    if lp_ not in times:
                        times[lp_] = (times[h][0] + [t], times[h][1] + [t + 1])
                    else:
                        times[lp_][1][-1] = t + 1
                    if lp_ not in confs:
                        confs[lp_] = confs[h] + [(-inf, -inf)]
                    confs[lp_][-1] = (max([float(confs[lp_][-1][0]), pc]), confs[lp_][-1][1])
                    if c == h[-1]:
                        nb_prev, b_prev = dp[h]
                        nb = _log_add_list([nb, pc + b_prev])
                        nb_l, b_l = nxt.get(h, (-inf, -inf))
                        nxt[h] = (_log_add_list([nb_l, pc + nb_prev]), b_l)
                        times[h][1][-1] = t + 1
                        confs[h][-1] = (max([float(confs[h][-1][0]), pc]), confs[h][-1][1])
                    else:
                        nb = _log_add_list([nb, pc + prev])
                    if lp_ not in hyps and lp_ in dp:
                        b = _log_add_list([b, float(p[blank]) + _log_add_list(list(dp[lp_]))])
                        nb = _log_add_list([nb, pc + dp[lp_][0]])
                    nxt[lp_] = (nb, b)
                    if lp_ not in new_hyps:
                        new_hyps.append(lp_)
            scores = {}
            for h in new_hyps:
                sc = ctc_weight * _log_add_list(list(nxt[h]))
                if len(h) > 1 and dec_w > 0:
                    root = h[:-1]
                    if root not in att:
                        rr = root[:-1]
                        att[root] = (decoder_row(bi, list(root)), att[rr][1] + float(att[rr][0][root[-1]]))
                    sc += (att[root][1] + float(att[root][0][h[-1]])) * dec_w
                    confs[h][-1] = (confs[h][-1][0], float(att[root][0][h[-1]]))
                sc += length_bonus * (len(h) - 1)
                scores[h] = sc
            rev = {}
            for k, v in scores.items():
                rev[v] = k
            keys = sorted(rev.keys())
            keys.reverse()
            hyps = [rev[s] for s in keys[:beam_size]]
            dp = dict(nxt)
        best = hyps[0]
        conf = torch.tensor([max(c[0], c[1]) for c in confs[best]])
        results.append(DecodeResult(list(best[1:]), torch.tensor([scores[best]]).item(), times=list(times[best][0][1:]),
                                    tokens_confidence=[math.exp(c.item()) for c in conf[1:]]))
    return results
