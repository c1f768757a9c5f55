"""`ASRModel.decode` — the operator boundary the kernels sit behind.

Same signature, argument meaning and result types as the reference's
`ASRModel.decode` (asr/wenet/transformer/asr_model.py:331-432); the body drives the native
plan (reverb_b200/engine.py) instead of a torch.nn graph:

    encoder (csrc/engine.cu) -> CTC head + top-k (csrc/ctc.cu) -> greedy / prefix beam (GPU)
    -> teacher-forced decoder over the n-best (GPU) -> score combination (host, search.py)
"""
from __future__ import annotations

import math
from typing import Dict, List, Optional

import numpy as np
import torch

from .engine import Engine, check_beam_size, nbest_lists
from .search import (DecodeResult, attention_beam_search, greedy_results,
                     joint_decoding_results, prefix_beam_results, rescoring_pick, rescoring_pick_batch,
                     time_sync_joint_search)

SUPPORTED_METHODS = ("attention", "ctc_greedy_search", "ctc_prefix_beam_search", "attention_rescoring", "joint_decoding")
JOINT_DECODING_SOS = 10000        # hard-coded in the reference (transformer/search.py:480)
JOINT_PRE_BEAM_RATIO = 1.5        # joint_decoding's default (search.py:457)


def cat_row(cat_embs, b: int):
    """Utterance b's mixing vector of a (num_langs,) or (B, num_langs) cat_embs."""
    if cat_embs is None or torch.as_tensor(cat_embs).dim() < 2:
        return cat_embs
    return torch.as_tensor(cat_embs)[b]


def alignment_result(a) -> DecodeResult:
    """engine.Alignment -> DecodeResult with `times` / `tokens_confidence` filled, so that it renders like a search
    result; the frame-level alignment travels as extra attributes."""
    T = len(a.frames)
    r = DecodeResult(tokens=list(a.tokens), score=float(a.score), confidence=math.exp(float(a.score) / T),
                     tokens_confidence=[math.exp(float(x)) for x in a.peak_logp], times=[int(t) for t in a.peak])
    r.alignment = a.frames
    r.first_frames, r.last_frames, r.loglik = a.first, a.last, a.loglik
    return r


class ASRModel:
    def __init__(self, engine: Engine, configs: Dict, vocab_size: int):
        self.engine = engine
        self.configs = configs
        self.vocab_size = vocab_size
        st = (configs.get("tokenizer_conf") or {}).get("special_tokens")
        # asr_model.py:79-82: eos is the same id as sos
        self.sos = vocab_size - 1 if st is None else st.get("<sos>", vocab_size - 1)
        self.eos = vocab_size - 1 if st is None else st.get("<eos>", vocab_size - 1)
        self.ignore_id = -1
        ds = configs.get("dataset_conf", {})
        self.lsl_enc = self.lsl_dec = bool(ds.get("pass_cat_emb", False))
        self.reverse_weight = configs.get("model_conf", {}).get("reverse_weight", 0.0)

    def sos_symbol(self) -> int:
        return self.sos

    def eos_symbol(self) -> int:
        return self.eos

    def eval(self):
        return self

    def to(self, device):
        return self

    # -- pieces of decode(), exposed for tests / profiling ---------------------------------------
    def attention_context(self, decoding_chunk_size: int, num_decoding_left_chunks: int):
        """The (chunk, left) pair add_optional_chunk_mask (utils/mask.py:126-197) would apply for this model's
        encoder_conf; (-1, -1) = full context."""
        ec = self.configs.get("encoder_conf", {})
        if ec.get("use_dynamic_chunk", False):
            if decoding_chunk_size < 0:
                return -1, -1
            if decoding_chunk_size > 0:
                return int(decoding_chunk_size), int(num_decoding_left_chunks)
            raise AssertionError("decoding_chunk_size == 0 selects the random training chunks")   # asr_model.py:377
        if ec.get("static_chunk_size", 0) > 0:
            return int(ec["static_chunk_size"]), int(num_decoding_left_chunks)
        return -1, -1

    def _forward_encoder(self, speech: torch.Tensor, speech_lengths, cat_embs=None, decoding_chunk_size: int = -1,
                         num_decoding_left_chunks: int = -1, simulate_streaming: bool = False):
        """-> (encoder_out (B, T', d) fp32 cuda, encoder_lens np.int32 (B,)).
        simulate_streaming with decoding_chunk_size > 0: encoder.forward_chunk_by_chunk (encoder.py:341-402), the
        cache-based chunk-by-chunk pass, evaluated as ONE masked pass with identical results (engine.cu
        rvb_encoder_forward_streaming).  Like the reference's it has no padding masks (every input frame counts) and
        serves one utterance at a time (`assert xs.size(0) == 1`, encoder.py:284).  The reference's decode() does not
        forward cat_embs on this path (asr_model.py:299-303) and therefore asserts on models with language-specific
        layers; here cat_embs is passed on, as encoder.forward_chunk_by_chunk itself expects."""
        lens = speech_lengths.detach().cpu().numpy() if torch.is_tensor(speech_lengths) else np.asarray(speech_lengths)
        if simulate_streaming and decoding_chunk_size > 0:
            assert speech.shape[0] == 1, "simulate_streaming decodes one utterance at a time (encoder.py:284)"
            return self.engine.forward_encoder(speech, lens, cat_embs, int(decoding_chunk_size),
                                               int(num_decoding_left_chunks), streaming=True)
        chunk, left = self.attention_context(decoding_chunk_size, num_decoding_left_chunks)
        return self.engine.forward_encoder(speech, lens, cat_embs, chunk, left)

    def ctc_logprobs(self, encoder_out: torch.Tensor, blank_penalty: float = 0.0, blank_id: int = 0) -> torch.Tensor:
        return self.engine.ctc_topk(encoder_out, 1, blank_penalty, blank_id, want_logp=True)[2]

    # -- decode() in three stages (A: everything that can be enqueued without looking at a result; B: the decoder
    # passes, which need the n-best lengths on the host; C: collect + host-side score combination), so that
    # decode_stream can overlap the host work of one batch with the GPU work of the next ones ----------------------
    def _stage_a(self, methods: List[str], speech: torch.Tensor, speech_lengths: torch.Tensor, beam_size: int,
                 decoding_chunk_size: int = -1, num_decoding_left_chunks: int = -1, ctc_weight: float = 0.0,
                 simulate_streaming: bool = False, reverse_weight: float = 0.0, context_graph=None,
                 blank_id: int = 0, blank_penalty: float = 0.0, length_penalty: float = 0.0,
                 infos: Optional[Dict[str, List[str]]] = None, cat_embs: Optional[torch.Tensor] = None,
                 cv=None, cv_lengths=None) -> dict:
        assert speech.shape[0] == speech_lengths.shape[0]
        assert decoding_chunk_size != 0
        check_beam_size(beam_size)
        unknown = [m for m in methods if m not in SUPPORTED_METHODS]
        if unknown:
            raise NotImplementedError(f"reverb_b200: decoding method(s) {unknown} are not built yet (SURVEY.md §8f)")
        if not speech.is_cuda:
            speech = speech.to(self.engine.device, non_blocking=True)
        speech = speech.to(torch.float32)
        encoder_out, encoder_lens = self._forward_encoder(speech, speech_lengths, cat_embs, decoding_chunk_size,
                                                          num_decoding_left_chunks, simulate_streaming)
        need_beam = "ctc_prefix_beam_search" in methods or "attention_rescoring" in methods
        k = beam_size if need_beam else 1
        joint = "joint_decoding" in methods
        if joint:
            # BeamSearchTimeSync looks at the int(1.5 * beam) best tokens of every frame (+ the blank's log-prob)
            pre_beam = int(JOINT_PRE_BEAM_RATIO * beam_size)
            if not 1 <= pre_beam <= 16:
                raise ValueError(f"reverb_b200: joint_decoding needs int(1.5 * beam_size) <= 16 (beam_size={beam_size})")
            if JOINT_DECODING_SOS >= self.vocab_size:
                # the reference indexes the embedding with sos = 10000 (IndexError there, SURVEY.md §8a quirk 3)
                raise IndexError(f"joint_decoding hard-codes sos={JOINT_DECODING_SOS}; vocabulary has {self.vocab_size} entries")
            k = max(k, pre_beam)
        topk_val, topk_idx, logp_full = self.engine.ctc_topk(encoder_out, k, blank_penalty, blank_id, want_logp=joint)
        st = {"methods": list(methods), "results": {}, "ticket": None, "cat_embs": cat_embs, "ctc_weight": ctc_weight,
              "reverse_weight": reverse_weight, "stage": 1}
        results = st["results"]
        if "attention" in methods:
            # autoregressive beam search with the left decoder (search.py:251-360); the decoder step runs on the GPU,
            # the beam bookkeeping on the host like the reference's
            # KV-cached step: one new position per hypothesis and step (the reference carries a per-layer cache too,
            # decoder.py:191-234); RVB_ATTENTION_STEP=recompute selects the cache-free step that re-runs the prefix
            import os as _os
            if _os.environ.get("RVB_ATTENTION_STEP", "cache") == "recompute":
                def step(hyps, parents=None):
                    return self.engine.decoder_step_topk(encoder_out, encoder_lens, hyps, beam_size, cat_embs, beam_size)
                results["attention"] = attention_beam_search(step, encoder_out.shape[0], encoder_out.shape[1],
                                                             beam_size, self.sos, self.eos, length_penalty)
            else:
                self.engine.decoder_cache_begin(encoder_out, encoder_lens, beam_size, encoder_out.shape[1], cat_embs)
                try:
                    def step(hyps, parents=None):
                        return self.engine.decoder_cache_step(hyps[:, -1], parents, beam_size)
                    results["attention"] = attention_beam_search(step, encoder_out.shape[0], encoder_out.shape[1],
                                                                 beam_size, self.sos, self.eos, length_penalty)
                finally:
                    self.engine.decoder_cache_end()
        if "ctc_greedy_search" in methods:
            results["ctc_greedy_search"] = greedy_results(self.engine.greedy_search(topk_idx, encoder_lens, blank_id))
        if joint:
            results["joint_decoding"] = self._joint_decoding(encoder_out, encoder_lens, topk_val, topk_idx, logp_full,
                                                             pre_beam, beam_size, ctc_weight, length_penalty, cat_embs)
            if need_beam and k != beam_size:                  # the searches below expect exactly beam_size candidates
                topk_val, topk_idx = topk_val[:, :, :beam_size].contiguous(), topk_idx[:, :, :beam_size].contiguous()
        if need_beam:
            # the n-best stays on the device between the search and the decoder (native ticket, include/rvb_b200.h);
            # with a context graph the search is the biased instantiation of the same kernel (search.py:124-248)
            st["ticket"] = self.engine.search_submit(topk_val, topk_idx, encoder_out, encoder_lens, beam_size, blank_id,
                                                     context=context_graph)
        return st

    def _joint_decoding(self, encoder_out, encoder_lens, topk_val, topk_idx, logp_full, pre_beam, beam_size,
                        ctc_weight, length_bonus, cat_embs) -> List[DecodeResult]:
        """transformer/search.py:450-496: per utterance, BeamSearchTimeSync over its valid frames with the LEFT decoder;
        decoder weight 1 - ctc_weight, `length_penalty` acts as the length bonus (asr_model.py:426-429)."""
        val = topk_val[:, :, :pre_beam].cpu().numpy()
        idx = topk_idx[:, :, :pre_beam].cpu().numpy()
        blank_lp = logp_full[:, :, 0].cpu().numpy()           # BeamSearchTimeSync's blank index is 0 (its default)
        per_utt = []
        for b in range(encoder_out.shape[0]):
            n = int(encoder_lens[b])
            mem = encoder_out[b:b + 1]
            mem_len = encoder_lens[b:b + 1]

            def rows(prefixes, mem=mem, mem_len=mem_len, cat=cat_row(cat_embs, b)):
                hy = np.asarray(prefixes, dtype=np.int32)
                return self.engine.decoder_step_logp(mem, mem_len, hy, hy.shape[0], cat)
            per_utt.append(time_sync_joint_search(val[b, :n], idx[b, :n], blank_lp[b, :n], rows, beam_size, ctc_weight,
                                                  length_bonus, JOINT_DECODING_SOS))
        return joint_decoding_results(per_utt)

    def _stage_b(self, st: dict) -> None:
        if st["stage"] != 1:
            return
        st["stage"] = 2
        if st["ticket"] is not None:
            self.engine.rescoring_submit(st["ticket"], st["cat_embs"], st["reverse_weight"],
                                         run_decoder="attention_rescoring" in st["methods"])

    def _stage_c(self, st: dict) -> Dict[str, List[DecodeResult]]:
        self._stage_b(st)
        results, methods = st["results"], st["methods"]
        if st["ticket"] is not None:
            toks, tims, olen, scores, nhyp, l2r, r2l = self.engine.rescoring_collect(st["ticket"])
            if "ctc_prefix_beam_search" in methods:
                results["ctc_prefix_beam_search"] = prefix_beam_results(nbest_lists(toks, tims, olen, scores, nhyp))
            if "attention_rescoring" in methods:
                results["attention_rescoring"] = rescoring_pick_batch(toks, tims, olen, scores, nhyp, l2r, r2l,
                                                                      st["ctc_weight"], st["reverse_weight"])
            st["ticket"] = None
        st["stage"] = 3
        return results

    @torch.no_grad()
    def decode(self, methods: List[str], speech: torch.Tensor, speech_lengths: torch.Tensor, beam_size: int,
               decoding_chunk_size: int = -1, num_decoding_left_chunks: int = -1, ctc_weight: float = 0.0,
               simulate_streaming: bool = False, reverse_weight: float = 0.0, context_graph=None,
               blank_id: int = 0, blank_penalty: float = 0.0, length_penalty: float = 0.0,
               infos: Optional[Dict[str, List[str]]] = None, cat_embs: Optional[torch.Tensor] = None,
               cv=None, cv_lengths=None) -> Dict[str, List[DecodeResult]]:
        """The reference's decode(); cat_embs, the language-specific mixing weights [v, 1 - v] of verbatimicity v, is
        (num_langs,) for the whole batch or (B, num_langs) with one row per utterance.  Row b decodes utterance b
        exactly as a batch whose every row carries cat_embs[b], in all six modes; all hypotheses of utterance b use
        cat_embs[b] (the reference's attention_rescoring / attention beam search at B = 1)."""
        st = self._stage_a(methods, speech, speech_lengths, beam_size, decoding_chunk_size, num_decoding_left_chunks,
                           ctc_weight, simulate_streaming, reverse_weight, context_graph, blank_id, blank_penalty,
                           length_penalty, infos, cat_embs, cv, cv_lengths)
        try:
            return self._stage_c(st)
        finally:
            self.engine.ticket_release(st["ticket"])

    @torch.no_grad()
    def decode_stream(self, batches, methods: List[str], beam_size: int, **kwargs):
        """decode() over an iterable of (speech, speech_lengths) batches, software-pipelined on the current stream by
        this one host thread; yields the per-batch result dicts in order.  A batch given as (speech, speech_lengths,
        cat_embs) decodes with its own cat_embs instead of the keyword argument's.  Chunks are independent units
        (cli/reverb.py:214-234), so the results equal the batch-by-batch loop of the reference.

        Schedule (A = encoder + CTC head + prefix beam, B = decoder passes, C = collect + host score combination):
            A(0) | A(1) B(0) | A(2) B(1) C(0) | A(3) B(2) C(1) | ...
        B(n-1) is enqueued right after A(n), so while the host waits for the n-best lengths of batch n-1 (they size
        the decoder batch) or combines the scores of batch n-2, the GPU still has a whole encoder pass queued."""
        inflight = []
        try:
            for batch in batches:
                kw = kwargs if len(batch) == 2 else dict(kwargs, cat_embs=batch[2])
                inflight.append(self._stage_a(methods, batch[0], batch[1], beam_size, **kw))
                if len(inflight) >= 2:
                    self._stage_b(inflight[-2])
                if len(inflight) >= 3:
                    yield self._stage_c(inflight.pop(0))
            while inflight:
                yield self._stage_c(inflight.pop(0))
        finally:
            for st in inflight:          # only non-empty when a stage raised or the consumer stopped early
                self.engine.ticket_release(st["ticket"])

    @torch.no_grad()
    def align(self, speech: torch.Tensor, speech_lengths, tokens, token_lengths, blank_id: int = 0, cat_embs=None,
              blank_penalty: float = 0.0, want_loglik: bool = False) -> List[DecodeResult]:
        """CTC forced alignment of known transcripts (the reference's force_align, utils/ctc_utils.py:105-161, driven by
        bin/alignment.py one utterance at a time): encoder -> CTC log-probs -> batched Viterbi on the GPU (csrc/align.cu).
        tokens (B, max_U) padded ids, token_lengths (B).  One DecodeResult per utterance: `tokens`, `times` = the peak
        frame of every token (the frame of its span with the largest log-prob: the prefix search's notion of a token
        time), `tokens_confidence` = exp(peak log-prob), `score` = Viterbi score, `confidence` = exp(score / T); plus
        `alignment` (the token id of every frame), `first_frames` / `last_frames` and, when asked for, `loglik`.
        ValueError when a transcript is empty or has more tokens (+ repeats) than the audio has encoder frames."""
        if not speech.is_cuda:
            speech = speech.to(self.engine.device, non_blocking=True)
        tok = np.asarray(tokens.cpu() if torch.is_tensor(tokens) else tokens)
        ulen = np.asarray(token_lengths.cpu() if torch.is_tensor(token_lengths) else token_lengths).reshape(-1)
        labels = [[int(x) for x in tok[b][:int(ulen[b])]] for b in range(speech.shape[0])]
        encoder_out, encoder_lens = self._forward_encoder(speech.to(torch.float32), speech_lengths, cat_embs)
        logp = self.ctc_logprobs(encoder_out, blank_penalty, blank_id)
        return [alignment_result(a) for a in
                self.engine.force_align(logp, encoder_lens, labels, blank_id, want_loglik)]

    def attention_rescoring(self, prefix_results: List[DecodeResult], encoder_out: torch.Tensor, encoder_lens,
                            ctc_weight: float = 0.0, reverse_weight: float = 0.0, cat_embs=None) -> List[DecodeResult]:
        """asr/wenet/transformer/search.py:363-448, batched over utterances x hypotheses."""
        nbest = [r.nbest for r in prefix_results]
        l2r, r2l = self.engine.rescoring_scores(encoder_out, encoder_lens, nbest, cat_embs, reverse_weight)
        out = []
        for b, r in enumerate(prefix_results):
            out.append(rescoring_pick(r.nbest, r.nbest_scores, r.nbest_times, l2r[b],
                                      None if r2l is None else r2l[b], ctc_weight, reverse_weight))
        return out
