"""ORACLE (test infrastructure, never shipped): fp32 CPU restatement, in plain torch
tensor ops over a flat state_dict, of the reference's model graph on the hot path:

  feats -> GlobalCMVN -> Conv2dSubsampling4 -> 18x (LSL) Conformer block -> after_norm
        -> CTC head (Linear + log_softmax)
  n-best -> (LSL) bi-transformer decoder, teacher forced -> log_softmax

Every function cites the reference file:line it follows (paths relative to
the reference's asr/wenet).  Pinned against outputs of the LIVE reference
(oracle/make_golden.py, make_golden_pins.py -> tests/golden/; checked by tests/test_oracle_golden.py and
tests/test_oracle_vs_reference.py).  The reference has no tests of its own
for this path (SURVEY.md §4), so "parity unpinned" by reference-held golden vectors;
pinned instead by outputs of the reference itself.

Only tests/, __graft_entry__.smoke() and bench.py's CPU-baseline / reference arm may
import this module.
"""
from __future__ import annotations

import math
from typing import Dict, List, Optional, Tuple

import torch
import torch.nn.functional as F

SD = Dict[str, torch.Tensor]

# Optional emulation of the CUDA path's storage precision (tests only): when EMULATE_BF16 is True every tensor the
# GPU engine stores as bf16 (GEMM operands, attention probabilities, conv activations) is rounded to bf16 at the same
# point of the graph, everything else stays fp32.  With it the oracle and the engine differ only by accumulation
# order, which lets the GPU parity tests use a ~10x tighter tolerance than against the pure-fp32 reference.
EMULATE_BF16 = False


def _q(x):
    return x.bfloat16().float() if EMULATE_BF16 else x


def _ln(x, sd: SD, p: str, eps: float):
    return F.layer_norm(x, (x.shape[-1],), sd[p + ".weight"], sd[p + ".bias"], eps)


def _lin(x, sd: SD, p: str):
    return F.linear(_q(x), _q(sd[p + ".weight"]), sd.get(p + ".bias"))


def make_pad_mask(lengths: torch.Tensor, max_len: int) -> torch.Tensor:
    """utils/mask.py:200-226 — True at padded positions."""
    return torch.arange(max_len)[None, :] >= lengths[:, None].long()


def sinusoid_pe(n: int, d: int) -> torch.Tensor:
    """transformer/embedding.py:39-56."""
    pe = torch.zeros(n, d)
    pos = torch.arange(0, n, dtype=torch.float32).unsqueeze(1)
    div = torch.exp(torch.arange(0, d, 2, dtype=torch.float32) * -(math.log(10000.0) / d))
    pe[:, 0::2] = torch.sin(pos * div)
    pe[:, 1::2] = torch.cos(pos * div)
    return pe


def subsample4(feats: torch.Tensor, lens: torch.Tensor, sd: SD) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """GlobalCMVN (transformer/cmvn.py:36-47) + Conv2dSubsampling4.forward
    (transformer/subsampling.py:201-226) + RelPositionalEncoding.forward
    (transformer/embedding.py:132-146)."""
    B, T, _ = feats.shape
    masks = ~make_pad_mask(lens, T).unsqueeze(1)                       # encoder.py:130
    x = (feats - sd["encoder.global_cmvn.mean"]) * sd["encoder.global_cmvn.istd"]
    x = x.unsqueeze(1)
    x = _q(F.relu(F.conv2d(x, sd["encoder.embed.conv.0.weight"], sd["encoder.embed.conv.0.bias"], stride=2)))
    x = _q(F.relu(F.conv2d(x, _q(sd["encoder.embed.conv.2.weight"]), sd["encoder.embed.conv.2.bias"], stride=2)))
    b, c, t, f = x.shape
    x = x.transpose(1, 2).contiguous().view(b, t, c * f)
    d = sd["encoder.embed.out.0.bias"].shape[0]
    if EMULATE_BF16:   # the engine folds xscale = sqrt(d) into the packed bf16 weight
        xs = math.sqrt(d)
        x = F.linear(x, _q(sd["encoder.embed.out.0.weight"] * xs), sd["encoder.embed.out.0.bias"] * xs)
    else:
        x = _lin(x, sd, "encoder.embed.out.0") * math.sqrt(d)
    pos_emb = sinusoid_pe(t, d).unsqueeze(0)
    masks = masks[:, :, 2::2][:, :, 2::2]
    return x, pos_emb, masks


def rel_attention(x, mask, pos_emb, sd: SD, p: str, H: int):
    """RelPositionMultiHeadedAttention.forward (transformer/attention.py:317-399); note the
    disabled rel_shift (:391-394): p is indexed by ABSOLUTE key position."""
    B, T, d = x.shape
    dk = d // H
    q = _q(_lin(x, sd, p + ".linear_q")).view(B, T, H, dk)
    k = _q(_lin(x, sd, p + ".linear_k")).view(B, T, H, dk).transpose(1, 2)
    v = _q(_lin(x, sd, p + ".linear_v")).view(B, T, H, dk).transpose(1, 2)
    pp = _q(F.linear(_q(pos_emb), _q(sd[p + ".linear_pos.weight"]))).view(1, -1, H, dk).transpose(1, 2)
    if EMULATE_BF16:
        # the wgmma attention folds the position term: s = q.(k + p) + (u.k + v.p), with K'' = bf16(k + p)
        kpp = _q(k + pp)
        cb = (sd[p + ".pos_bias_u"].unsqueeze(1) * k).sum(-1) + (sd[p + ".pos_bias_v"].unsqueeze(1) * pp).sum(-1)
        scores = (torch.matmul(q.transpose(1, 2), kpp.transpose(-2, -1)) + cb.unsqueeze(-2)) / math.sqrt(dk)
        return _attend(v, scores, mask, sd, p)
    qu = (q + sd[p + ".pos_bias_u"]).transpose(1, 2)
    qv = (q + sd[p + ".pos_bias_v"]).transpose(1, 2)
    ac = torch.matmul(qu, k.transpose(-2, -1))
    bd = torch.matmul(qv, pp.transpose(-2, -1))
    scores = (ac + bd) / math.sqrt(dk)
    return _attend(v, scores, mask, sd, p)


def _attend(v, scores, mask, sd: SD, p: str):
    """MultiHeadedAttention.forward_attention (transformer/attention.py:81-127)."""
    B = v.shape[0]
    m = mask.unsqueeze(1).eq(0)
    scores = scores.masked_fill(m, -float("inf"))
    if EMULATE_BF16:   # probabilities are rounded to bf16 for P.V, the normaliser is the fp32 sum
        mx = scores.amax(dim=-1, keepdim=True)
        mx = torch.where(torch.isinf(mx), torch.zeros_like(mx), mx)
        e = torch.exp(scores - mx).masked_fill(m, 0.0)
        den = e.sum(dim=-1, keepdim=True)
        x = torch.matmul(_q(e), v) / torch.where(den > 0, den, torch.ones_like(den))
        x = _q(x)
    else:
        attn = torch.softmax(scores, dim=-1).masked_fill(m, 0.0)
        x = torch.matmul(attn, v)
    x = x.transpose(1, 2).contiguous().view(B, -1, v.shape[1] * v.shape[3])
    return _lin(x, sd, p + ".linear_out")


def mha(q_in, kv_in, mask, sd: SD, p: str, H: int):
    """MultiHeadedAttention.forward (transformer/attention.py:129-175)."""
    B, Tq, d = q_in.shape
    dk = d // H
    q = _q(_lin(q_in, sd, p + ".linear_q")).view(B, Tq, H, dk).transpose(1, 2)
    k = _q(_lin(kv_in, sd, p + ".linear_k")).view(B, -1, H, dk).transpose(1, 2)
    v = _q(_lin(kv_in, sd, p + ".linear_v")).view(B, -1, H, dk).transpose(1, 2)
    scores = torch.matmul(q, k.transpose(-2, -1)) / math.sqrt(dk)
    return _attend(v, scores, mask, sd, p)


def conv_module(x, mask_pad, sd: SD, p: str, K: int, causal: bool, layer_norm: bool):
    """ConvolutionModule.forward (transformer/convolution.py:89-144)."""
    x = x.transpose(1, 2)
    x = x.masked_fill(~mask_pad, 0.0)
    if causal:
        x = F.pad(x, (K - 1, 0), "constant", 0.0)
    # (bf16 emulation: the CUDA path applies GLU to the fp32 accumulators in the GEMM epilogue and stores bf16 once)
    x = F.conv1d(_q(x), _q(sd[p + ".pointwise_conv1.weight"]), sd[p + ".pointwise_conv1.bias"])
    x = _q(F.glu(x, dim=1))
    x = F.conv1d(x, sd[p + ".depthwise_conv.weight"], sd[p + ".depthwise_conv.bias"],
                 padding=0 if causal else (K - 1) // 2, groups=x.shape[1])
    if layer_norm:
        x = F.silu(_ln(x.transpose(1, 2), sd, p + ".norm", 1e-5)).transpose(1, 2)
    else:
        x = F.silu(F.batch_norm(x, sd[p + ".norm.running_mean"], sd[p + ".norm.running_var"],
                                sd[p + ".norm.weight"], sd[p + ".norm.bias"], False, 0.0, 1e-5))
    x = F.conv1d(_q(x), _q(sd[p + ".pointwise_conv2.weight"]), sd[p + ".pointwise_conv2.bias"])
    x = x.masked_fill(~mask_pad, 0.0)
    return x.transpose(1, 2)


def ffn(x, sd: SD, p: str, act):
    """PositionwiseFeedForward.forward (transformer/positionwise_feed_forward.py:47-55)."""
    return _lin(_q(act(_lin(x, sd, p + ".w_1"))), sd, p + ".w_2")


def lsl_mix(x, sd: SD, p: str, cat_embs: torch.Tensor):
    """y = sum_i cat_embs[i] * language_layers[i](x)  (encoder_layer.py:376-390)."""
    if EMULATE_BF16:   # the engine folds W = sum_i c_i W_i (fp32) and stores it as bf16
        w = sum(cat_embs[i] * sd[f"{p}.language_layers.{i}.weight"] for i in range(cat_embs.shape[0]))
        b = sum(cat_embs[i] * sd[f"{p}.language_layers.{i}.bias"] for i in range(cat_embs.shape[0]))
        return F.linear(_q(x), _q(w), b)
    y = None
    for i in range(cat_embs.shape[0]):
        t = cat_embs[i] * _lin(x, sd, f"{p}.language_layers.{i}")
        y = t if y is None else y + t
    return y


def encoder_block(x, mask, pos_emb, mask_pad, sd: SD, p: str, cfg, cat_embs, lsl: bool):
    """ConformerEncoderLayer.forward (transformer/encoder_layer.py:164-244) and
    LanguageSpecificConformerEncoderLayer.forward (:305-402)."""
    ec = cfg["encoder_conf"]
    H, K = ec["attention_heads"], ec["cnn_module_kernel"]
    x = x + 0.5 * ffn(_ln(x, sd, p + ".norm_ff_macaron", 1e-5), sd, p + ".feed_forward_macaron", F.silu)
    x = x + rel_attention(_ln(x, sd, p + ".norm_mha", 1e-5), mask, pos_emb, sd, p + ".self_attn", H)
    x = x + conv_module(_ln(x, sd, p + ".norm_conv", 1e-5), mask_pad, sd, p + ".conv_module", K,
                        ec.get("causal", False), ec.get("cnn_module_norm", "batch_norm") == "layer_norm")
    n = _ln(x, sd, p + ".norm_ff", 1e-5)
    if lsl:
        y = lsl_mix(n, sd, p, cat_embs)
        x = x + 0.5 * ffn(y, sd, p + ".feed_forward", F.silu)
        x = _ln(x, sd, p + ".norm_final", 1e-5)
        return x + y
    x = x + 0.5 * ffn(n, sd, p + ".feed_forward", F.silu)
    return _ln(x, sd, p + ".norm_final", 1e-5)


def subsequent_chunk_mask(size: int, chunk_size: int, num_left_chunks: int = -1) -> torch.Tensor:
    """utils/mask.py:88-123."""
    ret = torch.zeros(size, size, dtype=torch.bool)
    for i in range(size):
        start = 0 if num_left_chunks < 0 else max((i // chunk_size - num_left_chunks) * chunk_size, 0)
        ending = min((i // chunk_size + 1) * chunk_size, size)
        ret[i, start:ending] = True
    return ret


def encoder_forward(feats, lens, sd: SD, cfg, cat_embs: Optional[torch.Tensor], decoding_chunk_size: int = -1,
                    num_decoding_left_chunks: int = -1):
    """BaseEncoder.forward (transformer/encoder.py:117-149).  decoding_chunk_size < 0: full-context decode
    (key-padding mask only, utils/mask.py:161-187); > 0: add_optional_chunk_mask's fixed chunk mask & pad mask for
    the attention (utils/mask.py:126-197; use_dynamic_chunk configs, else static_chunk_size), the pad mask alone for
    the convolution module.  Returns (encoder_out (B,T',d), encoder_lens (B,), masks (B,1,T'))."""
    x, pos_emb, masks = subsample4(feats, lens, sd)
    ec = cfg["encoder_conf"]
    att_masks = masks
    chunk = left = -1
    if ec.get("use_dynamic_chunk", False):
        if decoding_chunk_size > 0:
            chunk, left = decoding_chunk_size, num_decoding_left_chunks
    elif ec.get("static_chunk_size", 0) > 0:
        chunk, left = ec["static_chunk_size"], num_decoding_left_chunks
    if chunk > 0:
        att_masks = masks & subsequent_chunk_mask(x.shape[1], chunk, left).unsqueeze(0)
    L = cfg["encoder_conf"]["num_blocks"]
    has_lsl = bool(cfg["dataset_conf"].get("pass_cat_emb", False))
    for i in range(L):
        lsl = has_lsl and (i == 0 or i == L - 1)
        x = encoder_block(x, att_masks, pos_emb, masks, sd, f"encoder.encoders.{i}", cfg, cat_embs, lsl)
    x = _ln(x, sd, "encoder.after_norm", 1e-5)
    return x, masks.squeeze(1).sum(1), masks


def encoder_forward_chunk_by_chunk(feats, sd: SD, cfg, cat_embs: Optional[torch.Tensor], decoding_chunk_size: int,
                                   num_decoding_left_chunks: int = -1):
    """BaseEncoder.forward_chunk_by_chunk (transformer/encoder.py:341-402) with forward_chunk (:231-339) — the
    CACHE-based streaming simulation, restated literally: overlapping feature windows through the subsampling, per layer
    an attention cache of the last `chunk * left` keys / values (attention.py:356-366) and, for causal models, a
    convolution cache of the last K - 1 conv-module inputs (convolution.py:113-123); no masks at all (att_mask and
    mask_pad are the (0, 0, 0) fakes).  feats (1, T, 80) -> (1, T', d).
    (ASRModel._forward_encoder forgets to pass cat_embs on this path, asr_model.py:299-303, so `decode(...,
    simulate_streaming=True)` asserts on models with language-specific layers; the encoder method itself takes it.)"""
    assert feats.shape[0] == 1 and decoding_chunk_size > 0
    ec = cfg["encoder_conf"]
    H, K, L, d = ec["attention_heads"], ec["cnn_module_kernel"], ec["num_blocks"], ec["output_size"]
    causal = ec.get("causal", False)
    layer_norm = ec.get("cnn_module_norm", "batch_norm") == "layer_norm"
    has_lsl = bool(cfg["dataset_conf"].get("pass_cat_emb", False))
    dk = d // H
    lorder = K - 1 if causal else 0
    context, stride = 7, 4 * decoding_chunk_size
    window = (decoding_chunk_size - 1) * 4 + context
    T = feats.shape[1]
    required = decoding_chunk_size * num_decoding_left_chunks
    pe = sinusoid_pe(5000, d)
    att_cache = [None] * L        # per layer (k, v): (1, H, t, dk)
    cnn_cache = [None] * L        # per layer (1, d, lorder)
    outs, offset = [], 0
    for cur in range(0, T - context + 1, stride):
        xs = feats[:, cur:min(cur + window, T)]
        x, _, _ = subsample4(xs, torch.tensor([xs.shape[1]]), sd)
        cache_t1 = 0 if att_cache[0] is None else att_cache[0][0].shape[2]
        key_size = cache_t1 + x.shape[1]
        pos_emb = pe[offset - cache_t1:offset - cache_t1 + key_size].unsqueeze(0)     # embedding.py position_encoding
        start = 0 if required < 0 else (key_size if required == 0 else max(key_size - required, 0))
        for i in range(L):
            p = f"encoder.encoders.{i}"
            lsl = has_lsl and (i == 0 or i == L - 1)
            x = x + 0.5 * ffn(_ln(x, sd, p + ".norm_ff_macaron", 1e-5), sd, p + ".feed_forward_macaron", F.silu)
            # rel-pos attention over [cache | chunk], no mask (attention.py:344-399)
            n = _ln(x, sd, p + ".norm_mha", 1e-5)
            q = _lin(n, sd, p + ".self_attn.linear_q").view(1, -1, H, dk)
            k = _lin(n, sd, p + ".self_attn.linear_k").view(1, -1, H, dk).transpose(1, 2)
            v = _lin(n, sd, p + ".self_attn.linear_v").view(1, -1, H, dk).transpose(1, 2)
            if att_cache[i] is not None:
                k = torch.cat([att_cache[i][0], k], dim=2)
                v = torch.cat([att_cache[i][1], v], dim=2)
            att_cache[i] = (k[:, :, start:], v[:, :, start:])
            pp = F.linear(pos_emb, sd[p + ".self_attn.linear_pos.weight"]).view(1, -1, H, dk).transpose(1, 2)
            qu = (q + sd[p + ".self_attn.pos_bias_u"]).transpose(1, 2)
            qv = (q + sd[p + ".self_attn.pos_bias_v"]).transpose(1, 2)
            scores = (torch.matmul(qu, k.transpose(-2, -1)) + torch.matmul(qv, pp.transpose(-2, -1))) / math.sqrt(dk)
            a = torch.matmul(torch.softmax(scores, dim=-1), v).transpose(1, 2).contiguous().view(1, -1, d)
            x = x + _lin(a, sd, p + ".self_attn.linear_out")
            # convolution module with the left-context cache (convolution.py:107-144), no padding mask
            c = _ln(x, sd, p + ".norm_conv", 1e-5).transpose(1, 2)
            if lorder > 0:
                c = F.pad(c, (lorder, 0), "constant", 0.0) if cnn_cache[i] is None else torch.cat((cnn_cache[i], c), dim=2)
                cnn_cache[i] = c[:, :, -lorder:]
            q_ = p + ".conv_module"
            c = F.glu(F.conv1d(c, sd[q_ + ".pointwise_conv1.weight"], sd[q_ + ".pointwise_conv1.bias"]), dim=1)
            c = F.conv1d(c, sd[q_ + ".depthwise_conv.weight"], sd[q_ + ".depthwise_conv.bias"],
                         padding=0 if causal else (K - 1) // 2, groups=c.shape[1])
            if layer_norm:
                c = F.silu(_ln(c.transpose(1, 2), sd, q_ + ".norm", 1e-5)).transpose(1, 2)
            else:
                c = F.silu(F.batch_norm(c, sd[q_ + ".norm.running_mean"], sd[q_ + ".norm.running_var"],
                                        sd[q_ + ".norm.weight"], sd[q_ + ".norm.bias"], False, 0.0, 1e-5))
            c = F.conv1d(c, sd[q_ + ".pointwise_conv2.weight"], sd[q_ + ".pointwise_conv2.bias"])
            x = x + c.transpose(1, 2)
            n = _ln(x, sd, p + ".norm_ff", 1e-5)
            if lsl:
                y = lsl_mix(n, sd, p, cat_embs)
                x = x + 0.5 * ffn(y, sd, p + ".feed_forward", F.silu)
                x = _ln(x, sd, p + ".norm_final", 1e-5) + y
            else:
                x = x + 0.5 * ffn(n, sd, p + ".feed_forward", F.silu)
                x = _ln(x, sd, p + ".norm_final", 1e-5)
        outs.append(_ln(x, sd, "encoder.after_norm", 1e-5))
        offset += x.shape[1]
    return torch.cat(outs, dim=1)


def ctc_logprobs(enc_out, sd: SD, blank_penalty: float = 0.0, blank_id: int = 0):
    """ASRModel.ctc_logprobs (transformer/asr_model.py:318-329) / CTC.log_softmax (ctc.py:106-114)."""
    logits = _lin(enc_out, sd, "ctc.ctc_lo")
    if blank_penalty > 0.0:
        logits[:, :, blank_id] -= blank_penalty
    return logits.log_softmax(dim=2)


def decoder_forward(memory, ys_in, ys_lens, sd: SD, cfg, side: str, cat_embs, mem_lens=None):
    """(LanguageSpecific)TransformerDecoder.forward (transformer/decoder.py:116-169, 308-383) with
    DecoderLayer.forward (decoder_layer.py:62-133) / LanguageSpecificDecoderLayer.forward (:251-340).
    memory (N,T,d) with an all-ones memory mask (asr_model.py:895-900) unless mem_lens is given (attention
    mode passes the encoder mask, search.py:268-269).  Returns logits (N,L,V)."""
    dc = cfg["decoder_conf"]
    H = dc["attention_heads"]
    nb = dc["num_blocks"] if side == "left_decoder" else dc["r_num_blocks"]
    has_lsl = bool(cfg["dataset_conf"].get("pass_cat_emb", False))
    p = f"decoder.{side}"
    N, L = ys_in.shape
    d = memory.shape[-1]
    tgt_mask = (~make_pad_mask(ys_lens, L)).unsqueeze(1) & torch.tril(torch.ones(L, L, dtype=torch.bool)).unsqueeze(0)
    mem_mask = torch.ones(N, 1, memory.shape[1], dtype=torch.bool)
    if mem_lens is not None:
        mem_mask = (~make_pad_mask(mem_lens, memory.shape[1])).unsqueeze(1)
    x = F.embedding(ys_in, sd[p + ".embed.0.weight"]) * math.sqrt(d) + sinusoid_pe(L, d).unsqueeze(0)
    for i in range(nb):
        q = f"{p}.decoders.{i}"
        lsl = has_lsl and (i == 0 or i == nb - 1)
        eps = 1e-12 if lsl else 1e-5        # decoder_layer.py:241-243 vs :53-55
        t = _ln(x, sd, q + ".norm1", eps)
        x = x + mha(t, t, tgt_mask, sd, q + ".self_attn", H)
        x = x + mha(_ln(x, sd, q + ".norm2", eps), memory, mem_mask, sd, q + ".src_attn", H)
        t = _ln(x, sd, q + ".norm3", eps)
        if lsl:
            t = lsl_mix(t, sd, q, cat_embs)
        x = x + ffn(t, sd, q + ".feed_forward", F.relu)
    x = _ln(x, sd, p + ".after_norm", 1e-5)
    return _lin(x, sd, p + ".output_layer")


def reverse_hyps(hyps_in: torch.Tensor, hyps_lens: torch.Tensor, eos: int) -> torch.Tensor:
    """Right-to-left decoder input built in ASRModel.forward_attention_decoder
    (transformer/asr_model.py:903-949): [sos, w_U..w_1, eos...]."""
    r_lens = hyps_lens - 1
    r = hyps_in[:, 1:]
    max_len = int(r_lens.max())
    idx_range = torch.arange(0, max_len)
    seq_mask = r_lens.unsqueeze(1) > idx_range
    index = ((r_lens.unsqueeze(1) - 1) - idx_range) * seq_mask
    r = torch.gather(r, 1, index)
    r = torch.where(seq_mask, r, eos)
    return torch.cat([hyps_in[:, 0:1], r], dim=1)


def decoder_step_logp(memory, mem_lens, hyps, sd: SD, cfg, cat_embs):
    """TransformerDecoder.forward_one_step (transformer/decoder.py:191-234) of the LEFT decoder
    (Bi / LanguageSpecificBi decoders delegate to it, :498-522, :640-664): log_softmax over the vocabulary at the
    LAST position of every running hypothesis.  The reference caches the previous positions' layer outputs
    (decoder_layer.py:86-103); with the causal mask that equals recomputing the whole prefix, which is what this
    restatement does.  memory (S,T,d), mem_lens (S,), hyps (S,i) incl. sos -> (S,V)."""
    S, L = hyps.shape
    lens = torch.full((S,), L, dtype=torch.long)
    logits = decoder_forward(memory, hyps, lens, sd, cfg, "left_decoder", cat_embs, mem_lens=mem_lens)
    return torch.log_softmax(logits[:, -1], dim=-1)
