"""Synthetic reverb_asr_v1-shaped model directories and synthetic 16 kHz audio.

The real `reverb_asr_v1` checkpoint lives on HuggingFace and cannot be fetched
offline, so benchmarks and parity tests run on synthetic weights with the SAME
directory layout the reference loads (asr/wenet/cli/reverb.py:324-357):

    <dir>/config.yaml  <dir>/<name>.pt  <dir>/cmvn  <dir>/tk.units.txt  <dir>/tk.model

The state_dict key names/shapes are exactly those produced by the reference's
`init_model` (asr/wenet/utils/init_model.py:99-277) for `encoder: conformer` with
language-specific first/last blocks and an (LSL) bi-transformer decoder
(SURVEY.md §8a quirk 9); `tests/test_oracle_vs_reference.py` checks this by a
strict `load_state_dict` into the live reference model.

This module does not depend on the reference; the GPU tests and the benchmark use it.
"""
from __future__ import annotations

import json
import math
import os
import wave
from statistics import NormalDist
from typing import Dict

import numpy as np
import torch
import yaml

# Synthetic benchmark default (SURVEY.md §8, BASELINE.md §3): ~639 M parameters.
BENCH_SHAPE = dict(d=1024, heads=16, ff=4096, blocks=18, kernel=15, vocab=10001,
                   dec_ff=2048, dec_blocks=3, r_dec_blocks=3, emb_len=2)
# Small shape used by the parity tests (oracle finishes in seconds).
TEST_SHAPE = dict(d=128, heads=2, ff=256, blocks=3, kernel=15, vocab=101,
                  dec_ff=256, dec_blocks=3, r_dec_blocks=3, emb_len=2)


def make_config(shape: Dict, causal: bool = True, cnn_module_norm: str = "layer_norm",
                reverse_weight: float = 0.3, checkpoint_name: str = "synth.pt") -> Dict:
    """config.yaml contents; keys are the ones the reference dereferences
    (SURVEY.md §5 'Config / flags', Appendix B.4)."""
    return {
        "cmvn": "global_cmvn",
        "cmvn_conf": {"cmvn_file": "cmvn", "is_json_cmvn": True},
        "tokenizer": "rev_bpe",
        "tokenizer_conf": {
            "symbol_table_path": "tk.units.txt",
            "bpe_path": "tk.model",
            "non_lang_syms_path": None,
            "split_with_space": False,
        },
        "ctc_conf": {"ctc_blank_id": 0},
        "input_dim": 80,
        "encoder": "conformer",
        "encoder_conf": {
            "output_size": shape["d"],
            "attention_heads": shape["heads"],
            "linear_units": shape["ff"],
            "num_blocks": shape["blocks"],
            "dropout_rate": 0.1,
            "positional_dropout_rate": 0.1,
            "attention_dropout_rate": 0.0,
            "input_layer": "conv2d",
            "pos_enc_layer_type": "rel_pos",
            "selfattention_layer_type": "rel_selfattn",
            "normalize_before": True,
            "activation_type": "swish",
            "macaron_style": True,
            "use_cnn_module": True,
            "cnn_module_kernel": shape["kernel"],
            "cnn_module_norm": cnn_module_norm,
            "causal": causal,
            "use_dynamic_chunk": True,
            "use_dynamic_left_chunk": False,
        },
        "decoder": "bitransformer",
        "decoder_conf": {
            "attention_heads": shape["heads"],
            "linear_units": shape["dec_ff"],
            "num_blocks": shape["dec_blocks"],
            "r_num_blocks": shape["r_dec_blocks"],
            "dropout_rate": 0.1,
            "positional_dropout_rate": 0.1,
            "self_attention_dropout_rate": 0.0,
            "src_attention_dropout_rate": 0.0,
        },
        "model_conf": {
            "ctc_weight": 0.3,
            "lsm_weight": 0.1,
            "length_normalized_loss": False,
            "reverse_weight": reverse_weight,
        },
        "dataset_conf": {
            "fbank_conf": {"num_mel_bins": 80, "frame_length": 25, "frame_shift": 10, "dither": 0.0},
            "pass_cat_emb": True,
            "cat_emb_conf": {"emb_len": shape["emb_len"],
                             "one_hot_ids": {"verbatim": 0, "nonverbatim": 1}},
        },
    }


def _lin(g, out_f, in_f, bias=True, prefix="", sd=None):
    bound = 1.0 / math.sqrt(in_f)
    sd[prefix + ".weight"] = (torch.rand(out_f, in_f, generator=g) * 2 - 1) * bound
    if bias:
        sd[prefix + ".bias"] = (torch.rand(out_f, generator=g) * 2 - 1) * bound


def _ln(g, n, prefix, sd):
    sd[prefix + ".weight"] = 1.0 + 0.1 * torch.randn(n, generator=g)
    sd[prefix + ".bias"] = 0.05 * torch.randn(n, generator=g)


def _mha(g, d, prefix, sd, rel=False, heads=1):
    for n in ("linear_q", "linear_k", "linear_v", "linear_out"):
        _lin(g, d, d, True, f"{prefix}.{n}", sd)
    if rel:
        _lin(g, d, d, False, f"{prefix}.linear_pos", sd)
        dk = d // heads
        bound = math.sqrt(6.0 / (heads + dk))
        sd[f"{prefix}.pos_bias_u"] = (torch.rand(heads, dk, generator=g) * 2 - 1) * bound
        sd[f"{prefix}.pos_bias_v"] = (torch.rand(heads, dk, generator=g) * 2 - 1) * bound


def make_state_dict(cfg: Dict, vocab: int, seed: int = 0, blank_rate: float = 0.8,
                    ctc_scale: float = 6.0) -> Dict[str, torch.Tensor]:
    """Random fp32 weights with the reference's key names (SURVEY.md §8a quirk 9).

    CTC head shaping, so that a random model behaves like a trained (peaky, blank-
    dominated) one: non-blank rows of ctc.ctc_lo.weight are scaled by `ctc_scale`
    (logit sigma ~= 0.577*ctc_scale on LayerNorm'ed encoder output), the blank row is
    zeroed and the blank bias is set to the z-sigma level at which blank is the arg-max
    on a fraction `blank_rate` of the frames.  That level sits far above the 10th-
    highest non-blank logit, so blank is always inside the top-N of every frame and
    the reference's `vs_ns` typo never leaves `times_ns` unfilled (SURVEY.md §8a quirk 2).
    """
    g = torch.Generator().manual_seed(seed)
    ec, dc = cfg["encoder_conf"], cfg["decoder_conf"]
    d, H, ff, L, K = ec["output_size"], ec["attention_heads"], ec["linear_units"], ec["num_blocks"], ec["cnn_module_kernel"]
    F = cfg["input_dim"]
    F2 = ((F - 1) // 2 - 1) // 2
    emb_len = cfg["dataset_conf"]["cat_emb_conf"]["emb_len"] if cfg["dataset_conf"].get("pass_cat_emb") else 0
    sd: Dict[str, torch.Tensor] = {}
    # global cmvn buffers (GlobalCMVN registers mean/istd, transformer/cmvn.py:21-34)
    sd["encoder.global_cmvn.mean"] = 10.0 + 2.0 * torch.randn(F, generator=g)
    sd["encoder.global_cmvn.istd"] = 1.0 / (3.0 + torch.rand(F, generator=g))
    # Conv2dSubsampling4 (transformer/subsampling.py:172-199)
    b1 = 1.0 / math.sqrt(9.0)
    sd["encoder.embed.conv.0.weight"] = (torch.rand(d, 1, 3, 3, generator=g) * 2 - 1) * b1
    sd["encoder.embed.conv.0.bias"] = (torch.rand(d, generator=g) * 2 - 1) * b1
    b2 = 1.0 / math.sqrt(9.0 * d)
    sd["encoder.embed.conv.2.weight"] = (torch.rand(d, d, 3, 3, generator=g) * 2 - 1) * b2
    sd["encoder.embed.conv.2.bias"] = (torch.rand(d, generator=g) * 2 - 1) * b2
    _lin(g, d, d * F2, True, "encoder.embed.out.0", sd)
    _ln(g, d, "encoder.after_norm", sd)
    for i in range(L):
        p = f"encoder.encoders.{i}"
        _mha(g, d, p + ".self_attn", sd, rel=True, heads=H)
        for ffn in ("feed_forward", "feed_forward_macaron"):
            _lin(g, ff, d, True, f"{p}.{ffn}.w_1", sd)
            _lin(g, d, ff, True, f"{p}.{ffn}.w_2", sd)
        # ConvolutionModule (transformer/convolution.py:40-84)
        sd[p + ".conv_module.pointwise_conv1.weight"] = (torch.rand(2 * d, d, 1, generator=g) * 2 - 1) / math.sqrt(d)
        sd[p + ".conv_module.pointwise_conv1.bias"] = (torch.rand(2 * d, generator=g) * 2 - 1) / math.sqrt(d)
        sd[p + ".conv_module.depthwise_conv.weight"] = (torch.rand(d, 1, K, generator=g) * 2 - 1) / math.sqrt(K)
        sd[p + ".conv_module.depthwise_conv.bias"] = (torch.rand(d, generator=g) * 2 - 1) / math.sqrt(K)
        if ec["cnn_module_norm"] == "layer_norm":
            _ln(g, d, p + ".conv_module.norm", sd)
        else:
            _ln(g, d, p + ".conv_module.norm", sd)
            sd[p + ".conv_module.norm.running_mean"] = 0.1 * torch.randn(d, generator=g)
            sd[p + ".conv_module.norm.running_var"] = 0.5 + torch.rand(d, generator=g)
            sd[p + ".conv_module.norm.num_batches_tracked"] = torch.tensor(100, dtype=torch.long)
        sd[p + ".conv_module.pointwise_conv2.weight"] = (torch.rand(d, d, 1, generator=g) * 2 - 1) / math.sqrt(d)
        sd[p + ".conv_module.pointwise_conv2.bias"] = (torch.rand(d, generator=g) * 2 - 1) / math.sqrt(d)
        for n in ("norm_ff", "norm_mha", "norm_ff_macaron", "norm_conv", "norm_final"):
            _ln(g, d, f"{p}.{n}", sd)
        if emb_len > 0 and (i == 0 or i == L - 1):
            for j in range(emb_len):
                _lin(g, d, d, True, f"{p}.language_layers.{j}", sd)
    # CTC head (transformer/ctc.py:47)
    _lin(g, vocab, d, True, "ctc.ctc_lo", sd)
    sd["ctc.ctc_lo.weight"] *= ctc_scale
    sd["ctc.ctc_lo.weight"][0] = 0.0
    sd["ctc.ctc_lo.bias"] *= 0.0
    sigma = ctc_scale / math.sqrt(3.0)
    z = NormalDist().inv_cdf(blank_rate ** (1.0 / max(vocab - 2, 1)))
    sd["ctc.ctc_lo.bias"][0] = z * sigma
    # (LSL) bi-transformer decoder (transformer/decoder.py:524-602)
    sides = [("left_decoder", dc["num_blocks"])]
    if dc.get("r_num_blocks", 0) > 0:
        sides.append(("right_decoder", dc["r_num_blocks"]))
    for side, nb in sides:
        p = f"decoder.{side}"
        sd[p + ".embed.0.weight"] = torch.randn(vocab, d, generator=g)
        _ln(g, d, p + ".after_norm", sd)
        _lin(g, vocab, d, True, p + ".output_layer", sd)
        for i in range(nb):
            q = f"{p}.decoders.{i}"
            _mha(g, d, q + ".self_attn", sd)
            _mha(g, d, q + ".src_attn", sd)
            _lin(g, dc["linear_units"], d, True, q + ".feed_forward.w_1", sd)
            _lin(g, d, dc["linear_units"], True, q + ".feed_forward.w_2", sd)
            for n in ("norm1", "norm2", "norm3"):
                _ln(g, d, f"{q}.{n}", sd)
            if emb_len > 0 and (i == 0 or i == nb - 1):
                # LanguageSpecificDecoderLayer also owns two unused concat linears
                # (transformer/decoder_layer.py:246-247)
                _lin(g, d, 2 * d, True, q + ".concat_linear1", sd)
                _lin(g, d, 2 * d, True, q + ".concat_linear2", sd)
                for j in range(emb_len):
                    _lin(g, d, d, True, f"{q}.language_layers.{j}", sd)
    return sd


def make_units(vocab: int):
    """tk.units.txt: '<blank> 0' ... '<sos/eos> V-1' (utils/file_utils.py:61-68); every 3rd
    piece starts a word; a couple of <...> special pieces exercise ctc_align's special path."""
    lines = ["<blank> 0", "<unk> 1"]
    for i in range(2, vocab - 1):
        if i % 17 == 5:
            piece = f"<sp{i}>"
        elif i % 3 == 0:
            piece = f"▁w{i}"
        else:
            piece = f"p{i}"
        lines.append(f"{piece} {i}")
    lines.append(f"<sos/eos> {vocab - 1}")
    return lines


def write_model_dir(path: str, shape: Dict = None, seed: int = 0, causal: bool = True,
                    cnn_module_norm: str = "layer_norm", reverse_weight: float = 0.3,
                    blank_rate: float = 0.8) -> str:
    """Create a model directory loadable by both the reference's and this repo's `load_model`."""
    shape = dict(TEST_SHAPE if shape is None else shape)
    os.makedirs(path, exist_ok=True)
    cfg = make_config(shape, causal=causal, cnn_module_norm=cnn_module_norm, reverse_weight=reverse_weight)
    with open(os.path.join(path, "config.yaml"), "w") as f:
        yaml.safe_dump(cfg, f, sort_keys=False)
    sd = make_state_dict(cfg, shape["vocab"], seed=seed, blank_rate=blank_rate)
    # JSON cmvn stats consistent with the mean/istd buffers (utils/cmvn.py:21-43)
    mean = sd["encoder.global_cmvn.mean"].double().numpy()
    istd = sd["encoder.global_cmvn.istd"].double().numpy()
    n = 1000.0
    var = 1.0 / (istd * istd)
    stats = {"mean_stat": (mean * n).tolist(), "var_stat": ((var + mean * mean) * n).tolist(), "frame_num": n}
    with open(os.path.join(path, "cmvn"), "w") as f:
        json.dump(stats, f)
    with open(os.path.join(path, "tk.units.txt"), "w", encoding="utf8") as f:
        f.write("\n".join(make_units(shape["vocab"])) + "\n")
    open(os.path.join(path, "tk.model"), "wb").close()
    torch.save(sd, os.path.join(path, "synth.pt"))
    return path


def synth_audio(seconds: float, seed: int = 1234, sample_rate: int = 16000) -> np.ndarray:
    """Speech-like int16 audio (SURVEY.md §8d): Gaussian noise sigma=3000 amplitude-modulated
    at 4 Hz + 3 harmonics of a 120 Hz tone, with ~20 % silent segments."""
    rng = np.random.default_rng(seed)
    n = int(round(seconds * sample_rate))
    t = np.arange(n, dtype=np.float64) / sample_rate
    x = rng.normal(0.0, 3000.0, n) * (0.55 + 0.45 * np.sin(2 * np.pi * 4.0 * t))
    for h in (1, 2, 3):
        x += (1500.0 / h) * np.sin(2 * np.pi * 120.0 * h * t + 0.3 * h)
    seg = sample_rate // 2
    nseg = (n + seg - 1) // seg
    silent = rng.random(nseg) < 0.2
    mask = np.repeat(~silent, seg)[:n]
    x = x * mask
    return np.clip(np.round(x), -32768, 32767).astype(np.int16)


def write_wav(path: str, pcm: np.ndarray, sample_rate: int = 16000) -> str:
    with wave.open(path, "wb") as w:
        w.setnchannels(1)
        w.setsampwidth(2)
        w.setframerate(sample_rate)
        w.writeframes(np.ascontiguousarray(pcm, dtype=np.int16).tobytes())
    return path


def context_phrases(n: int, vocab: int, seed: int = 0, blank_id: int = 0, max_len: int = 4):
    """`n` seeded biasing phrases of 1..max_len non-blank token ids (duplicates and shared prefixes included, as in a
    real list) — for the context biasing tests and tools/context_bench.py."""
    rng = np.random.default_rng(seed)
    toks = np.setdiff1d(np.arange(vocab), [blank_id])
    return [rng.choice(toks, size=int(rng.integers(1, max_len + 1))).tolist() for _ in range(n)]


def context_topk(B: int, T: int, k: int, vocab: int, phrases, seed: int = 0, blank_id: int = 0):
    """Seeded per-frame top-k CTC log-probs (val (B, T, k) float32 descending, idx (B, T, k) int32) in which the tokens
    of `phrases` appear often: every utterance walks through a script of phrase tokens and random tokens, each held a
    few frames between blank runs; the script token is ranked first or, about a third of the time, just below a
    competitor by a small margin — where a context bonus can change the n-best."""
    rng = np.random.default_rng(seed)
    pool = np.unique(np.concatenate([np.asarray(p, dtype=np.int64) for p in phrases] + [np.arange(vocab)]))
    pool = pool[pool != blank_id]
    idx = np.empty((B, T, k), dtype=np.int32)
    val = np.empty((B, T, k), dtype=np.float32)
    for b in range(B):
        script = []
        while len(script) < T:
            script += list(phrases[int(rng.integers(len(phrases)))]) if rng.random() < 0.6 else \
                rng.choice(pool, size=int(rng.integers(1, 4))).tolist()
        pos, t = 0, 0
        while t < T:
            run = [blank_id] * int(rng.integers(0, 3)) + [script[pos]] * int(rng.integers(1, 4))
            pos += 1
            for tok in run[:T - t]:
                others = rng.choice(pool, size=k + 1, replace=False)
                others = [int(o) for o in others if o != tok][:k - 1]
                if tok != blank_id and blank_id not in others and rng.random() < 0.7:
                    others[-1] = blank_id
                order = [tok] + others
                if tok != blank_id and rng.random() < 0.35:
                    order[0], order[1] = order[1], order[0]           # the script token trails a competitor
                logits = np.sort(rng.normal(0.0, 1.0, k))[::-1] * 2.0
                logits[0] = logits[1] + (rng.uniform(0.05, 1.0) if rng.random() < 0.5 else rng.uniform(1.0, 6.0))
                lse = np.log(np.exp(logits - logits[0]).sum() + 1e-3) + logits[0]
                idx[b, t] = order
                val[b, t] = (logits - lse).astype(np.float32)
                t += 1
    return val, idx
