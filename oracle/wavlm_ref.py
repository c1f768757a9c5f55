"""CPU oracle of reverb-diarization-v2's segmentation network — TEST INFRASTRUCTURE ONLY.

pyannote's `SSeRiouSS` (pyannote.audio 3.3.1, restated from its published source): torchaudio's `wavlm_base()`
`extract_features` -> softmax(wav2vec_weights)-weighted sum of the 12 layer outputs -> 4-layer bidirectional
LSTM(128) -> 2 x [Linear(128) + LeakyReLU] -> Linear(7) -> LogSoftmax.  Written here with stock torch ops only
(F.conv1d, F.group_norm, F.layer_norm, F.scaled_dot_product_attention, nn.LSTM) so that GPU tests can import it
without torchaudio.  tests/test_wavlm_oracle.py pins the WavLM part against `torchaudio.models.wavlm_base`; the head
is unpinned (pyannote's source and the HF weights are absent), like all of v1 (oracle/diar_ref.py).

Only tests/, __graft_entry__.smoke() and the benchmark tools may import this module.
"""
from __future__ import annotations

import math
from typing import Dict, List, Optional, Tuple

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

CONV = ((10, 5), (3, 2), (3, 2), (3, 2), (3, 2), (2, 2), (2, 2))
P = "wav2vec."


def num_frames(num_samples: int) -> int:
    n = num_samples
    for k, s in CONV:
        n = (n - k) // s + 1 if n >= k else 0
    return n


def relative_positions_bucket(rel: torch.Tensor, num_buckets: int = 320, max_distance: int = 800) -> torch.Tensor:
    """torchaudio `WavLMSelfAttention._relative_positions_bucket` (bidirectional), float32 log and truncation."""
    nb = num_buckets // 2
    buckets = (rel > 0).to(torch.long) * nb
    rel = torch.abs(rel)
    max_exact = nb // 2
    is_small = rel < max_exact
    large = max_exact + (torch.log(rel.float() / max_exact) / math.log(max_distance / max_exact)
                         * (nb - max_exact)).to(torch.long)
    large = torch.minimum(large, torch.full_like(large, nb - 1))
    return buckets + torch.where(is_small, rel, large)


def fold_weight_norm(g: torch.Tensor, v: torch.Tensor) -> torch.Tensor:
    """weight_norm(dim=2): w[o, i, k] = g[k] v[o, i, k] / ||v[:, :, k]||"""
    return g * v / v.pow(2).sum(dim=(0, 1), keepdim=True).sqrt()


def stored_bf16(sd) -> List[str]:
    """The tensors WavLMSegRef(stored_weights=True) rounds to bf16, as csrc/diar_wavlm.cu finalize stores them: conv
    layers 1-6, the feature projection, in/out-proj and the two FFN weights of every layer (the folded positional conv
    weight is rounded too, see WavLMSegRef)."""
    names = [f"{P}feature_extractor.conv_layers.{i}.conv.weight" for i in range(1, len(CONV))]
    names.append(P + "encoder.feature_projection.projection.weight")
    for k in sd:
        if k.startswith(P + "encoder.transformer.layers.") and k.endswith((
                ".attention.attention.in_proj_weight", ".attention.attention.out_proj.weight",
                ".feed_forward.intermediate_dense.weight", ".feed_forward.output_dense.weight")):
            names.append(k)
    return names


class WavLMSegRef(nn.Module):
    """The network in `dtype` on `device` (float32 on the CPU by default).  With `stored_weights` it runs on the
    weights the network stores: `stored_bf16(sd)` rounded to bf16 (round to nearest even), and the positional conv's
    weight norm folded in float64, cast to float32, then rounded to bf16; everything else stays fp32."""

    def __init__(self, sd: Dict[str, np.ndarray], num_heads: int = 12, lstm_hidden: int = 128, lstm_layers: int = 4,
                 dtype: torch.dtype = torch.float32, device="cpu", stored_weights: bool = False):
        super().__init__()
        t32 = {k: torch.from_numpy(np.asarray(v, np.float32)) for k, v in sd.items()}
        if stored_weights:
            for k in stored_bf16(sd):
                t32[k] = t32[k].to(torch.bfloat16).float()
        self.t = t = {k: v.to(device=device, dtype=dtype) for k, v in t32.items()}
        self.H = num_heads
        self.L = sum(1 for k in t if k.startswith(P + "encoder.transformer.layers.") and k.endswith(".final_layer_norm.weight"))
        pc = P + "encoder.transformer.pos_conv_embed.conv."
        if pc + "parametrizations.weight.original0" in t:
            g, v = t[pc + "parametrizations.weight.original0"], t[pc + "parametrizations.weight.original1"]
        else:
            g, v = t[pc + "weight_g"], t[pc + "weight_v"]
        if stored_weights:
            self.pos_w = fold_weight_norm(g.double(), v.double()).float().to(torch.bfloat16).to(dtype)
        else:
            self.pos_w = fold_weight_norm(g, v)
        D = self.pos_w.shape[0]
        self.lstm = nn.LSTM(D, lstm_hidden, num_layers=lstm_layers, bidirectional=True, batch_first=True,
                            device=device, dtype=dtype)
        with torch.no_grad():
            for name, p in self.lstm.named_parameters():
                p.copy_(t["lstm." + name])
        self.n_linear = sum(1 for k in t if k.startswith("linear.") and k.endswith(".weight"))

    @torch.no_grad()
    def conv_features(self, wav: torch.Tensor) -> torch.Tensor:
        """(B, N) -> (B, T, 512)"""
        t = self.t
        fe = P + "feature_extractor.conv_layers."
        x = wav.unsqueeze(1)
        for i, (_, s) in enumerate(CONV):
            x = F.conv1d(x, t[f"{fe}{i}.conv.weight"], stride=s)
            if i == 0:
                x = F.group_norm(x, x.shape[1], t[fe + "0.layer_norm.weight"], t[fe + "0.layer_norm.bias"])
            x = F.gelu(x)
        return x.transpose(1, 2)

    @torch.no_grad()
    def front(self, feats: torch.Tensor) -> torch.Tensor:
        """(B, T, 512) conv features -> (B, T, 768) input of layer 0: LayerNorm, projection, positional conv, and the
        transformer's LayerNorm."""
        t = self.t
        fp = P + "encoder.feature_projection."
        x = F.linear(F.layer_norm(feats, (feats.shape[-1],), t[fp + "layer_norm.weight"], t[fp + "layer_norm.bias"]),
                     t[fp + "projection.weight"], t[fp + "projection.bias"])
        D = x.shape[-1]
        K, groups = self.pos_w.shape[-1], D // self.pos_w.shape[1]
        pc = F.conv1d(x.transpose(1, 2), self.pos_w, t[P + "encoder.transformer.pos_conv_embed.conv.bias"],
                      padding=K // 2, groups=groups)
        x = x + F.gelu(pc[..., :-1] if K % 2 == 0 else pc).transpose(1, 2)
        # torchaudio builds the post-LN wavlm_base with Transformer.layer_norm_first = True: the transformer's LayerNorm
        # runs once here, before layer 0, and never after the last layer
        return F.layer_norm(x, (D,), t[P + "encoder.transformer.layer_norm.weight"],
                            t[P + "encoder.transformer.layer_norm.bias"])

    def _rel_bias(self, T: int) -> torch.Tensor:
        """(H, T, T) relative-position bias; the buckets are integers computed the float32 way in every dtype"""
        emb = self.t[P + "encoder.transformer.layers.0.attention.rel_attn_embed.weight"]
        pos = torch.arange(T)
        return emb[relative_positions_bucket(pos[None, :] - pos[:, None]).to(emb.device)].permute(2, 0, 1)

    @torch.no_grad()
    def layer(self, l: int, x: torch.Tensor, bias: Optional[torch.Tensor] = None) -> torch.Tensor:
        """Transformer layer l on its input (B, T, 768) -> its output (B, T, 768)."""
        t = self.t
        B, T, D = x.shape
        if bias is None:
            bias = self._rel_bias(T)
        H, dh = self.H, D // self.H
        q = f"{P}encoder.transformer.layers.{l}."
        xh = x.view(B, T, H, dh).permute(0, 2, 1, 3)
        ga, gb = torch.sigmoid(F.linear(xh, t[q + "attention.gru_rel_pos_linear.weight"],
                                        t[q + "attention.gru_rel_pos_linear.bias"]).view(B, H, T, 2, 4).sum(-1)).chunk(2, -1)
        gate = ga * (gb * t[q + "attention.gru_rel_pos_const"].view(1, H, 1, 1) - 1.0) + 2.0   # (B, H, T, 1)
        qkv = F.linear(x, t[q + "attention.attention.in_proj_weight"], t[q + "attention.attention.in_proj_bias"])
        qq, kk, vv = (z.view(B, T, H, dh).transpose(1, 2) for z in qkv.chunk(3, -1))
        a = F.scaled_dot_product_attention(qq, kk, vv, attn_mask=gate * bias.unsqueeze(0))
        a = F.linear(a.transpose(1, 2).reshape(B, T, D), t[q + "attention.attention.out_proj.weight"],
                     t[q + "attention.attention.out_proj.bias"])
        x = F.layer_norm(x + a, (D,), t[q + "layer_norm.weight"], t[q + "layer_norm.bias"])
        ff = F.linear(F.gelu(F.linear(x, t[q + "feed_forward.intermediate_dense.weight"],
                                      t[q + "feed_forward.intermediate_dense.bias"])),
                      t[q + "feed_forward.output_dense.weight"], t[q + "feed_forward.output_dense.bias"])
        return F.layer_norm(x + ff, (D,), t[q + "final_layer_norm.weight"], t[q + "final_layer_norm.bias"])

    @torch.no_grad()
    def layers(self, feats: torch.Tensor) -> List[torch.Tensor]:
        """(B, T, 512) -> the 12 layer outputs (B, T, 768)"""
        x = self.front(feats)
        bias = self._rel_bias(x.shape[1])
        out = []
        for l in range(self.L):
            x = self.layer(l, x, bias)
            out.append(x)
        return out

    @torch.no_grad()
    def head(self, layers: List[torch.Tensor]) -> torch.Tensor:
        t = self.t
        w = F.softmax(t["wav2vec_weights"], dim=0)
        x = sum(w[i] * layers[i] for i in range(len(layers)))
        x, _ = self.lstm(x)
        for i in range(self.n_linear):
            x = F.leaky_relu(F.linear(x, t[f"linear.{i}.weight"], t[f"linear.{i}.bias"]))
        return F.log_softmax(F.linear(x, t["classifier.weight"], t["classifier.bias"]), dim=-1)

    @torch.no_grad()
    def forward(self, wav: torch.Tensor) -> Tuple[torch.Tensor, List[torch.Tensor], torch.Tensor]:
        """(B, N) -> (conv features, layer outputs, log-probabilities)"""
        feats = self.conv_features(wav)
        layers = self.layers(feats)
        return feats, layers, self.head(layers)
