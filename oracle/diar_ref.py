"""CPU oracle of the diarization forward (SURVEY.md §8f rank 1) — TEST INFRASTRUCTURE ONLY.

** parity unpinned **  The reference runs `pyannote.audio==3.3.1` behind
`Pipeline.from_pretrained('Revai/reverb-diarization-v1')` (diarization/infer_pyannote3.0.py:14,33-40;
diarization/requirements.txt:1).  Neither the package, its source nor the model weights are available offline or in
the reference repository, and the reference holds no tests or golden vectors for this path.  This file restates the PUBLISHED
architecture of that pipeline's two networks from the upstream project's public description:

  * segmentation  `PyanNet`  (pyannote/audio/models/segmentation/PyanNet.py, v3.3.1): SincNet front-end
    (InstanceNorm1d(1) -> ParamSincFB(80, 251, stride 10) |.| -> 3 x [MaxPool1d(3) -> InstanceNorm1d -> LeakyReLU] with
    Conv1d(80,60,5), Conv1d(60,60,5)) -> 4-layer bidirectional LSTM(hidden 128) -> 2 x [Linear(128) + LeakyReLU] ->
    Linear(7) -> LogSoftmax over the powerset classes of <= 3 speakers, <= 2 simultaneously (10 s window -> 589 frames);
  * embedding  `WeSpeakerResNet34` (pyannote/audio/models/embedding/wespeaker/): Kaldi fbank (80 mel, hamming window,
    waveform * 2^15, per-utterance mean subtraction) -> ResNet34 (BasicBlock [3,4,6,3], 32..256 channels, BatchNorm,
    ReLU) -> weighted temporal statistics pooling (mean, std) -> Linear(5120, 256).

They are built here from stock torch modules (nn.LSTM, F.conv1d, nn.BatchNorm2d ...) so that the CUDA kernels are
compared against torch's own arithmetic for the same architecture and the same (synthetic) weights.  What this oracle
cannot establish is that the architecture constants above equal the shipped checkpoints' — that needs the pyannote
3.3.1 source and the HuggingFace `config.yaml`, which a later session must supply.

Only tests/, __graft_entry__.smoke() and bench.py's CPU legs may import this module.
"""
from __future__ import annotations

import math
from typing import Dict, List, Optional, Tuple

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

# --------------------------------------------------------------------------------------------------------------------
# segmentation: PyanNet


def sinc_filters(low_hz_: torch.Tensor, band_hz_: torch.Tensor, kernel_size: int = 251, sample_rate: float = 16000.0,
                 min_low_hz: float = 50.0, min_band_hz: float = 50.0) -> torch.Tensor:
    """ParamSincFB.filters() (asteroid-filterbanks `param_sinc_fb.py`): n_filters/2 cosine + n_filters/2 sine band-pass
    filters from the learnt (low, band) cut-offs, half Hamming window mirrored around the centre tap.  -> (2C, kernel)."""
    half = kernel_size // 2
    like = dict(dtype=low_hz_.dtype, device=low_hz_.device)
    n_lin = torch.linspace(0, kernel_size / 2 - 1, steps=half, **like)
    window = 0.54 - 0.46 * torch.cos(2 * math.pi * n_lin / kernel_size)
    n_ = 2 * math.pi * torch.arange(-half, 0.0, **like).view(1, -1) / sample_rate
    low = min_low_hz + torch.abs(low_hz_.view(-1, 1))
    high = torch.clamp(low + min_band_hz + torch.abs(band_hz_.view(-1, 1)), min_low_hz, sample_rate / 2)
    band = (high - low)[:, 0]
    ft_low = torch.matmul(low, n_)
    ft_high = torch.matmul(high, n_)
    out = []
    for kind in ("cos", "sin"):
        if kind == "cos":
            left = ((torch.sin(ft_high) - torch.sin(ft_low)) / (n_ / 2)) * window
            center = 2 * band.view(-1, 1)
            right = torch.flip(left, dims=[1])
        else:
            left = ((torch.cos(ft_low) - torch.cos(ft_high)) / (n_ / 2)) * window
            center = torch.zeros_like(band.view(-1, 1))
            right = -torch.flip(left, dims=[1])
        bp = torch.cat([left, center, right], dim=1)
        out.append(bp / (2 * band[:, None]))
    return torch.cat(out, dim=0)


def _tensors(sd: Dict[str, np.ndarray], dtype: torch.dtype, device) -> Dict[str, torch.Tensor]:
    return {k: torch.from_numpy(np.asarray(v, np.float32)).to(device=device, dtype=dtype) for k, v in sd.items()}


def bf16_round(x: torch.Tensor) -> torch.Tensor:
    """x rounded to bfloat16 (round to nearest even, like the library's host-side f2bf / __float2bfloat16), in x's dtype."""
    return x.float().to(torch.bfloat16).to(x.dtype)


def _instance_norm(x: torch.Tensor, weight: torch.Tensor, bias: torch.Tensor) -> torch.Tensor:
    """F.instance_norm, which refuses a single position; there x - mean = 0 and the output is the bias (a 991-sample
    window has one frame)."""
    if x.shape[-1] == 1:
        return bias.view(1, -1, 1).expand_as(x).clone()
    return F.instance_norm(x, weight=weight, bias=bias)


class PyanNetRef(nn.Module):
    """Forward of PyanNet on (B, num_samples) waveforms -> (B, frames, classes) log-probabilities, in `dtype` on
    `device` (float32 on the CPU by default).  The network stores every weight in fp32, so there is no stored-weights
    variant."""

    def __init__(self, sd: Dict[str, np.ndarray], lstm_hidden: int = 128, lstm_layers: int = 4,
                 dtype: torch.dtype = torch.float32, device="cpu"):
        super().__init__()
        t = _tensors(sd, dtype, device)
        self.t = t
        self.filters = sinc_filters(t["sincnet.conv1d.0.filterbank.low_hz_"], t["sincnet.conv1d.0.filterbank.band_hz_"])
        in_dim = t["sincnet.conv1d.2.weight"].shape[0]
        self.lstm = nn.LSTM(in_dim, lstm_hidden, num_layers=lstm_layers, bidirectional=True, batch_first=True,
                            device=device, dtype=dtype)
        with torch.no_grad():
            for name, p in self.lstm.named_parameters():
                p.copy_(t["lstm." + name])
        self.n_linear = sum(1 for k in t if k.startswith("linear.") and k.endswith(".weight"))

    @torch.no_grad()
    def sincnet(self, wav: torch.Tensor) -> torch.Tensor:
        t = self.t
        x = F.instance_norm(wav.unsqueeze(1), weight=t["sincnet.wav_norm1d.weight"], bias=t["sincnet.wav_norm1d.bias"])
        x = torch.abs(F.conv1d(x, self.filters.unsqueeze(1), stride=10))
        x = F.leaky_relu(_instance_norm(F.max_pool1d(x, 3, 3), t["sincnet.norm1d.0.weight"], t["sincnet.norm1d.0.bias"]))
        for i in (1, 2):
            x = F.conv1d(x, t[f"sincnet.conv1d.{i}.weight"], t[f"sincnet.conv1d.{i}.bias"])
            x = F.leaky_relu(_instance_norm(F.max_pool1d(x, 3, 3), t[f"sincnet.norm1d.{i}.weight"],
                                            t[f"sincnet.norm1d.{i}.bias"]))
        return x                                                     # (B, 60, frames)

    @torch.no_grad()
    def forward(self, wav: torch.Tensor) -> torch.Tensor:
        return self.head(self.sincnet(wav).transpose(1, 2))

    @torch.no_grad()
    def head(self, x: torch.Tensor) -> torch.Tensor:
        """(B, frames, 60) SincNet features -> (B, frames, classes) log-probabilities: LSTM, linears, classifier."""
        t = self.t
        x, _ = self.lstm(x)
        for i in range(self.n_linear):
            x = F.leaky_relu(F.linear(x, t[f"linear.{i}.weight"], t[f"linear.{i}.bias"]))
        x = F.linear(x, t["classifier.weight"], t["classifier.bias"])
        return F.log_softmax(x, dim=-1)


def seg_num_frames(num_samples: int) -> int:
    n = (num_samples - 251) // 10 + 1
    n = n // 3
    for _ in range(2):
        n = (n - 4) // 3
    return n


# --------------------------------------------------------------------------------------------------------------------
# embedding: WeSpeaker ResNet34


def wespeaker_fbank(wav: torch.Tensor) -> torch.Tensor:
    """(num_samples,) in [-1, 1] -> (frames, 80): Kaldi fbank on wav * 2^15 with a hamming window, no dither, minus the
    mean over time (pyannote `WeSpeakerResNet34.compute_fbank`)."""
    import torchaudio.compliance.kaldi as kaldi
    f = kaldi.fbank(wav.view(1, -1) * (1 << 15), num_mel_bins=80, frame_length=25, frame_shift=10, dither=0.0,
                    sample_frequency=16000, window_type="hamming", use_energy=False)
    return f - f.mean(dim=0, keepdim=True)


class ResNet34Ref(nn.Module):
    """WeSpeaker ResNet34 on (B, frames, 80) features (+ optional (B, frames') pooling weights) -> (B, 256), in `dtype`
    on `device` (float32 on the CPU by default).

    With `stored_weights` every convolution runs with the weights the network stores (csrc/diar_emb.cu finalize):
    BatchNorm folded into the convolution in fp32 (scale = gamma / sqrtf(var + 1e-5), weight * scale, bias = beta -
    mean * scale), then the weights of every convolution but the first rounded to bf16 (`resnet_stored_bf16` names them)."""

    BLOCKS = (3, 4, 6, 3)

    def __init__(self, sd: Dict[str, np.ndarray], dtype: torch.dtype = torch.float32, device="cpu",
                 stored_weights: bool = False):
        super().__init__()
        self.t = _tensors(sd, dtype, device)
        self.folded = None
        if stored_weights:
            t32 = _tensors(sd, torch.float32, device)
            self.folded = {}
            rounded = set(resnet_stored_bf16(sd))
            for conv, bn in resnet_convs(sd):
                scale = t32[bn + ".weight"] / torch.sqrt(t32[bn + ".running_var"] + 1e-5)
                w = t32[conv] * scale.view(-1, 1, 1, 1)
                if conv in rounded:
                    w = bf16_round(w)
                self.folded[conv] = (w.to(dtype), (t32[bn + ".bias"] - t32[bn + ".running_mean"] * scale).to(dtype))

    def _conv_bn(self, x, conv, bn, **kw):
        if self.folded is not None:
            w, b = self.folded[conv]
            return F.conv2d(x, w, b, **kw)
        t = self.t
        return F.batch_norm(F.conv2d(x, t[conv], **kw), t[bn + ".running_mean"], t[bn + ".running_var"],
                            t[bn + ".weight"], t[bn + ".bias"], False, 0.0, 1e-5)

    @torch.no_grad()
    def trunk(self, feats: torch.Tensor) -> torch.Tensor:
        t = self.t
        x = feats.permute(0, 2, 1).unsqueeze(1)                      # (B, 1, F, T)
        x = F.relu(self._conv_bn(x, "resnet.conv1.weight", "resnet.bn1", padding=1))
        for li, nb in enumerate(self.BLOCKS, start=1):
            for bi in range(nb):
                p = f"resnet.layer{li}.{bi}"
                stride = 2 if (li > 1 and bi == 0) else 1
                y = F.relu(self._conv_bn(x, p + ".conv1.weight", p + ".bn1", stride=stride, padding=1))
                y = self._conv_bn(y, p + ".conv2.weight", p + ".bn2", padding=1)
                if (p + ".shortcut.0.weight") in t:
                    x = self._conv_bn(x, p + ".shortcut.0.weight", p + ".shortcut.1", stride=stride)
                x = F.relu(y + x)
        return x                                                     # (B, 256, F/8, T/8)

    @torch.no_grad()
    def forward(self, feats: torch.Tensor, weights: Optional[torch.Tensor] = None) -> torch.Tensor:
        t = self.t
        x = self.trunk(feats)
        B, C, Fq, T = x.shape
        seq = x.reshape(B, C * Fq, T)
        stats = stats_pool(seq, weights)
        return F.linear(stats, t["resnet.seg_1.weight"], t["resnet.seg_1.bias"])


_BN_OF = ((".conv1.weight", ".bn1"), (".conv2.weight", ".bn2"), (".shortcut.0.weight", ".shortcut.1"))


def resnet_convs(sd) -> List[Tuple[str, str]]:
    """(convolution weight, its BatchNorm prefix) of every convolution of the trunk, in state_dict order."""
    out = []
    for k in sd:
        if k == "resnet.conv1.weight":
            out.append((k, "resnet.bn1"))
        elif k.startswith("resnet.layer"):
            out += [(k, k[:-len(w)] + bn) for w, bn in _BN_OF if k.endswith(w)]
    return out


def resnet_stored_bf16(sd) -> List[str]:
    """The tensors ResNet34Ref(stored_weights=True) rounds to bf16: every trunk convolution but the first."""
    return [conv for conv, _ in resnet_convs(sd) if conv != "resnet.conv1.weight"]


def stats_pool(seq: torch.Tensor, weights: Optional[torch.Tensor]) -> torch.Tensor:
    """pyannote `StatsPool`: (B, D, T) [+ (B, T_w) weights, nearest-interpolated to T] -> (B, 2D) = [mean, std]."""
    if weights is None:
        return torch.cat([seq.mean(dim=-1), seq.std(dim=-1, correction=1)], dim=-1)
    w = weights.unsqueeze(1)
    if w.shape[-1] != seq.shape[-1]:
        w = F.interpolate(w, size=seq.shape[-1], mode="nearest")
    v1 = w.sum(dim=-1) + 1e-8
    mean = (seq * w).sum(dim=-1) / v1
    dx2 = (seq - mean.unsqueeze(-1)) ** 2
    v2 = (w * w).sum(dim=-1)
    var = (dx2 * w).sum(dim=-1) / (v1 - v2 / v1 + 1e-8)
    return torch.cat([mean, torch.sqrt(var)], dim=-1)
