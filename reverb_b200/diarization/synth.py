"""Synthetic weights for the two diarization networks, under pyannote's state_dict names.

The `Revai/reverb-diarization-v1` checkpoints live on HuggingFace and cannot be fetched offline (SURVEY.md §8c), so
parity tests and the diarization benchmark run on seeded random weights of the published shapes.
"""
from __future__ import annotations

import math
from typing import Dict

import numpy as np

SEG_SHAPE = dict(sample_rate=16000, sinc_filters=80, sinc_kernel=251, sinc_stride=10, conv_channels=60, conv_kernel=5,
                 lstm_hidden=128, lstm_layers=4, linear_dim=128, linear_layers=2, num_classes=7)


def _uniform(rng, shape, bound):
    return rng.uniform(-bound, bound, size=shape).astype(np.float32)


def segmentation_state_dict(seed: int = 0, shape: Dict = SEG_SHAPE) -> Dict[str, np.ndarray]:
    """PyanNet weights: SincNet cut-offs mel-spaced like ParamSincFB's initialisation (+ jitter), PyTorch-default
    uniform initialisation elsewhere; the classifier is scaled up so the log-probabilities are not flat."""
    rng = np.random.default_rng(seed)
    sd: Dict[str, np.ndarray] = {}
    half = shape["sinc_filters"] // 2
    sr = shape["sample_rate"]

    def to_mel(hz):
        return 2595 * np.log10(1 + hz / 700)

    def to_hz(mel):
        return 700 * (10 ** (mel / 2595) - 1)

    mel = np.linspace(to_mel(30.0), to_mel(sr / 2 - 100.0), half + 1)
    hz = to_hz(mel)
    sd["sincnet.wav_norm1d.weight"] = np.array([1.1], np.float32)
    sd["sincnet.wav_norm1d.bias"] = np.array([0.02], np.float32)
    sd["sincnet.conv1d.0.filterbank.low_hz_"] = (hz[:-1] * rng.uniform(0.95, 1.05, half)).astype(np.float32).reshape(-1, 1)
    sd["sincnet.conv1d.0.filterbank.band_hz_"] = (np.diff(hz) * rng.uniform(0.9, 1.1, half)).astype(np.float32).reshape(-1, 1)
    chans = [shape["sinc_filters"], shape["conv_channels"], shape["conv_channels"]]
    for i, c in enumerate(chans):
        sd[f"sincnet.norm1d.{i}.weight"] = rng.uniform(0.5, 1.5, c).astype(np.float32)
        sd[f"sincnet.norm1d.{i}.bias"] = rng.uniform(-0.2, 0.2, c).astype(np.float32)
    k = shape["conv_kernel"]
    for i in (1, 2):
        cin = chans[i - 1]
        bound = 1.0 / math.sqrt(cin * k)
        sd[f"sincnet.conv1d.{i}.weight"] = _uniform(rng, (shape["conv_channels"], cin, k), bound)
        sd[f"sincnet.conv1d.{i}.bias"] = _uniform(rng, (shape["conv_channels"],), bound)
    _head_state_dict(rng, sd, shape["conv_channels"], shape)
    return sd


def _head_state_dict(rng, sd: Dict[str, np.ndarray], in_dim: int, shape: Dict) -> None:
    """PyanNet's head (LSTM, linears, classifier) on `in_dim` input features, drawn from `rng` in that order."""
    H = shape["lstm_hidden"]
    bound = 1.0 / math.sqrt(H)
    for layer in range(shape["lstm_layers"]):
        cin = in_dim if layer == 0 else 2 * H
        for sfx in ("", "_reverse"):
            # larger than PyTorch's default so that the random network reacts to its input (default-init LSTMs are flat)
            sd[f"lstm.weight_ih_l{layer}{sfx}"] = _uniform(rng, (4 * H, cin), 4.0 * bound)
            sd[f"lstm.weight_hh_l{layer}{sfx}"] = _uniform(rng, (4 * H, H), 2.0 * bound)
            sd[f"lstm.bias_ih_l{layer}{sfx}"] = _uniform(rng, (4 * H,), bound)
            sd[f"lstm.bias_hh_l{layer}{sfx}"] = _uniform(rng, (4 * H,), bound)
    cin = 2 * H
    for i in range(shape["linear_layers"]):
        bound = 3.0 / math.sqrt(cin)
        sd[f"linear.{i}.weight"] = _uniform(rng, (shape["linear_dim"], cin), bound)
        sd[f"linear.{i}.bias"] = _uniform(rng, (shape["linear_dim"],), bound)
        cin = shape["linear_dim"]
    bound = 6.0 / math.sqrt(cin)
    sd["classifier.weight"] = _uniform(rng, (shape["num_classes"], cin), bound)
    sd["classifier.bias"] = _uniform(rng, (shape["num_classes"],), 0.5)


# reverb-diarization-v2: pyannote SSeRiouSS on torchaudio's wavlm_base(), PyanNet's head
WAVLM_SEG_SHAPE = dict(sample_rate=16000, conv_channels=512, embed_dim=768, num_layers=12, num_heads=12, ffn_dim=3072,
                       pos_conv_kernel=128, pos_conv_groups=16, num_buckets=320, max_distance=800, lstm_hidden=128,
                       lstm_layers=4, linear_dim=128, linear_layers=2, num_classes=7)
WAVLM_CONV = ((10, 5), (3, 2), (3, 2), (3, 2), (3, 2), (2, 2), (2, 2))   # (kernel, stride) of the feature extractor


def wavlm_segmentation_state_dict(seed: int = 0, shape: Dict = WAVLM_SEG_SHAPE) -> Dict[str, np.ndarray]:
    """SSeRiouSS weights under pyannote's names (`wav2vec.` + torchaudio's wavlm_base names, `wav2vec_weights`, the
    head's): PyTorch-default uniform initialisation, norms and gates away from the identity so that every term is
    exercised."""
    rng = np.random.default_rng(seed)
    sd: Dict[str, np.ndarray] = {}
    C, D, H, F = shape["conv_channels"], shape["embed_dim"], shape["num_heads"], shape["ffn_dim"]
    p = "wav2vec."
    fe = p + "feature_extractor.conv_layers."
    cin = 1
    for i, (k, _) in enumerate(WAVLM_CONV):
        sd[f"{fe}{i}.conv.weight"] = _uniform(rng, (C, cin, k), math.sqrt(3.0 / (cin * k)))
        cin = C
    sd[fe + "0.layer_norm.weight"] = rng.uniform(0.8, 1.2, C).astype(np.float32)
    sd[fe + "0.layer_norm.bias"] = rng.uniform(-0.1, 0.1, C).astype(np.float32)
    fp = p + "encoder.feature_projection."
    sd[fp + "layer_norm.weight"] = rng.uniform(0.8, 1.2, C).astype(np.float32)
    sd[fp + "layer_norm.bias"] = rng.uniform(-0.1, 0.1, C).astype(np.float32)
    sd[fp + "projection.weight"] = _uniform(rng, (D, C), 1.0 / math.sqrt(C))
    sd[fp + "projection.bias"] = _uniform(rng, (D,), 1.0 / math.sqrt(C))
    K, G = shape["pos_conv_kernel"], shape["pos_conv_groups"]
    pc = p + "encoder.transformer.pos_conv_embed.conv."
    sd[pc + "bias"] = _uniform(rng, (D,), 0.1)
    sd[pc + "parametrizations.weight.original0"] = rng.uniform(0.5, 1.5, (1, 1, K)).astype(np.float32)
    sd[pc + "parametrizations.weight.original1"] = rng.normal(0, 1, (D, D // G, K)).astype(np.float32)
    sd[p + "encoder.transformer.layer_norm.weight"] = rng.uniform(0.8, 1.2, D).astype(np.float32)
    sd[p + "encoder.transformer.layer_norm.bias"] = rng.uniform(-0.1, 0.1, D).astype(np.float32)
    for l in range(shape["num_layers"]):
        q = f"{p}encoder.transformer.layers.{l}."
        if l == 0:
            sd[q + "attention.rel_attn_embed.weight"] = rng.normal(0, 1, (shape["num_buckets"], H)).astype(np.float32)
        b = 1.0 / math.sqrt(D)
        sd[q + "attention.attention.in_proj_weight"] = _uniform(rng, (3 * D, D), math.sqrt(3.0) * b)
        sd[q + "attention.attention.in_proj_bias"] = _uniform(rng, (3 * D,), b)
        sd[q + "attention.attention.out_proj.weight"] = _uniform(rng, (D, D), b)
        sd[q + "attention.attention.out_proj.bias"] = _uniform(rng, (D,), b)
        sd[q + "attention.gru_rel_pos_const"] = rng.uniform(0.5, 1.5, (1, H, 1, 1)).astype(np.float32)
        sd[q + "attention.gru_rel_pos_linear.weight"] = _uniform(rng, (8, D // H), 1.0 / math.sqrt(D // H))
        sd[q + "attention.gru_rel_pos_linear.bias"] = _uniform(rng, (8,), 1.0 / math.sqrt(D // H))
        for n in ("layer_norm", "final_layer_norm"):
            sd[q + n + ".weight"] = rng.uniform(0.8, 1.2, D).astype(np.float32)
            sd[q + n + ".bias"] = rng.uniform(-0.1, 0.1, D).astype(np.float32)
        sd[q + "feed_forward.intermediate_dense.weight"] = _uniform(rng, (F, D), b)
        sd[q + "feed_forward.intermediate_dense.bias"] = _uniform(rng, (F,), b)
        sd[q + "feed_forward.output_dense.weight"] = _uniform(rng, (D, F), 1.0 / math.sqrt(F))
        sd[q + "feed_forward.output_dense.bias"] = _uniform(rng, (D,), 1.0 / math.sqrt(F))
    sd["wav2vec_weights"] = rng.uniform(-1.0, 1.0, shape["num_layers"]).astype(np.float32)
    _head_state_dict(rng, sd, D, shape)
    return sd


def synthetic_speech(seconds: float, seed: int = 0, sample_rate: int = 16000, turns: int = 0) -> np.ndarray:
    """Speech-like float32 waveform in [-1, 1]: amplitude-modulated noise + harmonics; `turns` > 0 alternates between
    that many synthetic 'speakers' (different pitch / spectral tilt) every few seconds with short silences."""
    rng = np.random.default_rng(seed)
    n = int(seconds * sample_rate)
    t = np.arange(n) / sample_rate
    out = np.zeros(n, np.float32)
    nspk = max(turns, 1)
    seg = 0
    pos = 0
    while pos < n:
        dur = int(rng.uniform(1.5, 4.0) * sample_rate)
        end = min(n, pos + dur)
        spk = seg % nspk
        f0 = 100.0 + 45.0 * spk
        tt = t[pos:end]
        env = 0.5 * (1 + np.sin(2 * np.pi * (3.0 + spk) * tt))
        sig = sum(np.sin(2 * np.pi * f0 * h * tt) / h for h in (1, 2, 3, 4))
        noise = rng.normal(0, 0.3, end - pos)
        out[pos:end] = (0.12 * env * (sig + noise)).astype(np.float32)
        pos = end + int(rng.uniform(0.1, 0.5) * sample_rate)
        seg += 1
    return np.clip(out, -1, 1)


EMB_SHAPE = dict(sample_rate=16000, num_mel_bins=80, m_channels=32, embed_dim=256, blocks=(3, 4, 6, 3))


def embedding_state_dict(seed: int = 0, shape: Dict = EMB_SHAPE) -> Dict[str, np.ndarray]:
    """WeSpeaker ResNet34 weights: Kaiming-normal convolutions, BatchNorm statistics / affine terms away from the
    identity so that the folding is exercised."""
    rng = np.random.default_rng(seed)
    sd: Dict[str, np.ndarray] = {}

    def conv(name, cout, cin, k):
        std = math.sqrt(2.0 / (cin * k * k))
        sd[name] = rng.normal(0, std, (cout, cin, k, k)).astype(np.float32)

    def bn(name, c):
        sd[name + ".weight"] = rng.uniform(0.6, 1.2, c).astype(np.float32)
        sd[name + ".bias"] = rng.uniform(-0.1, 0.1, c).astype(np.float32)
        sd[name + ".running_mean"] = rng.uniform(-0.1, 0.1, c).astype(np.float32)
        sd[name + ".running_var"] = rng.uniform(0.6, 1.4, c).astype(np.float32)

    c0 = shape["m_channels"]
    conv("resnet.conv1.weight", c0, 1, 3)
    bn("resnet.bn1", c0)
    cin = c0
    for li, nb in enumerate(shape["blocks"]):
        cout = c0 << li
        for bi in range(nb):
            p = f"resnet.layer{li + 1}.{bi}"
            stride = 2 if (li > 0 and bi == 0) else 1
            conv(p + ".conv1.weight", cout, cin, 3)
            bn(p + ".bn1", cout)
            conv(p + ".conv2.weight", cout, cout, 3)
            bn(p + ".bn2", cout)
            sd[p + ".bn2.weight"] *= 0.5          # keeps the residual stream from growing over 16 blocks
            if stride != 1 or cin != cout:
                conv(p + ".shortcut.0.weight", cout, cin, 1)
                bn(p + ".shortcut.1", cout)
            cin = cout
    fq = shape["num_mel_bins"]
    for _ in range(3):
        fq = (fq - 1) // 2 + 1
    d = 2 * cin * fq
    bound = 1.0 / math.sqrt(d)
    sd["resnet.seg_1.weight"] = _uniform(rng, (shape["embed_dim"], d), bound)
    sd["resnet.seg_1.bias"] = _uniform(rng, (shape["embed_dim"],), bound)
    return sd
