"""Shapes, inputs and readouts of the float64 tests of the diarization networks (tests/test_gpu_diar_f64.py).

* Tile constants read from the CUDA sources (`source_const`): `SC_PT` pooled positions per `sinc_conv_pool_kernel`
  CTA, `CP_PT` per `conv1d_pool_kernel` CTA, `LS_BT` windows per LSTM cluster, `WL_MAX_BATCH` windows per WavLM pass.
* `SEG_N`: PyanNet window lengths whose stage lengths sit on both sides of those tiles (`seg_lengths`); `WAVLM_T`:
  WavLM frame counts around the 64-key attention tile, plus T = 714 (distance 713, where torch's float32 bucket value
  is 4 ulp below a truncation boundary) and T = 849 (distances >= 800, the clamped buckets); `EMB_T`: ResNet frame
  counts of both parities at each stride-2 stage.
* `signal`: speech, silence, a DC offset under low-level noise, near full scale, and the pipeline's zero-padded last
  window (`padded_last_window`, cut by `SpeakerDiarization.windows`).
* The ResNet readout: `readout_state_dict` replaces `resnet.seg_1` by the 5120 x 5120 identity with zero bias, so the
  network's fp32 output is its pooled statistics, exactly (every product of the GEMM is x * 1 or x * 0).  With the
  S = T' one-hot masks of `one_hot_masks` (Tw = T': source index t, v1 = 1 + 1e-8f == 1.0f), row s of the mean half is
  the trunk's bf16 activation at frame s; `trunk_from_readout` reshapes it to (B, 256, 10, T').
* `interp_index`: the pooling kernel's float formula for the nearest-interpolation source index.
* `frame_errors`: the worst frame of a comparison and where it is.
"""
from __future__ import annotations

import os
import re
from typing import Dict

import numpy as np
import torch

from . import wavlm_ref

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "reverb_b200", "csrc")


def source_const(name: str, file: str) -> int:
    """The integer value of `constexpr int ... name = value` in csrc/<file>."""
    with open(os.path.join(CSRC, file)) as f:
        m = re.search(r"constexpr int [^;]*\b" + name + r"\s*=\s*(\d+)", f.read())
    assert m, f"{name} not found in {file}"
    return int(m.group(1))


ATT_KEY_TILE = source_const("AT_BN", "attention_tc.cu")   # keys per tile of attention_tc_kernel

# ------------------------------------------------------------------------------------------------------------ PyanNet


def seg_lengths(n: int) -> Dict[str, int]:
    """Stage lengths of PyanNet on n samples: `L1` pooled SincNet positions (sinc_conv_pool_kernel tiles), `L2` pooled
    positions of the first k = 5 conv and `T` of the second (conv1d_pool_kernel tiles; T = output frames)."""
    l1 = ((n - 251) // 10 + 1) // 3 if n >= 251 else 0
    l2 = max(l1 - 4, 0) // 3
    t = max(l2 - 4, 0) // 3
    return {"L1": l1, "L2": l2, "T": t}


def smallest_seg_n(stage: str, length: int) -> int:
    """The fewest samples whose `stage` length is `length`."""
    n = 251
    while seg_lengths(n)[stage] < length:
        n += 1
    return n


# T = 1; L1 = 64 / 65 (one full sinc tile, one more); T = 32 / 33 and 64 / 65 (conv1d_pool tiles of the second conv)
SEG_N = (991, 2161, 2191, 9361, 9631, 18001, 18271)
SEG_10S = 160000
SEG_BATCHES = (1, 8, 9, 33, 264)   # 264 windows: the pipeline's largest call, 33 clusters of the LSTM

# ---------------------------------------------------------------------------------------------------------------- WavLM
WAVLM_T = (1, 63, 64, 65, 128, 129, 499, 714, 849)
NEAR_TIE = 713                  # torch: log(713 / 80) / log(10) * 80 = 75.99997 in float32 -> bucket 80 + 75
CLAMP_FROM = 800                # max_distance: every distance from here on is clamped to bucket nb - 1


def wavlm_samples(t: int) -> int:
    """The fewest samples that give t WavLM frames."""
    n = 400 + 320 * (t - 1)
    assert wavlm_ref.num_frames(n) == t and wavlm_ref.num_frames(n - 1) == t - 1
    return n


# ------------------------------------------------------------------------------------------------------------- ResNet34
EMB_T = (8, 9, 10, 11)          # fbank frames: both parities at each of the three stride-2 stages


def emb_samples(t: int) -> int:
    return 400 + 160 * (t - 1)


def emb_trunk_frames(t: int) -> int:
    for _ in range(3):
        t = (t - 1) // 2 + 1
    return t


READOUT_DIM = 2 * 256 * 10      # [mean | std] over 256 channels x 10 frequencies


def readout_state_dict(sd: Dict[str, np.ndarray]) -> Dict[str, np.ndarray]:
    out = dict(sd)
    out["resnet.seg_1.weight"] = np.eye(READOUT_DIM, dtype=np.float32)
    out["resnet.seg_1.bias"] = np.zeros(READOUT_DIM, np.float32)
    return out


def readout_shape(shape: Dict) -> Dict:
    return dict(shape, embed_dim=READOUT_DIM)


def one_hot_masks(batch: int, tp: int) -> torch.Tensor:
    """(B, T', T') weights: row s selects trunk frame s."""
    return torch.eye(tp, dtype=torch.float32).expand(batch, tp, tp).contiguous()


def trunk_from_readout(stats: torch.Tensor) -> torch.Tensor:
    """(B, T', 5120) statistics of the one-hot masks -> (B, 256, 10, T') trunk output (feature j = c * 10 + f)."""
    B, tp, _ = stats.shape
    return stats[..., :READOUT_DIM // 2].reshape(B, tp, 256, 10).permute(0, 2, 3, 1)


def interp_index(t_out: int, t_in: int) -> np.ndarray:
    """stats_pool_kernel's source index of each of t_out frames: min(floor(t * (float(Tw) / float(T))), Tw - 1) in
    float32."""
    t = np.arange(t_out, dtype=np.float32)
    return np.minimum(np.floor(t * (np.float32(t_in) / np.float32(t_out))).astype(np.int64), t_in - 1)


def pool_masks(batch: int, tw: int, seed: int) -> torch.Tensor:
    """(B, 3, Tw) weights: a positive random ramp, then per window one of all-zero, all-ones and a single frame, then
    another ramp."""
    rng = np.random.default_rng(seed)
    m = np.zeros((batch, 3, tw), np.float32)
    x = np.linspace(0.0, 1.0, tw, dtype=np.float32)
    for b in range(batch):
        m[b, 0] = rng.uniform(0.05, 0.3) + rng.uniform(0.2, 1.0) * x + rng.uniform(0.0, 0.1, tw)
        kind = b % 3
        if kind == 1:
            m[b, 1] = 1.0
        elif kind == 2:
            m[b, 1, rng.integers(0, tw)] = 1.0
        m[b, 2] = rng.uniform(0.05, 0.3) + rng.uniform(0.2, 1.0) * x[::-1] + rng.uniform(0.0, 0.1, tw)
    return torch.from_numpy(m)


# ------------------------------------------------------------------------------------------------------------- inputs
def padded_last_window(seconds: float = 23.7, seed: int = 80) -> np.ndarray:
    """The zero-padded last 10 s window the pipeline cuts from a recording of `seconds`."""
    from reverb_b200.diarization import synth
    from reverb_b200.diarization.pipeline import SpeakerDiarization
    audio = torch.from_numpy(synth.synthetic_speech(seconds, seed=seed, turns=2))
    w = SpeakerDiarization(None, None, device="cpu").windows(audio)[-1]
    assert float(w[-1600:].abs().max()) == 0.0
    return w.numpy().copy()


SIGNALS = ("speech", "padded", "silence", "dc", "loud")


def signal(kind: str, n: int, seed: int) -> np.ndarray:
    """(n,) float32 window of one input family."""
    from reverb_b200.diarization import synth
    rng = np.random.default_rng(seed)
    if kind == "speech":
        s = synth.synthetic_speech(n / 16000 + 1.0, seed=seed, turns=2 + seed % 2)
        off = int(rng.integers(0, 16000))
        return s[off:off + n].astype(np.float32)
    if kind == "padded":        # the pipeline's last window; other lengths: its first n samples, the last third zeroed
        w = padded_last_window(seed=seed)
        if n > w.shape[0]:
            return np.pad(w, (0, n - w.shape[0]))
        if n < w.shape[0]:
            w = w[:n].copy()
            w[n - n // 3:] = 0.0
        return w
    if kind == "silence":
        return np.zeros(n, np.float32)
    if kind == "dc":
        return (0.3 + rng.normal(0, 1e-3, n)).astype(np.float32)
    if kind == "loud":
        s = synth.synthetic_speech(n / 16000 + 0.5, seed=seed, turns=2)[:n]
        return (0.99 * s / np.abs(s).max()).astype(np.float32)
    raise ValueError(kind)


def batch(kinds, n: int, seed: int) -> torch.Tensor:
    return torch.from_numpy(np.stack([signal(k, n, seed + i) for i, k in enumerate(kinds)]))


# ---------------------------------------------------------------------------------------------------------- reporting
def frame_errors(got: torch.Tensor, ref: torch.Tensor, floor: float = 1e-6) -> Dict:
    """got, ref (B, T, ...): per frame ||got - ref|| / max(||ref||, floor) and max |got - ref|; the worst of each and its
    (window, frame)."""
    got = torch.as_tensor(got).double().cpu()
    ref = torch.as_tensor(ref).double().cpu()
    assert got.shape == ref.shape, (got.shape, ref.shape)
    assert bool(torch.isfinite(got).all()), "non-finite output"
    B, T = got.shape[:2]
    diff = (got - ref).reshape(B, T, -1)
    rel = diff.norm(dim=-1) / ref.reshape(B, T, -1).norm(dim=-1).clamp_min(floor)
    ab = diff.abs().amax(dim=-1)
    r, a = int(rel.argmax()), int(ab.argmax())
    return {"rel": float(rel.flatten()[r]), "rel_at": divmod(r, T), "abs": float(ab.flatten()[a]),
            "abs_at": divmod(a, T), "frames": B * T}


def describe(tag: str, err: Dict) -> str:
    return (f"{tag}: worst frame rel {err['rel']:.3e} at {err['rel_at']}, abs {err['abs']:.3e} at {err['abs_at']} "
            f"({err['frames']} frames)")
