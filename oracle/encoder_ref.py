"""Float64 reference of the Conformer encoder, and the models and lengths its tests run.

* `VARIANTS`: two-block encoders at the production width (d = 1024, plus three at d = 640) that between them reach every
  path of elementwise.cu `launch_conv_mid`: the register-halo depthwise conv for K = 15 / 31 / 7, the generic tap loop
  (K = 9, K = 33 whose halo is wider than the 16-frame tile, the accurate mode, the chunk-local streaming conv), the
  LayerNorm tail (`conv_norm_silu_kernel`) and the BatchNorm tail, causal and symmetric, and at d = 640 a last
  128-pair channel slice that is only partly filled.  `conv_mid_path` restates the dispatch, so that the CPU tests can
  check the matrix reaches every branch.
* `encoder_f64` / `chunk_by_chunk_f64`: `model_ref.encoder_forward` / `encoder_forward_chunk_by_chunk` on the state
  dict and the inputs cast to float64, on any torch device.
* `FRONT_T`, `RAGGED`, `front_lens`: batch lengths that reach both parities of the conv1 output, encoder lengths
  T' = 1, 2, 3, 15, 16, 127, 128, 129 and 748, rows with no valid encoder frame and valid lengths below K.
* `poison`: feature frames past each row's length set to +-1e3; `frame_errors`: the worst valid frame.
"""
from __future__ import annotations

import contextlib
import os
from dataclasses import dataclass
from typing import Dict, List, Sequence

import numpy as np
import torch

from . import fbank_np, model_ref

SEED = 11
VOCAB = 101
CAT = (0.25, 0.75)              # cat_embs: both language-specific layers contribute
CM_TT = 16                      # frames per depthwise-conv tile (elementwise.cu)


@dataclass(frozen=True)
class Variant:
    name: str
    d: int
    causal: bool
    norm: str                   # "layer_norm" | "batch_norm"
    K: int

    @property
    def layer_norm(self) -> bool:
        return self.norm == "layer_norm"

    def shape(self) -> Dict:
        """Two encoder blocks (the first and the last carry language-specific layers), heads of 64, ff = 4 d, and the
        smallest decoder the loader takes: one left block, no right decoder."""
        return dict(d=self.d, heads=self.d // 64, ff=4 * self.d, blocks=2, kernel=self.K, vocab=VOCAB, dec_ff=256,
                    dec_blocks=1, r_dec_blocks=0, emb_len=2)

    def write(self, path: str) -> str:
        from reverb_b200 import synth
        return synth.write_model_dir(path, shape=self.shape(), seed=SEED, causal=self.causal, cnn_module_norm=self.norm,
                                     reverse_weight=0.0)


VARIANTS = [
    Variant("causal_ln_k15", 1024, True, "layer_norm", 15),       # production
    Variant("sym_ln_k15", 1024, False, "layer_norm", 15),
    Variant("causal_bn_k15", 1024, True, "batch_norm", 15),
    Variant("sym_bn_k15", 1024, False, "batch_norm", 15),
    Variant("sym_ln_k31", 1024, False, "layer_norm", 31),
    Variant("causal_bn_k7", 1024, True, "batch_norm", 7),
    Variant("causal_ln_k9", 1024, True, "layer_norm", 9),          # generic tap loop
    Variant("sym_bn_k33", 1024, False, "batch_norm", 33),         # generic, halo wider than a tile
    Variant("causal_ln_k7", 1024, True, "layer_norm", 7),          # the fused kernel's K = 7
    Variant("d640_causal_ln_k15", 640, True, "layer_norm", 15),   # C / 2 = 320: last channel slice 64 of 128
    Variant("d640_sym_bn_k31", 640, False, "batch_norm", 31),
    Variant("d640_sym_ln_k7", 640, False, "layer_norm", 7),
]
BY_NAME = {v.name: v for v in VARIANTS}
PRECISIONS = ("bf16", "fp32")

# RVB_CONV_FUSED=1 cases: LayerNorm, bf16, K in {7, 15}, d in {640, 1024}, causal and symmetric
FUSED = ["causal_ln_k15", "sym_ln_k15", "causal_ln_k7", "d640_causal_ln_k15", "d640_sym_ln_k7"]
# simulate_streaming (chunk-local conv of a symmetric model) and its decoding chunk sizes
STREAMING = ["sym_ln_k15", "sym_ln_k31"]
STREAM_CHUNKS = (16, 37)
# the front end runs every length of FRONT_T on these
FRONT = ["causal_ln_k15", "sym_bn_k15"]

# one ragged batch at T = 3000: full length, odd length, T' = 717 (not a multiple of 16), T' = 128, T' = 1, no frame
RAGGED = [3000, 2999, 2871, 515, 10, 6]
# T = 7 ... 16: both conv1 parities and T' = 1, 2, 3; then T' = 15, 16, 127, 128, 129 and 748 with both parities
FRONT_T = list(range(7, 17)) + [63, 67, 511, 515, 519, 2998, 2999, 3000]


def conv1_frames(T: int) -> int:
    """Conv2dSubsampling4's first conv output frames T1 (kernel 3, stride 2)."""
    return (T - 1) // 2


def encoder_frames(T: int) -> int:
    t1 = conv1_frames(T)
    return 0 if t1 < 1 else (t1 - 1) // 2


def valid_frames(feat_len: int, T: int) -> int:
    """Valid encoder frames of a row of `feat_len` feature frames in a T-frame batch (the reference's mask)."""
    feat_len = min(feat_len, T)
    return min((feat_len - 3) // 4 if feat_len >= 7 else 0, encoder_frames(T))


def front_lens(T: int) -> List[int]:
    """Three rows for a T-frame batch: full length, a row a little over half as long, and one shorter than 7 frames
    (no valid encoder frame) or, for long batches, with T' below every K of the matrix."""
    return [T, max(1, T // 2 + 3), max(1, min(T - 5, 37))]


def conv_mid_path(v: Variant, precision: str, fused: bool = False, streaming: bool = False) -> tuple:
    """The kernels elementwise.cu `launch_conv_mid` runs for this model: (depthwise kernel, norm tail)."""
    x3 = precision == "fp32"
    C2 = v.d // 2
    conv_chunk = streaming and not v.causal
    if fused and v.layer_norm and not x3 and not conv_chunk and v.K in (15, 7) and C2 <= 512:
        return (f"conv_dw_ln_fused_kernel<{v.K}>", "fused")
    if x3:
        dw = "conv_dw_kernel<0, true>"
    elif conv_chunk or v.K not in (15, 31, 7):
        dw = "conv_dw_kernel<0, false>"
    else:
        dw = f"conv_dw_kernel<{v.K}, false>"
    if not v.layer_norm:
        return (dw, "batch_norm")
    nv = (v.d // 4 + 31) // 32
    NV = next(n for n in (1, 2, 4, 8, 16, 32) if nv <= n or n == 32)
    return (dw, f"conv_norm_silu_kernel<{NV}, {'true' if x3 else 'false'}>")


def channel_slices(d: int):
    """(slices, channel pairs in the last slice) of conv_dw_kernel's grid.z."""
    C2 = d // 2
    return (C2 + 127) // 128, C2 - 128 * ((C2 - 1) // 128)


# ------------------------------------------------------------------------------------------------------------------
def features(B: int, T: int, seed: int = 0) -> torch.Tensor:
    """(B, T, 80) float32 log-mel features of seeded speech-like audio (one recording per row)."""
    from reverb_b200 import synth
    secs = (T - 1) * 0.01 + 0.025 + 0.01
    rows = [fbank_np.fbank(synth.synth_audio(secs, seed=seed + b).astype(np.float32))[:T] for b in range(B)]
    assert all(r.shape[0] == T for r in rows)
    return torch.from_numpy(np.stack(rows))


def zero_pad(feats: torch.Tensor, lens: Sequence[int]) -> torch.Tensor:
    out = feats.clone()
    for b, n in enumerate(lens):
        out[b, n:] = 0.0
    return out


def poison(feats: torch.Tensor, lens: Sequence[int], value: float = 1e3, seed: int = 0) -> torch.Tensor:
    """The frames past each row's length set to +-value (random signs); valid frames unchanged."""
    g = torch.Generator().manual_seed(seed)
    out = feats.clone()
    sign = torch.randint(0, 2, feats.shape, generator=g).to(feats.dtype) * 2 - 1
    for b, n in enumerate(lens):
        out[b, n:] = value * sign[b, n:]
    return out


def load_sd(model_dir: str):
    import yaml
    with open(os.path.join(model_dir, "config.yaml")) as f:
        cfg = yaml.safe_load(f)
    sd = torch.load(os.path.join(model_dir, "synth.pt"))
    return {k: v for k, v in sd.items() if v.is_floating_point()}, cfg


@contextlib.contextmanager
def _float64_on(device):
    """model_ref builds masks and position tables with factory functions: make them float64 on `device`."""
    old = torch.get_default_dtype()
    torch.set_default_dtype(torch.float64)
    try:
        with torch.device(device):
            yield
    finally:
        torch.set_default_dtype(old)


def _sd64(sd, device):
    return {k: v.to(device=device, dtype=torch.float64) for k, v in sd.items() if k.startswith("encoder.")}


def encoder_f64(sd, cfg, feats: torch.Tensor, lens: Sequence[int], cat=CAT, device="cpu"):
    """model_ref.encoder_forward in float64 -> (out (B, T', d) float64 on the CPU, valid frames (B,) list)."""
    assert not model_ref.EMULATE_BF16
    with _float64_on(device):
        out, enc_lens, _ = model_ref.encoder_forward(
            feats.to(device=device, dtype=torch.float64), torch.as_tensor(list(lens), device=device), _sd64(sd, device),
            cfg, torch.tensor(cat, dtype=torch.float64, device=device))
    return out.cpu(), [int(x) for x in enc_lens.cpu()]


def chunk_by_chunk_f64(sd, cfg, feats: torch.Tensor, chunk: int, cat=CAT, device="cpu"):
    """model_ref.encoder_forward_chunk_by_chunk in float64: (1, T, 80) -> (1, T', d) float64 on the CPU."""
    with _float64_on(device):
        out = model_ref.encoder_forward_chunk_by_chunk(feats.to(device=device, dtype=torch.float64), _sd64(sd, device),
                                                       cfg, torch.tensor(cat, dtype=torch.float64, device=device), chunk)
    return out.cpu()


def frame_errors(got, ref, enc_lens: Sequence[int]) -> Dict:
    """Per valid frame: ||got - ref|| / ||ref|| and max |got - ref|; returns the worst of each and where it is."""
    got = torch.as_tensor(got).double().cpu()
    ref = torch.as_tensor(ref).double().cpu()
    assert got.shape == ref.shape, (got.shape, ref.shape)
    worst = {"rel": 0.0, "rel_at": None, "abs": 0.0, "abs_at": None, "frames": 0}
    for b, n in enumerate(enc_lens):
        if n == 0:
            continue
        diff = got[b, :n] - ref[b, :n]
        assert bool(torch.isfinite(got[b, :n]).all()), f"non-finite output in row {b}"
        rel = diff.norm(dim=-1) / ref[b, :n].norm(dim=-1)
        ab = diff.abs().amax(dim=-1)
        t = int(rel.argmax())
        if float(rel[t]) > worst["rel"]:
            worst["rel"], worst["rel_at"] = float(rel[t]), (b, t)
        t = int(ab.argmax())
        if float(ab[t]) > worst["abs"]:
            worst["abs"], worst["abs_at"] = float(ab[t]), (b, t)
        worst["frames"] += n
    return worst
