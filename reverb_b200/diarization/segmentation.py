"""Segmentation models on the GPU through the C ABI of include/rvb_diar.h: PyanNet (reverb-diarization-v1,
csrc/diar_seg.cu) and WavLM / SSeRiouSS (reverb-diarization-v2, csrc/diar_wavlm.cu).

Mirror of what the reference obtains from `pyannote.audio` (`Model` called on (batch, channel, sample) windows inside
`SpeakerDiarization.get_segmentations`, behind diarization/infer_pyannote3.0.py:33-40), plus the
powerset -> multilabel conversion (`pyannote.audio.utils.powerset.Powerset.to_multilabel`).  ** parity unpinned **:
see include/rvb_diar.h.  No CPU fallback: construction fails without the CUDA library / a CUDA device.
"""
from __future__ import annotations

import ctypes as C
import itertools
from typing import Dict, Optional

import numpy as np
import torch

from .. import _lib
from .synth import SEG_SHAPE, WAVLM_CONV, WAVLM_SEG_SHAPE


def powerset_mapping(num_speakers: int = 3, max_set_size: int = 2) -> np.ndarray:
    """(num_powerset_classes, num_speakers) 0/1 matrix in pyannote's class order: the empty set, then all sets of size
    1, size 2, ... in `itertools.combinations` order."""
    rows = []
    for size in range(0, max_set_size + 1):
        for combo in itertools.combinations(range(num_speakers), size):
            r = np.zeros(num_speakers, np.float32)
            r[list(combo)] = 1.0
            rows.append(r)
    return np.stack(rows)


def powerset_to_multilabel(logp: torch.Tensor, mapping: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Hard conversion: arg-max powerset class per frame -> its speaker set.  (B, T, classes) -> (B, T, speakers)."""
    if mapping is None:
        mapping = torch.from_numpy(powerset_mapping()).to(logp.device)
    return mapping[logp.argmax(dim=-1)]


def _receptive_field(layers) -> tuple:
    """(size, step) in samples of a stack of unpadded (kernel, stride) layers: frame i covers [i * step, i * step + size)."""
    size, step = 1, 1
    for kernel, stride in reversed(layers):
        size = (size - 1) * stride + kernel
    for _, stride in layers:
        step *= stride
    return size, step


class SegmentationModel:
    # SincNet (k 251, stride 10), then MaxPool(3) / Conv(5) / MaxPool(3) / Conv(5) / MaxPool(3): 991 / 270 samples
    receptive_field = _receptive_field([(251, 10), (3, 3), (5, 1), (3, 3), (5, 1), (3, 3)])

    def __init__(self, state_dict: Dict[str, np.ndarray], shape: Dict = SEG_SHAPE, device: int = 0):
        if not torch.cuda.is_available():
            raise RuntimeError("reverb_b200.diarization needs a CUDA device (no CPU fallback)")
        self.lib = _lib.load()
        self.device = torch.device("cuda", device)
        self.shape = dict(shape)
        cfg = _lib.SegConfig(**{k: int(shape[k]) for k, _ in _lib.SegConfig._fields_})
        with torch.cuda.device(self.device):
            self.h = self.lib.rvb_seg_create(C.byref(cfg))
            if not self.h:
                raise RuntimeError(f"rvb_seg_create failed: {_lib.last_error()}")
            for name, arr in state_dict.items():
                a = np.ascontiguousarray(np.asarray(arr, np.float32))
                _lib.check(self.lib.rvb_seg_set_tensor(self.h, name.encode(), a.ctypes.data, a.size), "rvb_seg_set_tensor")
            _lib.check(self.lib.rvb_seg_finalize(self.h), "rvb_seg_finalize")

    def __del__(self):
        h, self.h = getattr(self, "h", None), None
        if h:
            self.lib.rvb_seg_destroy(h)

    def num_frames(self, num_samples: int) -> int:
        return int(self.lib.rvb_seg_num_frames(self.h, int(num_samples)))

    def forward(self, waveforms: torch.Tensor, return_sincnet: bool = False):
        """(B, num_samples) fp32 CUDA windows -> (B, frames, classes) log-probabilities."""
        assert waveforms.is_cuda and waveforms.dtype == torch.float32 and waveforms.dim() == 2
        w = waveforms.contiguous()
        B, N = w.shape
        T = self.num_frames(N)
        if T <= 0:
            raise ValueError(f"{N} samples are too few for one segmentation frame")
        out = torch.empty(B, T, self.shape["num_classes"], device=w.device, dtype=torch.float32)
        sinc = torch.empty(B, T, self.shape["conv_channels"], device=w.device, dtype=torch.float32) if return_sincnet else None
        stream = torch.cuda.current_stream(w.device).cuda_stream
        with torch.cuda.device(w.device):
            _lib.check(self.lib.rvb_seg_forward(self.h, w.data_ptr(), B, N, out.data_ptr(),
                                                sinc.data_ptr() if sinc is not None else None, stream), "rvb_seg_forward")
        return (out, sinc) if return_sincnet else out

    __call__ = forward


class WavLMSegmentationModel:
    """reverb-diarization-v2's segmentation network (pyannote `SSeRiouSS` on WavLM Base); same call as
    SegmentationModel.  `state_dict` under pyannote's names (`wav2vec.*`, `wav2vec_weights`, `lstm.*`, `linear.*`,
    `classifier.*`)."""
    receptive_field = _receptive_field(list(WAVLM_CONV))   # 400 / 320 samples

    def __init__(self, state_dict: Dict[str, np.ndarray], shape: Dict = WAVLM_SEG_SHAPE, device: int = 0):
        if not torch.cuda.is_available():
            raise RuntimeError("reverb_b200.diarization needs a CUDA device (no CPU fallback)")
        self.lib = _lib.load()
        self.device = torch.device("cuda", device)
        self.shape = dict(shape)
        cfg = _lib.WavlmSegConfig(**{k: int(shape[k]) for k, _ in _lib.WavlmSegConfig._fields_})
        with torch.cuda.device(self.device):
            self.h = self.lib.rvb_wavlm_seg_create(C.byref(cfg))
            if not self.h:
                raise RuntimeError(f"rvb_wavlm_seg_create failed: {_lib.last_error()}")
            for name, arr in state_dict.items():
                a = np.ascontiguousarray(np.asarray(arr, np.float32))
                _lib.check(self.lib.rvb_wavlm_seg_set_tensor(self.h, name.encode(), a.ctypes.data, a.size),
                           "rvb_wavlm_seg_set_tensor")
            _lib.check(self.lib.rvb_wavlm_seg_finalize(self.h), "rvb_wavlm_seg_finalize")

    def __del__(self):
        h, self.h = getattr(self, "h", None), None
        if h:
            self.lib.rvb_wavlm_seg_destroy(h)

    def num_frames(self, num_samples: int) -> int:
        return int(self.lib.rvb_wavlm_seg_num_frames(self.h, int(num_samples)))

    def forward(self, waveforms: torch.Tensor, return_intermediate: bool = False):
        """(B, num_samples) fp32 CUDA windows -> (B, frames, classes) log-probabilities; with return_intermediate also
        the conv extractor output (B, frames, 512) and the stacked layer outputs (layers, B, frames, 768)."""
        assert waveforms.is_cuda and waveforms.dtype == torch.float32 and waveforms.dim() == 2
        w = waveforms.contiguous()
        B, N = w.shape
        T = self.num_frames(N)
        if T <= 0:
            raise ValueError(f"{N} samples are too few for one segmentation frame")
        out = torch.empty(B, T, self.shape["num_classes"], device=w.device, dtype=torch.float32)
        conv = layers = None
        if return_intermediate:
            conv = torch.empty(B, T, self.shape["conv_channels"], device=w.device, dtype=torch.float32)
            layers = torch.empty(self.shape["num_layers"], B, T, self.shape["embed_dim"], device=w.device,
                                 dtype=torch.float32)
        stream = torch.cuda.current_stream(w.device).cuda_stream
        with torch.cuda.device(w.device):
            _lib.check(self.lib.rvb_wavlm_seg_forward(self.h, w.data_ptr(), B, N, out.data_ptr(),
                                                      conv.data_ptr() if conv is not None else None,
                                                      layers.data_ptr() if layers is not None else None, stream),
                       "rvb_wavlm_seg_forward")
        return (out, conv, layers) if return_intermediate else out

    __call__ = forward


def segmentation_model(state_dict: Dict[str, np.ndarray], device: int = 0):
    """The model a segmentation checkpoint holds: WavLM (v2) when its keys carry the `wav2vec.` prefix, else PyanNet."""
    if any(k.startswith("wav2vec.") for k in state_dict):
        return WavLMSegmentationModel(state_dict, device=device)
    return SegmentationModel(state_dict, device=device)
