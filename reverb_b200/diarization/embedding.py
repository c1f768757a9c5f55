"""WeSpeaker ResNet34 speaker-embedding model on the GPU (csrc/diar_emb.cu through include/rvb_diar.h).

Mirror of what the reference obtains from `pyannote.audio` (`PyannoteAudioPretrainedSpeakerEmbedding.__call__(waveforms,
masks)` inside `SpeakerDiarization.get_embeddings`, behind diarization/infer_pyannote3.0.py:33-40).
** parity unpinned **: see include/rvb_diar.h.  No CPU fallback.
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, Optional

import numpy as np
import torch

from .. import _lib
from .synth import EMB_SHAPE


class EmbeddingModel:
    def __init__(self, state_dict: Dict[str, np.ndarray], shape: Dict = EMB_SHAPE, device: int = 0):
        if not torch.cuda.is_available():
            raise RuntimeError("reverb_b200.diarization needs a CUDA device (no CPU fallback)")
        self.lib = _lib.load()
        self.device = torch.device("cuda", device)
        self.shape = dict(shape)
        cfg = _lib.EmbConfig(sample_rate=shape["sample_rate"], num_mel_bins=shape["num_mel_bins"],
                             m_channels=shape["m_channels"], embed_dim=shape["embed_dim"],
                             blocks=(C.c_int * 4)(*shape["blocks"]))
        with torch.cuda.device(self.device):
            self.h = self.lib.rvb_emb_create(C.byref(cfg))
            if not self.h:
                raise RuntimeError(f"rvb_emb_create failed: {_lib.last_error()}")
            for name, arr in state_dict.items():
                if name.endswith("num_batches_tracked"):
                    continue
                a = np.ascontiguousarray(np.asarray(arr, np.float32))
                _lib.check(self.lib.rvb_emb_set_tensor(self.h, name.encode(), a.ctypes.data, a.size), "rvb_emb_set_tensor")
            _lib.check(self.lib.rvb_emb_finalize(self.h), "rvb_emb_finalize")

    def __del__(self):
        h, self.h = getattr(self, "h", None), None
        if h:
            self.lib.rvb_emb_destroy(h)

    @property
    def dimension(self) -> int:
        return int(self.shape["embed_dim"])

    def num_frames(self, num_samples: int) -> int:
        return int(self.lib.rvb_emb_num_frames(self.h, int(num_samples)))

    def forward(self, waveforms: torch.Tensor, weights: Optional[torch.Tensor] = None, return_fbank: bool = False):
        """waveforms (B, num_samples) fp32 CUDA in [-1, 1]; weights (B, S, Tw) fp32 CUDA or None
        -> (B, S, embed_dim) (S = 1 without weights)."""
        assert waveforms.is_cuda and waveforms.dtype == torch.float32 and waveforms.dim() == 2
        w = waveforms.contiguous()
        B, N = w.shape
        if weights is not None:
            assert weights.is_cuda and weights.dtype == torch.float32 and weights.dim() == 3 and weights.shape[0] == B
            weights = weights.contiguous()
            S, Tw = int(weights.shape[1]), int(weights.shape[2])
        else:
            S, Tw = 1, 0
        out = torch.empty(B, S, self.dimension, device=w.device, dtype=torch.float32)
        fb = torch.empty(B, self.num_frames(N), self.shape["num_mel_bins"], device=w.device) if return_fbank else None
        stream = torch.cuda.current_stream(w.device).cuda_stream
        with torch.cuda.device(w.device):
            _lib.check(self.lib.rvb_emb_forward(self.h, w.data_ptr(), B, N, weights.data_ptr() if weights is not None else None,
                                                S, Tw, out.data_ptr(), fb.data_ptr() if fb is not None else None, stream),
                       "rvb_emb_forward")
        return (out, fb) if return_fbank else out

    __call__ = forward
