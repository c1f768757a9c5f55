"""`python -m reverb_b200.diarization.infer AUDIO... --out-dir DIR [--pipeline-model DIR | --synthetic]`

CLI mirror of diarization/infer_pyannote3.0.py:16-42 (positional audios, --out-dir, --pipeline-model,
--hf-access-token; output `<out-dir>/<basename>.rttm`).  Differences forced by the environment: there is no network, so
`--pipeline-model` names a LOCAL directory holding `segmentation.pt` and `embedding.pt` (torch state_dicts under
pyannote's key names, what `Model.from_pretrained(...).state_dict()` saves for the pipeline's two models) and the
HuggingFace token is accepted and ignored; `--synthetic` runs seeded random weights of v1, `--synthetic-v2` of v2
(benchmarks, smoke tests).
A segmentation checkpoint whose keys start with `wav2vec.` is reverb-diarization-v2's WavLM model, any other PyanNet
(v1).  Both use the pyannote 3.1 pipeline hyper-parameters (v2's own are not available offline).
"""
from __future__ import annotations

import argparse
import os
from pathlib import Path
from typing import Dict

import numpy as np
import torch

from . import synth
from .embedding import EmbeddingModel
from .pipeline import SpeakerDiarization
from .segmentation import segmentation_model


def _load_state_dict(path: str) -> Dict[str, np.ndarray]:
    sd = torch.load(path, map_location="cpu", weights_only=True)
    if isinstance(sd, dict) and "state_dict" in sd:
        sd = sd["state_dict"]
    return {k: v.float().numpy() for k, v in sd.items() if torch.is_tensor(v) and v.is_floating_point()}


def load_pipeline(model_dir: str = None, synthetic=False, device: int = 0, **kwargs) -> SpeakerDiarization:
    """synthetic: False (load `model_dir`), True or "v1" (seeded PyanNet weights), "v2" (seeded WavLM weights)."""
    if synthetic not in (False, None, True, "v1", "v2"):
        raise ValueError(f"synthetic must be 'v1' or 'v2', not {synthetic!r}")
    if synthetic:
        seg_sd = (synth.wavlm_segmentation_state_dict(0) if synthetic == "v2" else synth.segmentation_state_dict(0))
        emb_sd = synth.embedding_state_dict(0)
    else:
        if not model_dir or not os.path.isdir(model_dir):
            raise ValueError(f"pipeline model directory {model_dir!r} not found (no network: pass a local directory with "
                             "segmentation.pt and embedding.pt, or --synthetic)")
        seg_sd = _load_state_dict(os.path.join(model_dir, "segmentation.pt"))
        emb_sd = _load_state_dict(os.path.join(model_dir, "embedding.pt"))
    return SpeakerDiarization(segmentation_model(seg_sd, device=device), EmbeddingModel(emb_sd, device=device), **kwargs)


def read_audio(path: str) -> np.ndarray:
    """mono float32 in [-1, 1] at 16 kHz (pyannote's Audio(sample_rate=16000, mono="downmix"))"""
    from .. import _lib, audio_io
    from ..resample import resampled_length, sinc_resample_kernel
    wav, sr = audio_io.load_audio(path)                           # (channels, samples), int16-valued or float
    integer_pcm = np.issubdtype(np.asarray(wav).dtype, np.integer)
    x = np.asarray(wav, np.float32)
    if x.ndim == 2:
        x = x.mean(axis=0)
    if integer_pcm:
        x = x / 32768.0
    if sr != 16000:                                               # torchaudio.transforms.Resample semantics, on the GPU
        lib = _lib.load()
        kern, orig, new, width = sinc_resample_kernel(int(sr), 16000)
        t = torch.from_numpy(np.ascontiguousarray(x)).cuda()
        table = torch.from_numpy(kern).cuda()
        out = torch.empty(resampled_length(t.shape[0], orig, new), dtype=torch.float32, device="cuda")
        _lib.check(lib.rvb_resample(t.data_ptr(), 0, t.shape[0], table.data_ptr(), orig, new, width, out.data_ptr(),
                                    out.shape[0], torch.cuda.current_stream().cuda_stream), "rvb_resample")
        x = out.cpu().numpy()
    return x


def main(argv=None) -> int:
    ap = argparse.ArgumentParser(description="Run speaker diarization on audio files")
    ap.add_argument("audios", nargs="+")
    ap.add_argument("--out-dir", type=Path, required=True)
    ap.add_argument("--hf-access-token", type=str, default=None, help="accepted for CLI compatibility; unused offline")
    ap.add_argument("--pipeline-model", type=str, default=None, help="local directory with segmentation.pt / embedding.pt")
    syn = ap.add_mutually_exclusive_group()
    syn.add_argument("--synthetic", action="store_true", help="seeded random weights (no checkpoint available offline)")
    syn.add_argument("--synthetic-v2", action="store_true",
                     help="seeded random weights of reverb-diarization-v2 (WavLM segmentation)")
    args = ap.parse_args(argv)
    os.makedirs(args.out_dir, exist_ok=True)
    pipe = load_pipeline(args.pipeline_model, synthetic="v2" if args.synthetic_v2 else args.synthetic)
    for audio in args.audios:
        print("Processing", audio)
        turns = pipe(read_audio(audio))
        uri = os.path.splitext(os.path.basename(audio))[0]
        with open(args.out_dir / f"{uri}.rttm", "w") as f:
            pipe.write_rttm(f, uri, turns)
    return 0


if __name__ == "__main__":
    raise SystemExit(main())
