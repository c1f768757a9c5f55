"""Import the LIVE reference (a revdotcom/reverb checkout, $RVB_REFERENCE_ROOT/asr) so it can serve as the parity
oracle's ground truth when the golden fixtures are (re)generated.

TEST INFRASTRUCTURE ONLY.  Nothing in the product path (reverb_b200/) may import
this module.  It only works where RVB_REFERENCE_ROOT points at a reference
checkout; the test suite uses the committed fixtures under tests/golden/.

Shims (SURVEY.md Appendix B):
  1. stub `whisper.tokenizer.LANGUAGES` (reference: asr/wenet/utils/common.py:23)
  2. re-export typing.Union/Optional into torch.nn.modules.conv
     (reference: asr/wenet/squeezeformer/conv2d.py:17, written for torch 2.2)
  3. replace torchaudio.load by a `wave` reader that returns int16-valued
     (C, N) tensors (reference: asr/wenet/cli/reverb.py:122, normalize=False)
"""
import os
import sys
import typing
import wave

import numpy as np
import torch

REFERENCE_ROOT = os.environ.get("RVB_REFERENCE_ROOT", "")
_HERE = os.path.dirname(os.path.abspath(__file__))


def available() -> bool:
    return os.path.isdir(os.path.join(REFERENCE_ROOT, "asr", "wenet"))


def _wave_load(path, normalize=False, **_kw):
    with wave.open(str(path), "rb") as w:
        assert w.getsampwidth() == 2, "only 16-bit PCM supported by the oracle loader"
        sr = w.getframerate()
        nch = w.getnchannels()
        pcm = np.frombuffer(w.readframes(w.getnframes()), dtype=np.int16)
    pcm = pcm.reshape(-1, nch).T.copy()
    t = torch.from_numpy(pcm)
    if normalize:
        t = t.to(torch.float32) / 32768.0
    return t, sr


def import_reference():
    """Returns the reference's `wenet` package (imported from asr)."""
    if not available():
        raise RuntimeError("reference tree not found: set RVB_REFERENCE_ROOT to a revdotcom/reverb checkout (now %r)"
                           % REFERENCE_ROOT)
    stub_dir = os.path.join(_HERE, "_stubs")
    ref_asr = os.path.join(REFERENCE_ROOT, "asr")
    # The repo root ships a drop-in `wenet` alias; make sure the reference wins here.
    for p in (ref_asr, stub_dir):
        if p in sys.path:
            sys.path.remove(p)
        sys.path.insert(0, p)
    for name in list(sys.modules):
        if name == "wenet" or name.startswith("wenet."):
            mod = sys.modules[name]
            f = getattr(mod, "__file__", "") or ""
            if not f.startswith(ref_asr):
                del sys.modules[name]
    import torch.nn.modules.conv as _c
    _c.Union = typing.Union
    _c.Optional = typing.Optional
    import torchaudio
    torchaudio.load = _wave_load
    import wenet  # noqa: E402
    assert wenet.__file__.startswith(ref_asr), wenet.__file__
    return wenet
