"""The Conformer encoder on the GPU against a float64 reference, frame by frame, at the production width.

Every model of oracle/encoder_ref.py's matrix (two blocks, d = 1024 and 640, causal / symmetric, LayerNorm /
BatchNorm, K = 7, 9, 15, 31, 33) runs in both precisions on a ragged batch; the production model and a symmetric one
run every front-end length; the symmetric LayerNorm models run simulate_streaming; the RVB_CONV_FUSED=1 kernel runs in
a subprocess.  Every valid encoder frame is compared with `model_ref.encoder_forward` in float64 (computed on the
GPU with torch's float64 operators, cached per module): ||got - ref|| / ||ref|| per frame, and the largest absolute
difference.  Padded frames of zero-padded inputs are compared too: the reference masks them the same way.  Inputs whose
padded feature frames hold +-1e3 must give valid frames bit-identical to the zero-padded run, and two launches the same
bytes.

Bounds are about 2x the worst frame measured on one H100 80GB HBM3 (700 W power limit, max SM clock 1980 MHz), over
every model, length and path here, valid and padded frames alike:
  bf16:  rel 4.35e-3 (d = 640, K = 15), abs 2.59e-2  ->  bounds 9e-3 / 5.5e-2
  fp32:  rel 2.44e-5, abs 1.88e-4                     ->  bounds 5e-5 / 4e-4
The spread between models, paths and lengths is small (bf16 rel 3.6e-3 ... 4.35e-3), so one bound per precision serves
all of them.  `pytest -s` prints the measured values.  The file runs in about 90 s.
"""
import os
import subprocess
import sys
import textwrap

import pytest
import torch

from conftest import ROOT
from oracle import encoder_ref as er

pytestmark = pytest.mark.gpu

# worst per-frame relative error ||got - ref|| / ||ref|| and largest absolute difference, valid and padded frames
REL = {"bf16": 9e-3, "fp32": 5e-5}
ABS = {"bf16": 5.5e-2, "fp32": 4e-4}


class _Models:
    """Model directories written on first use, float64 references cached per (model, batch)."""

    def __init__(self, root):
        self.root, self.dirs, self.sd, self.refs = root, {}, {}, {}

    def dir(self, name):
        if name not in self.dirs:
            self.dirs[name] = er.BY_NAME[name].write(str(self.root / name))
        return self.dirs[name]

    def ref(self, name, key, fn):
        if (name, key) not in self.refs:
            if name not in self.sd:
                self.sd[name] = er.load_sd(self.dir(name))
            self.refs[(name, key)] = fn(*self.sd[name])
        return self.refs[(name, key)]


@pytest.fixture(scope="module")
def models(tmp_path_factory):
    return _Models(tmp_path_factory.mktemp("enc_f64"))


@pytest.fixture(scope="module")
def ragged():
    lens = er.RAGGED
    feats = er.features(len(lens), max(lens), seed=100)
    return lens, er.zero_pad(feats, lens), er.poison(feats, lens, seed=1)


def _asr(model_dir, precision):
    import reverb_b200
    return reverb_b200.ReverbASR(os.path.join(model_dir, "config.yaml"), os.path.join(model_dir, "synth.pt"), gpu=0,
                                 precision=precision)


def _run(asr, feats, lens):
    enc, enc_lens = asr.model._forward_encoder(feats.cuda(), torch.tensor(lens, dtype=torch.int32),
                                               torch.tensor(er.CAT))
    torch.cuda.synchronize()
    return enc.cpu(), [int(x) for x in enc_lens]


def _check(tag, got, ref, enc_lens, precision, padded=True):
    """Valid frames (and, for zero-padded inputs, padded frames) within the bounds; prints the worst frames."""
    err = er.frame_errors(got, ref, enc_lens)
    line = f"{tag} {precision}: worst frame rel {err['rel']:.3e} at {err['rel_at']}, abs {err['abs']:.3e} at " \
           f"{err['abs_at']} ({err['frames']} frames)"
    ok = err["rel"] <= REL[precision] and err["abs"] <= ABS[precision]
    if padded and sum(got.shape[1] - n for n in enc_lens):
        pad = er.frame_errors(torch.cat([got[b, n:] for b, n in enumerate(enc_lens)])[None],
                              torch.cat([ref[b, n:] for b, n in enumerate(enc_lens)])[None],
                              [sum(got.shape[1] - n for n in enc_lens)])
        line += f"; padded frames rel {pad['rel']:.3e}, abs {pad['abs']:.3e} ({pad['frames']})"
        ok = ok and pad["rel"] <= REL[precision] and pad["abs"] <= ABS[precision]
    print(line)
    assert ok, line
    return err


def _bit_equal_valid(a, b, enc_lens):
    for r, n in enumerate(enc_lens):
        assert torch.equal(a[r, :n], b[r, :n]), f"row {r}: valid frames depend on the padded feature frames"


@pytest.mark.parametrize("name", [v.name for v in er.VARIANTS])
def test_variant_ragged_batch_vs_f64(models, ragged, name):
    """One ragged T = 3000 batch (T' = 748, 748, 717, 128, 1, 0) per model and precision; the poisoned rerun gives the
    same valid bytes, and so does a second launch."""
    lens, zero, bad = ragged
    ref, ref_lens = models.ref(name, "ragged", lambda sd, cfg: er.encoder_f64(sd, cfg, zero, lens, device="cuda"))
    for precision in er.PRECISIONS:
        asr = _asr(models.dir(name), precision)
        got, enc_lens = _run(asr, zero, lens)
        assert enc_lens == ref_lens
        _check(name, got, ref, enc_lens, precision)
        again, _ = _run(asr, zero, lens)
        assert torch.equal(got, again), "two launches differ"
        poisoned, _ = _run(asr, bad, lens)
        _bit_equal_valid(got, poisoned, enc_lens)
        del asr


@pytest.mark.parametrize("name", er.FRONT)
def test_front_end_lengths_vs_f64(models, name):
    """Every front-end length (T = 7 ... 16, 63, 67, 511, 515, 519, 2998 - 3000) at B = 3 with ragged rows."""
    asrs = {p: _asr(models.dir(name), p) for p in er.PRECISIONS}
    for T in er.FRONT_T:
        lens = er.front_lens(T)
        feats = er.features(len(lens), T, seed=200 + T)
        zero, bad = er.zero_pad(feats, lens), er.poison(feats, lens, seed=T)
        ref, ref_lens = models.ref(name, ("front", T), lambda sd, cfg: er.encoder_f64(sd, cfg, zero, lens, device="cuda"))
        for precision, asr in asrs.items():
            got, enc_lens = _run(asr, zero, lens)
            assert enc_lens == ref_lens and got.shape[1] == er.encoder_frames(T)
            _check(f"{name} T={T} lens={lens}", got, ref, enc_lens, precision)
            poisoned, _ = _run(asr, bad, lens)
            _bit_equal_valid(got, poisoned, enc_lens)


@pytest.mark.parametrize("name", er.STREAMING)
def test_streaming_chunk_local_conv_vs_f64(models, name):
    """simulate_streaming of a symmetric model (the chunk-local depthwise conv) against the cache-based float64
    chunk-by-chunk pass, for two decoding chunk sizes."""
    T = 3000
    feats = er.features(1, T, seed=300)
    asrs = {p: _asr(models.dir(name), p) for p in er.PRECISIONS}
    for chunk in er.STREAM_CHUNKS:
        ref = models.ref(name, ("stream", chunk), lambda sd, cfg: er.chunk_by_chunk_f64(sd, cfg, feats, chunk, device="cuda"))
        for precision, asr in asrs.items():
            enc, _ = asr.model._forward_encoder(feats.cuda(), torch.tensor([T], dtype=torch.int32),
                                                torch.tensor(er.CAT), decoding_chunk_size=chunk, simulate_streaming=True)
            got = enc.cpu()
            assert got.shape == ref.shape
            _check(f"{name} streaming chunk={chunk}", got, ref, [got.shape[1]], precision, padded=False)


_FUSED_SCRIPT = """
import os, sys, torch
sys.path.insert(0, {root!r})
from oracle import encoder_ref as er
import reverb_b200
lens = er.RAGGED
zero = er.zero_pad(er.features(len(lens), max(lens), seed=100), lens)
for name, d in {dirs!r}.items():
    asr = reverb_b200.ReverbASR(os.path.join(d, "config.yaml"), os.path.join(d, "synth.pt"), gpu=0, precision="bf16")
    outs = []
    for _ in range(2):
        enc, enc_lens = asr.model._forward_encoder(zero.cuda(), torch.tensor(lens, dtype=torch.int32), torch.tensor(er.CAT))
        outs.append(enc.cpu())
    torch.save({{"enc": outs, "lens": [int(x) for x in enc_lens]}}, os.path.join({out!r}, name + ".pt"))
    del asr
"""


def test_fused_conv_kernel_vs_f64(models, ragged, tmp_path):
    """RVB_CONV_FUSED=1 (conv_dw_ln_fused_kernel, read once per process): LayerNorm models, bf16, K = 7 and 15,
    d = 640 and 1024, causal and symmetric, in a subprocess; compared with the same float64 references."""
    lens, zero, _ = ragged
    dirs = {n: models.dir(n) for n in er.FUSED}
    script = tmp_path / "fused.py"
    script.write_text(textwrap.dedent(_FUSED_SCRIPT.format(root=ROOT, dirs=dirs, out=str(tmp_path))))
    env = dict(os.environ, RVB_CONV_FUSED="1")
    r = subprocess.run([sys.executable] + (["-s"] if sys.flags.no_user_site else []) + [str(script)], env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    for n in er.FUSED:
        out = torch.load(tmp_path / (n + ".pt"))
        ref, ref_lens = models.ref(n, "ragged", lambda sd, cfg: er.encoder_f64(sd, cfg, zero, lens, device="cuda"))
        assert out["lens"] == ref_lens
        assert torch.equal(out["enc"][0], out["enc"][1]), "two launches differ"
        default, _ = _run(_asr(models.dir(n), "bf16"), zero, lens)
        assert not torch.equal(default, out["enc"][0]), "the subprocess did not run the fused kernel"
        _check(f"{n} RVB_CONV_FUSED=1", out["enc"][0], ref, ref_lens, "bf16")
