"""reverb-diarization-v2's WavLM segmentation network on the H100 (csrc/diar_wavlm.cu) against the stock-torch oracle
(oracle/wavlm_ref.py, itself pinned to torchaudio's wavlm_base by tests/test_wavlm_oracle.py), on seeded weights.

Errors are relative to the reference's largest magnitude; the bars are about twice the errors of the first H100 run
(DESIGN.md §7).  bf16 tensor-core operands against an fp32 reference.
"""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import wavlm_ref
from reverb_b200.diarization import synth
from reverb_b200.diarization.segmentation import WavLMSegmentationModel, segmentation_model

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def sd():
    return synth.wavlm_segmentation_state_dict(0)


@pytest.fixture(scope="module")
def model(sd):
    return WavLMSegmentationModel(sd)


@pytest.fixture(scope="module")
def ref(sd):
    return wavlm_ref.WavLMSegRef(sd)


def _rel(a, b):
    return float((a - b).abs().max() / b.abs().max())


@pytest.mark.parametrize("seconds,batch", [(2.0, 1), (4.0, 3), (10.0, 2)])
def test_stages_match_oracle(model, ref, seconds, batch):
    wav = torch.from_numpy(np.stack([synth.synthetic_speech(seconds, seed=40 + i, turns=2 + i) for i in range(batch)]))
    logp, conv, layers = model(wav.cuda(), return_intermediate=True)
    r_conv, r_layers, r_logp = ref(wav)
    e_conv = _rel(conv.cpu(), r_conv)
    e_layers = [_rel(layers[l].cpu(), r_layers[l]) for l in range(12)]
    e_logp = float((logp.cpu() - r_logp).abs().max())
    agree = float((logp.argmax(-1).cpu() == r_logp.argmax(-1)).float().mean())
    print(f"\n[wavlm {seconds}s x{batch}] conv {e_conv:.2e} layers max {max(e_layers):.2e} "
          f"({' '.join(f'{e:.1e}' for e in e_layers)}) logp abs {e_logp:.2e} argmax agree {agree:.4f}")
    assert e_conv < 1.5e-2
    assert max(e_layers) < 2e-2
    assert agree >= 0.96
    assert e_logp < 0.5


def test_window_is_batch_invariant(model):
    """alone, in a batch of 32, and in a batch of 40 (two passes of at most 32 windows)"""
    wav = torch.from_numpy(np.stack([synth.synthetic_speech(10.0, seed=60 + i, turns=3) for i in range(40)])).cuda()
    alone = model(wav[5:6].contiguous())
    assert torch.equal(alone[0], model(wav[:32].contiguous())[5])
    big = model(wav)
    assert torch.equal(alone[0], big[5])
    assert torch.equal(model(wav[35:36].contiguous())[0], big[35])


def test_frames_and_rejections(model, sd):
    assert model.num_frames(160000) == 499
    assert model.num_frames(399) == 0
    with pytest.raises(ValueError):
        model(torch.zeros(1, 399, device="cuda"))
    bad = dict(sd)
    bad["wav2vec.encoder.transformer.layers.0.attention.not_a_tensor"] = np.zeros(3, np.float32)
    with pytest.raises(RuntimeError, match="unknown tensor"):
        WavLMSegmentationModel(bad)
    short = dict(sd)
    short["wav2vec.encoder.feature_projection.projection.bias"] = np.zeros(5, np.float32)
    with pytest.raises(RuntimeError, match="elements"):
        WavLMSegmentationModel(short)
    missing = {k: v for k, v in sd.items() if k != "wav2vec_weights"}
    with pytest.raises(RuntimeError, match="not provided"):
        WavLMSegmentationModel(missing)


def test_weight_norm_legacy_names(model, sd):
    pc = "wav2vec.encoder.transformer.pos_conv_embed.conv."
    legacy = {k: v for k, v in sd.items() if "parametrizations" not in k}
    legacy[pc + "weight_g"] = sd[pc + "parametrizations.weight.original0"]
    legacy[pc + "weight_v"] = sd[pc + "parametrizations.weight.original1"]
    wav = torch.from_numpy(synth.synthetic_speech(3.0, seed=7)).view(1, -1).cuda()
    assert torch.equal(WavLMSegmentationModel(legacy)(wav), model(wav))


def test_dispatch(sd):
    assert isinstance(segmentation_model(sd), WavLMSegmentationModel)


def _three_speaker_wav(tmp_path):
    import wave
    pcm = (synth.synthetic_speech(40.0, seed=5, turns=3) * 32767).astype(np.int16)
    path = tmp_path / "three.wav"
    with wave.open(str(path), "wb") as w:
        w.setnchannels(1)
        w.setsampwidth(2)
        w.setframerate(16000)
        w.writeframes(pcm.tobytes())
    return str(path)


@pytest.fixture(scope="module")
def v2_dir(tmp_path_factory):
    """a pipeline directory as diarization.infer --pipeline-model reads it, with v2's segmentation checkpoint"""
    d = tmp_path_factory.mktemp("v2_pipeline")
    for name, sdict in (("segmentation.pt", synth.wavlm_segmentation_state_dict(0)),
                        ("embedding.pt", synth.embedding_state_dict(0))):
        torch.save({k: torch.from_numpy(v) for k, v in sdict.items()}, str(d / name))
    return str(d)


def test_infer_cli_v2_writes_rttm(tmp_path, v2_dir):
    wav = _three_speaker_wav(tmp_path)
    outs = {}
    for tag, flags in (("synthetic", ["--synthetic-v2"]), ("dir", ["--pipeline-model", v2_dir])):
        r = subprocess.run([sys.executable, "-m", "reverb_b200.diarization.infer", wav, "--out-dir", str(tmp_path / tag),
                            *flags], cwd=ROOT, capture_output=True, text=True, timeout=600)
        assert r.returncode == 0, r.stderr[-2000:]
        outs[tag] = (tmp_path / tag / "three.rttm").read_text()
    lines = outs["synthetic"].splitlines()
    assert lines and all(l.startswith("SPEAKER three 1 ") for l in lines)
    assert outs["dir"] == outs["synthetic"]          # the checkpoint directory loads the same v2 network


def test_recognize_wav_with_v2_model_dir_writes_stm_and_rttm(model_dirs, tmp_path, v2_dir):
    from reverb_b200 import recognize_wav
    from reverb_b200.diarization import infer
    wav = _three_speaker_wav(tmp_path)
    assert infer.main([wav, "--out-dir", str(tmp_path / "chain"), "--pipeline-model", v2_dir]) == 0
    out = tmp_path / "cli"
    recognize_wav.main(["--model", model_dirs["causal_ln"][0], "--audio_file", wav, "--result_dir", str(out),
                        "--modes", "ctc_prefix_beam_search", "--chunk_size", "300", "--batch_size", "4",
                        "--diarization_model", v2_dir])
    rttm = (out / "rttm" / "three.rttm").read_text()
    assert rttm == (tmp_path / "chain" / "three.rttm").read_text()
    from reverb_b200.diarization.words2speakers import stm_text
    ctm = (out / "ctc_prefix_beam_search" / "three.ctm").read_text()
    stm = (out / "ctc_prefix_beam_search" / "three.stm").read_text()
    assert stm and stm == stm_text("three", rttm, ctm)
