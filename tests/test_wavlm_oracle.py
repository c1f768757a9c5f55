"""The WavLM segmentation oracle (oracle/wavlm_ref.py) against torchaudio's own wavlm_base() (no GPU).

torchaudio is the third-party pin of reverb-diarization-v2's WavLM part, as its kaldi.fbank pins the ASR front end.
The SSeRiouSS head after the layer sum is not pinned (pyannote's source and weights are absent offline).
"""
import numpy as np
import pytest
import torch

from oracle import wavlm_ref
from reverb_b200.diarization import synth
from reverb_b200.diarization.segmentation import SegmentationModel, WavLMSegmentationModel

torchaudio = pytest.importorskip("torchaudio", reason="torchaudio is not installed: the WavLM oracle cannot be pinned")


@pytest.fixture(scope="module")
def sd():
    return synth.wavlm_segmentation_state_dict(0)


def _torchaudio_model(sd):
    m = torchaudio.models.wavlm_base().eval()
    own = {k[len("wav2vec."):]: torch.from_numpy(v) for k, v in sd.items() if k.startswith("wav2vec.")}
    m.load_state_dict(own, strict=True)
    return m


def test_state_dict_matches_torchaudio_names_and_shapes(sd):
    ref = torchaudio.models.wavlm_base().state_dict()
    own = {k[len("wav2vec."):]: v for k, v in sd.items() if k.startswith("wav2vec.")}
    assert set(own) == set(ref)
    for k, v in ref.items():
        assert tuple(own[k].shape) == tuple(v.shape), k
    assert sd["wav2vec_weights"].shape == (12,)
    assert sd["lstm.weight_ih_l0"].shape == (512, 768)


@pytest.mark.parametrize("seconds", [1.0, 2.37])
def test_layers_match_torchaudio(sd, seconds):
    torch.manual_seed(0)
    wav = torch.from_numpy(np.stack([synth.synthetic_speech(seconds, seed=s, turns=2) for s in (1, 2)]))
    m = _torchaudio_model(sd)
    with torch.no_grad():
        feats, _ = m.feature_extractor(wav, None)
        want = m.extract_features(wav)[0]
    ref = wavlm_ref.WavLMSegRef(sd)
    got_feats = ref.conv_features(wav)
    assert torch.equal(got_feats, feats)
    got = ref.layers(got_feats)
    assert len(got) == len(want) == 12
    for l, (a, b) in enumerate(zip(got, want)):
        rel = float((a - b).abs().max() / b.abs().max())
        assert rel <= 1e-5, (l, rel)


def test_bucket_matches_torchaudio_past_max_distance():
    att = torchaudio.models.wavlm_base().encoder.transformer.layers[0].attention
    pos = torch.arange(1000)
    rel = pos[None, :] - pos[:, None]
    assert torch.equal(wavlm_ref.relative_positions_bucket(rel), att._relative_positions_bucket(rel, True))


def test_weight_norm_fold(sd):
    m = _torchaudio_model(sd)
    pc = "wav2vec.encoder.transformer.pos_conv_embed.conv.parametrizations.weight."
    w = wavlm_ref.fold_weight_norm(torch.from_numpy(sd[pc + "original0"]), torch.from_numpy(sd[pc + "original1"]))
    torch.testing.assert_close(w, m.encoder.transformer.pos_conv_embed.conv.weight.detach(), rtol=1e-6, atol=1e-7)


@pytest.mark.parametrize("n", [400, 719, 720, 32000, 64000, 160000])
def test_frames_and_receptive_field(n):
    m = torchaudio.models.wavlm_base().eval()
    with torch.no_grad():
        feats, _ = m.feature_extractor(torch.zeros(1, n), None)
    assert wavlm_ref.num_frames(n) == feats.shape[1]
    size, step = WavLMSegmentationModel.receptive_field
    assert (size, step) == (400, 320)
    assert (n - size) // step + 1 == feats.shape[1]
    assert wavlm_ref.num_frames(399) == 0
    assert wavlm_ref.num_frames(160000) == 499
    assert SegmentationModel.receptive_field == (991, 270)
