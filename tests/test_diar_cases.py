"""The shapes, inputs and readouts of tests/test_gpu_diar_f64.py reach what they claim, from shapes alone (no GPU):
the tile edges of the PyanNet, WavLM and ResNet kernels, the bucket near-tie and clamp of WavLM's relative position
bias, the pooling kernel's interpolation index, the exactness of the ResNet readout, and the weights the float64
references round to bf16 (oracle/diar_cases.py, oracle/diar_ref.py, oracle/wavlm_ref.py)."""
import math
import re

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import diar_cases as dc
from oracle import diar_ref, wavlm_ref
from reverb_b200.diarization import synth

SC_PT = dc.source_const("SC_PT", "diar_seg.cu")
CP_PT = dc.source_const("CP_PT", "diar_seg.cu")
LS_BT = dc.source_const("LS_BT", "diar_seg.cu")


def test_tile_constants_are_the_ones_the_matrix_was_built_for():
    assert (SC_PT, CP_PT, LS_BT) == (64, 32, 8)
    assert dc.source_const("WL_MAX_BATCH", "diar_wavlm.cu") == 32
    assert dc.ATT_KEY_TILE == 64


def test_pyannet_lengths_sit_on_the_tile_edges():
    """Each N is the fewest samples for its stage length: T = 1; L1 = one and one more sinc_conv_pool tile; T = one
    and one more, two and one more conv1d_pool tiles."""
    want = [("T", 1), ("L1", SC_PT), ("L1", SC_PT + 1), ("T", CP_PT), ("T", CP_PT + 1), ("T", 2 * CP_PT),
            ("T", 2 * CP_PT + 1)]
    assert tuple(dc.smallest_seg_n(stage, length) for stage, length in want) == dc.SEG_N
    for n, (stage, length) in zip(dc.SEG_N, want):
        assert dc.seg_lengths(n)[stage] == length and dc.seg_lengths(n - 1)[stage] == length - 1
        assert dc.seg_lengths(n)["T"] == diar_ref.seg_num_frames(n)
    assert dc.seg_lengths(dc.SEG_10S)["T"] == 589
    # batches: one window, one full LSTM cluster, one more, and the pipeline's 264 windows = 33 clusters
    assert dc.SEG_BATCHES == (1, LS_BT, LS_BT + 1, 33, 33 * LS_BT)


def test_wavlm_frames_reach_the_key_tiles_the_near_tie_and_the_clamp():
    tile = dc.ATT_KEY_TILE
    assert {tile - 1, tile, tile + 1, 2 * tile, 2 * tile + 1} <= set(dc.WAVLM_T)
    for t in dc.WAVLM_T:
        assert wavlm_ref.num_frames(dc.wavlm_samples(t)) == t
    assert wavlm_ref.num_frames(160000) == 499 and 499 in dc.WAVLM_T
    # distance 713: torch's float32 value 75.99997 is a few ulp below 76 and truncates to 75
    v = torch.log(torch.tensor([float(dc.NEAR_TIE)]) / 80) / math.log(800 / 80) * (160 - 80)
    assert 75.9999 < float(v) < 76.0 and float(v) + 5 * float(torch.finfo(torch.float32).eps) * 76 >= 76.0
    rel = torch.tensor([dc.NEAR_TIE, -dc.NEAR_TIE, dc.NEAR_TIE + 1])
    assert wavlm_ref.relative_positions_bucket(rel).tolist() == [160 + 155, 155, 160 + 156]
    assert max(dc.WAVLM_T) - 1 >= dc.CLAMP_FROM and dc.NEAR_TIE + 1 in dc.WAVLM_T
    # the largest window reaches clamped buckets, and the distances where a clamp at nb - 2 would differ
    d = torch.arange(max(dc.WAVLM_T))
    b = wavlm_ref.relative_positions_bucket(d)
    assert int(b.max()) == 160 + 159 and int((b == 160 + 159).sum()) > 50
    assert int(d[b == 160 + 159].min()) <= dc.CLAMP_FROM


def test_resnet_frames_cover_both_parities_at_each_stride_2_stage():
    seen = set()
    for t in dc.EMB_T:
        assert synth_frames(dc.emb_samples(t)) == t
        x = t
        for stage in range(3):
            seen.add((stage, x % 2))
            x = (x - 1) // 2 + 1
    assert seen == {(s, p) for s in range(3) for p in (0, 1)}
    assert [dc.emb_samples(t) for t in dc.EMB_T] == [1520, 1680, 1840, 2000]
    assert dc.emb_trunk_frames(synth_frames(dc.SEG_10S)) == 125


def synth_frames(n):
    return 1 + (n - 400) // 160


@pytest.mark.parametrize("tw,t", [(589, 125), (499, 125), (589, 1), (589, 2), (499, 1), (499, 2), (589, 6), (499, 3),
                                  (125, 125)])
def test_interpolation_index_is_torch_nearest(tw, t):
    src = torch.arange(tw, dtype=torch.float32).view(1, 1, -1)
    want = F.interpolate(src, size=t, mode="nearest").view(-1).long().numpy()
    assert np.array_equal(dc.interp_index(t, tw), want)


def test_readout_identities():
    assert np.float32(1.0) + np.float32(1e-8) == np.float32(1.0)
    assert np.array_equal(dc.interp_index(125, 125), np.arange(125))
    # one-hot weights: the kernel's fmaf chain returns the selected bf16 value exactly, and the identity seg_1 passes it
    rng = np.random.default_rng(0)
    x = torch.from_numpy(rng.normal(0, 30, 125).astype(np.float32)).bfloat16().float().numpy()
    for s in (0, 61, 124):
        w = np.zeros(125, np.float32)
        w[s] = 1.0
        m = np.float32(0.0)
        for t in range(125):
            m = np.float32(np.float64(w[t]) * np.float64(x[t]) + np.float64(m))   # fmaf: one rounding
        v1 = np.float32(w.sum()) + np.float32(1e-8)
        assert np.float32(m / v1) == x[s]
    sd = dc.readout_state_dict(synth.embedding_state_dict(0))
    assert sd["resnet.seg_1.weight"].shape == (dc.READOUT_DIM, dc.READOUT_DIM)
    stats = torch.randn(3, 125, dc.READOUT_DIM)
    trunk = dc.trunk_from_readout(stats)
    assert trunk.shape == (3, 256, 10, 125)
    assert float(trunk[1, 7, 3, 11]) == float(stats[1, 11, 7 * 10 + 3])


def _source(name):
    with open(f"{dc.CSRC}/{name}") as f:
        return f.read()


def test_resnet_stored_weights_round_what_finalize_rounds():
    sd = synth.embedding_state_dict(0)
    src = _source("diar_emb.cu")
    # finalize packs every block convolution through emb_conv (bf16) and keeps resnet.conv1 in fp32
    suffixes = set(re.findall(r'emb_conv\(m, p \+ "([^"]+)"', src))
    assert suffixes == {".conv1.weight", ".conv2.weight", ".shortcut.0.weight"}
    assert '"resnet.conv1.weight"' in src and "emb_conv(m, \"resnet.conv1" not in src
    names = diar_ref.resnet_stored_bf16(sd)
    assert set(names) == {k for k in sd if k.startswith("resnet.layer") and k.endswith(tuple(suffixes))}
    ref = diar_ref.ResNet34Ref(sd, stored_weights=True)
    for conv, _ in diar_ref.resnet_convs(sd):
        w = ref.folded[conv][0]
        assert torch.equal(w, diar_ref.bf16_round(w)) == (conv in names), conv
    # the fold is finalize's: fp32 scale = gamma / sqrt(var + 1e-5), rounded after the product
    p = "resnet.layer2.0"
    g, v = sd[p + ".bn1.weight"], sd[p + ".bn1.running_var"]
    scale = g / np.sqrt(v + np.float32(1e-5))
    want = torch.from_numpy(sd[p + ".conv1.weight"] * scale[:, None, None, None]).bfloat16().float()
    assert torch.equal(ref.folded[p + ".conv1.weight"][0], want)
    # without stored_weights the reference is the plain fp32 one
    assert diar_ref.ResNet34Ref(sd).folded is None


def test_wavlm_stored_weights_round_what_finalize_rounds():
    sd = synth.wavlm_segmentation_state_dict(0)
    src = _source("diar_wavlm.cu")
    suffixes = set(re.findall(r'up_bf16\(st, \w+ \+ "([^"]+)"', src))
    assert suffixes == {"projection.weight", "attention.attention.in_proj_weight", "attention.attention.out_proj.weight",
                        "feed_forward.intermediate_dense.weight", "feed_forward.output_dense.weight"}
    # the other two to_bf16_host calls: conv layers 1-6 (permuted) and the folded positional conv
    assert src.count("to_bf16_host(") == 4 and "to_bf16_host(perm.data()" in src and "to_bf16_host(w.data()" in src
    assert "for (int i = 1; i < WL_NCONV; ++i)" in src
    names = wavlm_ref.stored_bf16(sd)
    conv = {f"wav2vec.feature_extractor.conv_layers.{i}.conv.weight" for i in range(1, 7)}
    assert set(names) == conv | {k for k in sd if k.endswith(tuple(suffixes)) and "feature_extractor" not in k}
    assert len(names) == 6 + 1 + 4 * 12
    ref = wavlm_ref.WavLMSegRef(sd, stored_weights=True)
    plain = wavlm_ref.WavLMSegRef(sd)
    for k, v in sd.items():
        t = ref.t[k]
        if k in names:
            assert torch.equal(t, diar_ref.bf16_round(t)) and not torch.equal(t, plain.t[k]), k
        else:
            assert torch.equal(t, plain.t[k]), k
    # positional conv: weight norm folded in float64, cast to float32, then rounded
    pc = "wav2vec.encoder.transformer.pos_conv_embed.conv.parametrizations.weight."
    w = wavlm_ref.fold_weight_norm(torch.from_numpy(sd[pc + "original0"]).double(),
                                   torch.from_numpy(sd[pc + "original1"]).double()).float()
    assert torch.equal(ref.pos_w, w.bfloat16().float())


def test_oracles_run_in_float64_and_default_to_float32():
    sd = synth.segmentation_state_dict(0)
    wav = torch.from_numpy(synth.synthetic_speech(1.0, seed=1)).view(1, -1)
    r32, r64 = diar_ref.PyanNetRef(sd), diar_ref.PyanNetRef(sd, dtype=torch.float64)
    a, b = r32(wav), r64(wav.double())
    assert a.dtype == torch.float32 and b.dtype == torch.float64
    assert float((a.double() - b).abs().max()) < 1e-3
    assert torch.equal(r32.head(r32.sincnet(wav).transpose(1, 2)), a)


def test_fbank_float64_hamming_path():
    from oracle import fbank_np
    w = synth.synthetic_speech(1.0, seed=2) * np.float32(1 << 15)
    f64 = fbank_np.fbank(w, window="hamming", dtype=np.float64)
    assert f64.dtype == np.float64 and f64.shape == (98, 80)
    ref = diar_ref.wespeaker_fbank(torch.from_numpy(w / np.float32(1 << 15))).double().numpy()
    assert np.abs((f64 - f64.mean(axis=0)) - ref).max() < 1e-2
    assert fbank_np.fbank(w).dtype == np.float32
