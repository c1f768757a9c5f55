"""The diarization networks on the GPU against float64 references, stage by stage and frame by frame.

References run on the GPU in torch float64 (oracle/diar_ref.py, oracle/wavlm_ref.py, oracle/fbank_np.py), once per
case.  Each stage is fed, where the network exposes it, the kernel's own output of the stage before, so a bound
measures that stage alone; bf16 networks run the reference on the weights the network stores (`stored_weights=True`),
so weight rounding is not part of the error.  Shapes and inputs come from oracle/diar_cases.py (tests/test_diar_cases.py
shows they reach the tile edges they claim).

* PyanNet (fp32): SincNet output against the float64 SincNet; log-probs against the float64 head on the kernel's SincNet
  output and end to end; arg-max equal wherever the float64 top-2 margin exceeds twice the bound.  10 s windows at
  B = 264 (33 LSTM clusters) and its first 1, 8, 9 and 33 windows (bit-equal), every tile-edge length, speech, the
  pipeline's zero-padded last window, silence, a DC offset under noise, near full scale.
* WavLM (bf16 GEMM operands): the conv extractor; layer 0 on `front` of the kernel's conv output; layer l >= 1 on the
  kernel's layer l - 1; the head on the kernel's 12 layers; end to end.  T = 1 ... 849, a 33-window call (the second
  32-window pass), and a probe of the relative-position bucket at distance 713.
* ResNet34 (bf16): the hamming fbank minus its time mean; the trunk, read out exactly through an identity `seg_1` and
  one-hot masks (oracle/diar_cases.py); the pooling against float64 pooling of the kernel's own trunk; `seg_1` against
  float64 on the kernel's statistics.

Errors: per frame ||got - ref|| / ||ref|| ("rel") and max |got - ref| ("abs"); `pytest -s` prints the worst frame of
every stage and case with its (window, frame).  Bounds are about 2x the worst value measured over every case on one
NVIDIA H100 80GB HBM3 (700 W power limit, max SM clock 1980 MHz):

  stage                                    measured rel / abs      bound rel / abs
  PyanNet SincNet                          5.46e-5 / 1.61e-4       1.1e-4 / 3.2e-4
  PyanNet head on the kernel's SincNet     1.22e-6 / 6.17e-6       2.5e-6 / 1.25e-5   (log-probs)
  PyanNet end to end                       3.71e-5 / 1.73e-4       7.5e-5 / 3.5e-4    (log-probs)
  WavLM conv extractor                     5.60e-3 / 2.21e-3       1.1e-2 / 4.5e-3
  WavLM front + layer 0                    2.49e-3 / 1.47e-2       5e-3 / 3e-2
  WavLM layers 1-11                        1.41e-3 / 7.03e-3       2.8e-3 / 1.4e-2
  WavLM head on the kernel's layers        3.73e-6 / 2.43e-5       7.5e-6 / 5e-5      (log-probs)
  WavLM end to end                         0.41 / 1.98             0.8 / 4.0          (log-probs, T = 849)
  ResNet fbank, bins >= 1e-3 of the frame  - / 8.95e-5             - / 1.8e-4         (74-75 % of the bins)
  ResNet fbank, the other bins             - / 3.01e-3             - / 6e-3
  ResNet trunk on the kernel's fbank       7.24e-3 / 11.4          1.5e-2 / 23
  pooling on the kernel's trunk            4.17e-7 / 1.69e-4       8.5e-7 / 3.4e-4
  seg_1 on the kernel's statistics         1.84e-6 / 3.37e-4       3.7e-6 / 7e-4

The fp32 PyanNet lands 11x below the 2e-3 bar of tests/test_gpu_diarization.py end to end.  The bf16 WavLM drifts
through 12 layers and a 4-layer LSTM end to end; the staged bounds are what pin its kernels.  The file runs in about
30 s.
"""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import diar_cases as dc
from oracle import diar_ref, fbank_np, wavlm_ref

pytestmark = pytest.mark.gpu

F64 = dict(dtype=torch.float64, device="cuda")

BOUNDS = {                      # (worst frame rel, largest abs difference)
    # PyanNet, fp32
    "seg.sinc": (1.1e-4, 3.2e-4),
    "seg.head": (2.5e-6, 1.25e-5),
    "seg.e2e": (7.5e-5, 3.5e-4),
    # WavLM, bf16 operands
    "wavlm.conv": (1.1e-2, 4.5e-3),
    "wavlm.layer0": (5e-3, 3e-2),
    "wavlm.layer": (2.8e-3, 1.4e-2),
    "wavlm.head": (7.5e-6, 5e-5),
    "wavlm.e2e": (0.8, 4.0),
    # ResNet34, bf16 operands
    "emb.fbank": (None, 1.8e-4),
    "emb.fbank_rest": (None, 6e-3),
    "emb.trunk": (1.5e-2, 23.0),
    "emb.pool": (8.5e-7, 3.4e-4),
    "emb.seg1": (3.7e-6, 7e-4),
}
FBANK_SHARE = 1e-3              # the tight fbank bound covers bins holding at least this share of their frame's energy


def _check(key, tag, got, ref, floor=1e-6):
    err = dc.frame_errors(got, ref, floor)
    rel, ab = BOUNDS[key]
    line = dc.describe(f"{key} {tag}", err) + f"  [bounds rel {rel:g}, abs {ab:g}]"
    print(line)
    assert err["rel"] <= rel and err["abs"] <= ab, line
    return err


# ================================================================================================= PyanNet (fp32)
@pytest.fixture(scope="module")
def seg():
    from reverb_b200.diarization import synth
    from reverb_b200.diarization.segmentation import SegmentationModel
    sd = synth.segmentation_state_dict(0)
    return SegmentationModel(sd), diar_ref.PyanNetRef(sd, **F64)


def _seg_compare(tag, model, ref, wav, got=None):
    """SincNet, head-on-kernel-SincNet and end-to-end checks of one batch; returns the kernel's log-probs."""
    logp, sinc = got if got is not None else model.forward(wav.cuda(), return_sincnet=True)
    ref_sinc = ref.sincnet(wav.to(**F64)).transpose(1, 2)
    _check("seg.sinc", tag, sinc, ref_sinc)
    head = ref.head(sinc.double())
    _check("seg.head", tag, logp, head)
    _check("seg.e2e", tag, logp, ref.head(ref_sinc))
    # arg-max equal wherever the reference's top-2 margin is clear of the bound
    top2 = head.topk(2, dim=-1).values
    clear = (top2[..., 0] - top2[..., 1]) > 2 * BOUNDS["seg.head"][1]
    same = logp.argmax(-1) == head.argmax(-1)
    print(f"seg.argmax {tag}: equal on {int(same[clear].sum())} of {int(clear.sum())} clear frames "
          f"({int(clear.numel())} frames)")
    assert bool(same[clear].all()), f"{tag}: arg-max differs at a clear frame"
    return logp


@pytest.fixture(scope="module")
def seg_264():
    kinds = [dc.SIGNALS[i % len(dc.SIGNALS)] for i in range(264)]
    wav = dc.batch(kinds, dc.SEG_10S, seed=1000)
    wav[263] = wav[8]
    return wav


def test_pyannet_264_windows_vs_f64(seg, seg_264):
    """The pipeline's largest call: 264 windows of every input family, 33 eight-window LSTM clusters."""
    model, ref = seg
    _seg_compare("10 s x 264", model, ref, seg_264)


def test_pyannet_window_is_batch_invariant(seg, seg_264):
    """The first 1, 8, 9 and 33 windows, and window 8 alone, are bit-equal to the same windows of the 264-batch, and
    so is window 263, which holds window 8's samples."""
    model, _ = seg
    wav = seg_264.cuda()
    big, big_sinc = model.forward(wav, return_sincnet=True)
    for b in dc.SEG_BATCHES[:-1]:
        part, part_sinc = model.forward(wav[:b].contiguous(), return_sincnet=True)
        assert torch.equal(part, big[:b]) and torch.equal(part_sinc, big_sinc[:b]), f"B = {b}"
    alone = model.forward(wav[8:9].contiguous())
    assert torch.equal(alone[0], big[8]) and torch.equal(alone[0], big[263])
    assert torch.equal(model.forward(wav), big), "two launches differ"


@pytest.mark.parametrize("n", dc.SEG_N)
def test_pyannet_tile_edges_vs_f64(seg, n):
    model, ref = seg
    kinds = ("speech", "padded", "dc", "loud", "silence")
    wav = dc.batch(kinds, n, seed=n)
    assert model.num_frames(n) == dc.seg_lengths(n)["T"]
    _seg_compare(f"N = {n} ({dc.seg_lengths(n)})", model, ref, wav)


# ================================================================================================ WavLM (bf16)
@pytest.fixture(scope="module")
def wavlm_sd():
    from reverb_b200.diarization import synth
    return synth.wavlm_segmentation_state_dict(0)


@pytest.fixture(scope="module")
def wavlm(wavlm_sd):
    from reverb_b200.diarization.segmentation import WavLMSegmentationModel
    return WavLMSegmentationModel(wavlm_sd), wavlm_ref.WavLMSegRef(wavlm_sd, stored_weights=True, **F64)


def _wavlm_staged(tag, ref, conv, layers, logp, idx=None):
    """Every stage of windows `idx` against the float64 reference fed with the kernel's previous stage."""
    if idx is not None:
        conv, layers, logp = conv[idx], layers[:, idx], logp[idx]
    x = ref.front(conv.double())
    for l in range(layers.shape[0]):
        _check("wavlm.layer0" if l == 0 else "wavlm.layer", f"{tag} layer {l}", layers[l], ref.layer(l, x))
        x = layers[l].double()
    head = ref.head([layers[l].double() for l in range(layers.shape[0])])
    _check("wavlm.head", tag, logp, head)
    return head


WAVLM_KINDS = ("speech", "padded", "silence", "dc")


@pytest.mark.parametrize("t", dc.WAVLM_T)
def test_wavlm_stages_vs_f64(wavlm, t):
    model, ref = wavlm
    n = dc.wavlm_samples(t)
    wav = dc.batch(WAVLM_KINDS, n, seed=2000 + t)
    logp, conv, layers = model(wav.cuda(), return_intermediate=True)
    tag = f"T = {t}"
    _check("wavlm.conv", tag, conv, ref.conv_features(wav.to(**F64)))
    _wavlm_staged(tag, ref, conv, layers, logp)
    e2e = ref(wav.to(**F64))[2]
    _check("wavlm.e2e", tag, logp, e2e)
    agree = float((logp.argmax(-1) == e2e.argmax(-1)).double().mean())
    print(f"wavlm.e2e {tag}: arg-max agreement {agree:.4f}")


def test_wavlm_second_pass_staged_outputs(wavlm):
    """33 windows: the staged outputs of the last window of the first 32-window pass and of the second pass."""
    model, ref = wavlm
    assert dc.source_const("WL_MAX_BATCH", "diar_wavlm.cu") == 32
    wav = dc.batch([WAVLM_KINDS[i % 4] for i in range(33)], dc.SEG_10S, seed=3000)
    logp, conv, layers = model(wav.cuda(), return_intermediate=True)
    idx = [31, 32]
    _check("wavlm.conv", "B = 33, windows 31 and 32", conv[idx], ref.conv_features(wav[idx].to(**F64)))
    _wavlm_staged("B = 33, windows 31 and 32", ref, conv, layers, logp, idx)
    alone, conv1, layers1 = model(wav[32:33].cuda(), return_intermediate=True)
    assert torch.equal(alone[0], logp[32]) and torch.equal(conv1[0], conv[32]) and torch.equal(layers1[:, 0], layers[:, 32])


def test_wavlm_bucket_at_distance_713(wavlm_sd):
    """torch's float32 bucket of distance 713 is 80 + 75 (value 75.99997); the next bucket starts at distance 714.  With
    the embedding rows of bucket 80 + 76 (both signs) raised by 12, a kernel that puts distance 713 in that bucket
    makes frames 0 and 713 of a T = 714 window attend to each other, far outside the layer bound; at T = 714 no pair of
    the reference reaches the raised rows."""
    from reverb_b200.diarization.segmentation import WavLMSegmentationModel
    sd = dict(wavlm_sd)
    key = "wav2vec.encoder.transformer.layers.0.attention.rel_attn_embed.weight"
    emb = sd[key].copy()
    emb[[156, 316]] += 12.0
    sd[key] = emb
    rel = torch.tensor([-dc.NEAR_TIE, dc.NEAR_TIE, -dc.NEAR_TIE - 1, dc.NEAR_TIE + 1])
    assert wavlm_ref.relative_positions_bucket(rel).tolist() == [155, 315, 156, 316]
    model, ref = WavLMSegmentationModel(sd), wavlm_ref.WavLMSegRef(sd, stored_weights=True, **F64)
    t = dc.NEAR_TIE + 1
    wav = dc.batch(("speech",), dc.wavlm_samples(t), seed=4000)
    _, conv, layers = model(wav.cuda(), return_intermediate=True)
    _check("wavlm.layer0", "distance-713 probe, layer 0", layers[0], ref.layer(0, ref.front(conv.double())))


# ============================================================================================== ResNet34 (bf16)
@pytest.fixture(scope="module")
def emb():
    from reverb_b200.diarization import synth
    from reverb_b200.diarization.embedding import EmbeddingModel
    sd = synth.embedding_state_dict(0)
    readout = EmbeddingModel(dc.readout_state_dict(sd), shape=dc.readout_shape(synth.EMB_SHAPE))
    return sd, EmbeddingModel(sd), readout, diar_ref.ResNet34Ref(sd, stored_weights=True, **F64)


def _fbank_f64(wav: torch.Tensor) -> torch.Tensor:
    """(B, N) -> (B, T, 80) float64 hamming fbank of wav * 2^15 minus its time mean, and (B, T, 80) each bin's share of
    its frame's mel energy."""
    out, share = [], []
    for w in wav.numpy():
        f = fbank_np.fbank(w * np.float32(1 << 15), window="hamming", dtype=np.float64)
        e = np.exp(f)
        share.append(e / e.sum(axis=1, keepdims=True))
        out.append(f - f.mean(axis=0, keepdims=True))
    return torch.from_numpy(np.stack(out)), torch.from_numpy(np.stack(share))


def _stats_pool_f64(seq: torch.Tensor, w) -> torch.Tensor:
    """diar_ref.stats_pool in float64, except that v1 = sum w + 1e-8 is formed in float32 as the network forms it: a
    single-frame mask gives v1 = 1 exactly and a zero std, where float64 would give a std of 6e-5 |x| from the 1e-8."""
    if w is None:
        return diar_ref.stats_pool(seq, None)
    w = F.interpolate(w[:, None].to(**F64), size=seq.shape[-1], mode="nearest")
    v1 = (w.sum(dim=-1).float() + 1e-8).double()
    mean = (seq * w).sum(dim=-1) / v1
    v2 = (w * w).sum(dim=-1)
    var = (((seq - mean.unsqueeze(-1)) ** 2) * w).sum(dim=-1) / (v1 - v2 / v1 + 1e-8)
    return torch.cat([mean, torch.sqrt(var)], dim=-1)


EMB_CASES = [(dc.SEG_10S, 32), (dc.SEG_10S, 33)] + [(dc.emb_samples(t), 5) for t in dc.EMB_T]


@pytest.mark.parametrize("n,b", EMB_CASES, ids=[f"N{n}xB{b}" for n, b in EMB_CASES])
def test_resnet_stages_vs_f64(emb, n, b):
    sd, prod, readout, ref = emb
    wav = dc.batch([dc.SIGNALS[i % len(dc.SIGNALS)] for i in range(b)], n, seed=5000 + b)
    tag = f"N = {n} x {b}"
    T = readout.num_frames(n)
    tp = dc.emb_trunk_frames(T)
    # fbank: the tight bound on bins with a fair share of their frame's energy, the other bound on the rest
    stats, fb = readout(wav.cuda(), dc.one_hot_masks(b, tp).cuda(), return_fbank=True)
    again = readout(wav.cuda(), dc.one_hot_masks(b, tp).cuda())
    assert torch.equal(stats, again), "two launches differ"
    ref_fb, share = _fbank_f64(wav)
    d = (fb.cpu().double() - ref_fb).abs()
    big = share >= FBANK_SHARE
    tight, rest = float(d[big].max()), float(d[~big].max()) if bool((~big).any()) else 0.0
    print(f"emb.fbank {tag}: max abs {tight:.3e} on {float(big.double().mean()):.4f} of the bins (share >= "
          f"{FBANK_SHARE:g}), {rest:.3e} on the rest  [bounds {BOUNDS['emb.fbank'][1]:g} / {BOUNDS['emb.fbank_rest'][1]:g}]")
    assert tight <= BOUNDS["emb.fbank"][1] and rest <= BOUNDS["emb.fbank_rest"][1]
    # trunk, frame by frame, on the kernel's fbank
    trunk = dc.trunk_from_readout(stats)                                   # (B, 256, 10, T')
    ref_trunk = ref.trunk(fb.double())
    _check("emb.trunk", tag, trunk.permute(0, 3, 1, 2), ref_trunk.permute(0, 3, 1, 2))
    # pooling on the kernel's own trunk: masks at both segmentation frame rates, and no masks.  With one trunk frame
    # the std is 0 / 0 in any float arithmetic (x - mean is a rounding error), so only the means are compared there.
    seq = trunk.double().reshape(b, -1, tp)
    half = slice(None) if tp > 1 else slice(0, dc.READOUT_DIM // 2)
    for tw in (589, 499):
        masks = dc.pool_masks(b, tw, seed=tw + b)
        got = readout(wav.cuda(), masks.cuda())
        want = torch.stack([_stats_pool_f64(seq, masks[:, s]) for s in range(3)], dim=1)
        _check("emb.pool", f"{tag}, Tw = {tw}", got[..., half], want[..., half])
        out = prod(wav.cuda(), masks.cuda())
        _check("emb.seg1", f"{tag}, Tw = {tw}", out,
               F.linear(got.double(), torch.from_numpy(sd["resnet.seg_1.weight"]).to(**F64),
                        torch.from_numpy(sd["resnet.seg_1.bias"]).to(**F64)))
    if tp > 1:                  # unweighted: pyannote's std(correction=1) needs two frames
        got = readout(wav.cuda())
        _check("emb.pool", f"{tag}, unweighted", got, _stats_pool_f64(seq, None)[:, None])
