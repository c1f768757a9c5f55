"""The model and length matrices of the float64 encoder tests (oracle/encoder_ref.py, tests/test_gpu_encoder_f64.py)
reach what they name, computed from shapes, and the float64 reference does not depend on padding."""
import os

import pytest
import torch

from conftest import ROOT
from oracle import encoder_ref as er
from reverb_b200 import corpus, synth


def _rows():
    """(model, feature lengths, batch T) of every batch the GPU tests compare with float64."""
    out = [(v, er.RAGGED, max(er.RAGGED)) for v in er.VARIANTS]
    out += [(er.BY_NAME[n], er.front_lens(T), T) for n in er.FRONT for T in er.FRONT_T]
    return out


def test_front_end_lengths():
    assert {er.conv1_frames(T) % 2 for T in er.FRONT_T} == {0, 1}
    assert {er.encoder_frames(T) for T in er.FRONT_T} >= {1, 2, 3, 15, 16, 127, 128, 129, 748}
    # the helpers agree with the product's own frame counts
    for T in er.FRONT_T + [max(er.RAGGED)]:
        assert er.encoder_frames(T) == corpus.encoder_out_frames(T)
        for n in er.front_lens(T) + er.RAGGED:
            assert er.valid_frames(n, T) == corpus.encoder_out_len(n, T)
    valid = [(v, er.valid_frames(n, T)) for v, lens, T in _rows() for n in lens if n <= T]
    assert any(e == 0 for _, e in valid), "no row without a valid encoder frame"
    assert any(e % 16 and e > 16 for _, e in valid), "every valid length is a multiple of the 16-frame tile"
    for causal in (True, False):
        assert any(0 < e < v.K for v, e in valid if v.causal == causal), f"no row with T' < K (causal={causal})"
    # rows of the front-end batches: full length, shorter, and below K or empty
    for n in er.FRONT:
        for T in er.FRONT_T:
            lens = er.front_lens(T)
            assert lens[0] == T and all(1 <= x <= T for x in lens)
            assert er.valid_frames(lens[2], T) < er.BY_NAME[n].K


def test_tail_lengths_are_planned_batch_lengths():
    """Two of the front-end lengths are what corpus.batch_frames picks for a recording's tail chunk at the default
    chunk of 2 998 frames: a 30.0 s + 5.15 s recording on the causal model, 30.0 s + 4.91 s on the symmetric one."""
    chunk = 2998
    causal, sym = er.BY_NAME[er.FRONT[0]], er.BY_NAME[er.FRONT[1]]
    assert causal.causal and not sym.causal
    for v, tail, want in ((causal, 515, 515), (sym, 491, 519)):
        right = corpus.right_context({"causal": v.causal, "cnn_module_kernel": v.K})
        batches = corpus.plan_window([chunk + tail], chunk, 4, right)
        assert [(b.T, b.lens) for b in batches] == [(chunk, [chunk]), (want, [tail])]
        assert want in er.FRONT_T


def test_every_conv_mid_path_runs():
    paths = {er.conv_mid_path(v, p) for v in er.VARIANTS for p in er.PRECISIONS}
    paths |= {er.conv_mid_path(er.BY_NAME[n], p, streaming=True) for n in er.STREAMING for p in er.PRECISIONS}
    fused = {er.conv_mid_path(er.BY_NAME[n], "bf16", fused=True) for n in er.FUSED}
    dw = {p[0] for p in paths}
    assert dw == {"conv_dw_kernel<15, false>", "conv_dw_kernel<31, false>", "conv_dw_kernel<7, false>",
                  "conv_dw_kernel<0, false>", "conv_dw_kernel<0, true>"}
    tails = {p[1] for p in paths}
    assert tails == {"batch_norm", "conv_norm_silu_kernel<8, false>", "conv_norm_silu_kernel<8, true>"}
    assert {p[0] for p in fused} == {"conv_dw_ln_fused_kernel<15>", "conv_dw_ln_fused_kernel<7>"}
    # the fused cases: causal and symmetric, both widths, both K
    fv = [er.BY_NAME[n] for n in er.FUSED]
    assert {v.causal for v in fv} == {True, False} and {v.d for v in fv} == {640, 1024} and {v.K for v in fv} == {7, 15}
    # the generic bf16 path from a K without a template, causal and with a halo (K - 1 = 32 frames) over twice the tile
    generic = [v for v in er.VARIANTS if er.conv_mid_path(v, "bf16")[0] == "conv_dw_kernel<0, false>"]
    assert any(v.causal for v in generic) and any(v.K - 1 > 2 * er.CM_TT - 1 for v in generic if not v.causal)
    # causal and symmetric models with each norm; both norms with a partly filled last channel slice
    for norm in ("layer_norm", "batch_norm"):
        assert {v.causal for v in er.VARIANTS if v.norm == norm} == {True, False}
        assert any(er.channel_slices(v.d)[1] < 128 for v in er.VARIANTS if v.norm == norm)
    assert er.channel_slices(640) == (3, 64) and er.channel_slices(1024) == (4, 128)
    # conv_norm_silu at d = 640: NV = 8 lanes' worth of float4 against nvec = 160, so the last pass is partly masked
    assert (640 // 4, er.conv_mid_path(er.BY_NAME["d640_causal_ln_k15"], "bf16")[1]) == (160, "conv_norm_silu_kernel<8, false>")


def test_conv_mid_dispatch_restated():
    """conv_mid_path restates launch_conv_mid; the conditions it relies on are still the ones in the source."""
    with open(os.path.join(ROOT, "reverb_b200", "csrc", "elementwise.cu")) as f:
        src = f.read()
    src = src[src.index("int launch_conv_mid("):]
    src = src[:src.index("\n}\n")]
    for line in ("if (fused_sel && use_ln && !x3 && conv_chunk <= 0 && (K == 15 || K == 7) && C2 <= 512)",
                 "if (x3) {", "RVB_DW(0, true);", "} else if (conv_chunk > 0) {", "RVB_DW(0, false);",
                 "} else if (K == 15) RVB_DW(15, false);", "else if (K == 31) RVB_DW(31, false);",
                 "else if (K == 7) RVB_DW(7, false);", "else RVB_DW(0, false);", "const int nv = (C / 4 + 31) / 32;",
                 "else if (nv <= 8) RVB_CNS(8);", "dim3 grid((T + CM_TT - 1) / CM_TT, B, (C2 + 127) / 128);"):
        assert line in src, line


def test_model_matrix_shapes(tmp_path):
    """A variant's model directory has the encoder it names."""
    from oracle.pipeline_ref import OracleASR
    v = er.BY_NAME["d640_sym_bn_k31"]
    sd, cfg = er.load_sd(v.write(str(tmp_path)))
    ec = cfg["encoder_conf"]
    assert (ec["output_size"], ec["attention_heads"], ec["linear_units"], ec["num_blocks"], ec["cnn_module_kernel"],
            ec["causal"], ec["cnn_module_norm"]) == (640, 10, 2560, 2, 31, False, "batch_norm")
    assert sd["encoder.encoders.1.conv_module.depthwise_conv.weight"].shape == (640, 1, 31)
    assert "encoder.encoders.1.language_layers.0.weight" in sd and "decoder.right_decoder.embed.0.weight" not in sd
    assert OracleASR(str(tmp_path)).vocab == er.VOCAB


@pytest.mark.parametrize("causal,norm,K", [(True, "layer_norm", 15), (True, "batch_norm", 31),
                                           (False, "batch_norm", 15), (False, "layer_norm", 31)])
def test_reference_ignores_padding(tmp_path, causal, norm, K):
    """Valid rows of the float64 reference are bit-identical whether padded feature frames hold zeros or +-1e3:
    valid encoder frame t reads feature frames up to 4 t + 6 <= feat_len - 1, and every later mixing of frames is
    masked.  The GPU poison test compares the kernels' valid rows on the same two inputs."""
    d = synth.write_model_dir(str(tmp_path), shape=dict(synth.TEST_SHAPE, blocks=2, kernel=K), seed=7, causal=causal,
                              cnn_module_norm=norm)
    sd, cfg = er.load_sd(d)
    T, lens = 303, [303, 211, 67, 10, 6]
    feats = er.features(len(lens), T, seed=3)
    zero, bad = er.zero_pad(feats, lens), er.poison(feats, lens)
    assert torch.equal(zero[0], bad[0]) and not torch.equal(zero[1], bad[1])
    a, la = er.encoder_f64(sd, cfg, zero, lens)
    b, lb = er.encoder_f64(sd, cfg, bad, lens)
    assert la == lb == [er.valid_frames(n, T) for n in lens] == [75, 52, 16, 1, 0]
    assert a.dtype == torch.float64
    for r, n in enumerate(la):
        assert torch.equal(a[r, :n], b[r, :n]), r
    assert not torch.equal(a[1], b[1])          # the padded rows themselves do see the poison
    err = er.frame_errors(b, a, la)
    assert err["rel"] == 0.0 and err["frames"] == sum(la)
