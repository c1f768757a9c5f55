"""Pins the oracle and the synthetic-model generator to the reference's own results, recorded from the live reference
by oracle/make_golden_pins.py into tests/golden/pins.{json,npz} and pins_conv.{json,npz}.  Encoder outputs are pinned by a seeded sample of
elements and the float64 sums of the whole tensor; both must match exactly."""
import json
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN


@pytest.fixture(scope="module")
def pins():
    with open(os.path.join(GOLDEN, "pins.json")) as f:
        meta = json.load(f)
    return meta, dict(np.load(os.path.join(GOLDEN, "pins.npz")))


def _assert_tensor_pinned(t, arrays, key, rec):
    a = t.detach().cpu().numpy().astype(np.float32)
    assert list(a.shape) == rec["enc_shape"]
    flat = a.reshape(-1)
    assert np.array_equal(flat[arrays[key + "_idx"]], arrays[key + "_val"])
    a64 = flat.astype(np.float64)
    assert float(a64.sum()) == rec["enc_sum"] and float((a64 * a64).sum()) == rec["enc_sumsq"]


def _assert_hyp(want, got, fields):
    for f in fields:
        w, g = want[f], getattr(got, f)
        if f == "tokens" or f == "nbest":
            g = [list(map(int, x)) for x in g] if f == "nbest" else [int(x) for x in g]
        if f == "score":
            g = float(g)
        assert g == w, f


def test_synthetic_state_dict_is_strictly_loadable(pins, model_dirs):
    meta, _ = pins
    d, _ = model_dirs["causal_ln"]
    sd = torch.load(os.path.join(d, "synth.pt"))
    assert set(meta["state_dict"].keys()) == set(sd.keys())
    for k in sd:
        assert list(sd[k].shape) == meta["state_dict"][k], k
    assert meta["encoder_layer_type"] == "LanguageSpecificConformerEncoderLayer"
    assert meta["decoder_type"] == "LanguageSpecificBiTransformerDecoder"


@pytest.mark.parametrize("case", ["causal_ln", "sym_bn"])
def test_oracle_equals_live_reference(pins, model_dirs, golden_cases, case):
    from oracle import pipeline_ref
    meta, arrays = pins
    rec = meta["cases"][case]
    _, garr = golden_cases[case]
    d, wav = model_dirs[case]
    orc = pipeline_ref.OracleASR(d)
    f_ref = torch.from_numpy(garr["feats"]).unsqueeze(0)          # the reference's compute_feats of this wav
    assert (f_ref - orc.compute_feats(wav)).abs().max().item() < 5e-4
    cat = torch.tensor([0.25, 0.75])
    modes = ["ctc_greedy_search", "ctc_prefix_beam_search", "attention_rescoring"]
    batches = list(orc.feats_batcher(f_ref, 350, 2))
    assert len(batches) == len(rec["decode"])
    for bi, (fb, fl) in enumerate(batches):
        want = rec["decode"][bi]["results"]
        got = orc.decode(modes, fb, fl, 7, ctc_weight=0.3, reverse_weight=0.5, cat_embs=cat, return_intermediates=True)
        _assert_tensor_pinned(got["_encoder_out"], arrays, f"{case}_enc_{bi}", rec["decode"][bi])
        for b in range(fb.shape[0]):
            _assert_hyp(want["ctc_greedy_search"][b], got["ctc_greedy_search"][b], ["tokens"])
            _assert_hyp(want["ctc_prefix_beam_search"][b], got["ctc_prefix_beam_search"][b],
                        ["nbest", "nbest_scores", "nbest_times"])
            _assert_hyp(want["attention_rescoring"][b], got["attention_rescoring"][b],
                        ["tokens", "score", "confidence", "tokens_confidence"])


@pytest.mark.parametrize("case", ["causal_ln", "sym_bn"])
def test_oracle_attention_mode_and_bounded_context_equal_live_reference(pins, model_dirs, golden_cases, case):
    """The later restatements — `attention` decode mode (search.py:251-360) and decoding_chunk_size > 0
    (utils/mask.py:88-197) — against the reference with settings the other fixtures do not use."""
    from oracle import pipeline_ref
    meta, arrays = pins
    rec = meta["cases"][case]
    _, garr = golden_cases[case]
    d, _ = model_dirs[case]
    orc = pipeline_ref.OracleASR(d)
    feats = torch.from_numpy(garr["feats"]).unsqueeze(0)
    cat = torch.tensor([0.4, 0.6])
    batches = list(orc.feats_batcher(feats, 300, 2))
    assert len(batches) == len(rec["attention_bounded"])
    for bi, (fb, fl) in enumerate(batches):
        want = rec["attention_bounded"][bi]
        got = orc.decode(["attention"], fb, fl, 5, cat_embs=cat, length_penalty=0.3)
        assert [[int(x) for x in r.tokens] for r in got["attention"]] == [w["tokens"] for w in want["attention"]]
        got_c = orc.decode(["ctc_prefix_beam_search"], fb, fl, 6, cat_embs=cat, return_intermediates=True,
                           decoding_chunk_size=12, num_decoding_left_chunks=1)
        _assert_tensor_pinned(got_c["_encoder_out"], arrays, f"{case}_encc_{bi}", want)
        assert len(got_c["ctc_prefix_beam_search"]) == len(want["prefix"])
        for w, c in zip(want["prefix"], got_c["ctc_prefix_beam_search"]):
            _assert_hyp(w, c, ["nbest", "nbest_scores", "nbest_times"])


@pytest.mark.parametrize("case", ["causal_ln_k7", "sym_bn_k31", "causal_bn_k15", "sym_ln_k15"])
def test_oracle_conv_variants_equal_live_reference(tmp_path, case):
    """The convolution-module variants the decoding pins leave out — K = 7 and K = 31, causal BatchNorm, symmetric
    LayerNorm — on a zero-padded ragged batch (full context) and, for the symmetric ones, the chunk-by-chunk streaming
    pass, against the reference's encoder (oracle/make_golden_pins.py conv_pins -> tests/golden/pins_conv.*)."""
    from oracle import make_golden_pins as mgp, model_ref, pipeline_ref
    from reverb_b200 import synth
    with open(os.path.join(GOLDEN, "pins_conv.json")) as f:
        meta = json.load(f)
    arrays = dict(np.load(os.path.join(GOLDEN, "pins_conv.npz")))
    assert (meta["T"], meta["lens"], meta["chunk"], meta["cat"]) == (mgp.CONV_T, mgp.CONV_LENS, mgp.CONV_CHUNK, mgp.CONV_CAT)
    rec = meta["cases"][case]
    assert {k: rec[k] for k in ("causal", "cnn_module_norm", "kernel")} == mgp.CONV_CASES[case]
    d = synth.write_model_dir(str(tmp_path), shape=dict(synth.TEST_SHAPE, kernel=rec["kernel"]), seed=rec["seed"],
                              causal=rec["causal"], cnn_module_norm=rec["cnn_module_norm"])
    orc = pipeline_ref.OracleASR(d)
    feats = mgp.conv_case_inputs()
    cat = torch.tensor(mgp.CONV_CAT)
    enc, _, _ = orc.forward_encoder(feats, torch.tensor(mgp.CONV_LENS, dtype=torch.int32), cat)
    _assert_tensor_pinned(enc, arrays, f"{case}_enc", rec["enc"])
    assert ("stream" in rec) == (not rec["causal"])
    if "stream" in rec:
        enc = model_ref.encoder_forward_chunk_by_chunk(feats[:1], orc.sd, orc.cfg, cat, mgp.CONV_CHUNK)
        _assert_tensor_pinned(enc, arrays, f"{case}_stream", rec["stream"])


def test_oracle_resample_equals_torchaudio():
    import torchaudio
    from oracle import resample_ref
    g = torch.Generator().manual_seed(3)
    x = torch.randn(2, 7777, generator=g) * 3000
    for rate in (8000, 32000, 44100):
        want = torchaudio.transforms.Resample(orig_freq=rate, new_freq=16000)(x)
        assert torch.equal(resample_ref.resample(x, rate, 16000), want)


def test_host_post_processing_equals_live_reference(pins, golden_cases, model_dirs):
    """reverb_b200's ctc_align / CTM rendering vs the reference's, on the reference's own hypotheses."""
    from reverb_b200 import ctc_align as mine
    from reverb_b200.text import PieceTokenizer
    meta, _ = golden_cases["causal_ln"]
    want = pins[0]["cases"]["causal_ln"]["post_processing"]
    d, _ = model_dirs["causal_ln"]
    tok = PieceTokenizer(os.path.join(d, "tk.units.txt"))
    assert len(want) == len(meta["batches"])
    for batch, wb in zip(meta["batches"], want):
        assert len(wb) == len(batch["attention_rescoring"])
        for r, a in zip(batch["attention_rescoring"], wb):
            b = mine.adjust_model_time_offset(mine.ctc_align(r["tokens"], r["times"], r["tokens_confidence"], tok, 40, 1230), 230)
            assert json.loads(json.dumps(b)) == a
