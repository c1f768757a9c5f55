"""Record the LIVE reference's results that pin the oracle and the synthetic-model generator
(tests/test_oracle_vs_reference.py) -> tests/golden/pins.json + pins.npz, and the encoder outputs of the convolution
module variants the decoding pins do not cover -> tests/golden/pins_conv.json + pins_conv.npz.

    python -m oracle.make_golden_pins [conv]   # needs RVB_REFERENCE_ROOT (oracle/refimport.py); `conv`: only the latter

Encoder outputs are stored as a fixed, seeded sample of elements plus float64 sums of the whole tensor, so that an
exact comparison stays possible without storing the tensors.
"""
import json
import os
import sys
import warnings

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
GOLDEN = os.path.join(ROOT, "tests", "golden")
N_SAMPLE = 2048


def tensor_pin(t: torch.Tensor, seed: int):
    """Seeded sample of flat indices / values and float64 sum and sum of squares of `t` (float32)."""
    a = t.detach().cpu().numpy().astype(np.float32).reshape(-1)
    idx = np.sort(np.random.default_rng(seed).choice(a.size, size=min(N_SAMPLE, a.size), replace=False))
    a64 = a.astype(np.float64)
    return idx.astype(np.int64), a[idx], float(a64.sum()), float((a64 * a64).sum())


def hyp(r):
    return {"tokens": [int(x) for x in r.tokens], "score": float(r.score) if r.score is not None else None,
            "confidence": r.confidence, "tokens_confidence": r.tokens_confidence,
            "nbest": [list(map(int, n)) for n in (r.nbest or [])], "nbest_scores": r.nbest_scores,
            "nbest_times": r.nbest_times}


def main():
    warnings.filterwarnings("ignore")
    from oracle import refimport
    from reverb_b200 import synth
    wenet_ref = refimport.import_reference()
    meta_out, arrays = {"cases": {}}, {}
    for case in ("causal_ln", "sym_bn"):
        with open(os.path.join(GOLDEN, case + ".json")) as f:
            meta = json.load(f)
        d = os.path.join("/tmp", f"rvb_pins_{case}")
        os.makedirs(d, exist_ok=True)
        synth.write_model_dir(d, causal=meta["causal"], cnn_module_norm=meta["cnn_module_norm"], seed=meta["model_seed"],
                              blank_rate=meta["blank_rate"])
        wav = synth.write_wav(os.path.join(d, "golden.wav"), synth.synth_audio(meta["audio_seconds"], seed=meta["audio_seed"]))
        m = wenet_ref.load_model(d)
        rec = {}
        if case == "causal_ln":
            sd = m.model.state_dict()
            meta_out["state_dict"] = {k: list(v.shape) for k, v in sd.items()}
            meta_out["encoder_layer_type"] = type(m.model.encoder.encoders[0]).__name__
            meta_out["decoder_type"] = type(m.model.decoder).__name__
        feats = m.compute_feats(wav, num_mel_bins=80, frame_length=25, frame_shift=10)
        # decode: chunk 350, batch 2, beam 7 (test_oracle_equals_live_reference)
        cat = torch.tensor([0.25, 0.75])
        modes = ["ctc_greedy_search", "ctc_prefix_beam_search", "attention_rescoring"]
        rec["decode"] = []
        for bi, (fb, fl) in enumerate(m.feats_batcher(feats, 350, 2)):
            with torch.no_grad():
                want = m.model.decode(modes, fb, fl, 7, ctc_weight=0.3, reverse_weight=0.5, cat_embs=cat,
                                      infos={"tasks": ["transcribe"], "langs": ["en"]})
                enc, _ = m.model._forward_encoder(fb, fl, cat_embs=cat)
            idx, val, s1, s2 = tensor_pin(enc, 1000 + bi)
            arrays[f"{case}_enc_{bi}_idx"], arrays[f"{case}_enc_{bi}_val"] = idx, val
            rec["decode"].append({"enc_shape": list(enc.shape), "enc_sum": s1, "enc_sumsq": s2,
                                  "results": {k: [hyp(r) for r in want[k]] for k in modes}})
        # attention mode and bounded context: chunk 300, batch 2
        cat = torch.tensor([0.4, 0.6])
        rec["attention_bounded"] = []
        for bi, (fb, fl) in enumerate(m.feats_batcher(feats, 300, 2)):
            with torch.no_grad():
                want = m.model.decode(["attention"], fb, fl, 5, length_penalty=0.3, cat_embs=cat,
                                      infos={"tasks": ["transcribe"], "langs": ["en"]})
                enc, _ = m.model._forward_encoder(fb, fl, decoding_chunk_size=12, num_decoding_left_chunks=1, cat_embs=cat)
                want_c = m.model.decode(["ctc_prefix_beam_search"], fb, fl, 6, decoding_chunk_size=12,
                                        num_decoding_left_chunks=1, cat_embs=cat, infos={"tasks": ["transcribe"], "langs": ["en"]})
            idx, val, s1, s2 = tensor_pin(enc, 2000 + bi)
            arrays[f"{case}_encc_{bi}_idx"], arrays[f"{case}_encc_{bi}_val"] = idx, val
            rec["attention_bounded"].append({"enc_shape": list(enc.shape), "enc_sum": s1, "enc_sumsq": s2,
                                             "attention": [hyp(r) for r in want["attention"]],
                                             "prefix": [hyp(r) for r in want_c["ctc_prefix_beam_search"]]})
        if case == "causal_ln":
            # the reference's CTM post-processing on its own hypotheses (golden causal_ln batches)
            from wenet.bin.ctc_align import adjust_model_time_offset as ref_adjust, ctc_align as ref_align
            rec["post_processing"] = [
                [ref_adjust(ref_align(r["tokens"], r["times"], r["tokens_confidence"], m.tokenizer, 40, 1230), 230)
                 for r in batch["attention_rescoring"]] for batch in meta["batches"]]
        meta_out["cases"][case] = rec
    np.savez_compressed(os.path.join(GOLDEN, "pins.npz"), **arrays)
    with open(os.path.join(GOLDEN, "pins.json"), "w") as f:
        json.dump(meta_out, f, separators=(",", ":"))


# Convolution-module variants at the test shape (d = 128): kernel sizes 7 and 31, causal BatchNorm, symmetric LayerNorm.
# Each runs one zero-padded ragged batch through the full-context encoder; the symmetric ones also run the cache-based
# chunk-by-chunk streaming pass.
CONV_CASES = {
    "causal_ln_k7": dict(causal=True, cnn_module_norm="layer_norm", kernel=7),
    "sym_bn_k31": dict(causal=False, cnn_module_norm="batch_norm", kernel=31),
    "causal_bn_k15": dict(causal=True, cnn_module_norm="batch_norm", kernel=15),
    "sym_ln_k15": dict(causal=False, cnn_module_norm="layer_norm", kernel=15),
}
CONV_T, CONV_LENS, CONV_CHUNK, CONV_CAT, CONV_SEED = 403, [403, 298, 61], 16, [0.25, 0.75], 5


def conv_case_inputs():
    from oracle import encoder_ref
    return encoder_ref.zero_pad(encoder_ref.features(len(CONV_LENS), CONV_T, seed=CONV_SEED), CONV_LENS)


def conv_pins():
    warnings.filterwarnings("ignore")
    from oracle import refimport
    from reverb_b200 import synth
    wenet_ref = refimport.import_reference()
    feats = conv_case_inputs()
    lens = torch.tensor(CONV_LENS, dtype=torch.int32)
    cat = torch.tensor(CONV_CAT)
    meta_out, arrays = {"T": CONV_T, "lens": CONV_LENS, "chunk": CONV_CHUNK, "cat": CONV_CAT, "cases": {}}, {}
    for ci, (case, kw) in enumerate(CONV_CASES.items()):
        d = os.path.join("/tmp", f"rvb_pins_conv_{case}")
        synth.write_model_dir(d, shape=dict(synth.TEST_SHAPE, kernel=kw["kernel"]), seed=CONV_SEED + ci,
                              causal=kw["causal"], cnn_module_norm=kw["cnn_module_norm"])
        m = wenet_ref.load_model(d)
        rec = dict(kw, seed=CONV_SEED + ci)
        with torch.no_grad():
            enc, _ = m.model._forward_encoder(feats, lens, cat_embs=cat)
        idx, val, s1, s2 = tensor_pin(enc, 3000 + ci)
        arrays[f"{case}_enc_idx"], arrays[f"{case}_enc_val"] = idx, val
        rec["enc"] = {"enc_shape": list(enc.shape), "enc_sum": s1, "enc_sumsq": s2}
        if not kw["causal"]:
            with torch.no_grad():
                enc, _ = m.model.encoder.forward_chunk_by_chunk(feats[:1], CONV_CHUNK, -1, cat_embs=cat)
            idx, val, s1, s2 = tensor_pin(enc, 4000 + ci)
            arrays[f"{case}_stream_idx"], arrays[f"{case}_stream_val"] = idx, val
            rec["stream"] = {"enc_shape": list(enc.shape), "enc_sum": s1, "enc_sumsq": s2}
        meta_out["cases"][case] = rec
    np.savez_compressed(os.path.join(GOLDEN, "pins_conv.npz"), **arrays)
    with open(os.path.join(GOLDEN, "pins_conv.json"), "w") as f:
        json.dump(meta_out, f, indent=1)


if __name__ == "__main__":
    if sys.argv[1:] != ["conv"]:
        main()
    conv_pins()
