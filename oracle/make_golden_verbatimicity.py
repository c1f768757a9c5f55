"""ORACLE tooling: golden vectors for per-utterance verbatimicity from the LIVE reference: the synthetic sym_bn model
of tests/golden/sym_bn.json, one batch of four chunks with a (B, 2) cat_embs whose rows hold 1, 0 and fractional
values -> encoder_out, ctc_greedy_search / ctc_prefix_beam_search (the reference's own 2-D cat_embs behaviour) and
attention_rescoring per row (the reference called one row at a time with that row's 1-D cat_embs)
-> tests/golden/verbatimicity.npz + verbatimicity.json.
Run from the repo root:  python oracle/make_golden_verbatimicity.py"""
import json
import os
import sys
import tempfile

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import refimport  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden")
CASE = "sym_bn"
CHUNK, BATCH = 220, 4
VALUES = [1.0, 0.0, 0.35, 0.7]
CTC_WEIGHT, REVERSE_WEIGHT, BEAM = 0.1, 0.0, 10


def cat_rows(values):
    return torch.tensor([[v, 1.0 - v] for v in values])


def main():
    sys.path.insert(0, ROOT)
    from reverb_b200 import synth
    wenet = refimport.import_reference()
    meta = json.load(open(os.path.join(GOLDEN, CASE + ".json")))
    d = tempfile.mkdtemp()
    synth.write_model_dir(d, causal=meta["causal"], cnn_module_norm=meta["cnn_module_norm"], seed=meta["model_seed"],
                          blank_rate=meta["blank_rate"])
    wav = synth.write_wav(os.path.join(d, "golden.wav"), synth.synth_audio(meta["audio_seconds"], seed=meta["audio_seed"]))
    m = wenet.load_model(d)
    feats = m.compute_feats(wav, num_mel_bins=80, frame_length=25, frame_shift=10)
    fb, fl = next(iter(m.feats_batcher(feats, CHUNK, BATCH)))
    assert fb.shape[0] == BATCH == len(VALUES)
    cat = cat_rows(VALUES)
    kw = dict(ctc_weight=CTC_WEIGHT, reverse_weight=REVERSE_WEIGHT, blank_id=m.blank_id,
              infos={"tasks": ["transcribe"], "langs": ["en"]})
    out = {"case": CASE, "chunk_size": CHUNK, "batch_size": BATCH, "values": VALUES, "beam_size": BEAM,
           "ctc_weight": CTC_WEIGHT, "reverse_weight": REVERSE_WEIGHT, "feats_lens": fl.tolist()}
    with torch.no_grad():
        enc, mask = m.model._forward_encoder(fb, fl, cat_embs=cat)
        res = m.model.decode(["ctc_greedy_search", "ctc_prefix_beam_search"], fb, fl, BEAM, cat_embs=cat, **kw)
        out["ctc_greedy_search"] = [list(map(int, r.tokens)) for r in res["ctc_greedy_search"]]
        out["ctc_prefix_beam_search"] = [{"tokens": list(map(int, r.tokens)),
                                          "nbest": [list(map(int, h)) for h in r.nbest],
                                          "nbest_scores": [float(s) for s in r.nbest_scores]}
                                         for r in res["ctc_prefix_beam_search"]]
        rows = []
        for b in range(BATCH):
            r = m.model.decode(["attention_rescoring"], fb[b:b + 1], fl[b:b + 1], BEAM, cat_embs=cat[b],
                               **kw)["attention_rescoring"][0]
            rows.append({"tokens": list(map(int, r.tokens)), "score": float(r.score)})
        out["attention_rescoring"] = rows
    arrays = {"feats": fb.numpy(), "encoder_out": enc.numpy(),
              "encoder_lens": mask.squeeze(1).sum(1).numpy().astype(np.int32)}
    np.savez_compressed(os.path.join(GOLDEN, "verbatimicity.npz"), **arrays)
    json.dump(out, open(os.path.join(GOLDEN, "verbatimicity.json"), "w"), indent=1)
    print({k: v.shape for k, v in arrays.items()})


if __name__ == "__main__":
    main()
