"""ORACLE tooling (test infrastructure): pins the `attention` decode mode (autoregressive beam search with the left
decoder, asr/wenet/transformer/search.py:251-360) against the LIVE reference (a reference checkout, see oracle/refimport.py).

Re-creates the two synthetic models of tests/golden/{causal_ln,sym_bn}.json from their stored seeds, runs the
reference's ASRModel.decode(['attention'], ...) batch by batch (two length penalties) and stores the token ids in
tests/golden/attention_mode.json.  Run from the repo root:  python oracle/make_golden_attention.py
"""
import json
import os
import sys
import tempfile

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import refimport  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden")


def main():
    sys.path.insert(0, ROOT)
    from reverb_b200 import synth
    wenet = refimport.import_reference()
    out = {"torch": torch.__version__, "beam_size": 10, "cases": {}}
    for name in ("causal_ln", "sym_bn"):
        meta = json.load(open(os.path.join(GOLDEN, name + ".json")))
        d = tempfile.mkdtemp()
        synth.write_model_dir(d, causal=meta["causal"], cnn_module_norm=meta["cnn_module_norm"],
                              seed=meta["model_seed"], blank_rate=meta["blank_rate"])
        wav = synth.write_wav(os.path.join(d, "golden.wav"), synth.synth_audio(meta["audio_seconds"], seed=meta["audio_seed"]))
        m = wenet.load_model(d)
        feats = m.compute_feats(wav, num_mel_bins=80, frame_length=25, frame_shift=10)
        cat = torch.tensor([meta["verbatimicity"], 1.0 - meta["verbatimicity"]])
        case = {}
        with torch.no_grad():
            for lp in (0.0, 0.6):
                batches = []
                for fb, fl in m.feats_batcher(feats, meta["chunk_size"], meta["batch_size"]):
                    res = m.model.decode(["attention"], fb, fl, 10, length_penalty=lp, cat_embs=cat, blank_id=m.blank_id,
                                         infos={"tasks": ["transcribe"], "langs": ["en"]})
                    batches.append([list(map(int, r.tokens)) for r in res["attention"]])
                case[f"length_penalty_{lp}"] = batches
        out["cases"][name] = case
        print(name, {k: [[len(t) for t in b] for b in v] for k, v in case.items()})
    with open(os.path.join(GOLDEN, "attention_mode.json"), "w") as f:
        json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
