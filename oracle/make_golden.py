"""Generate tests/golden/*.npz|json by running the LIVE reference (a revdotcom/reverb checkout named by
RVB_REFERENCE_ROOT, oracle/refimport.py).  Test infrastructure; run as `python -m oracle.make_golden`.

The tests must not depend on the Python reference, so its outputs on seeded synthetic
inputs are committed as small fixtures.  Inputs (model weights, audio) are regenerated
deterministically from seeds by reverb_b200/synth.py; a checksum of the weights is stored
so that a drifted generator is detected instead of silently compared.
"""
import json
import os
import sys
import tempfile
import warnings

import numpy as np
import torch

warnings.filterwarnings("ignore")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import refimport  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden")

CASES = [
    # name, causal, cnn norm, model seed, audio seconds, audio seed, chunk, batch, verbatimicity, reverse_weight
    ("causal_ln", True, "layer_norm", 0, 11.3, 1234, 400, 2, 0.7, 0.3),
    ("sym_bn", False, "batch_norm", 1, 9.0, 77, 330, 3, 1.0, 0.0),
]


def weights_checksum(sd):
    return float(sum(v.double().abs().sum().item() for k, v in sorted(sd.items()) if v.is_floating_point()))


def dr_to_dict(r):
    def f(x):
        if x is None:
            return None
        if isinstance(x, torch.Tensor):
            return float(x)
        return x
    return {
        "tokens": list(r.tokens), "score": f(r.score), "confidence": f(r.confidence),
        "tokens_confidence": r.tokens_confidence, "times": r.times,
        "nbest": [list(h) for h in r.nbest] if r.nbest is not None else None,
        "nbest_scores": r.nbest_scores, "nbest_times": r.nbest_times,
    }


def main():
    sys.path.insert(0, ROOT)
    import importlib.util
    spec = importlib.util.spec_from_file_location("rvb_synth", os.path.join(ROOT, "reverb_b200", "synth.py"))
    synth = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(synth)
    wenet = refimport.import_reference()
    os.makedirs(GOLDEN, exist_ok=True)
    modes = ["ctc_greedy_search", "ctc_prefix_beam_search", "attention_rescoring"]
    for name, causal, norm, mseed, secs, aseed, chunk, batch, verb, rw in CASES:
        d = tempfile.mkdtemp()
        synth.write_model_dir(d, causal=causal, cnn_module_norm=norm, seed=mseed, blank_rate=0.5)
        wav = synth.write_wav(os.path.join(d, "golden.wav"), synth.synth_audio(secs, seed=aseed))
        m = wenet.load_model(d)
        sd = torch.load(os.path.join(d, "synth.pt"))
        feats = m.compute_feats(wav, num_mel_bins=80, frame_length=25, frame_shift=10)
        cat = torch.tensor([verb, 1.0 - verb])
        arrays = {"feats": feats[0].numpy()}
        meta = {"name": name, "causal": causal, "cnn_module_norm": norm, "model_seed": mseed,
                "audio_seconds": secs, "audio_seed": aseed, "chunk_size": chunk, "batch_size": batch,
                "verbatimicity": verb, "reverse_weight": rw, "ctc_weight": 0.1, "beam_size": 10,
                "blank_rate": 0.5, "weights_checksum": weights_checksum(sd), "torch": torch.__version__,
                "batches": []}
        with torch.no_grad():
            for bi, (fb, fl) in enumerate(m.feats_batcher(feats, chunk, batch)):
                enc, mask = m.model._forward_encoder(fb, fl, cat_embs=cat)
                ctc = m.model.ctc_logprobs(enc)
                res = m.model.decode(modes, fb, fl, 10, ctc_weight=0.1, reverse_weight=rw,
                                     cat_embs=cat, blank_id=m.blank_id,
                                     infos={"tasks": ["transcribe"], "langs": ["en"]})
                arrays[f"enc_out_{bi}"] = enc.numpy()
                arrays[f"enc_lens_{bi}"] = mask.squeeze(1).sum(1).numpy()
                arrays[f"ctc_probs_{bi}"] = ctc.numpy()
                arrays[f"feats_lens_{bi}"] = fl.numpy()
                meta["batches"].append({k: [dr_to_dict(r) for r in v] for k, v in res.items()})
        # end-to-end strings through the reference's public API
        meta["transcribe"] = {}
        for mode in ("ctc_prefix_beam_search", "attention_rescoring"):
            for fmt in ("ctm", "txt"):
                meta["transcribe"][f"{mode}.{fmt}"] = m.transcribe(
                    wav, mode=mode, format=fmt, verbatimicity=verb, chunk_size=chunk, batch_size=batch,
                    beam_size=10, ctc_weight=0.1, reverse_weight=rw)
        np.savez_compressed(os.path.join(GOLDEN, f"{name}.npz"), **arrays)
        with open(os.path.join(GOLDEN, f"{name}.json"), "w") as f:
            json.dump(meta, f, indent=1)
        print("wrote", name, {k: v.shape for k, v in arrays.items()})

    # fbank-only fixtures straight from torchaudio (edge cases: N<400 -> empty; exactly one frame)
    from torchaudio.compliance import kaldi
    fb = {}
    for i, n in enumerate([400, 559, 560, 16000, 48123]):  # torchaudio asserts N >= 400
        pcm = synth.synth_audio(n / 16000.0 + 1e-9, seed=100 + i)[:n]
        assert pcm.shape[0] == n
        w = torch.from_numpy(pcm.astype(np.float32)).unsqueeze(0)
        out = kaldi.fbank(w, num_mel_bins=80, frame_length=25, frame_shift=10, dither=0.0,
                          energy_floor=0.0, sample_frequency=16000)
        fb[f"n{n}_seed{100 + i}"] = out.numpy().reshape(-1, 80)
    np.savez_compressed(os.path.join(GOLDEN, "fbank.npz"), **fb)
    print("wrote fbank", {k: v.shape for k, v in fb.items()})


if __name__ == "__main__":
    main()
