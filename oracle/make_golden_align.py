"""ORACLE tooling (test infrastructure): pins CTC forced alignment — `force_align` (asr/wenet/utils/ctc_utils.py:105-161)
— against the LIVE reference.

Input = the CTC log-probabilities the reference itself recorded for the two small fixtures (tests/golden/{causal_ln,
sym_bn}.npz, ctc_probs_0, the valid frames of each utterance), and for the one case that needs more states than a warp
of the trellis kernel holds, the valid frames of all utterances of a fixture joined in time ("concat").  Label
sequences per utterance: the reference's own prefix-beam-search best hypothesis and every other n-best entry, random
labels, labels with adjacent repeats, a single label, and a sequence that fills the frames exactly (T == U + repeats).
Stored in tests/golden/align.json (cases: where the log-probs come from, the labels) and align.npz (frames_<i>: the
reference's output).  Every case is also checked here against oracle/align_ref.py.
Run from the repo root:  RVB_REFERENCE_ROOT=<reverb checkout> python oracle/make_golden_align.py
"""
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import align_ref  # noqa: E402
import refimport  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden")


def with_repeats(rng, U, V):
    y = [int(x) for x in rng.integers(1, V, U)]
    for i in range(1, U, 3):
        y[i] = y[i - 1]
    return y


def fill_exactly(rng, T, V):
    """Labels with U + #(adjacent repeats) == T."""
    y = [int(rng.integers(1, V))]
    need = 1
    while need < T:
        if need + 2 <= T and rng.random() < 0.3:
            y.append(y[-1])
            need += 2
        else:
            nxt = int(rng.integers(1, V))
            while nxt == y[-1]:
                nxt = int(rng.integers(1, V))
            y.append(nxt)
            need += 1
    return y


def main():
    refimport.import_reference()
    from wenet.transformer import search as rsearch
    from wenet.utils import ctc_utils
    rng = np.random.default_rng(11)
    cases, arrays = [], {}

    def add(fixture, source, kind, logp, labels):
        assert align_ref.feasible(labels, logp.shape[0]), (fixture, source, kind)
        ref = ctc_utils.force_align(torch.from_numpy(logp), torch.tensor(labels, dtype=torch.long), 0)
        ref = np.asarray([int(x) for x in ref], dtype=np.int32)
        mine = align_ref.force_align(logp, labels, 0)
        assert np.array_equal(ref, mine), f"oracle/align_ref.py disagrees with the reference on {fixture}/{source}/{kind}"
        arrays[f"frames_{len(cases)}"] = ref
        cases.append({"fixture": fixture, "source": source, "kind": kind, "labels": [int(x) for x in labels]})
        print(fixture, source, kind, "T", logp.shape[0], "U", len(labels))

    for name in ("causal_ln", "sym_bn"):
        arr = np.load(os.path.join(GOLDEN, name + ".npz"))
        meta = json.load(open(os.path.join(GOLDEN, name + ".json")))
        probs, lens = arr["ctc_probs_0"], arr["enc_lens_0"]
        V = probs.shape[2]
        nbest = rsearch.ctc_prefix_beam_search(torch.from_numpy(probs), torch.from_numpy(lens), int(meta["beam_size"]), None, 0)
        for b in range(probs.shape[0]):
            T = int(lens[b])
            logp = np.ascontiguousarray(probs[b, :T])
            for r, hyp in enumerate(nbest[b].nbest):
                if len(hyp):
                    add(name, b, "best" if r == 0 else f"nbest{r}", logp, list(map(int, hyp)))
            add(name, b, "random", logp, [int(x) for x in rng.integers(1, V, T // 3)])
            add(name, b, "repeats", logp, with_repeats(rng, T // 3, V))
            add(name, b, "single", logp, [int(rng.integers(1, V))])
            add(name, b, "limit", logp, fill_exactly(rng, T, V))
        joined = np.concatenate([probs[b, :int(lens[b])] for b in range(probs.shape[0])])
        add(name, "concat", "long", joined, with_repeats(rng, 130, V))
    with open(os.path.join(GOLDEN, "align.json"), "w") as f:
        json.dump({"torch": torch.__version__, "blank_id": 0, "cases": cases}, f)
    np.savez_compressed(os.path.join(GOLDEN, "align.npz"), **arrays)
    print("wrote tests/golden/align.{json,npz}:", len(cases), "cases")


if __name__ == "__main__":
    main()
