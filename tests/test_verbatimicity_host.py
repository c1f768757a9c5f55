"""Per-utterance verbatimicity on the host: the CPU oracle against the live reference's (B, 2) cat_embs golden data
(tests/golden/verbatimicity.*, oracle/make_golden_verbatimicity.py), and the argument checks of transcribe_files and
the command line."""
import json

import numpy as np
import pytest
import torch


def _golden():
    meta = json.load(open("tests/golden/verbatimicity.json"))
    return meta, dict(np.load("tests/golden/verbatimicity.npz"))


def test_oracle_per_row_cat_embs_vs_reference_golden(model_dirs):
    from oracle import lsl_rows_ref, pipeline_ref
    meta, arr = _golden()
    orc = pipeline_ref.OracleASR(model_dirs[meta["case"]][0])
    fb = torch.from_numpy(arr["feats"])
    fl = torch.tensor(meta["feats_lens"], dtype=torch.int32)
    cat = torch.tensor([[v, 1.0 - v] for v in meta["values"]])
    with lsl_rows_ref.per_row_cat_embs():
        out = orc.decode(["ctc_greedy_search", "ctc_prefix_beam_search"], fb, fl, meta["beam_size"],
                         ctc_weight=meta["ctc_weight"], reverse_weight=meta["reverse_weight"], cat_embs=cat,
                         return_intermediates=True)
    np.testing.assert_array_equal(out["_encoder_out"].numpy(), arr["encoder_out"])
    assert out["_encoder_lens"].tolist() == arr["encoder_lens"].tolist()
    assert [list(r.tokens) for r in out["ctc_greedy_search"]] == meta["ctc_greedy_search"]
    for r, g in zip(out["ctc_prefix_beam_search"], meta["ctc_prefix_beam_search"]):
        assert list(r.tokens) == g["tokens"] and [list(h) for h in r.nbest] == g["nbest"]
        assert list(r.nbest_scores) == g["nbest_scores"]
    for b, g in enumerate(meta["attention_rescoring"]):
        r = orc.decode(["attention_rescoring"], fb[b:b + 1], fl[b:b + 1], meta["beam_size"],
                       ctc_weight=meta["ctc_weight"], reverse_weight=meta["reverse_weight"],
                       cat_embs=cat[b])["attention_rescoring"][0]
        assert list(r.tokens) == g["tokens"] and float(r.score) == g["score"]


def test_golden_rows_differ_by_verbatimicity():
    """The fixture exercises the per-row mixing: rows of different values give different encoder outputs than the
    first row's value would (row 0 is verbatim, row 1 non-verbatim)."""
    meta, arr = _golden()
    assert meta["values"][0] == 1.0 and meta["values"][1] == 0.0 and 0.0 < meta["values"][2] < 1.0
    assert not np.array_equal(arr["encoder_out"][0], arr["encoder_out"][1])


class _NoModel:
    """Stands in for a loaded ReverbASR: transcribe_files must reject the arguments before touching the model."""


def test_transcribe_files_rejects_wrong_value_count():
    from reverb_b200.reverb import ReverbASR
    files = ["/nonexistent/a.wav", "/nonexistent/b.wav", "/nonexistent/c.wav"]
    for values in ([1.0, 0.0], [1.0, 0.0, 0.5, 0.5], []):
        with pytest.raises(ValueError, match="one per file"):
            next(iter(ReverbASR.transcribe_files(_NoModel(), files, ["ctc_prefix_beam_search"],
                                                 verbatimicity=values)))


def test_cli_verbatimicity_counts():
    from reverb_b200.recognize_wav import get_args
    base = ["--model", "m", "--result_dir", "out", "--audio_file", "a.wav", "b.wav", "c.wav"]
    assert get_args(base).verbatimicity == 1.0
    assert get_args(base + ["--verbatimicity", "0.3"]).verbatimicity == 0.3
    assert get_args(base + ["--verbatimicity", "0", "1", "0.5"]).verbatimicity == [0.0, 1.0, 0.5]
    with pytest.raises(SystemExit):
        get_args(base + ["--verbatimicity", "0", "1"])


def test_oracle_per_row_mix_restores_the_one_vector_form():
    """Equal rows give the 1-D result, the bf16-emulating branch folds per row, and the block leaves model_ref as it was."""
    from oracle import lsl_rows_ref, model_ref
    g = torch.Generator().manual_seed(0)
    d = 16
    sd = {f"l.language_layers.{i}.{k}": torch.randn(*( (d, d) if k == "weight" else (d,)), generator=g)
          for i in range(2) for k in ("weight", "bias")}
    x = torch.randn(3, 5, d, generator=g)
    cat = torch.tensor([[0.35, 0.65], [1.0, 0.0], [0.35, 0.65]])
    orig = model_ref.lsl_mix
    with lsl_rows_ref.per_row_cat_embs():
        assert model_ref.lsl_mix is not orig
        y = model_ref.lsl_mix(x, sd, "l", cat)
        for b in range(3):
            torch.testing.assert_close(y[b], orig(x[b:b + 1], sd, "l", cat[b])[0], rtol=1e-6, atol=1e-6)
        model_ref.EMULATE_BF16 = True
        try:
            ye = model_ref.lsl_mix(x, sd, "l", cat)
            for b in range(3):
                assert torch.equal(ye[b], orig(x[b:b + 1], sd, "l", cat[b])[0])
        finally:
            model_ref.EMULATE_BF16 = False
    assert model_ref.lsl_mix is orig
