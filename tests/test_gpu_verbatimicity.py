"""Per-utterance verbatimicity: a (B, num_langs) cat_embs decodes row b exactly as a batch whose every row carries
cat_embs[b].  Checked at three levels: the grouped language-specific GEMM against plain launches of each group's
folded weight, ASRModel.decode rows against each other, and transcribe_files / the CLI against one call per file."""
import ctypes as C
import math
import os
from pathlib import Path

import numpy as np
import pytest
import torch

from reverb_b200 import synth

pytestmark = pytest.mark.gpu

CS = 300                                   # 3 s chunks: several chunks per file, files share batches
VALUES = [1.0, 0.0, 0.35, 1.0, 0.7]


def _p(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _check(rc):
    from reverb_b200 import _lib
    assert rc == 0, _lib.last_error()


@pytest.fixture(scope="module")
def lib():
    from reverb_b200 import _lib
    return _lib.load()


# 1. the grouped GEMM ------------------------------------------------------------------------------------------------

def _groups(G, B, seed):
    """Group of each of B utterances: runs of equal groups (so that whole tiles miss groups), every group present."""
    rng = np.random.default_rng(seed)
    g = np.sort(rng.integers(0, G, B)) if G > 1 else np.zeros(B, dtype=np.int64)
    g[:G] = np.arange(G)                     # every group present, the first G utterances one each
    return torch.tensor(g, dtype=torch.int32)


@pytest.mark.parametrize("G", [1, 2, 64])
@pytest.mark.parametrize("kind", ["f32", "bf16", "f32_x3", "bf16_pair"])
@pytest.mark.parametrize("rpb", [200, 3])
def test_grouped_gemm_bit_equal_to_plain_launches(lib, G, kind, rpb):
    x3 = kind.endswith("x3") or kind == "bf16_pair"
    out_mode = 1 if kind.startswith("f32") else 0
    d, K = 512, 512
    B = max(G, 70 if rpb == 200 else 300)
    M = B * rpb                                             # rpb = 200: M tiles straddle utterances
    g = torch.Generator(device="cuda").manual_seed(G * 7 + rpb)
    Af = torch.randn(M, K, device="cuda", generator=g) * 0.5
    Wf = torch.randn(G * d, K, device="cuda", generator=g) / math.sqrt(K)
    bias = torch.randn(G * d, device="cuda", generator=g)
    if x3:
        A = torch.empty(M, 2 * K, device="cuda", dtype=torch.bfloat16)
        W = torch.empty(G * d, 2 * K, device="cuda", dtype=torch.bfloat16)
        _check(lib.rvb_f32_to_bf16_pair(_p(Af), _p(A), M, K, _stream()))
        _check(lib.rvb_f32_to_bf16_pair(_p(Wf), _p(W), G * d, K, _stream()))
    else:
        A, W = Af.bfloat16(), Wf.bfloat16()
    width = d * (2 if (x3 and out_mode == 0) else 1)
    dt = torch.float32 if out_mode == 1 else torch.bfloat16
    grp = _groups(G, B, G + rpb)
    grp_d = grp.cuda()
    out = torch.full((M, width), 12345.0, device="cuda", dtype=dt)
    _check(lib.rvb_gemm_grouped(_p(A), _p(W), _p(bias), M, G * d, K, out_mode, _p(out), 0, _p(grp_d), rpb, d, int(x3),
                                _stream()))
    want = torch.empty_like(out)
    row_grp = grp.repeat_interleave(rpb).cuda()
    for k in range(G):
        part = torch.empty(M, width, device="cuda", dtype=dt)
        fn = lib.rvb_gemm_bf16x3 if x3 else lib.rvb_gemm_bf16
        _check(fn(_p(A), _p(W[k * d:(k + 1) * d]), _p(bias[k * d:(k + 1) * d]), M, d, K, 0, out_mode, 1.0, _p(part), 0,
                  _stream()))
        rows = row_grp == k
        want[rows] = part[rows]
    torch.cuda.synchronize()
    assert torch.equal(out.view(torch.int16) if dt == torch.bfloat16 else out.view(torch.int32),
                       want.view(torch.int16) if dt == torch.bfloat16 else want.view(torch.int32)), (G, kind, rpb)


def test_grouped_gemm_rejects_bad_groups(lib):
    A = torch.zeros(256, 512, device="cuda", dtype=torch.bfloat16)
    W = torch.zeros(2 * 96, 512, device="cuda", dtype=torch.bfloat16)
    out = torch.zeros(256, 96, device="cuda")
    grp = torch.zeros(2, dtype=torch.int32, device="cuda")
    assert lib.rvb_gemm_grouped(_p(A), _p(W), None, 256, 192, 512, 1, _p(out), 0, _p(grp), 128, 96, 0, _stream()) != 0


# 2. ASRModel.decode rows ---------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def asr(model_dirs):
    import reverb_b200
    return {n: reverb_b200.load_model(d) for n, (d, _) in model_dirs.items()}


@pytest.fixture(scope="module")
def asr_fp32(model_dirs):
    import reverb_b200
    return {n: reverb_b200.load_model(d, precision="fp32") for n, (d, _) in model_dirs.items()}


def _batch(m, model_dirs, case, B=4, T=CS):
    wav = synth.write_wav(os.path.join(model_dirs[case][0], "rows.wav"), synth.synth_audio(20.0, seed=31))
    feats = m.compute_feats(wav, num_mel_bins=80, frame_length=25, frame_shift=10)[0]
    x = torch.stack([feats[T * b:T * (b + 1)] for b in range(B)]).contiguous()
    return x, torch.full((B,), T, dtype=torch.int32)


def _cat(rows):
    return torch.tensor([[v, 1.0 - v] for v in rows])


METHODS = ["ctc_greedy_search", "ctc_prefix_beam_search", "attention_rescoring", "attention"]


def _summary(res, b):
    return {k: (list(r[b].tokens), r[b].score, list(getattr(r[b], "nbest", []) or []),
                list(getattr(r[b], "nbest_scores", []) or [])) for k, r in res.items()}


@pytest.mark.parametrize("precision", ["bf16", "fp32"])
@pytest.mark.parametrize("flat", [False, True])
def test_decode_rows_independent(asr, asr_fp32, model_dirs, monkeypatch, precision, flat):
    if flat:
        monkeypatch.setenv("RVB_RESCORE", "flat")
        monkeypatch.setenv("RVB_ATTENTION_STEP", "recompute")
    m = (asr if precision == "bf16" else asr_fp32)["sym_bn"]
    x, lens = _batch(m, model_dirs, "sym_bn")
    kw = dict(ctc_weight=0.3, reverse_weight=0.3, blank_id=m.blank_id)
    runs = {}
    for name, rows in (("a", [0.35, 1.0, 0.0, 0.7]), ("b", [0.35, 0.35, 0.5, 0.0]), ("u", [0.35] * 4)):
        cat = _cat(rows)
        enc, _ = m.model._forward_encoder(x.cuda(), lens, cat)
        res = m.model.decode(METHODS, x, lens, 4, cat_embs=cat, **kw)
        runs[name] = (enc, res)
    one = torch.tensor([0.35, 1.0 - 0.35])
    enc1, _ = m.model._forward_encoder(x.cuda(), lens, one)
    res1 = m.model.decode(METHODS, x, lens, 4, cat_embs=one, **kw)
    # row 0 does not depend on what the other rows carry
    assert torch.equal(runs["a"][0][0], runs["b"][0][0])
    assert _summary(runs["a"][1], 0) == _summary(runs["b"][1], 0)
    # equal rows are the one-vector call, bit for bit
    assert torch.equal(runs["u"][0], enc1)
    for b in range(4):
        assert _summary(runs["u"][1], b) == _summary(res1, b)
    # row b of a mixed batch is row b of a uniform batch at cat[b]
    for b, v in enumerate([0.35, 1.0, 0.0, 0.7]):
        cat_b = torch.tensor([v, 1.0 - v])
        enc_b, _ = m.model._forward_encoder(x.cuda(), lens, cat_b)
        assert torch.equal(runs["a"][0][b], enc_b[b])
        assert _summary(runs["a"][1], b) == _summary(m.model.decode(METHODS, x, lens, 4, cat_embs=cat_b, **kw), b)


def test_rescoring_scores_rows(asr, model_dirs):
    """ASRModel.attention_rescoring with a (B, 2) cat_embs: each row's decoder scores are the uniform call's."""
    m = asr["causal_ln"]
    x, lens = _batch(m, model_dirs, "causal_ln", B=3)
    rows = [0.0, 1.0, 0.6]
    pre = m.model.decode(["ctc_prefix_beam_search"], x, lens, 5, cat_embs=_cat(rows))["ctc_prefix_beam_search"]
    enc, el = m.model._forward_encoder(x.cuda(), lens, _cat(rows))
    nb = [r.nbest for r in pre]
    l2r, r2l = m.engine.rescoring_scores(enc, el, nb, _cat(rows), 0.3)
    for b, v in enumerate(rows):
        u2r, u2l = m.engine.rescoring_scores(enc, el, nb, torch.tensor([v, 1.0 - v]), 0.3)
        assert np.array_equal(np.asarray(l2r[b]), np.asarray(u2r[b]))
        if r2l is not None:
            assert np.array_equal(np.asarray(r2l[b]), np.asarray(u2l[b]))


def test_wrong_cat_length_is_an_error(asr, model_dirs):
    m = asr["sym_bn"]
    x, lens = _batch(m, model_dirs, "sym_bn", B=3)
    with pytest.raises(RuntimeError, match="one per utterance"):
        m.model._forward_encoder(x.cuda(), lens, torch.tensor([[1.0, 0.0], [0.0, 1.0]]))
    enc, el = m.model._forward_encoder(x.cuda(), lens, torch.tensor([1.0, 0.0]))
    with pytest.raises(RuntimeError, match="one per utterance"):
        m.engine.rescoring_scores(enc, el, [[(1, 2)]] * 3, torch.zeros(5), 0.0)


# 3. transcribe_files and the CLI --------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def wavs(tmp_path_factory):
    d = tmp_path_factory.mktemp("verbatimicity")
    out = []
    for i, secs in enumerate([5.0, 2.0, 7.3, 1.0, 4.0]):
        out.append(synth.write_wav(str(d / f"f{i}.wav"), synth.synth_audio(secs, seed=40 + i)))
    return out


def _per_file(m, files, values, modes, **kw):
    return {f: m.transcribe_modes(f, modes, verbatimicity=v, **kw) for f, v in zip(files, values)}


SETTINGS = [
    # (precision, lanes, env, decode keywords)
    ("bf16", 0, {}, dict(batch_size=3)),
    ("bf16", 0, {"RVB_RESCORE": "flat", "RVB_ATTENTION_STEP": "recompute"}, dict(batch_size=4)),
    ("fp32", 0, {}, dict(batch_size=3, decoding_chunk_size=16, num_decoding_left_chunks=2)),
    ("bf16", 2, {}, dict(batch_size=2)),
    ("fp32", 2, {"RVB_RESCORE": "flat", "RVB_ATTENTION_STEP": "recompute"}, dict(batch_size=3)),
    ("bf16", 0, {}, dict(batch_size=1, decoding_chunk_size=16, simulate_streaming=True)),
]


@pytest.mark.parametrize("setting", range(len(SETTINGS)))
def test_transcribe_files_per_file_values_equal_single_file(asr, asr_fp32, wavs, monkeypatch, setting):
    precision, lanes, env, kw = SETTINGS[setting]
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    m = (asr if precision == "bf16" else asr_fp32)["sym_bn" if setting % 2 == 0 else "causal_ln"]
    # (the attention mode's hypotheses carry no token times, which both output formats need: it is checked through
    # ASRModel.decode above)
    modes = ["ctc_prefix_beam_search", "attention_rescoring"]
    for fmt in ("ctm", "txt"):
        want = _per_file(m, wavs, VALUES, modes, format=fmt, chunk_size=CS, reverse_weight=0.3, **kw)
        if lanes:
            m.set_lanes(lanes)
        try:
            got = list(m.transcribe_files(wavs, modes, format=fmt, verbatimicity=VALUES, chunk_size=CS,
                                          reverse_weight=0.3, **kw))
        finally:
            if lanes:
                m.set_lanes(1)
        assert [f for f, _ in got] == wavs
        for f, outs in got:
            assert outs == want[f], (f, fmt, SETTINGS[setting])


def test_joint_decoding_rows(bench_model_dir):
    """joint_decoding needs a vocabulary above its hard-coded sos (10000): the benchmark-shaped model.  Row b of a
    (B, 2) cat_embs decodes as the one-vector call at cat_embs[b]."""
    import reverb_b200
    m = reverb_b200.load_model(bench_model_dir)
    wav = synth.write_wav(os.path.join(bench_model_dir, "joint.wav"), synth.synth_audio(10.0, seed=61))
    feats = m.compute_feats(wav, num_mel_bins=80, frame_length=25, frame_shift=10)[0]
    x = torch.stack([feats[CS * b:CS * (b + 1)] for b in range(3)]).contiguous()
    lens = torch.full((3,), CS, dtype=torch.int32)
    rows = [0.0, 1.0, 0.35]
    kw = dict(ctc_weight=0.3, blank_id=m.blank_id)
    got = m.model.decode(["joint_decoding", "attention_rescoring"], x, lens, 4, cat_embs=_cat(rows), **kw)
    for b, v in enumerate(rows):
        one = m.model.decode(["joint_decoding", "attention_rescoring"], x, lens, 4, cat_embs=torch.tensor([v, 1.0 - v]),
                             **kw)
        assert _summary(got, b) == _summary(one, b), b


def test_transcribe_files_length_mismatch(asr, wavs):
    with pytest.raises(ValueError, match="one per file"):
        next(iter(asr["sym_bn"].transcribe_files(wavs + ["/nonexistent.wav"], ["ctc_prefix_beam_search"],
                                                 verbatimicity=VALUES)))


def test_cli_two_files_two_values(model_dirs, wavs, tmp_path):
    from reverb_b200 import recognize_wav
    d = model_dirs["sym_bn"][0]
    base = ["--model", d, "--chunk_size", str(CS), "--batch_size", "4", "--modes", "attention_rescoring",
            "ctc_prefix_beam_search"]
    recognize_wav.main(base + ["--audio_file", wavs[0], wavs[2], "--verbatimicity", "0.0", "0.8",
                               "--result_dir", str(tmp_path / "both")])
    for f, v in ((wavs[0], "0.0"), (wavs[2], "0.8")):
        recognize_wav.main(base + ["--audio_file", f, "--verbatimicity", v, "--result_dir", str(tmp_path / "one")])
    for mode in ("attention_rescoring", "ctc_prefix_beam_search"):
        for f in (wavs[0], wavs[2]):
            name = Path(f).with_suffix(".ctm").name
            assert (tmp_path / "both" / mode / name).read_text() == (tmp_path / "one" / mode / name).read_text()


# 4. the live reference -------------------------------------------------------------------------------------------------

def test_accurate_mode_per_row_cat_embs_matches_the_reference_golden(asr_fp32):
    """precision='fp32' with a (B, 2) cat_embs against tests/golden/verbatimicity.* (the live reference's 2-D cat_embs
    for the encoder and the CTC modes, row-by-row 1-D calls for attention_rescoring): encoder_out rel-RMS < 2e-5 (the
    bar of the one-vector golden test) and every token identical."""
    import json
    meta = json.load(open("tests/golden/verbatimicity.json"))
    arr = dict(np.load("tests/golden/verbatimicity.npz"))
    m = asr_fp32[meta["case"]]
    fb = torch.from_numpy(arr["feats"]).cuda()
    fl = torch.tensor(meta["feats_lens"], dtype=torch.int32)
    cat = _cat(meta["values"])
    enc, enc_lens = m.model._forward_encoder(fb, fl, cat)
    assert enc_lens.tolist() == arr["encoder_lens"].tolist()
    for b in range(fb.shape[0]):
        n = int(enc_lens[b])
        e, r = enc[b, :n].cpu().double().numpy(), arr["encoder_out"][b, :n].astype(np.float64)
        assert np.sqrt(np.mean((e - r) ** 2) / np.mean(r ** 2)) < 2e-5, b
    got = m.model.decode(["ctc_greedy_search", "ctc_prefix_beam_search", "attention_rescoring"], fb, fl,
                         meta["beam_size"], ctc_weight=meta["ctc_weight"], reverse_weight=meta["reverse_weight"],
                         cat_embs=cat, blank_id=0)
    assert [list(r.tokens) for r in got["ctc_greedy_search"]] == meta["ctc_greedy_search"]
    for r, g in zip(got["ctc_prefix_beam_search"], meta["ctc_prefix_beam_search"]):
        assert list(r.tokens) == g["tokens"] and [list(h) for h in r.nbest] == g["nbest"]
    assert [list(r.tokens) for r in got["attention_rescoring"]] == [g["tokens"] for g in meta["attention_rescoring"]]
