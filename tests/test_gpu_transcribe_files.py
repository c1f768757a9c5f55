"""`ReverbASR.transcribe_files`: many recordings per call, chunks of several recordings per batch, tail chunks at a
trimmed length.  Every recording's output must be byte-equal to the one-recording path with padded tails
(decode_stream over feats_batcher), and a trimmed batch's valid encoder rows bit-equal to the padded batch's."""
import os
import struct
from itertools import chain
from pathlib import Path

import numpy as np
import pytest
import torch

from reverb_b200 import corpus, synth
from reverb_b200.context_graph import ContextGraph

pytestmark = pytest.mark.gpu

CS = 300                                  # chunk_size of the per-file tests: 3 s chunks keep the corpus small
MODES = ["ctc_prefix_beam_search", "attention_rescoring"]


@pytest.fixture(scope="module")
def asr(model_dirs):
    import reverb_b200
    return {n: reverb_b200.load_model(d) for n, (d, _) in model_dirs.items()}


@pytest.fixture(scope="module")
def asr_fp32(model_dirs):
    import reverb_b200
    return {n: reverb_b200.load_model(d, precision="fp32") for n, (d, _) in model_dirs.items()}


def _write_wav(path, samples, rate, fmt_tag=1):
    """RIFF/WAVE with (n, channels) int16 (fmt_tag 1) or float32 (fmt_tag 3) samples."""
    samples = np.asarray(samples)
    if samples.ndim == 1:
        samples = samples[:, None]
    data = np.ascontiguousarray(samples.astype(np.int16 if fmt_tag == 1 else np.float32)).tobytes()
    ch, width = samples.shape[1], 2 if fmt_tag == 1 else 4
    fmt = struct.pack("<HHIIHH", fmt_tag, ch, rate, rate * ch * width, ch * width, 8 * width)
    with open(path, "wb") as f:
        f.write(b"RIFF" + struct.pack("<I", 4 + 8 + len(fmt) + 8 + len(data)) + b"WAVE")
        f.write(b"fmt " + struct.pack("<I", len(fmt)) + fmt + b"data" + struct.pack("<I", len(data)) + data)
    return str(path)


def _samples_for(frames):
    return 400 + 160 * (frames - 1)


@pytest.fixture(scope="module")
def corpus_wavs(tmp_path_factory):
    d = tmp_path_factory.mktemp("corpus")
    a = lambda s, seed: synth.synth_audio(s, seed=seed)          # noqa: E731
    files = [
        _write_wav(d / "just_over_400.wav", a(1.0, 1)[:420], 16000),
        _write_wav(d / "one_s.wav", a(1.0, 2), 16000),
        _write_wav(d / "five_s.wav", a(5.0, 3), 16000),
        _write_wav(d / "exact_chunk.wav", a(4.0, 4)[:_samples_for(CS)], 16000),
        _write_wav(d / "chunk_plus_1.wav", a(4.0, 5)[:_samples_for(CS + 1)], 16000),
        _write_wav(d / "two_and_a_half.wav", a(8.0, 6)[:_samples_for(int(2.5 * CS))], 16000),
        _write_wav(d / "seven_chunks.wav", a(22.0, 7)[:_samples_for(7 * CS)], 16000),
        _write_wav(d / "eight_k.wav", synth.synth_audio(3.0, seed=8, sample_rate=8000), 8000),
        _write_wav(d / "float_44k.wav", synth.synth_audio(4.0, seed=9, sample_rate=44100) / 32768.0, 44100, 3),
        _write_wav(d / "stereo.wav", np.stack([a(2.0, 10), a(2.0, 11)], 1), 16000),
        _write_wav(d / "short_tail.wav", a(7.0, 12)[:_samples_for(2 * CS + 5)], 16000),
        _write_wav(d / "twelve_s.wav", a(12.0, 13), 16000),
    ]
    return files


def _padded_outputs(m, wav, modes, formats=("ctm", "txt"), verbatimicity=1.0, chunk_size=2051, batch_size=1,
                    beam_size=10, decoding_chunk_size=-1, num_decoding_left_chunks=-1, ctc_weight=0.1,
                    simulate_streaming=False, reverse_weight=0.0, blank_penalty=0.0, length_penalty=0.0,
                    timings_adjustment=230, context_graph=None):
    """The one-recording path with zero-padded tails: decode_stream over feats_batcher, output per format."""
    from reverb_b200 import reverb
    feats = m.compute_feats(wav, num_mel_bins=80, frame_length=25, frame_shift=10)
    kw = dict(decoding_chunk_size=decoding_chunk_size, num_decoding_left_chunks=num_decoding_left_chunks,
              ctc_weight=ctc_weight, simulate_streaming=simulate_streaming, reverse_weight=reverse_weight,
              context_graph=context_graph, blank_id=m.blank_id, blank_penalty=blank_penalty,
              length_penalty=length_penalty, infos={"tasks": ["transcribe"], "langs": ["en"]},
              cat_embs=torch.tensor([verbatimicity, 1.0 - verbatimicity]))
    res = list(m.model.decode_stream(m.feats_batcher(feats, chunk_size, batch_size), modes, beam_size, **kw))
    return {fmt: [reverb.get_output(fmt, m.tokenizer, Path(wav).name, list(chain(*(r[mode] for r in res))),
                                    timings_adjustment, chunk_size, m.input_frame_length, m.output_frame_length)
                  for mode in modes] for fmt in formats}


def _check_files(m, files, modes, formats=("ctm", "txt"), **kw):
    want = {f: _padded_outputs(m, f, modes, formats, **kw) for f in files}
    for fmt in formats:
        got = list(m.transcribe_files(files, modes, format=fmt, **kw))
        assert [f for f, _ in got] == list(files)
        for f, outs in got:
            assert outs == want[f][fmt], (f, fmt, kw)
    return want


# 1. the trimming rule ---------------------------------------------------------------------------------------------

@pytest.mark.parametrize("precision", ["bf16", "fp32"])
@pytest.mark.parametrize("case", ["causal_ln", "sym_bn"])
@pytest.mark.parametrize("chunked", [False, True])
def test_trimmed_tail_batch_rows_bit_equal(asr, asr_fp32, model_dirs, case, precision, chunked):
    m = (asr if precision == "bf16" else asr_fp32)[case]
    cs = 2051
    right = corpus.right_context(m.configs["encoder_conf"])
    t_ref = corpus.encoder_out_frames(cs)
    feats = m.compute_feats(synth.write_wav(os.path.join(model_dirs[case][0], "rows.wav"),
                                            synth.synth_audio(40.0, seed=21)),
                            num_mel_bins=80, frame_length=25, frame_shift=10)[0]
    near = 4 * (t_ref - max(right, 1)) + 3 + 2          # e within r of T'_ref
    groups = [[near, 1500, 300], [900, 500, 40], [5, 20, 7 + 4 * right - 1, 3], [cs - 1]]
    dcs, left = (16, 2) if chunked else (-1, -1)
    cat = torch.tensor([0.7, 0.3])
    for lens in groups:
        T_b = corpus.batch_frames(lens, cs, right)
        assert T_b <= cs
        padded = torch.zeros(len(lens), cs, 80, device=feats.device)
        for b, n in enumerate(lens):
            padded[b, :n] = feats[700 * b:700 * b + n]
        trimmed = padded[:, :T_b].contiguous()
        fl = torch.tensor(lens, dtype=torch.int32)
        # trimmed before and after the padded batch: the positional cache is computed at either length
        outs = [m.model._forward_encoder(x, fl, cat, dcs, left) for x in (trimmed, padded, trimmed)]
        (e0, l0), (e1, l1), (e2, l2) = outs
        assert l0.tolist() == l1.tolist() == l2.tolist()
        tk = [m.engine.ctc_topk(e, 10, 0.0, 0) for e in (e0, e1, e2)]
        for b, e in enumerate(l1.tolist()):
            assert torch.equal(e0[b, :e], e1[b, :e]), (case, precision, lens, b)
            assert torch.equal(e2[b, :e], e1[b, :e]), (case, precision, lens, b)
            for (v, i, _) in (tk[0], tk[2]):
                assert torch.equal(v[b, :e], tk[1][0][b, :e]) and torch.equal(i[b, :e], tk[1][1][b, :e])


# 2. per-file outputs ------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("batch_size", [1, 3, 64])
@pytest.mark.parametrize("case", ["causal_ln", "sym_bn"])
def test_per_file_outputs_equal_single_file_path(asr, corpus_wavs, case, batch_size):
    m = asr[case]
    _check_files(m, corpus_wavs, MODES, chunk_size=CS, batch_size=batch_size, reverse_weight=0.0)
    # transcribe_modes is the one-file call of the same path
    f = corpus_wavs[6]
    assert m.transcribe_modes(f, MODES, format="ctm", chunk_size=CS, batch_size=batch_size) == \
        _padded_outputs(m, f, MODES, chunk_size=CS, batch_size=batch_size)["ctm"]


def test_attention_mode_subset(asr, corpus_wavs, monkeypatch):
    """The attention mode's outputs raise in get_output (reference quirk), so compare the hypotheses themselves."""
    from reverb_b200 import reverb
    monkeypatch.setattr(reverb, "get_output",
                        lambda fmt, tok, name, hyps, *a: repr([(list(h.tokens), h.score) for h in hyps]))
    for case in ("causal_ln", "sym_bn"):
        _check_files(asr[case], corpus_wavs[4:8], ["attention", "attention_rescoring"], formats=("txt",),
                     chunk_size=CS, batch_size=3)


def test_fp32_subset(asr_fp32, corpus_wavs):
    for case in ("causal_ln", "sym_bn"):
        _check_files(asr_fp32[case], corpus_wavs[:7:2], MODES, chunk_size=CS, batch_size=3)


# 3. other decode options ------------------------------------------------------------------------------------------

@pytest.mark.parametrize("option", ["context_graph", "verbatimicity", "reverse_weight", "chunked", "streaming"])
def test_decode_options(asr, corpus_wavs, option):
    m = asr["causal_ln"]
    kw = dict(chunk_size=CS, batch_size=4)
    if option == "context_graph":
        kw["context_graph"] = ContextGraph(context_score=3.0, token_lists=synth.context_phrases(40, 100, seed=3))
    elif option == "verbatimicity":
        kw["verbatimicity"] = 0.3
    elif option == "reverse_weight":
        kw["reverse_weight"] = 0.3
    elif option == "chunked":
        kw.update(decoding_chunk_size=16, num_decoding_left_chunks=2)
    else:                                   # one utterance per batch on the streaming path
        kw.update(decoding_chunk_size=16, num_decoding_left_chunks=2, simulate_streaming=True, batch_size=1)
    _check_files(m, corpus_wavs, MODES, **kw)


# 4. order, lanes and windows --------------------------------------------------------------------------------------

def test_order_lanes_and_windows(asr, corpus_wavs, monkeypatch):
    m = asr["sym_bn"]
    kw = dict(chunk_size=CS, batch_size=5, format="ctm")
    base = dict(m.transcribe_files(corpus_wavs, MODES, **kw))
    perm = [corpus_wavs[i] for i in np.random.default_rng(4).permutation(len(corpus_wavs))]
    got = list(m.transcribe_files(perm, MODES, **kw))
    assert [f for f, _ in got] == perm and dict(got) == base
    m.set_lanes(2)
    try:
        assert dict(m.transcribe_files(corpus_wavs, MODES, **kw)) == base
    finally:
        m.set_lanes(1)
    monkeypatch.setattr(corpus, "WINDOW_BATCHES", 0)          # every recording is a window of its own
    assert dict(m.transcribe_files(corpus_wavs, MODES, **kw)) == base
    assert list(m.transcribe_files([], MODES, **kw)) == []


# 5. errors ----------------------------------------------------------------------------------------------------------

def test_errors(asr, corpus_wavs, tmp_path):
    m = asr["causal_ln"]
    short = _write_wav(tmp_path / "too_short.wav", synth.synth_audio(0.1, seed=1)[:300], 16000)
    files = corpus_wavs[:3] + [short] + corpus_wavs[3:5]
    yielded = []
    with pytest.raises(AssertionError, match="too_short.wav"):
        for f, outs in m.transcribe_files(files, MODES, chunk_size=CS, batch_size=4):
            yielded.append(f)
    assert yielded == corpus_wavs[:3]
    with pytest.raises(AssertionError, match="choose a window size 400"):
        m.transcribe(short)
    missing = str(tmp_path / "missing.wav")
    with pytest.raises(FileNotFoundError, match="missing.wav"):
        list(m.transcribe_files(corpus_wavs[:2] + [missing], MODES, chunk_size=CS))
    for mode in ("ctc_greedy_search", "attention"):
        with pytest.raises(TypeError) as single:
            m.transcribe(corpus_wavs[1], mode=mode, chunk_size=CS)
        with pytest.raises(TypeError) as many:
            list(m.transcribe_files(corpus_wavs[:2], [mode], chunk_size=CS))
        assert str(single.value) == str(many.value)


# 6. command line ----------------------------------------------------------------------------------------------------

def test_cli_several_files(model_dirs, corpus_wavs, tmp_path):
    from reverb_b200 import recognize_wav
    d = model_dirs["causal_ln"][0]
    base = ["--config", os.path.join(d, "config.yaml"), "--checkpoint", os.path.join(d, "synth.pt"),
            "--chunk_size", str(CS), "--batch_size", "4", "--modes"] + MODES
    files = [corpus_wavs[i] for i in (2, 6, 9)]
    recognize_wav.main(base + ["--result_dir", str(tmp_path / "many"), "--audio_file"] + files)
    for f in files:
        recognize_wav.main(base + ["--result_dir", str(tmp_path / "one"), "--audio_file", f])
    for mode in MODES:
        for f in files:
            name = Path(f).with_suffix(".ctm").name
            one = (tmp_path / "one" / mode / name).read_text()
            assert one and (tmp_path / "many" / mode / name).read_text() == one
