"""G.711 and ADPCM WAV decoding on the GPU (csrc/wav_codec.cu through audio_io.load_audio): bit-equal to the oracle's
host decoders (oracle/wav_codec_ref.py) over every G.711 code, every IMA step index at 1, 2 and 6 channels, every MS
ADPCM predictor with a custom eighth pair, clamping, partial last blocks with and without `fact`; the hand-worked MS
blocks; a one-hour 8 kHz IMA file; invalid headers named by block and byte; and every entry point giving the same
output for a codec WAV as for the PCM16 WAV of its decoded samples."""
import struct

import numpy as np
import pytest

from oracle import flac_ref as F
from oracle import wav_codec_ref as W
from reverb_b200.audio_io import load_audio

pytestmark = pytest.mark.gpu


def _signal(nch, n, seed, square_blocks=0, spb=1):
    """random-walk speech stand-in; the first `square_blocks` blocks are a full-scale square wave (drives the clamps)"""
    rng = np.random.default_rng(seed)
    x = np.clip(np.cumsum(rng.normal(0, 700, (nch, n)), 1), -32768, 32767).astype(np.int64)
    m = min(n, square_blocks * spb)
    x[:, :m] = np.where((np.arange(m) // 23 + np.arange(nch)[:, None]) % 2, 32767, -32768)
    return x


def _load(tmp_path, data, name="x.wav"):
    p = tmp_path / name
    p.write_bytes(data)
    return load_audio(str(p))


def _check(tmp_path, wav, payload, tag, nch, ba, frames, coefs=W.MS_COEFS):
    pcm, rate = _load(tmp_path, wav)
    want = W.decode(payload, tag, nch, ba, frames, coefs)
    assert rate == 8000 and pcm.dtype == np.int16 and pcm.shape == (nch, frames)
    assert np.array_equal(pcm, want)
    return pcm


@pytest.mark.parametrize("tag", [W.MULAW, W.ALAW])
@pytest.mark.parametrize("nch", [1, 2])
def test_every_g711_code(tmp_path, tag, nch):
    payload = bytes(range(256)) * 3 + bytes(range(0, 256, 7))        # a trailing partial frame at 2 channels
    wav = W.write_wav(payload, tag, nch, 8000, nch, 8)
    pcm = _check(tmp_path, wav, payload, tag, nch, nch, len(payload) // nch)
    table = W.ulaw_table() if tag == W.MULAW else W.alaw_table()
    assert np.array_equal(np.sort(np.unique(pcm)), np.unique(table))


def test_g711_inside_extensible(tmp_path):
    payload = bytes(range(256))
    ext = struct.pack("<HI", 8, 4) + struct.pack("<H", W.MULAW) + bytes(14)
    wav = W.write_wav(payload, 0xFFFE, 1, 8000, 1, 8, ext)
    pcm, _ = _load(tmp_path, wav)
    assert np.array_equal(pcm[0], W.ulaw_table())


@pytest.mark.parametrize("ba_per_ch", [256, 512, 1024, 2048])
@pytest.mark.parametrize("nch", [1, 2, 6])
@pytest.mark.parametrize("fact", [False, True])
def test_ima_every_step_index(tmp_path, ba_per_ch, nch, fact):
    ba = ba_per_ch * nch
    spb = W.ima_spb(nch, ba)
    n = 90 * spb + spb // 3                                          # 91 blocks, the last one partial
    x = _signal(nch, n, seed=ba + nch, square_blocks=4, spb=spb)
    idx = (np.arange(91)[:, None] * 7 + np.arange(nch)) % 89         # every step index, per block and channel
    wav, payload = W.codec_wav(x, 8000, W.IMA_ADPCM, ba, fact=fact, step_index=idx, last="full" if fact else "short")
    frames = n if fact else W.frames_in(len(payload), W.IMA_ADPCM, nch, ba)
    pcm = _check(tmp_path, wav, payload, W.IMA_ADPCM, nch, ba, frames)
    assert pcm.max() == 32767 and pcm.min() == -32768                 # the clamps were reached


@pytest.mark.parametrize("nch,ba", [(1, 256), (1, 1024), (2, 512), (2, 2048)])
@pytest.mark.parametrize("fact", [False, True])
def test_ms_every_predictor_and_a_custom_table(tmp_path, nch, ba, fact):
    coefs = list(W.MS_COEFS) + [(300, -100)]
    spb = W.ms_spb(nch, ba)
    nblk = 64
    n = (nblk - 1) * spb + spb // 2 + 1
    x = _signal(nch, n, seed=ba * nch, square_blocks=3, spb=spb)
    pred = (np.arange(nblk)[:, None] + 3 * np.arange(nch)) % 8         # the seven standard pairs and the eighth
    delta = np.where(np.arange(nblk) % 5 == 0, 16, np.where(np.arange(nblk) % 5 == 1, 4000, 100 + np.arange(nblk)))
    wav, payload = W.codec_wav(x, 8000, W.MS_ADPCM, ba, fact=fact, coefs=coefs, predictor=pred, delta=delta,
                               last="full" if fact else "short")
    frames = n if fact else W.frames_in(len(payload), W.MS_ADPCM, nch, ba)
    pcm = _check(tmp_path, wav, payload, W.MS_ADPCM, nch, ba, frames, coefs)
    assert pcm.max() == 32767 and pcm.min() == -32768


def test_hand_worked_ms_blocks(tmp_path):
    from test_wav_codec_host import hand_ms_blocks
    for i, (wav, _payload, want) in enumerate(hand_ms_blocks()):
        pcm, _ = _load(tmp_path, wav, f"hand{i}.wav")
        assert pcm.dtype == np.int16 and np.array_equal(pcm, want), i


def test_one_hour_8k_ima(tmp_path):
    from reverb_b200 import synth
    x = synth.synth_audio(3600.0, seed=41, sample_rate=8000).astype(np.int64)[None]
    wav, payload = W.codec_wav(x, 8000, W.IMA_ADPCM, 256)
    _check(tmp_path, wav, payload, W.IMA_ADPCM, 1, 256, x.shape[1])


def test_bad_headers_name_the_block(tmp_path):
    x = _signal(2, 505 * 20, seed=5)
    wav, payload = W.codec_wav(x, 8000, W.IMA_ADPCM, 512)
    data_off = len(wav) - len(payload)
    bad = bytearray(wav)
    bad[data_off + 13 * 512 + 4 + 2] = 89                            # channel 1's step index in block 13
    bad[data_off + 17 * 512 + 2] = 200                               # and a later block: the lowest one is named
    with pytest.raises(ValueError, match=rf"ima\.wav: format tag 0x0011 \(IMA ADPCM\): block 13 at byte "
                                         rf"{data_off + 13 * 512}: IMA ADPCM step index above 88"):
        _load(tmp_path, bytes(bad), "ima.wav")
    wav, payload = W.codec_wav(x[:1], 8000, W.MS_ADPCM, 256)
    data_off = len(wav) - len(payload)
    bad = bytearray(wav)
    bad[data_off + 7 * 256] = 7                                      # predictor 7 with a 7-pair table
    with pytest.raises(ValueError, match=rf"ms\.wav: format tag 0x0002 \(MS ADPCM\): block 7 at byte "
                                         rf"{data_off + 7 * 256}: MS ADPCM predictor index"):
        _load(tmp_path, bytes(bad), "ms.wav")
    pcm, _ = _load(tmp_path, wav)                                    # the intact file still decodes
    assert pcm.shape == (1, x.shape[1])


# ------------------------------------------------------------------------------------------------ end to end
CODECS = {"ulaw": (W.MULAW, 0), "alaw": (W.ALAW, 0), "ima": (W.IMA_ADPCM, 256), "ms": (W.MS_ADPCM, 256)}


def _pcm16_wav(x: np.ndarray, rate: int) -> bytes:
    nch = x.shape[0]
    raw = np.ascontiguousarray(x.T).astype("<i2").tobytes()
    return W.write_wav(raw, 1, nch, rate, 2 * nch, 16)


@pytest.fixture(scope="module")
def pairs(tmp_path_factory):
    """<codec><rate>: (codec WAV, PCM16 WAV of its decoded samples); also a FLAC of the 16 kHz mono PCM"""
    from reverb_b200 import synth
    root = tmp_path_factory.mktemp("codec_pairs")
    out = {}
    for rate, seconds in ((8000, 9.0), (16000, 7.0)):
        x = synth.synth_audio(seconds, seed=rate // 1000, sample_rate=rate).astype(np.int64)[None]
        for name, (tag, ba) in CODECS.items():
            wav, payload = W.codec_wav(x, rate, tag, ba)
            dec = W.decode(payload, tag, 1, ba, x.shape[1])
            stem = f"{name}{rate // 1000}k"
            (root / f"{stem}.codec.wav").write_bytes(wav)
            (root / f"{stem}.wav").write_bytes(_pcm16_wav(dec, rate))
            out[stem] = (str(root / f"{stem}.codec.wav"), str(root / f"{stem}.wav"))
        if rate == 16000:
            (root / "flac16k.flac").write_bytes(F.encode(x, rate, 16))
            out["flac16k"] = (str(root / "flac16k.flac"), None)
    return out


@pytest.fixture(scope="module")
def models(model_dirs):
    import reverb_b200
    d = model_dirs["causal_ln"][0]
    return {p: reverb_b200.load_model(d, precision=p) for p in ("bf16", "fp32")}


def _same(a: str, b: str):
    assert a.replace(".codec.wav", ".wav") == b and a


def test_load_audio_returns_the_pcm_samples(pairs):
    for stem, (codec, pcm) in pairs.items():
        if pcm:
            (a, ra), (b, rb) = load_audio(codec), load_audio(pcm)
            assert ra == rb and a.dtype == b.dtype == np.int16 and np.array_equal(a, b), stem


@pytest.mark.parametrize("precision", ["bf16", "fp32"])
def test_transcribe_codec_equals_pcm(models, pairs, precision):
    m = models[precision]
    kw = dict(mode="ctc_prefix_beam_search", format="ctm", chunk_size=300, batch_size=2)
    for stem, (codec, pcm) in pairs.items():
        if pcm:
            _same(m.transcribe(codec, **kw), m.transcribe(pcm, **kw))


@pytest.mark.parametrize("precision", ["bf16", "fp32"])
def test_transcribe_files_over_pcm_flac_and_codecs(models, pairs, precision):
    m = models[precision]
    modes = ["attention_rescoring", "ctc_prefix_beam_search"]
    files = [pairs["ima8k"][0], pairs["flac16k"][0], pairs["ulaw16k"][1], pairs["ms16k"][0], pairs["alaw8k"][0],
             pairs["ima8k"][1]]
    got = list(m.transcribe_files(files, modes, format="ctm", chunk_size=300, batch_size=4))
    assert [p for p, _ in got] == files
    single = {p: m.transcribe_modes(p, modes, format="ctm", chunk_size=300, batch_size=4) for p in set(files)}
    for p, outs in got:
        assert outs == single[p]
    assert [o.replace(".codec.wav", ".wav") for o in got[0][1]] == got[5][1]


@pytest.mark.parametrize("precision", ["bf16", "fp32"])
def test_align_codec_equals_pcm(models, pairs, precision):
    m = models[precision]
    ids = [3, 4, 7, 6, 8, 9, 10, 22, 12, 13]
    for stem in ("ima8k", "ms16k"):
        codec, pcm = pairs[stem]
        _same(m.align(codec, ids, chunk_size=300), m.align(pcm, ids, chunk_size=300))


def test_diarization_rttm_codec_equals_pcm(pairs, tmp_path):
    from reverb_b200.diarization import infer
    for stem in ("alaw8k", "ima16k"):
        codec, pcm = pairs[stem]
        assert infer.main([codec, "--out-dir", str(tmp_path / "c"), "--synthetic"]) == 0
        assert infer.main([pcm, "--out-dir", str(tmp_path / "p"), "--synthetic"]) == 0
        a = (tmp_path / "c" / f"{stem}.codec.rttm").read_text()
        b = (tmp_path / "p" / f"{stem}.rttm").read_text()
        assert a.replace(f"{stem}.codec", stem) == b and a


@pytest.mark.parametrize("precision", ["bf16", "fp32"])
def test_recognize_wav_cli_codec_ctm(model_dirs, pairs, tmp_path, monkeypatch, precision):
    from reverb_b200 import recognize_wav
    monkeypatch.setenv("RVB_PRECISION", precision)
    d = model_dirs["causal_ln"][0]
    stems = ("ulaw8k", "ima8k", "alaw16k", "ms16k")
    for kind, idx in (("c", 0), ("p", 1)):
        recognize_wav.main(["--model", d, "--audio_file", *[pairs[s][idx] for s in stems],
                            "--result_dir", str(tmp_path / kind), "--modes", "ctc_prefix_beam_search",
                            "--chunk_size", "300", "--batch_size", "2"])
    for stem in stems:
        a = (tmp_path / "c" / "ctc_prefix_beam_search" / f"{stem}.codec.ctm").read_text()
        b = (tmp_path / "p" / "ctc_prefix_beam_search" / f"{stem}.ctm").read_text()
        assert a.replace(f"{stem}.codec", stem) == b and a
