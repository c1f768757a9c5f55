"""FLAC decoding on the GPU (csrc/flac.cu through audio_io.load_audio): bit-exact against the oracle encoder's input
across sizes, rates, subframe types, stereo modes and residual codings; hand-assembled frames; a planted false sync
code; a one-hour libFLAC-layout stream; loud errors; and every entry point giving the same output for the same PCM as
WAV and as FLAC."""
import hashlib
import struct

import numpy as np
import pytest

from oracle import flac_ref as F
from reverb_b200.audio_io import load_audio, parse_flac_metadata

pytestmark = pytest.mark.gpu

S = F.SubSpec
SPECS = [S("verbatim"), S("fixed", order=0), S("fixed", order=1), S("fixed", order=2), S("fixed", order=3),
         S("fixed", order=4), S("lpc", order=1, precision=15), S("lpc", order=8, precision=12),
         S("lpc", order=12, precision=10), S("lpc", order=32, precision=15, rice_width=5)]


def _signal(nch, n, bps, seed=0, step_bits=8):
    rng = np.random.default_rng(seed)
    x = np.cumsum(rng.normal(0, 2.0 ** (bps - step_bits), (nch, n)), 1)
    lim = 2 ** (bps - 1)
    return np.clip(np.round(x), -lim, lim - 1).astype(np.int64)


def _decode(tmp_path, data, name="x.flac"):
    p = tmp_path / name
    p.write_bytes(data)
    return load_audio(str(p))


def _check(tmp_path, data, x, rate, bps):
    pcm, r = _decode(tmp_path, data)
    assert r == rate
    dt, width = (np.int16, 16) if bps <= 16 else (np.int32, 32)
    assert pcm.dtype == dt and pcm.shape == x.shape
    assert np.array_equal(pcm.astype(np.int64), x << (width - bps))
    vals = pcm.astype(np.int64) >> (width - bps)                 # the codec's values, for STREAMINFO's MD5
    w = (bps + 7) // 8
    md5 = hashlib.md5(np.ascontiguousarray(vals.T).astype("<i8").view(np.uint8).reshape(-1, 8)[:, :w].tobytes())
    assert md5.digest() == parse_flac_metadata(data).md5


def _mixed_frames(x, bs, seed):
    """Frames cycling through every subframe type per channel; one frame constant, one with wasted bits."""
    nch, n = x.shape
    frames, s, i = [], 0, 0
    while s < n:
        b = min(bs, n - s)
        frames.append(F.FrameSpec(b, sub=[SPECS[(i + c + seed) % len(SPECS)] if b > 32 else S("verbatim")
                                          for c in range(nch)]))
        s, i = s + b, i + 1
    frames[1].sub = [S("constant")] * nch
    x[:, bs:2 * bs] = x[:, bs:bs + 1]
    x[:, 2 * bs:3 * bs] &= ~np.int64(3)                          # 2 wasted bits (auto-detected)
    frames[2].sub = [S("lpc", order=4, precision=9)] * nch
    return frames


@pytest.mark.parametrize("bps,nch", [(4, 1), (8, 2), (12, 3), (16, 1), (16, 8), (17, 4), (20, 5), (24, 2), (24, 6),
                                     (31, 7), (32, 1), (32, 2)])
def test_sizes_channels_and_subframe_types(tmp_path, bps, nch):
    x = _signal(nch, 1024 * 13 + 77, bps, seed=bps * 10 + nch, step_bits=max(3, bps - 8) if bps < 12 else 8)
    frames = _mixed_frames(x, 1024, bps)
    _check(tmp_path, F.encode(x, 48000, bps, frames=frames), x, 48000, bps)


@pytest.mark.parametrize("bps", [16, 24, 32])
def test_every_stereo_mode(tmp_path, bps):
    x = _signal(2, 4096 * 9, bps, seed=bps)
    x[1] = (x[0] * 3 + x[1]) // 4                                 # correlated channels
    modes = ["independent", "left_side", "side_right", "mid_side"]
    frames = [F.FrameSpec(4096, stereo=modes[i % 4], sub=SPECS[(i * 3) % len(SPECS)]) for i in range(9)]
    _check(tmp_path, F.encode(x, 44100, bps, frames=frames), x, 44100, bps)


def test_every_block_size_code_with_variable_blocking_and_unknown_total(tmp_path):
    sizes = [(192, None), (576, None), (1152, None), (2304, None), (4608, None)] + \
        [(1 << k, None) for k in range(8, 16)] + [(100, 6), (1000, 7), (256, 6), (4096, 7), (65535, 7), (17, None)]
    x = _signal(2, sum(b for b, _ in sizes), 16, seed=3)
    frames = [F.FrameSpec(b, bs_code=c, stereo="mid_side" if i % 2 else "independent",
                          sub=S("lpc", order=min(8, b // 2), precision=12)) for i, (b, c) in enumerate(sizes)]
    data = F.encode(x, 16000, 16, frames=frames, variable=True, total_samples=0, id3=F.id3v2(),
                    blocks=[("SEEKTABLE", F.seektable([(0, 0, 192)])), ("VORBIS_COMMENT", F.vorbis_comment()),
                            ("APPLICATION", b"test1234"), ("CUESHEET", bytes(396)), ("PICTURE", bytes(50)),
                            ("PADDING", bytes(64))])
    _check(tmp_path, data, x, 16000, 16)


@pytest.mark.parametrize("rate,code", [(88200, None), (176400, None), (192000, None), (8000, None), (16000, None),
                                       (22050, None), (24000, None), (32000, None), (44100, None), (48000, None),
                                       (96000, None), (11000, 12), (11025, 13), (655350, 14), (12345, 0), (16000, 13),
                                       (16000, 0)])
def test_every_sample_rate_code(tmp_path, rate, code):
    x = _signal(1, 700, 16, seed=rate % 97)
    frames = [F.FrameSpec(256, rate_code=code, bps_code=0 if code == 0 else None), F.FrameSpec(256, rate_code=code),
              F.FrameSpec(188, rate_code=code)]
    data = F.encode(x, rate, 16, frames=frames)
    _check(tmp_path, data, x, rate, 16)


def test_partition_orders_parameter_widths_and_escapes(tmp_path):
    n = 32768
    x = _signal(1, n * 18, 16, seed=5)
    frames = [F.FrameSpec(n, sub=S("fixed", order=1, partition_order=po, rice_width=4 if po % 2 else 5))
              for po in range(16)]
    # explicit large 5-bit parameters; escaped partitions, one of them all-zero (0 bits per sample)
    x[0, 17 * n:17 * n + n // 4] = np.arange(n // 4) * 3 - 5000       # linear: FIXED order 2 residual is 0
    frames.append(F.FrameSpec(n, sub=S("fixed", order=2, partition_order=3, rice_width=5,
                                        rice_params=[29, 20, 5, 9, 0, 14, 3, 7])))
    frames.append(F.FrameSpec(n, sub=S("fixed", order=2, partition_order=2, escape=(0, 2), rice_width=4)))
    _check(tmp_path, F.encode(x, 16000, 16, frames=frames), x, 16000, 16)


def test_lpc_sums_beyond_32_bits(tmp_path):
    """24-bit audio with 15-bit coefficients: the predictor sums need 64 bits (RFC 9639 §9.2.6)"""
    x = _signal(2, 8192, 24, seed=9, step_bits=12)
    x = np.clip(x * 4, -2 ** 23, 2 ** 23 - 1)
    q, shift = F.quantize_coefs(F.lpc_coefs(x[:, :4096], 32), 15)
    acc = sum(q[:, j:j + 1] * x[:, 31 - j:4095 - j] for j in range(32))
    assert np.abs(acc).max() > 2 ** 31
    frames = [F.FrameSpec(4096, sub=S("lpc", order=32, precision=15, rice_width=5), stereo="left_side"),
              F.FrameSpec(4096, sub=S("lpc", order=32, precision=15))]
    _check(tmp_path, F.encode(x, 48000, 24, frames=frames), x, 48000, 24)


def test_hand_assembled_frames(tmp_path):
    from test_flac_host import hand_streams
    for i, (data, want) in enumerate(hand_streams()):
        pcm, rate = _decode(tmp_path, data, f"hand{i}.flac")
        assert rate == 16000 and pcm.dtype == np.int16 and np.array_equal(pcm, want)


def test_planted_sync_code_in_verbatim_data(tmp_path):
    x = _signal(1, 4096 * 3, 16, seed=11)
    fake = F.frame_header(7, 4096, 16000, 0, 16, False, F.FrameSpec(4096))   # a valid header, CRC-8 included
    assert len(fake) % 2 == 0
    words = np.frombuffer(fake, ">i2").astype(np.int64)
    x[0, 4096 + 100:4096 + 100 + len(words)] = words             # frame 1, VERBATIM: samples are byte-aligned
    frames = [F.FrameSpec(4096), F.FrameSpec(4096, sub=S("verbatim")), F.FrameSpec(4096)]
    data = F.encode(x, 16000, 16, frames=frames)
    assert data.count(fake) == 1
    _check(tmp_path, data, x, 16000, 16)


def test_one_hour_libflac_layout(tmp_path):
    from reverb_b200 import synth
    x = synth.synth_audio(3600.0, seed=21).astype(np.int64)[None]
    data = F.encode_libflac(x, 16000, 16)
    _check(tmp_path, data, x, 16000, 16)


def _frame_offsets(x, rate, bps, bs):
    """byte offset of every frame of F.encode(x, block_size=bs): a prefix of the frames encodes to the same bytes"""
    n = x.shape[1]
    return [len(F.encode(x[:, :k * bs], rate, bps, block_size=bs)) for k in range(1, (n + bs - 1) // bs)]


def test_corrupt_crc16_and_cut_file_name_the_frame(tmp_path):
    x = _signal(1, 4096 * 6, 16, seed=13)
    data = bytearray(F.encode(x, 16000, 16))
    offs = _frame_offsets(x, 16000, 16, 4096)
    bad = bytearray(data)
    bad[offs[3] - 1] ^= 0x5A                                     # last CRC-16 byte of frame 3
    with pytest.raises(ValueError, match=rf"bad\.flac: frame 3 at byte {offs[2]}: CRC-16 mismatch"):
        _decode(tmp_path, bytes(bad), "bad.flac")
    with pytest.raises(ValueError, match=rf"cut\.flac: frame 4 at byte {offs[3]}: missing"):
        _decode(tmp_path, bytes(data[:offs[3]]), "cut.flac")
    pcm, _ = _decode(tmp_path, bytes(data))                       # the intact file still decodes
    assert np.array_equal(pcm[0], x[0])


# ------------------------------------------------------------------------------------------------ end to end
def _riff(pcm: np.ndarray, rate: int, bits: int) -> bytes:
    nch = pcm.shape[0]
    if bits == 16:
        raw = np.ascontiguousarray(pcm.T).astype("<i2").tobytes()
    else:
        v = np.ascontiguousarray(pcm.T).astype("<i4").reshape(-1)
        raw = np.stack([v & 0xFF, (v >> 8) & 0xFF, (v >> 16) & 0xFF], 1).astype(np.uint8).tobytes()
    block = nch * bits // 8
    fmt = struct.pack("<HHIIHH", 1, nch, rate, rate * block, block, bits)
    chunks = b"fmt " + struct.pack("<I", 16) + fmt + b"data" + struct.pack("<I", len(raw)) + raw
    return b"RIFF" + struct.pack("<I", 4 + len(chunks)) + b"WAVE" + chunks


@pytest.fixture(scope="module")
def pairs(tmp_path_factory):
    """the same PCM as WAV (wav/<stem>.wav) and FLAC (flac/<stem>.flac)"""
    from reverb_b200 import synth
    root = tmp_path_factory.mktemp("flac_pairs")
    (root / "wav").mkdir()
    (root / "flac").mkdir()
    mono = synth.synth_audio(9.0, seed=31).astype(np.int64)[None]
    st = np.stack([synth.synth_audio(7.0, seed=32, sample_rate=44100), synth.synth_audio(7.0, seed=33, sample_rate=44100)])
    st = st.astype(np.int64)
    hi = synth.synth_audio(8.0, seed=34, sample_rate=48000).astype(np.int64)[None] * 256 + \
        np.random.default_rng(0).integers(-128, 128, (1, 384000))
    cases = {"mono16k": (mono, 16000, 16, None), "stereo44k": (st, 44100, 16, "mid_side"),
             "hi48k": (hi, 48000, 24, None)}
    out = {}
    for stem, (x, rate, bits, stereo) in cases.items():
        (root / "wav" / f"{stem}.wav").write_bytes(_riff(x, rate, bits))
        n = x.shape[1]
        frames = [F.FrameSpec(min(4096, n - s), stereo=stereo or "independent",
                              sub=S("lpc", order=min(8, (n - s) // 2), precision=12)) for s in range(0, n, 4096)]
        (root / "flac" / f"{stem}.flac").write_bytes(F.encode(x, rate, bits, frames=frames))
        out[stem] = (str(root / "wav" / f"{stem}.wav"), str(root / "flac" / f"{stem}.flac"))
    return out


@pytest.fixture(scope="module")
def models(model_dirs):
    import reverb_b200
    d = model_dirs["causal_ln"][0]
    return {p: reverb_b200.load_model(d, precision=p) for p in ("bf16", "fp32")}


def _same(a: str, b: str):
    assert a.replace(".flac", ".wav") == b and a


def test_load_audio_returns_the_wav_samples(pairs):
    for wav, flac in pairs.values():
        (a, ra), (b, rb) = load_audio(wav), load_audio(flac)
        assert ra == rb and a.dtype == b.dtype and np.array_equal(a, b)


@pytest.mark.parametrize("precision", ["bf16", "fp32"])
def test_transcribe_ctm_wav_equals_flac(models, pairs, precision):
    m = models[precision]
    for stem in ("mono16k", "stereo44k", "hi48k"):
        wav, flac = pairs[stem]
        kw = dict(mode="ctc_prefix_beam_search", format="ctm", chunk_size=300, batch_size=2)
        _same(m.transcribe(flac, **kw), m.transcribe(wav, **kw))


@pytest.mark.parametrize("precision", ["bf16", "fp32"])
def test_transcribe_files_over_mixed_containers(models, pairs, precision):
    m = models[precision]
    files = [pairs["mono16k"][1], pairs["stereo44k"][0], pairs["hi48k"][1], pairs["mono16k"][0]]
    got = list(m.transcribe_files(files, ["attention_rescoring", "ctc_prefix_beam_search"], format="ctm", chunk_size=300,
                                  batch_size=4))
    assert [p for p, _ in got] == files
    single = {p: m.transcribe_modes(p, ["attention_rescoring", "ctc_prefix_beam_search"], format="ctm", chunk_size=300,
                                    batch_size=4) for p in set(files)}
    for p, outs in got:
        assert outs == single[p]
    assert [o.replace(".flac", ".wav") for o in got[0][1]] == got[3][1]


@pytest.mark.parametrize("precision", ["bf16", "fp32"])
def test_align_wav_equals_flac(models, pairs, precision):
    m = models[precision]
    wav, flac = pairs["mono16k"]
    ids = [3, 4, 7, 6, 8, 9, 10, 22, 12, 13]
    _same(m.align(flac, ids, chunk_size=300), m.align(wav, ids, chunk_size=300))


def test_diarization_rttm_wav_equals_flac(pairs, tmp_path):
    from reverb_b200.diarization import infer
    wav, flac = pairs["stereo44k"]
    assert infer.main([wav, "--out-dir", str(tmp_path / "w"), "--synthetic"]) == 0
    assert infer.main([flac, "--out-dir", str(tmp_path / "f"), "--synthetic"]) == 0
    a, b = (tmp_path / "w" / "stereo44k.rttm").read_text(), (tmp_path / "f" / "stereo44k.rttm").read_text()
    assert a == b and a


@pytest.mark.parametrize("precision", ["bf16", "fp32"])
def test_recognize_wav_cli_flac_ctm(model_dirs, pairs, tmp_path, monkeypatch, precision):
    from reverb_b200 import recognize_wav
    monkeypatch.setenv("RVB_PRECISION", precision)
    d = model_dirs["causal_ln"][0]
    for kind, idx in (("w", 0), ("f", 1)):
        recognize_wav.main(["--model", d, "--audio_file", pairs["mono16k"][idx], pairs["stereo44k"][idx],
                            "--result_dir", str(tmp_path / kind), "--modes", "ctc_prefix_beam_search",
                            "--chunk_size", "300", "--batch_size", "2"])
    for stem in ("mono16k", "stereo44k"):
        a = (tmp_path / "f" / "ctc_prefix_beam_search" / f"{stem}.ctm").read_text()
        b = (tmp_path / "w" / "ctc_prefix_beam_search" / f"{stem}.ctm").read_text()
        _same(a, b)
