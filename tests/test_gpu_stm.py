"""transcribe(format="stm", diarization=...) is byte-equal to the three command lines run on files:
diarization.infer (RTTM) -> recognize_wav (CTM) -> words2speakers (STM); recognize_wav --diarization_synthetic writes
the same .stm and .rttm files."""
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

MODES = ["attention_rescoring", "ctc_prefix_beam_search"]


@pytest.fixture(scope="module")
def recordings(tmp_path_factory):
    """a mono call, and a stereo one whose channels differ (the ASR hears channel 0, diarization the downmix)"""
    import wave
    from reverb_b200.diarization import synth
    d = tmp_path_factory.mktemp("stm_audio")
    mono = (np.clip(synth.synthetic_speech(40.0, seed=5, turns=2), -1, 1) * 32767).astype(np.int16)[None]
    left = synth.synthetic_speech(30.0, seed=7, turns=3)
    right = synth.synthetic_speech(30.0, seed=8, turns=2)
    stereo = (np.clip(np.stack([left, right]), -1, 1) * 32767).astype(np.int16)
    paths = []
    for name, pcm in (("call_a.wav", mono), ("call_b.wav", stereo)):
        p = str(d / name)
        with wave.open(p, "wb") as w:
            w.setnchannels(pcm.shape[0])
            w.setsampwidth(2)
            w.setframerate(16000)
            w.writeframes(pcm.T.tobytes())
        paths.append(p)
    return paths


@pytest.fixture(scope="module")
def diarization():
    from reverb_b200.diarization.infer import load_pipeline
    return load_pipeline(synthetic=True)


def _file_chain(model_dir, wavs, out):
    from reverb_b200 import recognize_wav
    from reverb_b200.diarization import infer, words2speakers
    assert infer.main(wavs + ["--out-dir", str(out / "rttm"), "--synthetic"]) == 0
    recognize_wav.main(["--model", model_dir, "--audio_file", *wavs, "--result_dir", str(out / "asr"),
                        "--modes", *MODES, "--chunk_size", "300", "--batch_size", "4"])
    stms = {}
    for w in wavs:
        stem = os.path.splitext(os.path.basename(w))[0]
        for mode in MODES:
            dst = out / f"{stem}.{mode}.stm"
            words2speakers.main([str(out / "rttm" / f"{stem}.rttm"), str(out / "asr" / mode / f"{stem}.ctm"), str(dst)])
            stms[(w, mode)] = dst.read_text()
    return stms


@pytest.mark.parametrize("precision", ["bf16", "fp32"])
def test_stm_api_equals_the_file_chain(model_dirs, recordings, diarization, tmp_path, monkeypatch, precision):
    import reverb_b200
    monkeypatch.setenv("RVB_PRECISION", precision)            # recognize_wav's model follows it
    model_dir = model_dirs["causal_ln"][0]
    want = _file_chain(model_dir, recordings, tmp_path)
    for w in recordings:
        stem = os.path.splitext(os.path.basename(w))[0]
        assert (tmp_path / "rttm" / f"{stem}.rttm").read_text(), f"no speaker turns in {w}"
    asr = reverb_b200.load_model(model_dir, precision=precision)
    got = list(asr.transcribe_files(recordings, MODES, format="stm", diarization=diarization, chunk_size=300,
                                    batch_size=4))
    assert [p for p, _ in got] == recordings
    for w, outputs in got:
        for mode, text in zip(MODES, outputs):
            assert text == want[(w, mode)], (w, mode)
    for w in recordings:
        assert asr.transcribe(w, mode=MODES[1], format="stm", diarization=diarization, chunk_size=300,
                              batch_size=4) == want[(w, MODES[1])]
    assert any(len({ln.split()[2] for ln in text.splitlines()}) > 1 for text in want.values()), \
        "no transcript has two speakers"


def test_recognize_wav_writes_stm_and_rttm(model_dirs, recordings, tmp_path):
    from reverb_b200 import recognize_wav
    model_dir = model_dirs["causal_ln"][0]
    want = _file_chain(model_dir, recordings, tmp_path / "chain")
    out = tmp_path / "cli"
    recognize_wav.main(["--model", model_dir, "--audio_file", *recordings, "--result_dir", str(out),
                        "--modes", *MODES, "--chunk_size", "300", "--batch_size", "4", "--diarization_synthetic"])
    for w in recordings:
        stem = os.path.splitext(os.path.basename(w))[0]
        assert (out / "rttm" / f"{stem}.rttm").read_text() == (tmp_path / "chain" / "rttm" / f"{stem}.rttm").read_text()
        for mode in MODES:
            assert (out / mode / f"{stem}.stm").read_text() == want[(w, mode)]
            assert (out / mode / f"{stem}.ctm").read_text() == \
                (tmp_path / "chain" / "asr" / mode / f"{stem}.ctm").read_text()
