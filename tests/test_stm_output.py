"""Speaker-attributed transcripts assembled in memory (words2speakers.stm_text, reverb.speaker_outputs) equal the file
chain RTTM file -> CTM file -> write_stm byte for byte, and format="stm" / diarization= are checked before any audio
is read."""
import wave

import numpy as np
import pytest

CTM = "\n".join([
    "call.wav 0 0.00 0.40 hello 1.00",
    "call.wav 0 0.52 0.31 there 0.97",
    "call.wav 0 1.90 0.00 uh 0.50",          # zero duration: no overlap, nearest turn
    "call.wav 0 2.95 0.30 both 0.88",        # overlaps two speakers
    "call.wav 0 4.40 0.20 gap 0.91",         # between turns
    "call.wav 0 9.00 0.25 late 0.99",        # after the last turn
])


def _turns():
    from reverb_b200.diarization.rttm import Turn
    return [Turn(0.017, 1.2345, "SPEAKER_00"), Turn(2.5, 3.1, "SPEAKER_01"), Turn(3.0, 4.0, "SPEAKER_00"),
            Turn(5.0, 7.25, "SPEAKER_01")]


def _file_chain(tmp_path, uri, turns, ctm):
    from reverb_b200.diarization.rttm import write_rttm
    from reverb_b200.diarization.words2speakers import write_stm
    with open(tmp_path / f"{uri}.rttm", "w") as f:
        write_rttm(f, uri, turns)
    (tmp_path / f"{uri}.ctm").write_text(ctm)
    write_stm(str(tmp_path / f"{uri}.rttm"), str(tmp_path / f"{uri}.ctm"), str(tmp_path / f"{uri}.stm"))
    return (tmp_path / f"{uri}.rttm").read_text(), (tmp_path / f"{uri}.stm").read_text()


@pytest.mark.parametrize("ctm", [CTM, CTM + "\n", "", CTM.replace("\n", "\r\n")])
def test_stm_text_equals_write_stm_on_files(tmp_path, ctm):
    from reverb_b200.diarization.words2speakers import rttm_text, stm_text
    rttm_file, stm_file = _file_chain(tmp_path, "call", _turns(), ctm)
    rttm = rttm_text("call", _turns())
    assert rttm == rttm_file
    assert stm_text("call", rttm, ctm) == stm_file
    if ctm:
        assert "SPEAKER_00" in stm_file and "SPEAKER_01" in stm_file


def test_speaker_outputs_diarizes_the_downmix_once(tmp_path):
    """speaker_outputs reads the recording the way diarization.infer does (all channels downmixed, / 32768) and turns
    one diarization into one STM per CTM."""
    from reverb_b200.diarization.infer import read_audio
    from reverb_b200.reverb import speaker_outputs
    rng = np.random.default_rng(0)
    pcm = (rng.normal(size=(16000, 2)) * 3000).astype(np.int16)
    path = tmp_path / "call.wav"
    with wave.open(str(path), "wb") as w:
        w.setnchannels(2)
        w.setsampwidth(2)
        w.setframerate(16000)
        w.writeframes(pcm.tobytes())
    seen = []

    def diarization(audio):
        seen.append(np.asarray(audio))
        return _turns()

    ctms = [CTM, CTM.replace("hello", "hi")]
    rttm, stms = speaker_outputs(diarization, str(path), ctms)
    assert len(seen) == 1
    assert np.array_equal(seen[0], read_audio(str(path)))
    assert np.allclose(seen[0], pcm.astype(np.float32).mean(axis=1) / 32768.0)
    rttm_file, stm0 = _file_chain(tmp_path, "call", _turns(), ctms[0])
    _, stm1 = _file_chain(tmp_path, "call", _turns(), ctms[1])
    assert rttm == rttm_file and stms == [stm0, stm1]


def test_stm_format_and_diarization_go_together():
    """Both mismatches raise ValueError before the (missing) file is opened."""
    from reverb_b200.reverb import ReverbASR
    asr = ReverbASR.__new__(ReverbASR)                 # the check precedes any use of the model
    with pytest.raises(ValueError, match="diarization"):
        asr.transcribe("does-not-exist.wav", format="stm")
    with pytest.raises(ValueError, match="diarization"):
        asr.transcribe_modes("does-not-exist.wav", ["attention_rescoring"], format="ctm", diarization=lambda a: [])
    with pytest.raises(ValueError, match="diarization"):
        next(asr.transcribe_files(["does-not-exist.wav"], ["ctc_greedy_search"], format="txt", diarization=lambda a: []))
