"""Host side of corpus decoding (reverb_b200/corpus.py, `reverb` with several --audio_file): chunking, batch lengths,
windows and batch order.  No GPU needed."""
import types

import numpy as np
import pytest
import torch

from reverb_b200 import corpus


def _batcher_chunks(n, chunk_size, batch_size):
    """(first frame, valid frames) of every chunk of ReverbASR.feats_batcher over an n-frame recording."""
    from reverb_b200.reverb import ReverbASR
    fake = types.SimpleNamespace(test_conf={"fbank_conf": {"num_mel_bins": 1}})
    feats = torch.arange(1, n + 1, dtype=torch.float32).reshape(1, n, 1)
    out = []
    for fb, lens in ReverbASR.feats_batcher(fake, feats, chunk_size, batch_size):
        for row, fl in zip(fb[:, :, 0], lens.tolist()):
            assert torch.all(row[fl:] == 0)
            out.append((int(row[0]) - 1, fl))
    return out


def _lengths(rng, chunk_size):
    fixed = [1, 3, 6, 7, chunk_size - 1, chunk_size, chunk_size + 1, 2 * chunk_size, 3 * chunk_size + 5]
    return fixed + [int(x) for x in rng.integers(1, 5 * chunk_size, size=30)]


@pytest.mark.parametrize("chunk_size", [50, 2051])
def test_chunks_match_feats_batcher(chunk_size):
    rng = np.random.default_rng(0)
    for n in _lengths(rng, chunk_size):
        lens = corpus.chunk_lengths(n, chunk_size)
        starts = [i * chunk_size for i in range(len(lens))]
        assert list(zip(starts, lens)) == _batcher_chunks(n, chunk_size, 3), n


def test_encoder_length_formulas_match_the_library():
    from reverb_b200 import _lib
    lib = _lib.load()
    for T in (1, 2, 3, 6, 7, 8, 11, 299, 2051, 2998):
        assert corpus.encoder_out_frames(T) == lib.rvb_encoder_out_frames(T)
        for n in (0, 1, 6, 7, 10, 11, T - 1, T, T + 9):
            assert corpus.encoder_out_len(n, T) == lib.rvb_encoder_out_len(n, T), (n, T)


def _check_plan(frames, chunk_size, batch_size, right, trim):
    plan = corpus.plan_window(frames, chunk_size, batch_size, right, trim)
    seen = []
    t_ref = corpus.encoder_out_frames(chunk_size)
    for b in plan:
        assert 1 <= len(b.slots) <= batch_size and len(b.lens) == len(b.slots)
        for (r, c), fl in zip(b.slots, b.lens):
            assert corpus.chunk_lengths(frames[r], chunk_size)[c] == fl
        assert max(b.lens) <= b.T <= chunk_size and b.T >= 7
        if not trim or max(b.lens) == chunk_size:
            assert b.T == chunk_size
        else:
            # the T_b rule: every encoder row a valid row reads is computed
            e = max(corpus.encoder_out_len(fl, chunk_size) for fl in b.lens)
            assert corpus.encoder_out_frames(b.T) >= min(t_ref, e + right)
            # ... and T_b is the shortest such length
            if b.T > max(max(b.lens), 7):
                assert corpus.encoder_out_frames(b.T - 1) < min(t_ref, e + right)
            for fl in b.lens:                 # valid rows do not depend on the batch length
                assert corpus.encoder_out_len(fl, b.T) == corpus.encoder_out_len(fl, chunk_size)
        seen += b.slots
    want = [(r, c) for r, n in enumerate(frames) for c in range(len(corpus.chunk_lengths(n, chunk_size)))]
    assert sorted(seen) == want                 # every chunk in exactly one batch
    if plan:
        assert all(len(plan[0].slots) * plan[0].T >= len(b.slots) * b.T for b in plan)   # largest batch first
    return plan


@pytest.mark.parametrize("right", [0, 7])
@pytest.mark.parametrize("trim", [True, False])
def test_plan_window_invariants(right, trim):
    rng = np.random.default_rng(1)
    for chunk_size in (50, 2051, 2998):
        for batch_size in (1, 3, 64):
            for _ in range(5):
                frames = _lengths(rng, chunk_size)
                rng.shuffle(frames)
                _check_plan(frames[:int(rng.integers(1, len(frames)))], chunk_size, batch_size, right, trim)


def test_plan_window_shapes():
    cs = 2051
    plan = corpus.plan_window([2 * cs + 100, 500, cs, 3], cs, 2, right=7)
    full = [b for b in plan if b.T == cs]
    assert [b.slots for b in full] == [[(0, 0), (0, 1)], [(2, 0)]]     # (recording, chunk) order
    tails = [b for b in plan if b.T < cs]
    assert [b.slots for b in tails] == [[(1, 0), (0, 2)], [(3, 0)]]    # longest first
    assert tails[0].T == 4 * ((500 - 3) // 4 + 7) + 3                  # e + r encoder rows
    assert tails[1].T == 4 * 7 + 3                                     # len < 7 + 4r
    # e within r of T'_ref: the batch runs at the full length
    t_ref = corpus.encoder_out_frames(cs)
    near = 4 * (t_ref - 3) + 3
    assert corpus.plan_window([near], cs, 4, right=7)[0].T == cs
    assert corpus.plan_window([near], cs, 4, right=0)[0].T == near
    # simulate_streaming / attention mode: no trimming
    assert all(b.T == cs for b in corpus.plan_window([100, 2 * cs + 1], cs, 4, right=0, trim=False))


def test_windows_keep_recordings_whole_and_in_order():
    rng = np.random.default_rng(2)
    frames = [int(x) for x in rng.integers(1, 9000, size=200)] + [50_000, 3, 12_000]
    for budget in (1, 5_000, 20_000, 10 ** 9):
        packer, windows = corpus.WindowPacker(budget), []
        for i, n in enumerate(frames):
            w = packer.add(n, i)
            if w:
                windows.append(w)
        windows.append(packer.flush())
        assert [i for w in windows for i in w] == list(range(len(frames)))    # input order, each once
        for w in windows:
            assert len(w) == 1 or sum(frames[i] for i in w) <= budget
    assert corpus.window_frames(64, 2998) == corpus.WINDOW_BATCHES * 64 * 2998


def test_cli_several_files_and_duplicate_stems(tmp_path):
    from reverb_b200.recognize_wav import get_args, main, output_names
    a = get_args(["--audio_file", "a.wav", "d/b.wav", "c.flac", "--result_dir", "o", "--model", "m"])
    assert a.audio_file == ["a.wav", "d/b.wav", "c.flac"]
    assert get_args(["--audio_file", "a.wav", "--result_dir", "o"]).audio_file == ["a.wav"]
    assert output_names(a.audio_file) == ["a.ctm", "b.ctm", "c.ctm"]
    with pytest.raises(SystemExit):
        get_args(["--audio_file", "--result_dir", "o"])
    # the same stem twice is refused before any model is loaded (the model directory does not exist)
    with pytest.raises(ValueError, match="a.ctm"):
        main(["--audio_file", "x/a.wav", "y/a.flac", "--result_dir", str(tmp_path), "--model", str(tmp_path / "no")])
    assert not (tmp_path / "attention_rescoring").exists()
