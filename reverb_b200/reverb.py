"""`ReverbASR` / `load_model` — the public Python API, a drop-in for the reference's
asr/wenet/cli/reverb.py (same class, method names, argument names, defaults and error
behaviour), running on the native H100 engine.

Differences that are deliberate and documented in DESIGN.md:
  * the model always runs on a CUDA device (`gpu < 0` selects the current device; there
    is no CPU path), whereas the reference's `load_model()` is CPU-only (reverb.py:354-357);
  * RIFF/WAVE audio (PCM 8/16/24/32 bit, float, extensible, multi-channel) is parsed by
    reverb_b200/audio_io.py with torchaudio.load(normalize=False) value conventions, other
    containers go through torchaudio when it has a decoder backend; a file that is not
    16 kHz is resampled on the GPU with torchaudio.transforms.Resample's algorithm
    (csrc/resample.cu + resample.py), where the reference calls torchaudio on the CPU.
"""
from __future__ import annotations

import logging
import math
import queue
import shutil
import threading
from collections import deque
from functools import partial
from math import ceil
from pathlib import Path
from typing import Dict, Generator, Iterator, List, Tuple

import numpy as np
import torch
import torch.nn.functional as F
import yaml

from . import corpus
from .asr_model import ASRModel, alignment_result
from .context_graph import ContextGraph, tokenize
from .ctc_align import adjust_model_time_offset, ctc_align, ctc_align_ms, frames_to_ms, hyps_to_ctm, hyps_to_txt
from .engine import Engine, check_alignable, check_beam_size
from .resample import resampled_length
from .search import DecodeResult
from .text import get_blank_id, init_tokenizer

_FRAME_DOWNSAMPLING_FACTOR = {"linear": 1, "conv2d": 4, "conv2d6": 6, "conv2d8": 8}
CACHED_MODELS_DIR = Path.home() / ".cache/reverb"
_MODELS = {"reverb_asr_v1": "https://huggingface.co/Revai/reverb-asr"}


def _read_wav(path: str, device=None) -> Tuple[np.ndarray, int]:
    """samples (channels, n) + sample rate — the `torchaudio.load(normalize=False)` contract (audio_io.py); FLAC
    frames are decoded on `device`."""
    from .audio_io import load_audio
    return load_audio(path, device)


def _load_state_dict(checkpoint: str) -> Dict[str, torch.Tensor]:
    """utils/checkpoint.py:29-80: flat state_dict, optional {'model0': sd} wrapper."""
    sd = torch.load(checkpoint, map_location="cpu", mmap=False)
    if isinstance(sd, dict) and "model0" in sd:
        sd = sd["model0"]
    return sd


class ReverbASR:
    def __init__(self, config, checkpoint, cmvn_path: str | None = None, tokenizer_symbols: str | None = None,
                 bpe_path: str | None = None, gpu: int = -1, overwrite_cmvn: bool = False,
                 precision: str | None = None):
        self.jit = False
        if not torch.cuda.is_available():
            raise RuntimeError("reverb_b200.ReverbASR needs a CUDA device (H100, sm_90a); no CPU fallback exists")
        self.device = torch.device("cuda", gpu if gpu >= 0 else torch.cuda.current_device())
        self.checkpoint = checkpoint
        with open(config, "r") as fin:
            self.configs = yaml.load(fin, Loader=yaml.FullLoader)
        self.configs["cmvn_conf"]["cmvn_file"] = self._make_path_absolute(
            self.configs["cmvn_conf"]["cmvn_file"], cmvn_path)
        self.configs["tokenizer_conf"]["symbol_table_path"] = self._make_path_absolute(
            self.configs["tokenizer_conf"]["symbol_table_path"], tokenizer_symbols)
        self.configs["tokenizer_conf"]["bpe_path"] = self._make_path_absolute(
            self.configs["tokenizer_conf"]["bpe_path"], bpe_path)
        self.tokenizer = init_tokenizer(self.configs)
        self.blank_id = get_blank_id(self.configs, self.tokenizer.symbol_table)
        self.configs["output_dim"] = len(self.tokenizer.symbol_table)

        sd = _load_state_dict(checkpoint)
        # utils/init_model.py:102-117 + load_checkpoint: GlobalCMVN exists only when `cmvn: global_cmvn`; it is built
        # from the stats file and then overwritten by the checkpoint's buffers when the checkpoint holds them.
        # cli/reverb.py:80-85: `overwrite_cmvn` puts the file's stats back (the reference reads the top-level
        # `cmvn_file` / `is_json_cmvn` keys there; the cmvn_conf entries are accepted as well).
        input_dim = self.configs.get("input_dim", 80)
        if self.configs.get("cmvn", None) == "global_cmvn":
            from .cmvn import load_cmvn
            have = "encoder.global_cmvn.mean" in sd and "encoder.global_cmvn.istd" in sd
            ow_file = self.configs.get("cmvn_file", self.configs["cmvn_conf"]["cmvn_file"]) if overwrite_cmvn else None
            if ow_file is not None:
                mean, istd = load_cmvn(ow_file, self.configs.get("is_json_cmvn", self.configs["cmvn_conf"]["is_json_cmvn"]))
                have = False
            elif not have:
                mean, istd = load_cmvn(self.configs["cmvn_conf"]["cmvn_file"], self.configs["cmvn_conf"]["is_json_cmvn"])
            if not have:
                sd["encoder.global_cmvn.mean"] = torch.from_numpy(np.asarray(mean)).float()
                sd["encoder.global_cmvn.istd"] = torch.from_numpy(np.asarray(istd)).float()
        else:
            # no GlobalCMVN module in the reference model: the engine's fused (x - mean) * istd becomes the identity
            sd["encoder.global_cmvn.mean"] = torch.zeros(input_dim)
            sd["encoder.global_cmvn.istd"] = torch.ones(input_dim)
        # precision: 'bf16' (default, throughput) or 'fp32' (bf16x3 wgmma passes + fp32 attention: reference-level
        # accuracy, engine.resolve_precision); None -> $RVB_PRECISION.  Not a reference argument: an extension.
        self.engine = Engine(self.configs, sd, self.configs["output_dim"], self.device, precision)
        self.model = ASRModel(self.engine, self.configs, self.configs["output_dim"])
        self.test_conf = self.configs["dataset_conf"]
        self.input_frame_length = self.test_conf["fbank_conf"]["frame_shift"]
        self.output_frame_length = self.input_frame_length * _FRAME_DOWNSAMPLING_FACTOR.get(
            self.configs["encoder_conf"]["input_layer"], 4)
        self._lanes = None

    def set_lanes(self, n_lanes: int):
        """Decode consecutive batches on `n_lanes` concurrent streams / host threads (reverb_b200/pipeline.py).
        1 (default) = the reference's strictly sequential batch loop.  Results do not depend on this setting."""
        from .pipeline import Lanes
        if self._lanes is not None:
            self._lanes.close()
        self._lanes = Lanes(self, n_lanes) if n_lanes > 1 else None

    def _make_path_absolute(self, config_path: str, alternate_path: str | None = None) -> str:
        if alternate_path:
            return alternate_path
        p = Path(config_path)
        if not p.is_absolute():
            p = Path(self.checkpoint).parent / p   # adjacent to the checkpoint
        return p.as_posix()

    # ---------------------------------------------------------------------------------------------
    def compute_feats(self, audio_file: str, resample_rate: int = 16000, num_mel_bins=23, frame_length=25,
                      frame_shift=10, dither=0.0) -> torch.Tensor:
        """(1, m, num_mel_bins) float32 on the device; kernel: csrc/fbank.cu."""
        _check_fbank_conf(num_mel_bins, frame_length, frame_shift, dither, resample_rate)
        rec = self._read_recording(audio_file, resample_rate)
        return self._recording_feats(rec, resample_rate).unsqueeze(0)

    def _read_recording(self, audio_file, resample_rate: int = 16000) -> "_Recording":
        """Reads channel 0 of a recording on the host.  Raises the front end's error for a recording that has fewer
        than 400 samples at `resample_rate`, before anything is uploaded."""
        pcm, sample_rate = _read_wav(audio_file, self.device)
        logging.info(f"detected sample rate: {sample_rate}")
        ch0 = np.array(pcm[0], copy=True)                      # channel 0 (kaldi.fbank channel=-1 -> 0)
        if ch0.dtype != np.int16:
            # `waveform.to(torch.float)` of the reference (cli/reverb.py:124): the sample VALUES as they are (uint8 /
            # int32 / float32) — the kernels take int16 or float32 input
            ch0 = ch0.astype(np.float32)
        n = ch0.shape[0]
        if sample_rate != resample_rate:
            g = math.gcd(int(sample_rate), int(resample_rate))
            n = resampled_length(n, int(sample_rate) // g, int(resample_rate) // g)
        if n < 400:
            raise AssertionError(f"choose a window size 400 that is [2, {n}]")  # torchaudio's check
        return _Recording(audio_file, ch0, sample_rate, int(self.engine.lib.rvb_fbank_num_frames(n)))

    def _recording_feats(self, rec: "_Recording", resample_rate: int = 16000) -> torch.Tensor:
        """Upload, resampling and fbank of one recording on the current stream -> (m, 80) float32."""
        wave_dev = torch.from_numpy(rec.pcm).pin_memory().to(self.device, non_blocking=True)
        if rec.sample_rate != resample_rate:
            # torchaudio.transforms.Resample on channel 0 (the reference resamples every channel, then keeps the first)
            wave_dev = self.engine.resample(wave_dev, rec.sample_rate, resample_rate)
        feats = self.engine.fbank(wave_dev)
        assert feats.shape[0] == rec.frames
        return feats

    def feats_batcher(self, infeats: torch.Tensor, chunk_size: int, batch_size: int
                      ) -> Generator[Tuple[torch.Tensor, torch.Tensor], None, None]:
        """Fixed-length chunks with no overlap; only the final chunk is zero-padded (in feature space)."""
        nbins = self.test_conf["fbank_conf"]["num_mel_bins"]
        per_batch = chunk_size * batch_size
        num_batches = ceil(infeats.shape[1] / per_batch)
        for b in range(num_batches):
            fb = infeats[:, b * per_batch:(b + 1) * per_batch, :]
            lens = torch.tensor([chunk_size] * batch_size, dtype=torch.int32)
            if b == num_batches - 1:
                last = ceil(fb.shape[1] / chunk_size)
                lens = torch.tensor([chunk_size] * last, dtype=torch.int32)
                pad = chunk_size * last - fb.shape[1]
                if pad > 0:
                    lens[-1] -= pad
                    fb = F.pad(fb, (0, 0, 0, pad, 0, 0), mode="constant", value=0)
            yield fb.reshape(-1, chunk_size, nbins), lens

    def transcribe_modes(self, audio_file, modes: List[str], format: str = "txt", verbatimicity: float = 1.0,
                         chunk_size: int = 2051, batch_size: int = 1, beam_size: int = 10,
                         decoding_chunk_size: int = -1, num_decoding_left_chunks: int = -1, ctc_weight: float = 0.1,
                         simulate_streaming: bool = False, reverse_weight: float = 0.0, blank_penalty: float = 0.0,
                         length_penalty: float = 0.0, timings_adjustment: float = 230, context_graph=None,
                         diarization=None) -> list[str]:
        """context_graph: phrases to boost in ctc_prefix_beam_search / attention_rescoring (ReverbASR.context_graph, or
        either ContextGraph form); the other modes ignore it, like the reference's decode().
        format="stm" with `diarization` (a SpeakerDiarization, e.g. diarization.infer.load_pipeline()): a speaker on
        every word, see transcribe_files."""
        for _, outputs in self.transcribe_files(
                [audio_file], modes, format=format, verbatimicity=verbatimicity, chunk_size=chunk_size,
                batch_size=batch_size, beam_size=beam_size, decoding_chunk_size=decoding_chunk_size,
                num_decoding_left_chunks=num_decoding_left_chunks, ctc_weight=ctc_weight,
                simulate_streaming=simulate_streaming, reverse_weight=reverse_weight, blank_penalty=blank_penalty,
                length_penalty=length_penalty, timings_adjustment=timings_adjustment, context_graph=context_graph,
                diarization=diarization):
            pass
        return outputs

    def transcribe_files(self, audio_files, modes: List[str], format: str = "txt", verbatimicity=1.0,
                         chunk_size: int = 2051, batch_size: int = 1, beam_size: int = 10,
                         decoding_chunk_size: int = -1, num_decoding_left_chunks: int = -1, ctc_weight: float = 0.1,
                         simulate_streaming: bool = False, reverse_weight: float = 0.0, blank_penalty: float = 0.0,
                         length_penalty: float = 0.0, timings_adjustment: float = 230,
                         context_graph=None, diarization=None) -> Iterator[Tuple[str, List[str]]]:
        """Transcribes many recordings with one set of decode settings -> (audio_file, [output per mode]) in input
        order, each as soon as it and every earlier recording are decoded.  Every output is the one
        `transcribe_modes(audio_file, ...)` gives on its own.

        verbatimicity: one value for every file, or a sequence with one value per file (0.0 = nonverbatim ... 1.0 =
        verbatim).  Files with different values still share batches: each chunk's row carries its file's value.

        Batches hold chunks of several recordings, and tail chunks run at a trimmed length (reverb_b200/corpus.py,
        DESIGN.md §4f).  Files are read and parsed on a background thread, one window of recordings ahead; upload,
        resampling, fbank and decoding run on the caller's thread and current stream (or the lanes of `set_lanes`).
        A file that cannot be read, or has under 400 samples, raises the error `transcribe` raises, naming the file,
        after the outputs of every earlier file; no batch holding its chunks is decoded.

        format="stm" needs `diarization` (a SpeakerDiarization, e.g. diarization.infer.load_pipeline()) and only it
        takes one.  Each output is then the STM that the file chain diarization.infer (RTTM, uri = the file's stem) ->
        recognize_wav (CTM) -> words2speakers writes, byte for byte.  Diarization runs once per recording, on all of its
        channels downmixed (infer.read_audio; the ASR reads channel 0), on the caller's thread and current stream as
        the recording is yielded."""
        audio_files = list(audio_files)
        per_file = isinstance(verbatimicity, (list, tuple, np.ndarray, torch.Tensor))
        if per_file:                      # fail before any audio is read
            verbatimicity = [float(v) for v in verbatimicity]
            if len(verbatimicity) != len(audio_files):
                raise ValueError(f"verbatimicity has {len(verbatimicity)} values for {len(audio_files)} audio files; "
                                 "give one value, or one per file")
        if (format == "stm") != (diarization is not None):   # fail before any audio is read
            raise ValueError('format="stm" and diarization= go together: a speaker-attributed transcript needs a '
                             'SpeakerDiarization, and only format="stm" uses one')
        check_beam_size(beam_size)        # fail before any audio is read / decoded (limit: engine.MAX_BEAM_SIZE)
        if context_graph is not None:     # upload (and check) the graph once, before any audio is read
            context_graph = self.engine.device_context_graph(context_graph, self.blank_id)
        fc = self.test_conf["fbank_conf"]
        _check_fbank_conf(fc["num_mel_bins"], fc["frame_length"], fc["frame_shift"])
        # tails keep the padded length where the padding is part of the result: simulate_streaming has no padding
        # mask, and the attention mode's beam search runs up to T' steps
        trim = not simulate_streaming and "attention" not in modes
        right = corpus.right_context(self.configs["encoder_conf"])
        cat_embs = None if per_file else torch.tensor([verbatimicity, 1.0 - verbatimicity])
        kw = dict(decoding_chunk_size=decoding_chunk_size, num_decoding_left_chunks=num_decoding_left_chunks,
                  ctc_weight=ctc_weight, simulate_streaming=simulate_streaming, reverse_weight=reverse_weight,
                  context_graph=context_graph, blank_id=self.blank_id, blank_penalty=blank_penalty,
                  length_penalty=length_penalty, infos={"tasks": ["transcribe"], "langs": ["en"]}, cat_embs=cat_embs)

        def decode_batch(model, batch):
            return model.decode(modes, batch[0], batch[1], beam_size, **(kw if len(batch) == 2 else
                                                                        dict(kw, cat_embs=batch[2])))

        first = [0]                          # input index of the next recording the reader hands over

        def window_batches(window):
            jobs = self._window_batches(window, chunk_size, batch_size, right, trim)
            if not per_file:
                return jobs
            v = verbatimicity[first[0]:first[0] + len(window)]
            first[0] += len(window)
            # one [v, 1 - v] row per chunk, built as the single-file call builds its vector
            return [(plan, fb, fl, torch.tensor([[v[r], 1.0 - v[r]] for r, _ in plan.slots]))
                    for plan, fb, fl in jobs]

        reader = _Reader(self, audio_files, corpus.window_frames(batch_size, chunk_size))
        waiting: deque = deque()             # recordings not yet yielded, in input order
        stream = None
        try:
            # decode() and decode_stream run without autograd themselves; no grad-mode context spans a yield here
            if self._lanes is not None:
                def decoded():
                    for window in reader:
                        waiting.extend(window)
                        jobs = window_batches(window)
                        for job, res in zip(jobs, self._lanes.run([job[1:] for job in jobs], decode_batch)):
                            yield (job[0], window), res
            else:
                plans: deque = deque()

                def batches():
                    for window in reader:
                        waiting.extend(window)
                        for plan, *batch in window_batches(window):
                            plans.append((plan, window))
                            yield tuple(batch)

                # one software-pipelined decode_stream across window boundaries
                stream = self.model.decode_stream(batches(), modes, beam_size, **kw)

                def decoded():
                    for res in stream:
                        plan, window = plans.popleft()
                        yield (plan, window), res

            for (plan, window), res in decoded():
                for s, (r, c) in enumerate(plan.slots):
                    rec = window[r]
                    for mode in modes:
                        rec.hyps.setdefault(mode, {})[c] = res[mode][s]
                    rec.left -= 1
                while waiting and waiting[0].left == 0:
                    rec = waiting.popleft()
                    outputs = [get_output("ctm" if diarization is not None else format, self.tokenizer,
                                          Path(rec.path).name, [rec.hyps[mode][c] for c in range(rec.chunks)],
                                          timings_adjustment, chunk_size, self.input_frame_length,
                                          self.output_frame_length) for mode in modes]
                    if diarization is not None:
                        outputs = speaker_outputs(diarization, rec.path, outputs)[1]
                    yield rec.path, outputs
        finally:
            if stream is not None:
                stream.close()
            reader.close()
        if reader.error is not None:
            raise reader.error

    def _window_batches(self, window: List["_Recording"], chunk_size: int, batch_size: int, right: int, trim: bool):
        """Features of a window of recordings -> [(corpus.Batch, feats (B, T, 80), lens (B,) int32)] in the order of
        corpus.plan_window.  A row is the chunk's frames followed by zeros, as feats_batcher pads the last chunk."""
        feats = [self._recording_feats(rec) for rec in window]
        for rec in window:
            rec.pcm = None
        nbins = feats[0].shape[1]
        for rec in window:
            rec.chunks = rec.left = len(corpus.chunk_lengths(rec.frames, chunk_size))
        plan = corpus.plan_window([rec.frames for rec in window], chunk_size, batch_size, right, trim)
        starts = np.cumsum([0] + [f.shape[0] for f in feats])
        flat = torch.cat(feats + [feats[0].new_zeros(1, nbins)])
        zero_row = int(starts[-1])
        out = []
        for b in plan:
            first = torch.tensor([int(starts[r]) + c * chunk_size for r, c in b.slots], dtype=torch.int64)
            lens = torch.tensor(b.lens, dtype=torch.int32)
            first_d = first.pin_memory().to(self.device, non_blocking=True)
            lens_d = lens.to(torch.int64).pin_memory().to(self.device, non_blocking=True)
            t = torch.arange(b.T, device=self.device)
            rows = torch.where(t < lens_d[:, None], first_d[:, None] + t, zero_row)
            out.append((b, flat.index_select(0, rows.reshape(-1)).view(len(b.slots), b.T, nbins), lens))
        return out

    def transcribe(self, audio_file, mode: str = "ctc_prefix_beam_search", format: str = "txt",
                   verbatimicity: float = 1.0, chunk_size: int = 2051, batch_size: int = 1, beam_size: int = 10,
                   decoding_chunk_size: int = -1, num_decoding_left_chunks: int = -1, ctc_weight: float = 0.1,
                   simulate_streaming: bool = False, reverse_weight: float = 0.0, blank_penalty: float = 0.0,
                   length_penalty: float = 0.0, timings_adjustment: float = 230, context_graph=None,
                   diarization=None) -> str:
        """format: "txt", "ctm", or "stm" with `diarization` (speaker-attributed words, see transcribe_files)."""
        return self.transcribe_modes(
            audio_file, modes=[mode], format=format, verbatimicity=verbatimicity, chunk_size=chunk_size,
            batch_size=batch_size, beam_size=beam_size, decoding_chunk_size=decoding_chunk_size,
            num_decoding_left_chunks=num_decoding_left_chunks, ctc_weight=ctc_weight,
            simulate_streaming=simulate_streaming, reverse_weight=reverse_weight, blank_penalty=blank_penalty,
            length_penalty=length_penalty, timings_adjustment=timings_adjustment, context_graph=context_graph,
            diarization=diarization)[0]

    def context_graph(self, phrases, score: float = 6.0) -> ContextGraph:
        """A context biasing graph over `phrases` — a file with one phrase per line, or a list of strings — tokenized
        with this model's symbol table and sentencepiece model like the reference's ContextGraph; `score` is the bonus
        per matched token.  Pass it as `context_graph=` to transcribe / transcribe_modes."""
        bpe = self.configs["tokenizer_conf"].get("bpe_path")
        return ContextGraph(context_score=score, token_lists=tokenize(phrases, self.tokenizer.symbol_table, bpe))


    def transcript_ids(self, transcript) -> List[int]:
        """A transcript as token ids: a string goes through the model's sentencepiece pieces (pieces outside the symbol
        table map to <unk> and are kept, so that every word keeps its place), a list of ids is taken as it is."""
        if isinstance(transcript, str):
            ids = self.tokenizer.tokens2ids(self.tokenizer.text2tokens(transcript))
        else:
            ids = [int(t) for t in transcript]
        if len(ids) == 0:
            raise ValueError("reverb_b200: the transcript is empty, nothing to align")
        bad = [t for t in ids if t is None or not 0 <= t < len(self.tokenizer.symbol_table) or t == self.blank_id]
        if bad:
            raise ValueError(f"reverb_b200: transcript token ids {bad[:5]} are not non-blank ids of the symbol table")
        return ids

    def align(self, audio_file, transcript, format: str = "ctm", verbatimicity: float = 1.0, chunk_size: int = 2051,
              batch_size: int = 1, blank_penalty: float = 0.0, timings_adjustment: float = 230) -> str:
        """Forced alignment of a known transcript (text or token ids) to a recording of any length -> CTM / text.
        The encoder runs in the usual independent chunks, `batch_size` at a time; the valid log-prob rows of every chunk
        are pushed into ONE Viterbi trellis (Engine.aligner, on the search side stream, under the next batch's encoder),
        so the transcript is aligned to the whole recording, with no anchoring."""
        if format not in ("ctm", "txt"):
            raise ValueError("Invalid output format.")
        result, times_ms = self.align_tokens(audio_file, self.transcript_ids(transcript), verbatimicity, chunk_size,
                                             batch_size, blank_penalty)
        words = ctc_align_ms(result.tokens, times_ms, result.tokens_confidence, self.tokenizer, self.output_frame_length)
        if timings_adjustment != 0:
            words = adjust_model_time_offset(words, timings_adjustment)
        if format == "txt":
            return " ".join(hyps_to_txt(words))
        return "\n".join(hyps_to_ctm(Path(audio_file).name, words))

    def align_tokens(self, audio_file, ids: List[int], verbatimicity: float = 1.0, chunk_size: int = 2051,
                     batch_size: int = 1, blank_penalty: float = 0.0, want_loglik: bool = False,
                     workspace_budget_bytes: int = 0) -> Tuple[DecodeResult, List[int]]:
        """-> (DecodeResult with frames counted over the valid encoder frames of all chunks, per-token peak time in ms)."""
        fc = self.test_conf["fbank_conf"]
        feats = self.compute_feats(audio_file, num_mel_bins=fc["num_mel_bins"], frame_length=fc["frame_length"],
                                   frame_shift=fc["frame_shift"])
        n = feats.shape[1]
        feat_lens = [chunk_size] * (n // chunk_size) + ([n % chunk_size] if n % chunk_size else [])
        chunk_frames = [int(self.engine.lib.rvb_encoder_out_len(fl, chunk_size)) for fl in feat_lens]
        check_alignable(ids, sum(chunk_frames))
        cat_embs = torch.tensor([verbatimicity, 1.0 - verbatimicity])
        aligner = self.engine.aligner(ids, sum(chunk_frames), self.blank_id, want_loglik, workspace_budget_bytes)
        try:
            with torch.no_grad():
                c = 0
                for feats_batch, feats_lengths in self.feats_batcher(feats, chunk_size, batch_size):
                    enc_out, enc_lens = self.model._forward_encoder(feats_batch, feats_lengths, cat_embs)
                    logp = self.model.ctc_logprobs(enc_out, blank_penalty, self.blank_id)
                    for b in range(logp.shape[0]):
                        assert int(enc_lens[b]) == chunk_frames[c]
                        aligner.push(logp[b, :chunk_frames[c]])
                        c += 1
            result = alignment_result(aligner.finish())
        finally:
            aligner.abort()
        return result, frames_to_ms(result.times, chunk_frames, chunk_size * self.input_frame_length,
                                    self.output_frame_length)


def _check_fbank_conf(num_mel_bins, frame_length, frame_shift, dither=0.0, resample_rate=16000):
    if num_mel_bins != 80 or frame_length != 25 or frame_shift != 10 or dither != 0.0 or resample_rate != 16000:
        raise NotImplementedError("reverb_b200 fbank kernel is built for 80 bins / 25 ms / 10 ms / no dither @16 kHz")


class _Recording:
    """One recording of a transcribe_files call: channel 0 on the host, and its chunks' results as they arrive."""

    def __init__(self, path, pcm: np.ndarray, sample_rate: int, frames: int):
        self.path, self.pcm, self.sample_rate, self.frames = path, pcm, sample_rate, frames
        self.chunks = self.left = 0
        self.hyps: Dict[str, Dict[int, DecodeResult]] = {}


def _name_file(e: BaseException, path) -> BaseException:
    """`e`, or the same kind of exception with the file's name in front of its message."""
    if str(path) in str(e):
        return e
    try:
        named = type(e)(f"{path}: {e}")
    except Exception:
        return e
    named.__cause__ = e
    return named


class _Reader:
    """Reads and parses recordings on one background thread and hands them over in windows (corpus.WindowPacker),
    one window ahead of the decoder.  Iteration ends before the first file that cannot be read; its error, naming
    the file, is then in `error`."""

    def __init__(self, asr: ReverbASR, files: list, budget: int):
        self.error = None
        self._q: queue.Queue = queue.Queue(maxsize=1)
        self._stop = threading.Event()
        self._thread = threading.Thread(target=self._run, args=(asr, files, budget), daemon=True,
                                        name="reverb-reader")
        self._thread.start()

    def _put(self, item) -> bool:
        while not self._stop.is_set():
            try:
                self._q.put(item, timeout=0.1)
                return True
            except queue.Full:
                pass
        return False

    def _run(self, asr, files, budget):
        packer = corpus.WindowPacker(budget)
        try:
            for f in files:
                try:
                    rec = asr._read_recording(f)
                except Exception as e:
                    window = packer.flush()
                    if not window or self._put(window):
                        self._put(_name_file(e, f))
                    return
                window = packer.add(rec.frames, rec)
                if window and not self._put(window):
                    return
            window = packer.flush()
            if window:
                self._put(window)
        finally:
            self._put(None)

    def __iter__(self):
        while True:
            item = self._q.get()
            if item is None:
                return
            if isinstance(item, BaseException):
                self.error = item
                return
            yield item

    def close(self):
        self._stop.set()
        self._thread.join()


def get_output(format: str, tokenizer, audio_name: str, hyps: List[DecodeResult], timings_adjustment_ms: int,
               chunk_size: int, input_frame_length: int, output_frame_length: int) -> str:
    """One hypothesis per chunk -> words -> CTM lines / text (reference: cli/reverb.py:292-321)."""
    if format == "txt":
        render, delimiter = hyps_to_txt, " "
    elif format == "ctm":
        render, delimiter = partial(hyps_to_ctm, audio_name), "\n"
    else:
        raise ValueError("Invalid output format.")
    lines: List[str] = []
    time_shift_ms = 0
    for hyp in hyps:
        words = ctc_align(hyp.tokens, hyp.times, hyp.tokens_confidence, tokenizer, output_frame_length, time_shift_ms)
        words = adjust_model_time_offset(words, timings_adjustment_ms)
        time_shift_ms += chunk_size * input_frame_length
        lines.extend(render(words))
    return delimiter.join(lines)


def speaker_outputs(diarization, audio_file, ctms: List[str]) -> Tuple[str, List[str]]:
    """Diarizes `audio_file` -> (its RTTM as diarization.infer writes it, [the STM words2speakers writes from each
    CTM]).  The turns and words round-trip through the RTTM and CTM text, so the STM is the file chain's."""
    import os
    from .diarization.infer import read_audio
    from .diarization.words2speakers import rttm_text, stm_text
    uri = os.path.splitext(os.path.basename(str(audio_file)))[0]
    device = getattr(getattr(diarization, "segmentation", None), "device", None)   # any callable diarizes
    rttm = rttm_text(uri, diarization(read_audio(str(audio_file), device)))
    return rttm, [stm_text(uri, rttm, ctm) for ctm in ctms]


def load_model(model: str, gpu: int = -1, precision: str | None = None) -> ReverbASR:
    """Loads a reverb model from a directory (config.yaml + first *.pt) or by pretrained name."""
    if Path(model).exists():
        model_dir = Path(model)
        config_path = model_dir / "config.yaml"
        checkpoint_path = list(model_dir.glob("*.pt"))[0]
    elif model in _MODELS:
        model_dir = CACHED_MODELS_DIR / model
        config_path = model_dir / "config.yaml"
        checkpoint_path = model_dir / f"{model}.pt"
        if not (CACHED_MODELS_DIR.exists() and model_dir.exists() and config_path.exists()
                and checkpoint_path.exists()):
            CACHED_MODELS_DIR.parent.mkdir(exist_ok=True, parents=True)
            shutil.rmtree(model_dir, ignore_errors=True)
            download_model(_MODELS[model], model_dir)
    else:
        raise ValueError("Please specify a local path to a model or one of our pretrained models: "
                         f"{','.join(get_available_models())}")
    config_path, checkpoint_path = config_path.resolve(), checkpoint_path.resolve()
    logging.info(f"Loading the model with {config_path = } and {checkpoint_path = }")
    return ReverbASR(str(config_path), str(checkpoint_path), gpu=gpu, precision=precision)


def get_available_models():
    return list(_MODELS.keys())


def download_model(url: str, root: str):
    """Clones the model repository at `url` into `root` (needs network + GitPython)."""
    from git import Repo
    Repo.clone_from(url, root)
