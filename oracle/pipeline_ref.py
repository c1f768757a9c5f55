"""ORACLE (test infrastructure, never shipped): the whole hot path on the CPU, assembled from
the restated pieces (fbank_np, model_ref, search_ref) — the CPU twin of the reference's
`ReverbASR.transcribe_modes` -> `ASRModel.decode` (asr/wenet/cli/reverb.py:176-248,
asr/wenet/transformer/asr_model.py:331-432).

Used (a) as the checker in tests/ and __graft_entry__.smoke(), (b) as the timed CPU
baseline / `--impl reference` arm of bench.py (the tests and the benchmark do not need the
Python reference itself).  It executes the same ATen CPU operators as the reference does
(conv2d / linear / matmul / softmax / layer_norm), so its timing is representative.
"""
from __future__ import annotations

import glob
import os
import wave
from typing import Dict, List

import numpy as np
import torch
import yaml

from . import fbank_np, model_ref, search_ref


def read_wav_int16(path: str):
    with wave.open(path, "rb") as w:
        assert w.getsampwidth() == 2
        sr, nch = w.getframerate(), w.getnchannels()
        pcm = np.frombuffer(w.readframes(w.getnframes()), dtype=np.int16).reshape(-1, nch)
    return pcm[:, 0].astype(np.float32), sr


class OracleASR:
    def __init__(self, model_dir: str):
        with open(os.path.join(model_dir, "config.yaml")) as f:
            self.cfg = yaml.safe_load(f)
        ckpt = sorted(glob.glob(os.path.join(model_dir, "*.pt")))[0]
        sd = torch.load(ckpt, map_location="cpu")
        if "model0" in sd:                      # utils/checkpoint.py:29-80
            sd = sd["model0"]
        self.sd = {k: v.float() for k, v in sd.items() if v.is_floating_point()}
        self.vocab = self.sd["ctc.ctc_lo.weight"].shape[0]
        self.sos = self.eos = self.vocab - 1    # asr_model.py:79-82
        self.blank_id = 0

    # asr/wenet/cli/reverb.py:113-140
    def compute_feats(self, wav_path: str) -> torch.Tensor:
        x, sr = read_wav_int16(wav_path)
        assert sr == 16000
        return torch.from_numpy(fbank_np.fbank(x)).unsqueeze(0)

    # asr/wenet/cli/reverb.py:142-174
    @staticmethod
    def feats_batcher(feats: torch.Tensor, chunk_size: int, batch_size: int):
        m = feats.shape[1]
        per = chunk_size * batch_size
        nb = -(-m // per)
        for b in range(nb):
            fb = feats[:, b * per:(b + 1) * per, :]
            nchunks = -(-fb.shape[1] // chunk_size)
            lens = torch.full((nchunks,), chunk_size, dtype=torch.int32)
            pad = nchunks * chunk_size - fb.shape[1]
            if pad > 0:
                lens[-1] -= pad
                fb = torch.nn.functional.pad(fb, (0, 0, 0, pad))
            yield fb.reshape(-1, chunk_size, feats.shape[2]), lens

    @torch.no_grad()
    def forward_encoder(self, feats, lens, cat_embs, decoding_chunk_size: int = -1, num_decoding_left_chunks: int = -1):
        return model_ref.encoder_forward(feats, lens, self.sd, self.cfg, cat_embs, decoding_chunk_size,
                                         num_decoding_left_chunks)

    @torch.no_grad()
    def decode(self, methods: List[str], feats: torch.Tensor, lens: torch.Tensor, beam_size: int = 10,
               ctc_weight: float = 0.0, reverse_weight: float = 0.0, cat_embs=None,
               blank_penalty: float = 0.0, return_intermediates: bool = False, length_penalty: float = 0.0,
               decoding_chunk_size: int = -1, num_decoding_left_chunks: int = -1) -> Dict:
        """asr/wenet/transformer/asr_model.py:331-432 (attention / greedy / prefix / rescoring)."""
        enc, enc_lens, _ = self.forward_encoder(feats, lens, cat_embs, decoding_chunk_size, num_decoding_left_chunks)
        ctc_probs = model_ref.ctc_logprobs(enc, self.sd, blank_penalty, self.blank_id)
        out = {}
        if "attention" in methods:
            out["attention"] = self.attention_beam_search(enc, enc_lens, beam_size, length_penalty, cat_embs)
        if "ctc_greedy_search" in methods:
            out["ctc_greedy_search"] = search_ref.ctc_greedy_search(ctc_probs, enc_lens, self.blank_id)
        prefix = None
        if "ctc_prefix_beam_search" in methods or "attention_rescoring" in methods:
            prefix = search_ref.ctc_prefix_beam_search(ctc_probs, enc_lens, beam_size, self.blank_id)
            if "ctc_prefix_beam_search" in methods:
                out["ctc_prefix_beam_search"] = prefix
        if "attention_rescoring" in methods:
            out["attention_rescoring"] = self.attention_rescoring(prefix, enc, enc_lens, ctc_weight,
                                                                  reverse_weight, cat_embs)
        if return_intermediates:
            out["_encoder_out"], out["_encoder_lens"], out["_ctc_probs"] = enc, enc_lens, ctc_probs
        return out

    @torch.no_grad()
    def attention_beam_search(self, enc, enc_lens, beam_size, length_penalty, cat_embs):
        """asr/wenet/transformer/search.py:251-360: every utterance's memory is repeated beam_size times (:266-269)."""
        B, Tp, d = enc.shape
        mem = enc.unsqueeze(1).repeat(1, beam_size, 1, 1).view(B * beam_size, Tp, d)
        mem_lens = enc_lens.view(-1, 1).repeat(1, beam_size).view(-1)

        def step(hyps):
            return model_ref.decoder_step_logp(mem, mem_lens, hyps, self.sd, self.cfg, cat_embs).topk(beam_size)
        return search_ref.attention_beam_search(step, B, Tp, beam_size, self.sos, self.eos, length_penalty)

    @torch.no_grad()
    def attention_rescoring(self, prefix_results, enc, enc_lens, ctc_weight, reverse_weight, cat_embs):
        """asr/wenet/transformer/search.py:363-448 + asr_model.py:868-978."""
        results = []
        use_right = reverse_weight > 0 and self.cfg["decoder_conf"].get("r_num_blocks", 0) > 0 \
            and any(k.startswith("decoder.right_decoder") for k in self.sd)
        for b in range(enc.shape[0]):
            hyps = prefix_results[b].nbest
            ys, ylens = search_ref.rescoring_inputs(hyps, self.sos, self.eos)
            mem = enc[b, :int(enc_lens[b])].unsqueeze(0).repeat(len(hyps), 1, 1)
            dec = model_ref.decoder_forward(mem, ys, ylens, self.sd, self.cfg, "left_decoder", cat_embs)
            dec = torch.log_softmax(dec, dim=-1)
            rdec = None
            if use_right:
                rys = model_ref.reverse_hyps(ys, ylens, self.eos)
                rdec = model_ref.decoder_forward(mem, rys, ylens, self.sd, self.cfg, "right_decoder", cat_embs)
                rdec = torch.log_softmax(rdec, dim=-1)
            results.append(search_ref.rescoring_combine(hyps, prefix_results[b].nbest_scores,
                                                        prefix_results[b].nbest_times, dec, rdec,
                                                        ctc_weight, reverse_weight, self.eos))
        return results

    def transcribe_hyps(self, wav_path: str, modes: List[str], chunk_size: int = 2051, batch_size: int = 1,
                        beam_size: int = 10, ctc_weight: float = 0.1, reverse_weight: float = 0.0,
                        verbatimicity: float = 1.0):
        feats = self.compute_feats(wav_path)
        cat = torch.tensor([verbatimicity, 1.0 - verbatimicity])
        res = []
        for fb, fl in self.feats_batcher(feats, chunk_size, batch_size):
            res.append(self.decode(modes, fb, fl, beam_size, ctc_weight=ctc_weight,
                                   reverse_weight=reverse_weight, cat_embs=cat))
        return {m: [h for r in res for h in r[m]] for m in modes}
