"""Host-side handle of the native model plan (librvb_b200.so): PyTorch tensors in, PyTorch
tensors / Python lists out.  PyTorch is used for device memory and streams only; every
FLOP of the hot path runs in the hand-written sm_90a kernels behind the C ABI.
"""
from __future__ import annotations

import ctypes as C
import weakref
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch

from . import _lib
from ._lib import ModelConfig, check


# beam width the search kernels are built for (PB_MAXBEAM in csrc/ctc.cu; top-k <= 16 in logsoftmax_topk_kernel).
# The reference accepts any --beam_size; its CLI default is 10.
MAX_BEAM_SIZE = 16


def check_beam_size(beam_size: int) -> None:
    if not 1 <= int(beam_size) <= MAX_BEAM_SIZE:
        raise ValueError(f"reverb_b200: beam_size={beam_size} is outside the supported range 1..{MAX_BEAM_SIZE} "
                         "(the GPU prefix-beam / top-k kernels keep the beam in shared memory)")


def _ptr(t: Optional[torch.Tensor]):
    return None if t is None else C.c_void_p(t.data_ptr())


def _np_ptr(a: Optional[np.ndarray]):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def nbest_lists(toks, tims, olen, scores, nhyp) -> List[Tuple[List[tuple], List[float], List[List[int]]]]:
    """An n-best as arrays (Engine.prefix_beam_search_raw, Engine.rescoring_collect) -> per utterance
    (nbest tokens [tuple], nbest scores [float], nbest times [list])."""
    out = []
    for b in range(toks.shape[0]):
        n = int(nhyp[b])
        out.append(([tuple(toks[b, r, :olen[b, r, 0]].tolist()) for r in range(n)],
                    [float(s) for s in scores[b, :n]],
                    [tims[b, r, :olen[b, r, 1]].tolist() for r in range(n)]))
    return out


PRECISIONS = {"bf16": 0, "fp32": 1, "bf16x3": 1}


def resolve_precision(precision: Optional[str]) -> str:
    """'bf16' (default: bf16 tensor-core operands, fp32 accumulation — the throughput mode) or 'fp32' (= 'bf16x3': every
    GEMM runs as three wgmma passes over (hi, lo) bf16 operand pairs and the attention in fp32 — reference-level
    accuracy at ~3x the tensor work).  None -> environment variable RVB_PRECISION, else 'bf16'."""
    import os
    p = precision if precision is not None else os.environ.get("RVB_PRECISION", "bf16")
    if p not in PRECISIONS:
        raise ValueError(f"reverb_b200: precision must be one of {sorted(PRECISIONS)}, got {p!r}")
    return "fp32" if PRECISIONS[p] == 1 else "bf16"


def model_config_from_yaml(configs: Dict, vocab: int, precision: str = "bf16") -> ModelConfig:
    """config.yaml (SURVEY.md §5) -> rvb_model_config.  Only the architecture the hot path supports
    (conformer encoder with conv2d input / rel_pos attention, (bi)transformer decoder) is accepted."""
    ec, dc = configs["encoder_conf"], configs.get("decoder_conf", {})
    if configs.get("encoder", "conformer") != "conformer":
        raise ValueError(f"unsupported encoder type {configs.get('encoder')!r} (only 'conformer')")
    if ec.get("input_layer", "conv2d") != "conv2d":
        raise ValueError("only input_layer: conv2d (Conv2dSubsampling4) is supported")
    if ec.get("pos_enc_layer_type", "rel_pos") != "rel_pos" or \
            ec.get("selfattention_layer_type", "rel_selfattn") != "rel_selfattn":
        raise ValueError("only rel_pos / rel_selfattn encoders are supported")
    if ec.get("activation_type", "swish") != "swish":
        raise ValueError("only activation_type: swish is supported")
    if not ec.get("macaron_style", True) or not ec.get("use_cnn_module", True) or not ec.get("normalize_before", True):
        raise ValueError("only macaron-style pre-norm Conformer blocks with the CNN module are supported")
    ds = configs.get("dataset_conf", {})
    num_langs = ds.get("cat_emb_conf", {}).get("emb_len", 0) if ds.get("pass_cat_emb", False) else 0
    r_blocks = dc.get("r_num_blocks", 0)
    cfg = ModelConfig()
    cfg.input_dim = configs.get("input_dim", 80)
    cfg.d_model = ec.get("output_size", 256)
    cfg.heads = ec.get("attention_heads", 4)
    cfg.ffn_dim = ec.get("linear_units", 2048)
    cfg.num_blocks = ec.get("num_blocks", 6)
    cfg.cnn_kernel = ec.get("cnn_module_kernel", 15)
    cfg.causal = int(bool(ec.get("causal", False)))
    cfg.cnn_layer_norm = int(ec.get("cnn_module_norm", "batch_norm") == "layer_norm")
    cfg.num_langs = num_langs
    cfg.vocab = vocab
    cfg.dec_heads = dc.get("attention_heads", 4)
    cfg.dec_ffn_dim = dc.get("linear_units", 2048)
    cfg.dec_blocks = dc.get("num_blocks", 6)
    cfg.r_dec_blocks = r_blocks
    # asr_model.py:79-82: <sos>/<eos> from tokenizer_conf.special_tokens, else vocab - 1 for both
    st = (configs.get("tokenizer_conf") or {}).get("special_tokens") or {}
    cfg.sos_id = int(st.get("<sos>", vocab - 1))
    cfg.eos_id = int(st.get("<eos>", vocab - 1))
    cfg.precision = PRECISIONS[precision]
    return cfg


class DeviceContextGraph:
    """A context biasing graph uploaded to the device once (include/rvb_b200.h rvb_context_graph_*), for searches
    whose vocabulary has `vocab` entries and whose blank is `blank_id`.  Built from either graph form
    (context_graph.device_tables); a malformed graph raises ValueError before anything reaches the device.  The native
    handle is freed with this object, after the searches enqueued with it have finished."""

    def __init__(self, graph, vocab: int, blank_id: int = 0, device: Optional[torch.device] = None):
        from .context_graph import check_device_tables, device_tables
        t = device_tables(graph)
        check_device_tables(t, int(vocab), int(blank_id))
        self.lib = _lib.load()
        self.vocab, self.blank_id, self.num_states = int(vocab), int(blank_id), int(t["fail"].shape[0])
        self._h = None
        a = {k: np.ascontiguousarray(v, dtype=np.float64 if v.dtype == np.float64 else np.int32) for k, v in t.items()}
        with torch.cuda.device(device if device is not None else torch.cuda.current_device()):
            h = self.lib.rvb_context_graph_create(self.num_states, _np_ptr(a["off"]), _np_ptr(a["tok"]),
                                                  _np_ptr(a["dst"]), _np_ptr(a["fail"]), _np_ptr(a["bonus"]),
                                                  _np_ptr(a["emit"]), _np_ptr(a["token_score"]), self.vocab,
                                                  self.blank_id)
        if not h:
            raise ValueError("rvb_context_graph_create failed: " + _lib.last_error())
        self._h = C.c_void_p(h)

    def __del__(self):
        try:
            if self._h is not None:
                self.lib.rvb_context_graph_destroy(self._h)
                self._h = None
        except Exception:
            pass


# host graph -> {(device index, vocab, blank): DeviceContextGraph}: a graph object is uploaded once, not per batch
_device_graphs: "weakref.WeakKeyDictionary" = weakref.WeakKeyDictionary()


class Engine:
    """Owns one `rvb_model` (packed weights + workspace) on one CUDA device."""

    def __init__(self, configs: Dict, state_dict: Dict[str, torch.Tensor], vocab: int, device: torch.device,
                 precision: Optional[str] = None):
        if device.type != "cuda" or not torch.cuda.is_available():
            raise RuntimeError("reverb_b200 needs a CUDA device (sm_90a); there is no CPU path")
        self.lib = _lib.load()
        self.device = device
        self.precision = resolve_precision(precision)
        self.cfg = model_config_from_yaml(configs, vocab, self.precision)
        self.d_model = self.cfg.d_model
        self.vocab = vocab
        self.num_langs = self.cfg.num_langs
        self._h = None
        with torch.cuda.device(device):
            h = self.lib.rvb_model_create(C.byref(self.cfg))
            if not h:
                raise RuntimeError("rvb_model_create failed: " + _lib.last_error())
            self._h = C.c_void_p(h)
            for name, t in state_dict.items():
                if not torch.is_tensor(t) or not t.is_floating_point():
                    continue
                a = t.detach().to("cpu", torch.float32).contiguous()
                check(self.lib.rvb_model_set_tensor(self._h, name.encode("utf8"), C.c_void_p(a.data_ptr()), a.numel()),
                      f"rvb_model_set_tensor({name})")
            check(self.lib.rvb_model_finalize(self._h), "rvb_model_finalize")
        self.has_right_decoder = any(k.startswith("decoder.right_decoder.") for k in state_dict)

    def fork(self) -> "Engine":
        """A second plan over the same device weights with its own workspace (for a second stream / host thread).
        The parent engine must stay alive as long as the fork is used."""
        other = Engine.__new__(Engine)
        other.lib, other.device, other.cfg = self.lib, self.device, self.cfg
        other.precision = self.precision
        other.d_model, other.vocab, other.num_langs = self.d_model, self.vocab, self.num_langs
        other.has_right_decoder = self.has_right_decoder
        other._parent = self
        with torch.cuda.device(self.device):
            h = self.lib.rvb_model_fork(self._h)
        if not h:
            raise RuntimeError("rvb_model_fork failed: " + _lib.last_error())
        other._h = C.c_void_p(h)
        return other

    def __del__(self):
        try:
            if self._h is not None and self.lib is not None:
                self.lib.rvb_model_destroy(self._h)
                self._h = None
        except Exception:
            pass

    # ------------------------------------------------------------------ helpers
    def _stream(self):
        return C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

    def _cat(self, cat_embs) -> Tuple[Optional[np.ndarray], int]:
        """cat_embs (num_langs,) or (B, num_langs), one row per utterance -> (flat float32 array, n_cat); the native
        call checks n_cat against both lengths."""
        if self.num_langs == 0:
            return None, 0
        if cat_embs is None:
            raise ValueError("cat_embs is required by a model with language-specific layers")
        a = np.ascontiguousarray(torch.as_tensor(cat_embs).detach().cpu().numpy().astype(np.float32).reshape(-1))
        return a, int(a.shape[0])

    def encoder_out_frames(self, T: int) -> int:
        return int(self.lib.rvb_encoder_out_frames(int(T)))

    # ------------------------------------------------------------------ hot path
    def fbank(self, wave: torch.Tensor) -> torch.Tensor:
        """(N,) float32 or int16 samples on the device (int16-VALUED) -> (m, 80) float32."""
        assert wave.is_cuda and wave.dim() == 1 and wave.is_contiguous()
        n = wave.numel()
        m = int(self.lib.rvb_fbank_num_frames(n))
        feats = torch.empty((m, 80), dtype=torch.float32, device=wave.device)
        with torch.cuda.device(self.device):
            if wave.dtype == torch.int16:
                check(self.lib.rvb_fbank_i16(_ptr(wave), n, _ptr(feats), m, self._stream()), "rvb_fbank_i16")
            elif wave.dtype == torch.float32:
                check(self.lib.rvb_fbank_f32(_ptr(wave), n, _ptr(feats), m, self._stream()), "rvb_fbank_f32")
            else:
                raise TypeError(f"fbank: unsupported dtype {wave.dtype}")
        return feats

    def resample(self, wave: torch.Tensor, orig_freq: int, new_freq: int) -> torch.Tensor:
        """(N,) float32 or int16 on the device -> (ceil(N * new / orig),) float32: torchaudio.transforms.Resample
        semantics (cli/reverb.py:125-128) with the convolution on the GPU."""
        from .resample import resampled_length, sinc_resample_kernel
        assert wave.is_cuda and wave.dim() == 1 and wave.stride(0) == 1
        if wave.dtype not in (torch.int16, torch.float32):
            raise TypeError(f"resample: unsupported dtype {wave.dtype}")
        kern, orig, new, width = sinc_resample_kernel(int(orig_freq), int(new_freq))
        key = (int(orig_freq), int(new_freq))
        if not hasattr(self, "_resample_tables"):
            self._resample_tables = {}
        if key not in self._resample_tables:
            self._resample_tables[key] = torch.from_numpy(kern).to(self.device)
        n_in = wave.shape[0]
        n_out = resampled_length(n_in, orig, new)
        out = torch.empty(n_out, dtype=torch.float32, device=wave.device)
        with torch.cuda.device(self.device):
            check(self.lib.rvb_resample(_ptr(wave), int(wave.dtype == torch.int16), n_in, _ptr(self._resample_tables[key]),
                                        orig, new, width, _ptr(out), n_out, self._stream()), "rvb_resample")
        return out

    def fbank_batch(self, waves: torch.Tensor) -> torch.Tensor:
        """(B, N) equal-length recordings (float32 or int16, on the device) -> (B, m, 80) float32, one launch."""
        assert waves.is_cuda and waves.dim() == 2 and waves.stride(1) == 1
        B, n = waves.shape
        if B == 1 and waves.stride(0) < n:        # a size-1 dimension may carry any stride
            waves = waves.reshape(-1).view(1, n)
        m = int(self.lib.rvb_fbank_num_frames(n))
        feats = torch.empty((B, m, 80), dtype=torch.float32, device=waves.device)
        if waves.dtype not in (torch.int16, torch.float32):
            raise TypeError(f"fbank: unsupported dtype {waves.dtype}")
        with torch.cuda.device(self.device):
            check(self.lib.rvb_fbank_batch(_ptr(waves), int(waves.dtype == torch.int16), B, waves.stride(0), n,
                                           _ptr(feats), m, self._stream()), "rvb_fbank_batch")
        return feats

    def forward_encoder(self, feats: torch.Tensor, feat_lens: Sequence[int], cat_embs=None, chunk_size: int = -1,
                        num_left_chunks: int = -1, streaming: bool = False):
        """(B, T, 80) fp32 cuda -> (encoder_out (B, T', d) fp32 cuda, encoder_lens np.int32 (B,)).
        chunk_size > 0: bounded attention context (decoding_chunk_size / num_decoding_left_chunks of the reference)."""
        assert feats.is_cuda and feats.dtype == torch.float32 and feats.dim() == 3
        feats = feats.contiguous()
        B, T, _ = feats.shape
        Tp = self.encoder_out_frames(T)
        lens = np.ascontiguousarray(np.asarray(feat_lens, dtype=np.int32).reshape(-1))
        assert lens.shape[0] == B
        enc_lens = np.zeros(B, dtype=np.int32)
        out = torch.empty((B, Tp, self.d_model), dtype=torch.float32, device=feats.device)
        cat, ncat = self._cat(cat_embs)
        with torch.cuda.device(self.device):
            if streaming:
                # forward_chunk_by_chunk semantics (simulate_streaming): no padding masks, chunk-local context
                assert chunk_size > 0
                check(self.lib.rvb_encoder_forward_streaming(self._h, _ptr(feats), B, T, _np_ptr(cat), ncat,
                                                             int(chunk_size), int(num_left_chunks), _ptr(out),
                                                             _np_ptr(enc_lens), self._stream()),
                      "rvb_encoder_forward_streaming")
            elif chunk_size > 0:
                check(self.lib.rvb_encoder_forward_chunked(self._h, _ptr(feats), _np_ptr(lens), B, T, _np_ptr(cat), ncat,
                                                           int(chunk_size), int(num_left_chunks), _ptr(out),
                                                           _np_ptr(enc_lens), self._stream()),
                      "rvb_encoder_forward_chunked")
            else:
                check(self.lib.rvb_encoder_forward(self._h, _ptr(feats), _np_ptr(lens), B, T, _np_ptr(cat), ncat,
                                                   _ptr(out), _np_ptr(enc_lens), self._stream()), "rvb_encoder_forward")
        return out, enc_lens

    def ctc_topk(self, enc_out: torch.Tensor, k: int, blank_penalty: float = 0.0, blank_id: int = 0,
                 want_logp: bool = False):
        B, Tp, _ = enc_out.shape
        val = torch.empty((B, Tp, k), dtype=torch.float32, device=enc_out.device)
        idx = torch.empty((B, Tp, k), dtype=torch.int32, device=enc_out.device)
        logp = torch.empty((B, Tp, self.vocab), dtype=torch.float32, device=enc_out.device) if want_logp else None
        with torch.cuda.device(self.device):
            check(self.lib.rvb_ctc_topk(self._h, _ptr(enc_out.contiguous()), B, Tp, k, float(blank_penalty),
                                        int(blank_id), _ptr(val), _ptr(idx), _ptr(logp), self._stream()),
                  "rvb_ctc_topk")
        return val, idx, logp

    def logp_topk(self, logp: torch.Tensor, k: int):
        """top-k of recorded log-probs (B, T, V) (no softmax)."""
        logp = logp.contiguous()
        B, T, V = logp.shape
        val = torch.empty((B, T, k), dtype=torch.float32, device=logp.device)
        idx = torch.empty((B, T, k), dtype=torch.int32, device=logp.device)
        with torch.cuda.device(self.device):
            check(self.lib.rvb_logp_topk(_ptr(logp), B * T, V, k, _ptr(val), _ptr(idx), self._stream()),
                  "rvb_logp_topk")
        return val, idx

    def greedy_search(self, topk_idx: torch.Tensor, enc_lens, blank_id: int = 0) -> List[List[int]]:
        B, Tp, k = topk_idx.shape
        lens = np.ascontiguousarray(np.asarray(enc_lens, dtype=np.int32))
        toks = np.zeros((B, Tp), dtype=np.int32)
        olen = np.zeros(B, dtype=np.int32)
        with torch.cuda.device(self.device):
            check(self.lib.rvb_ctc_greedy_search(_ptr(topk_idx), k, _np_ptr(lens), B, Tp, int(blank_id),
                                                 _np_ptr(toks), _np_ptr(olen), self._stream()),
                  "rvb_ctc_greedy_search")
        return [toks[b, :olen[b]].tolist() for b in range(B)]

    def device_context_graph(self, graph, blank_id: int = 0) -> DeviceContextGraph:
        """The device copy of a context graph (either form, or a DeviceContextGraph, returned as it is), uploaded on
        first use and cached for as long as the host graph object lives."""
        if isinstance(graph, DeviceContextGraph):
            if graph.blank_id != int(blank_id):
                raise ValueError(f"context graph was checked against blank {graph.blank_id}, the search uses {blank_id}")
            return graph
        key = (self.device.index, self.vocab, int(blank_id))
        try:
            per_graph = _device_graphs.setdefault(graph, {})
        except TypeError:                                  # not weak-referenceable: upload for this call only
            return DeviceContextGraph(graph, self.vocab, blank_id, self.device)
        dg = per_graph.get(key)
        if dg is None:
            dg = per_graph[key] = DeviceContextGraph(graph, self.vocab, blank_id, self.device)
        return dg

    def prefix_beam_search_raw(self, topk_val: torch.Tensor, topk_idx: torch.Tensor, enc_lens, beam: int,
                               blank_id: int = 0, context=None):
        """n-best as arrays: tokens/times (B, beam, max_len) int32, lens (B, beam, 2) = {n_tokens, n_times},
        scores (B, beam) float64, n_hyp (B,).  context: a context graph (biased search, see device_context_graph)."""
        B, Tp, k = topk_idx.shape
        lens = np.ascontiguousarray(np.asarray(enc_lens, dtype=np.int32))
        max_len = max(int(lens.max()) if B else 1, 1)
        toks = np.zeros((B, beam, max_len), dtype=np.int32)
        tims = np.zeros((B, beam, max_len), dtype=np.int32)
        olen = np.zeros((B, beam, 2), dtype=np.int32)
        scores = np.zeros((B, beam), dtype=np.float64)
        nhyp = np.zeros(B, dtype=np.int32)
        dg = None if context is None else self.device_context_graph(context, blank_id)
        fn, graph = ((self.lib.rvb_ctc_prefix_beam_search, ()) if dg is None else
                     (self.lib.rvb_ctc_prefix_beam_search_biased, (dg._h,)))
        with torch.cuda.device(self.device):
            check(fn(_ptr(topk_val), _ptr(topk_idx), k, _np_ptr(lens), B, Tp, beam, int(blank_id), max_len, _np_ptr(toks),
                     _np_ptr(tims), _np_ptr(olen), _np_ptr(scores), _np_ptr(nhyp), *graph, self._stream()), fn.__name__)
        return toks, tims, olen, scores, nhyp

    def prefix_beam_search(self, topk_val: torch.Tensor, topk_idx: torch.Tensor, enc_lens, beam: int,
                           blank_id: int = 0, context=None):
        """-> per utterance (nbest tokens [tuple], nbest scores [float], nbest times [list])."""
        return nbest_lists(*self.prefix_beam_search_raw(topk_val, topk_idx, enc_lens, beam, blank_id, context))

    # ---- prefix beam search (+ attention rescoring) as three stages around a native ticket, so that one host thread
    # can software-pipeline consecutive batches (asr_model.ASRModel.decode_stream): see include/rvb_b200.h
    def search_submit(self, topk_val: torch.Tensor, topk_idx: torch.Tensor, enc_out: torch.Tensor, enc_lens, beam: int,
                      blank_id: int = 0, context=None) -> dict:
        """Enqueue ctc_prefix_beam_search (biased by the context graph `context` when given); returns the ticket (a
        dict that keeps every buffer of the batch, and the device graph, alive)."""
        B, Tp, k = topk_idx.shape
        lens = np.ascontiguousarray(np.asarray(enc_lens, dtype=np.int32))
        enc_out = enc_out.contiguous()
        dg = None if context is None else self.device_context_graph(context, blank_id)
        fn, graph = (self.lib.rvb_search_submit, ()) if dg is None else (self.lib.rvb_search_submit_biased, (dg._h,))
        with torch.cuda.device(self.device):
            tid = fn(self._h, _ptr(topk_val), _ptr(topk_idx), k, _ptr(enc_out), _np_ptr(lens), B, Tp, beam, int(blank_id),
                     *graph, self._stream())
        if tid < 0:
            raise RuntimeError("rvb_search_submit failed: " + _lib.last_error())
        return {"id": tid, "B": B, "Tp": Tp, "beam": beam, "cap": max(int(lens.max()) if B else 1, 1),
                "keep": (topk_val, topk_idx, enc_out, lens, dg), "stage": 1}

    def rescoring_submit(self, t: dict, cat_embs=None, reverse_weight: float = 0.0, run_decoder: bool = True) -> None:
        """Wait for the hypothesis lengths of ticket `t`, then enqueue the decoder passes (attention rescoring) and the
        device -> host copies of the results into page-locked buffers owned by the ticket."""
        B, beam, cap = t["B"], t["beam"], t["cap"]
        n = B * beam
        use_r = run_decoder and reverse_weight > 0.0 and self.has_right_decoder
        # page-locked result buffers: the native call copies straight into them (no staging copy)
        t["toks"] = torch.empty(n * cap, dtype=torch.int32, pin_memory=True)
        t["tims"] = torch.empty(n * cap, dtype=torch.int32, pin_memory=True)
        t["l2r"] = torch.empty(n * (cap + 1), dtype=torch.float32, pin_memory=True) if run_decoder else None
        t["r2l"] = torch.empty(n * (cap + 1), dtype=torch.float32, pin_memory=True) if use_r else None
        L = C.c_int(0)
        cat, ncat = self._cat(cat_embs) if run_decoder else (None, 0)
        with torch.cuda.device(self.device):
            check(self.lib.rvb_rescoring_submit(self._h, t["id"], _np_ptr(cat), ncat, float(reverse_weight), cap,
                                                int(bool(run_decoder)), _ptr(t["toks"]), _ptr(t["tims"]), _ptr(t["l2r"]),
                                                _ptr(t["r2l"]), C.byref(L), self._stream()), "rvb_rescoring_submit")
        t["L"], t["use_r"], t["run_decoder"], t["stage"] = L.value, use_r, bool(run_decoder), 2

    def rescoring_collect(self, t: dict):
        """-> (toks, tims (B, beam, L) int32, olen (B, beam, 2), ctc scores (B, beam) float64, n_hyp (B,), l2r, r2l
        (B, beam, L+1) float32; l2r / r2l None when unused)."""
        B, beam, L = t["B"], t["beam"], t["L"]
        n = B * beam
        olen = np.empty((B, beam, 2), dtype=np.int32)
        scores = np.empty((B, beam), dtype=np.float64)
        nhyp = np.empty(B, dtype=np.int32)
        check(self.lib.rvb_rescoring_collect(self._h, t["id"], _np_ptr(olen), _np_ptr(scores), _np_ptr(nhyp)),
              "rvb_rescoring_collect")
        t["stage"] = 3
        # bytes copied device -> host for this batch (lengths, counts, CTC scores, tokens, times, decoder scores)
        self.last_d2h_bytes = (olen.nbytes + nhyp.nbytes + scores.nbytes + 2 * n * L * 4
                               + (n * (L + 1) * 4 * (2 if t["use_r"] else 1) if t["run_decoder"] else 0))
        toks = t["toks"].numpy()[:n * L].reshape(B, beam, L)
        tims = t["tims"].numpy()[:n * L].reshape(B, beam, L)
        l2r = t["l2r"].numpy()[:n * (L + 1)].reshape(B, beam, L + 1) if t["l2r"] is not None else None
        r2l = t["r2l"].numpy()[:n * (L + 1)].reshape(B, beam, L + 1) if t["r2l"] is not None else None
        return toks, tims, olen, scores, nhyp, l2r, r2l

    def ticket_release(self, t: Optional[dict]) -> None:
        """Abandon a ticket that will not be collected (error paths)."""
        if t is not None and t.get("stage", 3) < 3:
            self.lib.rvb_ticket_release(self._h, t["id"])
            t["stage"] = 3

    def beam_search_rescoring(self, topk_val: torch.Tensor, topk_idx: torch.Tensor, enc_out: torch.Tensor, enc_lens,
                              beam: int, blank_id: int = 0, cat_embs=None, reverse_weight: float = 0.0):
        """ctc_prefix_beam_search + attention_rescoring decoder scores, the n-best never leaving the device in between
        (the three stages above back to back).  -> see rescoring_collect."""
        t = self.search_submit(topk_val, topk_idx, enc_out, enc_lens, beam, blank_id)
        self.rescoring_submit(t, cat_embs, reverse_weight, True)
        return self.rescoring_collect(t)

    def decoder_step_topk(self, enc_out: torch.Tensor, enc_lens, hyps: np.ndarray, n_per_utt: int, cat_embs=None,
                          k: int = 10):
        """One step of `attention` mode: hyps (B*N, L) running hypotheses (sos first) -> log_softmax top-k of the
        left decoder at the last position: (val (B*N, k) float32, idx (B*N, k) int32)."""
        B, Tp, _ = enc_out.shape
        hyps = np.ascontiguousarray(hyps, dtype=np.int32)
        S, L = hyps.shape
        assert S == B * n_per_utt
        lens = np.ascontiguousarray(np.asarray(enc_lens, dtype=np.int32))
        val = np.empty((S, k), dtype=np.float32)
        idx = np.empty((S, k), dtype=np.int32)
        cat, ncat = self._cat(cat_embs)
        with torch.cuda.device(self.device):
            check(self.lib.rvb_decoder_step_topk(self._h, _ptr(enc_out.contiguous()), _np_ptr(lens), B, Tp, n_per_utt,
                                                 _np_ptr(hyps), L, _np_ptr(cat), ncat, k, _np_ptr(val), _np_ptr(idx),
                                                 self._stream()), "rvb_decoder_step_topk")
        return val, idx

    # ---- KV-cached autoregressive decoder step (`attention` mode)
    def decoder_cache_begin(self, enc_out: torch.Tensor, enc_lens, n_per_utt: int, max_steps: int, cat_embs=None) -> None:
        """Project the source-attention keys / values of enc_out once and size the per-layer self-attention caches for
        `max_steps` positions of B * n_per_utt hypotheses (include/rvb_b200.h rvb_decoder_cache_*)."""
        B, Tp, _ = enc_out.shape
        lens = np.ascontiguousarray(np.asarray(enc_lens, dtype=np.int32))
        cat, ncat = self._cat(cat_embs)
        self._cache_keep = enc_out.contiguous()
        self._cache_S = B * n_per_utt
        with torch.cuda.device(self.device):
            check(self.lib.rvb_decoder_cache_begin(self._h, _ptr(self._cache_keep), _np_ptr(lens), B, Tp, n_per_utt,
                                                   int(max_steps), _np_ptr(cat), ncat, self._stream()),
                  "rvb_decoder_cache_begin")

    def decoder_cache_step(self, last_tokens: np.ndarray, parents: Optional[np.ndarray], k: int):
        """last_tokens (S,): the newest token of every hypothesis; parents (S,): the hypothesis (previous order) each
        one extends, None at the first step.  -> (val (S, k) float32, idx (S, k) int32) log_softmax top-k."""
        tok = np.ascontiguousarray(last_tokens, dtype=np.int32).reshape(-1)
        assert tok.shape[0] == self._cache_S
        par = None if parents is None else np.ascontiguousarray(parents, dtype=np.int32).reshape(-1)
        val = np.empty((self._cache_S, k), dtype=np.float32)
        idx = np.empty((self._cache_S, k), dtype=np.int32)
        with torch.cuda.device(self.device):
            check(self.lib.rvb_decoder_cache_step(self._h, _np_ptr(tok), _np_ptr(par), k, _np_ptr(val), _np_ptr(idx),
                                                  self._stream()), "rvb_decoder_cache_step")
        return val, idx

    def decoder_cache_end(self) -> None:
        self.lib.rvb_decoder_cache_end(self._h)
        self._cache_keep = None

    def decoder_step_logp(self, enc_out: torch.Tensor, enc_lens, hyps: np.ndarray, n_per_utt: int, cat_embs=None):
        """hyps (B*N, L) running hypotheses (sos first) -> the full log_softmax rows of the left decoder at the last
        position, (B*N, vocab) float32 (decoder.forward_one_step_with_attn of the reference, for joint_decoding)."""
        B, Tp, _ = enc_out.shape
        hyps = np.ascontiguousarray(hyps, dtype=np.int32)
        S, L = hyps.shape
        assert S == B * n_per_utt
        lens = np.ascontiguousarray(np.asarray(enc_lens, dtype=np.int32))
        out = np.empty((S, self.vocab), dtype=np.float32)
        cat, ncat = self._cat(cat_embs)
        with torch.cuda.device(self.device):
            check(self.lib.rvb_decoder_step_logp(self._h, _ptr(enc_out.contiguous()), _np_ptr(lens), B, Tp, n_per_utt,
                                                 _np_ptr(hyps), L, _np_ptr(cat), ncat, _np_ptr(out), self._stream()),
                  "rvb_decoder_step_logp")
        return out

    def rescoring_scores_raw(self, enc_out: torch.Tensor, enc_lens, toks: np.ndarray, hlen: np.ndarray, cat_embs=None,
                             reverse_weight: float = 0.0):
        """toks (B, N, L) int32 padded hypotheses, hlen (B, N) their lengths (-1 = absent).
        -> (l2r, r2l) float32 (B, N, Lmax+1), see rvb_attention_rescoring; r2l is None when unused."""
        B, Tp, _ = enc_out.shape
        N = toks.shape[1]
        max_len = max(int(hlen.max()), 1)
        toks = np.ascontiguousarray(toks[:, :, :max_len], dtype=np.int32)
        hlen = np.ascontiguousarray(hlen, dtype=np.int32)
        lens = np.ascontiguousarray(np.asarray(enc_lens, dtype=np.int32))
        l2r = np.zeros((B, N, max_len + 1), dtype=np.float32)
        use_r = reverse_weight > 0.0 and self.has_right_decoder
        r2l = np.zeros((B, N, max_len + 1), dtype=np.float32) if use_r else None
        cat, ncat = self._cat(cat_embs)
        with torch.cuda.device(self.device):
            check(self.lib.rvb_attention_rescoring(self._h, _ptr(enc_out.contiguous()), _np_ptr(lens), B, Tp,
                                                   _np_ptr(toks), _np_ptr(hlen), N, max_len, _np_ptr(cat), ncat,
                                                   float(reverse_weight), _np_ptr(l2r), _np_ptr(r2l), self._stream()),
                  "rvb_attention_rescoring")
        return l2r, r2l

    def rescoring_scores(self, enc_out: torch.Tensor, enc_lens, nbest: List[List[tuple]], cat_embs=None,
                         reverse_weight: float = 0.0):
        """Teacher-forced decoder log-probs of every hypothesis token (hypotheses given as lists of tuples)."""
        B = enc_out.shape[0]
        N = max(len(h) for h in nbest)
        max_len = max([len(h) for hs in nbest for h in hs] + [1])
        toks = np.zeros((B, N, max_len), dtype=np.int32)
        hlen = np.full((B, N), -1, dtype=np.int32)
        for b, hs in enumerate(nbest):
            for i, h in enumerate(hs):
                hlen[b, i] = len(h)
                if len(h):
                    toks[b, i, :len(h)] = np.asarray(h, dtype=np.int32)
        return self.rescoring_scores_raw(enc_out, enc_lens, toks, hlen, cat_embs, reverse_weight)


    # ---- CTC forced alignment (csrc/align.cu; include/rvb_b200.h rvb_ctc_force_align / rvb_aligner_*)
    def force_align(self, logp: torch.Tensor, enc_lens, labels: Sequence[Sequence[int]], blank_id: int = 0,
                    want_loglik: bool = False) -> List["Alignment"]:
        """logp (B, Tp, V) fp32 log-probs on the device, one label list per utterance -> one Alignment each."""
        assert logp.is_cuda and logp.dtype == torch.float32 and logp.dim() == 3
        logp = logp.contiguous()
        B, Tp, V = logp.shape
        lens = np.ascontiguousarray(np.asarray(enc_lens, dtype=np.int32).reshape(-1))
        assert lens.shape[0] == B and len(labels) == B
        for b in range(B):
            check_alignable(labels[b], int(lens[b]), f"utterance {b}")
        ulen = np.asarray([len(y) for y in labels], dtype=np.int32)
        max_U = int(ulen.max())
        lab = np.zeros((B, max_U), dtype=np.int32)
        for b, y in enumerate(labels):
            lab[b, :len(y)] = np.asarray(y, dtype=np.int32)
        out = _AlignBuffers(B, Tp, max_U, want_loglik)
        with torch.cuda.device(self.device):
            check(self.lib.rvb_ctc_force_align(_ptr(logp), V, _np_ptr(lens), B, Tp, _np_ptr(lab), _np_ptr(ulen), max_U,
                                               int(blank_id), *out.pointers(), self._stream()), "rvb_ctc_force_align")
        return [out.alignment(b, labels[b], int(lens[b])) for b in range(B)]

    def aligner(self, labels: Sequence[int], total_frames: int, blank_id: int = 0, want_loglik: bool = False,
                budget_bytes: int = 0, side_stream: bool = True) -> "Aligner":
        """One trellis over `total_frames` frames, fed piecewise (Aligner.push) — the form that crosses the encoder
        batches of a long recording.  budget_bytes > 0 bounds the device workspace (Aligner.workspace_bytes)."""
        return Aligner(self, labels, total_frames, blank_id, want_loglik, budget_bytes, side_stream)


class Alignment:
    """Forced alignment of one label sequence: `frames` the token id of every frame (what the reference's force_align
    returns), per label its `first` / `last` / `peak` frame and `peak_logp`, the Viterbi `score` (float32) and, when
    asked for, `loglik` = log p(y | x)."""

    def __init__(self, tokens, frames, first, last, peak, peak_logp, score, loglik=None):
        self.tokens, self.frames, self.first, self.last, self.peak = tokens, frames, first, last, peak
        self.peak_logp, self.score, self.loglik = peak_logp, score, loglik


def check_alignable(labels: Sequence[int], n_frames: int, what: str = "transcript") -> None:
    """An alignment exists iff U >= 1 and T >= U + #(adjacent equal labels): a repeat needs a blank frame in between."""
    U = len(labels)
    if U == 0:
        raise ValueError(f"reverb_b200: {what} is empty, nothing to align")
    need = U + sum(1 for a, b in zip(labels[:-1], labels[1:]) if a == b)
    if n_frames < need:
        raise ValueError(f"reverb_b200: {what} is infeasible: {U} tokens need at least {need} encoder frames, "
                         f"the audio has {n_frames}")


class _AlignBuffers:
    def __init__(self, B: int, T: int, max_U: int, want_loglik: bool):
        self.frames = np.zeros((B, T), dtype=np.int32)
        self.first, self.last, self.peak = (np.zeros((B, max_U), dtype=np.int32) for _ in range(3))
        self.peak_logp = np.zeros((B, max_U), dtype=np.float32)
        self.score = np.zeros(B, dtype=np.float32)
        self.loglik = np.zeros(B, dtype=np.float64) if want_loglik else None

    def pointers(self):
        return [_np_ptr(a) for a in (self.frames, self.first, self.last, self.peak, self.peak_logp, self.score,
                                     self.loglik)]

    def alignment(self, b: int, labels, T: int) -> Alignment:
        U = len(labels)
        return Alignment(list(labels), self.frames[b, :T].copy(), self.first[b, :U].copy(), self.last[b, :U].copy(),
                         self.peak[b, :U].copy(), self.peak_logp[b, :U].copy(), np.float32(self.score[b]),
                         None if self.loglik is None else float(self.loglik[b]))


class Aligner:
    """Handle of the resumable alignment (rvb_aligner_*).  push() enqueues and returns; finish() synchronises."""

    def __init__(self, engine: Engine, labels: Sequence[int], total_frames: int, blank_id: int, want_loglik: bool,
                 budget_bytes: int, side_stream: bool):
        self.engine, self.labels, self.total = engine, [int(t) for t in labels], int(total_frames)
        self.want_loglik = bool(want_loglik)
        check_alignable(self.labels, self.total)
        lab = np.ascontiguousarray(self.labels, dtype=np.int32)
        self._h = None
        with torch.cuda.device(engine.device):
            h = engine.lib.rvb_aligner_begin(engine._h if side_stream else None, _np_ptr(lab), len(self.labels),
                                             self.total, engine.vocab, int(blank_id), int(self.want_loglik),
                                             int(budget_bytes), engine._stream())
        if not h:
            raise RuntimeError("rvb_aligner_begin failed: " + _lib.last_error())
        self._h = C.c_void_p(h)

    @staticmethod
    def workspace_bytes(n_labels: int, total_frames: int, want_loglik: bool = False) -> int:
        return int(_lib.load().rvb_aligner_workspace_bytes(int(n_labels), int(total_frames), int(want_loglik)))

    def push(self, logp_rows: torch.Tensor) -> None:
        """(n, V) fp32 log-probs of the next n frames, on the device."""
        assert logp_rows.is_cuda and logp_rows.dtype == torch.float32 and logp_rows.dim() == 2
        assert logp_rows.shape[1] == self.engine.vocab
        rows = logp_rows.contiguous()
        with torch.cuda.device(self.engine.device):
            check(self.engine.lib.rvb_aligner_push(self._h, _ptr(rows), rows.shape[0], self.engine._stream()),
                  "rvb_aligner_push")

    def finish(self) -> Alignment:
        out = _AlignBuffers(1, self.total, len(self.labels), self.want_loglik)
        h, self._h = self._h, None                     # the native call frees the handle, also when it fails
        with torch.cuda.device(self.engine.device):
            check(self.engine.lib.rvb_aligner_finish(h, *out.pointers(), self.engine._stream()), "rvb_aligner_finish")
        return out.alignment(0, self.labels, self.total)

    def abort(self) -> None:
        if self._h is not None:
            self.engine.lib.rvb_aligner_abort(self._h)
            self._h = None

    def __del__(self):
        try:
            self.abort()
        except Exception:
            pass


def launch_count() -> int:
    return int(_lib.load().rvb_launch_count())
