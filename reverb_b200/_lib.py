"""ctypes binding of the C ABI declared in include/rvb_b200.h (librvb_b200.so, sm_90a).

This is the only place the Python host code touches native code.  There is no CPU
fallback: if the shared library is missing or a call fails, a RuntimeError is raised.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Optional

_HERE = os.path.dirname(os.path.abspath(__file__))
# RVB_LIB_PATH: A/B tuning aid (tools/gemm_bench.py against an older build); the product always loads the in-tree library
LIB_PATH = os.environ.get("RVB_LIB_PATH") or os.path.join(_HERE, "librvb_b200.so")


class ModelConfig(C.Structure):
    """Mirror of `rvb_model_config` (include/rvb_b200.h)."""
    _fields_ = [(n, C.c_int) for n in (
        "input_dim", "d_model", "heads", "ffn_dim", "num_blocks", "cnn_kernel", "causal",
        "cnn_layer_norm", "num_langs", "vocab", "dec_heads", "dec_ffn_dim", "dec_blocks", "r_dec_blocks",
        "sos_id", "eos_id", "precision")]


class SegConfig(C.Structure):
    """Mirror of `rvb_seg_config` (include/rvb_diar.h)."""
    _fields_ = [(n, C.c_int) for n in (
        "sample_rate", "sinc_filters", "sinc_kernel", "sinc_stride", "conv_channels", "conv_kernel", "lstm_hidden",
        "lstm_layers", "linear_dim", "linear_layers", "num_classes")]


class WavlmSegConfig(C.Structure):
    """Mirror of `rvb_wavlm_seg_config` (include/rvb_diar.h)."""
    _fields_ = [(n, C.c_int) for n in (
        "sample_rate", "conv_channels", "embed_dim", "num_layers", "num_heads", "ffn_dim", "pos_conv_kernel",
        "pos_conv_groups", "num_buckets", "max_distance", "lstm_hidden", "lstm_layers", "linear_dim", "linear_layers",
        "num_classes")]


class EmbConfig(C.Structure):
    """Mirror of `rvb_emb_config` (include/rvb_diar.h)."""
    _fields_ = [("sample_rate", C.c_int), ("num_mel_bins", C.c_int), ("m_channels", C.c_int), ("embed_dim", C.c_int),
                ("blocks", C.c_int * 4)]


_vp, _i, _f, _ll = C.c_void_p, C.c_int, C.c_float, C.c_longlong

# name -> (restype, argtypes); must list every symbol the header declares (tests/test_abi.py checks)
SIGNATURES = {
    "rvb_last_error": (C.c_char_p, []),
    "rvb_launch_count": (C.c_ulonglong, []),
    "rvb_held_bytes": (_i, [_vp, _vp]),
    "rvb_set_gemm_impl": (_i, [_i]),
    "rvb_get_gemm_impl": (_i, []),
    "rvb_gemm_profile_begin": (_i, []),
    "rvb_gemm_profile_end": (_i, [_vp, _vp, _vp]),
    "rvb_model_create": (_vp, [C.POINTER(ModelConfig)]),
    "rvb_model_set_tensor": (_i, [_vp, C.c_char_p, _vp, _ll]),
    "rvb_model_finalize": (_i, [_vp]),
    "rvb_model_fork": (_vp, [_vp]),
    "rvb_model_destroy": (None, [_vp]),
    "rvb_encoder_out_frames": (_i, [_i]),
    "rvb_encoder_out_len": (_i, [_i, _i]),
    "rvb_fbank_num_frames": (_ll, [_ll]),
    "rvb_fbank_f32": (_i, [_vp, _ll, _vp, _ll, _vp]),
    "rvb_fbank_i16": (_i, [_vp, _ll, _vp, _ll, _vp]),
    "rvb_fbank_batch": (_i, [_vp, _i, _i, _ll, _ll, _vp, _ll, _vp]),
    "rvb_encoder_forward": (_i, [_vp, _vp, _vp, _i, _i, _vp, _i, _vp, _vp, _vp]),
    "rvb_encoder_forward_chunked": (_i, [_vp, _vp, _vp, _i, _i, _vp, _i, _i, _i, _vp, _vp, _vp]),
    "rvb_encoder_forward_streaming": (_i, [_vp, _vp, _i, _i, _vp, _i, _i, _i, _vp, _vp, _vp]),
    "rvb_ctc_topk": (_i, [_vp, _vp, _i, _i, _i, _f, _i, _vp, _vp, _vp, _vp]),
    "rvb_logp_topk": (_i, [_vp, _i, _i, _i, _vp, _vp, _vp]),
    "rvb_ctc_greedy_search": (_i, [_vp, _i, _vp, _i, _i, _i, _vp, _vp, _vp]),
    "rvb_resample": (_i, [_vp, _i, _ll, _vp, _i, _i, _i, _vp, _ll, _vp]),
    "rvb_ctc_prefix_beam_search": (_i, [_vp, _vp, _i, _vp, _i, _i, _i, _i, _i, _vp, _vp, _vp, _vp, _vp, _vp]),
    "rvb_beam_search_rescoring": (_i, [_vp, _vp, _vp, _i, _vp, _vp, _i, _i, _i, _i, _vp, _i, _f, _i, _vp, _vp, _vp, _vp, _vp,
                                       _vp, _vp, _vp, _vp]),
    "rvb_search_submit": (_i, [_vp, _vp, _vp, _i, _vp, _vp, _i, _i, _i, _i, _vp]),
    "rvb_search_submit_biased": (_i, [_vp, _vp, _vp, _i, _vp, _vp, _i, _i, _i, _i, _vp, _vp]),
    "rvb_context_graph_create": (_vp, [_i, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i]),
    "rvb_context_graph_destroy": (None, [_vp]),
    "rvb_ctc_prefix_beam_search_biased": (_i, [_vp, _vp, _i, _vp, _i, _i, _i, _i, _i, _vp, _vp, _vp, _vp, _vp, _vp,
                                               _vp]),
    "rvb_rescoring_submit": (_i, [_vp, _i, _vp, _i, _f, _i, _i, _vp, _vp, _vp, _vp, _vp, _vp]),
    "rvb_rescoring_collect": (_i, [_vp, _i, _vp, _vp, _vp]),
    "rvb_ticket_release": (_i, [_vp, _i]),
    "rvb_decoder_step_topk": (_i, [_vp, _vp, _vp, _i, _i, _i, _vp, _i, _vp, _i, _i, _vp, _vp, _vp]),
    "rvb_decoder_cache_begin": (_i, [_vp, _vp, _vp, _i, _i, _i, _i, _vp, _i, _vp]),
    "rvb_decoder_cache_step": (_i, [_vp, _vp, _vp, _i, _vp, _vp, _vp]),
    "rvb_decoder_cache_end": (_i, [_vp]),
    "rvb_decoder_step_logp": (_i, [_vp, _vp, _vp, _i, _i, _i, _vp, _i, _vp, _i, _vp, _vp]),
    "rvb_attention_rescoring": (_i, [_vp, _vp, _vp, _i, _i, _vp, _vp, _i, _i, _vp, _i, _f, _vp, _vp, _vp]),
    "rvb_ctc_force_align": (_i, [_vp, _i, _vp, _i, _i, _vp, _vp, _i, _i, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "rvb_aligner_workspace_bytes": (_ll, [_i, _i, _i]),
    "rvb_aligner_begin": (_vp, [_vp, _vp, _i, _i, _i, _i, _i, _ll, _vp]),
    "rvb_aligner_push": (_i, [_vp, _vp, _i, _vp]),
    "rvb_aligner_finish": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "rvb_aligner_abort": (None, [_vp]),
    "rvb_gemm_bf16": (_i, [_vp, _vp, _vp, _i, _i, _i, _i, _i, _f, _vp, _i, _vp]),
    "rvb_gemm_bf16_rows": (_i, [_vp, _vp, _vp, _i, _i, _i, _i, _i, _f, _vp, _i, _vp, _i, _vp]),
    "rvb_gemm_bf16x3": (_i, [_vp, _vp, _vp, _i, _i, _i, _i, _i, _f, _vp, _i, _vp]),
    "rvb_gemm_grouped": (_i, [_vp, _vp, _vp, _i, _i, _i, _i, _vp, _i, _vp, _i, _i, _i, _vp]),
    "rvb_f32_to_bf16_pair": (_i, [_vp, _vp, _ll, _i, _vp]),
    "rvb_gemm_logsoftmax_gather_ws_bytes": (_ll, [_i, _i]),
    "rvb_gemm_logsoftmax_gather": (_i, [_vp, _vp, _vp, _i, _i, _i, _vp, _vp, _vp, _vp]),
    "rvb_layernorm": (_i, [_vp, _vp, _vp, _f, _i, _i, _vp, _vp, _vp]),
    "rvb_attention": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _vp, _vp,
                           _i, _f, _vp]),
    "rvb_attention_tc_chunked": (_i, [_vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _i, _i, _vp, _vp, _i, _i, _f, _vp]),
    "rvb_attention_tc": (_i, [_vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _i, _i, _vp, _vp, _i, _f, _vp]),
    "rvb_attention_tc_bits": (_i, [_vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _i, _i, _vp, _vp, _i, _vp, _i, _f,
                                   _vp]),
    "rvb_attention_tc_blocks_per_sm": (_i, [_i, _i, _i, _i]),
    "rvb_relpos_prep": (_i, [_vp, _i, _vp, _i, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _vp]),
    "rvb_f32_to_bf16": (_i, [_vp, _vp, _ll, _vp]),
    # include/rvb_diar.h
    "rvb_seg_create": (_vp, [C.POINTER(SegConfig)]),
    "rvb_seg_set_tensor": (_i, [_vp, C.c_char_p, _vp, _ll]),
    "rvb_seg_finalize": (_i, [_vp]),
    "rvb_seg_destroy": (None, [_vp]),
    "rvb_seg_num_frames": (_i, [_vp, _i]),
    "rvb_seg_forward": (_i, [_vp, _vp, _i, _i, _vp, _vp, _vp]),
    "rvb_wavlm_seg_create": (_vp, [C.POINTER(WavlmSegConfig)]),
    "rvb_wavlm_seg_set_tensor": (_i, [_vp, C.c_char_p, _vp, _ll]),
    "rvb_wavlm_seg_finalize": (_i, [_vp]),
    "rvb_wavlm_seg_destroy": (None, [_vp]),
    "rvb_wavlm_seg_num_frames": (_i, [_vp, _i]),
    "rvb_wavlm_seg_forward": (_i, [_vp, _vp, _i, _i, _vp, _vp, _vp, _vp]),
    "rvb_attention_tc_relbias": (_i, [_vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _vp, _vp, _f, _vp]),
    "rvb_emb_create": (_vp, [C.POINTER(EmbConfig)]),
    "rvb_emb_set_tensor": (_i, [_vp, C.c_char_p, _vp, _ll]),
    "rvb_emb_finalize": (_i, [_vp]),
    "rvb_emb_destroy": (None, [_vp]),
    "rvb_emb_num_frames": (_i, [_vp, _i]),
    "rvb_emb_forward": (_i, [_vp, _vp, _i, _i, _vp, _i, _i, _vp, _vp, _vp]),
    "rvb_centroid_linkage_workspace_bytes": (_ll, [_i]),
    "rvb_centroid_linkage": (_i, [_vp, _i, _i, _vp, _vp, _vp, _ll, _vp]),
}

_lib: Optional[C.CDLL] = None


def load() -> C.CDLL:
    """Load librvb_b200.so (built in-tree by reverb_b200/build.py).  Fails loudly if absent."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            f"{LIB_PATH} is missing: build it with `python -m reverb_b200.build` "
            "(or __graft_entry__.build()). reverb_b200 has no CPU fallback.")
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        if os.environ.get("RVB_LIB_PATH") and not hasattr(lib, name):
            continue                                  # an older build lacks the newer entry points
        fn = getattr(lib, name)
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def last_error() -> str:
    msg = load().rvb_last_error()
    return msg.decode("utf8", "replace") if msg else ""


def check(rc: int, what: str) -> None:
    if rc != 0:
        raise RuntimeError(f"{what} failed ({rc}): {last_error()}")
