"""reverb_b200 — Hopper-native (sm_90a, H100) inference engine behind the revdotcom/reverb API.

Public surface (same names as the reference's `wenet` package, asr/wenet/__init__.py:1-6):
    load_model, ReverbASR, get_available_models, download_model
"""
from .reverb import ReverbASR, download_model, get_available_models, load_model  # noqa: F401

__all__ = ["ReverbASR", "download_model", "get_available_models", "load_model"]
