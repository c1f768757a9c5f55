"""ORACLE (test infrastructure, never shipped): per-utterance cat_embs for the oracle model graph.

The reference's language-specific layers accept a (B, num_langs) cat_embs and weigh row b of their input with
cat_embs[b] (transformer/encoder_layer.py:376-390, decoder_layer.py:318-331 and :410-422:
`cat_embs[:, i].unsqueeze(-1).unsqueeze(-1) * layer(x)`).  oracle/model_ref.lsl_mix restates the 1-D form; the
context manager here puts a mixing function that also takes the 2-D form in its place for the duration of a call, so
that the unchanged graph functions of model_ref (encoder_forward, decoder_forward, ...) run the reference's 2-D
behaviour.  Running the oracle once per row is not a substitute: the batched GEMMs of the reference round differently
from B = 1 ones in the last bits.
"""
from __future__ import annotations

import contextlib

import torch

from . import model_ref


def lsl_mix_rows(x, sd, p: str, cat_embs: torch.Tensor, mix_1d=None):
    """sum_i cat_embs[:, i] * language_layers[i](x) with row b of x (B, T, d) weighed by cat_embs[b]; a 1-D cat_embs
    goes to `mix_1d` (model_ref's lsl_mix).  Under model_ref.EMULATE_BF16 each row uses the engine's fold of its own
    vector (W = sum_i c_i W_i, stored as bf16)."""
    mix_1d = mix_1d or model_ref.lsl_mix
    if cat_embs.dim() == 1:
        return mix_1d(x, sd, p, cat_embs)
    if model_ref.EMULATE_BF16:
        return torch.stack([mix_1d(x[b:b + 1], sd, p, cat_embs[b])[0] for b in range(x.shape[0])])
    y = None
    for i in range(cat_embs.shape[1]):
        t = cat_embs[:, i].unsqueeze(-1).unsqueeze(-1) * model_ref._lin(x, sd, f"{p}.language_layers.{i}")
        y = t if y is None else y + t
    return y


@contextlib.contextmanager
def per_row_cat_embs():
    """Within the block, model_ref's graph functions accept a (B, num_langs) cat_embs as the reference does."""
    orig = model_ref.lsl_mix
    model_ref.lsl_mix = lambda x, sd, p, cat_embs: lsl_mix_rows(x, sd, p, cat_embs, orig)
    try:
        yield
    finally:
        model_ref.lsl_mix = orig
