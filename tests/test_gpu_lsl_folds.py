"""The folds of the language-specific linears live in one stack per side (encoder, decoders) of each plan, one slot per
distinct cat_embs vector of a call.  A plan that has folded other vectors before, grown its stack, or been forked,
decodes every call byte for byte as a fresh plan does; a slot is refolded only when its vector changes."""
import ctypes as C
import gc
import os

import numpy as np
import pytest
import torch
import yaml

pytestmark = pytest.mark.gpu

V, W, U = 0.35, 1.0, 0.7
B, T = 3, 200


@pytest.fixture(scope="module")
def asr(tmp_path_factory):
    """(configs, state_dict, vocab) of the synthetic test-shape model"""
    from reverb_b200 import synth
    d = str(tmp_path_factory.mktemp("lsl_folds_model"))
    synth.write_model_dir(d, seed=11)
    with open(os.path.join(d, "config.yaml")) as f:
        configs = yaml.safe_load(f)
    return configs, torch.load(os.path.join(d, "synth.pt")), synth.TEST_SHAPE["vocab"]


def _engine(asr, precision="bf16"):
    from reverb_b200.engine import Engine
    configs, sd, vocab = asr
    return Engine(configs, sd, vocab, torch.device("cuda", 0), precision=precision)


def _cat(values):
    """one value -> the (num_langs,) vector of the whole call; a list -> one row per utterance"""
    if isinstance(values, float):
        return torch.tensor([values, 1.0 - values])
    return torch.tensor([[v, 1.0 - v] for v in values])


def _feats():
    g = torch.Generator().manual_seed(3)
    return (10.0 + 3.0 * torch.randn(B, T, 80, generator=g)).cuda(), [T, 170, 130]


def _nbest(vocab):
    rng = np.random.default_rng(5)
    return [[tuple(int(t) for t in rng.integers(1, vocab - 1, n)) for n in (4, 7, 1)] for _ in range(B)]


def _bits(a):
    return None if a is None else np.ascontiguousarray(a).view(np.int32).copy()


def _call(eng, cat):
    """encoder output and both rescoring decoders' scores of one call, as bits"""
    feats, lens = _feats()
    enc, el = eng.forward_encoder(feats, lens, cat)
    l2r, r2l = eng.rescoring_scores(enc, el, _nbest(eng.vocab), cat, reverse_weight=0.3)
    torch.cuda.synchronize()
    return enc.view(torch.int32).cpu(), _bits(l2r), _bits(r2l)


def _same(a, b):
    assert torch.equal(a[0], b[0]), "encoder output"
    assert np.array_equal(a[1], b[1]), "left-to-right scores"
    assert (a[2] is None) == (b[2] is None) and (a[2] is None or np.array_equal(a[2], b[2])), "right-to-left scores"


# uniform, two groups, growth to three slots with slots 0 and 1 unchanged, the same three vectors reordered, uniform
CALLS = [V, [V, W, W], [V, W, U], [W, V, U], V]


@pytest.mark.parametrize("precision", ["bf16", "fp32"])
def test_one_plan_equals_fresh_plans(asr, precision):
    eng = _engine(asr, precision)
    for values in CALLS:
        got = _call(eng, _cat(values))
        fresh = _engine(asr, precision)
        _same(got, _call(fresh, _cat(values)))
        del fresh


def _cache_run(eng, enc, el, cat, between=None):
    """attention-mode steps through the decoder cache; `between` is called after decoder_cache_begin and after the
    first step"""
    N, steps = 3, 5
    S = B * N
    rng = np.random.default_rng(9)
    eng.decoder_cache_begin(enc, el, N, steps, cat)
    out = []
    for s in range(steps):
        if between is not None and s < 2:
            between()
        tok = np.full(S, eng.vocab - 1, np.int32) if s == 0 else rng.integers(1, eng.vocab - 1, S).astype(np.int32)
        par = None if s == 0 else np.concatenate([b * N + rng.permutation(N) for b in range(B)]).astype(np.int32)
        val, idx = eng.decoder_cache_step(tok, par, 4)
        out.append((val.view(np.int32).copy(), idx.copy()))
    eng.decoder_cache_end()
    return out


@pytest.mark.parametrize("precision", ["bf16", "fp32"])
@pytest.mark.parametrize("cache_cat, other", [([V, W, W], U), (V, [W, U, W])])
def test_decoder_cache_survives_calls_in_between(asr, precision, cache_cat, other):
    ref = _engine(asr, precision)
    feats, lens = _feats()
    enc, el = ref.forward_encoder(feats, lens, _cat(V))
    want = _cache_run(ref, enc, el, _cat(cache_cat))
    eng = _engine(asr, precision)
    got = _cache_run(eng, enc, el, _cat(cache_cat),
                     between=lambda: eng.rescoring_scores(enc, el, _nbest(eng.vocab), _cat(other), 0.3))
    for s, (g, w) in enumerate(zip(got, want)):
        assert np.array_equal(g[0], w[0]) and np.array_equal(g[1], w[1]), f"step {s}"


def test_fork_folds_its_own_vectors(asr):
    eng = _engine(asr)
    v_before = _call(eng, _cat(V))
    fork = eng.fork()
    fork_w = _call(fork, _cat(W))
    _same(_call(eng, _cat(V)), v_before)
    _same(fork_w, _call(eng, _cat(W)))
    del fork


def _held():
    from reverb_b200 import _lib
    dev, pin = C.c_longlong(-1), C.c_longlong(-1)
    _lib.check(_lib.load().rvb_held_bytes(C.byref(dev), C.byref(pin)), "rvb_held_bytes")
    return dev.value, pin.value


def test_fork_allocates_nothing(asr):
    eng = _engine(asr)
    _call(eng, _cat(V))
    gc.collect()
    base = _held()
    fork = eng.fork()
    assert _held() == base
    del fork
    gc.collect()
    assert _held() == base


def test_slots_refold_only_when_their_vector_changes(asr):
    from reverb_b200.engine import launch_count
    eng = _engine(asr)
    feats, lens = _feats()

    def launches(values):
        l0 = launch_count()
        eng.forward_encoder(feats, lens, _cat(values))
        torch.cuda.synchronize()
        return launch_count() - l0

    launches(V)                          # first call: positional tables, the fold of v
    launches([V, W, W])                  # the stack grows to two slots: v and w are folded into it
    plain = launches(V)                  # slot 0 holds v: folds nothing
    grouped = launches([V, W, W])        # folds nothing
    assert launches(V) == plain and launches([V, W, W]) == grouped, "alternating one and two vectors refolds nothing"
    fold = launches([V, U, U]) - grouped  # slot 1 refolds for u, slot 0 keeps v
    assert fold > 0
    assert launches(W) == plain + fold   # slot 0 refolds for w: one vector's folds
