"""The native models give back every byte they hold.  rvb_held_bytes counts the device memory of all workspaces and
weights and the page-locked host memory of the library; each case reads it first and requires both counters to return
exactly to that baseline once its models are destroyed (or, for the synchronous searches, once their thread has
exited).  The whole-device figure of cudaMemGetInfo would not do: other processes share the GPU."""
import ctypes as C
import gc
import os
import threading
import time

import numpy as np
import pytest
import torch
import yaml

pytestmark = pytest.mark.gpu

CAT = [1.0, 0.0]


def _held():
    from reverb_b200 import _lib
    dev, pin = C.c_longlong(-1), C.c_longlong(-1)
    _lib.check(_lib.load().rvb_held_bytes(C.byref(dev), C.byref(pin)), "rvb_held_bytes")
    return dev.value, pin.value


def _baseline():
    gc.collect()   # models an earlier test left to the collector go first
    return _held()


@pytest.fixture(scope="module")
def asr(tmp_path_factory):
    """(configs, state_dict, vocab) of the synthetic test-shape model"""
    from reverb_b200 import synth
    d = str(tmp_path_factory.mktemp("lifetime_model"))
    synth.write_model_dir(d, seed=5)
    with open(os.path.join(d, "config.yaml")) as f:
        configs = yaml.safe_load(f)
    return configs, torch.load(os.path.join(d, "synth.pt")), synth.TEST_SHAPE["vocab"]


def _engine(asr):
    from reverb_b200.engine import Engine
    configs, sd, vocab = asr
    return Engine(configs, sd, vocab, torch.device("cuda", 0))


def _topk(eng, B=2, T=60, k=4, seed=0):
    g = torch.Generator().manual_seed(seed)
    logp = torch.log_softmax(torch.randn(B, T, eng.vocab, generator=g), -1).cuda()
    return eng.logp_topk(logp, k)


def test_plan_and_fork_free_everything(asr):
    base = _baseline()
    eng = _engine(asr)
    fork = eng.fork()
    g = torch.Generator().manual_seed(1)
    feats = (10.0 + 3.0 * torch.randn(2, 200, 80, generator=g)).cuda()
    enc, enc_lens = fork.forward_encoder(feats, [200, 160], CAT)
    val, idx, _ = fork.ctc_topk(enc, 4)
    t = fork.search_submit(val, idx, enc, enc_lens, 4)
    fork.rescoring_submit(t, CAT, reverse_weight=0.3)
    fork.rescoring_collect(t)
    fork.decoder_cache_begin(enc, enc_lens, 2, 8, CAT)   # left open: destroying the plan frees the cache
    torch.cuda.synchronize()
    during = _held()
    assert during[0] > base[0] and during[1] > base[1]
    del t, fork
    gc.collect()
    after_fork = _held()
    assert base[0] < after_fork[0] < during[0], "the fork's workspace and folds are freed, the parent's weights stay"
    del eng
    gc.collect()
    assert _held() == base


def test_failed_finalize_frees_what_it_uploaded(asr):
    from reverb_b200 import _lib
    from reverb_b200.engine import model_config_from_yaml
    configs, sd, vocab = asr
    lib = _lib.load()
    base = _baseline()
    cfg = model_config_from_yaml(configs, vocab)
    with torch.cuda.device(0):
        h = lib.rvb_model_create(C.byref(cfg))
        assert h
        h = C.c_void_p(h)
        try:
            for name, t in sd.items():
                if name == "ctc.ctc_lo.weight" or not t.is_floating_point():
                    continue
                a = t.detach().to("cpu", torch.float32).contiguous()
                _lib.check(lib.rvb_model_set_tensor(h, name.encode(), C.c_void_p(a.data_ptr()), a.numel()), name)
            assert lib.rvb_model_finalize(h) != 0
            assert _lib.last_error() == "model: tensor 'ctc.ctc_lo.weight' was not provided"
            assert _held()[0] > base[0], "the encoder was uploaded before the missing tensor was found"
        finally:
            lib.rvb_model_destroy(h)
    assert _held() == base


def test_diarization_models_free_everything():
    from reverb_b200.diarization import synth
    from reverb_b200.diarization.embedding import EmbeddingModel
    from reverb_b200.diarization.segmentation import SegmentationModel
    base = _baseline()
    wav = torch.from_numpy(np.stack([synth.synthetic_speech(5.0, seed=20 + i) for i in range(2)])).cuda()
    seg = SegmentationModel(synth.segmentation_state_dict(0))
    emb = EmbeddingModel(synth.embedding_state_dict(0))
    seg.forward(wav)
    emb.forward(wav)
    torch.cuda.synchronize()
    assert _held()[0] > base[0]
    del seg, emb
    gc.collect()
    assert _held() == base


def test_search_buffers_are_freed_when_their_thread_exits(asr):
    base = _baseline()
    eng = _engine(asr)
    val, idx = _topk(eng)
    lens = np.array([60, 45], np.int32)
    before = _held()
    seen = {}

    def searches():
        with torch.cuda.device(0):
            seen["greedy"] = eng.greedy_search(idx, lens)
            seen["beam"] = eng.prefix_beam_search(val, idx, lens, 4)
            seen["held"] = _held()

    th = threading.Thread(target=searches)
    th.start()
    th.join()
    assert len(seen["greedy"]) == 2 and len(seen["beam"]) == 2
    assert seen["held"][0] > before[0] and seen["held"][1] > before[1], "the searches use per-thread buffers"
    # join() may return before the thread-local destructors of the native library have run
    deadline = time.monotonic() + 2.0
    while _held() != before and time.monotonic() < deadline:
        time.sleep(0.01)
    assert _held() == before
    del eng
    gc.collect()
    assert _held() == base
