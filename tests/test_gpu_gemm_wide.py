"""The 128 x 256 GEMM tiles (csrc/gemm.cu `gemm_wide_kernel`) against the 128 x 128 ping-pong kernel and against an
fp64 product of the same bf16 operands.  launch_gemm takes the wide tiles for bf16 outputs with bias / ReLU / SiLU,
N % 256 == 0 and at least one wave of tiles; RVB_GEMM_WIDE=0 keeps every shape on 128 x 128 tiles.

Both kernels give every output element the same wgmma k16 steps in the same k-block order and the same epilogue
arithmetic, so the outputs must be the same bits.  The tile counts include CTAs with an odd number of tiles (the
output-tile barrier phases wrap) and K values that start consecutive tiles at different places of the 3-stage ring."""
import ctypes as C
import math
import os
import tempfile

import pytest
import torch

pytestmark = pytest.mark.gpu


def _p(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


@pytest.fixture(scope="module")
def lib():
    from reverb_b200 import _lib
    return _lib.load()


def _check(rc):
    from reverb_b200 import _lib
    assert rc == 0, _lib.last_error()


def _num_sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _kernel_names(fn):
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]


def _both(fn):
    """fn() with the default tile choice and with RVB_GEMM_WIDE=0; asserts which kernel each run took."""
    out = {}
    for wide in (True, False):
        if not wide:
            os.environ["RVB_GEMM_WIDE"] = "0"
        try:
            names = _kernel_names(lambda: out.__setitem__(wide, fn()))
        finally:
            os.environ.pop("RVB_GEMM_WIDE", None)
        assert any("gemm_wide_kernel" in n for n in names) == wide, names
    return out[True], out[False]


# (M, N, K): N = 256, 1024, 4096; M not a multiple of 128.  On 132 SMs the 265, 397, 268 and 400 tiles leave some CTAs
# with an odd number of tiles (3, 3, 3 and 3); K = 320 (5 k-blocks) and 1088 (17) start tiles at every ring stage
SHAPES = [(128 * 264 + 77, 256, 320), (128 * 396 + 77, 256, 1088), (128 * 66 + 5, 1024, 1088),
          (128 * 24 + 100, 4096, 320)]


@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "x".join(map(str, s)))
@pytest.mark.parametrize("act", [0, 1, 2], ids=["bias", "relu", "silu"])
def test_wide_equals_square_tiles_and_fp64(lib, shape, act):
    M, N, K = shape
    assert math.ceil(M / 128) * (N // 256) >= _num_sms()
    g = torch.Generator(device="cuda").manual_seed(M + N + act)
    A = (torch.randn(M, K, device="cuda", generator=g) * 0.5).bfloat16()
    W = (torch.randn(N, K, device="cuda", generator=g) / math.sqrt(K)).bfloat16()
    bias = torch.randn(N, device="cuda", generator=g)

    def run():
        out = torch.full((M, N), 7.0, device="cuda", dtype=torch.bfloat16)
        _check(lib.rvb_gemm_bf16(_p(A), _p(W), _p(bias), M, N, K, act, 0, 1.0, _p(out), N, _stream()))
        return out

    wide, square = _both(run)
    assert torch.equal(wide, square)
    ref = A.double() @ W.double().t() + bias.double()
    ref = torch.relu(ref) if act == 1 else torch.nn.functional.silu(ref) if act == 2 else ref
    torch.testing.assert_close(wide.double(), ref, rtol=1e-2, atol=1e-2)


def test_wide_without_bias_and_with_row_mask(lib):
    """No bias (the kernel adds +0, as the 128 x 128 epilogue does) and masked rows, which stay untouched."""
    M, N, K, rpb = 128 * 140 - 3, 512, 192, 300
    g = torch.Generator(device="cuda").manual_seed(5)
    A = (torch.randn(M, K, device="cuda", generator=g) * 0.5).bfloat16()
    W = (torch.randn(N, K, device="cuda", generator=g) / math.sqrt(K)).bfloat16()
    nb = (M + rpb - 1) // rpb
    lens = torch.randint(0, rpb + 1, (nb,), device="cuda", dtype=torch.int32, generator=g)

    def run():
        out = torch.full((M, N), 7.0, device="cuda", dtype=torch.bfloat16)
        _check(lib.rvb_gemm_bf16_rows(_p(A), _p(W), None, M, N, K, 2, 0, 1.0, _p(out), N, _p(lens), rpb, _stream()))
        return out

    wide, square = _both(run)
    assert torch.equal(wide, square)
    pos = torch.arange(M, device="cuda") % rpb
    keep = pos < lens.long()[torch.arange(M, device="cuda") // rpb]
    assert bool((wide[~keep] == 7.0).all())
    ref = torch.nn.functional.silu(A.double() @ W.double().t())
    torch.testing.assert_close(wide[keep].double(), ref[keep], rtol=1e-2, atol=1e-2)


def test_below_one_wave_keeps_square_tiles(lib):
    M, N, K = 128 * 10, 1024, 128   # 40 wide tiles
    A = torch.ones(M, K, device="cuda", dtype=torch.bfloat16)
    W = torch.ones(N, K, device="cuda", dtype=torch.bfloat16)
    out = torch.empty(M, N, device="cuda", dtype=torch.bfloat16)
    names = _kernel_names(lambda: _check(lib.rvb_gemm_bf16(_p(A), _p(W), None, M, N, K, 0, 0, 1.0, _p(out), N,
                                                           _stream())))
    assert not any("gemm_wide_kernel" in n for n in names) and any("gemm_wg_kernel" in n for n in names)
    assert bool((out == K).all())


@pytest.fixture(scope="module")
def small_model():
    import reverb_b200
    from reverb_b200 import synth
    d = tempfile.mkdtemp(prefix="rvb_wide_")
    shape = dict(synth.TEST_SHAPE, d=256, heads=4, ff=1024, blocks=1)
    synth.write_model_dir(d, shape=shape, seed=11)
    return reverb_b200.load_model(d)


def test_conv2_implicit_gemm_wide_equals_square(small_model):
    """The subsampling conv2 (implicit GEMM over 4-D TMA boxes, ReLU) at d = 256, B = 8: 8 * 19 = 152 wide tiles.
    The whole encoder output must be the same bits with either tile width."""
    m = small_model
    g = torch.Generator(device="cuda").manual_seed(3)
    B, T = 8, 301
    feats = torch.randn(B, T, 80, device="cuda", generator=g)
    lens = torch.tensor([301, 301, 250, 301, 77, 301, 180, 301])
    cat = torch.tensor([1.0, 0.0])

    def run():
        enc, enc_lens = m.model._forward_encoder(feats, lens, cat)
        return enc.clone(), list(enc_lens)

    (enc_w, lens_w), (enc_s, lens_s) = _both(run)
    assert lens_w == lens_s
    assert torch.equal(enc_w, enc_s)
