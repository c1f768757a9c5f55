"""Tile scheduling of the persistent wgmma GEMM (csrc/gemm.cu): a CTA takes tiles blockIdx.x, blockIdx.x + #SMs, ...
and its two consumer warpgroups take every other one of them.  Shapes with 1, 2, 131, 133, 264, 265 and 3 * 264 + 1
tiles give CTAs with 0, 1, an even and an odd number of tiles, and warpgroups without a tile, on a 132-SM H100.  Every
tile must be drained exactly once, into the right rows, and the same launch must give the same bytes."""
import ctypes as C
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

TILE_COUNTS = [1, 2, 131, 133, 264, 265, 3 * 264 + 1]
IMPLS = pytest.mark.parametrize("impl", [0, 2], ids=["wide", "narrow"])
K = 192   # 3 k-blocks: consecutive tiles start at different places of the 4-stage ring


def _p(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


@pytest.fixture(scope="module")
def lib():
    from reverb_b200 import _lib
    return _lib.load()


@pytest.fixture
def gemm_impl(lib, impl):
    lib.rvb_set_gemm_impl(impl)
    yield impl
    lib.rvb_set_gemm_impl(-1)


def _check(rc):
    from reverb_b200 import _lib
    assert rc == 0, _lib.last_error()


def _tile_n(impl):
    return 64 if impl == 2 else 128     # column tile width of plain epilogues (launch_gemm)


def _shape(impl, tiles):
    """(M, N): tiles x 1 column tile for odd counts, tiles/2 x 2 for even ones; ragged last row and column tile."""
    bn = _tile_n(impl)
    tiles_n = 2 if tiles % 2 == 0 else 1
    tiles_m = tiles // tiles_n
    N = tiles_n * bn - 8
    M = 128 * (tiles_m - 1) + 77
    assert (math.ceil(M / 128) * math.ceil(N / bn)) == tiles
    return M, N


def _operands(M, N, K, seed, wscale=1.0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    A = (torch.randn(M, K, device="cuda", generator=g) * 0.5).bfloat16()
    W = (torch.randn(N, K, device="cuda", generator=g) * (wscale / math.sqrt(K))).bfloat16()
    bias = torch.randn(N, device="cuda", generator=g)
    return A, W, bias


@IMPLS
@pytest.mark.parametrize("tiles", TILE_COUNTS)
def test_tile_totals_bf16_silu_and_fp32(lib, gemm_impl, tiles):
    M, N = _shape(gemm_impl, tiles)
    A, W, bias = _operands(M, N, K, tiles)
    ref = A.float() @ W.float().t() + bias
    ldo = (N + 7) & ~7
    out = torch.zeros(M, ldo, device="cuda")
    _check(lib.rvb_gemm_bf16(_p(A), _p(W), _p(bias), M, N, K, 0, 1, 1.0, _p(out), ldo, _stream()))
    torch.testing.assert_close(out[:, :N], ref, rtol=1e-3, atol=1e-3)
    assert bool((out[:, N:] == 0).all())
    out_b = torch.zeros(M, ldo, device="cuda", dtype=torch.bfloat16)
    _check(lib.rvb_gemm_bf16(_p(A), _p(W), _p(bias), M, N, K, 2, 0, 1.0, _p(out_b), ldo, _stream()))
    torch.testing.assert_close(out_b[:, :N].float(), torch.nn.functional.silu(ref), rtol=2e-2, atol=2e-2)
    assert bool((out_b[:, N:] == 0).all())


@IMPLS
@pytest.mark.parametrize("tiles", TILE_COUNTS)
def test_tile_totals_glu(lib, gemm_impl, tiles):
    bn = _tile_n(gemm_impl)
    tiles_n = 2 if tiles % 2 == 0 else 1
    Cc = tiles_n * bn // 2                  # output channels; the GEMM has 2 * Cc columns
    M = 128 * (tiles // tiles_n - 1) + 77
    A, W, bias = _operands(M, 2 * Cc, K, 100 + tiles)
    ref = torch.nn.functional.glu(A.float() @ W.float().t() + bias, dim=1)
    c = torch.arange(Cc, device="cuda")
    ra = 64 * (c // 32) + (c % 32)          # interleaved value / gate rows (include/rvb_b200.h)
    Wp, bp = torch.empty_like(W), torch.empty_like(bias)
    Wp[ra], Wp[ra + 32] = W[:Cc], W[Cc:]
    bp[ra], bp[ra + 32] = bias[:Cc], bias[Cc:]
    out = torch.zeros(M, Cc, device="cuda", dtype=torch.bfloat16)
    _check(lib.rvb_gemm_bf16(_p(A), _p(Wp), _p(bp), M, 2 * Cc, K, 3, 0, 1.0, _p(out), Cc, _stream()))
    torch.testing.assert_close(out.float(), ref, rtol=2e-2, atol=2e-2)


@IMPLS
@pytest.mark.parametrize("tiles", [t for t in TILE_COUNTS if t > 1])
def test_tile_totals_logsoftmax_gather(lib, gemm_impl, tiles):
    # the log-sum-exp epilogue always uses 128-wide tiles and needs N > 128: tiles_n = the smallest divisor >= 2
    tiles_n = next(d for d in range(2, tiles + 1) if tiles % d == 0)
    M, N = 128 * (tiles // tiles_n - 1) + 77, tiles_n * 128 - 40
    A, W, bias = _operands(M, N, K, 200 + tiles, wscale=3.0)
    g = torch.Generator(device="cuda").manual_seed(tiles)
    gather = torch.randint(0, N, (M,), device="cuda", dtype=torch.int32, generator=g)
    gather[::7] = -1
    gather[1 % M] = N - 1
    ws = torch.empty(int(lib.rvb_gemm_logsoftmax_gather_ws_bytes(M, N)), device="cuda", dtype=torch.uint8)
    out = torch.full((M,), 123.0, device="cuda")
    _check(lib.rvb_gemm_logsoftmax_gather(_p(A), _p(W), _p(bias), M, N, K, _p(gather), _p(ws), _p(out), _stream()))
    logp = torch.log_softmax(A.float() @ W.float().t() + bias, dim=-1)
    want = torch.where(gather >= 0, logp.gather(1, gather.long().clamp(min=0)[:, None])[:, 0], torch.zeros(M, device="cuda"))
    torch.testing.assert_close(out, want, rtol=1e-3, atol=2e-3)


@IMPLS
@pytest.mark.parametrize("tiles", TILE_COUNTS)
def test_residual_is_written_exactly_once(lib, gemm_impl, tiles):
    """Two residual launches into one zeroed buffer give 2x the product: a tile drained twice or skipped does not."""
    M, N = _shape(gemm_impl, tiles)
    A, W, bias = _operands(M, N, K, 300 + tiles)
    ref = A.float() @ W.float().t() + bias
    ldo = (N + 7) & ~7
    res = torch.zeros(M, ldo, device="cuda")
    for _ in range(2):
        _check(lib.rvb_gemm_bf16(_p(A), _p(W), _p(bias), M, N, K, 0, 2, 1.0, _p(res), ldo, _stream()))
    torch.testing.assert_close(res[:, :N], 2 * ref, rtol=1e-3, atol=2e-3)
    assert bool((res[:, N:] == 0).all())


@IMPLS
@pytest.mark.parametrize("tiles", [2, 133, 3 * 264 + 1])
def test_row_mask_writes_valid_rows_only(lib, gemm_impl, tiles):
    M, N = _shape(gemm_impl, tiles)
    A, W, bias = _operands(M, N, K, 400 + tiles)
    rows_per_batch = 300
    nb = (M + rows_per_batch - 1) // rows_per_batch
    g = torch.Generator().manual_seed(tiles)
    lens = torch.randint(0, rows_per_batch + 1, (nb,), generator=g, dtype=torch.int32)
    lens[0] = rows_per_batch
    ldo = (N + 7) & ~7
    out = torch.full((M, ldo), float("nan"), device="cuda", dtype=torch.bfloat16)
    _check(lib.rvb_gemm_bf16_rows(_p(A), _p(W), _p(bias), M, N, K, 0, 0, 1.0, _p(out), ldo, _p(lens.cuda()),
                                  rows_per_batch, _stream()))
    m = torch.arange(M)
    valid = ((m % rows_per_batch) < lens[m // rows_per_batch].long()).cuda()
    ref = (A.float() @ W.float().t() + bias)
    torch.testing.assert_close(out[valid, :N].float(), ref[valid], rtol=2e-2, atol=2e-2)
    assert bool(torch.isnan(out[~valid].float()).all())
    assert bool(torch.isnan(out[:, N:].float()).all())


@IMPLS
def test_same_launch_same_bytes(lib, gemm_impl):
    M, N = _shape(gemm_impl, 3 * 264 + 1)
    A, W, bias = _operands(M, N, 1024, 7)
    ldo = (N + 7) & ~7
    outs = []
    for out_mode, dt in ((0, torch.bfloat16), (1, torch.float32)):
        for _ in range(2):
            out = torch.zeros(M, ldo, device="cuda", dtype=dt)
            _check(lib.rvb_gemm_bf16(_p(A), _p(W), _p(bias), M, N, 1024, 2 if out_mode == 0 else 0, out_mode, 1.0,
                                     _p(out), ldo, _stream()))
            outs.append(out)
    assert torch.equal(outs[0].view(torch.int16), outs[1].view(torch.int16))
    assert torch.equal(outs[2].view(torch.int32), outs[3].view(torch.int32))
