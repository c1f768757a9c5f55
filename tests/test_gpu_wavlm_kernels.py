"""The two kernels reverb-diarization-v2 adds, against float64 references on the H100:

  * attention_tc_kernel<MASK_RELB> (rvb_attention_tc_relbias): softmax(q k^T / 8 + gate[i] rb[j - i]) v, H = 12, at
    T across the 64-key tile edges, T = 1 (a one-entry table) and T = 1000 (the largest table in shared memory);
    gate = 0 is the plain key-length attention bit for bit;
  * the erf-GELU GEMM epilogue (rvb_gemm_bf16, act 4) through both of its stores (16-byte aligned rows and not).

The attention bar is about twice the largest error of the first H100 run (DESIGN.md §7b).
"""
import ctypes as C
import math

import pytest
import torch

from reverb_b200 import _lib

pytestmark = pytest.mark.gpu

H, DK = 12, 64


@pytest.fixture(scope="module")
def lib():
    return _lib.load()


def _p(t):
    return C.c_void_p(t.data_ptr())


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _check(rc):
    assert rc == 0, _lib.last_error()


def _qkv(B, T, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    d = H * DK
    qkv = (torch.randn(B * T, 3 * d, device="cuda", generator=g) * 0.8).bfloat16()
    gate = torch.rand(B, H, T, device="cuda", generator=g) * 2.0 + 0.5          # the gate's range (0.5 .. 3)
    rb = torch.randn(H, 2 * T - 1, device="cuda", generator=g) * 2.0
    return qkv, gate, rb


def _relbias(lib, qkv, gate, rb, B, T):
    d = H * DK
    out = torch.zeros(B * T, d, device="cuda", dtype=torch.bfloat16)
    base = qkv.data_ptr()
    _check(lib.rvb_attention_tc_relbias(C.c_void_p(base), C.c_void_p(base + 2 * d), C.c_void_p(base + 4 * d), _p(out),
                                        3 * d, 3 * d, 3 * d, d, B, T, H, _p(gate), _p(rb), 1.0 / 8.0, _stream()))
    torch.cuda.synchronize()
    return out


def _reference(qkv, gate, rb, B, T):
    d = H * DK
    x = qkv.double().view(B, T, 3, H, DK)
    q, k, v = (x[:, :, i].transpose(1, 2) for i in range(3))                   # (B, H, T, DK)
    idx = torch.arange(T, device=qkv.device)
    table = rb.double()[:, (idx[None, :] - idx[:, None]) + T - 1]                # (H, T, T)
    s = q @ k.transpose(-1, -2) / 8.0 + gate.double()[..., None] * table[None]
    return (torch.softmax(s, -1) @ v).transpose(1, 2).reshape(B * T, d)


@pytest.mark.parametrize("T", [1, 63, 64, 65, 499, 1000])
def test_relbias_attention_vs_float64(lib, T):
    B = 2
    qkv, gate, rb = _qkv(B, T, T)
    got = _relbias(lib, qkv, gate, rb, B, T).double()
    ref = _reference(qkv, gate, rb, B, T)
    err = float((got - ref).abs().max() / ref.abs().max())
    print(f"\n[relbias attention T={T}] max abs err / max abs ref {err:.2e}")
    assert err < 6e-3


@pytest.mark.parametrize("T", [1, 65, 499])
def test_relbias_attention_with_zero_gate_is_plain_attention(lib, T):
    B = 2
    d = H * DK
    qkv, gate, rb = _qkv(B, T, 100 + T)
    got = _relbias(lib, qkv, torch.zeros_like(gate), rb, B, T)
    plain = torch.zeros_like(got)
    base = qkv.data_ptr()
    _check(lib.rvb_attention_tc(C.c_void_p(base), C.c_void_p(base + 2 * d), C.c_void_p(base + 4 * d), _p(plain),
                                3 * d, 3 * d, 3 * d, d, B, T, T, H, DK, None, None, 0, 1.0 / 8.0, _stream()))
    torch.cuda.synchronize()
    assert torch.equal(got, plain)


def test_relbias_attention_rejects_missing_table(lib):
    qkv, gate, _ = _qkv(1, 64, 1)
    out = torch.zeros(64, H * DK, device="cuda", dtype=torch.bfloat16)
    base = qkv.data_ptr()
    d = H * DK
    assert lib.rvb_attention_tc_relbias(C.c_void_p(base), C.c_void_p(base + 2 * d), C.c_void_p(base + 4 * d), _p(out),
                                        3 * d, 3 * d, 3 * d, d, 1, 64, H, _p(gate), None, 0.125, _stream()) != 0


@pytest.mark.parametrize("ldo_pad", [0, 1])
def test_gelu_epilogue_vs_float64(lib, ldo_pad):
    """Pre-activations set exactly (one-hot A rows pick a bf16 weight, bias added in fp32) over [-6, 6], where erf and
    tanh GELU differ by up to 10 % for x < -3.  Every output is the float64 erf GELU within one bf16 rounding step
    plus 2^-22 |x|: like torch's CUDA gelu, the kernel forms 1 + erf(x / sqrt 2) in fp32, whose absolute error that
    term bounds (it dominates for x < -4, where the result is below 1e-4).  ldo_pad 1 gives rows that are not
    16 bytes apart (the per-element store)."""
    M, N, K = 256, 200, 64
    g = torch.Generator(device="cuda").manual_seed(7 + ldo_pad)
    A = torch.zeros(M, K, device="cuda", dtype=torch.bfloat16)
    A[torch.arange(M), torch.arange(M) % K] = 1.0
    W = (torch.rand(N, K, device="cuda", generator=g) * 12.0 - 6.0).bfloat16()
    bias = (torch.rand(N, device="cuda", generator=g) * 0.5 - 0.25)
    ldo = N + ldo_pad
    out = torch.zeros(M, ldo, device="cuda", dtype=torch.bfloat16)
    _check(lib.rvb_gemm_bf16(_p(A), _p(W), _p(bias), M, N, K, 4, 0, 1.0, _p(out), ldo, _stream()))
    torch.cuda.synchronize()
    x = (A.float() @ W.float().t() + bias).double()                                # exact: one product per row
    ref = 0.5 * x * (1.0 + torch.special.erf(x / math.sqrt(2.0)))
    got = out[:, :N].double()
    ulp = torch.exp2(torch.floor(torch.log2(ref.abs().clamp_min(1e-30))) - 7)     # bf16 spacing at |ref|
    tol = ulp + 2.0 ** -22 * x.abs()
    steps = float(((got - ref).abs() / tol).max())
    tanh = 0.5 * x * (1.0 + torch.tanh(math.sqrt(2.0 / math.pi) * (x + 0.044715 * x ** 3)))
    tanh_steps = float(((got - tanh).abs() / tol).max())
    print(f"\n[gelu epilogue ldo={ldo}] max error {steps:.2f} tolerances (tanh form: {tanh_steps:.1f})")
    assert steps <= 1.0
    assert tanh_steps > 4.0
