"""wgmma attention (csrc/attention_tc.cu): the mask-specialised instantiations, the CTAs per SM they run with, and the
encoder shape of the benchmark.

The kernel has one instantiation per mask kind: key lengths only, chunk / causal, and key_bits (with the chunk /
causal mask when given).  Masks that hide the same keys must give the same bits whichever instantiation runs them."""
import ctypes as C
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

DK = 64


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


class SelfAttn:
    """Seeded self-attention inputs in the encoder's layout: rows of [q | k | v], groups of Tq == Tk rows."""

    def __init__(self, G, T, H, klens, seed):
        torch.manual_seed(seed)
        self.G, self.T, self.H, self.d = G, T, H, H * DK
        self.qkv = (torch.randn(G, T, 3 * self.d, device="cuda") * 0.7).bfloat16()
        self.bias = torch.randn(G, H, T, device="cuda") * 0.5
        self.klens = torch.tensor(klens, dtype=torch.int32, device="cuda")
        self.scale = 1.0 / math.sqrt(DK)

    def _ptrs(self, out):
        d = self.d
        return (_p(self.qkv), C.c_void_p(self.qkv.data_ptr() + 2 * d), C.c_void_p(self.qkv.data_ptr() + 4 * d), _p(out),
                3 * d, 3 * d, 3 * d, d, self.G, self.T, self.T, self.H, DK, _p(self.bias), _p(self.klens))

    def new_out(self):
        return torch.full((self.G, self.T, self.d), 7.0, device="cuda", dtype=torch.bfloat16)

    def lens_only(self, lib, causal=0):
        out = self.new_out()
        _check(lib.rvb_attention_tc(*self._ptrs(out), causal, self.scale, _stream()))
        return out

    def chunked(self, lib, chunk, left):
        out = self.new_out()
        _check(lib.rvb_attention_tc_chunked(*self._ptrs(out), chunk, left, self.scale, _stream()))
        return out

    def with_bits(self, lib, bits, bits_ld, causal=0):
        out = self.new_out()
        _check(lib.rvb_attention_tc_bits(*self._ptrs(out), causal, _p(bits), bits_ld, self.scale, _stream()))
        return out

    def visible_bits(self):
        """key_bits with the bit of every key below the group's key length set, for every query row"""
        bits_ld = 2 * ((self.T + 63) // 64)
        j = torch.arange(bits_ld * 32, device="cuda")
        vis = (j[None, :] < self.klens[:, None].long()).long()                   # (G, bits_ld * 32)
        words = (vis.view(self.G, bits_ld, 32) << torch.arange(32, device="cuda")).sum(-1)
        words = words.to(torch.int64).bitwise_and(0xFFFFFFFF)
        words = torch.where(words >= 2 ** 31, words - 2 ** 32, words).to(torch.int32)
        return words[:, None, :].expand(self.G, self.T, bits_ld).contiguous(), bits_ld

    def reference(self, causal=False, g0=0, g1=None):
        """the fp32 formula for groups [g0, g1)"""
        T, H, d = self.T, self.H, self.d
        qkv, bias, klens = self.qkv[g0:g1], self.bias[g0:g1], self.klens[g0:g1]
        G = qkv.shape[0]
        q = qkv[..., :d].float().view(G, T, H, DK).transpose(1, 2)
        k = qkv[..., d:2 * d].float().view(G, T, H, DK).transpose(1, 2)
        v = qkv[..., 2 * d:].float().view(G, T, H, DK).transpose(1, 2)
        s = (q @ k.transpose(-1, -2) + bias[:, :, None, :]) * self.scale
        i = torch.arange(T, device="cuda")
        mask = (i[None, None, :] >= klens[:, None, None])
        if causal:
            mask = mask | (i[None, :] > i[:, None])[None]
        s = s.masked_fill(mask[:, None], -float("inf"))
        a = torch.nan_to_num(torch.softmax(s, -1), nan=0.0)
        return (a @ v).transpose(1, 2).reshape(G, T, d)


@pytest.mark.parametrize("T", [1, 64, 65, 748])
def test_mask_instantiations_give_identical_bits(lib, T):
    """Key lengths only, a chunk mask with chunk >= Tk, and key_bits with every visible key's bit set hide the same
    keys, so the three instantiations must write the same bits; so must causal with and without all-visible key_bits."""
    x = SelfAttn(3, T, 2, [T, max(1, (T + 1) // 2), 0], seed=T)
    bits, bits_ld = x.visible_bits()
    plain = x.lens_only(lib)
    chunk_t = x.chunked(lib, T, -1)
    chunk_big = x.chunked(lib, 4 * T + 3, 2)
    with_bits = x.with_bits(lib, bits, bits_ld)
    causal = x.lens_only(lib, causal=1)
    causal_bits = x.with_bits(lib, bits, bits_ld, causal=1)
    torch.cuda.synchronize()
    for other in (chunk_t, chunk_big, with_bits):
        assert torch.equal(plain.view(torch.int16), other.view(torch.int16))
    assert torch.equal(causal.view(torch.int16), causal_bits.view(torch.int16))
    assert float(plain[2].float().abs().max()) == 0.0       # key length 0: zero rows
    torch.testing.assert_close(plain.float(), x.reference(), rtol=3e-2, atol=3e-2)
    torch.testing.assert_close(causal.float(), x.reference(causal=True), rtol=3e-2, atol=3e-2)


def test_encoder_shape_repeatable_and_matches_reference(lib):
    """The benchmarked encoder shape (B = 64, T' = 748, H = 16): two launches write the same bytes, and the output
    matches the fp32 formula."""
    B, T, H = 64, 748, 16
    klens = [T] * (B - 4) + [700, 513, 65, 1]
    x = SelfAttn(B, T, H, klens, seed=1234)
    a = x.lens_only(lib)
    b = x.lens_only(lib)
    torch.cuda.synchronize()
    assert torch.equal(a.view(torch.int16), b.view(torch.int16))
    for g0 in range(0, B, 8):              # the fp32 scores of 8 groups at a time
        torch.testing.assert_close(a[g0:g0 + 8].float(), x.reference(g0=g0, g1=g0 + 8), rtol=3e-2, atol=3e-2)


def test_two_ctas_per_sm(lib):
    """Every instantiation runs two CTAs per SM at the encoder's Tk; key rows too long for two CTAs' shared memory
    fall back to one."""
    for causal, chunk, bits in ((0, 0, 0), (1, 0, 0), (0, 16, 0), (1, 0, 1), (0, 0, 1)):
        assert lib.rvb_attention_tc_blocks_per_sm(748, causal, chunk, bits) == 2
        assert lib.rvb_attention_tc_blocks_per_sm(4096, causal, chunk, bits) == 2
        assert lib.rvb_attention_tc_blocks_per_sm(9000, causal, chunk, bits) == 1


def test_long_keys_one_cta_per_sm(lib):
    """Cross-attention over 9 000 keys (one CTA per SM) still matches the fp32 formula."""
    torch.manual_seed(3)
    H = 2
    d = H * DK
    G, Tq, Tk = 2, 130, 9000
    assert lib.rvb_attention_tc_blocks_per_sm(Tk, 0, 0, 0) == 1
    qx = (torch.randn(G, Tq, d, device="cuda") * 0.7).bfloat16()
    kv = (torch.randn(G, Tk, 2 * d, device="cuda") * 0.7).bfloat16()
    klens = torch.tensor([Tk, 4321], dtype=torch.int32, device="cuda")
    out = torch.zeros(G, Tq, d, device="cuda", dtype=torch.bfloat16)
    scale = 1.0 / math.sqrt(DK)
    _check(lib.rvb_attention_tc(_p(qx), _p(kv), C.c_void_p(kv.data_ptr() + 2 * d), _p(out), d, 2 * d, 2 * d, d,
                                G, Tq, Tk, H, DK, None, _p(klens), 0, scale, _stream()))
    q = qx.float().view(G, Tq, H, DK).transpose(1, 2)
    k = kv[..., :d].float().view(G, Tk, H, DK).transpose(1, 2)
    v = kv[..., d:].float().view(G, Tk, H, DK).transpose(1, 2)
    s = (q @ k.transpose(-1, -2)) * scale
    mask = torch.arange(Tk, device="cuda")[None, :] >= klens[:, None]
    s = s.masked_fill(mask[:, None, None, :], -float("inf"))
    ref = (torch.softmax(s, -1) @ v).transpose(1, 2).reshape(G, Tq, d)
    torch.testing.assert_close(out.float(), ref, rtol=3e-2, atol=3e-2)
