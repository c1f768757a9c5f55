"""Encoder-shaped attention micro-benchmark: wgmma kernel (incl. the K''/bias pre-kernel) vs the mma.sync kernel."""
import ctypes as C, json, math, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from reverb_b200 import _lib
lib = _lib.load()
p = lambda t: C.c_void_p(t.data_ptr())
B, T, H, dk = 64, 748, 16, 64
d = H * dk
torch.manual_seed(0)
qkv = (torch.randn(B, T, 3 * d, device="cuda") * 0.7).bfloat16()
pos = (torch.randn(T, d, device="cuda") * 0.7).bfloat16()
u = torch.randn(H, dk, device="cuda") * 0.3
v = torch.randn(H, dk, device="cuda") * 0.3
klens = torch.full((B,), T, dtype=torch.int32, device="cuda")
kpp = torch.empty(B, T, d, device="cuda", dtype=torch.bfloat16)
cb = torch.empty(B, H, T, device="cuda")
out = torch.empty(B, T, d, device="cuda", dtype=torch.bfloat16)
out2 = torch.empty_like(out)
st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
scale = 1 / math.sqrt(dk)
def tc():
    lib.rvb_relpos_prep(C.c_void_p(qkv.data_ptr() + 2 * d), 3 * d, p(pos), d, p(u), p(v), p(kpp), p(cb), B, T, H, dk, st)
    lib.rvb_attention_tc(p(qkv), p(kpp), C.c_void_p(qkv.data_ptr() + 4 * d), p(out), 3 * d, d, 3 * d, d, B, T, T, H, dk, p(cb), p(klens), 0, scale, st)
def prep():
    lib.rvb_relpos_prep(C.c_void_p(qkv.data_ptr() + 2 * d), 3 * d, p(pos), d, p(u), p(v), p(kpp), p(cb), B, T, H, dk, st)
def mma():
    lib.rvb_attention(p(qkv), C.c_void_p(qkv.data_ptr() + 2 * d), C.c_void_p(qkv.data_ptr() + 4 * d), p(pos), p(u), p(v), p(out2),
                      3 * d, 3 * d, 3 * d, d, d, B, T, T, H, dk, 1, p(klens), None, 0, scale, st)
def timeit(fn, n=10):
    for _ in range(3): fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize(); e0.record()
    for _ in range(n): fn()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n
flop = 2.0 * B * H * T * T * dk * 2
r = {"tc_total_ms": timeit(tc), "prep_ms": timeit(prep), "mma_ms": timeit(mma)}
r["tc_attn_tflops"] = flop / ((r["tc_total_ms"] - r["prep_ms"]) * 1e-3) / 1e12
r["mma_tflops_equiv"] = flop / (r["mma_ms"] * 1e-3) / 1e12
r["max_abs_diff"] = float((out.float() - out2.float()).abs().max())
print(json.dumps(r))
if "--sweep" in sys.argv:
    # per-CTA fixed cost vs per-key-tile cost: the same launch with the key lengths capped (ceil(klen / 64) tiles visited)
    def only_attn():
        lib.rvb_attention_tc(p(qkv), p(kpp), C.c_void_p(qkv.data_ptr() + 4 * d), p(out), 3 * d, d, 3 * d, d, B, T, T, H, dk, p(cb), p(klens), 0, scale, st)
    rows = []
    for L in (64, 128, 256, 384, 512, 640, 748):
        klens.fill_(L)
        rows.append({"klen": L, "tiles": (L + 63) // 64, "ms": timeit(only_attn, 20)})
    klens.fill_(T)
    print(json.dumps({"sweep": rows}))
