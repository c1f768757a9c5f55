"""Encoder-shaped attention micro-benchmark: wgmma kernel (incl. the K''/bias pre-kernel) vs the mma.sync kernel.

    python tools/attn_bench.py [--sweep] [--save PATH | --compare PATH]

Prints the card, its power limit and max SM clock, the CTAs per SM of the launched instantiation, then one JSON line:
per-launch times at B = 64, T = 748, H = 16 (d_k = 64) and the attention kernel's rate.  `--save` writes the wgmma
output of the fixed seeded inputs; `--compare` checks that this build's output is bit-equal to one saved from another
build (select it with RVB_LIB_PATH).  `--sweep` separates the per-CTA fixed cost from the per-key-tile cost."""
import ctypes as C, json, math, os, subprocess, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
from reverb_b200 import _lib


def arg(flag):
    return sys.argv[sys.argv.index(flag) + 1] if flag in sys.argv else None


lib = _lib.load()
p = lambda t: C.c_void_p(t.data_ptr())
B, T, H, dk = 64, 748, 16, 64
d = H * dk
q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i",
                    str(torch.cuda.current_device())], capture_output=True, text=True)
print(f"card: {q.stdout.strip() or torch.cuda.get_device_name()}  library: {_lib.LIB_PATH}", file=sys.stderr)
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
def prep():
    lib.rvb_relpos_prep(C.c_void_p(qkv.data_ptr() + 2 * d), 3 * d, p(pos), d, p(u), p(v), p(kpp), p(cb), B, T, H, dk, st)
def attn():
    lib.rvb_attention_tc(p(qkv), p(kpp), C.c_void_p(qkv.data_ptr() + 4 * d), p(out), 3 * d, d, 3 * d, d, B, T, T, H, dk, p(cb), p(klens), 0, scale, st)
def tc():
    prep()
    attn()
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
# an older build may lack the occupancy query
occ = lib.rvb_attention_tc_blocks_per_sm(T, 0, 0, 0) if hasattr(lib, "rvb_attention_tc_blocks_per_sm") else None
r = {"ctas_per_sm": occ, "tc_total_ms": timeit(tc), "prep_ms": timeit(prep), "attn_ms": timeit(attn, 100),
     "mma_ms": timeit(mma)}
r["tc_attn_tflops"] = flop / (r["attn_ms"] * 1e-3) / 1e12
r["mma_tflops_equiv"] = flop / (r["mma_ms"] * 1e-3) / 1e12
tc()
torch.cuda.synchronize()
r["max_abs_diff"] = float((out.float() - out2.float()).abs().max())
if arg("--save"):
    np.save(arg("--save"), out.view(torch.int16).cpu().numpy())
if arg("--compare"):
    ref = torch.from_numpy(np.load(arg("--compare"))).cuda().view(torch.bfloat16)
    r["bit_equal"] = bool(torch.equal(out.view(torch.int16), ref.view(torch.int16)))
    r["mismatched_elements"] = int((out.view(torch.int16) != ref.view(torch.int16)).sum())
print(json.dumps(r))
if "--sweep" in sys.argv:
    # per-CTA fixed cost vs per-key-tile cost: the same launch with the key lengths capped (ceil(klen / 64) tiles visited)
    rows = []
    for L in (64, 128, 256, 384, 512, 640, 748):
        klens.fill_(L)
        rows.append({"klen": L, "tiles": (L + 63) // 64, "ms": timeit(attn, 20)})
    klens.fill_(T)
    print(json.dumps({"sweep": rows}))
if arg("--compare") and not r["bit_equal"]:
    sys.exit(1)
