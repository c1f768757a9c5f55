// reverb_b200 — fp32 attention of the ACCURATE ("bf16x3") precision mode.
//
// In that mode every activation is a bf16 pair (hi, lo) with v = hi + lo to ~16 mantissa bits (GemmArgs::x3, kernels.h)
// and the projections run as three wgmma passes.  The attention itself is only ~5 % of the encoder FLOPs, so here it
// is evaluated directly in fp32 on the CUDA cores, operation for operation like the reference
// (asr/wenet/transformer/attention.py:344-399 rel-pos, :102-127 forward_attention; decoder: MultiHeadedAttention):
//     s[i,j] = ((q_i + u) . k_j + (q_i + v) . p_j) / sqrt(d_k)      (p: absolute key position, no rel_shift)
//     s[mask == 0] = -inf ; a = softmax_j(s) ; a[mask == 0] = 0 ; o_i = sum_j a[i,j] v_j
// The throughput path is attention_tc.cu (wgmma, bf16 operands); this kernel exists so that a whole decode can be
// run at fp32-level accuracy for parity with the reference (token ids bit-exact, logits to ~1e-4).
// One warp per query row; the row's scores live in shared memory.
#include <math.h>

#include "kernels.h"

namespace rvb {

__device__ __forceinline__ float ld_pair(const bf16* p, int lo) {
  return __bfloat162float(p[0]) + (lo ? __bfloat162float(p[lo]) : 0.f);
}

// dot(w[0..8), x[0..8)) with x = hi (+ lo): two 16-byte loads per 8 elements (rows / heads are 16-byte aligned)
__device__ __forceinline__ float dot8_pair(const float* w, const bf16* p, int lo, float acc) {
  const uint4 hv = *reinterpret_cast<const uint4*>(p);
  float x[8];
  float2 t;
  t = unpack_bf16x2(hv.x); x[0] = t.x; x[1] = t.y;
  t = unpack_bf16x2(hv.y); x[2] = t.x; x[3] = t.y;
  t = unpack_bf16x2(hv.z); x[4] = t.x; x[5] = t.y;
  t = unpack_bf16x2(hv.w); x[6] = t.x; x[7] = t.y;
  if (lo) {
    const uint4 lv = *reinterpret_cast<const uint4*>(p + lo);
    t = unpack_bf16x2(lv.x); x[0] += t.x; x[1] += t.y;
    t = unpack_bf16x2(lv.y); x[2] += t.x; x[3] += t.y;
    t = unpack_bf16x2(lv.z); x[4] += t.x; x[5] += t.y;
    t = unpack_bf16x2(lv.w); x[6] += t.x; x[7] += t.y;
  }
#pragma unroll
  for (int e = 0; e < 8; ++e) acc = fmaf(w[e], x[e], acc);
  return acc;
}

constexpr int AF_WARPS = 8;

__global__ void __launch_bounds__(AF_WARPS * 32)
attention_f32_kernel(AttnF32Args a) {
  extern __shared__ float af_smem[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int i = blockIdx.x * AF_WARPS + warp;  // query row inside the group
  const int h = blockIdx.y, g = blockIdx.z;
  float* sc = af_smem + (size_t)warp * (a.Tk + 2 * a.dk);  // [Tk] scores, then q+u [dk], q+v [dk]
  float* qu = sc + a.Tk;
  float* qv = qu + a.dk;
  if (i >= a.Tq) return;
  int klen = a.Tk;
  if (a.k_lens) klen = min(klen, a.k_lens[g]);
  // visible keys [lo, hi): key-length mask, causal (chunk = 1) or streaming chunk mask (utils/mask.py:88-123)
  int lo = 0, hi = klen;
  const int* klist = nullptr;  // prefix-tree attention: explicit key rows (the node's ancestors)
  if (a.key_list) {
    klist = a.key_list + ((long long)g * a.Tq + i) * a.key_list_ld;
    hi = min(a.Tk, a.key_list_len[(long long)g * a.Tq + i]);
  }
  if (a.chunk > 0) {
    hi = min(hi, (i / a.chunk + 1) * a.chunk);
    if (a.left >= 0) lo = max(0, (i / a.chunk - a.left) * a.chunk);
  }
  const bf16* qrow = a.q + ((long long)g * a.Tq + i) * a.ldq + h * a.dk;
  for (int c = lane; c < a.dk; c += 32) {
    const float q = ld_pair(qrow + c, a.q_lo);
    qu[c] = q + (a.bias_u ? a.bias_u[h * a.dk + c] : 0.f);
    qv[c] = q + (a.bias_v ? a.bias_v[h * a.dk + c] : 0.f);
  }
  __syncwarp();
  const float rs = sqrtf((float)a.dk);
  float m = -INFINITY;
  for (int j = lo + lane; j < hi; j += 32) {   // only the visible keys [lo, hi) are ever touched
    float s = -INFINITY;
    {
      const long long kr = klist ? (long long)klist[j] : (long long)g * a.Tk + j;
      const bf16* krow = a.k + kr * a.ldk + h * a.dk;
      float ac = 0.f, bd = 0.f;
      for (int c = 0; c < a.dk; c += 8) ac = dot8_pair(qu + c, krow + c, a.k_lo, ac);
      if (a.p) {
        const bf16* prow = a.p + (long long)j * a.ldp + h * a.dk;
        for (int c = 0; c < a.dk; c += 8) bd = dot8_pair(qv + c, prow + c, a.p_lo, bd);
      }
      s = (ac + bd) / rs;
    }
    sc[j] = s;
    m = fmaxf(m, s);
  }
  m = warp_max(m);
  float sum = 0.f;
  for (int j = lo + lane; j < hi; j += 32) {
    const float e = (m == -INFINITY) ? 0.f : expf(sc[j] - m);
    sc[j] = e;
    sum += e;
  }
  sum = warp_sum(sum);
  __syncwarp();
  const float inv = sum > 0.f ? 1.f / sum : 0.f;  // fully masked row -> zeros (softmax NaN -> masked_fill 0 in the reference)
  bf16* orow = a.out + ((long long)g * a.Tq + i) * a.ldo + h * a.dk;
  // o = sum_j a_j v_j: a lane owns two adjacent columns (one 4-byte load per key row, the warp reads the row's d_k * 2 bytes
  // contiguously); four keys in flight per lane
  for (int c = 2 * lane; c < a.dk; c += 64) {
    float o0 = 0.f, o1 = 0.f;
    auto vrow_of = [&](int j) -> const bf16* {
      const long long vr = klist ? (long long)klist[j] : (long long)g * a.Tk + j;
      return a.v + vr * a.ldv + h * a.dk + c;
    };
    auto ld2 = [&](const bf16* vp) -> float2 {
      float2 t = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(vp));
      if (a.v_lo) {
        const float2 u = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(vp + a.v_lo));
        t.x += u.x;
        t.y += u.y;
      }
      return t;
    };
    int j = lo;
    for (; j + 4 <= hi; j += 4) {
      const float2 v0 = ld2(vrow_of(j)), v1 = ld2(vrow_of(j + 1)), v2 = ld2(vrow_of(j + 2)), v3 = ld2(vrow_of(j + 3));
      const float w0 = sc[j] * inv, w1 = sc[j + 1] * inv, w2 = sc[j + 2] * inv, w3 = sc[j + 3] * inv;
      o0 = fmaf(w0, v0.x, o0); o1 = fmaf(w0, v0.y, o1);
      o0 = fmaf(w1, v1.x, o0); o1 = fmaf(w1, v1.y, o1);
      o0 = fmaf(w2, v2.x, o0); o1 = fmaf(w2, v2.y, o1);
      o0 = fmaf(w3, v3.x, o0); o1 = fmaf(w3, v3.y, o1);
    }
    for (; j < hi; ++j) {
      const float2 v0 = ld2(vrow_of(j));
      const float w0 = sc[j] * inv;
      o0 = fmaf(w0, v0.x, o0);
      o1 = fmaf(w0, v0.y, o1);
    }
    const bf16 h0 = __float2bfloat16(o0), h1 = __float2bfloat16(o1);
    *reinterpret_cast<__nv_bfloat162*>(orow + c) = __nv_bfloat162(h0, h1);
    if (a.o_lo)
      *reinterpret_cast<__nv_bfloat162*>(orow + a.o_lo + c) =
          __nv_bfloat162(__float2bfloat16(o0 - __bfloat162float(h0)), __float2bfloat16(o1 - __bfloat162float(h1)));
  }
}

int launch_attention_f32(const AttnF32Args& a, cudaStream_t stream) {
  RVB_REQUIRE(a.q && a.k && a.v && a.out && a.dk > 0 && a.dk <= 256 && a.dk % 8 == 0, "attention_f32: bad arguments");
  RVB_REQUIRE(a.ldk % 8 == 0 && a.ldp % 8 == 0 && a.k_lo % 8 == 0 && a.p_lo % 8 == 0 &&
                  ((uintptr_t)a.k & 15) == 0 && ((uintptr_t)a.p & 15) == 0,
              "attention_f32: key rows must be 16-byte aligned");
  RVB_REQUIRE(a.ldv % 2 == 0 && a.v_lo % 2 == 0 && a.ldo % 2 == 0 && a.o_lo % 2 == 0 && ((uintptr_t)a.v & 3) == 0 &&
                  ((uintptr_t)a.out & 3) == 0,
              "attention_f32: value / output rows must be 4-byte aligned");
  RVB_REQUIRE((a.chunk <= 0) || a.Tq == a.Tk, "attention_f32: causal / chunk masks need Tq == Tk");
  if (a.groups <= 0 || a.Tq <= 0) return 0;
  const size_t smem = (size_t)AF_WARPS * (a.Tk + 2 * a.dk) * sizeof(float);
  RVB_REQUIRE(smem <= 227 * 1024, "attention_f32: Tk=%d needs %zu B of shared memory", a.Tk, smem);
  static DynSmemOptIn optin;
  if (optin.ensure(attention_f32_kernel, smem)) return -1;
  dim3 grid((a.Tq + AF_WARPS - 1) / AF_WARPS, a.H, a.groups);
  attention_f32_kernel<<<grid, AF_WARPS * 32, smem, stream>>>(a);
  RVB_COUNT_LAUNCH();
  RVB_CHECK_LAUNCH();
  return 0;
}

}  // namespace rvb
