// reverb_b200 — fused (flash-style) multi-head attention for the Conformer encoder and the rescoring decoder.
//
// Encoder (reference: asr/wenet/transformer/attention.py:317-399, rel_shift disabled at :391-394):
//     s[i,j] = ((q_i + u_h) . k_j + (q_i + v_h) . p_j) / sqrt(d_k),  key-padding mask, softmax, masked_fill(0), . V
//   p_j = linear_pos(pos_emb)[j] is indexed by the ABSOLUTE key position, so the "bd" term is just a second
//   QK^T-shaped product against a batch-shared key matrix: both accumulate into the same score tile.
// Decoder (attention.py:129-200): plain scaled dot product with a causal+length mask (self-attn) or no mask
//   (src-attn over one utterance's encoder output, shared by its N hypotheses: q_per_kv = N de-duplicates the
//   reference's `encoder_out.repeat(N,1,1)`, asr_model.py:895).
//
// Scores are never materialised in HBM (the reference writes (B,H,T',T') fp32 = 2.29 GB per layer at B=64).
// Round-1 implementation: bf16 mma.sync.m16n8k16 with fp32 accumulation, online softmax in registers, K/V/P tiles
// double-buffered through shared memory with cp.async.  (attention_tc.cu is the wgmma version.)
#include "kernels.h"

namespace rvb {

constexpr int ATT_BM = 128;  // queries per CTA (16 per warp, 8 warps): halves the K/V/P re-reads vs 64
constexpr int ATT_THREADS = ATT_BM * 2;
constexpr int ATT_BN = 64;   // keys per tile
constexpr int ATT_PAD = 8;   // bf16 padding per smem row (keeps ldmatrix conflict-free)

__device__ __forceinline__ void cp_async16(void* smem, const void* gmem, bool valid) {
  uint32_t s = smem_u32(smem);
  int sz = valid ? 16 : 0;
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(s), "l"(gmem), "r"(sz) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
  asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}
__device__ __forceinline__ void ldmatrix_x4(uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3, const void* p) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3)
               : "r"(smem_u32(p)));
}
__device__ __forceinline__ void ldmatrix_x4_trans(uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3,
                                                  const void* p) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3)
               : "r"(smem_u32(p)));
}
__device__ __forceinline__ void mma_bf16(float* c, const uint32_t* a, uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

struct AttnKParams {
  const bf16* q;
  const bf16* k;
  const bf16* v;
  const bf16* p;
  const float* bias_u;
  const float* bias_v;
  bf16* out;
  long long ldq, ldk, ldv, ldp, ldo;
  int Tq, Tk, H, q_per_kv;
  const int* k_lens;
  const int* q_lens;
  int causal;
  float scale_log2;  // scale * log2(e)
};

template <int DK, bool HAS_POS>
__global__ void __launch_bounds__(ATT_THREADS, (DK <= 64) ? 2 : 1) attention_kernel(const AttnKParams prm) {
  constexpr int LDS = DK + ATT_PAD;          // smem row stride (elements)
  constexpr int TILE = ATT_BN * LDS;         // elements per staged matrix
  constexpr int NMAT = HAS_POS ? 3 : 2;      // K, V, (P)
  constexpr int KSTEPS = DK / 16;
  constexpr int NT_S = ATT_BN / 8;           // score n-tiles per key tile
  constexpr int NT_O = DK / 8;               // output n-tiles
  extern __shared__ __align__(16) uint8_t smem_att[];
  bf16* sbuf = reinterpret_cast<bf16*>(smem_att);  // [2][NMAT][TILE]

  const int qtile = blockIdx.x, h = blockIdx.y, bq = blockIdx.z;
  const int bk = bq / prm.q_per_kv;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane >> 2, t4 = lane & 3;
  const int q0 = qtile * ATT_BM;

  int klen = prm.Tk;
  if (prm.k_lens) klen = min(klen, __ldg(prm.k_lens + bk));
  if (prm.q_lens) klen = min(klen, __ldg(prm.q_lens + bq));
  int kend = klen;
  if (prm.causal) kend = min(kend, q0 + ATT_BM);
  const int ntiles = (kend + ATT_BN - 1) / ATT_BN;

  const bf16* kbase = prm.k + (long long)bk * prm.Tk * prm.ldk + h * DK;
  const bf16* vbase = prm.v + (long long)bk * prm.Tk * prm.ldv + h * DK;
  const bf16* pbase = HAS_POS ? (prm.p + h * DK) : nullptr;

  auto load_tile = [&](int tile, int buf) {
    bf16* dst = sbuf + (size_t)buf * NMAT * TILE;
    constexpr int CH = DK / 8;  // 16-byte chunks per row
    for (int i = threadIdx.x; i < ATT_BN * CH; i += ATT_THREADS) {
      int r = i / CH, c = i - r * CH;
      int key = tile * ATT_BN + r;
      bool ok = key < prm.Tk;
      long long kr = ok ? key : 0;
      cp_async16(dst + r * LDS + c * 8, kbase + kr * prm.ldk + c * 8, ok);
      cp_async16(dst + TILE + r * LDS + c * 8, vbase + kr * prm.ldv + c * 8, ok);
      if (HAS_POS) cp_async16(dst + 2 * TILE + r * LDS + c * 8, pbase + kr * prm.ldp + c * 8, ok);
    }
  };

  if (ntiles > 0) load_tile(0, 0);
  cp_async_commit();

  // ---- Q fragments (registers), with the per-head position biases folded in
  uint32_t qa[KSTEPS][4];
  uint32_t qb[HAS_POS ? KSTEPS : 1][4];
  {
    const int r0 = q0 + warp * 16 + g, r1 = r0 + 8;
    const bf16* qr0 = prm.q + ((long long)bq * prm.Tq + min(r0, prm.Tq - 1)) * prm.ldq + h * DK;
    const bf16* qr1 = prm.q + ((long long)bq * prm.Tq + min(r1, prm.Tq - 1)) * prm.ldq + h * DK;
#pragma unroll
    for (int ks = 0; ks < KSTEPS; ++ks) {
#pragma unroll
      for (int half = 0; half < 2; ++half) {
        const int col = ks * 16 + half * 8 + 2 * t4;
        uint32_t u0 = *reinterpret_cast<const uint32_t*>(qr0 + col);
        uint32_t u1 = *reinterpret_cast<const uint32_t*>(qr1 + col);
        if (HAS_POS) {
          float2 f0 = unpack_bf16x2(u0), f1 = unpack_bf16x2(u1);
          const float bu0 = __ldg(prm.bias_u + h * DK + col), bu1 = __ldg(prm.bias_u + h * DK + col + 1);
          const float bv0 = __ldg(prm.bias_v + h * DK + col), bv1 = __ldg(prm.bias_v + h * DK + col + 1);
          qa[ks][half * 2 + 0] = pack_bf16x2(f0.x + bu0, f0.y + bu1);
          qa[ks][half * 2 + 1] = pack_bf16x2(f1.x + bu0, f1.y + bu1);
          qb[ks][half * 2 + 0] = pack_bf16x2(f0.x + bv0, f0.y + bv1);
          qb[ks][half * 2 + 1] = pack_bf16x2(f1.x + bv0, f1.y + bv1);
        } else {
          qa[ks][half * 2 + 0] = u0;
          qa[ks][half * 2 + 1] = u1;
        }
      }
    }
  }

  float o[NT_O][4];
#pragma unroll
  for (int i = 0; i < NT_O; ++i) o[i][0] = o[i][1] = o[i][2] = o[i][3] = 0.f;
  float mrow[2] = {-INFINITY, -INFINITY};
  float lrow[2] = {0.f, 0.f};
  const int row_g[2] = {q0 + warp * 16 + g, q0 + warp * 16 + g + 8};

  for (int tile = 0; tile < ntiles; ++tile) {
    const int buf = tile & 1;
    if (tile + 1 < ntiles) load_tile(tile + 1, buf ^ 1);
    cp_async_commit();
    cp_async_wait<1>();
    __syncthreads();
    const bf16* sK = sbuf + (size_t)buf * NMAT * TILE;
    const bf16* sV = sK + TILE;
    const bf16* sP = sK + 2 * TILE;

    float s[NT_S][4];
#pragma unroll
    for (int i = 0; i < NT_S; ++i) s[i][0] = s[i][1] = s[i][2] = s[i][3] = 0.f;
#pragma unroll
    for (int ks = 0; ks < KSTEPS; ++ks) {
#pragma unroll
      for (int np = 0; np < NT_S / 2; ++np) {
        // four 8x8 matrices: (keys np*16 + {0,8}) x (k cols ks*16 + {0,8})
        const int mid = lane >> 3, r = lane & 7;
        const int krow = np * 16 + (mid >> 1) * 8 + r;
        const int kcol = ks * 16 + (mid & 1) * 8;
        uint32_t b0, b1, b2, b3;
        ldmatrix_x4(b0, b1, b2, b3, sK + krow * LDS + kcol);
        mma_bf16(s[2 * np], qa[ks], b0, b1);
        mma_bf16(s[2 * np + 1], qa[ks], b2, b3);
        if (HAS_POS) {
          ldmatrix_x4(b0, b1, b2, b3, sP + krow * LDS + kcol);
          mma_bf16(s[2 * np], qb[ks], b0, b1);
          mma_bf16(s[2 * np + 1], qb[ks], b2, b3);
        }
      }
    }
    // ---- mask + online softmax (log2 domain)
    float mnew[2] = {mrow[0], mrow[1]};
#pragma unroll
    for (int nt = 0; nt < NT_S; ++nt) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int key = tile * ATT_BN + nt * 8 + 2 * t4 + (e & 1);
        const int rr = e >> 1;
        bool ok = key < klen;
        if (prm.causal) ok = ok && (key <= row_g[rr]);
        float x = ok ? s[nt][e] * prm.scale_log2 : -INFINITY;
        s[nt][e] = x;
        mnew[rr] = fmaxf(mnew[rr], x);
      }
    }
#pragma unroll
    for (int rr = 0; rr < 2; ++rr) {
      mnew[rr] = fmaxf(mnew[rr], __shfl_xor_sync(0xffffffffu, mnew[rr], 1));
      mnew[rr] = fmaxf(mnew[rr], __shfl_xor_sync(0xffffffffu, mnew[rr], 2));
    }
    float corr[2], msub[2];
#pragma unroll
    for (int rr = 0; rr < 2; ++rr) {
      msub[rr] = (mnew[rr] == -INFINITY) ? 0.f : mnew[rr];
      corr[rr] = exp2f(mrow[rr] - msub[rr]);  // mrow = -inf -> 0
      mrow[rr] = mnew[rr];
      lrow[rr] *= corr[rr];
    }
#pragma unroll
    for (int i = 0; i < NT_O; ++i) {
      o[i][0] *= corr[0];
      o[i][1] *= corr[0];
      o[i][2] *= corr[1];
      o[i][3] *= corr[1];
    }
    uint32_t pa[NT_S / 2][4];
#pragma unroll
    for (int nt = 0; nt < NT_S; ++nt) {
      float p0 = exp2f(s[nt][0] - msub[0]), p1 = exp2f(s[nt][1] - msub[0]);
      float p2 = exp2f(s[nt][2] - msub[1]), p3 = exp2f(s[nt][3] - msub[1]);
      lrow[0] += p0 + p1;
      lrow[1] += p2 + p3;
      pa[nt >> 1][(nt & 1) * 2 + 0] = pack_bf16x2(p0, p1);
      pa[nt >> 1][(nt & 1) * 2 + 1] = pack_bf16x2(p2, p3);
    }
    // ---- O += P . V
#pragma unroll
    for (int kk = 0; kk < ATT_BN / 16; ++kk) {
#pragma unroll
      for (int np = 0; np < NT_O / 2; ++np) {
        const int mid = lane >> 3, r = lane & 7;
        const int vrow = kk * 16 + (mid & 1) * 8 + r;
        const int vcol = np * 16 + (mid >> 1) * 8;
        uint32_t b0, b1, b2, b3;
        ldmatrix_x4_trans(b0, b1, b2, b3, sV + vrow * LDS + vcol);
        mma_bf16(o[2 * np], pa[kk], b0, b1);
        mma_bf16(o[2 * np + 1], pa[kk], b2, b3);
      }
    }
    __syncthreads();
  }
  cp_async_wait<0>();

  // ---- finalize
#pragma unroll
  for (int rr = 0; rr < 2; ++rr) {
    lrow[rr] += __shfl_xor_sync(0xffffffffu, lrow[rr], 1);
    lrow[rr] += __shfl_xor_sync(0xffffffffu, lrow[rr], 2);
  }
  const float inv0 = lrow[0] > 0.f ? 1.f / lrow[0] : 0.f;
  const float inv1 = lrow[1] > 0.f ? 1.f / lrow[1] : 0.f;
#pragma unroll
  for (int nt = 0; nt < NT_O; ++nt) {
    const int col = h * DK + nt * 8 + 2 * t4;
    if (row_g[0] < prm.Tq)
      *reinterpret_cast<uint32_t*>(prm.out + ((long long)bq * prm.Tq + row_g[0]) * prm.ldo + col) =
          pack_bf16x2(o[nt][0] * inv0, o[nt][1] * inv0);
    if (row_g[1] < prm.Tq)
      *reinterpret_cast<uint32_t*>(prm.out + ((long long)bq * prm.Tq + row_g[1]) * prm.ldo + col) =
          pack_bf16x2(o[nt][2] * inv1, o[nt][3] * inv1);
  }
}

template <int DK, bool HAS_POS>
static int launch_attn_t(const AttnKParams& p, int Bq, cudaStream_t stream) {
  constexpr int NMAT = HAS_POS ? 3 : 2;
  const size_t smem = (size_t)2 * NMAT * ATT_BN * (DK + ATT_PAD) * sizeof(bf16);
  static DynSmemOptIn optin;
  if (optin.ensure(attention_kernel<DK, HAS_POS>, smem)) return -1;
  dim3 grid((p.Tq + ATT_BM - 1) / ATT_BM, p.H, Bq);
  attention_kernel<DK, HAS_POS><<<grid, ATT_THREADS, smem, stream>>>(p);
  RVB_COUNT_LAUNCH();
  RVB_CHECK_LAUNCH();
  return 0;
}

int launch_attention(const AttnArgs& a, cudaStream_t stream) {
  RVB_REQUIRE(a.q && a.k && a.v && a.out, "attention: null pointer");
  RVB_REQUIRE(a.dk == 32 || a.dk == 64 || a.dk == 128, "attention: d_k=%d unsupported (32/64/128)", a.dk);
  RVB_REQUIRE(a.ldq % 8 == 0 && a.ldk % 8 == 0 && a.ldv % 8 == 0 && a.ldo % 2 == 0 && (a.p == nullptr || a.ldp % 8 == 0),
              "attention: leading dimensions must be multiples of 8 elements");
  if (a.Bq <= 0 || a.Tq <= 0) return 0;
  AttnKParams p;
  p.q = a.q; p.k = a.k; p.v = a.v; p.p = a.p;
  p.bias_u = a.bias_u; p.bias_v = a.bias_v;
  p.out = a.out;
  p.ldq = a.ldq; p.ldk = a.ldk; p.ldv = a.ldv; p.ldp = a.ldp; p.ldo = a.ldo;
  p.Tq = a.Tq; p.Tk = a.Tk; p.H = a.H;
  p.q_per_kv = a.q_per_kv > 0 ? a.q_per_kv : 1;
  p.k_lens = a.k_lens; p.q_lens = a.q_lens;
  p.causal = a.causal;
  p.scale_log2 = a.scale * 1.4426950408889634f;
  const bool pos = a.p != nullptr;
  if (pos) RVB_REQUIRE(a.bias_u && a.bias_v, "attention: rel-pos needs bias_u / bias_v");
#define RVB_ATT(DKV)                                                    \
  return pos ? launch_attn_t<DKV, true>(p, a.Bq, stream) : launch_attn_t<DKV, false>(p, a.Bq, stream)
  if (a.dk == 32) { RVB_ATT(32); }
  if (a.dk == 64) { RVB_ATT(64); }
  RVB_ATT(128);
#undef RVB_ATT
}

}  // namespace rvb
