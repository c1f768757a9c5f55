// reverb_b200 — wgmma / TMA attention for the long (encoder self-attention, decoder source-attention) cases, sm_90a.
//
// Rel-pos scores without the second product.  The reference computes (asr/wenet/transformer/attention.py:378-397)
//     s[i,j] = ((q_i + u) . k_j + (q_i + v) . p_j) / sqrt(d_k)          (p_j: ABSOLUTE key position, no rel_shift)
// which is algebraically
//     s[i,j] = ( q_i . (k_j + p_j)  +  (u . k_j + v . p_j) ) / sqrt(d_k) =  ( q_i . K''_j + c_j ) / sqrt(d_k)
// so a small pre-kernel (or the projection GEMM's epilogue) builds K'' = k + p (bf16) and the per-key bias c (fp32)
// once per layer, and the attention itself is ONE tensor-core product per key tile plus a key bias.
//
// Kernel (one CTA = 128 query rows of one (group, head), 256 threads, two CTAs per SM):
//   thread 0   : also issues the TMA loads — Q once, then K'' and V tiles of 64 keys through AT_ST-deep rings
//   warps 0..7 : two warpgroups of 64 query rows each; per key tile
//                  S[64 x 64]  = Q . K''^T        wgmma m64n64k16 x 4, both operands from shared memory
//                  online softmax on the S fragments in registers (scale, key bias, masks, running max / sum)
//                  O[64 x 64] += P~ . V           wgmma m64n64k16 x 4, P~ (bf16) from registers, V MN-major
//                PV of tile j and S of tile j+1 go out as one wgmma group, so a warpgroup waits on the tensor cores
//                once per tile; the other three warpgroups of the SM fill that wait.
// Scores / probabilities never touch shared memory or HBM.
#include <cuda.h>
#include <math.h>
#include <stdlib.h>

#include <algorithm>
#include <type_traits>

#include "kernels.h"

namespace rvb {

constexpr int AT_BM = 128;  // query rows per CTA
constexpr int AT_BN = 64;   // keys per tile
constexpr int AT_DK = 64;
constexpr int AT_ST = 4;    // K'' / V ring stages
// Two warpgroups and no separate producer warp: the register file of each of the SM's four sub-partitions holds 16K
// registers, so two CTAs of 8 warps (4 per sub-partition) may use 128 registers per thread, two CTAs of 9 warps only 96.
constexpr int AT_THREADS = 256;
constexpr uint32_t AT_Q_BYTES = AT_BM * AT_DK * 2;     // 16 KB
constexpr uint32_t AT_TILE_BYTES = AT_BN * AT_DK * 2;  // 8 KB
constexpr uint32_t AT_SMEM_FIXED = AT_Q_BYTES + 2 * AT_ST * AT_TILE_BYTES + 256 /*barriers*/ + 1024 /*align slack*/;

__device__ __forceinline__ float fast_exp2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

struct AttnTcParams {
  bf16* out;
  long long ldo;
  const float* key_bias;  // (groups_kv, H, Tk) fp32 or nullptr
  const int* k_lens;      // per kv group, or nullptr
  int Tq, Tk, H;
  int chunk;   // > 0: chunk mask (utils/mask.py subsequent_chunk_mask): key j visible to query row i iff
               //      max(0, (i/chunk - left) * chunk) [0 when left < 0] <= j < (i/chunk + 1) * chunk; chunk 1 = causal
  int left;    // number of left chunks, < 0 = all
  const uint32_t* key_bits;  // optional per-(query row, key) visibility bits (AttnTcArgs::key_bits)
  int bits_ld;
  float scale_log2;
};

// Which masks a launch applies on top of the key lengths.  Each kind is its own instantiation, so the encoder's
// kernel carries no mask code.
enum AttnMask : int {
  MASK_LENS = 0,   // key lengths only (encoder self-attention, cross-attention)
  MASK_CHUNK = 1,  // chunk / causal mask, p.chunk > 0
  MASK_BITS = 2,   // key_bits, and the chunk / causal mask when p.chunk > 0 (prefix-tree self-attention)
};

// one S = Q . K''^T tile product into s (not committed)
__device__ __forceinline__ void attn_issue_s(float* s, uint64_t qdesc, const uint8_t* k_tile) {
  const uint64_t kdesc = make_sw128_desc(smem_u32(k_tile));
#pragma unroll
  for (int k = 0; k < AT_DK / 16; ++k) wgmma_m64n64k16_ss(s, qdesc + 2 * k, kdesc + 2 * k, k != 0);
}

template <int MASK>
__global__ void __launch_bounds__(AT_THREADS, 2)
attention_tc_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                    const __grid_constant__ CUtensorMap tmV, const AttnTcParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sQ = smem;
  uint8_t* sK = sQ + AT_Q_BYTES;               // AT_ST stages
  uint8_t* sV = sK + AT_ST * AT_TILE_BYTES;    // AT_ST stages
  uint64_t* bars = reinterpret_cast<uint64_t*>(sV + AT_ST * AT_TILE_BYTES);
  uint64_t* q_full = bars;
  uint64_t* k_full = bars + 1;             // [AT_ST]
  uint64_t* k_empty = k_full + AT_ST;      // [AT_ST]
  uint64_t* v_full = k_empty + AT_ST;      // [AT_ST]
  uint64_t* v_empty = v_full + AT_ST;      // [AT_ST]
  static_assert(1 + 4 * AT_ST <= 32, "barrier block is 256 bytes");
  float* s_bias = reinterpret_cast<float*>(bars + 32);   // [ntiles * AT_BN]: key bias * scale*log2e, -inf when masked

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int qtile = blockIdx.x, h = blockIdx.y, g = blockIdx.z;
  const int q0 = qtile * AT_BM;
  int klen = p.Tk;
  if (p.k_lens) klen = min(klen, __ldg(p.k_lens + g));
  // chunk mask: only the key tiles some row of this query tile can see are visited: [jt0, jt0 + ntiles)
  const bool chunked = MASK == MASK_CHUNK || (MASK == MASK_BITS && p.chunk > 0);
  auto vis_lo = [&](int i) { return (chunked && p.left >= 0) ? max(0, (i / p.chunk - p.left) * p.chunk) : 0; };
  auto vis_hi = [&](int i) { return chunked ? min(klen, (i / p.chunk + 1) * p.chunk) : klen; };
  const int jt0 = vis_lo(q0) / AT_BN;
  const int ntiles = max(0, (vis_hi(q0 + AT_BM - 1) + AT_BN - 1) / AT_BN - jt0);
  const long long krow0 = (long long)g * p.Tk;
  // K'' and V tile n into ring stage n % AT_ST (thread 0 only)
  auto load_tile = [&](int n) {
    const int st = n % AT_ST;
    const int krow = (int)(krow0 + (jt0 + n) * AT_BN);
    mbar_expect_tx(&k_full[st], AT_TILE_BYTES);
    tma_load_2d(sK + st * AT_TILE_BYTES, &tmK, &k_full[st], h * AT_DK, krow);
    mbar_expect_tx(&v_full[st], AT_TILE_BYTES);
    tma_load_2d(sV + st * AT_TILE_BYTES, &tmV, &v_full[st], h * AT_DK, krow);
  };

  // Thread 0 issues every load: Q and the first AT_ST tiles right after the barrier init, so they are in flight while
  // the key-bias table is filled; later tiles from the main loop.
  if (threadIdx.x == 0) {
    mbar_init(q_full, 1);
    for (int i = 0; i < AT_ST; ++i) {
      mbar_init(&k_full[i], 1);
      mbar_init(&k_empty[i], 8);   // lane 0 of every warp
      mbar_init(&v_full[i], 1);
      mbar_init(&v_empty[i], 8);
    }
    fence_barrier_init();
    if (ntiles > 0) {
      mbar_expect_tx(q_full, AT_Q_BYTES);
      tma_load_2d(sQ, &tmQ, q_full, h * AT_DK, (int)((long long)g * p.Tq + q0));
      for (int n = 0; n < min(ntiles, AT_ST); ++n) load_tile(n);
    }
  }
  {
    // key bias row of this (group, head), pre-scaled; masked keys -> -inf
    const float* kb = p.key_bias ? p.key_bias + ((long long)g * p.H + h) * p.Tk : nullptr;
    for (int kk = threadIdx.x; kk < ntiles * AT_BN; kk += AT_THREADS) {
      const int key = jt0 * AT_BN + kk;
      s_bias[kk] = (key < klen) ? (kb ? __ldg(kb + key) * p.scale_log2 : 0.f) : -INFINITY;
    }
  }
  __syncthreads();

  const int wg = warp >> 2, wl = warp & 3;
  // this thread's two query rows (fragment rows l/4 and l/4 + 8 of the warp's 16) and its key / dk columns
  // 8j + 2(l%4) + {0, 1}, j = 0..7
  const int rloc = wg * 64 + wl * 16 + (lane >> 2);
  const int row[2] = {q0 + rloc, q0 + rloc + 8};
  const int cq = 2 * (lane & 3);
  float o[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) o[i] = 0.f;
  float m_run[2] = {-INFINITY, -INFINITY}, row_sum[2] = {0.f, 0.f};   // row_sum: this thread's columns only
  const uint64_t qdesc = make_sw128_desc(smem_u32(sQ + wg * (AT_Q_BYTES / 2)));
  // s holds S of the tile being worked on; S(0) goes out here, S(j+1) with PV(j)
  float s[32];
  if (ntiles > 0) {
    mbar_wait(q_full, 0);
    mbar_wait(&k_full[0], 0);
    wgmma_fence_regs<32>(s);
    wgmma_fence();
    attn_issue_s(s, qdesc, sK);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs<32>(s);
    if (lane == 0) mbar_arrive(&k_empty[0]);
  }
  // one key tile; NEXT (every tile but the last) also issues S(j+1).  The last tile is a separate copy, so no branch
  // sits between the products of one wgmma group.
  auto tile = [&](const int j, auto next_tag) {
    constexpr bool next = decltype(next_tag)::value;
    const int st = j % AT_ST, ph = (j / AT_ST) & 1;
    // ---- refill the stage of tile j - 1 once all 8 warps have released it; the ring stays AT_ST - 1 tiles ahead
    if (threadIdx.x == 0 && j > 0 && j - 1 + AT_ST < ntiles) {
      const int n = j - 1 + AT_ST, ph_free = ((n / AT_ST) & 1) ^ 1;
      mbar_wait(&k_empty[n % AT_ST], ph_free);
      mbar_wait(&v_empty[n % AT_ST], ph_free);
      load_tile(n);
    }
    __syncwarp();
    // ---- x = s * scale*log2e + key bias, masks, tile maximum per row
    const int kbase = (jt0 + j) * AT_BN;
    const float* bias = s_bias + j * AT_BN;
    float tmax[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int jj = 0; jj < 8; ++jj) {
      const float2 b2 = *reinterpret_cast<const float2*>(bias + 8 * jj + cq);
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        s[4 * jj + 2 * i] = fmaf(s[4 * jj + 2 * i], p.scale_log2, b2.x);
        s[4 * jj + 2 * i + 1] = fmaf(s[4 * jj + 2 * i + 1], p.scale_log2, b2.y);
      }
    }
    if (chunked) {
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        const int lo = vis_lo(row[i]) - kbase, hi = vis_hi(row[i]) - kbase;   // visible columns: lo <= c < hi
#pragma unroll
        for (int jj = 0; jj < 8; ++jj)
#pragma unroll
          for (int c = 0; c < 2; ++c) {
            const int col = 8 * jj + cq + c;
            if (col < lo || col >= hi) s[4 * jj + 2 * i + c] = -INFINITY;
          }
      }
    }
    if (MASK == MASK_BITS) {
      // arbitrary visibility (prefix-tree self-attention: a node sees its ancestors): one bit per key of the row
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        const uint32_t* mw = p.key_bits + ((long long)g * p.Tq + min(row[i], p.Tq - 1)) * p.bits_ld + (kbase >> 5);
        const uint32_t w0 = __ldg(mw), w1 = __ldg(mw + 1);
#pragma unroll
        for (int jj = 0; jj < 8; ++jj)
#pragma unroll
          for (int c = 0; c < 2; ++c) {
            const int col = 8 * jj + cq + c;
            const uint32_t word = (col < 32) ? w0 : w1;
            if (!((word >> (col & 31)) & 1u)) s[4 * jj + 2 * i + c] = -INFINITY;
          }
      }
    }
#pragma unroll
    for (int jj = 0; jj < 8; ++jj)
#pragma unroll
      for (int i = 0; i < 2; ++i) tmax[i] = fmaxf(tmax[i], fmaxf(s[4 * jj + 2 * i], s[4 * jj + 2 * i + 1]));
    // the four threads of a quad hold the same two rows
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      tmax[i] = fmaxf(tmax[i], __shfl_xor_sync(0xffffffffu, tmax[i], 1));
      tmax[i] = fmaxf(tmax[i], __shfl_xor_sync(0xffffffffu, tmax[i], 2));
    }
    // ---- running maximum: O and the row sums move to the new maximum (rows without a visible key so far keep
    // m = -inf and O = 0; exp2(-inf) = 0 gives them zero weights)
    float m_eff[2];
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const float m_new = fmaxf(m_run[i], tmax[i]);
      const float f = (m_new == -INFINITY || m_run[i] == m_new) ? 1.f : fast_exp2(m_run[i] - m_new);
      m_run[i] = m_new;
      row_sum[i] *= f;
#pragma unroll
      for (int jj = 0; jj < 8; ++jj) {
        o[4 * jj + 2 * i] *= f;
        o[4 * jj + 2 * i + 1] *= f;
      }
      m_eff[i] = (m_new == -INFINITY) ? 0.f : m_new;
    }
    // ---- P~ = exp2(x - m) rounded to bf16, packed as the A fragments of the PV product (k-step ks = keys
    // [16ks, 16ks+16) = accumulator column groups 2ks and 2ks+1); the row sums add the same rounded values
    uint32_t pa[16];
#pragma unroll
    for (int jj = 0; jj < 8; ++jj)
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        const uint32_t w = pack_bf16x2(fast_exp2(s[4 * jj + 2 * i] - m_eff[i]), fast_exp2(s[4 * jj + 2 * i + 1] - m_eff[i]));
        const float2 pr = unpack_bf16x2(w);
        row_sum[i] += pr.x + pr.y;
        pa[2 * jj + i] = w;   // ks = jj / 2: regs {jj even: a0 (row), a1 (row + 8); jj odd: a2, a3}
      }
    // ---- O += P~ . V, then S of the next tile into s (free now that P~ is packed); groups retire in order, so one
    // wait covers both
    const int st1 = (j + 1) % AT_ST;
    mbar_wait(&v_full[st], ph);
    if (next) mbar_wait(&k_full[st1], ((j + 1) / AT_ST) & 1);
    {
      const uint64_t vdesc = make_sw128_desc(smem_u32(sV + st * AT_TILE_BYTES));
      wgmma_fence_regs<32>(o);
      wgmma_fence_regs<32>(s);
      wgmma_fence();
#pragma unroll
      for (int ks = 0; ks < AT_BN / 16; ++ks)
        wgmma_m64n64k16_rs_tb(o, pa + 4 * ks, vdesc + (uint64_t)((ks * 16 * 128) >> 4));   // 16 key rows of 128 B
      if (next) attn_issue_s(s, qdesc, sK + st1 * AT_TILE_BYTES);
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_regs<32>(o);
      wgmma_fence_regs<32>(s);
    }
    if (lane == 0) {
      mbar_arrive(&v_empty[st]);
      if (next) mbar_arrive(&k_empty[st1]);
    }
  };
#pragma unroll 1
  for (int j = 0; j + 1 < ntiles; ++j) tile(j, std::true_type());
  if (ntiles > 0) tile(ntiles - 1, std::false_type());
  // ---- epilogue: O / row_sum -> bf16 -> global (rows without a visible key: zeros)
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    float sum = row_sum[i];
    sum += __shfl_xor_sync(0xffffffffu, sum, 1);
    sum += __shfl_xor_sync(0xffffffffu, sum, 2);
    const float inv = sum > 0.f ? 1.f / sum : 0.f;
    if (row[i] < p.Tq) {
      bf16* orow = p.out + ((long long)g * p.Tq + row[i]) * p.ldo + h * AT_DK;
#pragma unroll
      for (int jj = 0; jj < 8; ++jj)
        *reinterpret_cast<uint32_t*>(orow + 8 * jj + cq) = pack_bf16x2(o[4 * jj + 2 * i] * inv, o[4 * jj + 2 * i + 1] * inv);
    }
  }
}

// K'' = k + p (bf16) and c[b,h,j] = u_h . k_j + v_h . p_j (fp32): one warp per (b, t) row.
__global__ void __launch_bounds__(256)
relpos_prep_kernel(const bf16* __restrict__ k, long long ldk, const bf16* __restrict__ pos, long long ldp,
                   const float* __restrict__ bias_u, const float* __restrict__ bias_v, bf16* __restrict__ kpp,
                   float* __restrict__ cbias, int B, int T, int H, int dk) {
  const long long row = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (row >= (long long)B * T) return;
  const int b = (int)(row / T), t = (int)(row - (long long)b * T);
  const int d = H * dk;
  const bf16* kr = k + row * ldk;
  const bf16* pr = pos + (long long)t * ldp;
  bf16* orow = kpp + row * d;
  for (int h = 0; h < H; ++h) {
    float acc = 0.f;
    for (int c = 2 * lane; c < dk; c += 64) {
      const int col = h * dk + c;
      float2 kv = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(kr + col));
      float2 pv = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(pr + col));
      *reinterpret_cast<uint32_t*>(orow + col) = pack_bf16x2(kv.x + pv.x, kv.y + pv.y);
      acc += __ldg(bias_u + col) * kv.x + __ldg(bias_u + col + 1) * kv.y + __ldg(bias_v + col) * pv.x +
             __ldg(bias_v + col + 1) * pv.y;
    }
    acc = warp_sum(acc);
    if (lane == 0) cbias[((long long)b * H + h) * T + t] = acc;
  }
}

// Same, vectorised: a lane owns 8 consecutive columns (16-byte loads / stores), a head is dk/8 adjacent lanes, so one
// warp pass covers 256 columns and the per-head dot products reduce with log2(dk/8) shuffles.
template <int LPH /* lanes per head = dk / 8 */>
__global__ void __launch_bounds__(256)
relpos_prep_vec_kernel(const bf16* __restrict__ k, long long ldk, const bf16* __restrict__ pos, long long ldp,
                       const float* __restrict__ bias_u, const float* __restrict__ bias_v, bf16* __restrict__ kpp,
                       float* __restrict__ cbias, int B, int T, int H) {
  const long long row = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (row >= (long long)B * T) return;
  const int b = (int)(row / T), t = (int)(row - (long long)b * T);
  const int d = H * LPH * 8;
  const bf16* kr = k + row * ldk;
  const bf16* pr = pos + (long long)t * ldp;
  bf16* orow = kpp + row * d;
  for (int c0 = 0; c0 < d; c0 += 256) {
    const int col = c0 + lane * 8;
    float acc = 0.f;
    if (col < d) {
      const uint4 kv = *reinterpret_cast<const uint4*>(kr + col);
      const uint4 pv = *reinterpret_cast<const uint4*>(pr + col);
      const float4 u0 = __ldg(reinterpret_cast<const float4*>(bias_u + col));
      const float4 u1 = __ldg(reinterpret_cast<const float4*>(bias_u + col) + 1);
      const float4 v0 = __ldg(reinterpret_cast<const float4*>(bias_v + col));
      const float4 v1 = __ldg(reinterpret_cast<const float4*>(bias_v + col) + 1);
      const float2 k0 = unpack_bf16x2(kv.x), k1 = unpack_bf16x2(kv.y), k2 = unpack_bf16x2(kv.z), k3 = unpack_bf16x2(kv.w);
      const float2 p0 = unpack_bf16x2(pv.x), p1 = unpack_bf16x2(pv.y), p2 = unpack_bf16x2(pv.z), p3 = unpack_bf16x2(pv.w);
      uint4 o;
      o.x = pack_bf16x2(k0.x + p0.x, k0.y + p0.y);
      o.y = pack_bf16x2(k1.x + p1.x, k1.y + p1.y);
      o.z = pack_bf16x2(k2.x + p2.x, k2.y + p2.y);
      o.w = pack_bf16x2(k3.x + p3.x, k3.y + p3.y);
      *reinterpret_cast<uint4*>(orow + col) = o;
      acc = u0.x * k0.x + u0.y * k0.y + u0.z * k1.x + u0.w * k1.y + u1.x * k2.x + u1.y * k2.y + u1.z * k3.x + u1.w * k3.y +
            v0.x * p0.x + v0.y * p0.y + v0.z * p1.x + v0.w * p1.y + v1.x * p2.x + v1.y * p2.y + v1.z * p3.x + v1.w * p3.y;
    }
#pragma unroll
    for (int o = LPH / 2; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if (col < d && (lane % LPH) == 0) cbias[((long long)b * H + col / (LPH * 8)) * T + t] = acc;
  }
}

int launch_relpos_prep(const bf16* k, int ldk, const bf16* pos, int ldp, const float* bias_u, const float* bias_v,
                       bf16* kpp, float* cbias, int B, int T, int H, int dk, cudaStream_t stream) {
  RVB_REQUIRE(dk % 2 == 0, "relpos_prep: d_k must be even");
  const long long rows = (long long)B * T;
  if (rows <= 0) return 0;
  const unsigned grid = (unsigned)((rows + 7) / 8);
  const bool aligned = (ldk % 8 == 0) && (ldp % 8 == 0) && ((reinterpret_cast<uintptr_t>(k) & 15) == 0) &&
                       ((reinterpret_cast<uintptr_t>(pos) & 15) == 0) && ((reinterpret_cast<uintptr_t>(kpp) & 15) == 0) &&
                       ((reinterpret_cast<uintptr_t>(bias_u) & 15) == 0) && ((reinterpret_cast<uintptr_t>(bias_v) & 15) == 0);
  if (aligned && dk == 64)
    relpos_prep_vec_kernel<8><<<grid, 256, 0, stream>>>(k, ldk, pos, ldp, bias_u, bias_v, kpp, cbias, B, T, H);
  else if (aligned && dk == 128)
    relpos_prep_vec_kernel<16><<<grid, 256, 0, stream>>>(k, ldk, pos, ldp, bias_u, bias_v, kpp, cbias, B, T, H);
  else if (aligned && dk == 32)
    relpos_prep_vec_kernel<4><<<grid, 256, 0, stream>>>(k, ldk, pos, ldp, bias_u, bias_v, kpp, cbias, B, T, H);
  else
    relpos_prep_kernel<<<grid, 256, 0, stream>>>(k, ldk, pos, ldp, bias_u, bias_v, kpp, cbias, B, T, H, dk);
  RVB_COUNT_LAUNCH();
  RVB_CHECK_LAUNCH();
  return 0;
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFn g_encode_att = nullptr;

static int tmap_2d(CUtensorMap* m, const void* base, long long cols, long long rows, long long ld_elems,
                   int box_rows) {
  cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  cuuint64_t str[1] = {(cuuint64_t)ld_elems * 2};
  cuuint32_t box[2] = {64, (cuuint32_t)box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = g_encode_att(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), dims, str, box, estr,
                            CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                            CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  RVB_REQUIRE(r == CUDA_SUCCESS, "attention: cuTensorMapEncodeTiled failed (%d)", (int)r);
  return 0;
}

static int attn_mask_kind(bool chunk_or_causal, bool key_bits) {
  return key_bits ? MASK_BITS : chunk_or_causal ? MASK_CHUNK : MASK_LENS;
}

// Q, both rings, barriers and the key-bias row: 86 272 B at Tk = 748.  Two CTAs fit the 228 KB of an SM (1 KB of it
// reserved per CTA) up to Tk = 8 128; longer key rows run one CTA per SM.
static size_t attn_smem_bytes(int Tk) { return AT_SMEM_FIXED + (size_t)((Tk + AT_BN - 1) / AT_BN) * AT_BN * sizeof(float); }

template <int MASK>
static int attn_opt_in(size_t smem) {
  static DynSmemOptIn optin;
  return optin.ensure(attention_tc_kernel<MASK>, smem);
}

template <int MASK>
static int attn_launch(dim3 grid, size_t smem, cudaStream_t stream, const CUtensorMap& tmQ, const CUtensorMap& tmK,
                       const CUtensorMap& tmV, const AttnTcParams& p) {
  if (attn_opt_in<MASK>(smem)) return -1;
  attention_tc_kernel<MASK><<<grid, AT_THREADS, smem, stream>>>(tmQ, tmK, tmV, p);
  return 0;
}

template <int MASK>
static int attn_blocks_per_sm(size_t smem, int* blocks) {
  if (attn_opt_in<MASK>(smem)) return -1;
  RVB_CHECK_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(blocks, attention_tc_kernel<MASK>, AT_THREADS, smem));
  return 0;
}

int attention_tc_blocks_per_sm(int Tk, bool chunk_or_causal, bool key_bits, int* blocks) {
  const size_t smem = attn_smem_bytes(Tk);
  switch (attn_mask_kind(chunk_or_causal, key_bits)) {
    case MASK_LENS: return attn_blocks_per_sm<MASK_LENS>(smem, blocks);
    case MASK_CHUNK: return attn_blocks_per_sm<MASK_CHUNK>(smem, blocks);
    default: return attn_blocks_per_sm<MASK_BITS>(smem, blocks);
  }
}

// q: (groups*Tq, ldq) rows with head h at columns [h*64, h*64+64) (+ the pointer offset already applied), same for k, v.
int launch_attention_tc(const AttnTcArgs& a, cudaStream_t stream) {
  RVB_REQUIRE(a.dk == AT_DK, "attention_tc: only d_k = 64 is built");
  RVB_REQUIRE(a.ldq % 8 == 0 && a.ldk % 8 == 0 && a.ldv % 8 == 0 && a.ldo % 8 == 0, "attention_tc: ld %% 8 != 0");
  RVB_REQUIRE(((uintptr_t)a.q & 15) == 0 && ((uintptr_t)a.k & 15) == 0 && ((uintptr_t)a.v & 15) == 0 &&
                  ((uintptr_t)a.out & 15) == 0,
              "attention_tc: operands must be 16-byte aligned");
  RVB_REQUIRE((!a.causal && a.chunk <= 0) || a.Tq == a.Tk, "attention_tc: causal / chunk masks need Tq == Tk");
  RVB_REQUIRE(!(a.causal && a.chunk > 0), "attention_tc: causal and chunk mask are exclusive");
  if (a.groups <= 0 || a.Tq <= 0) return 0;
  if (g_encode_att == nullptr) {
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult qres;
    RVB_CHECK_CUDA(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres));
    RVB_REQUIRE(fn != nullptr && qres == cudaDriverEntryPointSuccess, "cuTensorMapEncodeTiled not available");
    g_encode_att = reinterpret_cast<EncodeTiledFn>(fn);
  }
  AttnTcParams p;
  p.out = a.out;
  p.ldo = a.ldo;
  p.key_bias = a.key_bias;
  p.k_lens = a.k_lens;
  p.Tq = a.Tq;
  p.Tk = a.Tk;
  p.H = a.H;
  p.chunk = a.causal ? 1 : (a.chunk > 0 ? a.chunk : 0);
  p.left = a.causal ? -1 : a.left_chunks;
  p.key_bits = a.key_bits;
  p.bits_ld = a.bits_ld;
  RVB_REQUIRE(a.key_bits == nullptr || a.bits_ld >= 2 * ((a.Tk + 63) / 64), "attention_tc: key_bits rows are too short");
  p.scale_log2 = a.scale * 1.4426950408889634f;
  CUtensorMap tmQ, tmK, tmV;
  if (tmap_2d(&tmQ, a.q, (long long)a.H * AT_DK, (long long)a.groups * a.Tq, a.ldq, AT_BM)) return -1;
  if (tmap_2d(&tmK, a.k, (long long)a.H * AT_DK, (long long)a.groups * a.Tk, a.ldk, AT_BN)) return -1;
  if (tmap_2d(&tmV, a.v, (long long)a.H * AT_DK, (long long)a.groups * a.Tk, a.ldv, AT_BN)) return -1;
  dim3 grid((a.Tq + AT_BM - 1) / AT_BM, a.H, a.groups);
  const size_t smem = attn_smem_bytes(a.Tk);
  RVB_REQUIRE(smem <= 227 * 1024, "attention_tc: Tk=%d needs %zu B of shared memory", a.Tk, smem);
  int rc;
  switch (attn_mask_kind(a.causal || a.chunk > 0, a.key_bits != nullptr)) {
    case MASK_LENS: rc = attn_launch<MASK_LENS>(grid, smem, stream, tmQ, tmK, tmV, p); break;
    case MASK_CHUNK: rc = attn_launch<MASK_CHUNK>(grid, smem, stream, tmQ, tmK, tmV, p); break;
    default: rc = attn_launch<MASK_BITS>(grid, smem, stream, tmQ, tmK, tmV, p); break;
  }
  if (rc) return rc;
  RVB_COUNT_LAUNCH();
  RVB_CHECK_LAUNCH();
  return 0;
}

}  // namespace rvb
