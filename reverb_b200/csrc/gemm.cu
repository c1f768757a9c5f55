// reverb_b200 — persistent, warp-specialised wgmma + TMA GEMM for sm_90a.
//
//   C[M,N] = A[M,K] . W[N,K]^T  (+bias, activation, residual)      A, W: bf16, K-major; fp32 accumulate
//
// One kernel serves every dense layer on the hot path: the Conformer FFN / attention projections / pointwise convs
// (reference: asr/wenet/transformer/positionwise_feed_forward.py:47-55, attention.py:52-79, convolution.py:129,139),
// the CTC / decoder output layers (ctc.py:106-114, decoder.py:164-166) and — with `conv_mode` — the second
// Conv2d(d,d,3,stride 2) of Conv2dSubsampling4 (subsampling.py:186-189) as an implicit GEMM whose A tiles are fetched
// straight out of the channels-last conv1 activation by 4-D TMA boxes (no im2col buffer).
//
// Structure per CTA (384 threads, 1 CTA / SM, grid = #SMs, static round-robin tile scheduler), see gemm_wg_kernel:
//   warpgroup 0    : TMA producer (one thread, 40 registers) — fills a 4-deep ring of {A 128x64, W BNx64} bf16 tiles
//                    (SWIZZLE_128B)
//   warpgroups 1-2 : ping-pong consumers (232 registers), alternate whole tiles: wgmma m64nBNk16 x 2 from shared memory
//                    into registers, then — while the other warpgroup runs the next tile's MMAs — the fused epilogue
//                    (bias / ReLU / SiLU / GLU / residual(+row mask) / log-sum-exp / rel-pos keys) on a shared-memory
//                    copy of the accumulator; outputs pass through a per-warp XOR-swizzled staging tile so global
//                    accesses are coalesced.
// Wide bf16-output layers (bias / ReLU / SiLU, N % 256 == 0, at least one wave of tiles: FFN1, the conv2 implicit GEMM)
// run on 128 x 256 tiles instead (gemm_wide_kernel): both consumer warpgroups share one tile and one 256-wide weight
// tile per k-block, and the producer warpgroup's idle warps store the bf16 output tile.  RVB_GEMM_WIDE=0 (read per
// call) keeps them on 128 x 128 tiles; the outputs are the same bits.
// Tuning aid (environment, read once): RVB_GEMM_SKIP_EPI=1|2|3 (main loop only / no global stores / accumulator
// reads + math only — results are wrong by construction; tools/gemm_bench.py).  RVB_GEMM=simt selects the CUDA-core
// bring-up kernel, RVB_GEMM=narrow 64-wide tiles wherever the epilogue allows them.
#include <cuda.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <mutex>
#include <vector>

#include "kernels.h"

namespace rvb {

static int g_gemm_impl = -1;
void set_gemm_impl(int impl) { g_gemm_impl = impl; }
int get_gemm_impl() {
  if (g_gemm_impl < 0) {
    const char* e = getenv("RVB_GEMM");
    // default: wgmma kernel; RVB_GEMM=simt -> CUDA-core bring-up kernel, RVB_GEMM=narrow -> wgmma with 64-wide tiles
    g_gemm_impl = (e && strcmp(e, "simt") == 0) ? 1 : (e && strcmp(e, "narrow") == 0) ? 2 : 0;
  }
  return g_gemm_impl;
}

struct GemmKParams {
  int M, N, K, num_k_blocks;
  int tiles_n, num_tiles;
  const float* bias;
  int act, out_mode;
  void* out;
  long long ldo;
  float alpha;
  const int* row_lens;
  int rows_per_batch;
  int conv_mode, conv_T2, conv_F2, conv_tt, conv_cblocks;
  int conv_orow_mul;   // rows of `ldo` elements per (b, t'): F2, or 2*F2 for the hi/lo pair output (conv_pair_out)
  const int* lse_gather;  // OUT_LSE (kernels.h)
  float2* lse_part;
  float* lse_tgt;
  int lse_nslab;
  const bf16* rp_pos;   // EPI_BF16_RELPOS (GemmArgs::rp_*)
  long long rp_ldp;
  int rp_T, rp_H, rp_col0;
  const float* rp_u;
  const float* rp_v;
  float* rp_cb;
  int x3;              // bf16x3 accurate mode: num_k_blocks = 3 * kb_seg, pass s reads A half (s == 1), W half (s == 2)
  int kb_seg;          // k-blocks per pass (K / 64)
  int a_lo_ofs;        // column offset (elements) of the lo half of A: K (plain) or C (conv_mode: channel offset)
  int w_lo_ofs;        // column offset of the lo half of W: K
  long long out_split; // > 0: bf16 outputs are written as a hi / lo pair, lo at column + out_split
  int debug_skip_epi;  // RVB_GEMM_SKIP_EPI=1 (tuning aid): epilogue warps only hand the accumulator back, no stores
  int glu_coalesced;   // ACT_GLU with 16-byte aligned output rows (always true after the launch checks)
  int bf16_coalesced;  // bf16 output rows are 16-byte aligned -> staged, coalesced epilogue (see drain_tile)
  int f32_coalesced;  // fp32 output rows are 16-byte aligned -> staged, coalesced epilogue (see drain_tile)
  const int* grp;      // grouped output (GemmArgs::grp): group of each utterance of rows_per_batch rows, or nullptr
  int group_n;         // output columns per group
  int grp_slots;       // grouped output: utterance slots per M tile (the most utterances 128 rows can touch)
  // simt fallback only
  const bf16* A;
  const bf16* W;
  long long lda, ldw;
  int conv_T1h, conv_F1, conv_C;
};

struct TileCoord {
  int n0;        // first accumulator column (of W / bias)
  int row0;      // plain: first row; conv: t0
  int b, f;      // conv only
  int g;         // grouped output: the group of the tile's N block (0 otherwise); output column = n - g * group_n
};

// Grouped output: the tiles of M tile mt are (slot u, column block j) — u-th utterance among the tile's rows, j-th BN
// block of that utterance's group — so a launch enumerates grp_slots * group_n / BN tiles per M tile, whatever G is.
__device__ __forceinline__ TileCoord decode_tile(const GemmKParams& p, int tile, int BN) {
  TileCoord t;
  int nb = tile % p.tiles_n;
  int mt = tile / p.tiles_n;
  t.n0 = nb * BN;
  t.g = 0;
  if (p.grp != nullptr) {
    const int nbg = p.group_n / BN;
    t.g = __ldg(p.grp + (mt * 128) / p.rows_per_batch + nb / nbg);
    t.n0 = t.g * p.group_n + (nb % nbg) * BN;
  }
  if (p.conv_mode) {
    t.f = mt % p.conv_F2;
    int r = mt / p.conv_F2;
    t.row0 = (r % p.conv_tt) * 128;
    t.b = r / p.conv_tt;
  } else {
    t.row0 = mt * 128;
    t.b = 0;
    t.f = 0;
  }
  return t;
}

// Whether a tile has rows to write: always, except under a grouped output, where its slot must hold an utterance of
// the tile's rows whose group no earlier slot of the tile has (each group present among the rows is computed once).
// The producer and both consumer warpgroups walk the CTA's tiles through this same predicate, so they agree on the
// ring order.
__device__ __forceinline__ bool tile_active(const GemmKParams& p, int tile, int BN) {
  if (p.grp == nullptr) return true;
  const int r0 = (tile / p.tiles_n) * 128;
  const int b0 = r0 / p.rows_per_batch;
  const int b = b0 + (tile % p.tiles_n) / (p.group_n / BN);
  if (b > (min(r0 + 128, p.M) - 1) / p.rows_per_batch) return false;
  const int g = __ldg(p.grp + b);
  for (int e = b0; e < b; ++e)
    if (__ldg(p.grp + e) == g) return false;
  return true;
}

__device__ __forceinline__ float apply_act(float v, int act) {
  if (act == ACT_RELU) return fmaxf(v, 0.0f);
  if (act == ACT_SILU) return silu_f(v);
  return v;
}

// Epilogue variants (compile-time): the hot combinations get straight-line code, everything else goes through the
// generic runtime path.  EPI_GENERIC reads act / out_mode from the kernel parameters.
enum Epi { EPI_BF16 = 0, EPI_BF16_RELU = 1, EPI_BF16_SILU = 2, EPI_F32 = 3, EPI_RESID = 4, EPI_GENERIC = 5, EPI_GLU = 6,
           EPI_LSE = 7, EPI_BF16_RELPOS = 8, EPI_BF16_GELU = 9 };

__host__ __device__ inline int select_epi(int act, int out_mode) {
  if (act == ACT_GLU) return EPI_GLU;
  if (out_mode == OUT_LSE) return EPI_LSE;
  if (act == ACT_GELU) return EPI_BF16_GELU;   // bf16 output only (checked at launch)
  if (out_mode == OUT_BF16) return act == ACT_NONE ? EPI_BF16 : act == ACT_RELU ? EPI_BF16_RELU : EPI_BF16_SILU;
  if (act == ACT_NONE) return out_mode == OUT_F32 ? EPI_F32 : EPI_RESID;
  return EPI_GENERIC;
}

__device__ __forceinline__ float fast_silu(float x) { return __fdividef(x, 1.0f + __expf(-x)); }

__device__ __forceinline__ float ex2_approx(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float rcp_approx(float x) {
  float y;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
// x * sigmoid(g) for two lanes at once with packed fp32 math (FMUL2 / FADD2 around the two MUFU pairs); x == g gives SiLU
__device__ __forceinline__ float2 gated2(float2 x, float2 g) {
  const float2 zero2 = make_float2(0.f, 0.f), one2 = make_float2(1.f, 1.f);
  const float2 t = ffma2(g, make_float2(-1.4426950408889634f, -1.4426950408889634f), zero2);
  const float2 e = make_float2(ex2_approx(t.x), ex2_approx(t.y));
  const float2 den = ffma2(e, one2, one2);
  return ffma2(x, make_float2(rcp_approx(den.x), rcp_approx(den.y)), zero2);
}

// One thread stores 32 consecutive output columns [n0, n0+32) of one output row (n0 % 32 == 0).
template <int EPI>
// n0: accumulator (bias) column; the output column is n0 - oshift (grouped output: the group's first column)
__device__ __forceinline__ void store_chunk(const GemmKParams& p, long long out_row, int n0, int oshift, const uint32_t* acc) {
  float v[32];
  const bool full = (n0 + 32 <= p.N);
  constexpr int OUT = (EPI <= EPI_BF16_SILU || EPI == EPI_BF16_GELU) ? OUT_BF16 : (EPI == EPI_F32) ? OUT_F32 : OUT_RESID_F32;
  const int out_mode = (EPI == EPI_GENERIC) ? p.out_mode : OUT;
  // bias (vectorised when the whole chunk is in range; bias + n0 is 16-byte aligned because n0 % 32 == 0)
  if (p.bias != nullptr) {
    if (full && ((reinterpret_cast<uintptr_t>(p.bias) & 15) == 0)) {
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float4 b4 = __ldg(reinterpret_cast<const float4*>(p.bias + n0) + j);
        v[4 * j + 0] = __uint_as_float(acc[4 * j + 0]) + b4.x;
        v[4 * j + 1] = __uint_as_float(acc[4 * j + 1]) + b4.y;
        v[4 * j + 2] = __uint_as_float(acc[4 * j + 2]) + b4.z;
        v[4 * j + 3] = __uint_as_float(acc[4 * j + 3]) + b4.w;
      }
    } else {
#pragma unroll
      for (int j = 0; j < 32; ++j) v[j] = __uint_as_float(acc[j]) + ((n0 + j < p.N) ? __ldg(p.bias + n0 + j) : 0.f);
    }
  } else {
#pragma unroll
    for (int j = 0; j < 32; ++j) v[j] = __uint_as_float(acc[j]);
  }
  if (EPI == EPI_BF16_RELU) {
#pragma unroll
    for (int j = 0; j < 32; ++j) v[j] = fmaxf(v[j], 0.f);
  } else if (EPI == EPI_BF16_SILU) {
#pragma unroll
    for (int j = 0; j < 32; ++j) v[j] = fast_silu(v[j]);
  } else if (EPI == EPI_BF16_GELU) {
#pragma unroll
    for (int j = 0; j < 32; ++j) v[j] = gelu_erf(v[j]);
  } else if (EPI == EPI_GENERIC) {
    if (p.act == ACT_RELU) {
#pragma unroll
      for (int j = 0; j < 32; ++j) v[j] = fmaxf(v[j], 0.f);
    } else if (p.act == ACT_SILU) {
#pragma unroll
      for (int j = 0; j < 32; ++j) v[j] = fast_silu(v[j]);
    }
  }
  if (out_mode == OUT_BF16) {
    bf16* o = reinterpret_cast<bf16*>(p.out) + out_row * p.ldo + n0 - oshift;
    if (full && ((reinterpret_cast<uintptr_t>(o) & 15) == 0)) {
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        uint4 u;
        u.x = pack_bf16x2(v[8 * j + 0], v[8 * j + 1]);
        u.y = pack_bf16x2(v[8 * j + 2], v[8 * j + 3]);
        u.z = pack_bf16x2(v[8 * j + 4], v[8 * j + 5]);
        u.w = pack_bf16x2(v[8 * j + 6], v[8 * j + 7]);
        reinterpret_cast<uint4*>(o)[j] = u;
      }
    } else {
      for (int j = 0; j < 32; ++j)
        if (n0 + j < p.N) o[j] = __float2bfloat16(v[j]);
    }
  } else if (out_mode == OUT_F32) {
    float* o = reinterpret_cast<float*>(p.out) + out_row * p.ldo + n0 - oshift;
    if (full && ((reinterpret_cast<uintptr_t>(o) & 15) == 0)) {
#pragma unroll
      for (int j = 0; j < 8; ++j)
        reinterpret_cast<float4*>(o)[j] = make_float4(v[4 * j], v[4 * j + 1], v[4 * j + 2], v[4 * j + 3]);
    } else {
      for (int j = 0; j < 32; ++j)
        if (n0 + j < p.N) o[j] = v[j];
    }
  } else {  // OUT_RESID_F32
    float* o = reinterpret_cast<float*>(p.out) + out_row * p.ldo + n0 - oshift;
    if (full && ((reinterpret_cast<uintptr_t>(o) & 15) == 0)) {
      float4 r[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) r[j] = reinterpret_cast<const float4*>(o)[j];
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        r[j].x += p.alpha * v[4 * j];
        r[j].y += p.alpha * v[4 * j + 1];
        r[j].z += p.alpha * v[4 * j + 2];
        r[j].w += p.alpha * v[4 * j + 3];
        reinterpret_cast<float4*>(o)[j] = r[j];
      }
    } else {
      for (int j = 0; j < 32; ++j)
        if (n0 + j < p.N) o[j] += p.alpha * v[j];
    }
  }
}

// ACT_GLU: one thread turns 32 "value" + 32 "gate" accumulator columns [n0, n0+64) of one row (interleaved weight
// rows, see kernels.h) into 32 bf16 outputs at column n0 / 2.  N %% 64 == 0 and 16-byte aligned rows are checked at launch.
__device__ __forceinline__ void store_glu(const GemmKParams& p, long long out_row, int n0, const uint32_t* av,
                                          const uint32_t* gv) {
  bf16* o = reinterpret_cast<bf16*>(p.out) + out_row * p.ldo + (n0 >> 1);
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    float v[8];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float4 ba = make_float4(0.f, 0.f, 0.f, 0.f), bg = ba;
      if (p.bias != nullptr) {
        ba = __ldg(reinterpret_cast<const float4*>(p.bias + n0) + 2 * j + h);
        bg = __ldg(reinterpret_cast<const float4*>(p.bias + n0 + 32) + 2 * j + h);
      }
      const int e = 8 * j + 4 * h;
      v[4 * h + 0] = __fdividef(__uint_as_float(av[e + 0]) + ba.x, 1.f + __expf(-(__uint_as_float(gv[e + 0]) + bg.x)));
      v[4 * h + 1] = __fdividef(__uint_as_float(av[e + 1]) + ba.y, 1.f + __expf(-(__uint_as_float(gv[e + 1]) + bg.y)));
      v[4 * h + 2] = __fdividef(__uint_as_float(av[e + 2]) + ba.z, 1.f + __expf(-(__uint_as_float(gv[e + 2]) + bg.z)));
      v[4 * h + 3] = __fdividef(__uint_as_float(av[e + 3]) + ba.w, 1.f + __expf(-(__uint_as_float(gv[e + 3]) + bg.w)));
    }
    uint4 u;
    u.x = pack_bf16x2(v[0], v[1]);
    u.y = pack_bf16x2(v[2], v[3]);
    u.z = pack_bf16x2(v[4], v[5]);
    u.w = pack_bf16x2(v[6], v[7]);
    reinterpret_cast<uint4*>(o)[j] = u;
  }
}

// Maps (tile, row-in-tile) to the output row; returns -1 when the row must not be written.
__device__ __forceinline__ long long output_row(const GemmKParams& p, const TileCoord& t, int r) {
  if (p.conv_mode) {
    int tp = t.row0 + r;
    if (tp >= p.conv_T2) return -1;
    return ((long long)t.b * p.conv_T2 + tp) * p.conv_orow_mul + t.f;
  }
  int m = t.row0 + r;
  if (m >= p.M) return -1;
  if (p.row_lens != nullptr) {
    int b = m / p.rows_per_batch;
    int pos = m - b * p.rows_per_batch;
    if (pos >= __ldg(p.row_lens + b)) return -1;
  }
  if (p.grp != nullptr && __ldg(p.grp + m / p.rows_per_batch) != t.g) return -1;   // another group's N block
  return m;
}

// The accumulator tile is copied from the wgmma fragments to shared memory as fp32 [BM][BN] with the 16-byte chunks of
// row r XOR-swizzled by r % 8: the fragment stores (8 rows x 32 bytes per instruction) and the row reads below (32 rows
// x 16 bytes) both spread over all banks.  One thread reads 32 consecutive columns [c, c+32) of its row (c % 32 == 0).
template <int BN>
__device__ __forceinline__ void acc_ld32(const float* accs, int row, int c, uint32_t* r) {
  const float* rp = accs + row * BN;
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    const float4 v = *reinterpret_cast<const float4*>(rp + ((((c >> 2) + k) ^ (row & 7)) << 2));
    r[4 * k + 0] = __float_as_uint(v.x);
    r[4 * k + 1] = __float_as_uint(v.y);
    r[4 * k + 2] = __float_as_uint(v.z);
    r[4 * k + 3] = __float_as_uint(v.w);
  }
}

// Drains columns [c0, c1) of the accumulator tile for the 32 output rows of one epilogue warp (one thread = one row,
// read from the tile's shared-memory copy, see acc_ld32).  The caller has synchronised the tile.
//
// fp32 outputs (EPI_F32, EPI_RESID) go through a warp-private 32x32 fp32 staging tile in shared memory (XOR-swizzled
// in 16-byte slots, conflict-free both ways) so that global accesses are coalesced: one warp instruction covers 4 rows
// x 128 contiguous bytes (4 L1 wavefronts) instead of 32 rows x 16 bytes (32 wavefronts) — the thread-per-row pattern
// made the LSU, not HBM, the limit of the residual GEMMs (out += alpha * (acc + bias) reads AND writes 128 B/row/chunk).
// The residual loads are software-pipelined: the first chunk's residual is requested BEFORE the wait on the
// accumulator barrier and chunk c+1's while chunk c is being converted.
// PAIR (compile time): bf16 outputs are written as the accurate mode's (hi, lo) pair, lo at column + p.out_split, and
// SiLU / GLU use exact exp / division — kept out of the throughput kernels (PAIR = false) so that their epilogue is the
// straight-line code it was before the accurate mode existed (a run-time flag adds work to every element).
template <int BN, int EPI, bool PAIR>
__device__ __forceinline__ void drain_tile(const GemmKParams& p, const TileCoord& t, int q, int lane, const float* accs,
                                           int c0, int c1, float* stage) {
  const int arow = q * 32 + lane;
  const long long orow = output_row(p, t, arow);
  const int n0_tile = t.n0;
  const int oshift = t.g * p.group_n;   // grouped output: columns of group g start at output column 0
  if (p.debug_skip_epi == 1) return;  // main-loop-only timing: wrong results by construction (2: everything but the stores)
  if constexpr (EPI == EPI_LSE) {
    // log-sum-exp partial of x = acc + bias over this thread's columns [c0, c1) of the tile (one 128-column slab when
    // 8 warps drain a 256-wide tile, two slabs with 4 warps) + the gather target if it falls inside
    const int g = (orow >= 0) ? __ldg(p.lse_gather + orow) : -1;
#pragma unroll 1
    for (int cs = c0; cs < c1; cs += 128) {
      float m = -INFINITY, ssum = 0.f;
#pragma unroll 1
      for (int c = cs; c < cs + 128 && c < c1; c += 32) {
        const int n0 = n0_tile + c;
        if (n0 >= p.N) break;
        uint32_t acc[32];
        acc_ld32<BN>(accs, arow, c, acc);
        float x[32];
        float cm = -INFINITY;
        if (n0 + 32 <= p.N && p.bias != nullptr && (reinterpret_cast<uintptr_t>(p.bias) & 15) == 0) {
          // full chunk: vector bias loads, packed adds
          const float2 one2 = make_float2(1.f, 1.f);
          float mx[4] = {-INFINITY, -INFINITY, -INFINITY, -INFINITY};
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            const float4 b4 = __ldg(reinterpret_cast<const float4*>(p.bias + n0) + j);
            const float2 lo = ffma2(make_float2(__uint_as_float(acc[4 * j]), __uint_as_float(acc[4 * j + 1])), one2,
                                    make_float2(b4.x, b4.y));
            const float2 hi = ffma2(make_float2(__uint_as_float(acc[4 * j + 2]), __uint_as_float(acc[4 * j + 3])), one2,
                                    make_float2(b4.z, b4.w));
            x[4 * j] = lo.x;
            x[4 * j + 1] = lo.y;
            x[4 * j + 2] = hi.x;
            x[4 * j + 3] = hi.y;
            mx[0] = fmaxf(mx[0], lo.x);
            mx[1] = fmaxf(mx[1], lo.y);
            mx[2] = fmaxf(mx[2], hi.x);
            mx[3] = fmaxf(mx[3], hi.y);
          }
          cm = fmaxf(fmaxf(mx[0], mx[1]), fmaxf(mx[2], mx[3]));
        } else {
#pragma unroll
          for (int j = 0; j < 32; ++j) {
            const bool in = n0 + j < p.N;
            x[j] = in ? __uint_as_float(acc[j]) + (p.bias ? __ldg(p.bias + n0 + j) : 0.f) : -INFINITY;
            cm = fmaxf(cm, x[j]);
          }
        }
        if (g >= n0 && g < n0 + 32) {
          float tg = 0.f;
#pragma unroll
          for (int j = 0; j < 32; ++j) tg = (g == n0 + j) ? x[j] : tg;
          p.lse_tgt[orow] = tg;
        }
        if (cm > m) {
          ssum *= ex2_approx((m - cm) * 1.4426950408889634f);  // exp2(-inf) = 0 on the first chunk
          m = cm;
        }
        // sum exp(x - m) = sum exp2(x * log2e - m * log2e): one packed FFMA2 + two ex2 + one packed add per pair
        const float2 l2 = make_float2(1.4426950408889634f, 1.4426950408889634f);
        const float2 nm = make_float2(-m * 1.4426950408889634f, -m * 1.4426950408889634f);
        float2 part01 = make_float2(0.f, 0.f), part23 = make_float2(0.f, 0.f);
#pragma unroll
        for (int j = 0; j < 32; j += 4) {
          const float2 t01 = ffma2(make_float2(x[j], x[j + 1]), l2, nm);
          const float2 t23 = ffma2(make_float2(x[j + 2], x[j + 3]), l2, nm);
          part01 = ffma2(make_float2(ex2_approx(t01.x), ex2_approx(t01.y)), make_float2(1.f, 1.f), part01);
          part23 = ffma2(make_float2(ex2_approx(t23.x), ex2_approx(t23.y)), make_float2(1.f, 1.f), part23);
        }
        ssum += (part01.x + part01.y) + (part23.x + part23.y);
      }
      if (orow >= 0 && n0_tile + cs < ((p.N + 255) / 256) * 256)
        p.lse_part[(size_t)orow * p.lse_nslab + ((n0_tile + cs) >> 7)] = make_float2(m, ssum);
    }
    // the last column tile also fills the slabs past the end of N (lse_slabs rounds up to 256 columns)
    if (orow >= 0 && c1 > c0 && n0_tile + c1 >= p.N)
      for (int sl = (n0_tile + c1) >> 7; sl < p.lse_nslab; ++sl)
        p.lse_part[(size_t)orow * p.lse_nslab + sl] = make_float2(-INFINITY, 0.f);
  } else if constexpr (EPI == EPI_GLU) {
    if (p.glu_coalesced && ((c1 - c0) & 127) == 0) {
      // 128 accumulator columns = 64 outputs = 128 bytes per row per round through the staging tile (as for bf16)
      const int slot = lane & 7, rsub = lane >> 3;
      long long ro[8];  // element offset of (row it*4+rsub, output column n0_tile/2 + slot*8), or -1
#pragma unroll
      for (int it = 0; it < 8; ++it) {
        const long long o = __shfl_sync(0xffffffffu, orow, it * 4 + rsub);
        ro[it] = (o >= 0) ? o * p.ldo + (n0_tile >> 1) + slot * 8 : -1;
      }
      bf16* out = reinterpret_cast<bf16*>(p.out);
      uint32_t* stage_u = reinterpret_cast<uint32_t*>(stage);
#pragma unroll 1
      for (int c = c0; c < c1; c += 128) {
        if (n0_tile + c >= p.N) break;
        // PAIR (bf16x3): the tile is written twice, first the hi halves, then the residues lo = v - hi
        constexpr int nparts = PAIR ? 2 : 1;
#pragma unroll 1
        for (int part = 0; part < nparts; ++part) {
#pragma unroll 1
        for (int hf = 0; hf < 2; ++hf) {  // two groups of 32 value + 32 gate columns -> 16-byte slots 4*hf .. 4*hf+3
          uint32_t av[32], gv[32];
          acc_ld32<BN>(accs, arow, c + 64 * hf, av);
          acc_ld32<BN>(accs, arow, c + 64 * hf + 32, gv);
          const int n0 = n0_tile + c + 64 * hf;
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            float v[8];
#pragma unroll
            for (int h2 = 0; h2 < 2; ++h2) {
              float4 ba = make_float4(0.f, 0.f, 0.f, 0.f), bg = ba;
              if (p.bias != nullptr) {
                ba = __ldg(reinterpret_cast<const float4*>(p.bias + n0) + 2 * j + h2);
                bg = __ldg(reinterpret_cast<const float4*>(p.bias + n0 + 32) + 2 * j + h2);
              }
              const int e = 8 * j + 4 * h2;
              const float2 one2 = make_float2(1.f, 1.f);
              const float2 a01 = ffma2(make_float2(__uint_as_float(av[e + 0]), __uint_as_float(av[e + 1])), one2, make_float2(ba.x, ba.y));
              const float2 a23 = ffma2(make_float2(__uint_as_float(av[e + 2]), __uint_as_float(av[e + 3])), one2, make_float2(ba.z, ba.w));
              const float2 g01 = ffma2(make_float2(__uint_as_float(gv[e + 0]), __uint_as_float(gv[e + 1])), one2, make_float2(bg.x, bg.y));
              const float2 g23 = ffma2(make_float2(__uint_as_float(gv[e + 2]), __uint_as_float(gv[e + 3])), one2, make_float2(bg.z, bg.w));
              float2 o01, o23;
              if constexpr (PAIR) {  // accurate mode: exact division / exp instead of the ex2 / rcp approximations
                o01 = make_float2(a01.x / (1.f + expf(-g01.x)), a01.y / (1.f + expf(-g01.y)));
                o23 = make_float2(a23.x / (1.f + expf(-g23.x)), a23.y / (1.f + expf(-g23.y)));
              } else {
                o01 = gated2(a01, g01);
                o23 = gated2(a23, g23);
              }
              v[4 * h2 + 0] = o01.x;
              v[4 * h2 + 1] = o01.y;
              v[4 * h2 + 2] = o23.x;
              v[4 * h2 + 3] = o23.y;
            }
            if (PAIR && part == 1) {
#pragma unroll
              for (int e = 0; e < 8; ++e) v[e] -= __bfloat162float(__float2bfloat16(v[e]));
            }
            const int sl = 4 * hf + j;
            *reinterpret_cast<uint4*>(stage_u + lane * 32 + ((sl ^ (lane & 7)) << 2)) =
                make_uint4(pack_bf16x2(v[0], v[1]), pack_bf16x2(v[2], v[3]), pack_bf16x2(v[4], v[5]),
                           pack_bf16x2(v[6], v[7]));
          }
        }
        __syncwarp();
#pragma unroll
        for (int it = 0; it < 8; ++it) {
          const int row = it * 4 + rsub;
          const uint4 u = *reinterpret_cast<const uint4*>(stage_u + row * 32 + ((slot ^ (row & 7)) << 2));
          if (ro[it] >= 0) *reinterpret_cast<uint4*>(out + ro[it] + (c >> 1) + (PAIR ? part * p.out_split : 0)) = u;
        }
        __syncwarp();
        }
      }
      return;
    }
#pragma unroll 1
    for (int c = c0; c < c1; c += 64) {
      if (n0_tile + c >= p.N) break;
      uint32_t av[32], gv[32];
      acc_ld32<BN>(accs, arow, c, av);
      acc_ld32<BN>(accs, arow, c + 32, gv);
      if (orow >= 0) store_glu(p, orow, n0_tile + c, av, gv);
    }
  } else if ((EPI == EPI_BF16 || EPI == EPI_BF16_RELU || EPI == EPI_BF16_SILU || EPI == EPI_BF16_RELPOS ||
              EPI == EPI_BF16_GELU) &&
             p.bf16_coalesced) {
    // bf16 outputs: 64 accumulator columns (= 128 bytes per row) per round through the warp's staging tile, so a
    // warp store covers 4 rows x 128 contiguous bytes instead of 32 rows x 16 bytes (8x fewer LSU wavefronts)
    const int slot = lane & 7, rsub = lane >> 3;
    long long ro[8];  // element offset of (row it*4+rsub, column n0_tile + slot*8), or -1
#pragma unroll
    for (int it = 0; it < 8; ++it) {
      const long long o = __shfl_sync(0xffffffffu, orow, it * 4 + rsub);
      ro[it] = (o >= 0) ? o * p.ldo + n0_tile - oshift + slot * 8 : -1;
    }
    bf16* out = reinterpret_cast<bf16*>(p.out);
    uint32_t* stage_u = reinterpret_cast<uint32_t*>(stage);
#pragma unroll 1
    for (int c = c0; c < c1; c += 64) {
      if (n0_tile + c >= p.N) break;
      if (n0_tile + c + 64 <= p.N) {
        uint32_t acc[64];
        acc_ld32<BN>(accs, arow, c, acc);
        acc_ld32<BN>(accs, arow, c + 32, acc + 32);
        const int n0 = n0_tile + c;
        // EPI_BF16_RELPOS: this 64-column chunk is one head of the KEY block -> K'' = k + pos[t], key bias u.k + vp
        bool kcols = false;
        int rp_t = 0, rp_hc = 0;
        float rp_part[8];   // u . k + v . pos over each 8-column slot, summed like relpos_prep_vec_kernel<8>
        if constexpr (EPI == EPI_BF16_RELPOS) {
          kcols = n0 >= p.rp_col0 && n0 < p.rp_col0 + p.rp_H * 64;
          rp_hc = n0 - p.rp_col0;
          rp_t = orow >= 0 ? (int)(orow % p.rp_T) : 0;
        }
        // PAIR (bf16x3): the tile is written twice, first hi = bf16(v), then the residue lo = bf16(v - hi)
        constexpr int nparts = PAIR ? 2 : 1;
#pragma unroll 1
        for (int part = 0; part < nparts; ++part) {
#pragma unroll
        for (int j = 0; j < 8; ++j) {  // 8 columns -> one 16-byte slot
          float v[8];
          const float2 one2 = make_float2(1.f, 1.f);
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            float4 b4 = make_float4(0.f, 0.f, 0.f, 0.f);
            if (p.bias != nullptr) b4 = __ldg(reinterpret_cast<const float4*>(p.bias + n0) + 2 * j + h);
            // bias add (and SiLU) on column pairs with packed fp32 instructions
            float2 lo = ffma2(make_float2(__uint_as_float(acc[8 * j + 4 * h + 0]), __uint_as_float(acc[8 * j + 4 * h + 1])),
                              one2, make_float2(b4.x, b4.y));
            float2 hi = ffma2(make_float2(__uint_as_float(acc[8 * j + 4 * h + 2]), __uint_as_float(acc[8 * j + 4 * h + 3])),
                              one2, make_float2(b4.z, b4.w));
            if (EPI == EPI_BF16_SILU) {
              if constexpr (PAIR) {  // accurate mode: exact exp / division
                lo = make_float2(lo.x / (1.f + expf(-lo.x)), lo.y / (1.f + expf(-lo.y)));
                hi = make_float2(hi.x / (1.f + expf(-hi.x)), hi.y / (1.f + expf(-hi.y)));
              } else {
                lo = gated2(lo, lo);
                hi = gated2(hi, hi);
              }
            }
            v[4 * h + 0] = lo.x;
            v[4 * h + 1] = lo.y;
            v[4 * h + 2] = hi.x;
            v[4 * h + 3] = hi.y;
          }
          if (EPI == EPI_BF16_RELU) {
#pragma unroll
            for (int e = 0; e < 8; ++e) v[e] = fmaxf(v[e], 0.f);
          }
          if (EPI == EPI_BF16_GELU) {
#pragma unroll
            for (int e = 0; e < 8; ++e) v[e] = gelu_erf(v[e]);
          }
          if constexpr (EPI == EPI_BF16_RELPOS) {
            if (kcols) {
              const uint4 pv = *reinterpret_cast<const uint4*>(p.rp_pos + (long long)rp_t * p.rp_ldp + rp_hc + 8 * j);
              const float4 u0 = __ldg(reinterpret_cast<const float4*>(p.rp_u + rp_hc + 8 * j));
              const float4 u1 = __ldg(reinterpret_cast<const float4*>(p.rp_u + rp_hc + 8 * j) + 1);
              const float uu[8] = {u0.x, u0.y, u0.z, u0.w, u1.x, u1.y, u1.z, u1.w};
              const float4 v0 = __ldg(reinterpret_cast<const float4*>(p.rp_v + rp_hc + 8 * j));
              const float4 v1 = __ldg(reinterpret_cast<const float4*>(p.rp_v + rp_hc + 8 * j) + 1);
              const float2 p0 = unpack_bf16x2(pv.x), p1 = unpack_bf16x2(pv.y), p2 = unpack_bf16x2(pv.z), p3 = unpack_bf16x2(pv.w);
              const float pp[8] = {p0.x, p0.y, p1.x, p1.y, p2.x, p2.y, p3.x, p3.y};
              float kq[8];
#pragma unroll
              for (int e = 0; e < 8; ++e) {
                kq[e] = __bfloat162float(__float2bfloat16(v[e]));   // the key as the projection would store it
                v[e] = kq[e] + pp[e];
              }
              // the same expression as the separate kernel, so that both paths give the same bias bit for bit
              rp_part[j] = uu[0] * kq[0] + uu[1] * kq[1] + uu[2] * kq[2] + uu[3] * kq[3] + uu[4] * kq[4] + uu[5] * kq[5] +
                           uu[6] * kq[6] + uu[7] * kq[7] + v0.x * pp[0] + v0.y * pp[1] + v0.z * pp[2] + v0.w * pp[3] +
                           v1.x * pp[4] + v1.y * pp[5] + v1.z * pp[6] + v1.w * pp[7];
            }
          }
          if (PAIR && part == 1) {
#pragma unroll
            for (int e = 0; e < 8; ++e) v[e] -= __bfloat162float(__float2bfloat16(v[e]));
          }
          if (p.debug_skip_epi == 3 && v[0] != 123.456f) continue;  // tuning aid: accumulator reads + math only
          *reinterpret_cast<uint4*>(stage_u + lane * 32 + ((j ^ (lane & 7)) << 2)) =
              make_uint4(pack_bf16x2(v[0], v[1]), pack_bf16x2(v[2], v[3]), pack_bf16x2(v[4], v[5]),
                         pack_bf16x2(v[6], v[7]));
        }
        if (p.debug_skip_epi == 3) continue;
        __syncwarp();
#pragma unroll
        for (int it = 0; it < 8; ++it) {
          const int row = it * 4 + rsub;
          const uint4 u = *reinterpret_cast<const uint4*>(stage_u + row * 32 + ((slot ^ (row & 7)) << 2));
          if (ro[it] >= 0 && p.debug_skip_epi != 2)
            *reinterpret_cast<uint4*>(out + ro[it] + c + (PAIR ? part * p.out_split : 0)) = u;
        }
        __syncwarp();
        }
        if constexpr (EPI == EPI_BF16_RELPOS) {
          if (kcols && orow >= 0) {
            const int hh = rp_hc >> 6;
            // the separate kernel's shuffle reduction over the head's 8 lanes (xor 4, 2, 1)
            p.rp_cb[((orow / p.rp_T) * p.rp_H + hh) * (long long)p.rp_T + rp_t] =
                ((rp_part[0] + rp_part[4]) + (rp_part[2] + rp_part[6])) + ((rp_part[1] + rp_part[5]) + (rp_part[3] + rp_part[7]));
          }
        }
      } else {
        for (int cc = c; cc < c + 64 && cc < c1; cc += 32) {
          if (n0_tile + cc >= p.N) break;
          uint32_t acc[32];
          acc_ld32<BN>(accs, arow, cc, acc);
          if (orow >= 0) store_chunk<EPI>(p, orow, n0_tile + cc, oshift, acc);
        }
      }
    }
  } else if ((EPI == EPI_RESID || EPI == EPI_F32) && p.f32_coalesced) {
    const int slot = lane & 7, rsub = lane >> 3;
    long long ro[8];  // element offset of (row it*4+rsub, column n0_tile + slot*4), or -1
#pragma unroll
    for (int it = 0; it < 8; ++it) {
      const long long o = __shfl_sync(0xffffffffu, orow, it * 4 + rsub);
      ro[it] = (o >= 0) ? o * p.ldo + n0_tile - oshift + slot * 4 : -1;
    }
    float* out = reinterpret_cast<float*>(p.out);
    float4 r[8];
    if (EPI == EPI_RESID && n0_tile + c0 + slot * 4 + 4 <= p.N) {
#pragma unroll
      for (int it = 0; it < 8; ++it)
        if (ro[it] >= 0) r[it] = *reinterpret_cast<const float4*>(out + ro[it] + c0);
    }
#pragma unroll 1
    for (int c = c0; c < c1; c += 32) {
      if (n0_tile + c >= p.N) break;
      uint32_t acc[32];
      acc_ld32<BN>(accs, arow, c, acc);
      const int n = n0_tile + c + slot * 4;       // first of this lane's 4 columns
      const bool vec = (n + 4 <= p.N);
      float4 rn[8];
      const bool pre_next = EPI == EPI_RESID && (c + 32 < c1) && (n + 32 + 4 <= p.N);
      if (pre_next) {
#pragma unroll
        for (int it = 0; it < 8; ++it)
          if (ro[it] >= 0) rn[it] = *reinterpret_cast<const float4*>(out + ro[it] + c + 32);
      }
      float4 b4 = make_float4(0.f, 0.f, 0.f, 0.f);
      if (p.bias != nullptr) {
        if (vec) {
          b4 = __ldg(reinterpret_cast<const float4*>(p.bias + n));
        } else {
          if (n + 0 < p.N) b4.x = __ldg(p.bias + n + 0);
          if (n + 1 < p.N) b4.y = __ldg(p.bias + n + 1);
          if (n + 2 < p.N) b4.z = __ldg(p.bias + n + 2);
        }
      }
#pragma unroll
      for (int j = 0; j < 8; ++j)
        *reinterpret_cast<uint4*>(stage + lane * 32 + ((j ^ (lane & 7)) << 2)) =
            make_uint4(acc[4 * j], acc[4 * j + 1], acc[4 * j + 2], acc[4 * j + 3]);
      __syncwarp();
#pragma unroll
      for (int it = 0; it < 8; ++it) {
        const int row = it * 4 + rsub;
        float4 v = *reinterpret_cast<const float4*>(stage + row * 32 + ((slot ^ (row & 7)) << 2));
        v.x += b4.x; v.y += b4.y; v.z += b4.z; v.w += b4.w;
        if (ro[it] < 0) continue;
        float* o = out + ro[it] + c;
        if (vec) {
          if (EPI == EPI_RESID) {
            r[it].x += p.alpha * v.x; r[it].y += p.alpha * v.y; r[it].z += p.alpha * v.z; r[it].w += p.alpha * v.w;
            *reinterpret_cast<float4*>(o) = r[it];
          } else {
            *reinterpret_cast<float4*>(o) = v;
          }
        } else {
          const float vv[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
          for (int k = 0; k < 3; ++k)
            if (n + k < p.N) o[k] = (EPI == EPI_RESID) ? o[k] + p.alpha * vv[k] : vv[k];
        }
      }
      __syncwarp();
      if (pre_next) {
#pragma unroll
        for (int it = 0; it < 8; ++it) r[it] = rn[it];
      }
    }
  } else {
#pragma unroll 1
    for (int c = c0; c < c1; c += 32) {
      if (n0_tile + c >= p.N) break;
      uint32_t acc[32];
      acc_ld32<BN>(accs, arow, c, acc);
      if (orow >= 0) store_chunk<EPI>(p, orow, n0_tile + c, oshift, acc);
    }
  }
}

// warpgroup 0: TMA producer (one thread), warpgroups 1-2: consumers, each owning whole 128 x BN tiles in turn
constexpr int kConsumerWGs = 2;
constexpr int kGemmThreads = 128 * (1 + kConsumerWGs);
// setmaxnreg budgets: 40 * 128 + 232 * 256 = 64 512 of the SM's 65 536 registers
constexpr int kProducerRegs = 40;
constexpr int kConsumerRegs = 232;

template <int BN>
struct GemmCfg {
  static constexpr int BM = 128;
  static constexpr int BK = 64;
  // 4 stages + the whole 64 KB accumulator tile.  A 5th stage fits only with the tile copied and drained one 64-row half
  // at a time; measured on the H100 that is slower (DESIGN.md §4): the drain loses half its parallelism and the second
  // half's accumulators stay live (and spill) through the first half's drain.
  static constexpr int STAGES = 4;
  static constexpr uint32_t A_BYTES = BM * BK * 2;
  static constexpr uint32_t B_BYTES = BN * BK * 2;
  static constexpr uint32_t STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr uint32_t ACC_BYTES = BM * BN * 4;   // fp32 accumulator tile (epilogue copy), shared by both consumers
  static constexpr uint32_t SMEM_BYTES = STAGES * STAGE_BYTES + ACC_BYTES + 4 * 4096 /*epilogue staging, 4 warps*/ +
                                         256 /*barriers*/ + 1024 /*align slack*/;
};

// Persistent, warp-specialised TMA + wgmma GEMM (1 CTA / SM, grid = min(#tiles, #SMs), static round-robin tiles of
// 128 x BN), with ping-pong consumer warpgroups.  The producer fills a STAGES-deep ring of {A 128x64, W BNx64} bf16
// tiles (SWIZZLE_128B) in the CTA's tile order.  The CTA's i-th tile belongs to consumer warpgroup i % 2, which
// multiplies the whole tile (2 x wgmma m64nBNk16 per k16 step, rows 0-63 and 64-127), releasing each stage as soon as
// its MMAs have retired, then copies its accumulator to the shared fp32 tile and drains it through the fused epilogue
// (drain_tile) while the other warpgroup already runs the next tile's MMAs.  Two pairs of mbarriers order the hand-offs:
//   turn[w]    : warpgroup w may start its K loop — the other one has issued the last MMA of the previous tile;
//   accfree[w] : warpgroup w may write the shared accumulator tile — the other one has drained the previous tile.
// Both are arrived by all 128 threads of the other warpgroup once per tile, so the CTA's tile i (i >= 1) waits for
// completion (i + 1) / 2 of its barrier, parity ((i - 1) / 2) & 1; tile 0 waits for nothing.  Because a warpgroup
// arrives only after it has itself waited for the previous completion, a barrier is never more than one phase ahead
// of its waiter.  Arrivals no tile waits for (the CTA's last tile, a warpgroup without tiles) are harmless.
template <int BN, int EPI, bool PAIR>
__global__ void __launch_bounds__(kGemmThreads, 1)
gemm_wg_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const GemmKParams p) {
  using Cfg = GemmCfg<BN>;
  constexpr int STAGES = Cfg::STAGES;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sA = smem;
  uint8_t* sB = smem + STAGES * Cfg::A_BYTES;
  float* accs = reinterpret_cast<float*>(smem + STAGES * Cfg::STAGE_BYTES);
  float* stage_epi = accs + Cfg::BM * BN;
  uint64_t* bars = reinterpret_cast<uint64_t*>(stage_epi + 4 * 1024);
  uint64_t* full = bars;
  uint64_t* empty = bars + STAGES;
  uint64_t* turn = bars + 2 * STAGES;
  uint64_t* accfree = turn + 2;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    for (int i = 0; i < STAGES; ++i) {
      mbar_init(&full[i], 1);
      mbar_init(&empty[i], 4);   // lane 0 of every warp of the consuming warpgroup
    }
    for (int w = 0; w < kConsumerWGs; ++w) {
      mbar_init(&turn[w], 128);
      mbar_init(&accfree[w], 128);
    }
    fence_barrier_init();
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
  }
  __syncthreads();
  const int nkb = p.num_k_blocks;

  if (warp < 4) {
    // ------------------------------------------------------------ TMA producer
    setmaxnreg_dec<kProducerRegs>();
    if (warp == 0 && lane == 0) {
      uint32_t stage = 0, phase = 0;
      for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
        if (!tile_active(p, tile, BN)) continue;
        TileCoord t = decode_tile(p, tile, BN);
        for (int kbx = 0; kbx < nkb; ++kbx) {
          // bf16x3: pass 0 = A_hi W_hi, pass 1 = A_lo W_hi, pass 2 = A_hi W_lo
          const int seg = p.x3 ? kbx / p.kb_seg : 0;
          const int kb = kbx - seg * p.kb_seg;
          const int a_ofs = (seg == 1) ? p.a_lo_ofs : 0, w_ofs = (seg == 2) ? p.w_lo_ofs : 0;
          mbar_wait(&empty[stage], phase ^ 1);
          mbar_expect_tx(&full[stage], Cfg::STAGE_BYTES);
          if (p.conv_mode) {
            int tap = kb / p.conv_cblocks;
            int cb = kb - tap * p.conv_cblocks;
            int kh = tap / 3, kw = tap - kh * 3;
            tma_load_4d(sA + stage * Cfg::A_BYTES, &tmA, &full[stage], cb * 64 + a_ofs, 2 * t.f + kw, t.row0 + (kh >> 1),
                        t.b * 2 + (kh & 1));
          } else {
            tma_load_4d(sA + stage * Cfg::A_BYTES, &tmA, &full[stage], kb * 64 + a_ofs, t.row0, 0, 0);
          }
          tma_load_2d(sB + stage * Cfg::B_BYTES, &tmB, &full[stage], kb * 64 + w_ofs, t.n0);
          if (++stage == STAGES) {
            stage = 0;
            phase ^= 1;
          }
        }
      }
    }
  } else {
    // ------------------------------------------------------------ consumer warpgroups
    setmaxnreg_inc<kConsumerRegs>();
    const int wg = (warp >> 2) - 1, wl = warp & 3;
    // one warpgroup drains at a time: warp wl takes rows [32 wl, 32 wl + 32) and all columns
    float* stage_w = stage_epi + wl * 1024;
    float acc[BN];   // rows 0-63 in acc[0, BN/2), rows 64-127 in acc[BN/2, BN) (wgmma fragment layout, common.cuh)
    // i counts the CTA's active tiles (tile_active), the producer's ring order; tile i belongs to warpgroup i % 2
    int active = 0;
    for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
      if (!tile_active(p, tile, BN)) continue;
      const int i = active++;
      if (i % kConsumerWGs != wg) continue;
      TileCoord t = decode_tile(p, tile, BN);
      // the ring is consumed in the CTA's tile order: tile i's k-blocks are ring uses [i * nkb, (i + 1) * nkb)
      const uint32_t u0 = (uint32_t)i * (uint32_t)nkb;
      uint32_t stage = u0 % STAGES, phase = (u0 / STAGES) & 1;
      const uint32_t hand_parity = ((i - 1) >> 1) & 1;   // see the comment above the kernel
#pragma unroll
      for (int e = 0; e < BN; ++e) acc[e] = 0.f;
      if (i > 0) mbar_wait(&turn[wg], hand_parity);
      int prev = -1;
      for (int kb = 0; kb < nkb; ++kb) {
        mbar_wait(&full[stage], phase);
        const uint64_t adesc = make_sw128_desc(smem_u32(sA + stage * Cfg::A_BYTES));
        const uint64_t bdesc = make_sw128_desc(smem_u32(sB + stage * Cfg::B_BYTES));
        constexpr uint64_t kHalfA = (Cfg::A_BYTES / 2) >> 4;   // rows 64-127 of the A stage, in descriptor units
        wgmma_fence_regs<BN>(acc);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          // advance 16 bf16 = 32 B along K inside the 128 B swizzle span: +2 in the (addr >> 4) field
          if constexpr (BN == 128) {
            wgmma_m64n128k16_ss(acc, adesc + 2 * k, bdesc + 2 * k, 1u);
            wgmma_m64n128k16_ss(acc + BN / 2, adesc + kHalfA + 2 * k, bdesc + 2 * k, 1u);
          } else {
            wgmma_m64n64k16_ss(acc, adesc + 2 * k, bdesc + 2 * k, 1u);
            wgmma_m64n64k16_ss(acc + BN / 2, adesc + kHalfA + 2 * k, bdesc + 2 * k, 1u);
          }
        }
        wgmma_commit();
        wgmma_wait<1>();   // the previous stage's MMAs have retired: hand its buffers back to the producer
        wgmma_fence_regs<BN>(acc);
        if (prev >= 0 && lane == 0) mbar_arrive(&empty[prev]);
        prev = (int)stage;
        if (++stage == STAGES) {
          stage = 0;
          phase ^= 1;
        }
      }
      mbar_arrive(&turn[wg ^ 1]);   // every MMA of this tile is issued: the other warpgroup's K loop may follow
      wgmma_wait<0>();
      wgmma_fence_regs<BN>(acc);
      if (prev >= 0 && lane == 0) mbar_arrive(&empty[prev]);
      // accumulator -> shared memory, once the other warpgroup has drained the previous tile out of it
      if (i > 0) mbar_wait(&accfree[wg], hand_parity);
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int r0 = h * 64 + wl * 16 + (lane >> 2);
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
          const int c = 8 * j + 2 * (lane & 3);
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int r = r0 + 8 * e;
            *reinterpret_cast<float2*>(accs + r * BN + ((((c >> 2)) ^ (r & 7)) << 2) + (c & 3)) =
                make_float2(acc[h * (BN / 2) + 4 * j + 2 * e], acc[h * (BN / 2) + 4 * j + 2 * e + 1]);
          }
        }
      }
      asm volatile("bar.sync %0, 128;" ::"r"(1 + wg) : "memory");
      drain_tile<BN, EPI, PAIR>(p, t, wl, lane, accs, 0, BN, stage_w);
      mbar_arrive(&accfree[wg ^ 1]);   // this thread's reads of the tile and of its staging slot are done
    }
  }
}

// 128 x 256 tiles for the wide bf16-output GEMMs (FFN1, the conv2 implicit GEMM, ...).  3 stages of 48 KB + the 64 KB
// bf16 output tile = 208 KB; a 4th stage does not fit beside the output tile.
struct WideCfg {
  static constexpr int BM = 128;
  static constexpr int BN = 256;
  static constexpr int BK = 64;
  static constexpr int STAGES = 3;
  static constexpr uint32_t A_BYTES = BM * BK * 2;
  static constexpr uint32_t B_BYTES = BN * BK * 2;
  static constexpr uint32_t STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr uint32_t OUT_BYTES = BM * BN * 2;
  static constexpr uint32_t SMEM_BYTES = STAGES * STAGE_BYTES + OUT_BYTES + 256 /*barriers*/ + 1024 /*align slack*/;
};

// Persistent TMA + wgmma GEMM on 128 x 256 tiles for the bf16-output epilogues without cross-column work (bias, ReLU,
// SiLU; EPI_BF16 / EPI_BF16_RELU / EPI_BF16_SILU, plain or conv_mode, no hi/lo pair).  Per k-block the SM pulls one
// 256-wide weight tile that both consumer warpgroups read: 48 KB per 4.2 MFLOP instead of 32 KB per 2.1 MFLOP.
//   warpgroup 0, warp 0 : TMA producer (one thread) — a 3-deep ring of {A 128x64, W 256x64} bf16 tiles (SWIZZLE_128B)
//   warpgroup 0, warps 1-3 : copy the bf16 output tile from shared memory to global memory (16-byte stores, one
//                    512-byte row per warp instruction) under the next tile's main loop
//   warpgroups 1-2 : consumers of the same tile, rows 0-63 and 64-127: wgmma m64n256k16 x 4 per k-block (the k order of
//                    gemm_wg_kernel), each stage released once all 8 consumer warps have retired their MMAs.  Then bias
//                    and activation in registers, with gemm_wg_kernel's arithmetic, into the bf16 output tile.
// One mbarrier pair guards the output tile:
//   ofull : arrived by the 256 consumer threads once tile i is written — the copy warps may read it;
//   ofree : arrived by the 96 copy threads once tile i is stored — the consumers may write tile i + 1.
// Each completes once per tile, so the CTA's tile i waits for completion i + 1 of ofull (parity i & 1), and tile i
// (i >= 1) waits for completion i of ofree (parity (i - 1) & 1); tile 0 writes without waiting.  A barrier is never
// more than one phase ahead of its waiter: ofull's next arrivals need ofree's previous completion and vice versa.
// RVB_GEMM_SKIP_EPI=1 skips the epilogue (main loop only), 2 the global stores; the barrier hand-offs stay.
template <int EPI>
__global__ void __launch_bounds__(kGemmThreads, 1)
gemm_wide_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const GemmKParams p) {
  using Cfg = WideCfg;
  constexpr int STAGES = Cfg::STAGES;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sA = smem;
  uint8_t* sB = smem + STAGES * Cfg::A_BYTES;
  uint8_t* sOut = smem + STAGES * Cfg::STAGE_BYTES;   // bf16 [128][256], 16-byte chunk c of row r at c ^ (r % 8)
  uint64_t* bars = reinterpret_cast<uint64_t*>(sOut + Cfg::OUT_BYTES);
  uint64_t* full = bars;
  uint64_t* empty = bars + STAGES;
  uint64_t* ofull = bars + 2 * STAGES;
  uint64_t* ofree = ofull + 1;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    for (int i = 0; i < STAGES; ++i) {
      mbar_init(&full[i], 1);
      mbar_init(&empty[i], 8);   // lane 0 of every consumer warp
    }
    mbar_init(ofull, 256);
    mbar_init(ofree, 96);
    fence_barrier_init();
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
  }
  __syncthreads();
  const int nkb = p.num_k_blocks;

  if (warp < 4) {
    setmaxnreg_dec<kProducerRegs>();
    if (warp == 0) {
      // ---------------------------------------------------------- TMA producer
      if (lane == 0) {
        uint32_t stage = 0, phase = 0;
        for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
          const TileCoord t = decode_tile(p, tile, Cfg::BN);
          for (int kb = 0; kb < nkb; ++kb) {
            mbar_wait(&empty[stage], phase ^ 1);
            mbar_expect_tx(&full[stage], Cfg::STAGE_BYTES);
            if (p.conv_mode) {
              const int tap = kb / p.conv_cblocks;
              const int cb = kb - tap * p.conv_cblocks;
              const int kh = tap / 3, kw = tap - kh * 3;
              tma_load_4d(sA + stage * Cfg::A_BYTES, &tmA, &full[stage], cb * 64, 2 * t.f + kw, t.row0 + (kh >> 1),
                          t.b * 2 + (kh & 1));
            } else {
              tma_load_4d(sA + stage * Cfg::A_BYTES, &tmA, &full[stage], kb * 64, t.row0, 0, 0);
            }
            tma_load_2d(sB + stage * Cfg::B_BYTES, &tmB, &full[stage], kb * 64, t.n0);
            if (++stage == STAGES) {
              stage = 0;
              phase ^= 1;
            }
          }
        }
      }
    } else {
      // ---------------------------------------------------------- output tile -> global memory (warps 1-3)
      const int cw = warp - 1;
      const bool store = p.debug_skip_epi == 0;
      bf16* out = reinterpret_cast<bf16*>(p.out);
      int i = 0;
      for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x, ++i) {
        const TileCoord t = decode_tile(p, tile, Cfg::BN);
        mbar_wait(ofull, i & 1);
        if (store) {
#pragma unroll 4
          for (int r = cw; r < Cfg::BM; r += 3) {
            const long long orow = output_row(p, t, r);
            const uint4 u = *reinterpret_cast<const uint4*>(sOut + r * (Cfg::BN * 2) + ((lane ^ (r & 7)) << 4));
            if (orow >= 0) *reinterpret_cast<uint4*>(out + orow * p.ldo + t.n0 + lane * 8) = u;
          }
        }
        mbar_arrive(ofree);
      }
    }
  } else {
    // ------------------------------------------------------------ consumer warpgroups
    setmaxnreg_inc<kConsumerRegs>();
    const int wg = (warp >> 2) - 1, wl = warp & 3;
    float acc[Cfg::BN / 2];   // rows 64 wg + [0, 64) of the tile (wgmma fragment layout, common.cuh)
    uint32_t stage = 0, phase = 0;
    int i = 0;
    for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x, ++i) {
      const TileCoord t = decode_tile(p, tile, Cfg::BN);
#pragma unroll
      for (int e = 0; e < Cfg::BN / 2; ++e) acc[e] = 0.f;
      int prev = -1;
      for (int kb = 0; kb < nkb; ++kb) {
        mbar_wait(&full[stage], phase);
        constexpr uint64_t kHalfA = (Cfg::A_BYTES / 2) >> 4;   // rows 64-127 of the A stage, in descriptor units
        const uint64_t adesc = make_sw128_desc(smem_u32(sA + stage * Cfg::A_BYTES)) + wg * kHalfA;
        const uint64_t bdesc = make_sw128_desc(smem_u32(sB + stage * Cfg::B_BYTES));
        wgmma_fence_regs<Cfg::BN / 2>(acc);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < 4; ++k) wgmma_m64n256k16_ss(acc, adesc + 2 * k, bdesc + 2 * k, 1u);
        wgmma_commit();
        wgmma_wait<1>();   // the previous stage's MMAs have retired: release it
        wgmma_fence_regs<Cfg::BN / 2>(acc);
        if (prev >= 0 && lane == 0) mbar_arrive(&empty[prev]);
        prev = (int)stage;
        if (++stage == STAGES) {
          stage = 0;
          phase ^= 1;
        }
      }
      wgmma_wait<0>();
      wgmma_fence_regs<Cfg::BN / 2>(acc);
      if (lane == 0) mbar_arrive(&empty[prev]);
      if (i > 0) mbar_wait(ofree, (i - 1) & 1);
      if (p.debug_skip_epi != 1) {
        // thread (wl, lane) holds rows r0 and r0 + 8, columns 8 j + 2 (lane % 4) + {0, 1}; the 4 lanes of a row fill
        // one 16-byte chunk, and the 8 rows of a warp store land in 8 distinct chunk slots (conflict-free)
        const int r0 = wg * 64 + wl * 16 + (lane >> 2);
        uint32_t* so = reinterpret_cast<uint32_t*>(sOut) + r0 * (Cfg::BN / 2) + (lane & 3);
        const float2 one2 = make_float2(1.f, 1.f);
#pragma unroll
        for (int j = 0; j < Cfg::BN / 8; ++j) {
          float2 b = make_float2(0.f, 0.f);
          if (p.bias != nullptr) b = __ldg(reinterpret_cast<const float2*>(p.bias + t.n0 + 8 * j + 2 * (lane & 3)));
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            float2 v = ffma2(make_float2(acc[4 * j + 2 * e], acc[4 * j + 2 * e + 1]), one2, b);
            if (EPI == EPI_BF16_SILU) v = gated2(v, v);
            if (EPI == EPI_BF16_RELU) v = make_float2(fmaxf(v.x, 0.f), fmaxf(v.y, 0.f));
            so[8 * e * (Cfg::BN / 2) + ((j ^ (lane >> 2)) << 2)] = pack_bf16x2(v.x, v.y);
          }
        }
      }
      mbar_arrive(ofull);
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------
// Debug / bring-up kernel: same contract on plain CUDA cores (RVB_GEMM=simt).  Never used by the benchmarks.
__device__ __forceinline__ float load_a_elem(const GemmKParams& p, const TileCoord& t, int r, int k) {
  if (k >= p.K) return 0.0f;
  if (p.conv_mode) {
    int tp = t.row0 + r;
    if (tp >= p.conv_T2) return 0.0f;
    int tap = k / p.conv_C;
    int c = k - tap * p.conv_C;
    int kh = tap / 3, kw = tap - kh * 3;
    long long idx = (((long long)(t.b * 2 + (kh & 1)) * p.conv_T1h + (tp + (kh >> 1))) * p.conv_F1 + (2 * t.f + kw)) *
                        p.conv_C + c;
    return __bfloat162float(p.A[idx]);
  }
  int m = t.row0 + r;
  if (m >= p.M) return 0.0f;
  return __bfloat162float(p.A[(long long)m * p.lda + k]);
}

__global__ void __launch_bounds__(256) gemm_simt_kernel(const GemmKParams p) {
  // tile: 128 rows x 32 cols, 256 threads, each thread 4 rows x 4 cols.  ACT_GLU: tiles run over the N/2 OUTPUT
  // columns; output column oc pairs weight rows 2*(oc & ~31) + (oc & 31) (value) and that + 32 (gate).
  __shared__ float sA[128][17];
  __shared__ float sW[32][17];
  __shared__ float sG[32][17];
  const bool glu = (p.act == ACT_GLU);
  for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
    // here tiles_n counts 32-wide column tiles
    TileCoord t = decode_tile(p, tile, 32);
    const int tx = threadIdx.x & 7, ty = threadIdx.x >> 3;
    const int wrow0 = glu ? 2 * t.n0 : t.n0;
    float acc[4][4], accg[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) acc[i][j] = accg[i][j] = 0.f;
    for (int k0 = 0; k0 < p.K; k0 += 16) {
      for (int e = threadIdx.x; e < 128 * 16; e += 256) {
        int r = e >> 4, kk = e & 15;
        sA[r][kk] = load_a_elem(p, t, r, k0 + kk);
      }
      for (int e = threadIdx.x; e < 32 * 16; e += 256) {
        int n = e >> 4, kk = e & 15;
        int gn = wrow0 + n, gk = k0 + kk;
        sW[n][kk] = (gn < p.N && gk < p.K) ? __bfloat162float(p.W[(long long)gn * p.ldw + gk]) : 0.f;
        sG[n][kk] = (glu && gn + 32 < p.N && gk < p.K) ? __bfloat162float(p.W[(long long)(gn + 32) * p.ldw + gk]) : 0.f;
      }
      __syncthreads();
#pragma unroll
      for (int kk = 0; kk < 16; ++kk) {
        float a[4], w[4], g[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) a[i] = sA[ty * 4 + i][kk];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          w[j] = sW[tx * 4 + j][kk];
          g[j] = sG[tx * 4 + j][kk];
        }
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            acc[i][j] = fmaf(a[i], w[j], acc[i][j]);
            accg[i][j] = fmaf(a[i], g[j], accg[i][j]);
          }
      }
      __syncthreads();
    }
    for (int i = 0; i < 4; ++i) {
      long long orow = output_row(p, t, ty * 4 + i);
      if (orow < 0) continue;
      for (int j = 0; j < 4; ++j) {
        int n = t.n0 + tx * 4 + j;
        if (glu) {
          if (2 * n >= p.N) continue;
          const int wr = wrow0 + tx * 4 + j;
          float va = acc[i][j], vg = accg[i][j];
          if (p.bias) {
            va += p.bias[wr];
            vg += p.bias[wr + 32];
          }
          reinterpret_cast<bf16*>(p.out)[orow * p.ldo + n] = __float2bfloat16(va / (1.f + expf(-vg)));
          continue;
        }
        if (n >= p.N) continue;
        float x = acc[i][j];
        if (p.bias) x += p.bias[n];
        x = apply_act(x, p.act);
        if (p.out_mode == OUT_BF16)
          reinterpret_cast<bf16*>(p.out)[orow * p.ldo + n] = __float2bfloat16(x);
        else if (p.out_mode == OUT_F32)
          reinterpret_cast<float*>(p.out)[orow * p.ldo + n] = x;
        else
          reinterpret_cast<float*>(p.out)[orow * p.ldo + n] += p.alpha * x;
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFn g_encode = nullptr;

static int get_encode_fn() {
  if (g_encode) return 0;
  void* fn = nullptr;
  cudaDriverEntryPointQueryResult qres;
  RVB_CHECK_CUDA(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres));
  RVB_REQUIRE(fn != nullptr && qres == cudaDriverEntryPointSuccess, "cuTensorMapEncodeTiled not available");
  g_encode = reinterpret_cast<EncodeTiledFn>(fn);
  return 0;
}

static int make_tmap(CUtensorMap* m, const void* base, int rank, const cuuint64_t* dims, const cuuint64_t* strides_bytes,
                     const cuuint32_t* box) {
  cuuint32_t estr[5] = {1, 1, 1, 1, 1};
  CUresult r = g_encode(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, rank, const_cast<void*>(base), dims, strides_bytes, box,
                        estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                        CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  RVB_REQUIRE(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled failed with %d (rank %d dims %llu %llu)", (int)r, rank,
              (unsigned long long)dims[0], (unsigned long long)dims[1]);
  return 0;
}

static int g_num_sms = 0;

// ---- optional per-launch timing (bench.py's live roofline): CUDA events on the launching stream
struct GemmProfRec {
  cudaEvent_t a, b;
  double flops;
};
static bool g_prof_on = false;
static std::vector<GemmProfRec> g_prof;
static std::mutex g_prof_mutex;
// Events are pooled per device and reused across profiling windows: creating two per launch inside the timed region
// would cost host time exactly where the step is host-sensitive.
constexpr int kProfMaxDev = 64;
static std::vector<cudaEvent_t> g_prof_pool[kProfMaxDev];
static size_t g_prof_pool_used[kProfMaxDev];

static int prof_event(cudaEvent_t* out) {
  int dev = 0;
  RVB_CHECK_CUDA(cudaGetDevice(&dev));
  RVB_REQUIRE(dev >= 0 && dev < kProfMaxDev, "gemm profile: device index %d out of range", dev);
  std::lock_guard<std::mutex> lock(g_prof_mutex);
  auto& pool = g_prof_pool[dev];
  if (g_prof_pool_used[dev] == pool.size()) {
    cudaEvent_t e;
    RVB_CHECK_CUDA(cudaEventCreate(&e));
    pool.push_back(e);
  }
  *out = pool[g_prof_pool_used[dev]++];
  return 0;
}

void gemm_profile_begin() {
  std::lock_guard<std::mutex> lock(g_prof_mutex);
  g_prof.clear();
  for (int d = 0; d < kProfMaxDev; ++d) g_prof_pool_used[d] = 0;
  g_prof_on = true;
}
int gemm_profile_end(double* total_ms, double* total_flops, long long* launches) {
  g_prof_on = false;
  double ms = 0.0, fl = 0.0;
  for (auto& r : g_prof) {
    float t = 0.f;
    RVB_CHECK_CUDA(cudaEventSynchronize(r.b));
    RVB_CHECK_CUDA(cudaEventElapsedTime(&t, r.a, r.b));
    ms += t;
    fl += r.flops;
  }
  if (total_ms) *total_ms = ms;
  if (total_flops) *total_flops = fl;
  if (launches) *launches = (long long)g_prof.size();
  g_prof.clear();
  return 0;
}

// BN = 256: gemm_wide_kernel (launch_gemm has checked that the epilogue is one it covers)
template <int BN>
static int launch_wg(const GemmArgs& a, GemmKParams& p, cudaStream_t stream) {
  constexpr uint32_t SMEM_BYTES = BN == 256 ? WideCfg::SMEM_BYTES : GemmCfg<BN>::SMEM_BYTES;
  CUtensorMap tmA, tmB;
  const int kmul = a.x3 ? 2 : 1;
  const long long lda = a.lda ? a.lda : (long long)a.K * kmul, ldw = a.ldw ? a.ldw : (long long)a.K * kmul;
  if (a.conv_mode) {
    const cuuint64_t Cp = (cuuint64_t)a.conv_C * (a.x3 ? 2 : 1);  // physical channels: [hi C | lo C] in bf16x3 mode
    cuuint64_t dims[4] = {Cp, (cuuint64_t)a.conv_F1, (cuuint64_t)a.conv_T1h, (cuuint64_t)(2 * a.conv_B)};
    cuuint64_t str[3] = {Cp * 2, (cuuint64_t)a.conv_F1 * Cp * 2, (cuuint64_t)a.conv_T1h * a.conv_F1 * Cp * 2};
    cuuint32_t box[4] = {64, 1, 128, 1};
    if (make_tmap(&tmA, a.A, 4, dims, str, box)) return -1;
  } else {
    cuuint64_t dims[4] = {(cuuint64_t)a.K * (a.x3 ? 2 : 1), (cuuint64_t)a.M, 1, 1};
    cuuint64_t str[3] = {(cuuint64_t)lda * 2, (cuuint64_t)lda * 2 * a.M, (cuuint64_t)lda * 2 * a.M};
    cuuint32_t box[4] = {64, 128, 1, 1};
    if (make_tmap(&tmA, a.A, 4, dims, str, box)) return -1;
  }
  {
    cuuint64_t dims[2] = {(cuuint64_t)a.K * (a.x3 ? 2 : 1), (cuuint64_t)a.N};
    cuuint64_t str[1] = {(cuuint64_t)ldw * 2};
    cuuint32_t box[2] = {64, (cuuint32_t)BN};
    if (make_tmap(&tmB, a.W, 2, dims, str, box)) return -1;
  }
  void (*kern)(const CUtensorMap, const CUtensorMap, const GemmKParams) = nullptr;
  if constexpr (BN == 256) {
    switch (select_epi(a.act, a.out_mode)) {
      case EPI_BF16: kern = gemm_wide_kernel<EPI_BF16>; break;
      case EPI_BF16_RELU: kern = gemm_wide_kernel<EPI_BF16_RELU>; break;
      default: kern = gemm_wide_kernel<EPI_BF16_SILU>; break;
    }
  } else {
    const bool pair = a.out_split > 0;
    switch (a.rp_pos ? (int)EPI_BF16_RELPOS : select_epi(a.act, a.out_mode)) {
      case EPI_BF16: kern = pair ? gemm_wg_kernel<BN, EPI_BF16, true> : gemm_wg_kernel<BN, EPI_BF16, false>; break;
      case EPI_BF16_RELU: kern = pair ? gemm_wg_kernel<BN, EPI_BF16_RELU, true> : gemm_wg_kernel<BN, EPI_BF16_RELU, false>; break;
      case EPI_BF16_SILU: kern = pair ? gemm_wg_kernel<BN, EPI_BF16_SILU, true> : gemm_wg_kernel<BN, EPI_BF16_SILU, false>; break;
      case EPI_F32: kern = gemm_wg_kernel<BN, EPI_F32, false>; break;
      case EPI_RESID: kern = gemm_wg_kernel<BN, EPI_RESID, false>; break;
      case EPI_GLU: kern = pair ? gemm_wg_kernel<BN, EPI_GLU, true> : gemm_wg_kernel<BN, EPI_GLU, false>; break;
      case EPI_LSE: kern = gemm_wg_kernel<BN, EPI_LSE, false>; break;
      case EPI_BF16_RELPOS: kern = gemm_wg_kernel<BN, EPI_BF16_RELPOS, false>; break;
      case EPI_BF16_GELU: kern = gemm_wg_kernel<BN, EPI_BF16_GELU, false>; break;
      default: kern = gemm_wg_kernel<BN, EPI_GENERIC, false>; break;
    }
  }
  RVB_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM_BYTES));
  p.tiles_n = a.grp ? p.grp_slots * (p.group_n / BN) : (a.N + BN - 1) / BN;
  int tiles_m = a.conv_mode ? a.conv_B * a.conv_F2 * p.conv_tt : (a.M + 127) / 128;
  p.num_tiles = tiles_m * p.tiles_n;
  int grid = p.num_tiles < g_num_sms ? p.num_tiles : g_num_sms;
  GemmProfRec rec;
  if (g_prof_on) {
    if (prof_event(&rec.a) || prof_event(&rec.b)) return -1;
    rec.flops = 2.0 * (double)a.M * (double)(a.grp ? a.group_n : a.N) * (double)a.K * (a.x3 ? 3.0 : 1.0);
    RVB_CHECK_CUDA(cudaEventRecord(rec.a, stream));
  }
  kern<<<grid, kGemmThreads, SMEM_BYTES, stream>>>(tmA, tmB, p);
  RVB_COUNT_LAUNCH();
  RVB_CHECK_LAUNCH();
  if (g_prof_on) {
    RVB_CHECK_CUDA(cudaEventRecord(rec.b, stream));
    {
      std::lock_guard<std::mutex> lock(g_prof_mutex);
      g_prof.push_back(rec);
    }
  }
  return 0;
}

int launch_gemm(const GemmArgs& a, cudaStream_t stream) {
  RVB_REQUIRE(a.A && a.W && (a.out || a.out_mode == OUT_LSE), "gemm: null pointer");
  RVB_REQUIRE(a.M > 0 && a.N > 0 && a.K > 0, "gemm: bad shape M=%d N=%d K=%d", a.M, a.N, a.K);
  if (g_num_sms == 0) {
    int dev = 0;
    RVB_CHECK_CUDA(cudaGetDevice(&dev));
    RVB_CHECK_CUDA(cudaDeviceGetAttribute(&g_num_sms, cudaDevAttrMultiProcessorCount, dev));
  }
  GemmKParams p;
  memset(&p, 0, sizeof(p));
  p.M = a.M;
  p.N = a.N;
  p.K = a.K;
  p.num_k_blocks = (a.K + 63) / 64;
  p.x3 = a.x3;
  p.kb_seg = p.num_k_blocks;
  p.out_split = a.out_split;
  if (a.x3) {
    RVB_REQUIRE(a.K % 64 == 0, "gemm: bf16x3 mode needs K %% 64 == 0 (K=%d)", a.K);
    RVB_REQUIRE(get_gemm_impl() != 1, "gemm: bf16x3 mode is not built for the simt bring-up kernel");
    p.num_k_blocks *= 3;
    p.a_lo_ofs = a.conv_mode ? a.conv_C : a.K;
    p.w_lo_ofs = a.K;
  }
  if (a.out_split > 0)
    RVB_REQUIRE((a.out_mode == OUT_BF16) && a.out_split % 8 == 0, "gemm: out_split needs an aligned bf16 output");
  p.bias = a.bias;
  p.act = a.act;
  p.out_mode = a.out_mode;
  p.out = a.out;
  if (a.grp) {
    RVB_REQUIRE(a.group_n > 0 && a.group_n % 64 == 0 && a.N % a.group_n == 0 && a.rows_per_batch > 0 &&
                    a.act == ACT_NONE && (a.out_mode == OUT_BF16 || a.out_mode == OUT_F32) && !a.conv_mode && !a.rp_pos,
                "gemm: a grouped output needs group_n %% 64 == 0 dividing N (N=%d group_n=%d), rows_per_batch, no "
                "activation and a plain bf16 / fp32 output", a.N, a.group_n);
    RVB_REQUIRE(get_gemm_impl() != 1, "gemm: grouped output is not built for the simt bring-up kernel");
  }
  p.grp = a.grp;
  p.group_n = a.grp ? a.group_n : a.N;
  if (a.grp) {   // rows [r0, r0 + 128) touch at most 127 / rpb + 2 utterances
    const int rpb = a.rows_per_batch, n_utt = (a.M + rpb - 1) / rpb;
    p.grp_slots = std::min(n_utt, 127 / rpb + 2);
  }
  p.ldo = a.ldo ? a.ldo : (long long)(a.act == ACT_GLU ? a.N / 2 : p.group_n) * (a.out_split > 0 ? 2 : 1);
  p.alpha = a.alpha;
  p.row_lens = a.row_lens;
  p.rows_per_batch = a.rows_per_batch > 0 ? a.rows_per_batch : a.M;
  p.conv_mode = a.conv_mode;
  p.lse_gather = a.lse_gather;
  p.lse_part = a.lse_part;
  p.lse_tgt = a.lse_tgt;
  p.lse_nslab = lse_slabs(a.N);
  p.rp_pos = a.rp_pos;
  p.rp_ldp = a.rp_ldp;
  p.rp_T = a.rp_T;
  p.rp_H = a.rp_H;
  p.rp_col0 = a.rp_col0;
  p.rp_u = a.rp_u;
  p.rp_v = a.rp_v;
  p.rp_cb = a.rp_cb;
  if (a.rp_pos) {
    RVB_REQUIRE(a.out_mode == OUT_BF16 && a.act == ACT_NONE && a.out_split == 0 && !a.conv_mode && a.rp_T > 0 &&
                    a.rp_col0 % 64 == 0 && a.rp_ldp % 8 == 0 && a.N % 64 == 0 && a.rp_u && a.rp_v && a.rp_cb &&
                    (reinterpret_cast<uintptr_t>(a.rp_pos) & 15) == 0 && (reinterpret_cast<uintptr_t>(a.rp_u) & 15) == 0 &&
                    (reinterpret_cast<uintptr_t>(a.rp_v) & 15) == 0,
                "gemm: rel-pos epilogue needs a plain bf16 output, 64-aligned key columns and 16-byte aligned tables");
    RVB_REQUIRE(get_gemm_impl() != 1, "gemm: rel-pos epilogue is not built for the simt bring-up kernel");
  }
  if (a.act == ACT_GELU) {
    RVB_REQUIRE(a.out_mode == OUT_BF16 && a.out_split == 0 && !a.x3 && !a.grp && !a.rp_pos,
                "gemm: ACT_GELU needs a plain bf16 output");
    RVB_REQUIRE(get_gemm_impl() != 1, "gemm: ACT_GELU is not built for the simt bring-up kernel");
  }
  if (a.out_mode == OUT_LSE) {
    RVB_REQUIRE(a.lse_gather && a.lse_part && a.lse_tgt && a.act == ACT_NONE && !a.conv_mode && a.N > 128,
                "gemm: OUT_LSE needs gather / partial / target buffers, no activation and N > 128");
    RVB_REQUIRE(get_gemm_impl() != 1, "gemm: OUT_LSE is not built for the simt bring-up kernel");
  }
  {
    static int skip = -1;
    if (skip < 0) {
      const char* e = getenv("RVB_GEMM_SKIP_EPI");
      skip = e ? atoi(e) : 0;
    }
    p.debug_skip_epi = skip;
  }
  p.glu_coalesced = (a.act == ACT_GLU);
  p.bf16_coalesced = (a.out_mode == OUT_BF16) && (a.act != ACT_GLU) && (p.ldo % 8 == 0) &&
                     ((reinterpret_cast<uintptr_t>(a.out) & 15) == 0) &&
                     (a.bias == nullptr || (reinterpret_cast<uintptr_t>(a.bias) & 15) == 0);
  p.f32_coalesced = (a.out_mode != OUT_BF16) && (p.ldo % 4 == 0) && ((reinterpret_cast<uintptr_t>(a.out) & 15) == 0) &&
                    (a.bias == nullptr || (reinterpret_cast<uintptr_t>(a.bias) & 15) == 0);
  p.A = a.A;
  p.W = a.W;
  p.lda = a.lda ? a.lda : (long long)a.K * (a.x3 ? 2 : 1);
  p.ldw = a.ldw ? a.ldw : (long long)a.K * (a.x3 ? 2 : 1);
  if (a.conv_mode) {
    RVB_REQUIRE(a.conv_C % 64 == 0, "conv implicit GEMM needs C %% 64 == 0 (C=%d)", a.conv_C);
    RVB_REQUIRE(a.K == 9 * a.conv_C && a.M == a.conv_B * a.conv_F2 * a.conv_T2, "conv implicit GEMM: bad M/K");
    p.conv_T2 = a.conv_T2;
    p.conv_F2 = a.conv_F2;
    p.conv_orow_mul = a.conv_pair_out ? 2 * a.conv_F2 : a.conv_F2;
    p.conv_tt = (a.conv_T2 + 127) / 128;
    p.conv_cblocks = a.conv_C / 64;
    p.conv_T1h = a.conv_T1h;
    p.conv_F1 = a.conv_F1;
    p.conv_C = a.conv_C;
  }
  if (a.out_split > 0)
    RVB_REQUIRE(a.N % 128 == 0 && (a.act == ACT_GLU ? p.glu_coalesced : p.bf16_coalesced),
                "gemm: a hi/lo output pair needs N %% 128 == 0 and 16-byte aligned rows (N=%d)", a.N);
  if (a.act == ACT_GLU) {
    RVB_REQUIRE(a.out_mode == OUT_BF16 && a.N % 64 == 0 && !a.conv_mode, "gemm: ACT_GLU needs bf16 output and N %% 64 == 0");
    RVB_REQUIRE((reinterpret_cast<uintptr_t>(a.out) & 15) == 0 && p.ldo % 8 == 0 &&
                    (a.bias == nullptr || (reinterpret_cast<uintptr_t>(a.bias) & 15) == 0),
                "gemm: ACT_GLU needs 16-byte aligned output rows and bias");
  }
  if (get_gemm_impl() == 1) {
    p.tiles_n = ((a.act == ACT_GLU ? a.N / 2 : a.N) + 31) / 32;
    int tiles_m = a.conv_mode ? a.conv_B * a.conv_F2 * p.conv_tt : (a.M + 127) / 128;
    p.num_tiles = tiles_m * p.tiles_n;
    int grid = p.num_tiles < g_num_sms * 8 ? p.num_tiles : g_num_sms * 8;
    gemm_simt_kernel<<<grid, 256, 0, stream>>>(p);
    RVB_COUNT_LAUNCH();
    RVB_CHECK_LAUNCH();
    return 0;
  }
  RVB_REQUIRE((reinterpret_cast<uintptr_t>(a.A) & 15) == 0 && (reinterpret_cast<uintptr_t>(a.W) & 15) == 0,
              "gemm: operands must be 16-byte aligned");
  RVB_REQUIRE((p.lda * 2) % 16 == 0 && (p.ldw * 2) % 16 == 0, "gemm: leading dimensions must be multiples of 8");
  if (get_encode_fn()) return -1;
  // 64-wide tiles for narrow outputs; RVB_GEMM=narrow (impl 2) takes them for every shape whose epilogue allows it:
  // all but the log-sum-exp partials (128-column slabs) and GLU hi/lo pairs (written 128 accumulator columns at a time)
  // (a grouped output takes the tiles a plain launch of one group's N columns would take)
  const bool narrow = p.group_n <= 64 || (get_gemm_impl() == 2 && a.out_mode != OUT_LSE && !(a.act == ACT_GLU && a.out_split > 0));
  RVB_REQUIRE(!a.grp || p.group_n % (narrow ? 64 : 128) == 0, "gemm: grouped output needs group_n %% %d == 0 (group_n=%d)",
              narrow ? 64 : 128, p.group_n);
  if (narrow) return launch_wg<64>(a, p, stream);
  // 128 x 256 tiles (gemm_wide_kernel) for a plain bf16 output with bias / ReLU / SiLU, N % 256 == 0 and at least one
  // wave of tiles; RVB_GEMM_WIDE=0 (read per call, so one process can A/B both) keeps every shape on 128 x 128 tiles
  const int epi = select_epi(a.act, a.out_mode);
  const long long wide_tiles = (long long)(a.conv_mode ? a.conv_B * a.conv_F2 * p.conv_tt : (a.M + 127) / 128) * (a.N / 256);
  const char* wide_env = getenv("RVB_GEMM_WIDE");
  if ((epi == EPI_BF16 || epi == EPI_BF16_RELU || epi == EPI_BF16_SILU) && !a.rp_pos && !a.grp && !a.x3 &&
      a.out_split == 0 && p.bf16_coalesced && a.N % 256 == 0 && wide_tiles >= g_num_sms &&
      !(wide_env && strcmp(wide_env, "0") == 0))
    return launch_wg<256>(a, p, stream);
  return launch_wg<128>(a, p, stream);
}

}  // namespace rvb
