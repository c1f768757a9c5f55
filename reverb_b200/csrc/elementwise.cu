// reverb_b200 — HBM-bound kernels of the Conformer stack: LayerNorm (single / fused pair), CMVN+conv1+ReLU,
// GLU + depthwise conv + norm + SiLU, decoder embedding, small casts.  Warp-shuffle reductions, 128-bit loads.
#include <math.h>

#include "kernels.h"

namespace rvb {

// bf16x3 ("fp32-accurate") mode: an activation is stored as the bf16 PAIR hi = bf16(v), lo = bf16(v - hi), side by side in
// one row: hi at column c, lo at column c + width (row stride 2 * width).  See GemmArgs::x3 (kernels.h).
__device__ __forceinline__ float bf16_residue(float v) { return v - __bfloat162float(__float2bfloat16(v)); }
__device__ __forceinline__ void store_pair4(bf16* row, int col, int width, bool x3, float4 o) {
  uint2 u;
  u.x = pack_bf16x2(o.x, o.y);
  u.y = pack_bf16x2(o.z, o.w);
  *reinterpret_cast<uint2*>(row + col) = u;
  if (x3) {
    u.x = pack_bf16x2(bf16_residue(o.x), bf16_residue(o.y));
    u.y = pack_bf16x2(bf16_residue(o.z), bf16_residue(o.w));
    *reinterpret_cast<uint2*>(row + width + col) = u;
  }
}

// ---------------------------------------------------------------------------------------------------------------
// LayerNorm: one warp per row, row cached in registers (NV float4 per lane), two-pass variance like ATen.
// reference: nn.LayerNorm uses of transformer/encoder_layer.py:149-159, encoder.py:107, decoder_layer.py:53-55,241-243
template <int NV, bool X3>
__global__ void __launch_bounds__(256) layernorm_kernel(const float* __restrict__ x, const float* __restrict__ gamma,
                                                        const float* __restrict__ beta, float eps, int M, int d,
                                                        bf16* __restrict__ out_bf16, float* __restrict__ out_f32,
                                                        const int* __restrict__ row_lens, int rows_per_batch,
                                                        int mask_rows) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (warp >= M) return;
  const int nvec = d >> 2;
  const float4* xr = reinterpret_cast<const float4*>(x + (long long)warp * d);
  bool masked = false;
  if (mask_rows && row_lens != nullptr) {
    int b = warp / rows_per_batch;
    masked = (warp - b * rows_per_batch) >= __ldg(row_lens + b);
  }
  float4 v[NV];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    int idx = lane + 32 * i;
    if (idx < nvec) {
      v[i] = xr[idx];
      s += (v[i].x + v[i].y) + (v[i].z + v[i].w);
    } else {
      v[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
  }
  const float mean = warp_sum(s) / (float)d;
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    int idx = lane + 32 * i;
    if (idx < nvec) {
      float a = v[i].x - mean, b = v[i].y - mean, c = v[i].z - mean, e = v[i].w - mean;
      q += (a * a + b * b) + (c * c + e * e);
    }
  }
  const float rstd = rsqrtf(warp_sum(q) / (float)d + eps);
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    int idx = lane + 32 * i;
    if (idx < nvec) {
      float4 g = __ldg(reinterpret_cast<const float4*>(gamma) + idx);
      float4 bb = __ldg(reinterpret_cast<const float4*>(beta) + idx);
      float4 o;
      o.x = (v[i].x - mean) * rstd * g.x + bb.x;
      o.y = (v[i].y - mean) * rstd * g.y + bb.y;
      o.z = (v[i].z - mean) * rstd * g.z + bb.z;
      o.w = (v[i].w - mean) * rstd * g.w + bb.w;
      if (masked) o = make_float4(0.f, 0.f, 0.f, 0.f);
      if (out_f32) reinterpret_cast<float4*>(out_f32 + (long long)warp * d)[idx] = o;
      if (out_bf16) store_pair4(out_bf16 + (long long)warp * d * (X3 ? 2 : 1), 4 * idx, d, X3, o);
    }
  }
}

int launch_layernorm(const float* x, const float* gamma, const float* beta, float eps, int M, int d, bf16* out_bf16,
                     float* out_f32, const int* row_lens, int rows_per_batch, int mask_rows, cudaStream_t stream,
                     int x3) {
  RVB_REQUIRE(d % 4 == 0 && d <= 4096, "layernorm: d=%d unsupported (need d %% 4 == 0, d <= 4096)", d);
  if (M <= 0) return 0;
  const int grid = (M + 7) / 8;
  const int nv = (d / 4 + 31) / 32;
  if (rows_per_batch <= 0) rows_per_batch = M;
#define RVB_LN(NV)                                                                                                  \
  do {                                                                                                              \
    if (x3) layernorm_kernel<NV, true><<<grid, 256, 0, stream>>>(x, gamma, beta, eps, M, d, out_bf16, out_f32, row_lens, \
                                                                 rows_per_batch, mask_rows);                        \
    else layernorm_kernel<NV, false><<<grid, 256, 0, stream>>>(x, gamma, beta, eps, M, d, out_bf16, out_f32, row_lens,   \
                                                               rows_per_batch, mask_rows);                          \
  } while (0)
  if (nv <= 1) RVB_LN(1);
  else if (nv <= 2) RVB_LN(2);
  else if (nv <= 4) RVB_LN(4);
  else if (nv <= 8) RVB_LN(8);
  else if (nv <= 16) RVB_LN(16);
  else RVB_LN(32);
#undef RVB_LN
  RVB_COUNT_LAUNCH();
  RVB_CHECK_LAUNCH();
  return 0;
}

// x2 = LN_a(x) (+ y_add) ; n = LN_b(x2).  Fuses `norm_final` of block i (and the LSL `x = x + y`,
// encoder_layer.py:397-400) with the first pre-norm of block i+1 (or encoder.after_norm): one read, two writes.
template <int NV, bool X3>
__global__ void __launch_bounds__(256)
double_layernorm_kernel(const float* __restrict__ x, const float* __restrict__ ga, const float* __restrict__ ba,
                        const float* __restrict__ y_add, float* __restrict__ x2, const float* __restrict__ gb,
                        const float* __restrict__ bb, float eps, int M, int d, bf16* __restrict__ n_out,
                        float* __restrict__ n_out_f32) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (warp >= M) return;
  const int nvec = d >> 2;
  const float4* xr = reinterpret_cast<const float4*>(x + (long long)warp * d);
  float4 v[NV];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    int idx = lane + 32 * i;
    if (idx < nvec) {
      v[i] = xr[idx];
      s += (v[i].x + v[i].y) + (v[i].z + v[i].w);
    } else {
      v[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
  }
  float mean = warp_sum(s) / (float)d;
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    int idx = lane + 32 * i;
    if (idx < nvec) {
      float a = v[i].x - mean, b = v[i].y - mean, c = v[i].z - mean, e = v[i].w - mean;
      q += (a * a + b * b) + (c * c + e * e);
    }
  }
  float rstd = rsqrtf(warp_sum(q) / (float)d + eps);
  s = 0.f;
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    int idx = lane + 32 * i;
    if (idx < nvec) {
      float4 g = __ldg(reinterpret_cast<const float4*>(ga) + idx);
      float4 b4 = __ldg(reinterpret_cast<const float4*>(ba) + idx);
      float4 o;
      o.x = (v[i].x - mean) * rstd * g.x + b4.x;
      o.y = (v[i].y - mean) * rstd * g.y + b4.y;
      o.z = (v[i].z - mean) * rstd * g.z + b4.z;
      o.w = (v[i].w - mean) * rstd * g.w + b4.w;
      if (y_add) {
        float4 y = reinterpret_cast<const float4*>(y_add + (long long)warp * d)[idx];
        o.x += y.x;
        o.y += y.y;
        o.z += y.z;
        o.w += y.w;
      }
      reinterpret_cast<float4*>(x2 + (long long)warp * d)[idx] = o;
      v[i] = o;
      s += (o.x + o.y) + (o.z + o.w);
    }
  }
  if (n_out == nullptr && n_out_f32 == nullptr) return;
  mean = warp_sum(s) / (float)d;
  q = 0.f;
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    int idx = lane + 32 * i;
    if (idx < nvec) {
      float a = v[i].x - mean, b = v[i].y - mean, c = v[i].z - mean, e = v[i].w - mean;
      q += (a * a + b * b) + (c * c + e * e);
    }
  }
  rstd = rsqrtf(warp_sum(q) / (float)d + eps);
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    int idx = lane + 32 * i;
    if (idx < nvec) {
      float4 g = __ldg(reinterpret_cast<const float4*>(gb) + idx);
      float4 b4 = __ldg(reinterpret_cast<const float4*>(bb) + idx);
      float4 o;
      o.x = (v[i].x - mean) * rstd * g.x + b4.x;
      o.y = (v[i].y - mean) * rstd * g.y + b4.y;
      o.z = (v[i].z - mean) * rstd * g.z + b4.z;
      o.w = (v[i].w - mean) * rstd * g.w + b4.w;
      if (n_out_f32) reinterpret_cast<float4*>(n_out_f32 + (long long)warp * d)[idx] = o;
      if (n_out) store_pair4(n_out + (long long)warp * d * (X3 ? 2 : 1), 4 * idx, d, X3, o);
    }
  }
}

int launch_double_layernorm(const float* x, const float* ga, const float* ba, const float* y_add, float* x2,
                            const float* gb, const float* bb, float eps, int M, int d, bf16* n_out,
                            float* n_out_f32, cudaStream_t stream, int x3) {
  RVB_REQUIRE(d % 4 == 0 && d <= 4096, "double_layernorm: d=%d unsupported", d);
  if (M <= 0) return 0;
  const int grid = (M + 7) / 8;
  const int nv = (d / 4 + 31) / 32;
#define RVB_DLN(NV)                                                                                                     \
  do {                                                                                                                  \
    if (x3) double_layernorm_kernel<NV, true><<<grid, 256, 0, stream>>>(x, ga, ba, y_add, x2, gb, bb, eps, M, d, n_out, n_out_f32); \
    else double_layernorm_kernel<NV, false><<<grid, 256, 0, stream>>>(x, ga, ba, y_add, x2, gb, bb, eps, M, d, n_out, n_out_f32);   \
  } while (0)
  if (nv <= 1) RVB_DLN(1);
  else if (nv <= 2) RVB_DLN(2);
  else if (nv <= 4) RVB_DLN(4);
  else if (nv <= 8) RVB_DLN(8);
  else if (nv <= 16) RVB_DLN(16);
  else RVB_DLN(32);
#undef RVB_DLN
  RVB_COUNT_LAUNCH();
  RVB_CHECK_LAUNCH();
  return 0;
}

// ---------------------------------------------------------------------------------------------------------------
// GlobalCMVN + Conv2d(1, C, 3, stride 2) + ReLU  (transformer/cmvn.py:36-47, subsampling.py:186-187).
// Output is channels-last bf16 with the time axis split by parity, (B, 2, T1h, F1, C), so that the second conv's
// implicit-GEMM A tiles (gemm.cu conv_mode) are plain unit-stride 4-D TMA boxes.  One CTA per (b, C1_ROWS output
// rows): a thread keeps the 8 x 9 weights of its channel group in registers (as 4 x 9 channel PAIRS for the packed
// FFMA2) and reuses them for every (row, f), so the weight fetch is amortised over C1_ROWS * F1 outputs; the
// 2*C1_ROWS+1 CMVN'd input rows sit in shared memory, each value duplicated {x, x} as the second FFMA2 operand.
constexpr int C1_ROWS = 4;

__global__ void __launch_bounds__(256)
conv1_kernel(const float* __restrict__ feats, const float* __restrict__ mean, const float* __restrict__ istd,
             const float* __restrict__ w, const float* __restrict__ bias, bf16* __restrict__ out, int T, int F, int C,
             int T1, int T1h, int F1, int x3) {
  extern __shared__ float2 s_in2[];  // (2*C1_ROWS+1) rows x F, CMVN applied, every value DUPLICATED {x, x} (FFMA2 operand)
  const int t1_0 = blockIdx.x * C1_ROWS;  // first output row of this CTA, 0 .. 2*T1h-1
  const int b = blockIdx.y;
  const int CG = C >> 3;
  constexpr int IN_ROWS = 2 * C1_ROWS + 1;
  for (int i = threadIdx.x; i < IN_ROWS * F; i += blockDim.x) {
    int kh = i / F, f = i - kh * F;
    int t = 2 * t1_0 + kh;
    float x = (t < T) ? feats[((long long)b * T + t) * F + f] : 0.f;
    x = (x - __ldg(mean + f)) * __ldg(istd + f);
    s_in2[i] = make_float2(x, x);
  }
  const int cg = threadIdx.x % CG;
  const int fstep = blockDim.x / CG;
  // channel pairs (2p, 2p+1) of this thread's 8 channels share one packed accumulator
  float2 wr[4][9], br[4];
#pragma unroll
  for (int pc = 0; pc < 4; ++pc) {
    const int c = cg * 8 + 2 * pc;
    br[pc] = make_float2(__ldg(bias + c), __ldg(bias + c + 1));
#pragma unroll
    for (int k = 0; k < 9; ++k) wr[pc][k] = make_float2(__ldg(w + c * 9 + k), __ldg(w + (c + 1) * 9 + k));
  }
  __syncthreads();
  for (int rr = 0; rr < C1_ROWS; ++rr) {
    const int t1 = t1_0 + rr;
    if (t1 >= 2 * T1h) break;
    const int par = t1 & 1, th = t1 >> 1;
    const int Cp = x3 ? 2 * C : C;  // physical channels: [hi C | lo C] in bf16x3 mode
    bf16* orow = out + (((long long)(b * 2 + par) * T1h + th) * F1) * Cp;
    if (t1 >= T1) {  // padding row (T1 odd): keep it finite
      for (int i = threadIdx.x; i < F1 * (Cp >> 3); i += blockDim.x)
        reinterpret_cast<uint4*>(orow)[i] = make_uint4(0u, 0u, 0u, 0u);
      continue;
    }
    const float2* s_r = s_in2 + 2 * rr * F;
    for (int f = threadIdx.x / CG; f < F1; f += fstep) {
      float2 in[9];
#pragma unroll
      for (int kh = 0; kh < 3; ++kh)
#pragma unroll
        for (int kw = 0; kw < 3; ++kw) in[kh * 3 + kw] = s_r[kh * F + 2 * f + kw];
      float2 o[4];
#pragma unroll
      for (int pc = 0; pc < 4; ++pc) {
        float2 a = br[pc];
#pragma unroll
        for (int k = 0; k < 9; ++k) a = ffma2(wr[pc][k], in[k], a);
        o[pc] = make_float2(fmaxf(a.x, 0.f), fmaxf(a.y, 0.f));
      }
      uint4 u;
      u.x = pack_bf16x2(o[0].x, o[0].y);
      u.y = pack_bf16x2(o[1].x, o[1].y);
      u.z = pack_bf16x2(o[2].x, o[2].y);
      u.w = pack_bf16x2(o[3].x, o[3].y);
      reinterpret_cast<uint4*>(orow + (long long)f * Cp)[cg] = u;
      if (x3) {
        u.x = pack_bf16x2(bf16_residue(o[0].x), bf16_residue(o[0].y));
        u.y = pack_bf16x2(bf16_residue(o[1].x), bf16_residue(o[1].y));
        u.z = pack_bf16x2(bf16_residue(o[2].x), bf16_residue(o[2].y));
        u.w = pack_bf16x2(bf16_residue(o[3].x), bf16_residue(o[3].y));
        reinterpret_cast<uint4*>(orow + (long long)f * Cp + C)[cg] = u;
      }
    }
  }
}

int launch_conv1(const float* feats, const float* mean, const float* istd, const float* w, const float* bias,
                 bf16* out, int B, int T, int F, int C, int T1, int T1h, int F1, cudaStream_t stream, int x3) {
  RVB_REQUIRE(C % 8 == 0 && C / 8 <= 256, "conv1: C=%d unsupported", C);
  const int CG = C / 8;
  const int threads = (256 / CG) * CG;
  dim3 grid((2 * T1h + C1_ROWS - 1) / C1_ROWS, B);
  conv1_kernel<<<grid, threads, (2 * C1_ROWS + 1) * F * sizeof(float2), stream>>>(feats, mean, istd, w, bias, out, T, F,
                                                                                 C, T1, T1h, F1, x3);
  RVB_COUNT_LAUNCH();
  RVB_CHECK_LAUNCH();
  return 0;
}

// ---------------------------------------------------------------------------------------------------------------
// Conformer convolution module, middle part (transformer/convolution.py:129-138):
//   [pointwise_conv1 + GLU: fused into the GEMM epilogue, ACT_GLU]
//   depthwise conv (K taps, causal left pad K-1 or symmetric (K-1)/2) + bias
//   -> LayerNorm over channels (or BatchNorm1d eval) -> SiLU.
// Input (B, T, C) bf16 = GLU(pointwise_conv1(x)); output (B, T, C) bf16 feeds pointwise_conv2.  Layout stays
// (B, T, C) end to end: no transposes.
//
// Kernel A (conv_dw_kernel): one (batch, CM_TT-frame tile, 128-channel-pair slice) per 128-thread CTA; a thread owns
// one channel pair, loads its CM_TT+K-1 halo values straight into registers (a warp reads 128 contiguous bytes per
// frame) and runs the fully unrolled sliding window.  No block-wide phases, several CTAs per SM, so the loads of one
// CTA overlap the FMAs of the others.  With LayerNorm it writes the fp32 conv result and accumulates per-frame
// sum / sum of squares into one slot per (frame, channel slice) — no atomics, deterministic; kernel B (conv_norm_silu_kernel, one warp per frame)
// normalises + SiLU -> bf16.  With BatchNorm (eval) kernel A applies norm + SiLU itself and writes bf16 directly.
// K = 0 instantiates the generic version (run-time tap count, halo re-read through L1).
//
// pad_glu (C fp32, causal mode): the reference left-pads K-1 zero frames BEFORE pointwise_conv1
// (convolution.py:113-114,129-130), so the pad frames reach the depthwise conv as GLU(bias), not zeros.
constexpr int CM_TT = 16;

template <int K, bool X3>
__global__ void __launch_bounds__(128)
conv_dw_kernel(const bf16* __restrict__ x, const float* __restrict__ pad_glu, const float* __restrict__ dw_w,
               const float* __restrict__ dw_b, const float* __restrict__ norm_w, const float* __restrict__ norm_b,
               const float* __restrict__ bn_mean, const float* __restrict__ bn_var, int use_ln, float eps,
               float* __restrict__ conv_out, float* __restrict__ stats, bf16* __restrict__ out, int T, int C,
               int Krt, int causal, int conv_chunk) {
  __shared__ float s_part[4][CM_TT][2];
  const int b = blockIdx.y;
  const int t0 = blockIdx.x * CM_TT;
  const int C2 = C >> 1;
  const int cp = blockIdx.z * 128 + threadIdx.x;
  const bool ok = cp < C2;
  const int KK = (K > 0) ? K : Krt;
  const int left = causal ? (KK - 1) : (KK - 1) / 2;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float b0 = 0.f, b1 = 0.f;
  float2 padv = make_float2(0.f, 0.f);
  if (ok) {
    b0 = __ldg(dw_b + 2 * cp);
    b1 = __ldg(dw_b + 2 * cp + 1);
    if (causal) padv = make_float2(__ldg(pad_glu + 2 * cp), __ldg(pad_glu + 2 * cp + 1));
  }
  float acc[CM_TT][2];
#pragma unroll
  for (int t = 0; t < CM_TT; ++t) {
    acc[t][0] = b0;
    acc[t][1] = b1;
  }
  // X3: rows are [hi C | lo C] (2C bf16 = C uint32 words); the value is hi + lo
  const int CW = X3 ? C : C2;  // row stride in uint32 words
  const uint32_t* xb = reinterpret_cast<const uint32_t*>(x + (long long)b * T * C * (X3 ? 2 : 1)) + cp;
  if constexpr (K > 0) {
    constexpr int ROWS = CM_TT + K - 1;
    uint32_t rv[ROWS];
    uint32_t rl[X3 ? ROWS : 1];
#pragma unroll
    for (int r = 0; r < ROWS; ++r) {
      const int t = t0 - left + r;
      rv[r] = 0u;
      if (X3) rl[r] = 0u;
      if (ok && t >= 0 && t < T) {
        rv[r] = __ldg(xb + (long long)t * CW);
        if (X3) rl[r] = __ldg(xb + (long long)t * CW + C2);
      }
    }
    float w0[K], w1[K];
#pragma unroll
    for (int k = 0; k < K; ++k) {
      w0[k] = ok ? __ldg(dw_w + (2 * cp) * K + k) : 0.f;
      w1[k] = ok ? __ldg(dw_w + (2 * cp + 1) * K + k) : 0.f;
    }
#pragma unroll
    for (int r = 0; r < ROWS; ++r) {
      const int tt = t0 - left + r;
      float2 v = (tt < 0) ? padv : unpack_bf16x2(rv[r]);  // rv is 0 beyond T
      if (X3 && tt >= 0) {
        const float2 l = unpack_bf16x2(rl[r]);
        v.x += l.x;
        v.y += l.y;
      }
#pragma unroll
      for (int k = 0; k < K; ++k) {
        const int t = r - k;  // compile-time after unrolling
        if (t >= 0 && t < CM_TT) {
          // the channel pair's two FMAs as one packed FFMA2
          const float2 a2 = ffma2(make_float2(w0[k], w1[k]), v, make_float2(acc[t][0], acc[t][1]));
          acc[t][0] = a2.x;
          acc[t][1] = a2.y;
        }
      }
    }
  } else if (ok) {  // generic tap count
    for (int k = 0; k < KK; ++k) {
      const float w0 = __ldg(dw_w + (2 * cp) * KK + k), w1 = __ldg(dw_w + (2 * cp + 1) * KK + k);
#pragma unroll
      for (int t = 0; t < CM_TT; ++t) {
        const int tt = t0 + t - left + k;
        float2 v = make_float2(0.f, 0.f);
        // conv_chunk > 0 (cache-based streaming simulation of a NON-causal model, encoder.py:341-402): every chunk is
        // convolved on its own, zero padded at its edges — taps outside the output frame's chunk contribute nothing
        if (conv_chunk > 0 && (tt < 0 || tt / conv_chunk != (t0 + t) / conv_chunk)) {
        } else if (tt < 0) v = padv;
        else if (tt < T) {
          v = unpack_bf16x2(__ldg(xb + (long long)tt * CW));
          if (X3) {
            const float2 l = unpack_bf16x2(__ldg(xb + (long long)tt * CW + C2));
            v.x += l.x;
            v.y += l.y;
          }
        }
        acc[t][0] = fmaf(w0, v.x, acc[t][0]);
        acc[t][1] = fmaf(w1, v.y, acc[t][1]);
      }
    }
  }
  if (!use_ln) {
    if (!ok) return;
    const int c0 = 2 * cp, c1 = 2 * cp + 1;
    const float g0 = __ldg(norm_w + c0), g1 = __ldg(norm_w + c1), be0 = __ldg(norm_b + c0), be1 = __ldg(norm_b + c1);
    const float m0 = __ldg(bn_mean + c0), m1 = __ldg(bn_mean + c1);
    const float r0 = rsqrtf(__ldg(bn_var + c0) + eps), r1 = rsqrtf(__ldg(bn_var + c1) + eps);
#pragma unroll
    for (int t = 0; t < CM_TT; ++t) {
      if (t0 + t >= T) continue;
      const float y0 = (acc[t][0] - m0) * r0 * g0 + be0, y1 = (acc[t][1] - m1) * r1 * g1 + be1;
      if (X3) {
        const float s0 = y0 / (1.f + expf(-y0)), s1 = y1 / (1.f + expf(-y1));
        uint32_t* orow = reinterpret_cast<uint32_t*>(out + ((long long)b * T + t0 + t) * C * 2);
        orow[cp] = pack_bf16x2(s0, s1);
        orow[C2 + cp] = pack_bf16x2(bf16_residue(s0), bf16_residue(s1));
      } else {
        reinterpret_cast<uint32_t*>(out + ((long long)b * T + t0 + t) * C)[cp] = pack_bf16x2(silu_f(y0), silu_f(y1));
      }
    }
    return;
  }
  // per-frame sum / sum of squares over the warp's 64 channels: the 2 x CM_TT partials of a lane are reduced with a
  // transposing butterfly (31 shuffles instead of 10 per value): afterwards lane l holds the total of value l
  static_assert(CM_TT == 16, "the statistics butterfly assumes 32 values per lane");
  float sv[32];
#pragma unroll
  for (int t = 0; t < CM_TT; ++t) {
    sv[t] = ok ? acc[t][0] + acc[t][1] : 0.f;
    sv[CM_TT + t] = ok ? acc[t][0] * acc[t][0] + acc[t][1] * acc[t][1] : 0.f;
    if (ok && t0 + t < T)
      reinterpret_cast<float2*>(conv_out + ((long long)b * T + t0 + t) * C)[cp] = make_float2(acc[t][0], acc[t][1]);
  }
#pragma unroll
  for (int ofs = 16; ofs >= 1; ofs >>= 1) {
    const bool up = (lane & ofs) != 0;
#pragma unroll
    for (int i = 0; i < ofs; ++i) {
      const float send = up ? sv[i] : sv[i + ofs];
      const float keep = up ? sv[i + ofs] : sv[i];
      sv[i] = keep + __shfl_xor_sync(0xffffffffu, send, ofs);
    }
  }
  s_part[warp][lane & (CM_TT - 1)][lane >> 4] = sv[0];   // lanes 0..15: sums of frames 0..15, lanes 16..31: squares
  __syncthreads();
  if (threadIdx.x < 2 * CM_TT) {
    const int t = threadIdx.x >> 1, which = threadIdx.x & 1;
    if (t0 + t < T) {
      // one slot per (frame, channel slice): no atomics, so the statistics (and everything after) are deterministic
      const float v = s_part[0][t][which] + s_part[1][t][which] + s_part[2][t][which] + s_part[3][t][which];
      stats[(((long long)b * T + t0 + t) * gridDim.z + blockIdx.z) * 2 + which] = v;
    }
  }
}

// Fused variant for LayerNorm when one CTA can hold the whole channel dimension (C / 2 <= 512 threads, i.e. d <= 1024): depthwise conv,
// per-frame statistics (warp butterfly + one shared-memory reduction across the CTA's warps), normalise + SiLU, bf16 out —
// the fp32 conv result never goes to HBM (conv_dw_kernel + conv_norm_silu_kernel move 588 MB per layer at the benchmark
// shape, this kernel 196 MB: read the GLU output once, write the bf16 operand of pointwise_conv2 once).
template <int K>
__global__ void __launch_bounds__(512)
conv_dw_ln_fused_kernel(const bf16* __restrict__ x, const float* __restrict__ pad_glu, const float* __restrict__ dw_w,
                        const float* __restrict__ dw_b, const float* __restrict__ norm_w,
                        const float* __restrict__ norm_b, float eps, bf16* __restrict__ out, int T, int C, int causal) {
  __shared__ float s_part[16][32];   // [warp][16 frame sums | 16 frame sums of squares]
  __shared__ float s_tot[32];
  const int b = blockIdx.y;
  const int t0 = blockIdx.x * CM_TT;
  const int C2 = C >> 1;
  const int cp = threadIdx.x;
  const bool ok = cp < C2;
  const int left = causal ? (K - 1) : (K - 1) / 2;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarps = blockDim.x >> 5;
  float b0 = 0.f, b1 = 0.f;
  float2 padv = make_float2(0.f, 0.f);
  if (ok) {
    b0 = __ldg(dw_b + 2 * cp);
    b1 = __ldg(dw_b + 2 * cp + 1);
    if (causal) padv = make_float2(__ldg(pad_glu + 2 * cp), __ldg(pad_glu + 2 * cp + 1));
  }
  float acc[CM_TT][2];
#pragma unroll
  for (int t = 0; t < CM_TT; ++t) {
    acc[t][0] = b0;
    acc[t][1] = b1;
  }
  const uint32_t* xb = reinterpret_cast<const uint32_t*>(x + (long long)b * T * C) + cp;
  constexpr int ROWS = CM_TT + K - 1;
  uint32_t rv[ROWS];
#pragma unroll
  for (int r = 0; r < ROWS; ++r) {
    const int t = t0 - left + r;
    rv[r] = 0u;
    if (ok && t >= 0 && t < T) rv[r] = __ldg(xb + (long long)t * C2);
  }
  float w0[K], w1[K];
#pragma unroll
  for (int k = 0; k < K; ++k) {
    w0[k] = ok ? __ldg(dw_w + (2 * cp) * K + k) : 0.f;
    w1[k] = ok ? __ldg(dw_w + (2 * cp + 1) * K + k) : 0.f;
  }
#pragma unroll
  for (int r = 0; r < ROWS; ++r) {
    const int tt = t0 - left + r;
    const float2 v = (tt < 0) ? padv : unpack_bf16x2(rv[r]);  // rv is 0 beyond T
#pragma unroll
    for (int k = 0; k < K; ++k) {
      const int t = r - k;  // compile-time after unrolling
      if (t >= 0 && t < CM_TT) {
        const float2 a2 = ffma2(make_float2(w0[k], w1[k]), v, make_float2(acc[t][0], acc[t][1]));
        acc[t][0] = a2.x;
        acc[t][1] = a2.y;
      }
    }
  }
  // per-frame sum / sum of squares over the CTA's channels
  static_assert(CM_TT == 16, "the statistics butterfly assumes 32 values per lane");
  float sv[32];
#pragma unroll
  for (int t = 0; t < CM_TT; ++t) {
    sv[t] = ok ? acc[t][0] + acc[t][1] : 0.f;
    sv[CM_TT + t] = ok ? acc[t][0] * acc[t][0] + acc[t][1] * acc[t][1] : 0.f;
  }
#pragma unroll
  for (int ofs = 16; ofs >= 1; ofs >>= 1) {
    const bool up = (lane & ofs) != 0;
#pragma unroll
    for (int i = 0; i < ofs; ++i) {
      const float send = up ? sv[i] : sv[i + ofs];
      const float keep = up ? sv[i + ofs] : sv[i];
      sv[i] = keep + __shfl_xor_sync(0xffffffffu, send, ofs);
    }
  }
  s_part[warp][lane] = sv[0];   // lane l: value l (l < 16: sum of frame l, l >= 16: sum of squares of frame l - 16)
  __syncthreads();
  if (threadIdx.x < 32) {
    float tot = 0.f;
    for (int w = 0; w < nwarps; ++w) tot += s_part[w][threadIdx.x];   // fixed order: bit-reproducible
    s_tot[threadIdx.x] = tot;
  }
  __syncthreads();
  if (!ok) return;
  const float g0 = __ldg(norm_w + 2 * cp), g1 = __ldg(norm_w + 2 * cp + 1);
  const float be0 = __ldg(norm_b + 2 * cp), be1 = __ldg(norm_b + 2 * cp + 1);
#pragma unroll
  for (int t = 0; t < CM_TT; ++t) {
    if (t0 + t >= T) break;
    const float mean = s_tot[t] / (float)C;
    const float var = fmaxf(s_tot[CM_TT + t] / (float)C - mean * mean, 0.f);
    const float rstd = rsqrtf(var + eps);
    const float y0 = (acc[t][0] - mean) * rstd * g0 + be0, y1 = (acc[t][1] - mean) * rstd * g1 + be1;
    reinterpret_cast<uint32_t*>(out + ((long long)b * T + t0 + t) * C)[cp] = pack_bf16x2(silu_f(y0), silu_f(y1));
  }
}

// y = SiLU(LN(conv_out)) with mean / variance from the accumulated (sum, sum of squares): one warp per frame
template <int NV, bool X3>
__global__ void __launch_bounds__(256)
conv_norm_silu_kernel(const float* __restrict__ conv_out, const float* __restrict__ stats, int nslice,
                      const float* __restrict__ gamma, const float* __restrict__ beta, float eps, long long M, int C,
                      bf16* __restrict__ out) {
  const long long row = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (row >= M) return;
  float sum = 0.f, sq = 0.f;
  for (int i = 0; i < nslice; ++i) {  // fixed order: bit-reproducible
    sum += stats[(row * nslice + i) * 2];
    sq += stats[(row * nslice + i) * 2 + 1];
  }
  const float mean = sum / (float)C;
  const float var = fmaxf(sq / (float)C - mean * mean, 0.f);
  const float rstd = rsqrtf(var + eps);
  const int nvec = C >> 2;
  const float4* xr = reinterpret_cast<const float4*>(conv_out + row * C);
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const int idx = lane + 32 * i;
    if (idx < nvec) {
      const float4 v = xr[idx];
      const float4 g = __ldg(reinterpret_cast<const float4*>(gamma) + idx);
      const float4 bb = __ldg(reinterpret_cast<const float4*>(beta) + idx);
      float4 y = make_float4((v.x - mean) * rstd * g.x + bb.x, (v.y - mean) * rstd * g.y + bb.y,
                             (v.z - mean) * rstd * g.z + bb.z, (v.w - mean) * rstd * g.w + bb.w);
      if constexpr (X3) {  // accurate mode: exact exp / division
        y = make_float4(y.x / (1.f + expf(-y.x)), y.y / (1.f + expf(-y.y)), y.z / (1.f + expf(-y.z)),
                        y.w / (1.f + expf(-y.w)));
      } else {
        y = make_float4(silu_f(y.x), silu_f(y.y), silu_f(y.z), silu_f(y.w));
      }
      store_pair4(out + row * C * (X3 ? 2 : 1), 4 * idx, C, X3, y);
    }
  }
}

int launch_conv_mid(const bf16* x, const float* pad_glu, const float* dw_w, const float* dw_b, const float* norm_w,
                    const float* norm_b, const float* bn_mean, const float* bn_var, int use_ln, float eps,
                    bf16* out, int B, int T, int C, int K, int causal, cudaStream_t stream, float* conv_tmp,
                    float* stats, int x3, int conv_chunk) {
  RVB_REQUIRE(C % 4 == 0 && C <= 4096 && K >= 1 && K <= 64, "conv_mid: unsupported C=%d K=%d", C, K);
  RVB_REQUIRE(!causal || pad_glu != nullptr, "conv_mid: causal mode needs the GLU(pointwise_conv1 bias) pad row");
  RVB_REQUIRE(!use_ln || (conv_tmp != nullptr && stats != nullptr), "conv_mid: LayerNorm needs the fp32 scratch");
  const int C2 = C / 2;
  dim3 grid((T + CM_TT - 1) / CM_TT, B, (C2 + 127) / 128);
  const int nslice = (int)grid.z;
#define RVB_DW(KK, XX)                                                                                                 \
  conv_dw_kernel<KK, XX><<<grid, 128, 0, stream>>>(x, pad_glu, dw_w, dw_b, norm_w, norm_b, bn_mean, bn_var, use_ln, eps, \
                                                   conv_tmp, stats, out, T, C, K, causal, conv_chunk)
  RVB_REQUIRE(conv_chunk <= 0 || !causal, "conv_mid: chunk-local convolution is the non-causal streaming mode");
  {
    // RVB_CONV_FUSED=1: the single-kernel variant (not the default): 512 threads x 98 registers leave one CTA per SM and
    // the three phases (taps, statistics, normalise) run back to back instead of overlapping across CTAs.  Kept as an
    // option; not timed on the H100.
    static int fused_sel = -1;
    if (fused_sel < 0) {
      const char* e = getenv("RVB_CONV_FUSED");
      fused_sel = (e && atoi(e) == 1) ? 1 : 0;
    }
    if (fused_sel && use_ln && !x3 && conv_chunk <= 0 && (K == 15 || K == 7) && C2 <= 512) {
      const int threads = ((C2 + 31) / 32) * 32;
      dim3 g1((T + CM_TT - 1) / CM_TT, B);
      if (K == 15)
        conv_dw_ln_fused_kernel<15><<<g1, threads, 0, stream>>>(x, pad_glu, dw_w, dw_b, norm_w, norm_b, eps, out, T, C, causal);
      else
        conv_dw_ln_fused_kernel<7><<<g1, threads, 0, stream>>>(x, pad_glu, dw_w, dw_b, norm_w, norm_b, eps, out, T, C, causal);
      RVB_COUNT_LAUNCH();
      RVB_CHECK_LAUNCH();
      return 0;
    }
  }
  if (x3) {  // accurate mode: the generic tap loop (no register-resident halo) is fast enough
    RVB_DW(0, true);
  } else if (conv_chunk > 0) {
    RVB_DW(0, false);
  } else if (K == 15) RVB_DW(15, false);
  else if (K == 31) RVB_DW(31, false);
  else if (K == 7) RVB_DW(7, false);
  else RVB_DW(0, false);
#undef RVB_DW
  RVB_COUNT_LAUNCH();
  RVB_CHECK_LAUNCH();
  if (use_ln) {
    const long long M = (long long)B * T;
    const int nv = (C / 4 + 31) / 32;
    const unsigned g2 = (unsigned)((M + 7) / 8);
#define RVB_CNS(NV)                                                                                                        \
  do {                                                                                                                    \
    if (x3) conv_norm_silu_kernel<NV, true><<<g2, 256, 0, stream>>>(conv_tmp, stats, nslice, norm_w, norm_b, eps, M, C, out);  \
    else conv_norm_silu_kernel<NV, false><<<g2, 256, 0, stream>>>(conv_tmp, stats, nslice, norm_w, norm_b, eps, M, C, out);    \
  } while (0)
    if (nv <= 1) RVB_CNS(1);
    else if (nv <= 2) RVB_CNS(2);
    else if (nv <= 4) RVB_CNS(4);
    else if (nv <= 8) RVB_CNS(8);
    else if (nv <= 16) RVB_CNS(16);
    else RVB_CNS(32);
#undef RVB_CNS
    RVB_COUNT_LAUNCH();
    RVB_CHECK_LAUNCH();
  }
  return 0;
}

// ---------------------------------------------------------------------------------------------------------------
__global__ void scale_cast_kernel(const float* __restrict__ x, float scale, float* __restrict__ of,
                                  bf16* __restrict__ ob, long long n) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (; i < n; i += stride) {
    float v = x[i] * scale;
    if (of) of[i] = v;
    if (ob) ob[i] = __float2bfloat16(v);
  }
}

int launch_scale_cast(const float* x, float scale, float* out_f32, bf16* out_bf16, long long n, cudaStream_t stream) {
  if (n <= 0) return 0;
  long long blocks = (n + 255) / 256;
  if (blocks > 132 * 16) blocks = 132 * 16;
  scale_cast_kernel<<<(int)blocks, 256, 0, stream>>>(x, scale, out_f32, out_bf16, n);
  RVB_COUNT_LAUNCH();
  RVB_CHECK_LAUNCH();
  return 0;
}

int launch_f32_to_bf16(const float* x, bf16* out, long long n, cudaStream_t stream) {
  return launch_scale_cast(x, 1.0f, nullptr, out, n, stream);
}

// (rows, width) fp32 -> the bf16 pair layout (rows, 2 * width) = [hi | lo] of the accurate mode
__global__ void f32_to_pair_kernel(const float* __restrict__ x, bf16* __restrict__ out, long long rows, int width) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long n = rows * width, stride = (long long)gridDim.x * blockDim.x;
  for (; i < n; i += stride) {
    const long long r = i / width;
    const int c = (int)(i - r * width);
    const float v = x[i];
    const bf16 h = __float2bfloat16(v);
    out[r * 2 * width + c] = h;
    out[r * 2 * width + width + c] = __float2bfloat16(v - __bfloat162float(h));
  }
}

int launch_f32_to_pair(const float* x, bf16* out, long long rows, int width, cudaStream_t stream) {
  const long long n = rows * width;
  if (n <= 0) return 0;
  long long blocks = (n + 255) / 256;
  if (blocks > 132 * 16) blocks = 132 * 16;
  f32_to_pair_kernel<<<(int)blocks, 256, 0, stream>>>(x, out, rows, width);
  RVB_COUNT_LAUNCH();
  RVB_CHECK_LAUNCH();
  return 0;
}

struct WSumPtrs {
  const float* p[8];
  float c[8];
};
__global__ void weighted_sum_kernel(WSumPtrs in, int n_in, long long n, bf16* __restrict__ ob, float* __restrict__ of) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (; i < n; i += stride) {
    // same association order as the reference: y = c0*L0(x); y = y + c1*L1(x); ...  (encoder_layer.py:378-390)
    float v = in.c[0] * in.p[0][i];
    for (int j = 1; j < n_in; ++j) v = v + in.c[j] * in.p[j][i];
    if (ob) ob[i] = __float2bfloat16(v);
    if (of) of[i] = v;
  }
}

int launch_weighted_sum_bf16(const float* const* ins, const float* coef, int n_in, long long n, bf16* out_bf16,
                             float* out_f32, cudaStream_t stream) {
  RVB_REQUIRE(n_in >= 1 && n_in <= 8, "weighted_sum: n_in=%d unsupported", n_in);
  WSumPtrs w;
  for (int i = 0; i < n_in; ++i) {
    w.p[i] = ins[i];
    w.c[i] = coef[i];
  }
  long long blocks = (n + 255) / 256;
  if (blocks > 132 * 16) blocks = 132 * 16;
  weighted_sum_kernel<<<(int)blocks, 256, 0, stream>>>(w, n_in, n, out_bf16, out_f32);
  RVB_COUNT_LAUNCH();
  RVB_CHECK_LAUNCH();
  return 0;
}

// sinusoidal positional table (transformer/embedding.py:39-56): pe[pos, 2i] = sin(pos * w_i), pe[pos, 2i+1] = cos(..)
__global__ void sinusoid_kernel(int T, int d, float nlod, float* __restrict__ of, bf16* __restrict__ ob) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)T * d) return;
  int pos = (int)(i / d), c = (int)(i - (long long)pos * d);
  int i2 = c & ~1;
  // torch: div_term = exp(arange(0, d, 2) * -(ln(10000)/d)) in fp32, then sin/cos(position * div_term) in fp32
  float div = expf((float)i2 * nlod);
  float ang = (float)pos * div;
  float v = (c & 1) ? cosf(ang) : sinf(ang);
  if (of) of[i] = v;
  if (ob) ob[i] = __float2bfloat16(v);
}

int launch_sinusoid(int T, int d, float* out_f32, bf16* out_bf16, cudaStream_t stream) {
  long long n = (long long)T * d;
  if (n <= 0) return 0;
  sinusoid_kernel<<<(int)((n + 255) / 256), 256, 0, stream>>>(T, d, (float)(-(log(10000.0) / (double)d)), out_f32,
                                                              out_bf16);
  RVB_COUNT_LAUNCH();
  RVB_CHECK_LAUNCH();
  return 0;
}

// decoder embedding + absolute positional encoding (transformer/decoder.py:147 `self.embed`,
// embedding.py:58-76: x * sqrt(d) + pe[:L])
__global__ void embed_posenc_kernel(const int* __restrict__ tok, const float* __restrict__ emb, int L, int d,
                                    float nlod, float* __restrict__ out, int pos0) {
  const int r = blockIdx.x;
  const int pos = pos0 + r % L;
  const int id = tok[r];
  const float xs = sqrtf((float)d);
  for (int c = threadIdx.x; c < d; c += blockDim.x) {
    int i2 = c & ~1;
    float div = expf((float)i2 * nlod);
    float ang = (float)pos * div;
    float pe = (c & 1) ? cosf(ang) : sinf(ang);
    out[(long long)r * d + c] = emb[(long long)id * d + c] * xs + pe;
  }
}

int launch_embed_posenc(const int* tokens, const float* emb, int N, int L, int d, float* out, cudaStream_t stream,
                        int pos0) {
  if (N * L <= 0) return 0;
  embed_posenc_kernel<<<N * L, 128, 0, stream>>>(tokens, emb, L, d, (float)(-(log(10000.0) / (double)d)), out, pos0);
  RVB_COUNT_LAUNCH();
  RVB_CHECK_LAUNCH();
  return 0;
}

__global__ void embed_posenc_rows_kernel(const int* __restrict__ tok, const int* __restrict__ posv,
                                         const float* __restrict__ emb, int d, float nlod, float* __restrict__ out) {
  const int r = blockIdx.x;
  const int pos = posv[r];
  const int id = tok[r];
  const float xs = sqrtf((float)d);
  for (int c = threadIdx.x; c < d; c += blockDim.x) {
    int i2 = c & ~1;
    float div = expf((float)i2 * nlod);
    float ang = (float)pos * div;
    float pe = (c & 1) ? cosf(ang) : sinf(ang);
    out[(long long)r * d + c] = emb[(long long)id * d + c] * xs + pe;
  }
}

int launch_embed_posenc_rows(const int* tokens, const int* pos, const float* emb, int R, int d, float* out,
                             cudaStream_t stream) {
  if (R <= 0) return 0;
  embed_posenc_rows_kernel<<<R, 128, 0, stream>>>(tokens, pos, emb, d, (float)(-(log(10000.0) / (double)d)), out);
  RVB_COUNT_LAUNCH();
  RVB_CHECK_LAUNCH();
  return 0;
}

// ---------------------------------------------------------------------------------------------------------------
// KV cache of the autoregressive decoder step (engine.cu decoder_cache_step; reference decoder.py:191-234 keeps the layer
// OUTPUTS of the previous positions and re-projects their keys / values each step — a key / value cache holds the
// same information with less work).  Rows are `width` bf16 wide ([k | v], or its hi/lo pair layout).
//   kv_append : cache[s, pos, 0..width) = kv[s, col0 .. col0 + width)   (kv: (S, ld); cache rows are row_stride wide)
//   kv_reorder: dst[s, 0..npos, :] = src[parent[s], 0..npos, :]   (beam reordering, torch.index_select in the reference)
__global__ void kv_append_kernel(const bf16* __restrict__ kv, long long ld, int col0, bf16* __restrict__ cache, int Lcap,
                                 int pos, int width, int row_stride) {
  const int s = blockIdx.x;
  const uint4* src = reinterpret_cast<const uint4*>(kv + (long long)s * ld + col0);
  uint4* dst = reinterpret_cast<uint4*>(cache + ((long long)s * Lcap + pos) * row_stride);
  for (int i = threadIdx.x; i < width / 8; i += blockDim.x) dst[i] = src[i];
}

int launch_kv_append(const bf16* kv, long long ld, int col0, bf16* cache, int S, int Lcap, int pos, int width,
                     int row_stride, cudaStream_t stream) {
  RVB_REQUIRE(width % 8 == 0 && ld % 8 == 0 && col0 % 8 == 0 && row_stride % 8 == 0, "kv_append: rows must be 16-byte aligned");
  if (S <= 0) return 0;
  kv_append_kernel<<<S, 128, 0, stream>>>(kv, ld, col0, cache, Lcap, pos, width, row_stride);
  RVB_COUNT_LAUNCH();
  RVB_CHECK_LAUNCH();
  return 0;
}

__global__ void kv_reorder_kernel(const bf16* __restrict__ src, bf16* __restrict__ dst, const int* __restrict__ parent,
                                  int Lcap, int npos, int width) {
  const int s = blockIdx.x, p = parent[s];
  const uint4* a = reinterpret_cast<const uint4*>(src + (long long)p * Lcap * width);
  uint4* b = reinterpret_cast<uint4*>(dst + (long long)s * Lcap * width);
  const long long n = (long long)npos * width / 8;
  for (long long i = threadIdx.x; i < n; i += blockDim.x) b[i] = a[i];
}

int launch_kv_reorder(const bf16* src, bf16* dst, const int* parent, int S, int Lcap, int npos, int width,
                      cudaStream_t stream) {
  if (S <= 0 || npos <= 0) return 0;
  kv_reorder_kernel<<<S, 256, 0, stream>>>(src, dst, parent, Lcap, npos, width);
  RVB_COUNT_LAUNCH();
  RVB_CHECK_LAUNCH();
  return 0;
}

__global__ void fill_int_kernel(int* p, int n, int v) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) p[i] = v;
}
int launch_fill_int(int* p, int n, int v, cudaStream_t stream) {
  if (n <= 0) return 0;
  fill_int_kernel<<<(n + 255) / 256, 256, 0, stream>>>(p, n, v);
  RVB_COUNT_LAUNCH();
  RVB_CHECK_LAUNCH();
  return 0;
}

}  // namespace rvb
