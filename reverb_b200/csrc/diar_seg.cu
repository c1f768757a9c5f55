// reverb_b200 — segmentation network of the diarization pipeline (PyanNet) on sm_90a, fp32.
//
// Replaces `pyannote.audio` `PyanNet.forward` behind `Pipeline.from_pretrained('Revai/reverb-diarization-v1')`
// (reference: diarization/infer_pyannote3.0.py:33-40).  ** parity unpinned ** — see include/rvb_diar.h.
//
//   waveform window (B, N) -> InstanceNorm1d(1) -> SincNet:  |sinc band-pass bank (80 x 251, stride 10)| -> MaxPool(3)
//   -> InstanceNorm -> LeakyReLU -> 2 x [Conv1d(k=5) -> MaxPool(3) -> InstanceNorm -> LeakyReLU]      (B, frames, 60)
//   -> 4 x bidirectional LSTM(128) -> 2 x [Linear(128) + LeakyReLU] -> Linear(classes) -> log_softmax
//
// Kernels (all fp32 — the whole network is 1.3 GMAC per 10 s window, small next to the ASR encoder):
//   wav_norm_kernel          one CTA per window, two-pass mean / variance
//   sinc_conv_pool_kernel    the filter bank in shared memory, thread = (pooled position, 20 filters), 60 accumulators
//   conv1d_pool_kernel       Conv1d(k=5) + bias + MaxPool(3): thread = (pooled position, 8 output channels)
//   inorm_lrelu_kernel       InstanceNorm (two-pass) + LeakyReLU, optional (B, L, C) transposed store for the LSTM
//   sgemm_bias_act_kernel    64x64x16 register-tiled fp32 GEMM (+bias, LeakyReLU): LSTM input projections, linears
//   lstm_rec_kernel          the recurrence: a CLUSTER OF TWO CTAs per (8 windows, direction); thread = one row of W_hh
//                            kept in 128 registers (the 256 KB matrix is exactly one SM-pair's worth of registers), h
//                            exchanged between the two CTAs through distributed shared memory, one cluster barrier per
//                            time step
//   logsoftmax_rows_kernel   log_softmax over the (7) classes
#include <math.h>
#include <string.h>

#include <algorithm>
#include <string>
#include <vector>

#include "../../include/rvb_diar.h"
#include "host_mem.h"
#include "kernels.h"

namespace rvb {

// ------------------------------------------------------------------------------------------------ small reductions
__device__ __forceinline__ float block_sum(float v, float* red) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
  v = warp_sum(v);
  __syncthreads();   // `red` may still be read from a previous call
  if (lane == 0) red[warp] = v;
  __syncthreads();
  float t = 0.f;
  for (int w = 0; w < nw; ++w) t += red[w];   // fixed order
  return t;
}

// y = (x - mean) / sqrt(var + eps) * w + b over each window (InstanceNorm1d(1, affine=True), biased variance)
__global__ void __launch_bounds__(1024)
wav_norm_kernel(const float* __restrict__ x, float* __restrict__ y, int N, float w, float b, float eps) {
  __shared__ float red[32];
  const float* xr = x + (size_t)blockIdx.x * N;
  float* yr = y + (size_t)blockIdx.x * N;
  float s = 0.f;
  for (int i = threadIdx.x; i < N; i += blockDim.x) s += xr[i];
  const float mean = block_sum(s, red) / (float)N;
  float q = 0.f;
  for (int i = threadIdx.x; i < N; i += blockDim.x) {
    const float d = xr[i] - mean;
    q += d * d;
  }
  const float rstd = rsqrtf(block_sum(q, red) / (float)N + eps);
  for (int i = threadIdx.x; i < N; i += blockDim.x) yr[i] = (xr[i] - mean) * rstd * w + b;
}

// out[b, f, p] = max_{q in 3p..3p+2} | sum_k filt[f, k] * x[b, stride*q + k] |
constexpr int SC_PT = 64;   // pooled positions per CTA
constexpr int SC_FG = 4;    // filter groups (threads = SC_PT * SC_FG)
template <int FPT>          // filters per thread (n_filters = SC_FG * FPT)
__global__ void __launch_bounds__(SC_PT * SC_FG)
sinc_conv_pool_kernel(const float* __restrict__ x, const float* __restrict__ filt, float* __restrict__ out, int N, int K,
                      int stride, int Lp) {
  extern __shared__ float sc_smem[];
  const int F = SC_FG * FPT;
  float* fs = sc_smem;            // [F][K]
  float* xs = fs + F * K;         // [span]
  const int b = blockIdx.y, p0 = blockIdx.x * SC_PT;
  const int span = (3 * SC_PT - 1) * stride + K;
  const float* xr = x + (size_t)b * N;
  const int x0 = 3 * p0 * stride;
  for (int i = threadIdx.x; i < F * K; i += blockDim.x) fs[i] = filt[i];
  for (int i = threadIdx.x; i < span; i += blockDim.x) xs[i] = (x0 + i < N) ? xr[x0 + i] : 0.f;
  __syncthreads();
  const int p = threadIdx.x % SC_PT, fg = threadIdx.x / SC_PT;
  float acc[FPT][3];
#pragma unroll
  for (int f = 0; f < FPT; ++f) acc[f][0] = acc[f][1] = acc[f][2] = 0.f;
  const float* xp = xs + 3 * p * stride;
  const float* fp = fs + (size_t)fg * FPT * K;
#pragma unroll 2
  for (int k = 0; k < K; ++k) {
    const float a0 = xp[k], a1 = xp[stride + k], a2 = xp[2 * stride + k];
#pragma unroll
    for (int f = 0; f < FPT; ++f) {
      const float w = fp[f * K + k];   // warp-uniform: broadcast
      acc[f][0] = fmaf(w, a0, acc[f][0]);
      acc[f][1] = fmaf(w, a1, acc[f][1]);
      acc[f][2] = fmaf(w, a2, acc[f][2]);
    }
  }
  if (p0 + p < Lp) {
#pragma unroll
    for (int f = 0; f < FPT; ++f)
      out[((size_t)b * F + fg * FPT + f) * Lp + p0 + p] = fmaxf(fmaxf(fabsf(acc[f][0]), fabsf(acc[f][1])), fabsf(acc[f][2]));
  }
}

// out[b, co, p] = max_{q in 3p..3p+2} ( bias[co] + sum_{ci, k} w[co, ci, k] * in[b, ci, q + k] ),  k < 5
constexpr int CP_PT = 32, CP_CG = 8, CP_K = 5;
__global__ void __launch_bounds__(CP_PT * CP_CG)
conv1d_pool_kernel(const float* __restrict__ in, const float* __restrict__ w, const float* __restrict__ bias,
                   float* __restrict__ out, int Cin, int Cout, int Lin, int Lp) {
  extern __shared__ float cp_smem[];   // [Cin][3*PT + K - 1 (+1 pad)]
  constexpr int ROW = 3 * CP_PT + CP_K - 1 + 1;
  const int b = blockIdx.y, p0 = blockIdx.x * CP_PT;
  const float* ib = in + (size_t)b * Cin * Lin;
  for (int i = threadIdx.x; i < Cin * ROW; i += blockDim.x) {
    const int ci = i / ROW, c = i - ci * ROW;
    const int l = 3 * p0 + c;
    cp_smem[i] = (c < ROW - 1 && l < Lin) ? ib[(size_t)ci * Lin + l] : 0.f;
  }
  __syncthreads();
  const int p = threadIdx.x % CP_PT, cg = threadIdx.x / CP_PT;
  constexpr int CPT = 8;   // output channels per thread
  float acc[CPT][3];
#pragma unroll
  for (int c = 0; c < CPT; ++c) acc[c][0] = acc[c][1] = acc[c][2] = 0.f;
  for (int ci = 0; ci < Cin; ++ci) {
    const float* xr = cp_smem + ci * ROW + 3 * p;
    float xv[CP_K + 2];
#pragma unroll
    for (int j = 0; j < CP_K + 2; ++j) xv[j] = xr[j];
#pragma unroll
    for (int c = 0; c < CPT; ++c) {
      const int co = cg * CPT + c;
      if (co < Cout) {   // warp-uniform
        const float* wr = w + ((size_t)co * Cin + ci) * CP_K;
#pragma unroll
        for (int k = 0; k < CP_K; ++k) {
          const float wv = __ldg(wr + k);
          acc[c][0] = fmaf(wv, xv[k], acc[c][0]);
          acc[c][1] = fmaf(wv, xv[k + 1], acc[c][1]);
          acc[c][2] = fmaf(wv, xv[k + 2], acc[c][2]);
        }
      }
    }
  }
  if (p0 + p < Lp) {
#pragma unroll
    for (int c = 0; c < CPT; ++c) {
      const int co = cg * CPT + c;
      if (co < Cout)
        out[((size_t)b * Cout + co) * Lp + p0 + p] = fmaxf(fmaxf(acc[c][0], acc[c][1]), acc[c][2]) + __ldg(bias + co);
    }
  }
}

// InstanceNorm1d(C, affine=True) over L (biased variance, eps) + LeakyReLU(0.01); in (B, C, L);
// out (B, C, L) or, transposed != 0, (B, L, C)
__global__ void __launch_bounds__(256)
inorm_lrelu_kernel(const float* __restrict__ in, const float* __restrict__ w, const float* __restrict__ bias,
                   float* __restrict__ out, int C, int L, float eps, int transposed) {
  __shared__ float red[32];
  const int c = blockIdx.x, b = blockIdx.y;
  const float* xr = in + ((size_t)b * C + c) * L;
  float s = 0.f;
  for (int i = threadIdx.x; i < L; i += blockDim.x) s += xr[i];
  const float mean = block_sum(s, red) / (float)L;
  float q = 0.f;
  for (int i = threadIdx.x; i < L; i += blockDim.x) {
    const float d = xr[i] - mean;
    q += d * d;
  }
  const float rstd = rsqrtf(block_sum(q, red) / (float)L + eps);
  const float g = w[c] * rstd, be = bias[c];
  for (int i = threadIdx.x; i < L; i += blockDim.x) {
    float y = (xr[i] - mean) * g + be;
    y = y > 0.f ? y : 0.01f * y;
    if (transposed) out[((size_t)b * L + i) * C + c] = y;
    else out[((size_t)b * C + c) * L + i] = y;
  }
}

// C[m, n] = act( sum_k A[m, k] * W[n, k] + bias[n] ),  act: 0 none, 1 LeakyReLU(0.01).  fp32, 64x64x16 tiles.
__global__ void __launch_bounds__(256)
sgemm_bias_act_kernel(const float* __restrict__ A, int lda, const float* __restrict__ W, int ldw,
                      const float* __restrict__ bias, float* __restrict__ C, int ldc, int M, int N, int K, int act) {
  __shared__ float As[16][64 + 4];
  __shared__ float Ws[16][64 + 4];
  const int m0 = blockIdx.y * 64, n0 = blockIdx.x * 64;
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;   // 16 x 16 threads, 4 x 4 outputs each
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
  const int lr = threadIdx.x >> 2, lc = (threadIdx.x & 3) * 4;   // loader: row 0..63, k offset 0,4,8,12
  for (int k0 = 0; k0 < K; k0 += 16) {
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int k = k0 + lc + j;
      As[lc + j][lr] = (m0 + lr < M && k < K) ? A[(size_t)(m0 + lr) * lda + k] : 0.f;
      Ws[lc + j][lr] = (n0 + lr < N && k < K) ? W[(size_t)(n0 + lr) * ldw + k] : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < 16; ++k) {
      const float4 a = *reinterpret_cast<const float4*>(&As[k][ty * 4]);
      const float4 w = *reinterpret_cast<const float4*>(&Ws[k][tx * 4]);
      const float av[4] = {a.x, a.y, a.z, a.w}, wv[4] = {w.x, w.y, w.z, w.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], wv[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int m = m0 + ty * 4 + i;
    if (m >= M) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int n = n0 + tx * 4 + j;
      if (n >= N) continue;
      float v = acc[i][j] + (bias ? bias[n] : 0.f);
      if (act == 1) v = v > 0.f ? v : 0.01f * v;
      C[(size_t)m * ldc + n] = v;
    }
  }
}

int launch_sgemm(const float* A, int lda, const float* W, int ldw, const float* bias, float* C, int ldc, int M, int N,
                 int K, int act, cudaStream_t stream) {
  if (M <= 0 || N <= 0) return 0;
  dim3 grid((N + 63) / 64, (M + 63) / 64);
  sgemm_bias_act_kernel<<<grid, 256, 0, stream>>>(A, lda, W, ldw, bias, C, ldc, M, N, K, act);
  RVB_COUNT_LAUNCH();
  RVB_CHECK_LAUNCH();
  return 0;
}

// ------------------------------------------------------------------------------------------------ LSTM recurrence
// One layer, both directions.  G (B, T, 2 * 4H): input projections + both biases, forward gates [i f g o] x H first,
// then the reverse direction's.  Whh (2, 4H, H).  out (B, T, 2H): [h_forward | h_reverse] (PyTorch layout).
// Cluster (2 CTAs) = (LS_BT windows, direction): CTA rank c owns hidden units [c*H/2, (c+1)*H/2) of all four gates.
constexpr int LS_H = 128, LS_BT = 8, LS_THREADS = 256;
__device__ __forceinline__ float sigmoid_x(float x) { return 1.f / (1.f + expf(-x)); }   // exact exp (not __expf)

__global__ void __cluster_dims__(2, 1, 1) __launch_bounds__(LS_THREADS, 1)
lstm_rec_kernel(const float* __restrict__ G, const float* __restrict__ Whh, float* __restrict__ out, int B, int T) {
  __shared__ __align__(16) float hs[2][LS_BT][LS_H];       // h of the previous / current step, all units (both CTAs)
  __shared__ float gs[LS_BT][LS_THREADS];                   // this CTA's gate pre-activations
  const uint32_t rank = cluster_ctarank();
  const int dir = blockIdx.y;
  const int b0 = (blockIdx.x >> 1) * LS_BT;
  const int gate = threadIdx.x >> 6, ul = threadIdx.x & 63;
  const int unit = (int)rank * (LS_H / 2) + ul;
  const int row = gate * LS_H + unit;                       // row of W_hh / column of G for this thread
  float w[LS_H];
  {
    const float4* wr = reinterpret_cast<const float4*>(Whh + ((size_t)dir * 4 * LS_H + row) * LS_H);
#pragma unroll
    for (int k = 0; k < LS_H / 4; ++k) {
      const float4 v = __ldg(wr + k);
      w[4 * k] = v.x;
      w[4 * k + 1] = v.y;
      w[4 * k + 2] = v.z;
      w[4 * k + 3] = v.w;
    }
  }
  for (int i = threadIdx.x; i < 2 * LS_BT * LS_H; i += blockDim.x) (&hs[0][0][0])[i] = 0.f;
  // cell state of the (window, unit) pairs this thread finishes: pair id = threadIdx.x + 256 * q
  float cst[2] = {0.f, 0.f};
  // address of the peer CTA's hs through distributed shared memory
  uint32_t peer_hs;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(peer_hs) : "r"(smem_u32(&hs[0][0][0])), "r"(rank ^ 1u));
  cluster_sync_all();
  const size_t gld = (size_t)2 * 4 * LS_H;                  // G row length
  for (int s = 0; s < T; ++s) {
    const int t = dir ? T - 1 - s : s;
    const int cur = s & 1, nxt = cur ^ 1;
    float acc[LS_BT];
#pragma unroll
    for (int b = 0; b < LS_BT; ++b)
      acc[b] = (b0 + b < B) ? __ldg(G + ((size_t)(b0 + b) * T + t) * gld + (size_t)dir * 4 * LS_H + row) : 0.f;
#pragma unroll
    for (int k = 0; k < LS_H; k += 4) {
#pragma unroll
      for (int b = 0; b < LS_BT; ++b) {
        const float4 h4 = *reinterpret_cast<const float4*>(&hs[cur][b][k]);   // broadcast
        acc[b] = fmaf(w[k], h4.x, acc[b]);
        acc[b] = fmaf(w[k + 1], h4.y, acc[b]);
        acc[b] = fmaf(w[k + 2], h4.z, acc[b]);
        acc[b] = fmaf(w[k + 3], h4.w, acc[b]);
      }
    }
#pragma unroll
    for (int b = 0; b < LS_BT; ++b) gs[b][threadIdx.x] = acc[b];
    __syncthreads();
#pragma unroll
    for (int q = 0; q < 2; ++q) {
      const int pid = threadIdx.x + LS_THREADS * q;
      const int b = pid >> 6, u = pid & 63;
      const float ig = sigmoid_x(gs[b][u]), fg = sigmoid_x(gs[b][64 + u]);
      const float gg = tanhf(gs[b][128 + u]), og = sigmoid_x(gs[b][192 + u]);
      cst[q] = fg * cst[q] + ig * gg;
      const float h = og * tanhf(cst[q]);
      const int hu = (int)rank * (LS_H / 2) + u;
      hs[nxt][b][hu] = h;
      const uint32_t off = (uint32_t)(((nxt * LS_BT + b) * LS_H + hu) * sizeof(float));
      asm volatile("st.shared::cluster.f32 [%0], %1;" ::"r"(peer_hs + off), "f"(h) : "memory");
      if (b0 + b < B) out[((size_t)(b0 + b) * T + t) * (2 * LS_H) + dir * LS_H + hu] = h;
    }
    cluster_sync_all();   // both halves of h(nxt) are in both CTAs; gs may be overwritten
  }
}

__global__ void logsoftmax_rows_kernel(const float* __restrict__ x, float* __restrict__ y, long long rows, int C) {
  const long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= rows) return;
  const float* xr = x + r * C;
  float m = -INFINITY;
  for (int c = 0; c < C; ++c) m = fmaxf(m, xr[c]);
  float s = 0.f;
  for (int c = 0; c < C; ++c) s += expf(xr[c] - m);
  const float l = m + logf(s);
  for (int c = 0; c < C; ++c) y[r * C + c] = xr[c] - l;
}

}  // namespace rvb

// =====================================================================================================================
struct rvb_seg_model {
  rvb_seg_config cfg;
  bool finalized = false;
  rvb::WeightStore store{"rvb_seg_finalize:"};
  float wav_w = 1.f, wav_b = 0.f;
  float* filt = nullptr;
  float* norm_w[3] = {nullptr, nullptr, nullptr};
  float* norm_b[3] = {nullptr, nullptr, nullptr};
  float* conv_w[2] = {nullptr, nullptr};
  float* conv_b[2] = {nullptr, nullptr};
  std::vector<float*> wih, whh, lbias;   // per layer: (2*4H, in), (2, 4H, H), (2*4H)
  std::vector<float*> lin_w, lin_b;
  float* cls_w = nullptr;
  float* cls_b = nullptr;
  rvb::DevBuf ws_a, ws_b, ws_g, ws_h0, ws_h1;
};

namespace rvb {

// ParamSincFB.filters() (asteroid-filterbanks): cosine and sine band-pass filters with a mirrored half Hamming window
static void sinc_filter_bank(const std::vector<float>& low_hz_, const std::vector<float>& band_hz_, int kernel,
                             double sample_rate, std::vector<float>* out) {
  const int C = (int)low_hz_.size(), half = kernel / 2;
  const double min_low = 50.0, min_band = 50.0;
  out->assign((size_t)2 * C * kernel, 0.f);
  std::vector<double> window(half), n_(half);
  for (int i = 0; i < half; ++i) {
    const double lin = (half > 1) ? (double)i * (kernel / 2.0 - 1.0) / (double)(half - 1) : 0.0;   // linspace(0, K/2-1, half)
    window[i] = 0.54 - 0.46 * cos(2.0 * M_PI * lin / (double)kernel);
    n_[i] = 2.0 * M_PI * (double)(i - half) / sample_rate;
  }
  for (int c = 0; c < C; ++c) {
    const double low = min_low + fabs((double)low_hz_[c]);
    double high = low + min_band + fabs((double)band_hz_[c]);
    if (high < min_low) high = min_low;
    if (high > sample_rate / 2) high = sample_rate / 2;
    const double band = high - low;
    float* fc = out->data() + (size_t)c * kernel;
    float* fsn = out->data() + (size_t)(C + c) * kernel;
    for (int i = 0; i < half; ++i) {
      const double l = ((sin(high * n_[i]) - sin(low * n_[i])) / (n_[i] / 2.0)) * window[i] / (2.0 * band);
      const double r = ((cos(low * n_[i]) - cos(high * n_[i])) / (n_[i] / 2.0)) * window[i] / (2.0 * band);
      fc[i] = (float)l;
      fc[kernel - 1 - i] = (float)l;
      fsn[i] = (float)r;
      fsn[kernel - 1 - i] = (float)(-r);
    }
    fc[half] = (float)(2.0 * band / (2.0 * band));
    fsn[half] = 0.f;
  }
}

static int seg_frames(const rvb_seg_config& c, int num_samples, int* l1, int* l2, int* l3) {
  int n = (num_samples - c.sinc_kernel) / c.sinc_stride + 1;
  if (num_samples < c.sinc_kernel) n = 0;
  const int a = n / 3;
  const int b = (a - (c.conv_kernel - 1)) > 0 ? (a - (c.conv_kernel - 1)) / 3 : 0;
  const int d = (b - (c.conv_kernel - 1)) > 0 ? (b - (c.conv_kernel - 1)) / 3 : 0;
  if (l1) *l1 = a;
  if (l2) *l2 = b;
  if (l3) *l3 = d;
  return d;
}

}  // namespace rvb

RVB_API rvb_seg_model* rvb_seg_create(const rvb_seg_config* cfg) {
  if (!cfg) {
    rvb::set_error("rvb_seg_create: null config");
    return nullptr;
  }
  if (cfg->lstm_hidden != rvb::LS_H || cfg->conv_kernel != rvb::CP_K || cfg->sinc_filters % rvb::SC_FG != 0 ||
      cfg->sinc_filters / rvb::SC_FG != 20 || cfg->conv_channels > 64 || cfg->lstm_layers < 1 || cfg->num_classes < 1 ||
      cfg->linear_layers < 0 || cfg->sinc_kernel < 3 || (cfg->sinc_kernel & 1) == 0 || cfg->sinc_stride < 1) {
    rvb::set_error("rvb_seg_create: unsupported shape (built for 80 sinc filters, k=5 convolutions with <= 64 channels, "
                   "LSTM hidden 128)");
    return nullptr;
  }
  rvb_seg_model* m = new rvb_seg_model();
  m->cfg = *cfg;
  return m;
}

RVB_API int rvb_seg_set_tensor(rvb_seg_model* m, const char* name, const float* host, long long count) {
  RVB_REQUIRE(m && name && host && count > 0, "rvb_seg_set_tensor: bad arguments");
  RVB_REQUIRE(!m->finalized, "rvb_seg_set_tensor: model already finalized");
  m->store.set(name, host, (size_t)count);
  return 0;
}

RVB_API int rvb_seg_finalize(rvb_seg_model* m) {
  using namespace rvb;
  RVB_REQUIRE(m && !m->finalized, "rvb_seg_finalize: bad model");
  const rvb_seg_config& c = m->cfg;
  const std::vector<float>* t = nullptr;
  const std::vector<float>* t2 = nullptr;
  if (m->store.need("sincnet.wav_norm1d.weight", 1, &t)) return -1;
  m->wav_w = (*t)[0];
  if (m->store.need("sincnet.wav_norm1d.bias", 1, &t)) return -1;
  m->wav_b = (*t)[0];
  const int half = c.sinc_filters / 2;
  if (m->store.need("sincnet.conv1d.0.filterbank.low_hz_", half, &t) ||
      m->store.need("sincnet.conv1d.0.filterbank.band_hz_", half, &t2))
    return -1;
  std::vector<float> bank;
  sinc_filter_bank(*t, *t2, c.sinc_kernel, (double)c.sample_rate, &bank);
  if (m->store.upload(bank.data(), bank.size(), &m->filt)) return -1;
  const int nch[3] = {c.sinc_filters, c.conv_channels, c.conv_channels};
  for (int i = 0; i < 3; ++i) {
    const std::string p = "sincnet.norm1d." + std::to_string(i);
    if (m->store.need(p + ".weight", nch[i], &t) || m->store.upload(t->data(), t->size(), &m->norm_w[i])) return -1;
    if (m->store.need(p + ".bias", nch[i], &t) || m->store.upload(t->data(), t->size(), &m->norm_b[i])) return -1;
  }
  for (int i = 0; i < 2; ++i) {
    const std::string p = "sincnet.conv1d." + std::to_string(i + 1);
    const int cin = nch[i];
    if (m->store.need(p + ".weight", (size_t)c.conv_channels * cin * c.conv_kernel, &t) ||
        m->store.upload(t->data(), t->size(), &m->conv_w[i]))
      return -1;
    if (m->store.need(p + ".bias", c.conv_channels, &t) || m->store.upload(t->data(), t->size(), &m->conv_b[i]))
      return -1;
  }
  const int H = c.lstm_hidden;
  for (int l = 0; l < c.lstm_layers; ++l) {
    const int in = l == 0 ? c.conv_channels : 2 * H;
    std::vector<float> wih((size_t)2 * 4 * H * in), whh((size_t)2 * 4 * H * H), bias((size_t)2 * 4 * H);
    for (int d = 0; d < 2; ++d) {
      const std::string sfx = "_l" + std::to_string(l) + (d ? "_reverse" : "");
      if (m->store.need("lstm.weight_ih" + sfx, (size_t)4 * H * in, &t)) return -1;
      memcpy(wih.data() + (size_t)d * 4 * H * in, t->data(), t->size() * sizeof(float));
      if (m->store.need("lstm.weight_hh" + sfx, (size_t)4 * H * H, &t)) return -1;
      memcpy(whh.data() + (size_t)d * 4 * H * H, t->data(), t->size() * sizeof(float));
      if (m->store.need("lstm.bias_ih" + sfx, (size_t)4 * H, &t) ||
          m->store.need("lstm.bias_hh" + sfx, (size_t)4 * H, &t2))
        return -1;
      for (int i = 0; i < 4 * H; ++i) bias[(size_t)d * 4 * H + i] = (*t)[i] + (*t2)[i];
    }
    float *a = nullptr, *b = nullptr, *cc = nullptr;
    if (m->store.upload(wih.data(), wih.size(), &a) || m->store.upload(whh.data(), whh.size(), &b) ||
        m->store.upload(bias.data(), bias.size(), &cc))
      return -1;
    m->wih.push_back(a);
    m->whh.push_back(b);
    m->lbias.push_back(cc);
  }
  int in = 2 * H;
  for (int i = 0; i < c.linear_layers; ++i) {
    const std::string p = "linear." + std::to_string(i);
    float *a = nullptr, *b = nullptr;
    if (m->store.need(p + ".weight", (size_t)c.linear_dim * in, &t) || m->store.upload(t->data(), t->size(), &a))
      return -1;
    if (m->store.need(p + ".bias", c.linear_dim, &t) || m->store.upload(t->data(), t->size(), &b)) return -1;
    m->lin_w.push_back(a);
    m->lin_b.push_back(b);
    in = c.linear_dim;
  }
  if (m->store.need("classifier.weight", (size_t)c.num_classes * in, &t) ||
      m->store.upload(t->data(), t->size(), &m->cls_w))
    return -1;
  if (m->store.need("classifier.bias", c.num_classes, &t) || m->store.upload(t->data(), t->size(), &m->cls_b))
    return -1;
  m->store.drop_host();
  m->finalized = true;
  return 0;
}

RVB_API void rvb_seg_destroy(rvb_seg_model* m) {
  if (!m) return;
  delete m;
}

RVB_API int rvb_seg_num_frames(const rvb_seg_model* m, int num_samples) {
  if (!m) return -1;
  return rvb::seg_frames(m->cfg, num_samples, nullptr, nullptr, nullptr);
}

RVB_API int rvb_seg_forward(rvb_seg_model* m, const float* d_wave, int B, int num_samples, float* d_logp,
                            float* d_sincnet, void* stream_) {
  using namespace rvb;
  cudaStream_t stream = (cudaStream_t)stream_;
  RVB_REQUIRE(m && m->finalized, "rvb_seg_forward: model not finalized");
  RVB_REQUIRE(d_wave && d_logp && B >= 0 && num_samples > 0, "rvb_seg_forward: bad arguments");
  if (B == 0) return 0;
  const rvb_seg_config& c = m->cfg;
  int L1 = 0, L2 = 0, L3 = 0;
  const int T = seg_frames(c, num_samples, &L1, &L2, &L3);
  RVB_REQUIRE(T > 0, "rvb_seg_forward: %d samples are too few for one output frame", num_samples);
  const int F = c.sinc_filters, Cc = c.conv_channels, H = c.lstm_hidden;
  const size_t big = std::max((size_t)B * num_samples, (size_t)B * F * L1);
  if (m->ws_a.ensure(big * sizeof(float)) || m->ws_b.ensure((size_t)B * F * L1 * sizeof(float)) ||
      m->ws_g.ensure((size_t)B * T * 8 * H * sizeof(float)) || m->ws_h0.ensure((size_t)B * T * 2 * H * sizeof(float)) ||
      m->ws_h1.ensure((size_t)B * T * 2 * H * sizeof(float)))
    return -1;
  float* a = m->ws_a.as<float>();
  float* b = m->ws_b.as<float>();
  // SincNet
  wav_norm_kernel<<<B, 1024, 0, stream>>>(d_wave, a, num_samples, m->wav_w, m->wav_b, 1e-5f);
  RVB_COUNT_LAUNCH();
  RVB_CHECK_LAUNCH();
  {
    const size_t smem = ((size_t)F * c.sinc_kernel + (size_t)(3 * SC_PT - 1) * c.sinc_stride + c.sinc_kernel) * sizeof(float);
    RVB_REQUIRE(smem <= 200 * 1024, "rvb_seg_forward: the sinc filter bank does not fit shared memory");
    static DynSmemOptIn optin;
    if (optin.ensure(sinc_conv_pool_kernel<20>, smem)) return -1;
    dim3 grid((L1 + SC_PT - 1) / SC_PT, B);
    sinc_conv_pool_kernel<20><<<grid, SC_PT * SC_FG, smem, stream>>>(a, m->filt, b, num_samples, c.sinc_kernel,
                                                                     c.sinc_stride, L1);
    RVB_COUNT_LAUNCH();
    RVB_CHECK_LAUNCH();
  }
  inorm_lrelu_kernel<<<dim3(F, B), 256, 0, stream>>>(b, m->norm_w[0], m->norm_b[0], a, F, L1, 1e-5f, 0);
  RVB_COUNT_LAUNCH();
  RVB_CHECK_LAUNCH();
  // a: (B, F, L1) -> conv -> b (B, Cc, L2) -> norm -> a -> conv -> b (B, Cc, L3) -> norm (transposed) -> h0 (B, T, Cc)
  const int cin[2] = {F, Cc}, lin[2] = {L1, L2}, lout[2] = {L2, L3};
  float* x_lstm = m->ws_h1.as<float>();   // (B, T, Cc) input of LSTM layer 0
  for (int i = 0; i < 2; ++i) {
    const size_t smem = (size_t)cin[i] * (3 * CP_PT + CP_K) * sizeof(float);
    static DynSmemOptIn optin;
    if (optin.ensure(conv1d_pool_kernel, smem)) return -1;
    dim3 grid((lout[i] + CP_PT - 1) / CP_PT, B);
    conv1d_pool_kernel<<<grid, CP_PT * CP_CG, smem, stream>>>(a, m->conv_w[i], m->conv_b[i], b, cin[i], Cc, lin[i], lout[i]);
    RVB_COUNT_LAUNCH();
    RVB_CHECK_LAUNCH();
    inorm_lrelu_kernel<<<dim3(Cc, B), 256, 0, stream>>>(b, m->norm_w[i + 1], m->norm_b[i + 1], i == 1 ? x_lstm : a, Cc,
                                                        lout[i], 1e-5f, i == 1 ? 1 : 0);
    RVB_COUNT_LAUNCH();
    RVB_CHECK_LAUNCH();
  }
  if (d_sincnet)
    RVB_CHECK_CUDA(cudaMemcpyAsync(d_sincnet, x_lstm, (size_t)B * T * Cc * sizeof(float), cudaMemcpyDeviceToDevice, stream));
  // LSTM stack
  const long long M = (long long)B * T;
  float* g = m->ws_g.as<float>();
  const float* xin = x_lstm;
  int in = Cc;
  float* hbuf[2] = {m->ws_h0.as<float>(), m->ws_h1.as<float>()};
  for (int l = 0; l < c.lstm_layers; ++l) {
    float* hout = hbuf[l & 1];   // layer 0 reads h1 (x_lstm) and writes h0, layer 1 reads h0 and writes h1, ...
    if (launch_sgemm(xin, in, m->wih[l], in, m->lbias[l], g, 8 * H, (int)M, 8 * H, in, 0, stream)) return -1;
    dim3 grid(2 * ((B + LS_BT - 1) / LS_BT), 2);
    lstm_rec_kernel<<<grid, LS_THREADS, 0, stream>>>(g, m->whh[l], hout, B, T);
    RVB_COUNT_LAUNCH();
    RVB_CHECK_LAUNCH();
    xin = hout;
    in = 2 * H;
  }
  // linear stack + classifier + log_softmax
  float* y0 = m->ws_a.as<float>();
  float* y1 = m->ws_b.as<float>();
  const float* cur = xin;
  for (int i = 0; i < c.linear_layers; ++i) {
    float* dst = (i & 1) ? y1 : y0;
    if (launch_sgemm(cur, in, m->lin_w[i], in, m->lin_b[i], dst, c.linear_dim, (int)M, c.linear_dim, in, 1, stream)) return -1;
    cur = dst;
    in = c.linear_dim;
  }
  float* logits = (cur == y0) ? y1 : y0;
  if (launch_sgemm(cur, in, m->cls_w, in, m->cls_b, logits, c.num_classes, (int)M, c.num_classes, in, 0, stream)) return -1;
  logsoftmax_rows_kernel<<<(unsigned)((M + 255) / 256), 256, 0, stream>>>(logits, d_logp, M, c.num_classes);
  RVB_COUNT_LAUNCH();
  RVB_CHECK_LAUNCH();
  return 0;
}
