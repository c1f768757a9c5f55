// reverb_b200 — WavLM segmentation network of the diarization pipeline v2 (pyannote `SSeRiouSS` on WavLM Base), sm_90a.
//
// Replaces the segmentation model behind `Pipeline.from_pretrained('Revai/reverb-diarization-v2')`.  The WavLM part is
// torchaudio's `wavlm_base()` `extract_features` (extractor_mode "group_norm", post-LN transformer); the head after the
// softmax-weighted layer sum is PyanNet's (diar_seg.cu, SegHead).
//
//   waveform window (B, N) -> Conv1d(1, 512, 10, 5) -> GroupNorm(512, 512) -> GELU                conv0_stats + conv0_apply
//   -> 6 x [Conv1d(512, 512, k, 2) -> GELU], k = 3, 3, 3, 3, 2, 2          im2col rows + wgmma GEMM with the GELU epilogue
//   -> LayerNorm(512) -> Linear(512, 768)                                                  launch_layernorm + wgmma GEMM
//   -> x + GELU(Conv1d(768, 768, 128, pad 64, 16 groups))[:T]           16 x (im2col_pos + GEMM N = 48) + posconv_residual
//   -> LayerNorm(768)   (torchaudio builds the post-LN wavlm_base with Transformer.layer_norm_first = True: the
//                        transformer's LayerNorm runs once, before layer 0)
//   -> 12 x post-LN layer:  x = LN(x + out_proj(attn(x)));  x = LN(x + W2 GELU(W1 x))
//        attn: softmax(q k^T / 8 + gate[b,h,i] rb[h, j - i]), the 4th instantiation of attention_tc_kernel (MASK_RELB)
//        gate from the layer input (gate_kernel), rb from layer 0's rel_attn_embed (rel_bias_kernel, once per forward)
//   -> sum_l softmax(wav2vec_weights)_l x_l (fp32, accumulated as each layer finishes)  -> SegHead (LSTM, linears, ...)
//
// bf16 tensor-core operands; the residual stream, norms, softmax and accumulators are fp32.  Every window is computed
// on its own rows, so a window's output does not depend on the batch it runs in.
#include <math.h>
#include <string.h>

#include <algorithm>
#include <set>
#include <string>
#include <vector>

#include "../../include/rvb_diar.h"
#include "host_mem.h"
#include "kernels.h"

namespace rvb {

constexpr int WL_NCONV = 7;
constexpr int WL_KERNEL[WL_NCONV] = {10, 3, 3, 3, 3, 2, 2};
constexpr int WL_STRIDE[WL_NCONV] = {5, 2, 2, 2, 2, 2, 2};
constexpr int WL_C = 512;     // conv channels (built for this width)
constexpr int WL_DH = 64;     // head dim (the attention kernel's d_k)
constexpr int WL_MAX_BATCH = 32;   // windows per pass through the network

// ---------------------------------------------------------------------------------------------------- conv layer 0
// GroupNorm(512, 512) normalises each channel over the window's whole time axis.  The convolution is linear in the
// samples, so the statistics of channel c follow from the window's 10-sample patch moments: mean_c = w_c . m,
// var_c = w_c^T S w_c (m: mean patch, S: patch covariance, both fp64 over all frames).  No fp32 pre-norm tensor is
// written.  aff[b, c] = (gamma_c * rstd_c, beta_c - mean_c * gamma_c * rstd_c).
constexpr int C0_K = 10, C0_S = 5, C0_NQ = C0_K * (C0_K + 1) / 2;
__global__ void __launch_bounds__(256)
conv0_stats_kernel(const float* __restrict__ wave, int N, int T0, const float* __restrict__ w, const float* __restrict__ gn_w,
                   const float* __restrict__ gn_b, float eps, float2* __restrict__ aff) {
  __shared__ double red[8][C0_K + C0_NQ];
  __shared__ double mom[C0_K + C0_NQ];
  const int b = blockIdx.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const float* x = wave + (size_t)b * N;
  double s[C0_K], q[C0_NQ];
#pragma unroll
  for (int i = 0; i < C0_K; ++i) s[i] = 0.0;
#pragma unroll
  for (int i = 0; i < C0_NQ; ++i) q[i] = 0.0;
  for (int t = threadIdx.x; t < T0; t += blockDim.x) {
    double p[C0_K];
#pragma unroll
    for (int k = 0; k < C0_K; ++k) p[k] = (double)__ldg(x + (size_t)C0_S * t + k);
    int e = 0;
#pragma unroll
    for (int i = 0; i < C0_K; ++i) {
      s[i] += p[i];
#pragma unroll
      for (int j = 0; j <= i; ++j) q[e++] += p[i] * p[j];
    }
  }
#pragma unroll
  for (int i = 0; i < C0_K + C0_NQ; ++i) {
    double v = i < C0_K ? s[i] : q[i - C0_K];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if (lane == 0) red[warp][i] = v;
  }
  __syncthreads();
  for (int i = threadIdx.x; i < C0_K + C0_NQ; i += blockDim.x) {
    double v = 0.0;
    for (int wv = 0; wv < 8; ++wv) v += red[wv][i];   // fixed order
    mom[i] = v / (double)T0;
  }
  __syncthreads();
  for (int c = threadIdx.x; c < WL_C; c += blockDim.x) {
    double wc[C0_K], mean = 0.0;
#pragma unroll
    for (int k = 0; k < C0_K; ++k) {
      wc[k] = (double)__ldg(w + c * C0_K + k);
      mean += wc[k] * mom[k];
    }
    double var = 0.0;
    int e = 0;
#pragma unroll
    for (int i = 0; i < C0_K; ++i)
#pragma unroll
      for (int j = 0; j <= i; ++j, ++e) {
        const double cov = mom[C0_K + e] - mom[i] * mom[j];
        var += (i == j ? 1.0 : 2.0) * wc[i] * wc[j] * cov;
      }
    var = fmax(var, 0.0);
    const double a = (double)__ldg(gn_w + c) / sqrt(var + (double)eps);
    aff[(size_t)b * WL_C + c] = make_float2((float)a, (float)((double)__ldg(gn_b + c) - mean * a));
  }
}

// out (B, T0, 512) bf16 channels-last = GELU(conv(x) * a_c + b_c); CTA = (32 frames, window), thread = 2 channels
constexpr int C0_TT = 32;
__global__ void __launch_bounds__(256)
conv0_apply_kernel(const float* __restrict__ wave, int N, int T0, const float* __restrict__ w,
                   const float2* __restrict__ aff, bf16* __restrict__ out) {
  __shared__ float xs[C0_S * C0_TT + C0_K];
  const int b = blockIdx.y, t0 = blockIdx.x * C0_TT;
  const float* x = wave + (size_t)b * N;
  for (int i = threadIdx.x; i < C0_S * C0_TT + C0_K; i += blockDim.x) {
    const long long idx = (long long)C0_S * t0 + i;
    xs[i] = idx < N ? __ldg(x + idx) : 0.f;
  }
  float wr[2][C0_K];
  float2 af[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int c = threadIdx.x + 256 * h;
#pragma unroll
    for (int k = 0; k < C0_K; ++k) wr[h][k] = __ldg(w + c * C0_K + k);
    af[h] = __ldg(aff + (size_t)b * WL_C + c);
  }
  __syncthreads();
  const int nt = min(C0_TT, T0 - t0);
  for (int t = 0; t < nt; ++t) {
    bf16* orow = out + ((size_t)b * T0 + t0 + t) * WL_C;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float y = 0.f;
#pragma unroll
      for (int k = 0; k < C0_K; ++k) y = fmaf(wr[h][k], xs[C0_S * t + k], y);
      orow[threadIdx.x + 256 * h] = __float2bfloat16(gelu_erf(fmaf(y, af[h].x, af[h].y)));
    }
  }
}

// ---------------------------------------------------------------------------------------------------- conv layers 1-6
// im2col of a stride-2 conv on channels-last rows: row (b, t) of A is the contiguous slice [2t*C, (2t+k)*C) of window b
// (the weight is permuted to (out, tap, in) at finalize).  One thread copies 16 bytes.
__global__ void im2col_rows_kernel(const bf16* __restrict__ x, bf16* __restrict__ col, int B, int Tin, int Tout, int k) {
  const int vpr = k * WL_C / 8;   // uint4 per row
  const long long total = (long long)B * Tout * vpr;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / vpr;
    const int v = (int)(i - r * vpr);
    const int b = (int)(r / Tout), t = (int)(r - (long long)b * Tout);
    const uint4* src = reinterpret_cast<const uint4*>(x + ((size_t)b * Tin + 2 * t) * WL_C);
    reinterpret_cast<uint4*>(col)[i] = src[v];
  }
}

__global__ void bf16_to_f32_kernel(const bf16* __restrict__ x, float* __restrict__ y, long long n) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    y[i] = __bfloat162float(x[i]);
}

// ---------------------------------------------------------------------------------------------------- positional conv
// im2col of one group of the grouped conv: col[(b, t), k*Cg + i] = x[b, t + k - K/2, g*Cg + i] (zero outside the window)
__global__ void im2col_pos_kernel(const bf16* __restrict__ x, bf16* __restrict__ col, int B, int T, int D, int K, int Cg,
                                  int g) {
  const int vpg = Cg / 8;
  const int vpr = K * vpg;
  const long long total = (long long)B * T * vpr;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / vpr;
    const int v = (int)(i - r * vpr);
    const int k = v / vpg, iv = v - k * vpg;
    const int b = (int)(r / T), t = (int)(r - (long long)b * T);
    const int ts = t + k - K / 2;
    uint4 val = make_uint4(0u, 0u, 0u, 0u);
    if (ts >= 0 && ts < T) val = *reinterpret_cast<const uint4*>(x + ((size_t)b * T + ts) * D + g * Cg + iv * 8);
    reinterpret_cast<uint4*>(col)[i] = val;
  }
}

// x += GELU(conv) (fp32)
__global__ void posconv_residual_kernel(float* __restrict__ x, const float* __restrict__ conv, long long n) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    x[i] += gelu_erf(conv[i]);
}

// ---------------------------------------------------------------------------------------------------- relative bias
// torchaudio `WavLMSelfAttention._relative_positions_bucket` (bidirectional), float32 log and truncation as written there
__device__ __forceinline__ int rel_bucket(int d, int num_buckets, int max_distance) {
  const int nb = num_buckets / 2;
  int ret = d > 0 ? nb : 0;
  const int a = d < 0 ? -d : d;
  const int max_exact = nb / 2;
  if (a < max_exact) return ret + a;
  const float lg = logf((float)a / (float)max_exact) / (float)log((double)max_distance / (double)max_exact);
  const int large = max_exact + (int)(lg * (float)(nb - max_exact));
  return ret + min(large, nb - 1);
}

// rb[h, d + T - 1] = rel_attn_embed[bucket(d), h], d = j - i in [-(T-1), T-1]
__global__ void rel_bias_kernel(const float* __restrict__ emb, int H, int T, int num_buckets, int max_distance,
                                float* __restrict__ rb) {
  const int n = 2 * T - 1;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n * H; i += gridDim.x * blockDim.x) {
    const int h = i / n, e = i - h * n;
    rb[i] = __ldg(emb + rel_bucket(e - (T - 1), num_buckets, max_distance) * H + h);
  }
}

// ---------------------------------------------------------------------------------------------------- gate
// gate[(b*H + h)*T + t] = a (bb * const_h - 1) + 2,  (a, bb) = sigmoid(sum of the two 4-groups of lin(x[b, t, h]))
// with x the layer input split into H heads of 64.  One warp per (row, head); lane = 2 of the 64 elements.
__global__ void __launch_bounds__(256)
gate_kernel(const float* __restrict__ x, const float* __restrict__ lw /*(8, 64)*/, const float* __restrict__ lb /*(8)*/,
            const float* __restrict__ cst /*(H)*/, float* __restrict__ gate, int B, int T, int H) {
  const long long wid = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (wid >= (long long)B * T * H) return;
  const long long row = wid / H;
  const int h = (int)(wid - row * H);
  const float2 xv = *reinterpret_cast<const float2*>(x + row * (H * WL_DH) + h * WL_DH + 2 * lane);
  float o[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const float2 wv = __ldg(reinterpret_cast<const float2*>(lw + j * WL_DH) + lane);
    o[j] = warp_sum(xv.x * wv.x + xv.y * wv.y) + __ldg(lb + j);
  }
  if (lane == 0) {
    const float a = sigmoid_f(((o[0] + o[1]) + o[2]) + o[3]);
    const float bb = sigmoid_f(((o[4] + o[5]) + o[6]) + o[7]);
    const int b = (int)(row / T), t = (int)(row - (long long)b * T);
    gate[((long long)b * H + h) * T + t] = a * (bb * __ldg(cst + h) - 1.f) + 2.f;
  }
}

// acc = (first ? 0 : acc) + w * x
__global__ void layer_sum_kernel(float* __restrict__ acc, const float* __restrict__ x, float w, int first, long long n) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    acc[i] = (first ? 0.f : acc[i]) + w * x[i];
}

static unsigned grid_for(long long n, int threads = 256) {
  return (unsigned)std::min<long long>((n + threads - 1) / threads, 148LL * 32);
}

static void to_bf16_host(const float* src, size_t n, std::vector<bf16>* out) {
  out->resize(n);
  for (size_t i = 0; i < n; ++i) {
    const uint16_t h = f2bf(src[i]);
    memcpy(&(*out)[i], &h, 2);
  }
}

static int wavlm_frames(int n, int* lens /* WL_NCONV, optional */) {
  int L = n;
  for (int i = 0; i < WL_NCONV; ++i) {
    L = L >= WL_KERNEL[i] ? (L - WL_KERNEL[i]) / WL_STRIDE[i] + 1 : 0;
    if (lens) lens[i] = L;
  }
  return L;
}

}  // namespace rvb

// =====================================================================================================================
using rvb::bf16;

struct rvb_wavlm_seg_model {
  rvb_wavlm_seg_config cfg;
  bool finalized = false;
  std::set<std::string> names;   // every tensor name set_tensor accepts
  rvb::WeightStore store{"rvb_wavlm_seg_finalize:"};
  float *c0_w = nullptr, *gn_w = nullptr, *gn_b = nullptr;
  bf16* conv_w[rvb::WL_NCONV] = {};   // layers 1-6: (512, k * 512), (out, tap, in)
  float *fp_ln_w = nullptr, *fp_ln_b = nullptr, *fp_b = nullptr;
  bf16* fp_w = nullptr;
  bf16* pos_w = nullptr;              // (768, K * 48): row o = output channel, column k * 48 + i (weight norm folded)
  float* pos_b = nullptr;
  float *tln_w = nullptr, *tln_b = nullptr;   // encoder.transformer.layer_norm
  float* rel_emb = nullptr;           // (num_buckets, H)
  struct Layer {
    bf16 *in_w = nullptr, *out_w = nullptr, *ff1_w = nullptr, *ff2_w = nullptr;
    float *in_b = nullptr, *out_b = nullptr, *ff1_b = nullptr, *ff2_b = nullptr;
    float *gl_w = nullptr, *gl_b = nullptr, *gconst = nullptr;
    float *ln_w = nullptr, *ln_b = nullptr, *fln_w = nullptr, *fln_b = nullptr;
  };
  std::vector<Layer> layers;
  std::vector<float> layer_w;         // softmax(wav2vec_weights)
  rvb::SegHead head;
  rvb::DevBuf ws_c0, ws_c1, ws_col, ws_aff, ws_feat, ws_xa, ws_xb, ws_xbf, ws_qkv, ws_att, ws_ffn, ws_gate, ws_rb, ws_acc,
      ws_g, ws_h0, ws_h1, ws_y0, ws_y1;
};

namespace rvb {

static const char* kWavlmPrefix = "wav2vec.";

static void wavlm_names(const rvb_wavlm_seg_config& c, std::set<std::string>* out) {
  const std::string p = kWavlmPrefix;
  auto add = [&](const std::string& s) { out->insert(s); };
  add(p + "feature_extractor.conv_layers.0.conv.weight");
  add(p + "feature_extractor.conv_layers.0.layer_norm.weight");
  add(p + "feature_extractor.conv_layers.0.layer_norm.bias");
  for (int i = 1; i < WL_NCONV; ++i) add(p + "feature_extractor.conv_layers." + std::to_string(i) + ".conv.weight");
  for (const char* s : {"layer_norm.weight", "layer_norm.bias", "projection.weight", "projection.bias"})
    add(p + "encoder.feature_projection." + s);
  const std::string pc = p + "encoder.transformer.pos_conv_embed.conv.";
  for (const char* s : {"bias", "parametrizations.weight.original0", "parametrizations.weight.original1", "weight_g", "weight_v"})
    add(pc + s);
  add(p + "encoder.transformer.layer_norm.weight");
  add(p + "encoder.transformer.layer_norm.bias");
  for (int l = 0; l < c.num_layers; ++l) {
    const std::string q = p + "encoder.transformer.layers." + std::to_string(l) + ".";
    if (l == 0) add(q + "attention.rel_attn_embed.weight");
    for (const char* s : {"attention.gru_rel_pos_const", "attention.gru_rel_pos_linear.weight",
                          "attention.gru_rel_pos_linear.bias", "attention.attention.in_proj_weight",
                          "attention.attention.in_proj_bias", "attention.attention.out_proj.weight",
                          "attention.attention.out_proj.bias", "layer_norm.weight", "layer_norm.bias",
                          "feed_forward.intermediate_dense.weight", "feed_forward.intermediate_dense.bias",
                          "feed_forward.output_dense.weight", "feed_forward.output_dense.bias", "final_layer_norm.weight",
                          "final_layer_norm.bias"})
      add(q + s);
  }
  add("wav2vec_weights");
  for (int l = 0; l < c.lstm_layers; ++l)
    for (const char* d : {"", "_reverse"})
      for (const char* s : {"weight_ih", "weight_hh", "bias_ih", "bias_hh"})
        add(std::string("lstm.") + s + "_l" + std::to_string(l) + d);
  for (int i = 0; i < c.linear_layers; ++i) {
    add("linear." + std::to_string(i) + ".weight");
    add("linear." + std::to_string(i) + ".bias");
  }
  add("classifier.weight");
  add("classifier.bias");
}

static int up_f32(WeightStore& st, const std::string& name, size_t n, float** dst) {
  const std::vector<float>* t = nullptr;
  if (st.need(name, n, &t)) return -1;
  return st.upload(t->data(), n, dst);
}

static int up_bf16(WeightStore& st, const std::string& name, size_t n, bf16** dst) {
  const std::vector<float>* t = nullptr;
  if (st.need(name, n, &t)) return -1;
  std::vector<bf16> h;
  to_bf16_host(t->data(), n, &h);
  return st.upload(h.data(), n, dst);
}

static int gemm(const bf16* A, int lda, const bf16* W, const float* bias, int M, int N, int K, int act, int out_mode,
                void* out, int ldo, cudaStream_t stream) {
  GemmArgs g;
  g.A = A;
  g.W = W;
  g.M = M;
  g.N = N;
  g.K = K;
  g.lda = lda;
  g.bias = bias;
  g.act = act;
  g.out_mode = out_mode;
  g.out = out;
  g.ldo = ldo;
  return launch_gemm(g, stream);
}

}  // namespace rvb

RVB_API rvb_wavlm_seg_model* rvb_wavlm_seg_create(const rvb_wavlm_seg_config* cfg) {
  if (!cfg) {
    rvb::set_error("rvb_wavlm_seg_create: null config");
    return nullptr;
  }
  const rvb_wavlm_seg_config& c = *cfg;
  if (c.conv_channels != rvb::WL_C || c.num_heads < 1 || c.embed_dim != c.num_heads * rvb::WL_DH || c.embed_dim % 64 != 0 ||
      c.ffn_dim < 64 || c.ffn_dim % 64 != 0 || c.num_layers < 1 || c.pos_conv_kernel < 2 || (c.pos_conv_kernel & 1) ||
      c.pos_conv_groups < 1 || c.embed_dim % c.pos_conv_groups != 0 || (c.embed_dim / c.pos_conv_groups) % 8 != 0 ||
      c.num_buckets < 4 || c.max_distance <= c.num_buckets / 4 || c.lstm_hidden != 128 || c.lstm_layers < 1 ||
      c.num_classes < 1 || c.linear_layers < 0) {
    rvb::set_error("rvb_wavlm_seg_create: unsupported shape (built for 512 conv channels, 64-wide heads, an even "
                   "positional-conv kernel, LSTM hidden 128)");
    return nullptr;
  }
  rvb_wavlm_seg_model* m = new rvb_wavlm_seg_model();
  m->cfg = c;
  rvb::wavlm_names(c, &m->names);
  return m;
}

RVB_API int rvb_wavlm_seg_set_tensor(rvb_wavlm_seg_model* m, const char* name, const float* host, long long count) {
  RVB_REQUIRE(m && name && host && count > 0, "rvb_wavlm_seg_set_tensor: bad arguments");
  RVB_REQUIRE(!m->finalized, "rvb_wavlm_seg_set_tensor: model already finalized");
  RVB_REQUIRE(m->names.count(name), "rvb_wavlm_seg_set_tensor: unknown tensor '%s'", name);
  m->store.set(name, host, (size_t)count);
  return 0;
}

RVB_API int rvb_wavlm_seg_finalize(rvb_wavlm_seg_model* m) {
  using namespace rvb;
  RVB_REQUIRE(m && !m->finalized, "rvb_wavlm_seg_finalize: bad model");
  const rvb_wavlm_seg_config& c = m->cfg;
  WeightStore& st = m->store;
  const std::string p = kWavlmPrefix;
  const std::string fe = p + "feature_extractor.conv_layers.";
  const int D = c.embed_dim, H = c.num_heads, F = c.ffn_dim;
  if (up_f32(st, fe + "0.conv.weight", (size_t)WL_C * C0_K, &m->c0_w) ||
      up_f32(st, fe + "0.layer_norm.weight", WL_C, &m->gn_w) || up_f32(st, fe + "0.layer_norm.bias", WL_C, &m->gn_b))
    return -1;
  const std::vector<float>* t = nullptr;
  for (int i = 1; i < WL_NCONV; ++i) {
    const int k = WL_KERNEL[i];
    if (st.need(fe + std::to_string(i) + ".conv.weight", (size_t)WL_C * WL_C * k, &t)) return -1;
    std::vector<float> perm((size_t)WL_C * WL_C * k);   // (out, in, tap) -> (out, tap, in)
    for (int o = 0; o < WL_C; ++o)
      for (int ci = 0; ci < WL_C; ++ci)
        for (int j = 0; j < k; ++j) perm[((size_t)o * k + j) * WL_C + ci] = (*t)[((size_t)o * WL_C + ci) * k + j];
    std::vector<bf16> h;
    to_bf16_host(perm.data(), perm.size(), &h);
    if (st.upload(h.data(), h.size(), &m->conv_w[i])) return -1;
  }
  const std::string fp = p + "encoder.feature_projection.";
  if (up_f32(st, fp + "layer_norm.weight", WL_C, &m->fp_ln_w) || up_f32(st, fp + "layer_norm.bias", WL_C, &m->fp_ln_b) ||
      up_bf16(st, fp + "projection.weight", (size_t)D * WL_C, &m->fp_w) || up_f32(st, fp + "projection.bias", D, &m->fp_b))
    return -1;
  {
    // weight norm over dim 2: w[o, i, k] = g[k] v[o, i, k] / ||v[:, :, k]||
    const std::string pc = p + "encoder.transformer.pos_conv_embed.conv.";
    const int K = c.pos_conv_kernel, Cg = D / c.pos_conv_groups;
    const bool param = st.find(pc + "parametrizations.weight.original0") != nullptr;
    const std::vector<float>* g = nullptr;
    const std::vector<float>* v = nullptr;
    if (st.need(pc + (param ? "parametrizations.weight.original0" : "weight_g"), K, &g) ||
        st.need(pc + (param ? "parametrizations.weight.original1" : "weight_v"), (size_t)D * Cg * K, &v))
      return -1;
    std::vector<double> nrm(K, 0.0);
    for (size_t e = 0; e < v->size(); ++e) nrm[e % K] += (double)(*v)[e] * (double)(*v)[e];
    std::vector<float> w((size_t)D * K * Cg);
    for (int o = 0; o < D; ++o)
      for (int i = 0; i < Cg; ++i)
        for (int k = 0; k < K; ++k)
          w[((size_t)o * K + k) * Cg + i] =
              (float)((double)(*g)[k] * (double)(*v)[((size_t)o * Cg + i) * K + k] / sqrt(nrm[k]));
    std::vector<bf16> h;
    to_bf16_host(w.data(), w.size(), &h);
    if (st.upload(h.data(), h.size(), &m->pos_w) || up_f32(st, pc + "bias", D, &m->pos_b)) return -1;
  }
  if (up_f32(st, p + "encoder.transformer.layer_norm.weight", D, &m->tln_w) ||
      up_f32(st, p + "encoder.transformer.layer_norm.bias", D, &m->tln_b))
    return -1;
  for (int l = 0; l < c.num_layers; ++l) {
    const std::string q = p + "encoder.transformer.layers." + std::to_string(l) + ".";
    rvb_wavlm_seg_model::Layer L;
    if (l == 0 && up_f32(st, q + "attention.rel_attn_embed.weight", (size_t)c.num_buckets * H, &m->rel_emb)) return -1;
    if (up_bf16(st, q + "attention.attention.in_proj_weight", (size_t)3 * D * D, &L.in_w) ||
        up_f32(st, q + "attention.attention.in_proj_bias", (size_t)3 * D, &L.in_b) ||
        up_bf16(st, q + "attention.attention.out_proj.weight", (size_t)D * D, &L.out_w) ||
        up_f32(st, q + "attention.attention.out_proj.bias", D, &L.out_b) ||
        up_f32(st, q + "attention.gru_rel_pos_linear.weight", 8 * WL_DH, &L.gl_w) ||
        up_f32(st, q + "attention.gru_rel_pos_linear.bias", 8, &L.gl_b) ||
        up_f32(st, q + "attention.gru_rel_pos_const", H, &L.gconst) ||
        up_f32(st, q + "layer_norm.weight", D, &L.ln_w) || up_f32(st, q + "layer_norm.bias", D, &L.ln_b) ||
        up_bf16(st, q + "feed_forward.intermediate_dense.weight", (size_t)F * D, &L.ff1_w) ||
        up_f32(st, q + "feed_forward.intermediate_dense.bias", F, &L.ff1_b) ||
        up_bf16(st, q + "feed_forward.output_dense.weight", (size_t)D * F, &L.ff2_w) ||
        up_f32(st, q + "feed_forward.output_dense.bias", D, &L.ff2_b) ||
        up_f32(st, q + "final_layer_norm.weight", D, &L.fln_w) || up_f32(st, q + "final_layer_norm.bias", D, &L.fln_b))
      return -1;
    m->layers.push_back(L);
  }
  if (st.need("wav2vec_weights", c.num_layers, &t)) return -1;
  {
    double mx = -INFINITY, s = 0.0;
    for (float v : *t) mx = std::max(mx, (double)v);
    for (float v : *t) s += exp((double)v - mx);
    for (float v : *t) m->layer_w.push_back((float)(exp((double)v - mx) / s));
  }
  m->head.hidden = c.lstm_hidden;
  m->head.lstm_layers = c.lstm_layers;
  m->head.linear_layers = c.linear_layers;
  m->head.linear_dim = c.linear_dim;
  m->head.num_classes = c.num_classes;
  if (seg_head_load(st, D, &m->head)) return -1;
  st.drop_host();
  m->finalized = true;
  return 0;
}

RVB_API void rvb_wavlm_seg_destroy(rvb_wavlm_seg_model* m) { delete m; }

RVB_API int rvb_wavlm_seg_num_frames(const rvb_wavlm_seg_model* m, int num_samples) {
  if (!m) return -1;
  return rvb::wavlm_frames(num_samples, nullptr);
}

namespace rvb {

// windows [b0, b0 + B) of a call over Btot windows; d_layers is (layers, Btot, T, D)
static int wavlm_forward_part(rvb_wavlm_seg_model* m, const float* d_wave, int B, int Btot, int b0, int num_samples,
                              float* d_logp, float* d_conv, float* d_layers, cudaStream_t stream) {
  const rvb_wavlm_seg_config& c = m->cfg;
  int lens[WL_NCONV];
  const int T = wavlm_frames(num_samples, lens);
  const int D = c.embed_dim, H = c.num_heads, F = c.ffn_dim, K = c.pos_conv_kernel, G = c.pos_conv_groups, Cg = D / G;
  const long long M = (long long)B * T;
  const size_t c0 = (size_t)B * lens[0] * WL_C, c1 = (size_t)B * lens[1] * WL_C;
  const size_t col = std::max((size_t)B * lens[1] * 3 * WL_C, (size_t)M * K * Cg);
  const size_t hd = std::max(c.linear_dim, c.num_classes);
  if (m->ws_c0.ensure(c0 * 2) || m->ws_c1.ensure(c1 * 2) || m->ws_col.ensure(col * 2) ||
      m->ws_aff.ensure((size_t)B * WL_C * sizeof(float2)) || m->ws_feat.ensure((size_t)M * WL_C * 4) ||
      m->ws_xa.ensure((size_t)M * D * 4) || m->ws_xb.ensure((size_t)M * D * 4) || m->ws_xbf.ensure((size_t)M * D * 2) ||
      m->ws_qkv.ensure((size_t)M * 3 * D * 2) || m->ws_att.ensure((size_t)M * D * 2) ||
      m->ws_ffn.ensure((size_t)M * F * 2) || m->ws_gate.ensure((size_t)M * H * 4) ||
      m->ws_rb.ensure((size_t)H * (2 * T - 1) * 4) || m->ws_acc.ensure((size_t)M * D * 4) ||
      m->ws_g.ensure((size_t)M * 8 * c.lstm_hidden * 4) || m->ws_h0.ensure((size_t)M * 2 * c.lstm_hidden * 4) ||
      m->ws_h1.ensure((size_t)M * 2 * c.lstm_hidden * 4) || m->ws_y0.ensure((size_t)M * hd * 4) ||
      m->ws_y1.ensure((size_t)M * hd * 4))
    return -1;
  // ---- conv feature extractor
  bf16* cbuf[2] = {m->ws_c0.as<bf16>(), m->ws_c1.as<bf16>()};
  conv0_stats_kernel<<<B, 256, 0, stream>>>(d_wave, num_samples, lens[0], m->c0_w, m->gn_w, m->gn_b, 1e-5f,
                                            m->ws_aff.as<float2>());
  RVB_COUNT_LAUNCH();
  RVB_CHECK_LAUNCH();
  conv0_apply_kernel<<<dim3((lens[0] + C0_TT - 1) / C0_TT, B), 256, 0, stream>>>(d_wave, num_samples, lens[0], m->c0_w,
                                                                                 m->ws_aff.as<float2>(), cbuf[0]);
  RVB_COUNT_LAUNCH();
  RVB_CHECK_LAUNCH();
  bf16* colb = m->ws_col.as<bf16>();
  for (int i = 1; i < WL_NCONV; ++i) {
    const int k = WL_KERNEL[i];
    const long long rows = (long long)B * lens[i];
    im2col_rows_kernel<<<grid_for(rows * k * WL_C / 8), 256, 0, stream>>>(cbuf[(i - 1) & 1], colb, B, lens[i - 1], lens[i], k);
    RVB_COUNT_LAUNCH();
    RVB_CHECK_LAUNCH();
    if (gemm(colb, k * WL_C, m->conv_w[i], nullptr, (int)rows, WL_C, k * WL_C, ACT_GELU, OUT_BF16, cbuf[i & 1], WL_C, stream))
      return -1;
  }
  float* feat = m->ws_feat.as<float>();
  bf16_to_f32_kernel<<<grid_for(M * WL_C), 256, 0, stream>>>(cbuf[(WL_NCONV - 1) & 1], feat, M * WL_C);
  RVB_COUNT_LAUNCH();
  RVB_CHECK_LAUNCH();
  if (d_conv) RVB_CHECK_CUDA(cudaMemcpyAsync(d_conv, feat, (size_t)M * WL_C * 4, cudaMemcpyDeviceToDevice, stream));
  // ---- feature projection
  float* xa = m->ws_xa.as<float>();
  float* xb = m->ws_xb.as<float>();
  bf16* xbf = m->ws_xbf.as<bf16>();
  if (launch_layernorm(feat, m->fp_ln_w, m->fp_ln_b, 1e-5f, (int)M, WL_C, colb, nullptr, nullptr, 0, 0, stream) ||
      gemm(colb, WL_C, m->fp_w, m->fp_b, (int)M, D, WL_C, ACT_NONE, OUT_F32, xa, D, stream) ||
      launch_f32_to_bf16(xa, xbf, M * D, stream))
    return -1;
  // ---- positional conv: one GEMM per group (N = 48, K = 128 * 48) into xb, then x += GELU(xb)
  for (int g = 0; g < G; ++g) {
    im2col_pos_kernel<<<grid_for(M * K * Cg / 8), 256, 0, stream>>>(xbf, colb, B, T, D, K, Cg, g);
    RVB_COUNT_LAUNCH();
    RVB_CHECK_LAUNCH();
    if (gemm(colb, K * Cg, m->pos_w + (size_t)g * Cg * K * Cg, m->pos_b + g * Cg, (int)M, Cg, K * Cg, ACT_NONE, OUT_F32,
             xb + g * Cg, D, stream))
      return -1;
  }
  posconv_residual_kernel<<<grid_for(M * D), 256, 0, stream>>>(xa, xb, M * D);
  RVB_COUNT_LAUNCH();
  RVB_CHECK_LAUNCH();
  if (launch_layernorm(xa, m->tln_w, m->tln_b, 1e-5f, (int)M, D, xbf, xb, nullptr, 0, 0, stream)) return -1;
  std::swap(xa, xb);
  // ---- relative-position bias table, shared by all layers
  float* rb = m->ws_rb.as<float>();
  rel_bias_kernel<<<grid_for((long long)H * (2 * T - 1)), 256, 0, stream>>>(m->rel_emb, H, T, c.num_buckets, c.max_distance, rb);
  RVB_COUNT_LAUNCH();
  RVB_CHECK_LAUNCH();
  // ---- transformer layers (post-LN); xa holds the layer input / output, xb the mid-layer residual stream
  bf16* qkv = m->ws_qkv.as<bf16>();
  bf16* att = m->ws_att.as<bf16>();
  bf16* ffn = m->ws_ffn.as<bf16>();
  float* gate = m->ws_gate.as<float>();
  float* acc = m->ws_acc.as<float>();
  for (int l = 0; l < c.num_layers; ++l) {
    const rvb_wavlm_seg_model::Layer& L = m->layers[l];
    gate_kernel<<<(unsigned)((M * H * 32 + 255) / 256), 256, 0, stream>>>(xa, L.gl_w, L.gl_b, L.gconst, gate, B, T, H);
    RVB_COUNT_LAUNCH();
    RVB_CHECK_LAUNCH();
    if (gemm(xbf, D, L.in_w, L.in_b, (int)M, 3 * D, D, ACT_NONE, OUT_BF16, qkv, 3 * D, stream)) return -1;
    AttnTcArgs a;
    a.q = qkv;
    a.k = qkv + D;
    a.v = qkv + 2 * D;
    a.out = att;
    a.ldq = a.ldk = a.ldv = 3 * D;
    a.ldo = D;
    a.groups = B;
    a.Tq = a.Tk = T;
    a.H = H;
    a.dk = WL_DH;
    a.scale = 1.0f / sqrtf((float)WL_DH);
    a.gate = gate;
    a.rel_bias = rb;
    if (launch_attention_tc(a, stream)) return -1;
    GemmArgs o;
    o.A = att;
    o.W = L.out_w;
    o.M = (int)M;
    o.N = D;
    o.K = D;
    o.bias = L.out_b;
    o.out_mode = OUT_RESID_F32;
    o.out = xa;
    if (launch_gemm(o, stream)) return -1;
    if (launch_layernorm(xa, L.ln_w, L.ln_b, 1e-5f, (int)M, D, xbf, xb, nullptr, 0, 0, stream)) return -1;
    if (gemm(xbf, D, L.ff1_w, L.ff1_b, (int)M, F, D, ACT_GELU, OUT_BF16, ffn, F, stream)) return -1;
    o.A = ffn;
    o.W = L.ff2_w;
    o.K = F;
    o.bias = L.ff2_b;
    o.out = xb;
    if (launch_gemm(o, stream)) return -1;
    if (launch_layernorm(xb, L.fln_w, L.fln_b, 1e-5f, (int)M, D, xbf, xa, nullptr, 0, 0, stream)) return -1;
    layer_sum_kernel<<<grid_for(M * D), 256, 0, stream>>>(acc, xa, m->layer_w[l], l == 0, M * D);
    RVB_COUNT_LAUNCH();
    RVB_CHECK_LAUNCH();
    if (d_layers)
      RVB_CHECK_CUDA(cudaMemcpyAsync(d_layers + ((size_t)l * Btot + b0) * T * D, xa, (size_t)M * D * 4,
                                     cudaMemcpyDeviceToDevice, stream));
  }
  // ---- PyanNet's head on the weighted layer sum
  return seg_head_forward(m->head, acc, D, B, T, m->ws_g.as<float>(), m->ws_h0.as<float>(), m->ws_h1.as<float>(),
                          m->ws_y0.as<float>(), m->ws_y1.as<float>(), d_logp, stream);
}

}  // namespace rvb

RVB_API int rvb_wavlm_seg_forward(rvb_wavlm_seg_model* m, const float* d_wave, int B, int num_samples, float* d_logp,
                                  float* d_conv, float* d_layers, void* stream_) {
  using namespace rvb;
  RVB_REQUIRE(m && m->finalized, "rvb_wavlm_seg_forward: model not finalized");
  RVB_REQUIRE(d_wave && d_logp && B >= 0 && num_samples > 0, "rvb_wavlm_seg_forward: bad arguments");
  const int T = wavlm_frames(num_samples, nullptr);
  RVB_REQUIRE(T > 0, "rvb_wavlm_seg_forward: %d samples are too few for one output frame (400 needed)", num_samples);
  // Windows run WL_MAX_BATCH at a time: the workspace (about 100 MB per 10 s window) stays bounded, and a window's
  // result does not depend on the batch it is in.
  for (int b0 = 0; b0 < B; b0 += WL_MAX_BATCH) {
    const int nb = std::min(WL_MAX_BATCH, B - b0);
    if (wavlm_forward_part(m, d_wave + (size_t)b0 * num_samples, nb, B, b0, num_samples,
                           d_logp + (size_t)b0 * T * m->cfg.num_classes,
                           d_conv ? d_conv + (size_t)b0 * T * WL_C : nullptr, d_layers, (cudaStream_t)stream_))
      return -1;
  }
  return 0;
}

RVB_API int rvb_attention_tc_relbias(const void* d_q, const void* d_k, const void* d_v, void* d_out, int ldq, int ldk,
                                     int ldv, int ldo, int groups, int T, int H, const float* d_gate,
                                     const float* d_rel_bias, float scale, void* stream) {
  RVB_REQUIRE(d_gate && d_rel_bias, "rvb_attention_tc_relbias: gate and bias table are required");
  rvb::AttnTcArgs a;
  a.q = reinterpret_cast<const bf16*>(d_q);
  a.k = reinterpret_cast<const bf16*>(d_k);
  a.v = reinterpret_cast<const bf16*>(d_v);
  a.out = reinterpret_cast<bf16*>(d_out);
  a.ldq = ldq;
  a.ldk = ldk;
  a.ldv = ldv;
  a.ldo = ldo;
  a.groups = groups;
  a.Tq = a.Tk = T;
  a.H = H;
  a.dk = rvb::WL_DH;
  a.gate = d_gate;
  a.rel_bias = d_rel_bias;
  a.scale = scale;
  return rvb::launch_attention_tc(a, (cudaStream_t)stream);
}
