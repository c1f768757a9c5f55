// reverb_b200 — speaker-embedding network of the diarization pipeline (WeSpeaker ResNet34) on sm_90a.
//
// Replaces `pyannote.audio` `WeSpeakerResNet34.forward(waveforms, weights)` behind
// `Pipeline.from_pretrained('Revai/reverb-diarization-v1')` (reference: diarization/infer_pyannote3.0.py:33-40).
// ** parity unpinned ** — see include/rvb_diar.h.
//
//   window in [-1, 1] -> x 2^15 -> Kaldi fbank (fbank.cu, hamming window) -> minus the mean over time
//   -> conv 3x3 (1 -> C) + BN + ReLU                                   direct kernel, fp32 input
//   -> 16 BasicBlocks: [conv 3x3 (stride s) + BN + ReLU, conv 3x3 + BN, (+ 1x1 stride-s conv + BN shortcut), add, ReLU]
//      every 3x3 / 1x1 convolution = im2col (bf16, NHWC, K ordered (kh, kw, c)) + the wgmma GEMM of gemm.cu with the
//      BatchNorm folded into its weights / bias and ReLU in its epilogue; the residual add reads the GEMM's fp32 output
//   -> weighted statistics pooling over time per (channel, frequency) -> Linear(embed_dim) in fp32
//
// Activations are bf16 NHWC (B, F', T', C): exactly the (M, N) row-major output of the GEMM, so no layout pass exists
// between layers.  The trunk runs once per window; S weight rows per window only repeat the pooling.
#include <math.h>
#include <string.h>

#include <algorithm>
#include <string>
#include <vector>

#include "../../include/rvb_diar.h"
#include "host_mem.h"
#include "kernels.h"

namespace rvb {

__global__ void scale_kernel(const float* __restrict__ x, float* __restrict__ y, long long n, float s) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (; i < n; i += stride) y[i] = x[i] * s;
}

// feats (B, T, F) -> x (B, F, T) = feats - mean over T (per window and mel bin); optionally the normalised (B, T, F) copy
__global__ void __launch_bounds__(256)
cmn_transpose_kernel(const float* __restrict__ feats, float* __restrict__ x, float* __restrict__ feats_out, int T, int F) {
  __shared__ float red[8];
  const int f = blockIdx.x, b = blockIdx.y;
  const float* fr = feats + (size_t)b * T * F + f;
  float s = 0.f;
  for (int t = threadIdx.x; t < T; t += blockDim.x) s += fr[(size_t)t * F];
  s = warp_sum(s);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  float tot = 0.f;
  for (int w = 0; w < 8; ++w) tot += red[w];
  const float mean = tot / (float)T;
  for (int t = threadIdx.x; t < T; t += blockDim.x) {
    const float v = fr[(size_t)t * F] - mean;
    x[((size_t)b * F + f) * T + t] = v;
    if (feats_out) feats_out[((size_t)b * T + t) * F + f] = v;
  }
}

// first convolution: x (B, H, W) fp32, w (C, 9) + bias (BN folded) -> out (B, H, W, C) bf16 = relu(conv3x3 pad 1)
template <int C>
__global__ void __launch_bounds__(256)
conv_in_kernel(const float* __restrict__ x, const float* __restrict__ w, const float* __restrict__ bias,
               bf16* __restrict__ out, int H, int W, long long total) {
  __shared__ float ws[C * 9 + C];
  for (int i = threadIdx.x; i < C * 9; i += blockDim.x) ws[i] = w[i];
  for (int i = threadIdx.x; i < C; i += blockDim.x) ws[C * 9 + i] = bias[i];
  __syncthreads();
  const long long m = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (m >= total) return;
  const int wo = (int)(m % W);
  const int ho = (int)((m / W) % H);
  const long long b = m / ((long long)W * H);
  float v[9];
#pragma unroll
  for (int kh = 0; kh < 3; ++kh)
#pragma unroll
    for (int kw = 0; kw < 3; ++kw) {
      const int h = ho + kh - 1, ww = wo + kw - 1;
      v[kh * 3 + kw] = (h >= 0 && h < H && ww >= 0 && ww < W) ? x[(b * H + h) * W + ww] : 0.f;
    }
  uint4* o = reinterpret_cast<uint4*>(out + m * C);
#pragma unroll
  for (int c8 = 0; c8 < C / 8; ++c8) {
    float r[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const int c = c8 * 8 + e;
      float a = ws[C * 9 + c];
#pragma unroll
      for (int k = 0; k < 9; ++k) a = fmaf(ws[c * 9 + k], v[k], a);
      r[e] = fmaxf(a, 0.f);
    }
    uint4 u;
    u.x = pack_bf16x2(r[0], r[1]);
    u.y = pack_bf16x2(r[2], r[3]);
    u.z = pack_bf16x2(r[4], r[5]);
    u.w = pack_bf16x2(r[6], r[7]);
    o[c8] = u;
  }
}

// im2col for a KSxKS convolution (pad = KS/2) with stride s on bf16 NHWC: out (B*Ho*Wo, KS*KS*C), k = (kh*KS + kw)*C + c.
// One thread per 8 channels of one tap.
__global__ void __launch_bounds__(256)
im2col_kernel(const bf16* __restrict__ in, bf16* __restrict__ out, int H, int W, int C, int Ho, int Wo, int KS, int stride,
              long long total) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int c8n = C >> 3;
  const int c8 = (int)(i % c8n);
  const int tap = (int)((i / c8n) % (KS * KS));
  const long long m = i / ((long long)c8n * KS * KS);
  const int wo = (int)(m % Wo);
  const int ho = (int)((m / Wo) % Ho);
  const long long b = m / ((long long)Wo * Ho);
  const int kh = tap / KS, kw = tap - kh * KS, pad = KS / 2;
  const int h = ho * stride + kh - pad, w = wo * stride + kw - pad;
  uint4 v = make_uint4(0u, 0u, 0u, 0u);
  if (h >= 0 && h < H && w >= 0 && w < W) v = *reinterpret_cast<const uint4*>(in + ((b * H + h) * W + w) * C + c8 * 8);
  *reinterpret_cast<uint4*>(out + (m * KS * KS + tap) * C + c8 * 8) = v;
}

// out = bf16(relu(y + shortcut)),  y fp32 (the second convolution of a block), shortcut bf16
__global__ void __launch_bounds__(256)
add_relu_kernel(const float* __restrict__ y, const bf16* __restrict__ sc, bf16* __restrict__ out, long long n8) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n8) return;
  const float4 a = reinterpret_cast<const float4*>(y)[2 * i], b = reinterpret_cast<const float4*>(y)[2 * i + 1];
  const uint4 s = reinterpret_cast<const uint4*>(sc)[i];
  const float2 s0 = unpack_bf16x2(s.x), s1 = unpack_bf16x2(s.y), s2 = unpack_bf16x2(s.z), s3 = unpack_bf16x2(s.w);
  uint4 u;
  u.x = pack_bf16x2(fmaxf(a.x + s0.x, 0.f), fmaxf(a.y + s0.y, 0.f));
  u.y = pack_bf16x2(fmaxf(a.z + s1.x, 0.f), fmaxf(a.w + s1.y, 0.f));
  u.z = pack_bf16x2(fmaxf(b.x + s2.x, 0.f), fmaxf(b.y + s2.y, 0.f));
  u.w = pack_bf16x2(fmaxf(b.z + s3.x, 0.f), fmaxf(b.w + s3.y, 0.f));
  reinterpret_cast<uint4*>(out)[i] = u;
}

// Weighted statistics pooling (pyannote StatsPool): act (B, Fq, T, C) bf16; feature j = c * Fq + f;
// weights (B, S, Tw) nearest-interpolated to T (source index floor(t * Tw / T)) or all ones.
// stats[(b*S + s), j] = mean, stats[.., C*Fq + j] = std with
//   v1 = sum w (+1e-8), mean = sum w x / v1, var = sum w (x - mean)^2 / (v1 - sum w^2 / v1 + 1e-8)
__global__ void __launch_bounds__(256)
stats_pool_kernel(const bf16* __restrict__ act, const float* __restrict__ weights, float* __restrict__ stats, int S, int Fq,
                  int T, int C, int Tw) {
  extern __shared__ float wsm[];   // [T]
  const int s = blockIdx.x % S, b = blockIdx.x / S;
  float v1p = 0.f, v2p = 0.f;
  for (int t = threadIdx.x; t < T; t += blockDim.x) {
    float w = 1.f;
    if (weights) {
      // F.interpolate(mode="nearest"): source index floor(dst * (in / out)) in float arithmetic
      const int src = min((int)floorf((float)t * ((float)Tw / (float)T)), Tw - 1);
      w = weights[((size_t)b * S + s) * Tw + src];
    }
    wsm[t] = w;
  }
  __syncthreads();
  for (int t = 0; t < T; ++t) {   // every thread sums the same T values in the same order
    v1p += wsm[t];
    v2p += wsm[t] * wsm[t];
  }
  const float v1 = v1p + 1e-8f, v2 = v2p;
  const float den = v1 - v2 / v1 + 1e-8f;
  const int D = C * Fq;
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    for (int f = 0; f < Fq; ++f) {
      const bf16* a = act + (((size_t)b * Fq + f) * T) * C + c;
      float m = 0.f;
      for (int t = 0; t < T; ++t) m = fmaf(wsm[t], __bfloat162float(a[(size_t)t * C]), m);
      m /= v1;
      float q = 0.f;
      for (int t = 0; t < T; ++t) {
        const float d = __bfloat162float(a[(size_t)t * C]) - m;
        q = fmaf(wsm[t] * d, d, q);
      }
      float* o = stats + ((size_t)b * S + s) * 2 * D;
      o[c * Fq + f] = m;
      o[D + c * Fq + f] = sqrtf(q / den);
    }
  }
}

struct ConvW {
  bf16* w = nullptr;    // (Cout, K) bf16, BN folded, K = ks*ks*Cin ordered (kh, kw, ci)
  float* b = nullptr;   // (Cout) folded BN bias
  int cin = 0, cout = 0, ks = 3, stride = 1;
};

}  // namespace rvb

struct rvb_emb_model {
  rvb_emb_config cfg;
  bool finalized = false;
  rvb::WeightStore store{"rvb_emb_finalize:"};
  float* in_w = nullptr;   // (C, 9) fp32, BN folded
  float* in_b = nullptr;
  struct Block {
    rvb::ConvW c1, c2, sc;
    bool has_sc = false;
  };
  std::vector<Block> blocks;
  float* seg_w = nullptr;
  float* seg_b = nullptr;
  rvb::DevBuf ws_wave, ws_feat, ws_x, ws_a0, ws_a1, ws_a2, ws_col, ws_y, ws_stats;
};

namespace rvb {

// BatchNorm2d (eval) folded into the convolution before it: scale[c] = gamma / sqrt(var + eps), shift = beta - mean * scale
static int emb_bn(rvb_emb_model* m, const std::string& p, int C, std::vector<float>* scale, std::vector<float>* shift) {
  const std::vector<float>*g, *b, *mu, *var;
  if (m->store.need(p + ".weight", C, &g) || m->store.need(p + ".bias", C, &b) ||
      m->store.need(p + ".running_mean", C, &mu) || m->store.need(p + ".running_var", C, &var))
    return -1;
  scale->resize(C);
  shift->resize(C);
  for (int c = 0; c < C; ++c) {
    const float sc = (*g)[c] / sqrtf((*var)[c] + 1e-5f);
    (*scale)[c] = sc;
    (*shift)[c] = (*b)[c] - (*mu)[c] * sc;
  }
  return 0;
}
// conv weight (Cout, Cin, ks, ks) fp32 + BN -> bf16 (Cout, ks*ks*Cin) ordered (kh, kw, ci)
static int emb_conv(rvb_emb_model* m, const std::string& wname, const std::string& bnname, int cin, int cout, int ks,
                    int stride, ConvW* out) {
  const std::vector<float>* w;
  if (m->store.need(wname, (size_t)cout * cin * ks * ks, &w)) return -1;
  std::vector<float> scale, shift;
  if (emb_bn(m, bnname, cout, &scale, &shift)) return -1;
  const int K = ks * ks * cin;
  std::vector<bf16> packed((size_t)cout * K);
  for (int co = 0; co < cout; ++co)
    for (int ci = 0; ci < cin; ++ci)
      for (int kh = 0; kh < ks; ++kh)
        for (int kw = 0; kw < ks; ++kw)
          packed[(size_t)co * K + (kh * ks + kw) * cin + ci] =
              __float2bfloat16((*w)[(((size_t)co * cin + ci) * ks + kh) * ks + kw] * scale[co]);
  if (m->store.upload(packed.data(), packed.size(), &out->w) ||
      m->store.upload(shift.data(), shift.size(), &out->b))
    return -1;
  out->cin = cin;
  out->cout = cout;
  out->ks = ks;
  out->stride = stride;
  return 0;
}

static inline int conv_out(int n, int stride) { return (n - 1) / stride + 1; }   // 3x3 pad 1 (and 1x1 pad 0) with stride

// out (B*Ho*Wo, cout) = conv(in (B, H, W, cin)); bf16 output (+ReLU) or fp32 output (no activation)
static int emb_run_conv(rvb_emb_model* m, const ConvW& cw, const bf16* in, int B, int H, int W, bool relu, bf16* out_bf16,
                        float* out_f32, cudaStream_t stream) {
  const int Ho = conv_out(H, cw.stride), Wo = conv_out(W, cw.stride);
  const long long M = (long long)B * Ho * Wo;
  const int K = cw.ks * cw.ks * cw.cin;
  const bf16* A = in;
  if (!(cw.ks == 1 && cw.stride == 1)) {
    if (m->ws_col.ensure((size_t)M * K * sizeof(bf16))) return -1;
    const long long total = M * cw.ks * cw.ks * (cw.cin / 8);
    im2col_kernel<<<(unsigned)((total + 255) / 256), 256, 0, stream>>>(in, m->ws_col.as<bf16>(), H, W, cw.cin, Ho, Wo, cw.ks,
                                                                      cw.stride, total);
    RVB_COUNT_LAUNCH();
    RVB_CHECK_LAUNCH();
    A = m->ws_col.as<bf16>();
  }
  RVB_REQUIRE(M < (1ll << 31), "rvb_emb_forward: batch too large for one GEMM (M = %lld)", M);
  GemmArgs g;
  g.A = A;
  g.W = cw.w;
  g.M = (int)M;
  g.N = cw.cout;
  g.K = K;
  g.bias = cw.b;
  g.act = relu ? ACT_RELU : ACT_NONE;
  g.out_mode = out_bf16 ? OUT_BF16 : OUT_F32;
  g.out = out_bf16 ? (void*)out_bf16 : (void*)out_f32;
  return launch_gemm(g, stream);
}

}  // namespace rvb

RVB_API rvb_emb_model* rvb_emb_create(const rvb_emb_config* cfg) {
  if (!cfg) {
    rvb::set_error("rvb_emb_create: null config");
    return nullptr;
  }
  if (cfg->num_mel_bins != 80 || cfg->m_channels != 32 || cfg->embed_dim < 1 || cfg->sample_rate != 16000) {
    rvb::set_error("rvb_emb_create: unsupported shape (built for 16 kHz, 80 mel bins, m_channels 32)");
    return nullptr;
  }
  for (int i = 0; i < 4; ++i)
    if (cfg->blocks[i] < 1) {
      rvb::set_error("rvb_emb_create: every ResNet stage needs at least one block");
      return nullptr;
    }
  rvb_emb_model* m = new rvb_emb_model();
  m->cfg = *cfg;
  return m;
}

RVB_API int rvb_emb_set_tensor(rvb_emb_model* m, const char* name, const float* host, long long count) {
  RVB_REQUIRE(m && name && host && count > 0, "rvb_emb_set_tensor: bad arguments");
  RVB_REQUIRE(!m->finalized, "rvb_emb_set_tensor: model already finalized");
  m->store.set(name, host, (size_t)count);
  return 0;
}

RVB_API int rvb_emb_finalize(rvb_emb_model* m) {
  using namespace rvb;
  RVB_REQUIRE(m && !m->finalized, "rvb_emb_finalize: bad model");
  const rvb_emb_config& c = m->cfg;
  const int C0 = c.m_channels;
  {
    const std::vector<float>* w;
    if (m->store.need("resnet.conv1.weight", (size_t)C0 * 9, &w)) return -1;
    std::vector<float> scale, shift;
    if (emb_bn(m, "resnet.bn1", C0, &scale, &shift)) return -1;
    std::vector<float> wf((size_t)C0 * 9);
    for (int co = 0; co < C0; ++co)
      for (int k = 0; k < 9; ++k) wf[(size_t)co * 9 + k] = (*w)[(size_t)co * 9 + k] * scale[co];
    if (m->store.upload(wf.data(), wf.size(), &m->in_w) || m->store.upload(shift.data(), shift.size(), &m->in_b))
      return -1;
  }
  int cin = C0;
  for (int li = 0; li < 4; ++li) {
    const int cout = C0 << li;
    for (int bi = 0; bi < c.blocks[li]; ++bi) {
      const std::string p = "resnet.layer" + std::to_string(li + 1) + "." + std::to_string(bi);
      const int stride = (li > 0 && bi == 0) ? 2 : 1;
      rvb_emb_model::Block blk;
      if (emb_conv(m, p + ".conv1.weight", p + ".bn1", cin, cout, 3, stride, &blk.c1)) return -1;
      if (emb_conv(m, p + ".conv2.weight", p + ".bn2", cout, cout, 3, 1, &blk.c2)) return -1;
      blk.has_sc = (stride != 1 || cin != cout);
      if (blk.has_sc && emb_conv(m, p + ".shortcut.0.weight", p + ".shortcut.1", cin, cout, 1, stride, &blk.sc)) return -1;
      m->blocks.push_back(blk);
      cin = cout;
    }
  }
  const int Fq = conv_out(conv_out(conv_out(c.num_mel_bins, 2), 2), 2);
  const int D = cin * Fq;
  const std::vector<float>* t;
  if (m->store.need("resnet.seg_1.weight", (size_t)c.embed_dim * 2 * D, &t) ||
      m->store.upload(t->data(), t->size(), &m->seg_w))
    return -1;
  if (m->store.need("resnet.seg_1.bias", c.embed_dim, &t) || m->store.upload(t->data(), t->size(), &m->seg_b))
    return -1;
  m->store.drop_host();
  m->finalized = true;
  return 0;
}

RVB_API void rvb_emb_destroy(rvb_emb_model* m) {
  if (!m) return;
  delete m;
}

RVB_API int rvb_emb_num_frames(const rvb_emb_model* m, int num_samples) {
  if (!m) return -1;
  return num_samples < 400 ? 0 : 1 + (num_samples - 400) / 160;
}

RVB_API int rvb_emb_forward(rvb_emb_model* m, const float* d_wave, int B, int num_samples, const float* d_weights, int S,
                            int Tw, float* d_emb, float* d_fbank, void* stream_) {
  using namespace rvb;
  cudaStream_t stream = (cudaStream_t)stream_;
  RVB_REQUIRE(m && m->finalized, "rvb_emb_forward: model not finalized");
  RVB_REQUIRE(d_wave && d_emb && B >= 0 && num_samples > 0, "rvb_emb_forward: bad arguments");
  RVB_REQUIRE((d_weights == nullptr && S == 1) || (d_weights != nullptr && S >= 1 && Tw >= 1),
              "rvb_emb_forward: weights (B, S, Tw) or none with S = 1");
  if (B == 0) return 0;
  const rvb_emb_config& c = m->cfg;
  const int F = c.num_mel_bins, C0 = c.m_channels;
  const int T = rvb_emb_num_frames(m, num_samples);
  RVB_REQUIRE(T >= 8, "rvb_emb_forward: %d samples are too few", num_samples);
  const size_t act0 = (size_t)B * F * T * C0;   // elements of the largest activation (stage 1)
  if (m->ws_wave.ensure((size_t)B * num_samples * 4) || m->ws_feat.ensure((size_t)B * T * F * 4) ||
      m->ws_x.ensure((size_t)B * T * F * 4) || m->ws_a0.ensure(act0 * 2) || m->ws_a1.ensure(act0 * 2) ||
      m->ws_a2.ensure(act0 * 2) || m->ws_y.ensure(act0 * 4))
    return -1;
  // front-end
  {
    const long long n = (long long)B * num_samples;
    scale_kernel<<<(unsigned)std::min<long long>((n + 255) / 256, 132 * 16), 256, 0, stream>>>(d_wave, m->ws_wave.as<float>(), n,
                                                                                           32768.f);
    RVB_COUNT_LAUNCH();
    RVB_CHECK_LAUNCH();
    if (launch_fbank_batch(m->ws_wave.as<float>(), 0, B, num_samples, num_samples, m->ws_feat.as<float>(), T, stream, 1))
      return -1;
    cmn_transpose_kernel<<<dim3(F, B), 256, 0, stream>>>(m->ws_feat.as<float>(), m->ws_x.as<float>(), d_fbank, T, F);
    RVB_COUNT_LAUNCH();
    RVB_CHECK_LAUNCH();
  }
  bf16* cur = m->ws_a0.as<bf16>();
  bf16* tmp = m->ws_a1.as<bf16>();
  bf16* alt = m->ws_a2.as<bf16>();
  {
    const long long total = (long long)B * F * T;
    conv_in_kernel<32><<<(unsigned)((total + 255) / 256), 256, 0, stream>>>(m->ws_x.as<float>(), m->in_w, m->in_b, cur, F, T,
                                                                           total);
    RVB_COUNT_LAUNCH();
    RVB_CHECK_LAUNCH();
  }
  int H = F, W = T, C = C0;
  for (const auto& blk : m->blocks) {
    const int Ho = conv_out(H, blk.c1.stride), Wo = conv_out(W, blk.c1.stride);
    // y1 = relu(bn1(conv1(x)))
    if (emb_run_conv(m, blk.c1, cur, B, H, W, true, tmp, nullptr, stream)) return -1;
    // y2 = bn2(conv2(y1)) in fp32
    if (emb_run_conv(m, blk.c2, tmp, B, Ho, Wo, false, nullptr, m->ws_y.as<float>(), stream)) return -1;
    // shortcut
    const bf16* sc = cur;
    if (blk.has_sc) {
      if (emb_run_conv(m, blk.sc, cur, B, H, W, false, tmp, nullptr, stream)) return -1;   // tmp (y1) is free again
      sc = tmp;
    }
    const long long n8 = (long long)B * Ho * Wo * blk.c2.cout / 8;
    add_relu_kernel<<<(unsigned)((n8 + 255) / 256), 256, 0, stream>>>(m->ws_y.as<float>(), sc, alt, n8);
    RVB_COUNT_LAUNCH();
    RVB_CHECK_LAUNCH();
    std::swap(cur, alt);
    H = Ho;
    W = Wo;
    C = blk.c2.cout;
  }
  // pooling + embedding layer
  const int D = C * H;
  if (m->ws_stats.ensure((size_t)B * S * 2 * D * 4)) return -1;
  stats_pool_kernel<<<B * S, 256, (size_t)W * sizeof(float), stream>>>(cur, d_weights, m->ws_stats.as<float>(), S, H, W, C,
                                                                     d_weights ? Tw : 1);
  RVB_COUNT_LAUNCH();
  RVB_CHECK_LAUNCH();
  return launch_sgemm(m->ws_stats.as<float>(), 2 * D, m->seg_w, 2 * D, m->seg_b, d_emb, c.embed_dim, B * S, c.embed_dim, 2 * D,
                      0, stream);
}
