// reverb_b200 — the model plan: packed weights + workspace + the launch sequences of the encoder, CTC head and
// rescoring decoder, and the C ABI on top (include/rvb_b200.h).
//
// Reference call chain replaced here (all paths relative to asr/wenet/):
//   ASRModel._forward_encoder (transformer/asr_model.py:288) -> BaseEncoder.forward (transformer/encoder.py:117-149)
//     -> GlobalCMVN, Conv2dSubsampling4, RelPositionalEncoding, 18 x (LanguageSpecific)ConformerEncoderLayer, after_norm
//   ASRModel.ctc_logprobs (asr_model.py:318)                    -> rvb_ctc_topk
//   ASRModel.forward_attention_decoder (asr_model.py:868-978)   -> rvb_attention_rescoring
// Data layout in HBM: residual stream fp32 (B*T', d); every GEMM operand bf16, K-major; conv activations
// channels-last; weights packed once at rvb_model_finalize (fused QKV, permuted conv2 / embed weights, sqrt(d) folded
// into the embed linear, language-specific linears folded per call with the caller's cat_embs).
#include <math.h>
#include <stdarg.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <atomic>
#include <memory>
#include <string>
#include <vector>

#include "../../include/rvb_b200.h"
#include "host_mem.h"
#include "kernels.h"

namespace rvb {

// ---------------------------------------------------------------------------------------------------------------
static thread_local char g_err[1024] = "";
std::atomic<unsigned long long> g_launch_count{0};
void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
const char* last_error() { return g_err; }

struct Linear {  // bf16 weight (N, K) + fp32 bias (N) on device
  bf16* w = nullptr;
  float* b = nullptr;
  int N = 0, K = 0;
};
struct Norm {
  float* g = nullptr;
  float* b = nullptr;
};

struct EncLayer {
  Norm norm_ffm, norm_mha, norm_conv, norm_ff, norm_final;
  Linear ffm1, ffm2, ff1, ff2, qkv, out, pw1, pw2;  // pw1 rows interleaved for the GLU epilogue (load_linear_glu)
  float* pad_glu = nullptr;                          // (d) GLU(pointwise_conv1 bias): value of the causal pad frames
  float* pos_u = nullptr;
  float* pos_v = nullptr;
  float* dw_w = nullptr;  // (d, K)
  float* dw_b = nullptr;
  Norm cnorm;             // conv-module norm (LayerNorm or BatchNorm affine)
  float* bn_mean = nullptr;
  float* bn_var = nullptr;
  bool lsl = false;
  int lsl_idx = -1;                    // index among the encoder's LSL layers (LangStack)
  std::vector<float*> lang_w, lang_b;  // fp32 device copies of language_layers.{i}
};

struct DecLayer {
  Norm n1, n2, n3;
  float eps = 1e-5f;
  Linear qkv, so, cq, ckv, co, ff1, ff2;
  bool lsl = false;
  int lsl_idx = -1;  // index among the LSL layers of both decoders (LangStack)
  std::vector<float*> lang_w, lang_b;
};

struct SearchTicket;
struct DecCache;

// The folds of the distinct mixing vectors of a call, slot g for its group g, side by side for every LSL layer of the
// encoder (or of the decoders): weight (slots*d, d) — the (slots*d, 2d) pair layout in the accurate mode — and bias
// (slots*d), grow-only and sized exactly, slots = key.size().  key[g] is the vector slot g holds (empty: none), so a
// slot refolds only when its vector changes; growing reallocates the buffers and so empties every key.
struct LangStack {
  std::vector<DevBuf> w, b;             // by lsl_idx
  std::vector<std::vector<float>> key;  // by slot
};

// The language-specific mixing of one call's utterances: one vector (G == 0: plain launches of slot 0 of st), or G
// groups with each utterance's group id on the device (owned by the call, its ticket or its decoder cache) and
// rows_per_batch GEMM rows per utterance.
struct CatRows {
  int G = 0;
  const int* d_grp = nullptr;
  const LangStack* st = nullptr;
  int rows_per_batch = 0;
  CatRows rows(int rpb) const {
    CatRows c = *this;
    c.rows_per_batch = rpb;
    return c;
  }
};

struct Decoder {
  float* emb = nullptr;  // (V, d) fp32
  std::vector<DecLayer> layers;
  Norm after;
  Linear outl;
  bool present = false;
};

// Row buffers of a decoder pass over R rows (grow-only): residual stream x (fp32), LayerNorm output n, projections qkv,
// attention output att, FFN hidden h, LSL mix ybf, and the source-attention [k | v] of Mem encoder frames.  Every bf16
// buffer is pm times as wide: the [hi | lo] pairs of the accurate mode.
struct DecRows {
  DevBuf x, n, qkv, att, h, ybf, kv;
  int ensure(long long R, long long Mem, int d, int ffn, size_t pm) {
    if (x.ensure((size_t)R * d * 4) || n.ensure((size_t)R * d * 2 * pm) || qkv.ensure((size_t)R * 3 * d * 2 * pm) ||
        att.ensure((size_t)R * d * 2 * pm) || kv.ensure((size_t)Mem * 2 * d * 2 * pm) ||
        h.ensure((size_t)R * ffn * 2 * pm) || ybf.ensure((size_t)R * d * 2 * pm))
      return -1;
    return 0;
  }
};

// The n-best of a CTC prefix beam search over B utterances, `beam` hypothesis slots each, in one device buffer and a
// page-locked host mirror with the same layout (ints, scores 8-byte aligned):
//   times (S rows) | encoder lens (B) | tokens (S rows) | (n_tokens, n_times) (S pairs) | nhyp (B) | pad | scores (S)
// S = B * beam; token / time rows have stride len_cap.  Encoder lens .. nhyp is what a caller-supplied n-best uploads,
// (n_tokens, n_times) .. scores the small region a search hands back before its tokens and times.
struct NBest {
  DevBuf dev;
  HostPinned host;
  int B = 0, beam = 0, len_cap = 0;
  struct Arrays {
    int *tim, *lens, *tok, *olen, *nhyp;
    double* sc;
  };
  size_t S() const { return (size_t)B * beam; }
  size_t ints() const { return (2 * S() * len_cap + 2 * S() + 2 * (size_t)B + 1) & ~(size_t)1; }  // up to scores
  size_t bytes() const { return ints() * sizeof(int) + S() * sizeof(double); }
  Arrays at(void* base) const {
    Arrays a;
    a.tim = static_cast<int*>(base);
    a.lens = a.tim + S() * len_cap;
    a.tok = a.lens + B;
    a.olen = a.tok + S() * len_cap;
    a.nhyp = a.olen + 2 * S();
    a.sc = reinterpret_cast<double*>(static_cast<int*>(base) + ints());
    return a;
  }
  Arrays d() const { return at(dev.p); }
  Arrays h() const { return at(host.p); }
  size_t upload_bytes() const { return (size_t)(h().nhyp + B - h().lens) * sizeof(int); }   // lens .. nhyp
  size_t small_bytes() const { return bytes() - (size_t)(h().olen - h().tim) * sizeof(int); }  // olen .. scores
  int ntok(size_t s) const { return (int)(s % beam) < h().nhyp[s / beam] ? h().olen[2 * s] : 0; }  // 0 when absent
  int ensure(int B_, int beam_, int len_cap_) {
    B = B_;
    beam = beam_;
    len_cap = len_cap_;
    return (dev.ensure(bytes()) || host.ensure(bytes())) ? -1 : 0;
  }
};

// The packed weights of a plan, uploaded by rvb_model_finalize into the plan's WeightStore and never written after it:
// a fork copies them as they are.
struct Weights {
  float* cmvn_mean = nullptr;
  float* cmvn_istd = nullptr;
  float* conv1_w = nullptr;  // (d, 9)
  float* conv1_b = nullptr;
  Linear conv2;    // (d, 9*d) ordered (kh, kw, c)
  Linear embed;    // (d, F2*d) ordered (f, c), scaled by sqrt(d)
  Linear pos_all;  // (L*d, d) stacked linear_pos weights, no bias
  std::vector<EncLayer> enc;
  Norm after_norm;
  Linear ctc;
  Decoder dec_l, dec_r;
};

}  // namespace rvb

using namespace rvb;

struct rvb_model {
  rvb_model_config cfg;
  WeightStore store{"model:"};  // raw reference tensors until finalize, and the device allocations of this plan
  bool finalized = false;
  Weights w;
  rvb::LangStack st_enc, st_dec;  // folds of the calls' cat_embs (encoder, decoders)
  DevBuf ws_grp;                  // group ids of attention_rescoring, which waits for its stream before it returns
  HostPinned pin_grp;
  bool x3 = false;             // cfg.precision == 1: bf16x3 "fp32-accurate" mode (GemmArgs::x3, kernels.h)
  int pm() const { return x3 ? 2 : 1; }  // physical width multiplier of every bf16 operand ([hi | lo] pairs)
  DevBuf ws_fold;              // fp32 scratch of the accurate mode (LSL folds, positional table)

  // workspace (grow-only)
  DevBuf ws_c1, ws_c2, ws_x, ws_n, ws_h, ws_qkv, ws_att, ws_pw, ws_cm, ws_y, ws_ybf, ws_pe, ws_pall, ws_lens;
  DevBuf ws_encbf, ws_logits, ws_misc, ws_kpp, ws_cbias;
  rvb::DecRows dec_rows;        // rows of the flat and prefix-tree decoder passes
  DevBuf ws_lse;                // output layer: OUT_LSE partials + target logits
  DevBuf ws_tree_idx, ws_edge_rows, ws_edge_scores;  // prefix-tree pass: node / edge indices, edge rows, edge scores
  DevBuf ws_step_rows;          // full log_softmax rows of the last position (decoder_step_logp)
  DevBuf ws_search;             // prefix beam search of the tickets: they all search on s_search, one at a time
  rvb::NBest nbest_in;          // the caller's hypotheses of rvb_attention_rescoring
  HostPinned pin_a, pin_b, pin_c;
  int pe_T = 0;
  int pall_T = 0;               // ws_pall holds linear_pos(pos_emb) for this many frames
  const void* pall_ptr = nullptr;
  int lens_slot = 0;
  int lens_cap = 0;             // batch rows per slot of the pinned length ring (the largest B seen)
  static constexpr int kTickets = 4;
  std::unique_ptr<rvb::SearchTicket[]> tickets;  // [kTickets], created on first use (search_submit_any)
  std::unique_ptr<rvb::DecCache> dcache;         // KV cache of the autoregressive decoder (decoder_cache_begin / _step)
  cudaStream_t s_search = nullptr;               // side stream of the prefix beam search (search_submit)
  cudaEvent_t ev_topk = nullptr;

  ~rvb_model();
  int F1() const { return (cfg.input_dim - 1) / 2; }
  int F2() const { return (F1() - 1) / 2; }
};

namespace rvb {

// GEMM weight (N, K) fp32 -> device bf16 (N, K), or the pair layout (N, 2K) = [hi | lo] in the accurate mode
static int upload_w(rvb_model* m, const float* src, size_t N, size_t K, bf16** dst) {
  const size_t pm = m->pm();
  std::vector<uint16_t> tmp(N * K * pm);
  for (size_t n = 0; n < N; ++n)
    for (size_t k = 0; k < K; ++k) {
      const float v = src[n * K + k];
      const uint16_t h = f2bf(v);
      tmp[n * pm * K + k] = h;
      if (pm == 2) tmp[n * pm * K + K + k] = f2bf(v - bf2f(h));
    }
  return m->store.upload(tmp.data(), tmp.size(), dst);
}

// nn.Linear `prefix`.{weight,bias}; bias optional (zeros when absent and `bias_optional`)
static int load_linear(rvb_model* m, const std::string& prefix, int N, int K, Linear* out, bool has_bias = true,
                       bool bias_optional = false) {
  const std::vector<float>* w;
  if (m->store.need(prefix + ".weight", (size_t)N * K, &w)) return -1;
  if (upload_w(m, w->data(), N, K, &out->w)) return -1;
  out->N = N;
  out->K = K;
  if (has_bias) {
    const std::vector<float>* b = m->store.find(prefix + ".bias");
    if (b == nullptr && bias_optional) {
      std::vector<float> z(N, 0.f);
      if (m->store.upload(z.data(), N, &out->b)) return -1;
    } else {
      if (m->store.need(prefix + ".bias", N, &b)) return -1;
      if (m->store.upload(b->data(), N, &out->b)) return -1;
    }
  }
  return 0;
}

// pointwise_conv1 (2C x C) for the fused GLU epilogue (ACT_GLU, kernels.h): weight / bias rows interleaved in groups of
// 32 — [64j, 64j+32) = value rows of channels [32j, 32j+32), [64j+32, 64j+64) = their gate rows (C + 32j ...).
// pad_glu[c] = bf16(bias_a[c] * sigmoid(bias_g[c])): what a zero input frame becomes after pointwise_conv1 + GLU.
static int load_linear_glu(rvb_model* m, const std::string& prefix, int C, int K, Linear* out, float** pad_glu) {
  const std::vector<float>*w, *b;
  RVB_REQUIRE(C % 32 == 0, "model: conv module channels (%d) must be a multiple of 32", C);
  if (m->store.need(prefix + ".weight", (size_t)2 * C * K, &w) || m->store.need(prefix + ".bias", (size_t)2 * C, &b))
    return -1;
  std::vector<float> pw((size_t)2 * C * K), pb((size_t)2 * C), pad(C);
  for (int c = 0; c < C; ++c) {
    const int ra = 64 * (c / 32) + (c % 32), rg = ra + 32;
    memcpy(&pw[(size_t)ra * K], &(*w)[(size_t)c * K], (size_t)K * sizeof(float));
    memcpy(&pw[(size_t)rg * K], &(*w)[(size_t)(C + c) * K], (size_t)K * sizeof(float));
    pb[ra] = (*b)[c];
    pb[rg] = (*b)[C + c];
    const float g = (*b)[c] / (1.f + expf(-(*b)[C + c]));
    pad[c] = m->x3 ? g : bf2f(f2bf(g));  // the engine stores GLU outputs as bf16 (a hi/lo pair in the accurate mode)
  }
  if (upload_w(m, pw.data(), (size_t)2 * C, K, &out->w) || m->store.upload(pb.data(), pb.size(), &out->b) ||
      m->store.upload(pad.data(), pad.size(), pad_glu))
    return -1;
  out->N = 2 * C;
  out->K = K;
  return 0;
}

static int load_norm(rvb_model* m, const std::string& prefix, int d, Norm* out) {
  const std::vector<float>*g, *b;
  if (m->store.need(prefix + ".weight", d, &g) || m->store.need(prefix + ".bias", d, &b)) return -1;
  if (m->store.upload(g->data(), d, &out->g) || m->store.upload(b->data(), d, &out->b)) return -1;
  return 0;
}

// fused [q; k; v] (or [k; v]) projection
static int load_fused(rvb_model* m, const std::string& prefix, const std::vector<std::string>& parts, int d,
                      Linear* out) {
  std::vector<float> w, b;
  for (const auto& part : parts) {
    const std::vector<float>* pw;
    if (m->store.need(prefix + "." + part + ".weight", (size_t)d * d, &pw)) return -1;
    w.insert(w.end(), pw->begin(), pw->end());
    const std::vector<float>* pb = m->store.find(prefix + "." + part + ".bias");
    if (pb) {
      RVB_REQUIRE(pb->size() == (size_t)d, "model: bad bias size for %s.%s", prefix.c_str(), part.c_str());
      b.insert(b.end(), pb->begin(), pb->end());
    } else {
      b.insert(b.end(), d, 0.f);  // key_bias = False
    }
  }
  if (upload_w(m, w.data(), (size_t)d * parts.size(), d, &out->w) || m->store.upload(b.data(), b.size(), &out->b))
    return -1;
  out->N = d * (int)parts.size();
  out->K = d;
  return 0;
}

static int load_lang(rvb_model* m, const std::string& prefix, int d, int n_lang, std::vector<float*>* lw,
                     std::vector<float*>* lb) {
  for (int i = 0; i < n_lang; ++i) {
    const std::vector<float>*w, *b;
    std::string p = prefix + ".language_layers." + std::to_string(i);
    if (m->store.need(p + ".weight", (size_t)d * d, &w) || m->store.need(p + ".bias", d, &b)) return -1;
    float *dw, *db;
    if (m->store.upload(w->data(), w->size(), &dw) || m->store.upload(b->data(), d, &db)) return -1;
    lw->push_back(dw);
    lb->push_back(db);
  }
  return 0;
}

static int load_decoder(rvb_model* m, const std::string& side, int nblocks, Decoder* dec, int* n_lsl) {
  const rvb_model_config& c = m->cfg;
  const int d = c.d_model, V = c.vocab;
  const std::string p = "decoder." + side;
  const std::vector<float>* e;
  if (m->store.need(p + ".embed.0.weight", (size_t)V * d, &e)) return -1;
  if (m->store.upload(e->data(), e->size(), &dec->emb)) return -1;
  if (load_norm(m, p + ".after_norm", d, &dec->after)) return -1;
  if (load_linear(m, p + ".output_layer", V, d, &dec->outl)) return -1;
  dec->layers.resize(nblocks);
  for (int i = 0; i < nblocks; ++i) {
    DecLayer& L = dec->layers[i];
    const std::string q = p + ".decoders." + std::to_string(i);
    L.lsl = c.num_langs > 0 && (i == 0 || i == nblocks - 1);
    L.eps = L.lsl ? 1e-12f : 1e-5f;  // decoder_layer.py:241-243 vs :53-55
    if (load_norm(m, q + ".norm1", d, &L.n1) || load_norm(m, q + ".norm2", d, &L.n2) ||
        load_norm(m, q + ".norm3", d, &L.n3))
      return -1;
    if (load_fused(m, q + ".self_attn", {"linear_q", "linear_k", "linear_v"}, d, &L.qkv)) return -1;
    if (load_linear(m, q + ".self_attn.linear_out", d, d, &L.so)) return -1;
    if (load_linear(m, q + ".src_attn.linear_q", d, d, &L.cq)) return -1;
    if (load_fused(m, q + ".src_attn", {"linear_k", "linear_v"}, d, &L.ckv)) return -1;
    if (load_linear(m, q + ".src_attn.linear_out", d, d, &L.co)) return -1;
    if (load_linear(m, q + ".feed_forward.w_1", c.dec_ffn_dim, d, &L.ff1)) return -1;
    if (load_linear(m, q + ".feed_forward.w_2", d, c.dec_ffn_dim, &L.ff2)) return -1;
    if (L.lsl && load_lang(m, q, d, c.num_langs, &L.lang_w, &L.lang_b)) return -1;
    if (L.lsl) L.lsl_idx = (*n_lsl)++;
  }
  dec->present = true;
  return 0;
}

static int finalize_model(rvb_model* m) {
  const rvb_model_config& c = m->cfg;
  const int d = c.d_model, F = c.input_dim, L = c.num_blocks, K = c.cnn_kernel;
  const int F2 = m->F2();
  RVB_REQUIRE(d % 64 == 0, "model: d_model=%d must be a multiple of 64", d);
  RVB_REQUIRE(d % c.heads == 0 && d % c.dec_heads == 0, "model: heads must divide d_model");
  const std::vector<float>* t;
  if (m->store.need("encoder.global_cmvn.mean", F, &t) || m->store.upload(t->data(), F, &m->w.cmvn_mean)) return -1;
  if (m->store.need("encoder.global_cmvn.istd", F, &t) || m->store.upload(t->data(), F, &m->w.cmvn_istd)) return -1;
  if (m->store.need("encoder.embed.conv.0.weight", (size_t)d * 9, &t) ||
      m->store.upload(t->data(), t->size(), &m->w.conv1_w))
    return -1;
  if (m->store.need("encoder.embed.conv.0.bias", d, &t) || m->store.upload(t->data(), d, &m->w.conv1_b)) return -1;
  {  // conv2 weight (o, c, kh, kw) -> (o, kh, kw, c)
    if (m->store.need("encoder.embed.conv.2.weight", (size_t)d * d * 9, &t)) return -1;
    std::vector<float> w((size_t)d * d * 9);
    for (int o = 0; o < d; ++o)
      for (int ci = 0; ci < d; ++ci)
        for (int k = 0; k < 9; ++k) w[((size_t)o * 9 + k) * d + ci] = (*t)[((size_t)o * d + ci) * 9 + k];
    if (upload_w(m, w.data(), d, (size_t)9 * d, &m->w.conv2.w)) return -1;
    if (m->store.need("encoder.embed.conv.2.bias", d, &t) || m->store.upload(t->data(), d, &m->w.conv2.b)) return -1;
    m->w.conv2.N = d;
    m->w.conv2.K = 9 * d;
  }
  {  // embed linear (o, c*F2 + f) -> (o, f*d + c), times sqrt(d) (RelPositionalEncoding xscale, embedding.py:144)
    if (m->store.need("encoder.embed.out.0.weight", (size_t)d * d * F2, &t)) return -1;
    const float xs = sqrtf((float)d);
    std::vector<float> w((size_t)d * d * F2);
    for (int o = 0; o < d; ++o)
      for (int ci = 0; ci < d; ++ci)
        for (int f = 0; f < F2; ++f)
          w[(size_t)o * d * F2 + (size_t)f * d + ci] = (*t)[(size_t)o * d * F2 + (size_t)ci * F2 + f] * xs;
    if (upload_w(m, w.data(), d, (size_t)d * F2, &m->w.embed.w)) return -1;
    if (m->store.need("encoder.embed.out.0.bias", d, &t)) return -1;
    std::vector<float> b(*t);
    for (auto& v : b) v *= xs;
    if (m->store.upload(b.data(), d, &m->w.embed.b)) return -1;
    m->w.embed.N = d;
    m->w.embed.K = d * F2;
  }
  if (load_norm(m, "encoder.after_norm", d, &m->w.after_norm)) return -1;
  m->w.enc.resize(L);
  std::vector<float> posw;
  for (int i = 0; i < L; ++i) {
    EncLayer& E = m->w.enc[i];
    const std::string p = "encoder.encoders." + std::to_string(i);
    E.lsl = c.num_langs > 0 && (i == 0 || i == L - 1);
    if (load_norm(m, p + ".norm_ff_macaron", d, &E.norm_ffm) || load_norm(m, p + ".norm_mha", d, &E.norm_mha) ||
        load_norm(m, p + ".norm_conv", d, &E.norm_conv) || load_norm(m, p + ".norm_ff", d, &E.norm_ff) ||
        load_norm(m, p + ".norm_final", d, &E.norm_final))
      return -1;
    if (load_linear(m, p + ".feed_forward_macaron.w_1", c.ffn_dim, d, &E.ffm1) ||
        load_linear(m, p + ".feed_forward_macaron.w_2", d, c.ffn_dim, &E.ffm2) ||
        load_linear(m, p + ".feed_forward.w_1", c.ffn_dim, d, &E.ff1) ||
        load_linear(m, p + ".feed_forward.w_2", d, c.ffn_dim, &E.ff2))
      return -1;
    if (load_fused(m, p + ".self_attn", {"linear_q", "linear_k", "linear_v"}, d, &E.qkv)) return -1;
    if (load_linear(m, p + ".self_attn.linear_out", d, d, &E.out)) return -1;
    if (m->store.need(p + ".self_attn.linear_pos.weight", (size_t)d * d, &t)) return -1;
    posw.insert(posw.end(), t->begin(), t->end());
    if (m->store.need(p + ".self_attn.pos_bias_u", d, &t) || m->store.upload(t->data(), d, &E.pos_u)) return -1;
    if (m->store.need(p + ".self_attn.pos_bias_v", d, &t) || m->store.upload(t->data(), d, &E.pos_v)) return -1;
    if (load_linear_glu(m, p + ".conv_module.pointwise_conv1", d, d, &E.pw1, &E.pad_glu) ||
        load_linear(m, p + ".conv_module.pointwise_conv2", d, d, &E.pw2))
      return -1;
    if (m->store.need(p + ".conv_module.depthwise_conv.weight", (size_t)d * K, &t) ||
        m->store.upload(t->data(), t->size(), &E.dw_w))
      return -1;
    if (m->store.need(p + ".conv_module.depthwise_conv.bias", d, &t) || m->store.upload(t->data(), d, &E.dw_b)) return -1;
    if (load_norm(m, p + ".conv_module.norm", d, &E.cnorm)) return -1;
    if (!c.cnn_layer_norm) {
      if (m->store.need(p + ".conv_module.norm.running_mean", d, &t) || m->store.upload(t->data(), d, &E.bn_mean))
        return -1;
      if (m->store.need(p + ".conv_module.norm.running_var", d, &t) || m->store.upload(t->data(), d, &E.bn_var))
        return -1;
    }
    if (E.lsl && load_lang(m, p, d, c.num_langs, &E.lang_w, &E.lang_b)) return -1;
    if (E.lsl) E.lsl_idx = i == 0 ? 0 : 1;
  }
  if (upload_w(m, posw.data(), (size_t)L * d, d, &m->w.pos_all.w)) return -1;
  m->w.pos_all.N = L * d;
  m->w.pos_all.K = d;
  if (load_linear(m, "ctc.ctc_lo", c.vocab, d, &m->w.ctc)) return -1;
  int n_dec_lsl = 0;
  if (c.dec_blocks > 0 && m->store.find("decoder.left_decoder.embed.0.weight")) {
    if (load_decoder(m, "left_decoder", c.dec_blocks, &m->w.dec_l, &n_dec_lsl)) return -1;
  }
  if (c.r_dec_blocks > 0 && m->store.find("decoder.right_decoder.embed.0.weight")) {
    if (load_decoder(m, "right_decoder", c.r_dec_blocks, &m->w.dec_r, &n_dec_lsl)) return -1;
  }
  m->store.drop_host();
  m->finalized = true;
  return 0;
}

// cat_embs of one call over B utterances: n_cat == num_langs (one vector) or B * num_langs (one per utterance).
// -> the distinct vectors in order of first appearance (rows with equal bits are one vector), each utterance's group.
static int group_cat(const rvb_model* m, const float* cat, int n_cat, int B, std::vector<float>* uniq,
                     std::vector<int>* grp) {
  const int L = m->cfg.num_langs;
  uniq->clear();
  grp->assign(B, 0);
  if (L == 0) return 0;
  RVB_REQUIRE(cat != nullptr && (n_cat == L || n_cat == B * L),
              "cat_embs of length %d (one vector) or %d (one per utterance, B = %d) required (got %d)", L, B * L, B,
              n_cat);
  for (int b = 0; b < (n_cat == L ? 1 : B); ++b) {
    const float* v = cat + (size_t)b * L;
    const int G = (int)uniq->size() / L;
    int g = 0;
    while (g < G && memcmp(uniq->data() + (size_t)g * L, v, sizeof(float) * L) != 0) ++g;
    if (g == G) uniq->insert(uniq->end(), v, v + L);
    (*grp)[b] = g;
  }
  return 0;
}

// fold sum_i c_i * language_layers[i] (encoder_layer.py:376-390, decoder_layer.py:318-331) of each of the G vectors of
// `cat` (G * num_langs) into slot g of the stack of the encoder's (dec = false) or the decoders' LSL layers, on the
// stream of the kernels that read them.  A slot that holds its vector already folds nothing.
static int fold_stack(rvb_model* m, bool dec, const std::vector<float>& cat, cudaStream_t stream) {
  const int d = m->cfg.d_model, L = m->cfg.num_langs;
  if (L == 0) return 0;
  LangStack& st = dec ? m->st_dec : m->st_enc;
  const int G = (int)cat.size() / L;
  if (G > (int)st.key.size()) st.key.assign(G, {});  // the buffers (key.size() slots, exactly) grow below
  std::vector<int> stale;
  for (int g = 0; g < G; ++g)
    if (st.key[g].size() != (size_t)L || memcmp(st.key[g].data(), &cat[(size_t)g * L], sizeof(float) * L) != 0) {
      st.key[g].clear();
      stale.push_back(g);
    }
  if (stale.empty()) return 0;
  const size_t pm = (size_t)m->pm(), slots = st.key.size();
  if (m->x3 && m->ws_fold.ensure((size_t)d * d * sizeof(float))) return -1;
  auto fold = [&](std::vector<float*>& lw, std::vector<float*>& lb, int idx) -> int {
    if ((int)st.w.size() <= idx) {
      st.w.resize(idx + 1);
      st.b.resize(idx + 1);
    }
    if (st.w[idx].ensure(slots * d * d * pm * sizeof(bf16), true) || st.b[idx].ensure(slots * d * sizeof(float), true))
      return -1;
    for (int g : stale) {
      const float* c = cat.data() + (size_t)g * L;
      bf16* w = st.w[idx].as<bf16>() + (size_t)g * d * d * pm;
      if (m->x3) {  // fold in fp32, then split into the (d, 2d) hi/lo pair
        float* tmp = m->ws_fold.as<float>();
        if (launch_weighted_sum_bf16(lw.data(), c, L, (long long)d * d, nullptr, tmp, stream)) return -1;
        if (launch_f32_to_pair(tmp, w, d, d, stream)) return -1;
      } else if (launch_weighted_sum_bf16(lw.data(), c, L, (long long)d * d, w, nullptr, stream)) return -1;
      if (launch_weighted_sum_bf16(lb.data(), c, L, d, nullptr, st.b[idx].as<float>() + (size_t)g * d, stream)) return -1;
    }
    return 0;
  };
  if (!dec) {
    for (auto& E : m->w.enc)
      if (E.lsl && fold(E.lang_w, E.lang_b, E.lsl_idx)) return -1;
  } else {
    for (Decoder* D : {&m->w.dec_l, &m->w.dec_r})
      if (D->present)
        for (auto& Ld : D->layers)
          if (Ld.lsl && fold(Ld.lang_w, Ld.lang_b, Ld.lsl_idx)) return -1;
  }
  for (int g : stale) st.key[g].assign(&cat[(size_t)g * L], &cat[(size_t)g * L] + L);
  return 0;
}

// The LSL mixing of one call over B utterances: the distinct vectors of its cat_embs (group_cat) folded into the stack
// of the encoder (dec = false) or of the decoders; G = 0 when there is one.  -> grp, each utterance's group, for the
// caller to upload where the call's lifetime requires (cr->d_grp, read when G > 1), and the vectors in uniq if asked.
static int cat_rows(rvb_model* m, bool dec, const float* cat, int n_cat, int B, CatRows* cr, std::vector<int>* grp,
                    cudaStream_t stream, std::vector<float>* uniq = nullptr) {
  std::vector<float> own;
  if (uniq == nullptr) uniq = &own;
  if (group_cat(m, cat, n_cat, B, uniq, grp) || fold_stack(m, dec, *uniq, stream)) return -1;
  const int L = m->cfg.num_langs, G = L ? (int)uniq->size() / L : 0;
  cr->G = G > 1 ? G : 0;
  cr->st = dec ? &m->st_dec : &m->st_enc;
  return 0;
}

// B group ids -> dev through the page-locked pin, on `stream`
static int upload_groups(const std::vector<int>& grp, HostPinned& pin, DevBuf& dev, cudaStream_t stream) {
  if (pin.ensure(grp.size() * sizeof(int)) || dev.ensure(grp.size() * sizeof(int))) return -1;
  memcpy(pin.p, grp.data(), grp.size() * sizeof(int));
  RVB_CHECK_CUDA(cudaMemcpyAsync(dev.p, pin.p, grp.size() * sizeof(int), cudaMemcpyHostToDevice, stream));
  return 0;
}

// <sos>/<eos>: tokenizer_conf.special_tokens when the config names them, else vocab - 1 for both (asr_model.py:79-82)
static inline int sos_id(const rvb_model_config& c) { return c.sos_id > 0 ? c.sos_id : c.vocab - 1; }
static inline int eos_id(const rvb_model_config& c) { return c.eos_id > 0 ? c.eos_id : c.vocab - 1; }

static int gemm(rvb_model* m, const bf16* A, const Linear& W, int M, int act, int out_mode, void* out, float alpha,
                cudaStream_t stream, const int* row_lens = nullptr, int rows_per_batch = 0, int ldo = 0,
                bool use_bias = true) {
  GemmArgs g;
  g.x3 = m->x3 ? 1 : 0;
  if (m->x3 && out_mode == OUT_BF16) g.out_split = (act == ACT_GLU) ? W.N / 2 : W.N;  // bf16 outputs become hi/lo pairs
  g.A = A;
  g.W = W.w;
  g.M = M;
  g.N = W.N;
  g.K = W.K;
  g.bias = use_bias ? W.b : nullptr;
  g.act = act;
  g.out_mode = out_mode;
  g.out = out;
  g.alpha = alpha;
  g.row_lens = row_lens;
  g.rows_per_batch = rows_per_batch;
  g.ldo = ldo;
  return launch_gemm(g, stream);
}

// The language-specific linear of one LSL layer over M rows, from the folds of layer lsl_idx of cr.st: a plain launch
// of slot 0 for one vector (cr.G == 0), else one grouped launch, every row taking its utterance's slot
static int lang_gemm(rvb_model* m, const bf16* A, int lsl_idx, const CatRows& cr, int M, int out_mode, void* out,
                     cudaStream_t stream) {
  const int d = m->cfg.d_model;
  const Linear slot0{cr.st->w[lsl_idx].as<bf16>(), cr.st->b[lsl_idx].as<float>(), d, d};
  if (cr.G == 0) return gemm(m, A, slot0, M, ACT_NONE, out_mode, out, 1.f, stream);
  GemmArgs g;
  g.x3 = m->x3 ? 1 : 0;
  if (m->x3 && out_mode == OUT_BF16) g.out_split = d;
  g.A = A;
  g.W = slot0.w;
  g.M = M;
  g.N = cr.G * d;
  g.K = d;
  g.bias = slot0.b;
  g.act = ACT_NONE;
  g.out_mode = out_mode;
  g.out = out;
  g.grp = cr.d_grp;
  g.group_n = d;
  g.rows_per_batch = cr.rows_per_batch;
  return launch_gemm(g, stream);
}

// 1 = wgmma attention (default when d_k == 64), 0 = mma.sync kernel (RVB_ATTN=mma)
static int attn_impl() {
  static int v = -1;
  if (v < 0) {
    const char* e = getenv("RVB_ATTN");
    v = (e && strcmp(e, "mma") == 0) ? 0 : 1;
  }
  return v;
}

// whether an attention of `dk`-wide heads runs on the wgmma kernel (bf16 mode only)
static bool wgmma_attn(const rvb_model* m, int dk) { return !m->x3 && attn_impl() == 1 && dk == 64; }

// One attention of the decoder.  q / k / v / out address column 0 of head 0, with their LOGICAL (plain bf16) row
// strides; group g owns query rows [g*Tq, (g+1)*Tq) and key rows [g*Tk, (g+1)*Tk).  In the accurate mode every operand
// is a [hi | lo] pair: physical stride 2 * ld, lo one logical width (ld) to the right.
struct DecAttn {
  const bf16* q = nullptr;
  const bf16* k = nullptr;
  const bf16* v = nullptr;
  bf16* out = nullptr;
  int ldq = 0, ldk = 0, ldv = 0, ldo = 0;
  int groups = 0, Tq = 0, Tk = 0, H = 0, dk = 0;
  float scale = 1.0f;
  // the mask: key lengths (k_lens, per group), causal (with Tq == Tk, on top of k_lens), key bits (on top of causal,
  // AttnTcArgs::key_bits) or key lists (AttnF32Args::key_list)
  const int* k_lens = nullptr;
  bool causal = false;
  const uint32_t* key_bits = nullptr;
  int bits_ld = 0;
  const int* key_list = nullptr;
  const int* key_list_len = nullptr;
  int key_list_ld = 0;
  bool f32 = false;  // the fp32 kernel in the bf16 mode too
};

// the kernel: fp32 in the accurate mode, when asked for, or for key lists; else wgmma (wgmma_attn); else mma.sync
static int dec_attention(const rvb_model* m, const DecAttn& a, cudaStream_t stream) {
  if (m->x3 || a.f32 || a.key_list) {
    const int pm = m->pm(), lo = m->x3 ? 1 : 0;
    AttnF32Args f;
    f.q = a.q; f.k = a.k; f.v = a.v; f.out = a.out;
    f.ldq = a.ldq * pm; f.ldk = a.ldk * pm; f.ldv = a.ldv * pm; f.ldo = a.ldo * pm;
    f.q_lo = a.ldq * lo; f.k_lo = a.ldk * lo; f.v_lo = a.ldv * lo; f.o_lo = a.ldo * lo;
    f.groups = a.groups; f.Tq = a.Tq; f.Tk = a.Tk; f.H = a.H; f.dk = a.dk;
    f.k_lens = a.k_lens;
    f.chunk = a.causal ? 1 : 0;  // chunk = 1, left < 0: causal
    f.key_list = a.key_list; f.key_list_len = a.key_list_len; f.key_list_ld = a.key_list_ld;
    return launch_attention_f32(f, stream);
  }
  if (wgmma_attn(m, a.dk)) {
    AttnTcArgs t;
    t.q = a.q; t.k = a.k; t.v = a.v; t.out = a.out;
    t.ldq = a.ldq; t.ldk = a.ldk; t.ldv = a.ldv; t.ldo = a.ldo;
    t.groups = a.groups; t.Tq = a.Tq; t.Tk = a.Tk; t.H = a.H; t.dk = a.dk;
    t.k_lens = a.k_lens;
    t.causal = a.causal;
    t.key_bits = a.key_bits; t.bits_ld = a.bits_ld;
    t.scale = a.scale;
    return launch_attention_tc(t, stream);
  }
  RVB_REQUIRE(a.key_bits == nullptr, "decoder attention: key bit masks need the wgmma kernel");
  AttnArgs s;
  s.q = a.q; s.k = a.k; s.v = a.v; s.out = a.out;
  s.ldq = a.ldq; s.ldk = a.ldk; s.ldv = a.ldv; s.ldo = a.ldo;
  s.Bq = a.groups; s.Tq = a.Tq; s.Tk = a.Tk; s.H = a.H; s.dk = a.dk;
  s.k_lens = a.k_lens;  // one query batch per key batch: the same key count as q_lens under the causal mask
  s.causal = a.causal;
  s.scale = a.scale;
  return launch_attention(s, stream);
}

// source attention of Tq query rows per utterance (row stride d) over its Tp encoder frames, kv = [k | v] rows (2d)
static DecAttn src_attention(bf16* q, const bf16* kv, bf16* out, int d, int B, int Tq, int Tp, int H,
                             const int* d_enc_lens) {
  DecAttn a;
  a.q = q;
  a.k = kv;
  a.v = kv + d;
  a.out = out;
  a.ldq = a.ldo = d;
  a.ldk = a.ldv = 2 * d;
  a.groups = B;
  a.Tq = Tq;
  a.Tk = Tp;
  a.H = H;
  a.dk = d / H;
  a.scale = 1.0f / sqrtf((float)a.dk);
  a.k_lens = d_enc_lens;
  return a;
}

// att_chunk > 0: bounded-context attention (add_optional_chunk_mask, utils/mask.py:126-197, with a fixed decoding chunk):
// query frame i attends keys [max(0, (i/chunk - left) * chunk) (0 when left < 0), (i/chunk + 1) * chunk) & pad mask.
static int encoder_forward(rvb_model* m, const float* d_feats, const int* h_feat_lens, int B, int T,
                           const float* h_cat, int n_cat, float* d_enc_out, int* h_enc_lens, cudaStream_t stream,
                           int att_chunk = 0, int att_left = -1, bool streaming = false) {
  const rvb_model_config& c = m->cfg;
  RVB_REQUIRE(m->finalized, "encoder_forward: model not finalized");
  const int d = c.d_model, F = c.input_dim, H = c.heads, dk = d / H, L = c.num_blocks;
  const int T1 = (T - 1) / 2, F1 = m->F1(), Tp = (T1 - 1) / 2, F2 = m->F2();
  RVB_REQUIRE(T >= 7 && Tp >= 1, "encoder_forward: chunk of %d frames is too short for Conv2dSubsampling4", T);
  RVB_REQUIRE(Tp <= 5000, "encoder_forward: %d encoder frames exceed the positional table (5000)", Tp);
  const int T1h = (T1 + 1) / 2;
  const long long M = (long long)B * Tp;
  RVB_REQUIRE(M * (long long)F2 < (1ll << 31), "encoder_forward: batch too large (B*T'*F2 overflows int)");
  std::vector<int> grp;
  CatRows cr;
  if (cat_rows(m, false, h_cat, n_cat, B, &cr, &grp, stream)) return -1;

  // lengths
  // pinned staging ring: a back-to-back call must not overwrite lengths an earlier async copy still reads.  Slots are
  // sized for the largest batch seen, so batches of varying B (corpus decoding) only wait when that maximum grows.
  // A slot holds the lengths (lens_cap) and then the utterances' LSL groups of a per-utterance cat_embs.
  constexpr int kRing = 16;
  if (B > m->lens_cap) {
    RVB_CHECK_CUDA(cudaStreamSynchronize(stream));
    if (m->pin_a.ensure(sizeof(int) * 2 * B * kRing) || m->ws_lens.ensure(sizeof(int) * 2 * B * kRing)) return -1;
    m->lens_cap = B;
  }
  const int slot = (m->lens_slot++) % kRing;
  int* h_lens = m->pin_a.as<int>() + (size_t)slot * 2 * m->lens_cap;
  for (int b = 0; b < B; ++b) {
    int e = rvb_encoder_out_len(h_feat_lens[b], T);
    h_lens[b] = e;
    if (h_enc_lens) h_enc_lens[b] = e;
  }
  int* d_lens = m->ws_lens.as<int>() + (size_t)slot * 2 * m->lens_cap;
  if (cr.G) memcpy(h_lens + m->lens_cap, grp.data(), sizeof(int) * B);
  RVB_CHECK_CUDA(cudaMemcpyAsync(d_lens, h_lens, sizeof(int) * (cr.G ? m->lens_cap + B : B), cudaMemcpyHostToDevice,
                                 stream));
  cr.d_grp = d_lens + m->lens_cap;
  cr.rows_per_batch = Tp;

  // workspace
  const bool x3 = m->x3;
  const size_t pm = (size_t)m->pm();  // bf16 operands are (hi, lo) pairs in the accurate mode: twice as wide
  if (m->ws_c1.ensure((size_t)B * 2 * T1h * F1 * d * 2 * pm) || m->ws_c2.ensure((size_t)M * F2 * d * 2 * pm) ||
      m->ws_x.ensure((size_t)M * d * 4) || m->ws_n.ensure((size_t)M * d * 2 * pm) ||
      m->ws_h.ensure((size_t)M * c.ffn_dim * 2 * pm) || m->ws_qkv.ensure((size_t)M * 3 * d * 2 * pm) ||
      m->ws_att.ensure((size_t)M * d * 2 * pm) || m->ws_pw.ensure((size_t)M * d * 2 * pm) ||
      m->ws_cm.ensure((size_t)M * d * 2 * pm) || m->ws_y.ensure((size_t)M * d * 4) ||
      m->ws_ybf.ensure((size_t)M * d * 2 * pm) || m->ws_pall.ensure((size_t)Tp * L * d * 2 * pm) ||
      m->ws_kpp.ensure((size_t)M * d * 2) ||
      m->ws_cbias.ensure(((size_t)B * H * Tp + (size_t)M * 2 * ((d / 2 + 127) / 128)) * 4))
    return -1;
  const bool tc_attn = wgmma_attn(m, dk);
  if (!tc_attn && !x3 && attn_impl() == 1) {   // say so once: a d_k != 64 model runs the (slower) mma.sync attention
    static std::atomic<bool> warned{false};
    if (!warned.exchange(true))
      fprintf(stderr, "reverb_b200: d_k = %d — the wgmma attention kernel is built for d_k = 64; using the mma.sync kernel\n", dk);
  }
  // rel-pos key transform inside the [q; k; v] projection's epilogue (default); RVB_RELPOS=prep keeps the separate kernel
  const char* rp_env = getenv("RVB_RELPOS");   // read per call: tests A/B the two paths in one process
  const bool relpos_fused = tc_attn && !(rp_env && strcmp(rp_env, "prep") == 0) && get_gemm_impl() != 1;
  bf16* c1 = m->ws_c1.as<bf16>();
  bf16* c2 = m->ws_c2.as<bf16>();
  float* x = m->ws_x.as<float>();
  bf16* n = m->ws_n.as<bf16>();
  bf16* h = m->ws_h.as<bf16>();
  bf16* qkv = m->ws_qkv.as<bf16>();
  bf16* att = m->ws_att.as<bf16>();
  bf16* pw = m->ws_pw.as<bf16>();
  bf16* cm = m->ws_cm.as<bf16>();
  float* y = m->ws_y.as<float>();
  bf16* ybf = m->ws_ybf.as<bf16>();
  bf16* pall = m->ws_pall.as<bf16>();

  // positional table + all layers' linear_pos(pos_emb) in one GEMM (attention.py:374; batch-shared)
  if (m->pe_T < Tp) {
    if (m->ws_pe.ensure((size_t)Tp * d * 2 * pm)) return -1;
    if (x3) {
      if (m->ws_fold.ensure((size_t)Tp * d * sizeof(float) > (size_t)d * d * sizeof(float) ? (size_t)Tp * d * sizeof(float)
                                                                                             : (size_t)d * d * sizeof(float)))
        return -1;
      if (launch_sinusoid(Tp, d, m->ws_fold.as<float>(), nullptr, stream)) return -1;
      if (launch_f32_to_pair(m->ws_fold.as<float>(), m->ws_pe.as<bf16>(), Tp, d, stream)) return -1;
    } else if (launch_sinusoid(Tp, d, nullptr, m->ws_pe.as<bf16>(), stream)) {
      return -1;
    }
    m->pe_T = Tp;
  }
  // ... where row t depends on t only (the GEMM computes rows independently): kept for the longest T' seen, and a
  // shorter batch reads its leading rows
  if (m->pall_T < Tp || m->pall_ptr != (const void*)pall) {
    if (gemm(m, m->ws_pe.as<bf16>(), m->w.pos_all, Tp, ACT_NONE, OUT_BF16, pall, 1.f, stream, nullptr, 0, 0, false))
      return -1;
    m->pall_T = Tp;
    m->pall_ptr = pall;
  }

  // subsampling: CMVN + conv1 + ReLU ; conv2 + ReLU as implicit GEMM ; Linear(19 d -> d) * sqrt(d)
  if (launch_conv1(d_feats, m->w.cmvn_mean, m->w.cmvn_istd, m->w.conv1_w, m->w.conv1_b, c1, B, T, F, d, T1, T1h, F1,
                   stream, x3))
    return -1;
  {
    GemmArgs g;
    g.A = c1;
    g.W = m->w.conv2.w;
    g.M = (int)(M * F2);
    g.N = d;
    g.K = 9 * d;
    g.bias = m->w.conv2.b;
    g.act = ACT_RELU;
    g.out_mode = OUT_BF16;
    g.out = c2;
    g.ldo = d;
    g.conv_mode = 1;
    g.conv_B = B;
    g.conv_T1h = T1h;
    g.conv_F1 = F1;
    g.conv_C = d;
    g.conv_T2 = Tp;
    g.conv_F2 = F2;
    if (x3) {  // output row (b, t') = [hi (F2*d) | lo (F2*d)]: directly the pair-layout A operand of the embed linear
      g.x3 = 1;
      g.out_split = F2 * d;
      g.conv_pair_out = 1;
    }
    if (launch_gemm(g, stream)) return -1;
  }
  if (gemm(m, c2, m->w.embed, (int)M, ACT_NONE, OUT_F32, x, 1.f, stream)) return -1;

  const float att_scale = 1.0f / sqrtf((float)dk);
  // first pre-norm of block 0
  if (launch_layernorm(x, m->w.enc[0].norm_ffm.g, m->w.enc[0].norm_ffm.b, 1e-5f, (int)M, d, n, nullptr, nullptr, 0, 0,
                       stream, x3))
    return -1;
  for (int l = 0; l < L; ++l) {
    EncLayer& E = m->w.enc[l];
    // macaron FFN: x += 0.5 * W2 SiLU(W1 n)                                   (encoder_layer.py:200-207)
    if (gemm(m, n, E.ffm1, (int)M, ACT_SILU, OUT_BF16, h, 1.f, stream)) return -1;
    if (gemm(m, h, E.ffm2, (int)M, ACT_NONE, OUT_RESID_F32, x, 0.5f, stream)) return -1;
    // rel-pos MHSA                                                            (encoder_layer.py:209-217)
    if (launch_layernorm(x, E.norm_mha.g, E.norm_mha.b, 1e-5f, (int)M, d, n, nullptr, nullptr, 0, 0, stream, x3)) return -1;
    if (relpos_fused) {
      GemmArgs g;
      g.A = n;
      g.W = E.qkv.w;
      g.M = (int)M;
      g.N = E.qkv.N;
      g.K = E.qkv.K;
      g.bias = E.qkv.b;
      g.act = ACT_NONE;
      g.out_mode = OUT_BF16;
      g.out = qkv;
      g.rp_pos = pall + (size_t)l * d;
      g.rp_ldp = L * d;
      g.rp_T = Tp;
      g.rp_H = H;
      g.rp_col0 = d;
      g.rp_u = E.pos_u;
      g.rp_v = E.pos_v;
      g.rp_cb = m->ws_cbias.as<float>();
      if (launch_gemm(g, stream)) return -1;
    } else if (gemm(m, n, E.qkv, (int)M, ACT_NONE, OUT_BF16, qkv, 1.f, stream)) {
      return -1;
    }
    if (x3) {
      // accurate mode: the reference's two-product rel-pos attention in fp32 (attention_f32.cu) on the hi/lo pairs
      AttnF32Args a;
      a.q = qkv;
      a.k = qkv + d;
      a.v = qkv + 2 * d;
      a.p = pall + (size_t)l * d;
      a.bias_u = E.pos_u;
      a.bias_v = E.pos_v;
      a.out = att;
      a.ldq = a.ldk = a.ldv = 6 * d;
      a.q_lo = a.k_lo = a.v_lo = 3 * d;
      a.ldp = 2 * L * d;
      a.p_lo = L * d;
      a.ldo = 2 * d;
      a.o_lo = d;
      a.groups = B;
      a.Tq = Tp;
      a.Tk = Tp;
      a.H = H;
      a.dk = dk;
      a.k_lens = d_lens;
      a.chunk = att_chunk > 0 ? att_chunk : 0;
      a.left = att_left;
      if (launch_attention_f32(a, stream)) return -1;
    } else if (tc_attn) {
      // s = (q . (k + p) + (u . k + v . p)) / sqrt(d_k): fold the position term into the keys and a key bias
      bf16* kpp = m->ws_kpp.as<bf16>();
      float* cb = m->ws_cbias.as<float>();
      if (!relpos_fused && launch_relpos_prep(qkv + d, 3 * d, pall + (size_t)l * d, L * d, E.pos_u, E.pos_v, kpp, cb, B, Tp, H,
                                              dk, stream))
        return -1;
      AttnTcArgs a;
      a.q = qkv;
      a.k = relpos_fused ? qkv + d : kpp;   // fused: the projection already wrote K'' over the key columns
      a.v = qkv + 2 * d;
      a.out = att;
      a.ldq = 3 * d;
      a.ldk = relpos_fused ? 3 * d : d;
      a.ldv = 3 * d;
      a.ldo = d;
      a.groups = B;
      a.Tq = Tp;
      a.Tk = Tp;
      a.H = H;
      a.dk = dk;
      a.key_bias = cb;
      a.k_lens = d_lens;
      a.chunk = att_chunk;
      a.left_chunks = att_left;
      a.scale = att_scale;
      if (launch_attention_tc(a, stream)) return -1;
    } else {
      RVB_REQUIRE(att_chunk <= 0, "encoder_forward: chunk-masked attention needs the wgmma kernel (d_k = 64)");
      AttnArgs a;
      a.q = qkv;
      a.k = qkv + d;
      a.v = qkv + 2 * d;
      a.p = pall + (size_t)l * d;
      a.bias_u = E.pos_u;
      a.bias_v = E.pos_v;
      a.out = att;
      a.ldq = a.ldk = a.ldv = 3 * d;
      a.ldp = L * d;
      a.ldo = d;
      a.Bq = B;
      a.Tq = Tp;
      a.Tk = Tp;
      a.H = H;
      a.dk = dk;
      a.k_lens = d_lens;
      a.scale = att_scale;
      if (launch_attention(a, stream)) return -1;
    }
    if (gemm(m, att, E.out, (int)M, ACT_NONE, OUT_RESID_F32, x, 1.f, stream)) return -1;
    // convolution module                                                       (encoder_layer.py:222-231)
    if (launch_layernorm(x, E.norm_conv.g, E.norm_conv.b, 1e-5f, (int)M, d, n, nullptr, d_lens, Tp, 1, stream, x3))
      return -1;
    if (gemm(m, n, E.pw1, (int)M, ACT_GLU, OUT_BF16, pw, 1.f, stream)) return -1;   // pw = GLU(pointwise_conv1), (M, d)
    if (launch_conv_mid(pw, E.pad_glu, E.dw_w, E.dw_b, E.cnorm.g, E.cnorm.b, E.bn_mean, E.bn_var, c.cnn_layer_norm, 1e-5f, cm, B,
                        Tp, d, c.cnn_kernel, c.causal, stream, y /*fp32 (M, d) scratch, free until the LSL mix*/,
                        m->ws_cbias.as<float>() + (size_t)B * H * Tp, x3,
                        (streaming && !c.causal) ? att_chunk : 0))
      return -1;
    if (gemm(m, cm, E.pw2, (int)M, ACT_NONE, OUT_RESID_F32, x, 1.f, stream, d_lens, Tp)) return -1;
    // FFN (+ language-specific mix on the first / last block)                   (encoder_layer.py:233-242, 372-400)
    if (launch_layernorm(x, E.norm_ff.g, E.norm_ff.b, 1e-5f, (int)M, d, n, nullptr, nullptr, 0, 0, stream, x3)) return -1;
    const bf16* ffn_in = n;
    if (E.lsl) {
      if (lang_gemm(m, n, E.lsl_idx, cr, (int)M, OUT_F32, y, stream)) return -1;
      if (x3 ? launch_f32_to_pair(y, ybf, M, d, stream) : launch_f32_to_bf16(y, ybf, M * d, stream)) return -1;
      ffn_in = ybf;
    }
    if (gemm(m, ffn_in, E.ff1, (int)M, ACT_SILU, OUT_BF16, h, 1.f, stream)) return -1;
    if (gemm(m, h, E.ff2, (int)M, ACT_NONE, OUT_RESID_F32, x, 0.5f, stream)) return -1;
    // x = norm_final(x) (+ y) ; then the next block's first pre-norm, or after_norm for the last block
    const bool last = (l == L - 1);
    const Norm& nx = last ? m->w.after_norm : m->w.enc[l + 1].norm_ffm;
    if (launch_double_layernorm(x, E.norm_final.g, E.norm_final.b, E.lsl ? y : nullptr, x, nx.g, nx.b, 1e-5f, (int)M,
                                d, last ? nullptr : n, last ? d_enc_out : nullptr, stream, x3))
      return -1;
  }
  return 0;
}

__global__ void sub_column_kernel(float* x, long long ld, int rows, int col, float v) {
  int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r < rows) x[(long long)r * ld + col] -= v;
}

// the encoder output (Mem, d) fp32 as a GEMM operand in ws_encbf: bf16, or the [hi | lo] pair in the accurate mode
static int enc_operand(rvb_model* m, const float* d_enc_out, long long Mem, bf16** out, cudaStream_t stream) {
  const int d = m->cfg.d_model;
  if (m->ws_encbf.ensure((size_t)Mem * d * 2 * m->pm())) return -1;
  *out = m->ws_encbf.as<bf16>();
  return m->x3 ? launch_f32_to_pair(d_enc_out, *out, Mem, d, stream) : launch_f32_to_bf16(d_enc_out, *out, Mem * d, stream);
}

static int ctc_topk(rvb_model* m, const float* d_enc_out, int B, int Tp, int k, float blank_penalty, int blank_id,
                    float* d_topk_val, int* d_topk_idx, float* d_logp, cudaStream_t stream) {
  const rvb_model_config& c = m->cfg;
  const long long M = (long long)B * Tp;
  const int V = c.vocab;
  const int ldv = (V + 3) & ~3;
  if (m->ws_logits.ensure((size_t)M * ldv * 4)) return -1;
  bf16* encbf;
  float* logits = m->ws_logits.as<float>();
  if (enc_operand(m, d_enc_out, M, &encbf, stream)) return -1;
  if (gemm(m, encbf, m->w.ctc, (int)M, ACT_NONE, OUT_F32, logits, 1.f, stream, nullptr, 0, ldv)) return -1;
  if (blank_penalty > 0.f) {
    sub_column_kernel<<<(int)((M + 255) / 256), 256, 0, stream>>>(logits, ldv, (int)M, blank_id, blank_penalty);
    RVB_COUNT_LAUNCH();
    RVB_CHECK_LAUNCH();
  }
  return launch_logsoftmax_topk(logits, ldv, (int)M, V, k, d_topk_val, d_topk_idx, d_logp, 1, stream);
}

// The layers of a (LanguageSpecific)TransformerDecoder over the R rows of w.x, then after_norm -> w.n
// (decoder_layer.py:95-110 / 286-301).  self_attn(l) attends from the [q | k | v] projection in w.qkv, src_attn(l) from
// the q projection in w.qkv (row stride d) over the encoder output; both write w.att.
// cr: the LSL mixing of the rows' utterances (cr.rows_per_batch rows each).
template <class SelfAttn, class SrcAttn>
static int decoder_layers(rvb_model* m, Decoder& D, DecRows& w, int R, const CatRows& cr, SelfAttn self_attn,
                          SrcAttn src_attn, cudaStream_t stream) {
  const int d = m->cfg.d_model;
  const bool x3 = m->x3;
  float* x = w.x.as<float>();
  bf16* n = w.n.as<bf16>();
  bf16* qkv = w.qkv.as<bf16>();
  bf16* att = w.att.as<bf16>();
  bf16* h = w.h.as<bf16>();
  bf16* ybf = w.ybf.as<bf16>();
  for (size_t l = 0; l < D.layers.size(); ++l) {
    DecLayer& Ld = D.layers[l];
    // masked self-attention
    if (launch_layernorm(x, Ld.n1.g, Ld.n1.b, Ld.eps, R, d, n, nullptr, nullptr, 0, 0, stream, x3)) return -1;
    if (gemm(m, n, Ld.qkv, R, ACT_NONE, OUT_BF16, qkv, 1.f, stream)) return -1;
    if (self_attn(l)) return -1;
    if (gemm(m, att, Ld.so, R, ACT_NONE, OUT_RESID_F32, x, 1.f, stream)) return -1;
    // source attention over the utterance's encoder output
    if (launch_layernorm(x, Ld.n2.g, Ld.n2.b, Ld.eps, R, d, n, nullptr, nullptr, 0, 0, stream, x3)) return -1;
    if (gemm(m, n, Ld.cq, R, ACT_NONE, OUT_BF16, qkv, 1.f, stream)) return -1;  // q -> first d cols, ld = d
    if (src_attn(l)) return -1;
    if (gemm(m, att, Ld.co, R, ACT_NONE, OUT_RESID_F32, x, 1.f, stream)) return -1;
    // feed forward (ReLU), language-specific mix first on LSL layers
    if (launch_layernorm(x, Ld.n3.g, Ld.n3.b, Ld.eps, R, d, n, nullptr, nullptr, 0, 0, stream, x3)) return -1;
    const bf16* ffn_in = n;
    if (Ld.lsl) {
      if (lang_gemm(m, n, Ld.lsl_idx, cr, R, OUT_BF16, ybf, stream)) return -1;
      ffn_in = ybf;
    }
    if (gemm(m, ffn_in, Ld.ff1, R, ACT_RELU, OUT_BF16, h, 1.f, stream)) return -1;
    if (gemm(m, h, Ld.ff2, R, ACT_NONE, OUT_RESID_F32, x, 1.f, stream)) return -1;
  }
  return launch_layernorm(x, D.after.g, D.after.b, 1e-5f, R, d, n, nullptr, nullptr, 0, 0, stream, x3);
}

// Output layer: log-probability of the gather target of each of the M rows of A (gather < 0 -> 0) -> out (M)
static int target_logp(rvb_model* m, const Decoder& D, const bf16* A, int M, const int* gather, float* out,
                       cudaStream_t stream) {
  const int V = m->cfg.vocab, ldv = (V + 3) & ~3;
  if (get_gemm_impl() != 1 && V > 128) {
    // log_softmax + gather fused into the output-layer GEMM: the (M, V) fp32 logits (4.2 GB at B = 64) are never
    // written; the epilogue leaves per-slab (max, sum-exp) partials and the target logit, a small kernel merges them
    const int slabs = lse_slabs(V);
    if (m->ws_lse.ensure((size_t)M * slabs * sizeof(float2) + (size_t)M * sizeof(float))) return -1;
    float2* part = m->ws_lse.as<float2>();
    float* tgt = reinterpret_cast<float*>(part + (size_t)M * slabs);
    GemmArgs g;
    g.x3 = m->x3 ? 1 : 0;
    g.A = A;
    g.W = D.outl.w;
    g.bias = D.outl.b;
    g.M = M;
    g.N = D.outl.N;
    g.K = D.outl.K;
    g.out_mode = OUT_LSE;
    g.lse_gather = gather;
    g.lse_part = part;
    g.lse_tgt = tgt;
    if (launch_gemm(g, stream)) return -1;
    return launch_lse_merge(part, slabs, tgt, gather, M, out, stream);
  }
  if (m->ws_logits.ensure((size_t)M * ldv * 4)) return -1;
  float* logits = m->ws_logits.as<float>();
  if (gemm(m, A, D.outl, M, ACT_NONE, OUT_F32, logits, 1.f, stream, nullptr, 0, ldv)) return -1;
  return launch_logsoftmax_gather(logits, ldv, M, V, gather, 1, out, stream);
}

// Output layer on the LAST of every Lp rows of n (S sequences): log_softmax + top-k -> val / idx (S, k), and the full
// log_softmax rows -> logp (S, V) when given
static int last_position_topk(rvb_model* m, const Decoder& D, const bf16* n, int S, int Lp, DevBuf& logits_buf, int k,
                              float* val, int* idx, float* logp, cudaStream_t stream) {
  const int d = m->cfg.d_model, V = m->cfg.vocab, ldv = (V + 3) & ~3, pm = m->pm();
  if (logits_buf.ensure((size_t)S * ldv * 4)) return -1;
  float* logits = logits_buf.as<float>();
  // rows s*Lp + (Lp-1): the A operand is the strided view (S, d) with leading dimension Lp*d
  GemmArgs g;
  g.x3 = m->x3 ? 1 : 0;
  g.A = n + (size_t)(Lp - 1) * d * pm;
  g.lda = Lp * d * pm;
  g.W = D.outl.w;
  g.bias = D.outl.b;
  g.M = S;
  g.N = D.outl.N;
  g.K = D.outl.K;
  g.act = ACT_NONE;
  g.out_mode = OUT_F32;
  g.out = logits;
  g.ldo = ldv;
  g.alpha = 1.f;
  if (launch_gemm(g, stream)) return -1;
  return launch_logsoftmax_topk(logits, ldv, S, V, k, val, idx, logp, 1, stream);
}

// One pass of the decoder over R = S * Lp rows (S sequences of Lp positions).
// Default: log-probability of the gather target at every position -> d_scores (attention rescoring).
// step_k > 0 (autoregressive `attention` mode): only the LAST position of every sequence goes through the output
// layer; log_softmax + top-step_k of it -> d_step_val / d_step_idx (S, step_k).
static int decoder_pass(rvb_model* m, Decoder& D, const bf16* enc_bf, const int* d_enc_lens, int B, int Tp, int N,
                        int Lp, const int* d_tokens, const int* d_seq_lens, const int* d_gather, float* d_scores,
                        const CatRows& cr, cudaStream_t stream, int step_k = 0, float* d_step_val = nullptr, int* d_step_idx = nullptr,
                        float* d_step_logp = nullptr /* (S, V): full log_softmax rows of the last position */) {
  const rvb_model_config& c = m->cfg;
  const int d = c.d_model, H = c.dec_heads, dk = d / H, V = c.vocab;
  const int S = B * N;
  const long long R = (long long)S * Lp;
  const long long Mem = (long long)B * Tp;
  const int ldv = (V + 3) & ~3;
  RVB_REQUIRE(R < (1ll << 31) && R * ldv < (1ll << 40), "rescoring: too many hypothesis rows");
  DecRows& w = m->dec_rows;
  if (w.ensure(R, Mem, d, c.dec_ffn_dim, m->pm())) return -1;
  bf16* qkv = w.qkv.as<bf16>();
  bf16* att = w.att.as<bf16>();
  bf16* kv = w.kv.as<bf16>();
  if (launch_embed_posenc(d_tokens, D.emb, S, Lp, d, w.x.as<float>(), stream)) return -1;
  auto self_attn = [&](size_t) {
    DecAttn a;  // one group per hypothesis, causal, keys beyond the hypothesis length masked
    a.q = qkv;
    a.k = qkv + d;
    a.v = qkv + 2 * d;
    a.out = att;
    a.ldq = a.ldk = a.ldv = 3 * d;
    a.ldo = d;
    a.groups = S;
    a.Tq = a.Tk = Lp;
    a.H = H;
    a.dk = dk;
    a.scale = 1.0f / sqrtf((float)dk);
    a.k_lens = d_seq_lens;
    a.causal = true;
    return dec_attention(m, a, stream);
  };
  auto src_attn = [&](size_t l) {
    // K/V projected ONCE per utterance; its N hypotheses share the keys: one group of N * Lp query rows per utterance
    if (gemm(m, enc_bf, D.layers[l].ckv, (int)Mem, ACT_NONE, OUT_BF16, kv, 1.f, stream)) return -1;
    return dec_attention(m, src_attention(qkv, kv, att, d, B, N * Lp, Tp, H, d_enc_lens), stream);
  };
  if (decoder_layers(m, D, w, (int)R, cr.rows(N * Lp), self_attn, src_attn, stream)) return -1;
  if (step_k > 0)
    return last_position_topk(m, D, w.n.as<bf16>(), S, Lp, m->ws_logits, step_k, d_step_val, d_step_idx, d_step_logp,
                              stream);
  return target_logp(m, D, w.n.as<bf16>(), (int)R, d_gather, d_scores, stream);
}

// One step of the autoregressive `attention` decode mode (decoder.forward_one_step + logp.topk, search.py:302-306):
// the left decoder runs over the S = B*N running hypotheses of length L (sos first); the reference's per-layer
// output cache is an optimisation of the same computation, here the prefix is simply recomputed.
static int decoder_step_topk(rvb_model* m, const float* d_enc_out, const int* h_enc_lens, int B, int Tp, int N,
                             const int* h_hyps, int L, const float* h_cat, int n_cat, int k, float* h_val, int* h_idx,
                             cudaStream_t stream, float* h_logp = nullptr /* (S, V) full rows, optional */) {
  const rvb_model_config& c = m->cfg;
  RVB_REQUIRE(m->finalized && m->w.dec_l.present, "decoder_step_topk: model has no decoder");
  RVB_REQUIRE(L >= 1 && k >= 1 && k <= 16 && k <= c.vocab, "decoder_step_topk: bad L=%d / k=%d", L, k);
  const int S = B * N;
  const long long R = (long long)S * L, Mem = (long long)B * Tp;
  std::vector<int> grp;
  CatRows cr;
  if (cat_rows(m, true, h_cat, n_cat, B, &cr, &grp, stream)) return -1;
  const size_t ints = (size_t)R + S + 2 * B;   // tokens | lengths | encoder lengths | LSL groups
  const size_t out_bytes = (size_t)S * k * (sizeof(float) + sizeof(int));
  const size_t row_bytes = h_logp ? (size_t)S * c.vocab * sizeof(float) : 0;
  if (m->pin_b.ensure(ints * sizeof(int)) || m->ws_misc.ensure(ints * sizeof(int) + out_bytes) ||
      m->pin_c.ensure(out_bytes + row_bytes) || (h_logp && m->ws_step_rows.ensure(row_bytes)))
    return -1;
  int* hp = m->pin_b.as<int>();
  for (long long r = 0; r < R; ++r) {
    RVB_REQUIRE(h_hyps[r] >= 0 && h_hyps[r] < c.vocab, "decoder_step_topk: token id %d out of range", h_hyps[r]);
    hp[r] = h_hyps[r];
  }
  for (int s = 0; s < S; ++s) hp[R + s] = L;
  for (int b = 0; b < B; ++b) hp[R + S + b] = h_enc_lens[b];
  for (int b = 0; b < B; ++b) hp[R + S + B + b] = grp[b];
  int* dp = m->ws_misc.as<int>();
  cr.d_grp = dp + R + S + B;
  RVB_CHECK_CUDA(cudaMemcpyAsync(dp, hp, ints * sizeof(int), cudaMemcpyHostToDevice, stream));
  float* d_val = reinterpret_cast<float*>(dp + ints);
  int* d_idx = reinterpret_cast<int*>(d_val + (size_t)S * k);
  bf16* encbf;
  if (enc_operand(m, d_enc_out, Mem, &encbf, stream)) return -1;
  float* d_rows = h_logp ? m->ws_step_rows.as<float>() : nullptr;
  if (decoder_pass(m, m->w.dec_l, encbf, dp + R + S, B, Tp, N, L, dp, dp + R, nullptr, nullptr, cr, stream, k, d_val,
                   d_idx, d_rows))
    return -1;
  RVB_CHECK_CUDA(cudaMemcpyAsync(m->pin_c.p, d_val, out_bytes, cudaMemcpyDeviceToHost, stream));
  if (h_logp)
    RVB_CHECK_CUDA(cudaMemcpyAsync(reinterpret_cast<char*>(m->pin_c.p) + out_bytes, d_rows, row_bytes,
                                   cudaMemcpyDeviceToHost, stream));
  RVB_CHECK_CUDA(cudaStreamSynchronize(stream));
  memcpy(h_val, m->pin_c.p, (size_t)S * k * sizeof(float));
  memcpy(h_idx, reinterpret_cast<char*>(m->pin_c.p) + (size_t)S * k * sizeof(float), (size_t)S * k * sizeof(int));
  if (h_logp) memcpy(h_logp, reinterpret_cast<char*>(m->pin_c.p) + out_bytes, row_bytes);
  return 0;
}

// ---------------------------------------------------------------------------------------------------------------
// Autoregressive decoding with a KEY / VALUE cache (`attention` mode, search.py:251-360).  The reference's
// decoder.forward_one_step (decoder.py:191-234) caches each layer's OUTPUT for the previous positions and re-projects
// their self-attention keys / values every step; here the projected keys / values themselves are cached per layer
// ((S, Lcap, [k | v])), the source-attention keys / values of the encoder output are projected ONCE per utterance, and a
// step touches exactly one new position per hypothesis: every GEMM has M = S = B * N rows.  Beam reordering
// (torch.index_select of the caches, search.py:341-346) is a gather between two cache buffers.
struct DecCache {
  int B = 0, Tp = 0, N = 0, S = 0, Lcap = 0, step = 0;
  bool flip = false;
  std::vector<DevBuf> self_a, self_b, cross;  // per layer
  DevBuf ints;   // enc lens (B) | key counts (S) | tokens (S) | parents (S)
  DecRows rows;  // S rows (kv unused: `cross` holds the source-attention keys / values)
  DevBuf logits, outv;
  HostPinned pin;
  std::vector<float> cat;  // the distinct LSL mixing vectors of decoder_cache_begin, refolded (if need be) every step
  CatRows cr;              // their mixing of the cached utterances, the groups in grp
  DevBuf grp;
  HostPinned grp_pin;
};

static int decoder_cache_begin(rvb_model* m, const float* d_enc_out, const int* h_enc_lens, int B, int Tp, int N,
                               int Lcap, const float* h_cat, int n_cat, cudaStream_t stream) {
  const rvb_model_config& c = m->cfg;
  RVB_REQUIRE(m->finalized && m->w.dec_l.present, "decoder_cache_begin: model has no decoder");
  RVB_REQUIRE(B > 0 && Tp > 0 && N > 0 && Lcap > 0, "decoder_cache_begin: bad shape");
  if (m->dcache == nullptr) m->dcache.reset(new DecCache());
  DecCache& dc = *m->dcache;
  Decoder& D = m->w.dec_l;
  const int d = c.d_model, S = B * N;
  const size_t pm = (size_t)m->pm(), nl = D.layers.size();
  const long long Mem = (long long)B * Tp;
  std::vector<int> grp;
  if (cat_rows(m, true, h_cat, n_cat, B, &dc.cr, &grp, stream, &dc.cat)) return -1;
  if (dc.cr.G && upload_groups(grp, dc.grp_pin, dc.grp, stream)) return -1;
  dc.cr.d_grp = dc.grp.as<int>();
  dc.cr.rows_per_batch = N;
  dc.B = B; dc.Tp = Tp; dc.N = N; dc.S = S; dc.Lcap = Lcap; dc.step = 0; dc.flip = false;
  dc.self_a.resize(nl); dc.self_b.resize(nl); dc.cross.resize(nl);
  const size_t kvw = (size_t)2 * d * pm;  // cache row: [k | v] (x2 for the hi / lo pair layout)
  for (size_t l = 0; l < nl; ++l)
    if (dc.self_a[l].ensure((size_t)S * Lcap * kvw * 2) || dc.self_b[l].ensure((size_t)S * Lcap * kvw * 2) ||
        dc.cross[l].ensure((size_t)Mem * kvw * 2))
      return -1;
  const int ldv = (c.vocab + 3) & ~3;
  if (dc.ints.ensure(sizeof(int) * ((size_t)B + 3 * S)) || dc.rows.ensure(S, 0, d, c.dec_ffn_dim, pm) ||
      dc.logits.ensure((size_t)S * ldv * 4) || dc.outv.ensure((size_t)S * 16 * 8) ||
      dc.pin.ensure(sizeof(int) * ((size_t)B + 2 * S) + (size_t)S * 16 * 8))
    return -1;
  int* hp = dc.pin.as<int>();
  memcpy(hp, h_enc_lens, sizeof(int) * B);
  RVB_CHECK_CUDA(cudaMemcpyAsync(dc.ints.p, hp, sizeof(int) * B, cudaMemcpyHostToDevice, stream));
  bf16* encbf;
  if (enc_operand(m, d_enc_out, Mem, &encbf, stream)) return -1;
  for (size_t l = 0; l < nl; ++l)   // source-attention keys / values: once per utterance, not once per step
    if (gemm(m, encbf, D.layers[l].ckv, (int)Mem, ACT_NONE, OUT_BF16, dc.cross[l].p, 1.f, stream)) return -1;
  return 0;
}

// One position for every running hypothesis: tokens[s] = last token of hypothesis s, parents[s] = index (in the previous
// step's order) of the hypothesis it extends (nullptr / ignored at step 0).  -> log_softmax top-k of the new position.
static int decoder_cache_step(rvb_model* m, const int* h_tokens, const int* h_parents, int k, float* h_val, int* h_idx,
                              cudaStream_t stream) {
  const rvb_model_config& c = m->cfg;
  RVB_REQUIRE(m->dcache != nullptr && m->dcache->S > 0, "decoder_cache_step: call decoder_cache_begin first");
  DecCache& dc = *m->dcache;
  Decoder& D = m->w.dec_l;
  const int d = c.d_model, H = c.dec_heads, V = c.vocab, S = dc.S, B = dc.B, N = dc.N, pos = dc.step;
  RVB_REQUIRE(pos < dc.Lcap, "decoder_cache_step: step %d exceeds the cache capacity %d", pos, dc.Lcap);
  RVB_REQUIRE(k >= 1 && k <= 16 && k <= V, "decoder_cache_step: bad k=%d", k);
  const bool x3 = m->x3;
  const int pm = m->pm();
  const int kvw = 2 * d * pm;
  int* d_elen = dc.ints.as<int>();
  int* d_klen = d_elen + B;
  int* d_tok = d_klen + S;
  int* d_par = d_tok + S;
  int* hp = dc.pin.as<int>() + B;
  for (int s = 0; s < S; ++s) {
    RVB_REQUIRE(h_tokens[s] >= 0 && h_tokens[s] < V, "decoder_cache_step: token id %d out of range", h_tokens[s]);
    hp[s] = h_tokens[s];
    hp[S + s] = (h_parents && pos > 0) ? h_parents[s] : s;
    RVB_REQUIRE(hp[S + s] >= 0 && hp[S + s] < S, "decoder_cache_step: bad parent index");
  }
  RVB_CHECK_CUDA(cudaMemcpyAsync(d_tok, hp, sizeof(int) * 2 * S, cudaMemcpyHostToDevice, stream));
  if (launch_fill_int(d_klen, S, pos + 1, stream)) return -1;
  std::vector<DevBuf>& cur = dc.flip ? dc.self_b : dc.self_a;
  std::vector<DevBuf>& nxt = dc.flip ? dc.self_a : dc.self_b;
  const bool reorder = h_parents != nullptr && pos > 0;
  if (fold_stack(m, true, dc.cat, stream)) return -1;  // a call in between may have folded other vectors
  const CatRows& cr = dc.cr;
  bf16* qkv = dc.rows.qkv.as<bf16>();
  bf16* att = dc.rows.att.as<bf16>();
  if (launch_embed_posenc(d_tok, D.emb, S, 1, d, dc.rows.x.as<float>(), stream, pos)) return -1;
  auto self_attn = [&](size_t l) {
    bf16* cache = cur[l].as<bf16>();
    if (reorder) {  // the hypotheses were re-ranked: their histories follow (search.py:341-346)
      if (launch_kv_reorder(cache, nxt[l].as<bf16>(), d_par, S, dc.Lcap, pos, kvw, stream)) return -1;
      cache = nxt[l].as<bf16>();
    }
    // cache row = [k | v] = columns [d, 3d) of the projection (and their lo halves at +3d in the pair layout)
    if (launch_kv_append(qkv, 3 * d * pm, d, cache, S, dc.Lcap, pos, 2 * d, kvw, stream)) return -1;
    if (x3 && launch_kv_append(qkv, 3 * d * pm, 3 * d + d, cache + 2 * d, S, dc.Lcap, pos, 2 * d, kvw, stream)) return -1;
    DecAttn a;  // the new position over its own history
    a.q = qkv;
    a.k = cache;
    a.v = cache + d;
    a.out = att;
    a.ldq = 3 * d;
    a.ldk = a.ldv = 2 * d;
    a.ldo = d;
    a.groups = S;
    a.Tq = 1;
    a.Tk = dc.Lcap;  // group stride; the visible keys are [0, pos]
    a.H = H;
    a.dk = d / H;
    a.k_lens = d_klen;
    a.f32 = true;
    return dec_attention(m, a, stream);
  };
  auto src_attn = [&](size_t l) {
    DecAttn a = src_attention(qkv, dc.cross[l].as<bf16>(), att, d, B, N, dc.Tp, H, d_elen);
    a.f32 = true;
    return dec_attention(m, a, stream);
  };
  if (decoder_layers(m, D, dc.rows, S, cr, self_attn, src_attn, stream)) return -1;
  if (reorder) dc.flip = !dc.flip;
  float* d_val = dc.outv.as<float>();
  int* d_idx = reinterpret_cast<int*>(d_val + (size_t)S * k);
  if (last_position_topk(m, D, dc.rows.n.as<bf16>(), S, 1, dc.logits, k, d_val, d_idx, nullptr, stream)) return -1;
  char* hout = reinterpret_cast<char*>(dc.pin.as<int>() + B + 2 * S);
  const size_t out_bytes = (size_t)S * k * (sizeof(float) + sizeof(int));
  RVB_CHECK_CUDA(cudaMemcpyAsync(hout, d_val, out_bytes, cudaMemcpyDeviceToHost, stream));
  RVB_CHECK_CUDA(cudaStreamSynchronize(stream));
  memcpy(h_val, hout, (size_t)S * k * sizeof(float));
  memcpy(h_idx, hout + (size_t)S * k * sizeof(float), (size_t)S * k * sizeof(int));
  dc.step = pos + 1;
  return 0;
}

// 1 = prefix-tree rescoring (default), 0 = one decoder row per (hypothesis, position) (RVB_RESCORE=flat)
static int rescore_trie() {
  const char* e = getenv("RVB_RESCORE");   // read per call: tests / benchmarks flip it between calls
  return (e && strcmp(e, "flat") == 0) ? 0 : 1;
}

// The teacher-forced decoder over the PREFIX TREE of every utterance's n-best (ctc.cu trie_build_kernel): R = B * P rows,
// one per distinct prefix (P = node slots per utterance), instead of B * N * Lp.  d_scores (B*N, Lp): the same
// per-(hypothesis, position) log-probabilities decoder_pass produces.
struct TrieView {
  const int* node_of;
  int nstride;
  const int* node_tok;
  const int* node_par;
  const int* node_dep;
  int cap;
  const int* n_nodes;
};

static int decoder_pass_trie(rvb_model* m, Decoder& D, const bf16* enc_bf, const int* d_enc_lens, int B, int Tp, int N,
                             int Lp, int P, const TrieView& tv, const int* d_olen, const int* d_nhyp, float* d_scores,
                             const CatRows& cr, cudaStream_t stream) {
  const rvb_model_config& c = m->cfg;
  const int d = c.d_model, H = c.dec_heads, dk = d / H;
  const long long R = (long long)B * P, E = (long long)B * (P + N), Mem = (long long)B * Tp;
  const long long S = (long long)B * N;
  const size_t pm = (size_t)m->pm();
  // self-attention of the tree on the wgmma kernel: dense over the utterance's P node slots, causal tile range (a
  // parent always precedes its children) plus an ancestor bit mask; otherwise fp32 over ancestor lists
  const bool tc_self = wgmma_attn(m, dk) && !(getenv("RVB_TRIE_ATTN") && strcmp(getenv("RVB_TRIE_ATTN"), "list") == 0);
  const int bits_ld = 2 * ((P + 63) / 64);
  const size_t n_int = (size_t)R * 3 + (size_t)R * Lp + (size_t)E * 2 + (size_t)S * Lp + (tc_self ? (size_t)R * bits_ld : 0);
  DecRows& w = m->dec_rows;
  if (w.ensure(R, Mem, d, c.dec_ffn_dim, pm) || m->ws_tree_idx.ensure(n_int * sizeof(int)) ||
      m->ws_edge_rows.ensure((size_t)E * d * 2 * pm) || m->ws_edge_scores.ensure((size_t)E * sizeof(float)))
    return -1;
  bf16* qkv = w.qkv.as<bf16>();
  bf16* att = w.att.as<bf16>();
  bf16* kv = w.kv.as<bf16>();
  int* tok_in = m->ws_tree_idx.as<int>();
  int* pos = tok_in + R;
  int* alen = pos + R;
  int* anc = alen + R;
  int* src = anc + (size_t)R * Lp;
  int* tgt = src + E;
  int* smap = tgt + E;
  uint32_t* anc_bits = tc_self ? reinterpret_cast<uint32_t*>(smap + (size_t)S * Lp) : nullptr;
  bf16* a_out = m->ws_edge_rows.as<bf16>();
  float* e_sc = m->ws_edge_scores.as<float>();
  if (launch_trie_inputs(tv.node_of, tv.nstride, tv.node_tok, tv.node_par, tv.node_dep, tv.cap, tv.n_nodes, d_olen, d_nhyp,
                         B, N, P, Lp, eos_id(c), tok_in, pos, anc, alen, src, tgt, smap, stream, anc_bits, bits_ld))
    return -1;
  if (launch_embed_posenc_rows(tok_in, pos, D.emb, (int)R, d, w.x.as<float>(), stream)) return -1;
  auto self_attn = [&](size_t) {
    DecAttn a;  // every node over its ancestors (= the causal mask of the flat layout)
    a.q = qkv;
    a.k = qkv + d;
    a.v = qkv + 2 * d;
    a.out = att;
    a.ldq = a.ldk = a.ldv = 3 * d;
    a.ldo = d;
    a.H = H;
    a.dk = dk;
    a.scale = 1.0f / sqrtf((float)dk);
    if (tc_self) {
      a.groups = B;
      a.Tq = a.Tk = P;
      a.causal = true;
      a.key_bits = anc_bits;
      a.bits_ld = bits_ld;
    } else {
      a.groups = 1;
      a.Tq = (int)R;
      a.Tk = Lp;
      a.key_list = anc;
      a.key_list_len = alen;
      a.key_list_ld = Lp;
    }
    return dec_attention(m, a, stream);
  };
  auto src_attn = [&](size_t l) {  // K/V projected once per utterance
    if (gemm(m, enc_bf, D.layers[l].ckv, (int)Mem, ACT_NONE, OUT_BF16, kv, 1.f, stream)) return -1;
    return dec_attention(m, src_attention(qkv, kv, att, d, B, P, Tp, H, d_enc_lens), stream);
  };
  if (decoder_layers(m, D, w, (int)R, cr.rows(P), self_attn, src_attn, stream)) return -1;
  // output layer on one row per EDGE of the tree (+ one per hypothesis end): hidden state of the edge's source node
  if (launch_gather_rows(w.n.as<bf16>(), src, a_out, (int)E, d * (int)pm, stream)) return -1;
  if (target_logp(m, D, a_out, (int)E, tgt, e_sc, stream)) return -1;
  return launch_gather_scores(e_sc, smap, d_scores, S * Lp, stream);
}

// The flat decoder passes over a device n-best, one row per (hypothesis, position) with Lp positions per hypothesis.
// rescoring_inputs_kernel lays out, in idx (4 R + S ints, R = S * Lp), the decoder inputs tok_l / tok_r
// [sos, w_1..w_U, eos..] and the reversed variant (asr_model.py:921-949), the gather targets gat_l / gat_r (-1 = none,
// search.py:417-430) and slen = U + 1; absent hypotheses are empty.  -> d_sc_l / d_sc_r (R) log-probs of the targets.
static int rescoring_flat(rvb_model* m, const NBest& nb, const float* d_enc_out, int Tp, int Lp, bool use_r, int* idx,
                          float* d_sc_l, float* d_sc_r, const CatRows& cr, cudaStream_t stream) {
  const NBest::Arrays d = nb.d();
  const size_t R = nb.S() * Lp;
  int *tok_l = idx, *tok_r = idx + R, *gat_l = idx + 2 * R, *gat_r = idx + 3 * R, *slen = idx + 4 * R;
  if (launch_rescoring_inputs(d.tok, nb.len_cap, d.olen, d.nhyp, nb.B, nb.beam, Lp, sos_id(m->cfg), eos_id(m->cfg), tok_l,
                              tok_r, gat_l, gat_r, slen, stream))
    return -1;
  bf16* encbf;
  if (enc_operand(m, d_enc_out, (long long)nb.B * Tp, &encbf, stream)) return -1;
  if (decoder_pass(m, m->w.dec_l, encbf, d.lens, nb.B, Tp, nb.beam, Lp, tok_l, slen, gat_l, d_sc_l, cr, stream)) return -1;
  if (use_r && decoder_pass(m, m->w.dec_r, encbf, d.lens, nb.B, Tp, nb.beam, Lp, tok_r, slen, gat_r, d_sc_r, cr, stream))
    return -1;
  return 0;
}

// Position j < U of the right-to-left pass scores token w_{U-1-j}: reverse [0, U) of every row in place to put the
// scores in hypothesis order.  Position U (eos) stays; positions past it are 0 from the device (gather target -1).
static void unreverse_r2l(const NBest& nb, int Lp, float* r2l) {
  for (size_t s = 0; s < nb.S(); ++s) std::reverse(r2l + s * Lp, r2l + s * Lp + nb.ntok(s));
}

static int attention_rescoring(rvb_model* m, const float* d_enc_out, const int* h_enc_lens, int B, int Tp,
                               const int* h_tok, const int* h_len, int N, int max_len, const float* h_cat, int n_cat,
                               float reverse_weight, float* h_l2r, float* h_r2l, cudaStream_t stream) {
  RVB_REQUIRE(m->finalized && m->w.dec_l.present, "attention_rescoring: model has no decoder");
  const int Lp = max_len + 1, S = B * N;
  const long long R = (long long)S * Lp;
  const bool use_r = reverse_weight > 0.f && m->w.dec_r.present && h_r2l != nullptr;
  std::vector<int> grp;
  CatRows cr;
  if (cat_rows(m, true, h_cat, n_cat, B, &cr, &grp, stream)) return -1;
  if (cr.G && upload_groups(grp, m->pin_grp, m->ws_grp, stream)) return -1;
  cr.d_grp = m->ws_grp.as<int>();
  // the caller's hypotheses as an n-best with every slot present: an absent row (length < 0) is an empty hypothesis
  NBest& nb = m->nbest_in;
  const size_t rints = (size_t)R * 4 + S;
  if (nb.ensure(B, N, max_len) || m->ws_misc.ensure(rints * sizeof(int) + (size_t)R * 2 * sizeof(float)) ||
      m->pin_c.ensure((size_t)R * 2 * sizeof(float)))
    return -1;
  const NBest::Arrays h = nb.h();
  memcpy(h.lens, h_enc_lens, sizeof(int) * B);
  memcpy(h.tok, h_tok, sizeof(int) * S * max_len);
  for (int s = 0; s < S; ++s) {
    const int U = h_len[s] < 0 ? 0 : h_len[s];
    RVB_REQUIRE(U <= max_len, "attention_rescoring: hypothesis longer than max_len");
    h.olen[2 * s] = U;
    h.olen[2 * s + 1] = 0;
  }
  for (int b = 0; b < B; ++b) h.nhyp[b] = N;
  RVB_CHECK_CUDA(cudaMemcpyAsync(nb.d().lens, h.lens, nb.upload_bytes(), cudaMemcpyHostToDevice, stream));
  int* idx = m->ws_misc.as<int>();
  float* d_sc_l = reinterpret_cast<float*>(idx + rints);
  float* d_sc_r = d_sc_l + R;
  if (rescoring_flat(m, nb, d_enc_out, Tp, Lp, use_r, idx, d_sc_l, d_sc_r, cr, stream)) return -1;
  float* hs = m->pin_c.as<float>();
  RVB_CHECK_CUDA(cudaMemcpyAsync(hs, d_sc_l, (size_t)R * (use_r ? 2 : 1) * sizeof(float), cudaMemcpyDeviceToHost,
                                 stream));
  RVB_CHECK_CUDA(cudaStreamSynchronize(stream));
  memcpy(h_l2r, hs, (size_t)R * sizeof(float));
  if (use_r) {
    unreverse_r2l(nb, Lp, hs + R);
    memcpy(h_r2l, hs + R, (size_t)R * sizeof(float));
  }
  return 0;
}

// ctc_prefix_beam_search + attention_rescoring with the n-best kept on the device in between (asr_model.py:259-308 does
// the same two steps through Python lists), split into three host calls around a TICKET so that consecutive batches
// can be software-pipelined on one stream by one host thread (no GPU idle time while the host picks the decoder batch):
//   search_submit     enqueue the prefix beam search + the small D2H copy (hypothesis lengths / counts / CTC scores)
//   rescoring_submit  wait for that copy (the ONLY data-dependent host decision of the path: the decoder batch is
//                     padded to the longest hypothesis), enqueue decoder-input assembly, the decoder passes and the
//                     D2H copies of tokens / times / decoder scores straight into the caller's (pinned) buffers
//   rescoring_collect wait for those copies, hand out the small arrays
// Between the calls the host is free to enqueue the NEXT batch's encoder, so the GPU always has a full step queued
// while the host waits for lengths or post-processes results.  Buffers that live across calls belong to the ticket.
struct SearchTicket {
  int state = 0;      // 0 free, 1 search submitted, 2 decoder submitted
  NBest nb;           // rows of Tp tokens: a prefix never has more tokens than frames
  DevBuf trie;        // prefix trees of the n-best (left-to-right and reversed): node_of | node_tok | par | dep | n_nodes
  HostPinned nodes;   // n_nodes of each tree (B per direction)
  int trie_cap = 0, trie_stride = 0;
  bool has_trie = false, has_rtrie = false;
  int* tr_node_of(int dir) { return trie.as<int>() + (size_t)dir * trie_ints(); }
  size_t trie_ints() const { return nb.S() * trie_stride + (size_t)3 * nb.B * trie_cap + nb.B; }
  TrieView trie_view(int dir) {
    int* base = tr_node_of(dir);
    TrieView v;
    v.node_of = base;
    v.nstride = trie_stride;
    v.node_tok = base + nb.S() * trie_stride;
    v.node_par = const_cast<int*>(v.node_tok) + (size_t)nb.B * trie_cap;
    v.node_dep = const_cast<int*>(v.node_par) + (size_t)nb.B * trie_cap;
    v.cap = trie_cap;
    v.n_nodes = const_cast<int*>(v.node_dep) + (size_t)nb.B * trie_cap;
    return v;
  }
  cudaEvent_t ev_search = nullptr, ev_done = nullptr;
  int Tp = 0;
  const float* d_enc_out = nullptr;
  int Lmax = 1;
  bool use_r = false;
  float* h_r2l = nullptr;
  DevBuf grp;          // LSL groups of the batch's utterances (per-utterance cat_embs)
  HostPinned grp_pin;
  ~SearchTicket() {
    if (ev_search) cudaEventDestroy(ev_search);
    if (ev_done) cudaEventDestroy(ev_done);
  }
};

int search_side_stream(rvb_model* m, cudaStream_t* out) {
  if (m->s_search == nullptr) RVB_CHECK_CUDA(cudaStreamCreateWithFlags(&m->s_search, cudaStreamNonBlocking));
  *out = m->s_search;
  return 0;
}

// The CTC prefix beam search into nb (rows of nb.len_cap tokens) on `stream`, with workspace ws: zeroes every output
// (token / time rows read 0 past a hypothesis' end, whatever the buffer held before), uploads the encoder lengths
// through nb's host mirror, then searches, context-biased when graph != nullptr.
static int prefix_beam_into(NBest& nb, const float* d_topk_val, const int* d_topk_idx, int k, const int* h_enc_lens,
                            int Tp, int blank_id, DevBuf& ws, ::rvb_context_graph* graph, cudaStream_t stream) {
  const NBest::Arrays d = nb.d(), h = nb.h();
  if (ws.ensure(prefix_beam_workspace_bytes(nb.B, Tp, nb.beam))) return -1;
  RVB_CHECK_CUDA(cudaMemsetAsync(d.tim, 0, (size_t)(d.nhyp + nb.B - d.tim) * sizeof(int), stream));
  memcpy(h.lens, h_enc_lens, sizeof(int) * nb.B);
  RVB_CHECK_CUDA(cudaMemcpyAsync(d.lens, h.lens, sizeof(int) * nb.B, cudaMemcpyHostToDevice, stream));
  if (graph == nullptr)
    return launch_ctc_prefix_beam(d_topk_val, d_topk_idx, k, d.lens, nb.B, Tp, nb.beam, blank_id, ws.p, ws.cap,
                                  nb.len_cap, d.tok, d.tim, d.olen, d.sc, d.nhyp, stream);
  if (launch_ctc_prefix_beam_biased(d_topk_val, d_topk_idx, k, d.lens, nb.B, Tp, nb.beam, blank_id, ws.p, ws.cap,
                                    nb.len_cap, d.tok, d.tim, d.olen, d.sc, d.nhyp, *context_graph_view(graph), stream))
    return -1;
  return context_graph_note_use(graph, stream);
}

// graph != nullptr: the biased search (context biasing with that graph)
static int search_submit(rvb_model* m, SearchTicket& t, const float* d_topk_val, const int* d_topk_idx, int k,
                         const float* d_enc_out, const int* h_enc_lens, int B, int Tp, int beam, int blank_id,
                         ::rvb_context_graph* graph, cudaStream_t stream) {
  t.Tp = Tp;
  t.d_enc_out = d_enc_out;
  // prefix trees of the n-best for the tree-structured rescoring decoder (left-to-right, and reversed when the model
  // has a right-to-left decoder): built right behind the search, their node counts travel with the lengths
  t.has_trie = rescore_trie() && m->w.dec_l.present && beam <= 16;
  t.has_rtrie = t.has_trie && m->w.dec_r.present;
  t.trie_stride = Tp + 1;
  t.trie_cap = beam * Tp + 1;
  const int ndir = t.has_trie ? (t.has_rtrie ? 2 : 1) : 0;
  if (t.nb.ensure(B, beam, Tp) || t.nodes.ensure(sizeof(int) * B * 2) ||
      (ndir && t.trie.ensure(t.trie_ints() * ndir * sizeof(int))))
    return -1;
  if (!t.ev_search) RVB_CHECK_CUDA(cudaEventCreateWithFlags(&t.ev_search, cudaEventDisableTiming));
  if (!t.ev_done) RVB_CHECK_CUDA(cudaEventCreateWithFlags(&t.ev_done, cudaEventDisableTiming));
  // The search runs on a SIDE stream: it is one CTA per utterance (64 of 132 SMs, latency-bound), so
  // in a pipelined decode the next batch's fbank / conv1 (bandwidth-bound, small CTAs) share the GPU with it instead of
  // queueing behind it.  The side stream starts after everything enqueued so far on `stream` (the CTC top-k);
  // rescoring_submit makes `stream` wait for ev_search before it touches the n-best.
  static int side = -1;
  if (side < 0) {
    const char* e = getenv("RVB_SEARCH_STREAM");   // RVB_SEARCH_STREAM=main: keep the search on the caller's stream
    side = (e && strcmp(e, "main") == 0) ? 0 : 1;
  }
  cudaStream_t ss = stream;
  if (side) {
    if (search_side_stream(m, &ss)) return -1;
    if (m->ev_topk == nullptr) RVB_CHECK_CUDA(cudaEventCreateWithFlags(&m->ev_topk, cudaEventDisableTiming));
    RVB_CHECK_CUDA(cudaEventRecord(m->ev_topk, stream));
    RVB_CHECK_CUDA(cudaStreamWaitEvent(ss, m->ev_topk, 0));
  }
  if (prefix_beam_into(t.nb, d_topk_val, d_topk_idx, k, h_enc_lens, Tp, blank_id, m->ws_search, graph, ss)) return -1;
  const NBest::Arrays d = t.nb.d();
  RVB_CHECK_CUDA(cudaMemcpyAsync(t.nb.h().olen, d.olen, t.nb.small_bytes(), cudaMemcpyDeviceToHost, ss));
  for (int dir = 0; dir < ndir; ++dir) {
    TrieView v = t.trie_view(dir);
    if (launch_trie_build(d.tok, Tp, d.olen, d.nhyp, B, beam, dir, sos_id(m->cfg), const_cast<int*>(v.node_of),
                          v.nstride, const_cast<int*>(v.node_tok), const_cast<int*>(v.node_par),
                          const_cast<int*>(v.node_dep), v.cap, const_cast<int*>(v.n_nodes), ss))
      return -1;
    RVB_CHECK_CUDA(cudaMemcpyAsync(t.nodes.as<int>() + B * dir, v.n_nodes, sizeof(int) * B, cudaMemcpyDeviceToHost, ss));
  }
  RVB_CHECK_CUDA(cudaEventRecord(t.ev_search, ss));
  t.state = 1;
  return 0;
}

// run_decoder == 0: ctc_prefix_beam_search only (tokens / times are copied, no decoder scores)
static int rescoring_submit(rvb_model* m, SearchTicket& t, const float* h_cat, int n_cat, float reverse_weight, int cap,
                            int run_decoder, int* h_tokens, int* h_times, float* h_l2r, float* h_r2l, int* out_max_len,
                            cudaStream_t stream) {
  RVB_REQUIRE(t.state == 1, "rescoring_submit: ticket has no submitted search");
  const int B = t.nb.B, N = t.nb.beam, S = B * N, Tp = t.Tp;
  RVB_CHECK_CUDA(cudaEventSynchronize(t.ev_search));
  RVB_CHECK_CUDA(cudaStreamWaitEvent(stream, t.ev_search, 0));   // the n-best was produced on the side stream
  const NBest::Arrays d = t.nb.d();
  const int* ol = t.nb.h().olen;
  const int* nh = t.nb.h().nhyp;
  int Lmax = 1;
  for (int b = 0; b < B; ++b)
    for (int i = 0; i < N; ++i) {
      const size_t s = (size_t)b * N + i;
      if (i < nh[b]) {
        Lmax = ol[2 * s] > Lmax ? ol[2 * s] : Lmax;
        Lmax = ol[2 * s + 1] > Lmax ? ol[2 * s + 1] : Lmax;
      }
    }
  RVB_REQUIRE(Lmax <= cap && Lmax <= Tp, "beam_search_rescoring: hypothesis of %d tokens exceeds capacity %d", Lmax, cap);
  *out_max_len = Lmax;
  t.Lmax = Lmax;
  // n-best tokens / times -> caller's host buffers (compact rows of Lmax), overlapping the decoder on the copy engine
  RVB_CHECK_CUDA(cudaMemcpy2DAsync(h_tokens, (size_t)Lmax * sizeof(int), d.tok, (size_t)Tp * sizeof(int),
                                   (size_t)Lmax * sizeof(int), (size_t)S, cudaMemcpyDeviceToHost, stream));
  RVB_CHECK_CUDA(cudaMemcpy2DAsync(h_times, (size_t)Lmax * sizeof(int), d.tim, (size_t)Tp * sizeof(int),
                                   (size_t)Lmax * sizeof(int), (size_t)S, cudaMemcpyDeviceToHost, stream));
  t.use_r = false;
  t.h_r2l = nullptr;
  if (run_decoder) {
    RVB_REQUIRE(m->finalized && m->w.dec_l.present, "beam_search_rescoring: model has no decoder");
    std::vector<int> grp;
    CatRows cr;
    if (cat_rows(m, true, h_cat, n_cat, B, &cr, &grp, stream)) return -1;
    if (cr.G && upload_groups(grp, t.grp_pin, t.grp, stream)) return -1;
    cr.d_grp = t.grp.as<int>();
    const int Lp = Lmax + 1;
    const long long R = (long long)S * Lp;
    const bool use_r = reverse_weight > 0.f && m->w.dec_r.present && h_r2l != nullptr;
    const size_t rints = (size_t)R * 4 + S;
    if (m->ws_misc.ensure(rints * sizeof(int) + (size_t)R * 2 * sizeof(float))) return -1;
    int* dp = m->ws_misc.as<int>();
    float* d_sc_l = reinterpret_cast<float*>(dp + rints);
    float* d_sc_r = d_sc_l + R;
    if (t.has_trie && (!use_r || t.has_rtrie)) {
      // tree-structured decoder: one row per distinct prefix of the utterance's n-best
      const int* hp_nodes = t.nodes.as<int>();
      bf16* encbf;
      if (enc_operand(m, t.d_enc_out, (long long)B * Tp, &encbf, stream)) return -1;
      for (int dir = 0; dir < (use_r ? 2 : 1); ++dir) {
        int P = 1;
        for (int b = 0; b < B; ++b) P = hp_nodes[dir * B + b] > P ? hp_nodes[dir * B + b] : P;
        P = (P + 7) & ~7;
        if (decoder_pass_trie(m, dir ? m->w.dec_r : m->w.dec_l, encbf, d.lens, B, Tp, N, Lp, P, t.trie_view(dir), d.olen,
                              d.nhyp, dir ? d_sc_r : d_sc_l, cr, stream))
          return -1;
      }
    } else if (rescoring_flat(m, t.nb, t.d_enc_out, Tp, Lp, use_r, dp, d_sc_l, d_sc_r, cr, stream)) {
      return -1;
    }
    RVB_CHECK_CUDA(cudaMemcpyAsync(h_l2r, d_sc_l, (size_t)R * sizeof(float), cudaMemcpyDeviceToHost, stream));
    if (use_r) {
      RVB_CHECK_CUDA(cudaMemcpyAsync(h_r2l, d_sc_r, (size_t)R * sizeof(float), cudaMemcpyDeviceToHost, stream));
      t.use_r = true;
      t.h_r2l = h_r2l;
    }
  }
  RVB_CHECK_CUDA(cudaEventRecord(t.ev_done, stream));
  t.state = 2;
  return 0;
}

static int rescoring_collect(SearchTicket& t, int* h_lens, double* h_scores, int* h_nhyp) {
  RVB_REQUIRE(t.state == 2, "rescoring_collect: ticket has no submitted decoder pass");
  RVB_CHECK_CUDA(cudaEventSynchronize(t.ev_done));
  const NBest::Arrays h = t.nb.h();
  memcpy(h_lens, h.olen, t.nb.S() * 2 * sizeof(int));
  memcpy(h_nhyp, h.nhyp, sizeof(int) * t.nb.B);
  memcpy(h_scores, h.sc, t.nb.S() * sizeof(double));
  if (t.use_r) unreverse_r2l(t.nb, t.Lmax + 1, t.h_r2l);
  t.state = 0;
  return 0;
}

}  // namespace rvb

// the buffers, the tickets and the decoder cache free themselves; a fork's weights belong to the parent's store
rvb_model::~rvb_model() {
  if (s_search) cudaStreamDestroy(s_search);
  if (ev_topk) cudaEventDestroy(ev_topk);
}

// ================================================================================================================
// C ABI
extern "C" {

RVB_API const char* rvb_last_error(void) { return rvb::last_error(); }
RVB_API unsigned long long rvb_launch_count(void) { return rvb::g_launch_count.load(); }
RVB_API int rvb_held_bytes(long long* device, long long* pinned) {
  RVB_REQUIRE(device && pinned, "rvb_held_bytes: bad arguments");
  *device = rvb::g_held_device.load();
  *pinned = rvb::g_held_pinned.load();
  return 0;
}
RVB_API int rvb_set_gemm_impl(int impl) {
  rvb::set_gemm_impl(impl);
  return 0;
}
RVB_API int rvb_get_gemm_impl(void) { return rvb::get_gemm_impl(); }
RVB_API int rvb_gemm_profile_begin(void) {
  rvb::gemm_profile_begin();
  return 0;
}
RVB_API int rvb_gemm_profile_end(double* total_ms, double* total_flops, long long* launches) {
  return rvb::gemm_profile_end(total_ms, total_flops, launches);
}

RVB_API rvb_model* rvb_model_create(const rvb_model_config* cfg) {
  if (cfg == nullptr) {
    rvb::set_error("rvb_model_create: null config");
    return nullptr;
  }
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
    rvb::set_error("rvb_model_create: no CUDA device (this library has no CPU path)");
    return nullptr;
  }
  if (cfg->precision != 0 && cfg->precision != 1) {
    rvb::set_error("rvb_model_create: precision must be 0 (bf16) or 1 (bf16x3, fp32-accurate)");
    return nullptr;
  }
  rvb_model* m = new rvb_model();
  m->cfg = *cfg;
  m->x3 = cfg->precision == 1;
  return m;
}

RVB_API int rvb_model_set_tensor(rvb_model* m, const char* name, const float* h_data, long long numel) {
  RVB_REQUIRE(m && name && h_data && numel >= 0, "rvb_model_set_tensor: bad arguments");
  RVB_REQUIRE(!m->finalized, "rvb_model_set_tensor: model already finalized");
  m->store.set(name, h_data, (size_t)numel);
  return 0;
}

RVB_API int rvb_model_finalize(rvb_model* m) {
  RVB_REQUIRE(m != nullptr, "rvb_model_finalize: null model");
  if (m->finalized) return 0;
  return rvb::finalize_model(m);
}

// A second plan over the SAME packed weights with its own workspace (and its own language-specific folds, made by its
// calls), so two host threads / CUDA streams can decode different batches concurrently.  The parent must outlive
// its forks.
RVB_API rvb_model* rvb_model_fork(rvb_model* m) {
  if (m == nullptr || !m->finalized) {
    rvb::set_error("rvb_model_fork: model not finalized");
    return nullptr;
  }
  rvb_model* f = new rvb_model();
  f->cfg = m->cfg;
  f->x3 = m->x3;
  f->finalized = true;
  f->w = m->w;
  return f;
}

RVB_API void rvb_model_destroy(rvb_model* m) {
  if (!m) return;
  delete m;
}

RVB_API int rvb_encoder_out_frames(int T) {
  if (T < 3) return 0;
  int t1 = (T - 1) / 2;
  return t1 < 1 ? 0 : (t1 - 1) / 2;
}

RVB_API int rvb_encoder_out_len(int feat_len, int T) {
  // x_mask[:, :, 2::2][:, :, 2::2] (transformer/subsampling.py:226): output frame j is valid iff 4j + 6 < feat_len
  int Tp = rvb_encoder_out_frames(T);
  if (feat_len > T) feat_len = T;
  int e = feat_len >= 7 ? (feat_len - 3) / 4 : 0;
  return e < Tp ? e : Tp;
}

RVB_API long long rvb_fbank_num_frames(long long n_samples) { return n_samples < 400 ? 0 : 1 + (n_samples - 400) / 160; }

RVB_API int rvb_fbank_f32(const float* d_wave, long long n_samples, float* d_feats, long long n_frames, void* stream) {
  return rvb::launch_fbank(d_wave, n_samples, d_feats, n_frames, (cudaStream_t)stream);
}
RVB_API int rvb_fbank_i16(const short* d_wave, long long n_samples, float* d_feats, long long n_frames, void* stream) {
  return rvb::launch_fbank_i16(d_wave, n_samples, d_feats, n_frames, (cudaStream_t)stream);
}

RVB_API int rvb_fbank_batch(const void* d_wave, int is_i16, int batch, long long wave_stride, long long n_samples,
                            float* d_feats, long long n_frames, void* stream) {
  return rvb::launch_fbank_batch(d_wave, is_i16, batch, wave_stride, n_samples, d_feats, n_frames,
                                 (cudaStream_t)stream);
}

RVB_API int rvb_encoder_forward(rvb_model* m, const float* d_feats, const int* h_feat_lens, int B, int T,
                        const float* h_cat_embs, int n_cat, float* d_enc_out, int* h_enc_lens, void* stream) {
  RVB_REQUIRE(m && d_feats && h_feat_lens && d_enc_out && B > 0, "rvb_encoder_forward: bad arguments");
  return rvb::encoder_forward(m, d_feats, h_feat_lens, B, T, h_cat_embs, n_cat, d_enc_out, h_enc_lens,
                              (cudaStream_t)stream);
}

RVB_API int rvb_encoder_forward_chunked(rvb_model* m, const float* d_feats, const int* h_feat_lens, int B, int T,
                                        const float* h_cat_embs, int n_cat, int chunk_size, int num_left_chunks,
                                        float* d_enc_out, int* h_enc_lens, void* stream) {
  RVB_REQUIRE(m && d_feats && h_feat_lens && d_enc_out && B > 0 && chunk_size > 0,
              "rvb_encoder_forward_chunked: bad arguments");
  return rvb::encoder_forward(m, d_feats, h_feat_lens, B, T, h_cat_embs, n_cat, d_enc_out, h_enc_lens,
                              (cudaStream_t)stream, chunk_size, num_left_chunks);
}

// BaseEncoder.forward_chunk_by_chunk (encoder.py:341-402) in ONE batched pass: the chunk mask inside the attention
// kernel reproduces the attention cache (a query sees the `left` previous chunks + its own), causal convolutions see
// the same left context as through the reference's cnn cache, non-causal ones are evaluated chunk by chunk (zero
// padded at the chunk edges); there are no padding masks on this path — every frame of the (B, T, .) input is real.
RVB_API int rvb_encoder_forward_streaming(rvb_model* m, const float* d_feats, int B, int T, const float* h_cat_embs,
                                          int n_cat, int chunk_size, int num_left_chunks, float* d_enc_out,
                                          int* h_enc_lens, void* stream) {
  RVB_REQUIRE(m && d_feats && d_enc_out && B > 0 && chunk_size > 0, "rvb_encoder_forward_streaming: bad arguments");
  std::vector<int> lens(B, T);
  return rvb::encoder_forward(m, d_feats, lens.data(), B, T, h_cat_embs, n_cat, d_enc_out, h_enc_lens,
                              (cudaStream_t)stream, chunk_size, num_left_chunks, true);
}

RVB_API int rvb_resample(const void* d_wave, int is_i16, long long n_in, const float* d_kernel, int orig, int new_, int width,
                         float* d_out, long long n_out, void* stream) {
  RVB_REQUIRE(d_wave && d_kernel && d_out && n_in >= 0, "rvb_resample: bad arguments");
  return rvb::launch_resample(d_wave, is_i16, n_in, d_kernel, orig, new_, width, d_out, n_out, (cudaStream_t)stream);
}

RVB_API int rvb_ctc_topk(rvb_model* m, const float* d_enc_out, int B, int Tp, int k, float blank_penalty, int blank_id,
                 float* d_topk_val, int* d_topk_idx, float* d_logp, void* stream) {
  RVB_REQUIRE(m && m->finalized && d_enc_out && d_topk_val && d_topk_idx && B > 0 && Tp > 0, "rvb_ctc_topk: bad arguments");
  return rvb::ctc_topk(m, d_enc_out, B, Tp, k, blank_penalty, blank_id, d_topk_val, d_topk_idx, d_logp,
                       (cudaStream_t)stream);
}

RVB_API int rvb_logp_topk(const float* d_logp, int rows, int V, int k, float* d_topk_val, int* d_topk_idx, void* stream) {
  return rvb::launch_logsoftmax_topk(d_logp, V, rows, V, k, d_topk_val, d_topk_idx, nullptr, 0, (cudaStream_t)stream);
}

// per host thread: two decoding lanes (threads) may run the searches concurrently.  The model-less synchronous
// searches only: the prefix beam search (workspace, n-best) and the greedy search (outputs, host copy).  Freed when
// the thread exits.
static thread_local rvb::DevBuf g_search_ws, g_search_out;
static thread_local rvb::HostPinned g_search_pin;
static thread_local rvb::NBest g_search_nb;

RVB_API int rvb_ctc_greedy_search(const int* d_topk_idx, int k, const int* h_enc_lens, int B, int Tp, int blank_id,
                          int* h_tokens, int* h_lens, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  RVB_REQUIRE(d_topk_idx && h_enc_lens && h_tokens && h_lens && B > 0 && Tp > 0, "rvb_ctc_greedy_search: bad arguments");
  const size_t n_out = (size_t)B * Tp + B;
  if (g_search_out.ensure((n_out + B) * sizeof(int)) || g_search_pin.ensure((n_out + B) * sizeof(int))) return -1;
  int* d_lens = g_search_out.as<int>();
  int* d_tok = d_lens + B;
  int* d_olen = d_tok + (size_t)B * Tp;
  int* hp = g_search_pin.as<int>();
  memcpy(hp, h_enc_lens, sizeof(int) * B);
  RVB_CHECK_CUDA(cudaMemcpyAsync(d_lens, hp, sizeof(int) * B, cudaMemcpyHostToDevice, stream));
  if (rvb::launch_ctc_greedy(d_topk_idx, k, d_lens, B, Tp, blank_id, d_tok, d_olen, stream)) return -1;
  RVB_CHECK_CUDA(cudaMemcpyAsync(hp + B, d_tok, n_out * sizeof(int), cudaMemcpyDeviceToHost, stream));
  RVB_CHECK_CUDA(cudaStreamSynchronize(stream));
  memcpy(h_tokens, hp + B, (size_t)B * Tp * sizeof(int));
  memcpy(h_lens, hp + B + (size_t)B * Tp, sizeof(int) * B);
  return 0;
}

static int prefix_beam_search(const float* d_topk_val, const int* d_topk_idx, int k, const int* h_enc_lens, int B, int Tp,
                              int beam, int blank_id, int max_len, int* h_tokens, int* h_times, int* h_lens,
                              double* h_scores, int* h_nhyp, rvb_context_graph* graph, cudaStream_t stream) {
  RVB_REQUIRE(d_topk_val && d_topk_idx && h_enc_lens && h_tokens && h_times && h_lens && h_scores && h_nhyp && B > 0 &&
                  Tp > 0 && max_len > 0,
              "rvb_ctc_prefix_beam_search: bad arguments");
  rvb::NBest& nb = g_search_nb;
  if (nb.ensure(B, beam, max_len)) return -1;
  const rvb::NBest::Arrays h = nb.h();
  if (rvb::prefix_beam_into(nb, d_topk_val, d_topk_idx, k, h_enc_lens, Tp, blank_id, g_search_ws, graph, stream))
    return -1;
  RVB_CHECK_CUDA(cudaMemcpyAsync(nb.host.p, nb.dev.p, nb.bytes(), cudaMemcpyDeviceToHost, stream));
  RVB_CHECK_CUDA(cudaStreamSynchronize(stream));
  const size_t n_tok = nb.S() * max_len;
  memcpy(h_tokens, h.tok, n_tok * sizeof(int));
  memcpy(h_times, h.tim, n_tok * sizeof(int));
  memcpy(h_lens, h.olen, nb.S() * 2 * sizeof(int));
  memcpy(h_nhyp, h.nhyp, sizeof(int) * B);
  memcpy(h_scores, h.sc, nb.S() * sizeof(double));
  for (size_t i = 0; i < (size_t)B * beam; ++i) {
    RVB_REQUIRE(h_lens[2 * i] <= max_len && h_lens[2 * i + 1] <= max_len,
                "rvb_ctc_prefix_beam_search: hypothesis of %d tokens exceeds max_len=%d", h_lens[2 * i], max_len);
  }
  return 0;
}

RVB_API int rvb_ctc_prefix_beam_search(const float* d_topk_val, const int* d_topk_idx, int k, const int* h_enc_lens, int B,
                               int Tp, int beam, int blank_id, int max_len, int* h_tokens, int* h_times, int* h_lens,
                               double* h_scores, int* h_nhyp, void* stream) {
  return prefix_beam_search(d_topk_val, d_topk_idx, k, h_enc_lens, B, Tp, beam, blank_id, max_len, h_tokens, h_times,
                            h_lens, h_scores, h_nhyp, nullptr, (cudaStream_t)stream);
}

RVB_API int rvb_ctc_prefix_beam_search_biased(const float* d_topk_val, const int* d_topk_idx, int k,
                                              const int* h_enc_lens, int B, int Tp, int beam, int blank_id, int max_len,
                                              int* h_tokens, int* h_times, int* h_lens, double* h_scores, int* h_nhyp,
                                              rvb_context_graph* graph, void* stream) {
  RVB_REQUIRE(graph != nullptr, "rvb_ctc_prefix_beam_search_biased: no context graph");
  return prefix_beam_search(d_topk_val, d_topk_idx, k, h_enc_lens, B, Tp, beam, blank_id, max_len, h_tokens, h_times,
                            h_lens, h_scores, h_nhyp, graph, (cudaStream_t)stream);
}

static rvb::SearchTicket* ticket_of(rvb_model* m, int id) {
  if (m == nullptr || m->tickets == nullptr || id < 0 || id >= rvb_model::kTickets) return nullptr;
  return &m->tickets[id];
}

static int search_submit_any(rvb_model* m, const float* d_topk_val, const int* d_topk_idx, int k, const float* d_enc_out,
                             const int* h_enc_lens, int B, int Tp, int beam, int blank_id, rvb_context_graph* graph,
                             void* stream) {
  RVB_REQUIRE(m && d_topk_val && d_topk_idx && d_enc_out && h_enc_lens && B > 0 && Tp > 0 && beam > 0,
              "rvb_search_submit: bad arguments");
  if (m->tickets == nullptr) m->tickets.reset(new rvb::SearchTicket[rvb_model::kTickets]);
  int id = -1;
  for (int i = 0; i < rvb_model::kTickets; ++i)
    if (m->tickets[i].state == 0) {
      id = i;
      break;
    }
  RVB_REQUIRE(id >= 0, "rvb_search_submit: all %d tickets of this plan are in flight (collect one first)",
              rvb_model::kTickets);
  if (rvb::search_submit(m, m->tickets[id], d_topk_val, d_topk_idx, k, d_enc_out, h_enc_lens, B, Tp, beam, blank_id,
                         graph, (cudaStream_t)stream)) {
    m->tickets[id].state = 0;
    return -1;
  }
  return id;
}

RVB_API int rvb_search_submit(rvb_model* m, const float* d_topk_val, const int* d_topk_idx, int k, const float* d_enc_out,
                              const int* h_enc_lens, int B, int Tp, int beam, int blank_id, void* stream) {
  return search_submit_any(m, d_topk_val, d_topk_idx, k, d_enc_out, h_enc_lens, B, Tp, beam, blank_id, nullptr, stream);
}

RVB_API int rvb_search_submit_biased(rvb_model* m, const float* d_topk_val, const int* d_topk_idx, int k,
                                     const float* d_enc_out, const int* h_enc_lens, int B, int Tp, int beam, int blank_id,
                                     rvb_context_graph* graph, void* stream) {
  RVB_REQUIRE(graph != nullptr, "rvb_search_submit_biased: no context graph");
  return search_submit_any(m, d_topk_val, d_topk_idx, k, d_enc_out, h_enc_lens, B, Tp, beam, blank_id, graph, stream);
}

RVB_API int rvb_rescoring_submit(rvb_model* m, int ticket, const float* h_cat_embs, int n_cat, float reverse_weight, int cap,
                                 int run_decoder, int* h_tokens, int* h_times, float* h_l2r, float* h_r2l,
                                 int* out_max_len, void* stream) {
  rvb::SearchTicket* t = ticket_of(m, ticket);
  RVB_REQUIRE(t && h_tokens && h_times && out_max_len && cap > 0 && (!run_decoder || h_l2r),
              "rvb_rescoring_submit: bad arguments");
  int rc = rvb::rescoring_submit(m, *t, h_cat_embs, n_cat, reverse_weight, cap, run_decoder, h_tokens, h_times, h_l2r,
                                 h_r2l, out_max_len, (cudaStream_t)stream);
  if (rc) t->state = 0;
  return rc;
}

RVB_API int rvb_rescoring_collect(rvb_model* m, int ticket, int* h_lens, double* h_scores, int* h_nhyp) {
  rvb::SearchTicket* t = ticket_of(m, ticket);
  RVB_REQUIRE(t && h_lens && h_scores && h_nhyp, "rvb_rescoring_collect: bad arguments");
  int rc = rvb::rescoring_collect(*t, h_lens, h_scores, h_nhyp);
  if (rc) t->state = 0;
  return rc;
}

RVB_API int rvb_ticket_release(rvb_model* m, int ticket) {
  rvb::SearchTicket* t = ticket_of(m, ticket);
  RVB_REQUIRE(t != nullptr, "rvb_ticket_release: bad ticket");
  if (t->state == 1 && t->ev_search) cudaEventSynchronize(t->ev_search);
  if (t->state == 2 && t->ev_done) cudaEventSynchronize(t->ev_done);   // copies into the caller's buffers have landed
  t->state = 0;
  return 0;
}

RVB_API int rvb_beam_search_rescoring(rvb_model* m, const float* d_topk_val, const int* d_topk_idx, int k,
                                      const float* d_enc_out, const int* h_enc_lens, int B, int Tp, int beam,
                                      int blank_id, const float* h_cat_embs, int n_cat, float reverse_weight, int cap,
                                      int* h_tokens, int* h_times, int* h_lens, double* h_scores, int* h_nhyp,
                                      float* h_l2r, float* h_r2l, int* out_max_len, void* stream) {
  RVB_REQUIRE(m && d_topk_val && d_topk_idx && d_enc_out && h_enc_lens && h_tokens && h_times && h_lens && h_scores &&
                  h_nhyp && h_l2r && out_max_len && B > 0 && Tp > 0 && cap > 0,
              "rvb_beam_search_rescoring: bad arguments");
  RVB_REQUIRE(m->finalized && m->w.dec_l.present, "beam_search_rescoring: model has no decoder");
  const int id = rvb_search_submit(m, d_topk_val, d_topk_idx, k, d_enc_out, h_enc_lens, B, Tp, beam, blank_id, stream);
  if (id < 0) return -1;
  if (rvb_rescoring_submit(m, id, h_cat_embs, n_cat, reverse_weight, cap, 1, h_tokens, h_times, h_l2r, h_r2l, out_max_len,
                           stream))
    return -1;
  return rvb_rescoring_collect(m, id, h_lens, h_scores, h_nhyp);
}

RVB_API int rvb_decoder_step_topk(rvb_model* m, const float* d_enc_out, const int* h_enc_lens, int B, int Tp, int N,
                                  const int* h_hyps, int L, const float* h_cat_embs, int n_cat, int k, float* h_topk_val,
                                  int* h_topk_idx, void* stream) {
  RVB_REQUIRE(m && d_enc_out && h_enc_lens && h_hyps && h_topk_val && h_topk_idx && B > 0 && Tp > 0 && N > 0,
              "rvb_decoder_step_topk: bad arguments");
  return rvb::decoder_step_topk(m, d_enc_out, h_enc_lens, B, Tp, N, h_hyps, L, h_cat_embs, n_cat, k, h_topk_val,
                                h_topk_idx, (cudaStream_t)stream);
}

RVB_API int rvb_decoder_cache_begin(rvb_model* m, const float* d_enc_out, const int* h_enc_lens, int B, int Tp, int N,
                                    int max_steps, const float* h_cat_embs, int n_cat, void* stream) {
  RVB_REQUIRE(m && d_enc_out && h_enc_lens, "rvb_decoder_cache_begin: bad arguments");
  return rvb::decoder_cache_begin(m, d_enc_out, h_enc_lens, B, Tp, N, max_steps, h_cat_embs, n_cat, (cudaStream_t)stream);
}

RVB_API int rvb_decoder_cache_step(rvb_model* m, const int* h_tokens, const int* h_parents, int k, float* h_topk_val,
                                   int* h_topk_idx, void* stream) {
  RVB_REQUIRE(m && h_tokens && h_topk_val && h_topk_idx, "rvb_decoder_cache_step: bad arguments");
  return rvb::decoder_cache_step(m, h_tokens, h_parents, k, h_topk_val, h_topk_idx, (cudaStream_t)stream);
}

RVB_API int rvb_decoder_cache_end(rvb_model* m) {
  if (m) m->dcache.reset();
  return 0;
}

RVB_API int rvb_decoder_step_logp(rvb_model* m, const float* d_enc_out, const int* h_enc_lens, int B, int Tp, int N,
                                  const int* h_hyps, int L, const float* h_cat_embs, int n_cat, float* h_logp,
                                  void* stream) {
  RVB_REQUIRE(m && d_enc_out && h_enc_lens && h_hyps && h_logp && B > 0 && Tp > 0 && N > 0,
              "rvb_decoder_step_logp: bad arguments");
  std::vector<float> val((size_t)B * N);
  std::vector<int> idx((size_t)B * N);
  return rvb::decoder_step_topk(m, d_enc_out, h_enc_lens, B, Tp, N, h_hyps, L, h_cat_embs, n_cat, 1, val.data(), idx.data(),
                                (cudaStream_t)stream, h_logp);
}

RVB_API int rvb_attention_rescoring(rvb_model* m, const float* d_enc_out, const int* h_enc_lens, int B, int Tp,
                            const int* h_hyp_tokens, const int* h_hyp_lens, int N, int max_len,
                            const float* h_cat_embs, int n_cat, float reverse_weight, float* h_l2r, float* h_r2l,
                            void* stream) {
  RVB_REQUIRE(m && d_enc_out && h_enc_lens && h_hyp_tokens && h_hyp_lens && h_l2r && B > 0 && N > 0 && max_len >= 0,
              "rvb_attention_rescoring: bad arguments");
  return rvb::attention_rescoring(m, d_enc_out, h_enc_lens, B, Tp, h_hyp_tokens, h_hyp_lens, N, max_len, h_cat_embs,
                                  n_cat, reverse_weight, h_l2r, h_r2l, (cudaStream_t)stream);
}

RVB_API int rvb_gemm_bf16(const void* d_A, const void* d_W, const float* d_bias, int M, int N, int K, int act, int out_mode,
                  float alpha, void* d_out, int ldo, void* stream) {
  rvb::GemmArgs g;
  g.A = reinterpret_cast<const rvb::bf16*>(d_A);
  g.W = reinterpret_cast<const rvb::bf16*>(d_W);
  g.M = M;
  g.N = N;
  g.K = K;
  g.bias = d_bias;
  g.act = act;
  g.out_mode = out_mode;
  g.alpha = alpha;
  g.out = d_out;
  g.ldo = ldo;
  return rvb::launch_gemm(g, (cudaStream_t)stream);
}

RVB_API int rvb_gemm_bf16_rows(const void* d_A, const void* d_W, const float* d_bias, int M, int N, int K, int act,
                               int out_mode, float alpha, void* d_out, int ldo, const int* d_row_lens, int rows_per_batch,
                               void* stream) {
  rvb::GemmArgs g;
  g.A = reinterpret_cast<const rvb::bf16*>(d_A);
  g.W = reinterpret_cast<const rvb::bf16*>(d_W);
  g.M = M;
  g.N = N;
  g.K = K;
  g.bias = d_bias;
  g.act = act;
  g.out_mode = out_mode;
  g.alpha = alpha;
  g.out = d_out;
  g.ldo = ldo;
  g.row_lens = d_row_lens;
  g.rows_per_batch = rows_per_batch;
  return rvb::launch_gemm(g, (cudaStream_t)stream);
}

RVB_API int rvb_gemm_bf16x3(const void* d_A, const void* d_W, const float* d_bias, int M, int N, int K, int act, int out_mode,
                            float alpha, void* d_out, int ldo, void* stream) {
  rvb::GemmArgs g;
  g.A = reinterpret_cast<const rvb::bf16*>(d_A);
  g.W = reinterpret_cast<const rvb::bf16*>(d_W);
  g.M = M;
  g.N = N;
  g.K = K;
  g.bias = d_bias;
  g.act = act;
  g.out_mode = out_mode;
  g.alpha = alpha;
  g.out = d_out;
  g.ldo = ldo;
  g.x3 = 1;
  if (out_mode == rvb::OUT_BF16) g.out_split = (act == rvb::ACT_GLU) ? N / 2 : N;
  return rvb::launch_gemm(g, (cudaStream_t)stream);
}

RVB_API int rvb_gemm_grouped(const void* d_A, const void* d_W, const float* d_bias, int M, int N, int K, int out_mode,
                             void* d_out, int ldo, const int* d_grp, int rows_per_batch, int group_n, int x3,
                             void* stream) {
  rvb::GemmArgs g;
  g.A = reinterpret_cast<const rvb::bf16*>(d_A);
  g.W = reinterpret_cast<const rvb::bf16*>(d_W);
  g.M = M;
  g.N = N;
  g.K = K;
  g.bias = d_bias;
  g.out_mode = out_mode;
  g.out = d_out;
  g.ldo = ldo;
  g.grp = d_grp;
  g.group_n = group_n;
  g.rows_per_batch = rows_per_batch;
  g.x3 = x3 ? 1 : 0;
  if (x3 && out_mode == rvb::OUT_BF16) g.out_split = group_n;
  RVB_REQUIRE(d_grp != nullptr, "rvb_gemm_grouped: null group array");
  return rvb::launch_gemm(g, (cudaStream_t)stream);
}

RVB_API int rvb_f32_to_bf16_pair(const float* d_x, void* d_out, long long rows, int width, void* stream) {
  return rvb::launch_f32_to_pair(d_x, reinterpret_cast<rvb::bf16*>(d_out), rows, width, (cudaStream_t)stream);
}

RVB_API long long rvb_gemm_logsoftmax_gather_ws_bytes(int M, int N) {
  return (long long)M * rvb::lse_slabs(N) * (long long)sizeof(float2) + (long long)M * (long long)sizeof(float);
}

RVB_API int rvb_gemm_logsoftmax_gather(const void* d_A, const void* d_W, const float* d_bias, int M, int N, int K,
                                       const int* d_gather, void* d_ws, float* d_out, void* stream) {
  RVB_REQUIRE(d_A && d_W && d_gather && d_ws && d_out, "rvb_gemm_logsoftmax_gather: bad arguments");
  const int slabs = rvb::lse_slabs(N);
  rvb::GemmArgs g;
  g.A = reinterpret_cast<const rvb::bf16*>(d_A);
  g.W = reinterpret_cast<const rvb::bf16*>(d_W);
  g.bias = d_bias;
  g.M = M;
  g.N = N;
  g.K = K;
  g.out_mode = rvb::OUT_LSE;
  g.lse_gather = d_gather;
  g.lse_part = reinterpret_cast<float2*>(d_ws);
  g.lse_tgt = reinterpret_cast<float*>(g.lse_part + (size_t)M * slabs);
  if (rvb::launch_gemm(g, (cudaStream_t)stream)) return -1;
  return rvb::launch_lse_merge(g.lse_part, slabs, g.lse_tgt, d_gather, M, d_out, (cudaStream_t)stream);
}

RVB_API int rvb_layernorm(const float* d_x, const float* d_gamma, const float* d_beta, float eps, int M, int d,
                  void* d_out_bf16, float* d_out_f32, void* stream) {
  return rvb::launch_layernorm(d_x, d_gamma, d_beta, eps, M, d, reinterpret_cast<rvb::bf16*>(d_out_bf16), d_out_f32,
                               nullptr, 0, 0, (cudaStream_t)stream);
}

RVB_API int rvb_attention(const void* d_q, const void* d_k, const void* d_v, const void* d_p, const float* d_bias_u,
                  const float* d_bias_v, void* d_out, int ldq, int ldk, int ldv, int ldp, int ldo, int Bq, int Tq, int Tk,
                  int H, int dk, int q_per_kv, const int* d_k_lens, const int* d_q_lens, int causal, float scale,
                  void* stream) {
  rvb::AttnArgs a;
  a.q = reinterpret_cast<const rvb::bf16*>(d_q);
  a.k = reinterpret_cast<const rvb::bf16*>(d_k);
  a.v = reinterpret_cast<const rvb::bf16*>(d_v);
  a.p = reinterpret_cast<const rvb::bf16*>(d_p);
  a.bias_u = d_bias_u;
  a.bias_v = d_bias_v;
  a.out = reinterpret_cast<rvb::bf16*>(d_out);
  a.ldq = ldq; a.ldk = ldk; a.ldv = ldv; a.ldp = ldp; a.ldo = ldo;
  a.Bq = Bq; a.Tq = Tq; a.Tk = Tk; a.H = H; a.dk = dk;
  a.q_per_kv = q_per_kv;
  a.k_lens = d_k_lens; a.q_lens = d_q_lens;
  a.causal = causal;
  a.scale = scale;
  return rvb::launch_attention(a, (cudaStream_t)stream);
}

RVB_API int rvb_attention_tc(const void* d_q, const void* d_k, const void* d_v, void* d_out, int ldq, int ldk, int ldv,
                             int ldo, int groups, int Tq, int Tk, int H, int dk, const float* d_key_bias,
                             const int* d_k_lens, int causal, float scale, void* stream) {
  rvb::AttnTcArgs a;
  a.q = reinterpret_cast<const rvb::bf16*>(d_q);
  a.k = reinterpret_cast<const rvb::bf16*>(d_k);
  a.v = reinterpret_cast<const rvb::bf16*>(d_v);
  a.out = reinterpret_cast<rvb::bf16*>(d_out);
  a.ldq = ldq; a.ldk = ldk; a.ldv = ldv; a.ldo = ldo;
  a.groups = groups; a.Tq = Tq; a.Tk = Tk; a.H = H; a.dk = dk;
  a.key_bias = d_key_bias;
  a.k_lens = d_k_lens;
  a.causal = causal;
  a.scale = scale;
  return rvb::launch_attention_tc(a, (cudaStream_t)stream);
}

RVB_API int rvb_attention_tc_bits(const void* d_q, const void* d_k, const void* d_v, void* d_out, int ldq, int ldk,
                                  int ldv, int ldo, int groups, int Tq, int Tk, int H, int dk, const float* d_key_bias,
                                  const int* d_k_lens, int causal, const void* d_key_bits, int bits_ld, float scale,
                                  void* stream) {
  rvb::AttnTcArgs a;
  a.q = reinterpret_cast<const rvb::bf16*>(d_q);
  a.k = reinterpret_cast<const rvb::bf16*>(d_k);
  a.v = reinterpret_cast<const rvb::bf16*>(d_v);
  a.out = reinterpret_cast<rvb::bf16*>(d_out);
  a.ldq = ldq; a.ldk = ldk; a.ldv = ldv; a.ldo = ldo;
  a.groups = groups; a.Tq = Tq; a.Tk = Tk; a.H = H; a.dk = dk;
  a.key_bias = d_key_bias;
  a.k_lens = d_k_lens;
  a.causal = causal;
  a.key_bits = reinterpret_cast<const uint32_t*>(d_key_bits);
  a.bits_ld = bits_ld;
  a.scale = scale;
  RVB_REQUIRE(d_key_bits != nullptr, "rvb_attention_tc_bits: d_key_bits is null");
  return rvb::launch_attention_tc(a, (cudaStream_t)stream);
}

RVB_API int rvb_attention_tc_blocks_per_sm(int Tk, int causal, int chunk, int with_key_bits) {
  int blocks = 0;
  if (rvb::attention_tc_blocks_per_sm(Tk, causal || chunk > 0, with_key_bits != 0, &blocks)) return -1;
  return blocks;
}

RVB_API int rvb_attention_tc_chunked(const void* d_q, const void* d_k, const void* d_v, void* d_out, int ldq, int ldk,
                                     int ldv, int ldo, int groups, int Tq, int Tk, int H, int dk, const float* d_key_bias,
                                     const int* d_k_lens, int chunk, int left_chunks, float scale, void* stream) {
  rvb::AttnTcArgs a;
  a.q = reinterpret_cast<const rvb::bf16*>(d_q);
  a.k = reinterpret_cast<const rvb::bf16*>(d_k);
  a.v = reinterpret_cast<const rvb::bf16*>(d_v);
  a.out = reinterpret_cast<rvb::bf16*>(d_out);
  a.ldq = ldq; a.ldk = ldk; a.ldv = ldv; a.ldo = ldo;
  a.groups = groups; a.Tq = Tq; a.Tk = Tk; a.H = H; a.dk = dk;
  a.key_bias = d_key_bias;
  a.k_lens = d_k_lens;
  a.chunk = chunk;
  a.left_chunks = left_chunks;
  a.scale = scale;
  return rvb::launch_attention_tc(a, (cudaStream_t)stream);
}

RVB_API int rvb_relpos_prep(const void* d_k, int ldk, const void* d_pos, int ldp, const float* d_bias_u,
                            const float* d_bias_v, void* d_kpp, float* d_cbias, int B, int T, int H, int dk,
                            void* stream) {
  return rvb::launch_relpos_prep(reinterpret_cast<const rvb::bf16*>(d_k), ldk, reinterpret_cast<const rvb::bf16*>(d_pos),
                                 ldp, d_bias_u, d_bias_v, reinterpret_cast<rvb::bf16*>(d_kpp), d_cbias, B, T, H, dk,
                                 (cudaStream_t)stream);
}

RVB_API int rvb_f32_to_bf16(const float* d_x, void* d_out, long long n, void* stream) {
  return rvb::launch_f32_to_bf16(d_x, reinterpret_cast<rvb::bf16*>(d_out), n, (cudaStream_t)stream);
}

}  // extern "C"
