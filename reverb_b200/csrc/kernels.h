// reverb_b200 — host-side launchers of the sm_90a kernels (internal; the public boundary is
// include/rvb_b200.h).  Every launcher enqueues on the given stream and returns 0 / <0.
#pragma once
#include <vector>

#include "common.cuh"

struct rvb_model;
struct rvb_context_graph;

namespace rvb {

// the side stream the prefix beam search runs on (engine.cu search_submit), created on first use; forced alignment
// (align.cu) puts its serial trellis there too
int search_side_stream(::rvb_model* m, cudaStream_t* out);

// ------------------------------------------------------------------ GEMM (gemm.cu)
// ACT_GLU (bf16 output only): the N = 2C weight rows are interleaved in groups of 32 — rows [64j, 64j+32) are the
// "value" half of output channels [32j, 32j+32), rows [64j+32, 64j+64) their gates — and the kernel writes
// out[m, 32j + i] = (acc_a + bias_a) * sigmoid(acc_g + bias_g), an (M, C) matrix (default ldo = N / 2).
// ACT_GELU (bf16 output only): torch's default erf GELU, 0.5 x (1 + erf(x / sqrt 2)).
enum GemmAct { ACT_NONE = 0, ACT_RELU = 1, ACT_SILU = 2, ACT_GLU = 3, ACT_GELU = 4 };
enum GemmOut {
  OUT_BF16 = 0,      // out_bf16[m, n] = act(acc + bias)
  OUT_F32 = 1,       // out_f32[m, n]  = act(acc + bias)
  OUT_RESID_F32 = 2, // out_f32[m, n] += alpha * act(acc + bias)   (rows masked by row_lens are left untouched)
  // no C matrix at all: per row m and per column slab (lse_slab(N) slabs of 128 columns) the epilogue emits the
  // partial (max, sum exp(x - max)) of x = acc + bias over the slab -> lse_part[m, slab], and x[m, lse_gather[m]]
  // -> lse_tgt[m] (rows with a negative gather index are skipped).  launch_lse_merge turns the partials into
  // out[m] = x[m, gather[m]] - logsumexp_n x[m, n]: log_softmax + gather without ever writing the logits.
  OUT_LSE = 3
};
inline int lse_slabs(int N) { return ((N + 255) / 256) * 2; }

struct GemmArgs {
  // C[M,N] = A[M,K] * W[N,K]^T ; A, W bf16 row-major (K contiguous)
  const bf16* A = nullptr;
  const bf16* W = nullptr;
  int M = 0, N = 0, K = 0;
  int lda = 0;  // elements; 0 -> K
  int ldw = 0;  // elements; 0 -> K
  const float* bias = nullptr;
  int act = ACT_NONE;
  int out_mode = OUT_BF16;
  void* out = nullptr;
  int ldo = 0;  // elements; 0 -> N
  float alpha = 1.0f;
  // optional second output for OUT_RESID_F32: nothing (kept simple)
  // row masking: row m belongs to batch m / rows_per_batch, position m % rows_per_batch;
  // valid iff position < row_lens[batch].  nullptr -> all rows valid.
  const int* row_lens = nullptr;
  int rows_per_batch = 0;
  // conv2d-subsampling second conv as implicit GEMM (A is the conv1 activation, see subsample.cu):
  //   A logical layout (B, 2, T1h, F1, C) bf16 (time split by parity), M = B*F2*T2 rows ordered (b, f, t'),
  //   K = 9*C ordered (kh, kw, c); output row (b, t', f) -> out[((b*T2 + t')*F2 + f) * ldo + n]
  int conv_mode = 0;
  int conv_B = 0, conv_T1h = 0, conv_F1 = 0, conv_C = 0, conv_T2 = 0, conv_F2 = 0;
  // fp32-accurate mode ("bf16x3"): every operand is a PAIR of bf16 matrices hi = bf16(v), lo = bf16(v - hi) stored side
  // by side — A physical (M, 2K) = [A_hi | A_lo] (lda >= 2K), W physical (N, 2K) = [W_hi | W_lo] (conv_mode: channels
  // [hi C | lo C] of the activation, W = [hi 9C | lo 9C]) — and the kernel runs THREE passes over K into the same fp32
  // accumulator: A_hi W_hi + A_lo W_hi + A_hi W_lo (the lo.lo term, ~2^-18 relative, is dropped).  bf16 outputs
  // (OUT_BF16, ACT_GLU) are written as the same kind of pair: hi at column n, lo at column n + out_split.
  int x3 = 0;
  int out_split = 0;  // elements; > 0: bf16 output pair (ldo must cover both halves)
  // conv_mode + out_split: output row (b, t') holds [hi (F2*N) | lo (F2*N)] (out_split = F2*N), i.e. element (b,t',f,n)
  // -> out[((b*T2 + t') * 2*F2 + f) * ldo + n] — the pair-layout A operand of the Linear(F2*C -> d) that follows
  int conv_pair_out = 0;
  // rel-pos attention folded into the fused [q; k; v] projection (OUT_BF16, no activation, d_k = 64): the epilogue
  // replaces the key columns [rp_col0, rp_col0 + rp_H*64) by K'' = bf16(k + pos[t]) (t = row % rp_T, pos row stride
  // rp_ldp) and writes the per-key bias rp_cb[(row / rp_T) * rp_H + h, t] = u_h . k + v_h . pos[t] — what the separate
  // relpos_prep kernel (attention_tc.cu) computes from the stored projection, in the same summation order, so that the
  // fused and the separate path give the same bias bit for bit (a precomputed v . pos table rounds differently, and the
  // encoder layers amplify that difference).  v . pos costs 8 FMAs per key column here, next to the pos load.
  const bf16* rp_pos = nullptr;
  int rp_ldp = 0, rp_T = 0, rp_H = 0, rp_col0 = 0;
  const float* rp_u = nullptr;
  const float* rp_v = nullptr;
  float* rp_cb = nullptr;
  // OUT_LSE
  const int* lse_gather = nullptr;   // (M) column index per row, < 0 = none
  float2* lse_part = nullptr;        // (M, lse_slabs(N)) {max, sum exp(x - max)}; slabs without columns hold {-inf, 0}
  float* lse_tgt = nullptr;          // (M) the gathered x
  // grouped output (language-specific linears with per-utterance mixing weights): W (N, K) and bias (N) stack N / group_n
  // blocks of group_n rows, one per group.  Row m belongs to utterance m / rows_per_batch and takes only the block of its
  // group g = grp[m / rows_per_batch] (int32, device), written at output column n - g * group_n (ldo 0 -> group_n).
  // Every element equals a plain launch of that group's block: same tile width, k-block order and epilogue.  Tiles whose
  // rows hold no utterance of their block's group are skipped.  act none, out_mode OUT_BF16 (or its pair) / OUT_F32.
  const int* grp = nullptr;
  int group_n = 0;
};
// out[m] = gather[m] >= 0 ? tgt[m] - logsumexp(partials of row m) : 0
int launch_lse_merge(const float2* part, int slabs, const float* tgt, const int* gather, int M, float* out,
                     cudaStream_t stream);

int launch_gemm(const GemmArgs& a, cudaStream_t stream);
// 0 = wgmma/TMA kernel (default), 1 = plain CUDA-core debug kernel (env RVB_GEMM=simt), 2 = wgmma with 64-wide tiles
void set_gemm_impl(int impl);
int get_gemm_impl();
// per-launch CUDA-event timing of the wgmma GEMM (algorithmic FLOPs = 2*M*N*K per launch)
void gemm_profile_begin();
int gemm_profile_end(double* total_ms, double* total_flops, long long* launches);

// ------------------------------------------------------------------ fbank (fbank.cu)
// polyphase sinc resampling (torchaudio.transforms.Resample semantics; table from reverb_b200/resample.py), resample.cu
int launch_resample(const void* x, int is_i16, long long n_in, const float* kern /*(new, 2*width+orig)*/, int orig, int new_,
                    int width, float* y, long long n_out, cudaStream_t stream);
int launch_fbank(const float* wave, long long n_samples, float* feats, long long n_frames, cudaStream_t stream);
// int16 PCM input variant (the host API's H2D format)
int launch_fbank_i16(const short* wave, long long n_samples, float* feats, long long n_frames, cudaStream_t stream);
// `batch` equal-length recordings `wave_stride` samples apart -> feats (batch, n_frames, 80)
// window_type: 0 = povey (ASR front-end), 1 = hamming (WeSpeaker embedding front-end)
int launch_fbank_batch(const void* wave, int is_i16, int batch, long long wave_stride, long long n_samples,
                       float* feats, long long n_frames, cudaStream_t stream, int window_type = 0);

// ------------------------------------------------------------------ diarization (diar_seg.cu / diar_emb.cu)
// C[m, n] = act(sum_k A[m, k] W[n, k] + bias[n]) in fp32 on the CUDA cores; act 1 = LeakyReLU(0.01)
int launch_sgemm(const float* A, int lda, const float* W, int ldw, const float* bias, float* C, int ldc, int M, int N,
                 int K, int act, cudaStream_t stream);
class WeightStore;
// The head both segmentation networks share (PyanNet and WavLM / SSeRiouSS): bidirectional LSTM stack -> linears with
// LeakyReLU -> classifier -> log_softmax, fp32, under pyannote's names lstm.*, linear.{i}.*, classifier.*.
struct SegHead {
  int hidden = 128, lstm_layers = 0, linear_layers = 0, linear_dim = 0, num_classes = 0;
  std::vector<float*> wih, whh, lbias;   // per layer: (2*4H, in), (2, 4H, H), (2*4H)
  std::vector<float*> lin_w, lin_b;
  float* cls_w = nullptr;
  float* cls_b = nullptr;
};
// uploads the head's tensors from the store (in_dim: width of the LSTM input); shape fields must be set
int seg_head_load(WeightStore& store, int in_dim, SegHead* h);
// x (B*T, in_dim) -> logp (B*T, classes).  Scratch: g (B*T, 8H), h0 / h1 (B*T, 2H) (x may be h1, not h0),
// y0 / y1 (B*T, max(linear_dim, classes))
int seg_head_forward(const SegHead& h, const float* x, int in_dim, int B, int T, float* g, float* h0, float* h1,
                     float* y0, float* y1, float* logp, cudaStream_t stream);

// ------------------------------------------------------------------ norms / conv pieces (elementwise.cu)
// y = LN(x) * gamma + beta ; rows with position >= row_lens[batch] are written as 0 when mask_rows != 0.
// out_bf16 and/or out_f32 may be null.
// x3 != 0 (all launchers below): bf16 outputs / inputs use the accurate mode's pair layout [hi | lo] (row stride
// 2 * width, lo at column + width), see GemmArgs::x3.
int launch_layernorm(const float* x, const float* gamma, const float* beta, float eps, int M, int d, bf16* out_bf16,
                     float* out_f32, const int* row_lens, int rows_per_batch, int mask_rows, cudaStream_t stream,
                     int x3 = 0);
// x2 = LN_a(x) (fp32, in place allowed) ; n = LN_b(x2) -> bf16.  (norm_final of block i fused with the first
// pre-norm of block i+1.)  y_add (optional, fp32) is added to x2 after LN_a (LSL "x = x + y").
int launch_double_layernorm(const float* x, const float* ga, const float* ba, const float* y_add, float* x2,
                            const float* gb, const float* bb, float eps, int M, int d, bf16* n_out,
                            float* n_out_f32, cudaStream_t stream, int x3 = 0);
// CMVN + Conv2d(1->C, 3x3, stride 2) + ReLU, output bf16 (B, 2, T1h, F1, C) (time split by parity)
int launch_conv1(const float* feats, const float* mean, const float* istd, const float* w /*[C][9]*/,
                 const float* bias, bf16* out, int B, int T, int F, int C, int T1, int T1h, int F1,
                 cudaStream_t stream, int x3 = 0);
// depthwise conv (K taps) + LayerNorm|BatchNorm(eval) + SiLU on the GLU'd pointwise_conv1 output (B, T, C) bf16
// (GEMM epilogue ACT_GLU) -> (B, T, C) bf16.  pad_glu (C, fp32): value of the K-1 causal left pad frames =
// GLU(pointwise_conv1 bias), not zeros.  conv_tmp (B*T, C) fp32 and stats (B*T, ceil(C/256), 2) scratch are needed with LayerNorm.
int launch_conv_mid(const bf16* x, const float* pad_glu, const float* dw_w /*[C][K]*/, const float* dw_b,
                    const float* norm_w, const float* norm_b, const float* bn_mean, const float* bn_var,
                    int use_layer_norm, float eps, bf16* out, int B, int T, int C, int K, int causal,
                    cudaStream_t stream, float* conv_tmp = nullptr, float* stats = nullptr, int x3 = 0,
                    int conv_chunk = 0 /* > 0: non-causal, every chunk of conv_chunk frames convolved on its own */);
// x[m, :] = x[m, :] * scale   (fp32 -> fp32 in place) and optional bf16 copy
int launch_scale_cast(const float* x, float scale, float* out_f32, bf16* out_bf16, long long n, cudaStream_t stream);
int launch_f32_to_bf16(const float* x, bf16* out, long long n, cudaStream_t stream);
// (rows, width) fp32 -> (rows, 2 * width) bf16 pair [hi | lo]
int launch_f32_to_pair(const float* x, bf16* out, long long rows, int width, cudaStream_t stream);
// out = sum_i c[i] * in_i   (fold of the language-specific linears; n elements, up to 8 inputs)
int launch_weighted_sum_bf16(const float* const* ins, const float* coef, int n_in, long long n, bf16* out_bf16,
                             float* out_f32, cudaStream_t stream);
// decoder input: x[r, :] = emb[tok[r], :] * sqrt(d) + pe[pos(r), :]   (fp32), r over (N, L)
int launch_embed_posenc(const int* tokens, const float* emb, int N, int L, int d, float* out, cudaStream_t stream,
                        int pos0 = 0 /* position of column 0 */);
// decoder KV cache helpers (elementwise.cu): rows of `width` bf16, caches (S, Lcap, width)
int launch_kv_append(const bf16* kv, long long ld, int col0, bf16* cache, int S, int Lcap, int pos, int width,
                     int row_stride, cudaStream_t stream);
int launch_kv_reorder(const bf16* src, bf16* dst, const int* parent, int S, int Lcap, int npos, int width,
                      cudaStream_t stream);
int launch_fill_int(int* p, int n, int v, cudaStream_t stream);
// sinusoidal table pe[pos, :] for pos < T (fp32 (T, d) and bf16 copy)
int launch_sinusoid(int T, int d, float* out_f32, bf16* out_bf16, cudaStream_t stream);

// ------------------------------------------------------------------ attention (attention.cu)
struct AttnArgs {
  const bf16* q = nullptr;  // (Bq, Tq, H, dk) with row stride ldq elements
  const bf16* k = nullptr;  // (Bk, Tk, H, dk) row stride ldk
  const bf16* v = nullptr;  // (Bk, Tk, H, dk) row stride ldv
  const bf16* p = nullptr;  // optional rel-pos keys (Tk, H, dk), row stride ldp (shared by the batch)
  const float* bias_u = nullptr;  // (H, dk) added to q for the content term (with p)
  const float* bias_v = nullptr;  // (H, dk) added to q for the position term (with p)
  bf16* out = nullptr;            // (Bq, Tq, H*dk) row stride ldo
  int ldq = 0, ldk = 0, ldv = 0, ldp = 0, ldo = 0;
  int Bq = 0, Tq = 0, Tk = 0, H = 0, dk = 0;
  int q_per_kv = 1;               // kv batch = q batch / q_per_kv
  const int* k_lens = nullptr;    // per kv batch valid key count (nullptr -> Tk)
  const int* q_lens = nullptr;    // per q batch: causal-with-length mask (key j valid iff j <= i and j < q_lens[b])
  int causal = 0;
  float scale = 1.0f;
};
int launch_attention(const AttnArgs& a, cudaStream_t stream);

// wgmma attention (attention_tc.cu): d_k = 64, key-length mask, optional per-key bias (rel-pos folded, see the
// kernel header).  Rows are grouped: group g owns query rows [g*Tq, (g+1)*Tq) and key rows [g*Tk, (g+1)*Tk);
// the q/k/v pointers address column 0 of head 0 (heads are 64 columns apart).
struct AttnTcArgs {
  const bf16* q = nullptr;
  const bf16* k = nullptr;
  const bf16* v = nullptr;
  bf16* out = nullptr;
  int ldq = 0, ldk = 0, ldv = 0, ldo = 0;
  int groups = 0, Tq = 0, Tk = 0, H = 0, dk = 0;
  const float* key_bias = nullptr;  // (groups, H, Tk) fp32, added to q.k before scaling
  const int* k_lens = nullptr;      // (groups) valid keys
  int causal = 0;                   // self-attention with Tq == Tk: key j visible to query i iff j <= i
  int chunk = 0, left_chunks = -1;  // chunk > 0: streaming chunk mask (utils/mask.py:88-123), left_chunks < 0 = all
  // arbitrary visibility on top of the masks above (prefix-tree self-attention): bit (j & 31) of
  // key_bits[(group*Tq + i) * bits_ld + (j >> 5)] set <=> key j visible to query row i; bits_ld >= 2 * ceil(Tk / 64)
  const uint32_t* key_bits = nullptr;
  int bits_ld = 0;
  float scale = 1.0f;
  // WavLM's gated relative-position bias (self-attention, Tq == Tk, no other mask or key bias): score(i, j) +=
  // gate[(group*H + h)*Tq + i] * rel_bias[h*(2Tk - 1) + j - i + Tk - 1], added after the scaling
  const float* gate = nullptr;
  const float* rel_bias = nullptr;
};
int launch_attention_tc(const AttnTcArgs& a, cudaStream_t stream);
// CTAs per SM of the instantiation launch_attention_tc runs for these masks and Tk
int attention_tc_blocks_per_sm(int Tk, bool chunk_or_causal, bool key_bits, int* blocks);
// K'' = k + pos (bf16, (B*T, H*dk) dense) and cbias[b,h,t] = u_h . k + v_h . pos
int launch_relpos_prep(const bf16* k, int ldk, const bf16* pos, int ldp, const float* bias_u, const float* bias_v,
                       bf16* kpp, float* cbias, int B, int T, int H, int dk, cudaStream_t stream);

// fp32 attention of the accurate (bf16x3) mode (attention_f32.cu): same grouping convention as AttnTcArgs; every operand
// is a bf16 pair (value = x[c] + x[c + *_lo], *_lo == 0: plain bf16).  p (optional): rel-pos keys (Tk, H*dk) shared by
// all groups, with bias_u / bias_v (H*dk) — the reference's two-product score ((q+u).k + (q+v).p) / sqrt(dk).
struct AttnF32Args {
  const bf16* q = nullptr;
  const bf16* k = nullptr;
  const bf16* v = nullptr;
  const bf16* p = nullptr;
  const float* bias_u = nullptr;
  const float* bias_v = nullptr;
  bf16* out = nullptr;
  int ldq = 0, ldk = 0, ldv = 0, ldp = 0, ldo = 0;
  int q_lo = 0, k_lo = 0, v_lo = 0, p_lo = 0, o_lo = 0;
  int groups = 0, Tq = 0, Tk = 0, H = 0, dk = 0;
  const int* k_lens = nullptr;
  int chunk = 0, left = -1;  // chunk > 0: streaming chunk mask; chunk = 1, left < 0 = causal
  // key lists (prefix-tree self-attention): query row i of group g attends the key_list_len[g*Tq + i] key ROWS listed at
  // key_list[(g*Tq + i) * key_list_ld ...] (absolute row indices into k / v); Tk = the longest list
  const int* key_list = nullptr;
  const int* key_list_len = nullptr;
  int key_list_ld = 0;
};
int launch_attention_f32(const AttnF32Args& a, cudaStream_t stream);

// ------------------------------------------------------------------ CTC head / searches (ctc.cu)
// per row: logp = log_softmax(logits) ; top-k (k <= 16) of logp with indices ; optional full logp output.
int launch_logsoftmax_topk(const float* logits, int ld, int M, int V, int k, float* topk_val, int* topk_idx,
                           float* logp_out /*nullable, ld = V*/, int apply_softmax, cudaStream_t stream);
// greedy: per utterance, arg-max ids (top-1) with padded frames -> blank, collapsed (repeats merged, blanks dropped)
int launch_ctc_greedy(const int* top1_idx, int idx_stride, const int* lens, int B, int T, int blank, int* out_tokens,
                      int* out_lens, cudaStream_t stream);
struct PrefixBeamWorkspace;
size_t prefix_beam_workspace_bytes(int B, int T, int beam);
// CTC prefix beam search, one CTA per utterance, fp64 scores (reference: transformer/search.py:124-248)
int launch_ctc_prefix_beam(const float* topk_val, const int* topk_idx, int k, const int* lens, int B, int T, int beam,
                           int blank, void* workspace, size_t workspace_bytes, int max_len, int* out_tokens,
                           int* out_times, int* out_lens, double* out_scores, int* out_nhyp, cudaStream_t stream);
// Context graph in read-only device memory (context.cu): children in CSR by state with token-sorted child lists,
// the root's children also as a dense token -> child table (-1 = none), fail links, and the float64 tables of
// utils/context_graph.py (node_score = bonus, output_score = emit, token_score).  State 0 is the root.
struct ContextGraphView {
  const int* off = nullptr;        // n_nodes + 1
  const int* tok = nullptr;        // n_edges, sorted within a state
  const int* dst = nullptr;        // n_edges
  const int* fail = nullptr;       // n_nodes
  const int* root_next = nullptr;  // vocab
  const double* bonus = nullptr;
  const double* emit = nullptr;
  const double* token_score = nullptr;
  int n_nodes = 0, vocab = 0;
};
// the same search with context biasing (the `context_graph` branches of search.py:124-248)
int launch_ctc_prefix_beam_biased(const float* topk_val, const int* topk_idx, int k, const int* lens, int B, int T,
                                  int beam, int blank, void* workspace, size_t workspace_bytes, int max_len,
                                  int* out_tokens, int* out_times, int* out_lens, double* out_scores, int* out_nhyp,
                                  const ContextGraphView& graph, cudaStream_t stream);
// the device tables of a graph handle (context.cu), and the bookkeeping that lets rvb_context_graph_destroy wait for
// searches enqueued with it: call after enqueueing such a search on `stream`
const ContextGraphView* context_graph_view(const ::rvb_context_graph* g);
int context_graph_note_use(::rvb_context_graph* g, cudaStream_t stream);

// ------------------------------------------------------------------ rescoring (ctc.cu)
// per row r: lse = logsumexp(logits[r, :V]); out[r, j] = logits[r, gather_idx[r*G + j]] - lse  (idx < 0 -> 0)
int launch_logsoftmax_gather(const float* logits, int ld, int M, int V, const int* gather_idx, int G, float* out,
                             cudaStream_t stream);
// decoder inputs / gather targets (B*N rows of Lp) from the device-resident n-best of launch_ctc_prefix_beam
int launch_rescoring_inputs(const int* d_tokens, int tok_stride, const int* d_out_lens, const int* d_nhyp, int B, int N,
                            int Lp, int sos, int eos, int* tok_l, int* tok_r, int* gat_l, int* gat_r, int* slen,
                            cudaStream_t stream);

// prefix-tree rescoring (ctc.cu): see trie_build_kernel / trie_inputs_kernel
int launch_trie_build(const int* tok, int tok_stride, const int* olen, const int* nhyp, int B, int N, int reverse, int sos,
                      int* node_of, int nstride, int* node_tok, int* node_par, int* node_dep, int cap, int* n_nodes,
                      cudaStream_t stream);
int launch_trie_inputs(const int* node_of, int nstride, const int* node_tok, const int* node_par, const int* node_dep,
                       int cap, const int* n_nodes, const int* olen, const int* nhyp, int B, int N, int P, int Lp, int eos,
                       int* tok_in, int* pos, int* anc, int* alen, int* src, int* tgt, int* smap, cudaStream_t stream,
                       uint32_t* anc_bits = nullptr, int bits_ld = 0);
int launch_gather_rows(const bf16* in, const int* idx, bf16* out, int rows, int width, cudaStream_t stream);
int launch_gather_scores(const float* vals, const int* map, float* out, long long n, cudaStream_t stream);
// decoder input with a per-row position: x[r, :] = emb[tok[r], :] * sqrt(d) + pe[pos[r], :]
int launch_embed_posenc_rows(const int* tokens, const int* pos, const float* emb, int R, int d, float* out,
                             cudaStream_t stream);

}  // namespace rvb
