/* reverb_b200 — C ABI of the H100-native hot path of revdotcom/reverb.
 *
 * The reference (100 % Python, asr/wenet) has no FFI of its own; this header is the boundary a maintainer binds
 * with ctypes (see INTEGRATION.md) to replace, one for one, the operator-level calls of the reference's hot path:
 *
 *   rvb_fbank_*                 <- torchaudio.compliance.kaldi.fbank call   asr/wenet/cli/reverb.py:130-138
 *   rvb_resample                <- torchaudio.transforms.Resample call      asr/wenet/cli/reverb.py:125-128
 *   rvb_encoder_forward[_chunked] <- ASRModel._forward_encoder              asr/wenet/transformer/asr_model.py:288-316
 *                                  (BaseEncoder.forward, transformer/encoder.py:117-149; chunk masks utils/mask.py:88-197)
 *   rvb_ctc_topk                <- ASRModel.ctc_logprobs + logp.topk        asr_model.py:318-329, search.py:111,155
 *   rvb_ctc_greedy_search       <- ctc_greedy_search                        transformer/search.py:106-121
 *   rvb_ctc_prefix_beam_search  <- ctc_prefix_beam_search                   transformer/search.py:124-248
 *   rvb_context_graph_*, *_biased <- ContextGraph + its search branches      utils/context_graph.py, search.py:124-248
 *   rvb_attention_rescoring     <- forward_attention_decoder + the gather   asr_model.py:868-978, search.py:410-436
 *   rvb_beam_search_rescoring   <- the two calls above back to back          asr_model.py:403-424 (n-best stays on the device)
 *   rvb_decoder_step_topk       <- decoder.forward_one_step + logp.topk     search.py:302-306 (`attention` mode)
 *   rvb_model_*                 <- init_model / load_checkpoint             utils/init_model.py:99-277,
 *                                                                           utils/checkpoint.py:29-80
 *
 * Conventions: plain pointers and sizes, no C++/torch types.  `d_` pointers are device memory owned by the caller
 * (e.g. torch tensors' data_ptr()), `h_` pointers are host memory owned by the caller.  All work is enqueued on the
 * given CUDA stream (a `cudaStream_t` passed as void*); functions that fill `h_` outputs synchronise that stream
 * before returning.  Return value 0 = success, < 0 = failure with a message available from rvb_last_error().
 * There is no CPU fallback: without a CUDA device every compute entry point fails.
 */
#ifndef RVB_B200_H_
#define RVB_B200_H_

#if defined(__GNUC__)
#define RVB_API __attribute__((visibility("default")))
#else
#define RVB_API
#endif

#ifdef __cplusplus
extern "C" {
#endif

typedef struct rvb_model rvb_model;

typedef struct rvb_model_config {
  int input_dim;        /* fbank bins, 80 (config.yaml: input_dim) */
  int d_model;          /* encoder_conf.output_size */
  int heads;            /* encoder_conf.attention_heads */
  int ffn_dim;          /* encoder_conf.linear_units */
  int num_blocks;       /* encoder_conf.num_blocks */
  int cnn_kernel;       /* encoder_conf.cnn_module_kernel */
  int causal;           /* encoder_conf.causal */
  int cnn_layer_norm;   /* 1: cnn_module_norm == layer_norm, 0: batch_norm (eval statistics) */
  int num_langs;        /* dataset_conf.cat_emb_conf.emb_len when pass_cat_emb, else 0 */
  int vocab;            /* len(symbol_table) */
  int dec_heads;        /* decoder_conf.attention_heads */
  int dec_ffn_dim;      /* decoder_conf.linear_units */
  int dec_blocks;       /* decoder_conf.num_blocks */
  int r_dec_blocks;     /* decoder_conf.r_num_blocks (0: no right-to-left decoder) */
  int sos_id;           /* tokenizer_conf.special_tokens["<sos>"]; <= 0: vocab - 1 (asr_model.py:79-82) */
  int eos_id;           /* tokenizer_conf.special_tokens["<eos>"]; <= 0: vocab - 1 */
  int precision;        /* 0: bf16 tensor-core operands, fp32 accumulate (throughput mode, default)
                         * 1: "bf16x3" fp32-accurate mode — every GEMM operand is a (hi, lo) bf16 pair and runs as three
                         *    wgmma passes hi.hi + lo.hi + hi.lo (~2^-16 relative), attention in fp32: for parity with
                         *    the reference's fp32 graph (bit-exact greedy ids); ~3x the tensor work */
} rvb_model_config;

/* ---- diagnostics -------------------------------------------------------------------------------------------- */
RVB_API const char* rvb_last_error(void);
/* number of CUDA kernels this library has launched so far in this process */
RVB_API unsigned long long rvb_launch_count(void);
/* bytes this library currently holds in the workspaces and weights of its models: device memory and page-locked
 * host memory, over every model and thread of the process */
RVB_API int rvb_held_bytes(long long* device, long long* pinned);
/* 0 = wgmma/TMA GEMM (default), 1 = plain CUDA-core bring-up GEMM (debug only), 2 = wgmma GEMM with 64-wide tiles */
RVB_API int rvb_set_gemm_impl(int impl);
RVB_API int rvb_get_gemm_impl(void);
/* Per-launch CUDA-event timing of the wgmma GEMM kernel between begin/end (the roofline numbers of bench.py):
 * total device time (ms), algorithmic FLOPs (2*M*N*K summed) and launch count.  end() synchronises. */
RVB_API int rvb_gemm_profile_begin(void);
RVB_API int rvb_gemm_profile_end(double* total_ms, double* total_flops, long long* launches);

/* ---- model lifecycle ---------------------------------------------------------------------------------------- */
RVB_API rvb_model* rvb_model_create(const rvb_model_config* cfg);
/* Register one tensor of the reference state_dict under its reference key name (fp32, host memory, copied). */
RVB_API int rvb_model_set_tensor(rvb_model* m, const char* name, const float* h_data, long long numel);
/* Pack the registered tensors into the device layout (bf16 GEMM operands, fused QKV, permuted conv weights). */
RVB_API int rvb_model_finalize(rvb_model* m);
/* Second plan over the same packed weights with its own workspace: lets a second host thread / CUDA stream decode
 * concurrently (a plan serves one stream at a time).  The parent must outlive its forks. */
RVB_API rvb_model* rvb_model_fork(rvb_model* m);
RVB_API void rvb_model_destroy(rvb_model* m);
/* T' = ((T-1)/2 - 1)/2 encoder frames for T feature frames (Conv2dSubsampling4) */
RVB_API int rvb_encoder_out_frames(int T);
/* encoder_lens for a feature length (subsampled padding mask, transformer/subsampling.py:226) */
RVB_API int rvb_encoder_out_len(int feat_len, int T);

/* ---- hot path ----------------------------------------------------------------------------------------------- */
/* Sample-rate conversion (torchaudio.transforms.Resample as called at cli/reverb.py:125-128): orig / new_ are the two
 * rates divided by their gcd, d_kernel the (new_, 2*width + orig) fp32 polyphase windowed-sinc table
 * (reverb_b200/resample.py builds it the way torchaudio does), n_out = ceil(new_ * n_in / orig). */
RVB_API int rvb_resample(const void* d_wave, int is_i16, long long n_in, const float* d_kernel, int orig, int new_, int width,
                         float* d_out, long long n_out, void* stream);
/* number of fbank frames for n_samples (snip_edges): 0 if n < 400 else 1 + (n - 400) / 160 */
RVB_API long long rvb_fbank_num_frames(long long n_samples);
RVB_API int rvb_fbank_f32(const float* d_wave, long long n_samples, float* d_feats, long long n_frames, void* stream);
RVB_API int rvb_fbank_i16(const short* d_wave, long long n_samples, float* d_feats, long long n_frames, void* stream);
/* `batch` equal-length recordings (fixed-length chunks), `wave_stride` samples apart -> d_feats (batch, n_frames, 80) */
RVB_API int rvb_fbank_batch(const void* d_wave, int is_i16, int batch, long long wave_stride, long long n_samples,
                            float* d_feats, long long n_frames, void* stream);

/* feats (B, T, input_dim) fp32 -> enc_out (B, T', d_model) fp32; h_enc_lens[B] receives encoder_lens.
 * h_cat_embs: the LSL mixing weights [verbatimicity, 1 - verbatimicity], one vector (n_cat == num_langs) or one per
 * utterance ((B, num_langs) row-major, n_cat == B * num_langs: utterance b decodes exactly as a batch whose every row
 * carries row b); may be NULL iff num_langs == 0.  The same two lengths are accepted, with B the call's utterance count,
 * by rvb_encoder_forward_chunked / _streaming, rvb_rescoring_submit, rvb_beam_search_rescoring,
 * rvb_attention_rescoring, rvb_decoder_step_topk / _logp and rvb_decoder_cache_begin; in the decoder calls every
 * hypothesis of utterance b uses row b.  Any other n_cat is an error. */
RVB_API int rvb_encoder_forward(rvb_model* m, const float* d_feats, const int* h_feat_lens, int B, int T,
                        const float* h_cat_embs, int n_cat, float* d_enc_out, int* h_enc_lens, void* stream);
/* Same with bounded attention context — BaseEncoder.forward with decoding_chunk_size > 0 (encoder.py:117-149,
 * add_optional_chunk_mask / subsequent_chunk_mask, utils/mask.py:88-197): encoder frame i attends the keys of its own
 * chunk and of num_left_chunks chunks before it (all previous ones when < 0), chunk_size in encoder frames. */
RVB_API int rvb_encoder_forward_chunked(rvb_model* m, const float* d_feats, const int* h_feat_lens, int B, int T,
                                        const float* h_cat_embs, int n_cat, int chunk_size, int num_left_chunks,
                                        float* d_enc_out, int* h_enc_lens, void* stream);

/* The cache-based streaming simulation — BaseEncoder.forward_chunk_by_chunk (encoder.py:341-402; `simulate_streaming`) —
 * evaluated in one batched pass: identical results to feeding the chunks one by one with attention / convolution
 * caches (every frame of d_feats (B, T, input_dim) is taken as real: that path has no padding masks). */
RVB_API int rvb_encoder_forward_streaming(rvb_model* m, const float* d_feats, int B, int T, const float* h_cat_embs,
                                          int n_cat, int chunk_size, int num_left_chunks, float* d_enc_out,
                                          int* h_enc_lens, void* stream);

/* CTC head: logits = ctc_lo(enc_out) (blank_penalty subtracted from the blank column), log_softmax, top-k.
 * d_topk_val/d_topk_idx: (B*Tp, k) sorted descending; d_logp (B*Tp, vocab) optional (NULL to skip the write). */
RVB_API int rvb_ctc_topk(rvb_model* m, const float* d_enc_out, int B, int Tp, int k, float blank_penalty, int blank_id,
                 float* d_topk_val, int* d_topk_idx, float* d_logp, void* stream);
/* top-k of an existing (rows, V) log-prob matrix (no softmax) — used to run the searches on recorded ctc_probs */
RVB_API int rvb_logp_topk(const float* d_logp, int rows, int V, int k, float* d_topk_val, int* d_topk_idx, void* stream);

/* h_tokens: (B, Tp) int32, h_lens: (B) */
RVB_API int rvb_ctc_greedy_search(const int* d_topk_idx, int k, const int* h_enc_lens, int B, int Tp, int blank_id,
                          int* h_tokens, int* h_lens, void* stream);
/* n-best per utterance: h_tokens/h_times (B, beam, max_len) int32, h_lens (B, beam, 2) = {n_tokens, n_times},
 * h_scores (B, beam) float64, h_nhyp (B).  Fails if a hypothesis is longer than max_len. */
RVB_API int rvb_ctc_prefix_beam_search(const float* d_topk_val, const int* d_topk_idx, int k, const int* h_enc_lens, int B,
                               int Tp, int beam, int blank_id, int max_len, int* h_tokens, int* h_times, int* h_lens,
                               double* h_scores, int* h_nhyp, void* stream);

/* ---- context biasing (utils/context_graph.py ContextGraph + the `context_graph` branches of search.py:124-248) ----
 * A graph is uploaded once and used read-only by any number of searches.  Tables (reverb_b200.context_graph
 * device_tables builds them from either graph form): n_nodes states, 0 = root; the children of state s are the edges
 * [h_child_off[s], h_child_off[s+1]) with tokens h_child_tok (strictly increasing within a state) and target states
 * h_child_dst (n_nodes - 1 edges: a trie); h_fail (n_nodes) fail links; h_bonus = node_score, h_emit = output_score,
 * h_token_score = token_score, float64.  Checked before anything is allocated: a trie reachable from the root, tokens in
 * [0, vocab) and != blank_id, fail links to strictly shallower states, finite scores; NULL + rvb_last_error() otherwise.
 * destroy waits for the searches enqueued with the graph, then frees it. */
typedef struct rvb_context_graph rvb_context_graph;
RVB_API rvb_context_graph* rvb_context_graph_create(int n_nodes, const int* h_child_off, const int* h_child_tok,
                                                    const int* h_child_dst, const int* h_fail, const double* h_bonus,
                                                    const double* h_emit, const double* h_token_score, int vocab,
                                                    int blank_id);
RVB_API void rvb_context_graph_destroy(rvb_context_graph* g);
/* rvb_ctc_prefix_beam_search with context biasing: prefixes are ranked by score + context score; h_scores receives
 * score - node_score of the prefix's final state (the reference's finalize), in beam order. */
RVB_API int rvb_ctc_prefix_beam_search_biased(const float* d_topk_val, const int* d_topk_idx, int k,
                                              const int* h_enc_lens, int B, int Tp, int beam, int blank_id, int max_len,
                                              int* h_tokens, int* h_times, int* h_lens, double* h_scores, int* h_nhyp,
                                              rvb_context_graph* graph, void* stream);

/* Teacher-forced (bi-)decoder over the n-best.  h_hyp_tokens (B, N, max_len), h_hyp_lens (B, N) (a negative length
 * marks an absent hypothesis).  h_l2r (B, N, max_len + 1): [j] = log p(w_j | ...) for j < U, [U] = log p(eos);
 * h_r2l likewise for the right-to-left decoder with [j] = r_logp[U-1-j][w_j], [U] = r_logp[U][eos]
 * (only written when reverse_weight > 0 and the model has a right decoder; may be NULL otherwise). */
RVB_API int rvb_attention_rescoring(rvb_model* m, const float* d_enc_out, const int* h_enc_lens, int B, int Tp,
                            const int* h_hyp_tokens, const int* h_hyp_lens, int N, int max_len,
                            const float* h_cat_embs, int n_cat, float reverse_weight, float* h_l2r, float* h_r2l,
                            void* stream);

/* ctc_prefix_beam_search + attention_rescoring in one call, the n-best staying on the device in between
 * (what ASRModel.decode does for method "attention_rescoring", asr_model.py:259-308 / search.py:124-248,378-444).
 * Host outputs are written COMPACT with row length L = *out_max_len (the longest hypothesis / times list, >= 1):
 * h_tokens / h_times (B, beam, L), 0 past each row's n_tokens / n_times, h_l2r / h_r2l (B, beam, L + 1); the caller
 * provides room for L = cap.
 * h_lens (B, beam, 2) = {n_tokens, n_times}, h_scores (B, beam) float64 CTC scores, h_nhyp (B).
 * h_r2l may be NULL (or reverse_weight == 0): the right-to-left decoder is skipped. */
RVB_API int rvb_beam_search_rescoring(rvb_model* m, const float* d_topk_val, const int* d_topk_idx, int k,
                                      const float* d_enc_out, const int* h_enc_lens, int B, int Tp, int beam,
                                      int blank_id, const float* h_cat_embs, int n_cat, float reverse_weight, int cap,
                                      int* h_tokens, int* h_times, int* h_lens, double* h_scores, int* h_nhyp,
                                      float* h_l2r, float* h_r2l, int* out_max_len, void* stream);

/* The same three stages as separate calls around a ticket (0 .. 3 per plan), so that ONE host thread can software-
 * pipeline consecutive batches on one stream: between the calls it enqueues the next batch's encoder, and the GPU never
 * waits for the host (the decoder batch is padded to the longest hypothesis, which the host must learn first).
 *   rvb_search_submit     enqueues the prefix beam search (+ the small copy of lengths / counts / CTC scores);
 *                         returns the ticket (>= 0) or < 0.  d_enc_out must stay valid until the ticket is collected.
 *   rvb_rescoring_submit  blocks until that small copy has landed, then enqueues the decoder passes (run_decoder != 0)
 *                         and the copies of tokens / times / decoder scores INTO THE CALLER'S h_ buffers, which must be
 *                         page-locked for the call to stay asynchronous and must stay valid until collect;
 *                         *out_max_len = L as in rvb_beam_search_rescoring.  run_decoder == 0: prefix beam search only.
 *   rvb_rescoring_collect blocks until those copies are done, fills h_lens / h_scores / h_nhyp, re-indexes h_r2l to
 *                         hypothesis order and frees the ticket. */
RVB_API int rvb_search_submit(rvb_model* m, const float* d_topk_val, const int* d_topk_idx, int k, const float* d_enc_out,
                              const int* h_enc_lens, int B, int Tp, int beam, int blank_id, void* stream);
/* rvb_search_submit with context biasing (see rvb_ctc_prefix_beam_search_biased); the rest of the ticket is unchanged.
 * The graph must not be destroyed before the ticket is collected or released. */
RVB_API int rvb_search_submit_biased(rvb_model* m, const float* d_topk_val, const int* d_topk_idx, int k,
                                     const float* d_enc_out, const int* h_enc_lens, int B, int Tp, int beam, int blank_id,
                                     rvb_context_graph* graph, void* stream);
RVB_API int rvb_rescoring_submit(rvb_model* m, int ticket, const float* h_cat_embs, int n_cat, float reverse_weight, int cap,
                                 int run_decoder, int* h_tokens, int* h_times, float* h_l2r, float* h_r2l,
                                 int* out_max_len, void* stream);
RVB_API int rvb_rescoring_collect(rvb_model* m, int ticket, int* h_lens, double* h_scores, int* h_nhyp);
/* abandon a ticket in any state (waits for its pending copies; used on error paths) */
RVB_API int rvb_ticket_release(rvb_model* m, int ticket);

/* One step of the autoregressive `attention` decode mode (attention_beam_search, search.py:251-360: the
 * decoder.forward_one_step + logp.topk(beam) pair of lines 302-306).  h_hyps (B*N, L) int32: the running hypotheses
 * (sos first), N per utterance, all of length L; runs the LEFT decoder over them against the utterance's encoder output
 * (keys >= h_enc_lens[b] masked) and returns log_softmax(top-k) of the last position: h_topk_val / h_topk_idx (B*N, k). */
RVB_API int rvb_decoder_step_topk(rvb_model* m, const float* d_enc_out, const int* h_enc_lens, int B, int Tp, int N,
                                  const int* h_hyps, int L, const float* h_cat_embs, int n_cat, int k, float* h_topk_val,
                                  int* h_topk_idx, void* stream);

/* The decoder step with a per-layer KEY / VALUE cache (decoder.forward_one_step with its `cache`, decoder.py:191-234, as
 * driven by attention_beam_search, search.py:290-346):
 *   begin  projects the source-attention keys / values of the encoder output once and sizes the caches for
 *          max_steps positions of B * N hypotheses;
 *   step   takes the LAST token of every running hypothesis (h_tokens (B*N)) and, from the second step on, the index
 *          of the hypothesis each one extends (h_parents (B*N): the caches are gathered accordingly — the
 *          torch.index_select of search.py:341-346; NULL = identity), runs ONE position through the left decoder and
 *          returns log_softmax top-k: h_topk_val / h_topk_idx (B*N, k);
 *   end    frees the caches.  Same values as rvb_decoder_step_topk, which recomputes the whole prefix every step. */
RVB_API int rvb_decoder_cache_begin(rvb_model* m, const float* d_enc_out, const int* h_enc_lens, int B, int Tp, int N,
                                    int max_steps, const float* h_cat_embs, int n_cat, void* stream);
RVB_API int rvb_decoder_cache_step(rvb_model* m, const int* h_tokens, const int* h_parents, int k, float* h_topk_val,
                                   int* h_topk_idx, void* stream);
RVB_API int rvb_decoder_cache_end(rvb_model* m);

/* The same decoder step returning the FULL log_softmax row of the last position, h_logp (B*N, vocab) — what
 * decoder.forward_one_step_with_attn (transformer/decoder.py:236-281) hands to BeamSearchTimeSync
 * (espnet/beam_search_timesync.py:156-164, 211-218: `joint_decoding`, search.py:450-496). */
RVB_API int rvb_decoder_step_logp(rvb_model* m, const float* d_enc_out, const int* h_enc_lens, int B, int Tp, int N,
                                  const int* h_hyps, int L, const float* h_cat_embs, int n_cat, float* h_logp,
                                  void* stream);

/* ---- CTC forced alignment of a known transcript (force_align, utils/ctc_utils.py:95-161; driver bin/alignment.py) ----
 * Viterbi over the states [b, y0, b, y1, ..., y_{U-1}, b] in fp32 with the reference's tie rules (stay, then s-1, then
 * s-2; end state S-1 unless S-2 is strictly better): the frame alignment is the reference's, bit for bit.
 * Batched form, B utterances that each fit one chunk: d_logp (B*Tp, V) fp32 log-probs (rvb_ctc_topk's d_logp),
 * h_labels (B, max_U) / h_label_lens (B).  Host outputs: h_frames (B, Tp) the token id of every frame (blank_id or a
 * label; -1 from h_enc_lens[b] on), h_first / h_last / h_peak (B, max_U) first, last and peak frame of every label (peak =
 * the frame of its span with the largest log-prob, first on ties), h_peak_logp (B, max_U) that log-prob, h_score (B)
 * the Viterbi score, h_loglik (B) log p(y | x) by the forward algorithm in float64 (NULL: skipped).
 * An alignment exists iff U >= 1 and enc_len >= U + #(adjacent equal labels); an empty or infeasible label sequence, a
 * label that is blank or >= V, or U > 12287 fails on the host, before any launch, naming the utterance. */
RVB_API int rvb_ctc_force_align(const float* d_logp, int V, const int* h_enc_lens, int B, int Tp, const int* h_labels,
                                const int* h_label_lens, int max_U, int blank_id, int* h_frames, int* h_first,
                                int* h_last, int* h_peak, float* h_peak_logp, float* h_score, double* h_loglik,
                                void* stream);

/* Resumable form, ONE trellis fed piecewise — what carries a transcript across the independent encoder chunks of a long
 * recording; any split of the rows gives exactly the result of a single push.
 *   begin   labels, the total number of frames that will be pushed, and a budget: the handle owns
 *           rvb_aligner_workspace_bytes() of device memory — per frame and label slot (U + 1 rounded up to 128, or to
 *           768 above 4095 labels) 1 byte of back-pointers and 4 bytes of emission log-prob, i.e. about
 *           5 * total_frames * (U + 1) bytes: 5.6 GB for one hour (90 500 frames) against 12 000 tokens.  A request
 *           over budget_bytes (> 0) fails before anything is allocated.  m may be NULL; with a model the trellis runs on
 *           the model's search side stream, so that it hides under the next encoder pass on `stream`.
 *   push    n_rows further rows of (n_rows, V) log-probs: only the valid frames of a chunk.  The rows are consumed in
 *           stream order on `stream` (they may be overwritten by later work on it); nothing is synchronised.
 *   finish  frames indexed over the whole recording, outputs as above with B = 1, Tp = total_frames, max_U = U;
 *           synchronises, then frees the handle — also when it fails.  abort frees a handle that will not be finished. */
typedef struct rvb_aligner rvb_aligner;
RVB_API long long rvb_aligner_workspace_bytes(int U, int total_frames, int want_loglik);
RVB_API rvb_aligner* rvb_aligner_begin(rvb_model* m, const int* h_labels, int U, int total_frames, int V, int blank_id,
                                       int want_loglik, long long budget_bytes, void* stream);
RVB_API int rvb_aligner_push(rvb_aligner* a, const float* d_logp, int n_rows, void* stream);
RVB_API int rvb_aligner_finish(rvb_aligner* a, int* h_frames, int* h_first, int* h_last, int* h_peak, float* h_peak_logp,
                               float* h_score, double* h_loglik, void* stream);
RVB_API void rvb_aligner_abort(rvb_aligner* a);

/* ---- kernel-level entry points (parity tests, profiling) ----------------------------------------------------- */
/* C[M,N] = A[M,K] W[N,K]^T + bias; act: 0 none 1 relu 2 silu 3 glu; out_mode: 0 bf16, 1 f32, 2 f32 residual += alpha*(.)
 * act 3 (pointwise_conv1 + GLU of the conformer conv module, convolution.py:129-130): bf16 output (M, N/2); W / bias
 * rows interleaved in groups of 32 — rows [64j, 64j+32) are the value half of output channels [32j, 32j+32), rows
 * [64j+32, 64j+64) their gates; out[m, c] = value * sigmoid(gate). */
RVB_API int rvb_gemm_bf16(const void* d_A, const void* d_W, const float* d_bias, int M, int N, int K, int act, int out_mode,
                  float alpha, void* d_out, int ldo, void* stream);
/* For tests and tools: rvb_gemm_bf16 with the row mask the encoder applies internally (not needed to run a model).
 * Row m is batch m / rows_per_batch, position m % rows_per_batch, and is written only if position < d_row_lens[batch]
 * (int32, device); masked rows of d_out are left untouched. */
RVB_API int rvb_gemm_bf16_rows(const void* d_A, const void* d_W, const float* d_bias, int M, int N, int K, int act,
                               int out_mode, float alpha, void* d_out, int ldo, const int* d_row_lens, int rows_per_batch,
                               void* stream);
/* The same GEMM in the fp32-accurate "bf16x3" mode (rvb_model_config.precision = 1): d_A (M, 2K) and d_W (N, 2K) hold
 * (hi | lo) bf16 pairs — hi = bf16(v), lo = bf16(v - hi), rvb_f32_to_bf16_pair builds them — and three wgmma passes
 * hi.hi + lo.hi + hi.lo accumulate in fp32.  bf16 outputs (out_mode 0) are written as such a pair too: (M, 2N), or
 * (M, N) = (value half | residue half) of the N/2 GLU outputs; ldo = 0 selects that width. */
RVB_API int rvb_gemm_bf16x3(const void* d_A, const void* d_W, const float* d_bias, int M, int N, int K, int act, int out_mode,
                            float alpha, void* d_out, int ldo, void* stream);
/* The grouped GEMM of the language-specific layers with per-utterance mixing weights: d_W (N, K) and d_bias (N) stack
 * N / group_n blocks of group_n rows (one folded linear per group).  Row m belongs to utterance m / rows_per_batch and is
 * computed with the block of its group d_grp[m / rows_per_batch] (int32, device) only, into output columns
 * [0, group_n) of d_out (ldo 0 -> group_n, or 2 * group_n for a bf16 pair).  Bit-equal to a plain rvb_gemm_bf16 /
 * rvb_gemm_bf16x3 (x3 = 1) launch with that group's block.  out_mode 0 (bf16) or 1 (f32), no activation. */
RVB_API int rvb_gemm_grouped(const void* d_A, const void* d_W, const float* d_bias, int M, int N, int K, int out_mode,
                             void* d_out, int ldo, const int* d_grp, int rows_per_batch, int group_n, int x3,
                             void* stream);
/* (rows, width) fp32 -> (rows, 2 * width) bf16 = [hi | lo] */
RVB_API int rvb_f32_to_bf16_pair(const float* d_x, void* d_out, long long rows, int width, void* stream);
/* out[m] = log_softmax(A W^T + bias)[m, gather[m]] (0 where gather[m] < 0) without materialising the (M, N) logits:
 * the GEMM epilogue emits per-slab (max, sum-exp) partials + the gathered logit into d_ws
 * (rvb_gemm_logsoftmax_gather_ws_bytes(M, N) bytes), a second kernel merges them.  This is the output layer +
 * log_softmax + per-token indexing of attention rescoring (asr_model.py:868-978, search.py:413-436).  N > 128. */
RVB_API long long rvb_gemm_logsoftmax_gather_ws_bytes(int M, int N);
RVB_API int rvb_gemm_logsoftmax_gather(const void* d_A, const void* d_W, const float* d_bias, int M, int N, int K,
                                       const int* d_gather, void* d_ws, float* d_out, void* stream);
RVB_API int rvb_layernorm(const float* d_x, const float* d_gamma, const float* d_beta, float eps, int M, int d,
                  void* d_out_bf16, float* d_out_f32, void* stream);
/* q/k/v/out bf16, (B, T, H, dk) with the given row strides; p (Tk, H, dk) optional rel-pos keys */
RVB_API int rvb_attention(const void* d_q, const void* d_k, const void* d_v, const void* d_p, const float* d_bias_u,
                  const float* d_bias_v, void* d_out, int ldq, int ldk, int ldv, int ldp, int ldo, int Bq, int Tq, int Tk,
                  int H, int dk, int q_per_kv, const int* d_k_lens, const int* d_q_lens, int causal, float scale,
                  void* stream);
/* wgmma attention (d_k = 64): group g owns query rows [g*Tq, ..) and key rows [g*Tk, ..); pointers address head 0;
 * d_key_bias (groups, H, Tk) fp32 optional (added to q.k before scaling), d_k_lens (groups) optional; causal != 0
 * (needs Tq == Tk): key j is visible to query i iff j <= i (decoder self-attention, utils/mask.py subsequent_mask). */
RVB_API int rvb_attention_tc(const void* d_q, const void* d_k, const void* d_v, void* d_out, int ldq, int ldk, int ldv,
                             int ldo, int groups, int Tq, int Tk, int H, int dk, const float* d_key_bias,
                             const int* d_k_lens, int causal, float scale, void* stream);
/* same with the streaming chunk mask of utils/mask.py:88-123 (Tq == Tk): query i sees keys
 * [max(0, (i/chunk - left_chunks) * chunk) (0 when left_chunks < 0), (i/chunk + 1) * chunk) */
RVB_API int rvb_attention_tc_chunked(const void* d_q, const void* d_k, const void* d_v, void* d_out, int ldq, int ldk,
                                     int ldv, int ldo, int groups, int Tq, int Tk, int H, int dk, const float* d_key_bias,
                                     const int* d_k_lens, int chunk, int left_chunks, float scale, void* stream);
/* For tests and tools: rvb_attention_tc with per-(query row, key) visibility bits on top of the key-length and causal
 * masks, as the prefix-tree rescoring applies internally.  Bit (j & 31) of d_key_bits[(g*Tq + i) * bits_ld + (j >> 5)]
 * (uint32, device) set <=> key j visible to query row i of group g; bits_ld >= 2 * ceil(Tk / 64). */
RVB_API int rvb_attention_tc_bits(const void* d_q, const void* d_k, const void* d_v, void* d_out, int ldq, int ldk,
                                  int ldv, int ldo, int groups, int Tq, int Tk, int H, int dk, const float* d_key_bias,
                                  const int* d_k_lens, int causal, const void* d_key_bits, int bits_ld, float scale,
                                  void* stream);
/* For tests and tools: CTAs per SM of the wgmma attention instantiation a launch with these masks and Tk runs
 * (chunk > 0: rvb_attention_tc_chunked; with_key_bits != 0: rvb_attention_tc_bits); -1 on error */
RVB_API int rvb_attention_tc_blocks_per_sm(int Tk, int causal, int chunk, int with_key_bits);
/* K'' = k + pos (bf16) and cbias[b,h,t] = u_h.k + v_h.pos for the folded rel-pos attention */
RVB_API int rvb_relpos_prep(const void* d_k, int ldk, const void* d_pos, int ldp, const float* d_bias_u,
                            const float* d_bias_v, void* d_kpp, float* d_cbias, int B, int T, int H, int dk,
                            void* stream);
RVB_API int rvb_f32_to_bf16(const float* d_x, void* d_out, long long n, void* stream);

/* ---- FLAC decoding (RFC 9639; csrc/flac.cu, DESIGN.md §4k) ------------------------------------------------------
 * The caller parses the metadata blocks on the host and uploads the whole file once (d_bytes, n_bytes); the frames
 * start at byte audio_offset, right after the last metadata block.  rvb_flac_index finds the frames, rvb_flac_decode
 * decodes them; both synchronise the stream before returning. */
typedef struct rvb_flac_info {
  int sample_rate;      /* STREAMINFO: Hz, > 0 */
  int channels;         /* 1..8 */
  int bits_per_sample;  /* 4..32 */
  int max_block_size;   /* samples per channel of the largest frame (a launch-shape hint; larger frames still decode) */
} rvb_flac_info;
/* device workspace rvb_flac_index needs for a file of n_bytes bytes; it holds the frame index rvb_flac_decode reads */
RVB_API long long rvb_flac_index_workspace_bytes(long long n_bytes);
/* Finds every frame header (sync code, valid fields, CRC-8) and keeps the chain of frames whose coded frame / sample
 * numbers are consecutive from the frame at audio_offset.  h_n_frames: frames in the chain, 0 when no valid frame
 * header is at audio_offset, -1 when the bytes hold more sync candidates than any FLAC stream of that size;
 * h_total_samples: their block sizes summed (STREAMINFO may state 0, "unknown"). */
RVB_API int rvb_flac_index(const void* d_bytes, long long n_bytes, long long audio_offset, const rvb_flac_info* info,
                           void* d_workspace, long long workspace_bytes, int* h_n_frames, long long* h_total_samples,
                           void* stream);
/* device workspace rvb_flac_decode needs; -1 on bad arguments */
RVB_API long long rvb_flac_decode_workspace_bytes(int n_frames, long long total_samples, const rvb_flac_info* info);
/* Decodes the indexed frames into d_out (channels, total_samples), left-justified: int16 (x << (16 - bps)) for
 * bits_per_sample <= 16, int32 (x << (32 - bps)) above.  Every frame is checked (header against STREAMINFO, subframe
 * syntax, bounds of every read, CRC-16, the frame ending where the next begins); h_bad_frame is the lowest failing frame
 * (-1: none), h_bad_offset the byte offset concerned and h_bad_status its cause: 1 bad header, 2 header disagrees with
 * STREAMINFO, 3 bad subframe, 4 bad residual coding, 5 frame truncated, 6 CRC-16 mismatch, 7 no frame header where the
 * frame ends.  Samples of a failing frame are not written. */
RVB_API int rvb_flac_decode(const void* d_bytes, long long n_bytes, const rvb_flac_info* info,
                            const void* d_index_workspace, int n_frames, long long total_samples, void* d_workspace,
                            long long workspace_bytes, void* d_out, int* h_bad_frame, long long* h_bad_offset,
                            int* h_bad_status, void* stream);

/* ---- compressed WAV decoding: G.711 and ADPCM (csrc/wav_codec.cu, DESIGN.md §4l) ---------------------------------
 * The caller parses and validates the fmt chunk on the host and uploads the data chunk once (d_data, n_bytes). */
typedef struct rvb_wav_codec {
  int format_tag;         /* WAVE format tag: 0x0007 mu-law, 0x0006 A-law, 0x0011 IMA ADPCM, 0x0002 MS ADPCM */
  int channels;           /* >= 1 (MS ADPCM: 1 or 2) */
  int block_align;        /* bytes per block; G.711: channels */
  int samples_per_block;  /* per channel, header samples included (ADPCM) */
  int n_coef;             /* MS ADPCM: coefficient pairs, 7..256 */
  short coef[512];        /* MS ADPCM: n_coef pairs (c1, c2) */
} rvb_wav_codec;
/* Decodes the first `frames` samples of every channel into d_out (channels, frames) int16; samples past `frames` are
 * not written and no read leaves its block or the data span.  G.711 expands every byte; an ADPCM block decodes from
 * the state in its header, one thread per (block, channel).  h_bad_block is the lowest block whose header is invalid
 * (-1: none) and h_bad_status its cause: 1 IMA step index above 88, 2 MS ADPCM predictor index >= n_coef.  Returns -2
 * when `frames` is more than the bytes hold.  Synchronises the stream before returning. */
RVB_API int rvb_wav_decode(const void* d_data, long long n_bytes, const rvb_wav_codec* info, long long frames,
                           void* d_out, int* h_bad_block, int* h_bad_status, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* RVB_B200_H_ */
