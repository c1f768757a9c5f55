// reverb_b200 — CTC forced alignment of a known transcript on the GPU (reference: force_align / insert_blank,
// utils/ctc_utils.py:95-161, driven by bin/alignment.py one utterance at a time in a Python double loop).
//
// Labels y[0..U) give the states z = [b, y0, b, y1, ..., b, y_{U-1}, b], S = 2U + 1.  The kernels work on "slots":
// slot u < U holds the state pair (2u: the blank before y_u, 2u+1: y_u), slot U holds the trailing blank (its label
// half stays -inf).  The Viterbi update of ctc_utils.py:128-144 in slot form, fp32, one add per cell:
//     B'[u] = max(B[u], L[u-1])                      + logp[t][blank]      ties -> stay
//     L'[u] = max(L[u], B[u], L[u-1] if y_u != y_{u-1}) + logp[t][y_u]     ties -> stay, then s-1, then s-2
// so a slot needs ONE value of its left neighbour per frame, L[u-1].
//
//   align_gather          (rows, V) log-probs -> compact emissions em (rows, E): column u = logp[y_u] (u < U), -inf for
//                         the padding columns, column P = logp[blank].  The trellis walks the frames serially, and a
//                         scattered 4-byte read of a 40 KB row per state and frame would be its limiter; the gather is
//                         embarrassingly parallel, and afterwards every thread of the trellis reads its own K contiguous
//                         floats per frame.  The emissions are also what the per-token peak needs once the path is known.
//   ctc_viterbi_forward   one CTA per utterance, K slots per thread in registers, L[u-1] from the left neighbour by
//                         shuffle (and one shared-memory word per warp); next frame's emissions prefetched into
//                         registers; one byte of back-pointers per slot and frame; alpha in / out for a frame range.
//   ctc_forward_loglik    the forward algorithm on the same trellis in float64 (log p(y | x)), optional.
//   ctc_viterbi_backtrace end state (S-1 unless S-2 is strictly better), score, state per frame.
//   align_reduce          token id per frame; first / last / peak frame and peak log-prob per label.
#include <math.h>
#include <string.h>

#include <vector>

#include "../../include/rvb_b200.h"
#include "kernels.h"

namespace rvb {

constexpr int AL_K_SMALL = 4, AL_THREADS_SMALL = 1024;   // up to 4096 slots
constexpr int AL_K_LARGE = 24, AL_THREADS_LARGE = 512;   // up to 12288 slots
constexpr int AL_MAX_LABELS = AL_K_LARGE * AL_THREADS_LARGE - 1;

struct AlignGeom {
  int K, threads, P, E;  // slots per thread, CTA size, padded slots (= threads * K), emission row stride (floats)
};
static AlignGeom align_geom(int max_U) {
  AlignGeom g;
  const int slots = max_U + 1;
  g.K = slots <= AL_K_SMALL * AL_THREADS_SMALL ? AL_K_SMALL : AL_K_LARGE;
  g.threads = (((slots + g.K - 1) / g.K) + 31) / 32 * 32;
  g.P = g.threads * g.K;
  g.E = g.P + 4;  // blank at column P; rows stay 16-byte aligned
  return g;
}

// ---------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
align_gather_kernel(const float* __restrict__ logp, int V, int rows_per_utt, const int* __restrict__ labels,
                    int lab_stride, const int* __restrict__ ulens, const int* __restrict__ lens, int blank,
                    float* __restrict__ em, int E, int P) {
  const int row = blockIdx.x, b = row / rows_per_utt, t = row - b * rows_per_utt;
  if (lens != nullptr && t >= lens[b]) return;
  const int U = ulens[b];
  const int* lab = labels + (size_t)b * lab_stride;
  const float* x = logp + (size_t)row * V;
  float* o = em + (size_t)row * E;
  for (int c = threadIdx.x; c < E; c += 256) o[c] = c < U ? x[lab[c]] : (c == P ? x[blank] : -INFINITY);
}

// ---------------------------------------------------------------------------------------------------------------
// Frames [t0, min(t1, lens[b])) of utterance b.  t0 == 0 starts the trellis (ctc_utils.py:124-126), otherwise alpha
// (B, 2, P) = [blank halves | label halves] is read; it is written back at the end, so that the calls on [0, a),
// [a, b), [b, T) perform exactly the operations of one call on [0, T).
template <int K, int THREADS>
__global__ void __launch_bounds__(THREADS)
ctc_viterbi_forward_kernel(const float* __restrict__ em, int E, int P, unsigned char* __restrict__ bp,
                           const int* __restrict__ labels, int lab_stride, const int* __restrict__ ulens,
                           const int* __restrict__ lens, int rows_per_utt, float* __restrict__ alpha, int t0, int t1) {
  __shared__ float s_bound[2][32];
  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int U = ulens[b], T = min(lens[b], t1), u0 = tid * K;
  const float* emb = em + (size_t)b * rows_per_utt * E;
  unsigned char* bpb = bp + (size_t)b * rows_per_utt * P;
  float* gB = alpha + (size_t)b * 2 * P;
  float* gL = gB + P;
  const int* lab = labels + (size_t)b * lab_stride;
  const bool multi = blockDim.x > 32;

  unsigned skip = 0;  // bit j: the s-2 transition into label u0 + j is allowed (ctc_utils.py:130-131)
#pragma unroll
  for (int j = 0; j < K; ++j) {
    const int u = u0 + j;
    if (u >= 1 && u < U && lab[u] != lab[u - 1]) skip |= 1u << j;
  }
  float aB[K], aL[K];
  int t = t0;
  if (t0 == 0) {
#pragma unroll
    for (int j = 0; j < K; ++j) aB[j] = aL[j] = -INFINITY;
    if (tid == 0) {
      aB[0] = emb[P];
      aL[0] = emb[0];
    }
    t = 1;
  } else {
#pragma unroll
    for (int j = 0; j < K; ++j) {
      aB[j] = gB[u0 + j];
      aL[j] = gL[u0 + j];
    }
  }
  float e[K], eb = 0.f;
  if (t < T) {
    const float4* r = reinterpret_cast<const float4*>(emb + (size_t)t * E + u0);
#pragma unroll
    for (int q = 0; q < K / 4; ++q) {
      const float4 v = r[q];
      e[4 * q] = v.x, e[4 * q + 1] = v.y, e[4 * q + 2] = v.z, e[4 * q + 3] = v.w;
    }
    eb = emb[(size_t)t * E + P];
  }
  for (; t < T; ++t) {
    // L[u0 - 1] of frame t - 1: the left neighbour's last label half
    float left = __shfl_up_sync(0xffffffffu, aL[K - 1], 1);
    if (multi) {
      if (lane == 31) s_bound[t & 1][warp] = aL[K - 1];
      __syncthreads();
      if (lane == 0) left = warp > 0 ? s_bound[t & 1][warp - 1] : -INFINITY;
    } else if (lane == 0) {
      left = -INFINITY;
    }
    float4 nx[K / 4];
    float nb = 0.f;
    if (t + 1 < T) {  // next frame's emissions travel while this frame is computed
      const float4* r = reinterpret_cast<const float4*>(emb + (size_t)(t + 1) * E + u0);
#pragma unroll
      for (int q = 0; q < K / 4; ++q) nx[q] = r[q];
      nb = emb[(size_t)(t + 1) * E + P];
    }
    uint32_t packed[K / 4];
#pragma unroll
    for (int q = 0; q < K / 4; ++q) packed[q] = 0u;
#pragma unroll
    for (int j = 0; j < K; ++j) {
      const float oldB = aB[j], oldL = aL[j];
      const bool fromL = left > oldB;  // torch.argmax: the first maximum, i.e. "stay" on ties
      float m = oldL;
      unsigned p = 0u;
      if (oldB > m) {
        m = oldB;
        p = 1u;
      }
      if (((skip >> j) & 1u) && left > m) {
        m = left;
        p = 2u;
      }
      aB[j] = (fromL ? left : oldB) + eb;
      aL[j] = m + e[j];
      packed[j >> 2] |= (p | (fromL ? 4u : 0u)) << (8 * (j & 3));
      left = oldL;
    }
    uint32_t* o = reinterpret_cast<uint32_t*>(bpb + (size_t)t * P + u0);
#pragma unroll
    for (int q = 0; q < K / 4; ++q) o[q] = packed[q];
    if (t + 1 < T) {
#pragma unroll
      for (int q = 0; q < K / 4; ++q)
        e[4 * q] = nx[q].x, e[4 * q + 1] = nx[q].y, e[4 * q + 2] = nx[q].z, e[4 * q + 3] = nx[q].w;
      eb = nb;
    }
  }
#pragma unroll
  for (int j = 0; j < K; ++j) {
    gB[u0 + j] = aB[j];
    gL[u0 + j] = aL[j];
  }
}

// ---------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ double log_add3(double a, double b, double c) {
  const double m = fmax(a, fmax(b, c));
  if (m == -INFINITY) return m;
  return m + log(exp(a - m) + exp(b - m) + exp(c - m));
}

// Forward algorithm over the states s < 2U + 1 in float64; a64 (B, 2, 2P): frame t lives in buffer t & 1, in global
// memory, so the same call sequence as the Viterbi pass resumes it.  *out is written once the last frame is in.
__global__ void __launch_bounds__(1024)
ctc_forward_loglik_kernel(const float* __restrict__ em, int E, int P, const int* __restrict__ labels, int lab_stride,
                          const int* __restrict__ ulens, const int* __restrict__ lens, int rows_per_utt,
                          double* __restrict__ a64, int t0, int t1, double* __restrict__ out) {
  const int b = blockIdx.x, U = ulens[b], S = 2 * U + 1, T = min(lens[b], t1);
  const float* emb = em + (size_t)b * rows_per_utt * E;
  const int* lab = labels + (size_t)b * lab_stride;
  double* a = a64 + (size_t)b * 4 * P;
  int t = t0;
  if (t0 == 0) {
    for (int s = threadIdx.x; s < S; s += blockDim.x)
      a[s] = s == 0 ? (double)emb[P] : (s == 1 ? (double)emb[0] : -INFINITY);
    t = 1;
    __syncthreads();
  }
  for (; t < T; ++t) {
    const double* prev = a + (size_t)((t - 1) & 1) * 2 * P;
    double* cur = a + (size_t)(t & 1) * 2 * P;
    const float* er = emb + (size_t)t * E;
    for (int s = threadIdx.x; s < S; s += blockDim.x) {
      const int u = s >> 1;
      const bool is_label = s & 1;
      const double c1 = s >= 1 ? prev[s - 1] : -INFINITY;
      const double c2 = (is_label && u >= 1 && lab[u] != lab[u - 1]) ? prev[s - 2] : -INFINITY;
      cur[s] = log_add3(prev[s], c1, c2) + (double)(is_label ? er[u] : er[P]);
    }
    __syncthreads();
  }
  if (threadIdx.x == 0 && T == lens[b] && T > t0) {
    const double* fin = a + (size_t)((T - 1) & 1) * 2 * P;
    out[b] = log_add3(fin[S - 1], fin[S - 2], -INFINITY);
  }
}

// ---------------------------------------------------------------------------------------------------------------
// One thread per utterance walks the back-pointers (ctc_utils.py:146-155); state (B, rows_per_utt) int32.
__global__ void ctc_viterbi_backtrace_kernel(const unsigned char* __restrict__ bp, int P, const float* __restrict__ alpha,
                                             const int* __restrict__ ulens, const int* __restrict__ lens,
                                             int rows_per_utt, int* __restrict__ state, float* __restrict__ score) {
  const int b = blockIdx.x;
  if (threadIdx.x != 0) return;
  const int U = ulens[b], T = lens[b];
  const float endB = alpha[(size_t)b * 2 * P + U], endL = alpha[(size_t)b * 2 * P + P + U - 1];
  int s = endL > endB ? 2 * U - 1 : 2 * U;  // ctc_utils.py:148-153: argmax([alpha[S-1], alpha[S-2]])
  score[b] = endL > endB ? endL : endB;
  const unsigned char* bpb = bp + (size_t)b * rows_per_utt * P;
  int* st = state + (size_t)b * rows_per_utt;
  for (int t = T - 1; t >= 0; --t) {
    st[t] = s;
    if (t > 0) {
      const unsigned v = bpb[(size_t)t * P + (s >> 1)];
      s -= (s & 1) ? (int)(v & 3u) : (int)((v >> 2) & 1u);
    }
  }
}

// One thread per frame: the frame's token id; the thread of a label's first frame scans its span for the peak — the
// frame with the largest logp[t][y_u], the first one on ties.
__global__ void __launch_bounds__(256)
align_reduce_kernel(const int* __restrict__ state, const float* __restrict__ em, int E, const int* __restrict__ labels,
                    int lab_stride, const int* __restrict__ lens, int rows_per_utt, int blank, int max_U,
                    int* __restrict__ frames, int* __restrict__ first, int* __restrict__ last, int* __restrict__ peak,
                    float* __restrict__ peak_logp) {
  const int b = blockIdx.y, t = blockIdx.x * 256 + threadIdx.x;
  if (t >= rows_per_utt) return;
  const int T = lens[b];
  int* fr = frames + (size_t)b * rows_per_utt;
  if (t >= T) {
    fr[t] = -1;
    return;
  }
  const int* st = state + (size_t)b * rows_per_utt;
  const int s = st[t], u = s >> 1;
  fr[t] = (s & 1) ? labels[(size_t)b * lab_stride + u] : blank;
  if (!(s & 1) || (t > 0 && st[t - 1] == s)) return;
  const float* eu = em + (size_t)b * rows_per_utt * E + u;
  float best = eu[(size_t)t * E];
  int bt = t, q = t + 1;
  for (; q < T && st[q] == s; ++q) {
    const float v = eu[(size_t)q * E];
    if (v > best) {
      best = v;
      bt = q;
    }
  }
  const size_t o = (size_t)b * max_U + u;
  first[o] = t;
  last[o] = q - 1;
  peak[o] = bt;
  peak_logp[o] = best;
}

// ---------------------------------------------------------------------------------------------------------------
// Everything the device needs for B trellises that share one geometry.  The host checks feasibility before any launch.
struct AlignDev {
  AlignGeom g;
  int B = 0, rows = 0, max_U = 0, blank = 0, V = 0;
  int* labels = nullptr;  // (B, max_U) | ulens (B) | lens (B)
  int *ulens = nullptr, *lens = nullptr;
  float* em = nullptr;
  unsigned char* bp = nullptr;
  float* alpha = nullptr;
  double* a64 = nullptr;  // (B, 2, 2P) + ll (B)
  double* ll = nullptr;
  int* out = nullptr;  // state | frames (B, rows) | first | last | peak (B, max_U) | peak_logp | score (B)
};

static size_t align_bytes(const AlignGeom& g, int B, long long rows, int max_U, bool loglik) {
  size_t n = (size_t)B * rows * ((size_t)g.E * 4 + g.P);                       // emissions + back-pointers
  n += (size_t)B * 2 * g.P * 4 + ((size_t)B * max_U + 2 * B) * 4;              // alpha, labels, lengths
  n += ((size_t)2 * B * rows + (size_t)4 * B * max_U + B) * 4;                 // outputs
  if (loglik) n += (size_t)B * (4 * g.P + 1) * 8;
  return n + 8 * 256;
}

static void align_free(AlignDev& d) {
  void* ptrs[] = {d.labels, d.em, d.bp, d.alpha, d.a64, d.out};
  for (void* p : ptrs)
    if (p) cudaFree(p);
  d = AlignDev();
}

static int align_alloc(AlignDev& d, int B, int rows, int max_U, int V, int blank, bool loglik) {
  d.g = align_geom(max_U);
  d.B = B, d.rows = rows, d.max_U = max_U, d.V = V, d.blank = blank;
  const AlignGeom& g = d.g;
  RVB_CHECK_CUDA(cudaMalloc(&d.labels, ((size_t)B * max_U + 2 * B) * sizeof(int)));
  d.ulens = d.labels + (size_t)B * max_U;
  d.lens = d.ulens + B;
  RVB_CHECK_CUDA(cudaMalloc(&d.em, (size_t)B * rows * g.E * sizeof(float)));
  RVB_CHECK_CUDA(cudaMalloc(&d.bp, (size_t)B * rows * g.P));
  RVB_CHECK_CUDA(cudaMalloc(&d.alpha, (size_t)B * 2 * g.P * sizeof(float)));
  if (loglik) {
    RVB_CHECK_CUDA(cudaMalloc(&d.a64, (size_t)B * (4 * g.P + 1) * sizeof(double)));
    d.ll = d.a64 + (size_t)B * 4 * g.P;
  }
  RVB_CHECK_CUDA(cudaMalloc(&d.out, ((size_t)2 * B * rows + (size_t)4 * B * max_U + B) * sizeof(int)));
  return 0;
}

// An alignment exists iff T >= U + #(adjacent equal labels), U >= 1 (every repeat needs a blank frame in between).
static int align_check(const char* who, int b, const int* lab, int U, long long T, int V, int blank) {
  RVB_REQUIRE(U >= 1, "%s: utterance %d has an empty label sequence", who, b);
  RVB_REQUIRE(U <= AL_MAX_LABELS, "%s: utterance %d has %d labels, the trellis kernel holds at most %d", who, b, U,
              AL_MAX_LABELS);
  long long need = U;
  for (int u = 0; u < U; ++u) {
    RVB_REQUIRE(lab[u] >= 0 && lab[u] < V && lab[u] != blank, "%s: utterance %d label %d = %d is not a non-blank id below %d",
                who, b, u, lab[u], V);
    if (u > 0 && lab[u] == lab[u - 1]) ++need;
  }
  RVB_REQUIRE(T >= need, "%s: utterance %d is infeasible: %lld frames cannot hold %d labels (%lld frames needed)", who, b,
              T, U, need);
  return 0;
}

static int align_upload(AlignDev& d, const int* h_labels, const int* h_label_lens, const int* h_lens, cudaStream_t s) {
  // pageable sources: cudaMemcpyAsync stages them before it returns
  RVB_CHECK_CUDA(cudaMemcpyAsync(d.labels, h_labels, (size_t)d.B * d.max_U * sizeof(int), cudaMemcpyHostToDevice, s));
  RVB_CHECK_CUDA(cudaMemcpyAsync(d.ulens, h_label_lens, d.B * sizeof(int), cudaMemcpyHostToDevice, s));
  RVB_CHECK_CUDA(cudaMemcpyAsync(d.lens, h_lens, d.B * sizeof(int), cudaMemcpyHostToDevice, s));
  return 0;
}

// gather rows [r0, r0 + n) of every utterance's block from d_logp (whose row 0 is the block's row r0)
static int align_gather(AlignDev& d, const float* d_logp, int r0, int n, bool mask_by_len, cudaStream_t s) {
  if (n <= 0) return 0;
  // B == 1 (resumable form): the rows of this push land at row offset r0; B > 1 always gathers whole blocks (r0 == 0)
  align_gather_kernel<<<d.B == 1 ? n : d.B * d.rows, 256, 0, s>>>(d_logp, d.V, d.B == 1 ? n : d.rows, d.labels, d.max_U,
                                                                 d.ulens, mask_by_len ? d.lens : nullptr, d.blank,
                                                                 d.em + (size_t)r0 * d.g.E, d.g.E, d.g.P);
  RVB_COUNT_LAUNCH();
  RVB_CHECK_LAUNCH();
  return 0;
}

static int align_forward(AlignDev& d, int t0, int t1, cudaStream_t s) {
  const AlignGeom& g = d.g;
  if (g.K == AL_K_SMALL)
    ctc_viterbi_forward_kernel<AL_K_SMALL, AL_THREADS_SMALL><<<d.B, g.threads, 0, s>>>(
        d.em, g.E, g.P, d.bp, d.labels, d.max_U, d.ulens, d.lens, d.rows, d.alpha, t0, t1);
  else
    ctc_viterbi_forward_kernel<AL_K_LARGE, AL_THREADS_LARGE><<<d.B, g.threads, 0, s>>>(
        d.em, g.E, g.P, d.bp, d.labels, d.max_U, d.ulens, d.lens, d.rows, d.alpha, t0, t1);
  RVB_COUNT_LAUNCH();
  RVB_CHECK_LAUNCH();
  if (d.a64) {
    ctc_forward_loglik_kernel<<<d.B, 1024, 0, s>>>(d.em, g.E, g.P, d.labels, d.max_U, d.ulens, d.lens, d.rows, d.a64, t0,
                                                  t1, d.ll);
    RVB_COUNT_LAUNCH();
    RVB_CHECK_LAUNCH();
  }
  return 0;
}

// backtrace + reduction, results to the host; synchronises `s`
static int align_finish(AlignDev& d, int* h_frames, int* h_first, int* h_last, int* h_peak, float* h_peak_logp,
                        float* h_score, double* h_loglik, cudaStream_t s) {
  const size_t nf = (size_t)d.B * d.rows, nu = (size_t)d.B * d.max_U;
  int* state = d.out;
  int* frames = state + nf;
  int* first = frames + nf;
  int* last = first + nu;
  int* peak = last + nu;
  float* plp = reinterpret_cast<float*>(peak + nu);
  float* score = plp + nu;
  RVB_CHECK_CUDA(cudaMemsetAsync(first, 0, (4 * nu + d.B) * sizeof(int), s));
  ctc_viterbi_backtrace_kernel<<<d.B, 32, 0, s>>>(d.bp, d.g.P, d.alpha, d.ulens, d.lens, d.rows, state, score);
  RVB_COUNT_LAUNCH();
  RVB_CHECK_LAUNCH();
  align_reduce_kernel<<<dim3((d.rows + 255) / 256, d.B), 256, 0, s>>>(state, d.em, d.g.E, d.labels, d.max_U, d.lens, d.rows,
                                                                     d.blank, d.max_U, frames, first, last, peak, plp);
  RVB_COUNT_LAUNCH();
  RVB_CHECK_LAUNCH();
  RVB_CHECK_CUDA(cudaMemcpyAsync(h_frames, frames, nf * sizeof(int), cudaMemcpyDeviceToHost, s));
  RVB_CHECK_CUDA(cudaMemcpyAsync(h_first, first, nu * sizeof(int), cudaMemcpyDeviceToHost, s));
  RVB_CHECK_CUDA(cudaMemcpyAsync(h_last, last, nu * sizeof(int), cudaMemcpyDeviceToHost, s));
  RVB_CHECK_CUDA(cudaMemcpyAsync(h_peak, peak, nu * sizeof(int), cudaMemcpyDeviceToHost, s));
  RVB_CHECK_CUDA(cudaMemcpyAsync(h_peak_logp, plp, nu * sizeof(float), cudaMemcpyDeviceToHost, s));
  RVB_CHECK_CUDA(cudaMemcpyAsync(h_score, score, d.B * sizeof(float), cudaMemcpyDeviceToHost, s));
  if (h_loglik) RVB_CHECK_CUDA(cudaMemcpyAsync(h_loglik, d.ll, d.B * sizeof(double), cudaMemcpyDeviceToHost, s));
  RVB_CHECK_CUDA(cudaStreamSynchronize(s));
  return 0;
}

}  // namespace rvb

// ---------------------------------------------------------------------------------------------------------------
struct rvb_aligner {
  rvb::AlignDev d;
  int total = 0, pushed = 0;
  cudaStream_t side = nullptr;  // the model's search side stream, or null: work stays on the caller's stream
  cudaEvent_t ev = nullptr;
};

extern "C" {

RVB_API int rvb_ctc_force_align(const float* d_logp, int V, const int* h_enc_lens, int B, int Tp, const int* h_labels,
                                const int* h_label_lens, int max_U, int blank_id, int* h_frames, int* h_first,
                                int* h_last, int* h_peak, float* h_peak_logp, float* h_score, double* h_loglik,
                                void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  RVB_REQUIRE(d_logp && h_enc_lens && h_labels && h_label_lens && h_frames && h_first && h_last && h_peak &&
                  h_peak_logp && h_score && B > 0 && Tp > 0 && V > 0 && max_U > 0 && blank_id >= 0 && blank_id < V,
              "rvb_ctc_force_align: bad arguments");
  for (int b = 0; b < B; ++b) {
    RVB_REQUIRE(h_label_lens[b] <= max_U && h_enc_lens[b] <= Tp, "rvb_ctc_force_align: utterance %d exceeds max_U / Tp", b);
    if (rvb::align_check("rvb_ctc_force_align", b, h_labels + (size_t)b * max_U, h_label_lens[b], h_enc_lens[b], V, blank_id))
      return -2;
  }
  rvb::AlignDev d;
  int rc = rvb::align_alloc(d, B, Tp, max_U, V, blank_id, h_loglik != nullptr);
  if (rc == 0) rc = rvb::align_upload(d, h_labels, h_label_lens, h_enc_lens, stream);
  if (rc == 0) rc = rvb::align_gather(d, d_logp, 0, Tp, true, stream);
  if (rc == 0) rc = rvb::align_forward(d, 0, Tp, stream);
  if (rc == 0) rc = rvb::align_finish(d, h_frames, h_first, h_last, h_peak, h_peak_logp, h_score, h_loglik, stream);
  if (rc != 0) cudaStreamSynchronize(stream);
  rvb::align_free(d);
  return rc;
}

RVB_API long long rvb_aligner_workspace_bytes(int U, int total_frames, int want_loglik) {
  if (U < 1 || U > rvb::AL_MAX_LABELS || total_frames < 1) return -1;
  return (long long)rvb::align_bytes(rvb::align_geom(U), 1, total_frames, U, want_loglik != 0);
}

RVB_API void rvb_aligner_abort(rvb_aligner* a) {
  if (!a) return;
  if (a->side) cudaStreamSynchronize(a->side);
  if (a->ev) cudaEventDestroy(a->ev);
  rvb::align_free(a->d);
  delete a;
}

RVB_API rvb_aligner* rvb_aligner_begin(rvb_model* m, const int* h_labels, int U, int total_frames, int V, int blank_id,
                                       int want_loglik, long long budget_bytes, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  auto fail = [](rvb_aligner* a) -> rvb_aligner* {
    rvb_aligner_abort(a);
    return nullptr;
  };
  if (!(h_labels && V > 0 && blank_id >= 0 && blank_id < V && total_frames >= 0)) {
    rvb::set_error("rvb_aligner_begin: bad arguments");
    return nullptr;
  }
  if (rvb::align_check("rvb_aligner_begin", 0, h_labels, U, total_frames, V, blank_id)) return nullptr;
  const long long need = rvb_aligner_workspace_bytes(U, total_frames, want_loglik);
  if (budget_bytes > 0 && need > budget_bytes) {
    rvb::set_error("rvb_aligner_begin: %d frames x %d labels need %lld bytes of workspace, the budget is %lld", total_frames,
                   U, need, budget_bytes);
    return nullptr;
  }
  rvb_aligner* a = new rvb_aligner();
  a->total = total_frames;
  if (rvb::align_alloc(a->d, 1, total_frames, U, V, blank_id, want_loglik != 0)) return fail(a);
  if (rvb::align_upload(a->d, h_labels, &U, &total_frames, stream)) return fail(a);
  if (cudaStreamSynchronize(stream) != cudaSuccess) {  // &U / &total_frames are locals
    rvb::set_error("rvb_aligner_begin: upload failed");
    return fail(a);
  }
  if (m != nullptr) {
    if (rvb::search_side_stream(m, &a->side)) return fail(a);
    if (cudaEventCreateWithFlags(&a->ev, cudaEventDisableTiming) != cudaSuccess) {
      rvb::set_error("rvb_aligner_begin: cudaEventCreate failed");
      return fail(a);
    }
  }
  return a;
}

RVB_API int rvb_aligner_push(rvb_aligner* a, const float* d_logp, int n_rows, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  RVB_REQUIRE(a && d_logp && n_rows >= 0, "rvb_aligner_push: bad arguments");
  RVB_REQUIRE(a->pushed + (long long)n_rows <= a->total, "rvb_aligner_push: %d + %d rows exceed the %d frames announced",
              a->pushed, n_rows, a->total);
  if (n_rows == 0) return 0;
  // the gather reads the caller's rows on the caller's stream (they may be reused as soon as this returns, in stream
  // order); the serial trellis then runs on the side stream, under whatever the caller enqueues next
  if (rvb::align_gather(a->d, d_logp, a->pushed, n_rows, false, stream)) return -1;
  cudaStream_t ts = stream;
  if (a->side) {
    RVB_CHECK_CUDA(cudaEventRecord(a->ev, stream));
    RVB_CHECK_CUDA(cudaStreamWaitEvent(a->side, a->ev, 0));
    ts = a->side;
  }
  if (rvb::align_forward(a->d, a->pushed, a->pushed + n_rows, ts)) return -1;
  a->pushed += n_rows;
  return 0;
}

RVB_API int rvb_aligner_finish(rvb_aligner* a, int* h_frames, int* h_first, int* h_last, int* h_peak, float* h_peak_logp,
                               float* h_score, double* h_loglik, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  RVB_REQUIRE(a, "rvb_aligner_finish: null handle");
  int rc = 0;
  if (!(h_frames && h_first && h_last && h_peak && h_peak_logp && h_score)) {
    rvb::set_error("rvb_aligner_finish: bad arguments");
    rc = -2;
  } else if (a->pushed != a->total) {
    rvb::set_error("rvb_aligner_finish: %d of the %d frames announced were pushed", a->pushed, a->total);
    rc = -2;
  } else if (h_loglik != nullptr && a->d.a64 == nullptr) {
    rvb::set_error("rvb_aligner_finish: log-likelihood was not requested at begin");
    rc = -2;
  } else {
    rc = rvb::align_finish(a->d, h_frames, h_first, h_last, h_peak, h_peak_logp, h_score, h_loglik,
                           a->side ? a->side : stream);
  }
  rvb_aligner_abort(a);
  return rc;
}

}  // extern "C"
