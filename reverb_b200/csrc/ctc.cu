// reverb_b200 — CTC head post-processing and searches on the GPU.
//
//   logsoftmax_topk : per frame log_softmax over V (reference: transformer/ctc.py:106-114) fused with the top-N
//                     selection that both searches start from (transformer/search.py:111,155) — the (B,T',V) log-prob
//                     tensor (1.9 GB at B=64) is only written when the caller asks for it.
//   ctc_greedy      : arg-max path, padded frames -> blank, collapse repeats, drop blanks (search.py:106-121,
//                     utils/ctc_utils.py:22-32).
//   ctc_prefix_beam : CTC prefix beam search with the reference's exact update rules, float64 score arithmetic and
//                     Viterbi time tracking (search.py:124-248, utils/common.py:355-363) — one warp per utterance,
//                     prefixes as canonical trie nodes, times as persistent linked lists.  The biased instantiation
//                     adds the context-graph state of every prefix (the `context_graph` branches of the same lines).
//   logsoftmax_gather : rescoring decoder output -> log-probs of the hypothesis tokens only (search.py:413-436).
#include <math.h>

#include "kernels.h"

namespace rvb {

// ---------------------------------------------------------------------------------------------------------------
struct ArgMax {
  float v;
  int i;
};
__device__ __forceinline__ ArgMax better(ArgMax a, ArgMax b) {
  if (b.v > a.v || (b.v == a.v && b.i < a.i)) return b;
  return a;
}
__device__ __forceinline__ ArgMax warp_argmax(ArgMax a) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    ArgMax b;
    b.v = __shfl_xor_sync(0xffffffffu, a.v, o);
    b.i = __shfl_xor_sync(0xffffffffu, a.i, o);
    a = better(a, b);
  }
  return a;
}

// One CTA per row.  Pass 1 stages the row in shared memory and keeps each thread's running (max, index); the 32
// "lane-group" maxima (max over the threads with the same lane id, i.e. over the elements with index = lane mod 32)
// are DISTINCT elements (a lane group without elements contributes (-inf, INT_MAX), which ranks below every element),
// so the k-th best of them (k <= 16 < 32) is a lower bound of the row's k-th best: pass 2 (which also accumulates
// sum exp(x - max)) collects the few elements that are not worse than it — typically k .. k+4 — and one warp ranks
// those.  The kernel falls back to k rounds of block arg-max when that bound is -inf (fewer than k lane groups hold a
// finite element) or when more than TOPK_CAP elements pass it (a lane group full of ties or high values).
//
// Order contract, on both paths: the k reported entries are the first k of a stable sort of the row by value,
// descending — ties go to the lower index.  -inf entries are ordinary entries: a row with fewer than k finite entries
// reports its finite ones first, then its lowest-index -inf columns in index order, with value -inf.  NaN entries
// compare false and are never reported; if fewer than k entries are not NaN, the remaining slots get index 0.
constexpr int TOPK_CAP = 64;

__global__ void __launch_bounds__(256)
logsoftmax_topk_kernel(const float* __restrict__ logits, long long ld, int V, int k, float* __restrict__ topk_val,
                       int* __restrict__ topk_idx, float* __restrict__ logp_out, int apply_softmax) {
  extern __shared__ float s_row[];  // V floats
  __shared__ float s_red[8];
  __shared__ ArgMax s_arg[2][8];
  __shared__ ArgMax s_grp[8][32];
  __shared__ ArgMax s_cand[TOPK_CAP];
  __shared__ ArgMax s_thresh;
  __shared__ float s_stat[2];
  __shared__ int s_ncand;
  const long long row = blockIdx.x;
  const float* x = logits + row * ld;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  ArgMax mine;
  mine.v = -INFINITY;
  mine.i = 0x7fffffff;
  for (int i = threadIdx.x; i < V; i += 256) {
    ArgMax e;
    e.v = x[i];
    e.i = i;
    s_row[i] = e.v;
    mine = better(mine, e);
  }
  s_grp[warp][lane] = mine;
  float m = warp_max(mine.v);
  if (lane == 0) s_red[warp] = m;
  if (threadIdx.x == 0) {
    s_ncand = 0;
    s_thresh.v = -INFINITY;  // overwritten below by the k-th best lane-group maximum
    s_thresh.i = 0x7fffffff;
  }
  __syncthreads();
  if (warp == 0) {
    ArgMax g = s_grp[0][lane];
#pragma unroll
    for (int w = 1; w < 8; ++w) g = better(g, s_grp[w][lane]);
    int cnt = 0;  // how many lane-group maxima are strictly better than mine (a total order: indices are distinct)
    for (int o = 0; o < 32; ++o) {
      ArgMax h;
      h.v = __shfl_sync(0xffffffffu, g.v, o);
      h.i = __shfl_sync(0xffffffffu, g.i, o);
      cnt += (h.v > g.v || (h.v == g.v && h.i < g.i)) ? 1 : 0;
    }
    if (cnt == k - 1) s_thresh = g;
    if (lane == 0) {
      float mm = s_red[0];
      for (int w = 1; w < 8; ++w) mm = fmaxf(mm, s_red[w]);
      s_stat[0] = mm;
    }
  }
  __syncthreads();
  const ArgMax th = s_thresh;
  const bool filter_ok = th.i != 0x7fffffff && th.v > -INFINITY;
  m = s_stat[0];
  float ssum = 0.f;
  for (int i = threadIdx.x; i < V; i += 256) {
    const float v = s_row[i];
    if (apply_softmax) ssum += expf(v - m);
    if (filter_ok && (v > th.v || (v == th.v && i <= th.i))) {
      const int slot = atomicAdd(&s_ncand, 1);
      if (slot < TOPK_CAP) {
        s_cand[slot].v = v;
        s_cand[slot].i = i;
      }
    }
  }
  float lse_shift = 0.f, logsum = 0.f;
  if (apply_softmax) {
    ssum = warp_sum(ssum);
    if (lane == 0) s_red[warp] = ssum;
  }
  __syncthreads();
  if (apply_softmax) {
    float t = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) t += s_red[w];
    lse_shift = m;
    logsum = logf(t);
  }
  if (logp_out != nullptr) {
    for (int i = threadIdx.x; i < V; i += 256) logp_out[row * V + i] = (s_row[i] - lse_shift) - logsum;
  }
  const int nc = s_ncand;
  if (filter_ok && nc >= k && nc <= TOPK_CAP) {
    if (warp == 0) {
      for (int c = lane; c < nc; c += 32) {
        const ArgMax a = s_cand[c];
        int rank = 0;
        for (int o = 0; o < nc; ++o) {
          const ArgMax h = s_cand[o];
          rank += (h.v > a.v || (h.v == a.v && h.i < a.i)) ? 1 : 0;
        }
        if (rank < k) {
          topk_val[row * k + rank] = (a.v - lse_shift) - logsum;
          topk_idx[row * k + rank] = a.i;
        }
      }
    }
    return;
  }
  // fallback: k rounds of block arg-max over per-thread running maxima (ties -> lowest index); only the thread that
  // owned the winner rescans its ~V/256 elements, one barrier per round.  The rescan keeps the elements strictly after
  // the winner in (value desc, index asc) order: those are exactly the owner's elements not reported yet, so a
  // reported -inf is never picked again and further -inf entries follow in index order.
  auto local_best_after = [&](ArgMax prev) {
    ArgMax a;
    a.v = -INFINITY;
    a.i = 0x7fffffff;
    for (int i = threadIdx.x; i < V; i += 256) {
      ArgMax e;
      e.v = s_row[i];
      e.i = i;
      if (e.v < prev.v || (e.v == prev.v && e.i > prev.i)) a = better(a, e);
    }
    return a;
  };
  for (int r = 0; r < k; ++r) {
    ArgMax a = warp_argmax(mine);
    if (lane == 0) s_arg[r & 1][warp] = a;
    __syncthreads();
    ArgMax best = s_arg[r & 1][0];
#pragma unroll
    for (int w = 1; w < 8; ++w) best = better(best, s_arg[r & 1][w]);
    if (best.i == 0x7fffffff) {  // only NaN entries left (see the order contract above TOPK_CAP)
      if (threadIdx.x == 0) {
        topk_val[row * k + r] = (best.v - lse_shift) - logsum;
        topk_idx[row * k + r] = 0;
      }
    } else if ((best.i & 255) == (int)threadIdx.x) {
      topk_val[row * k + r] = (best.v - lse_shift) - logsum;
      topk_idx[row * k + r] = best.i;
      mine = local_best_after(best);
    }
  }
}

int launch_logsoftmax_topk(const float* logits, int ld, int M, int V, int k, float* topk_val, int* topk_idx,
                           float* logp_out, int apply_softmax, cudaStream_t stream) {
  RVB_REQUIRE(k >= 1 && k <= 16 && k <= V, "logsoftmax_topk: k=%d unsupported", k);
  if (M <= 0) return 0;
  const size_t smem = (size_t)V * sizeof(float);
  RVB_REQUIRE(smem <= 200 * 1024, "logsoftmax_topk: V=%d too large for the shared-memory row cache", V);
  static DynSmemOptIn optin;
  if (optin.ensure(logsoftmax_topk_kernel, smem)) return -1;
  logsoftmax_topk_kernel<<<M, 256, smem, stream>>>(logits, ld, V, k, topk_val, topk_idx, logp_out, apply_softmax);
  RVB_COUNT_LAUNCH();
  RVB_CHECK_LAUNCH();
  return 0;
}

// ---------------------------------------------------------------------------------------------------------------
__global__ void ctc_greedy_kernel(const int* __restrict__ top1, int stride, const int* __restrict__ lens, int T,
                                  int blank, int* __restrict__ out_tokens, int* __restrict__ out_lens) {
  const int b = blockIdx.x, lane = threadIdx.x;
  const int len = min(lens[b], T);
  int prev = -1, count = 0;
  for (int t0 = 0; t0 < T; t0 += 32) {
    int t = t0 + lane;
    int id = blank;
    if (t < len) id = top1[((long long)b * T + t) * stride];
    int left = __shfl_up_sync(0xffffffffu, id, 1);
    if (lane == 0) left = prev;
    bool keep = (t < T) && (id != blank) && (id != left);
    unsigned mask = __ballot_sync(0xffffffffu, keep);
    if (keep) out_tokens[(long long)b * T + count + __popc(mask & ((1u << lane) - 1u))] = id;
    count += __popc(mask);
    prev = __shfl_sync(0xffffffffu, id, 31);
  }
  if (lane == 0) out_lens[b] = count;
}

int launch_ctc_greedy(const int* top1_idx, int idx_stride, const int* lens, int B, int T, int blank, int* out_tokens,
                      int* out_lens, cudaStream_t stream) {
  if (B <= 0) return 0;
  ctc_greedy_kernel<<<B, 32, 0, stream>>>(top1_idx, idx_stride, lens, T, blank, out_tokens, out_lens);
  RVB_COUNT_LAUNCH();
  RVB_CHECK_LAUNCH();
  return 0;
}

// ---------------------------------------------------------------------------------------------------------------
// CTC prefix beam search.
constexpr int PB_MAXBEAM = 16;
constexpr int PB_MAXSLOTS = PB_MAXBEAM + PB_MAXBEAM * PB_MAXBEAM;
#define PB_NEG_INF (-INFINITY)

__device__ __forceinline__ double log_add2(double a, double b) {
  // utils/common.py:355-363 for two arguments: a_max + log(exp(a - a_max) + exp(b - a_max)).  One of the two
  // exponentials is exp(0) == 1 exactly and IEEE addition commutes, so a single exp() gives the same double.
  if (a == PB_NEG_INF) return b;
  if (b == PB_NEG_INF) return a;
  const double mx = a > b ? a : b;
  const double mn = a > b ? b : a;
  return mx + log(1.0 + exp(mn - mx));
}

struct PBLayout {
  size_t per_utt_ints;
  int pool_cap, hash_cap, times_cap;
};
__host__ __device__ inline PBLayout pb_layout(int T, int beam) {
  PBLayout l;
  l.pool_cap = beam * T + 2;
  int h = 64;
  while (h < 2 * l.pool_cap) h <<= 1;
  l.hash_cap = h;
  l.times_cap = 2 * beam * T + 2;
  l.per_utt_ints = (size_t)2 * l.pool_cap + l.hash_cap + (size_t)2 * l.times_cap;
  return l;
}
size_t prefix_beam_workspace_bytes(int B, int T, int beam) {
  PBLayout l = pb_layout(T, beam);
  return l.per_utt_ints * sizeof(int) * (size_t)B;
}

struct PBSlot {
  double s, ns, vs, vns, ctp;
  int times_s;           // times list node (-1 = empty list)
  int tns_src, tns_op;   // times_ns recipe: op 0 = none, 1 = append t to list tns_src, 2 = replace last of tns_src by t
  int src, tok;          // extension slots: source beam entry and token; stay slots: src = own index, tok = -1
};

constexpr int PB_THREADS = 128;
constexpr int PB_EXT_THREADS = PB_THREADS - 32;  // warps 0..2: extension candidates; last warp: stay slots
constexpr int PB_KEY_NONE = 0x7fffffff;

// Context biasing (biased instantiation only).  A prefix's context state and score depend on its token sequence alone
// (blank and repeat keep them, an extension takes one automaton step from its parent), so they travel with the beam
// entry and the reference's "first writer sets has_context" rule never has to be replayed.  These arrays live in dynamic
// shared memory in front of the trie, so the plain search's static layout is untouched.
struct PBCtx {
  double csc[2][PB_MAXBEAM];       // context score of every beam entry (both beam buffers)
  double slot_csc[PB_MAXSLOTS];    // context score of every slot of the frame
  double slot_tot[PB_MAXSLOTS];    // rank key of every slot: score() + context score (PrefixScore.total_score)
  int cst[2][PB_MAXBEAM];          // context state of every beam entry
  int slot_cst[PB_MAXSLOTS];
};
static_assert(sizeof(PBCtx) % 16 == 0, "the trie follows PBCtx in dynamic shared memory");

// One automaton step (utils/context_graph.py forward_one_step / fail walk; context_graph.py of this package): the
// child of `s` on `u` if there is one (token_score), else the fail walk from fail[s] that stops at the root, then the
// root's child if the walk ended there (bonus difference); plus the output bonus of the state reached.
__device__ __forceinline__ int ctx_child(const ContextGraphView& g, int s, int u) {
  if (s == 0) return u < g.vocab ? __ldg(g.root_next + u) : -1;
  int lo = __ldg(g.off + s);
  const int end = __ldg(g.off + s + 1);
  int hi = end;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (__ldg(g.tok + mid) < u) lo = mid + 1;
    else hi = mid;
  }
  return (lo < end && __ldg(g.tok + lo) == u) ? __ldg(g.dst + lo) : -1;
}
__device__ __forceinline__ double ctx_step(const ContextGraphView& g, int s, int u, int* next) {
  int n = ctx_child(g, s, u);
  double gained;
  if (n >= 0) {
    gained = __ldg(g.token_score + n);
  } else {
    int f = __ldg(g.fail + s);
    while ((n = ctx_child(g, f, u)) < 0) {
      f = __ldg(g.fail + f);
      if (f == 0) {
        n = ctx_child(g, 0, u);
        break;
      }
    }
    if (n < 0) n = f;
    gained = __ldg(g.bonus + n) - __ldg(g.bonus + s);
  }
  *next = n;
  return gained + __ldg(g.emit + n);
}

// The beam entering a frame: score()/viterbi_score()/times() of every prefix are derived when the entry is created.
struct PBBeam {
  double s[PB_MAXBEAM], ns[PB_MAXBEAM], vs[PB_MAXBEAM], vns[PB_MAXBEAM], score[PB_MAXBEAM], vit[PB_MAXBEAM];
  int node[PB_MAXBEAM], ts[PB_MAXBEAM], tns[PB_MAXBEAM], tnsp[PB_MAXBEAM], times[PB_MAXBEAM];
  int last[PB_MAXBEAM], par[PB_MAXBEAM];
};

// One CTA (4 warps) per utterance, two block barriers per frame:
//   P1  "stay" slots (prefix unchanged; last warp, a lane PAIR per prefix): at most three updates land on prefix j —
//       blank (lane 0 of the pair: s, v_s, times_s), repeat of its last token and the one extension
//       parent(j)+last(j) that equals j (lane 1: ns, v_ns, times_ns, replayed in the reference's iteration order);
//       extension slots (warps 0..2): one thread per (token, prefix) pair, final at once unless it collides with a
//       stay slot; every slot's score() is computed on the spot (extension slots have s = -inf: no transcendental)
//   P3  rank (score desc, dict insertion order asc; branch-free count), keep top `beam`, materialise survivors into
//       the OTHER beam buffer: canonical trie node (find-or-create in a shared-memory hash), times list nodes
// The next frame's top-k is prefetched into registers during P1.  Prefix identity = canonical trie node id, so the
// dict-merge semantics of the reference hold exactly.
// kBiased: context biasing with graph `cg` — P3 ranks by score() + context score, the recursion itself still uses
// score() / viterbi_score() alone, and the emitted score is score() - bonus[state] (finalize, search.py:226-233).
// The plain instantiation ignores `cg` and compiles to the code it had before biasing existed.
template <bool kBiased>
__global__ void __launch_bounds__(PB_THREADS)
ctc_prefix_beam_kernel(const float* __restrict__ topk_val, const int* __restrict__ topk_idx, int k,
                       const int* __restrict__ lens, int T, int beam, int blank, int* __restrict__ workspace,
                       int trie_in_smem, int max_len, int* __restrict__ out_tokens, int* __restrict__ out_times,
                       int* __restrict__ out_lens, double* __restrict__ out_scores, int* __restrict__ out_nhyp,
                       ContextGraphView cg) {
  extern __shared__ int pb_dyn[];
  const int b = blockIdx.x, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const PBLayout L = pb_layout(T, beam);
  int* ws = workspace + (size_t)b * L.per_utt_ints;
  PBCtx* cx = reinterpret_cast<PBCtx*>(pb_dyn);
  int* trie_parent = trie_in_smem ? (kBiased ? pb_dyn + sizeof(PBCtx) / sizeof(int) : pb_dyn) : ws;
  int* trie_tok = trie_parent + L.pool_cap;
  int* hash = trie_parent + 2 * L.pool_cap;  // -1 = empty
  int* times_parent = ws + 2 * L.pool_cap + L.hash_cap;
  int* times_t = times_parent + L.times_cap;

  __shared__ PBSlot slots[PB_MAXSLOTS];
  __shared__ double slot_score[PB_MAXSLOTS];
  __shared__ int slot_key[PB_MAXSLOTS];
  __shared__ PBBeam beams[2];
  __shared__ double s_tv[2][PB_MAXBEAM];
  __shared__ int s_ti[2][PB_MAXBEAM];
  __shared__ int s_pool, s_times, s_nlive[2];

  const int len = min(lens[b], T);
  const int kk = min(k, beam);
  if (trie_in_smem)
    for (int i = tid; i < L.hash_cap; i += PB_THREADS) hash[i] = -1;
  if (tid == 0) {
    trie_parent[0] = -1;
    trie_tok[0] = -1;
    s_pool = 1;
    s_times = 0;
    s_nlive[0] = s_nlive[1] = 0;
    PBBeam& C = beams[0];
    C.node[0] = 0;
    C.s[0] = 0.0;
    C.ns[0] = PB_NEG_INF;
    C.vs[0] = 0.0;
    C.vns[0] = 0.0;
    C.score[0] = 0.0;  // log_add([0, -inf])
    C.vit[0] = 0.0;    // v_s > v_ns is false -> v_ns
    C.ts[0] = -1;
    C.tns[0] = -1;
    C.tnsp[0] = -1;
    C.times[0] = -1;
    C.last[0] = -1;
    C.par[0] = -1;
    if constexpr (kBiased) {
      cx->cst[0][0] = 0;  // the root
      cx->csc[0][0] = 0.0;
    }
  }
  if (tid < kk && len > 0) {
    s_tv[0][tid] = (double)topk_val[((long long)b * T) * k + tid];
    s_ti[0][tid] = topk_idx[((long long)b * T) * k + tid];
  }
  int nb = 1;
  __syncthreads();

  for (int t = 0; t < len; ++t) {
    const int cur = t & 1;
    const PBBeam& C = beams[cur];
    PBBeam& N = beams[cur ^ 1];
    const double* tv = s_tv[cur];
    const int* ti = s_ti[cur];
    float pre_v = 0.f;
    int pre_i = 0;
    if (tid < kk && t + 1 < len) {
      pre_v = topk_val[((long long)b * T + t + 1) * k + tid];
      pre_i = topk_idx[((long long)b * T + t + 1) * k + tid];
    }
    const int ncand = kk * nb;
    const int nslots = nb + ncand;
    int mylive = 0;
    if (warp == PB_THREADS / 32 - 1) {
      // ---- P1a: stay slots, lane pair (2j, 2j+1) per prefix j
      const int j = lane >> 1, h = lane & 1;
      const bool act = j < nb;
      double s_new = PB_NEG_INF, vs_new = PB_NEG_INF;
      int times_s = -1, key = PB_KEY_NONE;
      double ns_new = PB_NEG_INF, vns_new = PB_NEG_INF, ctp = PB_NEG_INF;
      int tns_src = -1, tns_op = 0;
      if (act) {
        const int last_j = C.last[j];
        const bool nonempty = C.node[j] != 0;
        int ui_blank = -1, ui_last = -1, ip = -1;
        for (int u = 0; u < kk; ++u) {
          if (ti[u] == blank) ui_blank = u;
          if (nonempty && ti[u] == last_j) ui_last = u;
        }
        if (h == 0) {
          if (ui_blank >= 0) {  // blank: prefix unchanged, ends in blank
            const double p = tv[ui_blank];
            key = 2 * (ui_blank * nb + j);
            s_new = C.score[j] + p;  // log_add([-inf, x]) == x
            vs_new = C.vit[j] + p;
            times_s = C.times[j];
          }
        } else if (ui_last >= 0) {
          const int par_j = C.par[j];
          for (int i = 0; i < nb; ++i)
            if (C.node[i] == par_j) ip = i;
          const double p = tv[ui_last];
          // candidate order c = ui * nb + i: the repeat (i = j) comes before the collision (i = ip) iff j < ip
          const int nev = (ip >= 0) ? 2 : 1;
          for (int a = 0; a < nev; ++a) {
            const bool repeat_ev = (nev == 1) || ((a == 0) == (j < ip));
            if (repeat_ev) {
              if (key == PB_KEY_NONE) key = 2 * (ui_last * nb + j);
              ns_new = log_add2(ns_new, C.ns[j] + p);
              if (vns_new < C.vns[j] + p) {
                // reference typo (`vs_ns`, search.py:178): v_ns is NOT updated here
                if (ctp < p) {
                  ctp = p;
                  tns_src = C.tnsp[j];  // parent of prefix j's times_ns list: "copy, then overwrite the last element"
                  tns_op = 2;
                }
              }
            } else {
              if (key == PB_KEY_NONE) key = 2 * (ui_last * nb + ip) + 1;
              const bool rep = (last_j == C.last[ip]) && (C.node[ip] != 0);
              const double add = rep ? C.s[ip] : C.score[ip];
              const double vit = rep ? C.vs[ip] : C.vit[ip];
              ns_new = log_add2(ns_new, add + p);
              if (vns_new < vit + p) {
                vns_new = vit + p;
                ctp = p;
                tns_src = rep ? C.ts[ip] : C.times[ip];
                tns_op = 1;
              }
            }
          }
        }
      }
      // lane 1 of the pair gathers the blank half and finishes the slot
      const double s_other = __shfl_xor_sync(0xffffffffu, s_new, 1);
      const int key_other = __shfl_xor_sync(0xffffffffu, key, 1);
      if (act) {
        PBSlot& n = slots[j];
        if (h == 0) {
          n.s = s_new;
          n.vs = vs_new;
          n.times_s = times_s;
          n.src = j;
          n.tok = -1;
        } else {
          const int kmin = key < key_other ? key : key_other;
          n.ns = ns_new;
          n.vns = vns_new;
          n.ctp = ctp;
          n.tns_src = tns_src;
          n.tns_op = tns_op;
          slot_key[j] = kmin;
          slot_score[j] = (kmin == PB_KEY_NONE) ? PB_NEG_INF : log_add2(s_other, ns_new);
          mylive = (kmin != PB_KEY_NONE);
          if constexpr (kBiased) {  // the prefix is unchanged: so are its context state and score
            const double csc = cx->csc[cur][j];
            cx->slot_cst[j] = cx->cst[cur][j];
            cx->slot_csc[j] = csc;
            cx->slot_tot[j] = (kmin == PB_KEY_NONE) ? PB_NEG_INF : slot_score[j] + csc;
          }
        }
      }
    } else {
      // ---- P1b: extension slots, one thread per (token, prefix) candidate
      for (int c = tid; c < ncand; c += PB_EXT_THREADS) {
        const int ui = c / nb, i = c - ui * nb;
        const int u = ti[ui];
        const double p = tv[ui];
        int key = PB_KEY_NONE;
        double sc = PB_NEG_INF, tot = PB_NEG_INF;
        if (u != blank) {
          const int node_i = C.node[i];
          bool collide = false;
          for (int j = 0; j < nb; ++j) collide |= (C.par[j] == node_i && C.last[j] == u && C.node[j] != 0);
          if (!collide) {
            PBSlot& e = slots[nb + c];
            const bool rep = (u == C.last[i]) && (node_i != 0);
            // a single contribution into a fresh PrefixScore (s = ns = v_s = v_ns = -inf): log_add([-inf, x]) == x
            const double add = rep ? C.s[i] : C.score[i];
            const double vit = rep ? C.vs[i] : C.vit[i];
            e.s = PB_NEG_INF;
            e.ns = add + p;
            e.vs = PB_NEG_INF;
            e.vns = PB_NEG_INF;
            e.ctp = PB_NEG_INF;
            e.times_s = -1;
            e.tns_src = -1;
            e.tns_op = 0;
            if (PB_NEG_INF < vit + p) {
              e.vns = vit + p;
              e.ctp = p;
              e.tns_src = rep ? C.ts[i] : C.times[i];
              e.tns_op = 1;
            }
            e.src = i;
            e.tok = u;
            key = 2 * c + 1;
            sc = add + p;  // score() = log_add([-inf, ns]) = ns
            ++mylive;
            if constexpr (kBiased) {  // one automaton step from the parent's state
              int nst;
              const double step = ctx_step(cg, cx->cst[cur][i], u, &nst);
              const double csc = cx->csc[cur][i] + step;
              cx->slot_cst[nb + c] = nst;
              cx->slot_csc[nb + c] = csc;
              tot = sc + csc;
            }
          }
        }
        slot_key[nb + c] = key;
        slot_score[nb + c] = sc;
        if constexpr (kBiased) cx->slot_tot[nb + c] = tot;
      }
    }
    mylive = __reduce_add_sync(0xffffffffu, mylive);
    if (lane == 0 && mylive) atomicAdd(&s_nlive[cur], mylive);
    __syncthreads();
    // ---- P3: second beam prune (stable w.r.t. dict insertion order) + materialise the survivors into beams[cur^1]
    const int nnew = min(beam, s_nlive[cur]);
    if (tid == 0) s_nlive[cur ^ 1] = 0;
    if (tid < kk && t + 1 < len) {
      s_tv[cur ^ 1][tid] = (double)pre_v;
      s_ti[cur ^ 1][tid] = pre_i;
    }
    // rank key: score(), or score() + context score when biased
    const double* rank_key = slot_score;
    if constexpr (kBiased) rank_key = cx->slot_tot;
    for (int a = tid; a < nslots; a += PB_THREADS) {
      const int key = slot_key[a];
      if (key == PB_KEY_NONE) continue;
      const double sc = rank_key[a];
      // dead slots carry (score -inf, key INT_MAX): they never count, so the loop needs no liveness branch
      // four independent counters: the compare -> add chains overlap instead of serialising on one register
      int r0 = 0, r1 = 0, r2 = 0, r3 = 0;
      int o = 0;
      for (; o + 4 <= nslots; o += 4) {
        const double s0 = rank_key[o], s1 = rank_key[o + 1], s2 = rank_key[o + 2], s3 = rank_key[o + 3];
        const int k0 = slot_key[o], k1 = slot_key[o + 1], k2 = slot_key[o + 2], k3 = slot_key[o + 3];
        r0 += (int)((s0 > sc) | ((s0 == sc) & (k0 < key)));
        r1 += (int)((s1 > sc) | ((s1 == sc) & (k1 < key)));
        r2 += (int)((s2 > sc) | ((s2 == sc) & (k2 < key)));
        r3 += (int)((s3 > sc) | ((s3 == sc) & (k3 < key)));
      }
      for (; o < nslots; ++o) {
        const double so = rank_key[o];
        r0 += (int)((so > sc) | ((so == sc) & (slot_key[o] < key)));
      }
      const int rank = (r0 + r1) + (r2 + r3);
      if (rank >= nnew) continue;
      const PBSlot& s = slots[a];
      int node;
      if (s.tok < 0) {
        node = C.node[s.src];
      } else {
        const int parent = C.node[s.src];
        unsigned h = ((unsigned)parent * 2654435761u) ^ ((unsigned)s.tok * 40503u + 0x9e3779b9u);
        h &= (unsigned)(L.hash_cap - 1);
        node = -1;
        int fresh = -1;
        while (true) {
          int cur_n = atomicAdd(&hash[h], 0);
          if (cur_n == -1) {
            if (fresh < 0) {
              fresh = atomicAdd(&s_pool, 1);
              trie_parent[fresh] = parent;
              trie_tok[fresh] = s.tok;
              __threadfence_block();
            }
            int old = atomicCAS(&hash[h], -1, fresh);
            if (old == -1) {
              node = fresh;
              break;
            }
            cur_n = old;
          }
          if (trie_parent[cur_n] == parent && trie_tok[cur_n] == s.tok) {
            node = cur_n;
            break;
          }
          h = (h + 1) & (unsigned)(L.hash_cap - 1);
        }
      }
      int tns = -1, tnsp = -1;
      if (s.tns_op != 0) {
        tns = atomicAdd(&s_times, 1);
        tnsp = s.tns_src;      // op 1: append to list tns_src; op 2: tns_src already is the parent to hang t on
        times_parent[tns] = tnsp;
        times_t[tns] = t;
      }
      const bool sb = s.vs > s.vns;
      N.node[rank] = node;
      N.s[rank] = s.s;
      N.ns[rank] = s.ns;
      N.vs[rank] = s.vs;
      N.vns[rank] = s.vns;
      N.score[rank] = kBiased ? slot_score[a] : sc;
      N.vit[rank] = sb ? s.vs : s.vns;
      N.ts[rank] = s.times_s;
      N.tns[rank] = tns;
      N.tnsp[rank] = tnsp;
      N.times[rank] = sb ? s.times_s : tns;
      N.last[rank] = (s.tok < 0) ? C.last[s.src] : s.tok;
      N.par[rank] = (s.tok < 0) ? C.par[s.src] : C.node[s.src];
      if constexpr (kBiased) {
        cx->cst[cur ^ 1][rank] = cx->slot_cst[a];
        cx->csc[cur ^ 1][rank] = cx->slot_csc[a];
      }
    }
    nb = nnew;
    __syncthreads();
  }

  // ---- emit the n-best: tokens, score() and times() per surviving prefix, in beam order
  const PBBeam& F = beams[len & 1];
  if (tid == 0) out_nhyp[b] = nb;
  if (tid < nb) {
    const int r = tid;
    int n = 0;
    for (int node = F.node[r]; node > 0; node = trie_parent[node]) ++n;
    int* tok_out = out_tokens + ((long long)b * beam + r) * max_len;
    int* tim_out = out_times + ((long long)b * beam + r) * max_len;
    int pos = n;
    for (int node = F.node[r]; node > 0; node = trie_parent[node]) {
      --pos;
      if (pos < max_len) tok_out[pos] = trie_tok[node];
    }
    const int tl = F.times[r];
    int nt = 0;
    for (int q = tl; q >= 0; q = times_parent[q]) ++nt;
    pos = nt;
    for (int q = tl; q >= 0; q = times_parent[q]) {
      --pos;
      if (pos < max_len) tim_out[pos] = times_t[q];
    }
    out_lens[(b * beam + r) * 2 + 0] = n;
    out_lens[(b * beam + r) * 2 + 1] = nt;
    if constexpr (kBiased) {
      // finalize: the context score becomes -bonus[state] (an unfinished match is taken back); no re-sort
      out_scores[b * beam + r] = F.score[r] + (-__ldg(cg.bonus + cx->cst[len & 1][r]));
    } else {
      out_scores[b * beam + r] = F.score[r];
    }
  }
}

template <bool kBiased>
static int launch_prefix_beam(const float* topk_val, const int* topk_idx, int k, const int* lens, int B, int T, int beam,
                              int blank, void* workspace, size_t workspace_bytes, int max_len, int* out_tokens,
                              int* out_times, int* out_lens, double* out_scores, int* out_nhyp,
                              const ContextGraphView& cg, cudaStream_t stream) {
  RVB_REQUIRE(beam >= 1 && beam <= PB_MAXBEAM, "prefix beam: beam_size=%d unsupported (1..%d)", beam, PB_MAXBEAM);
  RVB_REQUIRE(k >= beam, "prefix beam: need top-k with k >= beam (k=%d beam=%d)", k, beam);
  const size_t need = prefix_beam_workspace_bytes(B, T, beam);
  RVB_REQUIRE(workspace_bytes >= need, "prefix beam: workspace too small (%zu < %zu)", workspace_bytes, need);
  if (B <= 0) return 0;
  const PBLayout L = pb_layout(T, beam);
  const size_t trie_bytes = ((size_t)2 * L.pool_cap + L.hash_cap) * sizeof(int);
  const int trie_in_smem = trie_bytes <= 150 * 1024;
  if (!trie_in_smem) RVB_CHECK_CUDA(cudaMemsetAsync(workspace, 0xFF, need, stream));  // hash tables = -1
  const size_t dyn = (trie_in_smem ? trie_bytes : 0) + (kBiased ? sizeof(PBCtx) : 0);
  static DynSmemOptIn optin;
  if (optin.ensure(ctc_prefix_beam_kernel<kBiased>, dyn)) return -1;
  ctc_prefix_beam_kernel<kBiased><<<B, PB_THREADS, dyn, stream>>>(topk_val, topk_idx, k, lens, T, beam, blank,
                                                                 reinterpret_cast<int*>(workspace), trie_in_smem,
                                                                 max_len, out_tokens, out_times, out_lens, out_scores,
                                                                 out_nhyp, cg);
  RVB_COUNT_LAUNCH();
  RVB_CHECK_LAUNCH();
  return 0;
}

int launch_ctc_prefix_beam(const float* topk_val, const int* topk_idx, int k, const int* lens, int B, int T, int beam,
                           int blank, void* workspace, size_t workspace_bytes, int max_len, int* out_tokens,
                           int* out_times, int* out_lens, double* out_scores, int* out_nhyp, cudaStream_t stream) {
  return launch_prefix_beam<false>(topk_val, topk_idx, k, lens, B, T, beam, blank, workspace, workspace_bytes, max_len,
                                   out_tokens, out_times, out_lens, out_scores, out_nhyp, ContextGraphView{}, stream);
}

int launch_ctc_prefix_beam_biased(const float* topk_val, const int* topk_idx, int k, const int* lens, int B, int T,
                                  int beam, int blank, void* workspace, size_t workspace_bytes, int max_len,
                                  int* out_tokens, int* out_times, int* out_lens, double* out_scores, int* out_nhyp,
                                  const ContextGraphView& graph, cudaStream_t stream) {
  RVB_REQUIRE(graph.off && graph.root_next && graph.bonus, "prefix beam: context graph not uploaded");
  return launch_prefix_beam<true>(topk_val, topk_idx, k, lens, B, T, beam, blank, workspace, workspace_bytes, max_len,
                                  out_tokens, out_times, out_lens, out_scores, out_nhyp, graph, stream);
}

// ---------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
logsoftmax_gather_kernel(const float* __restrict__ logits, long long ld, int V, const int* __restrict__ gidx, int G,
                         float* __restrict__ out) {
  __shared__ float s_red[8];
  __shared__ float s_stat[2];
  const long long row = blockIdx.x;
  const float* x = logits + row * ld;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float m = -INFINITY;
  for (int i = threadIdx.x; i < V; i += 256) m = fmaxf(m, x[i]);
  m = warp_max(m);
  if (lane == 0) s_red[warp] = m;
  __syncthreads();
  m = s_red[0];
  for (int w = 1; w < 8; ++w) m = fmaxf(m, s_red[w]);
  __syncthreads();
  float s = 0.f;
  for (int i = threadIdx.x; i < V; i += 256) s += expf(x[i] - m);
  s = warp_sum(s);
  if (lane == 0) s_red[warp] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
    for (int w = 0; w < 8; ++w) t += s_red[w];
    s_stat[0] = m;
    s_stat[1] = logf(t);
  }
  __syncthreads();
  for (int j = threadIdx.x; j < G; j += 256) {
    int id = gidx[row * G + j];
    out[row * G + j] = (id >= 0 && id < V) ? (x[id] - s_stat[0]) - s_stat[1] : 0.f;
  }
}

int launch_logsoftmax_gather(const float* logits, int ld, int M, int V, const int* gather_idx, int G, float* out,
                             cudaStream_t stream) {
  if (M <= 0) return 0;
  logsoftmax_gather_kernel<<<M, 256, 0, stream>>>(logits, ld, V, gather_idx, G, out);
  RVB_COUNT_LAUNCH();
  RVB_CHECK_LAUNCH();
  return 0;
}

// ---------------------------------------------------------------------------------------------------------------
// Decoder inputs of attention rescoring, built on the device from the n-best the prefix beam search left there:
// hypothesis s = (b, i) has U tokens w (0 when i >= nhyp[b]);  sos / eos from the model config (asr_model.py:79-82)
//   tok_l = [sos, w_1..w_U, eos..]                 tok_r = [sos, w_U..w_1, eos..]          (asr_model.py:921-949)
//   gat_l = [w_1..w_U, eos, -1..]                  gat_r = [w_U..w_1, eos, -1..]           (search.py:417-430)
__global__ void rescoring_inputs_kernel(const int* __restrict__ tok, int tok_stride, const int* __restrict__ olen,
                                        const int* __restrict__ nhyp, int N, int Lp, int sos, int eos,
                                        int* __restrict__ tok_l, int* __restrict__ tok_r, int* __restrict__ gat_l,
                                        int* __restrict__ gat_r, int* __restrict__ slen) {
  const int s = blockIdx.x, b = s / N, i = s - b * N;
  int U = (i < nhyp[b]) ? olen[2 * s] : 0;
  U = min(U, Lp - 1);
  const int* wv = tok + (size_t)s * tok_stride;
  for (int j = threadIdx.x; j < Lp; j += blockDim.x) {
    const size_t r = (size_t)s * Lp + j;
    tok_l[r] = (j == 0) ? sos : (j <= U ? wv[j - 1] : eos);
    tok_r[r] = (j == 0) ? sos : (j <= U ? wv[U - j] : eos);
    gat_l[r] = (j < U) ? wv[j] : (j == U ? eos : -1);
    gat_r[r] = (j < U) ? wv[U - 1 - j] : (j == U ? eos : -1);
  }
  if (threadIdx.x == 0) slen[s] = U + 1;
}

int launch_rescoring_inputs(const int* d_tokens, int tok_stride, const int* d_out_lens, const int* d_nhyp, int B, int N,
                            int Lp, int sos, int eos, int* tok_l, int* tok_r, int* gat_l, int* gat_r, int* slen,
                            cudaStream_t stream) {
  if (B * N <= 0) return 0;
  rescoring_inputs_kernel<<<B * N, 128, 0, stream>>>(d_tokens, tok_stride, d_out_lens, d_nhyp, N, Lp, sos, eos, tok_l,
                                                     tok_r, gat_l, gat_r, slen);
  RVB_COUNT_LAUNCH();
  RVB_CHECK_LAUNCH();
  return 0;
}

// ---------------------------------------------------------------------------------------------------------------
// Second half of the fused log_softmax + gather (GEMM epilogue OUT_LSE, gemm.cu): combine the per-slab partials
// (max, sum exp(x - max)) of a row into logsumexp and subtract it from the gathered logit.  One warp per row.
__global__ void __launch_bounds__(256)
lse_merge_kernel(const float2* __restrict__ part, int slabs, const float* __restrict__ tgt, const int* __restrict__ gather,
                 int M, float* __restrict__ out) {
  const int row = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (row >= M) return;
  const float2* pr = part + (size_t)row * slabs;
  float m = -INFINITY;
  for (int i = lane; i < slabs; i += 32) m = fmaxf(m, pr[i].x);
  m = warp_max(m);
  float s = 0.f;
  for (int i = lane; i < slabs; i += 32) {
    const float2 v = pr[i];
    s += (v.x == -INFINITY) ? 0.f : v.y * expf(v.x - m);
  }
  s = warp_sum(s);
  if (lane == 0) out[row] = (gather[row] >= 0) ? tgt[row] - (m + logf(s)) : 0.f;
}

int launch_lse_merge(const float2* part, int slabs, const float* tgt, const int* gather, int M, float* out,
                     cudaStream_t stream) {
  if (M <= 0) return 0;
  lse_merge_kernel<<<(M * 32 + 255) / 256, 256, 0, stream>>>(part, slabs, tgt, gather, M, out);
  RVB_COUNT_LAUNCH();
  RVB_CHECK_LAUNCH();
  return 0;
}

// ---------------------------------------------------------------------------------------------------------------
// Prefix-TREE attention rescoring.  The reference decodes each of the N hypotheses of an utterance on its own
// (search.py:382-411, asr_model.py:895 repeats the memory N times), although the n-best of a prefix beam search share
// most of their prefixes and a causal decoder gives identical outputs for identical prefixes.  Here the decoder runs
// once per DISTINCT prefix ("node" of the utterance's prefix tree): rows = nodes (~6x fewer than hypotheses x positions
// on real n-best lists), self-attention over the node's ancestors, and every (hypothesis, position) score is read from
// the edge it walks.  Same arithmetic per row as the flat path, so the scores agree to rounding.
//
// trie_build_kernel — one CTA per utterance.  Hypotheses are inserted in n-best order; hypothesis i shares the nodes of
// the earlier hypothesis with the longest common prefix and appends new nodes for the rest.
//   node 0 = the empty prefix (decoder input <sos>, depth 0); a node at depth j carries token w_j.
//   node_of[(b*N + i) * nstride + j] = node of the first j tokens of hypothesis i (j = 0 .. U_i).
// reverse != 0: the hypotheses are read back to front (right-to-left decoder, asr_model.py:921-949).
__global__ void __launch_bounds__(128)
trie_build_kernel(const int* __restrict__ tok, int tok_stride, const int* __restrict__ olen,
                  const int* __restrict__ nhyp, int N, int reverse, int sos, int* __restrict__ node_of, int nstride,
                  int* __restrict__ node_tok, int* __restrict__ node_par, int* __restrict__ node_dep, int cap,
                  int* __restrict__ n_nodes) {
  __shared__ int s_lcp[16];
  __shared__ int s_next, s_best, s_bestlen;
  const int b = blockIdx.x, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int n = min(nhyp[b], N);
  int* ntok = node_tok + (size_t)b * cap;
  int* npar = node_par + (size_t)b * cap;
  int* ndep = node_dep + (size_t)b * cap;
  if (tid == 0) {
    ntok[0] = sos;
    npar[0] = -1;
    ndep[0] = 0;
    s_next = 1;
  }
  __syncthreads();
  auto len_of = [&](int i) { return i < n ? olen[2 * ((size_t)b * N + i)] : 0; };
  auto tok_of = [&](int i, int U, int j) {  // j-th token (0-based) of hypothesis i in decoding order
    const int* w = tok + ((size_t)b * N + i) * tok_stride;
    return reverse ? w[U - 1 - j] : w[j];
  };
  for (int i = 0; i < N; ++i) {
    const int U = len_of(i);
    int* mine = node_of + ((size_t)b * N + i) * nstride;
    // longest common prefix with every earlier hypothesis (one warp per earlier hypothesis)
    for (int ip = warp; ip < i; ip += 4) {
      const int Up = len_of(ip), lim = min(U, Up);
      int first = lim;
      for (int j = lane; j < lim; j += 32)
        if (tok_of(i, U, j) != tok_of(ip, Up, j)) {
          first = j;
          break;
        }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) first = min(first, __shfl_xor_sync(0xffffffffu, first, o));
      if (lane == 0) s_lcp[ip] = first;
    }
    __syncthreads();
    if (tid == 0) {
      int best = -1, bl = 0;
      for (int ip = 0; ip < i; ++ip)
        if (s_lcp[ip] > bl) {
          bl = s_lcp[ip];
          best = ip;
        }
      s_best = best;
      s_bestlen = bl;
    }
    __syncthreads();
    const int L = s_bestlen, base = s_next;
    const int* theirs = node_of + ((size_t)b * N + (s_best < 0 ? 0 : s_best)) * nstride;
    for (int j = tid; j <= U; j += blockDim.x) {
      if (j == 0) mine[0] = 0;
      else if (j <= L) mine[j] = theirs[j];
      else {
        const int id = base + (j - L - 1);
        mine[j] = id;
        ntok[id] = tok_of(i, U, j - 1);
        ndep[id] = j;
        npar[id] = (j == L + 1) ? (L == 0 ? 0 : theirs[L]) : id - 1;
      }
    }
    __syncthreads();
    if (tid == 0) s_next = base + (U - L);
    __syncthreads();
  }
  if (tid == 0) n_nodes[b] = s_next;
}

int launch_trie_build(const int* tok, int tok_stride, const int* olen, const int* nhyp, int B, int N, int reverse, int sos,
                      int* node_of, int nstride, int* node_tok, int* node_par, int* node_dep, int cap, int* n_nodes,
                      cudaStream_t stream) {
  RVB_REQUIRE(N >= 1 && N <= 16, "trie_build: beam %d unsupported", N);
  if (B <= 0) return 0;
  trie_build_kernel<<<B, 128, 0, stream>>>(tok, tok_stride, olen, nhyp, N, reverse, sos, node_of, nstride, node_tok,
                                           node_par, node_dep, cap, n_nodes);
  RVB_COUNT_LAUNCH();
  RVB_CHECK_LAUNCH();
  return 0;
}

// trie_inputs_kernel — one CTA per utterance, once the host knows P (node slots per utterance) and Lp:
//   rows r = b*P + node:   tok_in[r], pos[r] (depth), anc[r*Lp + t] = row of the ancestor at depth t (t <= depth),
//                          alen[r] = depth + 1;  unused slots: <eos> at position 0 attending only themselves
//   score rows e = b*(P+N) + slot:  slot < P: the edge INTO node `slot` (src = its parent's row, target = its token),
//                          slot P + i: hypothesis i ends (src = its last node, target = <eos>);  -1 target = unused
//   smap[(b*N + i)*Lp + j] = score row of position j of hypothesis i (j <= U_i), else -1
__global__ void __launch_bounds__(256)
trie_inputs_kernel(const int* __restrict__ node_of, int nstride, const int* __restrict__ node_tok,
                   const int* __restrict__ node_par, const int* __restrict__ node_dep, int cap,
                   const int* __restrict__ n_nodes, const int* __restrict__ olen, const int* __restrict__ nhyp, int N,
                   int P, int Lp, int eos, int* __restrict__ tok_in, int* __restrict__ pos, int* __restrict__ anc,
                   int* __restrict__ alen, int* __restrict__ src, int* __restrict__ tgt, int* __restrict__ smap,
                   uint32_t* __restrict__ anc_bits, int bits_ld) {
  const int b = blockIdx.x;
  const int nn = n_nodes[b], n = min(nhyp[b], N);
  const int* ntok = node_tok + (size_t)b * cap;
  const int* npar = node_par + (size_t)b * cap;
  const int* ndep = node_dep + (size_t)b * cap;
  for (int node = threadIdx.x; node < P; node += blockDim.x) {
    const size_t r = (size_t)b * P + node;
    if (anc_bits) {  // the same ancestor set as a bit row over the utterance's node slots (wgmma attention mask)
      uint32_t* br = anc_bits + r * bits_ld;
      for (int w = 0; w < bits_ld; ++w) br[w] = 0u;
      int cur = node;
      if (node < nn)
        for (int t = ndep[node]; t >= 0; --t) {
          br[cur >> 5] |= 1u << (cur & 31);
          cur = npar[cur];
        }
      else
        br[node >> 5] = 1u << (node & 31);
    }
    if (node < nn) {
      const int dep = ndep[node];
      tok_in[r] = ntok[node];
      pos[r] = dep;
      alen[r] = dep + 1;
      int cur = node;
      for (int t = dep; t >= 0; --t) {
        anc[r * Lp + t] = b * P + cur;
        cur = npar[cur];
      }
    } else {
      tok_in[r] = eos;
      pos[r] = 0;
      alen[r] = 1;
      anc[r * Lp] = (int)r;
    }
  }
  for (int e = threadIdx.x; e < P + N; e += blockDim.x) {
    const size_t sr = (size_t)b * (P + N) + e;
    int s_ = b * P, t_ = -1;
    if (e >= 1 && e < nn) {
      s_ = b * P + npar[e];
      t_ = ntok[e];
    } else if (e >= P) {
      const int i = e - P;
      const int U = i < n ? olen[2 * ((size_t)b * N + i)] : 0;
      s_ = b * P + node_of[((size_t)b * N + i) * nstride + U];
      t_ = eos;
    }
    src[sr] = s_;
    tgt[sr] = t_;
  }
  for (int q = threadIdx.x; q < N * Lp; q += blockDim.x) {
    const int i = q / Lp, j = q - i * Lp;
    const int U = i < n ? olen[2 * ((size_t)b * N + i)] : 0;
    int mrow = -1;
    if (j < U) mrow = b * (P + N) + node_of[((size_t)b * N + i) * nstride + j + 1];
    else if (j == U) mrow = b * (P + N) + P + i;
    smap[((size_t)b * N + i) * Lp + j] = mrow;
  }
}

int launch_trie_inputs(const int* node_of, int nstride, const int* node_tok, const int* node_par, const int* node_dep,
                       int cap, const int* n_nodes, const int* olen, const int* nhyp, int B, int N, int P, int Lp, int eos,
                       int* tok_in, int* pos, int* anc, int* alen, int* src, int* tgt, int* smap, cudaStream_t stream,
                       uint32_t* anc_bits, int bits_ld) {
  if (B <= 0) return 0;
  RVB_REQUIRE(anc_bits == nullptr || bits_ld * 32 >= P, "trie_inputs: %d mask words cannot hold %d node slots", bits_ld, P);
  trie_inputs_kernel<<<B, 256, 0, stream>>>(node_of, nstride, node_tok, node_par, node_dep, cap, n_nodes, olen, nhyp, N,
                                            P, Lp, eos, tok_in, pos, anc, alen, src, tgt, smap, anc_bits, bits_ld);
  RVB_COUNT_LAUNCH();
  RVB_CHECK_LAUNCH();
  return 0;
}

// out[r, :] = in[idx[r], :]  (rows of `width` bf16, 16-byte aligned)
__global__ void gather_rows_kernel(const bf16* __restrict__ in, const int* __restrict__ idx, bf16* __restrict__ out,
                                   int width) {
  const uint4* a = reinterpret_cast<const uint4*>(in + (size_t)idx[blockIdx.x] * width);
  uint4* o = reinterpret_cast<uint4*>(out + (size_t)blockIdx.x * width);
  for (int i = threadIdx.x; i < width / 8; i += blockDim.x) o[i] = a[i];
}
int launch_gather_rows(const bf16* in, const int* idx, bf16* out, int rows, int width, cudaStream_t stream) {
  RVB_REQUIRE(width % 8 == 0, "gather_rows: width %% 8 != 0");
  if (rows <= 0) return 0;
  gather_rows_kernel<<<rows, 128, 0, stream>>>(in, idx, out, width);
  RVB_COUNT_LAUNCH();
  RVB_CHECK_LAUNCH();
  return 0;
}

// out[i] = map[i] >= 0 ? vals[map[i]] : 0
__global__ void gather_scores_kernel(const float* __restrict__ vals, const int* __restrict__ map, float* __restrict__ out,
                                     long long n) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = map[i] >= 0 ? vals[map[i]] : 0.f;
}
int launch_gather_scores(const float* vals, const int* map, float* out, long long n, cudaStream_t stream) {
  if (n <= 0) return 0;
  gather_scores_kernel<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(vals, map, out, n);
  RVB_COUNT_LAUNCH();
  RVB_CHECK_LAUNCH();
  return 0;
}

}  // namespace rvb
