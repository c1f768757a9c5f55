// reverb_b200 — centroid-linkage agglomerative clustering of speaker embeddings on sm_90a.
//
// Replaces `scipy.cluster.hierarchy.linkage(emb, method="centroid", metric="euclidean")` inside pyannote's
// `AgglomerativeClustering.cluster` (diarization/pipeline.py).  The result is scipy's Z bit for bit whenever no two
// candidate merge heights tie (oracle/linkage_ref.py restates the algorithm in numpy and pins it against scipy):
//
//   1. distances   d(i,j) = sqrt(sum_k (x_ik - x_jk)^2), summed over k in index order with no FMA (= scipy's pdist)
//   2. merges      n - 1 times: the globally closest active pair (a, b), a < b; the merged cluster keeps slot b,
//                  slot a is retired.  Ties: smallest height, then smallest (a, b)
//   3. update      d(k,b) <- sqrt(((sa*d_ak*d_ak) + (sb*d_bk*d_bk) - (sa*sb*d*d)/s) / s), s = sa + sb, in exactly
//                  this operation order (Lance-Williams for centroids on Euclidean distances)
//   4. output      rows in merge order, not sorted (centroid linkage has inversions; scipy keeps them)
//   5. labels      row r joins the clusters holding slots a and b (smaller id first) into cluster n + r; column 3 is
//                  the size.  Slot s always holds the cluster that contains point s, so a per-slot label is the
//                  union-find root without any find.
//
// Kernels: a 64 x 64 tiled distance kernel writes the condensed matrix into the caller's workspace (the memory scipy
// needs on the host); a row kernel fills each row's nearest-neighbour cache; then ONE persistent launch of a cluster of
// kLinkCta CTAs runs every merge, two cluster barriers per merge and no host round trip.  Each CTA owns a contiguous
// range of rows and keeps their (nearest value, index) cache exact: after a merge it rescans only the rows whose
// neighbour was a or b, plus row b, and lowers the cache of any row whose new d(k,b) is smaller.
//
// Every arithmetic step of the distances and the update is an explicit round-to-nearest intrinsic, so nvcc cannot
// contract any of them into an FMA.  Data that other threads write between barriers is read with ld.global.cg (L2).
#include <cooperative_groups.h>
#include <limits.h>
#include <math.h>

#include "../../include/rvb_diar.h"
#include "common.cuh"

namespace cg = cooperative_groups;

namespace rvb {
namespace {

constexpr int kPdTile = 64;      // distance tile: 64 x 64 pairs per 256-thread block, 4 x 4 per thread
constexpr int kPdK = 16;         // embedding dimensions staged in shared memory per step
constexpr int kLinkCta = 8;      // CTAs of the merge cluster (the portable cluster size)
constexpr int kLinkThreads = 1024;

// condensed index of the pair i < j (scipy's pdist order)
__device__ __forceinline__ long long cidx(long long i, long long j, long long n) {
  return i * n - i * (i + 1) / 2 + (j - i - 1);
}
__device__ __forceinline__ double pair_dist(const double* D, int i, int j, int n) {
  return __ldcg(D + (i < j ? cidx(i, j, n) : cidx(j, i, n)));
}

// NaN (a negative centroid distance under rounding) ranks with +inf, so a valid pair is always found
__device__ __forceinline__ double rank_key(double v) { return isnan(v) ? INFINITY : v; }
// (value, index): smaller value, then smaller index
__device__ __forceinline__ bool before(double v1, int j1, double v2, int j2) {
  const double k1 = rank_key(v1), k2 = rank_key(v2);
  return k1 < k2 || (k1 == k2 && j1 < j2);
}
// (height, a, b): smaller height, then smaller (a, b)
__device__ __forceinline__ bool pair_before(double v1, int a1, int b1, double v2, int a2, int b2) {
  const double k1 = rank_key(v1), k2 = rank_key(v2);
  return k1 < k2 || (k1 == k2 && (a1 < a2 || (a1 == a2 && b1 < b2)));
}

__device__ __forceinline__ void warp_argmin(double& v, int& j) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const double ov = __shfl_xor_sync(0xffffffffu, v, o);
    const int oj = __shfl_xor_sync(0xffffffffu, j, o);
    if (before(ov, oj, v, j)) {
      v = ov;
      j = oj;
    }
  }
}
__device__ __forceinline__ void warp_pairmin(double& v, int& a, int& b) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const double ov = __shfl_xor_sync(0xffffffffu, v, o);
    const int oa = __shfl_xor_sync(0xffffffffu, a, o), ob = __shfl_xor_sync(0xffffffffu, b, o);
    if (pair_before(ov, oa, ob, v, a, b)) {
      v = ov;
      a = oa;
      b = ob;
    }
  }
}
// every thread of the block returns the block's minimum; sv / sj hold one entry per warp
__device__ __forceinline__ void block_argmin(double& v, int& j, double* sv, int* sj) {
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31, nw = blockDim.x >> 5;
  warp_argmin(v, j);
  __syncthreads();
  if (l == 0) {
    sv[w] = v;
    sj[w] = j;
  }
  __syncthreads();
  v = l < nw ? sv[l] : INFINITY;
  j = l < nw ? sj[l] : INT_MAX;
  warp_argmin(v, j);
}

}  // namespace

__global__ void __launch_bounds__(256) pdist_kernel(const double* __restrict__ x, int n, int dim, double* __restrict__ D) {
  const int bi = blockIdx.y, bj = blockIdx.x;
  if (bj < bi) return;                                    // upper triangle of tiles only
  __shared__ double xi[kPdTile][kPdK + 1], xj[kPdTile][kPdK + 1];
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  double acc[4][4];
#pragma unroll
  for (int r = 0; r < 4; ++r)
#pragma unroll
    for (int c = 0; c < 4; ++c) acc[r][c] = 0.0;
  for (int k0 = 0; k0 < dim; k0 += kPdK) {
    for (int e = threadIdx.x; e < kPdTile * kPdK; e += 256) {
      const int r = e / kPdK, c = e % kPdK, k = k0 + c;
      const int gi = bi * kPdTile + r, gj = bj * kPdTile + r;
      // padding is zero in both operands: (0 - 0)^2 adds nothing
      xi[r][c] = (gi < n && k < dim) ? x[(long long)gi * dim + k] : 0.0;
      xj[r][c] = (gj < n && k < dim) ? x[(long long)gj * dim + k] : 0.0;
    }
    __syncthreads();
#pragma unroll
    for (int c = 0; c < kPdK; ++c) {
      double a[4], b[4];
#pragma unroll
      for (int r = 0; r < 4; ++r) {
        a[r] = xi[ty + 16 * r][c];
        b[r] = xj[tx + 16 * r][c];
      }
#pragma unroll
      for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int s = 0; s < 4; ++s) {
          const double t = __dsub_rn(a[r], b[s]);
          acc[r][s] = __dadd_rn(acc[r][s], __dmul_rn(t, t));
        }
    }
    __syncthreads();
  }
#pragma unroll
  for (int r = 0; r < 4; ++r)
#pragma unroll
    for (int s = 0; s < 4; ++s) {
      const int i = bi * kPdTile + ty + 16 * r, j = bj * kPdTile + tx + 16 * s;
      if (i < j && j < n) D[cidx(i, j, n)] = __dsqrt_rn(acc[r][s]);
    }
}

// one block per row: the row's nearest neighbour, and the per-slot state of the merge loop
__global__ void __launch_bounds__(256) link_init_kernel(const double* __restrict__ D, int n, double* nn_v, int* nn_j,
                                                        double* size, int* active, int* label) {
  __shared__ double sv[32];
  __shared__ int sj[32];
  const int k = blockIdx.x;
  double bv = INFINITY;
  int bj = INT_MAX;
  for (int j = threadIdx.x; j < n; j += blockDim.x) {
    if (j == k) continue;
    const double v = pair_dist(D, k, j, n);
    if (before(v, j, bv, bj)) {
      bv = v;
      bj = j;
    }
  }
  block_argmin(bv, bj, sv, sj);
  if (threadIdx.x == 0) {
    nn_v[k] = bv;
    nn_j[k] = bj;
    size[k] = 1.0;
    active[k] = 1;
    label[k] = k;
  }
}

// The whole merge loop.  Per merge:
//   A  (each CTA) rescan its stale rows, then publish the best (height, a, b) over its active rows in shared memory
//   -- cluster barrier --
//   B  (each CTA) read the kLinkCta candidates through DSMEM and take the same global minimum; update d(k, b) for its
//      own rows, lower or mark their caches; the owner of a retires it, the owner of b marks row b stale, CTA 0 writes
//      the Z row
//   -- cluster barrier --
// size[b] is read by every CTA in B, so its owner writes the new size in the next A.
__global__ void __cluster_dims__(kLinkCta, 1, 1) __launch_bounds__(kLinkThreads, 1)
    link_merge_kernel(double* D, int n, double* nn_v, int* nn_j, double* size, int* active, int* label, int* stale,
                      double* Z) {
  cg::cluster_group cluster = cg::this_cluster();
  const int rank = (int)cluster.block_rank();
  const int R = (n + kLinkCta - 1) / kLinkCta;
  const int r0 = min(n, rank * R), r1 = min(n, r0 + R);
  int* my_stale = stale + (long long)rank * R;            // at most R rows of this CTA are stale at once
  __shared__ double cand_v;                               // this CTA's best pair, read by the whole cluster
  __shared__ int cand_a, cand_b;
  __shared__ double sel_v;
  __shared__ int sel_a, sel_b;
  __shared__ int n_stale;
  __shared__ double red_v[32];
  __shared__ int red_a[32], red_b[32];
  int pend_b = -1;                                        // thread 0: size[pend_b] = pend_s, one phase late
  double pend_s = 0.0;
  if (threadIdx.x == 0) n_stale = 0;
  __syncthreads();

  for (int step = 0; step < n - 1; ++step) {
    // ---- A
    if (threadIdx.x == 0 && pend_b >= 0) size[pend_b] = pend_s;
    const int ns = n_stale;
    for (int q = 0; q < ns; ++q) {
      const int k = __ldcg(my_stale + q);
      double bv = INFINITY;
      int bj = INT_MAX;
      for (int j = threadIdx.x; j < n; j += blockDim.x) {
        if (j == k || !__ldcg(active + j)) continue;
        const double v = pair_dist(D, k, j, n);
        if (before(v, j, bv, bj)) {
          bv = v;
          bj = j;
        }
      }
      block_argmin(bv, bj, red_v, red_a);
      if (threadIdx.x == 0) {
        nn_v[k] = bv;
        nn_j[k] = bj;
      }
    }
    __syncthreads();                                      // every thread has read n_stale; thread 0's caches are out
    if (threadIdx.x == 0) n_stale = 0;
    {
      double bv = INFINITY;
      int ba = INT_MAX, bb = INT_MAX;
      for (int i = r0 + threadIdx.x; i < r1; i += blockDim.x) {
        if (!__ldcg(active + i)) continue;
        const int j = __ldcg(nn_j + i);
        const double v = __ldcg(nn_v + i);
        const int a = min(i, j), b = max(i, j);
        if (pair_before(v, a, b, bv, ba, bb)) {
          bv = v;
          ba = a;
          bb = b;
        }
      }
      warp_pairmin(bv, ba, bb);
      const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
      if (l == 0) {
        red_v[w] = bv;
        red_a[w] = ba;
        red_b[w] = bb;
      }
      __syncthreads();
      if (w == 0) {
        bv = red_v[l];
        ba = red_a[l];
        bb = red_b[l];
        warp_pairmin(bv, ba, bb);
        if (l == 0) {
          cand_v = bv;
          cand_a = ba;
          cand_b = bb;
        }
      }
    }
    cluster.sync();
    // ---- B
    if (threadIdx.x < 32) {
      double v = INFINITY;
      int a = INT_MAX, b = INT_MAX;
      if (threadIdx.x < kLinkCta) {
        v = *cluster.map_shared_rank(&cand_v, threadIdx.x);
        a = *cluster.map_shared_rank(&cand_a, threadIdx.x);
        b = *cluster.map_shared_rank(&cand_b, threadIdx.x);
      }
      warp_pairmin(v, a, b);
      if (threadIdx.x == 0) {
        sel_v = v;
        sel_a = a;
        sel_b = b;
      }
    }
    __syncthreads();
    const double d = sel_v;
    const int a = sel_a, b = sel_b;
    const double sa = __ldcg(size + a), sb = __ldcg(size + b);
    const double s = __dadd_rn(sa, sb);
    const double t3 = __ddiv_rn(__dmul_rn(__dmul_rn(__dmul_rn(sa, sb), d), d), s);
    for (int k = r0 + threadIdx.x; k < r1; k += blockDim.x) {
      if (k == a || k == b || !__ldcg(active + k)) continue;
      const double dak = pair_dist(D, a, k, n), dbk = pair_dist(D, b, k, n);
      const double t1 = __dmul_rn(__dmul_rn(sa, dak), dak);
      const double t2 = __dmul_rn(__dmul_rn(sb, dbk), dbk);
      const double v = __dsqrt_rn(__ddiv_rn(__dsub_rn(__dadd_rn(t1, t2), t3), s));
      D[k < b ? cidx(k, b, n) : cidx(b, k, n)] = v;
      const int nk = __ldcg(nn_j + k);
      if (nk == a || nk == b) {
        my_stale[atomicAdd(&n_stale, 1)] = k;
      } else if (before(v, b, __ldcg(nn_v + k), nk)) {
        nn_v[k] = v;
        nn_j[k] = b;
      }
    }
    if (threadIdx.x == 0) {
      if (a >= r0 && a < r1) active[a] = 0;
      pend_b = -1;
      if (b >= r0 && b < r1) {
        my_stale[atomicAdd(&n_stale, 1)] = b;
        pend_b = b;
        pend_s = s;
      }
      if (rank == 0) {
        const int la = label[a], lb = label[b];
        double* z = Z + 4LL * step;
        z[0] = (double)min(la, lb);
        z[1] = (double)max(la, lb);
        z[2] = d;
        z[3] = s;
        label[b] = n + step;
      }
    }
    cluster.sync();                                       // also: no CTA exits while another reads its shared memory
  }
}

namespace {

struct LinkLayout {
  long long dist, nn_v, size, nn_j, active, label, stale, total;
};

long long align256(long long b) { return (b + 255) & ~255LL; }

LinkLayout link_layout(long long n) {
  LinkLayout L;
  const long long R = (n + kLinkCta - 1) / kLinkCta;
  long long o = 0;
  L.dist = o;
  o += align256(n * (n - 1) / 2 * 8);
  L.nn_v = o;
  o += align256(n * 8);
  L.size = o;
  o += align256(n * 8);
  L.nn_j = o;
  o += align256(n * 4);
  L.active = o;
  o += align256(n * 4);
  L.label = o;
  o += align256(n * 4);
  L.stale = o;
  o += align256(R * kLinkCta * 4);
  L.total = o;
  return L;
}

}  // namespace
}  // namespace rvb

RVB_API long long rvb_centroid_linkage_workspace_bytes(int n) {
  // past 1e9 points the condensed matrix alone (4e18 bytes) overflows no counter yet exceeds any device
  if (n < 2 || n > 1000000000) return -1;
  return rvb::link_layout(n).total;
}

RVB_API int rvb_centroid_linkage(const double* d_emb, int n, int dim, double* d_Z, double* d_dist, void* d_workspace,
                                 long long workspace_bytes, void* stream_) {
  using namespace rvb;
  cudaStream_t stream = (cudaStream_t)stream_;
  RVB_REQUIRE(d_emb && d_Z && d_workspace && n >= 2 && dim >= 1, "rvb_centroid_linkage: bad arguments");
  const long long need = rvb_centroid_linkage_workspace_bytes(n);
  RVB_REQUIRE(need > 0, "rvb_centroid_linkage: %d embeddings are too many", n);
  RVB_REQUIRE(workspace_bytes >= need, "rvb_centroid_linkage: %d embeddings need %lld bytes of workspace, %lld given", n,
              need, workspace_bytes);
  const int tiles = (n + kPdTile - 1) / kPdTile;
  RVB_REQUIRE(tiles <= 65535, "rvb_centroid_linkage: %d embeddings exceed the distance kernel's grid", n);
  const LinkLayout L = link_layout(n);
  char* ws = static_cast<char*>(d_workspace);
  double* D = reinterpret_cast<double*>(ws + L.dist);
  double* nn_v = reinterpret_cast<double*>(ws + L.nn_v);
  double* size = reinterpret_cast<double*>(ws + L.size);
  int* nn_j = reinterpret_cast<int*>(ws + L.nn_j);
  int* active = reinterpret_cast<int*>(ws + L.active);
  int* label = reinterpret_cast<int*>(ws + L.label);
  int* stale = reinterpret_cast<int*>(ws + L.stale);

  pdist_kernel<<<dim3(tiles, tiles), 256, 0, stream>>>(d_emb, n, dim, D);
  RVB_COUNT_LAUNCH();
  RVB_CHECK_LAUNCH();
  if (d_dist) RVB_CHECK_CUDA(cudaMemcpyAsync(d_dist, D, (size_t)n * (n - 1) / 2 * 8, cudaMemcpyDeviceToDevice, stream));
  link_init_kernel<<<n, 256, 0, stream>>>(D, n, nn_v, nn_j, size, active, label);
  RVB_COUNT_LAUNCH();
  RVB_CHECK_LAUNCH();
  link_merge_kernel<<<kLinkCta, kLinkThreads, 0, stream>>>(D, n, nn_v, nn_j, size, active, label, stale, d_Z);
  RVB_COUNT_LAUNCH();
  RVB_CHECK_LAUNCH();
  return 0;
}
