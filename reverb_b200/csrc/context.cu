// reverb_b200 — context biasing graph in device memory (the automaton of utils/context_graph.py, reverb_b200/context_graph.py).
//
// The host compiles a graph to flat tables (context_graph.device_tables); rvb_context_graph_create checks them and
// uploads them once, read-only, for every search that uses the graph: children in CSR by state with token-sorted child
// lists, a dense token -> child table for the root (the fail walk of most steps ends there, and a root with thousands
// of children would otherwise cost a long binary search), fail links and the float64 bonus / emit / token_score values
// exactly as the host holds them.  The device step itself is ctx_step in ctc.cu.
//
// The graph records an event on every stream a search using it was enqueued on; destroy waits for those events, so a
// handle can be dropped while searches that use it are still in flight.
#include <math.h>
#include <stdlib.h>
#include <string.h>

#include <mutex>
#include <utility>
#include <vector>

#include "../../include/rvb_b200.h"
#include "kernels.h"

struct rvb_context_graph {
  void* dev = nullptr;
  rvb::ContextGraphView view;
  std::mutex mu;
  std::vector<std::pair<cudaStream_t, cudaEvent_t>> uses;
};

namespace rvb {

const ContextGraphView* context_graph_view(const ::rvb_context_graph* g) { return g ? &g->view : nullptr; }

int context_graph_note_use(::rvb_context_graph* g, cudaStream_t stream) {
  std::lock_guard<std::mutex> lock(g->mu);
  for (auto& u : g->uses)
    if (u.first == stream) {
      RVB_CHECK_CUDA(cudaEventRecord(u.second, stream));
      return 0;
    }
  cudaEvent_t ev;
  RVB_CHECK_CUDA(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
  g->uses.emplace_back(stream, ev);
  RVB_CHECK_CUDA(cudaEventRecord(ev, stream));
  return 0;
}

// Structural checks: a trie rooted at state 0 (every other state has exactly one parent edge), tokens in [0, V) and
// not the blank, strictly increasing within a state, fail links that point to a strictly shallower state (so every fail
// walk reaches the root), finite scores.
static int check_tables(int n, const int* off, const int* tok, const int* dst, const int* fail, const double* bonus,
                        const double* emit, const double* token_score, int V, int blank, std::vector<int>& depth) {
  RVB_REQUIRE(n >= 1 && V >= 1 && blank >= 0 && blank < V, "context graph: bad sizes (nodes=%d vocab=%d blank=%d)", n, V,
              blank);
  RVB_REQUIRE(off[0] == 0 && off[n] == n - 1, "context graph: %d edges for %d states (a trie has states - 1)", off[n], n);
  for (int s = 0; s < n; ++s) RVB_REQUIRE(off[s] <= off[s + 1], "context graph: child offsets decrease at state %d", s);
  depth.assign(n, -1);
  depth[0] = 0;
  // states are not numbered breadth first in general: walk the trie from the root
  std::vector<int> order(1, 0);
  for (size_t h = 0; h < order.size(); ++h) {
    const int s = order[h];
    for (int e = off[s]; e < off[s + 1]; ++e) {
      RVB_REQUIRE(tok[e] >= 0 && tok[e] < V && tok[e] != blank,
                  "context graph: state %d has a child on token %d (vocab %d, blank %d)", s, tok[e], V, blank);
      RVB_REQUIRE(e == off[s] || tok[e - 1] < tok[e], "context graph: children of state %d not sorted by token", s);
      const int c = dst[e];
      RVB_REQUIRE(c > 0 && c < n && depth[c] < 0, "context graph: state %d reached twice or out of range", c);
      depth[c] = depth[s] + 1;
      order.push_back(c);
    }
  }
  RVB_REQUIRE((int)order.size() == n, "context graph: %d of %d states unreachable from the root", n - (int)order.size(), n);
  RVB_REQUIRE(fail[0] == 0, "context graph: the root must fail to itself");
  for (int s = 1; s < n; ++s)
    RVB_REQUIRE(fail[s] >= 0 && fail[s] < n && depth[fail[s]] < depth[s],
                "context graph: fail link %d -> %d does not lead toward the root", s, fail[s]);
  for (int s = 0; s < n; ++s)
    RVB_REQUIRE(isfinite(bonus[s]) && isfinite(emit[s]) && isfinite(token_score[s]),
                "context graph: non-finite score at state %d", s);
  return 0;
}

}  // namespace rvb

RVB_API rvb_context_graph* rvb_context_graph_create(int n_nodes, const int* h_child_off, const int* h_child_tok,
                                                    const int* h_child_dst, const int* h_fail, const double* h_bonus,
                                                    const double* h_emit, const double* h_token_score, int vocab,
                                                    int blank_id) {
  if (n_nodes < 1 || !h_child_off || !h_fail || !h_bonus || !h_emit || !h_token_score ||
      (n_nodes > 1 && (!h_child_tok || !h_child_dst))) {
    rvb::set_error("rvb_context_graph_create: bad arguments");
    return nullptr;
  }
  std::vector<int> depth;
  if (rvb::check_tables(n_nodes, h_child_off, h_child_tok, h_child_dst, h_fail, h_bonus, h_emit, h_token_score, vocab,
                        blank_id, depth))
    return nullptr;
  const size_t n = (size_t)n_nodes, ne = (size_t)n_nodes - 1;
  std::vector<int> root_next((size_t)vocab, -1);
  for (int e = h_child_off[0]; e < h_child_off[1]; ++e) root_next[h_child_tok[e]] = h_child_dst[e];
  // doubles first (8-byte aligned), then the int tables
  const size_t dbl = 3 * n * sizeof(double);
  const size_t ints = (n + 1) + 2 * ne + n + (size_t)vocab;
  rvb_context_graph* g = new rvb_context_graph;
  if (cudaMalloc(&g->dev, dbl + ints * sizeof(int)) != cudaSuccess) {
    cudaGetLastError();
    rvb::set_error("rvb_context_graph_create: cudaMalloc of %zu bytes failed", dbl + ints * sizeof(int));
    delete g;
    return nullptr;
  }
  std::vector<char> host(dbl + ints * sizeof(int));
  double* hd = reinterpret_cast<double*>(host.data());
  memcpy(hd, h_bonus, n * sizeof(double));
  memcpy(hd + n, h_emit, n * sizeof(double));
  memcpy(hd + 2 * n, h_token_score, n * sizeof(double));
  int* hi = reinterpret_cast<int*>(host.data() + dbl);
  memcpy(hi, h_child_off, (n + 1) * sizeof(int));
  if (ne) {
    memcpy(hi + n + 1, h_child_tok, ne * sizeof(int));
    memcpy(hi + n + 1 + ne, h_child_dst, ne * sizeof(int));
  }
  memcpy(hi + n + 1 + 2 * ne, h_fail, n * sizeof(int));
  memcpy(hi + 2 * n + 1 + 2 * ne, root_next.data(), (size_t)vocab * sizeof(int));
  if (cudaMemcpy(g->dev, host.data(), host.size(), cudaMemcpyHostToDevice) != cudaSuccess) {
    cudaGetLastError();
    rvb::set_error("rvb_context_graph_create: upload failed");
    cudaFree(g->dev);
    delete g;
    return nullptr;
  }
  const double* dd = reinterpret_cast<const double*>(g->dev);
  const int* di = reinterpret_cast<const int*>(reinterpret_cast<const char*>(g->dev) + dbl);
  rvb::ContextGraphView& v = g->view;
  v.bonus = dd;
  v.emit = dd + n;
  v.token_score = dd + 2 * n;
  v.off = di;
  v.tok = di + n + 1;
  v.dst = di + n + 1 + ne;
  v.fail = di + n + 1 + 2 * ne;
  v.root_next = di + 2 * n + 1 + 2 * ne;
  v.n_nodes = n_nodes;
  v.vocab = vocab;
  return g;
}

RVB_API void rvb_context_graph_destroy(rvb_context_graph* g) {
  if (g == nullptr) return;
  {
    std::lock_guard<std::mutex> lock(g->mu);
    for (auto& u : g->uses) {
      cudaEventSynchronize(u.second);  // searches enqueued with this graph have finished reading it
      cudaEventDestroy(u.second);
    }
    g->uses.clear();
  }
  cudaFree(g->dev);
  delete g;
}
