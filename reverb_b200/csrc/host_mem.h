// reverb_b200 — who owns the device and page-locked memory of the native models (the ASR plan, segmentation,
// embedding): grow-only workspaces and the weight store.  Each frees what it holds when it is destroyed, and every byte
// held is counted (rvb_held_bytes, include/rvb_b200.h).
#pragma once
#include <atomic>
#include <map>
#include <string>
#include <vector>

#include "common.cuh"

namespace rvb {

// bytes currently held by DevBufs and WeightStores (device) and by HostPinneds (page-locked host memory)
inline std::atomic<long long> g_held_device{0}, g_held_pinned{0};

// Grow-only buffer: ensure(n) keeps the allocation when it already holds n bytes, else replaces it by one of
// n + n/8 + 256 bytes (device) or n + 256 bytes (page-locked host), or of exactly n bytes when `exact` (a buffer that
// grows in rare, whole steps, such as a fold stack slot by slot).  Move-only: the destructor frees.
template <bool Pinned>
struct GrowBuf {
  void* p = nullptr;
  size_t cap = 0;
  GrowBuf() = default;
  GrowBuf(const GrowBuf&) = delete;
  GrowBuf& operator=(const GrowBuf&) = delete;
  GrowBuf(GrowBuf&& o) noexcept : p(o.p), cap(o.cap) {
    o.p = nullptr;
    o.cap = 0;
  }
  GrowBuf& operator=(GrowBuf&& o) noexcept {
    if (this != &o) {
      release();
      p = o.p;
      cap = o.cap;
      o.p = nullptr;
      o.cap = 0;
    }
    return *this;
  }
  ~GrowBuf() { release(); }
  int ensure(size_t bytes, bool exact = false) {
    if (bytes <= cap) return 0;
    release();
    const size_t want = exact ? bytes : Pinned ? bytes + 256 : bytes + (bytes >> 3) + 256;
    void* q = nullptr;
    RVB_CHECK_CUDA(Pinned ? cudaMallocHost(&q, want) : cudaMalloc(&q, want));
    p = q;
    cap = want;
    held() += (long long)want;
    return 0;
  }
  void release() {
    if (p) {
      if (Pinned) cudaFreeHost(p);
      else cudaFree(p);
      held() -= (long long)cap;
    }
    p = nullptr;
    cap = 0;
  }
  template <typename T>
  T* as() const { return reinterpret_cast<T*>(p); }
  static std::atomic<long long>& held() { return Pinned ? g_held_pinned : g_held_device; }
};
using DevBuf = GrowBuf<false>;
using HostPinned = GrowBuf<true>;

// The named host tensors of a model until it is finalized, and every device allocation made from them.  `what`
// prefixes the error messages of need() ("model:", "rvb_seg_finalize:", ...).
class WeightStore {
 public:
  explicit WeightStore(const char* what) : what_(what) {}
  WeightStore(const WeightStore&) = delete;
  WeightStore& operator=(const WeightStore&) = delete;
  ~WeightStore() {
    for (void* p : owned_) cudaFree(p);
    g_held_device -= (long long)owned_bytes_;
  }

  void set(const std::string& name, const float* data, size_t n) { host_[name].assign(data, data + n); }
  const std::vector<float>* find(const std::string& name) const {
    auto it = host_.find(name);
    return it == host_.end() ? nullptr : &it->second;
  }
  // the tensor `name`, which must have `numel` elements
  int need(const std::string& name, size_t numel, const std::vector<float>** out) const {
    const std::vector<float>* v = find(name);
    RVB_REQUIRE(v != nullptr, "%s tensor '%s' was not provided", what_, name.c_str());
    RVB_REQUIRE(v->size() == numel, "%s tensor '%s' has %zu elements, expected %zu", what_, name.c_str(), v->size(),
                numel);
    *out = v;
    return 0;
  }
  void drop_host() { host_.clear(); }

  // a device copy of n elements of T from src (16 pad bytes behind them), owned by the store
  template <typename T>
  int upload(const void* src, size_t n, T** dst) {
    void* p = nullptr;
    if (alloc(n * sizeof(T), &p)) return -1;
    RVB_CHECK_CUDA(cudaMemcpy(p, src, n * sizeof(T), cudaMemcpyHostToDevice));
    *dst = reinterpret_cast<T*>(p);
    return 0;
  }

 private:
  static constexpr size_t kPad = 16;
  int alloc(size_t bytes, void** out) {
    void* p = nullptr;
    RVB_CHECK_CUDA(cudaMalloc(&p, bytes + kPad));
    owned_.push_back(p);
    owned_bytes_ += bytes + kPad;
    g_held_device += (long long)(bytes + kPad);
    *out = p;
    return 0;
  }
  const char* what_;
  std::map<std::string, std::vector<float>> host_;
  std::vector<void*> owned_;
  size_t owned_bytes_ = 0;
};

}  // namespace rvb
