// Shared host/device helpers for libarroyo_b200 (sm_90a only).
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#include <climits>
#include <cstdio>
#include <cstring>
#include <map>
#include <mutex>
#include <stdexcept>
#include <string>
#include <vector>

#include "../../include/arroyo_b200.h"

namespace ab {

// ---------------------------------------------------------------------------------------------
// errors
// ---------------------------------------------------------------------------------------------
struct Error : std::runtime_error {
  int32_t status;
  Error(int32_t s, const std::string& m) : std::runtime_error(m), status(s) {}
};

inline void cuda_check(cudaError_t e, const char* what, const char* file, int line) {
  if (e != cudaSuccess) {
    char buf[512];
    snprintf(buf, sizeof buf, "CUDA error %s (%d) at %s:%d: %s", cudaGetErrorName(e), (int)e, file, line, what);
    throw Error(ARROYO_B200_FATAL, buf);
  }
}
#define AB_CUDA(x) ::ab::cuda_check((x), #x, __FILE__, __LINE__)
#define AB_REQUIRE(cond, status, msg)                  \
  do {                                                 \
    if (!(cond)) throw ::ab::Error((status), (msg));   \
  } while (0)

// Key dictionaries (dict.cuh, bdict.cuh): the id of a slot not yet published, the id of a key that found no room,
// and the key of an empty slot (the INT64_MIN key itself gets a reserved id instead of a slot).
constexpr uint32_t ID_UNSET = 0xFFFFFFFFu;
constexpr uint32_t ID_OVERFLOW = 0xFFFFFFFEu;
constexpr long long EMPTY_KEY = LLONG_MIN;

// ---------------------------------------------------------------------------------------------
// exact unsigned 64-bit division by an invariant divisor (d >= 2), branch free.
// Used for `bin = ts - ts % width` (tumbling_aggregating_window.rs:65-73): one mulhi instead of
// a ~40-instruction 64-bit division per row.
// ---------------------------------------------------------------------------------------------
struct FastDivU64 {
  uint64_t magic;
  uint32_t shift;
  uint32_t pad;
  uint64_t d;

  static FastDivU64 make(uint64_t d) {
    FastDivU64 r{};
    r.d = d;
    int fl = 63 - __builtin_clzll(d);
    if ((d & (d - 1)) == 0) {
      r.magic = 0;
      r.shift = (uint32_t)(fl - 1);
    } else {
      unsigned __int128 num = ((unsigned __int128)1 << (64 + fl));
      uint64_t m = (uint64_t)(num / d);
      uint64_t rem = (uint64_t)(num % d);
      m += m;
      uint64_t twice = rem + rem;
      if (twice >= d || twice < rem) m += 1;
      r.magic = m + 1;
      r.shift = (uint32_t)fl;
    }
    return r;
  }
#ifdef __CUDACC__
  __device__ __forceinline__ uint64_t div(uint64_t n) const {
    uint64_t q = __umul64hi(magic, n);
    uint64_t t = ((n - q) >> 1) + q;
    return t >> shift;
  }
#endif
  uint64_t div_host(uint64_t n) const {
    uint64_t q = (uint64_t)(((unsigned __int128)magic * n) >> 64);
    uint64_t t = ((n - q) >> 1) + q;
    return t >> shift;
  }
};

// 64-bit key hash (splitmix64 finaliser).  The reference routes with ahash(HASH_SEEDS) over
// DataFusion create_hashes (arroyo-operator/src/context.rs:513-517); which subtask owns a key never
// changes a result, so the function is ours (SURVEY.md 8(c)(iii)).  Same function in oracle mix64.
__host__ __device__ __forceinline__ uint64_t mix64(uint64_t x) {
  uint64_t z = x + 0x9E3779B97F4A7C15ull;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}

// ---------------------------------------------------------------------------------------------
// RAII device / pinned buffers
// ---------------------------------------------------------------------------------------------
struct DevBuf {
  void* p = nullptr;
  size_t bytes = 0;
  DevBuf() = default;
  explicit DevBuf(size_t n) { alloc(n); }
  DevBuf(const DevBuf&) = delete;
  DevBuf& operator=(const DevBuf&) = delete;
  DevBuf(DevBuf&& o) noexcept : p(o.p), bytes(o.bytes) { o.p = nullptr; o.bytes = 0; }
  DevBuf& operator=(DevBuf&& o) noexcept {
    if (this != &o) { release(); p = o.p; bytes = o.bytes; o.p = nullptr; o.bytes = 0; }
    return *this;
  }
  ~DevBuf() { release(); }
  void alloc(size_t n) {
    release();
    if (n == 0) return;
    AB_CUDA(cudaMalloc(&p, n));
    bytes = n;
  }
  void release() {
    if (p) cudaFree(p);
    p = nullptr;
    bytes = 0;
  }
  template <class T> T* as() const { return reinterpret_cast<T*>(p); }
};

struct PinnedBuf {
  void* p = nullptr;
  size_t bytes = 0;
  PinnedBuf() = default;
  explicit PinnedBuf(size_t n) { alloc(n); }
  PinnedBuf(const PinnedBuf&) = delete;
  PinnedBuf& operator=(const PinnedBuf&) = delete;
  PinnedBuf(PinnedBuf&& o) noexcept : p(o.p), bytes(o.bytes) { o.p = nullptr; o.bytes = 0; }
  PinnedBuf& operator=(PinnedBuf&& o) noexcept {
    if (this != &o) { release(); p = o.p; bytes = o.bytes; o.p = nullptr; o.bytes = 0; }
    return *this;
  }
  ~PinnedBuf() { release(); }
  void alloc(size_t n) {
    release();
    if (n == 0) return;
    AB_CUDA(cudaHostAlloc(&p, n, cudaHostAllocDefault));
    bytes = n;
  }
  void release() {
    if (p) cudaFreeHost(p);
    p = nullptr;
    bytes = 0;
  }
  template <class T> T* as() const { return reinterpret_cast<T*>(p); }
};

// Process-wide pool of pinned host buffers (power-of-two size classes).  Output Arrow arrays
// borrow from it and give the memory back from their `release` callback, which may run on any
// thread, hence the mutex.  Intentionally leaked at exit (callbacks may outlive static dtors).
class PinnedPool {
 public:
  static PinnedPool& get() {
    static PinnedPool* inst = new PinnedPool();
    return *inst;
  }
  void* alloc(size_t bytes) {
    size_t cls = 256;
    while (cls < bytes) cls <<= 1;
    {
      std::lock_guard<std::mutex> g(mu_);
      auto it = free_.find(cls);
      if (it != free_.end() && !it->second.empty()) {
        void* p = it->second.back();
        it->second.pop_back();
        live_[p] = cls;
        return p;
      }
    }
    void* p = nullptr;
    AB_CUDA(cudaHostAlloc(&p, cls, cudaHostAllocDefault));
    std::lock_guard<std::mutex> g(mu_);
    live_[p] = cls;
    return p;
  }
  void free(void* p) {
    if (!p) return;
    std::lock_guard<std::mutex> g(mu_);
    auto it = live_.find(p);
    if (it == live_.end()) return;
    free_[it->second].push_back(p);
    live_.erase(it);
  }

 private:
  std::mutex mu_;
  std::map<size_t, std::vector<void*>> free_;
  std::map<void*, size_t> live_;
};

}  // namespace ab
