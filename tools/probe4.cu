// Micro-probe 4 (not product code; written at the end of round 1, to be run first thing in round 2).
//
// The ingest kernel is bound by the scattered-access path (L2 62 % busy, 3 sectors touched per row: dictionary slot,
// rows[id], sum[id]).  Which layout change buys the most?
//
//   A  today's shape      : persistent dictionary {key, id} 16 B -> id; RED rows[id], RED sum[id]   (3 sectors, 3 L2 ops)
//   B  slot-resident      : per-pane table of 32-byte slots {key, rows, sum, pad}: find-or-claim the slot, then two REDs
//                           into the same sector                                                     (1 sector, 3 L2 ops)
//   C  slot-resident AoS16: per-pane 16-byte slots {key, packed} with packed = rows << 40 | (sum & 2^40-1): ONE RED per row
//                           (upper bound for a guarded packed accumulator: only exact while a key has < 2^24 rows and
//                           |sum| < 2^39 in one pane)                                                (1 sector, 2 L2 ops)
//   D  A with the accumulators interleaved {rows, sum} 16 B per id (AoS)                             (2 sectors, 3 L2 ops)
//
// Same input as probe3: 16 Mi rows, 1 Mi distinct 64-bit keys, every table sized at load factor 0.25 / 0.5.
#include <cuda_runtime.h>
#include <climits>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <vector>
#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("CUDA %s at %d\n", cudaGetErrorString(e), __LINE__); exit(1);} } while (0)
__host__ __device__ inline uint64_t mix64(uint64_t x) {
  uint64_t z = x + 0x9E3779B97F4A7C15ull; z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull; z = (z ^ (z >> 27)) * 0x94D049BB133111EBull; return z ^ (z >> 31);
}
__host__ __device__ inline uint32_t home_of(long long key, uint32_t cap) { return (uint32_t)(((mix64((uint64_t)key) >> 32) * (uint64_t)cap) >> 32); }
constexpr long long EMPTY = LLONG_MIN;
struct alignas(16) Slot16 { long long key; unsigned long long v; };
struct alignas(32) Slot32 { long long key; unsigned long long rows, sum, pad; };

__device__ __forceinline__ void red_u64(unsigned long long* p, unsigned long long v) {
  asm volatile("red.global.add.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}

// A / D: persistent dictionary -> id -> accumulators (SoA or AoS)
template <int AOS>
__global__ void __launch_bounds__(256, 4) dict_kernel(const long long* __restrict__ key, const long long* __restrict__ val, long long n,
                                                      const Slot16* __restrict__ dict, uint32_t cap, unsigned long long* acc, unsigned long long K) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (; i < n; i += stride) {
    const long long k = __ldcs(key + i), v = __ldcs(val + i);
    uint32_t pos = home_of(k, cap);
    ulonglong2 raw = __ldcg(reinterpret_cast<const ulonglong2*>(dict + pos));
    while ((long long)raw.x != k) { pos = pos + 1 == cap ? 0 : pos + 1; raw = __ldcg(reinterpret_cast<const ulonglong2*>(dict + pos)); }
    const unsigned long long id = raw.y;
    if (AOS) { red_u64(acc + 2 * id, 1ull); red_u64(acc + 2 * id + 1, (unsigned long long)v); }
    else { red_u64(acc + id, 1ull); red_u64(acc + K + id, (unsigned long long)v); }
  }
}

// B: per-pane 32-byte slots; first touch claims the slot with a CAS on the key
__global__ void __launch_bounds__(256, 4) slot32_kernel(const long long* __restrict__ key, const long long* __restrict__ val, long long n,
                                                        Slot32* __restrict__ tab, uint32_t cap) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (; i < n; i += stride) {
    const long long k = __ldcs(key + i), v = __ldcs(val + i);
    uint32_t pos = home_of(k, cap);
    while (true) {
      long long cur = *(volatile long long*)&tab[pos].key;
      if (cur == EMPTY) cur = (long long)atomicCAS((unsigned long long*)&tab[pos].key, (unsigned long long)EMPTY, (unsigned long long)k), cur = cur == EMPTY ? k : cur;
      if (cur == k) break;
      pos = pos + 1 == cap ? 0 : pos + 1;
    }
    red_u64(&tab[pos].rows, 1ull);
    red_u64(&tab[pos].sum, (unsigned long long)v);
  }
}

// C: per-pane 16-byte slots, one packed RED per row
__global__ void __launch_bounds__(256, 4) slot16_kernel(const long long* __restrict__ key, const long long* __restrict__ val, long long n,
                                                        Slot16* __restrict__ tab, uint32_t cap) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (; i < n; i += stride) {
    const long long k = __ldcs(key + i), v = __ldcs(val + i);
    uint32_t pos = home_of(k, cap);
    while (true) {
      long long cur = *(volatile long long*)&tab[pos].key;
      if (cur == EMPTY) cur = (long long)atomicCAS((unsigned long long*)&tab[pos].key, (unsigned long long)EMPTY, (unsigned long long)k), cur = cur == EMPTY ? k : cur;
      if (cur == k) break;
      pos = pos + 1 == cap ? 0 : pos + 1;
    }
    red_u64(&tab[pos].v, (1ull << 40) + ((unsigned long long)v & ((1ull << 40) - 1)));
  }
}

template <class T>
__global__ void init_kernel(T* t, uint64_t n) {
  uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  for (; i < n; i += (uint64_t)gridDim.x * blockDim.x) { T s{}; s.key = EMPTY; t[i] = s; }
}

int main() {
  const long long n = 1ll << 24; const unsigned long long K = 1ull << 20;
  long long *k, *v;
  CK(cudaMalloc(&k, n * 8)); CK(cudaMalloc(&v, n * 8));
  std::vector<long long> hk(n), hv(n), keys(K);
  for (unsigned long long i = 0; i < K; ++i) keys[i] = (long long)mix64(i * 7919 + 1);
  uint64_t st = 42; unsigned long long want_sum = 0;
  for (long long i = 0; i < n; ++i) { st = mix64(st + i); hk[i] = keys[st % K]; hv[i] = (long long)((st >> 20) % 100000000); want_sum += (unsigned long long)hv[i]; }
  CK(cudaMemcpy(k, hk.data(), n * 8, cudaMemcpyHostToDevice)); CK(cudaMemcpy(v, hv.data(), n * 8, cudaMemcpyHostToDevice));
  cudaEvent_t e0, e1; CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
  const int grid = 132 * 8;
  auto timeit = [&](const char* name, auto launch, auto reset) {
    reset(); launch(); CK(cudaDeviceSynchronize()); CK(cudaGetLastError());
    float best = 1e9f;
    for (int r = 0; r < 5; ++r) {
      reset(); CK(cudaDeviceSynchronize());
      CK(cudaEventRecord(e0)); launch(); CK(cudaEventRecord(e1)); CK(cudaEventSynchronize(e1));
      float ms; CK(cudaEventElapsedTime(&ms, e0, e1)); best = ms < best ? ms : best;
    }
    printf("%-64s %7.3f ms  %7.2f Grows/s\n", name, best, n / best / 1e6);
  };
  for (double spi : {3.5, 2.0}) {
    const uint32_t cap = (uint32_t)(K * spi);
    printf("---- %.1f slots per key (cap %u) ----\n", spi, cap);
    // A / D
    std::vector<Slot16> hd(cap, Slot16{EMPTY, 0});
    for (unsigned long long i = 0; i < K; ++i) { uint32_t pos = home_of(keys[i], cap); while (hd[pos].key != EMPTY) pos = pos + 1 == cap ? 0 : pos + 1; hd[pos].key = keys[i]; hd[pos].v = i; }
    Slot16* dict; CK(cudaMalloc(&dict, (size_t)cap * 16)); CK(cudaMemcpy(dict, hd.data(), (size_t)cap * 16, cudaMemcpyHostToDevice));
    unsigned long long* acc; CK(cudaMalloc(&acc, K * 16));
    timeit("A dictionary 16 B -> id, SoA rows[] sum[] (today)", [&] { dict_kernel<0><<<grid, 256>>>(k, v, n, dict, cap, acc, K); }, [&] { CK(cudaMemsetAsync(acc, 0, K * 16)); });
    timeit("D dictionary 16 B -> id, AoS {rows, sum}", [&] { dict_kernel<1><<<grid, 256>>>(k, v, n, dict, cap, acc, K); }, [&] { CK(cudaMemsetAsync(acc, 0, K * 16)); });
    // B
    Slot32* t32; CK(cudaMalloc(&t32, (size_t)cap * 32));
    timeit("B per-pane 32 B slots {key, rows, sum}: claim + 2 RED, one sector", [&] { slot32_kernel<<<grid, 256>>>(k, v, n, t32, cap); },
           [&] { init_kernel<<<grid, 256>>>(t32, (uint64_t)cap); });
    {  // check B
      std::vector<Slot32> h(cap); CK(cudaMemcpy(h.data(), t32, (size_t)cap * 32, cudaMemcpyDeviceToHost));
      unsigned long long rows = 0, sum = 0, used = 0; for (auto& s : h) if (s.key != EMPTY) { rows += s.rows; sum += s.sum; ++used; }
      if (rows != (unsigned long long)n || sum != want_sum || used != K) printf("   !! B wrong: rows %llu sum %s keys %llu\n", rows, sum == want_sum ? "ok" : "BAD", used);
    }
    // B steady state: the table already holds every key (panes after the first reuse the slots' keys)
    timeit("B' same, keys already claimed (no CAS): load + 2 RED, one sector", [&] { slot32_kernel<<<grid, 256>>>(k, v, n, t32, cap); }, [&] {});
    // C
    Slot16* t16; CK(cudaMalloc(&t16, (size_t)cap * 16));
    timeit("C per-pane 16 B slots {key, rows<<40 | sum}: claim + 1 RED", [&] { slot16_kernel<<<grid, 256>>>(k, v, n, t16, cap); },
           [&] { init_kernel<<<grid, 256>>>(t16, (uint64_t)cap); });
    timeit("C' same, keys already claimed: load + 1 RED", [&] { slot16_kernel<<<grid, 256>>>(k, v, n, t16, cap); }, [&] {});
    CK(cudaFree(dict)); CK(cudaFree(acc)); CK(cudaFree(t32)); CK(cudaFree(t16));
  }
  return 0;
}
