// Micro-probe 3 (not product code): is "partition rows by dictionary home range, then aggregate each
// range in shared memory" faster than one global probe + two global REDs per row (probe2: 46 G rows/s)?
//
//   pass A  partition_kernel : rows (key, val, ts) -> bucket regions of 16-byte records {key, val32 | pane << 32}
//                              bucket = home slot >> LOG_SPB, one shared-memory atomic per row for the rank,
//                              one global atomic per (tile, bucket) for the base
//   pass B  aggregate_kernel : one block per bucket: dictionary slot range -> shared memory, rows probe it
//                              there and add into shared accumulators, then one RED per touched key
//
// The partition buffer of one sub-chunk is meant to stay in L2 (sub-chunk rows x 16 B).
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
struct alignas(16) Slot { long long key; uint32_t id; uint32_t pad; };

constexpr int A_THREADS = 1024;
template <int RPT>
__global__ void __launch_bounds__(A_THREADS, 1)
partition_kernel(const long long* __restrict__ key, const long long* __restrict__ val, const long long* __restrict__ ts, long long n,
                 uint32_t cap, int log_spb, uint32_t P, ulonglong2* __restrict__ region, uint32_t RC,
                 unsigned int* __restrict__ cursor, unsigned int* __restrict__ n_defer, long long wm, unsigned long long slide_inv,
                 long long slide) {
  extern __shared__ unsigned int s_mem[];
  unsigned int* s_cnt = s_mem;
  unsigned int* s_base = s_mem + P;
  const long long tile = (long long)A_THREADS * RPT;
  for (long long base = (long long)blockIdx.x * tile; base < n; base += (long long)gridDim.x * tile) {
    for (uint32_t i = threadIdx.x; i < P; i += A_THREADS) s_cnt[i] = 0;
    __syncthreads();
    long long k[RPT]; uint32_t v[RPT]; uint32_t br[RPT]; uint32_t rk[RPT];
#pragma unroll
    for (int j = 0; j < RPT; ++j) {
      const long long r = base + j * A_THREADS + threadIdx.x;
      br[j] = 0xFFFFFFFFu;
      if (r < n) {
        k[j] = __ldcs(key + r);
        const long long vv = __ldcs(val + r);
        const long long t = __ldcs(ts + r);
        const unsigned long long q = __umul64hi((unsigned long long)t, slide_inv);  // pane number (approx, probe only)
        if (t >= wm) {
          const uint32_t b = home_of(k[j], cap) >> log_spb;
          br[j] = b;
          v[j] = (uint32_t)vv;
          rk[j] = atomicAdd(&s_cnt[b], 1u) | ((uint32_t)(q & 0xFF) << 24);
        }
      }
    }
    __syncthreads();
    for (uint32_t i = threadIdx.x; i < P; i += A_THREADS) {
      const unsigned int c = s_cnt[i];
      s_base[i] = c ? atomicAdd(&cursor[i], c) : 0u;
    }
    __syncthreads();
    unsigned int dropped = 0;
#pragma unroll
    for (int j = 0; j < RPT; ++j) {
      if (br[j] != 0xFFFFFFFFu) {
        const uint32_t pos = s_base[br[j]] + (rk[j] & 0xFFFFFFu);
        if (pos < RC) {
          ulonglong2 rec;
          rec.x = (unsigned long long)k[j];
          rec.y = (unsigned long long)v[j] | ((unsigned long long)(rk[j] >> 24) << 32);
          region[(size_t)br[j] * RC + pos] = rec;
        } else {
          ++dropped;
        }
      }
    }
    if (dropped) atomicAdd(n_defer, dropped);
    __syncthreads();
  }
}

template <int THREADS>
__global__ void __launch_bounds__(THREADS)
aggregate_kernel(const Slot* __restrict__ slots, uint32_t cap, int log_spb, int margin, const ulonglong2* __restrict__ region,
                 uint32_t RC, unsigned int* __restrict__ cursor, unsigned long long* __restrict__ acc_rows,
                 unsigned long long* __restrict__ acc_sum, unsigned int* __restrict__ n_defer) {
  extern __shared__ unsigned long long s_u64[];
  const int spb = 1 << log_spb;
  const int S = spb + margin;
  long long* s_key = reinterpret_cast<long long*>(s_u64);
  unsigned long long* s_sum = s_u64 + S;
  unsigned int* s_id = reinterpret_cast<unsigned int*>(s_u64 + 2 * S);
  unsigned int* s_rows = s_id + S;
  const uint32_t b = blockIdx.x;
  const uint32_t lo = b << log_spb;
  for (int i = threadIdx.x; i < S; i += THREADS) {
    uint32_t g = lo + i;
    if (g >= cap) g -= cap;
    const ulonglong2 raw = __ldcg(reinterpret_cast<const ulonglong2*>(slots + g));
    s_key[i] = (long long)raw.x;
    s_id[i] = (uint32_t)raw.y;
    s_rows[i] = 0;
    s_sum[i] = 0;
  }
  __syncthreads();
  const uint32_t nb = min(cursor[b], RC);
  const ulonglong2* rows = region + (size_t)b * RC;
  unsigned int missed = 0;
  for (uint32_t i = threadIdx.x; i < nb; i += THREADS) {
    const ulonglong2 rec = __ldcs(rows + i);
    const long long key = (long long)rec.x;
    int p = (int)(home_of(key, cap) - lo);
    bool hit = false;
    while (p < S) {
      const long long kk = s_key[p];
      if (kk == key) { hit = true; break; }
      if (kk == EMPTY) break;
      ++p;
    }
    if (hit) {
      atomicAdd(&s_rows[p], 1u);
      atomicAdd(&s_sum[p], (unsigned long long)(long long)(int)(uint32_t)rec.y);
    } else {
      ++missed;
    }
  }
  if (missed) atomicAdd(n_defer, missed);
  __syncthreads();
  for (int i = threadIdx.x; i < S; i += THREADS) {
    const unsigned int r = s_rows[i];
    if (r) {
      const uint32_t id = s_id[i];
      asm volatile("red.global.add.u64 [%0], %1;" ::"l"(acc_rows + id), "l"((unsigned long long)r) : "memory");
      asm volatile("red.global.add.u64 [%0], %1;" ::"l"(acc_sum + id), "l"(s_sum[i]) : "memory");
    }
  }
  if (threadIdx.x == 0) cursor[b] = 0;
}

// the current product shape for comparison: one global probe + two REDs per row
__global__ void __launch_bounds__(256, 4)
direct_kernel(const long long* __restrict__ key, const long long* __restrict__ val, const long long* __restrict__ ts, long long n,
              const Slot* __restrict__ slots, uint32_t cap, unsigned long long* acc_rows, unsigned long long* acc_sum, long long wm) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (; i < n; i += stride) {
    const long long k = __ldcs(key + i), v = __ldcs(val + i), t = __ldcs(ts + i);
    if (t < wm) continue;
    uint32_t pos = home_of(k, cap);
    ulonglong2 raw = __ldcg(reinterpret_cast<const ulonglong2*>(slots + pos));
    while ((long long)raw.x != k) { pos = pos + 1 == cap ? 0 : pos + 1; raw = __ldcg(reinterpret_cast<const ulonglong2*>(slots + pos)); }
    const uint32_t id = (uint32_t)raw.y;
    asm volatile("red.global.add.u64 [%0], %1;" ::"l"(acc_rows + id), "l"(1ull) : "memory");
    asm volatile("red.global.add.u64 [%0], %1;" ::"l"(acc_sum + id), "l"((unsigned long long)v) : "memory");
  }
}

int main() {
  const long long n = 1ll << 24; const unsigned long long K = 1ull << 20;
  long long *k, *v, *t;
  CK(cudaMalloc(&k, n * 8)); CK(cudaMalloc(&v, n * 8)); CK(cudaMalloc(&t, n * 8));
  std::vector<long long> hk(n), hv(n), ht(n), keys(K);
  for (unsigned long long i = 0; i < K; ++i) keys[i] = (long long)mix64(i * 7919 + 1);
  uint64_t st = 42; unsigned long long want_sum = 0;
  for (long long i = 0; i < n; ++i) { st = mix64(st + i); hk[i] = keys[st % K]; hv[i] = (long long)((st >> 20) % 100000000); ht[i] = 1700000000000000000ll + (long long)((st >> 8) % 1000000000); want_sum += (unsigned long long)hv[i]; }
  CK(cudaMemcpy(k, hk.data(), n * 8, cudaMemcpyHostToDevice)); CK(cudaMemcpy(v, hv.data(), n * 8, cudaMemcpyHostToDevice)); CK(cudaMemcpy(t, ht.data(), n * 8, cudaMemcpyHostToDevice));
  unsigned long long *acc; CK(cudaMalloc(&acc, K * 2 * 8 + 64));
  unsigned int* n_defer; CK(cudaMalloc(&n_defer, 4));
  cudaEvent_t e0, e1; CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
  const long long wm = 1700000000000000000ll; const long long slide = 1000000000ll; const unsigned long long slide_inv = ~0ull / (unsigned long long)slide;
  std::vector<unsigned long long> hacc(K * 2);
  auto check = [&](const char* what) {
    CK(cudaMemcpy(hacc.data(), acc, K * 2 * 8, cudaMemcpyDeviceToHost));
    unsigned long long rows = 0, sum = 0; for (unsigned long long i = 0; i < K; ++i) { rows += hacc[i]; sum += hacc[K + i]; }
    unsigned int nd; CK(cudaMemcpy(&nd, n_defer, 4, cudaMemcpyDeviceToHost));
    if (rows + nd != (unsigned long long)n || (nd == 0 && sum != want_sum)) printf("   !! %s: rows %llu deferred %u (want %lld) sum %s\n", what, rows, nd, n, sum == want_sum ? "ok" : "BAD");
    return nd;
  };
  for (double spi : {3.5, 2.0, 1.5}) for (int order = 0; order < 2; ++order) {
    const uint32_t cap = (uint32_t)(K * spi);
    std::vector<Slot> hd(cap, Slot{EMPTY, 0xFFFFFFFFu, 0});
    for (unsigned long long i = 0; i < K; ++i) { uint32_t pos = home_of(keys[i], cap); while (hd[pos].key != EMPTY) pos = pos + 1 == cap ? 0 : pos + 1; hd[pos].key = keys[i]; hd[pos].id = (uint32_t)i; }
    if (order == 1) { uint32_t id = 0; for (uint32_t p = 0; p < cap; ++p) if (hd[p].key != EMPTY) hd[p].id = id++; }
    Slot* slots; CK(cudaMalloc(&slots, (size_t)cap * 16)); CK(cudaMemcpy(slots, hd.data(), (size_t)cap * 16, cudaMemcpyHostToDevice));
    printf("---- dict %.2f slots/id (%.0f MB), ids in %s order ----\n", spi, cap * 16.0 / 1e6, order ? "slot" : "arrival");
    {
      CK(cudaMemset(acc, 0, K * 16)); CK(cudaMemset(n_defer, 0, 4));
      direct_kernel<<<132 * 8, 256>>>(k, v, t, n, slots, cap, acc, acc + K, wm); CK(cudaDeviceSynchronize()); check("direct");
      CK(cudaEventRecord(e0));
      for (int r = 0; r < 5; ++r) direct_kernel<<<132 * 8, 256>>>(k, v, t, n, slots, cap, acc, acc + K, wm);
      CK(cudaEventRecord(e1)); CK(cudaEventSynchronize(e1)); float ms; CK(cudaEventElapsedTime(&ms, e0, e1)); ms /= 5;
      printf("direct probe + 2 RED                                         %7.3f ms  %7.2f Grows/s\n", ms, n / ms / 1e6);
    }
    for (int log_spb : {11, 12}) for (long long n_sub : {1ll << 20, 1ll << 21, 1ll << 22, 1ll << 23}) {
      const int margin = 64;
      const uint32_t P = (cap + (1u << log_spb) - 1) >> log_spb;
      const uint32_t RC = (uint32_t)(n_sub / P * 5 / 4 + 256);
      ulonglong2* region; CK(cudaMalloc(&region, (size_t)P * RC * 16));
      unsigned int* cursor; CK(cudaMalloc(&cursor, P * 4)); CK(cudaMemset(cursor, 0, P * 4));
      const int S = (1 << log_spb) + margin;
      const size_t smemB = (size_t)S * 24, smemA = (size_t)P * 8;
      constexpr int RPT = 8; constexpr int BT = 512;
      CK(cudaFuncSetAttribute(aggregate_kernel<BT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smemB));
      CK(cudaFuncSetAttribute(partition_kernel<RPT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smemA));
      int occB = 0; CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occB, aggregate_kernel<BT>, BT, smemB));
      const int gridA = (int)std::min<long long>((n_sub + A_THREADS * RPT - 1) / (A_THREADS * RPT), 132 * 2);
      auto pass = [&]() {
        for (long long off = 0; off < n; off += n_sub) {
          partition_kernel<RPT><<<gridA, A_THREADS, smemA>>>(k + off, v + off, t + off, n_sub, cap, log_spb, P, region, RC, cursor, n_defer, wm, slide_inv, slide);
          aggregate_kernel<BT><<<P, BT, smemB>>>(slots, cap, log_spb, margin, region, RC, cursor, acc, acc + K, n_defer);
        }
      };
      CK(cudaMemset(acc, 0, K * 16)); CK(cudaMemset(n_defer, 0, 4));
      pass(); CK(cudaDeviceSynchronize()); CK(cudaGetLastError());
      unsigned int nd = check("partitioned");
      CK(cudaEventRecord(e0));
      for (int r = 0; r < 5; ++r) pass();
      CK(cudaEventRecord(e1)); CK(cudaEventSynchronize(e1)); float ms; CK(cudaEventElapsedTime(&ms, e0, e1)); ms /= 5;
      // pass A alone / pass B alone
      CK(cudaEventRecord(e0));
      for (int r = 0; r < 5; ++r) for (long long off = 0; off < n; off += n_sub) { partition_kernel<RPT><<<gridA, A_THREADS, smemA>>>(k + off, v + off, t + off, n_sub, cap, log_spb, P, region, RC, cursor, n_defer, wm, slide_inv, slide); CK(cudaMemsetAsync(cursor, 0, P * 4)); }
      CK(cudaEventRecord(e1)); CK(cudaEventSynchronize(e1)); float msA; CK(cudaEventElapsedTime(&msA, e0, e1)); msA /= 5;
      printf("partitioned spb=%4d P=%5u sub=%2lldMi smemB=%3zuKB occB=%d deferred=%u  %7.3f ms  %7.2f Grows/s   (A alone %7.3f ms)\n",
             1 << log_spb, P, n_sub >> 20, smemB >> 10, occB, nd, ms, n / ms / 1e6, msA);
      CK(cudaFree(region)); CK(cudaFree(cursor));
    }
    CK(cudaFree(slots));
  }
  return 0;
}
