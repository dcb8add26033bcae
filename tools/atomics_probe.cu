// Micro-probe (not product code): how fast can an H100 do the scatter part of a keyed aggregate?
// Measures, for R random rows into K keys: (a) 1/2/3 x RED.64 into dense L2-resident arrays,
// (b) the same preceded by a 16-byte dictionary probe, (c) u32 vs u64 counters, (d) AoS vs SoA.
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o tools/atomics_probe tools/atomics_probe.cu
#include <cuda_runtime.h>
#include <cstdio>
#include <cstdlib>
#include <cstdint>
#include <vector>

#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("CUDA %s at %d\n", cudaGetErrorString(e), __LINE__); exit(1);} } while (0)

__host__ __device__ inline uint64_t mix64(uint64_t x) {
  uint64_t z = x + 0x9E3779B97F4A7C15ull;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}

// MODE bits: 1 = rows RED, 2 = sum RED, 4 = f64 RED, 8 = dictionary probe first, 16 = u32 rows, 32 = AoS, 64 = no atomics (loads only)
template <int MODE>
__global__ void __launch_bounds__(256) probe(const long long* __restrict__ key, const long long* __restrict__ val,
                                             const long long* __restrict__ ts, long long n, unsigned long long K,
                                             unsigned long long* acc, const ulonglong2* dict, uint32_t dmask,
                                             unsigned long long* sink) {
  long long i = ((long long)blockIdx.x * blockDim.x + threadIdx.x) * 2;
  long long stride = (long long)gridDim.x * blockDim.x * 2;
  unsigned long long s = 0;
  for (; i + 1 < n; i += stride) {
    longlong2 k2 = __ldcs((const longlong2*)(key + i));
    longlong2 v2 = __ldcs((const longlong2*)(val + i));
    longlong2 t2 = __ldcs((const longlong2*)(ts + i));
    long long kk[2] = {k2.x, k2.y}, vv[2] = {v2.x, v2.y}, tt[2] = {t2.x, t2.y};
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      uint64_t id = (uint64_t)kk[j];
      if (MODE & 8) {
        uint32_t pos = (uint32_t)mix64((uint64_t)kk[j]) & dmask;
        ulonglong2 sl = __ldcg(dict + pos);
        while ((long long)sl.x != kk[j]) { pos = (pos + 1) & dmask; sl = __ldcg(dict + pos); }
        id = (uint32_t)sl.y;
      }
      s += tt[j] & 1;
      if (MODE & 64) { s += id + vv[j]; continue; }
      if (MODE & 32) {
        unsigned long long* b = acc + id * 4;
        if (MODE & 1) atomicAdd(b, 1ull);
        if (MODE & 2) atomicAdd(b + 1, (unsigned long long)vv[j]);
        if (MODE & 4) atomicAdd((double*)(b + 2), (double)vv[j]);
      } else {
        if (MODE & 1) { if (MODE & 16) atomicAdd((unsigned int*)acc + id, 1u); else atomicAdd(acc + id, 1ull); }
        if (MODE & 2) atomicAdd(acc + K + id, (unsigned long long)vv[j]);
        if (MODE & 4) atomicAdd((double*)(acc + 2 * K + id), (double)vv[j]);
      }
    }
  }
  if (s == 0x123456789ull) *sink = s;
}

template <int MODE>
float run(const char* name, const long long* k, const long long* v, const long long* t, long long n, unsigned long long K,
          unsigned long long* acc, const ulonglong2* dict, uint32_t dmask, unsigned long long* sink, int reps) {
  cudaEvent_t e0, e1; CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
  int grid = 132 * 8;
  for (int w = 0; w < 2; ++w) probe<MODE><<<grid, 256>>>(k, v, t, n, K, acc, dict, dmask, sink);
  CK(cudaDeviceSynchronize());
  CK(cudaEventRecord(e0));
  for (int r = 0; r < reps; ++r) probe<MODE><<<grid, 256>>>(k, v, t, n, K, acc, dict, dmask, sink);
  CK(cudaEventRecord(e1)); CK(cudaEventSynchronize(e1));
  float ms; CK(cudaEventElapsedTime(&ms, e0, e1)); ms /= reps;
  printf("%-44s K=%8llu  %8.3f ms  %7.2f Grows/s  %7.1f GB/s(24B/row)\n", name, K, ms, n / ms / 1e6, n * 24.0 / ms / 1e6);
  return ms;
}

int main(int argc, char** argv) {
  long long n = 1ll << 24;  // one pane of the headline config
  int reps = 5;
  long long *k, *v, *t; unsigned long long *acc, *sink; ulonglong2* dict;
  CK(cudaMalloc(&k, n * 8)); CK(cudaMalloc(&v, n * 8)); CK(cudaMalloc(&t, n * 8)); CK(cudaMalloc(&sink, 8));
  for (unsigned long long K : {1ull << 14, 1ull << 20, 1ull << 23}) {
    std::vector<long long> hk(n), hv(n), ht(n);
    uint64_t st = 42;
    for (long long i = 0; i < n; ++i) { st = mix64(st + i); hk[i] = (long long)(st % K); hv[i] = (long long)((st >> 20) % 100000000); ht[i] = 1700000000000000000ll + i * 59; }
    CK(cudaMemcpy(k, hk.data(), n * 8, cudaMemcpyHostToDevice)); CK(cudaMemcpy(v, hv.data(), n * 8, cudaMemcpyHostToDevice)); CK(cudaMemcpy(t, ht.data(), n * 8, cudaMemcpyHostToDevice));
    CK(cudaMalloc(&acc, K * 4 * 8)); CK(cudaMemset(acc, 0, K * 4 * 8));
    uint32_t dcap = 1; while (dcap < 4 * K) dcap <<= 1;  // load 0.25..0.5
    dcap >>= 1;
    std::vector<ulonglong2> hd(dcap, ulonglong2{0x8000000000000000ull, 0xffffffffull});
    for (unsigned long long key = 0; key < K; ++key) { uint32_t pos = (uint32_t)mix64(key) & (dcap - 1); while (hd[pos].x != 0x8000000000000000ull) pos = (pos + 1) & (dcap - 1); hd[pos].x = key; hd[pos].y = key; }
    CK(cudaMalloc(&dict, (size_t)dcap * 16)); CK(cudaMemcpy(dict, hd.data(), (size_t)dcap * 16, cudaMemcpyHostToDevice));
    run<64>("loads only (stream 24 B/row)", k, v, t, n, K, acc, dict, dcap - 1, sink, reps);
    run<64 | 8>("loads + dict probe", k, v, t, n, K, acc, dict, dcap - 1, sink, reps);
    run<1>("RED rows(u64)", k, v, t, n, K, acc, dict, dcap - 1, sink, reps);
    run<1 | 16>("RED rows(u32)", k, v, t, n, K, acc, dict, dcap - 1, sink, reps);
    run<1 | 2>("RED rows+sum", k, v, t, n, K, acc, dict, dcap - 1, sink, reps);
    run<1 | 2 | 4>("RED rows+sum+f64", k, v, t, n, K, acc, dict, dcap - 1, sink, reps);
    run<1 | 2 | 4 | 32>("RED rows+sum+f64 AoS(32B)", k, v, t, n, K, acc, dict, dcap - 1, sink, reps);
    run<1 | 2 | 4 | 8>("probe + RED rows+sum+f64", k, v, t, n, K, acc, dict, dcap - 1, sink, reps);
    run<1 | 2 | 8>("probe + RED rows+sum", k, v, t, n, K, acc, dict, dcap - 1, sink, reps);
    run<1 | 2 | 4 | 8 | 32>("probe + RED rows+sum+f64 AoS", k, v, t, n, K, acc, dict, dcap - 1, sink, reps);
    CK(cudaFree(acc)); CK(cudaFree(dict));
  }
  return 0;
}
