// Micro-probe 2 (not product code): what limits the random 16-byte dictionary probe on an H100, and which
// issue pattern gets the most probes in flight?  Variants: rows per thread (MLP), ldcg vs ldg(nc) vs
// cp.async-to-shared, threads per block.
#include <cuda_runtime.h>
#include <cstdio>
#include <cstdlib>
#include <cstdint>
#include <vector>
#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("CUDA %s at %d\n", cudaGetErrorString(e), __LINE__); exit(1);} } while (0)
__host__ __device__ inline uint64_t mix64(uint64_t x) {
  uint64_t z = x + 0x9E3779B97F4A7C15ull; z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull; z = (z ^ (z >> 27)) * 0x94D049BB133111EBull; return z ^ (z >> 31);
}
// LOAD: 0 = ldcg, 1 = ldg (nc), 2 = cp.async.cg -> smem
template <int RPT, int LOAD, int RED>
__global__ void probe(const long long* __restrict__ key, const long long* __restrict__ val, long long n,
                      const ulonglong2* __restrict__ dict, uint32_t dmask, unsigned long long* acc, unsigned long long K,
                      unsigned long long* sink) {
  extern __shared__ ulonglong2 s_buf[];
  const long long tile = (long long)blockDim.x * RPT;
  unsigned long long s = 0;
  for (long long base = (long long)blockIdx.x * tile; base + tile <= n; base += (long long)gridDim.x * tile) {
    long long k[RPT], v[RPT]; uint32_t pos[RPT]; ulonglong2 sl[RPT];
#pragma unroll
    for (int j = 0; j < RPT; ++j) { k[j] = __ldcs(key + base + j * blockDim.x + threadIdx.x); if (RED) v[j] = __ldcs(val + base + j * blockDim.x + threadIdx.x); }
#pragma unroll
    for (int j = 0; j < RPT; ++j) pos[j] = (uint32_t)mix64((uint64_t)k[j]) & dmask;
    if (LOAD == 2) {
#pragma unroll
      for (int j = 0; j < RPT; ++j) {
        unsigned sa = (unsigned)__cvta_generic_to_shared(&s_buf[j * blockDim.x + threadIdx.x]);
        asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(sa), "l"(dict + pos[j]));
      }
      asm volatile("cp.async.commit_group;\ncp.async.wait_group 0;" ::: "memory");
#pragma unroll
      for (int j = 0; j < RPT; ++j) sl[j] = s_buf[j * blockDim.x + threadIdx.x];
    } else {
#pragma unroll
      for (int j = 0; j < RPT; ++j) sl[j] = LOAD == 0 ? __ldcg(dict + pos[j]) : __ldg(dict + pos[j]);
    }
#pragma unroll
    for (int j = 0; j < RPT; ++j) {
      while ((long long)sl[j].x != k[j]) { pos[j] = (pos[j] + 1) & dmask; sl[j] = __ldcg(dict + pos[j]); }
      uint32_t id = (uint32_t)sl[j].y;
      if (RED) { atomicAdd(acc + id, 1ull); atomicAdd(acc + K + id, (unsigned long long)v[j]); }
      else s += id;
    }
  }
  if (s == 0x123456789ull) *sink = s;
}
template <int RPT, int LOAD, int RED>
void run(const char* name, int threads, const long long* k, const long long* v, long long n, const ulonglong2* d, uint32_t dm,
         unsigned long long* acc, unsigned long long K, unsigned long long* sink) {
  cudaEvent_t e0, e1; CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
  size_t smem = LOAD == 2 ? (size_t)threads * RPT * 16 : 0;
  if (smem > 48 * 1024) CK(cudaFuncSetAttribute(probe<RPT, LOAD, RED>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  int occ = 0; CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, probe<RPT, LOAD, RED>, threads, smem));
  int grid = 132 * (occ > 0 ? occ : 1);
  for (int w = 0; w < 2; ++w) probe<RPT, LOAD, RED><<<grid, threads, smem>>>(k, v, n, d, dm, acc, K, sink);
  CK(cudaDeviceSynchronize());
  CK(cudaEventRecord(e0));
  for (int r = 0; r < 5; ++r) probe<RPT, LOAD, RED><<<grid, threads, smem>>>(k, v, n, d, dm, acc, K, sink);
  CK(cudaEventRecord(e1)); CK(cudaEventSynchronize(e1));
  float ms; CK(cudaEventElapsedTime(&ms, e0, e1)); ms /= 5;
  printf("%-28s rpt=%d thr=%4d occ=%2d  %7.3f ms  %7.2f Grows/s\n", name, RPT, threads, occ, ms, n / ms / 1e6);
}
int main() {
  long long n = 1ll << 24; unsigned long long K = 1ull << 20;
  long long *k, *v; unsigned long long *acc, *sink; ulonglong2* dict;
  CK(cudaMalloc(&k, n * 8)); CK(cudaMalloc(&v, n * 8)); CK(cudaMalloc(&sink, 8));
  std::vector<long long> hk(n), hv(n); uint64_t st = 42;
  for (long long i = 0; i < n; ++i) { st = mix64(st + i); hk[i] = (long long)(st % K); hv[i] = (long long)((st >> 20) % 100000000); }
  CK(cudaMemcpy(k, hk.data(), n * 8, cudaMemcpyHostToDevice)); CK(cudaMemcpy(v, hv.data(), n * 8, cudaMemcpyHostToDevice));
  CK(cudaMalloc(&acc, K * 4 * 8)); CK(cudaMemset(acc, 0, K * 4 * 8));
  for (uint32_t dcap : {1u << 21, 1u << 22}) {
    std::vector<ulonglong2> hd(dcap, ulonglong2{0x8000000000000000ull, 0xffffffffull});
    for (unsigned long long key = 0; key < K; ++key) { uint32_t pos = (uint32_t)mix64(key) & (dcap - 1); while (hd[pos].x != 0x8000000000000000ull) pos = (pos + 1) & (dcap - 1); hd[pos].x = key; hd[pos].y = key; }
    CK(cudaMalloc(&dict, (size_t)dcap * 16)); CK(cudaMemcpy(dict, hd.data(), (size_t)dcap * 16, cudaMemcpyHostToDevice));
    printf("---- dict slots %u (load %.2f) ----\n", dcap, (double)K / dcap);
#define R(RPT, LOAD, RED, THR, NAME) run<RPT, LOAD, RED>(NAME, THR, k, v, n, dict, dcap - 1, acc, K, sink)
    R(1, 0, 0, 256, "ldcg probe only"); R(2, 0, 0, 256, "ldcg probe only"); R(4, 0, 0, 256, "ldcg probe only"); R(8, 0, 0, 256, "ldcg probe only");
    R(4, 0, 0, 512, "ldcg probe only"); R(4, 0, 0, 1024, "ldcg probe only"); R(2, 0, 0, 128, "ldcg probe only");
    R(2, 1, 0, 256, "ldg(nc) probe only"); R(4, 1, 0, 256, "ldg(nc) probe only"); R(8, 1, 0, 256, "ldg(nc) probe only");
    R(2, 2, 0, 256, "cp.async probe only"); R(4, 2, 0, 256, "cp.async probe only"); R(8, 2, 0, 256, "cp.async probe only"); R(16, 2, 0, 256, "cp.async probe only");
    R(2, 0, 1, 256, "ldcg probe + 2 RED"); R(4, 0, 1, 256, "ldcg probe + 2 RED"); R(8, 0, 1, 256, "ldcg probe + 2 RED");
    R(4, 1, 1, 256, "ldg(nc) probe + 2 RED"); R(4, 2, 1, 256, "cp.async probe + 2 RED"); R(8, 2, 1, 256, "cp.async probe + 2 RED");
    CK(cudaFree(dict));
  }
  return 0;
}
