// Validity of a nullable output column: one byte per row on the device, exported as an Arrow validity bitmap (the
// joins' nullable sides, the window function's LAG / LEAD / NTH_VALUE).
#pragma once

#include "arrow_io.h"
#include "common.cuh"

namespace ab {

// validity bytes -> Arrow validity bitmap (LSB first)
static __global__ void pack_bits_kernel(const unsigned char* __restrict__ bytes, long long n, unsigned int* __restrict__ words) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  long long n_pad = (n + 31) / 32 * 32;
  long long stride = (long long)gridDim.x * blockDim.x;
  for (; i < n_pad; i += stride) {
    bool v = i < n && bytes[i];
    unsigned int b = __ballot_sync(0xffffffffu, v);
    if ((threadIdx.x & 31) == 0) words[i >> 5] = b;
  }
}

// Gives `col` the validity of its `n` rows from the device bytes `bytes`: packed into `words` ((n + 31) / 32 of them)
// by `grid` blocks of `threads` on `s`, copied to a pinned buffer and counted.  The call waits for `s`, so `words` may
// be reused as soon as it returns.  With no NULL row the column carries no bitmap.
inline void export_validity(OutColumn& col, const unsigned char* bytes, int64_t n, unsigned int* words, int grid,
                            int threads, cudaStream_t s, ArroyoB200Stats& st) {
  const size_t n_words = (size_t)((n + 31) / 32);
  pack_bits_kernel<<<grid, threads, 0, s>>>(bytes, n, words);
  AB_CUDA(cudaGetLastError());
  ++st.kernel_launches;
  col.validity = d2h_pinned(words, n_words * 4, s, &st.d2h_bytes);
  AB_CUDA(cudaStreamSynchronize(s));
  const unsigned int* w = (const unsigned int*)col.validity;
  int64_t set = 0;
  for (size_t i = 0; i < n_words; ++i) set += __builtin_popcount(w[i]);
  col.null_count = n - set;
  col.nullable = true;
  if (col.null_count == 0) {
    PinnedPool::get().free(col.validity);
    col.validity = nullptr;
  }
}

}  // namespace ab
