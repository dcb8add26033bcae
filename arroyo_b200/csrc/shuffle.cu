// Key-hash shuffle partitioner on sm_90a (H100): the device half of the Shuffle edge.
//
// Replaces ArrowCollector::collect -> repartition (arroyo-operator/src/context.rs:506-541) and
// server_for_hash_array (arroyo-operator/src/lib.rs:30-41): hash the routing key, dest =
// (hash / (u64::MAX / n)) % n, bucket rows per destination.  The reference sorts the whole batch by
// destination and gathers every column (K2/K6); here it is histogram -> scan -> scatter, and the
// per-destination segments are the send buffers of the NCCL all-to-all.
#include <climits>

#include "common.cuh"

namespace ab {
namespace {

constexpr int PT_THREADS = 256;
constexpr int PT_ROWS = 2048;  // rows per block
constexpr int MAX_DEST = 256;
constexpr int MAX_PCOLS = ARROYO_B200_MAX_COLS;

__device__ __forceinline__ uint32_t dest_of(long long key, uint64_t range, uint32_t n_dest) {
  return (uint32_t)((mix64((uint64_t)key) / range) % n_dest);
}

__global__ void __launch_bounds__(PT_THREADS) hist_kernel(const long long* __restrict__ key, long long n,
                                                          uint64_t range, uint32_t n_dest,
                                                          unsigned int* __restrict__ block_hist) {
  __shared__ unsigned int s_hist[MAX_DEST];
  for (int i = threadIdx.x; i < (int)n_dest; i += PT_THREADS) s_hist[i] = 0;
  __syncthreads();
  const long long base = (long long)blockIdx.x * PT_ROWS;
  for (int i = threadIdx.x; i < PT_ROWS; i += PT_THREADS) {
    long long r = base + i;
    if (r < n) atomicAdd(&s_hist[dest_of(__ldcs(key + r), range, n_dest)], 1u);
  }
  __syncthreads();
  for (int i = threadIdx.x; i < (int)n_dest; i += PT_THREADS)
    block_hist[(size_t)i * gridDim.x + blockIdx.x] = s_hist[i];  // dest-major
}

// One warp per destination: exclusive scan of that destination's per-block counts; then the
// destination bases.  block_hist is overwritten with per-(dest, block) start offsets relative to
// the destination's segment; counts/offsets (int64) receive the segment sizes and starts.
__global__ void scan_kernel(unsigned int* __restrict__ block_hist, uint32_t n_blocks, uint32_t n_dest,
                            long long* __restrict__ counts, long long* __restrict__ offsets) {
  __shared__ long long s_total[MAX_DEST];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int n_warps = blockDim.x >> 5;
  for (uint32_t d = warp; d < n_dest; d += n_warps) {
    unsigned int* h = block_hist + (size_t)d * n_blocks;
    unsigned long long carry = 0;
    for (uint32_t b0 = 0; b0 < n_blocks; b0 += 32) {
      uint32_t b = b0 + lane;
      unsigned int v = b < n_blocks ? h[b] : 0u;
      unsigned int x = v;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        unsigned int y = __shfl_up_sync(0xffffffffu, x, o);
        if (lane >= o) x += y;
      }
      if (b < n_blocks) h[b] = (unsigned int)(carry + x - v);
      carry += __shfl_sync(0xffffffffu, x, 31);
    }
    if (lane == 0) s_total[d] = (long long)carry;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    long long off = 0;
    for (uint32_t d = 0; d < n_dest; ++d) {
      counts[d] = s_total[d];
      offsets[d] = off;
      off += s_total[d];
    }
  }
}

// WatermarkGenerator::process_batch (arroyo-worker/src/arrow/watermark_generator.rs:150-197): the two
// reductions it runs on every batch -- max(_timestamp) and min(_timestamp) (the watermark expression is
// `_timestamp - delay`, so its minimum is min(_timestamp) - delay).
__global__ void __launch_bounds__(256) minmax_kernel(const long long* __restrict__ ts, long long n,
                                                     long long* __restrict__ out /* [min, max] */) {
  long long mn = LLONG_MAX, mx = LLONG_MIN;
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (; i < n; i += stride) {
    const long long t = __ldcs(ts + i);
    mn = min(mn, t);
    mx = max(mx, t);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    mn = min(mn, __shfl_xor_sync(0xffffffffu, mn, o));
    mx = max(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  }
  if ((threadIdx.x & 31) == 0 && mn != LLONG_MAX) {
    atomicMin(out, mn);
    atomicMax(out + 1, mx);
  }
}

struct ScatterParams {
  const long long* in[MAX_PCOLS];
  long long* out[MAX_PCOLS];
  int n_cols;
  int key_col;
  long long n;
  uint64_t range;
  uint32_t n_dest;
  const unsigned int* block_off;
  const long long* offsets;
  // packed layout (one all-to-all instead of one per column): destination d owns the element range
  // [n_cols * offsets[d], n_cols * (offsets[d] + counts[d])) of `packed`, its columns back to back
  long long* packed;
  const long long* counts;
};

__global__ void __launch_bounds__(PT_THREADS) scatter_kernel(const __grid_constant__ ScatterParams p) {
  __shared__ unsigned int s_cursor[MAX_DEST];
  __shared__ long long s_base[MAX_DEST];
  __shared__ long long s_count[MAX_DEST];
  for (int i = threadIdx.x; i < (int)p.n_dest; i += PT_THREADS) {
    s_cursor[i] = 0;
    const long long in_seg = (long long)p.block_off[(size_t)i * gridDim.x + blockIdx.x];
    if (p.packed) {
      s_base[i] = (long long)p.n_cols * p.offsets[i] + in_seg;
      s_count[i] = p.counts[i];
    } else {
      s_base[i] = p.offsets[i] + in_seg;
    }
  }
  __syncthreads();
  const long long base = (long long)blockIdx.x * PT_ROWS;
  for (int i = threadIdx.x; i < PT_ROWS; i += PT_THREADS) {
    long long r = base + i;
    if (r < p.n) {
      uint32_t d = dest_of(__ldcs(p.in[p.key_col] + r), p.range, p.n_dest);
      long long o = s_base[d] + (long long)atomicAdd(&s_cursor[d], 1u);
      if (p.packed) {
        const long long stride = s_count[d];
#pragma unroll 4
        for (int c = 0; c < p.n_cols; ++c) p.packed[o + c * stride] = __ldcs(p.in[c] + r);
      } else {
#pragma unroll 4
        for (int c = 0; c < p.n_cols; ++c) p.out[c][o] = __ldcs(p.in[c] + r);
      }
    }
  }
}

}  // namespace
}  // namespace ab

using namespace ab;

struct ArroyoB200Partitioner {
  int device;
  cudaStream_t stream;
  bool own_stream;
  int n_dest, n_cols, key_col;
  int64_t max_rows;
  DevBuf hist;
};

extern "C" {

int32_t arroyo_b200_ts_minmax(int32_t device, uint64_t stream, uint64_t ts_dev, int64_t n_rows, int64_t* out_min,
                               int64_t* out_max) {
  if (!ts_dev || n_rows < 0 || !out_min || !out_max) return ARROYO_B200_INVALID_ARGUMENT;
  try {
    AB_CUDA(cudaSetDevice(device));
    static thread_local long long* d_out = nullptr;
    static thread_local int d_dev = -1;
    static thread_local int d_sms = 0;
    if (!d_out || d_dev != device) {
      AB_CUDA(cudaMalloc(&d_out, 2 * sizeof(long long)));
      AB_CUDA(cudaDeviceGetAttribute(&d_sms, cudaDevAttrMultiProcessorCount, device));
      d_dev = device;
    }
    cudaStream_t st = (cudaStream_t)stream;
    const long long init[2] = {LLONG_MAX, LLONG_MIN};
    AB_CUDA(cudaMemcpyAsync(d_out, init, sizeof init, cudaMemcpyHostToDevice, st));
    if (n_rows > 0) {
      int grid = (int)std::min<int64_t>((n_rows + 255) / 256, (int64_t)d_sms * 8);
      minmax_kernel<<<grid, 256, 0, st>>>((const long long*)ts_dev, n_rows, d_out);
      AB_CUDA(cudaGetLastError());
    }
    long long h[2];
    AB_CUDA(cudaMemcpyAsync(h, d_out, sizeof h, cudaMemcpyDeviceToHost, st));
    AB_CUDA(cudaStreamSynchronize(st));
    *out_min = h[0];
    *out_max = h[1];
    return ARROYO_B200_OK;
  } catch (const Error& e) {
    return e.status;
  } catch (...) {
    return ARROYO_B200_RUNTIME;
  }
}

int32_t arroyo_b200_partitioner_create(int32_t device, uint64_t stream, int32_t n_dest, int32_t n_cols,
                                       int32_t key_col, int64_t max_rows, ArroyoB200Partitioner** out) {
  if (!out) return ARROYO_B200_INVALID_ARGUMENT;
  *out = nullptr;
  if (n_dest < 1 || n_dest > MAX_DEST || n_cols < 1 || n_cols > MAX_PCOLS || key_col < 0 || key_col >= n_cols ||
      max_rows < 1)
    return ARROYO_B200_INVALID_ARGUMENT;
  try {
    int count = 0;
    if (cudaGetDeviceCount(&count) != cudaSuccess || device < 0 || device >= count) {
      cudaGetLastError();
      return ARROYO_B200_FATAL;
    }
    AB_CUDA(cudaSetDevice(device));
    auto* p = new ArroyoB200Partitioner();
    p->device = device;
    p->n_dest = n_dest;
    p->n_cols = n_cols;
    p->key_col = key_col;
    p->max_rows = max_rows;
    if (stream) {
      p->stream = (cudaStream_t)stream;
      p->own_stream = false;
    } else {
      AB_CUDA(cudaStreamCreateWithFlags(&p->stream, cudaStreamNonBlocking));
      p->own_stream = true;
    }
    size_t n_blocks = (size_t)((max_rows + PT_ROWS - 1) / PT_ROWS);
    p->hist.alloc(n_blocks * (size_t)n_dest * sizeof(unsigned int));
    *out = p;
    return ARROYO_B200_OK;
  } catch (const Error& e) {
    return e.status;
  } catch (...) {
    return ARROYO_B200_RUNTIME;
  }
}

void arroyo_b200_partitioner_destroy(ArroyoB200Partitioner* p) {
  if (!p) return;
  cudaSetDevice(p->device);
  cudaStreamSynchronize(p->stream);
  if (p->own_stream) cudaStreamDestroy(p->stream);
  delete p;
}

static int32_t partition_impl(ArroyoB200Partitioner* p, const uint64_t* in_cols, int64_t n_rows,
                              const uint64_t* out_cols, uint64_t packed_dev, uint64_t counts_dev,
                              uint64_t offsets_dev) {
  if (!p || !in_cols || (!out_cols && !packed_dev) || !counts_dev || !offsets_dev || n_rows < 0 ||
      n_rows > p->max_rows)
    return ARROYO_B200_INVALID_ARGUMENT;
  try {
    AB_CUDA(cudaSetDevice(p->device));
    const uint32_t n_blocks = (uint32_t)std::max<int64_t>((n_rows + PT_ROWS - 1) / PT_ROWS, 1);
    const uint64_t range = UINT64_MAX / (uint64_t)p->n_dest;
    hist_kernel<<<n_blocks, PT_THREADS, 0, p->stream>>>((const long long*)in_cols[p->key_col], n_rows, range,
                                                        (uint32_t)p->n_dest, p->hist.as<unsigned int>());
    AB_CUDA(cudaGetLastError());
    scan_kernel<<<1, 1024, 0, p->stream>>>(p->hist.as<unsigned int>(), n_blocks, (uint32_t)p->n_dest,
                                           (long long*)counts_dev, (long long*)offsets_dev);
    AB_CUDA(cudaGetLastError());
    ScatterParams sp{};
    for (int c = 0; c < p->n_cols; ++c) {
      sp.in[c] = (const long long*)in_cols[c];
      sp.out[c] = out_cols ? (long long*)out_cols[c] : nullptr;
    }
    sp.packed = (long long*)packed_dev;
    sp.counts = (const long long*)counts_dev;
    sp.n_cols = p->n_cols;
    sp.key_col = p->key_col;
    sp.n = n_rows;
    sp.range = range;
    sp.n_dest = (uint32_t)p->n_dest;
    sp.block_off = p->hist.as<unsigned int>();
    sp.offsets = (const long long*)offsets_dev;
    scatter_kernel<<<n_blocks, PT_THREADS, 0, p->stream>>>(sp);
    AB_CUDA(cudaGetLastError());
    return ARROYO_B200_OK;
  } catch (const Error& e) {
    return e.status;
  } catch (...) {
    return ARROYO_B200_RUNTIME;
  }
}

int32_t arroyo_b200_partition(ArroyoB200Partitioner* p, const uint64_t* in_cols, int64_t n_rows,
                              const uint64_t* out_cols, uint64_t counts_dev, uint64_t offsets_dev) {
  if (!out_cols) return ARROYO_B200_INVALID_ARGUMENT;
  return partition_impl(p, in_cols, n_rows, out_cols, 0, counts_dev, offsets_dev);
}

int32_t arroyo_b200_partition_packed(ArroyoB200Partitioner* p, const uint64_t* in_cols, int64_t n_rows,
                                     uint64_t packed_dev, uint64_t counts_dev, uint64_t offsets_dev) {
  if (!packed_dev) return ARROYO_B200_INVALID_ARGUMENT;
  return partition_impl(p, in_cols, n_rows, nullptr, packed_dev, counts_dev, offsets_dev);
}

}  // extern "C"
