// Window function on sm_90a (H100): the GPU side of `WindowFunctionOperator` (arroyo-worker/src/arrow/window_fn.rs),
// for ROW_NUMBER / RANK / DENSE_RANK () OVER (PARTITION BY window [, key] ORDER BY k1 [DESC], ...), optionally fused
// with the `WHERE fn <= N` that usually follows it (top N per window), for COUNT(*) / SUM / AVG / MIN / MAX (x)
// OVER (PARTITION BY window [, key] [ORDER BY ...]) over the default frame or an explicit ROWS / RANGE / GROUPS frame,
// and for LAG / LEAD / FIRST_VALUE / LAST_VALUE / NTH_VALUE (x, ...) and PERCENT_RANK / CUME_DIST () over the same
// partitions (FIRST_VALUE / LAST_VALUE / NTH_VALUE over an explicit frame too).  The planner
// (plan/window_fn.rs:101-105) drops the `window` column from PARTITION BY: each upstream window stamps its rows with one
// `_timestamp`, so the rows are bucketed by `_timestamp` ("instant") and the remaining PARTITION BY column, if any,
// splits each instant further.
//
//   store   every accepted row, SoA, one 64-bit array per flat input column; a row's index is its arrival sequence.
//           The host doubles the store before a launch that could overfill it, from the rows it has handed over since
//           it last read the row count;
//   ingest  per launch: flag the rows that stay (ts >= the last watermark, filter_by_time in arroyo-rpc/src/df.rs:
//           211-231; a negative ts is reported, the reference panics on it), device_exclusive_scan, append them in
//           order behind the stored rows;
//   emit    at watermark w every instant < w leaves (window_fn.rs:178-201): flag and compact the indices of the rows
//           with ts < w, then stable LSD radix passes (CUB) starting from arrival order: the ORDER BY keys last to
//           first, the partition key, `_timestamp`.  Each key is sorted in an unsigned order-preserving form (sign bit
//           flipped for signed types, all bits complemented for DESC).  A rank pass flags segment starts (instant,
//           partition) and peer starts (every sort key) and scans them, ballots within a warp and a two-level scan
//           across 1024-row tiles: ROW_NUMBER = position in the segment + 1, RANK = position of the first peer + 1,
//           DENSE_RANK = peer starts in the segment so far.  An aggregate adds a segmented scan of its argument with the
//           same tiling, read at each peer group's last row (see "aggregates" below); the other functions add index
//           arithmetic on the rank scan and a read of the argument (see "value functions" below).  The fused filter, a
//           compaction and a gather of every column write the output in sorted order; the rows that stay are compacted
//           to the front of the store, in arrival order, so device memory tracks the open rows;
//   state   table "input": a checkpoint writes the rows accepted since the previous one (one store index marks them,
//           re-based when the store is compacted), one batch per instant, in the input layout.  on_start appends the
//           restored rows first and does not late-filter them, as the reference re-feeds them (:130-145).
// Rows that tie on every sort key leave in arrival order, restored rows first; DataFusion's sort promises no order
// there, and RANK and DENSE_RANK do not depend on it.  Output rows of one emission leave in one batch (the reference
// emits one batch per instant; the rows and their order are the same).  Device-resident output is refused.
#include <algorithm>
#include <climits>
#include <functional>

#include <cub/device/device_radix_sort.cuh>

#include "op.h"
#include "scan.cuh"
#include "validity.cuh"

namespace ab {
namespace {

constexpr int WF_THREADS = 256;
constexpr int WF_TILE = 1024;  // rows per rank tile: one per thread, 32 warps
constexpr unsigned FULL = 0xffffffffu;
constexpr uint64_t WF_MAX_ROWS = 1ull << 31;
constexpr int MAX_SORT_COLS = 2 + ARROYO_B200_MAX_ORDER_KEYS;  // _timestamp, the partition key, the ORDER BY keys

struct WCounters {
  unsigned long long n_store;  // rows in the store
  unsigned long long late;
  unsigned long long total;     // scan total
  unsigned long long instants;  // instants of the last emission
  unsigned int neg_ts;          // a row with a negative _timestamp arrived
  unsigned int pad;
};

struct WCols {
  unsigned long long* c[ARROYO_B200_MAX_COLS];
};

// flag[i] = row i of a launch stays: ts >= late_wm (LLONG_MIN: no watermark yet) and ts >= 0.  Counts late rows and
// notes negative timestamps.  The loop bound is uniform per warp, so every lane reaches the warp reduction.
__global__ void __launch_bounds__(WF_THREADS) wf_flag_kernel(const long long* __restrict__ ts, long long n,
                                                             long long late_wm, unsigned int* __restrict__ flag,
                                                             WCounters* counters) {
  const unsigned lane = threadIdx.x & 31;
  const long long stride = (long long)gridDim.x * blockDim.x;
  unsigned int late = 0;
  bool neg = false;
  for (long long row0 = (long long)blockIdx.x * blockDim.x + (threadIdx.x & ~31u); row0 < n; row0 += stride) {
    const long long i = row0 + lane;
    if (i >= n) continue;
    const long long t = __ldcs(ts + i);
    neg |= t < 0;
    late += (t >= 0 && t < late_wm) ? 1u : 0u;
    flag[i] = (t >= 0 && t >= late_wm) ? 1u : 0u;
  }
  const unsigned int wl = __reduce_add_sync(FULL, late);
  if (lane == 0 && wl) atomicAdd(&counters->late, (unsigned long long)wl);
  if (neg) counters->neg_ts = 1u;
}

// The flagged rows of a launch, appended in order behind the `*n_store` stored rows.
struct WAppend {
  const unsigned long long* in[ARROYO_B200_MAX_COLS];
  WCols store;
  int n_cols;
  const unsigned int* flag;
  const unsigned long long* off;
  long long n;
  const unsigned long long* n_store;
};
__global__ void __launch_bounds__(WF_THREADS) wf_append_kernel(const __grid_constant__ WAppend p) {
  const unsigned long long base = *p.n_store;
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (; i < p.n; i += stride) {
    if (!p.flag[i]) continue;
    const unsigned long long d = base + p.off[i];
    for (int c = 0; c < p.n_cols; ++c) p.store.c[c][d] = __ldcs(p.in[c] + i);
  }
}

// *n_store += the launch's scan total (a kernel of its own: every thread of the append reads the old count)
__global__ void wf_advance_kernel(WCounters* c) { c->n_store += c->total; }
__global__ void wf_set_rows_kernel(WCounters* c, unsigned long long n) { c->n_store = n; }

// flag[i] = stored row i leaves at watermark w
__global__ void wf_mark_kernel(const long long* __restrict__ ts, long long n, long long w, unsigned int* __restrict__ flag) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (; i < n; i += stride) flag[i] = ts[i] < w ? 1u : 0u;
}

// the flagged rows' store indices, compacted in arrival order
__global__ void wf_select_kernel(const unsigned int* __restrict__ flag, const unsigned long long* __restrict__ off,
                                 long long n, unsigned int* __restrict__ idx) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (; i < n; i += stride)
    if (flag[i]) idx[off[i]] = (unsigned int)i;
}

__global__ void wf_iota_kernel(unsigned int* __restrict__ idx, unsigned int first, long long n) {
  long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (; j < n; j += stride) idx[j] = first + (unsigned int)j;
}

// k[j] = the sort key of row idx[j] in its unsigned order-preserving form: col ^ flip
__global__ void wf_key_kernel(const unsigned long long* __restrict__ col, const unsigned int* __restrict__ idx, long long n,
                              unsigned long long flip, unsigned long long* __restrict__ k) {
  long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (; j < n; j += stride) k[j] = col[idx[j]] ^ flip;
}

// ---- ranks ------------------------------------------------------------------------------------------------------------
// The scan that turns the segment and peer starts of the sorted rows into ranks.  An element is row j's
// {seg = j + 1 if a segment starts there else 0, peer = the same for a peer group, dcnt = 1 if a peer group starts there};
// over a range, seg / peer are the last starts in it and dcnt counts the peer starts from its last segment start on (all
// of them when none starts in it).  A segment start is always a peer start.
struct RankVal {
  unsigned int seg, peer, dcnt;
  __device__ static RankVal zero() { return {0u, 0u, 0u}; }
};
__device__ __forceinline__ RankVal combine(RankVal a, RankVal b) {
  return {b.seg ? b.seg : a.seg, b.peer ? b.peer : a.peer, b.seg ? b.dcnt : a.dcnt + b.dcnt};
}
__device__ __forceinline__ RankVal shfl_up(RankVal v, int o) {
  return {__shfl_up_sync(FULL, v.seg, o), __shfl_up_sync(FULL, v.peer, o), __shfl_up_sync(FULL, v.dcnt, o)};
}

// Inclusive scan of one tile of WF_TILE rows (one per thread, `bits`: 2 = segment start, 4 = peer start), positions
// from `j` of the calling thread; the tile's total goes to `*total`.  Within a warp the starts are two ballots: the last
// start at or below a lane is the highest set bit of its ballot prefix.  Every thread of the block calls it.
__device__ __forceinline__ RankVal tile_inclusive(unsigned int bits, long long j, RankVal* total) {
  __shared__ RankVal s_warp[WF_TILE / 32];
  const unsigned lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const unsigned sb = __ballot_sync(FULL, bits & 2u), pb = __ballot_sync(FULL, bits & 4u);
  const unsigned le = lane == 31 ? FULL : (2u << lane) - 1u;
  const unsigned s = sb & le, p = pb & le;
  const long long lane0 = j - (long long)lane;
  RankVal v;
  v.seg = s ? (unsigned int)(lane0 + (31 - __clz(s))) + 1u : 0u;
  v.peer = p ? (unsigned int)(lane0 + (31 - __clz(p))) + 1u : 0u;
  v.dcnt = s ? (unsigned int)__popc(p & ~((1u << (31 - __clz(s))) - 1u)) : (unsigned int)__popc(p);
  if (lane == 31) s_warp[w] = v;
  __syncthreads();
  if (w == 0) {
    RankVal x = s_warp[lane];
    for (int o = 1; o < 32; o <<= 1) {
      const RankVal y = shfl_up(x, o);
      if ((int)lane >= o) x = combine(y, x);
    }
    s_warp[lane] = x;
  }
  __syncthreads();
  if (w > 0) v = combine(s_warp[w - 1], v);
  *total = s_warp[WF_TILE / 32 - 1];
  return v;
}

struct WRank {
  const unsigned long long* col[MAX_SORT_COLS];  // _timestamp, the partition key (keyed), the ORDER BY keys
  int n_col;
  int keyed;
  const unsigned int* idx;  // sorted
  long long n;
  unsigned char* bits;  // per sorted row: 1 = instant start, 2 = segment start, 4 = peer start
  RankVal* tiles;       // per tile: its total, then (wf_carry_kernel) the scan of the tiles before it
  unsigned long long* instants;
  int fn;
  long long top_n;
  unsigned long long* fn_out;
  unsigned int* keep;  // the fused filter
};

// pass 1: the starts of each sorted row (against the row before it), the instants, and each tile's total
__global__ void __launch_bounds__(WF_TILE) wf_rank_flags_kernel(const __grid_constant__ WRank p) {
  const long long j = (long long)blockIdx.x * WF_TILE + threadIdx.x;
  unsigned int bits = 0;
  if (j < p.n) {
    if (j == 0) {
      bits = 7u;
    } else {
      const unsigned int a = p.idx[j], b = p.idx[j - 1];
      const bool inst = p.col[0][a] != p.col[0][b];
      bool seg = inst;
      if (p.keyed) seg |= p.col[1][a] != p.col[1][b];
      bool peer = seg;
      for (int c = 1 + p.keyed; c < p.n_col; ++c) peer |= p.col[c][a] != p.col[c][b];
      bits = (inst ? 1u : 0u) | (seg ? 2u : 0u) | (peer ? 4u : 0u);
    }
    p.bits[j] = (unsigned char)bits;
  }
  const int starts = __syncthreads_count(bits & 1u);
  if (threadIdx.x == 0 && starts) atomicAdd(p.instants, (unsigned long long)starts);
  RankVal total;
  tile_inclusive(bits, j, &total);
  if (threadIdx.x == 0) p.tiles[blockIdx.x] = total;
}

// pass 2, one block: tiles[t] becomes the exclusive scan of the totals of tiles [0, t), 1024 tiles per round.  T is a
// scan element with combine / shfl_up overloads and an identity T::zero() (RankVal, AggVal).
template <class T>
__global__ void __launch_bounds__(1024) wf_carry_kernel(T* tiles, long long n_tiles) {
  __shared__ T s_warp[32];
  __shared__ T s_carry;
  const unsigned lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const T zero = T::zero();
  if (threadIdx.x == 0) s_carry = zero;
  __syncthreads();
  for (long long base = 0; base < n_tiles; base += 1024) {
    const long long i = base + threadIdx.x;
    const T v = i < n_tiles ? tiles[i] : zero;
    T x = v;
    for (int o = 1; o < 32; o <<= 1) {
      const T y = shfl_up(x, o);
      if ((int)lane >= o) x = combine(y, x);
    }
    T ex = shfl_up(x, 1);  // exclusive within the warp
    if (lane == 0) ex = zero;
    if (lane == 31) s_warp[w] = x;
    __syncthreads();
    if (w == 0) {
      T t = s_warp[lane];
      for (int o = 1; o < 32; o <<= 1) {
        const T y = shfl_up(t, o);
        if ((int)lane >= o) t = combine(y, t);
      }
      s_warp[lane] = t;  // inclusive over warps
    }
    __syncthreads();
    const T carry = s_carry;
    T before = w > 0 ? combine(carry, s_warp[w - 1]) : carry;
    if (i < n_tiles) tiles[i] = combine(before, ex);
    __syncthreads();
    if (threadIdx.x == 0) s_carry = combine(carry, s_warp[31]);
    __syncthreads();
  }
}

// pass 3: each sorted row's function value and whether the fused filter keeps it
__global__ void __launch_bounds__(WF_TILE) wf_rank_apply_kernel(const __grid_constant__ WRank p) {
  const long long j = (long long)blockIdx.x * WF_TILE + threadIdx.x;
  const unsigned int bits = j < p.n ? p.bits[j] : 0u;
  RankVal total;
  const RankVal v = tile_inclusive(bits, j, &total);
  if (j >= p.n) return;
  const RankVal s = combine(p.tiles[blockIdx.x], v);
  unsigned long long f;
  if (p.fn == ARROYO_B200_FN_ROW_NUMBER) f = (unsigned long long)(j + 2) - s.seg;
  else if (p.fn == ARROYO_B200_FN_RANK) f = (unsigned long long)(s.peer - s.seg) + 1ull;
  else f = s.dcnt;
  p.fn_out[j] = f;
  p.keep[j] = (p.top_n == 0 || f <= (unsigned long long)p.top_n) ? 1u : 0u;
}

// ---- aggregates -------------------------------------------------------------------------------------------------------
// SUM / COUNT / AVG / MIN / MAX over the default frame: from the segment start through the row's last peer (without
// ORDER BY every row of a segment is a peer).  A segmented inclusive scan of the argument over the sorted rows, reset at
// segment starts, gives each peer group's last row its frame's value; that row writes it at the group's first row, and
// the gather reads it there for every row of the group.  AggOp<K>: the scan's value, identity and operator, the
// argument's value for a row, and the function value from the frame's scan value and row count (AVG: the f64 sum over
// the count; COUNT scans ones).
template <int K> struct AggOp;
template <> struct AggOp<ARROYO_B200_AGG_COUNT_STAR> {
  using V = unsigned long long;
  __device__ static V identity() { return 0ull; }
  __device__ static V op(V a, V b) { return a + b; }
  __device__ static V load(const unsigned long long*, unsigned int) { return 1ull; }
  __device__ static unsigned long long result(V v, unsigned long long) { return v; }
};
template <> struct AggOp<ARROYO_B200_AGG_SUM_I64> {
  using V = unsigned long long;  // wrapping
  __device__ static V identity() { return 0ull; }
  __device__ static V op(V a, V b) { return a + b; }
  __device__ static V load(const unsigned long long* arg, unsigned int i) { return arg[i]; }
  __device__ static unsigned long long result(V v, unsigned long long) { return v; }
};
template <> struct AggOp<ARROYO_B200_AGG_MIN_I64> {
  using V = long long;
  __device__ static V identity() { return LLONG_MAX; }
  __device__ static V op(V a, V b) { return a < b ? a : b; }
  __device__ static V load(const unsigned long long* arg, unsigned int i) { return (long long)arg[i]; }
  __device__ static unsigned long long result(V v, unsigned long long) { return (unsigned long long)v; }
};
template <> struct AggOp<ARROYO_B200_AGG_MAX_I64> {
  using V = long long;
  __device__ static V identity() { return LLONG_MIN; }
  __device__ static V op(V a, V b) { return a > b ? a : b; }
  __device__ static V load(const unsigned long long* arg, unsigned int i) { return (long long)arg[i]; }
  __device__ static unsigned long long result(V v, unsigned long long) { return (unsigned long long)v; }
};
template <> struct AggOp<ARROYO_B200_AGG_AVG_I64> {
  using V = double;
  __device__ static V identity() { return 0.0; }
  __device__ static V op(V a, V b) { return a + b; }
  __device__ static V load(const unsigned long long* arg, unsigned int i) { return (double)(long long)arg[i]; }
  __device__ static unsigned long long result(V v, unsigned long long n) {
    return (unsigned long long)__double_as_longlong(v / (double)n);
  }
};

// The scan element: seg = a segment starts in the range, v = the operator over the range's rows from its last segment
// start on (all of them when none starts in it).
template <int K>
struct AggVal {
  unsigned int seg;
  typename AggOp<K>::V v;
  __device__ static AggVal zero() { return {0u, AggOp<K>::identity()}; }
};
template <int K>
__device__ __forceinline__ AggVal<K> combine(AggVal<K> a, AggVal<K> b) {
  return {a.seg | b.seg, b.seg ? b.v : AggOp<K>::op(a.v, b.v)};
}
template <int K>
__device__ __forceinline__ AggVal<K> shfl_up(AggVal<K> x, int o) {
  return {__shfl_up_sync(FULL, x.seg, o), __shfl_up_sync(FULL, x.v, o)};  // a 64-bit v moves as two 32-bit shuffles
}

struct WAgg {
  const unsigned long long* arg;  // the argument column (COUNT: unused)
  const unsigned int* idx;        // sorted
  const unsigned char* bits;      // wf_rank_flags_kernel's starts
  long long n;
  const RankVal* rank_tiles;      // after wf_carry_kernel<RankVal>
  void* tiles;                    // AggVal<K> per tile: its total, then the scan of the tiles before it
  unsigned long long* fv;         // at each peer group's first sorted row: the group's function value
  unsigned int* at;               // per sorted row: its peer group's first sorted row
};

template <int K>
__device__ __forceinline__ AggVal<K> agg_element(const WAgg& p, long long j, unsigned int bits) {
  AggVal<K> x = AggVal<K>::zero();
  if (j < p.n) {
    x.seg = (bits >> 1) & 1u;
    x.v = AggOp<K>::load(p.arg, p.idx[j]);
  }
  return x;
}

// Inclusive segmented scan of one tile of WF_TILE rows (one per thread); the tile's total goes to `*total`.  Every
// thread of the block calls it.
template <int K>
__device__ __forceinline__ AggVal<K> agg_tile_inclusive(AggVal<K> x, AggVal<K>* total) {
  __shared__ AggVal<K> s_warp[WF_TILE / 32];
  const unsigned lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  for (int o = 1; o < 32; o <<= 1) {
    const AggVal<K> y = shfl_up(x, o);
    if ((int)lane >= o) x = combine(y, x);
  }
  if (lane == 31) s_warp[w] = x;
  __syncthreads();
  if (w == 0) {
    AggVal<K> t = s_warp[lane];
    for (int o = 1; o < 32; o <<= 1) {
      const AggVal<K> y = shfl_up(t, o);
      if ((int)lane >= o) t = combine(y, t);
    }
    s_warp[lane] = t;
  }
  __syncthreads();
  if (w > 0) x = combine(s_warp[w - 1], x);
  *total = s_warp[WF_TILE / 32 - 1];
  return x;
}

// pass 1: each tile's total
template <int K>
__global__ void __launch_bounds__(WF_TILE) wf_agg_tiles_kernel(const __grid_constant__ WAgg p) {
  const long long j = (long long)blockIdx.x * WF_TILE + threadIdx.x;
  const unsigned int bits = j < p.n ? p.bits[j] : 0u;
  AggVal<K> total;
  agg_tile_inclusive<K>(agg_element<K>(p, j, bits), &total);
  if (threadIdx.x == 0) static_cast<AggVal<K>*>(p.tiles)[blockIdx.x] = total;
}

// pass 3 (after wf_carry_kernel over the tiles): each row's peer group, and at each group's last row the frame's
// value, written at the group's first row
template <int K>
__global__ void __launch_bounds__(WF_TILE) wf_agg_apply_kernel(const __grid_constant__ WAgg p) {
  const long long j = (long long)blockIdx.x * WF_TILE + threadIdx.x;
  const unsigned int bits = j < p.n ? p.bits[j] : 0u;
  RankVal rt;
  const RankVal rv = tile_inclusive(bits, j, &rt);
  AggVal<K> at;
  const AggVal<K> av = agg_tile_inclusive<K>(agg_element<K>(p, j, bits), &at);
  if (j >= p.n) return;
  const RankVal r = combine(p.rank_tiles[blockIdx.x], rv);
  const AggVal<K> s = combine(static_cast<const AggVal<K>*>(p.tiles)[blockIdx.x], av);
  const unsigned int first = r.peer - 1u;
  p.at[j] = first;
  if (j + 1 == p.n || (p.bits[j + 1] & 4u))
    p.fv[first] = AggOp<K>::result(s.v, (unsigned long long)(j + 2) - r.seg);
}

template <int K>
void launch_aggregate(const WAgg& p, uint64_t n_tiles, cudaStream_t stream) {
  static_assert(sizeof(AggVal<K>) == 16, "WindowFnOp::aggregate sizes the tile totals for 16 bytes");
  wf_agg_tiles_kernel<K><<<(unsigned)n_tiles, WF_TILE, 0, stream>>>(p);
  AB_CUDA(cudaGetLastError());
  wf_carry_kernel<AggVal<K>><<<1, 1024, 0, stream>>>(static_cast<AggVal<K>*>(p.tiles), (long long)n_tiles);
  AB_CUDA(cudaGetLastError());
  wf_agg_apply_kernel<K><<<(unsigned)n_tiles, WF_TILE, 0, stream>>>(p);
  AB_CUDA(cudaGetLastError());
}

// ---- value functions --------------------------------------------------------------------------------------------------
// LAG / LEAD / FIRST_VALUE / LAST_VALUE / NTH_VALUE, PERCENT_RANK and CUME_DIST are index arithmetic on the rank scan.
// For sorted row j the scan gives its segment's first row s and its peer group's first row g; the bounds pass adds the
// segment's last row e and the peer group's last row f (the default frame's end: without ORDER BY every row of a segment
// is a peer, so f = e): the last row of each peer group writes its index at the group's first row, and the last row of
// each segment does the same at the segment's first row.  The apply pass then reads the argument at the row the function
// names, LAG j - k, LEAD j + k, FIRST_VALUE s, LAST_VALUE f, NTH_VALUE s + n - 1, or takes the default (LAG / LEAD) or
// NULL when that row is outside [s, e] (NTH_VALUE: [s, f]).  PERCENT_RANK = (g - s) / (e - s), 0 when s = e, and
// CUME_DIST = (f - s + 1) / (e - s + 1), both in f64.  The argument's 64 bits move unchanged.
struct WValue {
  const unsigned long long* arg;  // the argument column (PERCENT_RANK / CUME_DIST: unused)
  const unsigned int* idx;        // sorted
  const unsigned char* bits;      // wf_rank_flags_kernel's starts
  long long n;
  const RankVal* rank_tiles;      // after wf_carry_kernel<RankVal>
  unsigned int* peer_last;        // at each peer group's first sorted row: the group's last sorted row
  unsigned int* seg_last;         // at each segment's first sorted row: the segment's last sorted row
  int fn;
  unsigned long long offset;      // LAG / LEAD: k; NTH_VALUE: n - 1
  unsigned long long dflt;        // LAG / LEAD: the default's bits (0 without one; a NULL row's value)
  unsigned long long* fv;         // per sorted row: the function's value
  unsigned char* valid;           // per sorted row: 0 = NULL; null when the function cannot give NULL
};

// Each row's segment and peer group first rows: the rank scan of its tile on top of the tiles before it.  Every thread
// of the block calls it.
__device__ __forceinline__ RankVal value_scan(const WValue& p, long long j, unsigned int bits) {
  RankVal total;
  const RankVal v = tile_inclusive(bits, j, &total);
  return combine(p.rank_tiles[blockIdx.x], v);
}

// pass 1: the last row of each peer group and of each segment, at its first row
__global__ void __launch_bounds__(WF_TILE) wf_bounds_kernel(const __grid_constant__ WValue p) {
  const long long j = (long long)blockIdx.x * WF_TILE + threadIdx.x;
  const unsigned int bits = j < p.n ? p.bits[j] : 0u;
  const RankVal r = value_scan(p, j, bits);
  if (j >= p.n) return;
  const unsigned int next = j + 1 < p.n ? p.bits[j + 1] : 6u;  // past the last row: a segment (and peer) start
  if (next & 4u) p.peer_last[r.peer - 1u] = (unsigned int)j;
  if (next & 2u) p.seg_last[r.seg - 1u] = (unsigned int)j;
}

// pass 2: each sorted row's value and validity
__global__ void __launch_bounds__(WF_TILE) wf_value_apply_kernel(const __grid_constant__ WValue p) {
  const long long j = (long long)blockIdx.x * WF_TILE + threadIdx.x;
  const unsigned int bits = j < p.n ? p.bits[j] : 0u;
  const RankVal r = value_scan(p, j, bits);
  if (j >= p.n) return;
  const unsigned int row = (unsigned int)j, s = r.seg - 1u, g = r.peer - 1u;
  const unsigned int f = p.peer_last[g], e = p.seg_last[s];
  unsigned long long v;
  bool ok = true;
  if (p.fn == ARROYO_B200_FN_PERCENT_RANK) {
    v = e == s ? 0ull : (unsigned long long)__double_as_longlong((double)(g - s) / (double)(e - s));
  } else if (p.fn == ARROYO_B200_FN_CUME_DIST) {
    v = (unsigned long long)__double_as_longlong((double)(f - s + 1u) / (double)(e - s + 1u));
  } else {
    // the offsets are compared before they are narrowed: k may be anything up to INT64_MAX
    unsigned int src;
    if (p.fn == ARROYO_B200_FN_LAG) {
      ok = p.offset <= (unsigned long long)(row - s);
      src = row - (unsigned int)p.offset;
    } else if (p.fn == ARROYO_B200_FN_LEAD) {
      ok = p.offset <= (unsigned long long)(e - row);
      src = row + (unsigned int)p.offset;
    } else if (p.fn == ARROYO_B200_FN_FIRST_VALUE) {
      src = s;
    } else if (p.fn == ARROYO_B200_FN_LAST_VALUE) {
      src = f;
    } else {
      ok = p.offset <= (unsigned long long)(f - s);
      src = s + (unsigned int)p.offset;
    }
    v = ok ? p.arg[p.idx[src]] : p.dflt;
  }
  p.fv[j] = v;
  if (p.valid) p.valid[j] = ok ? 1u : 0u;
}

// ---- explicit frames --------------------------------------------------------------------------------------------------
// An aggregate or FIRST_VALUE / LAST_VALUE / NTH_VALUE over `{ROWS | RANGE | GROUPS} BETWEEN start AND end`.  Sorted
// row j of a segment [s, e] gets the half-open frame [lo, hi) of sorted rows, clipped to [s, e + 1); lo >= hi is an
// empty frame.  Each bound is found from the rank scan (s, the peer group's first row g, the dense rank d) and
// wf_bounds_kernel's e and peer-group ends:
//   ROWS    row j - n / j / j + n (an end one past it);
//   GROUPS  the first row of peer group d - n / d / d + n (an end: of the group after it), through a map from each
//           segment's group ordinals to their first rows (wf_groups_kernel);
//   RANGE   CURRENT ROW: g, or one past the peer group's last row; n PRECEDING / FOLLOWING: a binary search in [s, e + 1)
//           of the one ORDER BY key in its sort's unsigned order-preserving form u, for u >= u(j) -/+ n (a start) or
//           u > u(j) -/+ n (an end); a limit u(j) -/+ n outside [0, 2^64) is before or after every row.  That form has
//           slope +-1, so under DESC "n PRECEDING" is keys up to x + n.
// ROWS and GROUPS offsets are clamped to 2^32 before any arithmetic: a segment has fewer than 2^31 rows, so a larger n
// reaches as far.  lo and hi are non-decreasing in j within a segment.  The values over [lo, hi):
//   COUNT hi - lo; SUM / AVG differences of prefix sums over the sorted rows, kept exact as the low 32 bits and the
//   high 32 bits (signed, biased by 2^31) of each value, so SUM wraps and AVG converts the exact sum to f64 once;
//   MIN / MAX a range-extremum query: 32-row blocks with in-block prefix and suffix extremes, a sparse table over the
//   block extremes, and a scan of at most 32 values when lo and hi - 1 share a block;
//   FIRST_VALUE / LAST_VALUE / NTH_VALUE the argument at lo, hi - 1, lo + n - 1 (NULL past hi - 1).
// Every function but COUNT is NULL on an empty frame.
constexpr unsigned long long FRAME_OFFSET_CAP = 1ull << 32;

struct WFrame {
  WValue b;                  // the rank scan, wf_bounds_kernel's peer_last / seg_last, fn, NTH_VALUE's n - 1, fv, valid
  int units, start_kind, end_kind;
  unsigned long long start_off, end_off;
  const unsigned long long* ukey;  // RANGE with an offset: per sorted row its ORDER BY key, unsigned order-preserving
  unsigned int* gfirst;            // GROUPS: at s + d - 1 the first row of the segment's d-th peer group
  unsigned int* gcount;            // GROUPS: at s the segment's number of peer groups
  const unsigned long long* pre_lo;  // SUM / AVG: at j (0 .. n) the sums over sorted rows [0, j) of the values' low
  const unsigned long long* pre_hi;  //   32 bits and of their high 32 bits + 2^31 (the signed high half, biased)
  const long long* v;              // MIN / MAX: per sorted row the argument
  const long long* in_pre;         //   per sorted row the extreme of its 32-row block's rows up to it
  const long long* in_suf;         //   ... and from it on
  const long long* table;          //   level k (k * n_blocks on): per block b the extreme of blocks [b, b + 2^k)
  long long n_blocks;
};

// GROUPS: each segment's peer groups by ordinal, and its group count
__global__ void __launch_bounds__(WF_TILE) wf_groups_kernel(const __grid_constant__ WFrame p) {
  const long long j = (long long)blockIdx.x * WF_TILE + threadIdx.x;
  const unsigned int bits = j < p.b.n ? p.b.bits[j] : 0u;
  const RankVal r = value_scan(p.b, j, bits);
  if (j >= p.b.n) return;
  const unsigned int s = r.seg - 1u;
  if (bits & 4u) p.gfirst[s + r.dcnt - 1u] = (unsigned int)j;
  const unsigned int next = j + 1 < p.b.n ? p.b.bits[j + 1] : 6u;
  if (next & 2u) p.gcount[s] = r.dcnt;
}

// the first row in [a, b) whose key is > t (`strict`) or >= t
__device__ __forceinline__ unsigned int key_search(const unsigned long long* u, unsigned int a, unsigned int b,
                                                   unsigned long long t, bool strict) {
  while (a < b) {
    const unsigned int m = a + (b - a) / 2;
    const unsigned long long x = u[m];
    if (strict ? x <= t : x < t) a = m + 1;
    else b = m;
  }
  return a;
}

// One end of row j's frame, in [s, e + 1]: the start (`end` false) or one past the end.
__device__ __forceinline__ unsigned int frame_edge(const WFrame& p, int kind, unsigned long long off, bool end,
                                                   unsigned int j, unsigned int s, unsigned int e, const RankVal& r) {
  if (kind == ARROYO_B200_BOUND_UNBOUNDED_PRECEDING) return s;
  if (kind == ARROYO_B200_BOUND_UNBOUNDED_FOLLOWING) return e + 1u;
  const bool cur = kind == ARROYO_B200_BOUND_CURRENT_ROW, back = kind == ARROYO_B200_BOUND_PRECEDING;
  if (p.units == ARROYO_B200_FRAME_RANGE) {
    const unsigned int g = r.peer - 1u;
    if (cur) return end ? p.b.peer_last[g] + 1u : g;
    // a limit past the key type's range lies before every row (PRECEDING) or after every row (FOLLOWING)
    const unsigned long long u = p.ukey[j];
    if (back ? u < off : off > ~u) return back ? s : e + 1u;
    return key_search(p.ukey, s, e + 1u, back ? u - off : u + off, end);
  }
  const long long n = cur ? 0 : (long long)(off < FRAME_OFFSET_CAP ? off : FRAME_OFFSET_CAP);
  const long long k = (back ? -n : n) + (end ? 1 : 0);
  if (p.units == ARROYO_B200_FRAME_ROWS) {
    const long long x = (long long)j + k;
    return x < (long long)s ? s : x > (long long)e + 1 ? e + 1u : (unsigned int)x;
  }
  const long long d = (long long)r.dcnt + k;  // GROUPS: the ordinal of the peer group the edge starts
  return d < 1 ? s : d > (long long)p.gcount[s] ? e + 1u : p.gfirst[s + (unsigned int)d - 1u];
}

// MIN / MAX of the sorted rows [a, b], a <= b
template <int K>
__device__ __forceinline__ long long range_extreme(const WFrame& p, unsigned int a, unsigned int b) {
  const unsigned int ba = a >> 5, bb = b >> 5;
  if (ba == bb) {
    long long x = p.v[a];
    for (unsigned int i = a + 1; i <= b; ++i) x = AggOp<K>::op(x, p.v[i]);
    return x;
  }
  long long x = AggOp<K>::op(p.in_suf[a], p.in_pre[b]);
  if (bb > ba + 1) {
    const unsigned int l = ba + 1, h = bb - 1;
    const int k = 31 - __clz(h - l + 1);
    const long long* t = p.table + (long long)k * p.n_blocks;
    x = AggOp<K>::op(x, AggOp<K>::op(t[l], t[h + 1 - (1u << k)]));
  }
  return x;
}

// each sorted row's frame and its value over it (F: an ArroyoB200AggKind, or FN_FIRST_VALUE .. FN_NTH_VALUE)
template <int F>
__global__ void __launch_bounds__(WF_TILE) wf_frame_apply_kernel(const __grid_constant__ WFrame p) {
  const long long j = (long long)blockIdx.x * WF_TILE + threadIdx.x;
  const unsigned int bits = j < p.b.n ? p.b.bits[j] : 0u;
  const RankVal r = value_scan(p.b, j, bits);
  if (j >= p.b.n) return;
  const unsigned int row = (unsigned int)j, s = r.seg - 1u, e = p.b.seg_last[s];
  const unsigned int lo = frame_edge(p, p.start_kind, p.start_off, false, row, s, e, r);
  const unsigned int hi = frame_edge(p, p.end_kind, p.end_off, true, row, s, e, r);
  bool ok = lo < hi;
  unsigned long long v = 0;
  if constexpr (F == ARROYO_B200_AGG_COUNT_STAR) {
    v = ok ? hi - lo : 0u;
    ok = true;
  } else if constexpr (F == ARROYO_B200_AGG_SUM_I64 || F == ARROYO_B200_AGG_AVG_I64) {
    if (ok) {
      const unsigned long long sl = p.pre_lo[hi] - p.pre_lo[lo];
      const long long sh = (long long)(p.pre_hi[hi] - p.pre_hi[lo] - ((unsigned long long)(hi - lo) << 31));
      if constexpr (F == ARROYO_B200_AGG_SUM_I64) v = ((unsigned long long)sh << 32) + sl;
      else v = (unsigned long long)__double_as_longlong((double)(((__int128)sh << 32) + (__int128)sl) / (double)(hi - lo));
    }
  } else if constexpr (F == ARROYO_B200_AGG_MIN_I64 || F == ARROYO_B200_AGG_MAX_I64) {
    if (ok) v = (unsigned long long)range_extreme<F>(p, lo, hi - 1u);
  } else {
    unsigned int src = lo;  // FIRST_VALUE
    if constexpr (F == ARROYO_B200_FN_LAST_VALUE) src = hi - 1u;
    if constexpr (F == ARROYO_B200_FN_NTH_VALUE) {
      ok = ok && p.b.offset < (unsigned long long)(hi - lo);  // compared before it is narrowed
      src = lo + (unsigned int)p.b.offset;
    }
    if (ok) v = p.b.arg[p.b.idx[src]];
  }
  p.b.fv[j] = v;
  if (p.b.valid) p.b.valid[j] = ok ? 1u : 0u;
}

// SUM / AVG: sorted row j's value as two 32-bit counts for device_exclusive_scan: lo[j] its low 32 bits, hi[j] its
// high 32 bits + 2^31
__global__ void wf_split_kernel(const unsigned long long* __restrict__ arg, const unsigned int* __restrict__ idx,
                                long long n, unsigned int* __restrict__ lo, unsigned int* __restrict__ hi) {
  long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (; j < n; j += stride) {
    const unsigned long long x = arg[idx[j]];
    lo[j] = (unsigned int)x;
    hi[j] = (unsigned int)(x >> 32) ^ 0x80000000u;
  }
}

// MIN / MAX: the sorted values, their in-block prefix and suffix extremes and level 0 of the sparse table (one warp per
// 32-row block; rows past n take the identity)
struct WRmq {
  const unsigned long long* arg;
  const unsigned int* idx;
  long long n;
  long long* v;
  long long* in_pre;
  long long* in_suf;
  long long* table;
  long long n_blocks;
};
template <int K>
__global__ void __launch_bounds__(WF_THREADS) wf_rmq_blocks_kernel(const __grid_constant__ WRmq p) {
  const long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const unsigned lane = threadIdx.x & 31;
  const long long x = j < p.n ? (long long)p.arg[p.idx[j]] : AggOp<K>::identity();
  long long up = x, down = x;
  for (int o = 1; o < 32; o <<= 1) {
    const long long a = __shfl_up_sync(FULL, up, o), b = __shfl_down_sync(FULL, down, o);
    if ((int)lane >= o) up = AggOp<K>::op(a, up);
    if ((int)lane + o < 32) down = AggOp<K>::op(down, b);
  }
  if (j < p.n) {
    p.v[j] = x;
    p.in_pre[j] = up;
    p.in_suf[j] = down;
  }
  if (lane == 0 && (j >> 5) < p.n_blocks) p.table[j >> 5] = down;
}

// level k of the sparse table from level k - 1 (a range past the last block is clipped to it)
template <int K>
__global__ void wf_rmq_level_kernel(long long* table, long long n_blocks, int k) {
  const long long* prev = table + (long long)(k - 1) * n_blocks;
  long long* cur = table + (long long)k * n_blocks;
  const long long half = 1ll << (k - 1);
  long long b = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (; b < n_blocks; b += stride) cur[b] = AggOp<K>::op(prev[b], prev[b + half < n_blocks ? b + half : n_blocks - 1]);
}

// out[c][o] = store[c][idx[j]] for the kept rows (keep null: every row, o = j), and the function column: fn[j], or
// fn[at[j]] when `at` is given, with its validity byte from `valid` when that is given
struct WGather {
  const unsigned long long* store[ARROYO_B200_MAX_COLS];
  WCols out;
  int n_cols;
  const unsigned int* idx;
  const unsigned int* keep;
  const unsigned long long* off;
  const unsigned long long* fn;
  const unsigned int* at;
  const unsigned char* valid;
  unsigned long long* fn_out;
  unsigned char* valid_out;
  long long n;
};
__global__ void __launch_bounds__(WF_THREADS) wf_gather_kernel(const __grid_constant__ WGather p) {
  long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (; j < p.n; j += stride) {
    if (p.keep && !p.keep[j]) continue;
    const unsigned long long o = p.keep ? p.off[j] : (unsigned long long)j;
    const unsigned int src = p.idx[j];
    for (int c = 0; c < p.n_cols; ++c) p.out.c[c][o] = p.store[c][src];
    if (p.fn_out) {
      const unsigned int f = p.at ? p.at[j] : (unsigned int)j;
      p.fn_out[o] = p.fn[f];
      if (p.valid) p.valid_out[o] = p.valid[f];
    }
  }
}

// the rows that stay, moved to [0, n - leaving) of `to` in arrival order: new index = i - (rows leaving below it)
struct WCompact {
  const unsigned long long* from[ARROYO_B200_MAX_COLS];
  WCols to;
  int n_cols;
  const unsigned int* flag;
  const unsigned long long* off;
  long long n;
};
__global__ void __launch_bounds__(WF_THREADS) wf_compact_kernel(const __grid_constant__ WCompact p) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (; i < p.n; i += stride) {
    if (p.flag[i]) continue;
    const unsigned long long d = (unsigned long long)i - p.off[i];
    for (int c = 0; c < p.n_cols; ++c) p.to.c[c][d] = p.from[c][i];
  }
}

// room for `bytes`, kept across calls (grown by half again so that a slowly growing need does not reallocate each time)
void reserve(DevBuf& b, size_t bytes) {
  if (b.bytes < bytes) b.alloc(std::max(bytes, b.bytes + b.bytes / 2));
}

bool sortable_format(const std::string& f) { return f == "l" || f == "L" || f.compare(0, 4, "tsn:") == 0; }

class WindowFnOp final : public OpBase {
 public:
  explicit WindowFnOp(const ArroyoB200OpConfig& c);
  ~WindowFnOp() override { drain_stream(); }
  void on_start(ArrowArray* state, ArrowSchema* schemas, int64_t n, int64_t watermark, int64_t table_min) override;
  void process_batch(uint32_t, uint32_t, ArrowArray* batch, const ArrowSchema* schema) override;
  void process_device_batch(uint32_t, uint32_t, const uint64_t* cols, int32_t n_cols, int64_t n_rows) override;
  void handle_watermark(int64_t wm, BatchesPriv* out_host, std::vector<ArroyoB200DeviceBatch>* out_dev) override;
  void handle_checkpoint(int64_t wm, BatchesPriv* out) override;
  void on_close(int, BatchesPriv*) override { flush(); }
  void flush() override {
    set_device();
    AB_CUDA(cudaStreamSynchronize(stream_));
  }
  void stats(ArroyoB200Stats* out) override {
    set_device();
    read_counters();
    *out = st_;
  }

 private:
  struct Store {
    DevBuf col[ARROYO_B200_MAX_COLS];
  };
  // The input layout, flat: one entry per 64-bit column; `nests_` re-nests the struct columns of host batches.
  struct Layout {
    std::vector<std::string> names, formats;
    std::vector<Nest> nests;
  };
  int n_cols_ = 0, ts_col_ = 0, key_col_ = -1, fn_ = 0;
  int agg_kind_ = 0;  // FN_AGGREGATE: the aggregate
  int arg_col_ = -1;  // the argument column of an aggregate (COUNT: none) or a value function
  int n_order_ = 0, order_col_[ARROYO_B200_MAX_ORDER_KEYS] = {}, order_desc_[ARROYO_B200_MAX_ORDER_KEYS] = {};
  int64_t top_n_ = 0;
  uint64_t offset_ = 0;      // LAG / LEAD: k; NTH_VALUE: n - 1
  uint64_t dflt_ = 0;        // LAG / LEAD: the default's bits
  bool has_default_ = false;
  ArroyoB200WindowFrame frame_{};  // units 0: the default frame (a default-equivalent frame is normalised to it)
  Layout layout_;
  bool typed_ = false;  // layout_ comes from a host or state batch (else: Int64 columns, no structs)
  int64_t late_wm_ = LLONG_MIN;
  Store cur_, alt_;  // alt_: where the rows that stay after an emission go (allocated on first use)
  uint64_t cap_ = 0;
  uint64_t n_store_ = 0;   // as of the last read
  uint64_t store_hi_ = 0;  // upper bound of the stored rows: n_store_ + rows handed over since
  uint64_t ckpt_from_ = 0; // rows [ckpt_from_, n) arrived since the last checkpoint
  DevBuf counters_, stage_;
  uint64_t stage_cap_ = 0;
  DevBuf flag_, off_, sums_, idx_[2], key_[2], cub_tmp_, bits_, tiles_, fnv_, keep_, off2_, agg_tiles_, at_;
  DevBuf seg_last_, valid_;  // value functions: each segment's last row at its first, each row's validity
  DevBuf gfirst_, gcount_, pre_, rmq_, table_;  // explicit frames: see WFrame
  DevBuf out_[ARROYO_B200_MAX_COLS], out_fn_, out_valid_, out_bits_;
  ArroyoB200Stats st_{};

  int grid_for(uint64_t n) const {
    return (int)std::max<uint64_t>(1, std::min<uint64_t>((n + WF_THREADS - 1) / WF_THREADS, (uint64_t)num_sms_ * 8));
  }
  WCounters* counters() const { return counters_.as<WCounters>(); }
  bool ranking() const { return fn_ <= ARROYO_B200_FN_DENSE_RANK; }
  bool value_fn() const { return fn_ >= ARROYO_B200_FN_LAG && fn_ <= ARROYO_B200_FN_NTH_VALUE; }
  // LAG / LEAD / NTH_VALUE, and under an explicit frame every function but COUNT, may give NULL; `null_rows()`: with
  // these arguments some row can be NULL
  bool nullable() const {
    if (frame_.units != ARROYO_B200_FRAME_DEFAULT)
      return !(fn_ == ARROYO_B200_FN_AGGREGATE && agg_kind_ == ARROYO_B200_AGG_COUNT_STAR);
    return fn_ == ARROYO_B200_FN_LAG || fn_ == ARROYO_B200_FN_LEAD || fn_ == ARROYO_B200_FN_NTH_VALUE;
  }
  bool null_rows() const { return nullable() && !has_default_; }
  const char* fn_name() const {
    static const char* const names[] = {"",          "row_number", "rank",       "dense_rank",   "",
                                        "lag",       "lead",       "first_value", "last_value",  "nth_value",
                                        "percent_rank", "cume_dist"};
    if (fn_ == ARROYO_B200_FN_AGGREGATE)
      return agg_kind_ == ARROYO_B200_AGG_COUNT_STAR ? "count"
             : agg_kind_ == ARROYO_B200_AGG_SUM_I64  ? "sum"
             : agg_kind_ == ARROYO_B200_AGG_AVG_I64  ? "avg"
             : agg_kind_ == ARROYO_B200_AGG_MIN_I64  ? "min"
                                                     : "max";
    return names[fn_];
  }
  // ranks are UInt64; count / sum / min / max Int64, avg Float64; a value function takes its argument's type,
  // PERCENT_RANK / CUME_DIST are Float64
  std::string fn_format() const {
    if (ranking()) return "L";
    if (value_fn()) return layout_.formats[arg_col_];
    if (fn_ != ARROYO_B200_FN_AGGREGATE) return "g";
    return agg_kind_ == ARROYO_B200_AGG_AVG_I64 ? "g" : "l";
  }
  void aggregate(const WRank& r, uint64_t n_tiles);
  void values(const WRank& r, uint64_t n_tiles);
  void framed(const WRank& r, uint64_t n_tiles);
  void check_frame(const ArroyoB200WindowFrame& f);
  unsigned long long flip_of(int col, bool desc) const;
  Layout layout_of(const std::vector<InColumn>& cols, const std::vector<Nest>& nests, const ArrowSchema* s) const;
  void check_layout(const Layout& l, int bad_type_status) const;
  void adopt(const Layout& l);
  std::vector<OutColumn> host_columns(const std::function<void*(int)>& data) const;
  void alloc_store(Store& s, uint64_t cap) const;
  void reserve_rows(uint64_t more);
  void read_counters();
  const unsigned long long* const* stage(const std::vector<InColumn>& cols, int64_t n, const unsigned long long** ptrs);
  void ingest(const unsigned long long* const* cols, int64_t n, long long late_wm);
  unsigned int* sort_rows(uint64_t e, bool by_ts_only);
  void emit(int64_t w, BatchesPriv* out);
};

WindowFnOp::WindowFnOp(const ArroyoB200OpConfig& c) {
  cfg = c;
  name = "window_function";
  AB_REQUIRE(c.window_fn >= ARROYO_B200_FN_ROW_NUMBER && c.window_fn <= ARROYO_B200_FN_CUME_DIST,
             ARROYO_B200_INVALID_ARGUMENT,
             "window function: window_fn must be ROW_NUMBER (1), RANK (2), DENSE_RANK (3), AGGREGATE (4), LAG (5), "
             "LEAD (6), FIRST_VALUE (7), LAST_VALUE (8), NTH_VALUE (9), PERCENT_RANK (10) or CUME_DIST (11)");
  fn_ = c.window_fn;
  const bool agg = fn_ == ARROYO_B200_FN_AGGREGATE;
  AB_REQUIRE(c.n_cols >= 1 && c.n_cols <= ARROYO_B200_MAX_COLS, ARROYO_B200_INVALID_ARGUMENT, "bad n_cols");
  n_cols_ = c.n_cols;
  AB_REQUIRE(c.timestamp_col >= 0 && c.timestamp_col < n_cols_, ARROYO_B200_INVALID_ARGUMENT, "bad timestamp_col");
  ts_col_ = c.timestamp_col;
  AB_REQUIRE(c.n_key_cols >= 0, ARROYO_B200_INVALID_ARGUMENT, "bad n_key_cols");
  AB_REQUIRE(c.n_key_cols <= 1, ARROYO_B200_UNSUPPORTED,
             "window function: PARTITION BY over more than one column besides the window is not supported");
  if (c.n_key_cols == 1) {
    AB_REQUIRE(c.key_col >= 0 && c.key_col < n_cols_, ARROYO_B200_INVALID_ARGUMENT, "bad key_col");
    key_col_ = c.key_col;
  }
  if (agg) {
    // aggs[0] is the aggregate, aggs[1 ..] the ORDER BY keys
    AB_REQUIRE(c.n_aggs >= 1 && c.n_aggs <= 1 + ARROYO_B200_MAX_ORDER_KEYS, ARROYO_B200_INVALID_ARGUMENT,
               "window function: an aggregate takes itself and 0 to 4 ORDER BY keys (n_aggs 1 to 5)");
    agg_kind_ = c.aggs[0].kind;
    AB_REQUIRE(agg_kind_ == ARROYO_B200_AGG_COUNT_STAR || agg_kind_ == ARROYO_B200_AGG_SUM_I64 ||
                   agg_kind_ == ARROYO_B200_AGG_AVG_I64 || agg_kind_ == ARROYO_B200_AGG_MIN_I64 ||
                   agg_kind_ == ARROYO_B200_AGG_MAX_I64,
               ARROYO_B200_INVALID_ARGUMENT,
               "window function: aggs[0] of an aggregate is COUNT_STAR, SUM_I64, AVG_I64, MIN_I64 or MAX_I64");
    if (agg_kind_ != ARROYO_B200_AGG_COUNT_STAR) {
      AB_REQUIRE(c.aggs[0].input_col >= 0 && c.aggs[0].input_col < n_cols_, ARROYO_B200_INVALID_ARGUMENT,
                 "window function: aggregate argument column out of range");
      arg_col_ = c.aggs[0].input_col;
    }
    AB_REQUIRE(c.slide_ns == 0, ARROYO_B200_INVALID_ARGUMENT,
               "window function: an aggregate takes no top N filter (slide_ns must be 0)");
  } else if (ranking()) {
    AB_REQUIRE(c.n_aggs >= 1 && c.n_aggs <= ARROYO_B200_MAX_ORDER_KEYS, ARROYO_B200_INVALID_ARGUMENT,
               "window function: ORDER BY takes 1 to 4 keys (n_aggs)");
    AB_REQUIRE(c.slide_ns >= 0, ARROYO_B200_INVALID_ARGUMENT, "window function: top N (slide_ns) must be >= 0");
    top_n_ = c.slide_ns;
  } else {
    if (value_fn()) {
      // aggs[0] is the argument, aggs[1 ..] the ORDER BY keys
      AB_REQUIRE(c.n_aggs >= 1 && c.n_aggs <= 1 + ARROYO_B200_MAX_ORDER_KEYS, ARROYO_B200_INVALID_ARGUMENT,
                 std::string("window function: ") + fn_name() +
                     " takes its argument and 0 to 4 ORDER BY keys (n_aggs 1 to 5)");
      AB_REQUIRE(c.aggs[0].kind == ARROYO_B200_FN_ARGUMENT, ARROYO_B200_INVALID_ARGUMENT,
                 std::string("window function: aggs[0] of ") + fn_name() + " is {FN_ARGUMENT (18), argument column}");
      AB_REQUIRE(c.aggs[0].input_col >= 0 && c.aggs[0].input_col < n_cols_, ARROYO_B200_INVALID_ARGUMENT,
                 "window function: argument column out of range");
      arg_col_ = c.aggs[0].input_col;
    } else {
      AB_REQUIRE(c.n_aggs >= 0 && c.n_aggs <= ARROYO_B200_MAX_ORDER_KEYS, ARROYO_B200_INVALID_ARGUMENT,
                 std::string("window function: ") + fn_name() + " takes 0 to 4 ORDER BY keys (n_aggs)");
    }
    AB_REQUIRE(c.slide_ns == 0, ARROYO_B200_INVALID_ARGUMENT,
               std::string("window function: ") + fn_name() + " takes no top N filter (slide_ns must be 0)");
    const bool lag_lead = fn_ == ARROYO_B200_FN_LAG || fn_ == ARROYO_B200_FN_LEAD;
    has_default_ = (c.flags & ARROYO_B200_FLAG_FN_DEFAULT) != 0;
    AB_REQUIRE(!has_default_ || lag_lead, ARROYO_B200_INVALID_ARGUMENT,
               std::string("window function: ") + fn_name() + " takes no default (ARROYO_B200_FLAG_FN_DEFAULT)");
    if (has_default_) dflt_ = (uint64_t)c.gap_ns;
    if (lag_lead) {
      AB_REQUIRE(c.width_ns >= 0, ARROYO_B200_UNSUPPORTED,
                 std::string("window function: ") + fn_name() + " with a negative offset is not supported");
      offset_ = (uint64_t)c.width_ns;
    } else if (fn_ == ARROYO_B200_FN_NTH_VALUE) {
      AB_REQUIRE(c.width_ns >= 0, ARROYO_B200_UNSUPPORTED,
                 "window function: nth_value with a negative n is not supported");
      AB_REQUIRE(c.width_ns != 0, ARROYO_B200_INVALID_ARGUMENT, "window function: nth_value's n (width_ns) must be >= 1");
      offset_ = (uint64_t)c.width_ns - 1;
    }
  }
  const int first_key = (agg || value_fn()) ? 1 : 0;
  n_order_ = c.n_aggs - first_key;
  for (int k = 0; k < n_order_; ++k) {
    const ArroyoB200Agg& a = c.aggs[first_key + k];
    AB_REQUIRE(a.kind == ARROYO_B200_ORDER_ASC || a.kind == ARROYO_B200_ORDER_DESC, ARROYO_B200_INVALID_ARGUMENT,
               "window function: an ORDER BY key's kind is ORDER_ASC (16) or ORDER_DESC (17)");
    AB_REQUIRE(a.input_col >= 0 && a.input_col < n_cols_, ARROYO_B200_INVALID_ARGUMENT,
               "window function: ORDER BY column out of range");
    order_col_[k] = a.input_col;
    order_desc_[k] = a.kind == ARROYO_B200_ORDER_DESC;
  }
  check_frame(c.frame);
  for (int f = 0; f < n_cols_; ++f) {
    layout_.names.push_back(f == ts_col_ ? "_timestamp" : "c" + std::to_string(f));
    layout_.formats.push_back(f == ts_col_ ? "tsn:" : "l");
  }
  open_device(c);
  counters_.alloc(sizeof(WCounters));
  AB_CUDA(cudaMemsetAsync(counters_.p, 0, sizeof(WCounters), stream_));
  cap_ = 1u << 16;
  alloc_store(cur_, cap_);
  AB_CUDA(cudaStreamSynchronize(stream_));
}

// The frame clause: refusals as DataFusion's planner refuses them (INVALID_ARGUMENT), a start after the end, which
// SQLite refuses and nothing here pins, UNSUPPORTED; a frame equal to the default is kept as units 0, so that it runs
// the default frame's kernels and gives their bits.
void WindowFnOp::check_frame(const ArroyoB200WindowFrame& f) {
  AB_REQUIRE(f.units >= ARROYO_B200_FRAME_DEFAULT && f.units <= ARROYO_B200_FRAME_GROUPS, ARROYO_B200_INVALID_ARGUMENT,
             "window function: frame.units must be DEFAULT (0), ROWS (1), RANGE (2) or GROUPS (3)");
  if (f.units == ARROYO_B200_FRAME_DEFAULT) return;
  const bool takes_frame = fn_ == ARROYO_B200_FN_AGGREGATE || fn_ == ARROYO_B200_FN_FIRST_VALUE ||
                           fn_ == ARROYO_B200_FN_LAST_VALUE || fn_ == ARROYO_B200_FN_NTH_VALUE;
  AB_REQUIRE(takes_frame, ARROYO_B200_INVALID_ARGUMENT,
             std::string("window function: ") + fn_name() + " takes no frame (frame.units must be 0)");
  auto bound_ok = [](int k) {
    return k >= ARROYO_B200_BOUND_UNBOUNDED_PRECEDING && k <= ARROYO_B200_BOUND_UNBOUNDED_FOLLOWING;
  };
  AB_REQUIRE(bound_ok(f.start_kind) && bound_ok(f.end_kind), ARROYO_B200_INVALID_ARGUMENT,
             "window function: frame.start_kind / end_kind must be ArroyoB200FrameBound codes (1 to 5)");
  AB_REQUIRE(f.start_kind != ARROYO_B200_BOUND_UNBOUNDED_FOLLOWING, ARROYO_B200_INVALID_ARGUMENT,
             "window function: a frame cannot start at UNBOUNDED FOLLOWING");
  AB_REQUIRE(f.end_kind != ARROYO_B200_BOUND_UNBOUNDED_PRECEDING, ARROYO_B200_INVALID_ARGUMENT,
             "window function: a frame cannot end at UNBOUNDED PRECEDING");
  auto offset = [](int k) { return k == ARROYO_B200_BOUND_PRECEDING || k == ARROYO_B200_BOUND_FOLLOWING; };
  AB_REQUIRE((!offset(f.start_kind) || f.start_offset >= 0) && (!offset(f.end_kind) || f.end_offset >= 0),
             ARROYO_B200_INVALID_ARGUMENT, "window function: a frame offset must be >= 0");
  AB_REQUIRE(f.units != ARROYO_B200_FRAME_RANGE || !(offset(f.start_kind) || offset(f.end_kind)) || n_order_ == 1,
             ARROYO_B200_INVALID_ARGUMENT, "window function: a RANGE frame with an offset takes exactly one ORDER BY key");
  AB_REQUIRE(f.units != ARROYO_B200_FRAME_GROUPS || n_order_ >= 1, ARROYO_B200_INVALID_ARGUMENT,
             "window function: a GROUPS frame takes an ORDER BY");
  const bool after = (f.start_kind == ARROYO_B200_BOUND_FOLLOWING && (f.end_kind == ARROYO_B200_BOUND_CURRENT_ROW ||
                                                                     f.end_kind == ARROYO_B200_BOUND_PRECEDING)) ||
                     (f.start_kind == ARROYO_B200_BOUND_CURRENT_ROW && f.end_kind == ARROYO_B200_BOUND_PRECEDING);
  AB_REQUIRE(!after, ARROYO_B200_UNSUPPORTED,
             "window function: a frame that starts after its end (n FOLLOWING AND CURRENT ROW | m PRECEDING, CURRENT "
             "ROW AND m PRECEDING) is not supported");
  const bool is_default =
      n_order_ > 0 ? f.units == ARROYO_B200_FRAME_RANGE && f.start_kind == ARROYO_B200_BOUND_UNBOUNDED_PRECEDING &&
                         f.end_kind == ARROYO_B200_BOUND_CURRENT_ROW
                   : f.start_kind == ARROYO_B200_BOUND_UNBOUNDED_PRECEDING &&
                         f.end_kind == ARROYO_B200_BOUND_UNBOUNDED_FOLLOWING;
  if (!is_default) frame_ = f;
}

// The flat layout of an imported batch: names and formats per flat column, and its struct columns.
WindowFnOp::Layout WindowFnOp::layout_of(const std::vector<InColumn>& cols, const std::vector<Nest>& nests,
                                         const ArrowSchema* s) const {
  Layout l;
  l.nests = nests;
  for (int64_t i = 0; i < s->n_children; ++i) {
    const ArrowSchema* cs = s->children[i];
    if (cs->format && !strcmp(cs->format, "+s")) {
      for (int64_t j = 0; j < cs->n_children; ++j) l.names.push_back(cs->children[j]->name ? cs->children[j]->name : "");
    } else {
      l.names.push_back(cs->name ? cs->name : "");
    }
  }
  for (const InColumn& c : cols) l.formats.push_back(c.format);
  return l;
}

// A batch's layout against the plan: its column count, the sort keys' types (`bad_type_status` when a key's type is
// not l, L or tsn:) and the argument's (an aggregate's not l, a value function's not l, L, g or tsn:), and, once the
// operator has its types, the same formats and struct columns.
void WindowFnOp::check_layout(const Layout& l, int bad_type_status) const {
  AB_REQUIRE((int)l.formats.size() == n_cols_, ARROYO_B200_INVALID_ARGUMENT,
             "window function: batch has " + std::to_string(l.formats.size()) + " flat columns, the plan " +
                 std::to_string(n_cols_));
  if (arg_col_ >= 0) {
    // an aggregate sums or compares Int64 values; a value function moves any 64-bit column of the operator unchanged
    const std::string& f = l.formats[arg_col_];
    const bool agg = fn_ == ARROYO_B200_FN_AGGREGATE;
    if (agg ? f != "l" : !(sortable_format(f) || f == "g"))
      throw Error(bad_type_status, "window function: " + std::string(fn_name()) + " argument of type '" + f +
                                       "' (supported: " + (agg ? "l" : "l, L, g, tsn:") + ")");
  }
  if (key_col_ >= 0 && !sortable_format(l.formats[key_col_]))
    throw Error(bad_type_status, "window function: PARTITION BY column of type '" + l.formats[key_col_] +
                                     "' (supported: l, L, tsn:)");
  for (int k = 0; k < n_order_; ++k)
    if (!sortable_format(l.formats[order_col_[k]]))
      throw Error(bad_type_status, "window function: ORDER BY column of type '" + l.formats[order_col_[k]] +
                                       "' (supported: l, L, tsn:; Float64 ordering is not supported)");
  if (!typed_) return;
  bool same = l.formats == layout_.formats && l.nests.size() == layout_.nests.size();
  for (size_t i = 0; same && i < l.nests.size(); ++i)
    same = l.nests[i].first == layout_.nests[i].first && l.nests[i].names.size() == layout_.nests[i].names.size();
  AB_REQUIRE(same, ARROYO_B200_INVALID_ARGUMENT,
             "window function: batch layout (column types or struct columns) differs from the operator's input layout");
}

void WindowFnOp::adopt(const Layout& l) {
  if (typed_) return;
  layout_ = l;
  typed_ = true;
}

// The columns of an output or state batch in the input layout, struct columns re-nested: `data(f)` gives flat column
// f's pinned host buffer.
std::vector<OutColumn> WindowFnOp::host_columns(const std::function<void*(int)>& data) const {
  std::vector<OutColumn> cols;
  auto column = [&](int f) {
    OutColumn c;
    c.name = layout_.names[f];
    c.format = layout_.formats[f];
    c.data = data(f);
    return c;
  };
  for (int f = 0; f < n_cols_;) {
    const Nest* nest = nullptr;
    for (const Nest& x : layout_.nests)
      if (x.first == f) nest = &x;
    if (!nest) {
      cols.push_back(column(f++));
      continue;
    }
    OutColumn s;
    s.name = nest->name;
    s.format = "+s";
    for (size_t k = 0; k < nest->names.size(); ++k) s.children.push_back(column(f + (int)k));
    cols.push_back(s);
    f += (int)nest->names.size();
  }
  return cols;
}

void WindowFnOp::alloc_store(Store& s, uint64_t cap) const {
  for (int c = 0; c < n_cols_; ++c) s.col[c].alloc(cap * 8);
}

// Reads the counters (waits for the stream): the stored rows, the late rows, and a negative timestamp, on which the
// reference panics.
void WindowFnOp::read_counters() {
  WCounters c{};
  AB_CUDA(cudaMemcpyAsync(&c, counters_.p, sizeof c, cudaMemcpyDeviceToHost, stream_));
  AB_CUDA(cudaStreamSynchronize(stream_));
  n_store_ = store_hi_ = c.n_store;
  st_.rows_late = c.late;
  if (c.neg_ts) {
    AB_CUDA(cudaMemsetAsync(&counters()->neg_ts, 0, 4, stream_));
    AB_CUDA(cudaStreamSynchronize(stream_));
    throw Error(ARROYO_B200_PANIC, "batch holds a negative _timestamp (before the Unix epoch): the reference panics on it");
  }
}

// Room for `more` rows: the bound is tightened from the device's count before the store doubles.  Past 2^31 rows the
// call is refused before anything changes.
void WindowFnOp::reserve_rows(uint64_t more) {
  if (store_hi_ + more <= cap_) return;
  read_counters();
  AB_REQUIRE(n_store_ + more <= WF_MAX_ROWS, ARROYO_B200_RUNTIME, "window function: more than 2^31 buffered rows");
  if (n_store_ + more <= cap_) return;
  uint64_t nc = cap_ * 2;
  while (nc < n_store_ + more) nc *= 2;
  nc = std::min<uint64_t>(nc, WF_MAX_ROWS);
  Store ns;
  alloc_store(ns, nc);
  for (int c = 0; c < n_cols_; ++c)
    if (n_store_) AB_CUDA(cudaMemcpyAsync(ns.col[c].p, cur_.col[c].p, n_store_ * 8, cudaMemcpyDeviceToDevice, stream_));
  AB_CUDA(cudaStreamSynchronize(stream_));
  cur_ = std::move(ns);
  alt_ = Store();
  cap_ = nc;
}

// Copies the `n` rows of a host batch's flat columns to the device; `ptrs` receives the device columns.  The host batch
// must outlive the copies.
const unsigned long long* const* WindowFnOp::stage(const std::vector<InColumn>& cols, int64_t n,
                                                   const unsigned long long** ptrs) {
  if ((uint64_t)n > stage_cap_) {
    AB_CUDA(cudaStreamSynchronize(stream_));
    stage_cap_ = std::max<uint64_t>((uint64_t)n, stage_cap_ * 2);
    stage_.alloc((size_t)n_cols_ * stage_cap_ * 8);
  }
  for (int c = 0; c < n_cols_; ++c) {
    unsigned long long* d = stage_.as<unsigned long long>() + (size_t)c * stage_cap_;
    AB_CUDA(cudaMemcpyAsync(d, cols[c].data, (size_t)n * 8, cudaMemcpyHostToDevice, stream_));
    ptrs[c] = d;
  }
  st_.h2d_bytes += (uint64_t)n * 8 * (uint64_t)n_cols_;
  return ptrs;
}

// Appends the rows of device columns `cols` with ts >= late_wm (and ts >= 0) to the store, in order.
void WindowFnOp::ingest(const unsigned long long* const* cols, int64_t n, long long late_wm) {
  reserve_rows((uint64_t)n);
  reserve(flag_, (size_t)n * 4);
  reserve(off_, (size_t)n * 8);
  wf_flag_kernel<<<grid_for((uint64_t)n), WF_THREADS, 0, stream_>>>((const long long*)cols[ts_col_], n, late_wm,
                                                                      flag_.as<unsigned int>(), counters());
  AB_CUDA(cudaGetLastError());
  device_exclusive_scan(flag_.as<unsigned int>(), n, off_.as<unsigned long long>(), &counters()->total, sums_, stream_);
  WAppend p{};
  for (int c = 0; c < n_cols_; ++c) {
    p.in[c] = cols[c];
    p.store.c[c] = cur_.col[c].as<unsigned long long>();
  }
  p.n_cols = n_cols_;
  p.flag = flag_.as<unsigned int>();
  p.off = off_.as<unsigned long long>();
  p.n = n;
  p.n_store = &counters()->n_store;
  wf_append_kernel<<<grid_for((uint64_t)n), WF_THREADS, 0, stream_>>>(p);
  AB_CUDA(cudaGetLastError());
  wf_advance_kernel<<<1, 1, 0, stream_>>>(counters());
  AB_CUDA(cudaGetLastError());
  st_.kernel_launches += 6;
  ++st_.ingest_launches;
  store_hi_ += (uint64_t)n;
}

void WindowFnOp::process_batch(uint32_t, uint32_t, ArrowArray* batch, const ArrowSchema* schema) {
  set_device();
  int64_t n = 0;
  std::vector<Nest> nests;
  const std::vector<InColumn> cols = import_batch(batch, schema, &n, -1, &nests);
  const Layout l = layout_of(cols, nests, schema);
  check_layout(l, ARROYO_B200_UNSUPPORTED);
  adopt(l);
  st_.rows_in += (uint64_t)n;
  if (n > 0) {
    const unsigned long long* ptrs[ARROYO_B200_MAX_COLS];
    ingest(stage(cols, n, ptrs), n, late_wm_);
    // the staging buffer is reused by the next batch, and a negative timestamp is reported with this batch
    read_counters();
  }
  if (batch->release) batch->release(batch);
  batch->release = nullptr;
}

void WindowFnOp::process_device_batch(uint32_t, uint32_t, const uint64_t* cols, int32_t n_cols, int64_t n_rows) {
  set_device();
  AB_REQUIRE(n_cols == n_cols_, ARROYO_B200_INVALID_ARGUMENT, "batch has the wrong number of columns");
  if (n_rows <= 0) return;
  st_.rows_in += (uint64_t)n_rows;
  ingest((const unsigned long long* const*)cols, n_rows, late_wm_);
}

// What a sort key's 64 bits are XORed with to sort as unsigned: the sign bit for signed types, every bit for DESC.
unsigned long long WindowFnOp::flip_of(int col, bool desc) const {
  const unsigned long long f = layout_.formats[col] == "L" ? 0ull : 1ull << 63;
  return desc ? ~f : f;
}

// Sorts the `e` store indices in idx_[0] and returns the buffer holding the sorted ones: stable LSD radix passes from
// arrival order, the ORDER BY keys last to first, the partition key, then `_timestamp` (`by_ts_only`: that pass alone).
unsigned int* WindowFnOp::sort_rows(uint64_t e, bool by_ts_only) {
  reserve(idx_[1], e * 4);
  reserve(key_[0], e * 8);
  reserve(key_[1], e * 8);
  struct Pass {
    int col;
    unsigned long long flip;
    int end_bit;
  };
  std::vector<Pass> passes;
  if (!by_ts_only) {
    for (int k = n_order_ - 1; k >= 0; --k) passes.push_back({order_col_[k], flip_of(order_col_[k], order_desc_[k]), 64});
    if (key_col_ >= 0) passes.push_back({key_col_, flip_of(key_col_, false), 64});
  }
  passes.push_back({ts_col_, 0ull, 63});  // timestamps are >= 0: bit 63 is never set
  cub::DoubleBuffer<unsigned long long> keys(key_[0].as<unsigned long long>(), key_[1].as<unsigned long long>());
  cub::DoubleBuffer<unsigned int> vals(idx_[0].as<unsigned int>(), idx_[1].as<unsigned int>());
  size_t tmp = 0;
  AB_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, tmp, keys, vals, (int64_t)e, 0, 64, stream_));
  reserve(cub_tmp_, std::max<size_t>(tmp, 1));
  for (const Pass& ps : passes) {
    // the keys of the rows in their current order
    wf_key_kernel<<<grid_for(e), WF_THREADS, 0, stream_>>>(cur_.col[ps.col].as<unsigned long long>(), vals.Current(),
                                                           (long long)e, ps.flip, keys.Current());
    AB_CUDA(cudaGetLastError());
    tmp = cub_tmp_.bytes;
    AB_CUDA(cub::DeviceRadixSort::SortPairs(cub_tmp_.p, tmp, keys, vals, (int64_t)e, 0, ps.end_bit, stream_));
    st_.kernel_launches += 2;
  }
  return vals.Current();
}

// handle_watermark (:178-201): every instant below `wm` leaves, in ascending order, and its rows are freed.
void WindowFnOp::handle_watermark(int64_t wm, BatchesPriv* out_host, std::vector<ArroyoB200DeviceBatch>*) {
  set_device();
  AB_REQUIRE(out_host != nullptr, ARROYO_B200_UNSUPPORTED, "window function: device-resident output is not implemented");
  read_counters();
  if (n_store_ > 0 && wm != LLONG_MIN) emit(wm, out_host);
  late_wm_ = std::max<int64_t>(late_wm_, wm);
}

void WindowFnOp::emit(int64_t w, BatchesPriv* out) {
  const uint64_t n = n_store_;
  reserve(flag_, n * 4);
  reserve(off_, n * 8);
  wf_mark_kernel<<<grid_for(n), WF_THREADS, 0, stream_>>>(cur_.col[ts_col_].as<long long>(), (long long)n, w,
                                                          flag_.as<unsigned int>());
  AB_CUDA(cudaGetLastError());
  device_exclusive_scan(flag_.as<unsigned int>(), (int64_t)n, off_.as<unsigned long long>(), &counters()->total, sums_,
                        stream_);
  st_.kernel_launches += 4;
  unsigned long long e = 0, below = 0;  // rows leaving; of them, rows below the checkpoint boundary
  AB_CUDA(cudaMemcpyAsync(&e, &counters()->total, 8, cudaMemcpyDeviceToHost, stream_));
  if (ckpt_from_ < n)
    AB_CUDA(cudaMemcpyAsync(&below, off_.as<unsigned long long>() + ckpt_from_, 8, cudaMemcpyDeviceToHost, stream_));
  AB_CUDA(cudaStreamSynchronize(stream_));
  if (e == 0) return;
  if (ckpt_from_ >= n) below = e;

  // the leaving rows, sorted
  reserve(idx_[0], e * 4);
  wf_select_kernel<<<grid_for(n), WF_THREADS, 0, stream_>>>(flag_.as<unsigned int>(), off_.as<unsigned long long>(),
                                                            (long long)n, idx_[0].as<unsigned int>());
  AB_CUDA(cudaGetLastError());
  ++st_.kernel_launches;
  const unsigned int* idx = sort_rows(e, false);

  // ranks and the fused filter, the aggregate, or a value function
  const bool agg = fn_ == ARROYO_B200_FN_AGGREGATE, rank = ranking();
  const uint64_t n_tiles = (e + WF_TILE - 1) / WF_TILE;
  reserve(bits_, e);
  reserve(tiles_, n_tiles * sizeof(RankVal));
  reserve(fnv_, e * 8);
  if (rank) {
    reserve(keep_, e * 4);
    reserve(off2_, e * 8);
  }
  AB_CUDA(cudaMemsetAsync(&counters()->instants, 0, 8, stream_));
  WRank r{};
  r.col[0] = cur_.col[ts_col_].as<unsigned long long>();
  r.n_col = 1;
  if (key_col_ >= 0) r.col[r.n_col++] = cur_.col[key_col_].as<unsigned long long>();
  for (int k = 0; k < n_order_; ++k) r.col[r.n_col++] = cur_.col[order_col_[k]].as<unsigned long long>();
  r.keyed = key_col_ >= 0 ? 1 : 0;
  r.idx = idx;
  r.n = (long long)e;
  r.bits = bits_.as<unsigned char>();
  r.tiles = tiles_.as<RankVal>();
  r.instants = &counters()->instants;
  r.fn = fn_;
  r.top_n = top_n_;
  r.fn_out = fnv_.as<unsigned long long>();
  r.keep = keep_.as<unsigned int>();
  wf_rank_flags_kernel<<<(unsigned)n_tiles, WF_TILE, 0, stream_>>>(r);
  AB_CUDA(cudaGetLastError());
  wf_carry_kernel<RankVal><<<1, 1024, 0, stream_>>>(r.tiles, (long long)n_tiles);
  AB_CUDA(cudaGetLastError());
  unsigned long long m = e, n_inst = 0;
  const bool frame = frame_.units != ARROYO_B200_FRAME_DEFAULT;
  if (frame) {
    framed(r, n_tiles);  // every row leaves
  } else if (agg) {
    aggregate(r, n_tiles);  // every row leaves
  } else if (!rank) {
    values(r, n_tiles);  // every row leaves
  } else {
    wf_rank_apply_kernel<<<(unsigned)n_tiles, WF_TILE, 0, stream_>>>(r);
    AB_CUDA(cudaGetLastError());
    device_exclusive_scan(keep_.as<unsigned int>(), (int64_t)e, off2_.as<unsigned long long>(), &counters()->total,
                          sums_, stream_);
    st_.kernel_launches += 6;
    AB_CUDA(cudaMemcpyAsync(&m, &counters()->total, 8, cudaMemcpyDeviceToHost, stream_));
  }
  AB_CUDA(cudaMemcpyAsync(&n_inst, &counters()->instants, 8, cudaMemcpyDeviceToHost, stream_));
  AB_CUDA(cudaStreamSynchronize(stream_));

  // the kept rows, in sorted order
  if (m > 0) {
    WGather g{};
    for (int c = 0; c < n_cols_; ++c) {
      reserve(out_[c], m * 8);
      g.store[c] = cur_.col[c].as<unsigned long long>();
      g.out.c[c] = out_[c].as<unsigned long long>();
    }
    reserve(out_fn_, m * 8);
    g.n_cols = n_cols_;
    g.idx = idx;
    g.keep = rank ? keep_.as<unsigned int>() : nullptr;
    g.off = rank ? off2_.as<unsigned long long>() : nullptr;
    g.fn = fnv_.as<unsigned long long>();
    g.at = agg && !frame ? at_.as<unsigned int>() : nullptr;
    g.fn_out = out_fn_.as<unsigned long long>();
    if (null_rows()) {
      reserve(out_valid_, m);
      g.valid = valid_.as<unsigned char>();
      g.valid_out = out_valid_.as<unsigned char>();
    }
    g.n = (long long)e;
    wf_gather_kernel<<<grid_for(e), WF_THREADS, 0, stream_>>>(g);
    AB_CUDA(cudaGetLastError());
    ++st_.kernel_launches;
    ++st_.emit_launches;
    std::vector<OutColumn> cols =
        host_columns([&](int f) { return d2h_pinned(out_[f].p, (size_t)m * 8, stream_, &st_.d2h_bytes); });
    OutColumn fc;
    fc.name = fn_name();
    fc.format = fn_format();
    fc.data = d2h_pinned(out_fn_.p, (size_t)m * 8, stream_, &st_.d2h_bytes);
    fc.nullable = nullable();
    if (g.valid) {
      reserve(out_bits_, (size_t)((m + 31) / 32) * 4);
      export_validity(fc, out_valid_.as<unsigned char>(), (int64_t)m, out_bits_.as<unsigned int>(), grid_for(m),
                      WF_THREADS, stream_, st_);
    }
    cols.push_back(fc);
    out->arrays.emplace_back();
    out->schemas.emplace_back();
    export_batch(cols, (int64_t)m, &out->arrays.back(), &out->schemas.back());
  }

  // the rows that stay, to the front of the store
  const uint64_t open = n - e;
  if (open) {
    if (!alt_.col[0].p) alloc_store(alt_, cap_);
    WCompact p{};
    for (int c = 0; c < n_cols_; ++c) {
      p.from[c] = cur_.col[c].as<unsigned long long>();
      p.to.c[c] = alt_.col[c].as<unsigned long long>();
    }
    p.n_cols = n_cols_;
    p.flag = flag_.as<unsigned int>();
    p.off = off_.as<unsigned long long>();
    p.n = (long long)n;
    wf_compact_kernel<<<grid_for(n), WF_THREADS, 0, stream_>>>(p);
    AB_CUDA(cudaGetLastError());
    ++st_.kernel_launches;
    std::swap(cur_, alt_);
  }
  wf_set_rows_kernel<<<1, 1, 0, stream_>>>(counters(), open);
  AB_CUDA(cudaGetLastError());
  ++st_.kernel_launches;
  AB_CUDA(cudaStreamSynchronize(stream_));  // the batch's copies have completed
  n_store_ = store_hi_ = open;
  ckpt_from_ -= std::min<uint64_t>(ckpt_from_, below);
  st_.rows_out += m;
  st_.windows_out += n_inst;
}

// The aggregate's segmented scan over the `r.n` sorted rows (after wf_rank_flags and the rank tiles' carry): fnv_ gets
// each peer group's value at its first row, at_ each row's group.
void WindowFnOp::aggregate(const WRank& r, uint64_t n_tiles) {
  reserve(agg_tiles_, n_tiles * 16);  // sizeof(AggVal<K>) for every K
  reserve(at_, (size_t)r.n * 4);
  WAgg p{};
  p.arg = arg_col_ >= 0 ? cur_.col[arg_col_].as<unsigned long long>() : nullptr;
  p.idx = r.idx;
  p.bits = r.bits;
  p.n = r.n;
  p.rank_tiles = r.tiles;
  p.tiles = agg_tiles_.p;
  p.fv = fnv_.as<unsigned long long>();
  p.at = at_.as<unsigned int>();
  switch (agg_kind_) {
    case ARROYO_B200_AGG_COUNT_STAR: launch_aggregate<ARROYO_B200_AGG_COUNT_STAR>(p, n_tiles, stream_); break;
    case ARROYO_B200_AGG_SUM_I64: launch_aggregate<ARROYO_B200_AGG_SUM_I64>(p, n_tiles, stream_); break;
    case ARROYO_B200_AGG_AVG_I64: launch_aggregate<ARROYO_B200_AGG_AVG_I64>(p, n_tiles, stream_); break;
    case ARROYO_B200_AGG_MIN_I64: launch_aggregate<ARROYO_B200_AGG_MIN_I64>(p, n_tiles, stream_); break;
    default: launch_aggregate<ARROYO_B200_AGG_MAX_I64>(p, n_tiles, stream_); break;
  }
  st_.kernel_launches += 5;  // with wf_rank_flags and the rank tiles' carry
}

// A value function, PERCENT_RANK or CUME_DIST over the `r.n` sorted rows (after wf_rank_flags and the rank tiles'
// carry): fnv_ gets each row's value and, when the function can give NULL, valid_ its validity.  at_ holds each peer
// group's last row, seg_last_ each segment's, at their first rows.
void WindowFnOp::values(const WRank& r, uint64_t n_tiles) {
  reserve(at_, (size_t)r.n * 4);
  reserve(seg_last_, (size_t)r.n * 4);
  WValue p{};
  p.arg = arg_col_ >= 0 ? cur_.col[arg_col_].as<unsigned long long>() : nullptr;
  p.idx = r.idx;
  p.bits = r.bits;
  p.n = r.n;
  p.rank_tiles = r.tiles;
  p.peer_last = at_.as<unsigned int>();
  p.seg_last = seg_last_.as<unsigned int>();
  p.fn = fn_;
  p.offset = offset_;
  p.dflt = dflt_;
  p.fv = fnv_.as<unsigned long long>();
  if (null_rows()) {
    reserve(valid_, (size_t)r.n);
    p.valid = valid_.as<unsigned char>();
  }
  wf_bounds_kernel<<<(unsigned)n_tiles, WF_TILE, 0, stream_>>>(p);
  AB_CUDA(cudaGetLastError());
  wf_value_apply_kernel<<<(unsigned)n_tiles, WF_TILE, 0, stream_>>>(p);
  AB_CUDA(cudaGetLastError());
  st_.kernel_launches += 4;  // with wf_rank_flags and the rank tiles' carry
}

// An aggregate or value function over the explicit frame (after wf_rank_flags and the rank tiles' carry): fnv_ gets
// each row's value and, unless the function is COUNT, valid_ its validity.  at_ holds each peer group's last row,
// seg_last_ each segment's, at their first rows.  The key buffers are free after the sort: key_[0] holds the RANGE
// key, key_[1] the split values of SUM / AVG or the sorted values of MIN / MAX.
void WindowFnOp::framed(const WRank& r, uint64_t n_tiles) {
  const uint64_t n = (uint64_t)r.n;
  reserve(at_, n * 4);
  reserve(seg_last_, n * 4);
  WFrame p{};
  WValue& b = p.b;
  b.arg = arg_col_ >= 0 ? cur_.col[arg_col_].as<unsigned long long>() : nullptr;
  b.idx = r.idx;
  b.bits = r.bits;
  b.n = r.n;
  b.rank_tiles = r.tiles;
  b.peer_last = at_.as<unsigned int>();
  b.seg_last = seg_last_.as<unsigned int>();
  b.fn = fn_;
  b.offset = offset_;
  b.fv = fnv_.as<unsigned long long>();
  if (null_rows()) {
    reserve(valid_, n);
    b.valid = valid_.as<unsigned char>();
  }
  p.units = frame_.units;
  p.start_kind = frame_.start_kind;
  p.end_kind = frame_.end_kind;
  p.start_off = (unsigned long long)frame_.start_offset;
  p.end_off = (unsigned long long)frame_.end_offset;
  wf_bounds_kernel<<<(unsigned)n_tiles, WF_TILE, 0, stream_>>>(b);
  AB_CUDA(cudaGetLastError());
  st_.kernel_launches += 4;  // with wf_rank_flags, the rank tiles' carry and the apply pass
  if (frame_.units == ARROYO_B200_FRAME_GROUPS) {
    reserve(gfirst_, n * 4);
    reserve(gcount_, n * 4);
    p.gfirst = gfirst_.as<unsigned int>();
    p.gcount = gcount_.as<unsigned int>();
    wf_groups_kernel<<<(unsigned)n_tiles, WF_TILE, 0, stream_>>>(p);
    AB_CUDA(cudaGetLastError());
    ++st_.kernel_launches;
  }
  auto offset = [](int k) { return k == ARROYO_B200_BOUND_PRECEDING || k == ARROYO_B200_BOUND_FOLLOWING; };
  if (frame_.units == ARROYO_B200_FRAME_RANGE && (offset(frame_.start_kind) || offset(frame_.end_kind))) {
    wf_key_kernel<<<grid_for(n), WF_THREADS, 0, stream_>>>(cur_.col[order_col_[0]].as<unsigned long long>(), r.idx,
                                                           r.n, flip_of(order_col_[0], order_desc_[0]),
                                                           key_[0].as<unsigned long long>());
    AB_CUDA(cudaGetLastError());
    ++st_.kernel_launches;
    p.ukey = key_[0].as<unsigned long long>();
  }
  const int kind = fn_ == ARROYO_B200_FN_AGGREGATE ? agg_kind_ : 0;
  if (kind == ARROYO_B200_AGG_SUM_I64 || kind == ARROYO_B200_AGG_AVG_I64) {
    // two exact prefix sums of 32-bit parts, each below 2^63 over 2^31 rows
    reserve(pre_, (n + 1) * 16);
    unsigned long long* lo = pre_.as<unsigned long long>();
    unsigned long long* hi = lo + n + 1;
    unsigned int* parts = key_[1].as<unsigned int>();
    wf_split_kernel<<<grid_for(n), WF_THREADS, 0, stream_>>>(b.arg, r.idx, r.n, parts, parts + n);
    AB_CUDA(cudaGetLastError());
    device_exclusive_scan(parts, (int64_t)n, lo, lo + n, sums_, stream_);
    device_exclusive_scan(parts + n, (int64_t)n, hi, hi + n, sums_, stream_);
    st_.kernel_launches += 7;
    p.pre_lo = lo;
    p.pre_hi = hi;
  } else if (kind == ARROYO_B200_AGG_MIN_I64 || kind == ARROYO_B200_AGG_MAX_I64) {
    WRmq q{};
    q.arg = b.arg;
    q.idx = r.idx;
    q.n = r.n;
    q.n_blocks = (long long)((n + 31) / 32);
    int levels = 1;
    while ((1ll << levels) <= q.n_blocks) ++levels;
    reserve(rmq_, n * 16);
    reserve(table_, (size_t)q.n_blocks * levels * 8);
    q.v = key_[1].as<long long>();
    q.in_pre = rmq_.as<long long>();
    q.in_suf = q.in_pre + n;
    q.table = table_.as<long long>();
    const bool mn = kind == ARROYO_B200_AGG_MIN_I64;
    const unsigned grid = (unsigned)((n + WF_THREADS - 1) / WF_THREADS);
    if (mn) wf_rmq_blocks_kernel<ARROYO_B200_AGG_MIN_I64><<<grid, WF_THREADS, 0, stream_>>>(q);
    else wf_rmq_blocks_kernel<ARROYO_B200_AGG_MAX_I64><<<grid, WF_THREADS, 0, stream_>>>(q);
    AB_CUDA(cudaGetLastError());
    for (int k = 1; k < levels; ++k) {
      const int lg = grid_for((uint64_t)q.n_blocks);
      if (mn) wf_rmq_level_kernel<ARROYO_B200_AGG_MIN_I64><<<lg, WF_THREADS, 0, stream_>>>(q.table, q.n_blocks, k);
      else wf_rmq_level_kernel<ARROYO_B200_AGG_MAX_I64><<<lg, WF_THREADS, 0, stream_>>>(q.table, q.n_blocks, k);
      AB_CUDA(cudaGetLastError());
    }
    st_.kernel_launches += (uint64_t)levels;
    p.v = q.v;
    p.in_pre = q.in_pre;
    p.in_suf = q.in_suf;
    p.table = q.table;
    p.n_blocks = q.n_blocks;
  }
  const unsigned grid = (unsigned)n_tiles;
  switch (fn_ == ARROYO_B200_FN_AGGREGATE ? agg_kind_ : fn_) {
    case ARROYO_B200_AGG_COUNT_STAR: wf_frame_apply_kernel<ARROYO_B200_AGG_COUNT_STAR><<<grid, WF_TILE, 0, stream_>>>(p); break;
    case ARROYO_B200_AGG_SUM_I64: wf_frame_apply_kernel<ARROYO_B200_AGG_SUM_I64><<<grid, WF_TILE, 0, stream_>>>(p); break;
    case ARROYO_B200_AGG_AVG_I64: wf_frame_apply_kernel<ARROYO_B200_AGG_AVG_I64><<<grid, WF_TILE, 0, stream_>>>(p); break;
    case ARROYO_B200_AGG_MIN_I64: wf_frame_apply_kernel<ARROYO_B200_AGG_MIN_I64><<<grid, WF_TILE, 0, stream_>>>(p); break;
    case ARROYO_B200_AGG_MAX_I64: wf_frame_apply_kernel<ARROYO_B200_AGG_MAX_I64><<<grid, WF_TILE, 0, stream_>>>(p); break;
    case ARROYO_B200_FN_FIRST_VALUE: wf_frame_apply_kernel<ARROYO_B200_FN_FIRST_VALUE><<<grid, WF_TILE, 0, stream_>>>(p); break;
    case ARROYO_B200_FN_LAST_VALUE: wf_frame_apply_kernel<ARROYO_B200_FN_LAST_VALUE><<<grid, WF_TILE, 0, stream_>>>(p); break;
    default: wf_frame_apply_kernel<ARROYO_B200_FN_NTH_VALUE><<<grid, WF_TILE, 0, stream_>>>(p); break;
  }
  AB_CUDA(cudaGetLastError());
}

// handle_checkpoint: table "input" gets the rows accepted since the previous checkpoint, one batch per instant in
// ascending order, each in arrival order and in the input layout (the reference flushes the batches it inserted under
// their instants since then).
void WindowFnOp::handle_checkpoint(int64_t, BatchesPriv* out) {
  set_device();
  read_counters();
  const uint64_t n = n_store_;
  if (n <= ckpt_from_) return;
  const uint64_t d = n - ckpt_from_;
  reserve(idx_[0], d * 4);
  wf_iota_kernel<<<grid_for(d), WF_THREADS, 0, stream_>>>(idx_[0].as<unsigned int>(), (unsigned int)ckpt_from_,
                                                          (long long)d);
  AB_CUDA(cudaGetLastError());
  ++st_.kernel_launches;
  const unsigned int* idx = sort_rows(d, true);
  WGather g{};
  for (int c = 0; c < n_cols_; ++c) {
    reserve(out_[c], d * 8);
    g.store[c] = cur_.col[c].as<unsigned long long>();
    g.out.c[c] = out_[c].as<unsigned long long>();
  }
  g.n_cols = n_cols_;
  g.idx = idx;
  g.n = (long long)d;
  wf_gather_kernel<<<grid_for(d), WF_THREADS, 0, stream_>>>(g);
  AB_CUDA(cudaGetLastError());
  ++st_.kernel_launches;
  // the columns once, on the host; each instant's rows are then a slice of them
  std::vector<void*> flat(n_cols_);
  for (int c = 0; c < n_cols_; ++c) flat[c] = d2h_pinned(out_[c].p, (size_t)d * 8, stream_, &st_.d2h_bytes);
  AB_CUDA(cudaStreamSynchronize(stream_));
  const uint64_t* ts = (const uint64_t*)flat[ts_col_];
  for (uint64_t s = 0; s < d;) {
    uint64_t e = s + 1;
    while (e < d && ts[e] == ts[s]) ++e;
    const std::vector<OutColumn> cols = host_columns([&](int f) {
      void* p = PinnedPool::get().alloc((size_t)(e - s) * 8);
      memcpy(p, (const uint64_t*)flat[f] + s, (size_t)(e - s) * 8);
      return p;
    });
    out->arrays.emplace_back();
    out->schemas.emplace_back();
    export_batch(cols, (int64_t)(e - s), &out->arrays.back(), &out->schemas.back());
    s = e;
  }
  for (void* p : flat) PinnedPool::get().free(p);
  ckpt_from_ = n;
}

// on_start (:130-145): the batches of table "input", in any order, appended to the store ahead of any later row and not
// late-filtered.  Every batch is checked against the input layout first: one that does not match => INVALID_ARGUMENT,
// nothing changed.  The restored watermark is the late watermark.
void WindowFnOp::on_start(ArrowArray* state, ArrowSchema* schemas, int64_t n, int64_t watermark, int64_t) {
  set_device();
  if (n > 0) AB_REQUIRE(state != nullptr && schemas != nullptr, ARROYO_B200_INVALID_ARGUMENT, "null state batches");
  std::vector<std::vector<InColumn>> cols((size_t)std::max<int64_t>(n, 0));
  std::vector<int64_t> rows(cols.size(), 0);
  uint64_t total = 0;
  Layout first;
  for (size_t b = 0; b < cols.size(); ++b) {
    std::vector<Nest> nests;
    Layout l;
    try {
      cols[b] = import_batch(&state[b], &schemas[b], &rows[b], -1, &nests);
      l = layout_of(cols[b], nests, &schemas[b]);
      check_layout(l, ARROYO_B200_INVALID_ARGUMENT);
    } catch (const Error& e) {
      throw Error(ARROYO_B200_INVALID_ARGUMENT, std::string("state batch: ") + e.what());
    }
    if (b == 0) first = l;
    AB_REQUIRE(l.formats == first.formats && l.nests.size() == first.nests.size(), ARROYO_B200_INVALID_ARGUMENT,
               "state batch: layout differs from the first state batch's");
    total += (uint64_t)rows[b];
  }
  if (total > 0) reserve_rows(total);  // may refuse: nothing has changed yet
  if (n > 0) adopt(first);
  if (total > 0) {
    for (size_t b = 0; b < cols.size(); ++b) {
      if (!rows[b]) continue;
      const unsigned long long* ptrs[ARROYO_B200_MAX_COLS];
      ingest(stage(cols[b], rows[b], ptrs), rows[b], LLONG_MIN);
    }
    read_counters();
    ckpt_from_ = n_store_;  // the table already holds them
  }
  if (watermark != INT64_MIN) late_wm_ = std::max<int64_t>(late_wm_, watermark);
  for (int64_t b = 0; b < n; ++b)
    if (state[b].release) state[b].release(&state[b]);
}

}  // namespace

OpBase* make_window_fn_op(const ArroyoB200OpConfig& cfg) { return new WindowFnOp(cfg); }

}  // namespace ab
