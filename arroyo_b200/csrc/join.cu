// Instant (windowed) join on sm_90a (H100).
//
// Replaces InstantJoin (arroyo-worker/src/arrow/instant_join.rs:109-172 process_side, :241-283
// process_batch_index / handle_watermark) and the DataFusion HashJoinExec it runs once per window instant
// (K10).  Both inputs carry window-stamped rows: every row of a window has the same `_timestamp`, and only
// rows with equal `_timestamp` may join.  The reference keeps one join exec per distinct timestamp; here
// rows of both sides are appended to device arenas and, at a watermark, every row with
// `_timestamp < watermark` is joined in ONE build / probe pass on the composite key (_timestamp, key):
// equal timestamps are part of the equality, so the result is the union of the per-instant joins.
//
//   build   : right rows -> open-addressing table of row indices (CAS claim, linear probing)
//   count   : left rows walk their chain and count matches (outer joins: unmatched rows count 1)
//   scan    : exclusive prefix sum of the counts = output offsets
//   write   : left rows walk again and write (left idx, right idx) pairs; matched right rows are flagged
//   append  : right / full joins: unmatched right rows appended with left idx = -1
//   gather  : output columns materialised from the pairs (+ validity bytes for the missing side),
//             `_timestamp = max(l._timestamp, r._timestamp)` (arroyo-planner/src/plan/join.rs:165-185)
//   compact : rows with `_timestamp >= watermark` are kept for later watermarks
//
// Output = [left payload cols..., right payload cols..., _timestamp]; the leading `_key_*` routing copies
// of each side are stripped like `unkeyed_batch` does (arroyo-rpc/src/df.rs:359-367).
#include <algorithm>
#include <climits>

#include "op.h"
#include "scan.cuh"

namespace ab {
namespace {

constexpr int JT = 256;

__device__ __forceinline__ uint64_t pair_hash(long long key, long long ts) {
  return mix64((uint64_t)key ^ mix64((uint64_t)ts));
}

// eligible[i] = ts[i] < wm; also min timestamp of all rows (panic check) and the eligible count
__global__ void mark_kernel(const long long* __restrict__ ts, long long n, long long wm, unsigned char* __restrict__ elig,
                            unsigned long long* __restrict__ n_elig, long long* __restrict__ min_ts) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  long long stride = (long long)gridDim.x * blockDim.x;
  unsigned long long c = 0;
  long long mn = LLONG_MAX;
  for (; i < n; i += stride) {
    long long t = ts[i];
    bool e = t < wm;
    elig[i] = e ? 1 : 0;
    c += e ? 1 : 0;
    mn = min(mn, t);
  }
  for (int o = 16; o > 0; o >>= 1) {
    c += __shfl_xor_sync(0xffffffffu, c, o);
    mn = min(mn, __shfl_xor_sync(0xffffffffu, mn, o));
  }
  if ((threadIdx.x & 31) == 0) {
    if (c) atomicAdd(n_elig, c);
    if (mn != LLONG_MAX) atomicMin(min_ts, mn);
  }
}

// Build-side table: 16-byte slots {key, row + 1, low 32 bits of the timestamp}: one sector per probe step, the
// key compared exactly and the timestamp pre-filtered in the slot; the full timestamp of a candidate is read
// from the build column only when both agree.  row + 1 == 0 marks an empty slot.
struct alignas(16) JSlot {
  long long key;
  unsigned int row1;
  unsigned int ts_lo;
};

__global__ void build_kernel(const long long* __restrict__ key, const long long* __restrict__ ts,
                             const unsigned char* __restrict__ elig, long long n, JSlot* __restrict__ tab, uint32_t mask) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  long long stride = (long long)gridDim.x * blockDim.x;
  for (; i < n; i += stride) {
    if (!elig[i]) continue;
    const long long k = key[i], t = ts[i];
    uint32_t pos = (uint32_t)pair_hash(k, t) & mask;
    while (atomicCAS(&tab[pos].row1, 0u, (unsigned int)i + 1u) != 0u) pos = (pos + 1) & mask;
    // the probe runs in a later kernel: plain stores are enough for the rest of the slot
    tab[pos].key = k;
    tab[pos].ts_lo = (unsigned int)(unsigned long long)t;
  }
}

// pass 0: cnt[i] = number of output rows of probe row i; pass 1: write the pairs at off[i].
// out_p / out_b receive the probe-side / build-side row of each pair (-1 = none).
template <int PASS>
__global__ void probe_kernel(const long long* __restrict__ pkey, const long long* __restrict__ pts,
                             const unsigned char* __restrict__ pelig, long long n_probe,
                             const long long* __restrict__ bts, const JSlot* __restrict__ tab, uint32_t mask,
                             int keep_unmatched_probe, unsigned int* __restrict__ cnt,
                             const unsigned long long* __restrict__ off, int* __restrict__ out_p, int* __restrict__ out_b,
                             unsigned char* __restrict__ b_matched) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  long long stride = (long long)gridDim.x * blockDim.x;
  for (; i < n_probe; i += stride) {
    if (!pelig[i]) {
      if (PASS == 0) cnt[i] = 0;
      continue;
    }
    const long long k = pkey[i], t = pts[i];
    const unsigned int tlo = (unsigned int)(unsigned long long)t;
    uint32_t pos = (uint32_t)pair_hash(k, t) & mask;
    unsigned int c = 0;
    unsigned long long o = PASS == 1 ? off[i] : 0;
    while (true) {
      const ulonglong2 raw = __ldg(reinterpret_cast<const ulonglong2*>(tab + pos));
      const unsigned int row1 = (unsigned int)raw.y;
      if (row1 == 0) break;
      if ((long long)raw.x == k && (unsigned int)(raw.y >> 32) == tlo) {
        const unsigned int j = row1 - 1;
        if (__ldg(bts + j) == t) {
          if (PASS == 1) {
            out_p[o + c] = (int)i;
            out_b[o + c] = (int)j;
            b_matched[j] = 1;
          }
          ++c;
        }
      }
      pos = (pos + 1) & mask;
    }
    if (c == 0 && keep_unmatched_probe) {
      if (PASS == 1) {
        out_p[o] = (int)i;
        out_b[o] = -1;
      }
      c = 1;
    }
    if (PASS == 0) cnt[i] = c;
  }
}

// outer joins: eligible build-side rows nobody matched, appended after the probe output
__global__ void append_unmatched_kernel(const unsigned char* __restrict__ elig, const unsigned char* __restrict__ matched,
                                        long long n, unsigned long long* __restrict__ cursor, int* __restrict__ out_p,
                                        int* __restrict__ out_b) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  long long stride = (long long)gridDim.x * blockDim.x;
  for (; i < n; i += stride) {
    bool take = elig[i] && !matched[i];
    unsigned int b = __ballot_sync(__activemask(), take);
    if (!take) continue;
    int lane = threadIdx.x & 31;
    int leader = __ffs(b) - 1;
    unsigned long long base = 0;
    if (lane == leader) base = atomicAdd(cursor, (unsigned long long)__popc(b));
    base = __shfl_sync(b, base, leader);
    unsigned long long o = base + __popc(b & ((1u << lane) - 1u));
    out_p[o] = -1;
    out_b[o] = (int)i;
  }
}

struct GatherParams {
  const int* idx;          // pair side to read
  const long long* src;    // source column
  long long* dst;
  unsigned char* valid;    // optional validity bytes
  long long n;
};
__global__ void gather_kernel(const __grid_constant__ GatherParams p) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  long long stride = (long long)gridDim.x * blockDim.x;
  for (; i < p.n; i += stride) {
    int j = p.idx[i];
    p.dst[i] = j >= 0 ? p.src[j] : 0;
    if (p.valid) p.valid[i] = j >= 0 ? 1 : 0;
  }
}
__global__ void gather_ts_kernel(const int* __restrict__ il, const int* __restrict__ ir, const long long* __restrict__ lts,
                                 const long long* __restrict__ rts, long long* __restrict__ dst, long long n) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  long long stride = (long long)gridDim.x * blockDim.x;
  for (; i < n; i += stride) {
    int a = il[i], b = ir[i];
    long long ta = a >= 0 ? lts[a] : LLONG_MIN, tb = b >= 0 ? rts[b] : LLONG_MIN;
    dst[i] = max(ta, tb);
  }
}
// validity bytes -> Arrow validity bitmap (LSB first)
__global__ void pack_bits_kernel(const unsigned char* __restrict__ bytes, long long n, unsigned int* __restrict__ words) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  long long n_pad = (n + 31) / 32 * 32;
  long long stride = (long long)gridDim.x * blockDim.x;
  for (; i < n_pad; i += stride) {
    bool v = i < n && bytes[i];
    unsigned int b = __ballot_sync(0xffffffffu, v);
    if ((threadIdx.x & 31) == 0) words[i >> 5] = b;
  }
}
// keep[i] = !elig[i] as counts for the compaction scan
__global__ void keep_counts_kernel(const unsigned char* __restrict__ elig, long long n, unsigned int* __restrict__ cnt) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  long long stride = (long long)gridDim.x * blockDim.x;
  for (; i < n; i += stride) cnt[i] = elig[i] ? 0u : 1u;
}
__global__ void compact_kernel(const long long* __restrict__ src, const unsigned char* __restrict__ elig,
                               const unsigned long long* __restrict__ off, long long n, long long* __restrict__ dst) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  long long stride = (long long)gridDim.x * blockDim.x;
  for (; i < n; i += stride)
    if (!elig[i]) dst[off[i]] = src[i];
}

struct Side : JoinSide {
  std::vector<DevBuf> cols_alt;  // compaction target of `cols`
  int64_t n = 0, cap = 0;
  DevBuf elig, cnt, off;
  int64_t scratch_cap = 0;
};

class InstantJoinOp final : public OpBase {
 public:
  explicit InstantJoinOp(const ArroyoB200OpConfig& c);
  ~InstantJoinOp() override;
  // on_start (instant_join.rs:205-247) IS a replay: the reference feeds every batch of table "left" to process_left and
  // every batch of table "right" to process_right.  The shim does the same through process_batch (the two tables need
  // two input indices, which this entry point does not carry); here only the restored watermark arrives, so that rows
  // older than it are refused exactly as process_side refuses them (:129-139).
  void on_start(ArrowArray* state, ArrowSchema* schemas, int64_t n, int64_t watermark, int64_t) override {
    AB_REQUIRE(n == 0, ARROYO_B200_UNSUPPORTED,
               "InstantJoin restore: pass the watermark here and replay the 'left' / 'right' tables through process_batch");
    (void)state;
    (void)schemas;
    if (watermark != INT64_MIN) last_wm_ = watermark;
  }
  void process_batch(uint32_t index, uint32_t in_partitions, ArrowArray* batch, const ArrowSchema* schema) override;
  void process_device_batch(uint32_t index, uint32_t in_partitions, const uint64_t* cols, int32_t n_cols,
                            int64_t n_rows) override;
  void handle_watermark(int64_t wm, BatchesPriv* out_host, std::vector<ArroyoB200DeviceBatch>* out_dev) override;
  void handle_checkpoint(int64_t, BatchesPriv*) override { flush(); }  // tables left/right are written by the shim
  void on_close(int, BatchesPriv*) override { flush(); }
  void flush() override {
    set_device();
    AB_CUDA(cudaStreamSynchronize(stream_));
    inputs_.release(true);
  }
  void stats(ArroyoB200Stats* out) override { *out = st_; }

 private:
  int join_type_;
  Side side_[2];
  int64_t last_wm_ = INT64_MIN;
  DevBuf scalars_;  // [0] n_elig L, [1] n_elig R, [2] min_ts L, [3] min_ts R, [4] total, [5] cursor
  PinnedBuf h_scalars_;
  DevBuf tab_, sums_, pair_l_, pair_r_, r_matched_;
  int64_t pair_cap_ = 0;
  std::vector<DevBuf> out_cols_;
  std::vector<DevBuf> out_valid_;
  DevBuf out_ts_;
  HeldInputs inputs_;  // host batches whose copies to the side columns may still run
  ArroyoB200Stats st_{};

  void reserve(Side& s, int64_t extra);
  void append(Side& s, const uint64_t* const* cols, int64_t n, bool host);
  int grid_for(int64_t n) const { return (int)std::max<int64_t>(1, std::min<int64_t>((n + JT - 1) / JT, (int64_t)num_sms_ * 8)); }
  void exclusive_scan(const unsigned int* cnt, int64_t n, unsigned long long* off, unsigned long long* total_dev);
  void compact(Side& s);
};

InstantJoinOp::InstantJoinOp(const ArroyoB200OpConfig& c) {
  cfg = c;
  name = "InstantJoin";
  join_type_ = c.join_type;
  AB_REQUIRE(join_type_ >= 0 && join_type_ <= 3, ARROYO_B200_INVALID_ARGUMENT, "bad join type");
  init_join_side(side_[0], c.n_cols, c.timestamp_col, c.left_key_col, c.left_n_routing);
  init_join_side(side_[1], c.right_n_cols, c.right_timestamp_col, c.right_key_col, c.right_n_routing);
  for (Side& s : side_) s.cols_alt.resize(s.n_cols);
  open_device(c);
  scalars_.alloc(8 * sizeof(unsigned long long));
  h_scalars_.alloc(8 * sizeof(unsigned long long));
}

InstantJoinOp::~InstantJoinOp() { drain_stream(); }

void InstantJoinOp::reserve(Side& s, int64_t extra) {
  if (s.n + extra <= s.cap) return;
  int64_t nc = std::max<int64_t>(s.cap * 2, 1 << 16);
  while (nc < s.n + extra) nc *= 2;
  // rows are numbered as int (pairs) and as row + 1 in 32 bits (table slots)
  AB_REQUIRE(nc < (1ll << 31), ARROYO_B200_RUNTIME, "join side holds more than 2^31 rows");
  for (int c = 0; c < s.n_cols; ++c) {
    if (c < s.n_routing) continue;
    DevBuf nb((size_t)nc * 8);
    if (s.n) AB_CUDA(cudaMemcpyAsync(nb.p, s.cols[c].p, (size_t)s.n * 8, cudaMemcpyDeviceToDevice, stream_));
    AB_CUDA(cudaStreamSynchronize(stream_));
    s.cols[c] = std::move(nb);
    s.cols_alt[c].release();
  }
  s.cap = nc;
}

void InstantJoinOp::append(Side& s, const uint64_t* const* cols, int64_t n, bool host) {
  reserve(s, n);
  for (int c = s.n_routing; c < s.n_cols; ++c)
    AB_CUDA(cudaMemcpyAsync(s.cols[c].as<long long>() + s.n, cols[c], (size_t)n * 8,
                            host ? cudaMemcpyHostToDevice : cudaMemcpyDeviceToDevice, stream_));
  if (host) st_.h2d_bytes += (uint64_t)n * 8 * (uint64_t)(s.n_cols - s.n_routing);
  s.n += n;
  st_.rows_in += (uint64_t)n;
}

void InstantJoinOp::process_batch(uint32_t index, uint32_t in_partitions, ArrowArray* batch, const ArrowSchema* schema) {
  set_device();
  AB_REQUIRE(in_partitions >= 2 && in_partitions % 2 == 0, ARROYO_B200_INVALID_ARGUMENT, "join needs an even number of inputs");
  const int sd = (int)(index / (in_partitions / 2));  // instant_join.rs:249-253
  AB_REQUIRE(sd == 0 || sd == 1, ARROYO_B200_INVALID_ARGUMENT, "bad input index");
  Side& s = side_[sd];
  int64_t n = 0;
  std::vector<InColumn> cols = import_batch(batch, schema, &n);
  AB_REQUIRE((int)cols.size() == s.n_cols, ARROYO_B200_INVALID_ARGUMENT, "join side has the wrong number of columns");
  require_join_key_type(cols[s.key_col].format, s.key_format, side_[1 - sd].key_format);
  AB_REQUIRE(n > 0, ARROYO_B200_PANIC, "should have max timestamp (empty batch; instant_join.rs:123)");
  for (int c = 0; c < s.n_cols; ++c) s.formats[c] = cols[c].format;
  s.key_format = cols[s.key_col].format;
  const uint64_t* ptrs[ARROYO_B200_MAX_COLS];
  for (int c = 0; c < s.n_cols; ++c) ptrs[c] = cols[c].data;
  append(s, ptrs, n, true);
  inputs_.hold(batch, stream_);
}

void InstantJoinOp::process_device_batch(uint32_t index, uint32_t in_partitions, const uint64_t* cols, int32_t n_cols,
                                         int64_t n_rows) {
  set_device();
  AB_REQUIRE(in_partitions >= 2 && in_partitions % 2 == 0, ARROYO_B200_INVALID_ARGUMENT, "join needs an even number of inputs");
  const int sd = (int)(index / (in_partitions / 2));
  AB_REQUIRE(sd == 0 || sd == 1, ARROYO_B200_INVALID_ARGUMENT, "bad input index");
  Side& s = side_[sd];
  AB_REQUIRE(n_cols == s.n_cols, ARROYO_B200_INVALID_ARGUMENT, "join side has the wrong number of columns");
  if (n_rows <= 0) return;
  const uint64_t* ptrs[ARROYO_B200_MAX_COLS];
  for (int c = 0; c < s.n_cols; ++c) ptrs[c] = (const uint64_t*)cols[c];
  append(s, ptrs, n_rows, false);
}

void InstantJoinOp::exclusive_scan(const unsigned int* cnt, int64_t n, unsigned long long* off, unsigned long long* total_dev) {
  device_exclusive_scan(cnt, n, off, total_dev, sums_, stream_);
  st_.kernel_launches += 3;
}

// keep rows that did not take part in this watermark's join
void InstantJoinOp::compact(Side& s) {
  if (s.n == 0) return;
  keep_counts_kernel<<<grid_for(s.n), JT, 0, stream_>>>(s.elig.as<unsigned char>(), s.n, s.cnt.as<unsigned int>());
  AB_CUDA(cudaGetLastError());
  unsigned long long* total = scalars_.as<unsigned long long>() + 4;
  exclusive_scan(s.cnt.as<unsigned int>(), s.n, s.off.as<unsigned long long>(), total);
  for (int c = s.n_routing; c < s.n_cols; ++c) {
    if (s.cols_alt[c].bytes < (size_t)s.cap * 8) s.cols_alt[c].alloc((size_t)s.cap * 8);
    compact_kernel<<<grid_for(s.n), JT, 0, stream_>>>(s.cols[c].as<long long>(), s.elig.as<unsigned char>(),
                                                     s.off.as<unsigned long long>(), s.n, s.cols_alt[c].as<long long>());
    AB_CUDA(cudaGetLastError());
    ++st_.kernel_launches;
  }
  AB_CUDA(cudaMemcpyAsync(h_scalars_.as<unsigned long long>() + 4, total, 8, cudaMemcpyDeviceToHost, stream_));
  AB_CUDA(cudaStreamSynchronize(stream_));
  for (int c = s.n_routing; c < s.n_cols; ++c) std::swap(s.cols[c], s.cols_alt[c]);
  s.n = (int64_t)h_scalars_.as<unsigned long long>()[4];
  ++st_.kernel_launches;
}

void InstantJoinOp::handle_watermark(int64_t wm, BatchesPriv* out_host, std::vector<ArroyoB200DeviceBatch>* out_dev) {
  set_device();
  // validated before any state changes: a refused call must leave the eligible rows where they are
  AB_REQUIRE(out_host != nullptr || join_type_ == ARROYO_B200_JOIN_INNER, ARROYO_B200_UNSUPPORTED,
             "device-resident join output is only available for inner joins (no validity bitmaps)");
  Side& L = side_[0];
  Side& R = side_[1];
  AB_REQUIRE(out_host != nullptr || L.payload.size() + R.payload.size() + 1 <= ARROYO_B200_MAX_COLS, ARROYO_B200_UNSUPPORTED,
             "device-resident join output has more than ARROYO_B200_MAX_COLS columns");
  unsigned long long* sc = scalars_.as<unsigned long long>();
  unsigned long long init[8] = {0, 0, (unsigned long long)LLONG_MAX, (unsigned long long)LLONG_MAX, 0, 0, 0, 0};
  AB_CUDA(cudaMemcpyAsync(sc, init, sizeof init, cudaMemcpyHostToDevice, stream_));
  for (int sd = 0; sd < 2; ++sd) {
    Side& s = side_[sd];
    if (s.scratch_cap < s.cap) {
      s.elig.alloc((size_t)s.cap);
      s.cnt.alloc((size_t)s.cap * 4);
      s.off.alloc((size_t)s.cap * 8);
      s.scratch_cap = s.cap;
    }
    if (s.n) {
      mark_kernel<<<grid_for(s.n), JT, 0, stream_>>>(s.cols[s.ts_col].as<long long>(), s.n, wm, s.elig.as<unsigned char>(),
                                                    sc + sd, (long long*)(sc + 2 + sd));
      AB_CUDA(cudaGetLastError());
      ++st_.kernel_launches;
    }
  }
  AB_CUDA(cudaMemcpyAsync(h_scalars_.p, sc, 8 * sizeof(unsigned long long), cudaMemcpyDeviceToHost, stream_));
  AB_CUDA(cudaStreamSynchronize(stream_));
  inputs_.release(true);
  const unsigned long long* hs = h_scalars_.as<unsigned long long>();
  const int64_t nl = (int64_t)hs[0], nr = (int64_t)hs[1];
  const int64_t min_ts = std::min<int64_t>((int64_t)hs[2], (int64_t)hs[3]);
  // rows older than the watermark that was in force when they arrived: the reference panics (:129-139)
  if (last_wm_ != INT64_MIN && min_ts < last_wm_ && (L.n || R.n)) {
    // only rows appended since the previous watermark can be that old: everything older was joined then
    throw Error(ARROYO_B200_PANIC, "shouldn't have a batch with a timestamp before the watermark (instant_join.rs:129-139)");
  }
  last_wm_ = wm;
  if (nl + nr == 0) return;

  const bool keep_l = join_type_ == ARROYO_B200_JOIN_LEFT || join_type_ == ARROYO_B200_JOIN_FULL;
  const bool keep_r = join_type_ == ARROYO_B200_JOIN_RIGHT || join_type_ == ARROYO_B200_JOIN_FULL;
  // Build on the side with fewer eligible rows (persons under auctions in q8), probe with the other.  The pair
  // arrays are filled through (probe side, build side) views, so everything downstream is side-agnostic.
  const int bsd = nl < nr ? 0 : 1;
  Side& Bs = side_[bsd];
  Side& Ps = side_[1 - bsd];
  const int64_t nb = bsd == 0 ? nl : nr;
  const bool keep_b = bsd == 0 ? keep_l : keep_r, keep_p = bsd == 0 ? keep_r : keep_l;
  uint64_t cap = 1024;
  while (cap < (uint64_t)nb * 2 + 2) cap <<= 1;
  AB_REQUIRE(cap <= (1ull << 31), ARROYO_B200_RUNTIME, "join build side too large");
  if (tab_.bytes < cap * sizeof(JSlot)) tab_.alloc(cap * sizeof(JSlot));
  AB_CUDA(cudaMemsetAsync(tab_.p, 0, cap * sizeof(JSlot), stream_));
  if (r_matched_.bytes < (size_t)std::max<int64_t>(Bs.n, 1)) r_matched_.alloc((size_t)std::max<int64_t>(Bs.cap, 1));
  if (Bs.n) AB_CUDA(cudaMemsetAsync(r_matched_.p, 0, (size_t)Bs.n, stream_));
  if (nb) {
    build_kernel<<<grid_for(Bs.n), JT, 0, stream_>>>(Bs.cols[Bs.key_col].as<long long>(), Bs.cols[Bs.ts_col].as<long long>(),
                                                    Bs.elig.as<unsigned char>(), Bs.n, tab_.as<JSlot>(), (uint32_t)(cap - 1));
    AB_CUDA(cudaGetLastError());
    ++st_.kernel_launches;
  }
  int64_t n_probe_out = 0;
  if (Ps.n) {
    probe_kernel<0><<<grid_for(Ps.n), JT, 0, stream_>>>(
        Ps.cols[Ps.key_col].as<long long>(), Ps.cols[Ps.ts_col].as<long long>(), Ps.elig.as<unsigned char>(), Ps.n,
        Bs.cols[Bs.ts_col].as<long long>(), tab_.as<JSlot>(), (uint32_t)(cap - 1), keep_p ? 1 : 0,
        Ps.cnt.as<unsigned int>(), nullptr, nullptr, nullptr, nullptr);
    AB_CUDA(cudaGetLastError());
    exclusive_scan(Ps.cnt.as<unsigned int>(), Ps.n, Ps.off.as<unsigned long long>(), sc + 4);
    AB_CUDA(cudaMemcpyAsync(h_scalars_.as<unsigned long long>() + 4, sc + 4, 8, cudaMemcpyDeviceToHost, stream_));
    AB_CUDA(cudaStreamSynchronize(stream_));
    n_probe_out = (int64_t)h_scalars_.as<unsigned long long>()[4];
    ++st_.kernel_launches;
  }
  const int64_t max_out = n_probe_out + (keep_b ? nb : 0);
  AB_REQUIRE(max_out < (int64_t)INT_MAX, ARROYO_B200_RUNTIME, "join output too large for one watermark");
  int64_t n_out = n_probe_out;
  if (max_out > 0) {
    if (pair_cap_ < max_out) {
      pair_l_.alloc((size_t)max_out * 4);
      pair_r_.alloc((size_t)max_out * 4);
      pair_cap_ = max_out;
    }
    int* pair_p = bsd == 0 ? pair_r_.as<int>() : pair_l_.as<int>();
    int* pair_b = bsd == 0 ? pair_l_.as<int>() : pair_r_.as<int>();
    if (n_probe_out) {
      probe_kernel<1><<<grid_for(Ps.n), JT, 0, stream_>>>(
          Ps.cols[Ps.key_col].as<long long>(), Ps.cols[Ps.ts_col].as<long long>(), Ps.elig.as<unsigned char>(), Ps.n,
          Bs.cols[Bs.ts_col].as<long long>(), tab_.as<JSlot>(), (uint32_t)(cap - 1), keep_p ? 1 : 0, nullptr,
          Ps.off.as<unsigned long long>(), pair_p, pair_b, r_matched_.as<unsigned char>());
      AB_CUDA(cudaGetLastError());
      ++st_.kernel_launches;
    }
    if (keep_b && nb) {
      unsigned long long cur = (unsigned long long)n_probe_out;
      AB_CUDA(cudaMemcpyAsync(sc + 5, &cur, 8, cudaMemcpyHostToDevice, stream_));
      append_unmatched_kernel<<<grid_for(Bs.n), JT, 0, stream_>>>(Bs.elig.as<unsigned char>(), r_matched_.as<unsigned char>(),
                                                                 Bs.n, sc + 5, pair_p, pair_b);
      AB_CUDA(cudaGetLastError());
      AB_CUDA(cudaMemcpyAsync(h_scalars_.as<unsigned long long>() + 5, sc + 5, 8, cudaMemcpyDeviceToHost, stream_));
      AB_CUDA(cudaStreamSynchronize(stream_));
      n_out = (int64_t)h_scalars_.as<unsigned long long>()[5];
      ++st_.kernel_launches;
    }
  }

  if (n_out > 0) {
    // gather [left payload..., right payload..., _timestamp]
    const size_t n_oc = L.payload.size() + R.payload.size();
    out_cols_.resize(n_oc);
    out_valid_.resize(n_oc);
    const bool l_nullable = keep_r, r_nullable = keep_l;
    size_t oc = 0;
    for (int sd = 0; sd < 2; ++sd) {
      Side& s = side_[sd];
      const bool nullable = sd == 0 ? l_nullable : r_nullable;
      for (int c : s.payload) {
        if (out_cols_[oc].bytes < (size_t)n_out * 8) out_cols_[oc].alloc((size_t)n_out * 8);
        if (nullable && out_valid_[oc].bytes < (size_t)n_out + 64) out_valid_[oc].alloc((size_t)n_out + 64);
        GatherParams gp{sd == 0 ? pair_l_.as<int>() : pair_r_.as<int>(), s.cols[c].as<long long>(),
                        out_cols_[oc].as<long long>(), nullable ? out_valid_[oc].as<unsigned char>() : nullptr, n_out};
        gather_kernel<<<grid_for(n_out), JT, 0, stream_>>>(gp);
        AB_CUDA(cudaGetLastError());
        ++st_.kernel_launches;
        ++oc;
      }
    }
    if (out_ts_.bytes < (size_t)n_out * 8) out_ts_.alloc((size_t)n_out * 8);
    gather_ts_kernel<<<grid_for(n_out), JT, 0, stream_>>>(pair_l_.as<int>(), pair_r_.as<int>(), L.cols[L.ts_col].as<long long>(),
                                                         R.cols[R.ts_col].as<long long>(), out_ts_.as<long long>(), n_out);
    AB_CUDA(cudaGetLastError());
    ++st_.kernel_launches;
    st_.rows_out += (uint64_t)n_out;
    ++st_.windows_out;

    if (out_host) {
      std::vector<OutColumn> cols;
      oc = 0;
      DevBuf bits;
      for (int sd = 0; sd < 2; ++sd) {
        Side& s = side_[sd];
        const bool nullable = sd == 0 ? l_nullable : r_nullable;
        for (int c : s.payload) {
          OutColumn o;
          o.name = std::string(sd == 0 ? "l" : "r") + std::to_string(c);
          o.format = s.formats[c];
          o.data = d2h_pinned(out_cols_[oc].p, (size_t)n_out * 8, stream_, &st_.d2h_bytes);
          if (nullable) {
            const size_t words = (size_t)((n_out + 31) / 32);
            if (bits.bytes < words * 4) bits.alloc(words * 4 + 64);
            pack_bits_kernel<<<grid_for(n_out), JT, 0, stream_>>>(out_valid_[oc].as<unsigned char>(), n_out, bits.as<unsigned int>());
            AB_CUDA(cudaGetLastError());
            o.validity = d2h_pinned(bits.p, words * 4, stream_, &st_.d2h_bytes);
            AB_CUDA(cudaStreamSynchronize(stream_));  // `bits` is reused by the next column
            const unsigned int* w = (const unsigned int*)o.validity;
            int64_t set = 0;
            for (size_t i = 0; i < words; ++i) set += __builtin_popcount(w[i]);
            o.null_count = n_out - set;
            o.nullable = true;
            if (o.null_count == 0) {
              PinnedPool::get().free(o.validity);
              o.validity = nullptr;
            }
          }
          cols.push_back(o);
          ++oc;
        }
      }
      OutColumn t;
      t.name = "_timestamp";
      t.format = "tsn:";
      t.data = d2h_pinned(out_ts_.p, (size_t)n_out * 8, stream_, &st_.d2h_bytes);
      cols.push_back(t);
      AB_CUDA(cudaStreamSynchronize(stream_));
      out_host->arrays.emplace_back();
      out_host->schemas.emplace_back();
      export_batch(cols, n_out, &out_host->arrays.back(), &out_host->schemas.back());
    } else {
      AB_REQUIRE(join_type_ == ARROYO_B200_JOIN_INNER, ARROYO_B200_UNSUPPORTED,
                 "device-resident join output is only available for inner joins (no validity bitmaps)");
      ArroyoB200DeviceBatch d{};
      d.n_rows = n_out;
      int c = 0;
      for (size_t i = 0; i < n_oc; ++i) d.cols[c++] = (uint64_t)out_cols_[i].p;
      d.cols[c++] = (uint64_t)out_ts_.p;
      d.n_cols = c;
      out_dev->push_back(d);
      AB_CUDA(cudaStreamSynchronize(stream_));
    }
  }
  // rows at or after the watermark stay for later
  compact(L);
  compact(R);
}

}  // namespace

OpBase* make_instant_join_op(const ArroyoB200OpConfig& cfg) { return new InstantJoinOp(cfg); }

}  // namespace ab
