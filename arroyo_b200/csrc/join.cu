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

#include "join_side.h"

namespace ab {
namespace {

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
  DevBuf elig, cnt, off;  // per-row scratch of the watermark, `cap` rows
};

class InstantJoinOp final : public JoinOpBase {
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

 private:
  int join_type_;
  Side side_[2];
  int64_t last_wm_ = INT64_MIN;
  DevBuf scalars_;  // [0] n_elig L, [1] n_elig R, [2] min_ts L, [3] min_ts R, [4] total, [5] cursor
  PinnedBuf h_scalars_;
  DevBuf tab_, r_matched_;
  HeldInputs inputs_;  // host batches whose copies to the side columns may still run

  void append(Side& s, const uint64_t* const* cols, int64_t n, bool host);
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

void InstantJoinOp::append(Side& s, const uint64_t* const* cols, int64_t n, bool host) {
  s.reserve(n, stream_, nullptr, &s.cols_alt);
  s.append(cols, n, host, stream_, st_);
  st_.rows_in += (uint64_t)n;
}

void InstantJoinOp::process_batch(uint32_t index, uint32_t in_partitions, ArrowArray* batch, const ArrowSchema* schema) {
  set_device();
  const int sd = side_of(index, in_partitions);
  Side& s = side_[sd];
  const JoinBatch b = s.import(batch, schema, s.key_format, side_[1 - sd]);
  AB_REQUIRE(b.n > 0, ARROYO_B200_PANIC, "should have max timestamp (empty batch; instant_join.rs:123)");
  s.take_formats(b.cols);
  append(s, b.data, b.n, true);
  inputs_.hold(batch, stream_);
}

void InstantJoinOp::process_device_batch(uint32_t index, uint32_t in_partitions, const uint64_t* cols, int32_t n_cols,
                                         int64_t n_rows) {
  set_device();
  Side& s = side_[side_of(index, in_partitions)];
  AB_REQUIRE(n_cols == s.n_cols, ARROYO_B200_INVALID_ARGUMENT, "join side has the wrong number of columns");
  if (n_rows <= 0) return;
  const uint64_t* ptrs[ARROYO_B200_MAX_COLS];
  for (int c = 0; c < s.n_cols; ++c) ptrs[c] = (const uint64_t*)cols[c];
  append(s, ptrs, n_rows, false);
}

// keep rows that did not take part in this watermark's join
void InstantJoinOp::compact(Side& s) {
  if (s.n == 0) return;
  keep_counts_kernel<<<grid_for(s.n), JOIN_THREADS, 0, stream_>>>(s.elig.as<unsigned char>(), s.n, s.cnt.as<unsigned int>());
  AB_CUDA(cudaGetLastError());
  unsigned long long* total = scalars_.as<unsigned long long>() + 4;
  device_exclusive_scan(s.cnt.as<unsigned int>(), s.n, s.off.as<unsigned long long>(), total, sums_, stream_);
  st_.kernel_launches += 3;
  for (int c = s.n_routing; c < s.n_cols; ++c) {
    if (s.cols_alt[c].bytes < (size_t)s.cap * 8) s.cols_alt[c].alloc((size_t)s.cap * 8);
    compact_kernel<<<grid_for(s.n), JOIN_THREADS, 0, stream_>>>(s.cols[c].as<long long>(), s.elig.as<unsigned char>(),
                                                               s.off.as<unsigned long long>(), s.n,
                                                               s.cols_alt[c].as<long long>());
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
    grow(s.elig, (size_t)s.cap);
    grow(s.cnt, (size_t)s.cap * 4);
    grow(s.off, (size_t)s.cap * 8);
    if (s.n) {
      mark_kernel<<<grid_for(s.n), JOIN_THREADS, 0, stream_>>>(s.cols[s.ts_col].as<long long>(), s.n, wm,
                                                              s.elig.as<unsigned char>(), sc + sd, (long long*)(sc + 2 + sd));
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
    build_kernel<<<grid_for(Bs.n), JOIN_THREADS, 0, stream_>>>(Bs.cols[Bs.key_col].as<long long>(),
                                                              Bs.cols[Bs.ts_col].as<long long>(), Bs.elig.as<unsigned char>(),
                                                              Bs.n, tab_.as<JSlot>(), (uint32_t)(cap - 1));
    AB_CUDA(cudaGetLastError());
    ++st_.kernel_launches;
  }
  int64_t n_probe_out = 0;
  if (Ps.n) {
    n_probe_out = count_pairs(
        [&] {
          probe_kernel<0><<<grid_for(Ps.n), JOIN_THREADS, 0, stream_>>>(
              Ps.cols[Ps.key_col].as<long long>(), Ps.cols[Ps.ts_col].as<long long>(), Ps.elig.as<unsigned char>(), Ps.n,
              Bs.cols[Bs.ts_col].as<long long>(), tab_.as<JSlot>(), (uint32_t)(cap - 1), keep_p ? 1 : 0,
              Ps.cnt.as<unsigned int>(), nullptr, nullptr, nullptr, nullptr);
        },
        Ps.cnt.as<unsigned int>(), Ps.n, Ps.off.as<unsigned long long>(), sc + 4, h_scalars_.as<unsigned long long>() + 4);
  }
  const int64_t max_out = n_probe_out + (keep_b ? nb : 0);
  AB_REQUIRE(max_out < (int64_t)INT_MAX, ARROYO_B200_RUNTIME, "join output too large for one watermark");
  int64_t n_out = n_probe_out;
  if (max_out > 0) {
    reserve_pairs(max_out);
    int* pair_p = pairs_[1 - bsd].as<int>();
    int* pair_b = pairs_[bsd].as<int>();
    if (n_probe_out) {
      probe_kernel<1><<<grid_for(Ps.n), JOIN_THREADS, 0, stream_>>>(
          Ps.cols[Ps.key_col].as<long long>(), Ps.cols[Ps.ts_col].as<long long>(), Ps.elig.as<unsigned char>(), Ps.n,
          Bs.cols[Bs.ts_col].as<long long>(), tab_.as<JSlot>(), (uint32_t)(cap - 1), keep_p ? 1 : 0, nullptr,
          Ps.off.as<unsigned long long>(), pair_p, pair_b, r_matched_.as<unsigned char>());
      AB_CUDA(cudaGetLastError());
      ++st_.kernel_launches;
    }
    if (keep_b && nb) {
      unsigned long long cur = (unsigned long long)n_probe_out;
      AB_CUDA(cudaMemcpyAsync(sc + 5, &cur, 8, cudaMemcpyHostToDevice, stream_));
      append_unmatched_kernel<<<grid_for(Bs.n), JOIN_THREADS, 0, stream_>>>(
          Bs.elig.as<unsigned char>(), r_matched_.as<unsigned char>(), Bs.n, sc + 5, pair_p, pair_b);
      AB_CUDA(cudaGetLastError());
      AB_CUDA(cudaMemcpyAsync(h_scalars_.as<unsigned long long>() + 5, sc + 5, 8, cudaMemcpyDeviceToHost, stream_));
      AB_CUDA(cudaStreamSynchronize(stream_));
      n_out = (int64_t)h_scalars_.as<unsigned long long>()[5];
      ++st_.kernel_launches;
    }
  }

  if (n_out > 0) write_output(L, R, n_out, keep_r, keep_l, out_host, out_dev);
  // rows at or after the watermark stay for later
  compact(L);
  compact(R);
}

}  // namespace

OpBase* make_instant_join_op(const ArroyoB200OpConfig& cfg) { return new InstantJoinOp(cfg); }

}  // namespace ab
