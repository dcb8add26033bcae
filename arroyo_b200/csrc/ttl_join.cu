// Non-windowed join with expiration on sm_90a (H100): the GPU side of `JoinWithExpiration`
// (arroyo-worker/src/arrow/join_with_expiration.rs:42-130), SURVEY.md 8(f) rank 3.  Inner joins of append-only inputs.
//
// The reference keeps each side's rows in a key-time table (`KeyTimeView`, arroyo-state/src/tables/
// expiring_time_key_map.rs:932-1050): an arriving batch is inserted into its side's table (:52, :83), the other
// side's stored rows of the batch's distinct keys are fetched (`get_batch`, :970-985) and the pair goes through the
// join plan (`compute_pair`, :110-130): every matching pair leaves exactly once, when its later row arrives.
//
// Here each side is a set of append-only device arenas (one per payload column) plus a persistent multimap
// key -> chain of row numbers: a 16-byte open-addressing slot {key, head row + 1} per distinct key and a `next`
// link per row.  A batch is
//   appended  to its side's arenas (H2D),
//   linked    into its side's multimap (one CAS to find / claim the key's slot, one atomicExch to push the row),
//   probed    against the OTHER side's multimap: count matches per new row -> exclusive scan -> write the pairs,
//   gathered  into the output columns [left payload..., right payload..., _timestamp = max(l, r)]
//             (arroyo-planner/src/plan/join.rs:165-185), which leave with the call (`process_batch_emit`).
// Rows leave the tables only through the state backend's retention (`ttl`, applied at restore / compaction), never
// inside a run: like the oracle, not restated.  Outer / updating joins are refused (ARROYO_B200_UNSUPPORTED).
//
// Restore (`restore_side`): the shim writes the key-time tables "left" / "right" from the host batches and hands
// what it reads back to the side they came from.  Those rows are appended and linked, the first step of a batch,
// and never probed: the reference's `insert_internal` (expiring_time_key_map.rs:1008-1049) stores restored rows
// without joining them, so no pair among them leaves again.
#include <algorithm>
#include <climits>

#include "op.h"
#include "scan.cuh"

namespace ab {
namespace {

constexpr int TJ = 256;

struct alignas(16) MSlot {
  long long key;
  unsigned int head1;  // newest row of the key + 1 (0: none yet)
  unsigned int used;   // 1 once the slot is claimed (the key may be any 64-bit value)
};

__device__ __forceinline__ uint32_t tj_home(long long key, uint32_t mask) { return (uint32_t)(mix64((uint64_t)key) >> 20) & mask; }

// links rows [first, first + n) of a side into its multimap
__global__ void tj_link_kernel(const long long* __restrict__ key, long long first, long long n, MSlot* __restrict__ tab,
                               uint32_t mask, int* __restrict__ next) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (; i < n; i += stride) {
    const long long row = first + i;
    const long long k = key[row];
    uint32_t pos = tj_home(k, mask);
    while (true) {
      const unsigned int was = atomicCAS(&tab[pos].used, 0u, 1u);
      if (was == 0u) {
        // claimed: publish the key (readers of a claimed slot wait for it through `used == 2`)
        tab[pos].key = k;
        __threadfence();
        atomicExch(&tab[pos].used, 2u);
        break;
      }
      unsigned int st = was;
      while (st == 1u) st = *(volatile unsigned int*)&tab[pos].used;
      if (*(volatile long long*)&tab[pos].key == k) break;
      pos = (pos + 1) & mask;
    }
    next[row] = (int)atomicExch(&tab[pos].head1, (unsigned int)row + 1u) - 1;
  }
}

// PASS 0: cnt[i] = matches of new row i in the other side; PASS 1: write (new row, stored row) pairs at off[i]
template <int PASS>
__global__ void tj_probe_kernel(const long long* __restrict__ pkey, long long first, long long n, const MSlot* __restrict__ tab,
                                uint32_t mask, const int* __restrict__ next, unsigned int* __restrict__ cnt,
                                const unsigned long long* __restrict__ off, int* __restrict__ out_new, int* __restrict__ out_old) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (; i < n; i += stride) {
    const long long k = pkey[first + i];
    uint32_t pos = tj_home(k, mask);
    int head = -1;
    while (true) {
      const ulonglong2 raw = __ldcg(reinterpret_cast<const ulonglong2*>(tab + pos));
      const unsigned int used = (unsigned int)(raw.y >> 32);
      if (used == 0u) break;
      if ((long long)raw.x == k) {
        head = (int)(unsigned int)raw.y - 1;
        break;
      }
      pos = (pos + 1) & mask;
    }
    unsigned int c = 0;
    unsigned long long o = PASS == 1 ? off[i] : 0;
    for (int r = head; r >= 0; r = next[r]) {
      if (PASS == 1) {
        out_new[o + c] = (int)(first + i);
        out_old[o + c] = r;
      }
      ++c;
    }
    if (PASS == 0) cnt[i] = c;
  }
}

__global__ void tj_rehash_kernel(const MSlot* __restrict__ old_tab, uint32_t old_cap, MSlot* __restrict__ tab, uint32_t mask) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  const uint32_t stride = gridDim.x * blockDim.x;
  for (; i < old_cap; i += stride) {
    const MSlot s = old_tab[i];
    if (!s.used) continue;
    uint32_t pos = tj_home(s.key, mask);
    while (atomicCAS(&tab[pos].used, 0u, 2u) != 0u) pos = (pos + 1) & mask;
    tab[pos].key = s.key;
    tab[pos].head1 = s.head1;
  }
}

struct TGather {
  const int* idx;
  const long long* src;
  long long* dst;
  long long n;
};
__global__ void tj_gather_kernel(const __grid_constant__ TGather p) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (; i < p.n; i += stride) p.dst[i] = p.src[p.idx[i]];
}
__global__ void tj_gather_ts_kernel(const int* __restrict__ il, const int* __restrict__ ir, const long long* __restrict__ lts,
                                    const long long* __restrict__ rts, long long* __restrict__ dst, long long n) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (; i < n; i += stride) dst[i] = max(lts[il[i]], rts[ir[i]]);
}

struct TSide : JoinSide {
  DevBuf next, tab;
  int64_t n = 0, cap = 0;
  uint32_t tab_cap = 0;
  uint64_t keys_bound = 0;  // rows linked so far: an upper bound of the distinct keys
};

class TtlJoinOp final : public OpBase {
 public:
  explicit TtlJoinOp(const ArroyoB200OpConfig& c);
  ~TtlJoinOp() override;
  void on_start(ArrowArray*, ArrowSchema*, int64_t n, int64_t, int64_t) override {
    AB_REQUIRE(n == 0, ARROYO_B200_UNSUPPORTED,
               "JoinWithExpiration restore: hand each key-time table to arroyo_b200_op_restore_side");
  }
  void restore_side(uint32_t side, ArrowArray* batches, ArrowSchema* schemas, int64_t n) override;
  void process_batch(uint32_t index, uint32_t parts, ArrowArray* batch, const ArrowSchema* schema) override {
    BatchesPriv sink;
    process_batch_emit(index, parts, batch, schema, &sink);
    for (auto& a : sink.arrays)
      if (a.release) a.release(&a);
    for (auto& s : sink.schemas)
      if (s.release) s.release(&s);
  }
  void process_batch_emit(uint32_t index, uint32_t parts, ArrowArray* batch, const ArrowSchema* schema, BatchesPriv* out) override;
  void process_device_batch(uint32_t, uint32_t, const uint64_t*, int32_t, int64_t) override {
    throw Error(ARROYO_B200_UNSUPPORTED, "JoinWithExpiration: device-resident input is not implemented");
  }
  void handle_watermark(int64_t, BatchesPriv*, std::vector<ArroyoB200DeviceBatch>*) override {}  // emits as rows arrive
  void handle_checkpoint(int64_t, BatchesPriv*) override { flush(); }
  void on_close(int, BatchesPriv*) override { flush(); }
  void flush() override {
    set_device();
    AB_CUDA(cudaStreamSynchronize(stream_));
  }
  void stats(ArroyoB200Stats* out) override { *out = st_; }

 private:
  TSide side_[2];
  DevBuf cnt_, off_, total_, sums_, pair_new_, pair_old_, out_ts_;
  std::vector<DevBuf> out_cols_;
  int64_t scratch_cap_ = 0, pair_cap_ = 0;
  bool took_input_ = false;  // process_batch has accepted a batch: restore_side is refused from then on
  ArroyoB200Stats st_{};

  int grid_for(int64_t n) const { return (int)std::max<int64_t>(1, std::min<int64_t>((n + TJ - 1) / TJ, (int64_t)num_sms_ * 8)); }
  void reserve(TSide& s, int64_t extra);
  void ensure_table(TSide& s, uint64_t more_rows);
};

TtlJoinOp::TtlJoinOp(const ArroyoB200OpConfig& c) {
  cfg = c;
  name = "JoinWithExpiration";
  AB_REQUIRE(c.join_type == ARROYO_B200_JOIN_INNER, ARROYO_B200_UNSUPPORTED,
             "JoinWithExpiration: only inner joins of append-only inputs are supported");
  init_join_side(side_[0], c.n_cols, c.timestamp_col, c.left_key_col, c.left_n_routing);
  init_join_side(side_[1], c.right_n_cols, c.right_timestamp_col, c.right_key_col, c.right_n_routing);
  open_device(c);
  total_.alloc(16);
}

TtlJoinOp::~TtlJoinOp() { drain_stream(); }

void TtlJoinOp::reserve(TSide& s, int64_t extra) {
  if (s.n + extra <= s.cap) return;
  int64_t nc = std::max<int64_t>(s.cap * 2, 1 << 16);
  while (nc < s.n + extra) nc *= 2;
  AB_REQUIRE(nc < (1ll << 31), ARROYO_B200_RUNTIME, "join side holds more than 2^31 rows");
  auto grow = [&](DevBuf& b, size_t elem) {
    DevBuf nb((size_t)nc * elem);
    if (s.n && b.p) AB_CUDA(cudaMemcpyAsync(nb.p, b.p, (size_t)s.n * elem, cudaMemcpyDeviceToDevice, stream_));
    AB_CUDA(cudaStreamSynchronize(stream_));
    b = std::move(nb);
  };
  for (int c = s.n_routing; c < s.n_cols; ++c) grow(s.cols[c], 8);
  grow(s.next, 4);
  s.cap = nc;
}

// the multimap stays at most half full of distinct keys (bounded by the rows linked so far)
void TtlJoinOp::ensure_table(TSide& s, uint64_t more_rows) {
  const uint64_t need = (s.keys_bound + more_rows) * 2 + 1024;
  if (s.tab_cap >= need) return;
  uint64_t nc = std::max<uint64_t>((uint64_t)s.tab_cap * 2, 1u << 16);
  while (nc < need) nc *= 2;
  AB_REQUIRE(nc <= (1ull << 31), ARROYO_B200_RUNTIME, "join side's key table would exceed 2^31 slots");
  DevBuf nt((size_t)nc * sizeof(MSlot));
  AB_CUDA(cudaMemsetAsync(nt.p, 0, (size_t)nc * sizeof(MSlot), stream_));
  if (s.tab_cap) {
    tj_rehash_kernel<<<grid_for(s.tab_cap), TJ, 0, stream_>>>(s.tab.as<MSlot>(), s.tab_cap, nt.as<MSlot>(), (uint32_t)(nc - 1));
    AB_CUDA(cudaGetLastError());
    ++st_.kernel_launches;
  }
  AB_CUDA(cudaStreamSynchronize(stream_));
  s.tab = std::move(nt);
  s.tab_cap = (uint32_t)nc;
}

// KeyTimeView::insert_internal (:1008-1049) for the batches of one side's table: every batch is checked before anything
// changes, then the call's rows are copied into consecutive arena ranges and linked by one launch.  A restore that
// succeeds takes every batch.
void TtlJoinOp::restore_side(uint32_t side, ArrowArray* batches, ArrowSchema* schemas, int64_t n) {
  AB_REQUIRE(side <= 1, ARROYO_B200_INVALID_ARGUMENT, "restore_side: side must be 0 (left) or 1 (right)");
  AB_REQUIRE(n >= 0 && (n == 0 || (batches != nullptr && schemas != nullptr)), ARROYO_B200_INVALID_ARGUMENT,
             "restore_side: null batches");
  AB_REQUIRE(!took_input_, ARROYO_B200_INVALID_ARGUMENT,
             "JoinWithExpiration: restore_side after process_batch (restore before the first batch)");
  TSide& s = side_[side];
  std::vector<std::vector<InColumn>> cols((size_t)n);
  std::vector<int64_t> rows((size_t)n, 0);
  std::string key_format = s.key_format;
  int64_t total = 0;
  for (int64_t b = 0; b < n; ++b) {
    cols[b] = import_batch(&batches[b], &schemas[b], &rows[b]);
    AB_REQUIRE((int)cols[b].size() == s.n_cols, ARROYO_B200_INVALID_ARGUMENT,
               "restore_side: batch does not have the side's number of columns");
    require_join_key_type(cols[b][s.key_col].format, key_format, side_[1 - side].key_format);
    key_format = cols[b][s.key_col].format;
    total += rows[b];
  }
  set_device();
  if (total > 0) {
    reserve(s, total);
    ensure_table(s, (uint64_t)total);
    long long at = s.n;
    for (int64_t b = 0; b < n; ++b) {
      for (int c = s.n_routing; c < s.n_cols; ++c)
        if (rows[b])
          AB_CUDA(cudaMemcpyAsync(s.cols[c].as<long long>() + at, cols[b][c].data, (size_t)rows[b] * 8,
                                  cudaMemcpyHostToDevice, stream_));
      at += rows[b];
    }
    st_.h2d_bytes += (uint64_t)total * 8 * (uint64_t)(s.n_cols - s.n_routing);
    tj_link_kernel<<<grid_for(total), TJ, 0, stream_>>>(s.cols[s.key_col].as<long long>(), s.n, total, s.tab.as<MSlot>(),
                                                      s.tab_cap - 1, s.next.as<int>());
    AB_CUDA(cudaGetLastError());
    ++st_.kernel_launches;
    AB_CUDA(cudaStreamSynchronize(stream_));
    s.n += total;
    s.keys_bound += (uint64_t)total;
  }
  if (n > 0) {
    for (int c = 0; c < s.n_cols; ++c) s.formats[c] = cols[n - 1][c].format;
    s.key_format = key_format;
  }
  for (int64_t b = 0; b < n; ++b)
    if (batches[b].release) batches[b].release(&batches[b]);
}

void TtlJoinOp::process_batch_emit(uint32_t index, uint32_t parts, ArrowArray* batch, const ArrowSchema* schema, BatchesPriv* out) {
  set_device();
  AB_REQUIRE(parts >= 2 && parts % 2 == 0, ARROYO_B200_INVALID_ARGUMENT, "join needs an even number of inputs");
  const int sd = (int)(index / (parts / 2));
  AB_REQUIRE(sd == 0 || sd == 1, ARROYO_B200_INVALID_ARGUMENT, "bad input index");
  TSide& s = side_[sd];
  TSide& o = side_[1 - sd];
  int64_t n = 0;
  std::vector<InColumn> cols = import_batch(batch, schema, &n);
  AB_REQUIRE((int)cols.size() == s.n_cols, ARROYO_B200_INVALID_ARGUMENT, "join side has the wrong number of columns");
  require_join_key_type(cols[s.key_col].format, s.key_format, o.key_format);
  for (int c = 0; c < s.n_cols; ++c) s.formats[c] = cols[c].format;
  s.key_format = cols[s.key_col].format;
  took_input_ = true;
  st_.rows_in += (uint64_t)n;
  if (n == 0) {
    if (batch->release) batch->release(batch);
    batch->release = nullptr;
    return;
  }
  // 1. append + link (insert into this side's key-time table, :52 / :83)
  reserve(s, n);
  ensure_table(s, (uint64_t)n);
  const long long first = s.n;
  for (int c = s.n_routing; c < s.n_cols; ++c)
    AB_CUDA(cudaMemcpyAsync(s.cols[c].as<long long>() + first, cols[c].data, (size_t)n * 8, cudaMemcpyHostToDevice, stream_));
  st_.h2d_bytes += (uint64_t)n * 8 * (uint64_t)(s.n_cols - s.n_routing);
  tj_link_kernel<<<grid_for(n), TJ, 0, stream_>>>(s.cols[s.key_col].as<long long>(), first, n, s.tab.as<MSlot>(), s.tab_cap - 1,
                                                s.next.as<int>());
  AB_CUDA(cudaGetLastError());
  ++st_.kernel_launches;
  ++st_.ingest_launches;
  s.n += n;
  s.keys_bound += (uint64_t)n;
  // 2. the other side's rows of these keys (get_batch, :59-64 / :90-95) x the batch (compute_pair)
  int64_t n_out = 0;
  if (o.n > 0) {
    if (n > scratch_cap_) {
      scratch_cap_ = std::max<int64_t>(n, scratch_cap_ * 2);
      cnt_.alloc((size_t)scratch_cap_ * 4);
      off_.alloc((size_t)scratch_cap_ * 8);
    }
    const long long* pkey = s.cols[s.key_col].as<long long>();
    tj_probe_kernel<0><<<grid_for(n), TJ, 0, stream_>>>(pkey, first, n, o.tab.as<MSlot>(), o.tab_cap - 1, o.next.as<int>(),
                                                       cnt_.as<unsigned int>(), nullptr, nullptr, nullptr);
    AB_CUDA(cudaGetLastError());
    device_exclusive_scan(cnt_.as<unsigned int>(), n, off_.as<unsigned long long>(), total_.as<unsigned long long>(), sums_, stream_);
    unsigned long long h_total = 0;
    AB_CUDA(cudaMemcpyAsync(&h_total, total_.p, 8, cudaMemcpyDeviceToHost, stream_));
    AB_CUDA(cudaStreamSynchronize(stream_));
    st_.kernel_launches += 4;
    n_out = (int64_t)h_total;
    if (n_out > 0) {
      if (n_out > pair_cap_) {
        pair_cap_ = std::max<int64_t>(n_out, pair_cap_ * 2);
        pair_new_.alloc((size_t)pair_cap_ * 4);
        pair_old_.alloc((size_t)pair_cap_ * 4);
        out_ts_.alloc((size_t)pair_cap_ * 8);
        out_cols_.clear();
      }
      tj_probe_kernel<1><<<grid_for(n), TJ, 0, stream_>>>(pkey, first, n, o.tab.as<MSlot>(), o.tab_cap - 1, o.next.as<int>(), nullptr,
                                                         off_.as<unsigned long long>(), pair_new_.as<int>(), pair_old_.as<int>());
      AB_CUDA(cudaGetLastError());
      ++st_.kernel_launches;
    }
  }
  // the host batch may go once its copies have been consumed
  AB_CUDA(cudaStreamSynchronize(stream_));
  if (batch->release) batch->release(batch);
  batch->release = nullptr;
  if (n_out == 0 || !out) return;
  // 3. output = [left payload..., right payload..., _timestamp = max(l, r)]
  const int* il = sd == 0 ? pair_new_.as<int>() : pair_old_.as<int>();
  const int* ir = sd == 0 ? pair_old_.as<int>() : pair_new_.as<int>();
  const size_t n_oc = side_[0].payload.size() + side_[1].payload.size();
  if (out_cols_.size() != n_oc) {
    out_cols_.clear();
    for (size_t i = 0; i < n_oc; ++i) out_cols_.emplace_back((size_t)pair_cap_ * 8);
  }
  std::vector<OutColumn> ocols;
  size_t oc = 0;
  for (int side = 0; side < 2; ++side) {
    TSide& z = side_[side];
    for (int c : z.payload) {
      TGather g{side == 0 ? il : ir, z.cols[c].as<long long>(), out_cols_[oc].as<long long>(), n_out};
      tj_gather_kernel<<<grid_for(n_out), TJ, 0, stream_>>>(g);
      AB_CUDA(cudaGetLastError());
      ++st_.kernel_launches;
      OutColumn col;
      col.name = (side == 0 ? "l" : "r") + std::to_string(c);
      col.format = z.formats[c];
      col.data = d2h_pinned(out_cols_[oc].p, (size_t)n_out * 8, stream_, &st_.d2h_bytes);
      ocols.push_back(col);
      ++oc;
    }
  }
  tj_gather_ts_kernel<<<grid_for(n_out), TJ, 0, stream_>>>(il, ir, side_[0].cols[side_[0].ts_col].as<long long>(),
                                                          side_[1].cols[side_[1].ts_col].as<long long>(), out_ts_.as<long long>(),
                                                          n_out);
  AB_CUDA(cudaGetLastError());
  ++st_.kernel_launches;
  ++st_.emit_launches;
  OutColumn t;
  t.name = "_timestamp";
  t.format = "tsn:";
  t.data = d2h_pinned(out_ts_.p, (size_t)n_out * 8, stream_, &st_.d2h_bytes);
  ocols.push_back(t);
  AB_CUDA(cudaStreamSynchronize(stream_));
  st_.rows_out += (uint64_t)n_out;
  ++st_.windows_out;
  out->arrays.emplace_back();
  out->schemas.emplace_back();
  export_batch(ocols, n_out, &out->arrays.back(), &out->schemas.back());
}

}  // namespace

OpBase* make_ttl_join_op(const ArroyoB200OpConfig& cfg) { return new TtlJoinOp(cfg); }

}  // namespace ab
