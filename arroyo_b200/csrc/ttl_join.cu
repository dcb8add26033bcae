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
#include <memory>

#include "join_side.h"

namespace ab {
namespace {

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

struct TSide : JoinSide {
  DevBuf next, tab;
  uint32_t tab_cap = 0;
  uint64_t keys_bound = 0;  // rows linked so far: an upper bound of the distinct keys
};

class TtlJoinOp final : public JoinOpBase {
 public:
  explicit TtlJoinOp(const ArroyoB200OpConfig& c);
  ~TtlJoinOp() override;
  void on_start(ArrowArray*, ArrowSchema*, int64_t n, int64_t, int64_t) override {
    AB_REQUIRE(n == 0, ARROYO_B200_UNSUPPORTED,
               "JoinWithExpiration restore: hand each key-time table to arroyo_b200_op_restore_side");
  }
  void restore_side(uint32_t side, ArrowArray* batches, ArrowSchema* schemas, int64_t n) override;
  void process_batch(uint32_t index, uint32_t parts, ArrowArray* batch, const ArrowSchema* schema) override {
    std::unique_ptr<BatchesPriv, void (*)(BatchesPriv*)> sink(new BatchesPriv(), discard);
    process_batch_emit(index, parts, batch, schema, sink.get());
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

 private:
  TSide side_[2];
  DevBuf cnt_, off_, total_;
  bool took_input_ = false;  // process_batch has accepted a batch: restore_side is refused from then on

  void ensure_table(TSide& s, uint64_t more_rows);
  void insert(TSide& s, const JoinBatch* in, int64_t n_batches, int64_t rows);
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
    tj_rehash_kernel<<<grid_for(s.tab_cap), JOIN_THREADS, 0, stream_>>>(s.tab.as<MSlot>(), s.tab_cap, nt.as<MSlot>(),
                                                                       (uint32_t)(nc - 1));
    AB_CUDA(cudaGetLastError());
    ++st_.kernel_launches;
  }
  AB_CUDA(cudaStreamSynchronize(stream_));
  s.tab = std::move(nt);
  s.tab_cap = (uint32_t)nc;
}

// Inserts accepted host batches of `rows` rows in all into side `s`'s key-time table (:52 / :83, insert_internal
// :1008-1049): one reserve and one table sizing for all of them, their rows copied into consecutive arena ranges,
// then linked into the multimap by one launch.
void TtlJoinOp::insert(TSide& s, const JoinBatch* in, int64_t n_batches, int64_t rows) {
  s.reserve(rows, stream_, &s.next);
  ensure_table(s, (uint64_t)rows);
  const int64_t first = s.n;
  for (int64_t b = 0; b < n_batches; ++b)
    if (in[b].n) s.append(in[b].data, in[b].n, true, stream_, st_);
  tj_link_kernel<<<grid_for(rows), JOIN_THREADS, 0, stream_>>>(s.cols[s.key_col].as<long long>(), first, rows,
                                                              s.tab.as<MSlot>(), s.tab_cap - 1, s.next.as<int>());
  AB_CUDA(cudaGetLastError());
  ++st_.kernel_launches;
  s.keys_bound += (uint64_t)rows;
}

// KeyTimeView::insert_internal (:1008-1049) for the batches of one side's table: every batch is checked before anything
// changes, then the call's rows are inserted without probing.  A restore that succeeds takes every batch.
void TtlJoinOp::restore_side(uint32_t side, ArrowArray* batches, ArrowSchema* schemas, int64_t n) {
  AB_REQUIRE(side <= 1, ARROYO_B200_INVALID_ARGUMENT, "restore_side: side must be 0 (left) or 1 (right)");
  AB_REQUIRE(n >= 0 && (n == 0 || (batches != nullptr && schemas != nullptr)), ARROYO_B200_INVALID_ARGUMENT,
             "restore_side: null batches");
  AB_REQUIRE(!took_input_, ARROYO_B200_INVALID_ARGUMENT,
             "JoinWithExpiration: restore_side after process_batch (restore before the first batch)");
  TSide& s = side_[side];
  std::vector<JoinBatch> in((size_t)n);
  int64_t total = 0;
  for (int64_t b = 0; b < n; ++b) {
    in[b] = s.import(&batches[b], &schemas[b], b ? in[b - 1].cols[s.key_col].format : s.key_format, side_[1 - side],
                     "restore_side: batch does not have the side's number of columns");
    total += in[b].n;
  }
  set_device();
  if (total > 0) {
    insert(s, in.data(), n, total);
    AB_CUDA(cudaStreamSynchronize(stream_));
  }
  if (n > 0) s.take_formats(in[n - 1].cols);
  for (int64_t b = 0; b < n; ++b)
    if (batches[b].release) batches[b].release(&batches[b]);
}

void TtlJoinOp::process_batch_emit(uint32_t index, uint32_t parts, ArrowArray* batch, const ArrowSchema* schema, BatchesPriv* out) {
  set_device();
  const int sd = side_of(index, parts);
  TSide& s = side_[sd];
  TSide& o = side_[1 - sd];
  const JoinBatch b = s.import(batch, schema, s.key_format, o);
  s.take_formats(b.cols);
  took_input_ = true;
  st_.rows_in += (uint64_t)b.n;
  const int64_t n = b.n;
  if (n == 0) {
    if (batch->release) batch->release(batch);
    batch->release = nullptr;
    return;
  }
  // 1. append + link (insert into this side's key-time table, :52 / :83)
  const long long first = s.n;
  insert(s, &b, 1, n);
  ++st_.ingest_launches;
  // 2. the other side's rows of these keys (get_batch, :59-64 / :90-95) x the batch (compute_pair)
  int64_t n_out = 0;
  if (o.n > 0) {
    grow(cnt_, (size_t)n * 4);
    grow(off_, (size_t)n * 8);
    const long long* pkey = s.cols[s.key_col].as<long long>();
    unsigned long long h_total = 0;
    n_out = count_pairs(
        [&] {
          tj_probe_kernel<0><<<grid_for(n), JOIN_THREADS, 0, stream_>>>(pkey, first, n, o.tab.as<MSlot>(), o.tab_cap - 1,
                                                                        o.next.as<int>(), cnt_.as<unsigned int>(), nullptr,
                                                                        nullptr, nullptr);
        },
        cnt_.as<unsigned int>(), n, off_.as<unsigned long long>(), total_.as<unsigned long long>(), &h_total);
    if (n_out > 0) {
      reserve_pairs(n_out);
      tj_probe_kernel<1><<<grid_for(n), JOIN_THREADS, 0, stream_>>>(pkey, first, n, o.tab.as<MSlot>(), o.tab_cap - 1,
                                                                    o.next.as<int>(), nullptr, off_.as<unsigned long long>(),
                                                                    pairs_[sd].as<int>(), pairs_[1 - sd].as<int>());
      AB_CUDA(cudaGetLastError());
      ++st_.kernel_launches;
    }
  }
  // the host batch may go once its copies have been consumed
  AB_CUDA(cudaStreamSynchronize(stream_));
  if (batch->release) batch->release(batch);
  batch->release = nullptr;
  if (n_out == 0) return;
  // 3. output = [left payload..., right payload..., _timestamp = max(l, r)]
  write_output(side_[0], side_[1], n_out, false, false, out, nullptr);
  ++st_.emit_launches;
}

}  // namespace

OpBase* make_ttl_join_op(const ArroyoB200OpConfig& cfg) { return new TtlJoinOp(cfg); }

}  // namespace ab
