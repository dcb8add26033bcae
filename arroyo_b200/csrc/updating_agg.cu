// Updating (non-windowed) keyed aggregate on sm_90a (H100): the GPU side of `IncrementalAggregatingFunc`
// (arroyo-worker/src/arrow/incremental_aggregator.rs), SURVEY.md 8(f) rank 2.
//
// The reference keeps one accumulator object per key and aggregate, updates them ONE ROW AT A TIME through dyn
// `Accumulator`s (:860-879), remembers for every key touched since the last flush the values it had before (:842-857)
// and, at a flush (every `flush_interval` tick, at checkpoints, at end of data), emits per touched key a retraction of
// the old values and an append of the new ones -- unless only the timestamp moved (:637-738).
//
// Here (append-only inputs: no `_updating_meta.is_retract` upstream; COUNT(*) / SUM / AVG / MIN / MAX over Int64):
//   ingest  one thread per row: dense id from the bucketed key dictionary (bdict.cuh), one RED per accumulator, the
//           trailing max(_timestamp) aggregate as a RED.max, and the key joins the touched list on its first row
//           since the last flush (atomicExch on a per-id flag).  A row whose bucket is out of ids is copied to a
//           deferral buffer; at the next host sync point the host doubles the bucket count and re-ingests it
//           (drain_deferred);
//   flush   one thread per touched key: compares the accumulators with their values at the previous flush (kept per
//           id: "the values it had before"), writes the retraction row (old values, old timestamp) and the append row
//           (new values), and rolls the snapshot forward.
// Output rows: [key?, aggregates..., _timestamp, is_retract] -- retractions first, then appends (a key's retraction
// must precede its append; the order between keys is unspecified in the reference too: it iterates a HashMap).
// The shim wraps `is_retract` into the `_updating_meta` struct together with the row id its metadata expression
// computes (:719-729).
//
// Not restated: retractions on the input (an updating upstream), count(distinct), TTL expiry (wall clock).  Such
// plans are refused at construction (ARROYO_B200_UNSUPPORTED) and stay on the stock operator.
#include <algorithm>
#include <climits>

#include "agg_plan.h"
#include "bdict.cuh"
#include "op.h"

namespace ab {
namespace {

struct UState {
  unsigned long long* cur;   // [n_acc][id_cap]; cur[0] = rows
  unsigned long long* prev;  // same layout: values at the previous flush (prev rows == 0: the key did not exist)
  long long* cur_ts;         // max(_timestamp)
  long long* prev_ts;
  unsigned int* touched;     // per id: in the touched list
  unsigned int* list;        // touched ids
  unsigned int* n_touched;
  unsigned long long id_cap;
  int n_acc;
  int acc_kind[MAX_ACC];
  int acc_val[MAX_ACC];
};

struct UIngest {
  const long long* key;
  const long long* ts;
  const long long* val[MAX_VALS];
  long long n;
  int keyed;
  int n_vals;
  BDict dict;
  UState st;
  // deferred rows: [key, ts, values...] columns with room for every row of the launch, and their count
  long long* d_key;
  long long* d_ts;
  long long* d_val[MAX_VALS];
  unsigned long long* deferred;
};

__device__ __noinline__ void upd_defer_row(const UIngest& p, long long i, long long key) {
  const unsigned long long d = atomicAdd(p.deferred, 1ull);
  p.d_key[d] = key;
  p.d_ts[d] = p.ts[i];
  for (int v = 0; v < p.n_vals; ++v) p.d_val[v][d] = p.val[v][i];
}

__global__ void __launch_bounds__(256) upd_ingest_kernel(const __grid_constant__ UIngest p) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (; i < p.n; i += stride) {
    uint32_t id = 0;
    if (p.keyed) {
      const long long key = __ldcs(p.key + i);
      id = bd_lookup_or_insert(p.dict, key);
      if (id >= ID_OVERFLOW) {  // the key's bucket is out of ids
        upd_defer_row(p, i, key);
        continue;
      }
    }
    atomicAdd(p.st.cur + id, 1ull);
#pragma unroll
    for (int a = 1; a < MAX_ACC; ++a) {
      if (a >= p.st.n_acc) break;
      const long long v = __ldcs(p.val[p.st.acc_val[a]] + i);
      unsigned long long* dst = p.st.cur + (unsigned long long)a * p.st.id_cap + id;
      switch (p.st.acc_kind[a]) {
        case ACC_SUM_I64: atomicAdd(dst, (unsigned long long)v); break;
        case ACC_SUM_F64: atomicAdd(reinterpret_cast<double*>(dst), (double)v); break;
        case ACC_MIN_I64: atomicMin(reinterpret_cast<long long*>(dst), v); break;
        case ACC_MAX_I64: atomicMax(reinterpret_cast<long long*>(dst), v); break;
      }
    }
    atomicMax(p.st.cur_ts + id, __ldcs(p.ts + i));
    if (atomicExch(p.st.touched + id, 1u) == 0u) p.st.list[atomicAdd(p.st.n_touched, 1u)] = id;
  }
}

struct UFlush {
  UState st;
  const long long* id_keys;
  unsigned int n;  // touched keys
  int keyed;
  int n_aggs;
  int agg_kind[ARROYO_B200_MAX_AGGS];
  int agg_acc[ARROYO_B200_MAX_AGGS];
  // output: retractions at [0, n_retract), appends at [n, n + n_append)
  long long* o_key;
  unsigned long long* o_agg[ARROYO_B200_MAX_AGGS];
  long long* o_ts;
  unsigned int* counts;  // [0] retractions, [1] appends
};

__global__ void __launch_bounds__(256) upd_flush_kernel(const __grid_constant__ UFlush p) {
  unsigned int i = blockIdx.x * blockDim.x + threadIdx.x;
  const unsigned int stride = gridDim.x * blockDim.x;
  for (; i < p.n; i += stride) {
    const unsigned int id = p.st.list[i];
    unsigned long long now[MAX_ACC], old[MAX_ACC];
    bool changed = false;
    for (int a = 0; a < p.st.n_acc; ++a) {
      now[a] = p.st.cur[(unsigned long long)a * p.st.id_cap + id];
      old[a] = p.st.prev[(unsigned long long)a * p.st.id_cap + id];
    }
    const bool had = old[0] != 0;
    // "don't bother emitting updates that just retract / append the same values (excluding the timestamp)" (:655-664):
    // compared on the OUTPUT values, like the reference compares ScalarValues
    for (int g = 0; g < p.n_aggs; ++g)
      changed = changed || agg_finalise(p.agg_kind[g], now[p.agg_acc[g]], now[0]) != agg_finalise(p.agg_kind[g], old[p.agg_acc[g]], old[0]);
    const long long now_ts = p.st.cur_ts[id], old_ts = p.st.prev_ts[id];
    const long long key = p.keyed ? p.id_keys[id] : 0;
    if (had && changed) {
      const unsigned int o = atomicAdd(p.counts + 0, 1u);
      if (p.keyed) p.o_key[o] = key;
      for (int g = 0; g < p.n_aggs; ++g) p.o_agg[g][o] = agg_finalise(p.agg_kind[g], old[p.agg_acc[g]], old[0]);
      p.o_ts[o] = old_ts;
    }
    if (!had || changed) {
      const unsigned int o = p.n + atomicAdd(p.counts + 1, 1u);
      if (p.keyed) p.o_key[o] = key;
      for (int g = 0; g < p.n_aggs; ++g) p.o_agg[g][o] = agg_finalise(p.agg_kind[g], now[p.agg_acc[g]], now[0]);
      p.o_ts[o] = now_ts;
    }
    for (int a = 0; a < p.st.n_acc; ++a) p.st.prev[(unsigned long long)a * p.st.id_cap + id] = now[a];
    p.st.prev_ts[id] = now_ts;
    p.st.touched[id] = 0;
  }
}

__global__ void upd_init_kernel(UState st, unsigned long long n) {
  unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
  const unsigned long long stride = (unsigned long long)gridDim.x * blockDim.x;
  for (; i < n; i += stride) {
    for (int a = 0; a < st.n_acc; ++a) {
      const unsigned long long v = acc_identity(st.acc_kind[a]);
      st.cur[(unsigned long long)a * st.id_cap + i] = v;
      st.prev[(unsigned long long)a * st.id_cap + i] = a == 0 ? 0 : v;
    }
    st.cur_ts[i] = LLONG_MIN;
    st.prev_ts[i] = LLONG_MIN;
    st.touched[i] = 0;
  }
}

// after the dictionary grew: new[map[i]] = old[i]
__global__ void upd_permute_kernel(UState o, UState n, const uint32_t* __restrict__ map, uint32_t old_ids) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  const uint32_t stride = gridDim.x * blockDim.x;
  for (; i < old_ids; i += stride) {
    const uint32_t m = map[i];
    if (m == ID_UNSET || m >= ID_OVERFLOW) continue;
    for (int a = 0; a < o.n_acc; ++a) {
      n.cur[(unsigned long long)a * n.id_cap + m] = o.cur[(unsigned long long)a * o.id_cap + i];
      n.prev[(unsigned long long)a * n.id_cap + m] = o.prev[(unsigned long long)a * o.id_cap + i];
    }
    n.cur_ts[m] = o.cur_ts[i];
    n.prev_ts[m] = o.prev_ts[i];
    n.touched[m] = o.touched[i];
  }
}
__global__ void upd_remap_list_kernel(unsigned int* list, unsigned int n, const uint32_t* __restrict__ map) {
  unsigned int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) list[i] = map[list[i]];
}

class UpdatingAggOp final : public OpBase {
 public:
  explicit UpdatingAggOp(const ArroyoB200OpConfig& c);
  ~UpdatingAggOp() override;
  void on_start(ArrowArray*, ArrowSchema*, int64_t n, int64_t, int64_t) override {
    AB_REQUIRE(n == 0, ARROYO_B200_UNSUPPORTED, "updating aggregate: state restore (tables 'a' / 'b') is not implemented");
  }
  void process_batch(uint32_t, uint32_t, ArrowArray* batch, const ArrowSchema* schema) override;
  void process_device_batch(uint32_t, uint32_t, const uint64_t* cols, int32_t n_cols, int64_t n_rows) override;
  // watermarks pass through an updating aggregate untouched (it emits on ticks, incremental_aggregator.rs:990-1004)
  void handle_watermark(int64_t, BatchesPriv*, std::vector<ArroyoB200DeviceBatch>*) override {}
  void handle_checkpoint(int64_t, BatchesPriv* out) override { flush_to(out); }  // :951-961
  void on_close(int end_of_data, BatchesPriv* out) override {                    // :1006-1018
    if (end_of_data && out) flush_to(out);
  }
  void handle_tick(BatchesPriv* out) override { flush_to(out); }  // :994-1004
  void flush() override {
    set_device();
    AB_CUDA(cudaStreamSynchronize(stream_));
  }
  void stats(ArroyoB200Stats* out) override {
    st_.n_keys = 0;
    if (plan_.keyed) {
      set_device();
      drain_deferred();  // also reads the dictionary's count (ids from BD_ID_BASE on)
      // id 0 is the INT64_MIN key's: it has rows once that key arrived
      unsigned long long min_key_rows = 0;
      AB_CUDA(cudaMemcpyAsync(&min_key_rows, cur_.p, 8, cudaMemcpyDeviceToHost, stream_));
      AB_CUDA(cudaStreamSynchronize(stream_));
      st_.n_keys = (uint64_t)total_keys_ + (min_key_rows ? 1 : 0);
    }
    *out = st_;
  }

 private:
  AggPlan plan_;
  std::string key_format_ = "l";
  // dictionary + state
  uint64_t n_buckets_ = 1, id_cap_ = 0;
  uint32_t total_keys_ = 0;
  DevBuf slots_, bucket_nkeys_, id_keys_, n_total_;
  DevBuf cur_, prev_, cur_ts_, prev_ts_, touched_, list_, counters_;  // counters_: [n_touched, retractions, appends, pad] u32 + deferred u64
  DevBuf staging_;
  uint64_t staging_cap_ = 0;
  // deferred rows (key, ts, values): two sets, one re-ingested while the other takes the rows that defer again
  DevBuf defer_[2][2 + MAX_VALS];
  uint64_t defer_cap_[2] = {0, 0};
  int defer_cur_ = 0;
  uint64_t out_cap_ = 0;
  DevBuf o_key_, o_ts_, o_agg_[ARROYO_B200_MAX_AGGS];
  ArroyoB200Stats st_{};

  BDict dict_view() const;
  UState state_view() const;
  void alloc_state(uint64_t n_buckets);
  void grow();
  void reserve_defer(int set, uint64_t rows);
  void drain_deferred();
  void ensure_room(uint64_t new_rows);
  void ingest(const long long* key, const long long* ts, const long long* const* vals, int64_t n);
  void flush_to(BatchesPriv* out);
};

UpdatingAggOp::UpdatingAggOp(const ArroyoB200OpConfig& c) {
  cfg = c;
  name = "UpdatingAggregatingFunc";
  AB_REQUIRE(!(c.flags & ARROYO_B200_FLAG_UPDATING_INPUT), ARROYO_B200_UNSUPPORTED,
             "updating aggregate over an updating input (retractions) is not supported");
  // AVG sums the inputs as f64, like the reference's accumulator (each value cast to f64, then added): an integer
  // sum would wrap and average to garbage once the values pass 2^63 in total
  plan_ = AggPlan(c, ACC_SUM_F64);
  open_device(c);
  counters_.alloc(32);
  AB_CUDA(cudaMemsetAsync(counters_.p, 0, 32, stream_));
  n_total_.alloc(4);
  AB_CUDA(cudaMemsetAsync(n_total_.p, 0, 4, stream_));
  alloc_state(plan_.keyed ? bd_buckets_for(c.expected_keys ? c.expected_keys : (1ull << 16)) : 1);
  AB_CUDA(cudaStreamSynchronize(stream_));
}

UpdatingAggOp::~UpdatingAggOp() { drain_stream(); }

BDict UpdatingAggOp::dict_view() const {
  BDict d{};
  d.slots = slots_.as<BSlot>();
  d.nkeys = bucket_nkeys_.as<unsigned int>();
  d.id_keys = id_keys_.as<long long>();
  d.n_total = n_total_.as<unsigned int>();
  d.n_buckets = (uint32_t)n_buckets_;
  return d;
}

UState UpdatingAggOp::state_view() const {
  UState s{};
  s.cur = cur_.as<unsigned long long>();
  s.prev = prev_.as<unsigned long long>();
  s.cur_ts = cur_ts_.as<long long>();
  s.prev_ts = prev_ts_.as<long long>();
  s.touched = touched_.as<unsigned int>();
  s.list = list_.as<unsigned int>();
  s.n_touched = counters_.as<unsigned int>();
  s.id_cap = id_cap_;
  s.n_acc = plan_.n_acc;
  for (int a = 0; a < plan_.n_acc; ++a) {
    s.acc_kind[a] = plan_.acc_kind[a];
    s.acc_val[a] = plan_.acc_val[a];
  }
  return s;
}

void UpdatingAggOp::alloc_state(uint64_t n_buckets) {
  n_buckets_ = n_buckets;
  id_cap_ = bd_id_cap(n_buckets_);
  AB_REQUIRE(id_cap_ < (1ull << 31), ARROYO_B200_RUNTIME, "key dictionary too large");
  id_keys_.alloc(id_cap_ * 8);
  bd_fill_keys_kernel<<<num_sms_ * 4, 256, 0, stream_>>>(id_keys_.as<long long>(), id_cap_);
  AB_CUDA(cudaGetLastError());
  bucket_nkeys_.alloc(n_buckets_ * 4);
  AB_CUDA(cudaMemsetAsync(bucket_nkeys_.p, 0, n_buckets_ * 4, stream_));
  if (plan_.keyed) {
    slots_.alloc(n_buckets_ * BD_KS * sizeof(BSlot));
    bd_init_kernel<<<num_sms_ * 4, 256, 0, stream_>>>(slots_.as<BSlot>(), n_buckets_ * BD_KS);
    AB_CUDA(cudaGetLastError());
  }
  cur_.alloc((size_t)plan_.n_acc * id_cap_ * 8);
  prev_.alloc((size_t)plan_.n_acc * id_cap_ * 8);
  cur_ts_.alloc(id_cap_ * 8);
  prev_ts_.alloc(id_cap_ * 8);
  touched_.alloc(id_cap_ * 4);
  list_.alloc(id_cap_ * 4);
  upd_init_kernel<<<num_sms_ * 4, 256, 0, stream_>>>(state_view(), id_cap_);
  AB_CUDA(cudaGetLastError());
  st_.kernel_launches += 2;
}

// Doubles the bucket count: keys are re-inserted (ids change), the per-id state and the touched list follow the map.
// A bucket's keys split between the two buckets that replace it, so the rehash itself never runs out of ids.
void UpdatingAggOp::grow() {
  // refused before anything moves: the operator stays usable
  AB_REQUIRE(bd_id_cap(n_buckets_ * 2) < (1ull << 31), ARROYO_B200_RUNTIME, "key dictionary too large");
  const BDict old_d = dict_view();
  const UState old_s = state_view();
  const uint32_t old_ids = (uint32_t)(BD_ID_BASE + n_buckets_ * BD_CAPB);
  const uint64_t old_cap = id_cap_;
  DevBuf k_slots = std::move(slots_), k_nk = std::move(bucket_nkeys_), k_keys = std::move(id_keys_), k_cur = std::move(cur_),
         k_prev = std::move(prev_), k_cts = std::move(cur_ts_), k_pts = std::move(prev_ts_), k_t = std::move(touched_),
         k_list = std::move(list_);
  unsigned int h_touched = 0;
  AB_CUDA(cudaMemcpyAsync(&h_touched, counters_.p, 4, cudaMemcpyDeviceToHost, stream_));
  AB_CUDA(cudaMemsetAsync(n_total_.p, 0, 4, stream_));
  AB_CUDA(cudaStreamSynchronize(stream_));
  alloc_state(n_buckets_ * 2);
  DevBuf map((size_t)old_cap * 4);
  const int grid = (int)std::min<uint64_t>((old_ids + 255) / 256, (uint64_t)num_sms_ * 8);
  bd_rehash_kernel<<<std::max(grid, 1), 256, 0, stream_>>>(old_d, dict_view(), old_ids, map.as<uint32_t>());
  AB_CUDA(cudaGetLastError());
  upd_permute_kernel<<<std::max(grid, 1), 256, 0, stream_>>>(old_s, state_view(), map.as<uint32_t>(), old_ids);
  AB_CUDA(cudaGetLastError());
  if (h_touched) {
    AB_CUDA(cudaMemcpyAsync(list_.p, k_list.p, (size_t)h_touched * 4, cudaMemcpyDeviceToDevice, stream_));
    upd_remap_list_kernel<<<(h_touched + 255) / 256, 256, 0, stream_>>>(list_.as<unsigned int>(), h_touched, map.as<uint32_t>());
    AB_CUDA(cudaGetLastError());
  }
  AB_CUDA(cudaMemcpyAsync(&total_keys_, n_total_.p, 4, cudaMemcpyDeviceToHost, stream_));
  AB_CUDA(cudaStreamSynchronize(stream_));
  st_.kernel_launches += 3;
}

void UpdatingAggOp::reserve_defer(int set, uint64_t rows) {
  if (rows <= defer_cap_[set]) return;
  defer_cap_[set] = std::max<uint64_t>(rows, defer_cap_[set] * 2);
  for (int c = 0; c < 2 + plan_.n_vals; ++c) defer_[set][c].alloc(defer_cap_[set] * 8);
}

// Re-ingests the rows the last launch deferred (their bucket was out of ids), doubling the bucket count before each
// pass.  Keys that share a bucket at several sizes need several passes; after DRAIN_STALLS passes in a row that placed
// none of the rows it gives up: RUNTIME, the rows are dropped and the operator stays usable.  Also reads the
// dictionary's key count into total_keys_.
void UpdatingAggOp::drain_deferred() {
  constexpr int DRAIN_STALLS = 4;
  unsigned long long* d_count = reinterpret_cast<unsigned long long*>((char*)counters_.p + 16);
  auto read = [&]() {
    unsigned long long n = 0;
    AB_CUDA(cudaMemcpyAsync(&n, d_count, 8, cudaMemcpyDeviceToHost, stream_));
    AB_CUDA(cudaMemcpyAsync(&total_keys_, n_total_.p, 4, cudaMemcpyDeviceToHost, stream_));
    AB_CUDA(cudaStreamSynchronize(stream_));
    return (uint64_t)n;
  };
  uint64_t n = read(), prev = UINT64_MAX;
  try {
    for (int stalls = 0; n > 0; prev = n, n = read()) {
      stalls = n < prev ? 0 : stalls + 1;
      AB_REQUIRE(stalls < DRAIN_STALLS, ARROYO_B200_RUNTIME,
                 "updating aggregate: rows whose dictionary bucket is out of ids still defer after the dictionary grew");
      st_.rows_deferred += n;
      grow();
      const int full = defer_cur_;
      defer_cur_ ^= 1;
      AB_CUDA(cudaMemsetAsync(d_count, 0, 8, stream_));
      const long long* vals[MAX_VALS] = {nullptr, nullptr, nullptr, nullptr};
      for (int v = 0; v < plan_.n_vals; ++v) vals[v] = defer_[full][2 + v].as<long long>();
      ingest(defer_[full][0].as<long long>(), defer_[full][1].as<long long>(), vals, (int64_t)n);
    }
  } catch (...) {
    cudaMemsetAsync(d_count, 0, 8, stream_);  // a failed drain must not fail every later call
    cudaStreamSynchronize(stream_);
    throw;
  }
}

// every row of the batch may bring a new key: keep the mean bucket fill at or under the target
void UpdatingAggOp::ensure_room(uint64_t new_rows) {
  if (!plan_.keyed) return;
  drain_deferred();
  while ((uint64_t)total_keys_ + new_rows > n_buckets_ * (uint64_t)BD_MEAN) grow();
}

void UpdatingAggOp::ingest(const long long* key, const long long* ts, const long long* const* vals, int64_t n) {
  if (n <= 0) return;
  UIngest p{};
  p.key = key;
  p.ts = ts;
  for (int v = 0; v < plan_.n_vals; ++v) p.val[v] = vals[v];
  p.n = n;
  p.keyed = plan_.keyed ? 1 : 0;
  p.n_vals = plan_.n_vals;
  p.dict = dict_view();
  p.st = state_view();
  if (plan_.keyed) {  // every row of the launch may defer (all rows of a key whose bucket is full do)
    reserve_defer(defer_cur_, (uint64_t)n);
    p.d_key = defer_[defer_cur_][0].as<long long>();
    p.d_ts = defer_[defer_cur_][1].as<long long>();
    for (int v = 0; v < plan_.n_vals; ++v) p.d_val[v] = defer_[defer_cur_][2 + v].as<long long>();
  }
  p.deferred = reinterpret_cast<unsigned long long*>((char*)counters_.p + 16);
  const int grid = (int)std::min<int64_t>((n + 255) / 256, (int64_t)num_sms_ * 8);
  upd_ingest_kernel<<<std::max(grid, 1), 256, 0, stream_>>>(p);
  AB_CUDA(cudaGetLastError());
  ++st_.kernel_launches;
  ++st_.ingest_launches;
}

void UpdatingAggOp::process_batch(uint32_t, uint32_t, ArrowArray* batch, const ArrowSchema* schema) {
  set_device();
  int64_t n = 0;
  std::vector<InColumn> cols = import_batch(batch, schema, &n);
  AB_REQUIRE((int)cols.size() == cfg.n_cols, ARROYO_B200_INVALID_ARGUMENT, "batch has the wrong number of columns");
  require_aggregate_input_types(cols, plan_.keyed ? plan_.key_col : -1, plan_.val_cols, plan_.n_vals);
  if (plan_.keyed) key_format_ = cols[plan_.key_col].format;
  st_.rows_in += (uint64_t)n;
  if (n == 0) {
    if (batch->release) batch->release(batch);
    return;
  }
  ensure_room((uint64_t)n);
  const int n_used = 2 + plan_.n_vals;
  if ((uint64_t)n > staging_cap_) {
    AB_CUDA(cudaStreamSynchronize(stream_));
    staging_cap_ = std::max<uint64_t>((uint64_t)n, staging_cap_ * 2);
    staging_.alloc((size_t)n_used * staging_cap_ * 8);
  }
  long long* base = staging_.as<long long>();
  const long long* vals[MAX_VALS] = {nullptr, nullptr, nullptr, nullptr};
  if (plan_.keyed) AB_CUDA(cudaMemcpyAsync(base, cols[plan_.key_col].data, (size_t)n * 8, cudaMemcpyHostToDevice, stream_));
  AB_CUDA(cudaMemcpyAsync(base + staging_cap_, cols[plan_.ts_col].data, (size_t)n * 8, cudaMemcpyHostToDevice, stream_));
  for (int v = 0; v < plan_.n_vals; ++v) {
    AB_CUDA(cudaMemcpyAsync(base + (size_t)(2 + v) * staging_cap_, cols[plan_.val_cols[v]].data, (size_t)n * 8, cudaMemcpyHostToDevice,
                            stream_));
    vals[v] = base + (size_t)(2 + v) * staging_cap_;
  }
  st_.h2d_bytes += (uint64_t)n * 8 * (uint64_t)((plan_.keyed ? 1 : 0) + 1 + plan_.n_vals);
  ingest(base, base + staging_cap_, vals, n);
  // the staging buffer is reused by the next batch: the copies and the kernel must have consumed the host batch
  AB_CUDA(cudaStreamSynchronize(stream_));
  if (batch->release) batch->release(batch);
  batch->release = nullptr;
}

void UpdatingAggOp::process_device_batch(uint32_t, uint32_t, const uint64_t* cols, int32_t n_cols, int64_t n_rows) {
  set_device();
  AB_REQUIRE(n_cols == cfg.n_cols, ARROYO_B200_INVALID_ARGUMENT, "batch has the wrong number of columns");
  if (n_rows <= 0) return;
  st_.rows_in += (uint64_t)n_rows;
  ensure_room((uint64_t)n_rows);
  const long long* vals[MAX_VALS] = {nullptr, nullptr, nullptr, nullptr};
  for (int v = 0; v < plan_.n_vals; ++v) vals[v] = (const long long*)cols[plan_.val_cols[v]];
  ingest(plan_.keyed ? (const long long*)cols[plan_.key_col] : nullptr, (const long long*)cols[plan_.ts_col], vals, n_rows);
}

static void* d2h_part(const void* dev, size_t off_rows, int64_t n, void* host, size_t host_off_rows, cudaStream_t s) {
  if (n > 0)
    AB_CUDA(cudaMemcpyAsync((char*)host + host_off_rows * 8, (const char*)dev + off_rows * 8, (size_t)n * 8, cudaMemcpyDeviceToHost, s));
  return host;
}

// flush (:637-738): one batch [key?, aggregates..., _timestamp, is_retract], or nothing when no key changed
void UpdatingAggOp::flush_to(BatchesPriv* out) {
  set_device();
  if (plan_.keyed) drain_deferred();
  struct {
    unsigned int touched, retracts, appends, pad;
  } h{};
  AB_CUDA(cudaMemcpyAsync(&h, counters_.p, 16, cudaMemcpyDeviceToHost, stream_));
  AB_CUDA(cudaStreamSynchronize(stream_));
  const unsigned int n = h.touched;
  if (n == 0 || !out) return;
  if (2ull * n > out_cap_) {
    out_cap_ = std::max<uint64_t>(2ull * n, 1024);
    o_key_.alloc(out_cap_ * 8);
    o_ts_.alloc(out_cap_ * 8);
    for (int g = 0; g < plan_.n_aggs; ++g) o_agg_[g].alloc(out_cap_ * 8);
  }
  UFlush p{};
  p.st = state_view();
  p.id_keys = id_keys_.as<long long>();
  p.n = n;
  p.keyed = plan_.keyed ? 1 : 0;
  p.n_aggs = plan_.n_aggs;
  for (int g = 0; g < plan_.n_aggs; ++g) {
    p.agg_kind[g] = plan_.agg_kind[g];
    p.agg_acc[g] = plan_.agg_acc[g];
    p.o_agg[g] = o_agg_[g].as<unsigned long long>();
  }
  p.o_key = o_key_.as<long long>();
  p.o_ts = o_ts_.as<long long>();
  p.counts = counters_.as<unsigned int>() + 1;
  const int grid = (int)std::min<unsigned int>((n + 255) / 256, (unsigned int)num_sms_ * 8);
  upd_flush_kernel<<<std::max(grid, 1), 256, 0, stream_>>>(p);
  AB_CUDA(cudaGetLastError());
  ++st_.kernel_launches;
  ++st_.emit_launches;
  AB_CUDA(cudaMemcpyAsync(&h, counters_.p, 16, cudaMemcpyDeviceToHost, stream_));
  AB_CUDA(cudaMemsetAsync(counters_.p, 0, 16, stream_));  // touched list and output counters start over
  AB_CUDA(cudaStreamSynchronize(stream_));
  const int64_t nr = h.retracts, na = h.appends, total = nr + na;
  if (total == 0) return;
  std::vector<OutColumn> cols;
  auto column = [&](const char* nm, const std::string& fmt, const void* dev) {
    OutColumn c;
    c.name = nm;
    c.format = fmt;
    void* host = PinnedPool::get().alloc((size_t)std::max<int64_t>(total, 1) * 8);
    d2h_part(dev, 0, nr, host, 0, stream_);
    d2h_part(dev, n, na, host, (size_t)nr, stream_);
    st_.d2h_bytes += (uint64_t)total * 8;
    c.data = host;
    cols.push_back(c);
  };
  if (plan_.keyed) column("key", key_format_, o_key_.p);
  for (int g = 0; g < plan_.n_aggs; ++g) column(("agg" + std::to_string(g)).c_str(), plan_.agg_format[g], o_agg_[g].p);
  column("_timestamp", "tsn:", o_ts_.p);
  {
    OutColumn r;
    r.name = "is_retract";
    r.format = "b";
    unsigned char* bits = (unsigned char*)PinnedPool::get().alloc((size_t)(total + 7) / 8 + 8);
    memset(bits, 0, (size_t)(total + 7) / 8 + 8);
    for (int64_t i = 0; i < nr; ++i) bits[i >> 3] |= (unsigned char)(1u << (i & 7));
    r.data = bits;
    cols.push_back(r);
  }
  AB_CUDA(cudaStreamSynchronize(stream_));
  st_.rows_out += (uint64_t)total;
  ++st_.windows_out;
  out->arrays.emplace_back();
  out->schemas.emplace_back();
  export_batch(cols, total, &out->arrays.back(), &out->schemas.back());
}

}  // namespace

OpBase* make_updating_agg_op(const ArroyoB200OpConfig& cfg) { return new UpdatingAggOp(cfg); }

}  // namespace ab
