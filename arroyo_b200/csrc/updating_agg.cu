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
//           (new values), and rolls the snapshot forward.  It also marks the id "flushed since the last state
//           export" (one byte store per key);
//   state   checkpoint_state writes table "a" (checkpoint_sliding :272-340, insert_batch :619-635): one row per marked
//           id, compacted from the snapshot, [key?, per aggregate its accumulator state, _timestamp, _generation].
//           The reference writes at every flush; writing at a checkpoint the keys flushed since the last export leaves
//           the same latest row per key.  Every export carries one generation, one above the last;
//   restore on_start (initialize :446-503) reads table "a" back: the keys go into the dictionary (BucketDict::place,
//           which grows it when a bucket runs out of ids), the row with the largest (_generation, position) wins per key and seeds both the
//           live accumulators and the previous-flush snapshot, so the first flush retracts what the uninterrupted run
//           would have retracted.
//   ttl     time-to-idle (UpdatingCache::with_time_to_idle, updating_cache.rs:42-62; time_out at every flush,
//           :688-705), on the clock the shim sets (arroyo_b200_op_set_clock; the library reads no clock).  Only when
//           the ttl (config gap_ns) is > 0: the ingest stamps each row's id with the clock of its call (a store only
//           when the stamp changes, so a hot key costs one load per row); rows that defer are drained before the
//           clock moves, so they keep the clock of the call that brought them.  After the flush kernel,
//           upd_expire_kernel evicts every live id with clock - stamp >= ttl: one retraction row of its previous-flush
//           values (what the reference's evaluate() returns after the flush), the id back to identity, and
//           flushed = 2: "evicted since the last export", which the export writes as a tombstone (null _timestamp,
//           the reference's deletion encoding in initialize :591-614) unless the key is flushed again first.  When
//           the ids that hold neither a live key nor a pending tombstone are half of the ids handed out (from 2^16
//           on), the dictionary is rebuilt from the kept keys (BucketDict::rebuild) and the per-id state follows the
//           old -> new id map, so device memory follows the live keys.  With ttl 0 none of this runs: the ingest is
//           the TTL = false instance, and the flush and export kernels do what they did without a ttl.
// Output rows: [key?, aggregates..., _timestamp, is_retract] -- retractions first, then appends (a key's retraction
// must precede its append; the order between keys is unspecified in the reference too: it iterates a HashMap), then
// the eviction retractions (the reference appends them last, :690-701).
// The shim wraps `is_retract` into the `_updating_meta` struct together with the row id its metadata expression
// computes (:719-729).
// Deviations with a ttl (INTEGRATION.md §3): eviction retractions leave even when the flush has no other row (the
// reference returns None then, :703-705, after it has evicted the keys); evicted keys leave tombstones in table "a",
// so a restore does not bring them back (the reference's table keeps their last rows).
//
// Not restated: retractions on the input (an updating upstream), count(distinct).  Such plans are refused at
// construction (ARROYO_B200_UNSUPPORTED) and stay on the stock operator.
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
  unsigned char* flushed;    // per id: flushed since the last state export
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
  // TTL only: per id the clock of its last row, the clock of this launch, and the live-key count (a key becomes live
  // on its first row after a flush that left it without rows: new, or back after an eviction)
  long long* last;
  long long now;
  unsigned int* n_live;
};

__device__ __noinline__ void upd_defer_row(const UIngest& p, long long i, long long key) {
  const unsigned long long d = atomicAdd(p.deferred, 1ull);
  p.d_key[d] = key;
  p.d_ts[d] = p.ts[i];
  for (int v = 0; v < p.n_vals; ++v) p.d_val[v][d] = p.val[v][i];
}

template <bool TTL>
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
    if (TTL && p.last[id] != p.now) p.last[id] = p.now;  // every writer stores the same value
    acc_red(ACC_ROWS, p.st.cur + id, 1ull);
#pragma unroll
    for (int a = 1; a < MAX_ACC; ++a) {
      if (a >= p.st.n_acc) break;
      const int kind = p.st.acc_kind[a];
      const long long v = __ldcs(p.val[p.st.acc_val[a]] + i);
      acc_red(kind, p.st.cur + (unsigned long long)a * p.st.id_cap + id, acc_of_value(kind, v));
    }
    acc_red(ACC_MAX_I64, reinterpret_cast<unsigned long long*>(p.st.cur_ts + id), (unsigned long long)__ldcs(p.ts + i));
    if (atomicExch(p.st.touched + id, 1u) == 0u) {
      p.st.list[atomicAdd(p.st.n_touched, 1u)] = id;
      if (TTL && p.st.prev[id] == 0) atomicAdd(p.n_live, 1u);  // prev rows == 0: no rows at the last flush
    }
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
#ifndef AB_UPDATING_NO_FLUSH_MARK  // measurement knob (tools/updating_state_rates.py): the flush without its store
    p.st.flushed[id] = 1;
#endif
  }
}

// Expiry (time_out, :690-701), after the flush kernel: every live id idle for at least the ttl leaves as one
// retraction row of its previous-flush values, compacted with one atomic per warp, and goes back to identity, marked
// flushed = 2 (a tombstone for the next export).  The touched list is empty here.
struct UExpire {
  UState st;
  const long long* id_keys;
  const long long* last;
  long long now, ttl;
  unsigned long long n_ids;  // ids to scan: [0, n_ids)
  int keyed;
  int n_aggs;
  int agg_kind[ARROYO_B200_MAX_AGGS];
  int agg_acc[ARROYO_B200_MAX_AGGS];
  long long* o_key;  // the eviction region of the flush's output
  unsigned long long* o_agg[ARROYO_B200_MAX_AGGS];
  long long* o_ts;
  unsigned int* count;   // rows written
  unsigned int* n_live;  // live keys, less the evicted ones
};

__global__ void __launch_bounds__(256) upd_expire_kernel(const __grid_constant__ UExpire p) {
  unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
  const unsigned long long stride = (unsigned long long)gridDim.x * blockDim.x;
  const unsigned int lane = threadIdx.x & 31;
  for (; i < p.n_ids; i += stride) {
    // clock >= every stamp >= 0: the difference cannot overflow
    const bool mine = p.st.prev[i] != 0 && p.now - p.last[i] >= p.ttl;
    const unsigned int active = __activemask();
    const unsigned int mask = __ballot_sync(active, mine);
    if (!mask) continue;
    const int leader = __ffs(active) - 1;
    unsigned int base = 0;
    if ((int)lane == leader) {
      base = atomicAdd(p.count, (unsigned int)__popc(mask));
      atomicSub(p.n_live, (unsigned int)__popc(mask));
    }
    base = __shfl_sync(active, base, leader);
    if (!mine) continue;
    const unsigned int o = base + __popc(mask & ((1u << lane) - 1u));
    unsigned long long old[MAX_ACC];
    for (int a = 0; a < p.st.n_acc; ++a) old[a] = p.st.prev[(unsigned long long)a * p.st.id_cap + i];
    if (p.keyed) p.o_key[o] = p.id_keys[i];
    for (int g = 0; g < p.n_aggs; ++g) p.o_agg[g][o] = agg_finalise(p.agg_kind[g], old[p.agg_acc[g]], old[0]);
    p.o_ts[o] = p.st.prev_ts[i];
    for (int a = 0; a < p.st.n_acc; ++a) {
      const unsigned long long v = acc_identity(p.st.acc_kind[a]);
      p.st.cur[(unsigned long long)a * p.st.id_cap + i] = v;
      p.st.prev[(unsigned long long)a * p.st.id_cap + i] = a == 0 ? 0 : v;
    }
    p.st.cur_ts[i] = LLONG_MIN;
    p.st.prev_ts[i] = LLONG_MIN;
    p.st.flushed[i] = 2;
  }
}

// Compaction: the ids to keep -- a live key (rows now or at the last flush) or one with a pending export row
__global__ void upd_keep_kernel(UState st, unsigned char* keep, uint32_t n_ids) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  const uint32_t stride = gridDim.x * blockDim.x;
  for (; i < n_ids; i += stride) keep[i] = st.cur[i] != 0 || st.prev[i] != 0 || st.flushed[i] != 0;
}

// State export: every id flushed since the last export leaves as one row of its previous-flush snapshot (the values
// the last flush emitted), compacted with one atomic per warp; an id evicted since (flushed = 2) leaves as a
// tombstone, o_dead[row] = 1 (o_dead is null without a ttl).
struct UExport {
  UState st;
  const long long* id_keys;
  unsigned long long n_ids;  // ids to scan: [0, n_ids)
  long long* o_key;
  unsigned long long* o_acc[MAX_ACC];
  long long* o_ts;
  unsigned int* count;
  unsigned char* o_dead;
};

__global__ void __launch_bounds__(256) upd_export_kernel(const __grid_constant__ UExport p) {
  unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
  const unsigned long long stride = (unsigned long long)gridDim.x * blockDim.x;
  const unsigned int lane = threadIdx.x & 31;
  for (; i < p.n_ids; i += stride) {
    const bool mine = p.st.flushed[i] != 0;
    const unsigned int active = __activemask();
    const unsigned int mask = __ballot_sync(active, mine);
    if (!mask) continue;
    const int leader = __ffs(active) - 1;
    unsigned int base = 0;
    if ((int)lane == leader) base = atomicAdd(p.count, (unsigned int)__popc(mask));
    base = __shfl_sync(active, base, leader);
    if (!mine) continue;
    const unsigned int o = base + __popc(mask & ((1u << lane) - 1u));
    if (p.o_dead) p.o_dead[o] = p.st.flushed[i] == 2;
    p.st.flushed[i] = 0;
    p.o_key[o] = p.id_keys[i];
    for (int a = 0; a < p.st.n_acc; ++a) p.o_acc[a][o] = p.st.prev[(unsigned long long)a * p.st.id_cap + i];
    p.o_ts[o] = p.st.prev_ts[i];
  }
}

// Restore: rows of table "a" in batch order, one thread per row.
struct URestore {
  UState st;
  const unsigned long long* gen;
  const unsigned long long* val[MAX_ACC];  // per accumulator; val[0] null: every row counts one
  const long long* ts;
  const unsigned int* ids;        // per row, from BucketDict::place
  unsigned long long* best_gen;   // per id
  long long* best_pos;            // per id, -1: no row
  long long n;
  const unsigned char* dead;      // per row, 1: a tombstone (null _timestamp); null when the table has none
  long long* last;                // TTL only: per id, stamped with `now`
  long long now;
  unsigned int* won;              // [0] keys restored live, [1] keys whose winning row is a tombstone
};

// the largest generation per id, then the last row of that generation
__global__ void __launch_bounds__(256) upd_restore_gen_kernel(const __grid_constant__ URestore p) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (; i < p.n; i += stride) atomicMax(p.best_gen + p.ids[i], p.gen[i]);
}
__global__ void __launch_bounds__(256) upd_restore_pos_kernel(const __grid_constant__ URestore p) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (; i < p.n; i += stride) {
    const unsigned int id = p.ids[i];
    if (p.gen[i] == p.best_gen[id]) atomicMax(p.best_pos + id, i);
  }
}

// the winning row seeds the live accumulators and the previous-flush snapshot alike; a winning tombstone leaves the
// id at identity (the key is absent)
__global__ void __launch_bounds__(256) upd_restore_seed_kernel(const __grid_constant__ URestore p) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (; i < p.n; i += stride) {
    const unsigned int id = p.ids[i];
    const bool win = p.best_pos[id] == i;
    const bool dead = win && p.dead && p.dead[i];
    const unsigned int active = __activemask();
    const unsigned int live_mask = __ballot_sync(active, win && !dead), dead_mask = __ballot_sync(active, dead);
    if ((int)(threadIdx.x & 31) == __ffs(active) - 1) {  // one atomic per warp
      if (live_mask) atomicAdd(p.won, (unsigned int)__popc(live_mask));
      if (dead_mask) atomicAdd(p.won + 1, (unsigned int)__popc(dead_mask));
    }
    if (!win || dead) continue;
    if (p.last) p.last[id] = p.now;
    for (int a = 0; a < p.st.n_acc; ++a) {
      const unsigned long long v = p.val[a] ? p.val[a][i] : 1ull;
      p.st.cur[(unsigned long long)a * p.st.id_cap + id] = v;
      p.st.prev[(unsigned long long)a * p.st.id_cap + id] = v;
    }
    p.st.cur_ts[id] = p.ts[i];
    p.st.prev_ts[id] = p.ts[i];
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
    st.flushed[i] = 0;
  }
}

// after the dictionary grew or was rebuilt: new[map[i]] = old[i]; o_last / n_last (the TTL stamps) may be null
__global__ void upd_permute_kernel(UState o, UState n, const long long* o_last, long long* n_last,
                                   const uint32_t* __restrict__ map, uint32_t old_ids) {
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
    n.flushed[m] = o.flushed[i];
    if (n_last) n_last[m] = o_last[i];
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
  void on_start(ArrowArray* state, ArrowSchema* schemas, int64_t n, int64_t, int64_t) override;
  void process_batch(uint32_t, uint32_t, ArrowArray* batch, const ArrowSchema* schema) override;
  void process_device_batch(uint32_t, uint32_t, const uint64_t* cols, int32_t n_cols, int64_t n_rows) override;
  // watermarks pass through an updating aggregate untouched (it emits on ticks, incremental_aggregator.rs:990-1004)
  void handle_watermark(int64_t, BatchesPriv*, std::vector<ArroyoB200DeviceBatch>*) override {}
  void handle_checkpoint(int64_t, BatchesPriv* out) override { flush_to(out); }  // :951-961
  void on_close(int end_of_data, BatchesPriv* out) override {                    // :1006-1018
    if (end_of_data && out) flush_to(out);
  }
  void handle_tick(BatchesPriv* out) override { flush_to(out); }  // :994-1004
  void checkpoint_state(BatchesPriv* out) override;
  void set_clock(int64_t now_ns) override;
  void flush() override {
    set_device();
    AB_CUDA(cudaStreamSynchronize(stream_));
  }
  void stats(ArroyoB200Stats* out) override {
    st_.n_keys = 0;
    if (plan_.keyed && ttl_ns_ > 0) {
      set_device();
      drain_deferred();
      st_.n_keys = read_live();
    } else if (plan_.keyed) {
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
  // dictionary (its key counter in n_total_) + per-id state
  BucketDict dict_;
  uint32_t total_keys_ = 0;
  DevBuf n_total_;
  DevBuf cur_, prev_, cur_ts_, prev_ts_, touched_, flushed_, list_, counters_;  // counters_: [n_touched, retractions, appends, pad] u32 + deferred u64
  AggStaging staging_;
  // deferred rows (key, ts, values): two sets, one re-ingested while the other takes the rows that defer again
  DevBuf defer_[2][2 + MAX_VALS];
  uint64_t defer_cap_[2] = {0, 0};
  int defer_cur_ = 0;
  uint64_t out_cap_ = 0;
  DevBuf o_key_, o_ts_, o_agg_[ARROYO_B200_MAX_AGGS];
  // state export: keys flushed since the last export (an upper bound: a key flushed twice counts twice), the
  // generation the next export writes, and the export's output buffers
  uint64_t unexported_ = 0, generation_ = 0, state_cap_ = 0;
  bool restored_ = false;
  DevBuf s_key_, s_ts_, s_acc_[MAX_ACC], s_dead_;
  ArroyoB200Stats st_{};
  // time-to-idle: the ttl (0: keys never expire), the clock, per id the clock of its last row, [live keys, evicted
  // by the last expiry pass] (u32), the evictions since the last export (an upper bound on the pending tombstones),
  // and the dictionary's size at construction (a compaction does not go below it)
  int64_t ttl_ns_ = 0, clock_ = 0;
  DevBuf last_, ttl_counters_;
  uint64_t tombstones_ = 0, min_buckets_ = 1;

  UState state_view() const;
  void alloc_state();
  void grow();
  void follow(const UState& old_s, const BdGrowth& g);
  uint32_t read_live();
  void maybe_compact(uint64_t live);
  void compact();
  void reserve_defer(int set, uint64_t rows);
  void drain_deferred();
  void ensure_room(uint64_t new_rows);
  void ingest(const AggCols& d, int64_t n);
  void flush_to(BatchesPriv* out);
  void launch_flush(unsigned int n);
  void launch_expire(unsigned int n);
  void export_state(BatchesPriv* out, unsigned int rows, bool dead);
};

UpdatingAggOp::UpdatingAggOp(const ArroyoB200OpConfig& c) {
  cfg = c;
  name = "UpdatingAggregatingFunc";
  AB_REQUIRE(!(c.flags & ARROYO_B200_FLAG_UPDATING_INPUT), ARROYO_B200_UNSUPPORTED,
             "updating aggregate over an updating input (retractions) is not supported");
  // AVG sums the inputs as f64, like the reference's accumulator (each value cast to f64, then added): an integer
  // sum would wrap and average to garbage once the values pass 2^63 in total
  plan_ = AggPlan(c, ACC_SUM_F64);
  AB_REQUIRE(c.gap_ns >= 0, ARROYO_B200_INVALID_ARGUMENT, "updating aggregate: negative ttl (gap_ns)");
  ttl_ns_ = c.gap_ns;
  open_device(c);
  counters_.alloc(32);
  AB_CUDA(cudaMemsetAsync(counters_.p, 0, 32, stream_));
  n_total_.alloc(4);
  AB_CUDA(cudaMemsetAsync(n_total_.p, 0, 4, stream_));
  if (ttl_ns_ > 0) {
    ttl_counters_.alloc(8);
    AB_CUDA(cudaMemsetAsync(ttl_counters_.p, 0, 8, stream_));
  }
  dict_.init(stream_, num_sms_, plan_.keyed, n_total_.as<unsigned int>(), &st_.kernel_launches);
  min_buckets_ = plan_.keyed ? bd_buckets_for(c.expected_keys ? c.expected_keys : (1ull << 16)) : 1;
  dict_.alloc(min_buckets_);
  alloc_state();
  AB_CUDA(cudaStreamSynchronize(stream_));
}

UpdatingAggOp::~UpdatingAggOp() { drain_stream(); }

UState UpdatingAggOp::state_view() const {
  UState s{};
  s.cur = cur_.as<unsigned long long>();
  s.prev = prev_.as<unsigned long long>();
  s.cur_ts = cur_ts_.as<long long>();
  s.prev_ts = prev_ts_.as<long long>();
  s.touched = touched_.as<unsigned int>();
  s.flushed = flushed_.as<unsigned char>();
  s.list = list_.as<unsigned int>();
  s.n_touched = counters_.as<unsigned int>();
  s.id_cap = dict_.id_cap();
  s.n_acc = plan_.n_acc;
  for (int a = 0; a < plan_.n_acc; ++a) {
    s.acc_kind[a] = plan_.acc_kind[a];
    s.acc_val[a] = plan_.acc_val[a];
  }
  return s;
}

// The per-id state for the dictionary's id capacity, every id at its identity.
void UpdatingAggOp::alloc_state() {
  const uint64_t id_cap = dict_.id_cap();
  cur_.alloc((size_t)plan_.n_acc * id_cap * 8);
  prev_.alloc((size_t)plan_.n_acc * id_cap * 8);
  cur_ts_.alloc(id_cap * 8);
  prev_ts_.alloc(id_cap * 8);
  touched_.alloc(id_cap * 4);
  flushed_.alloc(id_cap);
  list_.alloc(id_cap * 4);
  if (ttl_ns_ > 0) {
    last_.alloc(id_cap * 8);
    AB_CUDA(cudaMemsetAsync(last_.p, 0, id_cap * 8, stream_));
  }
  upd_init_kernel<<<num_sms_ * 4, 256, 0, stream_>>>(state_view(), id_cap);
  AB_CUDA(cudaGetLastError());
  ++st_.kernel_launches;
}

// Doubles the bucket count (BucketDict::grow, refused before anything moves: the operator stays usable); the per-id
// state and the touched list follow the old -> new id map.
void UpdatingAggOp::grow() {
  const UState old_s = state_view();
  follow(old_s, dict_.grow());
}

// The per-id state (viewed by `old_s`), the TTL stamps and the touched list move to the dictionary's new ids.
void UpdatingAggOp::follow(const UState& old_s, const BdGrowth& g) {
  DevBuf k_cur = std::move(cur_), k_prev = std::move(prev_), k_cts = std::move(cur_ts_), k_pts = std::move(prev_ts_),
         k_t = std::move(touched_), k_f = std::move(flushed_), k_list = std::move(list_), k_last = std::move(last_);
  unsigned int h_touched = 0;
  AB_CUDA(cudaMemcpyAsync(&h_touched, counters_.p, 4, cudaMemcpyDeviceToHost, stream_));
  AB_CUDA(cudaStreamSynchronize(stream_));
  alloc_state();
  const int grid = (int)std::min<uint64_t>((g.old_ids + 255) / 256, (uint64_t)num_sms_ * 8);
  upd_permute_kernel<<<std::max(grid, 1), 256, 0, stream_>>>(old_s, state_view(), k_last.as<long long>(),
                                                             last_.as<long long>(), g.map.as<uint32_t>(), g.old_ids);
  AB_CUDA(cudaGetLastError());
  ++st_.kernel_launches;
  if (h_touched) {
    AB_CUDA(cudaMemcpyAsync(list_.p, k_list.p, (size_t)h_touched * 4, cudaMemcpyDeviceToDevice, stream_));
    upd_remap_list_kernel<<<(h_touched + 255) / 256, 256, 0, stream_>>>(list_.as<unsigned int>(), h_touched, g.map.as<uint32_t>());
    AB_CUDA(cudaGetLastError());
    ++st_.kernel_launches;
  }
  AB_CUDA(cudaMemcpyAsync(&total_keys_, n_total_.p, 4, cudaMemcpyDeviceToHost, stream_));
  AB_CUDA(cudaStreamSynchronize(stream_));
}

// TTL only: the live-key count
uint32_t UpdatingAggOp::read_live() {
  uint32_t live = 0;
  AB_CUDA(cudaMemcpyAsync(&live, ttl_counters_.p, 4, cudaMemcpyDeviceToHost, stream_));
  AB_CUDA(cudaStreamSynchronize(stream_));
  return live;
}

// After an expiry pass or an export (TTL only): once the ids handed out that hold neither a live key (`live` of
// them) nor a pending tombstone are at least half of them, from 2^16 ids on, the dictionary is rebuilt from the kept
// keys and the per-id state follows.  Id 0 (the INT64_MIN key) keeps its place.
void UpdatingAggOp::maybe_compact(uint64_t live) {
  constexpr uint64_t COMPACT_MIN_IDS = 1ull << 16;
  if (!plan_.keyed || total_keys_ < COMPACT_MIN_IDS) return;
  const uint64_t kept = std::min<uint64_t>(live + tombstones_, total_keys_);
  if (2 * (total_keys_ - kept) < total_keys_) return;
  compact();
}

// Rebuilds the dictionary from the keys of the ids that hold a live key or a pending export row.
void UpdatingAggOp::compact() {
  const UState old_s = state_view();
  const uint32_t n_ids = dict_.n_ids();
  DevBuf keep(n_ids);
  const int grid = (int)std::min<uint64_t>((n_ids + 255) / 256, (uint64_t)num_sms_ * 8);
  upd_keep_kernel<<<std::max(grid, 1), 256, 0, stream_>>>(old_s, keep.as<unsigned char>(), n_ids);
  AB_CUDA(cudaGetLastError());
  ++st_.kernel_launches;
  follow(old_s, dict_.rebuild(keep.as<unsigned char>(), min_buckets_));
}

void UpdatingAggOp::set_clock(int64_t now_ns) {
  AB_REQUIRE(now_ns >= clock_, ARROYO_B200_INVALID_ARGUMENT,
             "updating aggregate: the clock moved backwards (" + std::to_string(now_ns) + " < " +
                 std::to_string(clock_) + ")");
  if (now_ns == clock_) return;
  // rows that deferred are stamped when they are re-ingested: with the clock of the call that brought them
  if (ttl_ns_ > 0 && plan_.keyed) {
    set_device();
    drain_deferred();
  }
  clock_ = now_ns;
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
      AggCols d;
      d.key = defer_[full][0].as<long long>();
      d.ts = defer_[full][1].as<long long>();
      for (int v = 0; v < plan_.n_vals; ++v) d.val[v] = defer_[full][2 + v].as<long long>();
      ingest(d, (int64_t)n);
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
  while ((uint64_t)total_keys_ + new_rows > dict_.n_buckets() * (uint64_t)BD_MEAN) grow();
}

void UpdatingAggOp::ingest(const AggCols& d, int64_t n) {
  if (n <= 0) return;
  UIngest p{};
  p.key = d.key;
  p.ts = d.ts;
  for (int v = 0; v < plan_.n_vals; ++v) p.val[v] = d.val[v];
  p.n = n;
  p.keyed = plan_.keyed ? 1 : 0;
  p.n_vals = plan_.n_vals;
  p.dict = dict_.view();
  p.st = state_view();
  if (plan_.keyed) {  // every row of the launch may defer (all rows of a key whose bucket is full do)
    reserve_defer(defer_cur_, (uint64_t)n);
    p.d_key = defer_[defer_cur_][0].as<long long>();
    p.d_ts = defer_[defer_cur_][1].as<long long>();
    for (int v = 0; v < plan_.n_vals; ++v) p.d_val[v] = defer_[defer_cur_][2 + v].as<long long>();
  }
  p.deferred = reinterpret_cast<unsigned long long*>((char*)counters_.p + 16);
  const int grid = (int)std::min<int64_t>((n + 255) / 256, (int64_t)num_sms_ * 8);
  if (ttl_ns_ > 0) {
    p.last = last_.as<long long>();
    p.now = clock_;
    p.n_live = ttl_counters_.as<unsigned int>();
    upd_ingest_kernel<true><<<std::max(grid, 1), 256, 0, stream_>>>(p);
  } else {
    upd_ingest_kernel<false><<<std::max(grid, 1), 256, 0, stream_>>>(p);
  }
  AB_CUDA(cudaGetLastError());
  ++st_.kernel_launches;
  ++st_.ingest_launches;
}

void UpdatingAggOp::process_batch(uint32_t, uint32_t, ArrowArray* batch, const ArrowSchema* schema) {
  set_device();
  AggCols d;
  const int64_t n = staging_.stage(plan_, batch, schema, stream_, &st_, &key_format_, &d);
  if (n == 0) {
    if (batch->release) batch->release(batch);
    return;
  }
  // ensure_room synchronises the stream before it can fail: a refused batch is no longer being copied
  ensure_room((uint64_t)n);
  ingest(d, n);
  // the staging buffer is reused by the next batch: the copies and the kernel must have consumed the host batch
  AB_CUDA(cudaStreamSynchronize(stream_));
  if (batch->release) batch->release(batch);
  batch->release = nullptr;
}

void UpdatingAggOp::process_device_batch(uint32_t, uint32_t, const uint64_t* cols, int32_t n_cols, int64_t n_rows) {
  set_device();
  const AggCols d = plan_.columns(cols, n_cols);
  if (n_rows <= 0) return;
  st_.rows_in += (uint64_t)n_rows;
  ensure_room((uint64_t)n_rows);
  ingest(d, n_rows);
}

static void* d2h_part(const void* dev, size_t off_rows, int64_t n, void* host, size_t host_off_rows, cudaStream_t s) {
  if (n > 0)
    AB_CUDA(cudaMemcpyAsync((char*)host + host_off_rows * 8, (const char*)dev + off_rows * 8, (size_t)n * 8, cudaMemcpyDeviceToHost, s));
  return host;
}

// flush (:637-738): one batch [key?, aggregates..., _timestamp, is_retract], or nothing when no key changed (and,
// with a ttl, none expired).  Output regions: retractions at [0, n), appends at [n, 2n), evictions at [2n, ...).
void UpdatingAggOp::flush_to(BatchesPriv* out) {
  set_device();
  if (plan_.keyed) drain_deferred();
  struct {
    unsigned int touched, retracts, appends, pad;
  } h{};
  const bool ttl = ttl_ns_ > 0;
  unsigned int ttl_h[2] = {0, 0};  // live keys, evicted
  AB_CUDA(cudaMemcpyAsync(&h, counters_.p, 16, cudaMemcpyDeviceToHost, stream_));
  if (ttl) AB_CUDA(cudaMemcpyAsync(ttl_h, ttl_counters_.p, 8, cudaMemcpyDeviceToHost, stream_));
  AB_CUDA(cudaStreamSynchronize(stream_));
  const unsigned int n = h.touched;
  const unsigned int live = ttl_h[0];  // the flush kernel does not change it: every key the expiry pass may evict
  if ((n == 0 && live == 0) || !out) return;
  unexported_ += n;
  const uint64_t cap = 2ull * n + live;
  if (cap > out_cap_) {
    out_cap_ = std::max<uint64_t>(cap, 1024);
    o_key_.alloc(out_cap_ * 8);
    o_ts_.alloc(out_cap_ * 8);
    for (int g = 0; g < plan_.n_aggs; ++g) o_agg_[g].alloc(out_cap_ * 8);
  }
  if (n) launch_flush(n);
  if (ttl) launch_expire(n);
  AB_CUDA(cudaMemcpyAsync(&h, counters_.p, 16, cudaMemcpyDeviceToHost, stream_));
  AB_CUDA(cudaMemsetAsync(counters_.p, 0, 16, stream_));  // touched list and output counters start over
  if (ttl) AB_CUDA(cudaMemcpyAsync(ttl_h, ttl_counters_.p, 8, cudaMemcpyDeviceToHost, stream_));
  AB_CUDA(cudaStreamSynchronize(stream_));
  const int64_t nr = h.retracts, na = h.appends, ne = ttl_h[1], total = nr + na + ne;
  unexported_ += (uint64_t)ne;
  tombstones_ += (uint64_t)ne;
  if (total > 0) {
    std::vector<OutColumn> cols;
    auto column = [&](const char* nm, const std::string& fmt, const void* dev) {
      OutColumn c;
      c.name = nm;
      c.format = fmt;
      void* host = PinnedPool::get().alloc((size_t)std::max<int64_t>(total, 1) * 8);
      d2h_part(dev, 0, nr, host, 0, stream_);
      d2h_part(dev, n, na, host, (size_t)nr, stream_);
      d2h_part(dev, 2ull * n, ne, host, (size_t)(nr + na), stream_);
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
      for (int64_t i = nr + na; i < total; ++i) bits[i >> 3] |= (unsigned char)(1u << (i & 7));
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
  if (ne) maybe_compact(live - (uint64_t)ne);
}

void UpdatingAggOp::launch_flush(unsigned int n) {
  UFlush p{};
  p.st = state_view();
  p.id_keys = dict_.id_keys();
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
}

// The expiry pass after the flush kernel of a flush with `n` touched keys: its rows go after the 2n of the flush.
void UpdatingAggOp::launch_expire(unsigned int n) {
  UExpire p{};
  p.st = state_view();
  p.id_keys = dict_.id_keys();
  p.last = last_.as<long long>();
  p.now = clock_;
  p.ttl = ttl_ns_;
  p.n_ids = plan_.keyed ? dict_.n_ids() : 1;
  p.keyed = plan_.keyed ? 1 : 0;
  p.n_aggs = plan_.n_aggs;
  for (int g = 0; g < plan_.n_aggs; ++g) {
    p.agg_kind[g] = plan_.agg_kind[g];
    p.agg_acc[g] = plan_.agg_acc[g];
    p.o_agg[g] = o_agg_[g].as<unsigned long long>() + 2ull * n;
  }
  p.o_key = o_key_.as<long long>() + 2ull * n;
  p.o_ts = o_ts_.as<long long>() + 2ull * n;
  p.n_live = ttl_counters_.as<unsigned int>();
  p.count = p.n_live + 1;
  AB_CUDA(cudaMemsetAsync(p.count, 0, 4, stream_));
  const int grid = (int)std::min<uint64_t>((p.n_ids + 255) / 256, (uint64_t)num_sms_ * 8);
  upd_expire_kernel<<<std::max(grid, 1), 256, 0, stream_>>>(p);
  AB_CUDA(cudaGetLastError());
  ++st_.kernel_launches;
  ++st_.emit_launches;
}


// checkpoint_sliding (:272-340): one batch of table "a" with the keys flushed since the last call, or nothing.
void UpdatingAggOp::checkpoint_state(BatchesPriv* out) {
  set_device();
  if (unexported_ == 0) return;
  const uint64_t n_ids = plan_.keyed ? dict_.n_ids() : 1;
  const uint64_t cap = std::min<uint64_t>(unexported_, n_ids);
  if (cap > state_cap_) {
    state_cap_ = std::max<uint64_t>(cap, 1024);
    s_key_.alloc(state_cap_ * 8);
    s_ts_.alloc(state_cap_ * 8);
    for (int a = 0; a < plan_.n_acc; ++a) s_acc_[a].alloc(state_cap_ * 8);
  }
  unsigned int* count = reinterpret_cast<unsigned int*>((char*)counters_.p + 24);
  AB_CUDA(cudaMemsetAsync(count, 0, 4, stream_));
  UExport p{};
  p.st = state_view();
  p.id_keys = dict_.id_keys();
  p.n_ids = n_ids;
  p.o_key = s_key_.as<long long>();
  for (int a = 0; a < plan_.n_acc; ++a) p.o_acc[a] = s_acc_[a].as<unsigned long long>();
  p.o_ts = s_ts_.as<long long>();
  p.count = count;
  const bool dead = tombstones_ > 0;  // evictions since the last export: rows may be tombstones
  if (dead) {
    if (s_dead_.bytes < cap) s_dead_.alloc(state_cap_);
    p.o_dead = s_dead_.as<unsigned char>();
  }
  const int grid = (int)std::min<uint64_t>((n_ids + 255) / 256, (uint64_t)num_sms_ * 8);
  upd_export_kernel<<<std::max(grid, 1), 256, 0, stream_>>>(p);
  AB_CUDA(cudaGetLastError());
  ++st_.kernel_launches;
  unsigned int rows = 0;
  AB_CUDA(cudaMemcpyAsync(&rows, count, 4, cudaMemcpyDeviceToHost, stream_));
  AB_CUDA(cudaStreamSynchronize(stream_));
  unexported_ = 0;
  tombstones_ = 0;
  if (rows > 0) export_state(out, rows, dead);
  if (dead) maybe_compact(read_live());
}

// The table-"a" batch (AggPlan::state_layout) of the `rows` rows the export kernel wrote; with `dead`, the rows it
// marked are tombstones: a null `_timestamp`.
void UpdatingAggOp::export_state(BatchesPriv* out, unsigned int rows, bool dead) {
  std::vector<OutColumn> cols = state_columns(plan_.state_layout(true), rows, plan_.keyed ? s_key_.p : nullptr,
                                              key_format_, s_acc_, s_ts_.p, stream_, &st_.d2h_bytes);
  const unsigned char* is_dead = dead ? (const unsigned char*)d2h_pinned(s_dead_.p, rows, stream_, &st_.d2h_bytes) : nullptr;
  AB_CUDA(cudaStreamSynchronize(stream_));
  if (is_dead) {
    OutColumn& ts = cols.back();
    uint8_t* valid = (uint8_t*)PinnedPool::get().alloc((size_t)rows / 8 + 8);
    memset(valid, 0, (size_t)rows / 8 + 8);
    for (unsigned int r = 0; r < rows; ++r) {
      if (is_dead[r]) ++ts.null_count;
      else valid[r >> 3] |= (uint8_t)(1u << (r & 7));
    }
    PinnedPool::get().free((void*)is_dead);
    ts.nullable = true;
    if (ts.null_count) ts.validity = valid;
    else PinnedPool::get().free(valid);
  }
  OutColumn g;
  g.name = "_generation";
  g.format = "L";
  g.data = PinnedPool::get().alloc((size_t)rows * 8);
  std::fill((uint64_t*)g.data, (uint64_t*)g.data + rows, (uint64_t)generation_);
  cols.push_back(g);
  ++generation_;
  out->arrays.emplace_back();
  out->schemas.emplace_back();
  export_batch(cols, rows, &out->arrays.back(), &out->schemas.back());
}

// initialize (:446-503): the batches of table "a", in any order and with any number of rows per key.  A restore that
// succeeds takes every batch once the copies have completed.
void UpdatingAggOp::on_start(ArrowArray* state, ArrowSchema* schemas, int64_t n, int64_t, int64_t) {
  if (n <= 0) return;
  const StateBatches sb(plan_, true, state, schemas, n);
  AB_REQUIRE(st_.rows_in == 0 && !restored_, ARROYO_B200_INVALID_ARGUMENT,
             "updating aggregate: restore into an operator that already holds rows or restored state");
  const int64_t total = sb.total;
  if (total == 0) {
    take_batches(state, n);
    return;
  }
  const int ts_col = sb.ts_col, gen_col = sb.ts_col + 1;
  set_device();
  if (plan_.keyed) {
    key_format_ = sb.cols[0][0].format;
    // the state is still empty: size the dictionary once to hold every restored key without growing
    const uint64_t b = bd_buckets_for((uint64_t)total);
    if (b > dict_.n_buckets()) {
      dict_.alloc(b);
      alloc_state();
    }
  }
  DevBuf d_key, d_gen, d_ts, d_val[MAX_ACC];
  if (plan_.keyed) sb.upload(0, 0, n, d_key, stream_, &st_.h2d_bytes);
  sb.upload(gen_col, 0, n, d_gen, stream_, &st_.h2d_bytes);
  sb.upload(ts_col, 0, n, d_ts, stream_, &st_.h2d_bytes);
  URestore p{};
  for (int a = 0; a < plan_.n_acc; ++a)
    if (sb.seed[a] >= 0) p.val[a] = sb.upload(sb.seed[a], 0, n, d_val[a], stream_, &st_.h2d_bytes);
  uint64_t max_gen = 0;
  for (int64_t b = 0; b < n; ++b)
    for (int64_t i = 0; i < sb.rows[b]; ++i) max_gen = std::max<uint64_t>(max_gen, sb.cols[b][gen_col].data[i]);
  // tombstones: the rows whose `_timestamp` is null
  DevBuf d_dead;
  bool any_dead = false;
  for (int64_t b = 0; b < n; ++b) any_dead = any_dead || sb.cols[b][ts_col].validity != nullptr;
  if (any_dead) {
    std::vector<unsigned char> h_dead((size_t)total, 0);
    int64_t off = 0;
    for (int64_t b = 0; b < n; ++b) {
      const InColumn& c = sb.cols[b][ts_col];
      for (int64_t i = 0; c.validity && i < sb.rows[b]; ++i) {
        const int64_t bit = c.validity_bit + i;
        h_dead[off + i] = !((c.validity[bit >> 3] >> (bit & 7)) & 1);
      }
      off += sb.rows[b];
    }
    d_dead.alloc((size_t)total);
    AB_CUDA(cudaMemcpyAsync(d_dead.p, h_dead.data(), (size_t)total, cudaMemcpyHostToDevice, stream_));
    AB_CUDA(cudaStreamSynchronize(stream_));  // h_dead goes when this block ends
    st_.h2d_bytes += (uint64_t)total;
    p.dead = d_dead.as<unsigned char>();
  }
  DevBuf ids((size_t)total * 4);
  dict_.place(plan_.keyed ? d_key.as<long long>() : nullptr, total, ids.as<uint32_t>(), [&] { grow(); });
  p.gen = d_gen.as<unsigned long long>();
  p.ts = d_ts.as<long long>();
  p.ids = ids.as<unsigned int>();
  p.n = total;
  const int grid = std::max(1, (int)std::min<int64_t>((total + 255) / 256, (int64_t)num_sms_ * 8));
  p.st = state_view();
  const uint64_t id_cap = dict_.id_cap();
  DevBuf best_gen(id_cap * 8), best_pos(id_cap * 8);
  AB_CUDA(cudaMemsetAsync(best_gen.p, 0, id_cap * 8, stream_));
  AB_CUDA(cudaMemsetAsync(best_pos.p, 0xFF, id_cap * 8, stream_));  // -1
  p.best_gen = best_gen.as<unsigned long long>();
  p.best_pos = best_pos.as<long long>();
  DevBuf won(8);
  AB_CUDA(cudaMemsetAsync(won.p, 0, 8, stream_));
  p.won = won.as<unsigned int>();
  if (ttl_ns_ > 0) {
    p.last = last_.as<long long>();
    p.now = clock_;
  }
  upd_restore_gen_kernel<<<grid, 256, 0, stream_>>>(p);
  AB_CUDA(cudaGetLastError());
  upd_restore_pos_kernel<<<grid, 256, 0, stream_>>>(p);
  AB_CUDA(cudaGetLastError());
  upd_restore_seed_kernel<<<grid, 256, 0, stream_>>>(p);
  AB_CUDA(cudaGetLastError());
  st_.kernel_launches += 3;
  if (ttl_ns_ > 0)  // the operator was empty: the live keys are the restored ones
    AB_CUDA(cudaMemcpyAsync(ttl_counters_.p, won.p, 4, cudaMemcpyDeviceToDevice, stream_));
  unsigned int h_won[2] = {0, 0};
  AB_CUDA(cudaMemcpyAsync(h_won, won.p, 8, cudaMemcpyDeviceToHost, stream_));
  AB_CUDA(cudaMemcpyAsync(&total_keys_, n_total_.p, 4, cudaMemcpyDeviceToHost, stream_));
  AB_CUDA(cudaStreamSynchronize(stream_));
  // keys whose latest row is a tombstone hold ids without state: give them back, so n_keys counts live keys
  if (h_won[1] && plan_.keyed) compact();
  generation_ = max_gen + 1;
  restored_ = true;
  take_batches(state, n);
}

}  // namespace

OpBase* make_updating_agg_op(const ArroyoB200OpConfig& cfg) { return new UpdatingAggOp(cfg); }

}  // namespace ab
