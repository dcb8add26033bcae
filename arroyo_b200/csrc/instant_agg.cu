// Instant-window aggregate on sm_90a (H100): the GPU side of `TumblingAggregatingWindowFunc` with width 0
// (arroyo-worker/src/arrow/tumbling_aggregating_window.rs), which the planner emits when a query aggregates a stream an
// upstream operator has already windowed (arroyo-planner extension/aggregate.rs:233-289, `instant_window_config`).
// Its bin is `_timestamp` itself (:65-73): every upstream window stamps its rows with one timestamp, so each upstream
// window is one bin ("instant").  Nexmark q5's MaxBids is this operator.
//
// Instants are sparse and can be numerous (behind a session window every session ends at its own timestamp), so the
// state is not the window operator's dense per-pane block but one group per (instant, key):
//   table   open addressing on the exact composite (instant, key), a `used` word per slot (every 64-bit key and
//           timestamp is legal), dense group ids from a counter.  Per id: the instant, the key and two SoA accumulator
//           blocks, `base` and `delta` (the rows since the last checkpoint).  The host grows the table before a launch
//           that could overfill it, from the rows it has handed over since it last read the group count;
//   ingest  one thread per row: the late test (ts < the last watermark, :280-291), find-or-insert of the group (its
//           creator sets both blocks to the accumulators' identities), then the lanes of a warp that carry the same
//           group combine their values (a log-step tree over the peer set) and one lane per group does the atomics
//           into `delta`.  The unkeyed aggregate of an upstream window sends every row into one group;
//   emit    at watermark w every group with instant < w leaves (:321-392): flag, compact (device_exclusive_scan),
//           CUB radix sort of (instant, id) by instant, finalise `base` + `delta` into the output columns, export
//           (the nested form's window{start = ts - W + 1, end = ts + 1} through export_window_batch).  The survivors
//           are then compacted to ids [0, n_open) and the table is rebuilt from them: device state stays proportional
//           to the open groups;
//   state   a checkpoint writes, per open instant, the partial rows of `delta` (:430-467, table "t" in partial_schema
//           [key?, state cols..., _timestamp = instant]) and folds `delta` into `base`: the shim's table keeps earlier
//           epochs, so writing the whole state again would count it twice on restore.  on_start merges partial rows
//           into `base`, one thread per row.
// Output rows of one emission leave in one batch, ordered by instant (the reference emits one batch per instant; the
// rows and their order are the same).  Device-resident output is refused (ARROYO_B200_UNSUPPORTED).
#include <algorithm>
#include <climits>

#include <cub/device/device_radix_sort.cuh>
#include <cuda/atomic>

#include "agg_plan.h"
#include "op.h"
#include "scan.cuh"

namespace ab {
namespace {

constexpr int IA_THREADS = 256;
constexpr unsigned FULL = 0xffffffffu;
constexpr uint32_t NO_GROUP = 0xffffffffu;
constexpr int64_t IA_CHUNK = 1 << 21;  // rows per ingest launch: the table is sized for the rows of one launch at a time

struct alignas(32) GSlot {
  long long inst;
  long long key;
  unsigned int used;  // 0 free, 1 being claimed, 2 published
  unsigned int id;
  unsigned long long pad;
};

// Device view of the groups.
struct IGroups {
  GSlot* tab;
  uint32_t mask;
  int n_acc;
  long long* inst;
  long long* key;
  unsigned long long* base;   // [n_acc][cap]; base[id] = rows
  unsigned long long* delta;  // same layout: rows since the last checkpoint
  unsigned long long cap;
  unsigned int* n_groups;
  int acc_kind[MAX_ACC];
};

struct ICounters {
  unsigned int n_groups;
  unsigned int neg_ts;  // a row with a negative _timestamp arrived
  unsigned long long late;
  unsigned long long instants;  // distinct instants of the last emission
  unsigned long long total;     // scan total
};

__device__ __forceinline__ uint32_t ia_home(long long inst, long long key, uint32_t mask) {
  return (uint32_t)mix64(mix64((uint64_t)inst) ^ (uint64_t)key) & mask;
}

__device__ __forceinline__ unsigned int ia_used(GSlot* s) {
  return cuda::atomic_ref<unsigned int, cuda::thread_scope_device>(s->used).load(cuda::memory_order_acquire);
}

// The group of (inst, key), created when it does not exist yet.  The creator sets both accumulator blocks to their
// identities before it publishes the slot, so whoever finds the slot may fold into them at once.
__device__ uint32_t ia_find_or_insert(const IGroups& g, long long inst, long long key) {
  uint32_t pos = ia_home(inst, key, g.mask);
  while (true) {
    GSlot* s = g.tab + pos;
    unsigned int u = ia_used(s);
    if (u == 0u) {
      u = atomicCAS(&s->used, 0u, 1u);
      if (u == 0u) {
        const uint32_t id = atomicAdd(g.n_groups, 1u);
        s->inst = inst;
        s->key = key;
        s->id = id;
        g.inst[id] = inst;
        g.key[id] = key;
        for (int a = 0; a < g.n_acc; ++a) {
          const unsigned long long v = acc_identity(g.acc_kind[a]);
          g.base[(unsigned long long)a * g.cap + id] = v;
          g.delta[(unsigned long long)a * g.cap + id] = v;
        }
        cuda::atomic_ref<unsigned int, cuda::thread_scope_device>(s->used).store(2u, cuda::memory_order_release);
        return id;
      }
    }
    while (u == 1u) u = ia_used(s);
    if (*(volatile long long*)&s->inst == inst && *(volatile long long*)&s->key == key) return *(volatile unsigned int*)&s->id;
    pos = (pos + 1) & g.mask;
  }
}

struct IIngest {
  IGroups g;
  const long long* key;
  const long long* ts;
  const long long* val[MAX_VALS];
  int acc_val[MAX_ACC];
  long long n;
  long long late_wm;  // rows with ts < late_wm are late (LLONG_MIN: no watermark yet)
  int keyed;
  ICounters* counters;
};

// Every lane of a warp runs every iteration (the loop bound is uniform per warp), so the peer sets of __match_any_sync
// are whole.  Lanes without a group carry NO_GROUP and are peers of each other only.
__global__ void __launch_bounds__(IA_THREADS) ia_ingest_kernel(const __grid_constant__ IIngest p) {
  const unsigned lane = threadIdx.x & 31;
  const long long stride = (long long)gridDim.x * blockDim.x;
  unsigned int late = 0;
  bool neg = false;
  for (long long row0 = (long long)blockIdx.x * blockDim.x + (threadIdx.x & ~31u); row0 < p.n; row0 += stride) {
    const long long i = row0 + lane;
    bool live = i < p.n;
    long long ts = 0, key = 0;
    if (live) {
      ts = __ldcs(p.ts + i);
      key = p.keyed ? __ldcs(p.key + i) : 0;
      if (ts < 0) {
        neg = true;
        live = false;
      } else if (ts < p.late_wm) {
        ++late;
        live = false;
      }
    }
    const uint32_t id = live ? ia_find_or_insert(p.g, ts, key) : NO_GROUP;
    unsigned long long v[MAX_ACC];
#pragma unroll
    for (int a = 1; a < MAX_ACC; ++a) {
      if (a >= p.g.n_acc) break;
      v[a] = acc_of_value(p.g.acc_kind[a], live ? __ldcs(p.val[p.acc_val[a]] + i) : 0);
    }
    // combine the peers' values: at each step a lane folds in the value of the next peer above it that is still in
    // play, then every peer of odd rank drops out; after at most five steps the lowest peer holds the whole set's
    const unsigned peers = __match_any_sync(FULL, id);
    const int leader = __ffs(peers) - 1;
    unsigned rest = lane == 31 ? 0u : peers & (FULL << (lane + 1));
    unsigned rank = __popc(peers & ((1u << lane) - 1u));
    while (__any_sync(FULL, rest != 0u)) {
      const int src = __ffs(rest) - 1;
#pragma unroll
      for (int a = 1; a < MAX_ACC; ++a) {
        if (a >= p.g.n_acc) break;
        const unsigned long long t = __shfl_sync(FULL, v[a], src < 0 ? (int)lane : src);
        if (src >= 0) v[a] = acc_merge(p.g.acc_kind[a], v[a], t);
      }
      rest &= ~__ballot_sync(FULL, rank & 1u);
      rank >>= 1;
    }
    if (live && (int)lane == leader) {
      acc_red(ACC_ROWS, p.g.delta + id, (unsigned long long)__popc(peers));
#pragma unroll
      for (int a = 1; a < MAX_ACC; ++a) {
        if (a >= p.g.n_acc) break;
        acc_red(p.g.acc_kind[a], p.g.delta + (unsigned long long)a * p.g.cap + id, v[a]);
      }
    }
  }
  const unsigned int wl = __reduce_add_sync(FULL, late);
  if (lane == 0 && wl) atomicAdd(&p.counters->late, (unsigned long long)wl);
  if (neg) p.counters->neg_ts = 1u;
}

// flag[id] = the group leaves: its instant is below the watermark (w != LLONG_MIN), or its delta block has rows
__global__ void ia_mark_kernel(const long long* __restrict__ inst, const unsigned long long* __restrict__ delta_rows,
                               unsigned int n, long long w, unsigned int* __restrict__ flag) {
  unsigned int i = blockIdx.x * blockDim.x + threadIdx.x;
  const unsigned int stride = gridDim.x * blockDim.x;
  for (; i < n; i += stride) flag[i] = w != LLONG_MIN ? (inst[i] < w ? 1u : 0u) : (delta_rows[i] ? 1u : 0u);
}

// the flagged groups' (instant, id) pairs, compacted
__global__ void ia_scatter_kernel(const unsigned int* __restrict__ flag, const unsigned long long* __restrict__ off,
                                  const long long* __restrict__ inst, unsigned int n, unsigned long long* __restrict__ sk,
                                  unsigned int* __restrict__ sv) {
  unsigned int i = blockIdx.x * blockDim.x + threadIdx.x;
  const unsigned int stride = gridDim.x * blockDim.x;
  for (; i < n; i += stride) {
    if (!flag[i]) continue;
    const unsigned long long o = off[i];
    sk[o] = (unsigned long long)inst[i];
    sv[o] = i;
  }
}

struct IFinal {
  IGroups g;
  const unsigned long long* inst;  // sorted
  const unsigned int* ids;
  long long n;
  int keyed;
  int n_aggs;
  int agg_kind[ARROYO_B200_MAX_AGGS];
  int agg_acc[ARROYO_B200_MAX_AGGS];
  int nested;
  long long width_m1;  // W - 1 of the nested form
  long long* o_key;
  unsigned long long* o_agg[ARROYO_B200_MAX_AGGS];
  long long* o_ts;
  long long* o_ws;
  long long* o_we;
  unsigned long long* instants;
};

// one output row per leaving group, in instant order: base + delta, finalised; counts the distinct instants
__global__ void __launch_bounds__(IA_THREADS) ia_final_kernel(const __grid_constant__ IFinal p) {
  const unsigned lane = threadIdx.x & 31;
  const long long stride = (long long)gridDim.x * blockDim.x;
  unsigned int firsts = 0;
  for (long long j0 = (long long)blockIdx.x * blockDim.x + (threadIdx.x & ~31u); j0 < p.n; j0 += stride) {
    const long long j = j0 + lane;
    if (j >= p.n) continue;
    const unsigned int id = p.ids[j];
    const long long inst = (long long)p.inst[j];
    if (j == 0 || (long long)p.inst[j - 1] != inst) ++firsts;
    unsigned long long m[MAX_ACC];
    for (int a = 0; a < p.g.n_acc; ++a) {
      const unsigned long long off = (unsigned long long)a * p.g.cap + id;
      m[a] = acc_merge(p.g.acc_kind[a], p.g.base[off], p.g.delta[off]);
    }
    if (p.keyed) p.o_key[j] = p.g.key[id];
    for (int g = 0; g < p.n_aggs; ++g) p.o_agg[g][j] = agg_finalise(p.agg_kind[g], m[p.agg_acc[g]], m[0]);
    p.o_ts[j] = inst;
    if (p.nested) {
      p.o_ws[j] = inst - p.width_m1;
      p.o_we[j] = inst + 1;
    }
  }
  const unsigned int wf = __reduce_add_sync(FULL, firsts);
  if (lane == 0 && wf) atomicAdd(p.instants, (unsigned long long)wf);
}

// partial rows of the groups with rows since the last checkpoint, in instant order: key, delta block, instant
struct IState {
  IGroups g;
  const unsigned long long* inst;
  const unsigned int* ids;
  long long n;
  long long* o_key;
  unsigned long long* o_acc[MAX_ACC];
  long long* o_ts;
};
__global__ void ia_state_kernel(const __grid_constant__ IState p) {
  long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (; j < p.n; j += stride) {
    const unsigned int id = p.ids[j];
    p.o_key[j] = p.g.key[id];
    for (int a = 0; a < p.g.n_acc; ++a) p.o_acc[a][j] = p.g.delta[(unsigned long long)a * p.g.cap + id];
    p.o_ts[j] = (long long)p.inst[j];
  }
}

// the groups that stay, moved to ids [0, n_open) of `to` in id order: new id = id - (groups leaving below it)
__global__ void ia_reclaim_kernel(const __grid_constant__ IGroups from, const __grid_constant__ IGroups to,
                                  const unsigned int* __restrict__ flag, const unsigned long long* __restrict__ off,
                                  unsigned int n) {
  unsigned int i = blockIdx.x * blockDim.x + threadIdx.x;
  const unsigned int stride = gridDim.x * blockDim.x;
  for (; i < n; i += stride) {
    if (flag[i]) continue;
    const unsigned int d = i - (unsigned int)off[i];
    to.inst[d] = from.inst[i];
    to.key[d] = from.key[i];
    for (int a = 0; a < from.n_acc; ++a) {
      to.base[(unsigned long long)a * to.cap + d] = from.base[(unsigned long long)a * from.cap + i];
      to.delta[(unsigned long long)a * to.cap + d] = from.delta[(unsigned long long)a * from.cap + i];
    }
  }
}

// the table of groups [0, n) in an all-free slot array (every (instant, key) is distinct); sets the group count
__global__ void ia_rebuild_kernel(const __grid_constant__ IGroups g, unsigned int n) {
  unsigned int i = blockIdx.x * blockDim.x + threadIdx.x;
  const unsigned int stride = gridDim.x * blockDim.x;
  if (i == 0) *g.n_groups = n;
  for (; i < n; i += stride) {
    const long long inst = g.inst[i], key = g.key[i];
    uint32_t pos = ia_home(inst, key, g.mask);
    while (atomicCAS(&g.tab[pos].used, 0u, 2u) != 0u) pos = (pos + 1) & g.mask;
    g.tab[pos].inst = inst;
    g.tab[pos].key = key;
    g.tab[pos].id = i;
  }
}

// Restore: partial rows merged into the `base` block of their group, one thread per row.  state[a] null: each row
// counts one (accumulator 0 of a plan whose partial state carries no row count).
struct IRestore {
  IGroups g;
  const long long* key;
  const long long* ts;
  const unsigned long long* state[MAX_ACC];
  long long n;
  int keyed;
};
__global__ void ia_restore_kernel(const __grid_constant__ IRestore p) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (; i < p.n; i += stride) {
    const uint32_t id = ia_find_or_insert(p.g, p.ts[i], p.keyed ? p.key[i] : 0);
    for (int a = 0; a < p.g.n_acc; ++a)
      acc_red(p.g.acc_kind[a], p.g.base + (unsigned long long)a * p.g.cap + id, p.state[a] ? p.state[a][i] : 1ull);
  }
}

class InstantAggOp final : public OpBase {
 public:
  explicit InstantAggOp(const ArroyoB200OpConfig& c);
  ~InstantAggOp() override { drain_stream(); }
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
    st_.n_keys = n_groups_;
    *out = st_;
  }

 private:
  struct Groups {
    DevBuf inst, key, base, delta;
  };
  AggPlan plan_;
  std::string key_format_ = "l";
  AggStaging staging_;
  bool nested_ = false;
  int64_t width_m1_ = 0;
  int64_t late_wm_ = LLONG_MIN;  // the last watermark: rows below it are late
  Groups cur_, alt_;             // alt_: where the survivors of an emission go (allocated on first use)
  uint64_t cap_ = 0;             // group ids per block
  DevBuf tab_;
  uint64_t tab_cap_ = 0;
  DevBuf counters_;
  uint64_t n_groups_ = 0;   // as of the last read
  uint64_t groups_hi_ = 0;  // upper bound of the groups on the device: n_groups_ + rows handed over since
  DevBuf flag_, off_, sums_, sk_, sv_, sk2_, sv2_, cub_tmp_;
  DevBuf o_key_, o_ts_, o_ws_, o_we_, o_agg_[ARROYO_B200_MAX_AGGS], o_acc_[MAX_ACC];
  ArroyoB200Stats st_{};

  int grid_for(uint64_t n) const {
    return (int)std::max<uint64_t>(1, std::min<uint64_t>((n + IA_THREADS - 1) / IA_THREADS, (uint64_t)num_sms_ * 8));
  }
  IGroups view(const Groups& g) const;
  void alloc_groups(Groups& g, uint64_t cap) const;
  void rebuild_table(uint64_t n);
  void reserve_groups(uint64_t more);
  void read_counters();
  void ingest(const AggCols& d, int64_t n);
  uint64_t select(long long w);  // flags, compacts and sorts the groups that leave; returns their count
  void emit(int64_t w, BatchesPriv* out);
  void reclaim(uint64_t g, uint64_t e);
  void export_state(uint64_t d, BatchesPriv* out);
};

// room for `bytes`, kept across calls (grown by half again so that a slowly growing need does not reallocate each time)
void reserve(DevBuf& b, size_t bytes) {
  if (b.bytes < bytes) b.alloc(std::max(bytes, b.bytes + b.bytes / 2));
}

InstantAggOp::InstantAggOp(const ArroyoB200OpConfig& c) {
  cfg = c;
  name = "instant_window";
  // AVG sums its inputs as f64 like the reference's accumulator
  plan_ = AggPlan(c, ACC_SUM_F64);
  AB_REQUIRE(c.partial_count_col_plus1 == 0, ARROYO_B200_UNSUPPORTED,
             "instant window aggregate over partial-aggregate inputs is not supported");
  nested_ = c.final_projection != 0;
  if (nested_) {
    AB_REQUIRE(c.width_ns > 0, ARROYO_B200_INVALID_ARGUMENT,
               "nested instant window: width_ns must be the upstream window's width (> 0)");
    width_m1_ = c.width_ns - 1;
  }
  open_device(c);
  counters_.alloc(sizeof(ICounters));
  AB_CUDA(cudaMemsetAsync(counters_.p, 0, sizeof(ICounters), stream_));
  cap_ = 1u << 16;
  alloc_groups(cur_, cap_);
  rebuild_table(0);
  AB_CUDA(cudaStreamSynchronize(stream_));
}

IGroups InstantAggOp::view(const Groups& g) const {
  IGroups v{};
  v.tab = tab_.as<GSlot>();
  v.mask = (uint32_t)(tab_cap_ - 1);
  v.n_acc = plan_.n_acc;
  v.inst = g.inst.as<long long>();
  v.key = g.key.as<long long>();
  v.base = g.base.as<unsigned long long>();
  v.delta = g.delta.as<unsigned long long>();
  v.cap = cap_;
  v.n_groups = &counters_.as<ICounters>()->n_groups;
  for (int a = 0; a < plan_.n_acc; ++a) v.acc_kind[a] = plan_.acc_kind[a];
  return v;
}

void InstantAggOp::alloc_groups(Groups& g, uint64_t cap) const {
  g.inst.alloc(cap * 8);
  g.key.alloc(cap * 8);
  g.base.alloc(cap * 8 * plan_.n_acc);
  g.delta.alloc(cap * 8 * plan_.n_acc);
}

// A free table of 2 * cap_ slots holding groups [0, n) of cur_; the group count becomes n.
void InstantAggOp::rebuild_table(uint64_t n) {
  const uint64_t want = cap_ * 2;
  if (tab_cap_ != want) {
    tab_.alloc(want * sizeof(GSlot));
    tab_cap_ = want;
  }
  AB_CUDA(cudaMemsetAsync(tab_.p, 0, tab_cap_ * sizeof(GSlot), stream_));
  ia_rebuild_kernel<<<grid_for(n), IA_THREADS, 0, stream_>>>(view(cur_), (unsigned int)n);
  AB_CUDA(cudaGetLastError());
  ++st_.kernel_launches;
}

// Reads the counters (waits for the stream): the group count, the late rows, and a negative timestamp, on which the
// reference panics.
void InstantAggOp::read_counters() {
  ICounters c{};
  AB_CUDA(cudaMemcpyAsync(&c, counters_.p, sizeof c, cudaMemcpyDeviceToHost, stream_));
  AB_CUDA(cudaStreamSynchronize(stream_));
  n_groups_ = groups_hi_ = c.n_groups;
  st_.rows_late = c.late;
  if (c.neg_ts) {
    AB_CUDA(cudaMemsetAsync(&counters_.as<ICounters>()->neg_ts, 0, 4, stream_));
    AB_CUDA(cudaStreamSynchronize(stream_));
    throw Error(ARROYO_B200_PANIC, "batch holds a negative _timestamp (before the Unix epoch): the reference panics on it");
  }
}

// Room for `more` new groups: every row handed over may open one.  The bound is tightened from the device's count
// before the blocks grow; growing doubles them, moves groups [0, n) and rebuilds the table.
void InstantAggOp::reserve_groups(uint64_t more) {
  if (groups_hi_ + more <= cap_) return;
  read_counters();
  if (n_groups_ + more <= cap_) return;
  uint64_t nc = cap_ * 2;
  while (nc < n_groups_ + more) nc *= 2;
  AB_REQUIRE(nc <= (1ull << 31), ARROYO_B200_RUNTIME, "instant window aggregate: more than 2^31 open groups");
  Groups ng;
  alloc_groups(ng, nc);
  const size_t n = (size_t)n_groups_;
  if (n) {
    AB_CUDA(cudaMemcpyAsync(ng.inst.p, cur_.inst.p, n * 8, cudaMemcpyDeviceToDevice, stream_));
    AB_CUDA(cudaMemcpyAsync(ng.key.p, cur_.key.p, n * 8, cudaMemcpyDeviceToDevice, stream_));
    for (int a = 0; a < plan_.n_acc; ++a) {
      AB_CUDA(cudaMemcpyAsync(ng.base.as<unsigned long long>() + (size_t)a * nc, cur_.base.as<unsigned long long>() + (size_t)a * cap_,
                              n * 8, cudaMemcpyDeviceToDevice, stream_));
      AB_CUDA(cudaMemcpyAsync(ng.delta.as<unsigned long long>() + (size_t)a * nc, cur_.delta.as<unsigned long long>() + (size_t)a * cap_,
                              n * 8, cudaMemcpyDeviceToDevice, stream_));
    }
  }
  AB_CUDA(cudaStreamSynchronize(stream_));
  cur_ = std::move(ng);
  alt_ = Groups();
  cap_ = nc;
  rebuild_table(n);
}

void InstantAggOp::ingest(const AggCols& d, int64_t n) {
  for (int64_t first = 0; first < n; first += IA_CHUNK) {
    const int64_t m = std::min<int64_t>(IA_CHUNK, n - first);
    reserve_groups((uint64_t)m);
    IIngest p{};
    p.g = view(cur_);
    p.key = d.key ? d.key + first : nullptr;
    p.ts = d.ts + first;
    for (int v = 0; v < plan_.n_vals; ++v) p.val[v] = d.val[v] + first;
    for (int a = 0; a < plan_.n_acc; ++a) p.acc_val[a] = plan_.acc_val[a];
    p.n = m;
    p.late_wm = late_wm_;
    p.keyed = plan_.keyed ? 1 : 0;
    p.counters = counters_.as<ICounters>();
    ia_ingest_kernel<<<grid_for((uint64_t)m), IA_THREADS, 0, stream_>>>(p);
    AB_CUDA(cudaGetLastError());
    ++st_.kernel_launches;
    ++st_.ingest_launches;
    groups_hi_ += (uint64_t)m;
  }
}

void InstantAggOp::process_batch(uint32_t, uint32_t, ArrowArray* batch, const ArrowSchema* schema) {
  set_device();
  AggCols d;
  const int64_t n = staging_.stage(plan_, batch, schema, stream_, &st_, &key_format_, &d);
  if (n > 0) {
    ingest(d, n);
    // the staging buffer is reused by the next batch, and a negative timestamp is reported with this batch
    read_counters();
  }
  if (batch->release) batch->release(batch);
  batch->release = nullptr;
}

void InstantAggOp::process_device_batch(uint32_t, uint32_t, const uint64_t* cols, int32_t n_cols, int64_t n_rows) {
  set_device();
  const AggCols d = plan_.columns(cols, n_cols);
  if (n_rows <= 0) return;
  st_.rows_in += (uint64_t)n_rows;
  ingest(d, n_rows);
}

// Flags the groups that leave -- instant < w, or (w == LLONG_MIN) rows since the last checkpoint -- and leaves their
// (instant, id) pairs sorted by instant in sk2_ / sv2_.  Needs n_groups_ current.
uint64_t InstantAggOp::select(long long w) {
  const uint64_t g = n_groups_;
  reserve(flag_, g * 4);
  reserve(off_, g * 8);
  ia_mark_kernel<<<grid_for(g), IA_THREADS, 0, stream_>>>(cur_.inst.as<long long>(), cur_.delta.as<unsigned long long>(),
                                                          (unsigned int)g, w, flag_.as<unsigned int>());
  AB_CUDA(cudaGetLastError());
  unsigned long long* total = &counters_.as<ICounters>()->total;
  device_exclusive_scan(flag_.as<unsigned int>(), (int64_t)g, off_.as<unsigned long long>(), total, sums_, stream_);
  unsigned long long e = 0;
  AB_CUDA(cudaMemcpyAsync(&e, total, 8, cudaMemcpyDeviceToHost, stream_));
  AB_CUDA(cudaStreamSynchronize(stream_));
  st_.kernel_launches += 4;
  if (e == 0) return 0;
  reserve(sk_, e * 8);
  reserve(sv_, e * 4);
  reserve(sk2_, e * 8);
  reserve(sv2_, e * 4);
  ia_scatter_kernel<<<grid_for(g), IA_THREADS, 0, stream_>>>(flag_.as<unsigned int>(), off_.as<unsigned long long>(),
                                                             cur_.inst.as<long long>(), (unsigned int)g,
                                                             sk_.as<unsigned long long>(), sv_.as<unsigned int>());
  AB_CUDA(cudaGetLastError());
  size_t tmp = 0;
  AB_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, tmp, sk_.as<unsigned long long>(), sk2_.as<unsigned long long>(),
                                          sv_.as<unsigned int>(), sv2_.as<unsigned int>(), (int64_t)e, 0, 63, stream_));
  reserve(cub_tmp_, std::max<size_t>(tmp, 1));
  tmp = cub_tmp_.bytes;
  // instants are non-negative: bit 63 is never set
  AB_CUDA(cub::DeviceRadixSort::SortPairs(cub_tmp_.p, tmp, sk_.as<unsigned long long>(), sk2_.as<unsigned long long>(),
                                          sv_.as<unsigned int>(), sv2_.as<unsigned int>(), (int64_t)e, 0, 63, stream_));
  st_.kernel_launches += 2;
  return e;
}

// handle_watermark (:321-392): every instant below `wm` leaves, in ascending order, and its groups are freed.
void InstantAggOp::handle_watermark(int64_t wm, BatchesPriv* out_host, std::vector<ArroyoB200DeviceBatch>*) {
  set_device();
  AB_REQUIRE(out_host != nullptr, ARROYO_B200_UNSUPPORTED,
             "instant window aggregate: device-resident output is not implemented");
  read_counters();
  if (n_groups_ > 0 && wm != LLONG_MIN) emit(wm, out_host);
  late_wm_ = std::max<int64_t>(late_wm_, wm);
}

void InstantAggOp::emit(int64_t w, BatchesPriv* out) {
  const uint64_t g = n_groups_;
  const uint64_t e = select(w);
  if (e == 0) return;
  reserve(o_key_, e * 8);
  reserve(o_ts_, e * 8);
  if (nested_) {
    reserve(o_ws_, e * 8);
    reserve(o_we_, e * 8);
  }
  for (int a = 0; a < plan_.n_aggs; ++a) reserve(o_agg_[a], e * 8);
  unsigned long long* instants = &counters_.as<ICounters>()->instants;
  AB_CUDA(cudaMemsetAsync(instants, 0, 8, stream_));
  IFinal p{};
  p.g = view(cur_);
  p.inst = sk2_.as<unsigned long long>();
  p.ids = sv2_.as<unsigned int>();
  p.n = (long long)e;
  p.keyed = plan_.keyed ? 1 : 0;
  p.n_aggs = plan_.n_aggs;
  for (int a = 0; a < plan_.n_aggs; ++a) {
    p.agg_kind[a] = plan_.agg_kind[a];
    p.agg_acc[a] = plan_.agg_acc[a];
    p.o_agg[a] = o_agg_[a].as<unsigned long long>();
  }
  p.nested = nested_ ? 1 : 0;
  p.width_m1 = width_m1_;
  p.o_key = o_key_.as<long long>();
  p.o_ts = o_ts_.as<long long>();
  p.o_ws = o_ws_.as<long long>();
  p.o_we = o_we_.as<long long>();
  p.instants = instants;
  ia_final_kernel<<<grid_for(e), IA_THREADS, 0, stream_>>>(p);
  AB_CUDA(cudaGetLastError());
  ++st_.kernel_launches;
  ++st_.emit_launches;
  // the window struct's position counts [key?, aggs...] (extension/aggregate.rs:392-452)
  const int wi = std::min<int>(std::max<int>(cfg.window_index, 0), (plan_.keyed ? 1 : 0) + plan_.n_aggs);
  export_window_batch(out, (int64_t)e, stream_, &st_.d2h_bytes, plan_.keyed ? o_key_.p : nullptr, key_format_, o_agg_,
                      plan_.agg_format, nested_ ? o_ws_.p : nullptr, o_we_.p, wi, o_ts_.p);
  unsigned long long n_inst = 0;
  AB_CUDA(cudaMemcpyAsync(&n_inst, instants, 8, cudaMemcpyDeviceToHost, stream_));
  reclaim(g, e);  // waits for the stream: the batch's copies have completed
  st_.rows_out += e;
  st_.windows_out += n_inst;
}

// Moves the g - e groups that stay to ids [0, g - e) and rebuilds the table from them.
void InstantAggOp::reclaim(uint64_t g, uint64_t e) {
  const uint64_t open = g - e;
  if (open) {
    if (!alt_.inst.p) alloc_groups(alt_, cap_);
    ia_reclaim_kernel<<<grid_for(g), IA_THREADS, 0, stream_>>>(view(cur_), view(alt_), flag_.as<unsigned int>(),
                                                               off_.as<unsigned long long>(), (unsigned int)g);
    AB_CUDA(cudaGetLastError());
    ++st_.kernel_launches;
    std::swap(cur_, alt_);
  }
  rebuild_table(open);
  AB_CUDA(cudaStreamSynchronize(stream_));
  n_groups_ = groups_hi_ = open;
}

// handle_checkpoint (:430-467): the partial rows of the rows received since the last checkpoint, one batch per
// instant, then `delta` folds into `base`.
void InstantAggOp::handle_checkpoint(int64_t, BatchesPriv* out) {
  set_device();
  read_counters();
  const uint64_t g = n_groups_;
  if (g == 0) return;
  const uint64_t d = select(LLONG_MIN);
  if (d > 0) export_state(d, out);
  FoldParams fp{};
  fp.base = cur_.base.as<unsigned long long>();
  fp.delta = cur_.delta.as<unsigned long long>();
  fp.cap = cap_;
  fp.n = (uint32_t)g;
  fp.n_acc = plan_.n_acc;
  for (int a = 0; a < plan_.n_acc; ++a) fp.acc_kind[a] = plan_.acc_kind[a];
  acc_fold_kernel<<<grid_for(g), IA_THREADS, 0, stream_>>>(fp);
  AB_CUDA(cudaGetLastError());
  ++st_.kernel_launches;
  AB_CUDA(cudaStreamSynchronize(stream_));
}

// Partial-state batches in `partial_schema` (AggPlan::state_layout), `_timestamp` = instant.  One batch per instant:
// the shim files a batch under its first row's timestamp and expires it by that time.
void InstantAggOp::export_state(uint64_t d, BatchesPriv* out) {
  reserve(o_key_, d * 8);
  reserve(o_ts_, d * 8);
  for (int a = 0; a < plan_.n_acc; ++a) reserve(o_acc_[a], d * 8);
  IState p{};
  p.g = view(cur_);
  p.inst = sk2_.as<unsigned long long>();
  p.ids = sv2_.as<unsigned int>();
  p.n = (long long)d;
  p.o_key = o_key_.as<long long>();
  for (int a = 0; a < plan_.n_acc; ++a) p.o_acc[a] = o_acc_[a].as<unsigned long long>();
  p.o_ts = o_ts_.as<long long>();
  ia_state_kernel<<<grid_for(d), IA_THREADS, 0, stream_>>>(p);
  AB_CUDA(cudaGetLastError());
  ++st_.kernel_launches;
  // the columns once, on the host; each instant's rows are then a slice of them
  const std::vector<OutColumn> cols = state_columns(plan_.state_layout(false), (int64_t)d, plan_.keyed ? o_key_.p : nullptr,
                                                    key_format_, o_acc_, o_ts_.p, stream_, &st_.d2h_bytes);
  AB_CUDA(cudaStreamSynchronize(stream_));
  const uint64_t* ts = (const uint64_t*)cols.back().data;
  for (uint64_t s = 0; s < d;) {
    uint64_t e = s + 1;
    while (e < d && ts[e] == ts[s]) ++e;
    std::vector<OutColumn> oc;
    for (const OutColumn& c : cols) {
      OutColumn o = c;
      o.data = PinnedPool::get().alloc((size_t)(e - s) * 8);
      memcpy(o.data, (const uint64_t*)c.data + s, (size_t)(e - s) * 8);
      oc.push_back(o);
    }
    out->arrays.emplace_back();
    out->schemas.emplace_back();
    export_batch(oc, (int64_t)(e - s), &out->arrays.back(), &out->schemas.back());
    s = e;
  }
  for (const OutColumn& c : cols) PinnedPool::get().free(c.data);
}

// on_start (:228-248): partial batches of table "t", in any order and with any number of rows per group, merged into
// their groups' `base` blocks.  The restored watermark is the late watermark.
void InstantAggOp::on_start(ArrowArray* state, ArrowSchema* schemas, int64_t n, int64_t watermark, int64_t) {
  set_device();
  const StateBatches sb(plan_, false, state, schemas, n);
  if (watermark != INT64_MIN) late_wm_ = std::max<int64_t>(late_wm_, watermark);
  if (sb.total > 0) {
    if (plan_.keyed) key_format_ = sb.cols[0][0].format;
    reserve_groups((uint64_t)sb.total);
    DevBuf d_key, d_ts, d_acc[MAX_ACC];
    IRestore p{};
    p.keyed = plan_.keyed ? 1 : 0;
    p.key = plan_.keyed ? (const long long*)sb.upload(0, 0, n, d_key, stream_, &st_.h2d_bytes) : nullptr;
    p.ts = (const long long*)sb.upload(sb.ts_col, 0, n, d_ts, stream_, &st_.h2d_bytes);
    for (int a = 0; a < plan_.n_acc; ++a)
      if (sb.seed[a] >= 0) p.state[a] = sb.upload(sb.seed[a], 0, n, d_acc[a], stream_, &st_.h2d_bytes);
    p.n = sb.total;
    p.g = view(cur_);
    ia_restore_kernel<<<grid_for((uint64_t)sb.total), IA_THREADS, 0, stream_>>>(p);
    AB_CUDA(cudaGetLastError());
    ++st_.kernel_launches;
    groups_hi_ += (uint64_t)sb.total;
    read_counters();
  }
  take_batches(state, n);
}

}  // namespace

OpBase* make_instant_agg_op(const ArroyoB200OpConfig& cfg) { return new InstantAggOp(cfg); }

}  // namespace ab
