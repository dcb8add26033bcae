// Session window aggregate on sm_90a (H100).
//
// Replaces SessionAggregatingWindowFunc (arroyo-worker/src/arrow/session_aggregating_window.rs:60-279 operator,
// :397-523 ActiveSession, :533-691 KeyComputingHolder, :850-895 process_batch) and the arrow-rs / DataFusion work
// it does per batch and per key (K7 late filter, K8 lexsort + partition + RowConverter, K9 per-key state machine,
// one AggregateExec(Single) per active session).
//
// The reference's semantics are defined by a sequential per-key state machine over "runs" (the rows of one key
// inside one input batch, sorted by time), including behaviour that is visible in results -- e.g. the row that
// ends ActiveSession::add_batch's scan is still sent to that session (:464-479), and the first row of a run never
// extends data_end in the scan path.  Parity therefore means executing that state machine, not a cleaned-up
// definition of a session.  Keys are independent, so the GPU runs it with one thread per key:
//
//   prep     per batch : late filter (ts >= watermark, :858-868), dense key id (shared dictionary), rows appended
//                        to the launch arena tagged with the batch sequence number, rows-per-key histogram
//   group    per launch: exclusive scan of the histogram + scatter = rows grouped by key (counting sort on the
//                        dense id; replaces lexsort_to_indices + take + partition)
//   apply    per launch: one thread per touched key: orders its rows by (batch, ts), cuts them into runs and
//                        feeds each run to KeyComputingHolder::add_batch (:645-677) restated on device state
//   advance  per watermark: one thread per key with state: KeyComputingHolder::watermark_update (:557-603) for the
//                        keys whose next_watermark_action < watermark (:62-74, :99-160); closed sessions are
//                        appended to the output columns [key, window.start, window.end, aggs..., _timestamp]
//
// Per-key state (SoA, indexed by dense id): active flag, data_start, data_end, accumulators, head of the pending
// run list.  Pending runs (`batches_by_start_time`, a BTreeMap<start, Vec<batch>>) are nodes of a pool, kept as a
// list ordered by (start, insertion); their rows live in a row pool.  Pools are bump-allocated by the kernels and
// grown / compacted by the host between launches.
#include <algorithm>
#include <climits>
#include <cstdlib>

#include <cub/device/device_segmented_sort.cuh>

#include "agg_plan.h"
#include "dict.cuh"
#include "op.h"
#include "scan.cuh"

namespace ab {
namespace {

constexpr int ST = 256;

struct SessCtx {
  long long gap;
  int n_vals, n_acc;
  int acc_kind[MAX_ACC], acc_val[MAX_ACC];
  unsigned long long id_cap;
  // per key
  int* active;
  long long* data_start;
  long long* data_end;
  unsigned long long* acc;  // [n_acc][id_cap]
  int* head;
  // node pool
  int* n_next;
  long long* n_start;
  long long* n_off;
  int* n_len;
  // row pool
  long long* r_ts;
  long long* r_val[MAX_VALS];
  // cursors / counters: [0] node cursor, [1] row cursor, [2] dead nodes, [3] dead rows, [4] out count,
  // [5] error flags, [6] arena cursor, [7] sessions open
  unsigned long long* ctr;
  unsigned long long node_cap, row_cap;
  // output
  const long long* id_keys;
  long long* o_key;
  long long* o_start;
  long long* o_end;
  long long* o_ts;
  unsigned long long* o_agg[ARROYO_B200_MAX_AGGS];
  int n_aggs, agg_kind[ARROYO_B200_MAX_AGGS], agg_acc[ARROYO_B200_MAX_AGGS];
  unsigned long long out_cap;
  int keyed;
};

enum : unsigned long long { ERR_POOL = 1, ERR_ADD_FLUSHED = 2, ERR_BEFORE_START = 4, ERR_OUT = 8, ERR_LOOP = 16, ERR_DICT = 32 };
// Every device loop over the linked lists is bounded: a corrupted list must surface as an error, never as a hang.  The
// bound is what a sound list can take: a list holds at most node_cap nodes; a fill visits each node at most twice
// (pop_first's walk, then add_batch) and allocates its remainders from the same pool; and every session a watermark
// opens consumes at least one pending row, so it opens and closes at most node_cap sessions.
__device__ __forceinline__ unsigned long long loop_guard(const SessCtx& c) { return 3 * c.node_cap + 8; }

struct RowsRef {
  const long long* ts;
  const long long* val[MAX_VALS];
  long long off;
  int n;
};

__device__ __forceinline__ void set_err(const SessCtx& c, unsigned long long e) { atomicOr(c.ctr + 5, e); }

// Bookkeeping a thread accumulates while it runs its keys' state machines; published once per warp at the end of
// the kernel.  (One global atomic per event on four shared counters serialised the whole kernel: tens of millions
// of same-address atomics per launch.)
struct Tally {
  unsigned long long dead_nodes = 0, dead_rows = 0;
  long long open = 0;
};
__device__ __forceinline__ void publish_tally(const SessCtx& c, const Tally& t) {
  unsigned long long dn = t.dead_nodes, dr = t.dead_rows;
  long long op = t.open;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    dn += __shfl_xor_sync(0xffffffffu, dn, o);
    dr += __shfl_xor_sync(0xffffffffu, dr, o);
    op += __shfl_xor_sync(0xffffffffu, op, o);
  }
  if ((threadIdx.x & 31) == 0) {
    if (dn) atomicAdd(c.ctr + 2, dn);
    if (dr) atomicAdd(c.ctr + 3, dr);
    if (op) atomicAdd(c.ctr + 7, (unsigned long long)op);
  }
}

__device__ void acc_reset(const SessCtx& c, uint32_t id) {
  for (int a = 0; a < c.n_acc; ++a) c.acc[(unsigned long long)a * c.id_cap + id] = acc_identity(c.acc_kind[a]);
}

// the session's Single-mode aggregate consumes rows [lo, hi) of r
__device__ void merge_rows(const SessCtx& c, uint32_t id, const RowsRef& r, int lo, int hi) {
  if (hi <= lo) return;
  for (int a = 0; a < c.n_acc; ++a) {
    unsigned long long* dst = c.acc + (unsigned long long)a * c.id_cap + id;
    const int kind = c.acc_kind[a];
    if (kind == ACC_ROWS) {
      *dst += (unsigned long long)(hi - lo);
      continue;
    }
    const long long* src = r.val[c.acc_val[a]] + r.off;
    // in row order, so an f64 sum rounds as the reference's sequential accumulator does
    *dst = acc_with_kind(kind, [&](auto k) {
      unsigned long long cur = *dst;
      for (int i = lo; i < hi; ++i) cur = acc_merge(k, cur, acc_of_value(k, src[i]));
      return cur;
    });
  }
}

// ActiveSession::add_batch (:425-492).  Returns true when rows [rem_lo, n) remain outside the session.
__device__ bool active_add_batch(const SessCtx& c, uint32_t id, const RowsRef& r, int* rem_lo) {
  const long long* ts = r.ts + r.off;
  const int n = r.n;
  const long long start = ts[0], end = ts[n - 1];
  long long ds = c.data_start[id], de = c.data_end[id];
  if (end < de + c.gap) {
    c.data_end[id] = max(de, end);
    c.data_start[id] = min(ds, start);
    merge_rows(c, id, r, 0, n);
    return false;
  }
  if (de + c.gap < start) {
    *rem_lo = 0;
    return true;
  }
  if (start < ds - c.gap) set_err(c, ERR_BEFORE_START);
  if (start < ds) c.data_start[id] = start;
  int index = 1;
  while (index < n) {
    const long long value = ts[index];
    ++index;
    if (value < de) continue;
    if (value < de + c.gap) {
      de = value;
      continue;
    }
    break;  // NB: `index` already points past the row that broke the scan (:464-479)
  }
  c.data_end[id] = de;
  if (index == n) {
    merge_rows(c, id, r, 0, n);
    return false;
  }
  merge_rows(c, id, r, 0, index);
  *rem_lo = index;
  return true;
}

__device__ int alloc_node(const SessCtx& c, long long start, long long off, int len) {
  const unsigned long long i = atomicAdd(c.ctr + 0, 1ull);
  if (i >= c.node_cap) {
    set_err(c, ERR_POOL);
    return -1;
  }
  c.n_next[i] = -1;
  c.n_start[i] = start;
  c.n_off[i] = off;
  c.n_len[i] = len;
  return (int)i;
}

// node `i` was reserved for the caller (apply_kernel hands every run the slot of its first row)
__device__ int init_node(const SessCtx& c, unsigned long long i, long long start, long long off, int len) {
  if (i >= c.node_cap) {
    set_err(c, ERR_POOL);
    return -1;
  }
  c.n_next[i] = -1;
  c.n_start[i] = start;
  c.n_off[i] = off;
  c.n_len[i] = len;
  return (int)i;
}

// by_start.entry(start).or_default().push(node): ordered by start, after the nodes with the same start
__device__ void pending_insert(const SessCtx& c, uint32_t id, int node) {
  if (node < 0) return;
  const long long start = c.n_start[node];
  int prev = -1, cur = c.head[id];
  unsigned long long guard = 0;
  const unsigned long long limit = loop_guard(c);
  while (cur >= 0 && c.n_start[cur] <= start) {
    prev = cur;
    cur = c.n_next[cur];
    if (++guard > limit) {
      set_err(c, ERR_LOOP);
      return;
    }
  }
  c.n_next[node] = cur;
  if (prev < 0) c.head[id] = node;
  else c.n_next[prev] = node;
}

__device__ RowsRef pool_rows(const SessCtx& c, int node) {
  RowsRef r;
  r.ts = c.r_ts;
  for (int v = 0; v < MAX_VALS; ++v) r.val[v] = c.r_val[v];
  r.off = c.n_off[node];
  r.n = c.n_len[node];
  return r;
}

// KeyComputingHolder::fill_active_session (:610-643)
__device__ void fill_active_session(const SessCtx& c, uint32_t id, Tally& tally) {
  unsigned long long guard = 0;
  const unsigned long long limit = loop_guard(c);
  while (true) {
    if (++guard > limit) {
      set_err(c, ERR_LOOP);
      return;
    }
    int h = c.head[id];
    if (h < 0) break;
    const long long first = c.n_start[h];
    if (c.data_end[id] + c.gap < first) break;
    // pop_first(): every run stored under this start time, in insertion order
    int tail = h;
    while (c.n_next[tail] >= 0 && c.n_start[c.n_next[tail]] == first) {
      tail = c.n_next[tail];
      if (++guard > limit) {
        set_err(c, ERR_LOOP);
        return;
      }
    }
    c.head[id] = c.n_next[tail];
    c.n_next[tail] = -1;
    for (int node = h; node >= 0;) {
      if (++guard > limit) {
        set_err(c, ERR_LOOP);
        return;
      }
      const int next = c.n_next[node];
      RowsRef r = pool_rows(c, node);
      int rem_lo = 0;
      if (active_add_batch(c, id, r, &rem_lo)) {
        const int nn = alloc_node(c, r.ts[r.off + rem_lo], r.off + rem_lo, r.n - rem_lo);
        pending_insert(c, id, nn);
        tally.dead_rows += (unsigned long long)rem_lo;
      } else {
        tally.dead_rows += (unsigned long long)r.n;
      }
      tally.dead_nodes += 1;
      node = next;
    }
  }
}

// ActiveSession::finish (:494-523) + to_record_batch (:316-382): one output row
__device__ void finish_session(const SessCtx& c, uint32_t id, Tally& tally) {
  const unsigned long long o = atomicAdd(c.ctr + 4, 1ull);
  if (o >= c.out_cap) {
    // cannot happen (the host sizes the output for one session per live row): still close the session so the
    // caller's loop makes progress, and report
    set_err(c, ERR_OUT);
    c.active[id] = 0;
    tally.open -= 1;
    return;
  }
  const long long start = c.data_start[id], end = c.data_end[id] + c.gap;
  if (c.keyed) c.o_key[o] = c.id_keys[id];
  c.o_start[o] = start;
  c.o_end[o] = end;
  c.o_ts[o] = end - 1;
  const unsigned long long rows = c.acc[id];
  for (int g = 0; g < c.n_aggs; ++g)
    c.o_agg[g][o] = agg_finalise(c.agg_kind[g], c.acc[(unsigned long long)c.agg_acc[g] * c.id_cap + id], rows);
  c.active[id] = 0;
  tally.open -= 1;
}

// KeyComputingHolder::watermark_update (:557-603)
__device__ void watermark_update(const SessCtx& c, uint32_t id, long long wm, bool in_add, Tally& tally) {
  unsigned long long guard = 0;
  const unsigned long long limit = loop_guard(c);
  while (true) {
    if (++guard > limit) {
      set_err(c, ERR_LOOP);
      return;
    }
    if (c.active[id]) {
      if (c.data_end[id] + c.gap < wm) {
        if (in_add) set_err(c, ERR_ADD_FLUSHED);  // "should not have flushed batches when adding a batch" (:672-675)
        finish_session(c, id, tally);
      } else {
        break;
      }
    } else {
      const int h = c.head[id];
      if (h < 0) break;
      const long long initial = c.n_start[h];
      if ((__int128)wm + c.gap < (__int128)initial) break;
      c.active[id] = 1;
      c.data_start[id] = initial;
      c.data_end[id] = initial;
      acc_reset(c, id);
      tally.open += 1;
      fill_active_session(c, id, tally);
    }
  }
}

// KeyComputingHolder::add_batch (:645-677) for one run of `id`.  The run's rows already sit in the row pool at
// `pool_off` (the grouping pass scatters straight into it) and `node` is the slot reserved for it.
__device__ void add_run(const SessCtx& c, uint32_t id, unsigned long long node, long long pool_off, int n, int has_wm,
                        long long wm, Tally& tally) {
  pending_insert(c, id, init_node(c, node, c.r_ts[pool_off], pool_off, n));
  if (!has_wm) return;
  if (c.active[id]) fill_active_session(c, id, tally);
  watermark_update(c, id, wm, true, tally);
}

// ---- kernels --------------------------------------------------------------------------------------------
struct PrepParams {
  const long long* key;
  const long long* ts;
  const long long* val[MAX_VALS];
  long long n;
  unsigned int seq;
  int has_wm;
  long long wm;
  int keyed, n_vals;
  DictView dict;
  unsigned int* min_key_seen;  // set when a row with the INT64_MIN key (id 0, not counted by the dictionary) is kept
  // launch arena (unordered)
  unsigned int* a_id;
  unsigned int* a_seq;
  long long* a_ts;
  long long* a_val[MAX_VALS];
  unsigned int* count;  // rows per id in this launch
  unsigned long long* ctr;
  unsigned long long arena_cap;
  unsigned long long* late;
  long long* earliest;  // min _timestamp of every row ever accepted (what `keys_by_start_time.first_key_value()` holds)
};

__global__ void __launch_bounds__(ST) prep_kernel(const __grid_constant__ PrepParams p) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long stride = (long long)gridDim.x * blockDim.x;
  unsigned long long late = 0;
  long long min_ts = LLONG_MAX;
  const int lane = threadIdx.x & 31;
  // uniform trip count: the arena slots of a warp's rows come from one atomic per warp iteration
  const long long n_round = (p.n + stride - 1) / stride * stride;
  for (; i < n_round; i += stride) {
    bool keep = i < p.n;
    long long ts = 0;
    uint32_t id = 0;
    if (keep) {
      ts = __ldcs(p.ts + i);
      if (p.has_wm && ts < p.wm) {  // K7: gt_eq(timestamp, watermark) filter (:858-868)
        ++late;
        keep = false;
      }
    }
    if (keep && p.keyed) {
      const long long key = __ldcs(p.key + i);
      if (key == EMPTY_KEY) *p.min_key_seen = 1u;
      id = key == EMPTY_KEY ? 0u : dict_insert(p.dict, key, dict_home((uint64_t)key, p.dict.cap));
      if (id >= ID_OVERFLOW) {  // the host sized ids and slots for every row of the launch: the batch fails, loudly
        atomicOr(p.ctr + 5, (unsigned long long)ERR_DICT);
        keep = false;
      }
    }
    const unsigned int kept = __ballot_sync(0xffffffffu, keep);
    if (!kept) continue;
    unsigned long long base = 0;
    if (lane == __ffs(kept) - 1) base = atomicAdd(p.ctr + 6, (unsigned long long)__popc(kept));
    base = __shfl_sync(0xffffffffu, base, __ffs(kept) - 1);
    if (!keep) continue;
    const unsigned long long o = base + __popc(kept & ((1u << lane) - 1u));
    if (o >= p.arena_cap) {
      atomicOr(p.ctr + 5, (unsigned long long)ERR_POOL);
      continue;
    }
    p.a_id[o] = id;
    p.a_seq[o] = p.seq;
    p.a_ts[o] = ts;
    min_ts = min(min_ts, ts);
    for (int v = 0; v < p.n_vals; ++v) p.a_val[v][o] = __ldcs(p.val[v] + i);
    atomicAdd(p.count + id, 1u);
  }
  if (late) atomicAdd(p.late, late);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) min_ts = min(min_ts, __shfl_xor_sync(0xffffffffu, min_ts, o));
  if (lane == 0 && min_ts != LLONG_MAX) atomicMin(p.earliest, min_ts);
}

struct GroupParams {
  const unsigned int* a_id;
  unsigned int* a_seq;  // written back only by the segmented sort of big keys, which parks rows here
  long long* a_ts;
  long long* a_val[MAX_VALS];
  unsigned long long n;
  int n_vals;
  const unsigned long long* offset;  // per id
  unsigned int* cursor;              // per id, zeroed
  unsigned int* g_seq;
  long long* g_ts;
  long long* g_val[MAX_VALS];
};

__global__ void __launch_bounds__(ST) group_kernel(const __grid_constant__ GroupParams p) {
  unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
  const unsigned long long stride = (unsigned long long)gridDim.x * blockDim.x;
  for (; i < p.n; i += stride) {
    const unsigned int id = p.a_id[i];
    const unsigned long long o = p.offset[id] + atomicAdd(p.cursor + id, 1u);
    p.g_seq[o] = p.a_seq[i];
    p.g_ts[o] = p.a_ts[i];
    for (int v = 0; v < p.n_vals; ++v) p.g_val[v][o] = p.a_val[v][i];
  }
}

// Keys with more rows than this in one launch are sorted by a device-wide segmented sort instead of one thread.
constexpr unsigned int SMALL_SORT = 16;

// the keys with more than SMALL_SORT rows in this launch: their grouped ranges [begin, end)
__global__ void big_keys_kernel(unsigned int n_ids, const unsigned int* count, const unsigned long long* offset,
                                unsigned int* seg_begin, unsigned int* seg_end, unsigned int* n_seg) {
  unsigned int id = blockIdx.x * blockDim.x + threadIdx.x;
  const unsigned int stride = gridDim.x * blockDim.x;
  for (; id < n_ids; id += stride) {
    const unsigned int cnt = count[id];
    if (cnt <= SMALL_SORT) continue;
    const unsigned int s = atomicAdd(n_seg, 1u);
    seg_begin[s] = (unsigned int)offset[id];
    seg_end[s] = (unsigned int)(offset[id] + cnt);
  }
}

// one block per big key: park its grouped rows in the (now unused) launch arena at the same positions, and seed the
// sort with the timestamps and the identity permutation
__global__ void big_park_kernel(const unsigned int* seg_begin, const unsigned int* seg_end, GroupParams g,
                                long long* key, unsigned int* idx) {
  const unsigned int b = seg_begin[blockIdx.x], e = seg_end[blockIdx.x];
  for (unsigned int i = b + threadIdx.x; i < e; i += blockDim.x) {
    g.a_seq[i] = g.g_seq[i];
    g.a_ts[i] = g.g_ts[i];
    for (int v = 0; v < g.n_vals; ++v) g.a_val[v][i] = g.g_val[v][i];
    key[i] = g.g_ts[i];
    idx[i] = i;
  }
}

// after the stable sort by ts: the batch number of each row, in that order, as the key of the second stable sort
__global__ void big_seq_kernel(const unsigned int* seg_begin, const unsigned int* seg_end, const unsigned int* a_seq,
                               const unsigned int* idx, unsigned int* seq) {
  const unsigned int b = seg_begin[blockIdx.x], e = seg_end[blockIdx.x];
  for (unsigned int i = b + threadIdx.x; i < e; i += blockDim.x) seq[i] = a_seq[idx[i]];
}

// rows back into the row pool in (batch, ts) order
__global__ void big_gather_kernel(const unsigned int* seg_begin, const unsigned int* seg_end, GroupParams g,
                                  const unsigned int* idx) {
  const unsigned int b = seg_begin[blockIdx.x], e = seg_end[blockIdx.x];
  for (unsigned int i = b + threadIdx.x; i < e; i += blockDim.x) {
    const unsigned int src = idx[i];
    g.g_seq[i] = g.a_seq[src];
    g.g_ts[i] = g.a_ts[src];
    for (int v = 0; v < g.n_vals; ++v) g.g_val[v][i] = g.a_val[v][src];
  }
}

struct ApplyParams {
  SessCtx c;
  unsigned int n_ids;
  unsigned int* count;
  unsigned int* cursor;
  const unsigned long long* offset;
  unsigned int* g_seq;
  long long* g_ts;       // row pool + row_base: the grouping pass wrote this launch's rows straight into the pool
  long long* g_val[MAX_VALS];
  unsigned long long row_base, node_base;  // pool positions of grouped row 0 / of the node slot of grouped row 0
  int has_wm;
  long long wm;
};

__global__ void __launch_bounds__(128) apply_kernel(const __grid_constant__ ApplyParams p) {
  unsigned int id = blockIdx.x * blockDim.x + threadIdx.x;
  const unsigned int stride = gridDim.x * blockDim.x;
  Tally tally;
  for (; id < p.n_ids; id += stride) {
    const unsigned int cnt = p.count[id];
    if (!cnt) continue;
    p.count[id] = 0;
    p.cursor[id] = 0;
    const unsigned long long off = p.offset[id];
    // order this key's rows by (batch, ts).  A key with more than SMALL_SORT rows in this launch was ordered by the
    // segmented sort (sort_big_keys); the few rows of any other key are ordered here, at a cost bounded by SMALL_SORT^2.
    for (unsigned int i = 1; i < cnt && cnt <= SMALL_SORT; ++i) {
      const unsigned int s = p.g_seq[off + i];
      const long long t = p.g_ts[off + i];
      long long vv[MAX_VALS];
      for (int v = 0; v < p.c.n_vals; ++v) vv[v] = p.g_val[v][off + i];
      long long j = (long long)i - 1;
      while (j >= 0 && (p.g_seq[off + j] > s || (p.g_seq[off + j] == s && p.g_ts[off + j] > t))) {
        p.g_seq[off + j + 1] = p.g_seq[off + j];
        p.g_ts[off + j + 1] = p.g_ts[off + j];
        for (int v = 0; v < p.c.n_vals; ++v) p.g_val[v][off + j + 1] = p.g_val[v][off + j];
        --j;
      }
      p.g_seq[off + j + 1] = s;
      p.g_ts[off + j + 1] = t;
      for (int v = 0; v < p.c.n_vals; ++v) p.g_val[v][off + j + 1] = vv[v];
    }
    // one run per input batch, in arrival order; a run's node is the slot of its first row
    unsigned int lo = 0, runs = 0;
    while (lo < cnt) {
      unsigned int hi = lo + 1;
      while (hi < cnt && p.g_seq[off + hi] == p.g_seq[off + lo]) ++hi;
      add_run(p.c, id, p.node_base + off + lo, (long long)(p.row_base + off + lo), (int)(hi - lo), p.has_wm, p.wm, tally);
      ++runs;
      lo = hi;
    }
    tally.dead_nodes += cnt - runs;  // reserved node slots that no run uses
  }
  publish_tally(p.c, tally);
}

struct AdvanceParams {
  SessCtx c;
  unsigned int n_ids;
  long long wm;
};

__global__ void __launch_bounds__(128) advance_kernel(const __grid_constant__ AdvanceParams p) {
  unsigned int id = blockIdx.x * blockDim.x + threadIdx.x;
  const unsigned int stride = gridDim.x * blockDim.x;
  Tally tally;
  for (; id < p.n_ids; id += stride) {
    const int h = p.c.head[id];
    const bool act = p.c.active[id] != 0;
    if (!act && h < 0) continue;
    // next_watermark_action (:536-546); only keys whose action time is before the watermark advance (:62-74)
    const __int128 action = act ? (__int128)p.c.data_end[id] + p.c.gap : (__int128)p.c.n_start[h] - p.c.gap;
    if (!(action < (__int128)p.wm)) continue;
    watermark_update(p.c, id, p.wm, false, tally);
  }
  publish_tally(p.c, tally);
}

// pool compaction: live nodes / rows per key -> offsets -> copy
__global__ void live_count_kernel(SessCtx c, unsigned int n_ids, unsigned int* cnt_nodes, unsigned int* cnt_rows) {
  unsigned int id = blockIdx.x * blockDim.x + threadIdx.x;
  const unsigned int stride = gridDim.x * blockDim.x;
  for (; id < n_ids; id += stride) {
    unsigned int nn = 0, nr = 0;
    for (int node = c.head[id]; node >= 0; node = c.n_next[node]) {
      ++nn;
      nr += (unsigned int)c.n_len[node];
    }
    cnt_nodes[id] = nn;
    cnt_rows[id] = nr;
  }
}
struct CompactDst {
  int* n_next;
  long long* n_start;
  long long* n_off;
  int* n_len;
  long long* r_ts;
  long long* r_val[MAX_VALS];
};
__global__ void compact_copy_kernel(SessCtx c, CompactDst d, unsigned int n_ids, const unsigned long long* node_off,
                                    const unsigned long long* row_off) {
  unsigned int id = blockIdx.x * blockDim.x + threadIdx.x;
  const unsigned int stride = gridDim.x * blockDim.x;
  for (; id < n_ids; id += stride) {
    int node = c.head[id];
    if (node < 0) continue;
    unsigned long long no = node_off[id], ro = row_off[id];
    c.head[id] = (int)no;
    while (node >= 0) {
      const int next = c.n_next[node];
      const int len = c.n_len[node];
      const long long so = c.n_off[node];
      d.n_start[no] = c.n_start[node];
      d.n_off[no] = (long long)ro;
      d.n_len[no] = len;
      d.n_next[no] = next >= 0 ? (int)(no + 1) : -1;
      for (int i = 0; i < len; ++i) {
        d.r_ts[ro + i] = c.r_ts[so + i];
        for (int v = 0; v < c.n_vals; ++v) d.r_val[v][ro + i] = c.r_val[v][so + i];
      }
      ro += (unsigned long long)len;
      ++no;
      node = next;
    }
  }
}

__global__ void fill_i32_kernel(int* p, int v, unsigned long long n) {
  unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
  const unsigned long long stride = (unsigned long long)gridDim.x * blockDim.x;
  for (; i < n; i += stride) p[i] = v;
}

// ---- host -----------------------------------------------------------------------------------------------
class SessionOp final : public OpBase {
 public:
  explicit SessionOp(const ArroyoB200OpConfig& c);
  ~SessionOp() override;
  void on_start(ArrowArray* state, ArrowSchema* schemas, int64_t n, int64_t watermark, int64_t start_time) override;
  void process_batch(uint32_t, uint32_t, ArrowArray* batch, const ArrowSchema* schema) override;
  void process_device_batch(uint32_t, uint32_t, const uint64_t* cols, int32_t n_cols, int64_t n_rows) override;
  void handle_watermark(int64_t wm, BatchesPriv* out_host, std::vector<ArroyoB200DeviceBatch>* out_dev) override;
  void handle_checkpoint(int64_t, BatchesPriv* out) override;
  void on_close(int, BatchesPriv*) override { flush(); }
  void flush() override;
  void stats(ArroyoB200Stats* out) override {
    unsigned long long late = 0;  // current, not as of the last watermark
    AB_CUDA(cudaMemcpyAsync(&late, late_.p, 8, cudaMemcpyDeviceToHost, stream_));
    AB_CUDA(cudaStreamSynchronize(stream_));
    st_.rows_late = late;
    st_.n_keys = 0;
    if (plan_.keyed) {
      // the dictionary's count (ids 1.., id 0 is INT64_MIN's) and whether an INT64_MIN key was accepted
      unsigned int nk[2] = {1, 0};
      AB_CUDA(cudaMemcpyAsync(nk, n_keys_dev_.p, sizeof nk, cudaMemcpyDeviceToHost, stream_));
      AB_CUDA(cudaStreamSynchronize(stream_));
      st_.n_keys = (uint64_t)(nk[0] - 1) + (nk[1] ? 1 : 0);
    }
    *out = st_;
  }

 private:
  AggPlan plan_;
  int64_t gap_;
  std::string key_format_ = "l";

  // dictionary + per-key state
  uint64_t id_cap_ = 0, dict_cap_ = 0;
  uint32_t n_keys_ = 1;
  DevBuf slots_, id_keys_, n_keys_dev_;
  DevBuf active_, data_start_, data_end_, acc_, head_, count_, cursor_, offset_;
  // pools
  uint64_t node_cap_ = 0, row_cap_ = 0;
  DevBuf n_next_, n_start_, n_off_, n_len_, r_ts_, r_val_[MAX_VALS];
  // compaction copies the live nodes / rows into a second set of pools and swaps the sets; both sets and the scratch
  // arrays persist (a cudaMalloc / cudaFree per step synchronises the device -- and, behind an NCCL edge, waits for the
  // peers' progress: 145 ms per step at N = 2 before they were kept)
  uint64_t sp_node_cap_ = 0, sp_row_cap_ = 0;
  DevBuf sp_next_, sp_start_, sp_off_, sp_len_, sp_rts_, sp_rval_[MAX_VALS];
  DevBuf c_cn_, c_cr_, c_on_, c_orow_, c_tot_;
  uint64_t c_cap_ = 0;
  DevBuf ctr_;
  PinnedBuf h_ctr_;
  // launch arena
  uint64_t arena_cap_ = 0;
  DevBuf a_id_, a_seq_, a_ts_, a_val_[MAX_VALS], g_seq_;
  // segmented sort of the keys with more than SMALL_SORT rows in a launch (sized on first use)
  uint64_t sort_cap_ = 0;
  DevBuf s_key_, s_key_out_, s_idx_, s_idx_out_, s_seq_, s_seq_out_, s_begin_, s_end_, s_nseg_, s_tmp_;
  uint64_t arena_rows_bound_ = 0;  // rows prepped since the last apply (upper bound incl. late rows)
  uint32_t seq_ = 0;
  bool has_wm_ = false;
  int64_t wm_ = 0;
  AggStaging staging_;
  DevBuf scan_sums_;
  // output
  uint64_t out_cap_ = 0;
  DevBuf o_key_, o_start_, o_end_, o_ts_, o_agg_[ARROYO_B200_MAX_AGGS];
  HeldInputs inputs_;  // host batches whose copies to staging_ may still run
  ArroyoB200Stats st_{};
  DevBuf late_, earliest_;
  uint64_t compact_min_ = 1u << 16;  // pools smaller than this are never compacted (ARROYO_B200_SESSION_COMPACT_MIN)

  int grid_for(uint64_t n, int threads) const {
    return (int)std::max<uint64_t>(1, std::min<uint64_t>((n + threads - 1) / threads, (uint64_t)num_sms_ * 16));
  }
  void alloc_keys(uint64_t cap);
  void grow_keys(uint64_t need);
  void ensure_pools(uint64_t add_nodes, uint64_t add_rows);
  void ensure_arena(uint64_t rows);
  SessCtx ctx();
  void read_ctr() {
    AB_CUDA(cudaMemcpyAsync(h_ctr_.p, ctr_.p, 8 * sizeof(unsigned long long), cudaMemcpyDeviceToHost, stream_));
    AB_CUDA(cudaStreamSynchronize(stream_));
  }
  void check_err();
  void prep(const AggCols& d, int64_t n);
  void apply_pending();
  void sort_big_keys(const GroupParams& g, uint64_t n);
  void maybe_compact();
};

SessionOp::SessionOp(const ArroyoB200OpConfig& c) {
  cfg = c;
  name = "session_window";
  AB_REQUIRE(c.gap_ns > 0, ARROYO_B200_INVALID_ARGUMENT, "session gap must be positive");
  gap_ = c.gap_ns;
  plan_ = AggPlan(c, ACC_SUM_F64);  // AVG: the sequential f64 sum per key
  open_device(c);
  if (const char* e = getenv("ARROYO_B200_SESSION_COMPACT_MIN")) compact_min_ = std::max<uint64_t>(1, strtoull(e, nullptr, 10));
  ctr_.alloc(8 * sizeof(unsigned long long));
  h_ctr_.alloc(8 * sizeof(unsigned long long));
  late_.alloc(8);
  earliest_.alloc(8);
  {
    const long long none = LLONG_MAX;
    AB_CUDA(cudaMemcpyAsync(earliest_.p, &none, 8, cudaMemcpyHostToDevice, stream_));
  }
  AB_CUDA(cudaMemsetAsync(ctr_.p, 0, 8 * sizeof(unsigned long long), stream_));
  AB_CUDA(cudaMemsetAsync(late_.p, 0, 8, stream_));
  n_keys_dev_.alloc(2 * sizeof(unsigned int));  // [dictionary count, INT64_MIN key seen]
  AB_CUDA(cudaMemsetAsync(n_keys_dev_.p, 0, 2 * sizeof(unsigned int), stream_));
  uint64_t want = c.expected_keys ? c.expected_keys : (1ull << 16);
  alloc_keys(plan_.keyed ? ((want + want / 8 + 2 + 1023) / 1024) * 1024 : 1024);
  AB_CUDA(cudaStreamSynchronize(stream_));
}

SessionOp::~SessionOp() { drain_stream(); }

void SessionOp::alloc_keys(uint64_t cap) {
  id_cap_ = cap;
  id_keys_.alloc(cap * 8);
  long long k0 = EMPTY_KEY;
  AB_CUDA(cudaMemcpyAsync(id_keys_.p, &k0, 8, cudaMemcpyHostToDevice, stream_));
  unsigned int one = 1;
  AB_CUDA(cudaMemcpyAsync(n_keys_dev_.p, &one, 4, cudaMemcpyHostToDevice, stream_));
  if (plan_.keyed) {
    dict_cap_ = dict_slots_for(cap);
    AB_REQUIRE(dict_cap_ <= (1ull << 31), ARROYO_B200_RUNTIME, "key dictionary too large");
    slots_.alloc(dict_cap_ * sizeof(Slot));
    dict_init_kernel<<<num_sms_ * 4, 256, 0, stream_>>>(slots_.as<Slot>(), dict_cap_);
    AB_CUDA(cudaGetLastError());
  }
  active_.alloc(cap * 4);
  data_start_.alloc(cap * 8);
  data_end_.alloc(cap * 8);
  acc_.alloc((size_t)plan_.n_acc * cap * 8);
  head_.alloc(cap * 4);
  count_.alloc(cap * 4);
  cursor_.alloc(cap * 4);
  offset_.alloc(cap * 8);
  AB_CUDA(cudaMemsetAsync(active_.p, 0, cap * 4, stream_));
  AB_CUDA(cudaMemsetAsync(count_.p, 0, cap * 4, stream_));
  AB_CUDA(cudaMemsetAsync(cursor_.p, 0, cap * 4, stream_));
  fill_i32_kernel<<<grid_for(cap, 256), 256, 0, stream_>>>(head_.as<int>(), -1, cap);
  AB_CUDA(cudaGetLastError());
}

// Doubles the dense id space until it can take `need` more keys.
void SessionOp::grow_keys(uint64_t need) {
  if ((uint64_t)n_keys_ + need <= id_cap_) return;
  // n_keys_ is a host-side upper bound between launches: fetch the real count before deciding
  unsigned int actual = 1;
  AB_CUDA(cudaMemcpyAsync(&actual, n_keys_dev_.p, 4, cudaMemcpyDeviceToHost, stream_));
  AB_CUDA(cudaStreamSynchronize(stream_));
  n_keys_ = (uint32_t)std::min<uint64_t>(actual, id_cap_);
  if ((uint64_t)n_keys_ + need <= id_cap_) return;
  uint64_t nc = id_cap_;
  while ((uint64_t)n_keys_ + need > nc) nc *= 2;
  const uint64_t oc = id_cap_;
  const uint64_t nv = n_keys_;
  auto regrow = [&](DevBuf& b, size_t elem, bool zero) {
    DevBuf nb(nc * elem);
    if (zero) AB_CUDA(cudaMemsetAsync(nb.p, 0, nc * elem, stream_));
    AB_CUDA(cudaMemcpyAsync(nb.p, b.p, nv * elem, cudaMemcpyDeviceToDevice, stream_));
    AB_CUDA(cudaStreamSynchronize(stream_));
    b = std::move(nb);
  };
  regrow(id_keys_, 8, false);
  regrow(active_, 4, true);
  regrow(data_start_, 8, false);
  regrow(data_end_, 8, false);
  regrow(count_, 4, true);
  regrow(cursor_, 4, true);
  {
    DevBuf nb(nc * 4);
    fill_i32_kernel<<<grid_for(nc, 256), 256, 0, stream_>>>(nb.as<int>(), -1, nc);
    AB_CUDA(cudaGetLastError());
    AB_CUDA(cudaMemcpyAsync(nb.p, head_.p, nv * 4, cudaMemcpyDeviceToDevice, stream_));
    AB_CUDA(cudaStreamSynchronize(stream_));
    head_ = std::move(nb);
  }
  {
    DevBuf nb((size_t)plan_.n_acc * nc * 8);
    for (int a = 0; a < plan_.n_acc; ++a)
      AB_CUDA(cudaMemcpyAsync(nb.as<unsigned long long>() + (size_t)a * nc, acc_.as<unsigned long long>() + (size_t)a * oc,
                              nv * 8, cudaMemcpyDeviceToDevice, stream_));
    AB_CUDA(cudaStreamSynchronize(stream_));
    acc_ = std::move(nb);
  }
  offset_.alloc(nc * 8);
  id_cap_ = nc;
  if (plan_.keyed) {
    dict_cap_ = dict_slots_for(nc);
    AB_REQUIRE(dict_cap_ <= (1ull << 31), ARROYO_B200_RUNTIME, "key dictionary too large");
    slots_.alloc(dict_cap_ * sizeof(Slot));
    dict_init_kernel<<<num_sms_ * 4, 256, 0, stream_>>>(slots_.as<Slot>(), dict_cap_);
    AB_CUDA(cudaGetLastError());
    if (nv > 1) {
      dict_rebuild_kernel<<<grid_for(nv, 256), 256, 0, stream_>>>(slots_.as<Slot>(), (uint32_t)dict_cap_,
                                                                  id_keys_.as<long long>(), (uint32_t)nv, 1u);
      AB_CUDA(cudaGetLastError());
    }
  }
  AB_CUDA(cudaStreamSynchronize(stream_));
}

void SessionOp::ensure_pools(uint64_t add_nodes, uint64_t add_rows) {
  read_ctr();
  const unsigned long long* h = h_ctr_.as<unsigned long long>();
  const uint64_t nodes = h[0], rows = h[1];
  auto regrow = [&](DevBuf& b, size_t elem, uint64_t used, uint64_t cap) {
    DevBuf nb(cap * elem);
    if (used) AB_CUDA(cudaMemcpyAsync(nb.p, b.p, used * elem, cudaMemcpyDeviceToDevice, stream_));
    AB_CUDA(cudaStreamSynchronize(stream_));
    b = std::move(nb);
  };
  if (nodes + add_nodes > node_cap_) {
    uint64_t nc = std::max<uint64_t>(node_cap_ * 2, 1 << 16);
    while (nodes + add_nodes > nc) nc *= 2;
    regrow(n_next_, 4, nodes, nc);
    regrow(n_start_, 8, nodes, nc);
    regrow(n_off_, 8, nodes, nc);
    regrow(n_len_, 4, nodes, nc);
    node_cap_ = nc;
  }
  if (rows + add_rows > row_cap_) {
    uint64_t rc = std::max<uint64_t>(row_cap_ * 2, 1 << 16);
    while (rows + add_rows > rc) rc *= 2;
    regrow(r_ts_, 8, rows, rc);
    for (int v = 0; v < plan_.n_vals; ++v) regrow(r_val_[v], 8, rows, rc);
    row_cap_ = rc;
  }
}

void SessionOp::ensure_arena(uint64_t rows) {
  if (rows <= arena_cap_) return;
  AB_REQUIRE(arena_rows_bound_ == 0, ARROYO_B200_RUNTIME, "arena growth with rows pending");
  uint64_t nc = std::max<uint64_t>(arena_cap_ * 2, 1 << 16);
  while (nc < rows) nc *= 2;
  a_id_.alloc(nc * 4);
  a_seq_.alloc(nc * 4);
  a_ts_.alloc(nc * 8);
  g_seq_.alloc(nc * 4);  // grouped timestamps / values go straight into the row pool (apply_pending)
  for (int v = 0; v < plan_.n_vals; ++v) a_val_[v].alloc(nc * 8);
  arena_cap_ = nc;
}

SessCtx SessionOp::ctx() {
  SessCtx c{};
  c.gap = gap_;
  c.n_vals = plan_.n_vals;
  c.n_acc = plan_.n_acc;
  for (int a = 0; a < plan_.n_acc; ++a) {
    c.acc_kind[a] = plan_.acc_kind[a];
    c.acc_val[a] = plan_.acc_val[a];
  }
  c.id_cap = id_cap_;
  c.active = active_.as<int>();
  c.data_start = data_start_.as<long long>();
  c.data_end = data_end_.as<long long>();
  c.acc = acc_.as<unsigned long long>();
  c.head = head_.as<int>();
  c.n_next = n_next_.as<int>();
  c.n_start = n_start_.as<long long>();
  c.n_off = n_off_.as<long long>();
  c.n_len = n_len_.as<int>();
  c.r_ts = r_ts_.as<long long>();
  for (int v = 0; v < MAX_VALS; ++v) c.r_val[v] = v < plan_.n_vals ? r_val_[v].as<long long>() : nullptr;
  c.ctr = ctr_.as<unsigned long long>();
  c.node_cap = node_cap_;
  c.row_cap = row_cap_;
  c.id_keys = id_keys_.as<long long>();
  c.o_key = o_key_.as<long long>();
  c.o_start = o_start_.as<long long>();
  c.o_end = o_end_.as<long long>();
  c.o_ts = o_ts_.as<long long>();
  c.n_aggs = plan_.n_aggs;
  for (int g = 0; g < plan_.n_aggs; ++g) {
    c.o_agg[g] = o_agg_[g].as<unsigned long long>();
    c.agg_kind[g] = plan_.agg_kind[g];
    c.agg_acc[g] = plan_.agg_acc[g];
  }
  c.out_cap = out_cap_;
  c.keyed = plan_.keyed ? 1 : 0;
  return c;
}

void SessionOp::check_err() {
  const unsigned long long e = h_ctr_.as<unsigned long long>()[5];
  if (!e) return;
  if (e & ERR_BEFORE_START)
    throw Error(ARROYO_B200_RUNTIME, "received a batch that starts before the current data_start - gap (session_aggregating_window.rs:452-456)");
  if (e & ERR_ADD_FLUSHED)
    throw Error(ARROYO_B200_RUNTIME, "should not have flushed batches when adding a batch (session_aggregating_window.rs:672-675)");
  if (e & ERR_LOOP) throw Error(ARROYO_B200_RUNTIME, "session operator: per-key list walk exceeded its bound (corrupted state)");
  if (e & ERR_DICT) throw Error(ARROYO_B200_RUNTIME, "session operator: a new key found no id or slot in the key dictionary");
  throw Error(ARROYO_B200_RUNTIME, "session operator pool / output capacity exceeded");
}

// one input batch -> launch arena
void SessionOp::prep(const AggCols& d, int64_t n) {
  if (n <= 0) return;
  // a launch never mixes rows that arrived under different watermarks, and is cut at 4 Mi rows
  if (arena_rows_bound_ + (uint64_t)n > (1ull << 22) && arena_rows_bound_ > 0) apply_pending();
  if (arena_rows_bound_ + (uint64_t)n > arena_cap_ && arena_rows_bound_ > 0) apply_pending();
  ensure_arena(arena_rows_bound_ + (uint64_t)n);
  if (plan_.keyed) grow_keys((uint64_t)n);
  PrepParams p{};
  p.key = d.key;
  p.ts = d.ts;
  for (int v = 0; v < plan_.n_vals; ++v) p.val[v] = d.val[v];
  p.n = n;
  p.seq = seq_++;
  p.has_wm = has_wm_ ? 1 : 0;
  p.wm = wm_;
  p.keyed = plan_.keyed ? 1 : 0;
  p.n_vals = plan_.n_vals;
  p.dict.slots = slots_.as<Slot>();
  p.dict.id_keys = id_keys_.as<long long>();
  p.dict.n_keys = n_keys_dev_.as<unsigned int>();
  p.min_key_seen = n_keys_dev_.as<unsigned int>() + 1;
  p.dict.cap = plan_.keyed ? (uint32_t)dict_cap_ : 1;
  p.dict.id_cap = (uint32_t)std::min<uint64_t>(id_cap_, 0xFFFFFFF0ull);
  p.a_id = a_id_.as<unsigned int>();
  p.a_seq = a_seq_.as<unsigned int>();
  p.a_ts = a_ts_.as<long long>();
  for (int v = 0; v < plan_.n_vals; ++v) p.a_val[v] = a_val_[v].as<long long>();
  p.count = count_.as<unsigned int>();
  p.ctr = ctr_.as<unsigned long long>();
  p.arena_cap = arena_cap_;
  p.late = late_.as<unsigned long long>();
  p.earliest = earliest_.as<long long>();
  prep_kernel<<<grid_for((uint64_t)n, ST), ST, 0, stream_>>>(p);
  AB_CUDA(cudaGetLastError());
  ++st_.kernel_launches;
  ++st_.ingest_launches;
  arena_rows_bound_ += (uint64_t)n;
  // n_keys grows with the rows seen; keep a conservative host bound for capacity planning
  n_keys_ = (uint32_t)std::min<uint64_t>((uint64_t)n_keys_ + (plan_.keyed ? (uint64_t)n : 0), id_cap_);
}

void SessionOp::process_batch(uint32_t, uint32_t, ArrowArray* batch, const ArrowSchema* schema) {
  set_device();
  AggCols d;
  const int64_t n = staging_.stage(plan_, batch, schema, stream_, &st_, &key_format_, &d);
  inputs_.release(false);
  if (n == 0) {
    if (batch->release) batch->release(batch);
    return;
  }
  inputs_.hold(batch, stream_);
  prep(d, n);
}

void SessionOp::process_device_batch(uint32_t, uint32_t, const uint64_t* cols, int32_t n_cols, int64_t n_rows) {
  set_device();
  const AggCols d = plan_.columns(cols, n_cols);
  if (n_rows <= 0) return;
  st_.rows_in += (uint64_t)n_rows;
  prep(d, n_rows);
}

// group the arena by key and run the per-key state machines over the new runs
void SessionOp::apply_pending() {
  if (arena_rows_bound_ == 0) return;
  read_ctr();
  check_err();
  const uint64_t n = h_ctr_.as<unsigned long long>()[6];
  unsigned int nk = 1;
  if (plan_.keyed) {
    AB_CUDA(cudaMemcpyAsync(&nk, n_keys_dev_.p, 4, cudaMemcpyDeviceToHost, stream_));
    AB_CUDA(cudaStreamSynchronize(stream_));
  }
  n_keys_ = (uint32_t)std::min<uint64_t>(nk, id_cap_);
  arena_rows_bound_ = 0;
  unsigned long long zero = 0;
  AB_CUDA(cudaMemcpyAsync(ctr_.as<unsigned long long>() + 6, &zero, 8, cudaMemcpyHostToDevice, stream_));
  if (n == 0) return;
  {
    // one node per new run, plus at most one remainder per row that can still be merged (new or already pending)
    const unsigned long long* hh = h_ctr_.as<unsigned long long>();
    const uint64_t live_rows = hh[1] - hh[3];
    ensure_pools(2 * n + live_rows + 16, n);
  }
  device_exclusive_scan(count_.as<unsigned int>(), n_keys_, offset_.as<unsigned long long>(),
                        ctr_.as<unsigned long long>() + 6 /* scratch: re-zeroed below */, scan_sums_, stream_);
  AB_CUDA(cudaMemcpyAsync(ctr_.as<unsigned long long>() + 6, &zero, 8, cudaMemcpyHostToDevice, stream_));
  GroupParams g{};
  g.a_id = a_id_.as<unsigned int>();
  g.a_seq = a_seq_.as<unsigned int>();
  g.a_ts = a_ts_.as<long long>();
  g.n = n;
  g.n_vals = plan_.n_vals;
  g.offset = offset_.as<unsigned long long>();
  g.cursor = cursor_.as<unsigned int>();
  // This launch's rows go straight into the row pool at [row_base, row_base + n) in grouped order, and grouped
  // row i owns node slot node_base + i: no allocation atomics in the per-key state machines (remainder nodes, the
  // only other allocation, come from the cursor behind the reserved range).
  const SessCtx cx = ctx();
  const unsigned long long row_base = h_ctr_.as<unsigned long long>()[1], node_base = h_ctr_.as<unsigned long long>()[0];
  AB_REQUIRE(row_base + n <= cx.row_cap && node_base + n <= cx.node_cap, ARROYO_B200_RUNTIME, "session pools too small");
  const unsigned long long cur2[2] = {node_base + n, row_base + n};
  AB_CUDA(cudaMemcpyAsync(ctr_.as<unsigned long long>(), cur2, sizeof cur2, cudaMemcpyHostToDevice, stream_));
  g.g_seq = g_seq_.as<unsigned int>();
  g.g_ts = cx.r_ts + row_base;
  for (int v = 0; v < plan_.n_vals; ++v) {
    g.a_val[v] = a_val_[v].as<long long>();
    g.g_val[v] = cx.r_val[v] + row_base;
  }
  group_kernel<<<grid_for(n, ST), ST, 0, stream_>>>(g);
  AB_CUDA(cudaGetLastError());
  sort_big_keys(g, n);
  ApplyParams a{};
  a.c = ctx();
  a.n_ids = n_keys_;
  a.count = count_.as<unsigned int>();
  a.cursor = cursor_.as<unsigned int>();
  a.offset = offset_.as<unsigned long long>();
  a.g_seq = g_seq_.as<unsigned int>();
  a.g_ts = cx.r_ts + row_base;
  for (int v = 0; v < plan_.n_vals; ++v) a.g_val[v] = cx.r_val[v] + row_base;
  a.row_base = row_base;
  a.node_base = node_base;
  a.has_wm = has_wm_ ? 1 : 0;
  a.wm = wm_;
  apply_kernel<<<grid_for(n_keys_, 128), 128, 0, stream_>>>(a);
  AB_CUDA(cudaGetLastError());
  st_.kernel_launches += 5;
  read_ctr();
  check_err();
}

// Orders the grouped rows of every key with more than SMALL_SORT rows in this launch by (batch, ts): two stable
// segmented sorts (by ts, then by batch) over those keys' ranges, then one gather.  The cost is O(n log n) in the
// key's rows, where one thread's insertion sort was O(n^2): a hot key, or the unkeyed operator, can hold millions of
// rows in one launch.
void SessionOp::sort_big_keys(const GroupParams& g, uint64_t n) {
  const uint64_t max_seg = n / (SMALL_SORT + 1);
  if (max_seg == 0) return;
  if (sort_cap_ < n) {
    sort_cap_ = std::max<uint64_t>(n, 2 * sort_cap_);
    s_key_.alloc(sort_cap_ * 8);
    s_key_out_.alloc(sort_cap_ * 8);
    s_idx_.alloc(sort_cap_ * 4);
    s_idx_out_.alloc(sort_cap_ * 4);
    s_seq_.alloc(sort_cap_ * 4);
    s_seq_out_.alloc(sort_cap_ * 4);
    s_begin_.alloc((sort_cap_ / (SMALL_SORT + 1) + 1) * 4);
    s_end_.alloc((sort_cap_ / (SMALL_SORT + 1) + 1) * 4);
    s_nseg_.alloc(4);
  }
  AB_CUDA(cudaMemsetAsync(s_nseg_.p, 0, 4, stream_));
  big_keys_kernel<<<grid_for(n_keys_, 256), 256, 0, stream_>>>(n_keys_, count_.as<unsigned int>(), offset_.as<unsigned long long>(),
                                                               s_begin_.as<unsigned int>(), s_end_.as<unsigned int>(),
                                                               s_nseg_.as<unsigned int>());
  AB_CUDA(cudaGetLastError());
  unsigned int n_seg = 0;
  AB_CUDA(cudaMemcpyAsync(&n_seg, s_nseg_.p, 4, cudaMemcpyDeviceToHost, stream_));
  AB_CUDA(cudaStreamSynchronize(stream_));
  st_.kernel_launches += 1;
  if (n_seg == 0) return;
  const unsigned int* sb = s_begin_.as<unsigned int>();
  const unsigned int* se = s_end_.as<unsigned int>();
  big_park_kernel<<<n_seg, ST, 0, stream_>>>(sb, se, g, s_key_.as<long long>(), s_idx_.as<unsigned int>());
  AB_CUDA(cudaGetLastError());
  size_t t1 = 0, t2 = 0;
  AB_CUDA(cub::DeviceSegmentedSort::StableSortPairs(nullptr, t1, s_key_.as<long long>(), s_key_out_.as<long long>(),
                                                    s_idx_.as<unsigned int>(), s_idx_out_.as<unsigned int>(), (int)n,
                                                    (int)n_seg, sb, se, stream_));
  AB_CUDA(cub::DeviceSegmentedSort::StableSortPairs(nullptr, t2, s_seq_.as<unsigned int>(), s_seq_out_.as<unsigned int>(),
                                                    s_idx_out_.as<unsigned int>(), s_idx_.as<unsigned int>(), (int)n,
                                                    (int)n_seg, sb, se, stream_));
  const size_t tb = std::max<size_t>(std::max(t1, t2), 1);
  if (s_tmp_.bytes < tb) s_tmp_.alloc(tb);
  AB_CUDA(cub::DeviceSegmentedSort::StableSortPairs(s_tmp_.p, t1, s_key_.as<long long>(), s_key_out_.as<long long>(),
                                                    s_idx_.as<unsigned int>(), s_idx_out_.as<unsigned int>(), (int)n,
                                                    (int)n_seg, sb, se, stream_));
  big_seq_kernel<<<n_seg, ST, 0, stream_>>>(sb, se, g.a_seq, s_idx_out_.as<unsigned int>(), s_seq_.as<unsigned int>());
  AB_CUDA(cudaGetLastError());
  t2 = s_tmp_.bytes;
  AB_CUDA(cub::DeviceSegmentedSort::StableSortPairs(s_tmp_.p, t2, s_seq_.as<unsigned int>(), s_seq_out_.as<unsigned int>(),
                                                    s_idx_out_.as<unsigned int>(), s_idx_.as<unsigned int>(), (int)n,
                                                    (int)n_seg, sb, se, stream_));
  big_gather_kernel<<<n_seg, ST, 0, stream_>>>(sb, se, g, s_idx_.as<unsigned int>());
  AB_CUDA(cudaGetLastError());
  st_.kernel_launches += 5;
}

void SessionOp::flush() {
  set_device();
  apply_pending();
  AB_CUDA(cudaStreamSynchronize(stream_));
  inputs_.release(true);
}

// handle_checkpoint (session_aggregating_window.rs:907-925): table "s" (the raw input batches) is written by the
// shim as the batches arrive; what the operator contributes is its entry of the global table "e",
// `earliest_batch_time()` = the first key of `keys_by_start_time` (:162-166).  Entries of that map are never
// removed (only the key sets inside them are emptied, :125-141, :244-262), so the value is the earliest data start
// the subtask has ever held = the smallest _timestamp of any row it accepted.  Returned as a one-column batch
// [earliest_batch_time: timestamp ns] with one row, or no rows when the subtask has not seen data.
void SessionOp::handle_checkpoint(int64_t, BatchesPriv* out) {
  flush();
  long long e = LLONG_MAX;
  AB_CUDA(cudaMemcpyAsync(&e, earliest_.p, 8, cudaMemcpyDeviceToHost, stream_));
  AB_CUDA(cudaStreamSynchronize(stream_));
  const int64_t n = e == LLONG_MAX ? 0 : 1;
  OutColumn c;
  c.name = "earliest_batch_time";
  c.format = "tsn:";
  long long* h = (long long*)PinnedPool::get().alloc(8);
  h[0] = e;
  c.data = h;
  std::vector<OutColumn> cols{c};
  out->arrays.emplace_back();
  out->schemas.emplace_back();
  export_batch(cols, n, &out->arrays.back(), &out->schemas.back());
}

// on_start (session_aggregating_window.rs:802-847).  `start_time` = the minimum over the subtasks' entries of table
// "e" (INT64_MIN: none, nothing is restored); `state` = the batches of table "s" from `start_time` on.  Every batch
// is filtered to rows at or after `start_time` and added exactly like a newly arrived batch under the watermark
// `start_time` (:826-835); then the sessions the restored watermark already closes are evicted and DROPPED (:837-845:
// they were emitted before the checkpoint).
void SessionOp::on_start(ArrowArray* state, ArrowSchema* schemas, int64_t n, int64_t watermark, int64_t start_time) {
  set_device();
  if (start_time != INT64_MIN) {
    has_wm_ = true;
    wm_ = start_time;
    // the replayed rows were counted by the operator that accepted them: rows_in and rows_late count only what the
    // caller hands in, so the counters are put back after the replay (rows before start_time count as late there)
    const uint64_t rows_in = st_.rows_in;
    unsigned long long late = 0;
    AB_CUDA(cudaMemcpyAsync(&late, late_.p, 8, cudaMemcpyDeviceToHost, stream_));
    for (int64_t i = 0; i < n; ++i) {
      AggCols d;
      const int64_t rows = staging_.stage(plan_, &state[i], &schemas[i], stream_, &st_, &key_format_, &d);
      prep(d, rows);
      apply_pending();  // every stored batch is its own input batch
      AB_CUDA(cudaStreamSynchronize(stream_));
      if (state[i].release) state[i].release(&state[i]);  // taken: its rows are in the operator's pools
    }
    st_.rows_in = rows_in;
    AB_CUDA(cudaMemcpyAsync(late_.p, &late, 8, cudaMemcpyHostToDevice, stream_));
    AB_CUDA(cudaStreamSynchronize(stream_));
  } else {
    AB_REQUIRE(n == 0, ARROYO_B200_INVALID_ARGUMENT, "session restore: state batches without a start time (table 'e')");
  }
  if (watermark == INT64_MIN) {
    has_wm_ = false;  // no watermark has been seen yet: later batches are not filtered (:858-868)
    flush();
    return;
  }
  if (start_time != INT64_MIN) {
    const ArroyoB200Stats before = st_;
    std::vector<ArroyoB200DeviceBatch> evicted;
    handle_watermark(watermark, nullptr, &evicted);
    AB_CUDA(cudaStreamSynchronize(stream_));
    st_.rows_out = before.rows_out;  // evicted results are not output
    st_.windows_out = before.windows_out;
  }
  has_wm_ = true;
  wm_ = watermark;
  flush();
}

// Pools are bump allocated; when more than half of what has been handed out is dead they are rebuilt from the
// per-key lists.
void SessionOp::maybe_compact() {
  const unsigned long long* h = h_ctr_.as<unsigned long long>();
  const uint64_t nodes = h[0], rows = h[1], dead_nodes = h[2], dead_rows = h[3];
  if (nodes < compact_min_ && rows < 4 * compact_min_) return;
  if (dead_nodes * 2 < nodes && dead_rows * 2 < rows) return;
  if (c_cap_ < n_keys_) {
    c_cap_ = std::max<uint64_t>(id_cap_, n_keys_);
    c_cn_.alloc(c_cap_ * 4);
    c_cr_.alloc(c_cap_ * 4);
    c_on_.alloc(c_cap_ * 8);
    c_orow_.alloc(c_cap_ * 8);
    c_tot_.alloc(16);
  }
  DevBuf &cn = c_cn_, &cr = c_cr_, &on = c_on_, &orow = c_orow_, &tot = c_tot_;
  SessCtx c = ctx();
  live_count_kernel<<<grid_for(n_keys_, 128), 128, 0, stream_>>>(c, n_keys_, cn.as<unsigned int>(), cr.as<unsigned int>());
  AB_CUDA(cudaGetLastError());
  device_exclusive_scan(cn.as<unsigned int>(), n_keys_, on.as<unsigned long long>(), tot.as<unsigned long long>(), scan_sums_, stream_);
  device_exclusive_scan(cr.as<unsigned int>(), n_keys_, orow.as<unsigned long long>(), tot.as<unsigned long long>() + 1, scan_sums_, stream_);
  unsigned long long t[2];
  AB_CUDA(cudaMemcpyAsync(t, tot.p, 16, cudaMemcpyDeviceToHost, stream_));
  AB_CUDA(cudaStreamSynchronize(stream_));
  const uint64_t live_nodes = t[0], live_rows = t[1];
  // the spare set takes the live entries; it is at least as large as the set in use, so a compaction allocates only
  // when the live data itself has outgrown it
  const uint64_t ncap = std::max<uint64_t>(std::max<uint64_t>(2 * live_nodes + 16, 1 << 16), node_cap_);
  const uint64_t rcap = std::max<uint64_t>(std::max<uint64_t>(2 * live_rows + 16, 1 << 16), row_cap_);
  if (sp_node_cap_ < ncap) {
    sp_next_.alloc(ncap * 4);
    sp_start_.alloc(ncap * 8);
    sp_off_.alloc(ncap * 8);
    sp_len_.alloc(ncap * 4);
    sp_node_cap_ = ncap;
  }
  if (sp_row_cap_ < rcap) {
    sp_rts_.alloc(rcap * 8);
    for (int v = 0; v < plan_.n_vals; ++v) sp_rval_[v].alloc(rcap * 8);
    sp_row_cap_ = rcap;
  }
  CompactDst d{};
  d.n_next = sp_next_.as<int>();
  d.n_start = sp_start_.as<long long>();
  d.n_off = sp_off_.as<long long>();
  d.n_len = sp_len_.as<int>();
  d.r_ts = sp_rts_.as<long long>();
  for (int v = 0; v < plan_.n_vals; ++v) d.r_val[v] = sp_rval_[v].as<long long>();
  compact_copy_kernel<<<grid_for(n_keys_, 128), 128, 0, stream_>>>(c, d, n_keys_, on.as<unsigned long long>(),
                                                                  orow.as<unsigned long long>());
  AB_CUDA(cudaGetLastError());
  unsigned long long nc[4] = {live_nodes, live_rows, 0, 0};
  AB_CUDA(cudaMemcpyAsync(ctr_.p, nc, sizeof nc, cudaMemcpyHostToDevice, stream_));
  AB_CUDA(cudaStreamSynchronize(stream_));
  std::swap(n_next_, sp_next_);
  std::swap(n_start_, sp_start_);
  std::swap(n_off_, sp_off_);
  std::swap(n_len_, sp_len_);
  std::swap(r_ts_, sp_rts_);
  for (int v = 0; v < plan_.n_vals; ++v) std::swap(r_val_[v], sp_rval_[v]);
  std::swap(node_cap_, sp_node_cap_);
  std::swap(row_cap_, sp_row_cap_);
  st_.kernel_launches += 8;
}

void SessionOp::handle_watermark(int64_t wm, BatchesPriv* out_host, std::vector<ArroyoB200DeviceBatch>* out_dev) {
  set_device();
  apply_pending();  // rows that arrived under the previous watermark
  // every session that can close: one per open session plus one per pending run at most
  read_ctr();
  const unsigned long long* h = h_ctr_.as<unsigned long long>();
  // every closed session holds at least one row: open sessions + pending rows bound the output, and every
  // remainder run created while filling consumes at least one pending row
  const uint64_t live_rows = h[1] - h[3];
  const uint64_t bound = h[7] + live_rows + 16;
  if (bound > out_cap_) {
    out_cap_ = std::max<uint64_t>(bound, out_cap_ * 2);
    o_key_.alloc(out_cap_ * 8);
    o_start_.alloc(out_cap_ * 8);
    o_end_.alloc(out_cap_ * 8);
    o_ts_.alloc(out_cap_ * 8);
    for (int g = 0; g < plan_.n_aggs; ++g) o_agg_[g].alloc(out_cap_ * 8);
  }
  ensure_pools(live_rows + 16, 0);  // remainders created while filling
  unsigned long long zero = 0;
  AB_CUDA(cudaMemcpyAsync(ctr_.as<unsigned long long>() + 4, &zero, 8, cudaMemcpyHostToDevice, stream_));
  AdvanceParams a{};
  a.c = ctx();
  a.n_ids = n_keys_;
  a.wm = wm;
  advance_kernel<<<grid_for(n_keys_, 128), 128, 0, stream_>>>(a);
  AB_CUDA(cudaGetLastError());
  ++st_.kernel_launches;
  ++st_.emit_launches;
  read_ctr();
  check_err();
  has_wm_ = true;
  wm_ = wm;
  const int64_t n = (int64_t)h_ctr_.as<unsigned long long>()[4];
  {
    unsigned long long late = 0;
    AB_CUDA(cudaMemcpyAsync(&late, late_.p, 8, cudaMemcpyDeviceToHost, stream_));
    AB_CUDA(cudaStreamSynchronize(stream_));
    st_.rows_late = late;
  }
  inputs_.release(false);
  if (n > 0) {
    st_.rows_out += (uint64_t)n;
    ++st_.windows_out;
    if (out_host) {
      // [key cols...] with the window struct inserted at window_index, [agg cols...], _timestamp
      // (session_aggregating_window.rs:316-382)
      const int wi = std::min<int>(std::max<int>(cfg.window_index, 0), plan_.keyed ? 1 : 0);
      export_window_batch(out_host, n, stream_, &st_.d2h_bytes, plan_.keyed ? o_key_.p : nullptr, key_format_, o_agg_,
                          plan_.agg_format, o_start_.p, o_end_.p, wi, o_ts_.p);
      AB_CUDA(cudaStreamSynchronize(stream_));
    } else {
      ArroyoB200DeviceBatch d{};
      d.n_rows = n;
      std::vector<uint64_t> cols;
      if (plan_.keyed) cols.push_back((uint64_t)o_key_.p);
      const int wi = std::min<int>(std::max<int>(cfg.window_index, 0), (int)cols.size());
      cols.insert(cols.begin() + wi, (uint64_t)o_end_.p);
      cols.insert(cols.begin() + wi, (uint64_t)o_start_.p);
      for (int g = 0; g < plan_.n_aggs; ++g) cols.push_back((uint64_t)o_agg_[g].p);
      cols.push_back((uint64_t)o_ts_.p);
      int c = 0;
      for (uint64_t v : cols) d.cols[c++] = v;
      d.n_cols = c;
      out_dev->push_back(d);
    }
  }
  maybe_compact();
}

}  // namespace

OpBase* make_session_op(const ArroyoB200OpConfig& cfg) { return new SessionOp(cfg); }

}  // namespace ab
