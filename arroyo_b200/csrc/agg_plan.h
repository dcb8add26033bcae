// The aggregate plan of the window, session and updating aggregates: which input columns the operator reads, which
// accumulators it keeps per key and how each aggregate is computed from them.
//
// Accumulators are 64-bit words in a per-key SoA block.  Accumulator 0 counts rows; every other one folds one value
// column with one kind, and aggregates of the same (kind, column) share it.  What each kind does on the device (its
// identity, the accumulator form of an input value, sequential and global merge, unmerge, AVG) is defined here and
// nowhere else.
#pragma once

#include <climits>
#include <string>
#include <type_traits>
#include <vector>

#include "arrow_io.h"
#include "common.cuh"

namespace ab {

constexpr int MAX_VALS = 4;                        // distinct value columns
constexpr int MAX_ACC = ARROYO_B200_MAX_AGGS + 1;  // accumulators, the row count included

// The columns an aggregate reads from one batch: the key (null when unkeyed), the timestamp and one per value slot.
struct AggCols {
  const long long* key = nullptr;
  const long long* ts = nullptr;
  const long long* val[MAX_VALS] = {};
};

enum AccKind : int { ACC_ROWS = 0, ACC_SUM_I64 = 1, ACC_SUM_F64 = 2, ACC_MIN_I64 = 3, ACC_MAX_I64 = 4 };

// What an accumulator of `kind` holds before its first row.
__host__ __device__ __forceinline__ unsigned long long acc_identity(int kind) {
  unsigned long long v = 0;
  if (kind == ACC_MIN_I64) v = (unsigned long long)LLONG_MAX;
  if (kind == ACC_MAX_I64) v = (unsigned long long)LLONG_MIN;
  return v;
}

// The accumulator-domain form of an Int64 input value `x` for an accumulator of `kind`: the bits of (double)x for
// ACC_SUM_F64, x itself for every other kind.
__device__ __forceinline__ unsigned long long acc_of_value(int kind, long long x) {
  return kind == ACC_SUM_F64 ? (unsigned long long)__double_as_longlong((double)x) : (unsigned long long)x;
}

// What folding `b` into `a` gives for an accumulator of `kind` (ACC_ROWS and ACC_SUM_I64 add, wrapping).
__device__ __forceinline__ unsigned long long acc_merge(int kind, unsigned long long a, unsigned long long b) {
  switch (kind) {
    case ACC_SUM_F64:
      return (unsigned long long)__double_as_longlong(__longlong_as_double((long long)a) + __longlong_as_double((long long)b));
    case ACC_MIN_I64: return (unsigned long long)min((long long)a, (long long)b);
    case ACC_MAX_I64: return (unsigned long long)max((long long)a, (long long)b);
    default: return a + b;
  }
}

// f(k) with `kind` as the compile-time constant k (std::integral_constant), which the functions above take as a kind:
// a loop over many values in f then folds with that kind's code alone instead of branching on the kind per value.
// ACC_ROWS is passed as ACC_SUM_I64, which folds the same way.
template <class F>
__device__ __forceinline__ auto acc_with_kind(int kind, F f) {
  switch (kind) {
    case ACC_SUM_F64: return f(std::integral_constant<int, ACC_SUM_F64>{});
    case ACC_MIN_I64: return f(std::integral_constant<int, ACC_MIN_I64>{});
    case ACC_MAX_I64: return f(std::integral_constant<int, ACC_MAX_I64>{});
    default: return f(std::integral_constant<int, ACC_SUM_I64>{});
  }
}

// What taking `b` back out of `a` gives: the inverse of acc_merge.  Defined only for the invertible kinds ACC_ROWS,
// ACC_SUM_I64 (exact, wrapping) and ACC_SUM_F64 (up to rounding); MIN and MAX cannot be unmerged.
__device__ __forceinline__ unsigned long long acc_unmerge(int kind, unsigned long long a, unsigned long long b) {
  if (kind == ACC_SUM_F64)
    return (unsigned long long)__double_as_longlong(__longlong_as_double((long long)a) - __longlong_as_double((long long)b));
  return a - b;
}

// Fire-and-forget global reductions (RED: no value comes back).  On a pointer loaded from memory, as accumulator
// blocks often are, the compiler only knows a generic address, and atomicAdd and friends compile to a generic ATOM
// with a shared-memory fallback; the explicit global address space makes every merge a RED.
__device__ __forceinline__ void red_add_u64(unsigned long long* dst, unsigned long long v) {
  asm volatile("red.global.add.u64 [%0], %1;" ::"l"(__cvta_generic_to_global(dst)), "l"(v) : "memory");
}

// acc_merge of `v`, already in the accumulator's domain, into the accumulator `*dst` in global memory, as one RED.
__device__ __forceinline__ void acc_red(int kind, unsigned long long* dst, unsigned long long v) {
  switch (kind) {
    case ACC_SUM_F64:
      asm volatile("red.global.add.f64 [%0], %1;" ::"l"(__cvta_generic_to_global(dst)),
                   "d"(__longlong_as_double((long long)v)) : "memory");
      break;
    case ACC_MIN_I64:
      asm volatile("red.global.min.s64 [%0], %1;" ::"l"(__cvta_generic_to_global(dst)), "l"((long long)v) : "memory");
      break;
    case ACC_MAX_I64:
      asm volatile("red.global.max.s64 [%0], %1;" ::"l"(__cvta_generic_to_global(dst)), "l"((long long)v) : "memory");
      break;
    default: red_add_u64(dst, v); break;
  }
}

// Two SoA accumulator blocks of `cap` ids each.  After a checkpoint has written `delta`, ids [0, n) fold it into
// `base` and start it over from the identities, so that the next checkpoint writes only the rows that arrive later.
struct FoldParams {
  unsigned long long* base;
  unsigned long long* delta;
  unsigned long long cap;
  uint32_t n;
  int n_acc;
  int acc_kind[MAX_ACC];
};
static __global__ void acc_fold_kernel(const __grid_constant__ FoldParams p) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  const uint32_t stride = gridDim.x * blockDim.x;
  for (; i < p.n; i += stride) {
    for (int a = 0; a < p.n_acc; ++a) {
      const unsigned long long off = (unsigned long long)a * p.cap + i;
      p.base[off] = acc_merge(p.acc_kind[a], p.base[off], p.delta[off]);
      p.delta[off] = acc_identity(p.acc_kind[a]);
    }
  }
}

// The f64 bits of AVG over `rows` rows from the sum accumulator `acc` of `kind`: the f64 sum (ACC_SUM_F64, DataFusion's
// AVG state) or the exact integer sum converted once (ACC_SUM_I64), over the rows.
__device__ __forceinline__ unsigned long long acc_mean(int kind, unsigned long long acc, unsigned long long rows) {
  const double num = kind == ACC_SUM_F64 ? __longlong_as_double((long long)acc) : (double)(long long)acc;
  return (unsigned long long)__double_as_longlong(num / (double)rows);
}

// Output value of an aggregate of `agg_kind` (ARROYO_B200_AGG_*) whose accumulator holds `acc`, in a plan whose AVG
// accumulators are ACC_SUM_F64: COUNT(*) is the row count, AVG acc_mean, anything else the accumulator itself.
__device__ __forceinline__ unsigned long long agg_finalise(int agg_kind, unsigned long long acc, unsigned long long rows) {
  if (agg_kind == ARROYO_B200_AGG_COUNT_STAR) return rows;
  if (agg_kind == ARROYO_B200_AGG_AVG_I64) return acc_mean(ACC_SUM_F64, acc, rows);
  return acc;
}

// One column of a checkpoint table after the key.
enum StateRole { S_ROWS, S_ACC, S_TS, S_GEN };
struct StateCol {
  std::string name;    // agg<g>[<field>], _timestamp or _generation
  const char* format;  // Arrow format ("tsn:": any timestamp[ns])
  int role;            // S_ROWS: the key's row count; S_ACC: accumulator `acc`
  int acc;             // 0 for every role but S_ACC
  bool count_star;     // the COUNT(*) aggregate's own row count
};

struct AggPlan {
  bool keyed = false;
  int n_cols = 0, key_col = 0, ts_col = 0;
  int n_vals = 0, val_cols[MAX_VALS];  // value slot -> input column
  int n_acc = 1, acc_kind[MAX_ACC] = {ACC_ROWS}, acc_val[MAX_ACC] = {0};
  int n_aggs = 0, agg_kind[ARROYO_B200_MAX_AGGS], agg_acc[ARROYO_B200_MAX_AGGS];
  std::vector<std::string> agg_format;  // Arrow format of each aggregate's output column

  AggPlan() = default;

  // Validates the column layout and the aggregates of `c`.  `avg_kind`: the accumulator an AVG folds its column
  // into, ACC_SUM_F64 (the sequential f64 sum, like the reference's accumulator) or ACC_SUM_I64 (the window's exact
  // integer sum, finalised as (double)sum / count).
  AggPlan(const ArroyoB200OpConfig& c, int avg_kind) {
    AB_REQUIRE(c.n_key_cols == 0 || c.n_key_cols == 1, ARROYO_B200_UNSUPPORTED,
               "only 0 or 1 group-by key columns are supported");
    keyed = c.n_key_cols == 1;
    n_cols = c.n_cols;
    key_col = c.key_col;
    ts_col = c.timestamp_col;
    AB_REQUIRE(c.n_cols >= 1 && c.n_cols <= ARROYO_B200_MAX_COLS, ARROYO_B200_INVALID_ARGUMENT, "bad n_cols");
    AB_REQUIRE(ts_col >= 0 && ts_col < c.n_cols, ARROYO_B200_INVALID_ARGUMENT, "bad timestamp_col");
    AB_REQUIRE(!keyed || (key_col >= 0 && key_col < c.n_cols), ARROYO_B200_INVALID_ARGUMENT, "bad key_col");
    AB_REQUIRE(c.n_aggs >= 1 && c.n_aggs <= ARROYO_B200_MAX_AGGS, ARROYO_B200_INVALID_ARGUMENT, "bad n_aggs");
    n_aggs = c.n_aggs;
    for (int g = 0; g < n_aggs; ++g) {
      const int kind = c.aggs[g].kind;
      agg_kind[g] = kind;
      agg_acc[g] = 0;
      if (kind == ARROYO_B200_AGG_COUNT_STAR) {
        agg_format.push_back("l");
        continue;
      }
      const int col = c.aggs[g].input_col;
      AB_REQUIRE(col >= 0 && col < c.n_cols, ARROYO_B200_INVALID_ARGUMENT, "aggregate input column out of range");
      const int vs = value_slot(col);
      int ak;
      switch (kind) {
        case ARROYO_B200_AGG_SUM_I64: ak = ACC_SUM_I64; agg_format.push_back("l"); break;
        case ARROYO_B200_AGG_AVG_I64: ak = avg_kind; agg_format.push_back("g"); break;
        case ARROYO_B200_AGG_MIN_I64: ak = ACC_MIN_I64; agg_format.push_back("l"); break;
        case ARROYO_B200_AGG_MAX_I64: ak = ACC_MAX_I64; agg_format.push_back("l"); break;
        default: throw Error(ARROYO_B200_UNSUPPORTED, "unsupported aggregate kind");
      }
      // share accumulators between identical (kind, column) pairs
      int found = -1;
      for (int a = 1; a < n_acc; ++a)
        if (acc_kind[a] == ak && acc_val[a] == vs) found = a;
      if (found < 0) {
        found = n_acc;
        acc_kind[n_acc] = ak;
        acc_val[n_acc] = vs;
        ++n_acc;
      }
      agg_acc[g] = found;
    }
  }

  // The value slot that carries input column `col`, taking the next free one on first use.
  int value_slot(int col) {
    for (int v = 0; v < n_vals; ++v)
      if (val_cols[v] == col) return v;
    AB_REQUIRE(n_vals < MAX_VALS, ARROYO_B200_UNSUPPORTED, "more than 4 distinct aggregate input columns");
    val_cols[n_vals] = col;
    return n_vals++;
  }

  // The columns of a batch handed over as one device pointer per input column.
  AggCols columns(const uint64_t* cols, int32_t n) const {
    AB_REQUIRE(n == n_cols, ARROYO_B200_INVALID_ARGUMENT, "batch has the wrong number of columns");
    AggCols d;
    if (keyed) d.key = (const long long*)cols[key_col];
    d.ts = (const long long*)cols[ts_col];
    for (int v = 0; v < n_vals; ++v) d.val[v] = (const long long*)cols[val_cols[v]];
    return d;
  }

  // The columns of a checkpoint table after the key, per aggregate in plan order, then `_timestamp`.
  //  - Table "t" of the window and instant aggregates (`partial_schema`, arroyo-planner builder.rs:163-192):
  //    COUNT(*) -> [count] Int64; SUM -> [sum] Int64; AVG -> [count] UInt64, [sum] Float64; MIN / MAX -> [min] /
  //    [max] Int64; `_timestamp` is the pane start or the instant.
  //  - Table "a" of the updating aggregate (`sliding_state_schema`, incremental_aggregator.rs:1083-1160): the same,
  //    but SUM -> [sum] Int64, [count] UInt64; `_timestamp` is max(_timestamp), then `_generation` UInt64.
  // Every count column holds the key's row count.
  std::vector<StateCol> state_layout(bool table_a) const {
    std::vector<StateCol> l;
    for (int g = 0; g < n_aggs; ++g) {
      const std::string p = "agg" + std::to_string(g);
      const int acc = agg_acc[g];
      switch (agg_kind[g]) {
        case ARROYO_B200_AGG_COUNT_STAR: l.push_back({p + "[count]", "l", S_ROWS, 0, true}); break;
        case ARROYO_B200_AGG_SUM_I64:
          l.push_back({p + "[sum]", "l", S_ACC, acc, false});
          if (table_a) l.push_back({p + "[count]", "L", S_ROWS, 0, false});
          break;
        case ARROYO_B200_AGG_AVG_I64:
          l.push_back({p + "[count]", "L", S_ROWS, 0, false});
          l.push_back({p + "[sum]", "g", S_ACC, acc, false});
          break;
        case ARROYO_B200_AGG_MIN_I64: l.push_back({p + "[min]", "l", S_ACC, acc, false}); break;
        case ARROYO_B200_AGG_MAX_I64: l.push_back({p + "[max]", "l", S_ACC, acc, false}); break;
      }
    }
    l.push_back({"_timestamp", "tsn:", S_TS, 0, false});
    if (table_a) l.push_back({"_generation", "L", S_GEN, 0, false});
    return l;
  }
};

// The batches of one checkpoint table handed to on_start, imported and checked against the plan's layout: a column
// count, key type or column type that is not the layout's is refused (INVALID_ARGUMENT) before the caller has changed
// anything.  Table "a" may hold nulls in `_timestamp` (tombstones).  The caller takes the batches (take_batches) only
// once its restore has succeeded.
struct StateBatches {
  std::vector<StateCol> layout;
  int kc = 0;                               // key columns: the layout's columns start at kc
  int ts_col = 0;                           // `_timestamp` (table "a": `_generation` follows it)
  std::vector<std::vector<InColumn>> cols;  // per batch
  std::vector<int64_t> rows;                // per batch
  int64_t total = 0;
  // The column each accumulator is restored from; -1: none, which only the row count can lack (each row then counts
  // one).  The row count comes from COUNT(*)'s column, else the first count column; an accumulator from its first
  // column, but an Int64 one before a Float64 one: an exact-sum AVG shares its integer accumulator with a SUM over the
  // same column, and the window aggregate keeps that sharing on restore only where the two columns agree.
  int seed[MAX_ACC];
  bool table_a = false;

  StateBatches(const AggPlan& plan, bool table_a_, const ArrowArray* state, const ArrowSchema* schemas, int64_t n)
      : layout(plan.state_layout(table_a_)), kc(plan.keyed ? 1 : 0), table_a(table_a_) {
    if (n > 0) AB_REQUIRE(state != nullptr && schemas != nullptr, ARROYO_B200_INVALID_ARGUMENT, "null state batches");
    ts_col = kc + (int)layout.size() - (table_a ? 2 : 1);
    cols.resize((size_t)std::max<int64_t>(n, 0));
    rows.assign(cols.size(), 0);
    for (size_t b = 0; b < cols.size(); ++b) {
      try {
        cols[b] = import_batch(&state[b], &schemas[b], &rows[b], table_a ? ts_col : -1);
      } catch (const Error& e) {
        throw Error(ARROYO_B200_INVALID_ARGUMENT, std::string("state batch: ") + e.what());
      }
      const std::vector<InColumn>& c = cols[b];
      AB_REQUIRE(c.size() == (size_t)kc + layout.size(), ARROYO_B200_INVALID_ARGUMENT,
                 "state batch has " + std::to_string(c.size()) + " columns, the plan's layout " +
                     std::to_string(kc + layout.size()));
      if (kc) {
        const std::string& f = c[0].format;
        AB_REQUIRE(f == "l" || f == "L" || f.compare(0, 4, "tsn:") == 0, ARROYO_B200_INVALID_ARGUMENT,
                   "state batch: key of type '" + f + "' (supported: l, L, tsn:)");
      }
      for (size_t j = 0; j < layout.size(); ++j) {
        const std::string& f = c[kc + j].format;
        const std::string want = layout[j].format;
        AB_REQUIRE(want == "tsn:" ? f.compare(0, 4, "tsn:") == 0 : f == want, ARROYO_B200_INVALID_ARGUMENT,
                   "state batch: column " + std::to_string(kc + j) + " has type '" + f + "', the layout '" + want + "'");
      }
      total += rows[b];
    }
    assign_seeds(plan);
  }

  // Fills `seed` for `plan`, which has the layout the batches were checked against: a plan that changed only which
  // accumulator an aggregate reads (the window aggregate's AVG promotion) restores from the same columns.
  void assign_seeds(const AggPlan& plan) {
    layout = plan.state_layout(table_a);
    for (int a = 0; a < MAX_ACC; ++a) seed[a] = -1;
    for (size_t j = 0; j < layout.size(); ++j) {
      const StateCol& sc = layout[j];
      const int c = kc + (int)j;
      if (sc.role == S_ROWS && (seed[0] < 0 || (sc.count_star && !layout[seed[0] - kc].count_star))) seed[0] = c;
      if (sc.role == S_ACC &&
          (seed[sc.acc] < 0 || (!strcmp(layout[seed[sc.acc] - kc].format, "g") && strcmp(sc.format, "g"))))
        seed[sc.acc] = c;
    }
  }

  // Column `c` of batches [b0, b1), concatenated in batch order into `dst` (a row's position is its index there),
  // copied on `s`; the copies count in `*h2d_bytes`.  The batches must outlive the copies.
  const unsigned long long* upload(int c, int64_t b0, int64_t b1, DevBuf& dst, cudaStream_t s,
                                   uint64_t* h2d_bytes) const {
    int64_t n = 0;
    for (int64_t b = b0; b < b1; ++b) n += rows[b];
    dst.alloc((size_t)n * 8);
    int64_t off = 0;
    for (int64_t b = b0; b < b1; ++b) {
      if (rows[b])
        AB_CUDA(cudaMemcpyAsync((char*)dst.p + off * 8, cols[b][c].data, (size_t)rows[b] * 8, cudaMemcpyHostToDevice, s));
      off += rows[b];
    }
    *h2d_bytes += (uint64_t)n * 8;
    return dst.as<unsigned long long>();
  }
};

// Takes the `n` state batches of a restore that succeeded.
inline void take_batches(ArrowArray* state, int64_t n) {
  for (int64_t b = 0; b < n; ++b)
    if (state[b].release) state[b].release(&state[b]);
}

// The columns of a checkpoint table's batch of `n` rows in `layout`, copied on `s` into pinned buffers (the copies
// count in `*d2h_bytes`): the key (`key` null: unkeyed), then the layout's columns from `acc` (one device column per
// accumulator, acc[0] the row count) and `ts`.  `_generation` is left to the caller.  Nothing may read the columns
// before `s` has passed the copies.
inline std::vector<OutColumn> state_columns(const std::vector<StateCol>& layout, int64_t n, const void* key,
                                            const std::string& key_format, const DevBuf* acc, const void* ts,
                                            cudaStream_t s, uint64_t* d2h_bytes) {
  std::vector<OutColumn> cols;
  auto column = [&](const std::string& name, const std::string& format, const void* dev) {
    OutColumn c;
    c.name = name;
    c.format = format;
    c.data = d2h_pinned(dev, (size_t)n * 8, s, d2h_bytes);
    cols.push_back(c);
  };
  if (key) column("key", key_format, key);
  for (const StateCol& sc : layout)
    if (sc.role != S_GEN) column(sc.name, sc.format, sc.role == S_TS ? ts : acc[sc.acc].p);
  return cols;
}

// The device copies of the columns an aggregate reads from its host batches, in one buffer reused in stream order.
struct AggStaging {
  DevBuf buf;
  uint64_t cap = 0;  // rows per column

  // Imports `batch`, checks it against `plan`, records its key's format in `*key_format` and counts its rows in
  // `st->rows_in`.  A batch with rows is then copied on `s` (the copies count in `st->h2d_bytes`) and `*dev` gets
  // the device columns.  Returns the row count.  The host batch must outlive the copies: the caller keeps it until
  // `s` has passed them.
  int64_t stage(const AggPlan& plan, ArrowArray* batch, const ArrowSchema* schema, cudaStream_t s,
                ArroyoB200Stats* st, std::string* key_format, AggCols* dev) {
    int64_t n = 0;
    const std::vector<InColumn> cols = import_batch(batch, schema, &n);
    AB_REQUIRE((int)cols.size() == plan.n_cols, ARROYO_B200_INVALID_ARGUMENT, "batch has the wrong number of columns");
    require_aggregate_input_types(cols, plan.keyed ? plan.key_col : -1, plan.val_cols, plan.n_vals);
    if (plan.keyed) *key_format = cols[plan.key_col].format;
    st->rows_in += (uint64_t)n;
    if (n == 0) return 0;
    if ((uint64_t)n > cap) {
      AB_CUDA(cudaStreamSynchronize(s));
      cap = std::max<uint64_t>((uint64_t)n, cap * 2);
      buf.alloc((size_t)(2 + plan.n_vals) * cap * 8);
    }
    long long* base = buf.as<long long>();
    auto copy = [&](int slot, int col) {
      long long* d = base + (size_t)slot * cap;
      AB_CUDA(cudaMemcpyAsync(d, cols[col].data, (size_t)n * 8, cudaMemcpyHostToDevice, s));
      return d;
    };
    if (plan.keyed) dev->key = copy(0, plan.key_col);
    dev->ts = copy(1, plan.ts_col);
    for (int v = 0; v < plan.n_vals; ++v) dev->val[v] = copy(2 + v, plan.val_cols[v]);
    st->h2d_bytes += (uint64_t)n * 8 * (uint64_t)((plan.keyed ? 1 : 0) + 1 + plan.n_vals);
    return n;
  }
};

}  // namespace ab
