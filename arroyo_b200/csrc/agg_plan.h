// The aggregate plan of the window, session and updating aggregates: which input columns the operator reads, which
// accumulators it keeps per key and how each aggregate is computed from them.
//
// Accumulators are 64-bit words in a per-key SoA block.  Accumulator 0 counts rows; every other one folds one value
// column with one kind, and aggregates of the same (kind, column) share it.
#pragma once

#include <climits>
#include <string>
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

// Output value of an aggregate of `agg_kind` (ARROYO_B200_AGG_*) whose accumulator holds `acc`: COUNT(*) is the row
// count, AVG the f64 sum over the rows, anything else the accumulator itself.
__device__ __forceinline__ unsigned long long agg_finalise(int agg_kind, unsigned long long acc, unsigned long long rows) {
  if (agg_kind == ARROYO_B200_AGG_COUNT_STAR) return rows;
  if (agg_kind == ARROYO_B200_AGG_AVG_I64)
    return (unsigned long long)__double_as_longlong(__longlong_as_double((long long)acc) / (double)rows);
  return acc;
}

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
};

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
