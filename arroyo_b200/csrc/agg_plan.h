// The aggregate plan of the window, session and updating aggregates: which input columns the operator reads, which
// accumulators it keeps per key and how each aggregate is computed from them.
//
// Accumulators are 64-bit words in a per-key SoA block.  Accumulator 0 counts rows; every other one folds one value
// column with one kind, and aggregates of the same (kind, column) share it.
#pragma once

#include <climits>
#include <string>
#include <vector>

#include "common.cuh"

namespace ab {

constexpr int MAX_VALS = 4;                        // distinct value columns
constexpr int MAX_ACC = ARROYO_B200_MAX_AGGS + 1;  // accumulators, the row count included

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
  int key_col = 0, ts_col = 0;
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
};

}  // namespace ab
