/*
 * arroyo_b200.h -- C ABI of libarroyo_b200.so: H100-native (sm_90a) window-assign /
 * keyed-aggregate / windowed-join operators behind Arroyo's ArrowOperator surface.
 *
 * This is the drop-in boundary (SURVEY.md 8(b)).  Every entry point cites the reference
 * interface it replaces; paths are relative to /root/reference/crates.  The reference side
 * binding (a Rust `extern "C"` block + a `GpuWindowConstructor` registered in
 * `construct_operator`, arroyo-worker/src/engine.rs:900-936) is shown in INTEGRATION.md.
 *
 * Conventions
 *  - plain C types only; batches cross the boundary as Arrow C Data Interface structs --
 *    the mechanism the reference already uses for UDF dylibs
 *    (arroyo-udf/arroyo-udf-common/src/lib.rs:12-69, arroyo-udf-host/src/lib.rs:96-99).
 *  - every call returns an int32 status: 0 = ok, >0 = error (see ArroyoB200Status);
 *    the message is available from arroyo_b200_op_last_error().  Nothing unwinds across the
 *    ABI.  The shim maps errors to DataflowError::InternalOperatorError
 *    (arroyo-rpc/src/errors.rs:45-60); ARROYO_B200_FATAL means the CUDA context is gone and
 *    the task must restart from its checkpoint.
 *  - a handle is thread-compatible, not thread-safe: `ArrowOperator: Send` and every trait
 *    method takes `&mut self` (arroyo-operator/src/operator.rs:1143-1144), so calls never
 *    overlap but may come from different OS threads; the library never relies on the
 *    thread's current CUDA device.
 *  - event time is int64 nanoseconds since the Unix epoch (arroyo-types/src/lib.rs:123-131).
 *    The end-of-data watermark `u64::MAX` ns (watermark_generator.rs:137-146) is passed as
 *    INT64_MAX.
 *  - there is NO CPU fallback: without a usable CUDA device op_create fails.
 */
#ifndef ARROYO_B200_H
#define ARROYO_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ---- Arrow C Data Interface (https://arrow.apache.org/docs/format/CDataInterface.html) ---- */
#ifndef ARROW_C_DATA_INTERFACE
#define ARROW_C_DATA_INTERFACE

#define ARROW_FLAG_DICTIONARY_ORDERED 1
#define ARROW_FLAG_NULLABLE 2
#define ARROW_FLAG_MAP_KEYS_SORTED 4

struct ArrowSchema {
  const char* format;
  const char* name;
  const char* metadata;
  int64_t flags;
  int64_t n_children;
  struct ArrowSchema** children;
  struct ArrowSchema* dictionary;
  void (*release)(struct ArrowSchema*);
  void* private_data;
};

struct ArrowArray {
  int64_t length;
  int64_t null_count;
  int64_t offset;
  int64_t n_buffers;
  int64_t n_children;
  const void** buffers;
  struct ArrowArray** children;
  struct ArrowArray* dictionary;
  void (*release)(struct ArrowArray*);
  void* private_data;
};
#endif /* ARROW_C_DATA_INTERFACE */

/* ---- status codes ---- */
typedef enum ArroyoB200Status {
  ARROYO_B200_OK = 0,
  ARROYO_B200_INVALID_ARGUMENT = 1, /* bad config / schema / null pointer            */
  ARROYO_B200_UNSUPPORTED = 2,      /* plan outside the supported subset: the shim   */
                                    /* must fall through to the stock CPU operator   */
  ARROYO_B200_RUNTIME = 3,          /* recoverable runtime error                     */
  ARROYO_B200_FATAL = 4,            /* sticky CUDA error; restart from checkpoint    */
  ARROYO_B200_PANIC = 5             /* a condition on which the reference panics     */
                                    /* (e.g. instant_join.rs:129-139)                */
} ArroyoB200Status;

/* ---- operator configuration ----
 * Derived by the shim from the protobuf operator configs
 * TumblingWindowAggregateOperator / SlidingWindowAggregateOperator /
 * SessionWindowAggregateOperator / JoinOperator (arroyo-rpc/proto/api.proto:39-80) after
 * pattern-matching the decoded DataFusion plans onto the supported subset. */
typedef enum ArroyoB200OpKind {
  ARROYO_B200_TUMBLING_AGGREGATE = 1, /* OperatorName::TumblingWindowAggregate */
  ARROYO_B200_SLIDING_AGGREGATE = 2,  /* OperatorName::SlidingWindowAggregate  */
  ARROYO_B200_SESSION_AGGREGATE = 3,  /* OperatorName::SessionWindowAggregate  */
  ARROYO_B200_INSTANT_JOIN = 4,       /* OperatorName::InstantJoin             */
  ARROYO_B200_UPDATING_AGGREGATE = 5, /* OperatorName::UpdatingAggregate: IncrementalAggregatingFunc,
                                       * arroyo-worker/src/arrow/incremental_aggregator.rs (append-only inputs;
                                       * COUNT(*) / SUM / AVG / MIN / MAX over Int64; emits on ticks, checkpoints and
                                       * end of data: rows [key?, aggregates..., _timestamp, is_retract bool])      */
  ARROYO_B200_TTL_JOIN = 6,           /* OperatorName::Join: JoinWithExpiration, arroyo-worker/src/arrow/
                                       * join_with_expiration.rs (inner joins of append-only inputs; same column fields as
                                       * INSTANT_JOIN; matches leave from arroyo_b200_op_process_batch_emit).  The shim
                                       * writes the key-time tables "left" / "right" from the input batches; a restart
                                       * hands them back through arroyo_b200_op_restore_side                           */
  ARROYO_B200_INSTANT_AGGREGATE = 7,  /* OperatorName::TumblingWindowAggregate with width_micros == 0: the instant window
                                       * the planner puts after an upstream window (extension/aggregate.rs:233-289).  The
                                       * bin is _timestamp itself; at watermark w every instant < w leaves in ascending
                                       * order.  Output [key?, aggregates..., _timestamp = instant], or with
                                       * final_projection the window{start = ts - (width_ns - 1), end = ts + 1} struct
                                       * inserted at window_index.  Checkpoints write table "t" (partial_schema, one
                                       * batch per instant, the rows since the previous checkpoint).  Host output only:
                                       * handle_watermark_device* => ARROYO_B200_UNSUPPORTED                           */
  ARROYO_B200_WINDOW_FUNCTION = 8     /* OperatorName::WindowFunction: WindowFunctionOperator, arroyo-worker/src/arrow/
                                       * window_fn.rs -- ROW_NUMBER / RANK / DENSE_RANK () OVER (PARTITION BY window
                                       * [, key] ORDER BY ...), optionally fused with the filter `fn <= N` after it,
                                       * COUNT(*) / SUM / AVG / MIN / MAX (x) OVER (PARTITION BY window [, key]
                                       * [ORDER BY ...]) with the default frame, LAG / LEAD / FIRST_VALUE / LAST_VALUE /
                                       * NTH_VALUE (x, ...) and PERCENT_RANK / CUME_DIST () OVER (PARTITION BY window
                                       * [, key] [ORDER BY ...]).
                                       * Config:
                                       *  - window_fn: ArroyoB200WindowFn; anything else => INVALID_ARGUMENT;
                                       *  - n_key_cols / key_col: the PARTITION BY column besides the window (the planner
                                       *    drops `window`, each upstream window stamping its rows with one _timestamp,
                                       *    plan/window_fn.rs:101-105): 0 or 1, of type l, L or tsn:; 2 or more =>
                                       *    UNSUPPORTED;
                                       *  - n_aggs / aggs[] of a ranking function: the ORDER BY list, 1 to 4 entries
                                       *    {ARROYO_B200_ORDER_ASC | _DESC, input_col} of type l, L or tsn: (a g column =>
                                       *    UNSUPPORTED, as DataFusion's float ordering and peers are not pinned here); 0
                                       *    or more than 4 entries, or another kind code => INVALID_ARGUMENT;
                                       *  - n_aggs / aggs[] of ARROYO_B200_FN_AGGREGATE: aggs[0] = {kind, input_col}, kind
                                       *    one of ARROYO_B200_AGG_COUNT_STAR, _SUM_I64, _AVG_I64, _MIN_I64, _MAX_I64
                                       *    (input_col ignored for COUNT; its column of another type than l =>
                                       *    UNSUPPORTED), then 0 to 4 ORDER BY entries as above; n_aggs 0 or more than 5,
                                       *    or another kind code => INVALID_ARGUMENT.  The frame is DataFusion's default:
                                       *    without ORDER BY the whole segment (instant, key), with ORDER BY `RANGE
                                       *    BETWEEN UNBOUNDED PRECEDING AND CURRENT ROW`, from the segment start through
                                       *    the row's last peer (peers tie on every ORDER BY key).  count / sum (wrapping)
                                       *    / min / max give Int64 (l); avg gives Float64 (g): the f64 sum of the values
                                       *    over the frame's row count;
                                       *  - n_aggs / aggs[] of a value function (FN_LAG .. FN_NTH_VALUE): aggs[0] =
                                       *    {ARROYO_B200_FN_ARGUMENT, x}, x any flat column of type l, L, g or tsn: (a
                                       *    window struct child included; another type => UNSUPPORTED), then 0 to 4
                                       *    ORDER BY entries as above; aggs[0] of another kind, or n_aggs 0 or more than
                                       *    5 => INVALID_ARGUMENT.  PERCENT_RANK / CUME_DIST: aggs[] is the ORDER BY list,
                                       *    0 to 4 entries.  For a row j of a segment (instant, key) spanning sorted rows
                                       *    [s, e], with f = the last row of j's peer group (the default frame's end; e
                                       *    without ORDER BY, where every row of the segment is a peer):
                                       *      LAG(x, k, d)    x at j - k if j - k >= s, else d        x's type, nullable
                                       *      LEAD(x, k, d)   x at j + k if j + k <= e, else d        x's type, nullable
                                       *      FIRST_VALUE(x)  x at s                                  x's type
                                       *      LAST_VALUE(x)   x at f                                  x's type
                                       *      NTH_VALUE(x, n) x at s + n - 1 if that is <= f, else NULL  x's type, nullable
                                       *      PERCENT_RANK()  (rank - 1) / (e - s), 0 when s = e      Float64 (g)
                                       *      CUME_DIST()     (f - s + 1) / (e - s + 1)               Float64 (g)
                                       *    The value functions move x's 64 bits unchanged (NaN payloads and -0.0
                                       *    included); LAG / LEAD ignore the frame.  width_ns is LAG / LEAD's k (>= 0)
                                       *    or NTH_VALUE's n (>= 1); every other function ignores it.  k < 0 or n < 0 =>
                                       *    UNSUPPORTED (DataFusion's reversed offsets are not pinned here), n = 0 =>
                                       *    INVALID_ARGUMENT.  With flags & ARROYO_B200_FLAG_FN_DEFAULT, LAG / LEAD's
                                       *    default d is the 64 bits in gap_ns, in x's type; without it d is NULL.  The
                                       *    flag on FN_FIRST_VALUE .. FN_CUME_DIST => INVALID_ARGUMENT (the ranking
                                       *    functions and the aggregates ignore flags, as before).  A nullable column
                                       *    carries an Arrow validity bitmap only when one of its rows is NULL;
                                       *  - frame (ArroyoB200WindowFrame): units 0 (a zeroed struct) is the default frame
                                       *    above.  ROWS / RANGE / GROUPS run the aggregates and FIRST_VALUE /
                                       *    LAST_VALUE / NTH_VALUE over [lo, hi), sorted rows clipped to [s, e + 1)
                                       *    (lo >= hi: an empty frame).  A start gives lo, an end hi:
                                       *      ROWS    n PRECEDING j - n, CURRENT ROW j, n FOLLOWING j + n; an end one
                                       *              past the row it names;
                                       *      RANGE   CURRENT ROW: the row's first peer / one past its last peer; n
                                       *              PRECEDING / FOLLOWING (exactly one ORDER BY key): the first row
                                       *              whose key is within n before / after the row's, or one past the
                                       *              last such row for an end.  "Before" is in sort order: under DESC
                                       *              "n PRECEDING" reaches keys up to x + n.  Computed on the sort's
                                       *              unsigned form of the key: a limit past the key type's range lies
                                       *              past every row, so the frame runs to the segment's edge or is
                                       *              empty (whether DataFusion errors on that overflow instead is not
                                       *              pinned here);
                                       *      GROUPS  the first row of the peer group n before / after the row's (an
                                       *              end: one past that group's last row);
                                       *      UNBOUNDED PRECEDING s, UNBOUNDED FOLLOWING e + 1.
                                       *    ROWS and GROUPS offsets may be anything up to INT64_MAX.  COUNT gives
                                       *    hi - lo; SUM the wrapping sum; AVG the exact sum converted to f64 once,
                                       *    over hi - lo; MIN / MAX the extremes; FIRST_VALUE / LAST_VALUE /
                                       *    NTH_VALUE x at lo / hi - 1 / lo + n - 1 (NULL unless < hi).  Every
                                       *    function but COUNT is NULL on an empty frame, and its column is nullable.
                                       *    A frame equal to the default (RANGE UNBOUNDED PRECEDING AND CURRENT ROW with
                                       *    ORDER BY; UNBOUNDED PRECEDING AND UNBOUNDED FOLLOWING in any unit without
                                       *    it) runs as units 0 and gives its bits.  INVALID_ARGUMENT: units outside 0
                                       *    to 3, a frame on any other function, a bound code outside 1 to 5, a start at
                                       *    UNBOUNDED FOLLOWING or an end at UNBOUNDED PRECEDING, a negative offset of
                                       *    n PRECEDING / FOLLOWING, RANGE with an offset and not exactly one ORDER BY
                                       *    key, GROUPS without ORDER BY.  UNSUPPORTED: a start after the end (n
                                       *    FOLLOWING AND CURRENT ROW | m PRECEDING, CURRENT ROW AND m PRECEDING),
                                       *    which SQLite refuses and nothing here pins.  Frames that are empty for
                                       *    every row (2 FOLLOWING AND 1 FOLLOWING) are accepted;
                                       *  - slide_ns: N of a fused `WHERE fn <= N` (`fn = 1` is the same as `<= 1` for all
                                       *    three ranking functions); 0 = every row leaves; < 0, or not 0 for any other
                                       *    function => INVALID_ARGUMENT;
                                       *  - n_cols / timestamp_col / key_col / input_col count FLAT columns: a host batch's
                                       *    struct columns (the upstream window{start, end}, children all 64-bit) are
                                       *    flattened in place, one level, for this kind only.
                                       * Columns pass through as raw 64 bits.  Device batches carry no types: the column
                                       * types are those of the first host or state batch (a zero-row host batch may
                                       * declare them), Int64 until then; a later batch of other types =>
                                       * INVALID_ARGUMENT.
                                       * Rows: _timestamp < the last watermark => late, dropped (filter_by_time keeps
                                       * ts >= w, arroyo-rpc/src/df.rs:211-231); a negative _timestamp => PANIC.
                                       * Watermark w: every instant < w leaves in ascending order (window_fn.rs:178-201),
                                       * in ONE batch per emission, rows ordered by (instant, partition key ASC, ORDER BY
                                       * keys); ties on every key by arrival order, restored rows first (DataFusion's sort
                                       * promises no order there; RANK and DENSE_RANK do not depend on it).  Output = the
                                       * input columns (struct columns re-nested as the host batches had them) then the
                                       * function: UInt64 (L) for a ranking function, named row_number / rank /
                                       * dense_rank, count / sum / avg / min / max as above for an aggregate, and lag /
                                       * lead / first_value / last_value / nth_value / percent_rank / cume_dist as
                                       * above.  Host output only: handle_watermark_device* => UNSUPPORTED.
                                       * Checkpoints write table "input" (retention 0): per open instant one batch of the
                                       * rows accepted since the previous checkpoint, in the input layout, in arrival
                                       * order.  on_start takes such batches in any order, does not late-filter them,
                                       * and the restored watermark becomes the late watermark.  More than 2^31 buffered
                                       * rows => RUNTIME, nothing changed.  Stats: rows_in, rows_late, rows_out (after
                                       * the fused filter), windows_out (instants emitted).                             */
} ArroyoB200OpKind;

/* WINDOW_FUNCTION: the function (config field `window_fn`) and the ORDER BY directions (`aggs[].kind`) */
typedef enum ArroyoB200WindowFn {
  ARROYO_B200_FN_ROW_NUMBER = 1,
  ARROYO_B200_FN_RANK = 2,
  ARROYO_B200_FN_DENSE_RANK = 3,
  ARROYO_B200_FN_AGGREGATE = 4,   /* the ArroyoB200AggKind in aggs[0] */
  ARROYO_B200_FN_LAG = 5,         /* value functions (5-9): aggs[0] = {ARROYO_B200_FN_ARGUMENT, x} */
  ARROYO_B200_FN_LEAD = 6,
  ARROYO_B200_FN_FIRST_VALUE = 7,
  ARROYO_B200_FN_LAST_VALUE = 8,
  ARROYO_B200_FN_NTH_VALUE = 9,
  ARROYO_B200_FN_PERCENT_RANK = 10,
  ARROYO_B200_FN_CUME_DIST = 11
} ArroyoB200WindowFn;
#define ARROYO_B200_ORDER_ASC 16
#define ARROYO_B200_ORDER_DESC 17
#define ARROYO_B200_FN_ARGUMENT 18 /* aggs[0].kind of a value function: input_col is its argument x */
#define ARROYO_B200_MAX_ORDER_KEYS 4

typedef enum ArroyoB200AggKind {
  ARROYO_B200_AGG_COUNT_STAR = 1, /* count(Int64(1)) -> Int64                          */
  ARROYO_B200_AGG_SUM_I64 = 2,    /* sum(Int64) -> Int64, wrapping                     */
  ARROYO_B200_AGG_AVG_I64 = 3,    /* avg(Int64) -> Float64; state (count u64, sum f64) */
  ARROYO_B200_AGG_MIN_I64 = 4,
  ARROYO_B200_AGG_MAX_I64 = 5
} ArroyoB200AggKind;

typedef enum ArroyoB200JoinType {
  ARROYO_B200_JOIN_INNER = 0,
  ARROYO_B200_JOIN_LEFT = 1,
  ARROYO_B200_JOIN_RIGHT = 2,
  ARROYO_B200_JOIN_FULL = 3
} ArroyoB200JoinType;

#define ARROYO_B200_MAX_AGGS 8
#define ARROYO_B200_MAX_COLS 16

typedef struct ArroyoB200Agg {
  int32_t kind;      /* ArroyoB200AggKind                              */
  int32_t input_col; /* index into the input batch; ignored for COUNT  */
} ArroyoB200Agg;

/* WINDOW_FUNCTION: an explicit frame clause, `{ROWS | RANGE | GROUPS} BETWEEN start AND end` (DataFusion's
 * WindowFrame).  units = ARROYO_B200_FRAME_DEFAULT (0, a zeroed struct) is DataFusion's default frame and the other
 * fields are ignored.  Otherwise start_kind / end_kind are ArroyoB200FrameBound codes and start_offset / end_offset
 * the n of `n PRECEDING` / `n FOLLOWING` (>= 0; ignored for the other bounds).  For RANGE over a Timestamp(ns) key
 * the offsets are nanoseconds.  The kind-8 contract above says which frames run and which are refused. */
typedef enum ArroyoB200FrameUnits {
  ARROYO_B200_FRAME_DEFAULT = 0,
  ARROYO_B200_FRAME_ROWS = 1,
  ARROYO_B200_FRAME_RANGE = 2,
  ARROYO_B200_FRAME_GROUPS = 3
} ArroyoB200FrameUnits;
typedef enum ArroyoB200FrameBound {
  ARROYO_B200_BOUND_UNBOUNDED_PRECEDING = 1,
  ARROYO_B200_BOUND_PRECEDING = 2,
  ARROYO_B200_BOUND_CURRENT_ROW = 3,
  ARROYO_B200_BOUND_FOLLOWING = 4,
  ARROYO_B200_BOUND_UNBOUNDED_FOLLOWING = 5
} ArroyoB200FrameBound;
typedef struct ArroyoB200WindowFrame {
  int32_t units;        /* ArroyoB200FrameUnits */
  int32_t start_kind;   /* ArroyoB200FrameBound */
  int32_t end_kind;     /* ArroyoB200FrameBound */
  int32_t pad;          /* 0 */
  int64_t start_offset;
  int64_t end_offset;
} ArroyoB200WindowFrame;

/* Input batches are the operator's `in_schemas[i]` (ArroyoSchema, arroyo-rpc/src/df.rs):
 * [key cols (routing copies)..., payload cols..., _timestamp]; all supported columns are
 * 64-bit fixed width (int64 "l", uint64 "L", timestamp[ns] "tsn:", float64 "g" for payload). */
typedef struct ArroyoB200OpConfig {
  int32_t kind;          /* ArroyoB200OpKind                                            */
  int32_t device;        /* CUDA ordinal                                                */
  uint64_t stream;       /* caller-owned cudaStream_t, or 0: the library creates a private non-blocking stream.
                          * STREAM-ORDERING CONTRACT: every kernel and copy of the handle is enqueued on this one
                          * stream.  Device buffers passed to process_device_batch(es) must have been produced on it
                          * (or the producer must have been synchronised with it before the call), and device output
                          * (handle_watermark_device) is ready for work enqueued on it.  With stream = 0 the private
                          * stream has NO ordering against any caller stream (the legacy default stream included): the
                          * caller must synchronise its producer before the call and arroyo_b200_op_flush before it
                          * reads device output or reuses the input buffers.  Host (Arrow) entry points need nothing:
                          * they synchronise internally before they return host data.                                 */
  uint32_t task_index;   /* TaskInfo.task_index  (arroyo-types/src/lib.rs TaskInfo)     */
  uint32_t parallelism;  /* TaskInfo.parallelism                                        */

  int64_t width_ns;      /* width_micros * 1000; 0 (the instant window) is refused here:*/
                         /* that plan is INSTANT_AGGREGATE                              */
                         /* INSTANT_AGGREGATE: read only when final_projection = 1, as  */
                         /* the upstream window's width W (> 0) of the window struct    */
  int64_t slide_ns;      /* slide_micros * 1000 (sliding only)                          */
  int64_t gap_ns;        /* gap_micros * 1000 (session)                                 */
                         /* UPDATING_AGGREGATE: the time-to-idle ttl in ns, 0 = keys    */
                         /* never expire, < 0 = INVALID_ARGUMENT.  A shim passes        */
                         /* ttl_micros * 1000, or 24 h when ttl_micros == 0, as the     */
                         /* reference does (incremental_aggregator.rs:1043-1048); see   */
                         /* arroyo_b200_op_set_clock                                    */

  int32_t n_cols;        /* columns in each input batch (join: left side)               */
  int32_t timestamp_col; /* ArroyoSchema.timestamp_index                                */
  int32_t n_key_cols;    /* 0 (global window) or 1; group-by column index below         */
  int32_t key_col;
  int32_t n_aggs;
  ArroyoB200Agg aggs[ARROYO_B200_MAX_AGGS];

  int32_t final_projection; /* 1: insert window{start,end} at window_index and set        */
                            /*    _timestamp = bin + width - 1 (planner                   */
                            /*    extension/aggregate.rs:292-390); 0: _timestamp = bin    */
  int32_t window_index;     /* position of the window struct among the output columns     */

  /* INSTANT_JOIN: left = input indices < in_partitions/2 (instant_join.rs:249-253).      */
  int32_t join_type;        /* ArroyoB200JoinType                                         */
  int32_t right_n_cols;
  int32_t right_timestamp_col;
  int32_t left_key_col;     /* equi-join columns (payload, after `unkeyed_batch`)         */
  int32_t right_key_col;
  int32_t left_n_routing;   /* leading `_key_*` routing copies stripped from each side    */
  int32_t right_n_routing;  /* (arroyo-rpc/src/df.rs:359-367)                             */

  /* Window aggregates fed with PARTIAL aggregates (the final stage of a partial -> shuffle -> final
   * plan: each upstream row stands for `count` original rows).  0 = inputs are raw rows; otherwise
   * 1 + the index of the input column that carries the row count.  SUM / MIN / MAX then merge the
   * upstream partial columns, COUNT(*) and AVG use the carried count. */
  int32_t partial_count_col_plus1;
  int32_t window_fn;        /* WINDOW_FUNCTION: ArroyoB200WindowFn; every other kind ignores it */

  uint64_t expected_keys;   /* capacity hint for the key dictionary (0 = default)         */
  uint32_t flags;           /* ARROYO_B200_FLAG_*                                         */
  uint32_t reserved;        /* 0, or log2(rows per ingest launch) in [16, 26] (default 24)     */

  /* ABI version 2 appended this field: the struct grew from 192 to 224 bytes, every earlier field keeping its
   * offset.  op_create reads the whole struct, so a caller built against version 1's declaration must be rebuilt
   * (arroyo_b200_abi_version tells the two apart); zero the field for today's behaviour. */
  ArroyoB200WindowFrame frame; /* WINDOW_FUNCTION: the frame clause (zeroed: the default frame); every other kind
                                * ignores it */
} ArroyoB200OpConfig;

#define ARROYO_B200_FLAG_PROFILE 1u       /* time kernels with CUDA events (op_stats)      */
#define ARROYO_B200_FLAG_REMERGE_ONLY 2u  /* sliding: always re-merge all panes per slide  */
                                          /* (the reference's algorithm) instead of the    */
                                          /* running add/evict window; same results        */
#define ARROYO_B200_FLAG_AVG_F64 8u       /* AVG(Int64) with its own f64 accumulator from the start  */
                                          /* (default: exact integer sum, promoted on demand)        */
#define ARROYO_B200_FLAG_COMBINE 4u       /* (default behaviour; kept for ABI stability)   */
#define ARROYO_B200_FLAG_ZERO_COPY 32u    /* accepted and ignored (pinned host batches were read in   */
                                          /* place over PCIe, which was slower than staging them      */
                                          /* with the copy engine; every host batch is staged now)    */
#define ARROYO_B200_FLAG_NO_COMBINE 16u   /* do not warp-combine equal keys before the     */
                                          /* atomics (measurement knob)                    */
#define ARROYO_B200_FLAG_NO_DIRECT 64u    /* accepted and ignored (round 1 mapped dense key ranges    */
                                          /* straight onto ids; every key is hashed now)              */
#define ARROYO_B200_FLAG_NO_TWO_PASS 128u /* always use the one-pass ingest kernel (probe + REDs per  */
                                          /* row) instead of partition + shared-memory aggregation     */
                                          /* (measurement knob; results are identical)                */
#define ARROYO_B200_FLAG_UPDATING_INPUT 512u /* UPDATING_AGGREGATE: the input is itself an updating stream (rows carry
                                          * `_updating_meta.is_retract`): refused, ARROYO_B200_UNSUPPORTED            */
#define ARROYO_B200_FLAG_TWO_PASS_ALWAYS 256u /* two-pass ingest for every eligible launch, however small  */
                                          /* (by default launches under 2^19 rows use the one-pass kernel: */
                                          /* the per-bucket set-up does not pay for them; test knob)       */
#define ARROYO_B200_FLAG_FN_DEFAULT 1024u /* WINDOW_FUNCTION, LAG / LEAD: gap_ns holds the default's 64 bits */

typedef struct ArroyoB200Op ArroyoB200Op;

/* A list of record batches owned by the library until released. Each batch is a struct
 * array (children = columns) + its schema.  `release` on the arrays / schemas, or
 * arroyo_b200_release_batches, returns the pinned buffers to the library's pool. */
typedef struct ArroyoB200Batches {
  int64_t n_batches;
  struct ArrowArray* arrays;
  struct ArrowSchema* schemas;
  void* private_data;
} ArroyoB200Batches;

/* Device-resident output of one emitted window (for chaining operators on the GPU and for
 * the device-resident throughput measurement).  Pointers stay valid until the next call on
 * the same handle. */
typedef struct ArroyoB200DeviceBatch {
  int64_t n_rows;
  int32_t n_cols;
  int32_t reserved;
  uint64_t cols[ARROYO_B200_MAX_COLS]; /* device pointers, one 64-bit column each */
} ArroyoB200DeviceBatch;

typedef struct ArroyoB200Stats {
  uint64_t rows_in;           /* rows handed to process_batch                          */
  uint64_t rows_late;         /* rows dropped by the late-bin rule                     */
  uint64_t rows_deferred;     /* rows re-ingested after ring / dictionary growth       */
  uint64_t rows_out;          /* rows emitted                                          */
  uint64_t windows_out;       /* windows (or sessions batches / join instants) emitted */
  uint64_t n_keys;            /* distinct keys in the dictionary                       */
  uint64_t kernel_launches;   /* CUDA kernels launched by this handle                  */
  uint64_t ingest_launches;
  uint64_t emit_launches;
  uint64_t h2d_bytes;
  uint64_t d2h_bytes;
  double ingest_ms;           /* CUDA-event time, ARROYO_B200_FLAG_PROFILE only        */
  double emit_ms;
  uint64_t ingest_rows_timed; /* rows covered by ingest_ms                             */
  uint64_t emit_rows_timed;   /* key slots scanned during emit_ms                      */
  double host_process_ms;     /* wall clock spent inside process_batch* calls          */
  double host_watermark_ms;   /* wall clock spent inside handle_watermark* calls       */
} ArroyoB200Stats;

/* ---- library ---- */
/* ABI version of this header (checked by the bindings): 2 since ArroyoB200OpConfig gained `frame`. */
int32_t arroyo_b200_abi_version(void);
/* Number of usable CUDA devices (0 on a box without a GPU). */
int32_t arroyo_b200_device_count(void);
/* Pinned host allocator for Arrow buffers handed to process_batch ("Arrow buffers pinned and
 * zero-copied to device"); pageable buffers are accepted too and staged internally. */
void* arroyo_b200_host_alloc(uint64_t bytes);
void arroyo_b200_host_free(void* p);

/* ---- operator lifecycle: mirrors trait ArrowOperator (arroyo-operator/src/operator.rs:1143-1257)
 * behind OperatorConstructor::with_config (operator.rs:56-63, arroyo-operator/src/lib.rs:135-151) ---- */

/* with_config(): build an operator; ARROYO_B200_UNSUPPORTED => use the stock operator.
 * `err`/`err_len` receive the message when creation fails (no handle to ask). */
int32_t arroyo_b200_op_create(const ArroyoB200OpConfig* config, ArroyoB200Op** out, char* err,
                              uint64_t err_len);
/* drop(): frees device memory, streams, pinned pools. */
void arroyo_b200_op_destroy(ArroyoB200Op* op);
/* Error text of the last failing call on this handle (valid until the next call). */
const char* arroyo_b200_op_last_error(const ArroyoB200Op* op);
/* ArrowOperator::name(). */
const char* arroyo_b200_op_name(const ArroyoB200Op* op);

/* ArrowOperator::on_start(ctx): restore.  `state` holds the batches the shim read from the
 * operator's state table (tumbling/sliding: table "t" in `partial_schema`
 * [key, state cols..., _timestamp = pane start], via
 * ExpiringTimeKeyView::all_batches_for_watermark, arroyo-state/src/tables/expiring_time_key_map.rs:858-872;
 * sliding_aggregating_window.rs:556-595, tumbling :228-248).  `n == 0` = fresh start.
 * `watermark_ns` = ctx.last_present_watermark() or INT64_MIN when there is none.
 * `table_min_time_ns` = ExpiringTimeKeyView::get_min_time() or INT64_MIN.
 * Ownership follows the Arrow C Data convention, as in process_batch: the library takes a state
 * batch by releasing it, which sets its `release` to NULL; a successful restore takes every array.
 * Whatever still has a non-null `release` after the call, successful or not, belongs to the caller,
 * and so do the schemas.
 * Window, instant and updating aggregates: a batch whose column count, column types or key type
 * (l, L or tsn:) is not the plan's layout of the table => ARROYO_B200_INVALID_ARGUMENT, with nothing
 * changed and every batch left to the caller.
 * Updating aggregate (incremental_aggregator.rs:446-503): `state` holds every batch of table "a"
 * (UncachedKeyValueView::get_all, in any order, not de-duplicated), in the layout
 * arroyo_b200_op_checkpoint_state writes; both time arguments are ignored.  Per key the row with the
 * largest `_generation` wins, a tie going to the later row (batch order, then row order); it seeds the
 * accumulators and the values the next flush retracts.  The dictionary is sized from the row count and
 * grows when a bucket runs out of ids; keys that still cannot be placed => ARROYO_B200_RUNTIME.
 * ARROYO_B200_INVALID_ARGUMENT, with nothing changed: an operator that has already taken rows or been
 * restored.  Restored rows do not count in
 * `rows_in`; their keys count in `n_keys`.
 * A null `_timestamp` (and only there) marks a tombstone: when it wins, its key stays absent (see
 * arroyo_b200_op_set_clock).  With a ttl, restored keys are stamped with the clock at this call.
 * TTL join: `n > 0` => ARROYO_B200_UNSUPPORTED; its tables go through arroyo_b200_op_restore_side. */
int32_t arroyo_b200_op_on_start(ArroyoB200Op* op, struct ArrowArray* state, struct ArrowSchema* schemas,
                                int64_t n, int64_t watermark_ns, int64_t table_min_time_ns);

/* The TTL join's restore: KeyTimeView::insert_internal (arroyo-state/src/tables/expiring_time_key_map.rs:1008-1049)
 * for the batches the shim read from table "left" (`side` 0) or "right" (`side` 1).  The reference loads both tables
 * at the first batch after a restart (get_key_time_view :200-236): batches whose newest `_timestamp` is below
 * last_present_watermark - ttl (UNIX_EPOCH without a watermark) are dropped by the shim, the rest are handed here.
 * The rows of the `n` batches, in the side's input layout (the layout process_batch takes), join that side's stored
 * rows.  Nothing is emitted, and pairs among restored rows never are; a later batch of the other side matches restored
 * rows exactly like rows it had received itself.
 *  - When: any number of calls, for either side, in any order, but only before the first batch process_batch /
 *    process_batch_emit accepts.  After that => ARROYO_B200_INVALID_ARGUMENT, nothing changed.
 *  - All `n` batches are checked before anything changes: the side's column count (INVALID_ARGUMENT), the key type
 *    rule of process_batch, counting earlier restored batches and the other side's key (UNSUPPORTED), no nulls
 *    (UNSUPPORTED).  On failure no row of the call is kept.  A restored key type binds later batches, as a first batch
 *    does.  Zero-row batches are accepted.  A side that would pass 2^31 rows => ARROYO_B200_RUNTIME, nothing changed.
 *  - Ownership as for on_start: the library takes the arrays on success, the caller keeps them on error, and the
 *    caller always keeps the schemas.
 *  - Restored rows count in no statistic but `h2d_bytes` and `kernel_launches`.
 * Every other operator kind => ARROYO_B200_UNSUPPORTED.  Device-resident input to the TTL join stays unsupported, so
 * a shim writes the tables only from host batches. */
int32_t arroyo_b200_op_restore_side(ArroyoB200Op* op, uint32_t side, struct ArrowArray* batches,
                                    struct ArrowSchema* schemas, int64_t n);

/* ArrowOperator::process_batch_index(index, in_partitions, batch, ctx, collector)
 * (operator.rs:1174-1188).  On success the library owns `batch` and calls its `release`
 * once the host->device copy has completed; on error the caller keeps ownership.
 * Non-zero `offset` is honoured; columns with null_count > 0 => ARROYO_B200_UNSUPPORTED.
 * Window operators emit nothing here (tumbling :250-319, sliding :598-674, session :850-895,
 * instant_join :109-172), so there is no collector argument. */
int32_t arroyo_b200_op_process_batch(ArroyoB200Op* op, uint32_t input_index, uint32_t in_partitions,
                                     struct ArrowArray* batch, const struct ArrowSchema* schema);

/* process_batch_index for operators that emit from it (operator.rs:1174-1188 hands them the collector): the TTL join
 * emits the pairs an arriving batch completes (join_with_expiration.rs:42-130).  For every other operator this is
 * arroyo_b200_op_process_batch with an empty `out`. */
int32_t arroyo_b200_op_process_batch_emit(ArroyoB200Op* op, uint32_t input_index, uint32_t in_partitions,
                                          struct ArrowArray* batch, const struct ArrowSchema* schema, ArroyoB200Batches* out);

/* Same, for a batch already resident on the operator's device: `cols[i]` are device pointers
 * to n_rows 64-bit values each.  The buffers must stay valid until the next call that
 * returns output (handle_watermark / handle_checkpoint / on_close / flush). */
int32_t arroyo_b200_op_process_device_batch(ArroyoB200Op* op, uint32_t input_index, uint32_t in_partitions,
                                            const uint64_t* cols, int32_t n_cols, int64_t n_rows);

/* A run of device-resident batches in one call (same semantics as calling
 * process_device_batch once per batch, in order): batch b has n_rows[b] rows and its column c
 * starts at cols[b * n_cols + c].  Exists so that hosts with a slow FFI (Python ctypes) do not
 * become the bottleneck of the device-resident path. */
int32_t arroyo_b200_op_process_device_batches(ArroyoB200Op* op, uint32_t input_index, uint32_t in_partitions,
                                              const uint64_t* cols, int32_t n_cols, const int64_t* n_rows,
                                              int64_t n_batches);

/* ArrowOperator::handle_watermark(watermark, ctx, collector) (operator.rs:1206-1214).
 * `watermark_ns` is ctx.last_present_watermark() after the run loop's min-merge over inputs
 * (WatermarkHolder, arroyo-operator/src/context.rs:35-86).  `out` receives, in ascending
 * window order, the batches the reference would pass to Collector::collect
 * (context.rs:490-494) before it forwards the watermark. */
int32_t arroyo_b200_op_handle_watermark(ArroyoB200Op* op, int64_t watermark_ns, ArroyoB200Batches* out);

/* handle_watermark in two halves, for shims that keep the run loop going while windows travel to the host -- the
 * mechanism the reference's own operators use for long-running work: ArrowOperator::future_to_poll /
 * handle_future_result (operator.rs:1190-1204; tumbling_aggregating_window.rs:394-428).
 *   begin: everything handle_watermark does, except that the device->host copies of the emitted windows are
 *          enqueued on a second stream and not awaited; the call returns as soon as they are enqueued.
 *   poll : `*ready` = 1 and `out` = the batches once those copies have completed (`block` != 0 waits for them),
 *          else `*ready` = 0.  The shim forwards the watermark after it has collected the batches
 *          (operator.rs:777-786).  `begin` with an uncollected emission outstanding is an error; the other
 *          entry points may be called in between (the copies overlap the next batches' host->device copies). */
/* ArrowOperator::handle_tick(tick, ctx, collector) (operator.rs:1233-1241), for operators whose `tick_interval()` is
 * set -- the updating aggregate flushes its change rows here (incremental_aggregator.rs:990-1004).  Other operators
 * emit nothing. */
int32_t arroyo_b200_op_handle_tick(ArroyoB200Op* op, ArroyoB200Batches* out);

int32_t arroyo_b200_op_handle_watermark_begin(ArroyoB200Op* op, int64_t watermark_ns);
int32_t arroyo_b200_op_handle_watermark_poll(ArroyoB200Op* op, int32_t block, ArroyoB200Batches* out, int32_t* ready);

/* The run loop of a single-input operator task for a run of queued batches, inside the library -- what the
 * subtask's loop does between two control messages (arroyo-operator/src/operator.rs:982-1062): for every batch
 * `process_batch`; when `watermarks[i]` != INT64_MIN the (already min-merged) watermark that follows batch i is
 * handled, with the begin / poll pair when `async_emit` != 0 (outstanding windows are collected before the next
 * emission begins and polled every few batches), else with the blocking call.  `out` receives the windows
 * collected during the call in emission order; with `async_emit` the last emission may still be outstanding on
 * return -- the next call, or handle_watermark_poll, delivers it.  Ownership of batches [0, *n_consumed) has moved
 * to the library (all of them on success).  For hosts whose per-call FFI cost is not negligible against a
 * 64 Ki-row batch's 28 us of PCIe time (Python ctypes; a Rust shim can as well loop itself). */
int32_t arroyo_b200_op_run_batches(ArroyoB200Op* op, struct ArrowArray* batches, const struct ArrowSchema* schema,
                                    int64_t n_batches, const int64_t* watermarks, int32_t async_emit,
                                    ArroyoB200Batches* out, int64_t* n_consumed);

/* Same, leaving the emitted windows on the device.  `out` must have room for `max_out`
 * entries; `*n_out` receives the number written.  Windows beyond the first `max_out` stay queued, in
 * order, and handle_watermark_device_poll returns them (again at most `max_out` per call): no emitted
 * window is lost.  While windows are queued, handle_watermark_device and _begin refuse a new emission
 * with INVALID_ARGUMENT (the queued windows live in the buffers it would write). */
int32_t arroyo_b200_op_handle_watermark_device(ArroyoB200Op* op, int64_t watermark_ns,
                                               ArroyoB200DeviceBatch* out, int64_t max_out, int64_t* n_out);

/* The same emission split in two, like handle_watermark_begin / _poll (the trait's future_to_poll /
 * handle_future_result pair, operator.rs:1190-1204):
 *   begin : plans the emission and enqueues its kernels; does NOT wait for the windows' row counts.
 *   poll  : waits for them and returns the windows (empty windows dropped).  At most one emission may be outstanding;
 *           handle_checkpoint / flush / on_close settle an outstanding one themselves (poll still returns it).
 * Between the two the caller typically hands over the next batches and calls `submit`, so the next ingest launch is
 * queued behind the emission and the device never waits for the host (bench.py: 0.48 -> 0.44 ms per step). */
int32_t arroyo_b200_op_handle_watermark_device_begin(ArroyoB200Op* op, int64_t watermark_ns);
int32_t arroyo_b200_op_handle_watermark_device_poll(ArroyoB200Op* op, ArroyoB200DeviceBatch* out, int64_t max_out,
                                                    int64_t* n_out);

/* ArrowOperator::handle_checkpoint(barrier, ctx, collector) (operator.rs:1216-1224):
 * `state_out` receives the partial-state batches the reference writes to its state table
 * (sliding :693-737, tumbling :430-467); the shim inserts them with
 * ExpiringTimeKeyView::insert(pane_start, batch) and flushes.  `watermark_ns` = ctx.watermark()
 * if it is an event time, else INT64_MIN. */
int32_t arroyo_b200_op_handle_checkpoint(ArroyoB200Op* op, int64_t watermark_ns, ArroyoB200Batches* state_out);

/* The updating aggregate's accumulator table "a" (incremental_aggregator.rs:619-635, checkpoint_sliding
 * :272-340): one batch with the latest state of every key flushed since the previous call, or no batch.
 * The shim calls it after handle_checkpoint and inserts the batches with
 * UncachedKeyValueView::insert_batch.  Columns: [key (the input key's type), per aggregate in plan
 * order: count(*) -> count Int64; sum -> sum Int64 (wrapping), count UInt64; avg -> count UInt64,
 * sum Float64; min -> min Int64; max -> max Int64; then _timestamp Timestamp(ns) = max(_timestamp),
 * _generation UInt64].  The unkeyed plan has no key column.  Every row of one call carries the same
 * generation, larger than any the operator wrote or restored before.  State rows count in no statistic
 * but `d2h_bytes`.  Every other operator kind returns no batches. */
int32_t arroyo_b200_op_checkpoint_state(ArroyoB200Op* op, ArroyoB200Batches* state_out);

/* The updating aggregate's clock for its time-to-idle ttl (`gap_ns`): the reference's `Instant::now()`, which the shim
 * reads from a monotonic source and passes in ns before every call that ingests, flushes or restores.  The library
 * never reads a clock of its own.  The clock starts at 0; a value below the current one => ARROYO_B200_INVALID_ARGUMENT,
 * nothing changed.  Every other operator kind => ARROYO_B200_UNSUPPORTED.
 * Time-to-idle (UpdatingCache::with_time_to_idle, updating_cache.rs:42-62; incremental_aggregator.rs:688-705):
 *  - every row ingested by process_batch, process_device_batch(es) or run_batches sets its key's last-update time to
 *    the clock at that call (rows deferred for dictionary growth included);
 *  - a flush (handle_tick, handle_checkpoint, on_close with end of data) first emits the change rows as without a
 *    ttl, then evicts every live key with clock - last update >= ttl: one retraction row with the values and
 *    `_timestamp` the key's last flush emitted, and its state is dropped.  A key that returns is a new key (append
 *    only).  The unkeyed plan's one group expires the same way.  Rows of one flush: retractions, appends, eviction
 *    retractions.  Eviction retractions leave even when the flush has no other row (the reference loses them then);
 *  - the next checkpoint_state writes a tombstone for every key evicted since the last export and not flushed again:
 *    a table-"a" row with a null `_timestamp` (the reference's deletion encoding, :591-614).  on_start accepts nulls
 *    in `_timestamp` only: a winning tombstone leaves its key absent; restored keys are stamped with the clock at
 *    on_start;
 *  - `n_keys` counts live keys; `rows_out` includes eviction retractions.  With ttl 0 nothing expires and the clock
 *    changes nothing. */
int32_t arroyo_b200_op_set_clock(ArroyoB200Op* op, int64_t now_ns);

/* ArrowOperator::on_close(final_message, ctx, collector) (operator.rs:1247-1256). */
int32_t arroyo_b200_op_on_close(ArroyoB200Op* op, int32_t end_of_data, ArroyoB200Batches* out);

/* Wait until every enqueued copy and kernel of this handle has finished and input batches
 * have been released. */
int32_t arroyo_b200_op_flush(ArroyoB200Op* op);

/* The operators batch input rows into launches of 2^reserved rows.  `submit` enqueues the rows
 * accepted so far without waiting for them (no reference counterpart: the reference's operators
 * run each batch to completion inside process_batch).  A host that knows its input queue is
 * empty calls it so that the device works while the host is idle. */
int32_t arroyo_b200_op_submit(ArroyoB200Op* op);

void arroyo_b200_release_batches(ArroyoB200Batches* batches);

int32_t arroyo_b200_op_stats(ArroyoB200Op* op, ArroyoB200Stats* out);

/* ---- key-hash shuffle: replaces ArrowCollector::collect -> repartition
 * (arroyo-operator/src/context.rs:506-541) + server_for_hash_array (arroyo-operator/src/lib.rs:30-41).
 * Device in, device out: rows of `n_cols` 64-bit columns are bucketed by
 * dest = (hash(key) / (u64::MAX / n_dest)) % n_dest into contiguous per-destination segments of
 * `out_cols` (same shapes as the inputs); `counts[d]` (device, n_dest int64) receives the rows
 * for destination d and `offsets[d]` their start.  The segments are the send buffers of the
 * NCCL all-to-all that carries the Shuffle edge. ---- */
typedef struct ArroyoB200Partitioner ArroyoB200Partitioner;
int32_t arroyo_b200_partitioner_create(int32_t device, uint64_t stream, int32_t n_dest, int32_t n_cols,
                                       int32_t key_col, int64_t max_rows, ArroyoB200Partitioner** out);
void arroyo_b200_partitioner_destroy(ArroyoB200Partitioner* p);
int32_t arroyo_b200_partition(ArroyoB200Partitioner* p, const uint64_t* in_cols, int64_t n_rows,
                              const uint64_t* out_cols, uint64_t counts_dev, uint64_t offsets_dev);
/* Same bucketing, one output buffer (`packed_dev`, n_rows * n_cols int64): destination d owns the
 * element range [n_cols * offsets[d], n_cols * (offsets[d] + counts[d])), holding its n_cols columns
 * back to back (counts[d] values each).  One all-to-all with element splits n_cols * counts then
 * carries every column of the edge; the receiver reads each sender's block as a columnar batch. */
int32_t arroyo_b200_partition_packed(ArroyoB200Partitioner* p, const uint64_t* in_cols, int64_t n_rows,
                                     uint64_t packed_dev, uint64_t counts_dev, uint64_t offsets_dev);
/* WatermarkGenerator::process_batch's reductions (arroyo-worker/src/arrow/watermark_generator.rs:160,176:
 * kernels::aggregate::max / min over the timestamp column) for a device-resident batch. Synchronous. */
int32_t arroyo_b200_ts_minmax(int32_t device, uint64_t stream, uint64_t ts_dev, int64_t n_rows, int64_t* out_min,
                               int64_t* out_max);
/* The hash used for routing (host-callable restatement for tests). */
uint64_t arroyo_b200_hash_key(int64_t key);
/* dest = (h / (u64::MAX / n)) % n -- arroyo-operator/src/lib.rs:30-41. */
uint32_t arroyo_b200_server_for_hash(uint64_t h, uint32_t n);

/* ---- host-only planner hooks (no CUDA): the window state machines, exposed so the host logic
 * can be tested on a box without a GPU.  `events` is a sequence of (kind, value) pairs:
 * kind 0 = on-time data touched pane `value`, kind 1 = watermark `value`, kind 2 = checkpoint.
 * The plan is written to `out` as int64 records {kind, a, b, c}:
 *   kind 1 = emit window [a, b) closing pane c (c = INT64_MIN if the pane had no exec)
 *   kind 2 = pane a joins the window store; kind 3 = pane a leaves it
 * Returns the number of records (or -1 if `out_cap` is too small). ---- */
int64_t arroyo_b200_plan_sliding(int64_t width_ns, int64_t slide_ns, const int64_t* events, int64_t n_events,
                                 int64_t* out, int64_t out_cap);
int64_t arroyo_b200_plan_tumbling(int64_t width_ns, const int64_t* events, int64_t n_events, int64_t* out,
                                  int64_t out_cap);

/* Host restatement of the kernels' window-bucket assignment `bin = ts - ts % width`
 * (tumbling_aggregating_window.rs:65-73), computed with the same multiply-high fast division the
 * device code uses, so the arithmetic can be pinned without a GPU. */
int64_t arroyo_b200_bin_start(int64_t ts_ns, int64_t width_ns);

#ifdef __cplusplus
}
#endif
#endif /* ARROYO_B200_H */
