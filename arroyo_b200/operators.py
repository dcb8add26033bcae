"""Host-side mirror of the reference's window operators over the C ABI.

Class and method names follow arroyo-worker/src/arrow/{tumbling,sliding}_aggregating_window.rs and
the ArrowOperator trait (arroyo-operator/src/operator.rs:1143-1257): name(), tables(), on_start(ctx),
process_batch(batch, ctx, collector), handle_watermark(watermark, ctx, collector),
handle_checkpoint(barrier, ctx, collector), on_close(final_message, ctx, collector).
Batches are pyarrow RecordBatches crossing the boundary through the Arrow C Data Interface."""
import ctypes as C
import functools
import struct
import time
from typing import List, Optional

import pyarrow as pa

from . import ffi
from .context import Collector, OperatorContext, clamp_watermark

TIMESTAMP = "_timestamp"
_AGG_KINDS = {"count": ffi.AGG_COUNT_STAR, "sum": ffi.AGG_SUM_I64, "avg": ffi.AGG_AVG_I64,
              "min": ffi.AGG_MIN_I64, "max": ffi.AGG_MAX_I64}


def _check(lib, handle, status):
    if status == ffi.OK:
        return
    msg = lib.arroyo_b200_op_last_error(handle)
    msg = msg.decode() if msg else ""
    if status == ffi.UNSUPPORTED:
        raise ffi.UnsupportedPlan(status, msg)
    raise ffi.ArroyoB200Error(status, msg)


def export_batch(batch: pa.RecordBatch):
    arr, sch = ffi.ArrowArray(), ffi.ArrowSchema()
    batch._export_to_c(C.addressof(arr), C.addressof(sch))
    return arr, sch


def _release(s):
    """Releases an exported Arrow C struct unless its consumer already took it (`release` set to NULL)."""
    if s.release:
        C.CFUNCTYPE(None, C.c_void_p)(s.release)(C.addressof(s))


def _agg_config(kind: int, c, names: List[str]) -> ffi.OpConfig:
    """The OpConfig of an aggregate over input columns `names`: its key column and aggregates from `c`."""
    cfg = ffi.OpConfig()
    cfg.kind = kind
    cfg.n_cols = len(names)
    cfg.timestamp_col = names.index(TIMESTAMP)
    if len(c.key_names) > 1:
        raise ffi.UnsupportedPlan(ffi.UNSUPPORTED, "more than one group-by key column")
    cfg.n_key_cols = len(c.key_names)
    cfg.key_col = names.index(c.key_names[0]) if c.key_names else 0
    cfg.n_aggs = len(c.aggs)
    for i, a in enumerate(c.aggs):
        if a.kind not in _AGG_KINDS:
            raise ffi.UnsupportedPlan(ffi.UNSUPPORTED, f"aggregate {a.kind}")
        cfg.aggs[i].kind = _AGG_KINDS[a.kind]
        cfg.aggs[i].input_col = names.index(a.col) if a.col is not None else 0
    return cfg


class ExportedBatches:
    """A run of record batches (same schema) exported once to Arrow C Data structs laid out as one C array -- the
    input of arroyo_b200_op_run_batches.  Export only builds descriptors: the buffers stay where they are."""

    def __init__(self, batches: List[pa.RecordBatch]):
        self.n = len(batches)
        self.names = list(batches[0].schema.names) if batches else []
        self.arrays = (ffi.ArrowArray * max(self.n, 1))()
        self.schema = ffi.ArrowSchema()
        step = C.sizeof(ffi.ArrowArray)
        base = C.addressof(self.arrays)
        for i, b in enumerate(batches):
            if i == 0:
                b._export_to_c(base, C.addressof(self.schema))
            else:
                b._export_to_c(base + i * step)

    def release_unconsumed(self, first: int):
        """Releases the batches the library did not take (after an error)."""
        for i in range(first, self.n):
            a = self.arrays[i]
            if a.release:
                C.CFUNCTYPE(None, C.c_void_p)(a.release)(C.addressof(a))

    def __del__(self):
        try:
            if self.schema.release:
                C.CFUNCTYPE(None, C.c_void_p)(self.schema.release)(C.addressof(self.schema))
        except Exception:
            pass


def import_batches(lib, out: ffi.Batches) -> List[pa.RecordBatch]:
    res = []
    try:
        for i in range(out.n_batches):
            res.append(pa.RecordBatch._import_from_c(C.addressof(out.arrays[i]), C.addressof(out.schemas[i])))
    finally:
        lib.arroyo_b200_release_batches(C.byref(out))
    return res


class _NativeOperator:
    """Owns one ArroyoB200Op handle."""

    kind = 0

    def __init__(self, device: int = 0, stream: int = 0, flags: int = 0, expected_keys: int = 0,
                 task_index: int = 0, parallelism: int = 1, chunk_log2: int = 0):
        self._lib = ffi.load()
        self._h = C.c_void_p()
        self._device = device
        self._stream = stream
        self._flags = flags
        self._expected_keys = expected_keys
        self._task_index = task_index
        self._parallelism = parallelism
        self._chunk_log2 = chunk_log2

    def _create(self, cfg: ffi.OpConfig):
        cfg.device = self._device
        cfg.stream = self._stream
        cfg.flags |= self._flags  # on top of the plan's own flags (WindowFunction's FLAG_FN_DEFAULT)
        cfg.expected_keys = self._expected_keys
        cfg.task_index = self._task_index
        cfg.parallelism = self._parallelism
        cfg.reserved = self._chunk_log2
        err = C.create_string_buffer(1024)
        st = self._lib.arroyo_b200_op_create(C.byref(cfg), C.byref(self._h), err, 1024)
        if st != ffi.OK:
            msg = err.value.decode()
            if st == ffi.UNSUPPORTED:
                raise ffi.UnsupportedPlan(st, msg)
            raise ffi.ArroyoB200Error(st, msg)

    @property
    def created(self) -> bool:
        return bool(self._h)

    def close(self):
        if self._h:
            self._lib.arroyo_b200_op_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def flush(self):
        _check(self._lib, self._h, self._lib.arroyo_b200_op_flush(self._h))

    def submit(self):
        """Enqueue the rows accepted so far without waiting (arroyo_b200_op_submit)."""
        if self.created:
            _check(self._lib, self._h, self._lib.arroyo_b200_op_submit(self._h))

    def stats(self) -> dict:
        s = ffi.Stats()
        _check(self._lib, self._h, self._lib.arroyo_b200_op_stats(self._h, C.byref(s)))
        return s.as_dict()

    def _process_batch(self, entry, index: int, parts: int, batch: pa.RecordBatch, out: Optional[ffi.Batches] = None):
        """Hands `batch` to `entry` (arroyo_b200_op_process_batch, or arroyo_b200_op_process_batch_emit with `out`).
        The library takes the array when the call succeeds; whatever it did not take is released here."""
        arr, sch = export_batch(batch)
        extra = () if out is None else (C.byref(out),)
        try:
            st = entry(self._h, index, parts, C.byref(arr), C.byref(sch), *extra)
        finally:
            _release(arr)
            _release(sch)
        _check(self._lib, self._h, st)

    def _hand_over_state(self, call, batches: List[pa.RecordBatch]):
        """Exports `batches` as C arrays and calls `call(arrays, schemas, n)` (on_start, restore_side).  The library
        takes the batches it consumed; the rest are released here."""
        n = len(batches)
        arrs = (ffi.ArrowArray * max(n, 1))()
        schs = (ffi.ArrowSchema * max(n, 1))()
        for i, b in enumerate(batches):
            b._export_to_c(C.addressof(arrs[i]), C.addressof(schs[i]))
        try:
            st = call(arrs, schs, n)
        finally:
            for s in list(arrs) + list(schs):
                _release(s)
        _check(self._lib, self._h, st)

    def _on_start(self, batches: List[pa.RecordBatch], wm: int, t: int):
        """arroyo_b200_op_on_start with `batches` as the state, the restored watermark `wm` and the table time `t`
        (ffi.INT64_MIN: none)."""
        self._hand_over_state(lambda a, s, n: self._lib.arroyo_b200_op_on_start(self._h, a, s, n, wm, t), batches)

    def _collect(self, out: ffi.Batches, collector: Optional[Collector]):
        """Imports the batches of `out` under `output_names()` into `collector` (None: they are dropped)."""
        names = self.output_names()
        for b in import_batches(self._lib, out):
            if collector is not None:
                collector.collect(pa.RecordBatch.from_arrays(b.columns, names=names))

    def _device_windows(self, call, max_out: int, drain: bool = True):
        """The windows of a device-resident emission, list of (n_rows, [device pointers]).  `call(out, max_out, n)`
        hands out at most `max_out` of them; with `drain`, arroyo_b200_op_handle_watermark_device_poll collects the
        ones the library queued beyond that."""
        out = getattr(self, "_dev_out", None)
        if out is None or len(out) < max_out:
            out = self._dev_out = (ffi.DeviceBatch * max_out)()  # reused: building it costs more than the call
        n = C.c_int64(0)
        got = []
        while True:
            _check(self._lib, self._h, call(out, max_out, C.byref(n)))
            got += [(out[i].n_rows, [out[i].cols[c] for c in range(out[i].n_cols)]) for i in range(n.value)]
            if not drain or n.value != max_out or max_out <= 0:
                return got
            call = functools.partial(self._lib.arroyo_b200_op_handle_watermark_device_poll, self._h)


class _WindowAggregate(_NativeOperator):
    def __init__(self, config, input_schema: Optional[pa.Schema] = None, **kw):
        super().__init__(**kw)
        self.config = config
        self._names: Optional[List[str]] = None
        if input_schema is not None:
            self._build(input_schema.names)

    # -- construction (OperatorConstructor::with_config) -------------------------------------
    def _build(self, names: List[str]):
        c = self.config
        if len(c.aggs) > ffi.MAX_AGGS:
            raise ffi.UnsupportedPlan(ffi.UNSUPPORTED, "too many aggregates")
        cfg = _agg_config(self.kind, c, names)
        cfg.width_ns = self._width_ns()
        cfg.slide_ns = int(getattr(c, "slide", 0) or 0)
        pc = getattr(c, "partial_count_col", None)
        cfg.partial_count_col_plus1 = names.index(pc) + 1 if pc else 0
        cfg.final_projection = 1 if c.final_projection else 0
        cfg.window_index = int(c.window_index)
        self._create(cfg)
        self._names = list(names)

    def _width_ns(self) -> int:
        return int(self.config.width)

    def output_names(self) -> List[str]:
        c = self.config
        names = list(c.key_names) + [a.name for a in c.aggs]
        if c.final_projection:
            names.insert(min(max(c.window_index, 0), len(names)), "window")
        return names + [TIMESTAMP]

    def partial_names(self) -> List[str]:
        c = self.config
        names = list(c.key_names)
        for a in c.aggs:
            if a.kind == "avg":
                names += [f"{a.name}[count]", f"{a.name}[sum]"]
            else:
                names.append(f"{a.name}[{a.kind}]")
        return names + [TIMESTAMP]

    # -- ArrowOperator ---------------------------------------------------------------------
    def tables(self):
        # table "t": partial aggregates, retention = width (tumbling :469-482, sliding :739-752)
        return {"t": int(self.config.width)}

    def on_start(self, ctx: OperatorContext):
        wm = ctx.last_present_watermark()
        table = ctx.table("t", int(self.config.width))
        batches = [b for _, b in table.all_batches_for_watermark(wm)]
        if not batches and not self.created:
            return
        if not self.created:
            raise ffi.ArroyoB200Error(ffi.INVALID_ARGUMENT, "restore needs input_schema at construction")
        mt = table.get_min_time()
        self._on_start(batches, ffi.INT64_MIN if wm is None else clamp_watermark(wm), ffi.INT64_MIN if mt is None else mt)

    def process_batch(self, batch: pa.RecordBatch, ctx: OperatorContext, collector: Collector):
        if not self.created:
            self._build(batch.schema.names)
        self._process_batch(self._lib.arroyo_b200_op_process_batch, 0, 1, batch)

    def process_device_batch(self, cols: List[int], n_rows: int):
        """`cols` = device pointers (ints), one per input column."""
        arr = (C.c_uint64 * len(cols))(*cols)
        st = self._lib.arroyo_b200_op_process_device_batch(self._h, 0, 1, arr, len(cols), n_rows)
        _check(self._lib, self._h, st)

    def process_device_batches(self, cols_flat, n_rows, n_cols: int):
        """A run of device batches in one FFI call; `cols_flat`/`n_rows` are prebuilt ctypes arrays
        ((c_uint64 * (n_batches * n_cols)), (c_int64 * n_batches))."""
        st = self._lib.arroyo_b200_op_process_device_batches(self._h, 0, 1, cols_flat, n_cols, n_rows, len(n_rows))
        _check(self._lib, self._h, st)

    def handle_watermark(self, watermark, ctx: OperatorContext, collector: Collector):
        wm = ctx.last_present_watermark()
        if wm is None or not self.created:
            return None if self.kind == ffi.SLIDING_AGGREGATE and wm is None else watermark
        out = ffi.Batches()
        _check(self._lib, self._h, self._lib.arroyo_b200_op_handle_watermark(self._h, clamp_watermark(wm), C.byref(out)))
        self._collect(out, collector)
        return watermark

    def handle_watermark_begin(self, watermark, ctx: OperatorContext) -> bool:
        """First half of handle_watermark (arroyo_b200_op_handle_watermark_begin): the emitted windows start their
        way to the host on a second stream.  Returns False when there was nothing to do (no watermark yet)."""
        wm = ctx.last_present_watermark()
        if wm is None or not self.created:
            return False
        _check(self._lib, self._h, self._lib.arroyo_b200_op_handle_watermark_begin(self._h, clamp_watermark(wm)))
        return True

    def handle_watermark_poll(self, collector: Collector, block: bool = True) -> bool:
        """Second half: collects the windows once their copies have completed (the future_to_poll /
        handle_future_result pair of the reference's operators).  Returns False while they are still in flight."""
        out = ffi.Batches()
        ready = C.c_int32(0)
        st = self._lib.arroyo_b200_op_handle_watermark_poll(self._h, 1 if block else 0, C.byref(out), C.byref(ready))
        _check(self._lib, self._h, st)
        if not ready.value:
            return False
        self._collect(out, collector)
        return True

    def run_batches(self, exported: "ExportedBatches", watermarks, collector: Collector, first: int = 0,
                    count: Optional[int] = None, async_emit: bool = True):
        """arroyo_b200_op_run_batches over exported[first : first + count]: the subtask run loop inside the library.
        `watermarks` is a (c_int64 * exported.n) array: the effective watermark that follows each batch, or
        ffi.NO_WATERMARK.  Windows collected during the call go to `collector`; with `async_emit` the last
        emission may still be outstanding (handle_watermark_poll, or the next call, delivers it)."""
        if not self.created:
            self._build(exported.names)
        count = exported.n - first if count is None else count
        out, taken = ffi.Batches(), C.c_int64(0)
        step = C.sizeof(ffi.ArrowArray)
        st = self._lib.arroyo_b200_op_run_batches(
            self._h, C.addressof(exported.arrays) + first * step, C.addressof(exported.schema), count,
            C.cast(C.addressof(watermarks) + 8 * first, C.POINTER(C.c_int64)), 1 if async_emit else 0, C.byref(out),
            C.byref(taken))
        self._collect(out, collector)
        _check(self._lib, self._h, st)

    def handle_watermark_device(self, wm: int, max_out: int = 64):
        """Emission left on the device: list of (n_rows, [device pointers]).  The library hands out at most `max_out`
        windows per call and queues the rest; they are collected here with further polls."""
        return self._device_windows(
            functools.partial(self._lib.arroyo_b200_op_handle_watermark_device, self._h, clamp_watermark(wm)), max_out)

    def handle_watermark_device_begin(self, wm: int):
        """First half of handle_watermark_device: the emission is enqueued, its row counts are not awaited."""
        _check(self._lib, self._h, self._lib.arroyo_b200_op_handle_watermark_device_begin(self._h, clamp_watermark(wm)))

    def handle_watermark_device_poll(self, max_out: int = 64, drain: bool = True):
        """Second half: the windows of the outstanding emission, list of (n_rows, [device pointers]).  With `drain`,
        polls until the library has no window queued (it hands out at most `max_out` per call)."""
        return self._device_windows(
            functools.partial(self._lib.arroyo_b200_op_handle_watermark_device_poll, self._h), max_out, drain)

    def handle_checkpoint(self, barrier, ctx: OperatorContext, collector: Collector):
        if not self.created:
            return
        w = ctx.watermark()
        wm = ffi.INT64_MIN if (w is None or w == "idle") else clamp_watermark(w)
        out = ffi.Batches()
        st = self._lib.arroyo_b200_op_handle_checkpoint(self._h, wm, C.byref(out))
        _check(self._lib, self._h, st)
        table = ctx.table("t", int(self.config.width))
        names = self.partial_names()
        for b in import_batches(self._lib, out):
            b = pa.RecordBatch.from_arrays(b.columns, names=names)
            table.insert(int(b.column(len(names) - 1)[0].value), b)

    def on_close(self, final_message, ctx: OperatorContext, collector: Collector):
        if self.created:
            self.flush()


class TumblingAggregatingWindowFunc(_WindowAggregate):
    """arroyo-worker/src/arrow/tumbling_aggregating_window.rs"""
    kind = ffi.TUMBLING_AGGREGATE

    def name(self):
        return "tumbling_window"


class SlidingAggregatingWindowFunc(_WindowAggregate):
    """arroyo-worker/src/arrow/sliding_aggregating_window.rs"""
    kind = ffi.SLIDING_AGGREGATE

    def name(self):
        return "sliding_window"


class InstantAggregatingWindowFunc(_WindowAggregate):
    """tumbling_aggregating_window.rs with width 0: the instant window the planner puts behind an upstream window
    (arroyo-planner extension/aggregate.rs:233-289).  Each `_timestamp` is one bin; at watermark w every instant < w
    leaves in ascending order.  `config.width` is 0.  `final_projection=False` gives [keys, aggs, _timestamp];
    `final_projection=True` is the nested form: window{start = ts - nested_width + 1, end = ts + 1} at `window_index`,
    `_timestamp = instant`.  Table "t" (retention 0) holds per instant the partial rows since the previous checkpoint."""
    kind = ffi.INSTANT_AGGREGATE

    def name(self):
        return "instant_window"

    def _width_ns(self) -> int:
        c = self.config
        if int(c.width) != 0:
            raise ffi.ArroyoB200Error(ffi.INVALID_ARGUMENT, "the instant window has width 0")
        return int(getattr(c, "nested_width", 0)) if c.final_projection else 0


_WINDOW_FNS = {"row_number": ffi.FN_ROW_NUMBER, "rank": ffi.FN_RANK, "dense_rank": ffi.FN_DENSE_RANK}
_WINDOW_AGGS = {"count": ffi.AGG_COUNT_STAR, "sum": ffi.AGG_SUM_I64, "avg": ffi.AGG_AVG_I64, "min": ffi.AGG_MIN_I64,
                "max": ffi.AGG_MAX_I64}
_WINDOW_VALUES = {"lag": ffi.FN_LAG, "lead": ffi.FN_LEAD, "first_value": ffi.FN_FIRST_VALUE,
                  "last_value": ffi.FN_LAST_VALUE, "nth_value": ffi.FN_NTH_VALUE}
_WINDOW_DISTS = {"percent_rank": ffi.FN_PERCENT_RANK, "cume_dist": ffi.FN_CUME_DIST}


def flat_names(schema: pa.Schema) -> List[str]:
    """The window function's flat columns: a struct column's children take its place as `<struct>_<child>`."""
    return [name for name, _ in _flat_fields(schema)]


def _flat_fields(schema: pa.Schema):
    fields = []
    for f in schema:
        if pa.types.is_struct(f.type):
            fields += [(f"{f.name}_{c.name}", c.type) for c in f.type]
        else:
            fields.append((f.name, f.type))
    return fields


_FRAME_UNITS = {"rows": ffi.FRAME_ROWS, "range": ffi.FRAME_RANGE, "groups": ffi.FRAME_GROUPS}
_FRAME_BOUNDS = {"unbounded_preceding": ffi.BOUND_UNBOUNDED_PRECEDING, "preceding": ffi.BOUND_PRECEDING,
                 "current_row": ffi.BOUND_CURRENT_ROW, "following": ffi.BOUND_FOLLOWING,
                 "unbounded_following": ffi.BOUND_UNBOUNDED_FOLLOWING}


def _frame_bound(bound):
    """A WindowFrame bound as (ArroyoB200FrameBound code, offset): a bare kind, or ("preceding" | "following", n).
    The library checks the offset's sign; one outside Int64 is refused here, before ctypes would wrap it."""
    kind, n = (bound, 0) if isinstance(bound, str) else bound
    if kind not in _FRAME_BOUNDS or (kind in ("preceding", "following")) != (not isinstance(bound, str)):
        raise ffi.ArroyoB200Error(ffi.INVALID_ARGUMENT, f"frame bound {bound!r}")
    if not ffi.INT64_MIN <= int(n) <= ffi.INT64_MAX:
        raise ffi.ArroyoB200Error(ffi.INVALID_ARGUMENT, f"frame offset {n} outside Int64")
    return _FRAME_BOUNDS[kind], int(n)


def _default_bits(value, arrow_type) -> int:
    """LAG / LEAD's default as the signed 64 bits of the argument's type: a Float64's IEEE bits, else the integer
    modulo 2^64."""
    if arrow_type is not None and pa.types.is_floating(arrow_type):
        return struct.unpack("<q", struct.pack("<d", float(value)))[0]
    return ((int(value) + (1 << 63)) % (1 << 64)) - (1 << 63)


class WindowFunction(_WindowAggregate):
    """window_fn.rs: ROW_NUMBER / RANK / DENSE_RANK per instant (each upstream window stamps its rows with one
    `_timestamp`) and partition key, with the fused `WHERE fn <= top_n`, COUNT / SUM / AVG / MIN / MAX of
    `config.argument` over the default frame, LAG / LEAD / FIRST_VALUE / LAST_VALUE / NTH_VALUE of `config.argument`,
    or PERCENT_RANK / CUME_DIST; the aggregates and FIRST_VALUE / LAST_VALUE / NTH_VALUE over `config.frame` when one is
    given.  At watermark w every instant < w leaves in one batch: the input columns, struct columns included, then the
    function column `config.name` (UInt64 for a rank, Float64 for avg, percent_rank and cume_dist, the argument's type
    for a value function, else Int64; lag / lead / nth_value, and under an explicit frame every function but count,
    are nullable).  Columns
    are named in the config by their flat names (`flat_names`).  Table "input" (retention 0) holds per instant the input
    rows since the previous checkpoint.  Device-resident input is flat; a schema given at construction declares the
    column types to the library, which device batches do not carry."""
    kind = ffi.WINDOW_FUNCTION

    def __init__(self, config, input_schema: Optional[pa.Schema] = None, **kw):
        _NativeOperator.__init__(self, **kw)
        self.config = config
        self._names: Optional[List[str]] = None
        if input_schema is not None:
            self._build(input_schema.names, input_schema)

    def name(self):
        return "window_function"

    def _build(self, names: List[str], schema: Optional[pa.Schema] = None):
        c = self.config
        agg, value = c.function in _WINDOW_AGGS, c.function in _WINDOW_VALUES
        codes = {**_WINDOW_FNS, **_WINDOW_VALUES, **_WINDOW_DISTS, **{f: ffi.FN_AGGREGATE for f in _WINDOW_AGGS}}
        if c.function not in codes:
            raise ffi.UnsupportedPlan(ffi.UNSUPPORTED, f"window function {c.function}")
        if c.function not in _WINDOW_FNS and c.top_n != 0:
            raise ffi.ArroyoB200Error(ffi.INVALID_ARGUMENT, f"{c.function} takes no top N filter")
        if c.default is not None and c.function not in ("lag", "lead"):
            raise ffi.ArroyoB200Error(ffi.INVALID_ARGUMENT, f"{c.function} takes no default")
        fields = [(n, None) for n in names] if schema is None else _flat_fields(schema)
        flat = [n for n, _ in fields]
        cfg = ffi.OpConfig()
        cfg.kind = self.kind
        cfg.window_fn = codes[c.function]
        cfg.n_cols = len(flat)
        cfg.timestamp_col = flat.index(TIMESTAMP)
        cfg.n_key_cols = 0 if c.partition_by is None else 1
        cfg.key_col = 0 if c.partition_by is None else flat.index(c.partition_by)
        if len(c.order_by) > ffi.MAX_ORDER_KEYS:
            raise ffi.ArroyoB200Error(ffi.INVALID_ARGUMENT, "more than 4 ORDER BY keys")
        first = 0
        if agg:  # aggs[0] is the aggregate, the ORDER BY keys follow
            cfg.aggs[0].kind = _WINDOW_AGGS[c.function]
            cfg.aggs[0].input_col = 0 if c.function == "count" else flat.index(c.argument)
            first = 1
        if value:  # aggs[0] is the argument, the ORDER BY keys follow
            cfg.aggs[0].kind = ffi.FN_ARGUMENT
            cfg.aggs[0].input_col = flat.index(c.argument)
            first = 1
            if c.function in ("lag", "lead", "nth_value"):
                cfg.width_ns = int(c.offset)
            if c.default is not None:
                cfg.flags |= ffi.FLAG_FN_DEFAULT
                cfg.gap_ns = _default_bits(c.default, fields[cfg.aggs[0].input_col][1])
        cfg.n_aggs = first + len(c.order_by)
        for i, (col, desc) in enumerate(c.order_by):
            cfg.aggs[first + i].kind = ffi.ORDER_DESC if desc else ffi.ORDER_ASC
            cfg.aggs[first + i].input_col = flat.index(col)
        cfg.slide_ns = int(c.top_n)
        if c.frame is not None:
            if c.frame.units not in _FRAME_UNITS:
                raise ffi.ArroyoB200Error(ffi.INVALID_ARGUMENT, f"frame units {c.frame.units!r}")
            cfg.frame.units = _FRAME_UNITS[c.frame.units]
            cfg.frame.start_kind, cfg.frame.start_offset = _frame_bound(c.frame.start)
            cfg.frame.end_kind, cfg.frame.end_offset = _frame_bound(c.frame.end)
        self._create(cfg)
        self._names = list(names)
        if schema is not None:
            # a zero-row batch declares the column types (device batches carry none)
            empty = pa.RecordBatch.from_arrays([pa.array([], f.type) for f in schema], schema=schema)
            self._process_batch(self._lib.arroyo_b200_op_process_batch, 0, 1, empty)

    def _ensure(self, schema: pa.Schema):
        if not self.created:
            self._build(schema.names, schema)

    def output_names(self) -> List[str]:
        return list(self._names) + [self.config.name]

    def state_names(self) -> List[str]:
        return list(self._names)

    def tables(self):
        return {"input": 0}

    def on_start(self, ctx: OperatorContext):
        wm = ctx.last_present_watermark()
        batches = [b for _, b in ctx.table("input", 0).all_batches_for_watermark(wm)]
        if not batches and not self.created:
            return
        if not self.created:
            self._ensure(batches[0].schema)
        self._on_start(batches, ffi.INT64_MIN if wm is None else clamp_watermark(wm), ffi.INT64_MIN)

    def process_batch(self, batch: pa.RecordBatch, ctx: OperatorContext, collector: Collector):
        self._ensure(batch.schema)
        self._process_batch(self._lib.arroyo_b200_op_process_batch, 0, 1, batch)

    def run_batches(self, exported: "ExportedBatches", watermarks, collector: Collector, first: int = 0,
                    count: Optional[int] = None, async_emit: bool = True):
        if not self.created:
            raise ffi.ArroyoB200Error(ffi.INVALID_ARGUMENT, "run_batches needs input_schema at construction")
        super().run_batches(exported, watermarks, collector, first, count, async_emit)

    def handle_checkpoint(self, barrier, ctx: OperatorContext, collector: Collector):
        if not self.created:
            return
        out = ffi.Batches()
        _check(self._lib, self._h, self._lib.arroyo_b200_op_handle_checkpoint(self._h, ffi.INT64_MIN, C.byref(out)))
        table = ctx.table("input", 0)
        names = self.state_names()
        for b in import_batches(self._lib, out):
            b = pa.RecordBatch.from_arrays(b.columns, names=names)
            table.insert(b.column(names.index(TIMESTAMP)).cast(pa.int64())[0].as_py(), b)


class SessionAggregatingWindowFunc(_NativeOperator):
    """arroyo-worker/src/arrow/session_aggregating_window.rs.  Output = [key cols...] with the window struct
    inserted at `window_index`, [agg cols...], `_timestamp = window.end - 1 ns` (:316-382)."""
    kind = ffi.SESSION_AGGREGATE

    def __init__(self, config, input_schema: Optional[pa.Schema] = None, **kw):
        super().__init__(**kw)
        self.config = config
        if input_schema is not None:
            self._build(input_schema.names)

    def name(self):
        return "session_window"

    def tables(self):
        # "s": raw sorted input batches, retention gap x 100; "e": earliest start per subtask (:927-941)
        return {"s": int(self.config.gap) * 100, "e": 0}

    def _build(self, names: List[str]):
        cfg = _agg_config(self.kind, self.config, names)
        cfg.gap_ns = int(self.config.gap)
        cfg.window_index = int(self.config.window_index)
        self._create(cfg)

    def output_names(self) -> List[str]:
        c = self.config
        names = list(c.key_names)
        names.insert(min(max(c.window_index, 0), len(names)), "window")
        return names + [a.name for a in c.aggs] + [TIMESTAMP]

    def _set_watermark(self, ctx: OperatorContext):
        """A new operator takes the last watermark before its first batch (on_start with nothing to restore): the
        library only learns watermarks from handle_watermark and on_start, and without one it would treat every row as
        on time."""
        wm = ctx.last_present_watermark()
        if wm is None or not self.created:
            return
        self._on_start([], clamp_watermark(wm), ffi.INT64_MIN)

    def process_batch(self, batch: pa.RecordBatch, ctx: OperatorContext, collector: Collector):
        if not self.created:
            self._build(batch.schema.names)
            self._set_watermark(ctx)
        # Table "s" holds the raw input rows that passed the late filter, keyed by the batch's newest timestamp
        # (session_aggregating_window.rs:858-883).  The shim owns the table: it keeps the on-time rows of the batch it
        # is about to hand over (the reference also sorts them; restore re-sorts, :829, so the order is not state).
        wm = ctx.last_present_watermark()
        kept = batch
        if wm is not None:
            import pyarrow.compute as pc
            ts = batch.column(batch.schema.names.index(TIMESTAMP)).cast(pa.int64())
            kept = batch.filter(pc.greater_equal(ts, min(wm, (1 << 63) - 1)))
        if kept.num_rows:
            ts = kept.column(kept.schema.names.index(TIMESTAMP)).cast(pa.int64())
            import pyarrow.compute as pc
            ctx.table("s", int(self.config.gap) * 100).insert(int(pc.max(ts).as_py()), kept)
        self._process_batch(self._lib.arroyo_b200_op_process_batch, 0, 1, batch)

    def process_device_batch(self, cols: List[int], n_rows: int):
        """Device-resident input (operator chaining): the rows never reach the host, so table "s" is not maintained
        and such a subtask cannot be restored from a checkpoint."""
        arr = (C.c_uint64 * len(cols))(*cols)
        _check(self._lib, self._h, self._lib.arroyo_b200_op_process_device_batch(self._h, 0, 1, arr, len(cols), n_rows))

    def handle_checkpoint(self, barrier, ctx: OperatorContext, collector: Collector):
        """session_aggregating_window.rs:907-925: flush table "s" at the watermark, publish this subtask's
        earliest_batch_time() in the global table "e"."""
        wm = ctx.last_present_watermark()
        ctx.table("s", int(self.config.gap) * 100).flush(wm)
        earliest = None
        if self.created:
            out = ffi.Batches()
            st = self._lib.arroyo_b200_op_handle_checkpoint(self._h, ffi.INT64_MIN if wm is None else clamp_watermark(wm),
                                                            C.byref(out))
            _check(self._lib, self._h, st)
            for b in import_batches(self._lib, out):
                if b.num_rows:
                    earliest = int(b.column(0).cast(pa.int64())[0].as_py())
        ctx.global_table("e")[ctx.task_index] = earliest

    def on_start(self, ctx: OperatorContext):
        """session_aggregating_window.rs:802-847."""
        starts = [v for v in ctx.global_table("e").values() if v is not None]
        if not starts:
            self._set_watermark(ctx)
            return
        start_time = min(starts)
        table = ctx.table("s", int(self.config.gap) * 100)
        batches = [b for _, b in table.all_batches_for_watermark(start_time)]
        if not self.created:
            if not batches:
                return
            self._build(batches[0].schema.names)
        wm = ctx.last_present_watermark()
        self._on_start(batches, ffi.INT64_MIN if wm is None else clamp_watermark(wm), start_time)

    def handle_watermark(self, watermark, ctx: OperatorContext, collector: Collector):
        wm = ctx.last_present_watermark()
        if wm is None or not self.created:
            return watermark
        out = ffi.Batches()
        _check(self._lib, self._h, self._lib.arroyo_b200_op_handle_watermark(self._h, clamp_watermark(wm), C.byref(out)))
        self._collect(out, collector)
        return watermark

    def handle_watermark_device(self, wm: int, max_out: int = 4):
        return self._device_windows(
            functools.partial(self._lib.arroyo_b200_op_handle_watermark_device, self._h, clamp_watermark(wm)), max_out)


class UpdatingAggregatingFunc(_NativeOperator):
    """arroyo-worker/src/arrow/incremental_aggregator.rs (`IncrementalAggregatingFunc`): the non-windowed GROUP BY.
    Change rows leave on ticks (`tick_interval` = flush interval, :990-1004), at checkpoints (:951-961) and at end of
    data (:1006-1018): [key cols..., aggregates..., _timestamp, _is_retract].  `config`: anything with `key_names`
    and `aggs` (oracle.updating_oracle.UpdatingAggConfig has the shape).  Append-only inputs only.

    State: a checkpoint also writes the accumulators of the keys flushed since the last checkpoint to the key-value
    table "a" (`state_names()` columns, :619-635), and `on_start` restores them from it (:446-503).

    Time-to-idle: `ttl` in ns, read as the reference reads `ttl_micros` (0 means 24 h, :1043-1048); a flush then
    retracts and drops every key idle for at least `ttl` on the clock `clock()` (ns, default time.monotonic_ns), which
    is passed to the library before every call that ingests, flushes or restores.  `ttl=None`: keys never expire and
    the clock is never read."""
    kind = ffi.UPDATING_AGGREGATE
    IS_RETRACT = "_is_retract"
    DEFAULT_TTL_NS = 24 * 60 * 60 * 1_000_000_000

    def __init__(self, config, input_schema: Optional[pa.Schema] = None, updating_input: bool = False,
                 ttl: Optional[int] = None, clock=None, **kw):
        super().__init__(**kw)
        self.config = config
        self.updating_input = updating_input
        self.ttl = None if ttl is None else (int(ttl) or self.DEFAULT_TTL_NS)
        self.clock = clock or time.monotonic_ns
        self._key_type = None
        if input_schema is not None:
            self._build(input_schema.names)
            self._note_key_type(input_schema)

    def name(self):
        return "UpdatingAggregatingFunc"

    def _note_key_type(self, schema: pa.Schema):
        if self.config.key_names:
            self._key_type = schema.field(self.config.key_names[0]).type

    def tables(self):
        # accumulator state / batch state (:963-988); "b" (count(distinct ...)) stays empty: such plans are refused
        return {"a": 0, "b": 0}

    def state_names(self) -> List[str]:
        """Columns of table "a": keys, each aggregate's accumulator state, `_timestamp`, `_generation`."""
        names = list(self.config.key_names)
        fields = {"count": ["count"], "sum": ["sum", "count"], "avg": ["count", "sum"], "min": ["min"], "max": ["max"]}
        for a in self.config.aggs:
            names += [f"{a.name}[{f}]" for f in fields[a.kind]]
        return names + [TIMESTAMP, "_generation"]

    def on_start(self, ctx: OperatorContext):
        batches = list(ctx.key_value_table("a").get_all())
        if not batches:
            return
        if not self.created:
            raise ffi.ArroyoB200Error(ffi.INVALID_ARGUMENT, "restore needs input_schema at construction")
        self._tick_clock()
        self._on_start(batches, ffi.INT64_MIN, ffi.INT64_MIN)

    def _build(self, names: List[str]):
        cfg = _agg_config(self.kind, self.config, names)
        cfg.gap_ns = self.ttl or 0
        if self.updating_input:
            self._flags |= ffi.FLAG_UPDATING_INPUT
        self._create(cfg)

    def _tick_clock(self):
        """arroyo_b200_op_set_clock(clock()) before a call that stamps, expires or restores (with a ttl only)."""
        if self.ttl is not None and self.created:
            _check(self._lib, self._h, self._lib.arroyo_b200_op_set_clock(self._h, int(self.clock())))

    def output_names(self) -> List[str]:
        return list(self.config.key_names) + [a.name for a in self.config.aggs] + [TIMESTAMP, self.IS_RETRACT]

    def process_batch(self, batch: pa.RecordBatch, ctx: OperatorContext, collector: Collector):
        if not self.created:
            self._build(batch.schema.names)
        self._note_key_type(batch.schema)
        self._tick_clock()
        self._process_batch(self._lib.arroyo_b200_op_process_batch, 0, 1, batch)

    def process_device_batch(self, cols: List[int], n_rows: int):
        """`cols` = device pointers (ints), one per input column; needs `input_schema` at construction."""
        arr = (C.c_uint64 * len(cols))(*cols)
        self._tick_clock()
        _check(self._lib, self._h, self._lib.arroyo_b200_op_process_device_batch(self._h, 0, 1, arr, len(cols), n_rows))

    def process_device_batches(self, cols_flat, n_rows, n_cols: int):
        """A run of device batches in one FFI call; `cols_flat`/`n_rows` are prebuilt ctypes arrays
        ((c_uint64 * (n_batches * n_cols)), (c_int64 * n_batches))."""
        self._tick_clock()
        st = self._lib.arroyo_b200_op_process_device_batches(self._h, 0, 1, cols_flat, n_cols, n_rows, len(n_rows))
        _check(self._lib, self._h, st)

    def handle_watermark(self, watermark, ctx: OperatorContext, collector: Collector):
        return watermark

    def _typed(self, out, names) -> List[pa.RecordBatch]:
        res = []
        for b in import_batches(self._lib, out):
            cols = b.columns
            # device batches carry no Arrow types: the key column leaves with the input schema's key type
            if self._key_type is not None and cols[0].type != self._key_type:
                cols = [cols[0].view(self._key_type)] + cols[1:]
            res.append(pa.RecordBatch.from_arrays(cols, names=names))
        return res

    def _emit(self, out, collector: Collector):
        for b in self._typed(out, self.output_names()):
            collector.collect(b)

    def handle_tick(self, tick, ctx: OperatorContext, collector: Collector):
        if not self.created:
            return
        out = ffi.Batches()
        self._tick_clock()
        _check(self._lib, self._h, self._lib.arroyo_b200_op_handle_tick(self._h, C.byref(out)))
        self._emit(out, collector)

    def handle_checkpoint(self, barrier, ctx: OperatorContext, collector: Collector):
        if not self.created:
            return
        out = ffi.Batches()
        self._tick_clock()
        _check(self._lib, self._h, self._lib.arroyo_b200_op_handle_checkpoint(self._h, ffi.INT64_MIN, C.byref(out)))
        self._emit(out, collector)
        if ctx is not None:  # then the state of the keys flushed since the last checkpoint (:951-961)
            self.checkpoint_state(ctx.key_value_table("a"))

    def checkpoint_state(self, table):
        """arroyo_b200_op_checkpoint_state: inserts the state rows of the keys flushed since the last call into
        `table` (a KeyValueTable)."""
        out = ffi.Batches()
        _check(self._lib, self._h, self._lib.arroyo_b200_op_checkpoint_state(self._h, C.byref(out)))
        for b in self._typed(out, self.state_names()):
            table.insert_batch(b)

    def on_close(self, final_message, ctx: OperatorContext, collector: Collector):
        if not self.created:
            return
        out = ffi.Batches()
        self._tick_clock()
        _check(self._lib, self._h, self._lib.arroyo_b200_op_on_close(self._h, 1 if final_message == "end_of_data" else 0,
                                                                      C.byref(out)))
        self._emit(out, collector)


_JOIN_TYPES = {"inner": ffi.JOIN_INNER, "left": ffi.JOIN_LEFT, "right": ffi.JOIN_RIGHT, "full": ffi.JOIN_FULL}


class InstantJoin(_NativeOperator):
    """arroyo-worker/src/arrow/instant_join.rs.  Inputs with index < in_partitions / 2 are the left side
    (:249-253).  The native operator needs both input layouts, so batches are buffered until each side's
    schema is known (pass `left_schema` / `right_schema` to skip that)."""
    kind = ffi.INSTANT_JOIN

    def __init__(self, config, left_schema: Optional[pa.Schema] = None, right_schema: Optional[pa.Schema] = None, **kw):
        super().__init__(**kw)
        self.config = config
        self._schemas = [left_schema, right_schema]
        self._buffered = []
        if left_schema is not None and right_schema is not None:
            self._build()

    def name(self):
        return "InstantJoin"

    def tables(self):
        return {"left": 0, "right": 0}  # instant_join.rs:305-328

    def _side_layout(self, side: int):
        c = self.config
        names = self._schemas[side].names
        routing = c.left_routing_keys if side == 0 else c.right_routing_keys
        on = c.left_on if side == 0 else c.right_on
        if len(on) != 1:
            raise ffi.UnsupportedPlan(ffi.UNSUPPORTED, "only single-column equi-joins are supported")
        if list(names[:len(routing)]) != list(routing):
            raise ffi.ArroyoB200Error(ffi.INVALID_ARGUMENT, "routing key columns must lead the schema")
        return len(names), names.index(TIMESTAMP), names.index(on[0]), len(routing)

    def _build(self):
        cfg = ffi.OpConfig()
        cfg.kind = self.kind
        cfg.join_type = _JOIN_TYPES[self.config.join_type]
        cfg.n_cols, cfg.timestamp_col, cfg.left_key_col, cfg.left_n_routing = self._side_layout(0)
        cfg.right_n_cols, cfg.right_timestamp_col, cfg.right_key_col, cfg.right_n_routing = self._side_layout(1)
        self._create(cfg)
        for index, parts, batch in self._buffered:
            self._send(index, parts, batch)
        self._buffered = []

    def output_names(self):
        out = []
        for side in (0, 1):
            names = self._schemas[side].names
            routing = self.config.left_routing_keys if side == 0 else self.config.right_routing_keys
            for n in names[len(routing):]:
                if n == TIMESTAMP:
                    continue
                out.append(n if n not in out else n + "_right")
        return out + [TIMESTAMP]

    def _send(self, index, parts, batch):
        self._process_batch(self._lib.arroyo_b200_op_process_batch, index, parts, batch)

    def on_start(self, ctx: OperatorContext):
        """instant_join.rs:205-247: every batch of table "left" goes back through process_left, every batch of table
        "right" through process_right (which also re-inserts them into the tables, :116-128)."""
        wm = ctx.last_present_watermark()
        replay = []
        for side, name in enumerate(("left", "right")):
            replay.append([b for _, b in ctx.table(name, 0).all_batches_for_watermark(wm)])
        if self.created and wm is not None:
            self._on_start([], clamp_watermark(wm), ffi.INT64_MIN)
        for side, batches in enumerate(replay):
            for b in batches:
                self.process_batch_index(side, 2, b, ctx, None)

    def handle_checkpoint(self, barrier, ctx: OperatorContext, collector: Collector):
        """instant_join.rs:285-303: both tables are flushed at the watermark (retention 0)."""
        wm = ctx.last_present_watermark()
        ctx.table("left", 0).flush(wm)
        ctx.table("right", 0).flush(wm)

    def process_batch_index(self, index: int, in_partitions: int, batch: pa.RecordBatch, ctx: OperatorContext,
                            collector: Collector):
        side = index // (in_partitions // 2)
        if batch.num_rows:
            # process_side (:116-128): the raw batch goes into the side's table under its newest timestamp
            import pyarrow.compute as pc
            ts = batch.column(batch.schema.names.index(TIMESTAMP)).cast(pa.int64())
            ctx.table("left" if side == 0 else "right", 0).insert(int(pc.max(ts).as_py()), batch)
        if self._schemas[side] is None:
            self._schemas[side] = batch.schema
        if not self.created:
            if self._schemas[0] is not None and self._schemas[1] is not None:
                self._build()
            else:
                self._buffered.append((index, in_partitions, batch))
                return
        self._send(index, in_partitions, batch)

    def handle_watermark(self, watermark, ctx: OperatorContext, collector: Collector):
        wm = ctx.last_present_watermark()
        if wm is None:
            return watermark
        if not self.created:
            # one side never produced a row: nothing can match; an inner join emits nothing
            if self.config.join_type == "inner":
                self._buffered = []
                return wm
            known = 0 if self._schemas[0] is not None else 1
            self._schemas[1 - known] = pa.schema([("__none", pa.int64()), (TIMESTAMP, pa.timestamp("ns"))])
            saved = (self.config.left_on, self.config.right_on)
            if known == 0:
                self.config.right_on = ["__none"]
            else:
                self.config.left_on = ["__none"]
            try:
                self._build()
            finally:
                self.config.left_on, self.config.right_on = saved
        out = ffi.Batches()
        _check(self._lib, self._h, self._lib.arroyo_b200_op_handle_watermark(self._h, clamp_watermark(wm), C.byref(out)))
        self._collect(out, collector)
        return wm


DAY_NS = 24 * 3600 * 10 ** 9


class JoinWithExpiration(InstantJoin):
    """arroyo-worker/src/arrow/join_with_expiration.rs: the non-windowed join (inner, append-only inputs).  Every
    matching pair leaves once, from the `process_batch_index` call that brings its later row (:42-108).

    State: every non-empty input batch goes into its side's key-time table, "left" or "right", under its newest
    `_timestamp` (KeyTimeView::insert, arroyo-state/src/tables/expiring_time_key_map.rs:997-1006), and a checkpoint
    flushes both tables at the watermark.  After `on_start` the first batch loads both tables from watermark - ttl on
    (get_key_time_view :200-236) and hands them to arroyo_b200_op_restore_side: the restored rows join their side's
    stored rows and are never paired with each other (insert_internal :1008-1049)."""
    kind = ffi.TTL_JOIN

    def __init__(self, config, left_schema: Optional[pa.Schema] = None, right_schema: Optional[pa.Schema] = None, **kw):
        self._restore_pending = False
        self._restored = [[], []]  # per side: table batches that wait for the operator to be built
        super().__init__(config, left_schema, right_schema, **kw)

    def name(self):
        return "JoinWithExpiration"

    def ttl(self) -> int:
        """The tables' retention in ns: `config.ttl`, where 0 means 24 h (join_with_expiration.rs:239-248)."""
        return int(getattr(self.config, "ttl", 0) or 0) or DAY_NS

    def tables(self):
        return {"left": self.ttl(), "right": self.ttl()}  # key-time tables (:228-262)

    def _table(self, ctx: OperatorContext, side: int):
        return ctx.table("left" if side == 0 else "right", self.ttl())

    def on_start(self, ctx: OperatorContext):
        """Nothing is read yet: like the reference, the first batch after the restart loads both tables, with the
        watermark of that moment (process_left / process_right -> get_key_time_table)."""
        self._restore_pending = True

    def _restore(self, ctx: OperatorContext):
        wm = ctx.last_present_watermark()
        for side in (0, 1):
            batches = [b for _, b in self._table(ctx, side).all_batches_for_watermark(wm)]
            if not batches:
                continue
            if self._schemas[side] is None:
                self._schemas[side] = batches[0].schema
            if self.created:
                self._restore_side(side, batches)
            else:
                self._restored[side] += batches
        if not self.created and self._schemas[0] is not None and self._schemas[1] is not None:
            self._build()

    def _restore_side(self, side: int, batches: List[pa.RecordBatch]):
        if batches:
            self._hand_over_state(
                lambda a, s, n: self._lib.arroyo_b200_op_restore_side(self._h, side, a, s, n), batches)

    def _build(self):
        """Creates the operator, then restores the table batches that waited for it, then sends the buffered input."""
        buffered, self._buffered = self._buffered, []
        super()._build()
        restored, self._restored = self._restored, [[], []]
        for side in (0, 1):
            self._restore_side(side, restored[side])
        for index, parts, batch in buffered:
            self._send(index, parts, batch)

    def handle_checkpoint(self, barrier, ctx: OperatorContext, collector: Collector):
        """The tables keep what is at or after watermark - ttl (the checkpointer, expiring_time_key_map.rs:747-760)."""
        wm = ctx.last_present_watermark()
        for side in (0, 1):
            self._table(ctx, side).flush(wm)

    def _send(self, index, parts, batch, collector=None):
        out = ffi.Batches()
        self._process_batch(self._lib.arroyo_b200_op_process_batch_emit, index, parts, batch, out)
        self._collect(out, collector)

    def process_batch_index(self, index: int, in_partitions: int, batch: pa.RecordBatch, ctx: OperatorContext,
                            collector: Collector):
        side = index // (in_partitions // 2)
        if self._restore_pending:
            self._restore_pending = False
            self._restore(ctx)
        if self._schemas[side] is None:
            self._schemas[side] = batch.schema
        if self.created or (self._schemas[0] is not None and self._schemas[1] is not None):
            if not self.created:
                self._build()
            self._send(index, in_partitions, batch, collector)
        else:
            self._buffered.append((index, in_partitions, batch))
        if batch.num_rows:  # the table takes the batches the operator took (KeyTimeView::insert)
            import pyarrow.compute as pc
            ts = batch.column(batch.schema.names.index(TIMESTAMP)).cast(pa.int64())
            self._table(ctx, side).insert(int(pc.max(ts).as_py()), batch)

    def handle_watermark(self, watermark, ctx: OperatorContext, collector: Collector):
        return watermark
