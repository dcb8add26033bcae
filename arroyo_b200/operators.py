"""Host-side mirror of the reference's window operators over the C ABI.

Class and method names follow arroyo-worker/src/arrow/{tumbling,sliding}_aggregating_window.rs and
the ArrowOperator trait (arroyo-operator/src/operator.rs:1143-1257): name(), tables(), on_start(ctx),
process_batch(batch, ctx, collector), handle_watermark(watermark, ctx, collector),
handle_checkpoint(barrier, ctx, collector), on_close(final_message, ctx, collector).
Batches are pyarrow RecordBatches crossing the boundary through the Arrow C Data Interface."""
import ctypes as C
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
        cfg.flags = self._flags
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
        cfg = ffi.OpConfig()
        cfg.kind = self.kind
        cfg.width_ns = int(c.width)
        cfg.slide_ns = int(getattr(c, "slide", 0) or 0)
        cfg.n_cols = len(names)
        cfg.timestamp_col = names.index(TIMESTAMP)
        if len(c.key_names) > 1:
            raise ffi.UnsupportedPlan(ffi.UNSUPPORTED, "more than one group-by key column")
        cfg.n_key_cols = len(c.key_names)
        cfg.key_col = names.index(c.key_names[0]) if c.key_names else 0
        if len(c.aggs) > ffi.MAX_AGGS:
            raise ffi.UnsupportedPlan(ffi.UNSUPPORTED, "too many aggregates")
        cfg.n_aggs = len(c.aggs)
        for i, a in enumerate(c.aggs):
            if a.kind not in _AGG_KINDS:
                raise ffi.UnsupportedPlan(ffi.UNSUPPORTED, f"aggregate {a.kind}")
            cfg.aggs[i].kind = _AGG_KINDS[a.kind]
            cfg.aggs[i].input_col = names.index(a.col) if a.col is not None else 0
        pc = getattr(c, "partial_count_col", None)
        cfg.partial_count_col_plus1 = names.index(pc) + 1 if pc else 0
        cfg.final_projection = 1 if c.final_projection else 0
        cfg.window_index = int(c.window_index)
        self._create(cfg)
        self._names = list(names)

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
        n = len(batches)
        arrs = (ffi.ArrowArray * max(n, 1))()
        schs = (ffi.ArrowSchema * max(n, 1))()
        for i, b in enumerate(batches):
            b._export_to_c(C.addressof(arrs[i]), C.addressof(schs[i]))
        mt = table.get_min_time()
        st = self._lib.arroyo_b200_op_on_start(
            self._h, arrs, schs, n, ffi.INT64_MIN if wm is None else clamp_watermark(wm),
            ffi.INT64_MIN if mt is None else mt)
        _check(self._lib, self._h, st)

    def process_batch(self, batch: pa.RecordBatch, ctx: OperatorContext, collector: Collector):
        if not self.created:
            self._build(batch.schema.names)
        arr, sch = export_batch(batch)
        st = self._lib.arroyo_b200_op_process_batch(self._h, 0, 1, C.byref(arr), C.byref(sch))
        if st != ffi.OK:
            # on error the caller keeps ownership of the exported structs
            for s in (arr, sch):
                if s.release:
                    C.CFUNCTYPE(None, C.c_void_p)(s.release)(C.addressof(s))
        _check(self._lib, self._h, st)
        # the schema struct stays ours
        if sch.release:
            C.CFUNCTYPE(None, C.c_void_p)(sch.release)(C.addressof(sch))

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
        st = self._lib.arroyo_b200_op_handle_watermark(self._h, clamp_watermark(wm), C.byref(out))
        _check(self._lib, self._h, st)
        names = self.output_names()
        for b in import_batches(self._lib, out):
            collector.collect(pa.RecordBatch.from_arrays(b.columns, names=names))
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
        names = self.output_names()
        for b in import_batches(self._lib, out):
            collector.collect(pa.RecordBatch.from_arrays(b.columns, names=names))
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
        names = self.output_names()
        for b in import_batches(self._lib, out):
            collector.collect(pa.RecordBatch.from_arrays(b.columns, names=names))
        _check(self._lib, self._h, st)

    def handle_watermark_device(self, wm: int, max_out: int = 64):
        """Emission left on the device: list of (n_rows, [device pointers]).  The library hands out at most `max_out`
        windows per call and queues the rest; they are collected here with further polls."""
        out = getattr(self, "_dev_out", None)
        if out is None or len(out) < max_out:
            out = self._dev_out = (ffi.DeviceBatch * max_out)()  # reused: building it costs more than the call
        n = C.c_int64(0)
        st = self._lib.arroyo_b200_op_handle_watermark_device(self._h, clamp_watermark(wm), out, max_out, C.byref(n))
        _check(self._lib, self._h, st)
        got = [(out[i].n_rows, [out[i].cols[c] for c in range(out[i].n_cols)]) for i in range(n.value)]
        return got + self._drain_device(max_out, n.value)

    def _drain_device(self, max_out: int, n: int):
        got = []
        while n == max_out and max_out > 0:
            more = self.handle_watermark_device_poll(max_out, drain=False)
            got += more
            n = len(more)
        return got

    def handle_watermark_device_begin(self, wm: int):
        """First half of handle_watermark_device: the emission is enqueued, its row counts are not awaited."""
        _check(self._lib, self._h, self._lib.arroyo_b200_op_handle_watermark_device_begin(self._h, clamp_watermark(wm)))

    def handle_watermark_device_poll(self, max_out: int = 64, drain: bool = True):
        """Second half: the windows of the outstanding emission, list of (n_rows, [device pointers]).  With `drain`,
        polls until the library has no window queued (it hands out at most `max_out` per call)."""
        out = getattr(self, "_dev_out", None)
        if out is None or len(out) < max_out:
            out = self._dev_out = (ffi.DeviceBatch * max_out)()
        n = C.c_int64(0)
        _check(self._lib, self._h, self._lib.arroyo_b200_op_handle_watermark_device_poll(self._h, out, max_out, C.byref(n)))
        got = [(out[i].n_rows, [out[i].cols[c] for c in range(out[i].n_cols)]) for i in range(n.value)]
        return got + (self._drain_device(max_out, n.value) if drain else [])

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
        c = self.config
        cfg = ffi.OpConfig()
        cfg.kind = self.kind
        cfg.gap_ns = int(c.gap)
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
        cfg.window_index = int(c.window_index)
        self._create(cfg)

    def output_names(self) -> List[str]:
        c = self.config
        names = list(c.key_names)
        names.insert(min(max(c.window_index, 0), len(names)), "window")
        return names + [a.name for a in c.aggs] + [TIMESTAMP]

    def _send(self, batch: pa.RecordBatch):
        arr, sch = export_batch(batch)
        st = self._lib.arroyo_b200_op_process_batch(self._h, 0, 1, C.byref(arr), C.byref(sch))
        if st != ffi.OK and arr.release:
            C.CFUNCTYPE(None, C.c_void_p)(arr.release)(C.addressof(arr))
        if sch.release:
            C.CFUNCTYPE(None, C.c_void_p)(sch.release)(C.addressof(sch))
        _check(self._lib, self._h, st)

    def process_batch(self, batch: pa.RecordBatch, ctx: OperatorContext, collector: Collector):
        if not self.created:
            self._build(batch.schema.names)
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
        self._send(batch)

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
            return
        start_time = min(starts)
        table = ctx.table("s", int(self.config.gap) * 100)
        batches = [b for _, b in table.all_batches_for_watermark(start_time)]
        if not self.created:
            if not batches:
                return
            self._build(batches[0].schema.names)
        n = len(batches)
        arrs = (ffi.ArrowArray * max(n, 1))()
        schs = (ffi.ArrowSchema * max(n, 1))()
        for i, b in enumerate(batches):
            b._export_to_c(C.addressof(arrs[i]), C.addressof(schs[i]))
        wm = ctx.last_present_watermark()
        st = self._lib.arroyo_b200_op_on_start(self._h, arrs, schs, n,
                                               ffi.INT64_MIN if wm is None else clamp_watermark(wm), start_time)
        _check(self._lib, self._h, st)

    def handle_watermark(self, watermark, ctx: OperatorContext, collector: Collector):
        wm = ctx.last_present_watermark()
        if wm is None or not self.created:
            return watermark
        out = ffi.Batches()
        st = self._lib.arroyo_b200_op_handle_watermark(self._h, clamp_watermark(wm), C.byref(out))
        _check(self._lib, self._h, st)
        names = self.output_names()
        for b in import_batches(self._lib, out):
            collector.collect(pa.RecordBatch.from_arrays(b.columns, names=names))
        return watermark

    def handle_watermark_device(self, wm: int, max_out: int = 4):
        out = (ffi.DeviceBatch * max_out)()
        n = C.c_int64(0)
        st = self._lib.arroyo_b200_op_handle_watermark_device(self._h, clamp_watermark(wm), out, max_out, C.byref(n))
        _check(self._lib, self._h, st)
        got = [(out[i].n_rows, [out[i].cols[c] for c in range(out[i].n_cols)]) for i in range(n.value)]
        while n.value == max_out and max_out > 0:  # windows beyond max_out stay queued in the library
            _check(self._lib, self._h, self._lib.arroyo_b200_op_handle_watermark_device_poll(self._h, out, max_out, C.byref(n)))
            got += [(out[i].n_rows, [out[i].cols[c] for c in range(out[i].n_cols)]) for i in range(n.value)]
        return got


class UpdatingAggregatingFunc(_NativeOperator):
    """arroyo-worker/src/arrow/incremental_aggregator.rs (`IncrementalAggregatingFunc`): the non-windowed GROUP BY.
    Change rows leave on ticks (`tick_interval` = flush interval, :990-1004), at checkpoints (:951-961) and at end of
    data (:1006-1018): [key cols..., aggregates..., _timestamp, _is_retract].  `config`: anything with `key_names`
    and `aggs` (oracle.updating_oracle.UpdatingAggConfig has the shape).  Append-only inputs only."""
    kind = ffi.UPDATING_AGGREGATE
    IS_RETRACT = "_is_retract"

    def __init__(self, config, input_schema: Optional[pa.Schema] = None, updating_input: bool = False, **kw):
        super().__init__(**kw)
        self.config = config
        self.updating_input = updating_input
        if input_schema is not None:
            self._build(input_schema.names)

    def name(self):
        return "UpdatingAggregatingFunc"

    def tables(self):
        return {"a": 0, "b": 0}  # accumulator state / batch state (:963-988): restore is not implemented

    def _build(self, names: List[str]):
        c = self.config
        cfg = ffi.OpConfig()
        cfg.kind = self.kind
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
        if self.updating_input:
            self._flags |= ffi.FLAG_UPDATING_INPUT
        self._create(cfg)

    def output_names(self) -> List[str]:
        return list(self.config.key_names) + [a.name for a in self.config.aggs] + [TIMESTAMP, self.IS_RETRACT]

    def process_batch(self, batch: pa.RecordBatch, ctx: OperatorContext, collector: Collector):
        if not self.created:
            self._build(batch.schema.names)
        arr, sch = export_batch(batch)
        st = self._lib.arroyo_b200_op_process_batch(self._h, 0, 1, C.byref(arr), C.byref(sch))
        if st != ffi.OK and arr.release:
            C.CFUNCTYPE(None, C.c_void_p)(arr.release)(C.addressof(arr))
        if sch.release:
            C.CFUNCTYPE(None, C.c_void_p)(sch.release)(C.addressof(sch))
        _check(self._lib, self._h, st)

    def handle_watermark(self, watermark, ctx: OperatorContext, collector: Collector):
        return watermark

    def _emit(self, out, collector: Collector):
        names = self.output_names()
        for b in import_batches(self._lib, out):
            collector.collect(pa.RecordBatch.from_arrays(b.columns, names=names))

    def handle_tick(self, tick, ctx: OperatorContext, collector: Collector):
        if not self.created:
            return
        out = ffi.Batches()
        _check(self._lib, self._h, self._lib.arroyo_b200_op_handle_tick(self._h, C.byref(out)))
        self._emit(out, collector)

    def handle_checkpoint(self, barrier, ctx: OperatorContext, collector: Collector):
        if not self.created:
            return
        out = ffi.Batches()
        _check(self._lib, self._h, self._lib.arroyo_b200_op_handle_checkpoint(self._h, ffi.INT64_MIN, C.byref(out)))
        self._emit(out, collector)

    def on_close(self, final_message, ctx: OperatorContext, collector: Collector):
        if not self.created:
            return
        out = ffi.Batches()
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
        arr, sch = export_batch(batch)
        st = self._lib.arroyo_b200_op_process_batch(self._h, index, parts, C.byref(arr), C.byref(sch))
        if st != ffi.OK and arr.release:
            C.CFUNCTYPE(None, C.c_void_p)(arr.release)(C.addressof(arr))
        if sch.release:
            C.CFUNCTYPE(None, C.c_void_p)(sch.release)(C.addressof(sch))
        _check(self._lib, self._h, st)

    def on_start(self, ctx: OperatorContext):
        """instant_join.rs:205-247: every batch of table "left" goes back through process_left, every batch of table
        "right" through process_right (which also re-inserts them into the tables, :116-128)."""
        wm = ctx.last_present_watermark()
        replay = []
        for side, name in enumerate(("left", "right")):
            replay.append([b for _, b in ctx.table(name, 0).all_batches_for_watermark(wm)])
        if self.created and wm is not None:
            empty = (ffi.ArrowArray * 1)()
            emptys = (ffi.ArrowSchema * 1)()
            _check(self._lib, self._h, self._lib.arroyo_b200_op_on_start(self._h, empty, emptys, 0, clamp_watermark(wm),
                                                                          ffi.INT64_MIN))
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
        st = self._lib.arroyo_b200_op_handle_watermark(self._h, clamp_watermark(wm), C.byref(out))
        _check(self._lib, self._h, st)
        names = self.output_names()
        for b in import_batches(self._lib, out):
            collector.collect(pa.RecordBatch.from_arrays(b.columns, names=names))
        return wm


class JoinWithExpiration(InstantJoin):
    """arroyo-worker/src/arrow/join_with_expiration.rs: the non-windowed join (inner, append-only inputs).  Every
    matching pair leaves once, from the `process_batch_index` call that brings its later row (:42-108)."""
    kind = ffi.TTL_JOIN

    def name(self):
        return "JoinWithExpiration"

    def tables(self):
        return {"left": 0, "right": 0}  # key-time tables with retention = ttl (:228-262); restore is a replay

    def on_start(self, ctx: OperatorContext):
        raise ffi.UnsupportedPlan(ffi.UNSUPPORTED, "JoinWithExpiration restore: replay the key-time tables through process_batch_index")

    def handle_checkpoint(self, barrier, ctx: OperatorContext, collector: Collector):
        return

    def _send(self, index, parts, batch, collector=None):
        arr, sch = export_batch(batch)
        out = ffi.Batches()
        st = self._lib.arroyo_b200_op_process_batch_emit(self._h, index, parts, C.byref(arr), C.byref(sch), C.byref(out))
        if st != ffi.OK and arr.release:
            C.CFUNCTYPE(None, C.c_void_p)(arr.release)(C.addressof(arr))
        if sch.release:
            C.CFUNCTYPE(None, C.c_void_p)(sch.release)(C.addressof(sch))
        _check(self._lib, self._h, st)
        names = self.output_names()
        for b in import_batches(self._lib, out):
            if collector is not None:
                collector.collect(pa.RecordBatch.from_arrays(b.columns, names=names))

    def process_batch_index(self, index: int, in_partitions: int, batch: pa.RecordBatch, ctx: OperatorContext,
                            collector: Collector):
        side = index // (in_partitions // 2)
        if self._schemas[side] is None:
            self._schemas[side] = batch.schema
        if not self.created:
            if self._schemas[0] is not None and self._schemas[1] is not None:
                self._build()
                pending, self._buffered = self._buffered, []
                for i, parts, b in pending:
                    self._send(i, parts, b, collector)
            else:
                self._buffered.append((index, in_partitions, batch))
                return
        self._send(index, in_partitions, batch, collector)

    def handle_watermark(self, watermark, ctx: OperatorContext, collector: Collector):
        return watermark
