"""Record batches crossing the C ABI: what every entry point that hands back an ArroyoB200Batches does with `out`, and
who owns the state batches given to arroyo_b200_op_on_start.  That follows the Arrow C Data convention: the library
takes a batch by releasing it, and whatever still has a `release` after the call belongs to the caller."""
import ctypes as C

import numpy as np
import pyarrow as pa
import pytest

import arroyo_b200 as ab
from arroyo_b200 import ffi
from arroyo_b200 import operators as native
from oracle import arroyo_oracle as O
from oracle import updating_oracle as U

S = 1_000_000_000


def _entry_points(lib):
    """name -> call(handle, out) of every entry point that hands back an ArroyoB200Batches."""
    return {
        "handle_watermark": lambda h, out: lib.arroyo_b200_op_handle_watermark(h, 0, out),
        "handle_tick": lambda h, out: lib.arroyo_b200_op_handle_tick(h, out),
        "handle_checkpoint": lambda h, out: lib.arroyo_b200_op_handle_checkpoint(h, ffi.INT64_MIN, out),
        "checkpoint_state": lambda h, out: lib.arroyo_b200_op_checkpoint_state(h, out),
        "on_close": lambda h, out: lib.arroyo_b200_op_on_close(h, 1, out),
        "process_batch_emit": lambda h, out: lib.arroyo_b200_op_process_batch_emit(h, 0, 2, None, None, out),
        "handle_watermark_poll": lambda h, out: lib.arroyo_b200_op_handle_watermark_poll(h, 1, out,
                                                                                         C.byref(C.c_int32())),
        "run_batches": lambda h, out: lib.arroyo_b200_op_run_batches(h, None, None, 0, None, 0, out,
                                                                     C.byref(C.c_int64())),
    }


ENTRY_POINTS = sorted(_entry_points(None))


@pytest.mark.parametrize("entry", ENTRY_POINTS)
def test_null_handle_is_refused_and_out_is_zeroed(entry):
    lib = ffi.load()
    call = _entry_points(lib)[entry]
    out = ffi.Batches()
    out.n_batches = 7
    out.arrays = C.cast(C.c_void_p(64), C.POINTER(ffi.ArrowArray))
    out.schemas = C.cast(C.c_void_p(64), C.POINTER(ffi.ArrowSchema))
    out.private_data = 64
    assert call(None, C.byref(out)) == ffi.INVALID_ARGUMENT
    assert out.n_batches == 0 and not out.arrays and not out.schemas and not out.private_data
    assert call(None, None) == ffi.INVALID_ARGUMENT


# ---- GPU ---------------------------------------------------------------------------------------------------------
AGGS = [O.Agg("count", None, "n"), O.Agg("sum", "value", "total"), O.Agg("avg", "value", "mean")]
SCHEMA = pa.schema([("key", pa.int64()), ("value", pa.int64()), (O.TIMESTAMP, pa.timestamp("ns"))])


def _batch(rng, t0):
    n = 1000
    ts = np.sort(rng.integers(t0, t0 + 2 * S, n))
    return pa.RecordBatch.from_arrays(
        [pa.array(rng.integers(0, 100, n)), pa.array(rng.integers(-1000, 1000, n)),
         pa.array(ts).cast(pa.timestamp("ns"))], schema=SCHEMA)


def _new(kind):
    if kind in ("tumbling", "sliding"):
        cls = native.TumblingAggregatingWindowFunc if kind == "tumbling" else native.SlidingAggregatingWindowFunc
        cfg = O.WindowAggConfig(width=4 * S, slide=S if kind == "sliding" else 0, key_names=["key"], aggs=AGGS,
                                window_index=1)
        return cls(cfg, input_schema=SCHEMA)
    if kind == "instant":
        cfg = O.WindowAggConfig(width=0, key_names=["key"], aggs=AGGS, final_projection=False)
        return native.InstantAggregatingWindowFunc(cfg, input_schema=SCHEMA)
    if kind == "session":
        return native.SessionAggregatingWindowFunc(O.SessionConfig(gap=S, key_names=["key"], aggs=AGGS, window_index=1),
                                                   input_schema=SCHEMA)
    return native.UpdatingAggregatingFunc(U.UpdatingAggConfig(["key"], AGGS), input_schema=SCHEMA)


def _state(kind):
    """Two batches of checkpointed state from a short run, and the time arguments on_start takes with them."""
    rng = np.random.default_rng(5)
    op, ctx, out = _new(kind), ab.OperatorContext(1), ab.Collector()
    for t0 in (0, 10 * S):
        op.process_batch(_batch(rng, t0), ctx, out)
        if kind == "updating":
            op.handle_checkpoint(None, ctx, out)  # one batch of table "a" per checkpoint
    if kind != "updating":
        op.handle_checkpoint(None, ctx, out)
    op.close()
    if kind == "updating":
        return list(ctx.key_value_table("a").get_all()), ffi.INT64_MIN, ffi.INT64_MIN
    if kind == "session":
        start = min(v for v in ctx.global_table("e").values() if v is not None)
        return [b for _, b in ctx.table("s").all_batches_for_watermark(start)], ffi.INT64_MIN, start
    table = ctx.table("t")
    return [b for _, b in table.all_batches_for_watermark(None)], ffi.INT64_MIN, table.get_min_time()


def _on_start(op, batches, wm, t):
    n = len(batches)
    arrs, schs = (ffi.ArrowArray * n)(), (ffi.ArrowSchema * n)()
    for i, b in enumerate(batches):
        b._export_to_c(C.addressof(arrs[i]), C.addressof(schs[i]))
    st = op._lib.arroyo_b200_op_on_start(op._h, arrs, schs, n, wm, t)
    return st, list(arrs), list(schs)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["tumbling", "sliding", "session", "updating"])
def test_on_start_takes_the_state_batches_it_restores(kind):
    batches, wm, t = _state(kind)
    assert len(batches) >= 2
    op = _new(kind)
    st, arrs, schs = _on_start(op, batches, wm, t)
    assert st == ffi.OK, op._lib.arroyo_b200_op_last_error(op._h)
    assert all(a.release is None for a in arrs)
    assert all(s.release is not None for s in schs)  # the schemas stay the caller's
    for s in schs:
        native._release(s)
    op.close()


def _broken(how, b):
    """`b` with the wrong column count ("columns"), or with its first state column, an Int64 one in the layout of
    tables "t" and "a", as Float64 ("type")."""
    if how == "columns":
        return b.drop_columns([b.schema.names[-2]])
    col = b.column(1)
    assert col.type == pa.int64()
    return b.set_column(1, b.schema.field(1).with_type(pa.float64()), col.cast(pa.float64()))


# "last": only the last batch has the wrong column count.  Table "s" of the session holds raw input rows, where a
# Float64 value is an unsupported input type rather than a broken layout: it keeps the column-count case only.
REFUSALS = [pytest.param(k, h, id=k if h == "columns" else f"{k}-{h}")
            for k in ("tumbling", "sliding", "instant", "session", "updating")
            for h in ("columns", "type", "last") if k != "session" or h == "columns"]


@pytest.mark.gpu
@pytest.mark.parametrize("kind,how", REFUSALS)
def test_a_refused_on_start_leaves_the_state_batches_to_the_caller(kind, how):
    batches, wm, t = _state(kind)
    assert len(batches) >= 2
    if how == "last":
        bad = batches[:-1] + [_broken("columns", batches[-1])]
    else:
        bad = [_broken(how, b) for b in batches]
    op = _new(kind)
    st, arrs, schs = _on_start(op, bad, wm, t)
    assert st == ffi.INVALID_ARGUMENT
    assert all(a.release is not None for a in arrs)
    for s in arrs + schs:
        C.CFUNCTYPE(None, C.c_void_p)(s.release)(C.addressof(s))
        assert s.release is None
    stats = op.stats()
    assert stats["rows_in"] == 0
    assert stats["n_keys"] == 0
    op.close()


@pytest.mark.gpu
@pytest.mark.parametrize("flags", [0, ffi.FLAG_ZERO_COPY], ids=["staged", "zero_copy_flag"])
def test_window_aggregate_releases_every_host_batch_by_flush(flags):
    """The tumbling / sliding aggregate holds the host batches it takes until their copies have run, in groups of 16,
    and flush hands every one of them back: the Arrow pool's bytes return to their baseline.  40 batches leave two
    sealed groups and 8 batches that only flush seals.  FLAG_ZERO_COPY is accepted and changes nothing."""
    rng = np.random.default_rng(6)
    op = native.SlidingAggregatingWindowFunc(
        O.WindowAggConfig(width=4 * S, slide=S, key_names=["key"], aggs=AGGS, window_index=1),
        input_schema=SCHEMA, flags=flags)
    ctx, out = ab.OperatorContext(1), ab.Collector()
    base = pa.total_allocated_bytes()
    for i in range(40):
        b = _batch(rng, i * S // 8)
        b = b.take(pa.array(np.arange(b.num_rows)))  # buffers from the Arrow pool, not wrapped numpy memory
        op.process_batch(b, ctx, out)
    del b
    assert pa.total_allocated_bytes() > base  # the batches taken since the last sealed group are still held
    op.flush()
    assert pa.total_allocated_bytes() == base
    assert op.stats()["rows_in"] == 40 * 1000
    op.close()


@pytest.mark.gpu
def test_null_out_is_refused_except_by_on_close():
    op = _new("updating")
    for name, call in _entry_points(op._lib).items():
        st = call(op._h, None)
        assert st == (ffi.OK if name == "on_close" else ffi.INVALID_ARGUMENT), (name, st)
    op.close()
