"""The window function operator's aggregates (WindowFunction with COUNT / SUM / AVG / MIN / MAX OVER (PARTITION BY
window [, key] [ORDER BY ...]), the default frame) on the GPU: the exact reference (tests/exact_window_agg_reference.py)
watermark by watermark, 2^24-row instants against numpy, the CUDA sliding aggregate of golden
`most_active_driver_last_hour` feeding SUM(count) OVER (PARTITION BY window [ORDER BY count DESC]), and refusals.

Integer columns and the row order are bit-exact; AVG agrees within 1e-6 relative (of the argument's magnitude when the
arguments reach +-2^63, where an f64 sum's rounding depends on its order)."""
import zlib

import numpy as np
import pyarrow as pa
import pytest

from oracle import arroyo_oracle as O
from tests.exact_window_agg_reference import window_agg_emissions
from tests.exact_window_fn_reference import TS
from tests import test_gpu_window_function as W
from tests.test_gpu_window_function import (INT64_MAX, INT64_MIN, ORIGIN, SEC, SHAPES, Stream, _create, _device_run,
                                            _ffi_config, host_rows)

FN_TYPE = {"count": pa.int64(), "sum": pa.int64(), "avg": pa.float64(), "min": pa.int64(), "max": pa.int64()}


class AggStream(Stream):
    """Batches of [p?, k0.., a, x, _timestamp]: the aggregate's argument `a` (values in [-1000, 1000), or from
    {INT64_MIN, INT64_MAX, ...} with pool "extreme").  `order` is the number of ORDER BY keys k0.. (k0 DESC, k1 ASC,
    ...) or "x": ORDER BY the arrival sequence, so no row has a peer."""

    def __init__(self, seed, keyed, order, pool=3):
        super().__init__(seed, keyed, 0 if order == "x" else order, pool=pool)
        self.order = order

    def names(self):
        return (["p"] if self.keyed else []) + [f"k{i}" for i in range(self.n_order)] + ["a", "x", TS]

    def order_by(self):
        return [("x", False)] if self.order == "x" else super().order_by()

    def _values(self, col, n):
        if col != "a":
            return super()._values(col, n)
        if self.pool == "extreme":
            return self.rng.choice(np.array([INT64_MIN, INT64_MAX, INT64_MAX - 1, 0, -1, 7], dtype=np.int64), n)
        return self.rng.integers(-1000, 1000, n).astype(np.int64)


def s_spans(st):
    """Segments over many 1024-row tiles next to 1-row instants."""
    st.at([ORIGIN], 5000)
    st.at(ORIGIN + SEC + np.arange(200), 1)
    st.at([ORIGIN + 2 * SEC], 9000)
    st.wm(ORIGIN + 2 * SEC)
    st.at([ORIGIN + 3 * SEC], 3000)
    st.wm(INT64_MAX)


AGG_SHAPES = {**SHAPES, "spans": s_spans}

CASES = [  # shape, function, keyed, ORDER BY (key count or "x"), entry, pool of the ORDER BY keys and argument
    ("ties", "sum", True, 1, "host", 3),
    ("ties", "count", False, 0, "device", 3),
    ("ties", "avg", True, 2, "sliced", 3),
    ("ties", "min", False, 4, "run_batches", 3),
    ("ties", "max", True, "x", "host", 3),
    ("ties", "sum", False, 1, "device", 1),
    ("edges", "avg", False, 1, "host", 3),
    ("edges", "max", True, 0, "run_batches", 3),
    ("edges", "count", True, 2, "sliced", 3),
    ("extremes", "sum", True, 1, "host", "extreme"),
    ("extremes", "min", False, 2, "device", "extreme"),
    ("extremes", "max", True, 0, "sliced", "extreme"),
    ("extremes", "avg", False, 1, "host", "extreme"),
    ("extremes", "sum", False, 0, "run_batches", "extreme"),
    ("backlog", "sum", True, 1, "device", 3),
    ("backlog", "avg", False, 0, "host", 3),
    ("spans", "sum", False, 1, "host", 3),
    ("spans", "min", True, "x", "device", 3),
    ("spans", "avg", False, 0, "sliced", 3),
    ("spans", "count", False, "x", "run_batches", 3),
    ("spans", "max", False, 1, "device", 1),
    ("restarts", "sum", True, 2, "host", 3),
    ("restarts", "avg", False, 1, "device", 3),
    ("restarts", "count", True, 0, "run_batches", 3),
    ("restarts", "min", True, 1, "sliced", 3),
    ("restarts", "max", False, 4, "host", 3),
]


def case_id(c):
    return f"{c[0]}-{c[1]}-{'keyed' if c[2] else 'unkeyed'}-order{c[3]}-{c[4]}-pool{c[5]}"


def typed_rows(rb):
    """host_rows keeping Float64 values as floats (host_rows makes every value an int)."""
    cols = {}
    for name, col in zip(rb.schema.names, rb.columns):
        if pa.types.is_struct(col.type):
            for f, child in zip(col.type, col.flatten()):
                cols[f"{name}_{f.name}"] = child
        else:
            cols[name] = col
    lists = {c: (v.cast(pa.int64()) if pa.types.is_timestamp(v.type) else v).to_pylist() for c, v in cols.items()}
    return [{c: v[i] for c, v in lists.items()} for i in range(rb.num_rows)]


def run_gpu(st, cfg, entry, monkeypatch):
    """test_gpu_window_function.run_gpu, its output rows read by typed_rows."""
    monkeypatch.setattr(W, "host_rows", typed_rows)
    return W.run_gpu(st, cfg, entry)


def assert_rows_equal(want, got, function, scale=1.0):
    assert len(got) == len(want)
    for i, (w, g) in enumerate(zip(want, got)):
        assert len(g) == len(w), ("watermark", i, len(g), len(w))
        for j, (a, b) in enumerate(zip(w, g)):
            if function == "avg":
                assert {**a, "fn": 0} == {**b, "fn": 0}, ("watermark", i, "row", j, a, b)
                assert abs(a["fn"] - b["fn"]) <= 1e-6 * max(abs(a["fn"]), scale), ("watermark", i, "row", j, a, b)
            else:
                assert a == b, ("watermark", i, "row", j, a, b)


@pytest.mark.gpu
@pytest.mark.parametrize("shape,function,keyed,order,entry,pool", CASES, ids=[case_id(c) for c in CASES])
def test_aggregate_against_exact_reference(shape, function, keyed, order, entry, pool, monkeypatch):
    from arroyo_b200 import config
    seed = zlib.crc32(f"agg/{shape}/{function}/{entry}".encode()) % 1000
    st = AggStream(seed, keyed, order, pool=pool)
    AGG_SHAPES[shape](st)
    cfg = config.WindowFunctionConfig(function, "p" if keyed else None, st.order_by(), "fn", argument="a")
    want, late, want_states = window_agg_emissions(st.events, cfg.partition_by, cfg.order_by, function, "a", "fn")
    got, states, rows_in, rows_late, schemas = run_gpu(st, cfg, entry, monkeypatch)
    assert_rows_equal(want, got, function, scale=2.0 ** 63 if pool == "extreme" else 1.0)
    assert states == want_states
    assert rows_in == sum(len(ev[1][TS]) for ev in st.events if ev[0] == "batch")
    assert rows_late == late
    assert schemas
    for s in schemas:
        assert s.names == st.names() + ["fn"] and s.field("fn").type == FN_TYPE[function]


# ---- scale ------------------------------------------------------------------------------------------------------------
def numpy_frames(p, k, a):
    """One instant: the stable order by (p, k DESC) (k None: by p alone) and per sorted row its segment's first index,
    its frame's last index and the sorted argument."""
    n = len(a)
    order = np.lexsort((np.arange(n), p) if k is None else (np.arange(n), ~k, p))
    sp = p[order]
    seg = np.r_[True, sp[1:] != sp[:-1]]
    peer_end = np.r_[seg[1:], True]
    if k is not None:
        sk = k[order]
        peer_end[:-1] |= sk[1:] != sk[:-1]
    seg_first = np.maximum.accumulate(np.where(seg, np.arange(n), 0))
    frame_last = np.flip(np.minimum.accumulate(np.flip(np.where(peer_end, np.arange(n), n))))
    return order, seg, seg_first, frame_last, a[order]


@pytest.mark.gpu
@pytest.mark.parametrize("ordered", [False, True], ids=["whole_partition", "order_by"])
@pytest.mark.parametrize("shape", ["one_instant_2_20_partitions", "one_partition"])
def test_scale_2_24_rows(shape, ordered):
    from arroyo_b200 import config
    n = 1 << 24
    rng = np.random.default_rng(37)
    t = ORIGIN + 5 * SEC
    keyed = shape != "one_partition"
    cols = {"p": rng.integers(0, 1 << 20, n).astype(np.int64), "k": rng.integers(-50, 50, n).astype(np.int64),
            "a": rng.integers(-1000, 1000, n).astype(np.int64), "x": np.arange(n, dtype=np.int64),
            TS: np.full(n, t, dtype=np.int64)}
    names = ["p", "k", "a", "x", TS]
    order, seg, seg_first, frame_last, sa = numpy_frames(cols["p"] if keyed else np.zeros(n, np.int64),
                                                         cols["k"] if ordered else None, cols["a"])
    starts = np.flatnonzero(seg)
    lengths = np.diff(np.r_[starts, n])
    count = frame_last - seg_first + 1
    if ordered:
        cs = np.cumsum(sa)
        sums = cs[frame_last] - np.where(seg_first > 0, cs[seg_first - 1], 0)
        seg_id = np.cumsum(seg) - 1
        run_max = np.maximum.accumulate(seg_id * 4096 + sa + 1024)  # segments ascend, so a max never crosses one
        want = {"sum": sums, "max": run_max[frame_last] - seg_id * 4096 - 1024, "avg": sums / count}
    else:
        want = {"sum": np.repeat(np.add.reduceat(sa, starts), lengths),
                "min": np.repeat(np.minimum.reduceat(sa, starts), lengths), "count": count}
    order_by = [("k", True)] if ordered else []
    for function, w in want.items():
        cfg = config.WindowFunctionConfig(function, "p" if keyed else None, order_by, "fn", argument="a")
        got, stats = _device_run(cols, names, cfg, t + 1)
        assert np.array_equal(got["x"], cols["x"][order]), function
        if function == "avg":
            assert np.allclose(got["fn"], w, rtol=1e-6, atol=0), function
        else:
            assert np.array_equal(got["fn"], w.astype(np.int64)), function
        assert stats["rows_out"] == n and stats["windows_out"] == 1


# ---- golden input: the CUDA sliding aggregate feeding SUM(count) OVER (PARTITION BY window [ORDER BY count DESC]) -----
def _share_of_window(inputs, device, order_by):
    """hop(1 min, 1 h) count(*) GROUP BY driver_id (CUDA sliding aggregate), then SUM(count) OVER (PARTITION BY window
    [ORDER BY count DESC]) (CUDA window function): per watermark the rows it emits."""
    import arroyo_b200 as ab
    from arroyo_b200 import config, operators as native
    from tests import golden_cases as GC
    from tests import gpu_ops as G
    s_cfg = O.WindowAggConfig(width=GC.HOUR, slide=GC.MIN, key_names=["driver_id"], aggs=[O.Agg("count", None, "count")],
                              window_index=1)
    sliding = native.SlidingAggregatingWindowFunc(s_cfg)
    w_cfg = config.WindowFunctionConfig("sum", None, order_by, "fn", argument="count")
    ts_t = pa.timestamp("ns")
    if device:
        schema = pa.schema([("driver_id", pa.int64()), ("window_start", ts_t), ("window_end", ts_t),
                            ("count", pa.int64()), (TS, ts_t)])
    else:
        schema = pa.schema([("driver_id", pa.int64()), ("window", pa.struct([("start", ts_t), ("end", ts_t)])),
                            ("count", pa.int64()), (TS, ts_t)])
    wf = native.WindowFunction(w_cfg, input_schema=schema)
    s_ctx, w_ctx, out = ab.OperatorContext(1), ab.OperatorContext(1), []

    def advance(wm):
        s_ctx.watermarks.set(0, wm)
        if device:
            for n, ptrs in sliding.handle_watermark_device(wm):
                wf.process_device_batch(ptrs, n)
            wf.flush()  # the sliding windows' buffers are reused by its next call
        else:
            col = ab.Collector()
            sliding.handle_watermark(wm, s_ctx, col)
            for rb in col.batches:
                wf.process_batch(rb, w_ctx, None)
        w_ctx.watermarks.set(0, wm)
        col = ab.Collector()
        wf.handle_watermark(wm, w_ctx, col)
        for rb in col.batches:
            assert rb.schema.names == schema.names + ["fn"] and rb.schema.field("fn").type == pa.int64()
        out.append([r for rb in col.batches for r in host_rows(rb)])

    gen = O.WatermarkGenerator(GC.HOUR)
    for b in O.source_batches({"driver_id": inputs["cars_driver_id"], TS: inputs["cars_ts"]}, GC.BATCH):
        sliding.process_batch(G.to_arrow(b), s_ctx, None)
        wm = gen.process_batch(b[TS])
        if wm is not None:
            advance(wm)
    advance(O.FINAL_WATERMARK)
    sliding.close()
    wf.close()
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("order_by", [[], [("count", True)]], ids=["share_of_window", "running_total"])
@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
def test_golden_input_sum_over_window(golden, device, order_by):
    """Equal to the exact reference fed by the numpy oracle's sliding aggregate.  Rows that tie on every sort key may
    arrive in another order from the two sliding aggregates; their values do not depend on it (peers share a frame),
    so each emission is compared as a multiset, and the sorted order by (window, count DESC) is checked."""
    from tests.golden_cases import multiset
    from tests.test_window_fn_reference import sliding_events
    inputs, _ = golden
    want, late, _ = window_agg_emissions(sliding_events(inputs), None, order_by, "sum", "count", "fn")
    got = _share_of_window(inputs, device, order_by)
    assert late == 0 and len(got) == len(want)
    cols = ("driver_id", "window_start", "window_end", "count", TS, "fn")
    assert sum(map(len, got)) > 1000
    for w, g in zip(want, got):
        assert multiset([{c: r[c] for c in cols} for r in g]) == multiset([{c: r[c] for c in cols} for r in w])
        assert [(r[TS], r["fn"]) for r in g] == [(r[TS], r["fn"]) for r in w]


# ---- refusals ---------------------------------------------------------------------------------------------------------
def _agg_config(kind, n_order=1, **kw):
    from arroyo_b200 import ffi
    cfg = _ffi_config(**{"window_fn": ffi.FN_AGGREGATE, "n_aggs": 1 + n_order, **kw})
    cfg.aggs[0].kind = kind
    cfg.aggs[0].input_col = 0
    for i in range(n_order):
        cfg.aggs[1 + i].kind = ffi.ORDER_DESC if i % 2 == 0 else ffi.ORDER_ASC
        cfg.aggs[1 + i].input_col = 1
    return cfg


@pytest.mark.gpu
def test_aggregate_refusals():
    import arroyo_b200 as ab
    from arroyo_b200 import config, ffi, operators as native
    for kind in (ffi.AGG_COUNT_STAR, ffi.AGG_SUM_I64, ffi.AGG_AVG_I64, ffi.AGG_MIN_I64, ffi.AGG_MAX_I64):
        for n_order in (0, 1, 4):
            assert _create(_agg_config(kind, n_order)) == ffi.OK, (kind, n_order)
    # aggs[0] not an aggregate kind
    assert _create(_agg_config(ffi.ORDER_DESC)) == ffi.INVALID_ARGUMENT
    assert _create(_agg_config(0)) == ffi.INVALID_ARGUMENT
    assert _create(_agg_config(6)) == ffi.INVALID_ARGUMENT
    # an ORDER BY entry that is not ASC / DESC
    bad_order = _agg_config(ffi.AGG_SUM_I64, 2)
    bad_order.aggs[2].kind = ffi.AGG_MAX_I64
    assert _create(bad_order) == ffi.INVALID_ARGUMENT
    # n_aggs 0 or more than 5
    assert _create(_agg_config(ffi.AGG_SUM_I64, 0, n_aggs=0)) == ffi.INVALID_ARGUMENT
    assert _create(_agg_config(ffi.AGG_SUM_I64, 4, n_aggs=6)) == ffi.INVALID_ARGUMENT
    # a fused top N
    assert _create(_agg_config(ffi.AGG_SUM_I64, 1, slide_ns=1)) == ffi.INVALID_ARGUMENT
    assert _create(_agg_config(ffi.AGG_SUM_I64, 1, slide_ns=-1)) == ffi.INVALID_ARGUMENT
    # the argument column out of range (COUNT ignores it)
    out_of_range = _agg_config(ffi.AGG_SUM_I64)
    out_of_range.aggs[0].input_col = 3
    assert _create(out_of_range) == ffi.INVALID_ARGUMENT
    out_of_range.aggs[0].kind = ffi.AGG_COUNT_STAR
    assert _create(out_of_range) == ffi.OK
    # ranking functions keep their rules: 0 ORDER BY keys
    assert _create(_ffi_config(n_aggs=0)) == ffi.INVALID_ARGUMENT
    assert _create(_ffi_config(window_fn=ffi.FN_RANK, n_aggs=0)) == ffi.INVALID_ARGUMENT

    ts_t = pa.timestamp("ns")
    schema = pa.schema([("key", pa.int64()), ("a", pa.int64()), (TS, ts_t)])
    with pytest.raises(ffi.ArroyoB200Error) as e:  # the Python config refuses a top N too
        native.WindowFunction(config.WindowFunctionConfig("sum", None, [], "s", 1, argument="a"), input_schema=schema)
    assert e.value.status == ffi.INVALID_ARGUMENT
    # an argument that is not Int64; COUNT takes any
    for t in (pa.float64(), pa.uint64(), ts_t):
        other = pa.schema([("key", pa.int64()), ("a", t), (TS, ts_t)])
        for function in ("sum", "avg", "min", "max"):
            with pytest.raises(ffi.UnsupportedPlan):
                native.WindowFunction(config.WindowFunctionConfig(function, "key", [], "s", argument="a"),
                                      input_schema=other)
        native.WindowFunction(config.WindowFunctionConfig("count", "key", [], "c", argument="a"),
                              input_schema=other).close()
    # a state batch whose argument is not Int64: INVALID_ARGUMENT, nothing taken
    op = native.WindowFunction(config.WindowFunctionConfig("sum", None, [("key", False)], "s", argument="a"),
                               input_schema=schema)
    bad = pa.RecordBatch.from_arrays([pa.array([1], pa.int64()), pa.array([2.0], pa.float64()),
                                      pa.array([ORIGIN], ts_t)], names=["key", "a", TS])
    with pytest.raises(ffi.ArroyoB200Error) as e:
        op._on_start([bad], ffi.INT64_MIN, ffi.INT64_MIN)
    assert e.value.status == ffi.INVALID_ARGUMENT
    # host output only
    with pytest.raises(ffi.UnsupportedPlan):
        op.handle_watermark_device(ORIGIN)
    with pytest.raises(ffi.UnsupportedPlan):
        op.handle_watermark_device_begin(ORIGIN)
    ctx, col = ab.OperatorContext(1), ab.Collector()
    ctx.watermarks.set(0, INT64_MAX)
    op.handle_watermark(INT64_MAX, ctx, col)
    assert not col.batches and op.stats()["rows_in"] == 0
    op.close()
