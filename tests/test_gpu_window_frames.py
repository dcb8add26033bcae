"""The window function operator's explicit frames (WindowFunction with COUNT / SUM / AVG / MIN / MAX and FIRST_VALUE /
LAST_VALUE / NTH_VALUE over ROWS / RANGE / GROUPS frames) on the GPU: the exact reference
(tests/exact_window_frame_reference.py) watermark by watermark, default-equivalent frames against the default-frame
operator bit for bit, 2^24-row instants against numpy, the CUDA sliding aggregate of golden
`most_active_driver_last_hour` feeding framed SUM(count) and FIRST_VALUE(driver_id), and refusals.  No reference golden
uses an explicit frame: the golden case feeds the frames from a golden workload's sliding aggregate.

Every column is compared as its 64 bits, a NULL as None; AVG within 1e-15 relative (the exact sum and the count each
rounded once to f64, against the exactly rounded quotient).  Every output batch passes pyarrow's full validation, and
a column carries a validity bitmap exactly when one of its rows is NULL."""
import struct
import zlib

import numpy as np
import pyarrow as pa
import pytest

from oracle import arroyo_oracle as O
from tests.exact_window_fn_reference import TS
from tests.exact_window_frame_reference import window_frame_emissions
from tests.test_gpu_window_aggregates import s_spans
from tests.test_gpu_window_function import INT64_MAX, INT64_MIN, ORIGIN, SEC, SHAPES, _create, _ffi_config
from tests.test_gpu_window_values import ARROW, ValueStream, bit_events, bit_rows, run_gpu

FN_TYPE = {"count": "l", "sum": "l", "avg": "g", "min": "l", "max": "l"}
AGGREGATES = ("count", "sum", "avg", "min", "max")


def s_wide(st):
    """Segments of 6000 and 12000 rows: frames far larger than a 1024-row tile, and a 1-row segment."""
    st.at([ORIGIN], 6000)
    st.at([ORIGIN + SEC], 1)
    st.at([ORIGIN + 2 * SEC], 12000)
    st.wm(INT64_MAX)


FRAME_SHAPES = {**SHAPES, "spans": s_spans, "wide": s_wide}


class FrameStream(ValueStream):
    """ValueStream with k0 ascending or descending (`desc`), and with pool "extreme" an Int64 argument from
    {INT64_MIN, INT64_MAX, ...}, so that sums wrap."""

    def __init__(self, seed, keyed, order, arg_type, desc=True, types=None, pool=3):
        super().__init__(seed, keyed, order, arg_type, types, pool)
        self.desc = desc

    def order_by(self):
        return [(c, not d if c == "k0" and not self.desc else d) for c, d in super().order_by()]

    def _values(self, col, n):
        if col == "a" and self.arg_type == "l" and self.pool == "extreme":
            return self.rng.choice(np.array([INT64_MIN, INT64_MAX, INT64_MAX - 1, 0, -1, 7], dtype=np.int64), n)
        return super()._values(col, n)


def f64(bits):
    return struct.unpack("<d", struct.pack("<q", bits))[0]


def frame_cfg(function, keyed, order_by, frame, offset=1):
    from arroyo_b200 import config
    argument = None if function == "count" else "a"
    return config.WindowFunctionConfig(function, "p" if keyed else None, order_by, "fn", argument=argument,
                                       offset=offset, frame=config.WindowFrame(*frame))


ROWS_SMALL = ("rows", ("preceding", 2), ("following", 1))
ROWS_TILES = ("rows", ("preceding", 1500), ("following", 40))  # crosses 1024-row tiles and 32-row blocks
ROWS_BEFORE = ("rows", ("preceding", 5000), ("preceding", 3000))  # wholly before the row
ROWS_AFTER = ("rows", ("following", 3000), ("following", 5000))  # wholly after it
ROWS_MAX = ("rows", ("preceding", INT64_MAX), ("following", 0))
ROWS_EMPTY = ("rows", ("following", 2), ("following", 1))  # empty everywhere
ROWS_ZERO = ("rows", ("preceding", 0), ("following", 0))
RANGE_SMALL = ("range", ("preceding", 1), "current_row")
RANGE_SKIP = ("range", ("following", 1), ("following", 1))  # skips the row's own peers
RANGE_MAX = ("range", ("preceding", INT64_MAX), ("following", INT64_MAX))
RANGE_ONE = ("range", ("preceding", 1), ("following", 1))
RANGE_CUR = ("range", "current_row", "unbounded_following")
GROUPS_SMALL = ("groups", ("preceding", 1), ("following", 1))
GROUPS_AHEAD = ("groups", ("following", 1), "unbounded_following")
GROUPS_MAX = ("groups", ("preceding", INT64_MAX), ("preceding", 1))

L_KEYS = {"k0": "L"}
TS_KEYS = {"k0": "tsn"}
I_KEYS = {"k0": "l"}

CASES = [  # shape, function, keyed, ORDER BY (key count or "x"), argument type, entry, frame, k0 DESC, key types
    ("ties", "sum", True, 1, "l", "host", ROWS_SMALL, True, None),
    ("ties", "count", False, 2, "l", "device", GROUPS_SMALL, True, None),
    ("ties", "avg", True, 1, "l", "sliced", RANGE_SMALL, False, None),
    ("ties", "min", False, 1, "l", "run_batches", RANGE_SKIP, True, None),
    ("ties", "max", True, 4, "l", "host", GROUPS_AHEAD, False, None),
    ("ties", "first_value", True, "x", "g", "device", ROWS_SMALL, True, None),
    ("ties", "last_value", False, 1, "g", "host", RANGE_ONE, True, None),
    ("ties", "nth_value", True, 2, "L", "sliced", GROUPS_SMALL, True, None),
    ("ties", "sum", False, 0, "l", "host", ("rows", "current_row", ("following", 3)), True, None),
    ("edges", "sum", True, 1, "l", "host", ROWS_ZERO, True, None),
    ("edges", "min", False, 1, "l", "device", ROWS_EMPTY, True, None),
    ("edges", "last_value", True, 1, "tsn", "run_batches", RANGE_CUR, True, None),
    ("extremes", "sum", True, 1, "l", "host", RANGE_MAX, True, I_KEYS),
    ("extremes", "count", False, 1, "l", "device", RANGE_ONE, False, I_KEYS),
    ("extremes", "max", True, 1, "l", "sliced", RANGE_MAX, False, L_KEYS),
    ("extremes", "count", False, 1, "l", "host", ("range", ("preceding", 1 << 62), ("following", 4)), True, L_KEYS),
    ("extremes", "first_value", True, 1, "g", "host", ("range", ("preceding", 1), "unbounded_following"), True, TS_KEYS),
    ("extremes", "count", False, 1, "l", "run_batches", ("range", ("following", 1), ("following", INT64_MAX)), False, TS_KEYS),
    ("extremes", "avg", True, 1, "l", "device", ROWS_SMALL, True, I_KEYS),
    ("extremes", "nth_value", False, 2, "g", "host", GROUPS_MAX, True, I_KEYS),
    ("backlog", "sum", True, 1, "l", "device", GROUPS_SMALL, True, None),
    ("backlog", "first_value", False, 0, "l", "host", ("rows", ("preceding", 1), "current_row"), True, None),
    ("spans", "sum", False, "x", "l", "host", ROWS_TILES, True, None),
    ("spans", "min", True, "x", "l", "device", ROWS_TILES, True, None),
    ("spans", "max", False, "x", "l", "sliced", ROWS_BEFORE, True, None),
    ("spans", "avg", False, "x", "l", "run_batches", ROWS_AFTER, True, None),
    ("spans", "count", False, 1, "l", "host", RANGE_SMALL, True, None),
    ("spans", "nth_value", False, "x", "l", "device", ROWS_TILES, True, None),
    ("wide", "min", False, "x", "l", "host", ROWS_MAX, True, None),
    ("wide", "max", False, "x", "l", "device", ("rows", ("preceding", 700), ("following", 900)), True, None),
    ("wide", "sum", False, 1, "l", "host", GROUPS_SMALL, True, None),
    ("wide", "last_value", False, "x", "tsn", "host", ROWS_BEFORE, True, None),
    ("restarts", "sum", True, 2, "l", "host", ROWS_SMALL, True, None),
    ("restarts", "avg", False, 1, "l", "device", RANGE_ONE, False, None),
    ("restarts", "min", True, 1, "l", "run_batches", GROUPS_SMALL, True, None),
    ("restarts", "first_value", False, "x", "L", "sliced", ROWS_EMPTY, True, None),
    ("restarts", "max", True, 0, "l", "host", ("rows", ("preceding", 3), "unbounded_following"), True, None),
]


def case_id(c):
    f = c[6]
    bounds = "-".join(b if isinstance(b, str) else f"{b[0]}{b[1]}" for b in f[1:])
    return f"{c[0]}-{c[1]}-{'keyed' if c[2] else 'unkeyed'}-order{c[3]}-{c[4]}-{c[5]}-{f[0]}-{bounds}" + \
        ("" if c[7] else "-asc") + ("" if c[8] is None else "-" + c[8]["k0"])


def assert_rows_equal(want, got, function):
    assert len(got) == len(want)
    for i, (w, g) in enumerate(zip(want, got)):
        assert len(g) == len(w), ("watermark", i, len(g), len(w))
        for j, (a, b) in enumerate(zip(w, g)):
            if function == "avg" and a["fn"] is not None and b["fn"] is not None:
                assert {**a, "fn": 0} == {**b, "fn": 0}, ("watermark", i, "row", j, a, b)
                assert f64(b["fn"]) == pytest.approx(a["fn"], rel=1e-15, abs=0), ("watermark", i, "row", j, a, b)
            else:
                assert a == b, ("watermark", i, "row", j, a, b)


@pytest.mark.gpu
@pytest.mark.parametrize("shape,function,keyed,order,arg_type,entry,frame,desc,types", CASES,
                         ids=[case_id(c) for c in CASES])
def test_frames_against_exact_reference(shape, function, keyed, order, arg_type, entry, frame, desc, types,
                                        monkeypatch):
    seed = zlib.crc32(f"frame/{shape}/{function}/{entry}".encode()) % 1000
    extreme = shape == "extremes"
    st = FrameStream(seed, keyed, order, arg_type, desc, types, "extreme" if extreme else 3)
    FRAME_SHAPES[shape](st)
    cfg = frame_cfg(function, keyed, st.order_by(), frame, 2)
    want, late, want_states = window_frame_emissions(bit_events(st.events), cfg.partition_by, cfg.order_by, function,
                                                     cfg.argument, frame, "fn", 2)
    got, states, rows_in, rows_late, schemas = run_gpu(st, cfg, entry, monkeypatch)
    assert_rows_equal(want, got, function)
    assert states == want_states
    assert rows_in == sum(len(ev[1][TS]) for ev in st.events if ev[0] == "batch")
    assert rows_late == late
    assert schemas
    fn_type = ARROW[FN_TYPE.get(function, arg_type)]
    for s in schemas:
        assert s.names == st.names() + ["fn"] and s.field("fn").type == fn_type
    if frame in (ROWS_EMPTY, RANGE_SKIP):
        assert any(r["fn"] in (None, 0) for rows in got for r in rows)


@pytest.mark.gpu
@pytest.mark.parametrize("function", AGGREGATES + ("first_value", "last_value", "nth_value"))
def test_default_equivalent_frames_are_bit_identical(function, monkeypatch):
    """RANGE UNBOUNDED PRECEDING AND CURRENT ROW with ORDER BY, and UNBOUNDED PRECEDING AND UNBOUNDED FOLLOWING in ROWS
    or RANGE without it (GROUPS takes an ORDER BY), run the default frame's kernels: the same bits as a default-frame
    operator, AVG included."""
    from arroyo_b200 import config
    for order, frames in ((1, [("range", "unbounded_preceding", "current_row")]),
                          (0, [(u, "unbounded_preceding", "unbounded_following") for u in ("rows", "range")])):
        st = FrameStream(zlib.crc32(f"default/{function}".encode()) % 1000, True, order, "l")
        SHAPES["ties"](st)
        argument = None if function == "count" else "a"
        base = config.WindowFunctionConfig(function, "p", st.order_by(), "fn", argument=argument, offset=2)
        want = run_gpu(st, base, "host", monkeypatch)[0]
        for frame in frames:
            got = run_gpu(st, frame_cfg(function, True, st.order_by(), frame, 2), "host", monkeypatch)[0]
            assert got == want, frame


@pytest.mark.gpu
def test_frame_ends_never_decrease_on_the_gpu():
    """The GPU's lo and hi are non-decreasing in the row within a segment.  The argument v = k0 * 2^32 + arrival rises
    strictly in sort order (k0 ASC, ties in arrival order) within each segment, so FIRST_VALUE(v) reads the row at lo
    and LAST_VALUE(v) the row at hi - 1: both must be non-decreasing over the rows whose frame is not empty, and COUNT
    must be hi - lo for them."""
    import arroyo_b200 as ab
    from arroyo_b200 import config, operators as native
    rng = np.random.default_rng(5)
    n = 20000
    cols = {"p": rng.integers(0, 5, n).astype(np.int64), "k0": rng.integers(-20, 20, n).astype(np.int64),
            "x": np.arange(n, dtype=np.int64), TS: (ORIGIN + rng.integers(0, 3, n) * SEC).astype(np.int64)}
    cols["v"] = cols["k0"] * (1 << 32) + cols["x"]
    names = ["p", "k0", "v", "x", TS]
    schema = pa.schema([(c, pa.timestamp("ns") if c == TS else pa.int64()) for c in names])
    rb = pa.RecordBatch.from_arrays([pa.array(cols[c]).cast(schema.field(c).type) for c in names], schema=schema)
    frames = [ROWS_SMALL, ROWS_TILES, ROWS_BEFORE, ROWS_AFTER, RANGE_ONE, RANGE_SKIP,
              ("range", ("preceding", 3), ("following", 5)), GROUPS_SMALL, GROUPS_AHEAD,
              ("groups", ("preceding", 2), ("preceding", 1))]
    for frame in frames:
        out = {}
        for function in ("first_value", "last_value", "count"):
            cfg = config.WindowFunctionConfig(function, "p", [("k0", False)], "fn",
                                              argument=None if function == "count" else "v",
                                              frame=config.WindowFrame(*frame))
            op = native.WindowFunction(cfg, input_schema=schema)
            ctx, col = ab.OperatorContext(1), ab.Collector()
            op.process_batch(rb, ctx, None)
            ctx.watermarks.set(0, INT64_MAX)
            op.handle_watermark(INT64_MAX, ctx, col)
            op.close()
            out[function] = [r for b in col.batches for r in bit_rows(b)]
        rows = out["count"]
        assert len(rows) == n and [r["x"] for r in out["first_value"]] == [r["x"] for r in rows]
        segments = {}
        for i, r in enumerate(rows):
            segments.setdefault((r[TS], r["p"]), []).append(i)
        pos = {r["v"]: i for i, r in enumerate(rows)}  # v is unique: the sorted row that holds it
        for idx in segments.values():
            lo = [pos[out["first_value"][i]["fn"]] for i in idx if rows[i]["fn"]]
            hi = [pos[out["last_value"][i]["fn"]] + 1 for i in idx if rows[i]["fn"]]
            assert lo == sorted(lo) and hi == sorted(hi), frame
            assert [h - l for l, h in zip(lo, hi)] == [rows[i]["fn"] for i in idx if rows[i]["fn"]], frame
            assert all(out["first_value"][i]["fn"] is None for i in idx if not rows[i]["fn"]), frame


# ---- scale ------------------------------------------------------------------------------------------------------------
def _device_run(cols, names, cfg, wm):
    """One device batch of `cols` through a fresh operator, then watermark `wm`: each output column's 64 bits and
    validity (None: no NULL) as numpy."""
    from tests.test_gpu_window_values import _device_run as run
    return run(cols, names, cfg, wm)


def _window_min(x, lo, hi, width):
    """min of x[lo:hi] per row, for frames of at most `width` rows."""
    out = np.full(len(x), np.iinfo(np.int64).max)
    for d in range(width):
        np.minimum(out, np.where(hi - lo > d, x[np.minimum(lo + d, len(x) - 1)], out), out=out)
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("shape", ["one_instant_2_20_partitions", "one_partition"])
def test_scale_2_24_rows(shape):
    """One instant of 2^24 rows ORDER BY k DESC, ROWS / RANGE / GROUPS frames: numpy's stable lexsort for the order,
    searchsorted for the frames, cumsum differences for COUNT / SUM / AVG and windows of at most 201 rows for MIN /
    MAX and the value functions."""
    n = 1 << 24
    rng = np.random.default_rng(43)
    t = ORIGIN + 5 * SEC
    keyed = shape != "one_partition"
    cols = {"p": rng.integers(0, 1 << 20, n).astype(np.int64), "k": rng.integers(-50, 50, n).astype(np.int64),
            "a": rng.integers(-(1 << 30), 1 << 30, n).astype(np.int64), "x": np.arange(n, dtype=np.int64),
            TS: np.full(n, t, dtype=np.int64)}
    names = ["p", "k", "a", "x", TS]
    y = 49 - cols["k"]  # ascending in sort order (k DESC)
    key = (cols["p"] if keyed else np.zeros(n, np.int64)) * 128 + y
    order = np.lexsort((np.arange(n), key))
    sk, sa, pos = key[order], cols["a"][order], np.arange(n)
    s = np.searchsorted(sk, sk // 128 * 128, "left")
    e1 = np.searchsorted(sk, sk // 128 * 128 + 128, "left")
    group_first = np.searchsorted(sk, sk, "left")
    rows_100 = ("rows", ("preceding", 100), ("following", 100))
    frames = {  # frame -> (lo, hi)
        ROWS_SMALL: (np.maximum(pos - 2, s), np.minimum(pos + 2, e1)),
        rows_100: (np.maximum(pos - 100, s), np.minimum(pos + 101, e1)),
        ("range", ("preceding", 3), ("following", 2)): (np.maximum(np.searchsorted(sk, sk - 3, "left"), s),
                                                        np.minimum(np.searchsorted(sk, sk + 2, "right"), e1)),
    }
    if not keyed:
        # one partition of 2^24 rows holds all 100 key values, so its peer groups are the key values
        frames[GROUPS_SMALL] = (np.searchsorted(sk, sk - 1, "left"), np.searchsorted(sk, sk + 1, "right"))
    cs = np.concatenate([[0], np.cumsum(sa)])
    for frame, (lo, hi) in frames.items():
        assert (hi > lo).all()
        count = hi - lo
        want = {"count": count, "sum": cs[hi] - cs[lo], "avg": (cs[hi] - cs[lo]) / count,
                "first_value": sa[lo], "last_value": sa[hi - 1]}
        if frame == ROWS_SMALL:
            want["min"] = _window_min(sa, lo, hi, 4)
        elif frame == rows_100 and not keyed:
            pad = np.concatenate([np.full(100, np.iinfo(np.int64).max), sa, np.full(100, np.iinfo(np.int64).max)])
            want["min"] = np.lib.stride_tricks.sliding_window_view(pad, 201).min(axis=1)
        elif frame[0] != "rows" and not keyed:
            # RANGE / GROUPS in one partition: the extreme over whole key values, from each value's extreme
            vmax = np.full(100 + 8, np.iinfo(np.int64).min)
            np.maximum.at(vmax, y[order] + 4, sa)
            w = np.lib.stride_tricks.sliding_window_view(vmax, 6 if frame[0] == "range" else 3).max(axis=1)
            want["max"] = w[y[order] + 4 - (3 if frame[0] == "range" else 1)]
        for function, w in want.items():
            cfg = frame_cfg(function, keyed, [("k", True)], frame)
            got, stats = _device_run(cols, names, cfg, t + 1)
            assert np.array_equal(got["x"][0], cols["x"][order]), (frame, function)
            values, valid = got["fn"]
            assert valid is None, (frame, function)
            if function == "avg":
                assert np.allclose(values.view(np.float64), w, rtol=1e-15, atol=0), frame
            else:
                assert np.array_equal(values, w.astype(np.int64)), (frame, function)
            assert stats["rows_out"] == n and stats["windows_out"] == 1


# ---- golden input: the CUDA sliding aggregate feeding framed SUM(count) and FIRST_VALUE(driver_id) -----------------
GOLDEN_ORDER = [("count", True), ("driver_id", True)]
GOLDEN_ROWS = ("rows", ("preceding", 1), ("following", 1))
GOLDEN_RANGE = ("range", ("preceding", 2), ("following", 5))


def _after_sliding(inputs, device, cfg):
    """hop(1 min, 1 h) count(*) GROUP BY driver_id (CUDA sliding aggregate), then the window function `cfg` (CUDA):
    per watermark the rows it emits."""
    import arroyo_b200 as ab
    from arroyo_b200 import operators as native
    from tests import golden_cases as GC
    from tests import gpu_ops as G
    s_cfg = O.WindowAggConfig(width=GC.HOUR, slide=GC.MIN, key_names=["driver_id"], aggs=[O.Agg("count", None, "count")],
                              window_index=1)
    sliding = native.SlidingAggregatingWindowFunc(s_cfg)
    ts_t = pa.timestamp("ns")
    if device:
        schema = pa.schema([("driver_id", pa.int64()), ("window_start", ts_t), ("window_end", ts_t),
                            ("count", pa.int64()), (TS, ts_t)])
    else:
        schema = pa.schema([("driver_id", pa.int64()), ("window", pa.struct([("start", ts_t), ("end", ts_t)])),
                            ("count", pa.int64()), (TS, ts_t)])
    wf = native.WindowFunction(cfg, input_schema=schema)
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
        out.append([r for rb in col.batches for r in bit_rows(rb)])

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
@pytest.mark.parametrize("function,argument,order_by,frame", [
    ("sum", "count", GOLDEN_ORDER, GOLDEN_ROWS), ("first_value", "driver_id", GOLDEN_ORDER, GOLDEN_ROWS),
    ("last_value", "window_start", GOLDEN_ORDER, GOLDEN_ROWS), ("sum", "count", [("count", True)], GOLDEN_RANGE)],
    ids=["sum-rows", "first_value-rows", "last_value-window_start-rows", "sum-range"])
@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
def test_golden_input_frames(golden, device, function, argument, order_by, frame):
    """Equal to the exact reference fed by the numpy oracle's sliding aggregate.  (count DESC, driver_id DESC) orders
    each window without ties, so the ROWS frames are compared row by row; the RANGE frame over count alone holds whole
    peer groups, so its rows are compared as a multiset and its values in order."""
    from arroyo_b200 import config
    from tests.golden_cases import multiset
    from tests.test_window_fn_reference import sliding_events
    inputs, _ = golden
    cfg = config.WindowFunctionConfig(function, None, order_by, "fn", argument=argument,
                                      frame=config.WindowFrame(*frame))
    want, late, _ = window_frame_emissions(sliding_events(inputs), None, order_by, function, argument, frame, "fn")
    got = _after_sliding(inputs, device, cfg)
    assert late == 0 and len(got) == len(want)
    cols = ("driver_id", "window_start", "window_end", "count", TS, "fn")
    assert sum(map(len, got)) > 1000
    for w, g in zip(want, got):
        g, w = [{c: r[c] for c in cols} for r in g], [{c: r[c] for c in cols} for r in w]
        if frame == GOLDEN_ROWS:
            assert g == w
        else:
            assert multiset(g) == multiset(w)
            assert [(r[TS], r["fn"]) for r in g] == [(r[TS], r["fn"]) for r in w]


# ---- refusals ---------------------------------------------------------------------------------------------------------
def _framed(fn, units, start, end, n_order=1, start_offset=1, end_offset=1, agg=None):
    from arroyo_b200 import ffi
    value = fn in (ffi.FN_FIRST_VALUE, ffi.FN_LAST_VALUE, ffi.FN_NTH_VALUE, ffi.FN_LAG, ffi.FN_LEAD)
    first = 1 if fn == ffi.FN_AGGREGATE or value else 0
    cfg = _ffi_config(window_fn=fn, n_aggs=first + n_order, width_ns=1 if fn in (ffi.FN_LAG, ffi.FN_LEAD,
                                                                                  ffi.FN_NTH_VALUE) else 0)
    if first:
        cfg.aggs[0].kind = agg if fn == ffi.FN_AGGREGATE else ffi.FN_ARGUMENT
        cfg.aggs[0].input_col = 0
    for i in range(n_order):
        cfg.aggs[first + i].kind = ffi.ORDER_DESC
        cfg.aggs[first + i].input_col = 1
    cfg.frame.units, cfg.frame.start_kind, cfg.frame.end_kind = units, start, end
    cfg.frame.start_offset, cfg.frame.end_offset = start_offset, end_offset
    return cfg


@pytest.mark.gpu
def test_frame_refusals():
    import arroyo_b200 as ab
    from arroyo_b200 import config, ffi, operators as native
    UP, P, CR, F, UF = (ffi.BOUND_UNBOUNDED_PRECEDING, ffi.BOUND_PRECEDING, ffi.BOUND_CURRENT_ROW, ffi.BOUND_FOLLOWING,
                        ffi.BOUND_UNBOUNDED_FOLLOWING)
    ROWS, RANGE, GROUPS = ffi.FRAME_ROWS, ffi.FRAME_RANGE, ffi.FRAME_GROUPS
    framed = [(ffi.FN_AGGREGATE, k) for k in (ffi.AGG_COUNT_STAR, ffi.AGG_SUM_I64, ffi.AGG_AVG_I64, ffi.AGG_MIN_I64,
                                               ffi.AGG_MAX_I64)] + \
        [(f, None) for f in (ffi.FN_FIRST_VALUE, ffi.FN_LAST_VALUE, ffi.FN_NTH_VALUE)]
    accepted = [(s, e) for s in (UP, P, CR, F) for e in (P, CR, F, UF)
                if (s, e) not in ((F, CR), (F, P), (CR, P))]
    for fn, agg in framed:
        for units in (ROWS, RANGE, GROUPS):
            for s, e in accepted:
                for so, eo in ((0, 0), (1, 3), (3, 1), (INT64_MAX, INT64_MAX)):
                    assert _create(_framed(fn, units, s, e, 1, so, eo, agg)) == ffi.OK, (fn, agg, units, s, e, so, eo)
            # a start after the end: UNSUPPORTED
            for s, e in ((F, CR), (F, P), (CR, P)):
                assert _create(_framed(fn, units, s, e, agg=agg)) == ffi.UNSUPPORTED, (fn, units, s, e)
            # UNBOUNDED FOLLOWING as a start, UNBOUNDED PRECEDING as an end, unknown bound codes
            for s, e in ((UF, UF), (UP, UP), (UF, CR), (CR, UP), (0, CR), (CR, 6), (-1, UF)):
                assert _create(_framed(fn, units, s, e, agg=agg)) == ffi.INVALID_ARGUMENT, (fn, units, s, e)
            # negative offsets (ignored where the bound takes none)
            assert _create(_framed(fn, units, P, CR, 1, -1, 0, agg)) == ffi.INVALID_ARGUMENT
            assert _create(_framed(fn, units, CR, F, 1, 0, -1, agg)) == ffi.INVALID_ARGUMENT
            assert _create(_framed(fn, units, UP, CR, 1, -1, -1, agg)) == ffi.OK
        # RANGE with an offset over other than one ORDER BY key; GROUPS without ORDER BY
        for n_order in (0, 2, 4):
            assert _create(_framed(fn, RANGE, P, CR, n_order, agg=agg)) == ffi.INVALID_ARGUMENT
            assert _create(_framed(fn, RANGE, CR, UF, n_order, agg=agg)) == ffi.OK
        assert _create(_framed(fn, GROUPS, P, F, 0, agg=agg)) == ffi.INVALID_ARGUMENT
        assert _create(_framed(fn, ROWS, P, F, 0, agg=agg)) == ffi.OK
        for units in (4, -1):
            assert _create(_framed(fn, units, P, F, agg=agg)) == ffi.INVALID_ARGUMENT
    # the functions that take no frame
    for fn in (ffi.FN_ROW_NUMBER, ffi.FN_RANK, ffi.FN_DENSE_RANK, ffi.FN_LAG, ffi.FN_LEAD, ffi.FN_PERCENT_RANK,
               ffi.FN_CUME_DIST):
        assert _create(_framed(fn, ROWS, UP, CR)) == ffi.INVALID_ARGUMENT, fn
        assert _create(_framed(fn, ffi.FRAME_DEFAULT, UF, UP, 1, -1, -1)) == ffi.OK, fn

    ts_t = pa.timestamp("ns")
    schema = pa.schema([("key", pa.int64()), ("a", pa.int64()), (TS, ts_t)])
    for frame in (config.WindowFrame("slices", "unbounded_preceding", "current_row"),
                  config.WindowFrame("rows", "preceding", "current_row"),
                  config.WindowFrame("rows", ("current_row", 1), "current_row"),
                  config.WindowFrame("rows", ("preceding", 1 << 63), "current_row")):
        with pytest.raises(ffi.ArroyoB200Error) as e:
            native.WindowFunction(config.WindowFunctionConfig("sum", None, [("key", False)], "f", argument="a",
                                                              frame=frame), input_schema=schema)
        assert e.value.status == ffi.INVALID_ARGUMENT, frame
    with pytest.raises(ffi.UnsupportedPlan):
        native.WindowFunction(config.WindowFunctionConfig(
            "sum", None, [("key", False)], "f", argument="a",
            frame=config.WindowFrame("rows", ("following", 1), "current_row")), input_schema=schema)
    # frames on non-Int64 aggregate arguments stay refused; host output only
    floats = pa.schema([("key", pa.int64()), ("a", pa.float64()), (TS, ts_t)])
    with pytest.raises(ffi.UnsupportedPlan):
        native.WindowFunction(config.WindowFunctionConfig("sum", None, [("key", False)], "f", argument="a",
                                                          frame=config.WindowFrame(*ROWS_SMALL)), input_schema=floats)
    op = native.WindowFunction(config.WindowFunctionConfig("max", None, [("key", False)], "f", argument="a",
                                                           frame=config.WindowFrame(*ROWS_SMALL)), input_schema=schema)
    with pytest.raises(ffi.UnsupportedPlan):
        op.handle_watermark_device(ORIGIN)
    ctx, col = ab.OperatorContext(1), ab.Collector()
    ctx.watermarks.set(0, INT64_MAX)
    op.handle_watermark(INT64_MAX, ctx, col)
    assert not col.batches and op.stats()["rows_in"] == 0
    op.close()


def test_frame_config_layout():
    """The frame is appended to the config: every earlier field keeps its offset, and a zeroed frame is the default."""
    import ctypes as C

    from arroyo_b200 import ffi
    fields = [f for f, _ in ffi.OpConfig._fields_]
    assert fields[-1] == "frame" and fields[-2] == "reserved"
    assert ffi.OpConfig.frame.offset == ffi.OpConfig.reserved.offset + 4
    assert C.sizeof(ffi.WindowFrame) == 32 and C.sizeof(ffi.OpConfig) % 8 == 0
    assert ffi.OpConfig().frame.units == ffi.FRAME_DEFAULT
