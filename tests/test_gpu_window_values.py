"""The window function operator's value and distribution functions (WindowFunction with LAG / LEAD / FIRST_VALUE /
LAST_VALUE / NTH_VALUE and PERCENT_RANK / CUME_DIST OVER (PARTITION BY window [, key] [ORDER BY ...])) on the GPU: the
exact reference (tests/exact_window_value_reference.py) watermark by watermark, 2^24-row instants against numpy, the
CUDA sliding aggregate of golden `most_active_driver_last_hour` feeding LAG(count) and CUME_DIST(), and refusals.

Every column is compared as its 64 bits (Float64 NaN payloads and -0.0 included), a NULL as None.  Every output batch
passes pyarrow's full validation, and a column carries a validity bitmap exactly when one of its rows is NULL."""
import struct
import zlib

import numpy as np
import pyarrow as pa
import pytest

from oracle import arroyo_oracle as O
from tests import test_gpu_window_function as W
from tests.exact_window_fn_reference import TS
from tests.exact_window_value_reference import DISTRIBUTIONS, window_value_emissions
from tests.test_gpu_window_aggregates import s_spans
from tests.test_gpu_window_function import INT64_MAX, INT64_MIN, ORIGIN, SEC, SHAPES, Stream, _create, _ffi_config

ARROW = {**W.ARROW, "g": pa.float64()}
F64_BITS = np.array([0x7FF8000000000001, 0xFFF8000000000ABC, 0x7FF0000000000001, 1 << 63, 0, 0x7FF0000000000000,
                     0xFFF0000000000000, 0x3FF8000000000000, 0xC00C000000000000], dtype=np.uint64).view(np.int64)
DEFAULTS = {"l": -7, "L": (1 << 64) - 3, "tsn": ORIGIN - 1, "g": -0.0}  # per argument type, as a user writes it


def f64_bits(v: float) -> int:
    return struct.unpack("<q", struct.pack("<d", v))[0]


def ref_default(arg_type, default):
    """The reference's default: the value as the reader gives it back (a Float64 as its bits)."""
    if default is None:
        return None
    return f64_bits(default) if arg_type == "g" else default


# ---- streams ----------------------------------------------------------------------------------------------------------
class ValueStream(Stream):
    """Batches of [p?, k0.., a, x, _timestamp]: the argument `a` of type `arg_type` (l, L, tsn or g; Float64 from
    special bit patterns, NaN payloads and -0.0 among them).  `order` is the number of ORDER BY keys k0.. (k0 DESC, k1
    ASC, ...) or "x": ORDER BY the arrival sequence, so no row has a peer."""

    def __init__(self, seed, keyed, order, arg_type, types=None, pool=3):
        super().__init__(seed, keyed, 0 if order == "x" else order, {**(types or {}), "a": arg_type}, pool=pool)
        self.order, self.arg_type = order, arg_type

    def names(self):
        return (["p"] if self.keyed else []) + [f"k{i}" for i in range(self.n_order)] + ["a", "x", TS]

    def order_by(self):
        return [("x", False)] if self.order == "x" else super().order_by()

    def _values(self, col, n):
        if col != "a":
            return super()._values(col, n)
        r, t = self.rng, self.arg_type
        if t == "g":
            return r.choice(F64_BITS, n).view(np.float64)
        if t == "L":
            return r.choice(np.array([0, 1, 1 << 63, (1 << 64) - 1, 12345], dtype=np.uint64), n)
        if t == "tsn":
            return r.choice(np.array([INT64_MIN, INT64_MAX, 0, ORIGIN, ORIGIN + 1], dtype=np.int64), n)
        return np.where(r.random(n) < 0.1, INT64_MIN, r.integers(-1000, 1000, n)).astype(np.int64)


def to_arrow(cols, types):
    """test_gpu_window_function.to_arrow with Float64 ("g") columns."""
    arrays = []
    for c, v in cols.items():
        t = "tsn" if c == TS else types.get(c, "l")
        if t == "g":
            arrays.append(pa.array(np.asarray(v, dtype=np.float64), type=pa.float64()))
        elif t == "L":
            arrays.append(pa.array(np.asarray(v, dtype=np.uint64), type=pa.uint64()))
        else:
            a = pa.array(np.asarray(v, dtype=np.int64), type=pa.int64())
            arrays.append(a.cast(ARROW[t]) if t == "tsn" else a)
    return pa.RecordBatch.from_arrays(arrays, names=list(cols))


def bit_rows(rb):
    """Rows of an output or state batch as dicts of each column's 64 bits as a Python int (UInt64 unsigned, others
    signed), None for NULL; struct children flattened as <struct>_<child>.  Checks the batch with pyarrow's full
    validation and that a column has a validity bitmap exactly when it has NULLs."""
    rb.validate(full=True)
    cols = {}
    for name, col in zip(rb.schema.names, rb.columns):
        if pa.types.is_struct(col.type):
            for f, child in zip(col.type, col.flatten()):
                cols[f"{name}_{f.name}"] = child
        else:
            cols[name] = col
    out = {}
    for name, col in cols.items():
        validity, data = col.buffers()[:2]
        assert (validity is None) == (col.null_count == 0), (name, col.null_count)
        dtype = np.uint64 if pa.types.is_unsigned_integer(col.type) else np.int64
        v = [int(x) for x in np.frombuffer(data, dtype=dtype)[col.offset:col.offset + len(col)]]
        if col.null_count:
            v = [None if null else x for x, null in zip(v, col.is_null().to_pylist())]
        out[name] = v
    return [{c: v[i] for c, v in out.items()} for i in range(rb.num_rows)]


def bit_events(events):
    """The events as the reference reads them: Float64 columns as their bits."""
    return [(ev[0], {c: (v.view(np.int64) if v.dtype == np.float64 else v) for c, v in ev[1].items()})
            if ev[0] == "batch" else ev for ev in events]


def want_bits(emissions, function):
    if function not in DISTRIBUTIONS:
        return emissions
    return [[{**r, "fn": f64_bits(r["fn"])} for r in rows] for rows in emissions]


def run_gpu(st, cfg, entry, monkeypatch):
    """test_gpu_window_function.run_gpu with Float64 input and its batches read by bit_rows."""
    monkeypatch.setattr(W, "to_arrow", to_arrow)
    monkeypatch.setattr(W, "host_rows", bit_rows)
    return W.run_gpu(st, cfg, entry)


VALUE_SHAPES = {**SHAPES, "spans": s_spans}
EXTREME_TYPES = {"p": "L", "k0": "L", "k1": "tsn", "k2": "l", "k3": "tsn"}

CASES = [  # shape, function, keyed, ORDER BY (key count or "x"), argument type, entry, offset, with a default
    ("ties", "lag", True, 1, "l", "host", 1, False),
    ("ties", "lead", False, 2, "g", "device", 3, True),
    ("ties", "first_value", True, 4, "L", "sliced", 1, False),
    ("ties", "last_value", False, 1, "tsn", "run_batches", 1, False),
    ("ties", "nth_value", True, 2, "g", "host", 2, False),
    ("ties", "percent_rank", True, 1, "l", "device", 1, False),
    ("ties", "cume_dist", False, 0, "l", "host", 1, False),
    ("ties", "last_value", True, 0, "g", "device", 1, False),
    ("ties", "lag", False, 0, "L", "sliced", 0, False),
    ("edges", "lag", True, 2, "tsn", "host", INT64_MAX, True),
    ("edges", "lead", True, 1, "l", "run_batches", INT64_MAX, False),
    ("edges", "nth_value", False, 1, "l", "device", INT64_MAX, False),
    ("edges", "percent_rank", False, 2, "g", "sliced", 1, False),
    ("edges", "lead", False, 0, "g", "host", 0, True),
    ("extremes", "lag", True, 2, "g", "host", 1, True),
    ("extremes", "first_value", True, 1, "L", "device", 1, False),
    ("extremes", "cume_dist", True, 2, "tsn", "run_batches", 1, False),
    ("extremes", "lead", False, 4, "tsn", "sliced", 2, False),
    ("extremes", "last_value", True, 3, "l", "host", 1, False),
    ("backlog", "lag", True, 1, "l", "device", 1, False),
    ("backlog", "cume_dist", False, 0, "l", "host", 1, False),
    ("spans", "lag", False, "x", "l", "device", 1000, False),
    ("spans", "lead", False, 1, "g", "host", 1, True),
    ("spans", "nth_value", False, "x", "l", "sliced", 1500, False),
    ("spans", "last_value", True, 1, "g", "run_batches", 1, False),
    ("spans", "percent_rank", False, "x", "l", "host", 1, False),
    ("spans", "cume_dist", True, 1, "L", "device", 1, False),
    ("restarts", "lag", True, 2, "l", "host", 1, False),
    ("restarts", "lead", False, 1, "g", "device", 2, True),
    ("restarts", "nth_value", True, 1, "tsn", "run_batches", 3, False),
    ("restarts", "cume_dist", True, 0, "L", "sliced", 1, False),
    ("restarts", "first_value", False, 4, "l", "host", 1, False),
    ("restarts", "percent_rank", True, 2, "l", "run_batches", 1, False),
]


def case_id(c):
    return f"{c[0]}-{c[1]}-{'keyed' if c[2] else 'unkeyed'}-order{c[3]}-{c[4]}-{c[5]}-off{c[6]}" + \
        ("-default" if c[7] else "")


@pytest.mark.gpu
@pytest.mark.parametrize("shape,function,keyed,order,arg_type,entry,offset,with_default", CASES,
                         ids=[case_id(c) for c in CASES])
def test_values_against_exact_reference(shape, function, keyed, order, arg_type, entry, offset, with_default,
                                        monkeypatch):
    from arroyo_b200 import config
    seed = zlib.crc32(f"value/{shape}/{function}/{entry}".encode()) % 1000
    extreme = shape == "extremes"
    st = ValueStream(seed, keyed, order, arg_type, EXTREME_TYPES if extreme else None, "extreme" if extreme else 3)
    VALUE_SHAPES[shape](st)
    default = DEFAULTS[arg_type] if with_default else None
    argument = None if function in DISTRIBUTIONS else "a"
    cfg = config.WindowFunctionConfig(function, "p" if keyed else None, st.order_by(), "fn", argument=argument,
                                      offset=offset, default=default)
    want, late, want_states = window_value_emissions(bit_events(st.events), cfg.partition_by, cfg.order_by, function,
                                                     argument, "fn", offset, ref_default(arg_type, default))
    want = want_bits(want, function)
    got, states, rows_in, rows_late, schemas = run_gpu(st, cfg, entry, monkeypatch)
    assert len(got) == len(want)
    for i, (w, g) in enumerate(zip(want, got)):
        assert len(g) == len(w), ("watermark", i, len(g), len(w))
        for j, (a, b) in enumerate(zip(w, g)):
            assert a == b, ("watermark", i, "row", j, a, b)
    assert states == want_states
    assert rows_in == sum(len(ev[1][TS]) for ev in st.events if ev[0] == "batch")
    assert rows_late == late
    assert schemas
    fn_type = pa.float64() if function in DISTRIBUTIONS else ARROW[arg_type]
    for s in schemas:
        assert s.names == st.names() + ["fn"] and s.field("fn").type == fn_type
        assert s.field("a").type == ARROW[arg_type]


@pytest.mark.gpu
def test_window_struct_argument_and_validity():
    """LAG / NTH_VALUE of the upstream window struct's children, from host batches that carry the struct: timestamps
    out, the struct re-nested, NULLs counted exactly; with a default or a reachable n, no bitmap at all."""
    import arroyo_b200 as ab
    from arroyo_b200 import config, operators as native
    ts_t = pa.timestamp("ns")
    win = pa.struct([("start", ts_t), ("end", ts_t)])
    schema = pa.schema([("p", pa.int64()), ("window", win), ("v", pa.int64()), (TS, ts_t)])
    rng = np.random.default_rng(3)
    n = 500
    cols = {"p": rng.integers(0, 5, n).astype(np.int64), "window_start": rng.integers(0, 1 << 62, n).astype(np.int64),
            "window_end": rng.integers(0, 1 << 62, n).astype(np.int64), "v": rng.permutation(n).astype(np.int64),
            TS: (ORIGIN + rng.integers(0, 3, n) * SEC).astype(np.int64)}
    rb = pa.RecordBatch.from_arrays(
        [pa.array(cols["p"]), pa.StructArray.from_arrays([pa.array(cols["window_start"]).cast(ts_t),
                                                          pa.array(cols["window_end"]).cast(ts_t)], fields=list(win)),
         pa.array(cols["v"]), pa.array(cols[TS]).cast(ts_t)], schema=schema)
    segments = len({(int(t), int(p)) for t, p in zip(cols[TS], cols["p"])})
    calls = [("lag", "window_start", 2, None, 2 * segments), ("lag", "window_end", 1, ORIGIN, 0),
             ("lead", "window_start", 1, None, segments), ("nth_value", "window_end", 2, None, segments),
             ("nth_value", "window_start", 1, None, 0)]
    for function, argument, offset, default, nulls in calls:
        cfg = config.WindowFunctionConfig(function, "p", [("v", True)], "fn", argument=argument, offset=offset,
                                          default=default)
        op = native.WindowFunction(cfg, input_schema=schema)
        ctx, col = ab.OperatorContext(1), ab.Collector()
        op.process_batch(rb, ctx, None)
        ctx.watermarks.set(0, INT64_MAX)
        op.handle_watermark(INT64_MAX, ctx, col)
        op.close()
        (out,) = col.batches
        assert out.schema.names == schema.names + ["fn"]
        assert [(f.name, f.type) for f in out.schema.field("window").type] == [(f.name, f.type) for f in win]
        assert out.schema.field("fn").type == ts_t
        fn = out.column(out.num_columns - 1)
        assert fn.null_count == nulls and (fn.buffers()[0] is None) == (nulls == 0), (function, argument)
        want, _, _ = window_value_emissions([("batch", cols), ("wm", INT64_MAX)], "p", [("v", True)], function,
                                            argument, "fn", offset, default)
        assert bit_rows(out) == want[0], (function, argument)


# ---- scale ------------------------------------------------------------------------------------------------------------
def _device_run(cols, names, cfg, wm):
    """One device batch of `cols` through a fresh operator, then watermark `wm`: each output column's 64 bits and
    validity (None: no NULL) as numpy."""
    import torch

    import arroyo_b200 as ab
    from arroyo_b200 import operators as native
    schema = pa.schema([(c, pa.timestamp("ns") if c == TS else pa.int64()) for c in names])
    op = native.WindowFunction(cfg, input_schema=schema)
    dev = [torch.from_numpy(cols[c]).cuda() for c in names]
    op.process_device_batch([t.data_ptr() for t in dev], len(cols[TS]))
    ctx, col = ab.OperatorContext(1), ab.Collector()
    ctx.watermarks.set(0, wm)
    op.handle_watermark(wm, ctx, col)
    stats = op.stats()
    op.close()
    (rb,) = col.batches
    out = {}
    for c, a in zip(rb.schema.names, rb.columns):
        validity, data = a.buffers()[:2]
        valid = None if validity is None else ~a.is_null().to_numpy(zero_copy_only=False)
        out[c] = (np.frombuffer(data, dtype=np.int64)[:len(a)], valid)
    return out, stats


@pytest.mark.gpu
@pytest.mark.parametrize("shape", ["one_instant_2_20_partitions", "one_partition"])
def test_scale_2_24_rows(shape):
    """One instant of 2^24 rows ORDER BY k DESC: numpy's stable lexsort for the order, shifts within segments for the
    value functions, searchsorted on the sorted keys for the segment and peer bounds."""
    from arroyo_b200 import config
    n = 1 << 24
    rng = np.random.default_rng(41)
    t = ORIGIN + 5 * SEC
    keyed = shape != "one_partition"
    cols = {"p": rng.integers(0, 1 << 20, n).astype(np.int64), "k": rng.integers(-50, 50, n).astype(np.int64),
            "a": rng.integers(INT64_MIN, INT64_MAX, n, dtype=np.int64), "x": np.arange(n, dtype=np.int64),
            TS: np.full(n, t, dtype=np.int64)}
    names = ["p", "k", "a", "x", TS]
    key = (cols["p"] if keyed else np.zeros(n, np.int64)) * 128 + (49 - cols["k"])  # ascending = (p, k DESC)
    order = np.lexsort((np.arange(n), key))
    sk, sa, pos = key[order], cols["a"][order], np.arange(n)
    s = np.searchsorted(sk, sk // 128 * 128, "left")
    e = np.searchsorted(sk, sk // 128 * 128 + 128, "left") - 1
    g = np.searchsorted(sk, sk, "left")
    f = np.searchsorted(sk, sk, "right") - 1
    want = {  # function, offset, default -> (values, validity or None)
        ("lag", 1, None): (sa[np.maximum(pos - 1, 0)], pos - 1 >= s),
        ("lead", 5, -1): (np.where(pos + 5 <= e, sa[np.minimum(pos + 5, n - 1)], -1), None),
        ("first_value", 1, None): (sa[s], None),
        ("last_value", 1, None): (sa[f], None),
        ("nth_value", 3, None): (sa[np.minimum(s + 2, n - 1)], s + 2 <= f),
        ("percent_rank", 1, None): (np.where(e == s, 0.0, (g - s) / np.maximum(e - s, 1)).view(np.int64), None),
        ("cume_dist", 1, None): (((f - s + 1) / (e - s + 1)).view(np.int64), None),
    }
    for (function, offset, default), (w, valid) in want.items():
        argument = None if function in DISTRIBUTIONS else "a"
        cfg = config.WindowFunctionConfig(function, "p" if keyed else None, [("k", True)], "fn", argument=argument,
                                          offset=offset, default=default)
        got, stats = _device_run(cols, names, cfg, t + 1)
        assert np.array_equal(got["x"][0], cols["x"][order]), function
        values, got_valid = got["fn"]
        if valid is None or valid.all():
            assert got_valid is None, function
            assert np.array_equal(values, w), function
        else:
            assert np.array_equal(got_valid, valid), function
            assert np.array_equal(values[valid], w[valid]), function
        assert stats["rows_out"] == n and stats["windows_out"] == 1


# ---- golden input: the CUDA sliding aggregate feeding LAG(count) and CUME_DIST() ---------------------------------------
GOLDEN_ORDER = [("count", True), ("driver_id", True)]


def _after_sliding(inputs, device, function):
    """hop(1 min, 1 h) count(*) GROUP BY driver_id (CUDA sliding aggregate), then `function` OVER (PARTITION BY window
    ORDER BY count DESC, driver_id DESC) (CUDA window function): per watermark the rows it emits."""
    import arroyo_b200 as ab
    from arroyo_b200 import config, operators as native
    from tests import golden_cases as GC
    from tests import gpu_ops as G
    s_cfg = O.WindowAggConfig(width=GC.HOUR, slide=GC.MIN, key_names=["driver_id"], aggs=[O.Agg("count", None, "count")],
                              window_index=1)
    sliding = native.SlidingAggregatingWindowFunc(s_cfg)
    argument = None if function in DISTRIBUTIONS else "count"
    w_cfg = config.WindowFunctionConfig(function, None, GOLDEN_ORDER, "fn", argument=argument)
    ts_t = pa.timestamp("ns")
    if device:
        schema = pa.schema([("driver_id", pa.int64()), ("window_start", ts_t), ("window_end", ts_t),
                            ("count", pa.int64()), (TS, ts_t)])
    else:
        schema = pa.schema([("driver_id", pa.int64()), ("window", pa.struct([("start", ts_t), ("end", ts_t)])),
                            ("count", pa.int64()), (TS, ts_t)])
    wf = native.WindowFunction(w_cfg, input_schema=schema)
    s_ctx, w_ctx, out = ab.OperatorContext(1), ab.OperatorContext(1), []
    fn_type = pa.float64() if function in DISTRIBUTIONS else pa.int64()

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
            assert rb.schema.names == schema.names + ["fn"] and rb.schema.field("fn").type == fn_type
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
@pytest.mark.parametrize("function", ["lag", "cume_dist"])
@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
def test_golden_input_gap_and_position(golden, device, function):
    """Equal, row by row, to the exact reference fed by the numpy oracle's sliding aggregate: (count DESC, driver_id
    DESC) orders each window without ties, so the rows and their values do not depend on arrival order."""
    from tests.test_window_fn_reference import sliding_events
    inputs, _ = golden
    argument = None if function in DISTRIBUTIONS else "count"
    want, late, _ = window_value_emissions(sliding_events(inputs), None, GOLDEN_ORDER, function, argument, "fn")
    want = want_bits(want, function)
    got = _after_sliding(inputs, device, function)
    assert late == 0 and len(got) == len(want)
    cols = ("driver_id", "window_start", "window_end", "count", TS, "fn")
    assert sum(map(len, got)) > 1000
    for w, g in zip(want, got):
        assert [{c: r[c] for c in cols} for r in g] == [{c: r[c] for c in cols} for r in w]
    if function == "lag":
        assert any(r["fn"] is None for rows in got for r in rows)


# ---- refusals ---------------------------------------------------------------------------------------------------------
def _value_config(fn, n_order=1, **kw):
    from arroyo_b200 import ffi
    value = fn <= ffi.FN_NTH_VALUE
    cfg = _ffi_config(**{"window_fn": fn, "n_aggs": (1 if value else 0) + n_order,
                         "width_ns": 1 if fn in (ffi.FN_LAG, ffi.FN_LEAD, ffi.FN_NTH_VALUE) else 0, **kw})
    first = 0
    if value:
        cfg.aggs[0].kind = ffi.FN_ARGUMENT
        cfg.aggs[0].input_col = 0
        first = 1
    for i in range(n_order):
        cfg.aggs[first + i].kind = ffi.ORDER_DESC if i % 2 == 0 else ffi.ORDER_ASC
        cfg.aggs[first + i].input_col = 1
    return cfg


@pytest.mark.gpu
def test_value_refusals():
    import arroyo_b200 as ab
    from arroyo_b200 import config, ffi, operators as native
    values = (ffi.FN_LAG, ffi.FN_LEAD, ffi.FN_FIRST_VALUE, ffi.FN_LAST_VALUE, ffi.FN_NTH_VALUE)
    dists = (ffi.FN_PERCENT_RANK, ffi.FN_CUME_DIST)
    for fn in values + dists:
        for n_order in (0, 1, 4):
            assert _create(_value_config(fn, n_order)) == ffi.OK, (fn, n_order)
        # a fused top N
        assert _create(_value_config(fn, slide_ns=1)) == ffi.INVALID_ARGUMENT
        assert _create(_value_config(fn, slide_ns=-1)) == ffi.INVALID_ARGUMENT
        # an ORDER BY entry that is not ASC / DESC
        bad_order = _value_config(fn, 2)
        bad_order.aggs[bad_order.n_aggs - 1].kind = ffi.AGG_MAX_I64
        assert _create(bad_order) == ffi.INVALID_ARGUMENT
        # a default on anything but LAG / LEAD
        with_default = _value_config(fn, flags=ffi.FLAG_FN_DEFAULT, gap_ns=5)
        assert _create(with_default) == (ffi.OK if fn in (ffi.FN_LAG, ffi.FN_LEAD) else ffi.INVALID_ARGUMENT)
    for fn in values:
        for kind in (ffi.ORDER_DESC, ffi.ORDER_ASC, 0, ffi.AGG_SUM_I64, 19):  # aggs[0] not the argument marker
            cfg = _value_config(fn)
            cfg.aggs[0].kind = kind
            assert _create(cfg) == ffi.INVALID_ARGUMENT, (fn, kind)
        assert _create(_value_config(fn, 0, n_aggs=0)) == ffi.INVALID_ARGUMENT
        assert _create(_value_config(fn, 4, n_aggs=6)) == ffi.INVALID_ARGUMENT
        out_of_range = _value_config(fn)
        out_of_range.aggs[0].input_col = 3
        assert _create(out_of_range) == ffi.INVALID_ARGUMENT
    for fn in dists:
        assert _create(_value_config(fn, 4, n_aggs=5)) == ffi.INVALID_ARGUMENT
        assert _create(_value_config(fn, 0, n_aggs=-1)) == ffi.INVALID_ARGUMENT
    # offsets: k >= 0 (INT64_MAX included), n >= 1; negative ones are unsupported
    for fn in (ffi.FN_LAG, ffi.FN_LEAD):
        assert _create(_value_config(fn, width_ns=0)) == ffi.OK
        assert _create(_value_config(fn, width_ns=INT64_MAX)) == ffi.OK
        assert _create(_value_config(fn, width_ns=-1)) == ffi.UNSUPPORTED
    assert _create(_value_config(ffi.FN_NTH_VALUE, width_ns=INT64_MAX)) == ffi.OK
    assert _create(_value_config(ffi.FN_NTH_VALUE, width_ns=0)) == ffi.INVALID_ARGUMENT
    assert _create(_value_config(ffi.FN_NTH_VALUE, width_ns=-2)) == ffi.UNSUPPORTED
    # every other code stays refused; the ranking functions keep their rules and ignore the flag
    for code in (0, 12, 13, 18, -1):
        assert _create(_ffi_config(window_fn=code)) == ffi.INVALID_ARGUMENT, code
    assert _create(_ffi_config(flags=ffi.FLAG_FN_DEFAULT)) == ffi.OK
    assert _create(_ffi_config(window_fn=ffi.FN_RANK, n_aggs=0)) == ffi.INVALID_ARGUMENT

    ts_t = pa.timestamp("ns")
    schema = pa.schema([("key", pa.int64()), ("a", pa.int64()), (TS, ts_t)])
    for cfg in (config.WindowFunctionConfig("lag", None, [], "f", 1, argument="a"),  # a top N
                config.WindowFunctionConfig("first_value", None, [], "f", argument="a", default=3),
                config.WindowFunctionConfig("cume_dist", None, [], "f", default=3)):
        with pytest.raises(ffi.ArroyoB200Error) as e:
            native.WindowFunction(cfg, input_schema=schema)
        assert e.value.status == ffi.INVALID_ARGUMENT
    with pytest.raises(ffi.UnsupportedPlan):  # NTILE stays on the stock operator
        native.WindowFunction(config.WindowFunctionConfig("ntile", None, [("a", False)], "f"), input_schema=schema)
    with pytest.raises(ffi.UnsupportedPlan):
        native.WindowFunction(config.WindowFunctionConfig("lead", None, [], "f", argument="a", offset=-1),
                              input_schema=schema)
    # an argument of a type the operator does not move (a duration); a Float64 one is taken
    durations = pa.schema([("key", pa.int64()), ("a", pa.duration("ns")), (TS, ts_t)])
    with pytest.raises(ffi.UnsupportedPlan):
        native.WindowFunction(config.WindowFunctionConfig("lag", None, [], "f", argument="a"), input_schema=durations)
    floats = pa.schema([("key", pa.int64()), ("a", pa.float64()), (TS, ts_t)])
    native.WindowFunction(config.WindowFunctionConfig("lag", None, [("key", True)], "f", argument="a"),
                          input_schema=floats).close()
    # a state batch of another layout: INVALID_ARGUMENT, nothing taken; host output only
    op = native.WindowFunction(config.WindowFunctionConfig("lead", "key", [], "f", argument="a"), input_schema=schema)
    bad = pa.RecordBatch.from_arrays([pa.array([1], pa.int64()), pa.array([2.0], pa.float64()),
                                      pa.array([ORIGIN], ts_t)], names=["key", "a", TS])
    with pytest.raises(ffi.ArroyoB200Error) as e:
        op._on_start([bad], ffi.INT64_MIN, ffi.INT64_MIN)
    assert e.value.status == ffi.INVALID_ARGUMENT
    with pytest.raises(ffi.UnsupportedPlan):
        op.handle_watermark_device(ORIGIN)
    ctx, col = ab.OperatorContext(1), ab.Collector()
    ctx.watermarks.set(0, INT64_MAX)
    op.handle_watermark(INT64_MAX, ctx, col)
    assert not col.batches and op.stats()["rows_in"] == 0
    op.close()
