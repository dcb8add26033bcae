"""The window function operator (WindowFunction: window_fn.rs, ROW_NUMBER / RANK / DENSE_RANK per instant and
partition key with the fused top N) on the GPU: golden `most_active_driver_last_hour` with the CUDA sliding aggregate
feeding it, the exact reference (tests/exact_window_fn_reference.py) watermark by watermark, scale against
np.lexsort-based ranks, memory reclamation and refusals.

Streams are lists of ("batch", {column: array}), ("wm", w) and ("restart",) events; a restart is handle_checkpoint, a
new operator and on_start from table "input"."""
import ctypes as C
import zlib

import numpy as np
import pyarrow as pa
import pytest

from oracle import arroyo_oracle as O
from tests.exact_window_fn_reference import TS, window_fn_emissions

SEC = 1_000_000_000
ORIGIN = 1_700_000_000 * SEC
INT64_MIN, INT64_MAX = -(1 << 63), (1 << 63) - 1
ARROW = {"l": pa.int64(), "L": pa.uint64(), "tsn": pa.timestamp("ns")}
NUMPY = {"l": np.int64, "L": np.uint64, "tsn": np.int64}


# ---- streams ----------------------------------------------------------------------------------------------------------
class Stream:
    """Batches of [p?, k0.., x, _timestamp]: partition key `p`, ORDER BY keys k0..k{n_order-1} (k0 DESC, k1 ASC, ...),
    payload `x`.  `types` maps p / k<i> to l, L or tsn (default l)."""

    def __init__(self, seed, keyed, n_order, types=None, pool=3):
        self.rng = np.random.default_rng(seed)
        self.keyed, self.n_order, self.types, self.pool = keyed, n_order, dict(types or {}), pool
        self.events, self.seq = [], 0

    def names(self):
        return (["p"] if self.keyed else []) + [f"k{i}" for i in range(self.n_order)] + ["x", TS]

    def order_by(self):
        return [(f"k{i}", i % 2 == 0) for i in range(self.n_order)]

    def _values(self, col, n):
        t = self.types.get(col, "l")
        r = self.rng
        if self.pool == "extreme":
            pools = {"l": [INT64_MIN, INT64_MAX, 0, -1, 7], "L": [1 << 63, (1 << 64) - 1, 0, 5, (1 << 63) + 9],
                     "tsn": [0, 1, ORIGIN, INT64_MAX]}
            return r.choice(np.array(pools[t], dtype=NUMPY[t]), n)
        v = r.integers(0, self.pool if col != "p" else 4, n)
        if t == "L":
            return (v.astype(np.uint64) + np.uint64(1 << 63))
        if t == "tsn":
            return (v + ORIGIN).astype(np.int64)
        return (v - 1).astype(np.int64)

    def batch(self, ts):
        ts = np.asarray(ts, dtype=np.int64)
        cols = {}
        for c in self.names()[:-2]:
            cols[c] = self._values(c, len(ts))
        cols["x"] = np.arange(self.seq, self.seq + len(ts), dtype=np.int64)  # arrival order, for the reader
        self.seq += len(ts)
        cols[TS] = self.rng.permutation(ts)
        self.events.append(("batch", cols))

    def at(self, instants, per):
        self.batch(np.repeat(np.asarray(instants, dtype=np.int64), per))

    def wm(self, w):
        self.events.append(("wm", w))

    def restart(self):
        self.events.append(("restart",))


def s_ties(st):
    for r in range(4):
        base = ORIGIN + r * 10 * SEC
        for _ in range(3):
            st.at(base + np.arange(3) * SEC, 700)
        st.wm(base + 10 * SEC)
    st.wm(INT64_MAX)


def s_edges(st):
    st.batch([])
    st.at([0, 5, ORIGIN], 3)
    st.wm(0)  # releases none
    st.wm(1)  # releases instant 0
    st.at([ORIGIN - 1, ORIGIN, ORIGIN + 1], 2)  # late at w - 1 once w = ORIGIN
    st.wm(ORIGIN)
    st.at([ORIGIN - 1, ORIGIN, ORIGIN + 3], 4)  # ORIGIN - 1 is late, ORIGIN is not
    st.batch([])
    st.at(ORIGIN + 10 + np.arange(300), 2)
    st.wm(ORIGIN + 400)  # hundreds
    st.at([INT64_MAX - 5, INT64_MAX - 1], 3)
    st.wm(INT64_MAX)


def s_backlog(st):
    st.at(ORIGIN + np.arange(1 << 16) * 7, 2)
    st.at(ORIGIN + np.arange(1 << 16) * 7, 1)
    st.wm(ORIGIN + (1 << 16) * 7)  # releases 2^16 instants
    st.wm(INT64_MAX)


def s_restarts(st):
    for r in range(6):
        base = ORIGIN + r * 10 * SEC
        st.at(base + np.arange(5) * SEC, 40)
        st.at(base + 12 * SEC + np.arange(3) * SEC, 30)  # stays open past the next watermark
        st.wm(base + 10 * SEC)
        st.restart()
    st.wm(INT64_MAX)


def s_extremes(st):
    s_edges(st)


SHAPES = {"ties": s_ties, "edges": s_edges, "backlog": s_backlog, "restarts": s_restarts, "extremes": s_extremes}


# ---- GPU driver -------------------------------------------------------------------------------------------------------
def to_arrow(cols, types):
    arrays = []
    for c, v in cols.items():
        t = "tsn" if c == TS else types.get(c, "l")
        if t == "L":
            arrays.append(pa.array(np.asarray(v, dtype=np.uint64), type=pa.uint64()))
        else:
            a = pa.array(np.asarray(v, dtype=np.int64), type=pa.int64())
            arrays.append(a.cast(ARROW[t]) if t == "tsn" else a)
    return pa.RecordBatch.from_arrays(arrays, names=list(cols))


def host_rows(rb):
    """Rows of an output batch as dicts of Python ints (struct children flattened as <struct>_<child>)."""
    cols = {}
    for name, col in zip(rb.schema.names, rb.columns):
        if pa.types.is_struct(col.type):
            for f, child in zip(col.type, col.flatten()):
                cols[f"{name}_{f.name}"] = child
        else:
            cols[name] = col
    out = {}
    for name, col in cols.items():
        if pa.types.is_timestamp(col.type):
            col = col.cast(pa.int64())
        out[name] = col.to_numpy(zero_copy_only=False)
    n = rb.num_rows
    return [{c: int(v[i]) for c, v in out.items()} for i in range(n)]


def wf_config(st, function, top_n, name="fn"):
    from arroyo_b200 import config
    return config.WindowFunctionConfig(function, "p" if st.keyed else None, st.order_by(), name, top_n)


def run_gpu(st, cfg, entry):
    """The CUDA operator on `st.events`: (per watermark the output rows in order, per restart table "input" as
    {instant: rows}, total rows_in, total rows_late, output schemas)."""
    import torch

    import arroyo_b200 as ab
    from arroyo_b200 import ffi, operators as native
    from arroyo_b200.context import clamp_watermark
    first = next(ev[1] for ev in st.events if ev[0] == "batch")
    schema = to_arrow(first, st.types).schema

    def make():
        return native.WindowFunction(cfg, input_schema=schema)

    op, ctx, outs, states, keep, pending, schemas, totals = make(), ab.OperatorContext(1), [], [], [], [], [], [0, 0]

    def rows_of(batches):
        schemas.extend(b.schema for b in batches)
        return [r for b in batches for r in host_rows(b)]

    def run_pending(wm):
        ex = native.ExportedBatches([to_arrow(b, st.types) for b in pending])
        wms = (C.c_int64 * len(pending))(*([ffi.NO_WATERMARK] * (len(pending) - 1) + [wm]))
        col = ab.Collector()
        op.run_batches(ex, wms, col)
        op.handle_watermark_poll(col, block=True)
        pending.clear()
        return col.batches

    def add_stats():
        s = op.stats()
        totals[0] += s["rows_in"]
        totals[1] += s["rows_late"]

    for ev in st.events:
        if ev[0] == "batch":
            b = ev[1]
            n = len(b[TS])
            if entry == "run_batches" and n:
                pending.append(b)
            elif entry == "sliced":
                rb, s, i = to_arrow(b, st.types), 0, 0
                while s < n:
                    z = min((1, 7, 1023, 2)[i % 4], n - s)
                    op.process_batch(rb.slice(s, z), ctx, None)
                    s, i = s + z, i + 1
            elif entry == "device":
                dev = [torch.from_numpy(np.ascontiguousarray(b[c]).view(np.int64)).cuda() for c in b]
                keep.append(dev)
                op.process_device_batch([t.data_ptr() for t in dev], n)
            else:
                op.process_batch(to_arrow(b, st.types), ctx, None)
        elif ev[0] == "wm":
            ctx.watermarks.set(0, ev[1])
            if entry == "run_batches" and pending:
                outs.append(rows_of(run_pending(clamp_watermark(ev[1]))))
            else:
                col = ab.Collector()
                op.handle_watermark(ev[1], ctx, col)
                outs.append(rows_of(col.batches))
        else:
            if pending:
                assert not run_pending(ffi.NO_WATERMARK)
            add_stats()
            table = ctx.table("input", 0)
            before = {t: len(bs) for t, bs in table.batches.items()}
            op.handle_checkpoint(None, ctx, None)
            state = {}
            for t, bs in table.batches.items():
                for rb in bs[before.get(t, 0):]:
                    assert rb.schema.names == list(schema.names)
                    assert [f.type for f in rb.schema] == [f.type for f in schema]
                    state.setdefault(t, []).extend(host_rows(rb))
            states.append(state)
            op.close()
            op = make()
            op.on_start(ctx)
    add_stats()
    op.close()
    return outs, states, totals[0], totals[1], schemas


CASES = [  # shape, function, keyed, types, ORDER BY keys, entry, top_n
    ("ties", "row_number", True, {}, 1, "host", 0),
    ("ties", "rank", True, {}, 2, "device", 0),
    ("ties", "dense_rank", False, {}, 1, "sliced", 0),
    ("ties", "rank", False, {}, 3, "run_batches", 3),
    ("ties", "row_number", True, {"p": "L", "k0": "L"}, 1, "device", 1),
    ("ties", "dense_rank", True, {"p": "tsn", "k1": "tsn"}, 2, "host", 1),
    ("edges", "row_number", True, {}, 4, "host", 0),
    ("edges", "dense_rank", False, {}, 2, "device", 3),
    ("edges", "rank", True, {"k0": "L", "k1": "tsn"}, 3, "run_batches", 1 << 40),
    ("edges", "row_number", False, {}, 1, "sliced", 1),
    ("extremes", "row_number", True, {}, 2, "host", 0),
    ("extremes", "rank", True, {"p": "L", "k0": "L", "k1": "L"}, 2, "device", 0),
    ("extremes", "dense_rank", True, {"p": "tsn", "k0": "tsn", "k1": "l", "k2": "L", "k3": "tsn"}, 4, "sliced", 0),
    ("backlog", "row_number", True, {}, 1, "device", 0),
    ("backlog", "dense_rank", False, {}, 2, "host", 1),
    ("restarts", "row_number", True, {}, 2, "host", 0),
    ("restarts", "rank", False, {"k0": "L"}, 1, "device", 1),
    ("restarts", "dense_rank", True, {}, 3, "run_batches", 0),
    ("restarts", "row_number", True, {"p": "tsn"}, 1, "sliced", 3),
]


def case_id(c):
    return f"{c[0]}-{c[1]}-{'keyed' if c[2] else 'unkeyed'}-{''.join(f'{k}{v}' for k, v in c[3].items()) or 'l'}-" \
           f"{c[4]}keys-{c[5]}-top{c[6]}"


@pytest.mark.gpu
@pytest.mark.parametrize("shape,function,keyed,types,n_order,entry,top_n", CASES, ids=[case_id(c) for c in CASES])
def test_window_function_against_exact_reference(shape, function, keyed, types, n_order, entry, top_n):
    seed = zlib.crc32(f"{shape}/{function}/{entry}".encode()) % 1000
    st = Stream(seed, keyed, n_order, types, pool="extreme" if shape == "extremes" else 3)
    SHAPES[shape](st)
    cfg = wf_config(st, function, top_n)
    want, late, want_states = window_fn_emissions(st.events, cfg.partition_by, cfg.order_by, function, "fn", top_n)
    got, states, rows_in, rows_late, schemas = run_gpu(st, cfg, entry)
    assert len(got) == len(want)
    for i, (w, g) in enumerate(zip(want, got)):
        assert len(g) == len(w), ("watermark", i, len(g), len(w))
        for j, (a, b) in enumerate(zip(w, g)):
            assert a == b, ("watermark", i, "row", j, a, b)
    assert states == want_states
    assert rows_in == sum(len(ev[1][TS]) for ev in st.events if ev[0] == "batch")
    assert rows_late == late
    for s in schemas:
        assert s.names == st.names() + ["fn"] and s.field("fn").type == pa.uint64()
        for c in st.names()[:-2]:
            assert s.field(c).type == ARROW[types.get(c, "l")]


# ---- golden: most_active_driver_last_hour, fully on the GPU ------------------------------------------------------------
def _most_active_driver(inputs, device, top_n):
    """hop(1 min, 1 h) count(*) GROUP BY driver_id (CUDA sliding aggregate), ROW_NUMBER() OVER (PARTITION BY window
    ORDER BY count DESC, driver_id DESC) (CUDA window function, fed at every watermark), restarted at 0.3 and 0.6 of
    the stream."""
    import arroyo_b200 as ab
    from arroyo_b200 import config, operators as native
    from tests import golden_cases as GC
    from tests import gpu_ops as G
    s_cfg = O.WindowAggConfig(width=GC.HOUR, slide=GC.MIN, key_names=["driver_id"], aggs=[O.Agg("count", None, "count")],
                              window_index=1)
    sliding = native.SlidingAggregatingWindowFunc(s_cfg)
    w_cfg = config.WindowFunctionConfig("row_number", None, [("count", True), ("driver_id", True)], "row_number", top_n)
    ts_t = pa.timestamp("ns")
    if device:
        schema = pa.schema([("driver_id", pa.int64()), ("window_start", ts_t), ("window_end", ts_t),
                            ("count", pa.int64()), (TS, ts_t)])
    else:
        schema = pa.schema([("driver_id", pa.int64()), ("window", pa.struct([("start", ts_t), ("end", ts_t)])),
                            ("count", pa.int64()), (TS, ts_t)])
    wf = native.WindowFunction(w_cfg, input_schema=schema)
    s_ctx, w_ctx, rows = ab.OperatorContext(1), ab.OperatorContext(1), []

    def advance(wm):
        nonlocal wf
        s_ctx.watermarks.set(0, wm)
        if device:
            wins = sliding.handle_watermark_device(wm)
            for n, ptrs in wins:
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
            want_names = schema.names + ["row_number"]
            assert rb.schema.names == want_names and rb.schema.field("row_number").type == pa.uint64()
            if not device:
                wt = rb.schema.field("window").type
                assert [(f.name, f.type) for f in wt] == [("start", ts_t), ("end", ts_t)]
            rows.extend(host_rows(rb))

    batches = O.source_batches({"driver_id": inputs["cars_driver_id"], TS: inputs["cars_ts"]}, GC.BATCH)
    restarts = {int(len(batches) * 0.3), int(len(batches) * 0.6)}
    gen = O.WatermarkGenerator(GC.HOUR)
    for i, b in enumerate(batches):
        sliding.process_batch(G.to_arrow(b), s_ctx, None)
        wm = gen.process_batch(b[TS])
        if wm is not None:
            advance(wm)
        if i in restarts:
            wf.handle_checkpoint(None, w_ctx, None)
            wf.close()
            wf = native.WindowFunction(w_cfg, input_schema=schema)
            wf.on_start(w_ctx)
    advance(O.FINAL_WATERMARK)
    sliding.close()
    wf.close()
    return [{"start": r["window_start"], "end": r["window_end"], "driver_id": r["driver_id"], "count": r["count"],
             "row_number": r["row_number"]} for r in rows if top_n or r["row_number"] == 1]


@pytest.mark.gpu
@pytest.mark.parametrize("top_n", [1, 0], ids=["top1", "filtered"])
@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
def test_most_active_driver_golden(golden, device, top_n):
    from tests.golden_cases import multiset
    inputs, expected = golden
    assert multiset(_most_active_driver(inputs, device, top_n)) == multiset(expected["most_active_driver_last_hour"])


# ---- scale ------------------------------------------------------------------------------------------------------------
def lexsort_ranks(ts, p, keys, descs, function):
    """Order (stable, by ts, p, keys) and function values computed with numpy."""
    n = len(ts)
    sort_keys = [np.arange(n)]
    for k, d in reversed(list(zip(keys, descs))):
        sort_keys.append(~k if d else k)
    sort_keys += [p, ts]
    order = np.lexsort(sort_keys)
    st, sp = ts[order], p[order]
    seg = np.r_[True, (st[1:] != st[:-1]) | (sp[1:] != sp[:-1])]
    peer = seg.copy()
    for k in keys:
        sk = k[order]
        peer[1:] |= sk[1:] != sk[:-1]
    pos = np.arange(n)
    seg_pos = np.maximum.accumulate(np.where(seg, pos, 0))
    if function == "row_number":
        return order, (pos - seg_pos + 1).astype(np.uint64)
    if function == "rank":
        return order, (np.maximum.accumulate(np.where(peer, pos, 0)) - seg_pos + 1).astype(np.uint64)
    cp = np.cumsum(peer)
    return order, (cp - cp[seg_pos] + 1).astype(np.uint64)


def _device_run(cols, names, cfg, wm):
    """One device batch of `cols` through a fresh operator, then watermark `wm`: the output columns as numpy."""
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
    out = {}
    for rb in col.batches:
        for c, a in zip(rb.schema.names, rb.columns):
            a = a.cast(pa.int64()) if pa.types.is_timestamp(a.type) else a
            out.setdefault(c, []).append(a.to_numpy(zero_copy_only=False))
    return {c: np.concatenate(v) for c, v in out.items()}, stats


@pytest.mark.gpu
@pytest.mark.parametrize("shape", ["one_instant_2_20_partitions", "one_partition"])
def test_scale_2_24_rows(shape):
    from arroyo_b200 import config
    n = 1 << 24
    rng = np.random.default_rng(31)
    t = ORIGIN + 5 * SEC
    keyed = shape != "one_partition"
    cols = {"p": rng.integers(0, 1 << 20, n).astype(np.int64), "k": rng.integers(-50, 50, n).astype(np.int64),
            "x": np.arange(n, dtype=np.int64), TS: np.full(n, t, dtype=np.int64)}
    names = ["p", "k", "x", TS]
    for function in ("row_number", "rank", "dense_rank"):
        cfg = config.WindowFunctionConfig(function, "p" if keyed else None, [("k", True)], "fn")
        got, stats = _device_run(cols, names, cfg, t + 1)
        order, want = lexsort_ranks(cols[TS], cols["p"] if keyed else np.zeros(n, np.int64), [cols["k"]], [True],
                                    function)
        assert np.array_equal(got["x"], cols["x"][order]), function
        assert np.array_equal(got["fn"], want), function
        assert stats["rows_out"] == n and stats["windows_out"] == 1
    assert keyed or int(want.max()) == 100  # dense_rank over 100 distinct keys; row_number reached 2^24 above


@pytest.mark.gpu
def test_sliding_1m_keys_device_top1():
    """2^20-key sliding windows fed device-resident for 20 slides, top_n = 1: per window the key with the largest sum,
    ties to the largest key."""
    import torch

    import arroyo_b200 as ab
    from arroyo_b200 import config, operators as native
    from tests.test_gpu_window_time import _Ptr
    keys, slide = 1 << 20, SEC
    s_cfg = O.WindowAggConfig(width=4 * slide, slide=slide, key_names=["key"], aggs=[O.Agg("sum", "v", "s")],
                              window_index=1)
    ts_t = pa.timestamp("ns")
    sliding = native.SlidingAggregatingWindowFunc(
        s_cfg, input_schema=pa.schema([("key", pa.int64()), ("v", pa.int64()), (TS, ts_t)]), expected_keys=keys)
    names = ["key", "window_start", "window_end", "s", TS]
    schema = pa.schema([(c, ts_t if c in ("window_start", "window_end", TS) else pa.int64()) for c in names])
    wf = native.WindowFunction(config.WindowFunctionConfig("row_number", None, [("s", True), ("key", True)], "rn", 1),
                               input_schema=schema)
    rng = np.random.default_rng(5)
    ctx, wctx, checked = ab.OperatorContext(1), ab.OperatorContext(1), 0
    for step in range(24):
        k = rng.permutation(keys).astype(np.int64)
        v = rng.integers(-1000, 1000, keys).astype(np.int64)
        ts = ORIGIN + step * slide + rng.integers(0, slide, keys).astype(np.int64)
        dev = [torch.from_numpy(a).cuda() for a in (k, v, ts)]
        sliding.process_device_batch([t.data_ptr() for t in dev], keys)
        wm = ORIGIN + step * slide
        if step < 4:
            continue
        wins = sliding.handle_watermark_device(wm)
        want = []
        for n, ptrs in wins:
            host = {c: torch.as_tensor(_Ptr(p, n, "<i8"), device="cuda").cpu().numpy() for c, p in zip(names, ptrs)}
            best = np.lexsort((host["key"], host["s"]))[-1]
            want.append({c: int(host[c][best]) for c in names})
            wf.process_device_batch(ptrs, n)
        wf.flush()
        wctx.watermarks.set(0, wm)
        col = ab.Collector()
        wf.handle_watermark(wm, wctx, col)
        got = [r for rb in col.batches for r in host_rows(rb)]
        assert [{c: r[c] for c in names} for r in got] == sorted(want, key=lambda r: r[TS])
        assert all(r["rn"] == 1 for r in got)
        checked += len(got)
    assert checked >= 20
    sliding.close()
    wf.close()


# ---- memory -----------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_emitted_rows_are_reclaimed():
    """500 watermarks, each releasing the previous round's instants: device memory in use stops growing."""
    import torch

    import arroyo_b200 as ab
    from arroyo_b200 import operators as native
    st = Stream(9, True, 2)
    rounds, per = 500, 200
    first = {c: np.zeros(1, np.int64) for c in st.names()}
    op = native.WindowFunction(wf_config(st, "rank", 0), input_schema=to_arrow(first, {}).schema)
    ctx = ab.OperatorContext(1)
    torch.cuda.init()
    free_at = {}
    for r in range(rounds):
        base = ORIGIN + r * per * SEC
        st.events.clear()
        st.at(base + np.arange(per, dtype=np.int64) * SEC, 5)
        op.process_batch(to_arrow(st.events[0][1], {}), ctx, None)
        ctx.watermarks.set(0, base)
        col = ab.Collector()
        op.handle_watermark(base, ctx, col)
        assert sum(b.num_rows for b in col.batches) == (0 if r == 0 else per * 5)
        if r in (20, rounds - 1):
            free_at[r] = torch.cuda.mem_get_info()[0]
    op.close()
    assert abs(free_at[rounds - 1] - free_at[20]) <= 4 << 20, free_at


# ---- refusals ---------------------------------------------------------------------------------------------------------
def _ffi_config(**kw):
    from arroyo_b200 import ffi
    cfg = ffi.OpConfig()
    cfg.kind = ffi.WINDOW_FUNCTION
    cfg.window_fn = ffi.FN_ROW_NUMBER
    cfg.n_cols = 3
    cfg.timestamp_col = 2
    cfg.n_aggs = 1
    cfg.aggs[0].kind = ffi.ORDER_DESC
    cfg.aggs[0].input_col = 1
    for k, v in kw.items():
        setattr(cfg, k, v)
    return cfg


def _create(cfg):
    from arroyo_b200 import ffi
    lib, h, err = ffi.load(), C.c_void_p(), C.create_string_buffer(256)
    st = lib.arroyo_b200_op_create(C.byref(cfg), C.byref(h), err, 256)
    if h:
        lib.arroyo_b200_op_destroy(h)
    return st


@pytest.mark.gpu
def test_refusals():
    import arroyo_b200 as ab
    from arroyo_b200 import config, ffi, operators as native
    assert _create(_ffi_config()) == ffi.OK
    assert _create(_ffi_config(n_key_cols=2)) == ffi.UNSUPPORTED
    assert _create(_ffi_config(n_aggs=0)) == ffi.INVALID_ARGUMENT
    assert _create(_ffi_config(n_aggs=5)) == ffi.INVALID_ARGUMENT
    assert _create(_ffi_config(window_fn=4)) == ffi.INVALID_ARGUMENT
    assert _create(_ffi_config(window_fn=0)) == ffi.INVALID_ARGUMENT
    assert _create(_ffi_config(slide_ns=-1)) == ffi.INVALID_ARGUMENT
    bad_kind = _ffi_config()
    bad_kind.aggs[0].kind = ffi.AGG_MAX_I64
    assert _create(bad_kind) == ffi.INVALID_ARGUMENT

    ts_t = pa.timestamp("ns")
    cfg = config.WindowFunctionConfig("rank", None, [("a", False)], "r")
    floats = pa.schema([("key", pa.int64()), ("a", pa.float64()), (TS, ts_t)])
    with pytest.raises(ffi.UnsupportedPlan):  # a Float64 ORDER BY key
        native.WindowFunction(cfg, input_schema=floats)
    schema = pa.schema([("key", pa.int64()), ("a", pa.int64()), (TS, ts_t)])
    op = native.WindowFunction(cfg, input_schema=schema)
    ctx = ab.OperatorContext(1)
    nulls = pa.RecordBatch.from_arrays([pa.array([1, None], pa.int64()), pa.array([1, 2], pa.int64()),
                                        pa.array([ORIGIN, ORIGIN], ts_t)], schema=schema)
    with pytest.raises(ffi.UnsupportedPlan):
        op.process_batch(nulls, ctx, None)
    negative = pa.RecordBatch.from_arrays([pa.array([1], pa.int64()), pa.array([1], pa.int64()),
                                           pa.array([-5], pa.int64()).cast(ts_t)], schema=schema)
    with pytest.raises(ffi.ArroyoB200Error) as e:
        op.process_batch(negative, ctx, None)
    assert e.value.status == ffi.PANIC
    with pytest.raises(ffi.UnsupportedPlan):
        op.handle_watermark_device(ORIGIN)
    with pytest.raises(ffi.UnsupportedPlan):
        op.handle_watermark_device_begin(ORIGIN)
    # state batches of the wrong layout: a missing column, a column of another type; nothing is taken
    good = pa.RecordBatch.from_arrays([pa.array([1], pa.int64()), pa.array([2], pa.int64()), pa.array([ORIGIN], ts_t)],
                                      schema=schema)
    fresh = native.WindowFunction(cfg, input_schema=schema)
    for bad in (pa.RecordBatch.from_arrays([pa.array([1], pa.int64()), pa.array([ORIGIN], ts_t)], names=["key", TS]),
                pa.RecordBatch.from_arrays([pa.array([1], pa.int64()), pa.array([2], pa.uint64()),
                                            pa.array([ORIGIN], ts_t)], names=["key", "a", TS])):
        with pytest.raises(ffi.ArroyoB200Error) as e:
            fresh._on_start([good, bad], ffi.INT64_MIN, ffi.INT64_MIN)
        assert e.value.status == ffi.INVALID_ARGUMENT
    col = ab.Collector()
    ctx2 = ab.OperatorContext(1)
    ctx2.watermarks.set(0, INT64_MAX)
    fresh.handle_watermark(INT64_MAX, ctx2, col)
    assert not col.batches and fresh.stats()["rows_in"] == 0
    fresh.close()
    op.close()
    # a struct column stays refused by every other kind
    inst = native.InstantAggregatingWindowFunc(
        config.WindowAggConfig(width=0, key_names=["key"], aggs=[config.Agg("max", "a", "m")], final_projection=False),
        input_schema=schema)
    nested = pa.RecordBatch.from_arrays(
        [pa.array([1], pa.int64()), pa.StructArray.from_arrays([pa.array([1], pa.int64())], names=["s"]),
         pa.array([ORIGIN], ts_t)], names=["key", "a", TS])
    with pytest.raises(ffi.UnsupportedPlan):
        inst.process_batch(nested, ctx, None)
    inst.close()
