"""The instant-window aggregate (InstantAggregatingWindowFunc: tumbling_aggregating_window.rs with width 0, what the
planner emits to aggregate an already-windowed stream) against its own exact reference, `instant_emissions`, watermark
by watermark: which rows are late, which instants each watermark releases, in what order, and every column.

Streams are lists of ("batch", cols), ("wm", w) and ("restart",) events (a restart is handle_checkpoint, a new operator
and on_start).  The CPU test pins the numpy oracle's width-0 operator to the same reference; the GPU tests also use the
oracle for the checkpoint interchange and restart runs."""
import ctypes as C
import zlib

import numpy as np
import pyarrow as pa
import pytest

from oracle import arroyo_oracle as O

A = O.Agg
TS = O.TIMESTAMP
SEC = 1_000_000_000
ORIGIN = 1_700_000_000 * SEC
INT64_MIN, INT64_MAX = -(1 << 63), (1 << 63) - 1
PLANS = {
    "ints": [A("count", None, "n"), A("sum", "a", "sa"), A("avg", "a", "ava")],
    "minmax": [A("count", None, "n"), A("min", "a", "mna"), A("max", "a", "mxa"), A("sum", "a", "sa")],
}


# ---- exact reference --------------------------------------------------------------------------------------------------
def _agg_value(kind, vals):
    if kind == "count":
        return len(vals)
    if kind == "sum":
        return (sum(vals) + (1 << 63)) % (1 << 64) - (1 << 63)  # Int64 SUM wraps
    if kind == "avg":
        return sum(float(v) for v in vals) / len(vals)
    return min(vals) if kind == "min" else max(vals)


def instant_emissions(events, key_name, aggs):
    """The instant window's event time (tumbling_aggregating_window.rs with width 0, :280-291 and :321-392):

    * bin(ts) = ts; the group is (instant, key), or the instant alone when unkeyed;
    * a row is late iff ts < w for the last watermark w before its batch; before the first watermark nothing is late;
    * watermark w releases every open instant < w, in ascending order; instants >= w stay; end of data is INT64_MAX;
    * a restart (checkpoint, new operator, on_start) changes nothing.

    Watermarks must not decrease.  Returns (per watermark the list of (instant, {key or None: row}) it releases, in
    order, the number of late rows).  Rows hold the key, the aggregates and `_timestamp` = instant."""
    cols_of = sorted({a.col for a in aggs if a.col is not None})
    open_, last_wm, late, out = {}, None, 0, []
    for ev in events:
        if ev[0] == "restart":
            continue
        if ev[0] == "batch":
            cols = ev[1].cols
            ts = [int(t) for t in cols[TS]]
            keys = [int(k) for k in cols[key_name]] if key_name else [None] * len(ts)
            for r, (t, k) in enumerate(zip(ts, keys)):
                if last_wm is not None and t < last_wm:
                    late += 1
                    continue
                open_.setdefault(t, {}).setdefault(k, []).append({c: int(cols[c][r]) for c in cols_of})
            continue
        w = min(int(ev[1]), INT64_MAX)
        assert last_wm is None or w >= last_wm, "watermarks must not decrease"
        last_wm = w
        released = []
        for t in sorted(x for x in open_ if x < w):
            rows = {}
            for k, vals in open_.pop(t).items():
                row = {a.name: _agg_value(a.kind, [v[a.col] for v in vals] if a.col else vals) for a in aggs}
                row[TS] = t
                if key_name:
                    row[key_name] = k
                rows[k] = row
            released.append((t, rows))
        out.append(released)
    return out, late


def check_emissions(want, got, key_name, who=""):
    """`got`: per watermark the output rows in emission order.  Instants must leave in ascending order, and the rows
    equal the reference's: integers exactly, AVG within 1e-6 relative."""
    assert len(got) == len(want), (who, len(got), len(want))
    for i, (w, g) in enumerate(zip(want, got)):
        inst = [int(r[TS]) for r in g]
        assert inst == sorted(inst), (who, "watermark", i, "instants out of order")
        exp = {(t, k): row for t, rows in w for k, row in rows.items()}
        seen = {}
        for r in g:
            gk = (int(r[TS]), int(r[key_name]) if key_name else None)
            assert gk not in seen, (who, "watermark", i, "group emitted twice", gk)
            seen[gk] = r
        assert sorted(seen, key=str) == sorted(exp, key=str), (who, "watermark", i, sorted(set(seen) ^ set(exp), key=str)[:8])
        for gk, row in exp.items():
            for c, v in row.items():
                if isinstance(v, float):
                    assert abs(float(seen[gk][c]) - v) <= 1e-6 * abs(v), (who, i, gk, c, seen[gk][c], v)
                else:
                    assert int(seen[gk][c]) == v, (who, i, gk, c, seen[gk][c], v)


# ---- streams ----------------------------------------------------------------------------------------------------------
class Stream:
    def __init__(self, seed, keys):
        self.rng = np.random.default_rng(seed)
        self.keys = keys
        self.events = []

    def _keys(self, n):
        r = self.rng
        if self.keys == "few":
            return r.integers(-1, 2, n).astype(np.int64)
        if self.keys == "many":
            return r.integers(0, 3000, n).astype(np.int64) * 7919 - 13
        if self.keys == "extreme":
            return r.choice(np.array([INT64_MIN, INT64_MAX, 0, -1], dtype=np.int64), n)
        if self.keys == "u64":
            return r.choice(np.array([1 << 63, (1 << 64) - 1, 0, 5], dtype=np.uint64), n)
        if self.keys == "tsn":
            return r.choice(np.array([0, 1, ORIGIN, INT64_MAX], dtype=np.int64), n)
        raise KeyError(self.keys)

    def batch(self, ts):
        ts = np.asarray(ts, dtype=np.int64)
        cols = {}
        if self.keys != "none":
            cols["key"] = self._keys(len(ts))
        cols["a"] = self.rng.integers(-1000, 1000, len(ts)).astype(np.int64)
        cols[TS] = self.rng.permutation(ts)
        self.events.append(("batch", O.Batch(cols)))

    def at(self, instants, per=3):
        self.batch(np.repeat(np.asarray(instants, dtype=np.int64), per))

    def wm(self, w):
        self.events.append(("wm", int(w)))

    def restart(self):
        self.events.append(("restart",))

    def end(self):
        self.wm(INT64_MAX)
        return self


def s_edges(seed, keys):
    st, o = Stream(seed, keys), ORIGIN
    st.wm(o - 1000 * SEC)  # before any row: releases nothing
    st.at([o + k * SEC for k in range(6)])
    st.wm(o - 500 * SEC)  # releases nothing
    st.wm(o + 1)  # releases one instant
    w = o + 2 * SEC
    st.wm(w)
    st.batch([w, w, w - 1, w - 1, w + 7, o, w])  # ts == w kept, w - 1 and o late
    st.batch([])
    st.wm(w)  # the same watermark again: nothing new
    st.at([o + k * SEC for k in range(10, 310)], per=2)
    st.wm(o + 400 * SEC)  # releases hundreds
    st.at([o + 400 * SEC, o + 400 * SEC - 1, o + 401 * SEC])
    st.wm(o + 400 * SEC + 1)
    return st.end()


def s_extremes(seed, keys):
    st = Stream(seed, keys)
    big = INT64_MAX - 2
    st.batch([0, 0, 1, 2, big, big + 1, big, INT64_MAX])  # INT64_MAX itself never leaves
    st.wm(1)  # releases 0
    st.batch([0, 1, 1, 3])
    st.wm(3)
    st.batch([big, big - 5])
    st.wm(big)
    st.batch([big - 1, big, big + 1])
    return st.end()


def s_backlog(seed, keys):
    st, o = Stream(seed, keys), ORIGIN
    for chunk in range(4):
        st.at([o + (chunk * 200 + k) * SEC - 1 for k in range(200)], per=2)
    st.wm(o + 500 * SEC)
    st.at([o + 700 * SEC, o + 900 * SEC])
    st.wm(o + 900 * SEC)
    return st.end()


def s_restarts(seed, keys):
    st, o = Stream(seed, keys), ORIGIN
    st.at([o + k * SEC for k in range(10)])
    st.restart()  # before any watermark
    st.wm(o + 3 * SEC)
    st.restart()
    st.restart()  # twice in a row, no new rows
    st.at([o + 2 * SEC, o + 3 * SEC, o + 12 * SEC])  # late, kept at ts == w, new
    st.wm(o + 5 * SEC)
    st.at([o + 6 * SEC, o + 9 * SEC])
    st.restart()  # open instants on both sides of the next watermark
    st.wm(o + 8 * SEC)
    st.restart()
    st.at([o + 8 * SEC, o + 7 * SEC, o + 20 * SEC])
    return st.end()


SHAPES = {"edges": s_edges, "extremes": s_extremes, "backlog": s_backlog, "restarts": s_restarts}


# ---- CPU: the oracle's width-0 operator is the reference ---------------------------------------------------------------
def _random_stream(seed, keys):
    st, o = Stream(seed, keys), ORIGIN
    w = None
    for _ in range(40):
        r = st.rng.random()
        if r < 0.5:
            lo = (w if w is not None else o) - 3 * SEC
            st.at(lo + st.rng.integers(0, 12, st.rng.integers(0, 6)) * SEC, per=int(st.rng.integers(1, 4)))
        elif r < 0.85:
            w = (w if w is not None else o) + int(st.rng.integers(0, 3)) * SEC + int(st.rng.integers(0, 2))
            st.wm(w)
        else:
            st.restart()
    return st.end()


@pytest.mark.parametrize("keys", ["none", "few", "many"])
@pytest.mark.parametrize("plan", ["ints", "minmax"])
def test_oracle_width_zero_matches_instant_emissions(keys, plan):
    for seed in range(6):
        st = _random_stream(seed * 31 + len(keys), keys)
        key = None if keys == "none" else "key"
        cfg = O.WindowAggConfig(width=0, key_names=[key] if key else [], aggs=PLANS[plan], final_projection=False)
        ctx, op, outs = O.OperatorContext(1), O.TumblingAggregatingWindowFunc(cfg), []
        for ev in st.events:
            if ev[0] == "batch":
                op.process_batch(ev[1], ctx, O.Collector())
            elif ev[0] == "wm":
                ctx.watermarks.set(0, ev[1])
                col = O.Collector()
                op.handle_watermark(ev[1], ctx, col)
                outs.append([r for b in col.batches for r in b.rows()])
            else:
                op.handle_checkpoint(ctx)
                op = O.TumblingAggregatingWindowFunc(cfg)
                op.on_start(ctx)
        want, _ = instant_emissions(st.events, key, cfg.aggs)
        check_emissions(want, outs, key, f"oracle seed {seed}")


# ---- GPU drivers ------------------------------------------------------------------------------------------------------
def to_arrow(batch, tsn_key=False):
    from tests.gpu_ops import to_arrow as base
    rb = base(batch)
    if not tsn_key:
        return rb
    cols = [c.cast(pa.timestamp("ns")) if n == "key" else c for n, c in zip(rb.schema.names, rb.columns)]
    return pa.RecordBatch.from_arrays(cols, names=rb.schema.names)


def gpu_config(keys, plan, **kw):
    from arroyo_b200 import config
    key_names = [] if keys == "none" else ["key"]
    aggs = [config.Agg(a.kind, a.col, a.name) for a in PLANS[plan]]
    return config.WindowAggConfig(width=0, key_names=key_names, aggs=aggs, final_projection=kw.pop("nested", False),
                                  **kw)


def run_gpu(st, cfg, entry, tsn_key=False):
    """The CUDA operator on `st.events`: (per watermark the output rows in order, rows_in, rows_late, out schemas)."""
    import torch

    import arroyo_b200 as ab
    from arroyo_b200 import ffi, operators as native
    from arroyo_b200.context import clamp_watermark
    from tests.gpu_ops import from_arrow
    first = next(ev[1] for ev in st.events if ev[0] == "batch")
    schema = to_arrow(first, tsn_key).schema
    names = list(schema.names)

    def make():
        return native.InstantAggregatingWindowFunc(cfg, input_schema=schema)

    op, ctx, outs, keep, pending, schemas = make(), ab.OperatorContext(1), [], [], [], []
    totals = [0, 0]

    def host_rows(batches):
        schemas.extend(b.schema for b in batches)
        return [r for b in batches for r in from_arrow(b).rows()]

    def run_pending(wm):
        ex = native.ExportedBatches([to_arrow(b, tsn_key) for b in pending])
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
            if entry == "run_batches" and b.num_rows:
                pending.append(b)
            elif entry == "sliced":
                rb, s, i = to_arrow(b, tsn_key), 0, 0
                while s < b.num_rows:
                    z = min((1, 7, 1023, 2)[i % 4], b.num_rows - s)
                    op.process_batch(rb.slice(s, z), ctx, None)
                    s, i = s + z, i + 1
            elif entry == "device":
                dev = [torch.from_numpy(np.ascontiguousarray(b[c]).view(np.int64)).cuda() for c in names]
                keep.append(dev)
                op.process_device_batch([t.data_ptr() for t in dev], b.num_rows)
            else:
                op.process_batch(to_arrow(b, tsn_key), ctx, None)
        elif ev[0] == "wm":
            w = ev[1]
            ctx.watermarks.set(0, w)
            if entry == "run_batches" and pending:
                outs.append(host_rows(run_pending(clamp_watermark(w))))
            else:
                col = ab.Collector()
                op.handle_watermark(w, ctx, col)
                outs.append(host_rows(col.batches))
        else:
            if pending:
                assert not run_pending(ffi.NO_WATERMARK)
            add_stats()
            op.handle_checkpoint(None, ctx, None)
            op.close()
            op = make()
            op.on_start(ctx)
    add_stats()
    op.close()
    return outs, totals[0], totals[1], schemas


CASES = [
    ("edges", "few", "ints", "host"),
    ("edges", "none", "minmax", "device"),
    ("edges", "many", "minmax", "sliced"),
    ("edges", "few", "ints", "run_batches"),
    ("extremes", "extreme", "minmax", "host"),
    ("extremes", "u64", "ints", "host"),
    ("extremes", "tsn", "minmax", "sliced"),
    ("extremes", "none", "ints", "run_batches"),
    ("extremes", "few", "minmax", "device"),
    ("backlog", "many", "ints", "device"),
    ("backlog", "none", "minmax", "host"),
    ("restarts", "few", "minmax", "host"),
    ("restarts", "many", "ints", "device"),
    ("restarts", "none", "ints", "sliced"),
    ("restarts", "u64", "minmax", "run_batches"),
]


@pytest.mark.gpu
@pytest.mark.parametrize("shape,keys,plan,entry", CASES, ids=["-".join(c) for c in CASES])
def test_instant_window_event_time(shape, keys, plan, entry):
    st = SHAPES[shape](zlib.crc32(f"{shape}/{keys}".encode()) % 1000, keys)
    cfg = gpu_config(keys, plan)
    key = None if keys == "none" else "key"
    want, late = instant_emissions(st.events, key, PLANS[plan])
    got, rows_in, rows_late, schemas = run_gpu(st, cfg, entry, tsn_key=keys == "tsn")
    check_emissions(want, got, key, "gpu")
    assert rows_in == sum(ev[1].num_rows for ev in st.events if ev[0] == "batch")
    assert rows_late == late
    if key and entry != "device":  # the key leaves with its input type
        want_type = {"u64": pa.uint64(), "tsn": pa.timestamp("ns")}.get(keys, pa.int64())
        assert all(s.field(0).type == want_type for s in schemas)


@pytest.mark.gpu
def test_watermark_releases_2_20_instants():
    """One watermark releases 2^20 instants (a session-window upstream ends every session at its own timestamp)."""
    import arroyo_b200 as ab
    from arroyo_b200 import operators as native
    from tests.gpu_ops import from_arrow
    n = 1 << 20
    rng = np.random.default_rng(3)
    inst = ORIGIN + np.arange(n, dtype=np.int64) * 3
    ts = np.concatenate([inst, inst[rng.integers(0, n, n // 2)]])
    a = rng.integers(-10**12, 10**12, len(ts)).astype(np.int64)
    perm = rng.permutation(len(ts))
    batch = O.Batch({"a": a[perm], TS: ts[perm]})
    cfg = gpu_config("none", "minmax")
    op = native.InstantAggregatingWindowFunc(cfg, input_schema=to_arrow(batch).schema)
    ctx, col = ab.OperatorContext(1), ab.Collector()
    op.process_batch(to_arrow(batch), ctx, None)
    ctx.watermarks.set(0, int(inst[-1]) + 1)
    op.handle_watermark(int(inst[-1]) + 1, ctx, col)
    got = O.Batch.concat([from_arrow(b) for b in col.batches])
    assert np.array_equal(got[TS], inst)
    order = np.argsort(ts, kind="stable")
    st, sa = ts[order], a[order]
    starts = np.flatnonzero(np.r_[True, st[1:] != st[:-1]])
    assert np.array_equal(got["n"], np.diff(np.r_[starts, len(st)]))
    assert np.array_equal(got["mna"], np.minimum.reduceat(sa, starts))
    assert np.array_equal(got["mxa"], np.maximum.reduceat(sa, starts))
    assert np.array_equal(got["sa"], np.add.reduceat(sa, starts))
    s = op.stats()
    assert s["windows_out"] == n and s["rows_out"] == n and s["n_keys"] == 0
    op.close()


@pytest.mark.gpu
def test_hot_group_is_bit_exact():
    """2^24 rows in one unkeyed instant: every warp's rows combine into one group before the atomics."""
    import arroyo_b200 as ab
    from arroyo_b200 import config, operators as native
    from tests.gpu_ops import from_arrow
    n = 1 << 24
    rng = np.random.default_rng(11)
    a = rng.integers(INT64_MIN, INT64_MAX, n, dtype=np.int64, endpoint=True)
    t = ORIGIN + 10 * SEC - 1
    batch = O.Batch({"a": a, TS: np.full(n, t, dtype=np.int64)})
    aggs = [config.Agg("count", None, "n"), config.Agg("sum", "a", "s"), config.Agg("min", "a", "lo"),
            config.Agg("max", "a", "hi")]
    cfg = config.WindowAggConfig(width=0, aggs=aggs, final_projection=False)
    op = native.InstantAggregatingWindowFunc(cfg, input_schema=to_arrow(batch).schema)
    ctx, col = ab.OperatorContext(1), ab.Collector()
    op.process_batch(to_arrow(batch), ctx, None)
    ctx.watermarks.set(0, t + 1)
    op.handle_watermark(t + 1, ctx, col)
    rows = [r for b in col.batches for r in from_arrow(b).rows()]
    assert len(rows) == 1
    r = rows[0]
    with np.errstate(over="ignore"):
        want_sum = int(np.add.reduce(a, dtype=np.int64))
    assert (int(r["n"]), int(r["s"]), int(r["lo"]), int(r["hi"]), int(r[TS])) == (n, want_sum, int(a.min()), int(a.max()), t)
    op.close()


@pytest.mark.gpu
def test_emitted_groups_are_reclaimed():
    """500 watermarks, each opening fresh instants and releasing the previous round's: n_keys is the open-group count
    after every emission, and device memory in use stops growing after the first rounds."""
    import torch

    import arroyo_b200 as ab
    from arroyo_b200 import operators as native
    st = Stream(21, "few")
    cfg = gpu_config("few", "ints")
    rounds, per = 500, 300
    first = O.Batch({"key": np.zeros(1, np.int64), "a": np.zeros(1, np.int64), TS: np.full(1, ORIGIN, np.int64)})
    op = native.InstantAggregatingWindowFunc(cfg, input_schema=to_arrow(first).schema)
    ctx = ab.OperatorContext(1)
    torch.cuda.init()
    free_at = {}
    for r in range(rounds):
        base = ORIGIN + r * per * SEC
        inst = base + np.arange(per, dtype=np.int64) * SEC
        ts = np.repeat(inst, 4)
        keys = np.tile(np.array([-1, 0, 1, 1], dtype=np.int64), per)
        b = O.Batch({"key": keys, "a": st.rng.integers(-9, 9, len(ts)).astype(np.int64), TS: ts})
        op.process_batch(to_arrow(b), ctx, None)
        ctx.watermarks.set(0, base)  # releases the previous round
        col = ab.Collector()
        op.handle_watermark(base, ctx, col)
        assert sum(x.num_rows for x in col.batches) == (0 if r == 0 else per * 3)
        assert op.stats()["n_keys"] == per * 3
        if r in (20, rounds - 1):
            free_at[r] = torch.cuda.mem_get_info()[0]
    op.close()
    assert abs(free_at[rounds - 1] - free_at[20]) <= 4 << 20, free_at


# ---- restarts ---------------------------------------------------------------------------------------------------------
def windowed_stream(seed, n_instants, per, keyed, batch=32):
    """An upstream window's output: rows stamped with window ends, instants in ascending order, in batches of 32."""
    rng = np.random.default_rng(seed)
    ts = np.repeat(ORIGIN + np.arange(1, n_instants + 1, dtype=np.int64) * 2 * SEC - 1, per)
    cols = {}
    if keyed:
        cols["key"] = rng.integers(0, 40, len(ts)).astype(np.int64)
    cols["a"] = rng.integers(-10**6, 10**6, len(ts)).astype(np.int64)
    cols[TS] = ts
    return O.source_batches(cols, batch)


@pytest.mark.gpu
@pytest.mark.parametrize("keyed", [True, False], ids=["keyed", "unkeyed"])
@pytest.mark.parametrize("frac", [0.3, 0.7])
def test_restart_matches_oracle(keyed, frac):
    from arroyo_b200 import operators as native
    from tests import gpu_ops as G
    from tests.restart_ops import GpuKit, RestartOps
    from tests.test_gpu_parity import assert_same

    class _GpuInstant(G._WindowOp):  # the tests.gpu_ops adapter, for the restart harness
        native_cls = native.InstantAggregatingWindowFunc

    batches = windowed_stream(5, 300, 9, keyed)
    aggs = PLANS["ints"] + [A("min", "a", "mna"), A("max", "a", "mxa")]
    cfg = O.WindowAggConfig(width=0, key_names=["key"] if keyed else [], aggs=aggs, final_projection=False)
    want = O.run_single_input(O.TumblingAggregatingWindowFunc(cfg), batches).batches
    harness = RestartOps(O, GpuKit, frac)
    op = _GpuInstant(cfg, input_schema=to_arrow(batches[0]).schema)
    got = harness.run_single_input(op, batches, ctx=GpuKit.make_ctx(1)).batches
    assert_same(want, got, float_cols=("ava",), ordered=False)


@pytest.mark.gpu
@pytest.mark.parametrize("plan", ["ints", "minmax"])
def test_checkpoint_interchange_with_oracle(plan):
    """Table "t" written by the oracle restores into the CUDA operator and the reverse, each continuing to the output
    of an uninterrupted run; both operators write the same per-instant state."""
    import arroyo_b200 as ab
    from arroyo_b200 import operators as native
    from tests.gpu_ops import from_arrow
    from tests.test_gpu_checkpoint_interchange import _merged, _run_prefix
    from tests.test_gpu_parity import assert_same
    batches = windowed_stream(8, 200, 7, True)
    cfg = O.WindowAggConfig(width=0, key_names=["key"], aggs=PLANS[plan], final_projection=False)
    want = O.run_single_input(O.TumblingAggregatingWindowFunc(cfg), batches).batches
    half = len(batches) // 2
    schema = to_arrow(batches[0]).schema
    o_op, o_ctx, o_out, o_gen = O.TumblingAggregatingWindowFunc(cfg), O.OperatorContext(1), O.Collector(), O.WatermarkGenerator()
    g_op = native.InstantAggregatingWindowFunc(cfg, input_schema=schema)
    g_ctx, g_out, g_gen = ab.OperatorContext(1), ab.Collector(), ab.WatermarkGenerator()
    for lo, hi in ((0, half - 3), (half - 3, half)):  # two checkpoints: the second one writes deltas only
        _run_prefix(o_op, o_ctx, o_out, o_gen, batches[lo:hi])
        _run_prefix(g_op, g_ctx, g_out, g_gen, batches[lo:hi], adapt=to_arrow)
        o_op.handle_checkpoint(o_ctx)
        g_op.handle_checkpoint(None, g_ctx, g_out)
    g_op.close()
    wm = o_ctx.last_present_watermark()
    assert wm == g_ctx.last_present_watermark()
    o_state = {t: bs for t, bs in o_ctx.table("t", 0).all_batches_for_watermark(wm)}
    g_state = {}
    for t, rb in g_ctx.table("t", 0).all_batches_for_watermark(wm):
        g_state.setdefault(t, []).append(from_arrow(rb))
    assert o_state and sorted(o_state) == sorted(g_state)
    for t in o_state:
        assert _merged(o_state[t]) == _merged(g_state[t]), f"instant {t}"
        for b in g_state[t]:
            assert bool((b[TS] == t).all()) and list(b.cols) == list(o_state[t][0].cols)
    rest = batches[half:]
    fcols = tuple(a.name for a in cfg.aggs if a.kind == "avg")

    def finish(op, ctx, out, gen, adapt=lambda b: b):
        _run_prefix(op, ctx, out, gen, rest, adapt=adapt)
        ctx.watermarks.set(0, O.FINAL_WATERMARK)
        op.handle_watermark(O.FINAL_WATERMARK, ctx, out)

    # oracle-written table -> CUDA operator
    r_ctx = ab.OperatorContext(1)
    r_ctx.watermarks.set(0, wm)
    for t, bs in o_state.items():
        for b in bs:
            r_ctx.table("t", 0).insert(t, to_arrow(b))
    r_op = native.InstantAggregatingWindowFunc(cfg, input_schema=schema)
    r_op.on_start(r_ctx)
    r_out, r_gen = ab.Collector(), ab.WatermarkGenerator()
    r_gen.__dict__.update(g_gen.__dict__)
    finish(r_op, r_ctx, r_out, r_gen, adapt=to_arrow)
    r_op.close()
    assert_same(want, [from_arrow(b) for b in g_out.batches + r_out.batches], float_cols=fcols, ordered=False)
    # CUDA-written table -> oracle operator
    c_ctx = O.OperatorContext(1)
    c_ctx.watermarks.set(0, wm)
    for t, bs in g_state.items():
        c_ctx.table("t", 0).flushed[t] = list(bs)
    c_op = O.TumblingAggregatingWindowFunc(cfg)
    c_op.on_start(c_ctx)
    c_out, c_gen = O.Collector(), O.WatermarkGenerator()
    c_gen.__dict__.update(o_gen.__dict__)
    finish(c_op, c_ctx, c_out, c_gen)
    assert_same(want, list(o_out.batches) + list(c_out.batches), float_cols=fcols, ordered=False)


# ---- nested form ------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("where", ["first", "middle", "last"])
def test_nested_form_window_struct(where):
    import arroyo_b200 as ab
    from arroyo_b200 import operators as native
    from tests.gpu_ops import from_arrow
    W = 10 * SEC
    st = s_edges(4, "few")
    wi = {"first": 0, "middle": 2, "last": 1 + len(PLANS["ints"])}[where]
    cfg = gpu_config("few", "ints", nested=True, nested_width=W, window_index=wi)
    want, _ = instant_emissions(st.events, "key", PLANS["ints"])
    op = native.InstantAggregatingWindowFunc(cfg, input_schema=to_arrow(st.events[1][1]).schema)
    ctx, got = ab.OperatorContext(1), []
    for ev in st.events:
        if ev[0] == "batch":
            op.process_batch(to_arrow(ev[1]), ctx, None)
            continue
        ctx.watermarks.set(0, ev[1])
        col = ab.Collector()
        op.handle_watermark(ev[1], ctx, col)
        rows = []
        for b in col.batches:
            names = ["key"] + [a.name for a in PLANS["ints"]]
            names.insert(wi, "window")
            assert b.schema.names == names + [TS], b.schema.names
            wt = b.schema.field("window").type
            assert [(f.name, f.type) for f in wt] == [("start", pa.timestamp("ns")), ("end", pa.timestamp("ns"))]
            rows += from_arrow(b).rows()
        for r in rows:
            assert int(r["window_start"]) == int(r[TS]) - W + 1 and int(r["window_end"]) == int(r[TS]) + 1
        got.append(rows)
    op.close()
    check_emissions(want, got, "key", "nested")


# ---- golden: Nexmark q5 with MaxBids on the instant window -------------------------------------------------------------
def _q5(inputs, device):
    """hop(2 s, 10 s) count(*) GROUP BY auction (CUDA sliding aggregate), MaxBids = max(num) per window (CUDA instant
    aggregate, nested form, W = 10 s, fed watermark by watermark), joined ON window.start (CUDA instant join)."""
    import arroyo_b200 as ab
    from arroyo_b200 import config, operators as native
    from tests import golden_cases as GC
    from tests import gpu_ops as G
    from tests.test_gpu_window_time import device_rows
    W = 10 * SEC
    s_cfg = O.WindowAggConfig(width=W, slide=2 * SEC, key_names=["auction"], aggs=[O.Agg("count", None, "num")],
                              window_index=1)
    sliding = native.SlidingAggregatingWindowFunc(s_cfg)
    m_cfg = config.WindowAggConfig(width=0, aggs=[config.Agg("max", "num", "maxn")], final_projection=True,
                                   nested_width=W, window_index=0)
    dev_names = ["auction", "window_start", "window_end", "num", TS]
    if device:
        schema = pa.schema([(n, pa.timestamp("ns") if n == TS else pa.int64()) for n in dev_names])
    else:
        schema = pa.schema([("num", pa.int64()), (TS, pa.timestamp("ns"))])
    maxbids = native.InstantAggregatingWindowFunc(m_cfg, input_schema=schema)
    s_ctx, m_ctx = ab.OperatorContext(1), ab.OperatorContext(1)
    left, right = [], []

    def advance(wm):
        s_ctx.watermarks.set(0, wm)
        if device:
            wins = sliding.handle_watermark_device(wm)
            for n, ptrs in wins:
                maxbids.process_device_batch(ptrs, n)
            maxbids.flush()  # the sliding windows' buffers are reused by its next call
            rows = device_rows(wins, dev_names)
            if rows:
                left.append(O.Batch({c: np.array([r[c] for r in rows], dtype=np.int64)
                                     for c in ("auction", "num", "window_start", TS)}))
        else:
            col = ab.Collector()
            sliding.handle_watermark(wm, s_ctx, col)
            for rb in col.batches:
                b = G.from_arrow(rb)
                left.append(O.Batch({"auction": b["auction"], "num": b["num"], "window_start": b["window_start"],
                                     TS: b[TS]}))
                maxbids.process_batch(pa.RecordBatch.from_arrays([rb.column("num"), rb.column(TS)], names=["num", TS]),
                                      m_ctx, None)
        m_ctx.watermarks.set(0, wm)
        col = ab.Collector()
        maxbids.handle_watermark(wm, m_ctx, col)
        for rb in col.batches:
            b = G.from_arrow(rb)
            assert np.array_equal(b["window_start"], b[TS] - W + 1)
            right.append(O.Batch({"w": b["window_start"], "maxn": b["maxn"], TS: b[TS]}))

    gen = O.WatermarkGenerator()
    for b in O.source_batches({"auction": inputs["bids_auction"], TS: inputs["bids_ts"]}, GC.BATCH):
        sliding.process_batch(G.to_arrow(b), s_ctx, None)
        wm = gen.process_batch(b[TS])
        if wm is not None:
            advance(wm)
    advance(O.FINAL_WATERMARK)
    assert maxbids.stats()["windows_out"] == sum(x.num_rows for x in right) > 0
    sliding.close()
    maxbids.close()
    join = G.InstantJoin(O.JoinConfig(left_on=["window_start"], right_on=["w"], join_type="inner"))
    out = GC._drive_join(G, join, left, right)
    return [{"auction": r["auction"], "count": r["num"]} for r in out.rows() if r["num"] >= r["maxn"]]


@pytest.mark.gpu
@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
def test_nexmark_q5_with_instant_window(golden, device):
    from tests.golden_cases import multiset
    inputs, expected = golden
    assert multiset(_q5(inputs, device)) == multiset(expected["nexmark_q5"])


# ---- refusals ---------------------------------------------------------------------------------------------------------
def _ffi_config(n_key_cols=0):
    from arroyo_b200 import ffi
    cfg = ffi.OpConfig()
    cfg.kind = ffi.INSTANT_AGGREGATE
    cfg.n_cols = 3
    cfg.timestamp_col = 2
    cfg.n_key_cols = n_key_cols
    cfg.n_aggs = 1
    cfg.aggs[0].kind = ffi.AGG_MAX_I64
    cfg.aggs[0].input_col = 1
    return cfg


def _create(cfg):
    from arroyo_b200 import ffi
    lib, h, err = ffi.load(), C.c_void_p(), C.create_string_buffer(256)
    st = lib.arroyo_b200_op_create(C.byref(cfg), C.byref(h), err, 256)
    if h:
        lib.arroyo_b200_op_destroy(h)
    return st, err.value


@pytest.mark.gpu
def test_refusals():
    import arroyo_b200 as ab
    from arroyo_b200 import config, ffi, operators as native
    assert _create(_ffi_config(n_key_cols=2))[0] == ffi.UNSUPPORTED
    assert _create(_ffi_config())[0] == ffi.OK
    cfg = _ffi_config()
    cfg.kind = ffi.TUMBLING_AGGREGATE
    assert _create(cfg)[0] == ffi.UNSUPPORTED  # width 0 stays refused by the tumbling kind
    cfg = _ffi_config()
    cfg.final_projection = 1  # the nested form needs the upstream width
    assert _create(cfg)[0] == ffi.INVALID_ARGUMENT

    aggs = [config.Agg("max", "a", "mx")]
    c = config.WindowAggConfig(width=0, key_names=["key"], aggs=aggs, final_projection=False)
    floats = pa.RecordBatch.from_arrays([pa.array([1], pa.int64()), pa.array([1.5], pa.float64()),
                                         pa.array([ORIGIN], pa.timestamp("ns"))], names=["key", "a", TS])
    op = native.InstantAggregatingWindowFunc(c, input_schema=floats.schema)
    with pytest.raises(ffi.UnsupportedPlan):
        op.process_batch(floats, ab.OperatorContext(1), None)
    with pytest.raises(ffi.UnsupportedPlan):
        op.handle_watermark_device(ORIGIN)
    with pytest.raises(ffi.UnsupportedPlan):
        op.handle_watermark_device_begin(ORIGIN)
    # state batches of the wrong layout: a missing column, a column of the wrong type
    bad = pa.RecordBatch.from_arrays([pa.array([1], pa.int64()), pa.array([ORIGIN], pa.timestamp("ns"))],
                                     names=["key", TS])
    with pytest.raises(ffi.ArroyoB200Error) as e:
        op._on_start([bad], ffi.INT64_MIN, ffi.INT64_MIN)
    assert e.value.status == ffi.INVALID_ARGUMENT
    wrong_type = pa.RecordBatch.from_arrays([pa.array([1], pa.int64()), pa.array([1.0], pa.float64()),
                                             pa.array([ORIGIN], pa.timestamp("ns"))], names=["key", "mx[max]", TS])
    with pytest.raises(ffi.ArroyoB200Error) as e:
        op._on_start([wrong_type], ffi.INT64_MIN, ffi.INT64_MIN)
    assert e.value.status == ffi.INVALID_ARGUMENT
    op.close()
