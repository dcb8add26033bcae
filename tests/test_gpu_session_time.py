"""Event time of the session window aggregate against tests/exact_reference.session_emissions, watermark by
watermark: which rows are late, which sessions exist, which watermark closes each of them, every column, and the
rows_in / rows_late / n_keys statistics.

Every stream is an explicit list of ("batch", cols), ("wm", w) and ("restart",) events (a restart is
handle_checkpoint, a new operator and on_start).  The shapes go where session.cu has edges: rows and watermarks exactly
on a gap boundary, the tie at the advance rule, runs that peel one row at a time, a key with 600,000 sessions, a hot key
with 10^6 rows in one launch, edge and UInt64 / timestamp keys, timestamps at both ends of their range, gaps from 1 ns
to 2^40 ns, and restarts with open sessions, pending runs and expired state.  Values are functions of the timestamp,
so rows with equal timestamps are interchangeable and every stream has one answer."""
import zlib

import numpy as np
import pyarrow as pa
import pytest

from oracle import arroyo_oracle as O
from tests import exact_reference as X

A = O.Agg
TS = O.TIMESTAMP
INT64_MIN = -(1 << 63)
INT64_MAX = (1 << 63) - 1
SEC = 1_000_000_000
ORIGIN = 1_700_000_000 * SEC
PLANS = {
    "count": [A("count", None, "n")],
    "sum": [A("sum", "a", "sa")],
    "min": [A("min", "a", "mna")],
    "max": [A("max", "a", "mxa")],
    "avg": [A("avg", "a", "ava")],
    # several columns, as in test_gpu_agg_plans.PLANS; "b" is large, so its sums wrap and AVG takes the f64 bound
    "mix2": [A("count", None, "n"), A("sum", "a", "sa"), A("avg", "b", "avb"), A("max", "b", "mxb")],
    "mix3": [A("min", "a", "mna"), A("sum", "b", "sb"), A("avg", "c", "avc"), A("count", None, "n"),
             A("max", "c", "mxc")],
    "mix4": [A("sum", "a", "sa"), A("min", "b", "mnb"), A("max", "c", "mxc"), A("avg", "d", "avd"),
             A("avg", "a", "ava")],
}
VALUE_COLS = ("a", "b", "c", "d")


def values(ts, col):
    """A column's values as a function of the timestamp: small for "a", up to 2^62 in magnitude for "b" and "d"."""
    with np.errstate(over="ignore"):
        salt = np.uint64((0x9E3779B97F4A7C15 * (1 + VALUE_COLS.index(col))) % (1 << 64))
        h = np.asarray(ts, dtype=np.int64).view(np.uint64) + salt
        h = (h ^ (h >> np.uint64(31))) * np.uint64(0xBF58476D1CE4E5B9)
        h ^= h >> np.uint64(29)
    if col in ("a", "c"):
        return (h % np.uint64(2001)).astype(np.int64) - 1000
    return (h >> np.uint64(1)).astype(np.int64) - (1 << 62)


class Stream:
    """`keys`: "one" (key 7), "few" (5 keys), "edge" (INT64_MIN, INT64_MAX, 0, -1), "u64" (keys >= 2^63), "ts"
    (timestamp-typed keys) or "none" (the unkeyed operator)."""

    KEYSETS = {"one": [7], "few": [3, 11, -5, 1 << 40, 99], "edge": [INT64_MIN, INT64_MAX, 0, -1],
               "u64": [(1 << 63), (1 << 64) - 1, (1 << 63) + 12345, 5], "ts": [0, SEC, ORIGIN, -1]}

    def __init__(self, seed, keys, gap, n_vals=4):
        self.rng = np.random.default_rng(seed)
        self.keys, self.gap, self.n_vals = keys, gap, n_vals
        self.events = []

    def keyset(self):
        return self.KEYSETS[self.keys]

    def batch(self, ts, key=None):
        """Rows at `ts`; `key`: None (random keys of the key set), a scalar or an array of keys."""
        ts = np.asarray(ts, dtype=np.int64).reshape(-1)
        n = len(ts)
        cols = {}
        if self.keys != "none":
            ks = self.keyset()
            if key is None:
                key = np.asarray(ks, dtype=object)[self.rng.integers(0, len(ks), n)]
            key = np.broadcast_to(np.asarray(key, dtype=object), (n,))
            cols["key"] = np.array([int(k) for k in key], dtype=np.uint64 if self.keys == "u64" else np.int64)
        for c in VALUE_COLS[:self.n_vals]:
            cols[c] = values(ts, c)
        cols[TS] = ts
        self.events.append(("batch", O.Batch(cols)))

    def per_key(self, ts):
        """The same timestamps once for every key of the key set, in one batch."""
        ks = [None] if self.keys == "none" else self.keyset()
        self.batch(np.tile(np.asarray(ts, dtype=np.int64), len(ks)), None if self.keys == "none" else np.repeat(
            np.asarray(ks, dtype=object), len(ts)))

    def wm(self, w):
        self.events.append(("wm", int(w)))

    def restart(self):
        self.events.append(("restart",))

    def end(self):
        self.wm(INT64_MAX)
        return self


# ---- stream shapes: f(seed, keys, gap) -> Stream ------------------------------------------------------------------------
def s_gap_edges(seed, keys, g):
    st, o = Stream(seed, keys, g), ORIGIN
    st.wm(o - 10 * g)
    # inside one run: g - 1, g and g + 1 apart, then equal timestamps
    st.per_key([o, o + g - 1, o + 2 * g - 1, o + 3 * g, o + 3 * g, o + 3 * g + 1, o + 4 * g + 2])
    st.wm(o - g)
    # across batches: a run whose first row is exactly de + gap, one g - 1 after, one g + 1 after
    st.per_key([o + 5 * g + 2])
    st.per_key([o + 6 * g + 1, o + 6 * g + 1])
    st.per_key([o + 7 * g + 3])
    st.wm(o + 3 * g)
    # a breaking row at index 1, in the middle, and last (the i == n case)
    st.per_key([o + 8 * g, o + 10 * g, o + 10 * g + 1])
    st.per_key([o + 8 * g + 1, o + 8 * g + 2, o + 9 * g + 3, o + 9 * g + 4, o + 12 * g])
    st.per_key([o + 9 * g + 5, o + 9 * g + 6, o + 14 * g])
    st.wm(o + 9 * g)
    st.per_key([o + 12 * g + 1, o + 13 * g])
    return st.end()


def s_wm_edges(seed, keys, g):
    st, o = Stream(seed, keys, g), ORIGIN
    st.wm(-5 * g)  # a negative watermark makes nothing late
    st.per_key([o, o + g // 2])
    st.wm(o - 30 * g)  # far behind the data
    st.wm(o - 30 * g)  # the same watermark twice
    de = o + g // 2
    st.wm(de + g)  # de + gap: does not close
    st.per_key([de + g])
    st.wm(de + g + 1)  # de + gap + 1: closes
    # a pending start of exactly w + gap is not opened by the watermark, but by a row for that key under the same w
    w = de + 5 * g
    st.per_key([w + g, w + g + 3])
    st.wm(w)
    st.per_key([w + 7])
    st.wm(w)
    st.per_key([w + 4 * g])
    st.wm(w + 2 * g)
    st.wm(w + 2 * g + 10)
    return st.end()


def s_no_wm(seed, keys, g):
    """No watermark until end of data; the batches arrive in reverse time order."""
    st, o = Stream(seed, keys, g), ORIGIN
    for j in range(12, -1, -1):
        st.batch(o + j * g * 3 // 4 + st.rng.integers(0, g // 4 + 1, 6))
    st.batch(o + np.arange(0, 20 * g, g, dtype=np.int64))
    return st.end()


def s_late(seed, keys, g):
    st, o = Stream(seed, keys, g), ORIGIN
    st.per_key([o, o + g // 3])
    w = o + 2 * g
    st.wm(w)
    st.per_key([w - 1, w, w + 1])  # w - 1 is late, w is not
    st.batch(w - 1 - st.rng.integers(0, 5 * g, 40))  # a whole late batch
    mixed = np.asarray([w - g, w + 2, w - 2, w + g, w - 3 * g, w + 2 * g - 1, w + 5 * g], dtype=np.int64)
    st.batch(st.rng.permutation(np.tile(mixed, 4)))  # late rows mixed into runs
    st.wm(w + 3 * g)
    st.batch(w + 3 * g - 1 + st.rng.integers(-2, 3, 30))
    return st.end()


def s_disorder(seed, keys, g):
    st, o = Stream(seed, keys, g), ORIGIN
    st.wm(o - g)
    st.per_key([o + g, o + g + g // 2])
    st.wm(o)  # opens the session at o + g
    st.per_key([o + g // 4, o + g // 2])  # starts before ds, within the gap
    st.per_key([o + g // 8 + 1, o + 3 * g])
    st.wm(o + g // 8 + 1)
    # evens and odds: two runs of one key 0.75 gap apart peel one row at a time (session_aggregating_window.rs:610-614)
    x, b = 3 * g // 4, o + 10 * g
    st.per_key([b + 2 * k * x for k in range(40)])
    st.per_key([b + (2 * k + 1) * x for k in range(40)])
    st.wm(b - g)
    st.per_key([b + 80 * x + 1])
    return st.end()


def s_many_sessions(seed, keys, g, n_sessions=600_000, per_batch=1000):
    """One key (or the unkeyed operator) with n_sessions sessions of two rows that only the final watermark closes; a
    watermark far behind the data follows every batch, so every launch stays small."""
    st, o = Stream(seed, keys, g, n_vals=1), ORIGIN
    st.wm(o - 10 * g)
    ts = o + np.arange(2 * n_sessions, dtype=np.int64) * (2 * g)  # every row breaks the scan: two rows per session
    for i in range(0, len(ts), 2 * per_batch):
        st.batch(ts[i:i + 2 * per_batch], None if keys == "none" else 7)
        st.wm(o - 10 * g)
    return st.end()


def s_hot_key(seed, keys, g, n=1_000_000):
    """One key with 10^6 rows in one batch, in random order, next to cold keys."""
    st, o = Stream(seed, keys, g, n_vals=2), ORIGIN
    ts = o + st.rng.integers(0, n // 3 * g // 8, n).astype(np.int64)
    cold = o + st.rng.integers(0, 8 * g, 3000).astype(np.int64)
    key = np.concatenate([np.full(n, 7, dtype=object), st.rng.integers(100, 1100, 3000).astype(object)])
    order = st.rng.permutation(n + 3000)
    st.wm(o - g)
    st.batch(np.concatenate([ts, cold])[order], key[order])
    st.wm(o + n // 12 * g // 8)
    return st.end()


def s_unkeyed_big(seed, keys, g, n=2_200_000):
    """The unkeyed operator with two batches of more than 4 Mi rows in all: the second crosses the launch arena's cut."""
    st, o = Stream(seed, keys, g, n_vals=1), ORIGIN
    for j in range(2):
        st.batch(o + st.rng.integers(0, n // 4 * g // 8, n).astype(np.int64) + j * (n // 8 * g // 8))
    st.wm(o + n // 16 * g // 8)
    return st.end()


def s_growing_keys(seed, keys, g, n_keys=100_000):
    """expected_keys = 1, growing to 10^5 keys while sessions are open and runs are pending."""
    st, o = Stream(seed, "few", g, n_vals=2), ORIGIN
    st.wm(o - g)
    for j in range(5):
        k = st.rng.permutation(n_keys)[: n_keys // 2 + j * n_keys // 10]
        ts = o + j * g // 2 + st.rng.integers(0, g, len(k)).astype(np.int64)
        far = st.rng.random(len(k)) < 0.2
        ts[far] += 10 * g  # pending far ahead
        st.batch(ts, k.astype(object) * 7919 - 3)
        st.wm(o + j * g // 4)
    return st.end()


def s_time_range(seed, keys, g):
    """ts = 0 and timestamps up to INT64_MAX - 2 gap."""
    st = Stream(seed, keys, g)
    st.per_key([0, 0, 1, g - 1])
    st.wm(-g)
    st.per_key([g, 3 * g])
    st.wm(0)
    top = INT64_MAX - 2 * g
    st.per_key([top - 3 * g, top - g - 1, top])
    st.wm(top - 5 * g)
    st.per_key([top - 1, top])
    st.wm(top - g)
    return st.end()


def s_restarts(seed, keys, g):
    st, o = Stream(seed, keys, g), ORIGIN
    st.per_key([o + g, o + 2 * g - 5])
    st.restart()  # before any watermark: no late filter afterwards
    st.per_key([o, o + 10 * g])
    st.wm(o + g // 2)
    st.per_key([o + 2 * g, o + 40 * g])  # an open session and runs pending far ahead
    st.restart()
    st.restart()  # twice in a row
    st.per_key([o + g // 2, o + 3 * g - 1])
    st.wm(o + 5 * g)  # closes the first session
    st.restart()  # right after a watermark that closed sessions: they are not emitted again
    st.per_key([o + 5 * g, o + 11 * g - 1])
    st.wm(o + 12 * g)
    return st.end()


def s_long_session(seed, keys, g):
    """A session longer than 100 gaps: table "s" drops its early rows at a checkpoint, so the restored session is
    shorter, and what it emits differs from the stream without the restart."""
    st, o = Stream(seed, keys, g), ORIGIN
    st.wm(o - 3 * g)
    for j in range(0, 150, 10):
        st.per_key(o + (j + np.arange(10, dtype=np.int64)) * (g // 2))
        st.wm(o + (j - 5) * (g // 2))
    st.restart()
    st.per_key([o + 75 * g])
    st.wm(o + 74 * g)
    st.restart()
    st.per_key([o + 200 * g])
    return st.end()


def s_restart_no_data(seed, keys, g):
    """A restart after a watermark but before any on-time row: table "e" is empty, nothing is restored, and the new
    operator must still treat rows older than the watermark as late."""
    st, o = Stream(seed, keys, g), ORIGIN
    st.wm(o)
    st.per_key([o - 1])
    st.restart()
    st.per_key([o - g, o - 1, o, o + 1])
    st.wm(o + g // 2)
    return st.end()


def s_compact(seed, keys, g):
    """Many short sessions and pending runs across restarts, for a pool that compacts at 64 nodes."""
    st, o = Stream(seed, keys, g), ORIGIN
    st.wm(o - 8 * g)
    for j in range(40):
        st.batch(o + 2 * j * g + st.rng.integers(0, 3 * g, 50).astype(np.int64))
        st.wm(o + 2 * (j - 3) * g)
        if j % 13 == 12:
            st.restart()
    return st.end()


SHAPES = {
    "gap_edges": s_gap_edges, "wm_edges": s_wm_edges, "no_wm": s_no_wm, "late": s_late, "disorder": s_disorder,
    "many_sessions": s_many_sessions, "hot_key": s_hot_key, "unkeyed_big": s_unkeyed_big,
    "growing_keys": s_growing_keys, "time_range": s_time_range, "restarts": s_restarts,
    "long_session": s_long_session, "compact": s_compact, "restart_no_data": s_restart_no_data,
}
GAPS = {"5s": 5 * SEC, "1ns": 1, "999ns": 999, "30d": 30 * 86400 * SEC, "2^40": 1 << 40}


def make(name, keys, gap="5s", **kw):
    seed = zlib.crc32(f"{name}/{keys}/{gap}".encode()) % 1000
    return SHAPES[name](seed, keys, GAPS[gap], **kw)


SLICES = (1, 7, 1023, 2)


def sliced_events(events):
    """The events as the `sliced` entry hands them over: every batch cut into slices of 1, 7, 1023, 2, 1, ... rows.
    Each slice is a batch of its own, and a session's runs follow its batches."""
    out = []
    for ev in events:
        if ev[0] != "batch":
            out.append(ev)
            continue
        b, s, i = ev[1], 0, 0
        while s < b.num_rows:
            z = min(SLICES[i % 4], b.num_rows - s)
            out.append(("batch", O.Batch({c: v[s:s + z] for c, v in b.cols.items()})))
            s, i = s + z, i + 1
    return out


def config(st, plan):
    key_names = [] if st.keys == "none" else ["key"]
    return O.SessionConfig(gap=st.gap, key_names=key_names, aggs=PLANS[plan], window_index=len(key_names))


def reference(st, cfg):
    return X.session_emissions(st.events, cfg.key_names[0] if cfg.key_names else None, cfg.aggs, cfg.gap)


def run_oracle(st, cfg, impl="numpy"):
    """The numpy or C oracle on the same events: one list of output rows per watermark."""
    from oracle import c_oracle
    cls = {"numpy": O.SessionAggregatingWindowFunc, "c": c_oracle.SessionAggregatingWindowFunc}[impl]
    ctx, op, outs = O.OperatorContext(1), cls(cfg), []
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
            op = cls(cfg)
            op.on_start(ctx)
    return outs


def check_emissions(want, got, cfg, who):
    key = cfg.key_names[0] if cfg.key_names else None
    assert len(got) == len(want), (who, len(got), len(want))
    for i, (w, g) in enumerate(zip(want, got)):
        for r in g:
            assert int(r[TS]) == int(r["window_end"]) - 1, (who, i, r)
        errs = X.mismatches(w, g, lambda r: (int(r[key]) if key else None, int(r["window_start"])))
        assert not errs, (who, "watermark", i, errs[:8])


# ---- the CUDA operator ---------------------------------------------------------------------------------------------------
def key_type(st):
    return {"u64": pa.uint64(), "ts": pa.timestamp("ns")}.get(st.keys, pa.int64())


def arrow_batch(st, b):
    from tests.gpu_ops import to_arrow
    rb = to_arrow(b)
    if st.keys == "ts":
        i = rb.schema.names.index("key")
        rb = rb.set_column(i, pa.field("key", pa.timestamp("ns")), rb.column(i).cast(pa.timestamp("ns")))
    return rb


class _Ptr:
    def __init__(self, ptr, n, typestr):
        self.__cuda_array_interface__ = {"shape": (n,), "typestr": typestr, "data": (ptr, False), "version": 2}


def device_rows(wins, names):
    import torch
    rows = []
    for n, ptrs in wins:
        assert len(ptrs) == len(names)
        host = {c: torch.as_tensor(_Ptr(p, n, "<f8" if c.startswith("av") else "<i8"), device="cuda").cpu().numpy()
                for c, p in zip(names, ptrs)}
        rows += O.Batch(host).rows()
    return rows


def run_gpu(st, cfg, entry, expected_keys=0):
    """The CUDA operator on the same events.  Returns (one list of output rows per watermark, rows_in, rows_late,
    n_keys after the last watermark).  `device` feeds device batches and takes every watermark on the device;
    `poll_host` feeds device batches and alternates host (even) and device (odd) watermarks."""
    import torch

    import arroyo_b200 as ab
    from arroyo_b200 import operators as native
    from tests.gpu_ops import from_arrow
    first = next(ev[1] for ev in st.events if ev[0] == "batch")
    schema = arrow_batch(st, first).schema
    names = list(schema.names)
    key_names = list(cfg.key_names)
    dev_names = key_names[:cfg.window_index] + ["window_start", "window_end"] + key_names[cfg.window_index:] + \
        [a.name for a in cfg.aggs] + [TS]

    def make_op():
        return native.SessionAggregatingWindowFunc(cfg, input_schema=schema, expected_keys=expected_keys)

    op, ctx, outs, keep = make_op(), ab.OperatorContext(1), [], []
    device_input = entry in ("device", "poll_host")
    totals = [0, 0]

    def host_rows(batches):
        rows = []
        for b in batches:
            if key_names and not device_input:
                # device columns carry no Arrow type: the key of their sessions leaves as Int64 with the same bits
                assert b.schema.field("key").type == key_type(st), b.schema
            r = from_arrow(b).rows()
            if st.keys == "u64":
                for x in r:
                    x["key"] = int(x["key"]) % (1 << 64)
            rows += r
        return rows

    def dev_rows(wins):
        rows = device_rows(wins, dev_names)
        if st.keys == "u64":
            for x in rows:
                x["key"] = int(x["key"]) % (1 << 64)
        return rows

    for ev in st.events:
        if ev[0] == "batch":
            b = ev[1]
            if entry == "sliced":
                rb, s, i = arrow_batch(st, b), 0, 0
                while s < b.num_rows:
                    z = min(SLICES[i % 4], b.num_rows - s)
                    op.process_batch(rb.slice(s, z), ctx, None)
                    s, i = s + z, i + 1
            elif entry in ("device", "poll_host"):
                dev = [torch.from_numpy(np.ascontiguousarray(b[c]).view(np.int64)).cuda() for c in names]
                keep.append(dev)
                del keep[:-4]
                op.process_device_batch([t.data_ptr() for t in dev], b.num_rows)
            else:
                op.process_batch(arrow_batch(st, b), ctx, None)
        elif ev[0] == "wm":
            w = ev[1]
            ctx.watermarks.set(0, w)
            if entry == "device" or (entry == "poll_host" and len(outs) % 2 == 1):
                outs.append(dev_rows(op.handle_watermark_device(w)))
            else:
                col = ab.Collector()
                op.handle_watermark(w, ctx, col)
                outs.append(host_rows(col.batches))
            torch.cuda.synchronize()
            keep.clear()
        else:
            assert entry in ("host", "sliced"), "device input keeps no table 's': restarts use host entry points"
            s = op.stats()
            totals[0] += s["rows_in"]
            totals[1] += s["rows_late"]
            op.handle_checkpoint(None, ctx, None)
            op.close()
            op = make_op()
            op.on_start(ctx)
    s = op.stats()
    totals[0] += s["rows_in"]
    totals[1] += s["rows_late"]
    op.close()
    return outs, totals[0], totals[1], s["n_keys"]


# (shape, keys, gap, plan, entry, expected_keys): a cross section, not the product
CASES = [
    ("gap_edges", "few", "5s", "mix2", "host"),
    ("gap_edges", "one", "1ns", "count", "sliced"),
    ("gap_edges", "edge", "999ns", "sum", "device"),
    ("gap_edges", "none", "30d", "min", "host"),
    ("gap_edges", "u64", "2^40", "mix3", "poll_host"),
    ("gap_edges", "ts", "5s", "max", "host"),
    ("wm_edges", "few", "5s", "avg", "host"),
    ("wm_edges", "edge", "1ns", "mix4", "device"),
    ("wm_edges", "none", "999ns", "mix2", "sliced"),
    ("wm_edges", "u64", "5s", "count", "host"),
    ("wm_edges", "ts", "30d", "sum", "poll_host"),
    ("no_wm", "few", "5s", "mix3", "host"),
    ("no_wm", "none", "2^40", "avg", "device"),
    ("no_wm", "edge", "999ns", "max", "sliced"),
    ("late", "few", "5s", "mix4", "sliced"),
    ("late", "one", "1ns", "mix2", "host"),
    ("late", "none", "5s", "sum", "poll_host"),
    ("late", "u64", "999ns", "min", "device"),
    ("disorder", "few", "5s", "mix2", "host"),
    ("disorder", "edge", "999ns", "avg", "sliced"),
    ("disorder", "none", "2^40", "mix3", "host"),
    ("disorder", "ts", "1ns", "count", "device"),
    ("time_range", "few", "5s", "mix4", "host"),
    ("time_range", "edge", "1ns", "sum", "device"),
    ("time_range", "none", "2^40", "max", "poll_host"),
    ("time_range", "u64", "30d", "mix2", "sliced"),
    ("restarts", "few", "5s", "mix2", "host"),
    ("restarts", "edge", "999ns", "mix3", "sliced"),
    ("restarts", "none", "30d", "avg", "host"),
    ("restarts", "u64", "1ns", "min", "host"),
    ("long_session", "few", "5s", "mix4", "host"),
    ("long_session", "none", "999ns", "sum", "sliced"),
    ("restart_no_data", "few", "5s", "mix2", "host"),
    ("restart_no_data", "none", "1ns", "count", "sliced"),
    ("compact", "few", "5s", "mix2", "host"),
    ("compact", "none", "999ns", "count", "host"),
]


def _counts(st, cfg, want, late, n_keys, got, rows_in, rows_late, n_keys_got):
    assert rows_in == sum(ev[1].num_rows for ev in st.events if ev[0] == "batch")
    assert rows_late == late
    if cfg.key_names:
        assert n_keys_got == n_keys


@pytest.mark.gpu
@pytest.mark.parametrize("shape,keys,gap,plan,entry", CASES, ids=["-".join(c) for c in CASES])
def test_session_event_time(shape, keys, gap, plan, entry, monkeypatch):
    if shape == "compact":
        monkeypatch.setenv("ARROYO_B200_SESSION_COMPACT_MIN", "64")
    st = make(shape, keys, gap)
    cfg = config(st, plan)
    ref = st
    if entry == "sliced":
        ref = Stream(0, keys, st.gap)
        ref.events = sliced_events(st.events)
    want, late, n_keys = reference(ref, cfg)
    got, rows_in, rows_late, nk = run_gpu(st, cfg, entry, expected_keys=64)
    check_emissions(want, got, cfg, "gpu")
    _counts(st, cfg, want, late, n_keys, got, rows_in, rows_late, nk)


# the shapes that are large, once each
BIG_CASES = [
    ("many_sessions", "one", "avg", "host"),
    ("many_sessions", "none", "sum", "device"),
    ("hot_key", "few", "mix2", "host"),
    ("hot_key", "few", "min", "poll_host"),
    ("unkeyed_big", "none", "avg", "host"),
    ("growing_keys", "few", "mix2", "host"),
    ("growing_keys", "few", "max", "device"),
]


@pytest.mark.gpu
@pytest.mark.parametrize("shape,keys,plan,entry", BIG_CASES, ids=["-".join(c) for c in BIG_CASES])
def test_session_event_time_large(shape, keys, plan, entry):
    st = make(shape, keys)
    cfg = config(st, plan)
    want, late, n_keys = reference(st, cfg)
    got, rows_in, rows_late, nk = run_gpu(st, cfg, entry, expected_keys=1 if shape == "growing_keys" else 64)
    check_emissions(want, got, cfg, "gpu")
    _counts(st, cfg, want, late, n_keys, got, rows_in, rows_late, nk)
    if shape == "many_sessions":
        assert len(want[-1]) >= 600_000
