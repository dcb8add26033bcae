"""The CUDA updating aggregate's time-to-idle ttl (arroyo_b200_op_set_clock, config gap_ns) against
tests/exact_ttl_reference.py, flush by flush, through the entry points of test_gpu_updating_restore.Driver.

* Int64, UInt64 and timestamp keys, the INT64_MIN key, the unkeyed plan; ttl shorter than, equal to and longer than
  the flush gap; flushes whose only rows are evictions; restarts after evictions (evicted keys stay gone, restored
  keys expire one ttl after the restart clock); statistics (n_keys counts live keys, rows_out the evictions).
* Crowded buckets from expected_keys = 256, with the clock moving between a call whose rows defer and their drain.
* ttl 0 with the clock moved far: the output and statistics of a run that never sets the clock.
* A clock that goes back, and set_clock on other operator kinds: refused, the stream unchanged afterwards.
* Table "a" interchange with the ttl oracle in both directions, and from a table written without tombstones.
* 2^24 rows over 2^20 keys, half of them expiring, bit-exact against a numpy group-by.
* Memory: 8 waves of 2^20 fresh keys, each expiring fully: n_keys returns to 0 and device memory stays flat."""
import zlib

import numpy as np
import pyarrow as pa
import pytest

from oracle import arroyo_oracle as O
from oracle import updating_oracle as U
from tests import test_gpu_updating_restore as R
from tests import updating_state_oracle as S
from tests import updating_ttl_oracle as L
from tests.exact_ttl_reference import updating_ttl
from tests.test_updating_restore_oracle import _Ctx
from tests.test_updating_ttl_oracle import STEP, TTLS, flush_errors, reference_events, table_errors, ttl_stream

pytestmark = pytest.mark.gpu
TS = O.TIMESTAMP


def rows_of(b):
    """Rows of an Arrow batch as dicts of Python values (timestamps as int, nulls as None)."""
    cols = {}
    for n in b.schema.names:
        a = b.column(n)
        cols[n] = (a.cast(pa.int64()) if pa.types.is_timestamp(a.type) else a).to_pylist()
    if "_is_retract" in cols:
        cols[U.IS_RETRACT] = cols.pop("_is_retract")
    return [dict(zip(cols, t)) for t in zip(*cols.values())]


class Driver(R.Driver):
    """test_gpu_updating_restore.Driver with a ttl and a clock the test moves (`now`)."""

    def __init__(self, st, aggs, entry, ttl, expected_keys=None):
        self.ttl, self.now = ttl, 0
        super().__init__(st, aggs, entry, expected_keys)

    def make(self, expected_keys):
        return self.native.UpdatingAggregatingFunc(self.cfg, input_schema=self.schema, expected_keys=expected_keys,
                                                   ttl=self.ttl, clock=lambda: self.now)

    def clock(self, t):
        self.send_pending()  # batches held for one call go with the clock of their own time
        self.now = t


def run(st, aggs, entry, ttl, checkpoints=(), restarts=(), expected_keys=None):
    """(rows per flush, table "a" rows after each checkpoint, stats at the end, rows_out since the last restart)."""
    d = Driver(st, aggs, entry, ttl, expected_keys)
    outs, tables, since, deferred = [], [], 0, 0
    for ev in st.events:
        if ev[0] == "clock":
            d.clock(ev[1])
        elif ev[0] == "batch":
            d.batch(ev[1])
        else:
            i = len(outs)
            cp = i in checkpoints or i in restarts
            g = d.flush("checkpoint" if cp else "tick")
            outs.append([] if g is None else rows_of(g))
            since += len(outs[-1])
            if cp:
                tables.append([rows_of(b) for b in d.ctx.key_value_table("a").batches])
            if i in restarts:
                deferred += d.op.stats()["rows_deferred"]
                d.restart()
                since = 0
    stats = d.op.stats()
    stats["rows_deferred"] += deferred  # over every operator of the run
    d.op.close()
    return outs, tables, stats, since


def live_keys(want):
    """The keys live after the last flush of exact_ttl_reference's flushes (restarts keep the live keys)."""
    live = set()
    for _, a, e in want:
        live = (live | set(a)) - set(e)
    return live


def check(st, aggs, ttl, outs, tables, want, want_tables, who):
    key = st.key_name()
    assert len(outs) == len(want), who
    for i, (g, w) in enumerate(zip(outs, want)):
        errs = flush_errors(g, w, key, ordered=True)
        assert not errs, (who, "flush", i, errs[:8])
    assert len(tables) == len(want_tables), who
    for j, (t, w) in enumerate(zip(tables, want_tables)):
        errs = table_errors(t, w, key, aggs)
        assert not errs, (who, "checkpoint", j, errs[:8])


def edge_keys(rng, n):
    return rng.choice(np.array([-(1 << 63), -(1 << 63) + 1, -1, 0, 1, (1 << 63) - 1, 42, 7919], dtype=np.int64), n)


def crowded(rng, n):
    """Keys that share bucket 0 of a 1- and a 2-bucket dictionary (expected_keys = 256): once more than a bucket's
    1280 ids arrive, rows defer until the dictionary has 4 buckets."""
    from tests import test_gpu_updating_changes as T
    return rng.choice(T.crowded_keys(2000, n_buckets=1), n)


# (shape, plan, entry, ttl, restarts: "none" | "mid" | "each")
CASES = [
    ("i64", "P2", "host", "equal", "mid"), ("i64", "P3", "sliced", "short", "mid"), ("u64", "P7", "device", "equal", "mid"),
    ("ts", "P8", "device_run", "short", "mid"), ("ts", "P1", "mixed", "equal", "none"), ("edge", "P2", "host", "equal", "mid"),
    ("edge", "COUNT", "device", "short", "each"), ("unkeyed", "P2", "host", "equal", "each"),
    ("unkeyed", "AMM", "sliced", "short", "mid"), ("i64", "MM", "mixed", "long", "mid"), ("i64", "P6a", "device", "equal", "each"),
    ("crowded", "P2", "host", "equal", "mid"), ("crowded", "P4", "device", "short", "none"),
    ("crowded", "COUNT", "device_run", "equal", "mid"),
]
KW = {"i64": {}, "u64": {"key_type": "u64"}, "ts": {"key_type": "ts"}, "unkeyed": {"key_type": None},
      "edge": {"keys_fn": edge_keys}, "crowded": {"keys_fn": crowded, "n_batches": 24, "expected_keys": 256}}


@pytest.mark.parametrize("shape,plan,entry,ttl,restarts", CASES, ids=["-".join(c) for c in CASES])
def test_flushes_equal_the_exact_reference(shape, plan, entry, ttl, restarts):
    from tests import test_gpu_updating_changes as T
    seed = zlib.crc32(f"{shape}/{plan}/{entry}/{ttl}".encode())
    st, aggs = ttl_stream(seed, **KW[shape]), T.PLANS[plan]
    key = st.key_name()
    n = sum(1 for ev in st.events if ev[0] == "flush")
    cps = set(range(1, n, 2))
    runs = {"none": [()], "mid": [(n // 2,)], "each": [(i,) for i in range(n - 1)]}[restarts]
    deferred = 0
    for r in runs:
        want, want_tables = updating_ttl(reference_events(st.events, cps, r), key, aggs, TTLS[ttl])
        outs, tables, stats, since = run(st, aggs, entry, TTLS[ttl], cps, r)
        deferred += stats["rows_deferred"]
        who = (shape, plan, entry, ttl, r)
        check(st, aggs, TTLS[ttl], outs, tables, want, want_tables, who)
        assert stats["rows_out"] == since, (who, stats["rows_out"], since)
        assert stats["n_keys"] == (len(live_keys(want)) if key else 0), (who, stats["n_keys"], len(live_keys(want)))
    if shape == "crowded":  # the stream did make rows defer
        assert deferred > 0


def _sortable(row):
    """A row as a sortable tuple: the GPU's row order inside a flush follows its atomics."""
    return tuple(sorted((k, str(v)) for k, v in row.items()))


def test_ttl_zero_with_the_clock_moved_is_a_run_without_a_clock():
    from tests import test_gpu_updating_changes as T
    st, aggs = ttl_stream(zlib.crc32(b"ttl0")), T.PLANS["P2"]
    results = []
    for move in (False, True):
        d = R.Driver(st, aggs, "host")
        outs = []
        for ev in st.events:
            if ev[0] == "clock":
                if move:
                    assert d.op._lib.arroyo_b200_op_set_clock(d.op._h, ev[1] * 10 ** 9) == 0
            elif ev[0] == "batch":
                d.batch(ev[1])
            else:
                g = d.flush("checkpoint")
                outs.append([] if g is None else rows_of(g))
        s = d.op.stats()
        d.op.close()
        table = [rows_of(b) for b in d.ctx.key_value_table("a").batches]
        results.append(([sorted(map(_sortable, o)) for o in outs], [sorted(map(_sortable, t)) for t in table],
                        {k: v for k, v in s.items() if not k.startswith("host_")}))
    assert results[0] == results[1]


def test_refused_clocks_change_nothing():
    from arroyo_b200 import ffi
    from arroyo_b200 import operators as native
    from tests import test_gpu_updating_changes as T
    st, aggs = ttl_stream(zlib.crc32(b"refused")), T.PLANS["P3"]
    want, _ = updating_ttl(reference_events(st.events), "k", aggs, STEP)
    d = Driver(st, aggs, "host", STEP)
    outs = []
    for ev in st.events:
        if ev[0] == "clock":
            d.clock(ev[1])
            assert d.op._lib.arroyo_b200_op_set_clock(d.op._h, ev[1]) == ffi.OK
            if ev[1] > 0:  # a clock that goes back: refused, the clock stays where it is
                assert d.op._lib.arroyo_b200_op_set_clock(d.op._h, ev[1] - 1) == ffi.INVALID_ARGUMENT
        elif ev[0] == "batch":
            d.batch(ev[1])
        else:
            g = d.flush("tick")
            outs.append([] if g is None else rows_of(g))
    d.op.close()
    for i, (g, w) in enumerate(zip(outs, want)):
        errs = flush_errors(g, w, "k", ordered=True)
        assert not errs, ("flush", i, errs[:8])
    # other kinds have no clock
    from arroyo_b200.config import WindowAggConfig
    w = native.TumblingAggregatingWindowFunc(WindowAggConfig(width=10, key_names=["k"], aggs=[O.Agg("count", None, "n")]),
                                             input_schema=st.schema())
    assert w._lib.arroyo_b200_op_set_clock(w._h, 5) == ffi.UNSUPPORTED
    w.close()
    # a negative ttl is refused at create
    with pytest.raises(ffi.ArroyoB200Error) as e:
        native.UpdatingAggregatingFunc(U.UpdatingAggConfig(["k"], aggs), input_schema=st.schema(), ttl=-1)
    assert e.value.status == ffi.INVALID_ARGUMENT


def _to_arrow_table(b, names, key_type):
    """An oracle table-"a" batch (tombstones: `_timestamp` None) as the Arrow batch the library reads."""
    arrays = []
    for n in names:
        v = b[n]
        if n == TS:
            arrays.append(pa.array([None if x is None else int(x) for x in v], type=pa.int64()).cast(pa.timestamp("ns")))
        elif key_type is not None and n == names[0]:
            k = np.array([int(x) % (1 << 64) for x in v], dtype=np.uint64)
            arrays.append(pa.array(k) if key_type == pa.uint64() else pa.array(k.view(np.int64)).cast(key_type))
        else:
            arrays.append(pa.array(np.asarray(v)))
    return pa.RecordBatch.from_arrays(arrays, names=names)


def _to_oracle(b):
    return O.Batch({c: np.array(col, dtype=object) for c, col in
                    ((n, [r[n] for r in rows_of(b)]) for n in b.schema.names)})


@pytest.mark.parametrize("reference", [False, True])
def test_table_interchange_with_the_ttl_oracle(reference):
    """oracle -> GPU at a cut (the oracle's table with tombstones, or like the reference's without), and GPU -> oracle;
    each continues to the exact reference of the restart."""
    from tests import test_gpu_updating_changes as T
    st, aggs = ttl_stream(zlib.crc32(f"interchange/{reference}".encode())), T.PLANS["P3"]
    n = sum(1 for ev in st.events if ev[0] == "flush")
    cut = (2 * n) // 3  # after the lone-eviction flush
    cfg = U.UpdatingAggConfig(["k"], aggs)
    names = S.state_names(cfg)
    want, _ = updating_ttl(reference_events(st.events, set(range(n)), {cut}), "k", aggs, STEP,
                           tombstones=not reference)
    # oracle -> GPU
    octx, oracle, d, got = _Ctx(), L.IncrementalAggregatingFunc(cfg, STEP, reference), None, []
    for ev in st.events:
        if ev[0] == "clock":
            (oracle.set_clock(ev[1]) if d is None else d.clock(ev[1]))
        elif ev[0] == "batch":
            (oracle.process_batch(O.Batch(ev[1])) if d is None else d.batch(ev[1]))
        elif d is None:
            b = oracle.handle_checkpoint(None, octx)
            got.append([] if b is None else b.rows())
            if len(got) - 1 == cut:
                d = Driver(st, aggs, "host", STEP, expected_keys=256)
                d.now = oracle.now
                for ob in octx.table.batches:
                    d.ctx.key_value_table("a").insert_batch(_to_arrow_table(ob, names, pa.int64()))
                d.op.on_start(d.ctx)
        else:
            g = d.flush("checkpoint")
            got.append([] if g is None else rows_of(g))
    d.op.close()
    for i, (g, w) in enumerate(zip(got, want)):
        if i <= cut and reference and not w[0] and not w[1]:
            assert g == []  # the reference drops a flush of evictions alone
            continue
        errs = flush_errors(g, w, "k", ordered=i > cut)
        assert not errs, ("oracle->gpu", reference, "flush", i, errs[:8])
    if reference:
        return
    # GPU -> oracle
    d, oracle, got = Driver(st, aggs, "device", STEP), None, []
    for ev in st.events:
        if ev[0] == "clock":
            (d.clock(ev[1]) if oracle is None else oracle.set_clock(ev[1]))
        elif ev[0] == "batch":
            (d.batch(ev[1]) if oracle is None else oracle.process_batch(O.Batch(ev[1])))
        elif oracle is None:
            g = d.flush("checkpoint")
            got.append([] if g is None else rows_of(g))
            if len(got) - 1 == cut:
                octx = _Ctx()
                for gb in d.ctx.key_value_table("a").batches:
                    assert gb.schema.names == names
                    octx.table.insert_batch(_to_oracle(gb))
                d.op.close()
                oracle = L.IncrementalAggregatingFunc(cfg, STEP)
                oracle.set_clock(d.now)
                oracle.on_start(octx)
        else:
            b = oracle.handle_checkpoint(None, octx)
            got.append([] if b is None else b.rows())
    for i, (g, w) in enumerate(zip(got, want)):
        errs = flush_errors(g, w, "k", ordered=i <= cut)
        assert not errs, ("gpu->oracle", "flush", i, errs[:8])


def _dev_cols(schema, cols):
    import torch
    ts = [torch.from_numpy(np.ascontiguousarray(cols[f.name]).view(np.int64)).cuda() for f in schema]
    torch.cuda.synchronize()
    return ts


def _group(keys, vals, ts):
    """numpy group-by: {key: (count, wrapped sum, min, max, max ts)}."""
    order = np.argsort(keys, kind="stable")
    k, v, t = keys[order], vals[order], ts[order]
    starts = np.flatnonzero(np.r_[True, k[1:] != k[:-1]])
    with np.errstate(over="ignore"):
        sums = np.add.reduceat(v, starts)
    return {int(kk): (int(c), int(s), int(mn), int(mx), int(tt)) for kk, c, s, mn, mx, tt in
            zip(k[starts], np.diff(np.r_[starts, len(k)]), sums, np.minimum.reduceat(v, starts),
                np.maximum.reduceat(v, starts), np.maximum.reduceat(t, starts))}


def test_2e24_rows_over_2e20_keys_half_expiring():
    import arroyo_b200 as ab
    from arroyo_b200 import operators as native
    aggs = [O.Agg("count", None, "n"), O.Agg("sum", "a", "s"), O.Agg("min", "a", "mn"), O.Agg("max", "a", "mx")]
    schema = pa.schema([("k", pa.int64()), ("a", pa.int64()), (TS, pa.timestamp("ns"))])
    rng = np.random.default_rng(24)
    n, nk, ttl = 1 << 24, 1 << 20, 10 ** 9
    now = [0]
    op = native.UpdatingAggregatingFunc(U.UpdatingAggConfig(["k"], aggs), input_schema=schema, ttl=ttl,
                                        clock=lambda: now[0])
    ctx = ab.OperatorContext(1)
    k1 = rng.integers(0, nk, n).astype(np.int64)
    c1 = {"k": k1, "a": rng.integers(-(1 << 62), 1 << 62, n), TS: rng.integers(0, 1 << 40, n)}
    keep = [_dev_cols(schema, c1)]
    op.process_device_batch([t.data_ptr() for t in keep[0]], n)
    col = ab.Collector()
    op.handle_tick(0, ctx, col)
    first = _group(c1["k"], c1["a"], c1[TS])
    assert sum(b.num_rows for b in col.batches) == len(first)
    # the even keys come back half a ttl later; a ttl after the first batch the odd keys expire
    now[0] = ttl // 2
    k2 = (rng.integers(0, nk // 2, n // 4) * 2).astype(np.int64)
    c2 = {"k": k2, "a": rng.integers(-(1 << 62), 1 << 62, n // 4), TS: rng.integers(0, 1 << 40, n // 4)}
    keep.append(_dev_cols(schema, c2))
    op.process_device_batch([t.data_ptr() for t in keep[1]], n // 4)
    now[0] = ttl
    col = ab.Collector()
    op.handle_tick(0, ctx, col)
    (b,) = col.batches
    allk = np.concatenate([k1, k2])
    both = _group(allk, np.concatenate([c1["a"], c2["a"]]), np.concatenate([c1[TS], c2[TS]]))
    r = b.column("_is_retract").to_numpy(zero_copy_only=False)
    k = b.column("k").to_numpy()
    cols = [b.column(c).to_numpy() for c in ("n", "s", "mn", "mx")] + [b.column(TS).cast(pa.int64()).to_numpy()]
    got_app = {int(k[i]): tuple(int(c[i]) for c in cols) for i in np.flatnonzero(~r)}
    touched = set(np.unique(k2).tolist())
    assert got_app == {kk: both[kk] for kk in touched}
    idle = set(first) - touched  # the odd keys, and the few even ones the second batch missed
    assert len(idle) >= len(first) // 2
    changed = touched & set(first)  # every key that came back changed its count
    ret = np.flatnonzero(r)
    changes, evictions = ret[:len(changed)], ret[len(changed):]
    assert {int(k[i]): tuple(int(c[i]) for c in cols) for i in changes} == {kk: first[kk] for kk in changed}
    assert {int(k[i]): tuple(int(c[i]) for c in cols) for i in evictions} == {kk: first[kk] for kk in idle}
    assert op.stats()["n_keys"] == len(touched)
    op.close()


def test_memory_follows_the_live_keys():
    import torch
    import arroyo_b200 as ab
    from arroyo_b200 import operators as native
    aggs = [O.Agg("count", None, "n"), O.Agg("sum", "a", "s")]
    schema = pa.schema([("k", pa.int64()), ("a", pa.int64()), (TS, pa.timestamp("ns"))])
    nk, ttl = 1 << 20, 1000
    now = [0]
    op = native.UpdatingAggregatingFunc(U.UpdatingAggConfig(["k"], aggs), input_schema=schema, ttl=ttl,
                                        clock=lambda: now[0])
    cols = [torch.empty(nk, dtype=torch.int64, device="cuda") for _ in range(3)]
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    levels = []
    for w in range(8):
        now[0] = w * 10 * ttl
        cols[0].copy_(torch.arange(w * nk, (w + 1) * nk, dtype=torch.int64))
        cols[1].fill_(w)
        cols[2].fill_(w)
        torch.cuda.synchronize()
        op.process_device_batch([c.data_ptr() for c in cols], nk)
        op.handle_tick(0, None, ab.Collector())
        if w == 0:
            footprint = free0 - torch.cuda.mem_get_info()[0]
        now[0] += ttl
        col = ab.Collector()
        op.handle_checkpoint(None, ab.OperatorContext(1), col)  # the evictions, then their tombstones leave
        assert sum(b.num_rows for b in col.batches) == nk
        assert op.stats()["n_keys"] == 0, w
        torch.cuda.synchronize()
        levels.append(torch.cuda.mem_get_info()[0])
    op.close()
    assert footprint > 0
    assert levels[7] >= levels[0] - footprint, (levels, footprint)
