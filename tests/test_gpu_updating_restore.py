"""The CUDA updating aggregate (csrc/updating_agg.cu) across a checkpoint and a restart: table "a" written by
arroyo_b200_op_checkpoint_state and read back by on_start.

* Restart at a flush: the operator is checkpointed, destroyed, and a new one with expected_keys = 256 is restored from
  table "a" and continues.  Every flush, before and after the restart, equals exact_reference.updating_changes of the
  uninterrupted stream, and the merged change stream equals exact_reference.updating_rows.
* Two restarts with the table's batches shuffled, so that only the generation rule can pick a key's latest row.
* Table contents: after every checkpoint, the latest row per key equals exact_state_reference.updating_state.
* Interchange: the oracle's table restores the GPU operator and the GPU's table restores the oracle; each continues
  to the uninterrupted result.
* The reference's goldens `grouped_aggregates` / `aggregates` across a restart at several cut points.
* Refusals (a state layout that is not the plan's, restore after rows): INVALID_ARGUMENT, and nothing changes.
* Stats: restored rows are not in `rows_in`, their keys are in `n_keys`, state rows are not in `rows_out`."""
import ctypes as C
import zlib

import numpy as np
import pyarrow as pa
import pytest

from oracle import arroyo_oracle as O
from oracle import updating_oracle as U
from tests import exact_reference as X
from tests import updating_state_oracle as S
from tests.exact_state_reference import updating_state
from tests import test_gpu_updating_changes as T
from tests.test_updating_restore_oracle import _Ctx, change_errors, latest_rows, state_errors

pytestmark = pytest.mark.gpu
TS = O.TIMESTAMP


def _host(arr):
    if pa.types.is_timestamp(arr.type):
        arr = arr.cast(pa.int64())
    return arr.to_numpy(zero_copy_only=False)


def arrow_rows(b):
    cols = {c: _host(b.column(c)).tolist() for c in b.schema.names}
    return [dict(zip(cols, t)) for t in zip(*cols.values())]


def state_to_arrow(b, names, key_type):
    """An oracle table-"a" batch (typed numpy columns, keys as Python ints) as the Arrow batch the library reads."""
    arrays = []
    for n in names:
        v = b[n]
        if n == TS:
            arrays.append(pa.array(np.asarray(v, dtype=np.int64)).cast(pa.timestamp("ns")))
        elif key_type is not None and n == names[0]:
            k = np.array([int(x) % (1 << 64) for x in v], dtype=np.uint64)
            arrays.append(pa.array(k) if key_type == pa.uint64() else pa.array(k.view(np.int64)).cast(key_type))
        else:
            arrays.append(pa.array(v))  # int64, uint64 or float64, as the oracle typed them
    return pa.RecordBatch.from_arrays(arrays, names=names)


def state_to_oracle(b):
    return O.Batch({c: _host(b.column(c)) for c in b.schema.names})


class Driver:
    """Feeds a stream of test_gpu_updating_changes to the GPU operator through `entry` (host, sliced, device,
    device_run, mixed); restarts after the flushes in `restarts`."""

    def __init__(self, st, aggs, entry, expected_keys=None):
        import arroyo_b200 as ab
        from arroyo_b200 import operators as native
        self.ab, self.native = ab, native
        self.st, self.aggs, self.entry = st, aggs, entry
        self.schema = st.schema()
        self.cfg = U.UpdatingAggConfig([st.key_name()] if st.key_type else [], aggs)
        self.ctx = ab.OperatorContext(1)
        self.op = self.make(st.expected_keys if expected_keys is None else expected_keys)
        self.pending, self.keep, self.n_batch = [], [], 0

    def make(self, expected_keys):
        return self.native.UpdatingAggregatingFunc(self.cfg, input_schema=self.schema, expected_keys=expected_keys)

    def _dev(self, cols):
        import torch
        ts = [torch.from_numpy(np.ascontiguousarray(cols[f.name]).view(np.int64)).cuda() for f in self.schema]
        torch.cuda.synchronize()
        self.keep.append(ts)
        return [t.data_ptr() for t in ts]

    def batch(self, cols):
        if self.entry in ("sliced", "device_run"):
            self.pending.append(cols)
        elif self.entry == "device" or (self.entry == "mixed" and self.n_batch % 2 == 1):
            self.op.process_device_batch(self._dev(cols), len(cols[TS]))
        else:
            self.op.process_batch(T.to_arrow(cols, self.schema), self.ctx, None)
        self.n_batch += 1

    def send_pending(self):
        if not self.pending:
            return
        if self.entry == "sliced":
            allc = {c: np.concatenate([p[c] for p in self.pending]) for c in self.schema.names}
            big, s, i = T.to_arrow(allc, self.schema), 0, 0
            while s < big.num_rows:
                z = min(T.SIZES[i % len(T.SIZES)], big.num_rows - s)
                self.op.process_batch(big.slice(s, z), self.ctx, None)
                s, i = s + z, i + 1
        else:
            ptrs = [p for cols in self.pending for p in self._dev(cols)]
            rows = [len(cols[TS]) for cols in self.pending]
            self.op.process_device_batches((C.c_uint64 * len(ptrs))(*ptrs), (C.c_int64 * len(rows))(*rows),
                                           len(self.schema))
        self.pending.clear()

    def flush(self, how):
        """how: tick, checkpoint or close; returns the flush's rows."""
        self.send_pending()
        col = self.ab.Collector()
        if how == "close":
            self.op.on_close("end_of_data", self.ctx, col)
        elif how == "tick":
            self.op.handle_tick(0, self.ctx, col)
        else:
            self.op.handle_checkpoint(None, self.ctx, col)
        self.keep.clear()
        assert len(col.batches) <= 1
        return col.batches[0] if col.batches else None

    def restart(self, rng=None, expected_keys=256):
        self.op.close()
        table = self.ctx.key_value_table("a")
        if rng is not None:
            table.batches = [table.batches[j] for j in rng.permutation(len(table.batches))]
        self.op = self.make(expected_keys)
        self.op.on_start(self.ctx)


def run(st, aggs, entry, restarts=(), checkpoints=None, seed=0):
    """Returns (batch or None per flush, table "a" batches after each flush, stats at the end, rows / keys fed since
    the last restart).  Flushes in `checkpoints` (default: every other one) and in `restarts` are checkpoints, the last
    flush is on_close(end_of_data), the others are ticks."""
    rng = np.random.default_rng(seed)
    d = Driver(st, aggs, entry)
    n_flush = sum(1 for ev in st.events if ev[0] == "flush")
    outs, tables, rows_since = [], [], 0
    for ev in st.events:
        if ev[0] == "batch":
            d.batch(ev[1])
            rows_since += len(ev[1][TS])
            continue
        i = len(outs)
        cp = i in restarts or (i % 2 == 1 if checkpoints is None else i in checkpoints)
        how = "close" if i == n_flush - 1 and i not in restarts else "checkpoint" if cp else "tick"
        outs.append(d.flush(how))
        tables.append([arrow_rows(b) for b in d.ctx.key_value_table("a").batches] if how == "checkpoint" else None)
        if i in restarts:
            d.restart(rng)
            rows_since = 0
    stats = d.op.stats()
    d.op.close()
    return outs, tables, stats, rows_since


def check_changes(st, aggs, outs, want, who):
    key = st.key_name()
    key_type = st.schema().field(key).type if key else None
    assert len(outs) == len(want), (who, len(outs), len(want))
    merged, n_out = [], []
    for i, (g, w) in enumerate(zip(outs, want)):
        if g is None:
            assert not w[0] and not w[1], (who, "flush", i, "emitted nothing")
            n_out.append(0)
            continue
        if key:
            assert g.schema.field(key).type == key_type, (who, g.schema)
        r = _host(g.column("_is_retract")).astype(bool)
        nr = int(r.sum())
        assert r[:nr].all() and not r[nr:].any(), (who, "flush", i, "a retraction after an append")
        rows = arrow_rows(g)
        errs = change_errors(rows, w, key)
        assert not errs, (who, "flush", i, errs[:8])
        n_out.append(len(rows))
        cols = {c: _host(g.column(c)) for c in g.schema.names if c != "_is_retract"}
        merged.append(O.Batch({**cols, U.IS_RETRACT: r}))
    batches = [O.Batch(ev[1]) for ev in st.events if ev[0] == "batch" and len(ev[1][TS])]
    exact = X.updating_rows(batches, key, aggs)
    final = U.merge_change_stream(merged, [key] if key else [])
    errs = X.mismatches({k: {c: v for c, v in r.items() if c != TS} for k, r in exact.items()}, final,
                        lambda row: int(row[key]) if key else None)
    assert not errs, (who, "merged", errs[:8])
    return n_out


def _keys_with_rows(st):
    return len({int(k) for ev in st.events if ev[0] == "batch" for k in ev[1].get("k", [])}) if st.key_type else 0


# (shape, plan, entry): the shapes of test_gpu_updating_changes across the entry points
CASES = [
    ("random", "P2", "host"), ("random", "P3", "sliced"), ("random", "P7", "device"), ("random", "AMM", "mixed"),
    ("random", "P6a", "device_run"), ("random_u64", "P2", "host"), ("random_u64", "P8", "device"),
    ("random_ts", "P3", "sliced"), ("random_ts", "P1", "device"),
    ("edge_keys", "P2", "host"), ("edge_keys", "COUNT", "device"), ("edge_keys", "P6b", "sliced"),
    ("edge_keys_u64", "P5", "host"), ("edge_values", "P3", "host"), ("edge_values", "P7", "device"),
    ("unkeyed", "P2", "host"), ("unkeyed", "AMM", "sliced"), ("unkeyed", "MM", "device"),
    ("growth_1e5", "P2", "host"), ("growth_1e5", "P4", "device"), ("growth_1e6", "COUNT", "device_run"),
    ("crowded_1300", "P2", "host"), ("crowded_1300", "P6a", "device"), ("hot", "P2", "host"), ("hot", "P4", "device"),
    ("quiet_MM", "MM", "host"), ("quiet_AMM", "AMM", "device"),
]


@pytest.mark.parametrize("shape,plan,entry", CASES, ids=["-".join(c) for c in CASES])
def test_restart_at_a_flush(shape, plan, entry):
    seed = zlib.crc32(f"{shape}/{plan}/{entry}".encode())
    st, aggs = T.SHAPES[shape](seed), T.PLANS[plan]
    want = X.updating_changes(st.events, st.key_name(), aggs)
    n = len(want)
    cut = max(0, n // 2 - 1)
    outs, tables, stats, rows_since = run(st, aggs, entry, restarts={cut}, seed=seed)
    who = f"{shape}/{plan}/{entry}"
    n_out = check_changes(st, aggs, outs, want, who)
    # table contents at every checkpoint
    exact = updating_state(st.events, st.key_name(), aggs)
    for i, t in enumerate(tables):
        if t is not None:
            errs = state_errors(latest_rows(t, st.key_name()), exact[i], st.key_name(), aggs)
            assert not errs, (who, "table after flush", i, errs[:8])
    # stats of the restored operator: rows since the restart, every key, rows emitted since the restart
    assert stats["rows_in"] == rows_since, (who, stats["rows_in"], rows_since)
    assert stats["n_keys"] == _keys_with_rows(st), (who, stats["n_keys"], _keys_with_rows(st))
    assert stats["rows_out"] == sum(n_out[cut + 1:]), (who, stats["rows_out"], sum(n_out[cut + 1:]))


TWICE = [("random", "P2", "host"), ("random", "P7", "device"), ("edge_keys", "P3", "sliced"), ("unkeyed", "P8", "host"),
         ("growth_1e5", "P1", "device_run"), ("crowded_1300", "COUNT", "host"), ("quiet_AMM", "AMM", "mixed")]


@pytest.mark.parametrize("shape,plan,entry", TWICE, ids=["-".join(c) for c in TWICE])
def test_two_restarts_with_shuffled_batches(shape, plan, entry):
    """Checkpoints only at the two restarts: a key touched before both has rows of two generations in table "a", and
    the batches arrive shuffled."""
    seed = zlib.crc32(f"twice/{shape}/{plan}/{entry}".encode())
    st, aggs = T.SHAPES[shape](seed), T.PLANS[plan]
    want = X.updating_changes(st.events, st.key_name(), aggs)
    n = len(want)
    r = {max(0, n // 3 - 1), max(1, (2 * n) // 3 - 1)}
    outs, tables, stats, _ = run(st, aggs, entry, restarts=r, checkpoints=set(), seed=seed)
    check_changes(st, aggs, outs, want, f"twice/{shape}/{plan}/{entry}")
    exact = updating_state(st.events, st.key_name(), aggs)
    last = max(r)
    errs = state_errors(latest_rows(tables[last], st.key_name()), exact[last], st.key_name(), aggs)
    assert not errs, errs[:8]
    assert stats["n_keys"] == _keys_with_rows(st)


INTERCHANGE = [("random", "P3"), ("random_u64", "P7"), ("edge_keys", "P2"), ("unkeyed", "AMM"), ("edge_values", "P5"),
               ("quiet_MM", "MM")]


@pytest.mark.parametrize("shape,plan", INTERCHANGE, ids=["-".join(c) for c in INTERCHANGE])
def test_interchange_with_the_oracle(shape, plan):
    """The oracle's checkpoint restores the GPU operator, and the GPU's checkpoint restores the oracle; both continue
    to the uninterrupted change stream."""
    seed = zlib.crc32(f"interchange/{shape}/{plan}".encode())
    st, aggs = T.SHAPES[shape](seed), T.PLANS[plan]
    key = st.key_name()
    key_type = st.schema().field(key).type if key else None
    want = X.updating_changes(st.events, key, aggs)
    cut = max(0, len(want) // 2 - 1)
    cfg = U.UpdatingAggConfig([key] if key else [], aggs)
    names = S.state_names(cfg)
    # oracle -> GPU
    octx, oracle, d = _Ctx(), S.IncrementalAggregatingFunc(cfg), None
    got, i = [], 0
    for ev in st.events:
        if ev[0] == "batch":
            (oracle.process_batch(O.Batch(ev[1])) if d is None else d.batch(ev[1]))
            continue
        if d is None:
            b = oracle.handle_checkpoint(None, octx) if i == cut else oracle.flush()
            got.append([] if b is None else b.rows())
            if i == cut:
                d = Driver(st, aggs, "host", expected_keys=256)
                for ob in octx.table.batches:
                    d.ctx.key_value_table("a").insert_batch(state_to_arrow(ob, names, key_type))
                d.op.on_start(d.ctx)
        else:
            g = d.flush("tick")
            got.append([] if g is None else arrow_rows(g))
        i += 1
    d.op.close()
    for j, (g, w) in enumerate(zip(got, want)):
        errs = change_errors(g, w, key)
        assert not errs, ("oracle->gpu", "flush", j, errs[:8])
    # GPU -> oracle
    d, oracle, got, i = Driver(st, aggs, "device"), None, [], 0
    for ev in st.events:
        if ev[0] == "batch":
            (d.batch(ev[1]) if oracle is None else oracle.process_batch(O.Batch(ev[1])))
            continue
        if oracle is None:
            g = d.flush("checkpoint" if i == cut else "tick")
            got.append([] if g is None else arrow_rows(g))
            if i == cut:
                octx = _Ctx()
                for gb in d.ctx.key_value_table("a").batches:
                    assert gb.schema.names == names
                    octx.table.insert_batch(state_to_oracle(gb))
                d.op.close()
                oracle = S.IncrementalAggregatingFunc(cfg)
                oracle.on_start(octx)
        else:
            b = oracle.flush()
            got.append([] if b is None else b.rows())
        i += 1
    for j, (g, w) in enumerate(zip(got, want)):
        errs = change_errors(g, w, key)
        assert not errs, ("gpu->oracle", "flush", j, errs[:8])


GOLDEN_AGGS = [O.Agg("min", "counter", "min"), O.Agg("max", "counter", "max"), O.Agg("sum", "counter", "sum"),
               O.Agg("count", None, "count"), O.Agg("avg", "counter", "avg")]


@pytest.mark.parametrize("keyed", [True, False])
def test_goldens_across_a_restart(golden, accumulator_golden, keyed):
    import arroyo_b200 as ab
    from arroyo_b200 import operators as native
    from tests.gpu_ops import to_arrow
    counter, ts = golden[0]["impulse_counter"], golden[0]["impulse_ts"]
    keys = ["counter_mod"] if keyed else []
    cols = {"counter": counter, TS: ts}
    if keyed:
        cols = {"counter_mod": counter % 5, **cols}
    batches = O.source_batches(cols, 32)
    cfg = U.UpdatingAggConfig(keys, GOLDEN_AGGS)
    n_flush = len(batches) // 3 + 1
    for cut in sorted({0, 1, n_flush // 2, n_flush - 2}):
        ctx = ab.OperatorContext(1)
        schema = to_arrow(batches[0]).schema
        op = native.UpdatingAggregatingFunc(cfg, input_schema=schema)
        got, f = [], 0
        for i, b in enumerate(batches):
            op.process_batch(to_arrow(b), ctx, None)
            if (i + 1) % 3 == 0 or i == len(batches) - 1:
                col = ab.Collector()
                if f == cut:
                    op.handle_checkpoint(None, ctx, col)
                    op.close()
                    op = native.UpdatingAggregatingFunc(cfg, input_schema=schema, expected_keys=256)
                    op.on_start(ctx)
                else:
                    op.handle_tick(0, ctx, col)
                for gb in col.batches:
                    c = {n: _host(gb.column(n)) for n in gb.schema.names}
                    c[U.IS_RETRACT] = c.pop("_is_retract").astype(bool)
                    got.append(O.Batch(c))
                f += 1
        op.close()
        assert U.merge_change_stream(got, keys) == accumulator_golden["grouped_aggregates" if keyed else "aggregates"], cut


def test_refusals_change_nothing():
    from arroyo_b200 import ffi
    st = T.s_random(5, every=1, n_batches=6)
    aggs = T.PLANS["P2"]
    want = X.updating_changes(st.events, "k", aggs)
    batches = [ev[1] for ev in st.events if ev[0] == "batch"]
    # a table "a" written by a checkpoint after the first flush
    d = Driver(st, aggs, "host")
    d.batch(batches[0])
    d.flush("checkpoint")
    table = list(d.ctx.key_value_table("a").batches)
    d.op.close()
    good = table[0]
    bad_tables = {
        "column missing": good.drop_columns([good.schema.names[1]]),
        "generation as Int64": good.set_column(len(good.schema) - 1, S.GENERATION,
                                               good.column(S.GENERATION).cast(pa.int64())),
        "AVG sum as Int64": good.set_column(2, good.schema.names[2], pa.array(np.zeros(good.num_rows, np.int64))),
        "key as Float64": good.set_column(0, "k", pa.array(np.zeros(good.num_rows))),
    }
    for what, bad in bad_tables.items():
        d = Driver(st, aggs, "host")
        d.ctx.key_value_table("a").insert_batch(good)
        d.ctx.key_value_table("a").insert_batch(bad)
        with pytest.raises(ffi.ArroyoB200Error) as e:
            d.op.on_start(d.ctx)
        assert e.value.status == ffi.INVALID_ARGUMENT, (what, e.value)
        s = d.op.stats()
        assert s["n_keys"] == 0 and s["rows_in"] == 0, (what, s)
        # the operator is still the fresh one: the stream runs as if no restore had been tried
        outs, i = [], 0
        for ev in st.events:
            if ev[0] == "batch":
                d.batch(ev[1])
            else:
                outs.append(d.flush("tick"))
        d.op.close()
        check_changes(st, aggs, outs, want, what)
    # restore after rows: refused, the rows and the change stream are untouched
    d = Driver(st, aggs, "host")
    d.ctx.key_value_table("a").insert_batch(good)
    outs = []
    for ev in st.events:
        if ev[0] == "batch":
            d.batch(ev[1])
            if len(outs) == 1:
                with pytest.raises(ffi.ArroyoB200Error) as e:
                    d.op.on_start(d.ctx)
                assert e.value.status == ffi.INVALID_ARGUMENT
        else:
            outs.append(d.flush("tick"))
    s = d.op.stats()
    d.op.close()
    check_changes(st, aggs, outs, want, "after rows")
    assert s["rows_in"] == sum(len(b[TS]) for b in batches)


def test_state_rows_leave_the_change_statistics_alone():
    """checkpoint_state twice in a row: the second call has nothing to write; rows_out / windows_out count change rows
    only; a plan with nothing flushed writes nothing."""
    import arroyo_b200 as ab
    st = T.s_random(9, every=0, n_batches=2)
    aggs = T.PLANS["P8"]
    d = Driver(st, aggs, "host")
    table = ab.context.KeyValueTable()
    d.op.checkpoint_state(table)
    assert table.batches == []
    d.batch(st.events[0][1])
    out = d.flush("tick")
    s0 = d.op.stats()
    d.op.checkpoint_state(table)
    d.op.checkpoint_state(table)
    assert len(table.batches) == 1 and table.batches[0].num_rows == out.num_rows
    assert set(table.batches[0].column(S.GENERATION).to_pylist()) == {0}
    s1 = d.op.stats()
    for f in ("rows_in", "rows_out", "windows_out", "n_keys"):
        assert s0[f] == s1[f], f
    d.op.close()
