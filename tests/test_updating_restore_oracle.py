"""The updating oracle's state table "a" and its restore (tests/updating_state_oracle.py: checkpoint_state, on_start)
against tests/exact_state_reference.py and tests/exact_reference.py, on CPU-sized streams of
tests/test_gpu_updating_changes.py.

* After every checkpoint, the latest row per key of table "a" (largest _generation, the later row on a tie) is the
  exact state of every key with rows: `exact_state_reference.updating_state`.
* An oracle checkpointed at a flush, dropped, and restored from table "a" into a fresh oracle continues with the change
  stream of the uninterrupted run (`exact_reference.updating_changes`), flush by flush: the retractions carry the
  restored values.  The table's batches are handed over shuffled, and streams restart twice, so only the generation
  rule can pick the latest row of a key.

The helpers here (`latest_rows`, `state_errors`, `change_errors`) are shared with tests/test_gpu_updating_restore.py."""
import zlib

import numpy as np
import pytest

from oracle import arroyo_oracle as O
from oracle import updating_oracle as U
from tests import exact_reference as X
from tests import updating_state_oracle as S
from tests.exact_state_reference import updating_state

A = O.Agg
GEN = S.GENERATION


def latest_rows(batches, key_name):
    """{key or None: row} of table "a": per key the row with the largest _generation, on a tie the later one (batch
    order, then row order)."""
    best = {}
    for b in batches:
        for r in b:
            k = int(r[key_name]) if key_name else None
            if k not in best or int(r[GEN]) >= int(best[k][GEN]):
                best[k] = r
    return best


def state_errors(got: dict, want: dict, key_name, aggs):
    """Differences between the latest table rows and the exact per-key state (empty: equal).  AVG sums are exact
    while a key's sum of |x| is below 2^53, else within n * 2u * sum|x| of the exact sum."""
    errs = []
    if set(got) != set(want):
        errs.append(f"keys: missing {sorted(set(want) - set(got))[:5]}, unexpected {sorted(set(got) - set(want))[:5]}")
    for k in set(got) & set(want):
        g, w = got[k], want[k]
        checks = [(X.TIMESTAMP, int(g[X.TIMESTAMP]), w[X.TIMESTAMP])]
        if key_name:
            checks.append((key_name, int(g[key_name]), k))
        for a in aggs:
            if a.kind in ("count", "sum", "avg"):
                checks.append((f"{a.name}[count]", int(g[f"{a.name}[count]"]), w["rows"]))
            if a.kind in ("sum", "min", "max"):
                f = f"{a.name}[{a.kind}]"
                checks.append((f, int(g[f]), w[a.name]))
            if a.kind == "avg":
                exact, abs_sum = w[a.name]
                s = float(g[f"{a.name}[sum]"])
                ok = s == float(exact) if abs_sum < 2 ** 53 else abs(s - exact) <= w["rows"] * 2 * X.U * abs_sum
                if not ok:
                    errs.append(f"key {k}: {a.name}[sum] = {s!r}, exact {exact} (sum|x| {abs_sum})")
        errs += [f"key {k}: {c} = {gv}, want {wv}" for c, gv, wv in checks if gv != wv]
    return errs


def change_errors(got_rows, want, key_name):
    """One flush's rows (dicts with an `_is_retract` flag) against updating_changes' (retractions, appends)."""
    wr, wa = want
    errs = []
    for part, w in (([r for r in got_rows if r[U.IS_RETRACT]], wr), ([r for r in got_rows if not r[U.IS_RETRACT]], wa)):
        errs += X.mismatches(w, part, lambda r: int(r[key_name]) if key_name else None)
    return errs


class _Ctx:
    """A context with nothing but table "a"."""

    def __init__(self):
        self.table = S.KeyValueTable()

    def key_value_table(self, name):
        assert name == "a"
        return self.table


def run_oracle(st, aggs, restarts=(), checkpoints=None, seed=0):
    """Runs the oracle over a stream of test_gpu_updating_changes.  Flushes whose index is in `checkpoints` (default:
    every flush) are checkpoints; after a flush whose index is in `restarts` the oracle is dropped and a fresh one is
    restored from table "a", its batches shuffled.  Returns (rows per flush, table "a" rows after each flush)."""
    rng = np.random.default_rng(seed)
    cfg = U.UpdatingAggConfig([st.key_name()] if st.key_type else [], aggs)
    ctx, op = _Ctx(), S.IncrementalAggregatingFunc(cfg)
    outs, tables = [], []
    for ev in st.events:
        if ev[0] == "batch":
            op.process_batch(O.Batch(ev[1]))
            continue
        i = len(outs)
        if checkpoints is None or i in checkpoints or i in restarts:
            b = op.handle_checkpoint(None, ctx)
        else:
            b = op.handle_tick()
        outs.append([] if b is None else b.rows())
        tables.append([b.rows() for b in ctx.table.batches])
        if i in restarts:
            order = rng.permutation(len(ctx.table.batches))
            ctx.table.batches = [ctx.table.batches[j] for j in order]
            op = S.IncrementalAggregatingFunc(cfg)
            op.on_start(ctx)
    return outs, tables


def _shapes():
    from tests import test_gpu_updating_changes as T
    return {
        "random": ("P2", lambda: T.s_random(1)), "random_u64": ("P7", lambda: T.s_random(2, "u64", every=3)),
        "random_ts": ("P8", lambda: T.s_random(3, "ts", every=1)), "quiet_AMM": ("AMM", lambda: T.s_quiet(6, "AMM")),
        "quiet_MM": ("MM", lambda: T.s_quiet(5, "MM")), "edge_keys": ("P5", lambda: T.s_edge_keys(13)),
        "unkeyed": ("P2", lambda: T.s_unkeyed(15)), "growth": ("P1", lambda: T.s_growth(16, 3000)),
        "edge_values": ("P3", lambda: T.s_edge_values(17)), "min_only": ("P6a", lambda: T.s_random(4, every=1)),
        "crowded_spread": ("P6b", lambda: T.s_crowded(18, 1400, True)),
    }


SHAPES = _shapes()


@pytest.mark.parametrize("shape", sorted(SHAPES))
def test_table_a_holds_the_exact_state(shape):
    from tests import test_gpu_updating_changes as T
    plan, make = SHAPES[shape]
    st, aggs = make(), T.PLANS[plan]
    key = st.key_name()
    n_flush = sum(1 for ev in st.events if ev[0] == "flush")
    # checkpoints at every other flush: a checkpoint also writes the keys the ticks before it flushed
    cps = set(range(1, n_flush, 2)) | {n_flush - 1}
    _, tables = run_oracle(st, aggs, checkpoints=cps)
    want = updating_state(st.events, key, aggs)
    for i in sorted(cps):
        errs = state_errors(latest_rows(tables[i], key), want[i], key, aggs)
        assert not errs, (shape, "flush", i, errs[:8])


def _restart_cases():
    cases = []
    for shape in sorted(SHAPES):
        cases += [(shape, "each"), (shape, "twice")]
    return cases


@pytest.mark.parametrize("shape,how", _restart_cases())
def test_restored_oracle_continues_the_uninterrupted_stream(shape, how):
    """"each": a restart after every flush in turn (one per run); "twice": two restarts in one run, with shuffled
    batches and checkpoints only at the restarts, so a key's rows of different generations sit in shuffled batches."""
    from tests import test_gpu_updating_changes as T
    plan, make = SHAPES[shape]
    st, aggs = make(), T.PLANS[plan]
    key = st.key_name()
    want = X.updating_changes(st.events, key, aggs)
    n = len(want)
    seed = zlib.crc32(f"{shape}/{how}".encode())
    runs = [({i}, None) for i in range(n - 1)] if how == "each" else [({n // 3, (2 * n) // 3}, set())]
    for restarts, cps in runs:
        got, _ = run_oracle(st, aggs, restarts=restarts, checkpoints=cps, seed=seed)
        assert len(got) == n
        for i, (g, w) in enumerate(zip(got, want)):
            errs = change_errors(g, w, key)
            assert not errs, (shape, sorted(restarts), "flush", i, errs[:8])


def test_restore_picks_the_largest_generation_then_the_later_row():
    aggs = [A("sum", "a", "s"), A("max", "a", "mx")]
    cfg = U.UpdatingAggConfig(["k"], aggs)
    names = S.state_names(cfg)
    assert names == ["k", "s[sum]", "s[count]", "mx[max]", X.TIMESTAMP, GEN]

    def batch(rows):
        return O.Batch({n: np.array([r[i] for r in rows], dtype=object) for i, n in enumerate(names)})

    ctx = _Ctx()
    # key 1: generation 5 wins over a later generation 3; key 2: a tie on 4 goes to the later row
    ctx.table.insert_batch(batch([(1, 10, 2, 7, 100, 5), (2, 1, 1, 1, 100, 4)]))
    ctx.table.insert_batch(batch([(1, 99, 9, 99, 999, 3), (2, 20, 3, 9, 200, 4)]))
    op = S.IncrementalAggregatingFunc(cfg)
    op.on_start(ctx)
    assert op.generation == 6
    op.process_batch(O.Batch({"k": np.array([1, 2]), "a": np.array([1, 1]), X.TIMESTAMP: np.array([50, 50])}))
    rows = op.flush().rows()
    got = {(r["k"], r[U.IS_RETRACT]): (r["s"], r["mx"], r[X.TIMESTAMP]) for r in rows}
    assert got == {(1, True): (10, 7, 100), (1, False): (11, 7, 100), (2, True): (20, 9, 200), (2, False): (21, 9, 200)}
    b = op.checkpoint_state()
    assert set(b[GEN].tolist()) == {6} and sorted(b["s[count]"].tolist()) == [3, 4]
