"""The ttl oracle (tests/updating_ttl_oracle.py) against the exact ttl reference (tests/exact_ttl_reference.py) on
random streams with clock steps: ttl shorter than the flush gap, equal to it (the >= boundary) and longer than the
stream; keys that go idle and come back; flushes whose only rows are evictions; restarts at every flush, after
evictions too; tables written with tombstones and, like the reference's own, without.

The helpers here (`ttl_stream`, `reference_events`, `flush_errors`, `table_errors`) are shared with
tests/test_gpu_updating_ttl.py."""
import zlib

import numpy as np
import pytest

from oracle import arroyo_oracle as O
from oracle import updating_oracle as U
from tests import exact_reference as X
from tests import updating_ttl_oracle as L
from tests.exact_ttl_reference import updating_ttl
from tests.test_updating_restore_oracle import _Ctx, latest_rows, state_errors

STEP = 1000  # clock steps are multiples of STEP


def ttl_stream(seed, key_type="i64", n_batches=18, n_keys=90, every=2, keys_fn=None, expected_keys=0):
    """A test_gpu_updating_changes.Stream with ("clock", t) events: before every batch and every flush the clock
    moves by 0, 1 or 2 STEPs.  Each batch draws from a window of a third of the keys that wanders, so keys go idle and
    come back.  Two thirds in, the clock jumps 5 STEPs to a flush with no batch since the last one (its only rows can
    be evictions).  `keys_fn(rng, n)`: the keys of a batch instead."""
    from tests import test_gpu_updating_changes as T
    st = T.Stream(seed, key_type, expected_keys)
    rng, clock = st.rng, 0

    def tick(k):
        nonlocal clock
        clock += k * STEP
        st.events.append(("clock", clock))

    for i in range(n_batches):
        tick(int(rng.integers(0, 3)))
        n = int(rng.integers(1, 300))
        if keys_fn is not None:
            keys = keys_fn(rng, n)
        else:
            lo = (i * n_keys) // n_batches
            keys = ((lo + rng.integers(0, n_keys // 3, n)) % n_keys) * 7919 - 500
        st.batch(keys=keys if key_type else None, n=n)
        if (i + 1) % every == 0:
            tick(int(rng.integers(0, 3)))
            st.flush()
        if i == (2 * n_batches) // 3:
            st.flush()
            tick(5)
            st.flush()
    tick(1)
    st.flush()
    return st


def reference_events(events, checkpoints=(), restarts=()):
    """The stream's events for exact_ttl_reference: flush i is a checkpoint when i is in `checkpoints` or `restarts`,
    and a restart follows each flush in `restarts`."""
    out, i = [], 0
    for ev in events:
        if ev[0] != "flush":
            out.append(ev)
            continue
        out.append(("checkpoint",) if i in checkpoints or i in restarts else ("flush",))
        if i in restarts:
            out.append(("restart",))
        i += 1
    return out


def flush_errors(got_rows, want, key_name, ordered=False):
    """One flush's rows, in output order (dicts with `_is_retract`), against (retractions, appends, evictions): the
    change rows come first, then the eviction retractions.  `ordered`: the change rows are all retractions, then all
    appends (the CUDA operator; the oracle keeps a key's retraction next to its append)."""
    wr, wa, we = want
    key_of = (lambda r: int(r[key_name])) if key_name else (lambda r: None)
    head, tail = got_rows[:len(wr) + len(wa)], got_rows[len(wr) + len(wa):]
    errs = []
    if ordered and any(not r[U.IS_RETRACT] for r in head[:len(wr)]):
        errs.append("an append before a retraction")
    for name, part, w in (("retractions", [r for r in head if r[U.IS_RETRACT]], wr),
                          ("appends", [r for r in head if not r[U.IS_RETRACT]], wa), ("evictions", tail, we)):
        if name == "evictions" and any(not r[U.IS_RETRACT] for r in part):
            errs.append("evictions: an append among them")
        errs += [f"{name}: {e}" for e in X.mismatches(w, part, key_of)]
    return errs


def table_errors(batches_rows, want, key_name, aggs):
    """Table "a" (lists of row dicts) against exact_ttl_reference's table: the latest row per key, a null
    `_timestamp` for a tombstone."""
    got = latest_rows(batches_rows, key_name)
    dead = {k for k, r in got.items() if r[X.TIMESTAMP] is None}
    want_dead = {k for k, r in want.items() if r is None}
    errs = [] if dead == want_dead else [f"tombstones: {sorted(dead ^ want_dead, key=str)[:8]}"]
    live = {k: r for k, r in got.items() if k not in dead}
    return errs + state_errors(live, {k: r for k, r in want.items() if r is not None}, key_name, aggs)


def run_oracle(st, aggs, ttl, checkpoints=(), restarts=(), reference=False):
    """(rows per flush, table "a" rows after each checkpoint) of the ttl oracle over a ttl_stream."""
    cfg = U.UpdatingAggConfig([st.key_name()] if st.key_type else [], aggs)
    ctx, op = _Ctx(), L.IncrementalAggregatingFunc(cfg, ttl, reference)
    outs, tables = [], []
    for ev in st.events:
        if ev[0] == "clock":
            op.set_clock(ev[1])
        elif ev[0] == "batch":
            op.process_batch(O.Batch(ev[1]))
        else:
            i = len(outs)
            cp = i in checkpoints or i in restarts
            b = op.handle_checkpoint(None, ctx) if cp else op.handle_tick()
            outs.append([] if b is None else b.rows())
            if cp:
                tables.append([b.rows() for b in ctx.table.batches])
            if i in restarts:
                now = op.now
                op = L.IncrementalAggregatingFunc(cfg, ttl, reference)
                op.set_clock(now)
                op.on_start(ctx)
    return outs, tables


TTLS = {"short": STEP // 2, "equal": STEP, "long": 10 ** 12}
SHAPES = {"i64": ("P2", {}), "u64": ("P7", {"key_type": "u64"}), "ts": ("P8", {"key_type": "ts"}),
          "unkeyed": ("P2", {"key_type": None}), "minmax": ("MM", {}), "avg": ("AMM", {"every": 3})}


def _cases():
    return [(s, t) for s in sorted(SHAPES) for t in sorted(TTLS)]


@pytest.mark.parametrize("shape,ttl", _cases())
def test_oracle_equals_the_exact_reference(shape, ttl):
    """Checkpoints at every other flush; no restart, then a restart after every flush in turn."""
    from tests import test_gpu_updating_changes as T
    plan, kw = SHAPES[shape]
    st, aggs = ttl_stream(zlib.crc32(f"{shape}/{ttl}".encode()), **kw), T.PLANS[plan]
    key = st.key_name()
    n = sum(1 for ev in st.events if ev[0] == "flush")
    cps = set(range(1, n, 2))
    for restarts in [()] + [(i,) for i in range(n - 1)]:
        want, want_tables = updating_ttl(reference_events(st.events, cps, restarts), key, aggs, TTLS[ttl])
        got, tables = run_oracle(st, aggs, TTLS[ttl], cps, restarts)
        assert len(got) == n
        for i, (g, w) in enumerate(zip(got, want)):
            errs = flush_errors(g, w, key)
            assert not errs, (shape, ttl, restarts, "flush", i, errs[:8])
        assert len(tables) == len(want_tables)
        for j, (t, w) in enumerate(zip(tables, want_tables)):
            errs = table_errors(t, w, key, aggs)
            assert not errs, (shape, ttl, restarts, "checkpoint", j, errs[:8])


def test_the_stream_exercises_every_case():
    """The streams above do evict, bring keys back, and have flushes whose only rows are evictions."""
    from tests import test_gpu_updating_changes as T
    st = ttl_stream(zlib.crc32(b"i64/equal"))
    want, _ = updating_ttl(reference_events(st.events), "k", T.PLANS["P2"], STEP)
    evicted, back, only = set(), 0, 0
    for r, a, e in want:
        back += len(evicted & set(a))
        evicted |= set(e)
        only += bool(e) and not r and not a
    assert evicted and back and only


@pytest.mark.parametrize("ttl", sorted(TTLS))
def test_reference_mode_keeps_evicted_rows_and_drops_lone_evictions(ttl):
    """reference=True: the table has no tombstones, a restart brings evicted keys back, and a flush whose only rows
    would be evictions emits nothing."""
    from tests import test_gpu_updating_changes as T
    st, aggs = ttl_stream(zlib.crc32(f"ref/{ttl}".encode())), T.PLANS["P3"]
    n = sum(1 for ev in st.events if ev[0] == "flush")
    cps = set(range(n))
    for restarts in [()] + [(i,) for i in range(0, n - 1, 3)]:
        want, want_tables = updating_ttl(reference_events(st.events, cps, restarts), "k", aggs, TTLS[ttl],
                                         tombstones=False)
        got, tables = run_oracle(st, aggs, TTLS[ttl], cps, restarts, reference=True)
        for i, (g, w) in enumerate(zip(got, want)):
            r, a, e = w
            if not r and not a:
                assert g == [], (ttl, restarts, "flush", i)
                continue
            errs = flush_errors(g, w, "k")
            assert not errs, (ttl, restarts, "flush", i, errs[:8])
        for j, (t, w) in enumerate(zip(tables, want_tables)):
            assert all(r is not None for r in w.values())
            errs = table_errors(t, w, "k", aggs)
            assert not errs, (ttl, restarts, "checkpoint", j, errs[:8])


def test_tables_without_tombstones_restore_evicted_keys():
    """A table written in reference mode restores a tombstone-mode oracle: the evicted keys come back, as the
    reference does, and are retracted one ttl after the restart."""
    from tests import test_gpu_updating_changes as T
    st, aggs = ttl_stream(zlib.crc32(b"interchange")), T.PLANS["P2"]
    n = sum(1 for ev in st.events if ev[0] == "flush")
    cut = n // 2
    cfg = U.UpdatingAggConfig(["k"], aggs)
    ctx, op, got = _Ctx(), L.IncrementalAggregatingFunc(cfg, STEP, reference=True), []
    for ev in st.events:
        if ev[0] == "clock":
            op.set_clock(ev[1])
        elif ev[0] == "batch":
            op.process_batch(O.Batch(ev[1]))
        else:
            b = op.handle_checkpoint(None, ctx)
            got.append([] if b is None else b.rows())
            if len(got) - 1 == cut:
                now = op.now
                op = L.IncrementalAggregatingFunc(cfg, STEP)
                op.set_clock(now)
                op.on_start(ctx)
    want, _ = updating_ttl(reference_events(st.events, set(range(n)), {cut}), "k", aggs, STEP, tombstones=False)
    for i, (g, w) in enumerate(zip(got, want)):
        if i <= cut and not w[0] and not w[1]:  # the reference-mode oracle before the cut drops lone evictions
            assert g == []
            continue
        errs = flush_errors(g, w, "k")
        assert not errs, ("flush", i, errs[:8])


def test_default_ttl_is_a_day():
    cfg = U.UpdatingAggConfig(["k"], [O.Agg("count", None, "n")])
    op = L.IncrementalAggregatingFunc(cfg, 0)
    assert op.ttl == 24 * 3600 * 10 ** 9
    op.process_batch(O.Batch({"k": np.array([1]), X.TIMESTAMP: np.array([5])}))
    op.set_clock(op.ttl - 1)
    assert [r[U.IS_RETRACT] for r in op.flush().rows()] == [False]
    op.set_clock(op.ttl)
    assert [(r["k"], r[U.IS_RETRACT]) for r in op.flush().rows()] == [(1, True)]
    with pytest.raises(ValueError):
        op.set_clock(0)
