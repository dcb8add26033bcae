"""The CUDA join with expiration across restarts: tables "left" / "right" written by the Python mirror
(operators.JoinWithExpiration), read back at the first batch after `on_start` and handed to
arroyo_b200_op_restore_side, against the exact restart reference (tests/ttl_join_state_oracle.expiring_join_restarts)
batch by batch and against the golden `updating_inner_join`.  Also: a restored hot chain, a 2^24-row restore whose
multimap then rehashes, interchange of tables with the state oracle, refused restores, and the statistics."""
import ctypes as C
import zlib

import numpy as np
import pyarrow as pa
import pytest

from oracle import arroyo_oracle as O
from tests import exact_reference as X
from tests import test_gpu_joins as J
from tests import ttl_join_state_oracle as S

pytestmark = pytest.mark.gpu

TS = X.TIMESTAMP
T0 = J.T0


def _config(st, ttl):
    import arroyo_b200 as ab
    return ab.JoinConfig(left_on=[st.on[0]], right_on=[st.on[1]], join_type="inner",
                         left_routing_keys=list(st.routing[0]), right_routing_keys=list(st.routing[1]), ttl=ttl)


def run_gpu(st, events, ttl, entry="host", ctx=None, seed=0):
    """Drives the CUDA join through `events` ((side, columns), ("wm", w), ("restart", None)).  A restart checkpoints the
    operator, destroys it and starts a new one on the same context.  Returns the output of each batch event (a list
    of record batches), one (stats, rows sent, rows emitted) per operator that was built, and the context."""
    import arroyo_b200 as ab
    from arroyo_b200 import operators as native
    rng = np.random.default_rng(seed)
    ctx = ctx or ab.OperatorContext(2)
    outs, ops = [], []
    op, sent, emitted = native.JoinWithExpiration(_config(st, ttl)), 0, 0

    def retire(op):
        if op.created:
            ops.append((op.stats(), sent, emitted))
        op.close()

    for ev, arg in events:
        if ev == "wm":
            ctx.watermarks.set(0, arg)
            ctx.watermarks.set(1, arg)
        elif ev == "restart":
            op.handle_checkpoint(None, ctx, None)
            retire(op)
            op, sent, emitted = native.JoinWithExpiration(_config(st, ttl)), 0, 0
            op.on_start(ctx)
        else:
            col = ab.Collector()
            rb = J.to_arrow(st.schemas[ev], arg)
            for piece in (J._slices(rb, rng) if entry == "sliced" and rb.num_rows else [rb]):
                op.process_batch_index(ev, 2, piece, ctx, col)
            outs.append(col.batches)
            sent += rb.num_rows
            emitted += sum(b.num_rows for b in col.batches)
    retire(op)
    return outs, ops, ctx


def reference(st, events, ttl, entry="host", seed=0):
    """The exact output of each batch event.  Sliced input reaches the tables slice by slice, so each slice is a batch
    of its own there (the slices `run_gpu` cuts with the same seed); a batch's output is that of its slices."""
    if entry != "sliced":
        return S.expiring_join_restarts(events, ttl, st.on[0], st.on[1], st.routing[0], st.routing[1])
    rng = np.random.default_rng(seed)
    pieces, per_batch = [], []
    for ev, arg in events:
        if ev not in (0, 1):
            pieces.append((ev, arg))
            continue
        rb = J.to_arrow(st.schemas[ev], arg)
        sizes = [p.num_rows for p in J._slices(rb, rng)] if rb.num_rows else [0]
        starts = np.cumsum([0] + sizes[:-1])
        pieces += [(ev, {c: v[o:o + z] for c, v in arg.items()}) for o, z in zip(starts, sizes)]
        per_batch.append(len(sizes))
    out = S.expiring_join_restarts(pieces, ttl, st.on[0], st.on[1], st.routing[0], st.routing[1])
    want, i = [], 0
    for m in per_batch:
        part = out[i:i + m]
        want.append(X.Rows(part[0].names, np.concatenate([r.vals for r in part]),
                           np.concatenate([r.valid for r in part])))
        i += m
    return want


def check_run(st, events, ttl, entry="host", what=""):
    want = reference(st, events, ttl, entry)
    got, ops, ctx = run_gpu(st, events, ttl, entry)
    assert len(got) == len(want)
    for i, (w, g) in enumerate(zip(want, got)):
        J.check(w, J.rows_of(g, w.names), (what, "batch", i))
    for stats, sent, emitted in ops:  # restored rows count in neither
        assert stats["rows_in"] == sent and stats["rows_out"] == emitted, (stats, sent, emitted)
    return want, ops, ctx


def with_restarts(events, at):
    """`events` with a restart before each batch event numbered in `at` (the number of batches: at the end)."""
    out, b = [], 0
    for ev in events:
        if ev[0] in (0, 1):
            out += [("restart", None)] * at.count(b)
            b += 1
        out.append(ev)
    return out + [("restart", None)] * at.count(b)


def with_watermarks(events):
    """A watermark at the newest timestamp so far after every batch, so that a restart's cutoff is watermark - ttl."""
    out, newest = [], None
    for ev, arg in events:
        out.append((ev, arg))
        if len(arg[TS]):
            newest = max(newest or -(1 << 63), int(np.max(arg[TS])))
        if newest is not None:
            out.append(("wm", newest))
    return out


def n_batches(events):
    return sum(1 for e in events if e[0] in (0, 1))


# ---------------------------------------------------------------------------------------------------------------
def golden_stream(golden, order):
    from tests.test_ttl_join_restore_oracle import golden_feed
    sch = [("counter", "l"), (TS, "tsn:")]
    st = J.Stream(np.random.default_rng(0), left=sch, right=sch, left_on="counter", right_on="counter")
    return st, [(s, dict(b.cols)) for s, b in golden_feed(golden, order)]


@pytest.mark.parametrize("order", ["left_first", "right_first", "alternating"])
def test_updating_inner_join_golden_across_a_restart(golden, accumulator_golden, order):
    """No pair is lost and none is emitted twice, wherever the restart falls."""
    from tests.golden_cases import multiset
    st, feed = golden_stream(golden, order)
    for k in range(n_batches(feed) + 1):
        got, _, _ = run_gpu(st, with_restarts(feed, [k]), 0)
        rows = []
        for g in got:
            for rb in g:
                rows += [{"left_count": a, "right_count": b}
                         for a, b in zip(rb.column(0).to_pylist(), rb.column(1).to_pylist())]
        assert multiset(rows) == multiset(accumulator_golden["updating_inner_join"]), (order, k)


RESTART_CASES = [(s, "host") for s in J.TSHAPES] + [("routing1", "sliced"), ("u64_keys", "sliced"),
                                                     ("edge_keys", "sliced")]


@pytest.mark.parametrize("shape,entry", RESTART_CASES, ids=[f"{s}-{e}" for s, e in RESTART_CASES])
def test_restarts_against_the_exact_reference(shape, entry):
    """Every join shape with a restart at three cuts, under a ttl that keeps everything and one that drops the older
    batches at the restart."""
    st = J.TSHAPES[shape](np.random.default_rng(zlib.crc32(shape.encode()) + 7))
    events = with_watermarks(st.events)
    n = n_batches(events)
    span = max(int(np.max(a[TS])) for e, a in events if e != "wm" and len(a[TS])) - T0
    dropped = False
    for ttl in (0, max(span // 3, 1)):
        full = sum(len(w) for w in reference(st, events, ttl))
        for k in sorted({1, n // 2, n - 1}):
            want, _, _ = check_run(st, with_restarts(events, [k]), ttl, entry, (shape, ttl, k))
            dropped |= sum(len(w) for w in want) < full
    assert dropped or shape in ("zero_rows", "one_key_batch", "long_chain", "one_side_first"), "no pair was dropped"


def test_two_restarts():
    st = J.TSHAPES["edge_keys"](np.random.default_rng(21))
    events = with_watermarks(st.events)
    n = n_batches(events)
    span = int(max(np.max(a[TS]) for e, a in events if e != "wm" and len(a[TS]))) - T0
    for at in ([4, 4], [3, 9], [0, n // 2], [n // 2, n]):
        for ttl in (0, span // 4):
            check_run(st, with_restarts(events, at), ttl, what=("two restarts", at, ttl))


def test_restarts_with_one_empty_side():
    """`one_side_first` sends six left batches before the first right one: a restart there leaves table "right" empty,
    so the new operator learns the right layout only from the right side's first batch; until then the restored left
    rows and the left batches that follow wait.  A restart before any batch finds both tables empty."""
    st = J.TSHAPES["one_side_first"](np.random.default_rng(22))
    events = st.events
    for at in ([0], [3], [6], [3, 5], [3, 9]):
        want, ops, _ = check_run(st, with_restarts(events, at), 0, what=("one side", at))
        assert sum(len(w) for w in want) > 0


def test_hot_chain_restored_then_probed():
    """A 2^20-row chain on one key, restored, then probed by 20 rows: 20 x 2^20 pairs."""
    rng = np.random.default_rng(23)
    st = J.Stream(rng)
    n = 1 << 20
    st.send(0, np.full(n, 5), T0 + np.arange(n))
    st.send(1, np.concatenate([np.full(20, 5), np.arange(100, 130)]), T0 + n + np.arange(50))
    events = with_restarts(st.events, [1])
    got, ops, _ = run_gpu(st, events, 0)
    assert sum(b.num_rows for b in got[1]) == 20 * n
    left, right = st.events[0][1], st.events[1][1]
    col = lambda name: np.concatenate([np.asarray(b.column(name)).view(np.int64) for b in got[1]])  # noqa: E731
    assert np.array_equal(np.sort(col("a")), np.sort(np.repeat(left["a"], 20)))
    assert np.array_equal(np.sort(col("b")), np.sort(np.repeat(right["b"][:20], n)))
    assert np.array_equal(np.sort(col(TS)), np.sort(np.tile(T0 + n + np.arange(20), n)))
    stats, sent, emitted = ops[-1]
    assert stats["rows_in"] == 50 and stats["rows_out"] == 20 * n


def test_large_restore_then_rehash():
    """2^24 left rows restored in one call, then 2^24 more left rows, which rehash the restored multimap, then a right
    batch that probes both."""
    import arroyo_b200 as ab
    from arroyo_b200 import operators as native
    rng = np.random.default_rng(24)
    m, keys = 1 << 24, 1 << 22
    lsch = pa.schema([("id", pa.int64()), (TS, pa.timestamp("ns"))])
    ctx = ab.OperatorContext(2)
    table = ctx.table("left", S.DAY_NS)
    lk = [rng.integers(0, keys, m), rng.integers(0, keys, m)]
    for i in range(16):  # the restored table: 16 batches of 2^20 rows
        part = slice(i << 20, (i + 1) << 20)
        table.insert(T0 + i, pa.RecordBatch.from_arrays(
            [pa.array(lk[0][part]), pa.array(np.full(1 << 20, T0 + i)).cast(pa.timestamp("ns"))], schema=lsch))
    st = J.Stream(rng, left=[("id", "l"), (TS, "tsn:")])
    op = native.JoinWithExpiration(_config(st, 0), left_schema=J.arrow_schema(st.schemas[0]),
                                   right_schema=J.arrow_schema(st.schemas[1]))
    op.on_start(ctx)
    col = ab.Collector()
    second = pa.RecordBatch.from_arrays([pa.array(lk[1]), pa.array(np.full(m, T0 + 20)).cast(pa.timestamp("ns"))],
                                        schema=lsch)
    op.process_batch_index(0, 2, second, ctx, col)
    assert not col.batches
    after = op.stats()
    assert after["rows_in"] == m and after["h2d_bytes"] >= 2 * m * 16  # the restore's copies and the batch's
    rk = rng.integers(0, keys, 4096)
    st.send(1, rk, np.full(4096, T0 + 30))
    op.process_batch_index(1, 2, J.to_arrow(st.schemas[1], st.events[-1][1]), ctx, col)
    got = J.rows_of(col.batches, ["id", "id_right", "b", TS])
    # every (left row, right row) with equal keys, from a sort of the 2^25 left keys
    allk = np.concatenate(lk)
    lts = np.concatenate([np.repeat(T0 + np.arange(16), 1 << 20), np.full(m, T0 + 20)])
    order = np.argsort(allk, kind="stable")
    lo, hi = np.searchsorted(allk[order], rk, "left"), np.searchsorted(allk[order], rk, "right")
    cnt = hi - lo
    ri = np.repeat(np.arange(4096), cnt)
    li = order[np.repeat(lo, cnt) + np.arange(cnt.sum()) - np.repeat(np.cumsum(cnt) - cnt, cnt)]
    b = st.events[-1][1]["b"]
    want = X.Rows.from_columns(["id", "id_right", "b", TS], [allk[li], rk[ri], b[ri], np.maximum(lts[li], T0 + 30)])
    assert len(want) > 10_000
    J.check(want, got, "large restore")
    op.close()


# ---------------------------------------------------------------------------------------------------------------
def _oracle_events(events):
    return [(e, O.Batch({k: np.asarray(v) for k, v in a.items()})) if e in (0, 1) else (e, a) for e, a in events]


@pytest.mark.parametrize("direction", ["oracle_to_gpu", "gpu_to_oracle"])
def test_checkpoint_interchange_with_the_state_oracle(direction):
    """Tables written by one implementation restore into the other; the output after the restart is exact."""
    import arroyo_b200 as ab
    st = J.TSHAPES["edge_keys"](np.random.default_rng(25))
    events = with_watermarks(st.events)
    n = n_batches(events)
    span = int(max(np.max(a[TS]) for e, a in events if e != "wm" and len(a[TS]))) - T0
    for k in (2, n // 2, n - 2):
        for ttl in (0, span // 3):
            full = with_restarts(events, [k])
            cut = full.index(("restart", None))
            want = reference(st, full, ttl)
            nb = n_batches(full[:cut])
            gctx, octx = ab.OperatorContext(2), O.OperatorContext(2)
            if direction == "oracle_to_gpu":
                _, octx = S.run_oracle(_oracle_events(full[:cut + 1]), ttl, *st.on, ctx=octx)
                for name in S.TABLES:
                    for t, batches in octx.table(name, S.retention(ttl)).all_batches_for_watermark(None):
                        for b in batches:
                            side = S.TABLES.index(name)
                            gctx.table(name, S.retention(ttl)).insert(t, J.to_arrow(st.schemas[side], b.cols))
                for i in (0, 1):
                    gctx.watermarks.set(i, octx.watermarks.watermarks[i])
                got, _, _ = run_gpu(st, [("restart", None)] + full[cut + 1:], ttl, ctx=gctx)
                got = [J.rows_of(g, w.names) for g, w in zip(got, want[nb:])]
            else:
                _, _, gctx = run_gpu(st, full[:cut + 1], ttl, ctx=gctx)
                for name in S.TABLES:
                    for t, b in gctx.table(name, S.retention(ttl)).all_batches_for_watermark(None):
                        octx.table(name, S.retention(ttl)).insert(
                            t, O.Batch({c: np.asarray(b.column(c)).view(np.int64) if b.schema.field(c).type != pa.uint64()
                                        else np.asarray(b.column(c)) for c in b.schema.names}))
                for i in (0, 1):
                    octx.watermarks.set(i, gctx.watermarks.watermarks[i])
                got, _ = S.run_oracle(_oracle_events([("restart", None)] + full[cut + 1:]), ttl, *st.on, ctx=octx,
                                      names=S.output_names(full))
            assert len(got) == len(want) - nb
            for i, (w, g) in enumerate(zip(want[nb:], got)):
                J.check(w, g, (direction, k, ttl, i))
            assert sum(len(w) for w in want[nb:]) > 0


# ---------------------------------------------------------------------------------------------------------------
def _restore(op, side, batches):
    """arroyo_b200_op_restore_side on exported `batches`; returns the status and whether each array was taken."""
    from arroyo_b200 import ffi, operators as native
    n = len(batches)
    arrs, schs = (ffi.ArrowArray * max(n, 1))(), (ffi.ArrowSchema * max(n, 1))()
    for i, b in enumerate(batches):
        b._export_to_c(C.addressof(arrs[i]), C.addressof(schs[i]))
    code = op._lib.arroyo_b200_op_restore_side(op._h, side, arrs, schs, n)
    taken = [not arrs[i].release for i in range(n)]
    assert all(schs[i].release for i in range(n))  # the schemas stay the caller's
    for s in list(arrs)[:n] + list(schs)[:n]:
        native._release(s)
    return code, taken


def _refusal_stream():
    rng = np.random.default_rng(26)
    st = J.Stream(rng)
    for i in range(6):
        st.send(i % 2, rng.integers(0, 40, 300), T0 + 1000 * i + np.arange(300))
    return st


def _made(st):
    from tests.test_gpu_joins import _make
    return _make("expiring", st)


def _continue_and_check(op, st, restored):
    """Sends the stream's batches after the restore of `restored` ((side, columns) list) and checks them exactly."""
    import arroyo_b200 as ab
    ctx = ab.OperatorContext(2)
    events = list(restored) + [("restart", None)] + st.events
    want = reference(st, events, 0)[len(restored):]
    got = []
    for side, cols in st.events:
        c = ab.Collector()
        op.process_batch_index(side, 2, J.to_arrow(st.schemas[side], cols), ctx, c)
        got.append(c.batches)
    for i, (w, g) in enumerate(zip(want, got)):
        J.check(w, J.rows_of(g, w.names), ("after refusal", i))
    assert sum(len(w) for w in want) > 0
    stats = op.stats()
    assert stats["rows_in"] == sum(len(c[TS]) for _, c in st.events)
    assert stats["rows_out"] == sum(len(w) for w in want)


def _table_batches(st, side, n, seed):
    rng = np.random.default_rng(seed)
    src = J.Stream(rng)
    for i in range(n):
        src.send(side, rng.integers(0, 40, 200), T0 - 10_000 + 500 * i + np.arange(200))
    return src.events


def test_restore_after_process_batch_is_refused():
    """Once a batch is in, a restore is refused with nothing taken, and the stream goes on as if it had not been
    asked for."""
    import arroyo_b200 as ab
    from arroyo_b200 import ffi
    st = _refusal_stream()
    op = _made(st)
    ctx = ab.OperatorContext(2)
    want = reference(st, st.events, 0)
    got = []
    for i, (side, cols) in enumerate(st.events):
        c = ab.Collector()
        op.process_batch_index(side, 2, J.to_arrow(st.schemas[side], cols), ctx, c)
        got.append(c.batches)
        if i == 0:
            table = [J.to_arrow(st.schemas[1], c) for _, c in _table_batches(st, 1, 2, 1)]
            assert _restore(op, 1, table) == (ffi.INVALID_ARGUMENT, [False, False])
    for i, (w, g) in enumerate(zip(want, got)):
        J.check(w, J.rows_of(g, w.names), ("after a late restore", i))
    assert op.stats()["rows_out"] == sum(len(w) for w in want) > 0
    op.close()


@pytest.mark.parametrize("what", ["columns", "key_type", "nulls"])
def test_refused_restore_keeps_nothing(what):
    """A call with one bad batch among good ones keeps no row of the call and takes no array; the same good batches
    then restore, and the stream joins exactly against them."""
    from arroyo_b200 import ffi
    st = _refusal_stream()
    op = _made(st)
    left = _table_batches(st, 0, 3, 2)
    right = _table_batches(st, 1, 2, 3)
    good = [J.to_arrow(st.schemas[0], c) for _, c in left]
    if what == "key_type":  # the right side restores Int64 keys first; a UInt64 left key then differs from them
        assert _restore(op, 1, [J.to_arrow(st.schemas[1], c) for _, c in right]) == (ffi.OK, [True, True])
        sch = [(n, "L" if n == "id" else c) for n, c in st.schemas[0]]
        bad = J.to_arrow(sch, {k: np.asarray(v).view(np.uint64) if k == "id" else v for k, v in left[0][1].items()})
        want_code = ffi.UNSUPPORTED
    elif what == "columns":
        bad = good[0].drop_columns(["a"])
        want_code = ffi.INVALID_ARGUMENT
    else:
        a = pa.array(list(range(199)) + [None], type=pa.int64())
        bad = pa.RecordBatch.from_arrays([good[0].column(0), a, good[0].column(2)], names=good[0].schema.names)
        want_code = ffi.UNSUPPORTED
    code, taken = _restore(op, 0, good[:2] + [bad] + good[2:])
    assert code == want_code and not any(taken), (code, op._lib.arroyo_b200_op_last_error(op._h))
    st0 = op.stats()
    assert st0["rows_in"] == 0 and st0["rows_out"] == 0
    assert _restore(op, 0, good) == (ffi.OK, [True] * 3)
    if what != "key_type":
        assert _restore(op, 1, [J.to_arrow(st.schemas[1], c) for _, c in right]) == (ffi.OK, [True, True])
    _continue_and_check(op, st, left + right)
    op.close()


def test_zero_row_and_empty_restores_are_accepted():
    from arroyo_b200 import ffi
    st = _refusal_stream()
    op = _made(st)
    empty = J.to_arrow(st.schemas[0], {n: np.zeros(0, J.NP[c]) for n, c in st.schemas[0]})
    assert _restore(op, 0, []) == (ffi.OK, [])
    assert _restore(op, 0, [empty]) == (ffi.OK, [True])
    assert op.stats()["kernel_launches"] == 0
    _continue_and_check(op, st, [])
    op.close()


@pytest.mark.parametrize("kind", ["tumbling", "session", "updating", "instant_join"])
def test_restore_side_is_only_for_the_join_with_expiration(kind):
    from arroyo_b200 import ffi
    if kind == "instant_join":
        st = _refusal_stream()
        from tests.test_gpu_joins import _make
        op = _make("instant", st)
        batch = J.to_arrow(st.schemas[0], st.events[0][1])
    else:
        from tests.test_abi_batches import _batch, _new
        op = _new(kind)
        batch = _batch(np.random.default_rng(0), 0)
    code, taken = _restore(op, 0, [batch])
    assert code == ffi.UNSUPPORTED and taken == [False]
    op.close()
