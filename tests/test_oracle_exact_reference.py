"""The oracles against the exact group-by of tests/exact_reference.py on the multi-column plans of
tests/test_gpu_agg_plans.py: tumbling and sliding windows (oracle/arroyo_oracle.py) and the updating aggregate
(oracle/updating_oracle.py), including AVG over inputs whose integer sum wraps."""
import numpy as np
import pytest

from oracle import arroyo_oracle as O
from oracle import updating_oracle as U
from tests import exact_reference as X
from tests.test_gpu_agg_plans import PLANS, run_updating, stream
from tests.test_gpu_parity import S, T0

A = O.Agg


@pytest.mark.parametrize("regime", ["R1", "R2", "R3"])
@pytest.mark.parametrize("kind", ["tumbling", "sliding"])
def test_window_oracle_matches_exact_reference(kind, regime):
    for i, (plan, aggs) in enumerate(PLANS.items()):
        keys = ("uniform", "hot", "u64", "none")[i % 4]
        key_names = [] if keys == "none" else ["key"]
        batches = stream(keys, regime, n_rows=8_000, batch=1_000, seed=i)
        if kind == "sliding":
            cfg = O.WindowAggConfig(width=4 * S, slide=S, key_names=key_names, aggs=aggs, window_index=len(key_names))
            op = O.SlidingAggregatingWindowFunc(cfg)
        else:
            cfg = O.WindowAggConfig(width=S, key_names=key_names, aggs=aggs, window_index=len(key_names))
            op = O.TumblingAggregatingWindowFunc(cfg)
        got = O.run_single_input(op, batches, S).batches
        want = X.window_rows(batches, key_names[0] if key_names else None, aggs, cfg.width, cfg.slide or None)
        rows = [r for b in got for r in b.rows()]
        errs = X.mismatches(want, rows, lambda r: (r["window_start"], r["key"] if key_names else None))
        assert not errs, (plan, errs[:10])


@pytest.mark.parametrize("regime", ["R1", "R2", "R3"])
def test_updating_oracle_matches_exact_reference(regime):
    for i, (plan, aggs) in enumerate(PLANS.items()):
        keys = ("uniform", "hot", "u64", "none")[i % 4]
        key_names = [] if keys == "none" else ["key"]
        batches = stream(keys, regime, n_rows=3_000, batch=250, seed=i)
        cfg = U.UpdatingAggConfig(key_names, aggs)
        final = U.merge_change_stream(run_updating(U.IncrementalAggregatingFunc(cfg), batches, 3), key_names)
        want = X.updating_rows(batches, key_names[0] if key_names else None, aggs)
        want = {k: {c: v for c, v in r.items() if c != X.TIMESTAMP} for k, r in want.items()}
        errs = X.mismatches(want, final, lambda r: r["key"] if key_names else None)
        assert not errs, (plan, errs[:10])
        # the oracle's AVG is the reference's own arithmetic: the f64 sum in row order
        for r in final:
            w = want[r["key"] if key_names else None]
            for a in aggs:
                if a.kind == "avg":
                    assert r[a.name] == w[a.name].seq, (plan, r, w[a.name])


def test_updating_oracle_avg_does_not_wrap():
    """Four rows of 2^62 on one key: the wrapping i64 sum is 0, the AVG is 2^62."""
    aggs = [A("avg", "a", "ava"), A("sum", "a", "sa"), A("count", None, "n")]
    cfg = U.UpdatingAggConfig(["key"], aggs)
    b = O.Batch({"key": np.array([7, 7, 7, 7, 8, 8], dtype=np.int64),
                 "a": np.array([1 << 62] * 4 + [3, -4], dtype=np.int64), O.TIMESTAMP: T0 + np.arange(6, dtype=np.int64)})
    final = {r["key"]: r for r in U.merge_change_stream(run_updating(U.IncrementalAggregatingFunc(cfg), [b], 0), ["key"])}
    assert final[7] == {"key": 7, "ava": float(1 << 62), "sa": 0, "n": 4}
    assert final[8] == {"key": 8, "ava": -0.5, "sa": -1, "n": 2}
    assert not X.mismatches({k: {c: v for c, v in r.items() if c != X.TIMESTAMP}
                             for k, r in X.updating_rows([b], "key", aggs).items()}, list(final.values()),
                            lambda r: r["key"])


def test_exact_reference_avg_rule():
    """The AVG rule itself: exact below 2^53 (a one-ulp slip fails), the summation bound above."""
    from fractions import Fraction
    m = X.Mean(Fraction(10, 3), 10)
    assert X.check_avg(10 / 3, m)
    assert not X.check_avg(np.nextafter(10 / 3, 4), m)
    assert not X.check_avg(float(np.float32(10 / 3)), m)
    big = X.Mean(Fraction(4 * (1 << 62) + 1, 4), 4 * (1 << 62) + 1)
    assert X.check_avg(float(1 << 62), big)
    assert not X.check_avg(0.0, big)



# ---- event time: the window oracle against window_emissions, watermark by watermark ----
TIME_SHAPES = ["T1", "T2", "T3", "T4:1", "T4:n-1", "T4:n", "T4:n+1", "T4:4095", "T4:4096", "T4:4097", "T4:1000000", "T5", "T5:wide",
               "T6:1", "T6:2", "T6:4", "T6:4095", "T6:4096", "T6:4097", "T6:5000", "T6:1000000", "T7:16", "T7:17",
               "T7:600", "T7:3600", "T7:4096", "T7:4097", "T8:zero", "T8:neg", "T8:big@30d", "T8:zero@2", "T8:zero@3",
               "T8:big@p", "T8:big@2^32-1", "T8:big@2^32+1", "T8:neg@p", "T9"]


@pytest.mark.parametrize("kind", ["tumbling", "running"])
def test_window_oracle_event_time_matches_exact_reference(kind):
    from tests import test_gpu_window_time as T
    for i, shape in enumerate(TIME_SHAPES):
        keys = ("few", "many", "none")[i % 3]
        plan = ("ints", "minmax")[i % 2]
        st = T._shape(shape, kind)(keys)
        cfg = T.config(st, kind, plan)
        want, _ = T.reference(st, cfg)
        T.check_emissions(want, T.run_oracle(st, kind, cfg), cfg, f"oracle {shape}")


def test_window_emissions_by_hand():
    """The event-time rules on a stream small enough to follow by hand (tumbling width 10, sliding 20 / 10)."""
    aggs = [A("count", None, "n"), A("sum", "a", "s")]
    b1 = {"a": np.array([1, 2, 3, 4], dtype=np.int64), X.TIMESTAMP: np.array([3, 12, 19, 25], dtype=np.int64)}
    b2 = {"a": np.array([10, 20, 30, 40], dtype=np.int64), X.TIMESTAMP: np.array([9, 10, 14, 15], dtype=np.int64)}
    ev = [("wm", -25), ("batch", b1), ("wm", 15), ("batch", b2), ("restart",), ("wm", 20), ("wm", 20), ("wm", X.INT64_MAX)]
    out, late = X.window_emissions(ev, None, aggs, 10)
    assert late == 1  # ts 9: bin 0 < bin(15) = 10; ts 10 and 14 are in [bin(w), w), ts 15 is at w
    assert [list(o) for o in out] == [[], [(0, None)], [(10, None)], [], [(20, None)]]
    assert out[1][(0, None)]["n"] == 1 and out[2][(10, None)]["s"] == 2 + 3 + 20 + 30 + 40
    out, late = X.window_emissions(ev, None, aggs, 20, 10)
    assert late == 1
    assert [list(o) for o in out] == [[], [(-10, None)], [(0, None)], [], [(10, None), (20, None)]]
    assert out[2][(0, None)]["n"] == 6 and out[4][(20, None)]["s"] == 4
    with pytest.raises(ValueError):
        X.window_emissions([("wm", 5), ("wm", 4)], None, aggs, 10)

# ---- joins: the oracles' InstantJoin (numpy and C) and JoinWithExpiration against the exact reference joins ----
INSTANT_SHAPES = ["left_smaller", "right_smaller", "equal", "zero_eligible", "left_only", "right_only", "build_1",
                  "build_511", "build_513", "edge_keys", "u64_keys", "ts_keys", "many_instants", "ts_2p32", "ts_eq_wm",
                  "routing1", "routing2"]
# join_oracle.c: Int64-compatible columns only, no routing columns, both layouts known before the first watermark
C_ORACLE_SHAPES = ["left_smaller", "right_smaller", "equal", "zero_eligible", "build_511", "edge_keys", "u64_keys",
                   "ts_2p32", "ts_eq_wm", "many_instants"]


def _oracle_instant(join, st):
    ctx, outs = O.OperatorContext(2), []
    for ev, arg in st.events:
        if ev == "wm":
            for i in (0, 1):
                ctx.watermarks.set(i, arg)
            col = O.Collector()
            join.handle_watermark(arg, ctx, col)
            outs.append(col.batches)
        else:
            join.process_batch_index(ev, 2, O.Batch(dict(arg)), ctx, O.Collector())
    return outs


def _oracle_rows(batches, names):
    if not batches:
        return X.Rows(names, np.zeros((0, len(names)), np.uint64), np.zeros((0, len(names)), bool))
    b = O.Batch.concat(batches)
    assert b.names() == names, (b.names(), names)
    return X.Rows.from_columns(names, [b[c] for c in names], b.valid)


@pytest.mark.parametrize("join_type", ["inner", "left", "right", "full"])
@pytest.mark.parametrize("impl", ["numpy", "c"])
def test_instant_join_oracle_matches_exact_reference(impl, join_type):
    from oracle import c_oracle
    from tests.test_gpu_joins import SHAPES
    for shape in INSTANT_SHAPES if impl == "numpy" else C_ORACLE_SHAPES:
        st = SHAPES[shape](np.random.default_rng(7))
        cfg = O.JoinConfig(left_on=[st.on[0]], right_on=[st.on[1]], join_type=join_type,
                           left_routing_keys=list(st.routing[0]), right_routing_keys=list(st.routing[1]))
        got = _oracle_instant(O.InstantJoin(cfg) if impl == "numpy" else c_oracle.InstantJoin(cfg), st)
        want = st.reference_instant(join_type)
        assert len(got) == len(want)
        for i, (w, g) in enumerate(zip(want, got)):
            errs = X.join_mismatches(w, _oracle_rows(g, w.names))
            assert not errs, (shape, i, errs)


def _dict_rows(rows, names):
    """Rows as dicts of Python values (floats by their bits, ints as 64-bit patterns) -> X.Rows."""
    vals = np.zeros((len(rows), len(names)), dtype=np.uint64)
    for i, r in enumerate(rows):
        assert list(r) == names, (list(r), names)
        for j, c in enumerate(names):
            v = r[c]
            vals[i, j] = np.array([v]).view(np.uint64)[0] if isinstance(v, float) else int(v) % (1 << 64)
    return X.Rows(names, vals, np.ones(vals.shape, bool))


def test_expiring_join_oracle_matches_exact_reference():
    from tests.test_gpu_joins import TSHAPES
    for shape in ["edge_keys", "u64_keys", "ts_keys", "zero_rows", "one_side_first", "routing0"]:
        st = TSHAPES[shape](np.random.default_rng(3))
        join = U.JoinWithExpiration(*st.on)
        want = st.reference_expiring()
        for i, ((side, cols), w) in enumerate(zip(st.events, want)):
            errs = X.join_mismatches(w, _dict_rows(join.process_batch_index(side, 2, O.Batch(dict(cols))), w.names))
            assert not errs, (shape, i, errs)


def test_exact_reference_joins_by_hand():
    """The reference joins on a stream small enough to follow by hand."""
    left = {"id": np.array([1, 1, 2, -1], dtype=np.int64), "a": np.array([10, 11, 12, 13], dtype=np.int64),
            X.TIMESTAMP: np.array([5, 5, 5, 9], dtype=np.int64)}
    right = {"id": np.array([1, 3, -1], dtype=np.int64), "a": np.array([20, 21, 22], dtype=np.int64),
             X.TIMESTAMP: np.array([5, 5, 7], dtype=np.int64)}
    out = X.instant_join([(0, left), (1, right), ("wm", 9), ("wm", 10)], "full", "id", "id")
    assert out[0].names == ["id", "a", "id_right", "a_right", X.TIMESTAMP]
    assert sorted(out[0].tuples(), key=str) == sorted([(1, 10, 1, 20, 5), (1, 11, 1, 20, 5), (2, 12, None, None, 5),
                                                       (None, None, 3, 21, 5), (None, None, (1 << 64) - 1, 22, 7)],
                                                      key=str)
    assert out[1].tuples() == [((1 << 64) - 1, 13, None, None, 9)]  # -1 at ts 9 != -1 at ts 7
    with pytest.raises(ValueError):
        X.instant_join([("wm", 6), (0, left)], "inner", "id", "id")
    out = X.expiring_join([(1, right), (0, left)], "id", "id")
    assert len(out[0]) == 0
    assert sorted(out[1].tuples()) == sorted([(1, 10, 1, 20, 5), (1, 11, 1, 20, 5),
                                              ((1 << 64) - 1, 13, (1 << 64) - 1, 22, 9)])
    a, b = out[1], X.Rows(out[1].names, out[1].vals[::-1], out[1].valid[::-1])
    assert not X.join_mismatches(a, b)
    b.vals[0, 1] ^= np.uint64(1)
    assert X.join_mismatches(a, b)
