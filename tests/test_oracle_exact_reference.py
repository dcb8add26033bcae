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


# ---- session windows: the numpy and C session oracles against exact_reference.session_emissions ----------------------
def _session_shapes():
    from tests import test_gpu_session_time as T
    # UInt64 keys are left out: the numpy oracle builds its output key column from Python ints and turns keys >= 2^63
    # into Float64 (the C oracle takes Int64 keys only)
    return [(s, k, g, p) for s, k, g, p, _ in T.CASES if k != "u64"]


@pytest.mark.parametrize("impl", ["numpy", "c"])
def test_session_oracle_matches_exact_reference(impl):
    from tests import test_gpu_session_time as T
    ran = 0
    for shape, keys, gap, plan in _session_shapes():
        st = T.make(shape, keys, gap)
        cfg = T.config(st, plan)
        # session_oracle.c: one value column, no checkpoint / restore
        if impl == "c" and (len({a.col for a in cfg.aggs if a.col}) > 1 or any(ev[0] == "restart" for ev in st.events)):
            continue
        want, _, _ = T.reference(st, cfg)
        T.check_emissions(want, T.run_oracle(st, cfg, impl), cfg, f"{impl} {shape}/{keys}/{gap}/{plan}")
        ran += 1
    assert ran >= (20 if impl == "numpy" else 10)


def _chain_stream(seed, keys, gap, n_batches=60):
    """At most one row per key per batch, no two rows of a key exactly `gap` apart, watermarks behind the data."""
    from tests import test_gpu_session_time as T
    st = T.Stream(seed, keys, gap)
    rng, o, used = st.rng, T.ORIGIN, {}
    ks = [None] if keys == "none" else st.keyset()
    st.wm(o - 10 * gap)
    for b in range(n_batches):
        tss, kk = [], []
        for k in ks:
            if rng.random() < 0.3:
                continue
            while True:
                t = o + int(rng.integers(0, 40 * gap)) + (b * gap) // 2
                if all(abs(t - u) != gap for u in used.get(k, ())):
                    break
            used.setdefault(k, []).append(t)
            tss.append(t)
            kk.append(k)
        if tss:
            st.batch(tss, None if keys == "none" else np.asarray(kk, dtype=object))
        if b % 7 == 6:
            st.wm(o + (b - 14) * gap // 2)
    return st.end()


@pytest.mark.parametrize("keys", ["few", "none", "edge"])
@pytest.mark.parametrize("gap", [1, 999, 5 * S])
def test_session_emissions_match_chains(keys, gap):
    """In the restricted class of streams, every emitted session is a maximal chain of the key's on-time rows whose
    consecutive distances are < gap: the rule statement of session_emissions against the declarative definition."""
    from tests import test_gpu_session_time as T
    st = _chain_stream(abs(hash((keys, gap))) % 1000, keys, gap)
    cfg = T.config(st, "count")
    out, _, _ = T.reference(st, cfg)
    got = {}
    for emitted in out:
        for (k, s), r in emitted.items():
            assert (k, s) not in got
            got[(k, s)] = (r["window_end"], r["n"])
    want = X.session_chains(st.events, cfg.key_names[0] if cfg.key_names else None, gap)
    assert got == want


def test_session_emissions_by_hand():
    """The session rules on streams small enough to follow by hand (gap 10)."""
    aggs = [A("count", None, "n"), A("sum", "a", "s")]

    def b(ts, a):
        return {"a": np.array(a, dtype=np.int64), X.TIMESTAMP: np.array(ts, dtype=np.int64)}

    # one run [0, 5, 25, 26] under a watermark: 25 breaks the scan and is taken without extending data_end
    out, late, n_keys = X.session_emissions([("wm", -100), ("batch", b([0, 5, 25, 26], [1, 2, 3, 4])),
                                             ("wm", 15), ("wm", 16), ("wm", X.INT64_MAX)], None, aggs, 10)
    assert late == 0 and n_keys == 1
    assert out[0] == {} and out[1] == {} and list(out[2]) == [(None, 0)]  # w = 15 = data_end + gap does not close
    assert out[2][(None, 0)]["n"] == 3 and out[2][(None, 0)]["window_end"] == 15 and out[2][(None, 0)]["s"] == 6
    assert list(out[3]) == [(None, 26)] and out[3][(None, 26)]["n"] == 1
    # inside one run, a row exactly gap after the first breaks the scan and is still taken; ts < w is late, ts = w not
    out, late, _ = X.session_emissions([("batch", b([0, 10], [1, 2])), ("wm", 10), ("wm", 11), ("batch", b([11, 9], [5, 6])),
                                        ("wm", 21), ("wm", 22)], None, aggs, 10)
    assert late == 1
    assert out[0] == {} and list(out[1]) == [(None, 0)] and out[1][(None, 0)]["n"] == 2
    assert out[1][(None, 0)]["window_end"] == 10 and out[2] == {} and out[3][(None, 11)]["s"] == 5
    # a restart after the session at 0 closed: table "s" replays from start = 0, the restored watermark drops it again
    out, _, _ = X.session_emissions([("batch", b([0], [1])), ("wm", 11), ("batch", b([30], [2])), ("restart",),
                                     ("wm", X.INT64_MAX)], None, aggs, 10)
    assert list(out[0]) == [(None, 0)] and list(out[1]) == [(None, 30)]


# ---- the updating aggregate: the oracle's change stream against exact_reference.updating_changes -------------------
def _oracle_changes(st, aggs):
    """The oracle on a stream of tests/test_gpu_updating_changes.py: one (retraction rows, append rows) per flush."""
    cfg = U.UpdatingAggConfig([st.key_name()] if st.key_type else [], aggs)
    op, out = U.IncrementalAggregatingFunc(cfg), []
    for ev in st.events:
        if ev[0] == "batch":
            op.process_batch(O.Batch(ev[1]))
            continue
        b = op.flush()
        rows = [] if b is None else b.rows()
        out.append(([r for r in rows if r[U.IS_RETRACT]], [r for r in rows if not r[U.IS_RETRACT]]))
    return out


def _updating_cpu_shapes():
    from tests import test_gpu_updating_changes as T
    return [
        ("random", "P2", lambda: T.s_random(1)), ("random_u64", "P7", lambda: T.s_random(2, "u64", every=3)),
        ("random_ts", "P8", lambda: T.s_random(3, "ts", every=1)), ("quiet_P1", "P1", lambda: T.s_quiet(4, "P1")),
        ("quiet_MM", "MM", lambda: T.s_quiet(5, "MM")), ("quiet_AMM", "AMM", lambda: T.s_quiet(6, "AMM")),
        ("quiet_flush_P1", "P1", lambda: T.s_quiet(7, "P1", whole_flush=True)),
        ("quiet_flush_AMM", "AMM", lambda: T.s_quiet(8, "AMM", "u64", whole_flush=True)),
        ("ts_backwards", "P1", lambda: T.s_ts_backwards(9)), ("double_tick", "P4", lambda: T.s_cadence(10, "double")),
        ("tick_first", "COUNT", lambda: T.s_cadence(11, "tick_first")),
        ("empty_and_one", "P3", lambda: T.s_cadence(12, "empty_and_one")),
        ("edge_keys", "P5", lambda: T.s_edge_keys(13)), ("edge_keys_u64", "P6b", lambda: T.s_edge_keys(14, "u64")),
        ("unkeyed", "P2", lambda: T.s_unkeyed(15)), ("growth", "P1", lambda: T.s_growth(16, 3000)),
        ("edge_values", "P3", lambda: T.s_edge_values(17)), ("crowded_spread", "P6a", lambda: T.s_crowded(18, 1400, True)),
    ]


@pytest.mark.parametrize("case", _updating_cpu_shapes(), ids=lambda c: c[0])
def test_updating_oracle_change_stream_matches_exact_reference(case):
    """Flush by flush, the oracle's retractions and appends equal updating_changes' on every column (the flag by the
    split, _timestamp exactly, AVG by its rule)."""
    from tests import test_gpu_updating_changes as T
    name, plan, make = case
    st = make()
    aggs = T.PLANS[plan]
    key = st.key_name()
    want = X.updating_changes(st.events, key, aggs)
    got = _oracle_changes(st, aggs)
    assert len(got) == len(want)
    n_rows = 0
    for i, ((gr, ga), (wr, wa)) in enumerate(zip(got, want)):
        for g, w in ((gr, wr), (ga, wa)):
            errs = X.mismatches(w, g, lambda r: int(r[key]) if key else None)
            assert not errs, (name, "flush", i, errs[:8])
        n_rows += len(gr) + len(ga)
    assert n_rows > 0
    if name.startswith("quiet_flush"):
        assert want[3] == ({}, {})  # a period of quiet rows only


def test_updating_changes_by_hand():
    """The change-stream rules on a stream small enough to follow by hand."""
    aggs = [A("sum", "a", "s"), A("max", "a", "mx")]

    def b(k, a, ts):
        return ("batch", {"k": np.array(k, dtype=np.int64), "a": np.array(a, dtype=np.int64),
                          X.TIMESTAMP: np.array(ts, dtype=np.int64)})
    ev = [("flush",), b([1, 2], [5, 3], [10, 20]), ("flush",),
          b([1, 1], [2, -2], [30, 31]),   # key 1: SUM and MAX unchanged, _timestamp 10 -> 31: suppressed
          ("flush",), ("flush",),
          b([1, 2], [7, 0], [5, 40]),     # key 1 changes: the retraction carries _timestamp 31; key 2 suppressed
          ("flush",)]
    out = X.updating_changes(ev, "k", aggs)
    assert out[0] == ({}, {})
    assert out[1][0] == {} and out[1][1] == {1: {"k": 1, "s": 5, "mx": 5, X.TIMESTAMP: 10},
                                             2: {"k": 2, "s": 3, "mx": 3, X.TIMESTAMP: 20}}
    assert out[2] == ({}, {}) and out[3] == ({}, {})
    assert out[4] == ({1: {"k": 1, "s": 5, "mx": 5, X.TIMESTAMP: 31}}, {1: {"k": 1, "s": 12, "mx": 7, X.TIMESTAMP: 31}})
    # unkeyed, SUM wrapping at 64 bits, and an AVG whose exact mean moves below one f64 ulp: suppressed
    big = (1 << 62)
    ev = [("batch", {"a": np.array([big, big], dtype=np.int64), X.TIMESTAMP: np.array([1, 2], dtype=np.int64)}),
          ("flush",),
          ("batch", {"a": np.array([big + 1], dtype=np.int64), X.TIMESTAMP: np.array([3], dtype=np.int64)}),
          ("flush",)]
    out = X.updating_changes(ev, None, [A("avg", "a", "av")])
    assert list(out[0][1]) == [None] and float(out[0][1][None]["av"].exact) == float(big)
    assert out[1] == ({}, {})
    out = X.updating_changes(ev, None, [A("sum", "a", "s")])
    assert out[0][1][None]["s"] == -(1 << 63) and out[1][0][None]["s"] == -(1 << 63)
    assert out[1][1][None]["s"] == -(1 << 63) + big + 1
