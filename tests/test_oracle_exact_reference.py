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
