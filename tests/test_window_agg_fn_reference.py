"""Pins the exact reference's aggregate window functions (tests/exact_window_agg_reference.py: COUNT / SUM / AVG / MIN /
MAX OVER (PARTITION BY window [, key] [ORDER BY ...]) with the default frame) to an independent engine, SQLite's
window functions, which take the same default frames: the whole partition without ORDER BY, `RANGE BETWEEN UNBOUNDED
PRECEDING AND CURRENT ROW` with it.  The arguments are bounded so that SQLite's checked Int64 sums cannot overflow;
wrapping SUM near +-2^63 is checked against numpy's int64 cumsum instead."""
import math
import sqlite3

import numpy as np
import pytest

from tests.exact_window_agg_reference import AGGREGATES, aggregate_rows, window_agg_emissions
from tests.exact_window_fn_reference import INT64_MAX, TS

ORDER_SETS = {0: [], 1: [("k0", True)], 2: [("k0", False), ("k1", True)],
              4: [("k0", True), ("k1", False), ("k2", True), ("k3", False)]}


def random_batch(seed, n=3000):
    """Rows with heavy ties: 6 instants, 4 partition keys, ORDER BY keys from 3 values, a unique `seq`."""
    rng = np.random.default_rng(seed)
    cols = {"p": rng.integers(0, 4, n), TS: rng.integers(0, 6, n) * 1000 + 7}
    for i in range(4):
        cols[f"k{i}"] = rng.integers(-1, 2, n)
    cols["x"] = rng.integers(-1_000_000, 1_000_001, n)
    cols["seq"] = np.arange(n)
    return {c: v.astype(np.int64) for c, v in cols.items()}


def sqlite_values(cols, keyed, order_by, function):
    """seq -> the function's value as SQLite computes it."""
    db = sqlite3.connect(":memory:")
    names = list(cols)
    columns = ", ".join(f'"{c}" INTEGER' for c in names)
    db.execute(f"CREATE TABLE t ({columns})")
    db.executemany(f"INSERT INTO t VALUES ({', '.join('?' * len(names))})",
                   zip(*[[int(v) for v in cols[c]] for c in names]))
    call = "COUNT(*)" if function == "count" else f"{function.upper()}(x)"
    part = f'"{TS}"' + (", p" if keyed else "")
    order = ", ".join(f"{c} {'DESC' if d else 'ASC'}" for c, d in order_by)
    over = f"PARTITION BY {part}" + (f" ORDER BY {order}" if order else "")
    got = dict(db.execute(f"SELECT seq, {call} OVER ({over}) FROM t"))
    db.close()
    return got


@pytest.mark.parametrize("n_order", sorted(ORDER_SETS))
@pytest.mark.parametrize("keyed", [True, False], ids=["keyed", "unkeyed"])
def test_aggregates_match_sqlite(keyed, n_order):
    cols = random_batch(100 * n_order + keyed)
    order_by = ORDER_SETS[n_order]
    for function in AGGREGATES:
        out, late, _ = window_agg_emissions([("batch", cols), ("wm", INT64_MAX)], "p" if keyed else None, order_by,
                                            function, "x", "f")
        assert late == 0 and len(out) == 1 and len(out[0]) == len(cols[TS])
        want = sqlite_values(cols, keyed, order_by, function)
        for r in out[0]:
            w = want[r["seq"]]
            if function == "avg":
                assert isinstance(r["f"], float)
                assert math.isclose(r["f"], w, rel_tol=1e-12), (function, r, w)
            else:
                assert isinstance(r["f"], int) and r["f"] == w, (function, r, w)


def test_output_order_and_frames():
    """Rows leave sorted as the ranking functions sort them; peers share the frame end, segments restart it."""
    rows = [{TS: 5, "k": 1, "v": v, "seq": i} for i, v in enumerate([3, 1, 3, 2])] + [{TS: 5, "k": 0, "v": 9, "seq": 4}]
    got = aggregate_rows(rows, "k", [("v", True)], "sum", "v", "s")
    assert [(r["seq"], r["s"]) for r in got] == [(4, 9), (0, 6), (2, 6), (3, 8), (1, 9)]
    whole = aggregate_rows(rows, "k", [], "sum", "v", "s")
    assert [(r["seq"], r["s"]) for r in whole] == [(4, 9), (0, 9), (1, 9), (2, 9), (3, 9)]
    assert [r["a"] for r in aggregate_rows(rows, None, [("v", False)], "avg", "v", "a")] == [1.0, 1.5, 2.25, 2.25, 3.6]


@pytest.mark.parametrize("ties", [False, True], ids=["unique", "ties"])
def test_wrapping_sum_matches_numpy_cumsum(ties):
    """SUM near +-2^63 wraps modulo 2^64: numpy's int64 cumsum, read at each peer group's last index."""
    rng = np.random.default_rng(11 + ties)
    n = 2000
    big = np.array([INT64_MAX, -INT64_MAX - 1, INT64_MAX - 5, -(1 << 62), 1 << 62, -1, 0, 3], dtype=np.int64)
    x = rng.choice(big, n)
    k = rng.integers(0, 40, n) if ties else rng.permutation(n)
    cols = {"k": k.astype(np.int64), "x": x, TS: np.full(n, 9, np.int64)}
    out, _, _ = window_agg_emissions([("batch", cols), ("wm", INT64_MAX)], None, [("k", False)], "sum", "x", "s")
    order = np.lexsort((np.arange(n), cols["k"]))
    with np.errstate(over="ignore"):
        cs = np.cumsum(x[order])
    sk = cols["k"][order]
    last = np.r_[sk[1:] != sk[:-1], True]
    group_end = np.flip(np.minimum.accumulate(np.flip(np.where(last, np.arange(n), n))))
    want = cs[group_end]
    assert [r["s"] for r in out[0]] == [int(v) for v in want]
    assert [r["x"] for r in out[0]] == [int(v) for v in x[order]]
    assert any(abs(int(v)) > 1 << 62 for v in want)
    # the whole frame without ORDER BY: the total, wrapped
    whole, _, _ = window_agg_emissions([("batch", cols), ("wm", INT64_MAX)], None, [], "sum", "x", "s")
    assert {r["s"] for r in whole[0]} == {int(cs[-1])}
