"""Pins the exact reference's value and distribution window functions (tests/exact_window_value_reference.py: LAG /
LEAD / FIRST_VALUE / LAST_VALUE / NTH_VALUE and PERCENT_RANK / CUME_DIST OVER (PARTITION BY window [, key] [ORDER BY
...])) to an independent engine, SQLite's window functions, which take the same default frames: the whole partition
without ORDER BY, `RANGE BETWEEN UNBOUNDED PRECEDING AND CURRENT ROW` with it.

SQLite orders the rows of a peer group in no stated way, and the reference by arrival.  So the value functions are
compared row by row on orders that a unique last ORDER BY key makes tie-free, and on heavy-tie orders with an argument
that is constant within each peer group, as multisets per (segment, peer group).  PERCENT_RANK and CUME_DIST do not
depend on the order within a peer group: they are compared row by row, bit for bit, on heavy ties."""
import sqlite3
import struct
from collections import Counter

import numpy as np
import pytest

from tests.exact_window_fn_reference import INT64_MAX, TS
from tests.exact_window_value_reference import DISTRIBUTIONS, value_rows, window_value_emissions

TIE_ORDERS = {0: [], 1: [("k0", True)], 2: [("k0", False), ("k1", True)],
              4: [("k0", True), ("k1", False), ("k2", True), ("k3", False)]}
UNIQUE_ORDERS = {1: [("seq", True)], 2: [("k0", False), ("seq", True)],
                 4: [("k0", True), ("k1", False), ("k2", True), ("seq", False)]}
BIG = 1_000_000  # larger than any segment
CALLS = ([("lag", k, d) for k in (0, 1, 3, BIG) for d in (None, -7)] +
         [("lead", k, d) for k in (0, 1, 3, BIG) for d in (None, -7)] +
         [("first_value", 1, None), ("last_value", 1, None)] + [("nth_value", n, None) for n in (1, 2, BIG)])


def random_batch(seed, n=3000):
    """Rows with heavy ties: 6 instants, 4 partition keys, ORDER BY keys from 3 values, a unique `seq`, an argument
    `x`."""
    rng = np.random.default_rng(seed)
    cols = {"p": rng.integers(0, 4, n), TS: rng.integers(0, 6, n) * 1000 + 7}
    for i in range(4):
        cols[f"k{i}"] = rng.integers(-1, 2, n)
    cols["x"] = rng.integers(-1_000_000, 1_000_001, n)
    cols["seq"] = np.arange(n)
    return {c: v.astype(np.int64) for c, v in cols.items()}


def sql_call(function, offset, default, argument):
    if function in ("lag", "lead"):
        return f"{function.upper()}({argument}, {offset}" + ("" if default is None else f", {default}") + ")"
    if function == "nth_value":
        return f"NTH_VALUE({argument}, {offset})"
    if function in DISTRIBUTIONS:
        return f"{function.upper()}()"
    return f"{function.upper()}({argument})"


def sqlite_values(cols, keyed, order_by, call):
    """seq -> the value of SQL window function `call` as SQLite computes it."""
    db = sqlite3.connect(":memory:")
    names = list(cols)
    db.execute(f"CREATE TABLE t ({', '.join(f'{chr(34)}{c}{chr(34)} INTEGER' for c in names)})")
    db.executemany(f"INSERT INTO t VALUES ({', '.join('?' * len(names))})",
                   zip(*[[int(v) for v in cols[c]] for c in names]))
    part = f'"{TS}"' + (", p" if keyed else "")
    order = ", ".join(f"{c} {'DESC' if d else 'ASC'}" for c, d in order_by)
    over = f"PARTITION BY {part}" + (f" ORDER BY {order}" if order else "")
    got = dict(db.execute(f"SELECT seq, {call} OVER ({over}) FROM t"))
    db.close()
    return got


def reference(cols, keyed, order_by, function, argument, offset=1, default=None):
    out, late, _ = window_value_emissions([("batch", cols), ("wm", INT64_MAX)], "p" if keyed else None, order_by,
                                          function, argument, "f", offset, default)
    assert late == 0 and len(out) == 1 and len(out[0]) == len(cols[TS])
    return out[0]


def bits(v):
    return struct.pack("<d", v)


@pytest.mark.parametrize("n_order", sorted(UNIQUE_ORDERS))
@pytest.mark.parametrize("keyed", [True, False], ids=["keyed", "unkeyed"])
def test_values_match_sqlite_row_by_row(keyed, n_order):
    cols = random_batch(300 + 10 * n_order + keyed)
    order_by = UNIQUE_ORDERS[n_order]
    for function, offset, default in CALLS:
        got = reference(cols, keyed, order_by, function, "x", offset, default)
        want = sqlite_values(cols, keyed, order_by, sql_call(function, offset, default, "x"))
        for r in got:
            assert r["f"] == want[r["seq"]], (function, offset, default, r, want[r["seq"]])
        assert any(r["f"] is not None for r in got) == (offset < BIG or default is not None)
        if function in ("lag", "lead") and offset > 0:
            assert any(r["f"] == (-7 if default is not None else None) for r in got)


@pytest.mark.parametrize("n_order", sorted(TIE_ORDERS))
@pytest.mark.parametrize("keyed", [True, False], ids=["keyed", "unkeyed"])
def test_distributions_match_sqlite_bit_for_bit_on_ties(keyed, n_order):
    cols = random_batch(500 + 10 * n_order + keyed)
    order_by = TIE_ORDERS[n_order]
    for function in DISTRIBUTIONS:
        got = reference(cols, keyed, order_by, function, None)
        want = sqlite_values(cols, keyed, order_by, sql_call(function, 1, None, None))
        for r in got:
            assert isinstance(r["f"], float) and bits(r["f"]) == bits(want[r["seq"]]), (function, r, want[r["seq"]])
        if n_order == 0:
            assert {r["f"] for r in got} == {0.0 if function == "percent_rank" else 1.0}


@pytest.mark.parametrize("n_order", sorted(TIE_ORDERS))
@pytest.mark.parametrize("keyed", [True, False], ids=["keyed", "unkeyed"])
def test_values_match_sqlite_per_peer_group_on_ties(keyed, n_order):
    """An argument `g` constant within each (segment, peer group): each group's multiset of values does not depend on
    the order of its rows."""
    cols = random_batch(700 + 10 * n_order + keyed)
    order_by = TIE_ORDERS[n_order]
    n = len(cols[TS])

    def group(i):
        return (int(cols[TS][i]), int(cols["p"][i]) if keyed else 0) + tuple(int(cols[c][i]) for c, _ in order_by)

    cols["g"] = np.array([hash(group(i)) % 1_000_003 for i in range(n)], dtype=np.int64)
    for function, offset, default in CALLS:
        got = reference(cols, keyed, order_by, function, "g", offset, default)
        want = sqlite_values(cols, keyed, order_by, sql_call(function, offset, default, "g"))
        got_groups, want_groups = {}, {}
        for r in got:
            got_groups.setdefault(group(r["seq"]), Counter())[r["f"]] += 1
        for seq, v in want.items():
            want_groups.setdefault(group(seq), Counter())[v] += 1
        assert got_groups == want_groups, (function, offset, default)


def test_frames_by_hand():
    """One segment of 5 rows ORDER BY v DESC, a second segment of 1 row: the rules of the module docstring."""
    rows = [{TS: 5, "k": 1, "v": v, "x": 10 * i, "seq": i} for i, v in enumerate([3, 1, 3, 2, 2])]
    rows.append({TS: 5, "k": 0, "v": 9, "x": 99, "seq": 5})
    order = [("v", True)]

    def run(function, offset=1, default=None):
        return [(r["seq"], r["f"]) for r in value_rows(rows, "k", order, function, "x", "f", offset, default)]

    # sorted: seq 5 | seq 0, 2 (v 3), 3, 4 (v 2), 1 (v 1)
    assert run("lag") == [(5, None), (0, None), (2, 0), (3, 20), (4, 30), (1, 40)]
    assert run("lag", 0) == [(5, 99), (0, 0), (2, 20), (3, 30), (4, 40), (1, 10)]
    assert run("lead", 2, -1) == [(5, -1), (0, 30), (2, 40), (3, 10), (4, -1), (1, -1)]
    assert run("first_value") == [(5, 99), (0, 0), (2, 0), (3, 0), (4, 0), (1, 0)]
    assert run("last_value") == [(5, 99), (0, 20), (2, 20), (3, 40), (4, 40), (1, 10)]
    assert run("nth_value", 3) == [(5, None), (0, None), (2, None), (3, 30), (4, 30), (1, 30)]
    assert run("percent_rank") == [(5, 0.0), (0, 0.0), (2, 0.0), (3, 0.5), (4, 0.5), (1, 1.0)]
    assert run("cume_dist") == [(5, 1.0), (0, 0.4), (2, 0.4), (3, 0.8), (4, 0.8), (1, 1.0)]
    whole = [(r["seq"], r["f"]) for r in value_rows(rows, "k", [], "last_value", "x", "f")]
    assert whole == [(5, 99), (0, 40), (1, 40), (2, 40), (3, 40), (4, 40)]


def test_emissions_follow_the_ranking_reference():
    """Late rows and watermarks come from the ranking reference: a late row never reaches LAG."""
    ev = [("batch", {TS: np.array([7, 7, 9], np.int64), "x": np.array([1, 2, 3], np.int64)}), ("wm", 8),
          ("batch", {TS: np.array([7, 9], np.int64), "x": np.array([4, 5], np.int64)}), ("wm", INT64_MAX)]
    out, late, _ = window_value_emissions(ev, None, [], "lag", "x", "f", 1, 0)
    assert late == 1
    assert [[(r[TS], r["x"], r["f"]) for r in rows] for rows in out] == [[(7, 1, 0), (7, 2, 1)],
                                                                          [(9, 3, 0), (9, 5, 3)]]
