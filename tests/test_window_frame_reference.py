"""Pins the exact reference's explicit frames (tests/exact_window_frame_reference.py: COUNT(*) / SUM / AVG / MIN / MAX
and FIRST_VALUE / LAST_VALUE / NTH_VALUE over ROWS / RANGE / GROUPS frames) to an independent engine, SQLite's window
functions, which run all three units with every bound, empty frames and DESC orders.

SQLite orders the rows of a peer group in no stated way, and the reference by arrival.  So ROWS frames and the value
functions are compared row by row on orders that a unique last ORDER BY key makes tie-free; the aggregates under RANGE
and GROUPS are compared row by row on heavy ties too, as those frames hold whole peer groups.  Arguments stay far from
+-2^63, where SQLite's SUM switches to REAL or fails: the edges are checked against hand-worked values instead."""
import itertools
import sqlite3

import numpy as np
import pytest

from tests.exact_window_agg_reference import aggregate_rows
from tests.exact_window_fn_reference import INT64_MAX, TS
from tests.exact_window_frame_reference import FUNCTIONS, frame_rows, segment_frames, window_frame_emissions
from tests.exact_window_value_reference import value_rows

INT64_MIN = -(1 << 63)
BIG = 1_000_000  # larger than any segment and any key distance here
AGGREGATES = ("count", "sum", "avg", "min", "max")
# every (start, end) shape SQLite and DataFusion accept; P / F take an offset
SHAPES = [("UP", "P"), ("UP", "CR"), ("UP", "F"), ("UP", "UF"), ("P", "P"), ("P", "CR"), ("P", "F"), ("P", "UF"),
          ("CR", "CR"), ("CR", "F"), ("CR", "UF"), ("F", "F"), ("F", "UF")]
REFUSED_SHAPES = [("F", "CR"), ("F", "P"), ("CR", "P")]  # a start after the end
OFFSET_PAIRS = [(0, 0), (1, 1), (2, 0), (1, 3), (3, 1), (0, 2), (BIG, 2), (2, BIG)]
_KINDS = {"UP": "unbounded_preceding", "P": "preceding", "CR": "current_row", "F": "following",
          "UF": "unbounded_following"}
TIE_FREE = [[("seq", False)], [("seq", True)], [("k", True), ("seq", False)]]
TIES = [[("k", False)], [("k", True)], [("k", True), ("k1", False)]]


def frames(units, one_key=True):
    """Every accepted frame of `units` (RANGE with offsets only when the order has one key)."""
    out = []
    for s, e in SHAPES:
        if units == "range" and not one_key and ("P" in (s, e) or "F" in (s, e)):
            continue
        n_offsets = (s in ("P", "F")) + (e in ("P", "F"))
        pairs = OFFSET_PAIRS if n_offsets == 2 else [(k, k) for k in (0, 1, 2, BIG)] if n_offsets else [(0, 0)]
        for a, b in pairs:
            start = (_KINDS[s], a) if s in ("P", "F") else _KINDS[s]
            end = (_KINDS[e], b) if e in ("P", "F") else _KINDS[e]
            out.append((units, start, end))
    return sorted(set(out), key=repr)


def sql_bound(b):
    if isinstance(b, str):
        return b.upper().replace("_", " ")
    return f"{b[1]} {b[0].upper()}"


def sql_frame(frame):
    units, start, end = frame
    return f"{units.upper()} BETWEEN {sql_bound(start)} AND {sql_bound(end)}"


def sql_call(function, argument, offset):
    if function == "count":
        return "COUNT(*)"
    if function == "nth_value":
        return f"NTH_VALUE({argument}, {offset})"
    return f"{function.upper()}({argument})"


def random_batch(seed, n=300):
    """Rows with heavy ties: 4 instants, 3 partition keys, ORDER BY keys k (20 values) and k1 (3 values), a unique
    `seq`, an argument `x`."""
    rng = np.random.default_rng(seed)
    cols = {"p": rng.integers(0, 3, n), TS: rng.integers(0, 4, n) * 1000 + 7, "k": rng.integers(-10, 10, n),
            "k1": rng.integers(-1, 2, n), "x": rng.integers(-1_000_000, 1_000_001, n), "seq": rng.permutation(n)}
    return {c: v.astype(np.int64) for c, v in cols.items()}


class SQLite:
    def __init__(self, cols):
        self.db = sqlite3.connect(":memory:")
        names = list(cols)
        self.db.execute(f"CREATE TABLE t ({', '.join(f'{chr(34)}{c}{chr(34)} INTEGER' for c in names)})")
        self.db.executemany(f"INSERT INTO t VALUES ({', '.join('?' * len(names))})",
                            zip(*[[int(v) for v in cols[c]] for c in names]))

    def values(self, keyed, order_by, call, frame):
        """seq -> `call` OVER (... frame) as SQLite computes it."""
        part = f'"{TS}"' + (", p" if keyed else "")
        order = ", ".join(f"{c} {'DESC' if d else 'ASC'}" for c, d in order_by)
        over = f"PARTITION BY {part}" + (f" ORDER BY {order}" if order else "") + " " + sql_frame(frame)
        return dict(self.db.execute(f"SELECT seq, {call} OVER ({over}) FROM t"))


def reference(cols, keyed, order_by, function, frame, offset=1):
    out, late, _ = window_frame_emissions([("batch", cols), ("wm", INT64_MAX)], "p" if keyed else None, order_by,
                                          function, "x", frame, "f", offset)
    assert late == 0 and len(out) == 1 and len(out[0]) == len(cols[TS])
    return out[0]


def check(db, cols, keyed, order_by, functions, frame):
    for function in functions:
        for offset in ((1, 2, BIG) if function == "nth_value" else (1,)):
            got = reference(cols, keyed, order_by, function, frame, offset)
            want = db.values(keyed, order_by, sql_call(function, "x", offset), frame)
            for r in got:
                w = want[r["seq"]]
                if function == "avg" and w is not None:
                    assert r["f"] == pytest.approx(w, rel=1e-12, abs=0), (frame, function, r, w)
                else:
                    assert r["f"] == w, (frame, function, offset, r, w)


@pytest.mark.parametrize("units", ["rows", "range", "groups"])
@pytest.mark.parametrize("order", range(len(TIE_FREE)))
@pytest.mark.parametrize("keyed", [True, False], ids=["keyed", "unkeyed"])
def test_tie_free_orders_match_sqlite_row_by_row(keyed, order, units):
    cols = random_batch(100 + 10 * order + keyed)
    order_by = TIE_FREE[order]
    db = SQLite(cols)
    for frame in frames(units, one_key=len(order_by) == 1):
        check(db, cols, keyed, order_by, FUNCTIONS, frame)


@pytest.mark.parametrize("units", ["range", "groups"])
@pytest.mark.parametrize("order", range(len(TIES)))
@pytest.mark.parametrize("keyed", [True, False], ids=["keyed", "unkeyed"])
def test_aggregates_on_heavy_ties_match_sqlite_row_by_row(keyed, order, units):
    cols = random_batch(300 + 10 * order + keyed)
    order_by = TIES[order]
    db = SQLite(cols)
    for frame in frames(units, one_key=len(order_by) == 1):
        check(db, cols, keyed, order_by, AGGREGATES, frame)


@pytest.mark.parametrize("keyed", [True, False], ids=["keyed", "unkeyed"])
def test_frames_without_order_by_match_sqlite(keyed):
    """Without ORDER BY every row of a segment is a peer: RANGE frames are the whole segment, ROWS frames follow the
    row order, which SQLite does not state, so only their aggregates over whole segments are compared."""
    cols = random_batch(500 + keyed)
    db = SQLite(cols)
    for frame in frames("range", one_key=False):
        check(db, cols, keyed, [], AGGREGATES, frame)
    check(db, cols, keyed, [], AGGREGATES, ("rows", "unbounded_preceding", "unbounded_following"))


def test_one_row_segments_and_empty_frames():
    """Every instant and key of its own: each frame holds the row or nothing."""
    n = 40
    cols = {"p": np.arange(n, dtype=np.int64), TS: np.full(n, 7, np.int64), "k": np.zeros(n, np.int64),
            "k1": np.zeros(n, np.int64), "x": np.arange(n, dtype=np.int64) * 3 - 50, "seq": np.arange(n, dtype=np.int64)}
    db = SQLite(cols)
    for units in ("rows", "range", "groups"):
        for frame in frames(units):
            check(db, cols, True, [("seq", True)], FUNCTIONS, frame)


def test_sqlite_refuses_what_the_operator_refuses():
    """A start after the end is refused by SQLite ("unsupported frame specification"), so nothing pins it and the
    operator refuses it as UNSUPPORTED; UNBOUNDED FOLLOWING as a start, UNBOUNDED PRECEDING as an end and RANGE with an
    offset over other than one ORDER BY key are refused by SQLite and DataFusion alike."""
    db = SQLite(random_batch(9, 20))
    refused = [("rows", (_KINDS[s], 1) if s in ("P", "F") else _KINDS[s], (_KINDS[e], 1) if e in ("P", "F") else _KINDS[e])
               for s, e in REFUSED_SHAPES]
    refused += [("rows", "unbounded_following", "unbounded_following"), ("rows", "unbounded_preceding",
                                                                          "unbounded_preceding")]
    for frame in refused:
        with pytest.raises(sqlite3.OperationalError):
            db.values(False, [("seq", False)], "SUM(x)", frame)
    for order_by in ([], [("k", False), ("seq", False)]):
        with pytest.raises(sqlite3.OperationalError, match="one ORDER BY"):
            db.values(False, order_by, "SUM(x)", ("range", ("preceding", 1), "current_row"))


def test_default_equivalent_frames_equal_the_default_frame_references():
    cols = random_batch(77)
    rows = [{c: int(v[i]) for c, v in cols.items()} for i in range(len(cols[TS]))]
    for order_by in ([("k", True)], [("k", False), ("k1", True)]):
        frame = ("range", "unbounded_preceding", "current_row")
        for function in AGGREGATES:
            want = aggregate_rows(rows, "p", order_by, function, "x", "f")
            got = frame_rows(rows, "p", order_by, function, "x", "f", frame)
            assert [r["f"] for r in got] == pytest.approx([r["f"] for r in want], rel=1e-12)
        for function in ("first_value", "last_value", "nth_value"):
            assert frame_rows(rows, "p", order_by, function, "x", "f", frame, 2) == \
                value_rows(rows, "p", order_by, function, "x", "f", 2)
    for units in ("rows", "range", "groups"):
        frame = (units, "unbounded_preceding", "unbounded_following")
        for function in AGGREGATES:
            want = aggregate_rows(rows, None, [], function, "x", "f")
            got = frame_rows(rows, None, [], function, "x", "f", frame)
            assert [r["f"] for r in got] == pytest.approx([r["f"] for r in want], rel=1e-12)
        for function in ("first_value", "last_value", "nth_value"):
            assert frame_rows(rows, None, [], function, "x", "f", frame, 3) == \
                value_rows(rows, None, [], function, "x", "f", 3)


@pytest.mark.parametrize("units", ["rows", "range", "groups"])
def test_frame_ends_never_decrease_within_a_segment(units):
    """The reference's lo and hi are non-decreasing in the row within a segment, for every accepted frame (the GPU's
    are checked in tests/test_gpu_window_frames.py)."""
    cols = random_batch(31, 200)
    rows = [{c: int(v[i]) for c, v in cols.items()} for i in range(len(cols[TS]))]
    for desc in (False, True):
        seg = sorted(rows, key=lambda r: (-r["k"] if desc else r["k"], r["seq"]))
        for frame in frames(units):
            bounds = segment_frames(seg, [("k", desc)], frame)
            for (a, b), (c, d) in zip(bounds, bounds[1:]):
                assert a <= c and b <= d, frame


def test_range_edges_by_hand():
    """RANGE bounds past a key type's range take everything up to the segment's edge: Int64 keys at INT64_MIN /
    INT64_MAX, UInt64 keys at 2^64 - 1, ASC and DESC."""
    def counts(keys, order_by, frame):
        rows = [{TS: 1, "k": k, "x": 1, "seq": i} for i, k in enumerate(keys)]
        return [r["f"] for r in frame_rows(rows, None, order_by, "count", "x", "f", frame)]

    keys = [INT64_MIN, -1, 0, INT64_MAX]
    back = ("range", ("preceding", INT64_MAX), "current_row")
    assert counts(keys, [("k", False)], back) == [1, 2, 2, 2]
    # DESC: "preceding" is the larger keys, up to x + n
    assert counts(keys, [("k", True)], back) == [1, 2, 2, 2]  # sorted MAX, 0, -1, MIN
    ahead = ("range", "current_row", ("following", INT64_MAX))
    assert counts(keys, [("k", False)], ahead) == [2, 2, 2, 1]
    unsigned = [0, 1 << 63, (1 << 64) - 2, (1 << 64) - 1]
    assert counts(unsigned, [("k", False)], ("range", ("preceding", 1), ("following", INT64_MAX))) == [1, 3, 2, 2]
    assert counts(unsigned, [("k", True)], ("range", ("following", 1), "unbounded_following")) == [3, 2, 1, 0]
    # a start FOLLOWING or an end PRECEDING past the range: empty, not the edge row
    assert counts(keys, [("k", False)], ("range", ("following", 1), ("following", INT64_MAX))) == [1, 1, 1, 0]
    assert counts(keys, [("k", False)], ("range", "unbounded_preceding", ("preceding", 1))) == [0, 1, 2, 3]
    assert counts(unsigned, [("k", False)], ("range", ("following", 1), "unbounded_following")) == [3, 2, 1, 0]
    # ROWS and GROUPS offsets up to INT64_MAX
    rows_max = ("rows", ("preceding", INT64_MAX), ("following", INT64_MAX))
    assert counts(keys, [("k", False)], rows_max) == [4, 4, 4, 4]
    assert counts(keys, [("k", False)], ("groups", ("following", INT64_MAX), "unbounded_following")) == [0, 0, 0, 0]


def test_sums_wrap_and_averages_are_exact_at_the_edges():
    rows = [{TS: 1, "x": x, "seq": i} for i, x in enumerate([INT64_MAX, INT64_MAX, 10 ** 18, 3, 4, INT64_MIN])]
    order = [("seq", False)]
    frame = ("rows", ("preceding", 1), "current_row")
    sums = [r["f"] for r in frame_rows(rows, None, order, "sum", "x", "f", frame)]
    assert sums == [INT64_MAX, -2, INT64_MAX + 10 ** 18 - (1 << 64), 10 ** 18 + 3, 7, INT64_MIN + 4]
    avgs = [r["f"] for r in frame_rows(rows, None, order, "avg", "x", "f", frame)]
    assert avgs == [float(INT64_MAX), float(INT64_MAX), (INT64_MAX + 10 ** 18) / 2, (10 ** 18 + 3) / 2, 3.5,
                    (INT64_MIN + 4) / 2]
    # one huge value ahead of a frame of small ones does not cancel into the small ones' average
    small = ("rows", ("preceding", 1), ("preceding", 0))
    assert [r["f"] for r in frame_rows(rows, None, order, "avg", "x", "f", small)][4] == 3.5


def test_emissions_follow_the_ranking_reference():
    """Late rows and watermarks come from the ranking reference: a late row never enters a frame."""
    ev = [("batch", {TS: np.array([7, 7, 9], np.int64), "x": np.array([1, 2, 3], np.int64)}), ("wm", 8),
          ("batch", {TS: np.array([7, 9], np.int64), "x": np.array([4, 5], np.int64)}), ("wm", INT64_MAX)]
    out, late, _ = window_frame_emissions(ev, None, [], "sum", "x", ("rows", ("preceding", 1), "current_row"))
    assert late == 1
    assert [[(r[TS], r["x"], r["fn"]) for r in rows] for rows in out] == [[(7, 1, 1), (7, 2, 3)],
                                                                          [(9, 3, 3), (9, 5, 8)]]


def test_frames_cover_every_accepted_shape():
    for units in ("rows", "range", "groups"):
        shapes = {(f[1] if isinstance(f[1], str) else f[1][0], f[2] if isinstance(f[2], str) else f[2][0])
                  for f in frames(units)}
        assert len(shapes) == len(SHAPES), units
    assert len(list(itertools.chain(*(frames(u) for u in ("rows", "range", "groups"))))) > 100
