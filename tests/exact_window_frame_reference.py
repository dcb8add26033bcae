"""An exact statement of the window function operator's explicit frames: COUNT(*) / SUM / AVG / MIN / MAX (x) and
FIRST_VALUE / LAST_VALUE / NTH_VALUE (x, n) OVER (PARTITION BY window [, key] [ORDER BY ...] {ROWS | RANGE | GROUPS}
BETWEEN start AND end), row by row in plain Python.  Rows, late rows, watermarks, restarts and the output order are
those of the ranking functions (tests/exact_window_fn_reference.py, which this builds on); what differs is the value
appended under `name`.

A frame is (units, start, end): units "rows", "range" or "groups"; each bound "unbounded_preceding", "current_row",
"unbounded_following", or ("preceding" | "following", n) with n >= 0.  Every row t of row j's segment has a coordinate
and the frame is the rows whose coordinate lies in [A, B], in exact integers (no bound saturates or wraps):

* ROWS: t's position; n PRECEDING / CURRENT ROW / n FOLLOWING stand for j - n / j / j + n;
* GROUPS, and RANGE's CURRENT ROW: t's peer group ordinal (peers tie on every ORDER BY key); the bounds stand for
  j's ordinal - n / + 0 / + n;
* RANGE with an offset (exactly one ORDER BY key x): x, negated under DESC so that it ascends in sort order; the bounds
  stand for that value of j - n / + n.  So under DESC "n PRECEDING" takes keys up to x(j) + n;
* UNBOUNDED PRECEDING / FOLLOWING: no limit.

A start gives A and an end gives B.  The frame is contiguous in sort order, [lo, hi); it is empty when no row lies in
[A, B].  Over it: count = its rows; sum wraps modulo 2^64; avg is the exact sum over the count, correctly rounded to a
float; min / max the extremes; first_value / last_value x at lo / hi - 1; nth_value x at lo + n - 1 if that is in the
frame.  An empty frame gives count 0 and None (NULL) for every other function.  The value functions only move x: the
tests pass Float64 arguments as their 64-bit patterns."""
from bisect import bisect_left, bisect_right
from fractions import Fraction
from typing import List, Optional, Sequence, Tuple

from tests.exact_window_agg_reference import wrap64
from tests.exact_window_fn_reference import TS, rank_rows, window_fn_emissions

FUNCTIONS = ("count", "sum", "avg", "min", "max", "first_value", "last_value", "nth_value")
_ORDER = "__arrival_rank"  # the ranking reference's ROW_NUMBER: only its sort is used


def bound(b) -> Tuple[str, int]:
    """A bound as (kind, n); n is 0 for the bounds without an offset."""
    return (b, 0) if isinstance(b, str) else (b[0], int(b[1]))


def _unpack(frame):
    return frame if isinstance(frame, tuple) else (frame.units, frame.start, frame.end)


def segment_frames(rows: List[dict], order_by: Sequence[Tuple[str, bool]], frame) -> List[Tuple[int, int]]:
    """Per row of one sorted segment its frame [lo, hi), as indices into the segment (lo >= hi: empty)."""
    units, start, end = _unpack(frame)
    (sk, sn), (ek, en) = bound(start), bound(end)
    n = len(rows)
    groups, g = [], -1
    for t, r in enumerate(rows):
        if t == 0 or any(r[c] != rows[t - 1][c] for c, _ in order_by):
            g += 1
        groups.append(g)
    offsets = units == "range" and (sk in ("preceding", "following") or ek in ("preceding", "following"))
    if offsets:
        assert len(order_by) == 1, "RANGE with an offset takes exactly one ORDER BY key"
        c, desc = order_by[0]
        coord = [-r[c] if desc else r[c] for r in rows]
    elif units == "rows":
        coord = list(range(n))
    else:
        coord = groups
    out = []
    for j in range(n):
        def limit(kind, k):
            return coord[j] - k if kind == "preceding" else coord[j] + k if kind == "following" else coord[j]
        lo = 0 if sk == "unbounded_preceding" else bisect_left(coord, limit(sk, sn))
        hi = n if ek == "unbounded_following" else bisect_right(coord, limit(ek, en))
        out.append((lo, hi))
    return out


def frame_value(xs: List[int], lo: int, hi: int, function: str, offset: int = 1):
    """`function` over xs[lo:hi] (None: NULL)."""
    if hi <= lo:
        return 0 if function == "count" else None
    if function == "count":
        return hi - lo
    if function == "sum":
        return wrap64(sum(xs[lo:hi]))
    if function == "avg":
        return float(Fraction(sum(xs[lo:hi]), hi - lo))
    if function == "min":
        return min(xs[lo:hi])
    if function == "max":
        return max(xs[lo:hi])
    if function == "first_value":
        return xs[lo]
    if function == "last_value":
        return xs[hi - 1]
    assert function == "nth_value" and offset >= 1, (function, offset)
    return xs[lo + offset - 1] if lo + offset - 1 < hi else None


def frame_sorted(ordered: List[dict], partition_by: Optional[str], order_by: Sequence[Tuple[str, bool]],
                 function: str, argument: Optional[str], name: str, frame, offset: int = 1) -> List[dict]:
    """Rows already sorted by (instant, partition key, ORDER BY keys, arrival), each with `function` of `argument`
    (count: ignored) over its frame under `name`.  `offset` is NTH_VALUE's n."""
    assert function in FUNCTIONS, function

    def segment(r):
        return r[TS], r[partition_by] if partition_by else None

    out, s = [], 0
    while s < len(ordered):
        e = s
        while e + 1 < len(ordered) and segment(ordered[e + 1]) == segment(ordered[s]):
            e += 1
        rows = ordered[s:e + 1]
        xs = [r[argument] if function != "count" else 0 for r in rows]
        for r, (lo, hi) in zip(rows, segment_frames(rows, order_by, frame)):
            out.append({**r, name: frame_value(xs, lo, hi, function, offset)})
        s = e + 1
    return out


def _strip(rows: List[dict]) -> List[dict]:
    return [{c: v for c, v in r.items() if c != _ORDER} for r in rows]


def frame_rows(rows: List[dict], partition_by: Optional[str], order_by: Sequence[Tuple[str, bool]], function: str,
               argument: Optional[str], name: str, frame, offset: int = 1) -> List[dict]:
    """The rows of one emission (in arrival order) sorted as the ranking functions sort them, each with its value."""
    ordered = _strip(rank_rows(rows, partition_by, order_by, "row_number", _ORDER))
    return frame_sorted(ordered, partition_by, order_by, function, argument, name, frame, offset)


def window_frame_emissions(events, partition_by: Optional[str], order_by: Sequence[Tuple[str, bool]], function: str,
                           argument: Optional[str], frame, name: str = "fn", offset: int = 1):
    """window_fn_emissions for a function over an explicit frame: runs `events` ("batch", ("wm", w), ("restart",)) and
    returns (per watermark the rows it emits, in order; the number of late rows; per restart the table "input" it
    writes)."""
    out, late, states = window_fn_emissions(events, partition_by, order_by, "row_number", _ORDER)
    return [frame_sorted(_strip(rows), partition_by, order_by, function, argument, name, frame, offset)
            for rows in out], late, states
