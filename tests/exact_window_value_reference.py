"""An exact statement of the window function operator's value and distribution functions, LAG / LEAD / FIRST_VALUE /
LAST_VALUE / NTH_VALUE (x, ...) and PERCENT_RANK / CUME_DIST () OVER (PARTITION BY window [, key] [ORDER BY ...]) with
DataFusion 48's defaults, row by row in plain Python.  Rows, late rows, watermarks, restarts and the output order are
those of the ranking functions (tests/exact_window_fn_reference.py, which this builds on); what differs is the value
appended under `name`.  For row j of a segment (instant, partition key) spanning sorted rows [s, e], with f the last
row of j's peer group (peers tie on every ORDER BY key; without ORDER BY every row of the segment is a peer):

* LAG(x, k, d): x at j - k if j - k >= s, else d (None, i.e. NULL, without a default); LEAD(x, k, d): x at j + k if
  j + k <= e, else d.  Both ignore the frame;
* FIRST_VALUE(x): x at s; LAST_VALUE(x): x at f, the default frame's end;
* NTH_VALUE(x, n): x at s + n - 1 if that row is at or before f, else None;
* PERCENT_RANK(): (rank - 1) / (rows - 1) as a float, 0.0 for a 1-row segment;
* CUME_DIST(): (rows up to f) / rows, a float;
* every row leaves (no fused filter).

k and n are literals, k >= 0 and n >= 1.  The value functions only move x: the tests pass Float64 arguments as their
64-bit patterns.  NTILE, negative offsets, IGNORE NULLS and explicit frames are not stated here: those stay on the stock
operator."""
from typing import List, Optional, Sequence, Tuple

from tests.exact_window_fn_reference import TS, rank_rows, window_fn_emissions

VALUES = ("lag", "lead", "first_value", "last_value", "nth_value")
DISTRIBUTIONS = ("percent_rank", "cume_dist")
FUNCTIONS = VALUES + DISTRIBUTIONS
NULLABLE = ("lag", "lead", "nth_value")
_ORDER = "__arrival_rank"  # the ranking reference's ROW_NUMBER: only its sort is used


def values_sorted(ordered: List[dict], partition_by: Optional[str], order_by: Sequence[Tuple[str, bool]],
                  function: str, argument: Optional[str], name: str, offset: int = 1, default=None) -> List[dict]:
    """Rows already sorted by (instant, partition key, ORDER BY keys, arrival), each with `function` under `name`.
    `offset` is LAG / LEAD's k or NTH_VALUE's n; `default` LAG / LEAD's default (None: NULL)."""
    assert function in FUNCTIONS, function
    assert offset >= (1 if function == "nth_value" else 0), offset

    def segment(r):
        return r[TS], r[partition_by] if partition_by else None

    out, s = [], 0
    while s < len(ordered):
        e = s
        while e + 1 < len(ordered) and segment(ordered[e + 1]) == segment(ordered[s]):
            e += 1
        rows = ordered[s:e + 1]
        n = len(rows)
        first, last = [0] * n, [0] * n  # per row: its peer group's first and last index in the segment
        a = 0
        while a < n:
            b = a
            while b + 1 < n and all(rows[b + 1][c] == rows[a][c] for c, _ in order_by):
                b += 1
            for t in range(a, b + 1):
                first[t], last[t] = a, b
            a = b + 1
        for t, r in enumerate(rows):
            if function == "lag":
                v = rows[t - offset][argument] if t - offset >= 0 else default
            elif function == "lead":
                v = rows[t + offset][argument] if t + offset <= n - 1 else default
            elif function == "first_value":
                v = rows[0][argument]
            elif function == "last_value":
                v = rows[last[t]][argument]
            elif function == "nth_value":
                v = rows[offset - 1][argument] if offset - 1 <= last[t] else None
            elif function == "percent_rank":
                v = 0.0 if n == 1 else first[t] / (n - 1)
            else:
                v = (last[t] + 1) / n
            out.append({**r, name: v})
        s = e + 1
    return out


def _strip(rows: List[dict]) -> List[dict]:
    return [{c: v for c, v in r.items() if c != _ORDER} for r in rows]


def value_rows(rows: List[dict], partition_by: Optional[str], order_by: Sequence[Tuple[str, bool]], function: str,
               argument: Optional[str], name: str, offset: int = 1, default=None) -> List[dict]:
    """The rows of one emission (in arrival order) sorted as the ranking functions sort them, each with its value."""
    ordered = _strip(rank_rows(rows, partition_by, order_by, "row_number", _ORDER))
    return values_sorted(ordered, partition_by, order_by, function, argument, name, offset, default)


def window_value_emissions(events, partition_by: Optional[str], order_by: Sequence[Tuple[str, bool]], function: str,
                           argument: Optional[str], name: str = "fn", offset: int = 1, default=None):
    """window_fn_emissions for a value or distribution function: runs `events` ("batch", ("wm", w), ("restart",)) and
    returns (per watermark the rows it emits, in order; the number of late rows; per restart the table "input" it
    writes)."""
    out, late, states = window_fn_emissions(events, partition_by, order_by, "row_number", _ORDER)
    return [values_sorted(_strip(rows), partition_by, order_by, function, argument, name, offset, default)
            for rows in out], late, states
