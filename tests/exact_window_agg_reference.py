"""An exact statement of the window function operator's aggregates, COUNT(*) / SUM / AVG / MIN / MAX (x) OVER
(PARTITION BY window [, key] [ORDER BY ...]) with DataFusion 48's default frames, row by row in plain Python.  Rows,
late rows, watermarks, restarts and the output order are those of the ranking functions
(tests/exact_window_fn_reference.py, which this builds on); what differs is the value appended under `name`:

* without ORDER BY the frame is the whole segment (instant, partition key): every row of a segment gets one value;
* with ORDER BY the frame is `RANGE BETWEEN UNBOUNDED PRECEDING AND CURRENT ROW`: from the segment start through the
  row's last peer (peers tie on every ORDER BY key, as for RANK);
* count, sum and min / max are Int64, sum wrapping modulo 2^64; avg is Float64, each value cast to f64 and summed in
  sorted order, then divided by the frame's row count;
* every row leaves (no fused filter).

An explicit frame, DISTINCT, FILTER or IGNORE NULLS are not stated here: those stay on the stock operator."""
from typing import List, Optional, Sequence, Tuple

from tests.exact_window_fn_reference import TS, rank_rows, window_fn_emissions

AGGREGATES = ("count", "sum", "avg", "min", "max")
_ORDER = "__arrival_rank"  # the ranking reference's ROW_NUMBER: only its sort is used


def wrap64(v: int) -> int:
    return ((v + (1 << 63)) % (1 << 64)) - (1 << 63)


def aggregate_sorted(ordered: List[dict], partition_by: Optional[str], order_by: Sequence[Tuple[str, bool]],
                     function: str, argument: Optional[str], name: str) -> List[dict]:
    """Rows already sorted by (instant, partition key, ORDER BY keys, arrival), each with the aggregate `function` of
    `argument` (count: ignored) over its frame under `name`."""
    assert function in AGGREGATES, function

    def segment(r):
        return r[TS], r[partition_by] if partition_by else None

    out, i = [], 0
    while i < len(ordered):
        seg = segment(ordered[i])
        n, total, fsum, lo, hi = 0, 0, 0.0, None, None
        while i < len(ordered) and segment(ordered[i]) == seg:
            # one peer group: every row of the segment without ORDER BY
            peers = tuple(ordered[i][c] for c, _ in order_by)
            j = i
            while j < len(ordered) and segment(ordered[j]) == seg and tuple(ordered[j][c] for c, _ in order_by) == peers:
                j += 1
            for r in ordered[i:j]:
                x = r[argument] if function != "count" else 0
                n += 1
                total = wrap64(total + x)
                fsum += float(x)
                lo = x if lo is None else min(lo, x)
                hi = x if hi is None else max(hi, x)
            value = {"count": n, "sum": total, "avg": fsum / n, "min": lo, "max": hi}[function]
            out += [{**r, name: value} for r in ordered[i:j]]
            i = j
    return out


def _strip(rows: List[dict]) -> List[dict]:
    return [{c: v for c, v in r.items() if c != _ORDER} for r in rows]


def aggregate_rows(rows: List[dict], partition_by: Optional[str], order_by: Sequence[Tuple[str, bool]], function: str,
                   argument: Optional[str], name: str) -> List[dict]:
    """The rows of one emission (in arrival order) sorted as the ranking functions sort them, each with its value."""
    ordered = _strip(rank_rows(rows, partition_by, order_by, "row_number", _ORDER))
    return aggregate_sorted(ordered, partition_by, order_by, function, argument, name)


def window_agg_emissions(events, partition_by: Optional[str], order_by: Sequence[Tuple[str, bool]], function: str,
                         argument: Optional[str], name: str = "fn"):
    """window_fn_emissions for an aggregate: runs `events` ("batch", ("wm", w), ("restart",)) and returns (per watermark
    the rows it emits, in order; the number of late rows; per restart the table "input" it writes)."""
    out, late, states = window_fn_emissions(events, partition_by, order_by, "row_number", _ORDER)
    return [aggregate_sorted(_strip(rows), partition_by, order_by, function, argument, name) for rows in out], late, states
