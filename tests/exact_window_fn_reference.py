"""An exact statement of the window function operator (WindowFunctionOperator, arroyo-worker/src/arrow/window_fn.rs),
row by row in plain Python, for the tests to compare the CUDA operator and the numpy oracle's pipelines against:

* rows are bucketed by `_timestamp` ("instant"): each upstream window stamps all its rows with one timestamp, so the
  planner drops `window` from PARTITION BY (plan/window_fn.rs:101-105); the remaining PARTITION BY column, if any,
  splits each instant into segments;
* a row is late, and dropped, iff `_timestamp < w` for the last watermark w before its batch (filter_by_time keeps
  ts >= w, arroyo-rpc/src/df.rs:211-231); before the first watermark nothing is late;
* watermark w releases every instant < w, in ascending order (window_fn.rs:178-201).  Within an instant the rows are
  ordered by the partition key (ascending), then the ORDER BY keys; rows that tie on every key keep their arrival order
  (DataFusion's sort promises none; the CUDA operator keeps this one);
* ROW_NUMBER is the position in the segment + 1, RANK the position of the row's first peer + 1 (peers tie on every
  ORDER BY key), DENSE_RANK the number of distinct peer groups up to the row's; the value is appended as the last
  column.  A fused `WHERE fn <= top_n` (top_n > 0) is applied last;
* a restart (checkpoint, new operator, on_start with table "input") changes nothing: the table holds, per open instant,
  the rows since the previous checkpoint in arrival order, and the restored rows come back ahead of every later row.

Column values are compared as Python ints of the given numpy arrays: an Int64 or timestamp column orders as signed, a
UInt64 column as unsigned."""
from typing import Dict, List, Optional, Sequence, Tuple

TS = "_timestamp"
INT64_MAX = (1 << 63) - 1


def rank_rows(rows: List[dict], partition_by: Optional[str], order_by: Sequence[Tuple[str, bool]], function: str,
              name: str, top_n: int = 0) -> List[dict]:
    """The rows of one emission (already in arrival order) sorted by (instant, partition key, ORDER BY keys, arrival),
    each with its function value under `name`, then filtered by `<= top_n` when top_n > 0."""
    def sort_key(ir):
        i, r = ir
        k = [r[TS], r[partition_by] if partition_by else 0]
        k += [-r[c] if desc else r[c] for c, desc in order_by]
        return k + [i]

    ordered = [r for _, r in sorted(enumerate(rows), key=sort_key)]
    out, seg, prev = [], None, None
    pos = first_peer = dense = 0
    for r in ordered:
        s = (r[TS], r[partition_by] if partition_by else None)
        peers = tuple(r[c] for c, _ in order_by)
        if s != seg:
            seg, pos, first_peer, dense, prev = s, 0, 0, 0, None
        if peers != prev:
            first_peer, dense, prev = pos, dense + 1, peers
        value = {"row_number": pos + 1, "rank": first_peer + 1, "dense_rank": dense}[function]
        pos += 1
        if top_n == 0 or value <= top_n:
            out.append({**r, name: value})
    return out


def window_fn_emissions(events, partition_by: Optional[str], order_by: Sequence[Tuple[str, bool]], function: str,
                        name: str = "fn", top_n: int = 0):
    """Runs `events`: ("batch", {column: array}), ("wm", w) and ("restart",).  Watermarks must not decrease; end of
    data is INT64_MAX.  Returns (per watermark the rows it emits, in order; the number of late rows; per restart the
    table "input" it writes: {instant: rows since the previous checkpoint, in arrival order})."""
    open_rows: List[dict] = []
    fresh: List[dict] = []  # rows accepted since the last checkpoint that are still open
    last_wm, late, out, states = None, 0, [], []
    for ev in events:
        if ev[0] == "restart":
            state: Dict[int, List[dict]] = {}
            for r in fresh:
                state.setdefault(r[TS], []).append(r)
            states.append(state)
            fresh = []
            continue
        if ev[0] == "batch":
            cols = ev[1]
            names = list(cols)
            n = len(cols[TS])
            for i in range(n):
                r = {c: int(cols[c][i]) for c in names}
                if last_wm is not None and r[TS] < last_wm:
                    late += 1
                    continue
                open_rows.append(r)
                fresh.append(r)
            continue
        w = min(int(ev[1]), INT64_MAX)
        assert last_wm is None or w >= last_wm, "watermarks must not decrease"
        last_wm = w
        leaving = [r for r in open_rows if r[TS] < w]
        open_rows = [r for r in open_rows if r[TS] >= w]
        fresh = [r for r in fresh if r[TS] >= w]
        out.append(rank_rows(leaving, partition_by, order_by, function, name, top_n))
    return out, late, states
