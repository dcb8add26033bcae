"""CPU restatement of the reference's updating (non-windowed) aggregate -- TEST INFRASTRUCTURE ONLY.

SURVEY.md 8(f) rank 2: `IncrementalAggregatingFunc` (arroyo-worker/src/arrow/incremental_aggregator.rs), the operator
behind `SELECT ... GROUP BY` without a window.  No CUDA operator exists for it yet; this restatement and its golden pins
come first (tests/test_updating_oracle.py).  Nothing under arroyo_b200/ may import this module.

What the reference does (line numbers of incremental_aggregator.rs):
  * state per key = one accumulator per aggregate (:49-175).  Aggregates whose DataFusion sliding accumulator supports
    `retract_batch` are kept as that accumulator ("Sliding": count, sum, avg); the others ("Batch": count(distinct ...),
    and any aggregate without retraction) keep a multiset {argument value -> count} and are re-evaluated from the values
    whose count is positive (:151-172, constructor :1083-1098).
  * process_batch (:826-883 keyed, :775-824 global): for every key of the batch that was not touched since the last
    flush, remember the values it had (None for a new key, :842-857); then apply every row as an append or -- when the
    input is itself an updating stream and `_updating_meta.is_retract` is set -- a retraction (:873-880).
  * flush (:637-738; on every tick of `flush_interval`, at checkpoints and at end of data): for each touched key evaluate
    the aggregates; if it had values before, skip it when nothing but the timestamp changed (:655-664), else emit a
    retraction row with the old values (:666-671); emit an append row with the new values unless the key has no rows
    left -- the last aggregate, max(_timestamp), is then NULL -- in which case the key is dropped (:674-688).
    Keys idle for `ttl` are retracted and dropped (:690-704); wall-clock driven, not restated here.

PARITY: pinned on the merged change stream (the reference's tests merge the Debezium output per primary key before
comparing, smoke_tests.rs:519-562) by `grouped_aggregates`, `aggregates` and `debezium_agg`.  MIN / MAX under
retractions are unpinned: DataFusion's sliding min / max accumulators claim retract support but retract in FIFO order;
here they are kept as multisets (exact under any retraction order)."""
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np

from .arroyo_oracle import TIMESTAMP, Agg, Batch

IS_RETRACT = "_is_retract"


class UpdatingAggConfig:
    def __init__(self, key_names: Sequence[str], aggs: Sequence[Agg]):
        """`aggs`: Agg(kind, col, name) with kind in count | sum | avg | min | max | count_distinct."""
        self.key_names = list(key_names)
        self.aggs = list(aggs)


class _KeyState:
    __slots__ = ("rows", "sums", "fsums", "multi", "ts")

    def __init__(self, n_aggs):
        self.rows = 0                                # count(*) / avg denominator / "has rows"
        self.sums = [0] * n_aggs                     # wrapping int64 sums (sum)
        self.fsums = [0.0] * n_aggs                  # f64 sums in row order (avg: each value cast to f64, then added)
        self.multi: List[Dict[int, int]] = [dict() for _ in range(n_aggs)]  # value -> count (min, max, count_distinct)
        self.ts: Dict[int, int] = {}                 # multiset of _timestamp (the trailing max(_timestamp) aggregate)


def _wrap(x: int) -> int:
    x &= (1 << 64) - 1
    return x - (1 << 64) if x >= (1 << 63) else x


class IncrementalAggregatingFunc:
    """Output rows: keys, aggregates, _timestamp = max(_timestamp) of the key's live rows, IS_RETRACT."""

    def __init__(self, cfg: UpdatingAggConfig):
        self.cfg = cfg
        self.state: Dict[Tuple[int, ...], _KeyState] = {}
        self.updated: Dict[Tuple[int, ...], Optional[Tuple]] = {}  # key -> values before the first touch of this flush

    def name(self):
        return "UpdatingAggregatingFunc"

    # ---- evaluation (:151-172, :222-230) ----
    def _evaluate(self, st: _KeyState) -> Tuple:
        out = []
        for a, agg in enumerate(self.cfg.aggs):
            k = agg.kind
            if k == "count":
                out.append(st.rows)
            elif k == "sum":
                out.append(_wrap(st.sums[a]) if st.rows else None)
            elif k == "avg":
                out.append(st.fsums[a] / st.rows if st.rows else None)
            else:
                live = [v for v, c in st.multi[a].items() if c > 0]
                if k == "count_distinct":
                    out.append(len(live))
                elif k == "min":
                    out.append(min(live) if live else None)
                elif k == "max":
                    out.append(max(live) if live else None)
                else:
                    raise ValueError(k)
        live_ts = [t for t, c in st.ts.items() if c > 0]
        out.append(max(live_ts) if live_ts else None)
        return tuple(out)

    def process_batch(self, batch: Batch, ctx=None, collector=None):
        n = batch.num_rows
        keys = [tuple(int(batch[k][i]) for k in self.cfg.key_names) for i in range(n)]
        retract = batch.cols.get(IS_RETRACT)
        # values before this flush period's first touch (:842-857)
        for k in keys:
            if k not in self.updated:
                st = self.state.get(k)
                self.updated[k] = self._evaluate(st) if st is not None else None
        ts = batch[TIMESTAMP]
        for i, k in enumerate(keys):
            st = self.state.get(k)
            if st is None:
                st = self.state[k] = _KeyState(len(self.cfg.aggs))
            sign = -1 if (retract is not None and bool(retract[i])) else 1
            st.rows = max(st.rows + sign, 0)
            t = int(ts[i])
            st.ts[t] = st.ts.get(t, 0) + sign
            for a, agg in enumerate(self.cfg.aggs):
                if agg.kind == "sum":
                    st.sums[a] += sign * int(batch[agg.col][i])
                elif agg.kind == "avg":
                    st.fsums[a] += sign * float(int(batch[agg.col][i]))
                elif agg.kind in ("min", "max", "count_distinct"):
                    v = int(batch[agg.col][i])
                    c = st.multi[a].get(v)
                    if sign > 0:
                        st.multi[a][v] = (c or 0) + 1
                    elif c:                      # retracting a missing / already-zero value is ignored (:128-147)
                        st.multi[a][v] = c - 1

    def flush(self) -> Optional[Batch]:
        rows = []
        for k, before in self.updated.items():
            st = self.state[k]
            now = self._evaluate(st)
            if before is not None:
                if before[:-1] == now[:-1]:      # only the timestamp moved: nothing to say (:655-664)
                    if now[-1] is None:
                        del self.state[k]
                    continue
                rows.append((k, before, True))
            if now[-1] is not None:
                rows.append((k, now, False))
            else:
                del self.state[k]                # no rows left under this key (:685-688)
        self.updated = {}
        if not rows:
            return None
        cols: Dict[str, list] = {name: [] for name in self.cfg.key_names}
        for agg in self.cfg.aggs:
            cols[agg.name] = []
        cols[TIMESTAMP] = []
        cols[IS_RETRACT] = []
        for k, vals, r in rows:
            for name, kv in zip(self.cfg.key_names, k):
                cols[name].append(kv)
            for agg, v in zip(self.cfg.aggs, vals[:-1]):
                cols[agg.name].append(v)
            cols[TIMESTAMP].append(vals[-1])
            cols[IS_RETRACT].append(r)
        return Batch({c: np.array(v, dtype=object) for c, v in cols.items()})

    # the reference flushes on ticks, checkpoints and end of data; callers decide when
    handle_tick = handle_checkpoint = on_close = lambda self, *a, **k: self.flush()


def merge_change_stream(batches: Sequence[Optional[Batch]], key_names: Sequence[str]) -> List[dict]:
    """What the reference's test harness does with a Debezium sink before comparing (smoke_tests.rs:519-562):
    apply appends and retractions per primary key; the surviving rows are the result."""
    state: Dict[Tuple, dict] = {}
    for b in batches:
        if b is None:
            continue
        for r in b.rows():
            k = tuple(r[c] for c in key_names)
            if r[IS_RETRACT]:
                if k not in state:
                    raise AssertionError(f"retraction for a row that is not there: {r}")
                del state[k]
            else:
                state[k] = {c: v for c, v in r.items() if c not in (IS_RETRACT, TIMESTAMP)}
    return [state[k] for k in sorted(state)]


class JoinWithExpiration:
    """SURVEY.md 8(f) rank 3, inner joins of append-only inputs only: arroyo-worker/src/arrow/join_with_expiration.rs.

    process_left / process_right (:42-108): the arriving batch is inserted into its side's key-time table
    (KeyTimeView::insert, arroyo-state/src/tables/expiring_time_key_map.rs:997-1046: rows grouped per key), the other
    side's stored rows of the batch's keys are fetched (get_batch :970-985) and the pair goes through the join plan
    (compute_pair :110-130) -- so every matching pair is emitted exactly once, when its later row arrives.  Rows leave
    the tables only through the state backend's retention (`ttl`, applied at restore / compaction), never inside a
    run: not restated.  Outer joins rely on the planner's updating-join rewrite and are out of this restatement.
    Output = [left payload..., right payload (clashing names get `_right`)..., _timestamp = max(l.ts, r.ts)]."""

    def __init__(self, left_on: str, right_on: str):
        self.on = (left_on, right_on)
        self.rows: List[Dict[int, List[dict]]] = [{}, {}]  # side -> key -> stored rows
        self.names: List[Optional[List[str]]] = [None, None]

    def name(self):
        return "JoinWithExpiration"

    def _pair(self, l: dict, r: dict) -> dict:
        out = {k: v for k, v in l.items() if k != TIMESTAMP}
        for k, v in r.items():
            if k != TIMESTAMP:
                out[k if k not in out else k + "_right"] = v
        out[TIMESTAMP] = max(l[TIMESTAMP], r[TIMESTAMP])
        return out

    def process_batch_index(self, index: int, total_inputs: int, batch: Batch, ctx=None, collector=None):
        side = index // (total_inputs // 2)
        other = 1 - side
        new_rows = batch.rows()
        for r in new_rows:                                   # insert first (:52, :83) ...
            self.rows[side].setdefault(r[self.on[side]], []).append(r)
        out = []
        for r in new_rows:                                   # ... then join the batch with the other side's rows
            for o in self.rows[other].get(r[self.on[side]], ()):
                out.append(self._pair(r, o) if side == 0 else self._pair(o, r))
        if out and collector is not None:
            cols = {k: np.array([x[k] for x in out]) for k in out[0]}
            collector.collect(Batch(cols))
        return out
