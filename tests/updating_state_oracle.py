"""CPU restatement of the updating aggregate's state table "a" and its restore -- TEST INFRASTRUCTURE ONLY.

It extends oracle/updating_oracle.py's `IncrementalAggregatingFunc` (which it leaves unchanged) with what the
reference does around it (line numbers of arroyo-worker/src/arrow/incremental_aggregator.rs):
  * state (checkpoint_sliding :272-340, written to the key-value table "a" at every flush :619-635): one row per key
    touched since the last write, [keys..., each aggregate's sliding-accumulator state, _timestamp, _generation].
    The per-aggregate fields are DataFusion 48's accumulator states (count: [count Int64]; sum: [sum Int64, count
    UInt64]; avg: [count UInt64, sum Float64]; min / max: [min / max Int64]); the last field, the trailing
    max(_timestamp) aggregate's state, is renamed `_timestamp` (sliding_state_schema :1083-1160).  Here the rows are
    written at a checkpoint for the keys flushed since the last one, which leaves the same latest row per key; every
    write carries one generation, one above the last one written or restored.
  * restore (initialize :446-503): table "a" arrives in any order and not de-duplicated (UncachedKeyValueView::get_all,
    arroyo-state/src/tables/expiring_time_key_map.rs:1096-1099); per key the row with the largest _generation wins,
    the later row on a tie.
Restatement limits: append-only inputs (MIN / MAX restore as one-value multisets), no count(distinct) (table "b")."""
from typing import Dict, List, Optional, Tuple

import numpy as np

from oracle.arroyo_oracle import TIMESTAMP, Batch
from oracle import updating_oracle as U

GENERATION = "_generation"
# table "a" fields per aggregate kind, and their numpy types
_STATE_FIELDS = {"count": [("count", np.int64)], "sum": [("sum", np.int64), ("count", np.uint64)],
                 "avg": [("count", np.uint64), ("sum", np.float64)], "min": [("min", np.int64)],
                 "max": [("max", np.int64)]}


def state_names(cfg: U.UpdatingAggConfig) -> List[str]:
    """Columns of table "a"."""
    names = list(cfg.key_names)
    for a in cfg.aggs:
        if a.kind not in _STATE_FIELDS:
            raise NotImplementedError(f"table 'a' state of {a.kind} (a Batch accumulator lives in table 'b')")
        names += [f"{a.name}[{f}]" for f, _ in _STATE_FIELDS[a.kind]]
    return names + [TIMESTAMP, GENERATION]


class KeyValueTable:
    """UncachedKeyValueView (arroyo-state/src/tables/expiring_time_key_map.rs:1073-1110): insert_batch appends,
    get_all yields every batch, unordered and not de-duplicated."""

    def __init__(self):
        self.batches: List[Batch] = []

    def insert_batch(self, batch):
        self.batches.append(batch)

    def get_all(self):
        yield from self.batches


def key_value_table(ctx, name: str):
    """ctx.table_manager.get_uncached_key_value_view(name), for any context object."""
    if hasattr(ctx, "key_value_table"):
        return ctx.key_value_table(name)
    return ctx.__dict__.setdefault("key_value_tables", {}).setdefault(name, KeyValueTable())


class IncrementalAggregatingFunc(U.IncrementalAggregatingFunc):
    """The updating oracle with checkpoint_sliding and initialize: flushes, ticks and end of data behave as the
    base class's; `handle_checkpoint(barrier, ctx)` also writes table "a", `on_start(ctx)` restores from it."""

    def __init__(self, cfg: U.UpdatingAggConfig):
        super().__init__(cfg)
        self.unexported: Dict[Tuple[int, ...], None] = {}  # keys flushed since the last state write (ordered set)
        self.generation = 0                                  # the generation the next state write carries

    def flush(self) -> Optional[Batch]:
        self.unexported.update(dict.fromkeys(self.updated))
        return super().flush()

    def handle_checkpoint(self, barrier=None, ctx=None, collector=None) -> Optional[Batch]:
        """Flushes; with a context, then writes the state of the keys flushed since the last write to table "a"."""
        out = self.flush()
        if ctx is not None:
            b = self.checkpoint_state()
            if b is not None:
                key_value_table(ctx, "a").insert_batch(b)
        return out

    def checkpoint_state(self) -> Optional[Batch]:
        """Table "a" rows of the keys flushed since the last call (None: no such key)."""
        keys = [k for k in self.unexported if k in self.state]
        self.unexported = {}
        if not keys:
            return None
        names = state_names(self.cfg)
        cols: Dict[str, list] = {n: [] for n in names}
        for k in keys:
            st = self.state[k]
            for name, kv in zip(self.cfg.key_names, k):
                cols[name].append(kv)
            for a, agg in enumerate(self.cfg.aggs):
                live = [v for v, c in st.multi[a].items() if c > 0]
                value = {"sum": U._wrap(st.sums[a]), "avg": st.fsums[a], "min": min(live) if live else None,
                         "max": max(live) if live else None}
                for f, _ in _STATE_FIELDS[agg.kind]:
                    cols[f"{agg.name}[{f}]"].append(st.rows if f == "count" else value[agg.kind])
            cols[TIMESTAMP].append(max(t for t, c in st.ts.items() if c > 0))
            cols[GENERATION].append(self.generation)
        self.generation += 1
        types = {f"{agg.name}[{f}]": t for agg in self.cfg.aggs for f, t in _STATE_FIELDS[agg.kind]}
        types.update({TIMESTAMP: np.int64, GENERATION: np.uint64})
        return Batch({n: np.array(v, dtype=types.get(n, object)) for n, v in cols.items()})

    def on_start(self, ctx):
        """Restores from the batches of table "a" (in any order, with several rows per key)."""
        batches = list(key_value_table(ctx, "a").get_all())
        if not batches:
            return
        if self.state or self.updated:
            raise ValueError("restore into an operator that already holds state")
        names = state_names(self.cfg)
        best: Dict[Tuple[int, ...], Tuple[int, dict]] = {}
        for b in batches:
            assert list(b.cols) == names, (list(b.cols), names)
            for r in b.rows():
                k = tuple(int(r[n]) for n in self.cfg.key_names)
                g = int(r[GENERATION])
                if k not in best or g >= best[k][0]:  # rows come in position order: a tie goes to the later one
                    best[k] = (g, r)
        # the row count: COUNT(*)'s, else a SUM's or AVG's count, else 1 (a MIN / MAX-only plan)
        counts = [f"{a.name}[count]" for a in self.cfg.aggs if a.kind == "count"]
        counts += [f"{a.name}[count]" for a in self.cfg.aggs if a.kind in ("sum", "avg")]
        for k, (g, r) in best.items():
            st = self.state[k] = U._KeyState(len(self.cfg.aggs))
            st.rows = int(r[counts[0]]) if counts else 1
            for a, agg in enumerate(self.cfg.aggs):
                if agg.kind == "sum":
                    st.sums[a] = int(r[f"{agg.name}[sum]"])
                elif agg.kind == "avg":
                    st.fsums[a] = float(r[f"{agg.name}[sum]"])
                elif agg.kind in ("min", "max"):
                    st.multi[a] = {int(r[f"{agg.name}[{agg.kind}]"]): 1}
            st.ts = {int(r[TIMESTAMP]): 1}
        self.generation = max(self.generation, max(g for g, _ in best.values()) + 1)
