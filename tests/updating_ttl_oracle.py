"""CPU restatement of the updating aggregate's time-to-idle ttl -- TEST INFRASTRUCTURE ONLY.

It extends tests/updating_state_oracle.py's `IncrementalAggregatingFunc` (which it leaves unchanged) with the
reference's `UpdatingCache::with_time_to_idle` (arroyo-worker/src/arrow/updating_cache.rs:42-62) under an explicit
clock (`set_clock`, standing for `Instant::now()`):
  * every row refreshes its key's idle clock (modify_and_update :215-236; a key's position in the eviction list is
    its last update);
  * every flush, after the change rows, runs time_out(now) (incremental_aggregator.rs:688-701): keys idle for at
    least ttl, oldest first, leave as one retraction of their current values and their state is dropped;
  * table "a": the key-value table keeps a key's last row; a row with a null `_timestamp` deletes the key at restore
    (initialize :591-614).  Restored keys are stamped with the clock at on_start (:480).
With `reference=False` (the default) it follows the CUDA operator's two deviations (INTEGRATION.md §3): eviction
retractions leave even when the flush has no other row (the reference returns None then, :703-705), and the next
state write carries a tombstone (null `_timestamp`) for every key evicted since the last write and not flushed again.
With `reference=True` it is the reference: evictions alone emit nothing, and evicted keys keep their last row."""
from typing import Dict, Optional, Tuple

import numpy as np

from oracle.arroyo_oracle import TIMESTAMP, Batch
from oracle import updating_oracle as U
from tests import updating_state_oracle as S

DEFAULT_TTL = 24 * 60 * 60 * 1_000_000_000  # ttl_micros == 0 (:1043-1048), in ns


class IncrementalAggregatingFunc(S.IncrementalAggregatingFunc):
    def __init__(self, cfg: U.UpdatingAggConfig, ttl: int, reference: bool = False):
        super().__init__(cfg)
        self.ttl = int(ttl) or DEFAULT_TTL
        self.reference = reference
        self.now = 0
        self.last: Dict[Tuple[int, ...], int] = {}  # the eviction list: key -> last update, oldest first
        # keys evicted since the last state write: None (a tombstone), or (reference) their last _KeyState
        self.gone: Dict[Tuple[int, ...], Optional[U._KeyState]] = {}

    def set_clock(self, now: int):
        if now < self.now:
            raise ValueError("the clock never goes back")
        self.now = now

    def process_batch(self, batch: Batch, ctx=None, collector=None):
        super().process_batch(batch, ctx, collector)
        for i in range(batch.num_rows):
            k = tuple(int(batch[n][i]) for n in self.cfg.key_names)
            self.last.pop(k, None)
            self.last[k] = self.now

    def flush(self) -> Optional[Batch]:
        for k in self.updated:
            self.gone.pop(k, None)  # flushed again: its next state row is a live one
        out = super().flush()
        evicted = []
        for k, t in list(self.last.items()):  # time_out (updating_cache.rs TTLIter): oldest first
            if self.now - t < self.ttl:
                break
            del self.last[k]
            st = self.state.pop(k)
            evicted.append((k, self._evaluate(st)))
            self.gone[k] = st if self.reference else None
        if not evicted or (self.reference and out is None):
            return out
        cols = {c: list(v) for c, v in out.cols.items()} if out is not None else \
            {c: [] for c in list(self.cfg.key_names) + [a.name for a in self.cfg.aggs] + [TIMESTAMP, U.IS_RETRACT]}
        for k, vals in evicted:
            for name, kv in zip(self.cfg.key_names, k):
                cols[name].append(kv)
            for agg, v in zip(self.cfg.aggs, vals[:-1]):
                cols[agg.name].append(v)
            cols[TIMESTAMP].append(vals[-1])
            cols[U.IS_RETRACT].append(True)
        return Batch({c: np.array(v, dtype=object) for c, v in cols.items()})

    handle_tick = on_close = lambda self, *a, **k: self.flush()

    def checkpoint_state(self) -> Optional[Batch]:
        gone, self.gone = self.gone, {}
        last_rows = {k: st for k, st in gone.items() if st is not None}  # reference: the key's last row
        live = self.state
        self.state = {**live, **last_rows}
        self.unexported.update(dict.fromkeys(last_rows))
        try:
            b = super().checkpoint_state()
        finally:
            self.state = live
        dead = [k for k, st in gone.items() if st is None]
        if not dead:
            return b
        gen = self.generation - 1 if b is not None else self.generation
        if b is None:
            self.generation += 1
        names = S.state_names(self.cfg)
        cols = {n: (list(b[n]) if b is not None else []) for n in names}
        for k in dead:
            for name, kv in zip(self.cfg.key_names, k):
                cols[name].append(kv)
            for agg in self.cfg.aggs:
                for f, t in S._STATE_FIELDS[agg.kind]:
                    cols[f"{agg.name}[{f}]"].append(t(0))
            cols[TIMESTAMP].append(None)
            cols[S.GENERATION].append(gen)
        types = {f"{agg.name}[{f}]": t for agg in self.cfg.aggs for f, t in S._STATE_FIELDS[agg.kind]}
        types[S.GENERATION] = np.uint64
        return Batch({n: np.array(v, dtype=types.get(n, object)) for n, v in cols.items()})

    def on_start(self, ctx):
        """Restores from table "a": per key the row with the largest _generation (the later one on a tie) wins, and a
        winning tombstone leaves the key absent.  Restored keys are stamped with the clock now."""
        batches = list(S.key_value_table(ctx, "a").get_all())
        if not batches:
            return
        best: Dict[Tuple[int, ...], Tuple[int, dict]] = {}
        for b in batches:
            for r in b.rows():
                k = tuple(int(r[n]) for n in self.cfg.key_names)
                g = int(r[S.GENERATION])
                if k not in best or g >= best[k][0]:
                    best[k] = (g, r)
        live = [r for _, r in best.values() if r[TIMESTAMP] is not None]
        tmp = S.KeyValueTable()
        if live:
            names = S.state_names(self.cfg)
            tmp.insert_batch(Batch({n: np.array([r[n] for r in live], dtype=object) for n in names}))
        holder = type("Ctx", (), {})()
        holder.key_value_tables = {"a": tmp}
        super().on_start(holder)
        self.generation = max(self.generation, max(g for g, _ in best.values()) + 1)
        self.last = dict.fromkeys(self.state, self.now)
