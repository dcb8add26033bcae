"""CPU oracle for the arroyo-b200 hot path.  TEST INFRASTRUCTURE ONLY.

This module is a plain numpy / pure-Python restatement of the *reference's* algorithm for
the per-batch window-assign / keyed-aggregate / windowed-join operators.  It is never
imported by the product package (`arroyo_b200/`): only `tests/`, `__graft_entry__.smoke()`
and `bench.py`'s `cpu_baseline` / `--impl reference` legs may use it, and only as the
checker.

Every class cites the reference file:line it follows (paths relative to
/root/reference/crates).  The arithmetic inside DataFusion 48.0.1 (fork
ArroyoSystems/arrow-datafusion@916b45f5) / arrow-rs 55.2.0 is not under /root/reference;
it is restated from its published semantics (SURVEY.md section 8(a), "dep-knowledge"):

  COUNT(*)        -> Int64, never NULL
  SUM(Int64)      -> Int64, wrapping add
  AVG(Int64)      -> Float64; partial state (count: UInt64, sum: Float64 of inputs cast
                     to f64 before summing); final = sum / count
  MIN/MAX         -> type preserving

Parity pinning: the oracle is checked against the reference's own golden vectors
(crates/arroyo-sql-testing/golden_outputs/*.json, re-encoded by tests/golden/make_golden.py)
in tests/test_oracle_golden.py.  PARITY UNPINNED (no reference vector exists): SUM/AVG
inside *windowed* aggregates, i64 SUM overflow, the ahash values of the shuffle (we use our
own 64-bit mixer; ownership of a key does not change any result), Nexmark q8.

Time is int nanoseconds since the Unix epoch everywhere (python ints: no overflow).
The end-of-data watermark is u64::MAX ns (arroyo-worker/src/arrow/watermark_generator.rs:137-146).
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np

U64_MAX = (1 << 64) - 1
FINAL_WATERMARK = U64_MAX  # watermark_generator.rs:137-146
TIMESTAMP = "_timestamp"


# --------------------------------------------------------------------------------------
# A tiny columnar record batch
# --------------------------------------------------------------------------------------
class Batch:
    """Ordered mapping column-name -> 1-D numpy array (all the same length).

    `valid[name]` (optional) is a boolean array; absent means "no nulls".
    """

    def __init__(self, cols: Dict[str, np.ndarray], valid: Optional[Dict[str, np.ndarray]] = None):
        self.cols = dict(cols)
        self.valid = dict(valid or {})
        n = {len(v) for v in self.cols.values()}
        assert len(n) <= 1, "ragged batch"

    @property
    def num_rows(self) -> int:
        for v in self.cols.values():
            return len(v)
        return 0

    def names(self) -> List[str]:
        return list(self.cols.keys())

    def __getitem__(self, name: str) -> np.ndarray:
        return self.cols[name]

    def take(self, idx) -> "Batch":
        return Batch({k: v[idx] for k, v in self.cols.items()}, {k: v[idx] for k, v in self.valid.items()})

    def slice(self, start: int, length: int) -> "Batch":
        return self.take(slice(start, start + length))

    @staticmethod
    def concat(batches: Sequence["Batch"]) -> "Batch":
        assert batches
        names = batches[0].names()
        cols = {k: np.concatenate([b.cols[k] for b in batches]) for k in names}
        valid = {}
        for k in names:
            if any(k in b.valid for b in batches):
                valid[k] = np.concatenate(
                    [b.valid.get(k, np.ones(b.num_rows, dtype=bool)) for b in batches]
                )
        return Batch(cols, valid)

    def rows(self) -> List[dict]:
        """Rows as python dicts (None for nulls); used for multiset comparison in tests."""
        out = []
        for i in range(self.num_rows):
            r = {}
            for k, v in self.cols.items():
                if k in self.valid and not self.valid[k][i]:
                    r[k] = None
                else:
                    x = v[i]
                    r[k] = x.item() if hasattr(x, "item") else x
            out.append(r)
        return out


def bin_start(ts: int, width: int) -> int:
    """`ts - ts % width`; width 0 = instant window (the timestamp itself).
    arroyo-worker/src/arrow/tumbling_aggregating_window.rs:65-73,
    sliding_aggregating_window.rs:89-99; planner emits date_bin(width, _timestamp)
    (arroyo-planner/src/builder.rs:201-224)."""
    if width == 0:
        return ts
    return ts - ts % width


def bin_start_array(ts: np.ndarray, width: int) -> np.ndarray:
    if width == 0:
        return ts.copy()
    # timestamps in the supported range are non-negative; numpy % on int64 is floor-mod
    # like date_bin for the epoch origin.
    return ts - ts % np.int64(width)


# --------------------------------------------------------------------------------------
# Watermarks
# --------------------------------------------------------------------------------------
IDLE = "idle"


class WatermarkHolder:
    """arroyo-operator/src/context.rs:35-86.  A watermark is an int (event time) or IDLE."""

    def __init__(self, n_inputs: int):
        self.watermarks: List[Optional[object]] = [None] * n_inputs
        self.cur_watermark: Optional[object] = None
        self.last_present_watermark: Optional[int] = None
        self._update()

    def _update(self):
        cur: Optional[object] = IDLE
        for w in self.watermarks:
            if w is None:
                cur = None
                break
            if cur == IDLE:
                cur = w
            elif w == IDLE:
                pass
            else:
                cur = min(cur, w)
        self.cur_watermark = cur
        if cur is not None and cur != IDLE:
            self.last_present_watermark = cur

    def set(self, idx: int, watermark) -> Optional[object]:
        self.watermarks[idx] = watermark
        self._update()
        return self.cur_watermark


class WatermarkGenerator:
    """arroyo-worker/src/arrow/watermark_generator.rs:150-197.

    `delay_ns`: the watermark expression is `_timestamp - delay` (default 1 s,
    arroyo-planner/src/rewriters.rs:71-82); `interval_ns` = 1 s
    (arroyo-planner/src/extension/watermark_node.rs:97).
    process_batch returns the watermark to broadcast, or None."""

    def __init__(self, delay_ns: int = 1_000_000_000, interval_ns: int = 1_000_000_000):
        self.delay = delay_ns
        self.interval = interval_ns
        self.last_watermark_emitted_at = 0  # UNIX_EPOCH
        self.max_watermark = 0
        self.idle = False

    def process_batch(self, ts: np.ndarray) -> Optional[int]:
        if len(ts) == 0:
            return None
        max_timestamp = int(ts.max())
        watermark = int(ts.min()) - self.delay
        self.max_watermark = max(self.max_watermark, watermark)
        if self.idle or max(max_timestamp - self.last_watermark_emitted_at, 0) > self.interval:
            self.last_watermark_emitted_at = max_timestamp
            self.idle = False
            return watermark
        return None


# --------------------------------------------------------------------------------------
# Keyed state view (host side, only what the operators' control flow observes)
# --------------------------------------------------------------------------------------
class ExpiringTimeKeyView:
    """arroyo-state/src/tables/expiring_time_key_map.rs:825-929 (control-flow-visible part)."""

    def __init__(self, retention: int):
        self.retention = retention
        self.flushed: Dict[int, List[Batch]] = {}
        self.to_flush: Dict[int, List[Batch]] = {}

    def insert(self, max_timestamp: int, batch: Batch):
        self.to_flush.setdefault(max_timestamp, []).append(batch)

    def flush(self, watermark: Optional[int]):
        for t in sorted(self.to_flush):
            batches = self.to_flush.pop(t)
            if watermark is not None and t < watermark - self.retention:
                continue
            self.flushed.setdefault(t, []).extend(batches)
        if watermark is not None:
            cutoff = watermark - self.retention
            self.flushed = {t: b for t, b in self.flushed.items() if t >= cutoff}

    def flush_timestamp(self, t: int):
        batches = self.to_flush.pop(t, None)
        if batches is None:
            return
        self.flushed.setdefault(t, []).extend(batches)

    def expire_timestamp(self, t: int):
        self.flushed.pop(t, None)
        self.to_flush.pop(t, None)

    def get_min_time(self) -> Optional[int]:
        keys = list(self.flushed) + list(self.to_flush)
        return min(keys) if keys else None

    def all_batches_for_watermark(self, watermark: Optional[int]):
        cutoff = 0 if watermark is None else watermark - self.retention
        for t in sorted(self.flushed):
            if t >= cutoff:
                yield t, self.flushed[t]
        for t in sorted(self.to_flush):
            if t >= cutoff:
                yield t, self.to_flush[t]


class OperatorContext:
    """arroyo-operator/src/context.rs:459-467 (fields the hot path reads)."""

    def __init__(self, n_inputs: int = 1, task_index: int = 0, parallelism: int = 1):
        self.watermarks = WatermarkHolder(n_inputs)
        self.tables: Dict[str, ExpiringTimeKeyView] = {}
        self.task_index = task_index
        self.parallelism = parallelism

    def last_present_watermark(self) -> Optional[int]:
        return self.watermarks.last_present_watermark

    def table(self, name: str, retention: int) -> ExpiringTimeKeyView:
        if name not in self.tables:
            self.tables[name] = ExpiringTimeKeyView(retention)
        return self.tables[name]

    def global_table(self, name: str) -> dict:
        """GlobalKeyedView (arroyo-state/src/tables/global_keyed_map.rs): one value per subtask."""
        if not hasattr(self, "global_tables"):
            self.global_tables = {}
        return self.global_tables.setdefault(name, {})


class Collector:
    """arroyo-operator/src/context.rs:490-494: collects output batches in emission order."""

    def __init__(self):
        self.batches: List[Batch] = []

    def collect(self, batch: Batch):
        self.batches.append(batch)

    def all(self) -> Optional[Batch]:
        return Batch.concat(self.batches) if self.batches else None


# --------------------------------------------------------------------------------------
# Aggregates (DataFusion partial / final accumulators, restated)
# --------------------------------------------------------------------------------------
@dataclass
class Agg:
    """One aggregate expression.  kind in {count, sum, avg, min, max}; `col` is the input
    column name (ignored for count(*)); `name` is the output column name."""

    kind: str
    col: Optional[str]
    name: str


def _group(keys: List[np.ndarray], n: int) -> Tuple[List[np.ndarray], np.ndarray, int]:
    """Group ids for rows by the tuple of key columns.  Returns (unique key columns,
    inverse index per row, number of groups).  No key columns => one global group."""
    if not keys:
        return [], np.zeros(n, dtype=np.int64), (1 if n > 0 else 0)
    if len(keys) == 1:
        uniq, inv = np.unique(keys[0], return_inverse=True)
        return [uniq], inv.astype(np.int64), len(uniq)
    rec = np.rec.fromarrays(keys)
    uniq, inv = np.unique(rec, return_inverse=True)
    return [np.asarray(uniq[f]) for f in uniq.dtype.names], inv.astype(np.int64), len(uniq)


def partial_state_names(aggs: Sequence[Agg]) -> List[str]:
    names = []
    for a in aggs:
        if a.kind == "avg":
            names += [f"{a.name}[count]", f"{a.name}[sum]"]
        else:
            names.append(f"{a.name}[{a.kind}]")
    return names


def partial_aggregate(batch: Batch, key_names: Sequence[str], aggs: Sequence[Agg]) -> Batch:
    """AggregateExec(Partial): rows -> [group cols..., accumulator state cols...]
    (call sites tumbling_aggregating_window.rs:302-309, sliding :657-664)."""
    n = batch.num_rows
    uk, inv, g = _group([batch[k] for k in key_names], n)
    cols: Dict[str, np.ndarray] = {k: u for k, u in zip(key_names, uk)}
    for a in aggs:
        if a.kind == "count":
            c = np.zeros(g, dtype=np.int64)
            np.add.at(c, inv, 1)
            cols[f"{a.name}[count]"] = c
        elif a.kind == "sum":
            v = batch[a.col]
            if v.dtype.kind == "f":
                s = np.zeros(g, dtype=np.float64)
            else:
                s = np.zeros(g, dtype=v.dtype)
            with np.errstate(over="ignore"):
                np.add.at(s, inv, v)  # integer add wraps
            cols[f"{a.name}[sum]"] = s
        elif a.kind == "avg":
            c = np.zeros(g, dtype=np.uint64)
            np.add.at(c, inv, np.uint64(1))
            s = np.zeros(g, dtype=np.float64)
            np.add.at(s, inv, batch[a.col].astype(np.float64))
            cols[f"{a.name}[count]"] = c
            cols[f"{a.name}[sum]"] = s
        elif a.kind in ("min", "max"):
            v = batch[a.col]
            if a.kind == "min":
                s = np.full(g, np.iinfo(v.dtype).max if v.dtype.kind in "iu" else np.inf, dtype=v.dtype)
                np.minimum.at(s, inv, v)
            else:
                s = np.full(g, np.iinfo(v.dtype).min if v.dtype.kind in "iu" else -np.inf, dtype=v.dtype)
                np.maximum.at(s, inv, v)
            cols[f"{a.name}[{a.kind}]"] = s
        else:
            raise ValueError(a.kind)
    return Batch(cols)


def final_aggregate(partials: Sequence[Batch], key_names: Sequence[str], aggs: Sequence[Agg]) -> Optional[Batch]:
    """AggregateExec(Final): merge partial batches by key and finalise
    (call sites tumbling :353-372, sliding :169-196).  Empty input => no rows (None)."""
    partials = [p for p in partials if p.num_rows > 0]
    if not partials:
        return None
    allp = Batch.concat(partials)
    n = allp.num_rows
    uk, inv, g = _group([allp[k] for k in key_names], n)
    cols: Dict[str, np.ndarray] = {k: u for k, u in zip(key_names, uk)}
    for a in aggs:
        if a.kind == "count":
            c = np.zeros(g, dtype=np.int64)
            np.add.at(c, inv, allp[f"{a.name}[count]"])
            cols[a.name] = c
        elif a.kind == "sum":
            v = allp[f"{a.name}[sum]"]
            s = np.zeros(g, dtype=v.dtype)
            with np.errstate(over="ignore"):
                np.add.at(s, inv, v)
            cols[a.name] = s
        elif a.kind == "avg":
            c = np.zeros(g, dtype=np.uint64)
            np.add.at(c, inv, allp[f"{a.name}[count]"])
            s = np.zeros(g, dtype=np.float64)
            np.add.at(s, inv, allp[f"{a.name}[sum]"])
            cols[a.name] = s / c.astype(np.float64)
        elif a.kind == "min":
            v = allp[f"{a.name}[min]"]
            s = np.full(g, np.iinfo(v.dtype).max if v.dtype.kind in "iu" else np.inf, dtype=v.dtype)
            np.minimum.at(s, inv, v)
            cols[a.name] = s
        elif a.kind == "max":
            v = allp[f"{a.name}[max]"]
            s = np.full(g, np.iinfo(v.dtype).min if v.dtype.kind in "iu" else -np.inf, dtype=v.dtype)
            np.maximum.at(s, inv, v)
            cols[a.name] = s
    return Batch(cols)


def single_aggregate(batch: Batch, key_names: Sequence[str], aggs: Sequence[Agg]) -> Optional[Batch]:
    """AggregateExec(Single) = Partial followed by Final over one input."""
    return final_aggregate([partial_aggregate(batch, key_names, aggs)], key_names, aggs)


@dataclass
class WindowAggConfig:
    """What the reference's protobuf operator config carries, reduced to the supported subset
    (arroyo-rpc/proto/api.proto:39-80; schemas SURVEY.md Appendix A).

    Input schema  : [key cols..., value cols..., _timestamp]
    Partial schema: [key cols..., state cols..., _timestamp = pane start]
    Output schema : final projection (arroyo-planner/src/extension/aggregate.rs:292-390):
                    [key cols..., agg cols...] with the window struct {start,end} inserted at
                    `window_index`, then `_timestamp = bin + width - 1`.  Here the struct is
                    flattened to two columns `window_start`, `window_end`.
                    `final_projection=False` (tumbling only) gives [keys, aggs, _timestamp = bin]."""

    width: int
    slide: int = 0  # sliding only
    key_names: List[str] = field(default_factory=list)
    aggs: List[Agg] = field(default_factory=list)
    final_projection: bool = True
    window_index: int = 0


def _project(final: Batch, cfg: WindowAggConfig, bin_ts: int, width: int) -> Batch:
    """add_bin_start_as_timestamp + final projection (tumbling :95-106/:373-385,
    sliding :197-222; planner extension/aggregate.rs:342-389)."""
    n = final.num_rows
    if not cfg.final_projection:
        cols = dict(final.cols)
        cols[TIMESTAMP] = np.full(n, bin_ts, dtype=np.int64)
        return Batch(cols)
    items = list(final.cols.items())
    win = [
        ("window_start", np.full(n, bin_ts, dtype=np.int64)),
        ("window_end", np.full(n, bin_ts + width, dtype=np.int64)),
    ]
    items[cfg.window_index:cfg.window_index] = win
    cols = dict(items)
    cols[TIMESTAMP] = np.full(n, bin_ts + width - 1, dtype=np.int64)
    return Batch(cols)


def _split_by_bin(batch: Batch, width: int) -> List[Tuple[int, Batch]]:
    """K1+K2: date_bin, sort_to_indices, take, partition (tumbling :256-277, sliding :604-625).
    Returns (bin, slice) in ascending bin order."""
    bins = bin_start_array(batch[TIMESTAMP], width)
    order = np.argsort(bins, kind="stable")
    sorted_batch = batch.take(order)
    sb = bins[order]
    out = []
    if len(sb) == 0:
        return out
    cuts = np.flatnonzero(np.diff(sb)) + 1
    starts = np.concatenate([[0], cuts])
    ends = np.concatenate([cuts, [len(sb)]])
    for s, e in zip(starts, ends):
        out.append((int(sb[s]), sorted_batch.slice(int(s), int(e - s))))
    return out


class _BinExec:
    """BinComputingHolder (tumbling :76-91, sliding :429-447): rows buffered in the running
    Partial exec (`active`) and the partial batches it has already produced (`finished`)."""

    def __init__(self):
        self.active: List[Batch] = []
        self.finished: List[Batch] = []

    def drain(self, cfg: WindowAggConfig) -> List[Batch]:
        """Close the sender and drain the partial exec -> its partial batches."""
        if not self.active:
            return []
        p = partial_aggregate(Batch.concat(self.active), cfg.key_names, cfg.aggs)
        self.active = []
        return [p]


# --------------------------------------------------------------------------------------
# Tumbling window aggregate
# --------------------------------------------------------------------------------------
class TumblingAggregatingWindowFunc:
    """arroyo-worker/src/arrow/tumbling_aggregating_window.rs:250-392, :430-467."""

    def __init__(self, cfg: WindowAggConfig):
        self.cfg = cfg
        self.width = cfg.width
        self.execs: Dict[int, _BinExec] = {}

    def name(self):
        return "tumbling_window"

    def tables(self):
        return {"t": self.width}

    def on_start(self, ctx: OperatorContext):
        table = ctx.table("t", self.width)
        for t, batches in table.all_batches_for_watermark(ctx.last_present_watermark()):
            b = bin_start(t, self.width)
            ex = self.execs.setdefault(b, _BinExec())
            for batch in batches:
                ex.finished.append(Batch({k: v for k, v in batch.cols.items() if k != TIMESTAMP}))

    def process_batch(self, batch: Batch, ctx: OperatorContext, collector: Collector):
        wm = ctx.last_present_watermark()
        for b, rows in _split_by_bin(batch, self.width):
            if wm is not None and b < bin_start(wm, self.width):
                continue  # :282-291 late bin, dropped
            self.execs.setdefault(b, _BinExec()).active.append(rows)

    def handle_watermark(self, watermark, ctx: OperatorContext, collector: Collector):
        wm = ctx.last_present_watermark()
        if wm is not None:
            wbin = bin_start(wm, self.width)
            while self.execs:
                first = min(self.execs)
                if not first < wbin:
                    break
                ex = self.execs.pop(first)
                ex.finished.extend(ex.drain(self.cfg))
                final = final_aggregate(ex.finished, self.cfg.key_names, self.cfg.aggs)
                if final is not None:
                    collector.collect(_project(final, self.cfg, first, self.width))
        return watermark

    def handle_checkpoint(self, ctx: OperatorContext):
        wm = ctx.watermarks.cur_watermark
        wm = None if (wm is None or wm == IDLE) else wm
        table = ctx.table("t", self.width)
        for b in sorted(self.execs):
            ex = self.execs[b]
            for p in ex.drain(self.cfg):
                cols = dict(p.cols)
                cols[TIMESTAMP] = np.full(p.num_rows, b, dtype=np.int64)
                table.insert(b, Batch(cols))
                ex.finished.append(p)
        table.flush(wm)


# --------------------------------------------------------------------------------------
# Sliding window aggregate
# --------------------------------------------------------------------------------------
class _Tier:
    """RecordBatchTier (sliding_aggregating_window.rs:236-324) incl. its quirks: after
    `delete_before` clears all panes `start_time` is left unchanged."""

    def __init__(self, width: int):
        self.width = width
        self.start_time: Optional[int] = None
        self.panes: List[List[Batch]] = []

    def insert(self, batch: Batch, ts: int):
        b = bin_start(ts, self.width)
        if self.start_time is None:
            self.start_time = b
            self.panes.append([batch])
            return
        if b < self.start_time:
            raise RuntimeError("SystemTime duration_since error: bin before tier start")
        idx = (b - self.start_time) // self.width
        while len(self.panes) <= idx:
            self.panes.append([])
        self.panes[idx].append(batch)

    def batches_for_timestamp(self, b: int) -> List[Batch]:
        if self.start_time is None or self.start_time > b:
            return []
        idx = (b - self.start_time) // self.width
        if len(self.panes) <= idx:
            return []
        return list(self.panes[idx])

    def delete_before(self, cutoff: int):
        b = bin_start(cutoff, self.width)
        if self.start_time is None or self.start_time >= b:
            return
        idx = (b - self.start_time) // self.width
        if idx >= len(self.panes):
            self.panes.clear()
            return
        del self.panes[:idx]
        self.start_time = b

    def is_empty(self) -> bool:
        return all(len(p) == 0 for p in self.panes)


class SlidingAggregatingWindowFunc:
    """arroyo-worker/src/arrow/sliding_aggregating_window.rs:102-210 (should_advance/advance),
    :556-595 (on_start), :598-674 (process_batch), :676-737 (watermark, checkpoint).
    Single tier of width = slide (:519-521)."""

    NO_DATA, ONLY_BUFFERED, IN_MEMORY = "NoData", "OnlyBufferedData", "InMemoryData"

    def __init__(self, cfg: WindowAggConfig):
        assert cfg.slide > 0 and cfg.width % cfg.slide == 0
        self.cfg = cfg
        self.width = cfg.width
        self.slide = cfg.slide
        self.execs: Dict[int, _BinExec] = {}
        self.tier = _Tier(self.slide)
        self.state: Tuple[str, Optional[int]] = (self.NO_DATA, None)

    def name(self):
        return "sliding_window"

    def on_start(self, ctx: OperatorContext):
        wm = ctx.last_present_watermark()
        table = ctx.table("t", self.width)
        wbin = bin_start(wm if wm is not None else 0, self.slide)
        for t, batches in table.all_batches_for_watermark(wm):
            b = bin_start(t, self.slide)
            stripped = [Batch({k: v for k, v in x.cols.items() if k != TIMESTAMP}) for x in batches]
            if b < wbin:
                for x in stripped:
                    self.tier.insert(x, b)
                continue
            self.execs.setdefault(b, _BinExec()).finished.extend(stripped)
        if self.tier.is_empty():
            mt = table.get_min_time()
            self.state = (self.ONLY_BUFFERED, bin_start(mt, self.slide)) if mt is not None else (self.NO_DATA, None)
        else:
            self.state = (self.IN_MEMORY, wbin)

    def process_batch(self, batch: Batch, ctx: OperatorContext, collector: Collector):
        wm = ctx.last_present_watermark()
        for b, rows in _split_by_bin(batch, self.slide):
            if wm is not None and b < bin_start(wm, self.slide):
                continue  # :631-633
            kind, t = self.state
            if kind == self.NO_DATA:
                self.state = (self.ONLY_BUFFERED, b)
            elif kind == self.ONLY_BUFFERED:
                self.state = (self.ONLY_BUFFERED, min(t, b))
            self.execs.setdefault(b, _BinExec()).active.append(rows)

    def should_advance(self, watermark: int) -> bool:
        wbin = bin_start(watermark, self.slide)
        kind, t = self.state
        if kind == self.NO_DATA:
            return False
        return t + self.slide <= wbin

    def advance(self, ctx: OperatorContext, collector: Collector):
        kind, b = self.state
        assert kind != self.NO_DATA
        table = ctx.table("t", self.width)
        bin_end = b + self.slide
        table.flush(bin_end)
        ex = self.execs.pop(b, None)
        if ex is not None:
            for p in ex.drain(self.cfg):
                cols = dict(p.cols)
                cols[TIMESTAMP] = np.full(p.num_rows, b, dtype=np.int64)
                table.insert(b, Batch(cols))
                ex.finished.append(p)
            for p in ex.finished:
                self.tier.insert(p, b)
        table.flush_timestamp(bin_end)
        # The reference expires bin_end - width + slide here: the oldest pane of the NEXT window, which its in-memory
        # tier still holds.  A checkpoint taken now would then restore that window without it.  Expire the pane that
        # has just left instead, so the table always holds what the tier holds.
        table.expire_timestamp(bin_end - self.width)
        interval_start, interval_end = bin_end - self.width, bin_end
        partials: List[Batch] = []
        cur = interval_start
        while cur < interval_end:
            partials.extend(self.tier.batches_for_timestamp(cur))
            cur += self.slide
        self.tier.delete_before(bin_end + self.slide - self.width)
        if self.tier.is_empty():
            # the reference consults only the table here and would never emit the panes still pending in `execs`
            # (rows that arrived while the store was non-empty and were not checkpointed): they are candidates too
            mt = table.get_min_time()
            if self.execs and (mt is None or min(self.execs) < mt):
                mt = min(self.execs)
            self.state = (self.ONLY_BUFFERED, bin_start(mt, self.slide)) if mt is not None else (self.NO_DATA, None)
        else:
            self.state = (self.IN_MEMORY, bin_end)
        final = final_aggregate(partials, self.cfg.key_names, self.cfg.aggs)
        if final is not None:
            collector.collect(_project(final, self.cfg, interval_start, self.width))

    def handle_watermark(self, watermark, ctx: OperatorContext, collector: Collector):
        wm = ctx.last_present_watermark()
        if wm is None:
            return None
        while self.should_advance(wm):
            self.advance(ctx, collector)
        return watermark

    def handle_checkpoint(self, ctx: OperatorContext):
        wm = ctx.watermarks.cur_watermark
        wm = None if (wm is None or wm == IDLE) else wm
        table = ctx.table("t", self.width)
        for b in sorted(self.execs):
            ex = self.execs[b]
            for p in ex.drain(self.cfg):
                cols = dict(p.cols)
                cols[TIMESTAMP] = np.full(p.num_rows, b, dtype=np.int64)
                table.insert(b, Batch(cols))
                ex.finished.append(p)
        table.flush(wm)


# --------------------------------------------------------------------------------------
# Session window aggregate
# --------------------------------------------------------------------------------------
@dataclass
class SessionConfig:
    """SessionWindowAggregateOperator (api.proto:39-80; planner extension/aggregate.rs:170-231).
    Output = [key cols...] with window_start/window_end inserted at window_index, agg cols,
    _timestamp = window_end - 1 (session_aggregating_window.rs:316-382)."""

    gap: int
    key_names: List[str] = field(default_factory=list)
    aggs: List[Agg] = field(default_factory=list)
    window_index: int = 0


class _ActiveSession:
    """session_aggregating_window.rs:397-523.  `rows` collects the batches sent to the
    session's Single-mode aggregate."""

    def __init__(self, initial_timestamp: int):
        self.data_start = initial_timestamp
        self.data_end = initial_timestamp
        self.rows: List[Batch] = []

    def add_batch(self, batch: Batch, gap: int) -> Optional[Tuple[int, Batch]]:
        ts = batch[TIMESTAMP]
        n = batch.num_rows
        start, end = int(ts[0]), int(ts[n - 1])
        if end < self.data_end + gap:
            self.data_end = max(self.data_end, end)
            self.data_start = min(self.data_start, start)
            self.rows.append(batch)
            return None
        if self.data_end + gap < start:
            return (start, batch)
        if start < self.data_start - gap:
            raise RuntimeError("received a batch that starts before the current data_start - gap")
        if start < self.data_start:
            self.data_start = start
        # :464-479 -- NB the reference increments `index` before testing the row, so the row
        # that breaks the loop is *included* in the slice sent to this session.  Restated as is.
        index = 1
        while index < n:
            value = int(ts[index])
            index += 1
            if value < self.data_end:
                continue
            if value < self.data_end + gap:
                self.data_end = value
                continue
            break
        if index == n:
            self.rows.append(batch)
            return None
        self.rows.append(batch.slice(0, index))
        rest = batch.slice(index, n - index)
        return (int(ts[index]), rest)


class _KeyComputingHolder:
    """session_aggregating_window.rs:533-691."""

    def __init__(self, cfg: SessionConfig):
        self.cfg = cfg
        self.active: Optional[_ActiveSession] = None
        self.by_start: Dict[int, List[Batch]] = {}

    def next_watermark_action(self) -> Optional[int]:
        if self.active is not None:
            return self.active.data_end + self.cfg.gap
        if self.by_start:
            return min(self.by_start) - self.cfg.gap
        return None

    def earliest_data(self) -> Optional[int]:
        if self.active is not None:
            return self.active.data_start
        return min(self.by_start) if self.by_start else None

    def is_empty(self) -> bool:
        return self.active is None and not self.by_start

    def fill_active_session(self):
        a = self.active
        assert a is not None
        while self.by_start:
            first = min(self.by_start)
            if a.data_end + self.cfg.gap < first:
                break
            batches = self.by_start.pop(first)
            for b in batches:
                rem = a.add_batch(b, self.cfg.gap)
                if rem is not None:
                    self.by_start.setdefault(rem[0], []).append(rem[1])

    def watermark_update(self, watermark: int) -> List[Tuple[int, int, Batch]]:
        results = []
        while True:
            if self.active is not None:
                if self.active.data_end + self.cfg.gap < watermark:
                    a = self.active
                    self.active = None
                    rows = Batch.concat(a.rows)
                    agg = single_aggregate(rows, [], self.cfg.aggs)
                    assert agg is not None and agg.num_rows == 1
                    results.append((a.data_start, a.data_end + self.cfg.gap, agg))
                else:
                    break
            else:
                if not self.by_start:
                    break
                initial = min(self.by_start)
                if watermark + self.cfg.gap < initial:
                    break
                self.active = _ActiveSession(initial)
                self.fill_active_session()
        return results

    def add_batch(self, batch: Batch, watermark: Optional[int]):
        if batch.num_rows == 0:
            return
        start_time = int(batch[TIMESTAMP][0])
        self.by_start.setdefault(start_time, []).append(batch)
        if watermark is None:
            return
        if self.active is not None:
            self.fill_active_session()
        flushed = self.watermark_update(watermark)
        if flushed:
            raise RuntimeError("should not have flushed batches when adding a batch")


class SessionAggregatingWindowFunc:
    """arroyo-worker/src/arrow/session_aggregating_window.rs:60-279, :850-895."""

    def __init__(self, cfg: SessionConfig):
        self.cfg = cfg
        self.key_computations: Dict[tuple, _KeyComputingHolder] = {}
        self.keys_by_next_watermark_action: Dict[int, set] = {}
        # `keys_by_start_time` (:50-54): only its first key is ever read (earliest_batch_time, :162-166), and its
        # entries are never removed -- :125-141 and :244-262 empty the key *sets* -- so the first key is the smallest
        # start time that was ever registered
        self.start_times_seen: Optional[int] = None

    def _note_start(self, t: Optional[int]):
        if t is not None and (self.start_times_seen is None or t < self.start_times_seen):
            self.start_times_seen = t

    def earliest_batch_time(self) -> Optional[int]:
        return self.start_times_seen

    def tables(self):
        return {"s": self.cfg.gap * 100, "e": 0}

    def on_start(self, ctx: OperatorContext):
        """:802-847."""
        starts = [v for v in ctx.global_table("e").values() if v is not None]
        if not starts:
            return
        start_time = min(starts)
        table = ctx.table("s", self.cfg.gap * 100)
        for _t, batches in list(table.all_batches_for_watermark(start_time)):
            for batch in list(batches):
                batch = batch.take(batch[TIMESTAMP] >= start_time)
                if batch.num_rows == 0:
                    continue
                self._add_at_watermark(self._sort(batch), start_time)
        wm = ctx.last_present_watermark()
        if wm is None:
            return
        self._results_at_watermark(wm)  # evicted results are dropped (:837-845)

    def handle_checkpoint(self, ctx: OperatorContext):
        """:907-925."""
        wm = ctx.last_present_watermark()
        ctx.table("s", self.cfg.gap * 100).flush(wm)
        ctx.global_table("e")[ctx.task_index] = self.earliest_batch_time()

    def name(self):
        return "session_window"

    def _sort(self, batch: Batch) -> Batch:
        # lexsort by (keys..., _timestamp) (:305-314; arroyo-rpc/src/df.rs:318-357)
        cols = [batch[TIMESTAMP]] + [batch[k] for k in reversed(self.cfg.key_names)]
        return batch.take(np.lexsort(cols))

    def _add_at_watermark(self, sorted_batch: Batch, watermark: Optional[int]):
        n = sorted_batch.num_rows
        if not self.cfg.key_names:
            ranges = [(0, n)]
        else:
            change = np.zeros(n, dtype=bool)
            for k in self.cfg.key_names:
                c = sorted_batch[k]
                change[1:] |= c[1:] != c[:-1]
            starts = np.concatenate([[0], np.flatnonzero(change)])
            ends = np.concatenate([starts[1:], [n]])
            ranges = list(zip(starts.tolist(), ends.tolist()))
        for s, e in ranges:
            kb = sorted_batch.slice(s, e - s)
            key = tuple(kb[k][0].item() for k in self.cfg.key_names)
            kc = self.key_computations.get(key)
            if kc is None:
                kc = self.key_computations[key] = _KeyComputingHolder(self.cfg)
            before = kc.next_watermark_action()
            kc.add_batch(kb, watermark)
            after = kc.next_watermark_action()
            assert after is not None
            self._note_start(kc.earliest_data())  # :228-262
            if before is not None and before != after:
                self.keys_by_next_watermark_action[before].discard(key)
                if not self.keys_by_next_watermark_action[before]:
                    del self.keys_by_next_watermark_action[before]
            if before is None or before != after:
                self.keys_by_next_watermark_action.setdefault(after, set()).add(key)

    def process_batch(self, batch: Batch, ctx: OperatorContext, collector: Collector):
        wm = ctx.last_present_watermark()
        if wm is not None:
            batch = batch.take(batch[TIMESTAMP] >= min(wm, np.iinfo(np.int64).max))  # :858-868
        if batch.num_rows == 0:
            return
        sorted_batch = self._sort(batch)
        ctx.table("s", self.cfg.gap * 100).insert(int(sorted_batch[TIMESTAMP].max()), sorted_batch)
        self._add_at_watermark(sorted_batch, wm)

    def _results_at_watermark(self, watermark: int):
        results = []
        while self.keys_by_next_watermark_action:
            first = min(self.keys_by_next_watermark_action)
            if not first < watermark:
                break
            keys = self.keys_by_next_watermark_action.pop(first)
            for key in sorted(keys):
                kc = self.key_computations[key]
                flushed = kc.watermark_update(watermark)
                if flushed:
                    results.append((key, flushed))
                if kc.is_empty():
                    del self.key_computations[key]
                else:
                    self._note_start(kc.earliest_data())  # :127-141
                    nxt = kc.next_watermark_action()
                    if nxt == first:
                        raise RuntimeError("next watermark action did not advance")
                    self.keys_by_next_watermark_action.setdefault(nxt, set()).add(key)
        return results

    def handle_watermark(self, watermark, ctx: OperatorContext, collector: Collector):
        wm = ctx.last_present_watermark()
        if wm is None:
            return watermark
        results = self._results_at_watermark(wm)
        if results:
            rows_keys, starts, ends, aggs = [], [], [], []
            for key, sessions in results:
                for s, e, agg in sessions:
                    rows_keys.append(key)
                    starts.append(s)
                    ends.append(e)
                    aggs.append(agg)
            items = []
            for i, k in enumerate(self.cfg.key_names):
                items.append((k, np.array([rk[i] for rk in rows_keys])))
            win = [
                ("window_start", np.array(starts, dtype=np.int64)),
                ("window_end", np.array(ends, dtype=np.int64)),
            ]
            items[self.cfg.window_index:self.cfg.window_index] = win
            merged = Batch.concat(aggs)
            items += list(merged.cols.items())
            cols = dict(items)
            cols[TIMESTAMP] = np.array(ends, dtype=np.int64) - 1
            collector.collect(Batch(cols))
        return watermark


# --------------------------------------------------------------------------------------
# Instant (windowed) join
# --------------------------------------------------------------------------------------
@dataclass
class JoinConfig:
    """JoinOperator (api.proto:39-80).  Inputs are [_key cols..., payload cols..., _timestamp];
    the `_key_*` routing copies are stripped before the join (`unkeyed_batch`,
    arroyo-rpc/src/df.rs:359-367) and the join is an equi-join of `left_on[i] = right_on[i]`
    payload columns.  join_type in {inner, left, right, full}.
    Output = [left payload cols..., right payload cols..., _timestamp = max(l.ts, r.ts)]
    (arroyo-planner/src/plan/join.rs:121-198); right-side columns that clash with a left
    name get the suffix `_right`."""

    left_on: List[str]
    right_on: List[str]
    join_type: str = "inner"
    left_routing_keys: List[str] = field(default_factory=list)
    right_routing_keys: List[str] = field(default_factory=list)


def hash_join(left: Optional[Batch], right: Optional[Batch], cfg: JoinConfig,
              left_names: List[str], right_names: List[str],
              left_dtypes: Dict[str, np.dtype], right_dtypes: Dict[str, np.dtype]) -> Optional[Batch]:
    """HashJoinExec restated as a sort-free nested grouping (K10).  Row order unspecified."""
    ln = left.num_rows if left is not None else 0
    rn = right.num_rows if right is not None else 0
    li: List[int] = []
    ri: List[int] = []
    index: Dict[tuple, List[int]] = {}
    for j in range(rn):
        index.setdefault(tuple(right[c][j].item() for c in cfg.right_on), []).append(j)
    matched_r = np.zeros(rn, dtype=bool)
    for i in range(ln):
        k = tuple(left[c][i].item() for c in cfg.left_on)
        js = index.get(k)
        if js:
            for j in js:
                li.append(i)
                ri.append(j)
                matched_r[j] = True
        elif cfg.join_type in ("left", "full"):
            li.append(i)
            ri.append(-1)
    if cfg.join_type in ("right", "full"):
        for j in np.flatnonzero(~matched_r):
            li.append(-1)
            ri.append(int(j))
    if not li:
        return None
    li_a = np.array(li, dtype=np.int64)
    ri_a = np.array(ri, dtype=np.int64)
    cols: Dict[str, np.ndarray] = {}
    valid: Dict[str, np.ndarray] = {}
    lvalid, rvalid = li_a >= 0, ri_a >= 0

    def gather(src: Optional[Batch], name: str, idx: np.ndarray, ok: np.ndarray, dt) -> np.ndarray:
        out = np.zeros(len(idx), dtype=dt)
        if src is not None and ok.any():
            out[ok] = src[name][idx[ok]]
        return out

    for c in left_names:
        if c == TIMESTAMP:
            continue
        cols[c] = gather(left, c, li_a, lvalid, left_dtypes[c])
        if not lvalid.all():
            valid[c] = lvalid.copy()
    for c in right_names:
        if c == TIMESTAMP:
            continue
        name = c if c not in cols else c + "_right"
        cols[name] = gather(right, c, ri_a, rvalid, right_dtypes[c])
        if not rvalid.all():
            valid[name] = rvalid.copy()
    lts = gather(left, TIMESTAMP, li_a, lvalid, np.int64)
    rts = gather(right, TIMESTAMP, ri_a, rvalid, np.int64)
    cols[TIMESTAMP] = np.where(lvalid & rvalid, np.maximum(lts, rts), np.where(lvalid, lts, rts))
    return Batch(cols, valid)


class InstantJoin:
    """arroyo-worker/src/arrow/instant_join.rs:109-172 (process_side), :241-283."""

    def __init__(self, cfg: JoinConfig):
        self.cfg = cfg
        self.execs: Dict[int, Tuple[List[Batch], List[Batch]]] = {}
        self.names: List[Optional[List[str]]] = [None, None]
        self.dtypes: List[Dict[str, np.dtype]] = [{}, {}]

    def name(self):
        return "InstantJoin"

    def tables(self):
        return {"left": 0, "right": 0}  # :305-328

    def on_start(self, ctx: OperatorContext):
        """:205-247: replay both tables through process_left / process_right."""
        wm = ctx.last_present_watermark()
        for side, name in enumerate(("left", "right")):
            batches = [b for _t, bs in ctx.table(name, 0).all_batches_for_watermark(wm) for b in bs]
            for b in batches:
                self._process_side(side, b, ctx)

    def handle_checkpoint(self, ctx: OperatorContext):
        """:285-303."""
        wm = ctx.last_present_watermark()
        ctx.table("left", 0).flush(wm)
        ctx.table("right", 0).flush(wm)

    def _process_side(self, side: int, batch: Batch, ctx: OperatorContext):
        if batch.num_rows == 0:
            raise RuntimeError("should have max timestamp")  # :123 expect()
        ts = batch[TIMESTAMP]
        ctx.table("left" if side == 0 else "right", 0).insert(int(ts.max()), batch)  # :116-128
        wm = ctx.last_present_watermark()
        if wm is not None and wm > int(ts.min()):
            raise RuntimeError("shouldn't have a batch with timestamp before the watermark")  # :129-139
        routing = self.cfg.left_routing_keys if side == 0 else self.cfg.right_routing_keys
        unkeyed = Batch({k: v for k, v in batch.cols.items() if k not in routing})
        if self.names[side] is None:
            self.names[side] = unkeyed.names()
            self.dtypes[side] = {k: v.dtype for k, v in unkeyed.cols.items()}
        for t in np.unique(ts):
            rows = unkeyed.take(ts == t)
            self.execs.setdefault(int(t), ([], []))[side].append(rows)

    def process_batch_index(self, index: int, total_inputs: int, batch: Batch, ctx: OperatorContext,
                            collector: Collector):
        self._process_side(index // (total_inputs // 2), batch, ctx)  # :249-253

    def handle_watermark(self, watermark, ctx: OperatorContext, collector: Collector):
        wm = ctx.last_present_watermark()
        if wm is None:
            return watermark
        for t in sorted(self.execs):
            if t >= wm:
                break
            lb, rb = self.execs.pop(t)
            left = Batch.concat(lb) if lb else None
            right = Batch.concat(rb) if rb else None
            if self.names[0] is None or self.names[1] is None:
                # one side never produced a batch: schema unknown to the restatement
                if self.cfg.join_type == "inner":
                    continue
            out = hash_join(left, right, self.cfg, self.names[0] or [], self.names[1] or [],
                            self.dtypes[0], self.dtypes[1])
            if out is not None:
                collector.collect(out)
        return wm


# --------------------------------------------------------------------------------------
# Key-hash shuffle
# --------------------------------------------------------------------------------------
def mix64(x: np.ndarray) -> np.ndarray:
    """Our 64-bit key hash (splitmix64 finaliser).  The reference hashes routing keys with
    DataFusion `create_hashes` + ahash(HASH_SEEDS) (arroyo-operator/src/context.rs:513-517);
    the exact ahash value is build dependent and only decides *which* subtask owns a key,
    never a result (SURVEY.md 8(c)(iii)) -- parity unpinned, by design."""
    z = x.astype(np.uint64) + np.uint64(0x9E3779B97F4A7C15)
    with np.errstate(over="ignore"):
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        z = z ^ (z >> np.uint64(31))
    return z


def server_for_hash_array(h: np.ndarray, n: int) -> np.ndarray:
    """arroyo-operator/src/lib.rs:30-41: (hash / (u64::MAX / n)) % n -- the formula the shuffle uses."""
    range_size = np.uint64(U64_MAX // n)
    return ((h // range_size) % np.uint64(n)).astype(np.uint64)


def server_for_hash(x: int, n: int) -> int:
    """arroyo-types/src/lib.rs:640-647."""
    if n == 1:
        return 0
    return x // (U64_MAX // n + 1)


def range_for_server(i: int, n: int) -> Tuple[int, int]:
    """arroyo-types/src/lib.rs:649-661 (inclusive range)."""
    if n == 1:
        return (0, U64_MAX)
    rs = U64_MAX // n + 1
    start = rs * i
    end = U64_MAX if i + 1 == n else start + rs - 1
    return (start, end)


def repartition(batch: Batch, key_names: Sequence[str], qs: int) -> List[Tuple[int, Batch]]:
    """arroyo-operator/src/context.rs:506-541 (keyed branch): hash -> dest -> sort by dest ->
    gather -> slice per dest.  Multi-column keys fold the per-column hashes."""
    h = np.zeros(batch.num_rows, dtype=np.uint64)
    for k in key_names:
        with np.errstate(over="ignore"):
            h = mix64(batch[k].astype(np.int64).view(np.uint64) ^ (h * np.uint64(31)))
    servers = server_for_hash_array(h, qs)
    order = np.argsort(servers, kind="stable")
    sb = batch.take(order)
    ss = servers[order]
    out = []
    if len(ss) == 0:
        return out
    cuts = np.flatnonzero(np.diff(ss)) + 1
    starts = np.concatenate([[0], cuts])
    ends = np.concatenate([cuts, [len(ss)]])
    for s, e in zip(starts, ends):
        out.append((int(ss[s]), sb.slice(int(s), int(e - s))))
    return out


# --------------------------------------------------------------------------------------
# A miniature single-subtask dataflow: source batches -> watermark generator -> operator
# --------------------------------------------------------------------------------------
def run_single_input(op, batches: Sequence[Batch], delay_ns: int = 1_000_000_000,
                     ctx: Optional[OperatorContext] = None) -> Collector:
    """Drive `op` the way the worker run loop does for one input partition
    (arroyo-operator/src/operator.rs:932-1066): each source batch goes through the
    WatermarkGenerator (forward batch, then maybe broadcast a watermark), and end of data
    broadcasts the final watermark (watermark_generator.rs:131-148)."""
    ctx = ctx or OperatorContext(1)
    out = Collector()
    gen = WatermarkGenerator(delay_ns)
    for b in batches:
        op.process_batch(b, ctx, out)
        wm = gen.process_batch(b[TIMESTAMP])
        if wm is not None:
            ctx.watermarks.set(0, wm)
            op.handle_watermark(wm, ctx, out)
    ctx.watermarks.set(0, FINAL_WATERMARK)
    op.handle_watermark(FINAL_WATERMARK, ctx, out)
    return out


def source_batches(cols: Dict[str, np.ndarray], batch_size: int) -> List[Batch]:
    n = len(next(iter(cols.values())))
    return [Batch({k: v[i:i + batch_size] for k, v in cols.items()}) for i in range(0, n, batch_size)]
