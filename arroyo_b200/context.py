"""Host-side mirror of the pieces of arroyo-operator the hot path talks to: WatermarkHolder
(context.rs:35-86), OperatorContext (context.rs:459-467), Collector (context.rs:490-494) and the
WatermarkGenerator's emission rule (arroyo-worker/src/arrow/watermark_generator.rs:150-197).
Pure control flow -- no row data is computed here."""
from typing import Dict, List, Optional

IDLE = "idle"
U64_MAX = (1 << 64) - 1
INT64_MAX = (1 << 63) - 1
FINAL_WATERMARK = U64_MAX  # end-of-data watermark, watermark_generator.rs:137-146


class WatermarkHolder:
    """Min-merge of the watermarks of all input partitions; Idle inputs are ignored; no watermark
    until every input has reported (context.rs:63-79)."""

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
            elif w != IDLE:
                cur = min(cur, w)
        self.cur_watermark = cur
        if cur is not None and cur != IDLE:
            self.last_present_watermark = cur

    def set(self, idx: int, watermark):
        self.watermarks[idx] = watermark
        self._update()
        return self.cur_watermark


class StateTable:
    """The slice of ExpiringTimeKeyView (arroyo-state/src/tables/expiring_time_key_map.rs:833-929) a
    checkpoint round trip needs: batches keyed by timestamp."""

    def __init__(self, retention: int):
        self.retention = retention
        self.batches: Dict[int, list] = {}

    def insert(self, ts: int, batch):
        self.batches.setdefault(ts, []).append(batch)

    def get_min_time(self) -> Optional[int]:
        return min(self.batches) if self.batches else None

    def flush(self, watermark: Optional[int]):
        """ExpiringTimeKeyView::flush (expiring_time_key_map.rs:853-893): what a checkpoint keeps = the entries at
        or after watermark - retention."""
        if watermark is not None:
            cutoff = watermark - self.retention
            self.batches = {t: b for t, b in self.batches.items() if t >= cutoff}

    def all_batches_for_watermark(self, watermark: Optional[int]):
        cutoff = 0 if watermark is None else watermark - self.retention
        for t in sorted(self.batches):
            if t >= cutoff:
                for b in self.batches[t]:
                    yield t, b


class KeyValueTable:
    """The slice of UncachedKeyValueView (arroyo-state/src/tables/expiring_time_key_map.rs:1073-1110) the updating
    aggregate uses: `insert_batch` appends a batch of rows, `get_all` yields every batch written so far, in no
    particular order and without de-duplication (a key may have rows in several batches; its `_generation` column
    tells which is the latest)."""

    def __init__(self):
        self.batches: list = []

    def insert_batch(self, batch):
        self.batches.append(batch)

    def get_all(self):
        yield from self.batches


class OperatorContext:
    def __init__(self, n_inputs: int = 1, task_index: int = 0, parallelism: int = 1):
        self.watermarks = WatermarkHolder(n_inputs)
        self.tables: Dict[str, StateTable] = {}
        self.task_index = task_index
        self.parallelism = parallelism

    def last_present_watermark(self) -> Optional[int]:
        return self.watermarks.last_present_watermark

    def watermark(self):
        return self.watermarks.cur_watermark

    def table(self, name: str, retention: int = 0) -> StateTable:
        if name not in self.tables:
            self.tables[name] = StateTable(retention)
        return self.tables[name]

    def key_value_table(self, name: str) -> KeyValueTable:
        """get_uncached_key_value_view(name)."""
        if not hasattr(self, "key_value_tables"):
            self.key_value_tables = {}
        return self.key_value_tables.setdefault(name, KeyValueTable())

    def global_table(self, name: str) -> dict:
        """GlobalKeyedView (arroyo-state/src/tables/global_keyed_map.rs): one value per subtask, all of them
        visible to every subtask on restore."""
        if not hasattr(self, "global_tables"):
            self.global_tables = {}
        return self.global_tables.setdefault(name, {})


class Collector:
    def __init__(self):
        self.batches = []

    def collect(self, batch):
        self.batches.append(batch)


class WatermarkGenerator:
    """Emission rule only (min/max of the batch's timestamps are supplied by the caller):
    watermark = min(ts) - delay, broadcast when max(ts) - last_emitted_at > interval."""

    def __init__(self, delay_ns: int = 1_000_000_000, interval_ns: int = 1_000_000_000):
        self.delay = delay_ns
        self.interval = interval_ns
        self.last_watermark_emitted_at = 0
        self.max_watermark = 0
        self.idle = False

    def process_device_batch(self, ts_ptr: int, n_rows: int, device: int = 0, stream: int = 0) -> Optional[int]:
        """The generator's two reductions run on the device (arroyo_b200_ts_minmax), then the emission rule."""
        import ctypes as C

        from . import ffi
        mn, mx = C.c_int64(0), C.c_int64(0)
        st = ffi.load().arroyo_b200_ts_minmax(device, stream, ts_ptr, n_rows, C.byref(mn), C.byref(mx))
        if st != ffi.OK:
            raise ffi.ArroyoB200Error(st, "ts_minmax failed")
        if n_rows == 0:
            return None
        return self.on_batch(mn.value, mx.value)

    def on_batch(self, min_ts: int, max_ts: int) -> Optional[int]:
        watermark = min_ts - self.delay
        self.max_watermark = max(self.max_watermark, watermark)
        if self.idle or max(max_ts - self.last_watermark_emitted_at, 0) > self.interval:
            self.last_watermark_emitted_at = max_ts
            self.idle = False
            return watermark
        return None


def clamp_watermark(wm: int) -> int:
    """The C ABI carries event time as int64 ns; the end-of-data watermark u64::MAX becomes INT64_MAX."""
    return INT64_MAX if wm > INT64_MAX else int(wm)
