"""CPU restatement of the join with expiration's key-time tables and their restore -- TEST INFRASTRUCTURE ONLY.

It extends oracle/updating_oracle.py's `JoinWithExpiration` (which it leaves unchanged) with what the reference does
around it (join_with_expiration.rs, arroyo-state/src/tables/expiring_time_key_map.rs):
  * insert (KeyTimeView::insert :997-1006): every arriving batch goes, raw, into its side's table "left" or "right",
    here under its newest `_timestamp`.
  * checkpoint: the checkpointer keeps what still holds data at or after watermark - retention (:747-760).  The
    retention is the join's ttl; a ttl of 0 means 24 h (join_with_expiration.rs:239-248).
  * restore is lazy: the first batch after a restart loads both tables with the watermark of that moment
    (get_key_time_table in process_left / process_right).  A batch whose newest `_timestamp` is below watermark - ttl
    (UNIX_EPOCH without a watermark) is dropped (get_key_time_view :200-236); the rest join their side's stored rows
    without being joined against the other side (insert_internal :1008-1049).

`expiring_join_restarts` is the exact reference of a stream with restarts, built on exact_reference.expiring_join."""
import numpy as np

from oracle import updating_oracle as U
from oracle.arroyo_oracle import TIMESTAMP
from tests import exact_reference as X

DAY_NS = 24 * 3600 * 10 ** 9
TABLES = ("left", "right")


def retention(ttl: int) -> int:
    return ttl or DAY_NS


def cutoff(watermark, ttl: int) -> int:
    """The oldest newest-timestamp a restored batch may have: watermark - retention, or 0 (UNIX_EPOCH) without a
    watermark (all_batches_for_watermark)."""
    return 0 if watermark is None else watermark - retention(ttl)


def newest(batch) -> int:
    return int(np.max(np.asarray(X._columns(batch)[TIMESTAMP]).astype(np.int64)))


class JoinWithExpiration(U.JoinWithExpiration):
    """The join oracle with its tables: `process_batch_index(..., ctx)` inserts into them, `handle_checkpoint(barrier,
    ctx)` flushes them, `on_start(ctx)` makes the next batch load them.  `ctx` is an oracle.arroyo_oracle
    OperatorContext."""

    def __init__(self, left_on: str, right_on: str, ttl: int = 0):
        super().__init__(left_on, right_on)
        self.ttl = retention(ttl)
        self.restore_pending = False

    def tables(self):
        return dict.fromkeys(TABLES, self.ttl)

    def on_start(self, ctx):
        self.restore_pending = True

    def handle_checkpoint(self, barrier=None, ctx=None, collector=None):
        wm = ctx.last_present_watermark()
        for name in TABLES:
            ctx.table(name, self.ttl).flush(wm)

    def _load(self, ctx):
        wm = ctx.last_present_watermark()
        for side, name in enumerate(TABLES):
            for _, batches in ctx.table(name, self.ttl).all_batches_for_watermark(wm):
                for b in batches:
                    for r in b.rows():  # insert_internal: stored, not probed
                        self.rows[side].setdefault(r[self.on[side]], []).append(r)

    def process_batch_index(self, index: int, total_inputs: int, batch, ctx=None, collector=None):
        side = index // (total_inputs // 2)
        if self.restore_pending:
            self.restore_pending = False
            self._load(ctx)
        if ctx is not None and batch.num_rows:
            ctx.table(TABLES[side], self.ttl).insert(newest(batch), batch)
        return super().process_batch_index(index, total_inputs, batch, ctx, collector)


def run_oracle(events, ttl, left_on, right_on, ctx=None, names=None):
    """Drives the oracle through `events` (as `expiring_join_restarts` takes them, batches as column dicts or
    oracle Batches).  A restart checkpoints the operator, drops it and starts a new one on the same context.  Returns
    each batch's output as X.Rows with the columns `names` (default: `output_names(events)`), and the context (its
    tables)."""
    from oracle import arroyo_oracle as O
    ctx = ctx or O.OperatorContext(2)
    op = JoinWithExpiration(left_on, right_on, ttl)
    outs = []
    for ev, arg in events:
        if ev == "wm":
            ctx.watermarks.set(0, arg)
            ctx.watermarks.set(1, arg)
        elif ev == "restart":
            op.handle_checkpoint(None, ctx)
            op = JoinWithExpiration(left_on, right_on, ttl)
            op.on_start(ctx)
        else:
            outs.append(op.process_batch_index(ev, 2, arg if isinstance(arg, O.Batch) else O.Batch(arg), ctx))
    names = names or output_names(events)
    return [X.Rows.from_columns(names, [np.array([int(r[c]) % (1 << 64) for r in out], dtype=np.uint64)
                                        for c in names]) for out in outs], ctx


def output_names(events):
    """The join's output columns for a stream without routing columns: each side's first batch names them."""
    first = [None, None]
    for ev, arg in events:
        if ev in (0, 1) and first[ev] is None:
            first[ev] = [c for c in X._columns(arg) if c != TIMESTAMP]
    names = list(first[0] or [])
    for c in first[1] or []:
        names.append(c if c not in names else c + "_right")
    return names + [TIMESTAMP]


def expiring_join_restarts(events, ttl, left_on, right_on, left_routing=(), right_routing=()):
    """The join with expiration across restarts.  `events`: (side, batch), ("wm", w) (the effective watermark) and
    ("restart", None).  A restart's cutoff `c` is the watermark in effect at the first batch after it, minus the
    retention (0 without a watermark).  With `kept` = the non-empty batches inserted so far, both sides in insertion
    order, whose newest `_timestamp` is at least `c`, the outputs of the batches up to the next restart are
    `expiring_join(kept + those batches)[len(kept):]`.  Returns one X.Rows per batch event."""
    inserted, kept, segment, out = [], [], [], []
    wm, restarted = None, False

    def close():
        out.extend(X.expiring_join(kept + segment, left_on, right_on, left_routing, right_routing)[len(kept):])

    for ev, arg in events:
        if ev == "wm":
            wm = arg
        elif ev == "restart":
            close()
            segment, restarted = [], True
        else:
            if restarted:  # the lazy load: the cutoff of the watermark at this batch
                c = cutoff(wm, ttl)
                kept = [e for e in inserted if newest(e[1]) >= c]
                restarted = False
            segment.append((ev, arg))
            if len(X._columns(arg)[TIMESTAMP]):
                inserted.append((ev, arg))
    close()
    # a run whose kept batches miss a side names only the other side's columns; it has no pairs either
    names = max((r.names for r in out), key=len, default=[])
    for i, r in enumerate(out):
        if r.names != names:
            assert len(r) == 0, (r.names, names)
            out[i] = X.Rows(names, np.zeros((0, len(names)), np.uint64), np.zeros((0, len(names)), bool))
    return out
