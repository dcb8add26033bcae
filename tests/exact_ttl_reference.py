"""The updating aggregate's change stream and table "a" under a time-to-idle ttl, stated directly from the rules --
for checking tests/updating_ttl_oracle.py and the CUDA operator.

Built from the same per-batch partials as tests/exact_reference.updating_changes (Python integers, no f64 sums), and
like that module it imports nothing from oracle/.  The rules (incremental_aggregator.rs:637-738, :826-883;
updating_cache.rs:42-62, 215-236):

* a key is live from its first row until it is evicted; every row stamps its key with the clock of its batch;
* a flush first emits the change rows of exact_reference.updating_changes, then evicts every live key with
  clock - stamp >= ttl: one retraction of its state (values and `_timestamp` as its last flush emitted them), and
  the key is dropped.  A key that comes back after an eviction is a new key: an append only;
* table "a" at a checkpoint: the state of every key flushed since the previous checkpoint, as of its last flush; a
  key evicted since then writes a tombstone (None) instead, unless `tombstones` is false (the reference's own table,
  which keeps the key's last row);
* a restart restores every key whose latest table row is not a tombstone, stamped with the clock at the restart.

`events`: ("clock", t) (t never decreases; the clock starts at 0), ("batch", cols), ("flush",), ("checkpoint",) -- a
flush, then the table write -- and ("restart",).  Returns (one (retractions, appends, evictions) per flush or
checkpoint, each {key or None: row} with the key column, every aggregate (AVG as a Mean) and `_timestamp`; one table
per checkpoint: {key or None: state row as exact_state_reference.updating_state writes it, or None for a tombstone},
the latest row of every key written so far)."""
from fractions import Fraction

from tests.exact_reference import TIMESTAMP, _batch_partials, _columns, _merge_state, _state_row, _wrap


def _outputs(st, aggs):
    return tuple(st[0] if a.kind == "count" else float(Fraction(st[i][0], st[0])) if a.kind == "avg"
                 else _wrap(st[i]) if a.kind == "sum" else st[i] for i, a in enumerate(aggs, 1))


def table_row(st, aggs):
    """A key's state as exact_state_reference.updating_state describes it."""
    row = {"rows": st[0], TIMESTAMP: st[-1]}
    for i, a in enumerate(aggs, 1):
        row[a.name] = (st[0] if a.kind == "count" else _wrap(st[i]) if a.kind == "sum"
                       else tuple(st[i]) if a.kind == "avg" else st[i])
    return row


def updating_ttl(events, key_name, aggs, ttl, tombstones=True):
    assert ttl > 0
    state, stamp, before = {}, {}, {}
    table, pending = {}, {}  # key -> state list, or None: a tombstone
    clock, flushes, tables = 0, [], []
    for ev in events:
        if ev[0] == "clock":
            assert ev[1] >= clock, "the clock never goes back"
            clock = ev[1]
        elif ev[0] == "batch":
            for k, part in _batch_partials(_columns(ev[1]), key_name, aggs).items():
                if k not in before:
                    before[k] = state.get(k)
                state[k] = _merge_state(state.get(k), part, aggs)
                stamp[k] = clock
        elif ev[0] in ("flush", "checkpoint"):
            retract, append = {}, {}
            for k, old in before.items():
                new = state[k]
                pending[k] = list(new)
                if old is not None:
                    if _outputs(old, aggs) == _outputs(new, aggs):
                        continue
                    retract[k] = _state_row(old, k, key_name, aggs)
                append[k] = _state_row(new, k, key_name, aggs)
            before = {}
            evict = {k: _state_row(st, k, key_name, aggs) for k, st in state.items() if clock - stamp[k] >= ttl}
            for k in evict:
                del state[k], stamp[k]
                if tombstones:
                    pending[k] = None
            flushes.append((retract, append, evict))
            if ev[0] == "checkpoint":
                table.update(pending)
                pending = {}
                tables.append({k: None if st is None else table_row(st, aggs) for k, st in table.items()})
        else:
            assert ev[0] == "restart", ev
            state = {k: list(st) for k, st in table.items() if st is not None}
            stamp = dict.fromkeys(state, clock)
            before, pending = {}, {}
    return flushes, tables
