"""The updating aggregate's exact per-key state at every flush, for checking its state table "a".

Built from the same per-batch partials as tests/exact_reference.updating_changes (Python integers, no f64 sums), and
like that module it imports nothing from oracle/."""
from tests.exact_reference import TIMESTAMP, _batch_partials, _columns, _merge_state, _wrap


def updating_state(events, key_name, aggs):
    """One {key or None: state} per flush, over every key with rows before that flush.  A state is {"rows": row
    count, `_timestamp`: max timestamp, and per aggregate: COUNT the row count, SUM the wrapped sum, MIN / MAX the
    value, AVG the pair (exact integer sum, sum of |x|)}.  `events`: ("batch", cols) and ("flush",)."""
    state, out = {}, []
    for ev in events:
        if ev[0] == "batch":
            for k, part in _batch_partials(_columns(ev[1]), key_name, aggs).items():
                state[k] = _merge_state(state.get(k), part, aggs)
            continue
        assert ev[0] == "flush", ev
        snap = {}
        for k, st in state.items():
            row = {"rows": st[0], TIMESTAMP: st[-1]}
            for i, a in enumerate(aggs, 1):
                row[a.name] = (st[0] if a.kind == "count" else _wrap(st[i]) if a.kind == "sum"
                               else tuple(st[i]) if a.kind == "avg" else st[i])
            snap[k] = row
        out.append(snap)
    return out
