"""Exact group-by reference for the window and updating aggregates, and exact reference joins (`instant_join`,
`expiring_join`), computed straight from the raw input rows with numpy and Python integers.  It shares no code or
arithmetic with oracle/, so it can catch mistakes the oracle and the CUDA operators would make together (an AVG taken
over a wrapped integer sum, a float32 or double-rounded mean, a join that matches on part of its key).

AVG rule (`check_avg`): when the absolute values of a group's inputs sum to less than 2^53, every f64 or exact-integer
AVG path is exact up to its one final division, so the result must be bit-identical to the correctly rounded mean.
Otherwise |got - mean| <= 2u * sum|x| + 2u * |mean| with u = 2^-53: that is n * 2u * sum|x| on the sum, the error
bound of an f64 sum of n terms in any order including the rounding of each input, divided by n, plus the final
division."""
import bisect
import heapq
import itertools
from fractions import Fraction

import numpy as np

U = 2.0 ** -53
TIMESTAMP = "_timestamp"


class Mean:
    """An exact mean (`exact`), the sum of the group's absolute values (`abs_sum`, an int), and for the updating
    aggregate the sequential f64 sum in row order divided by the count (`seq`), the reference's own arithmetic."""
    __slots__ = ("exact", "abs_sum", "seq")

    def __init__(self, exact: Fraction, abs_sum: int, seq=None):
        self.exact, self.abs_sum, self.seq = exact, abs_sum, seq

    def __repr__(self):
        return f"Mean({float(self.exact)!r}, abs_sum={self.abs_sum}, seq={self.seq!r})"


def check_avg(got: float, want: Mean) -> bool:
    exact = float(want.exact)
    if want.abs_sum < 2 ** 53:
        return float(got) == exact
    err = abs(Fraction(float(got)) - want.exact)
    return err <= Fraction(2 * U) * want.abs_sum + Fraction(2 * U) * abs(want.exact)


def _split_sum(x_u64: np.ndarray, inv: np.ndarray, n_groups: int):
    """Exact per-group sums of unsigned 64-bit values as Python ints: the high and low 32-bit halves are summed
    separately (no int64 overflow below 2^31 rows per group)."""
    hi = np.zeros(n_groups, dtype=np.int64)
    lo = np.zeros(n_groups, dtype=np.int64)
    np.add.at(hi, inv, (x_u64 >> np.uint64(32)).astype(np.int64))
    np.add.at(lo, inv, (x_u64 & np.uint64(0xFFFFFFFF)).astype(np.int64))
    return [(int(h) << 32) + int(l) for h, l in zip(hi, lo)]


def _exact_sums(v: np.ndarray, inv: np.ndarray, n_groups: int):
    """(exact signed sum, exact sum of |v|) per group, as Python ints."""
    u = v.view(np.uint64)
    neg = v < 0
    total = _split_sum(u, inv, n_groups)
    n_neg = np.zeros(n_groups, dtype=np.int64)
    np.add.at(n_neg, inv, neg.astype(np.int64))
    signed = [t - (int(k) << 64) for t, k in zip(total, n_neg)]  # a negative v is u - 2^64
    absu = np.where(neg, (~u) + np.uint64(1), u)                   # |INT64_MIN| = 2^63 fits in u64
    return signed, _split_sum(absu, inv, n_groups)


def _aggregate(cols, inv, n_groups, aggs, order=None):
    """{agg name: per-group values}; order = row order for the sequential f64 AVG (updating aggregate)."""
    out = {}
    count = np.bincount(inv, minlength=n_groups)
    for a in aggs:
        if a.kind == "count":
            out[a.name] = [int(c) for c in count]
            continue
        v = np.ascontiguousarray(cols[a.col]).astype(np.int64, copy=False)
        if a.kind == "sum":
            s = np.zeros(n_groups, dtype=np.int64)
            with np.errstate(over="ignore"):
                np.add.at(s, inv, v)  # wraps like the operators' i64 SUM
            out[a.name] = [int(x) for x in s]
        elif a.kind in ("min", "max"):
            ii = np.iinfo(np.int64)
            s = np.full(n_groups, ii.max if a.kind == "min" else ii.min, dtype=np.int64)
            (np.minimum if a.kind == "min" else np.maximum).at(s, inv, v)
            out[a.name] = [int(x) for x in s]
        elif a.kind == "avg":
            signed, abs_sum = _exact_sums(v, inv, n_groups)
            seq = None
            if order is not None:
                seq = [0.0] * n_groups
                for g, x in zip(inv.tolist(), v.tolist()):
                    seq[g] += float(x)
            out[a.name] = [Mean(Fraction(signed[g], int(count[g])), abs_sum[g],
                                None if seq is None else seq[g] / int(count[g])) for g in range(n_groups)]
        else:
            raise ValueError(a.kind)
    return out


def _concat(batches):
    names = list(batches[0].cols)
    return {c: np.concatenate([np.asarray(b[c]) for b in batches]) for c in names}


def _group_keys(key: np.ndarray, extra: np.ndarray = None):
    """Group ids for (extra, key) rows; keys are grouped by value (UInt64 keys as UInt64)."""
    k = key.view(np.int64) if key.dtype == np.uint64 else key.astype(np.int64, copy=False)
    parts = [k] if extra is None else [extra.astype(np.int64, copy=False), k]
    uniq, inv = np.unique(np.stack(parts), axis=1, return_inverse=True)
    return uniq, inv.reshape(-1), uniq.shape[1]


def window_rows(batches, key_name, aggs, width, slide=None):
    """Expected output of a tumbling (slide None) or sliding window aggregate over rows that are never late:
    {(window_start, key or None): {column: value}} with window_end, _timestamp = window_end - 1 and the
    aggregates (AVG as a Mean)."""
    emitted, _ = window_emissions([("batch", b) for b in batches] + [("wm", INT64_MAX)], key_name, aggs, width, slide)
    return emitted[0]


def _bin(t: int, slide: int) -> int:
    return t - t % slide  # Python's % floors: a negative watermark bins below zero


class _Panes:
    """Per-(pane, key) partial states of the on-time rows: {pane: {key: [rows, state per aggregate]}}.  A state is
    the wrapping-free exact sum (SUM), the value (MIN / MAX) or (exact sum, sum of |x|) (AVG); COUNT uses `rows`."""

    def __init__(self, key_name, aggs, slide):
        self.key_name, self.aggs, self.slide = key_name, list(aggs), slide
        self.by_pane = {}

    def add(self, cols, ts):
        n = len(ts)
        if n == 0:
            return
        panes = ts - ts % np.int64(self.slide)
        key = np.asarray(cols[self.key_name]) if self.key_name else np.zeros(n, dtype=np.int64)
        uniq, inv, n_groups = _group_keys(key, panes)
        vals = _aggregate(cols, inv, n_groups, self.aggs)
        count = np.bincount(inv, minlength=n_groups)
        for g in range(n_groups):
            pane, k = int(uniq[0, g]), int(uniq[1, g])
            new = [int(count[g])]
            for a in self.aggs:
                v = vals[a.name][g]
                new.append((int(v.exact * int(count[g])), v.abs_sum) if a.kind == "avg" else int(v))
            keys = self.by_pane.setdefault(pane, {})
            old = keys.get(k)
            keys[k] = new if old is None else self._merge(old, new)

    def _merge(self, x, y):
        out = [x[0] + y[0]]
        for i, a in enumerate(self.aggs, 1):
            if a.kind == "min":
                out.append(min(x[i], y[i]))
            elif a.kind == "max":
                out.append(max(x[i], y[i]))
            elif a.kind == "avg":
                out.append((x[i][0] + y[i][0], x[i][1] + y[i][1]))
            else:  # count (unused: rows), sum (exact, wrapped on output)
                out.append(x[i] + y[i])
        return out

    def windows(self, starts, width, key_out):
        """Rows of the windows starting at `starts` (ascending) that hold at least one row, in (start, key) order."""
        per_key = {}
        for pane in sorted(self.by_pane):
            for k, st in self.by_pane[pane].items():
                per_key.setdefault(k, []).append((pane, st))
        starts = np.asarray(starts, dtype=object)
        rows = []
        for k, items in per_key.items():
            bins = [p for p, _ in items]
            i0 = [bisect.bisect_left(bins, s) for s in starts]
            i1 = [bisect.bisect_left(bins, s + width) for s in starts]
            pre = [list(itertools.accumulate((st[0] for _, st in items), initial=0))]
            mins = {}
            for i, a in enumerate(self.aggs, 1):
                if a.kind in ("min", "max"):
                    mins[i] = _RangeExtreme([st[i] for _, st in items], a.kind)
                    pre.append(None)
                elif a.kind == "avg":
                    pre.append((list(itertools.accumulate((st[i][0] for _, st in items), initial=0)),
                                list(itertools.accumulate((st[i][1] for _, st in items), initial=0))))
                else:
                    pre.append(list(itertools.accumulate((st[i] for _, st in items), initial=0)))
            for s, a0, a1 in zip(starts, i0, i1):
                if a1 <= a0:
                    continue
                n = pre[0][a1] - pre[0][a0]
                row = {"window_start": int(s), "window_end": int(s) + width, TIMESTAMP: int(s) + width - 1}
                if self.key_name:
                    row[self.key_name] = key_out(k)
                for i, a in enumerate(self.aggs, 1):
                    if a.kind == "count":
                        row[a.name] = n
                    elif a.kind == "sum":
                        row[a.name] = _wrap(pre[i][a1] - pre[i][a0])
                    elif a.kind == "avg":
                        ex, ab = pre[i]
                        row[a.name] = Mean(Fraction(ex[a1] - ex[a0], n), ab[a1] - ab[a0])
                    else:
                        row[a.name] = mins[i].query(a0, a1)
                rows.append(row)
        rows.sort(key=lambda r: (r["window_start"], -1 if r.get(self.key_name) is None else r[self.key_name]))
        return rows

    def prune(self, below: int):
        for p in [p for p in self.by_pane if p < below]:
            del self.by_pane[p]


def _wrap(x: int) -> int:
    x &= (1 << 64) - 1
    return x - (1 << 64) if x >= 1 << 63 else x


class _RangeExtreme:
    """MIN or MAX over index ranges [i0, i1) of a list: a sparse table."""

    def __init__(self, vals, kind):
        self.f = min if kind == "min" else max
        self.levels = [list(vals)]
        j = 1
        while 2 * j <= len(vals):
            prev = self.levels[-1]
            self.levels.append([self.f(prev[i], prev[i + j]) for i in range(len(prev) - j)])
            j *= 2

    def query(self, i0, i1):
        lv = (i1 - i0).bit_length() - 1
        t = self.levels[lv]
        return self.f(t[i0], t[i1 - (1 << lv)])


def window_emissions(events, key_name, aggs, width, slide=None):
    """The event-time behaviour of the tumbling (slide None) and sliding window aggregates, from these rules
    (tumbling_aggregating_window.rs:282-291 and :321-392, sliding_aggregating_window.rs:631-633 and :676-691):

    * bin(t) = t - t mod slide with floor division (tumbling: slide = width);
    * a row is late iff bin(ts) < bin(w) for the last watermark w before its batch; before the first watermark nothing
      is late; a late row counts in no window;
    * an on-time row belongs to the windows starting at bin(ts) - k * slide, 0 <= k < width / slide;
    * watermark w emits, in ascending window_start, every window that holds an on-time row, has not been emitted
      and ends at or before bin(w) (start + width <= bin(w)); end of data is INT64_MAX;
    * a restart (checkpoint, new operator, on_start) changes nothing.

    `events`: ("batch", cols), ("wm", w) or ("restart",); watermarks must not decrease.  Returns (one
    {(window_start, key or None): row} per watermark, in emission order, the number of late rows)."""
    slide = slide or width
    assert width % slide == 0 and slide > 0
    panes = _Panes(key_name, aggs, slide)
    last_wm, bound, late = None, None, 0
    dtype = None
    out = []
    for ev in events:
        if ev[0] == "restart":
            continue
        if ev[0] == "batch":
            cols = {c: np.asarray(v) for c, v in _columns(ev[1]).items()}
            ts = cols[TIMESTAMP].astype(np.int64)
            if key_name and len(ts):
                dtype = cols[key_name].dtype
            keep = np.ones(len(ts), dtype=bool)
            if last_wm is not None:
                keep = (ts - ts % np.int64(slide)) >= _bin(last_wm, slide)
            late += int((~keep).sum())
            panes.add({c: v[keep] for c, v in cols.items()}, ts[keep])
            continue
        assert ev[0] == "wm", ev
        w = min(int(ev[1]), INT64_MAX)
        if last_wm is not None and w < last_wm:
            raise ValueError("watermarks must not decrease")
        last_wm = w
        new_bound = _bin(w, slide)
        lo = None if bound is None else bound - width  # windows starting at or below lo were emitted
        hi = new_bound - width
        # the windows a pane belongs to start in [pane - width + slide, pane]: merge those runs, keep (lo, hi]
        starts, run = [], None
        for pane in sorted(panes.by_pane):
            a, b = pane - width + slide, min(pane, hi)
            if lo is not None:
                a = max(a, lo + slide)
            if a > b:
                continue
            if run is not None and a <= run[1] + slide:
                run[1] = max(run[1], b)
                continue
            if run is not None:
                starts.extend(range(run[0], run[1] + 1, slide))
            run = [a, b]
        if run is not None:
            starts.extend(range(run[0], run[1] + 1, slide))
        key_out = (lambda k: int(np.int64(k).view(np.uint64))) if dtype == np.uint64 else int
        rows = panes.windows(starts, width, key_out)
        out.append({(r["window_start"], r[key_name] if key_name else None): r for r in rows})
        bound = new_bound if bound is None else max(bound, new_bound)
        panes.prune(bound - width + 1)
    return out, late


def updating_rows(batches, key_name, aggs):
    """Final per-key state of the updating aggregate after the last flush: {key or None: {column: value}} with
    _timestamp = max(_timestamp) of the key's rows and AVG as a Mean carrying the sequential f64 mean."""
    cols = _concat(batches)
    n_rows = len(cols[TIMESTAMP])
    key = cols[key_name] if key_name else np.zeros(n_rows, dtype=np.int64)
    uniq, inv, n = _group_keys(key)
    vals = _aggregate(cols, inv, n, aggs, order=True)
    ts = np.full(n, np.iinfo(np.int64).min, dtype=np.int64)
    np.maximum.at(ts, inv, cols[TIMESTAMP].astype(np.int64))
    out = {}
    for g in range(n):
        kv = None
        if key_name:
            kv = int(np.int64(uniq[0, g]).view(np.uint64)) if key.dtype == np.uint64 else int(uniq[0, g])
        row = {TIMESTAMP: int(ts[g])}
        if key_name:
            row[key_name] = kv
        for a in aggs:
            row[a.name] = vals[a.name][g]
        out[kv] = row
    return out


def _batch_partials(cols, key_name, aggs):
    """{key or None: [rows, state per aggregate, max ts]} of one batch's rows.  A state is the exact sum (SUM), the
    value (MIN / MAX) or [exact sum, sum of |x|] (AVG); COUNT uses `rows`."""
    ts = np.asarray(cols[TIMESTAMP]).astype(np.int64)
    n = len(ts)
    if n == 0:
        return {}
    key = np.asarray(cols[key_name]) if key_name else np.zeros(n, dtype=np.int64)
    uniq, inv, n_groups = _group_keys(key)
    count = np.bincount(inv, minlength=n_groups)
    tmax = np.full(n_groups, np.iinfo(np.int64).min, dtype=np.int64)
    np.maximum.at(tmax, inv, ts)
    per_agg = []
    for a in aggs:
        if a.kind == "count":
            per_agg.append(None)
            continue
        v = np.ascontiguousarray(cols[a.col]).astype(np.int64, copy=False)
        if a.kind in ("sum", "avg"):
            signed, abs_sum = _exact_sums(v, inv, n_groups)
            per_agg.append(signed if a.kind == "sum" else list(zip(signed, abs_sum)))
        else:
            ii = np.iinfo(np.int64)
            s = np.full(n_groups, ii.max if a.kind == "min" else ii.min, dtype=np.int64)
            (np.minimum if a.kind == "min" else np.maximum).at(s, inv, v)
            per_agg.append(s.tolist())
    keys = [None] * n_groups
    if key_name:
        keys = uniq[0].view(np.uint64).tolist() if key.dtype == np.uint64 else uniq[0].tolist()
    out = {}
    counts, tmaxs = count.tolist(), tmax.tolist()
    for g in range(n_groups):
        st = [counts[g]]
        for a, vals in zip(aggs, per_agg):
            st.append(None if vals is None else (list(vals[g]) if a.kind == "avg" else vals[g]))
        st.append(tmaxs[g])
        out[keys[g]] = st
    return out


def _merge_state(old, new, aggs):
    if old is None:
        return new
    out = [old[0] + new[0]]
    for i, a in enumerate(aggs, 1):
        x, y = old[i], new[i]
        out.append(None if a.kind == "count" else min(x, y) if a.kind == "min" else max(x, y) if a.kind == "max"
                   else [x[0] + y[0], x[1] + y[1]] if a.kind == "avg" else x + y)
    out.append(max(old[-1], new[-1]))
    return out


def _state_row(st, key, key_name, aggs):
    row = {TIMESTAMP: st[-1]}
    if key_name:
        row[key_name] = key
    for i, a in enumerate(aggs, 1):
        if a.kind == "count":
            row[a.name] = st[0]
        elif a.kind == "sum":
            row[a.name] = _wrap(st[i])
        elif a.kind == "avg":
            row[a.name] = Mean(Fraction(st[i][0], st[0]), st[i][1])
        else:
            row[a.name] = st[i]
    return row


def updating_changes(events, key_name, aggs):
    """The updating (non-windowed GROUP BY) aggregate's change stream, flush by flush, from these rules
    (incremental_aggregator.rs:637-738, :826-883), over append-only rows:

    * state_f(k) is the aggregates of every row of key k received before flush f, and `_timestamp` = the max of those
      rows' timestamps.  COUNT is exact, SUM wraps at 64 bits, MIN and MAX are exact, AVG is a Mean;
    * k is touched at flush f if at least one of its rows arrived since flush f - 1 (the start, for the first flush);
    * only touched keys appear in flush f.  A key that had no rows at flush f - 1 gets an append of state_f only.
      Otherwise, if any output other than `_timestamp` differs between state_{f-1} and state_f, it gets a retraction
      of state_{f-1} (its `_timestamp` included) and an append of state_f; else it is suppressed;
    * AVG counts as changed when the correctly rounded f64 means (float of the exact mean) differ;
    * the retraction carries state_{f-1} even when flush f - 1 suppressed the key: its `_timestamp` moved then, and
      the reference reads its "before" values at the key's first touch after flush f - 1.

    With a key whose sum of |x| reaches 2^53, put COUNT in the plan: the operators sum AVG inputs in f64, in an order
    the caller does not control, so suppression must not depend on an AVG alone.

    `events`: ("batch", cols) and ("flush",).  Returns one (retractions, appends) per flush, each {key or None: row}
    with the key column (keyed), every aggregate (AVG as a Mean) and `_timestamp`."""
    def outputs(st):
        return tuple(st[0] if a.kind == "count" else float(Fraction(st[i][0], st[0])) if a.kind == "avg"
                     else _wrap(st[i]) if a.kind == "sum" else st[i] for i, a in enumerate(aggs, 1))

    state, before, out = {}, {}, []
    for ev in events:
        if ev[0] == "batch":
            for k, part in _batch_partials(_columns(ev[1]), key_name, aggs).items():
                old = state.get(k)
                if k not in before:
                    before[k] = old  # the values at the previous flush (None: the key had no rows)
                state[k] = _merge_state(old, part, aggs)
            continue
        assert ev[0] == "flush", ev
        retract, append = {}, {}
        for k, old in before.items():
            new = state[k]
            if old is not None:
                if outputs(old) == outputs(new):
                    continue
                retract[k] = _state_row(old, k, key_name, aggs)
            append[k] = _state_row(new, k, key_name, aggs)
        out.append((retract, append))
        before = {}
    return out


def mismatches(want: dict, got_rows, key_of):
    """Compares output rows (dicts) with `want` ({group: row}); `key_of(row)` gives a row's group.  Integer columns
    must be equal, AVG columns must pass `check_avg`.  Returns a list of readable differences (empty: all equal)."""
    errs = []
    seen = set()
    for r in got_rows:
        g = key_of(r)
        if g in seen:
            errs.append(f"group {g} emitted twice")
            continue
        seen.add(g)
        w = want.get(g)
        if w is None:
            errs.append(f"unexpected group {g}: {r}")
            continue
        for c, wv in w.items():
            if c not in r:
                errs.append(f"group {g}: column {c} missing")
            elif isinstance(wv, Mean):
                if not check_avg(r[c], wv):
                    errs.append(f"group {g}: {c} = {float(r[c])!r}, want {wv}")
            elif int(r[c]) != wv:
                errs.append(f"group {g}: {c} = {r[c]}, want {wv}")
    for g in want.keys() - seen:
        errs.append(f"missing group {g}")
    return errs


# ---- joins ------------------------------------------------------------------------------------------------------
# A join input batch is a mapping {column name: numpy array of a 64-bit type} in schema order (or anything with such
# a mapping as `.cols`).  Keys are grouped by their Python value (`tolist()`: Int64 signed, UInt64 unsigned), every
# other value travels as its 64-bit pattern, so Float64 payloads keep NaN payloads and -0.0 and UInt64 values >= 2^63
# stay exact.  Output columns: the left side's columns that are neither routing nor `_timestamp`, then the right
# side's (a name the left side already has gets `_right`), then `_timestamp`.
INT64_MAX = (1 << 63) - 1


def _columns(batch):
    return batch.cols if hasattr(batch, "cols") else batch


def _bits(a) -> np.ndarray:
    a = np.ascontiguousarray(a)
    if a.dtype.itemsize != 8:
        raise TypeError(f"join columns are 64-bit, got {a.dtype}")
    return a.view(np.uint64)


class Rows:
    """A multiset of join output rows: `names`, `vals` ((n, k) uint64, each value's 64-bit pattern, 0 where null) and
    `valid` ((n, k) bool)."""

    def __init__(self, names, vals, valid):
        self.names = list(names)
        k = len(self.names)
        self.vals = np.asarray(vals, dtype=np.uint64).reshape(-1, k)
        self.valid = np.asarray(valid, dtype=bool).reshape(self.vals.shape)
        self.vals = np.where(self.valid, self.vals, np.uint64(0))

    @classmethod
    def from_columns(cls, names, cols, valid=None):
        """`cols`: one 64-bit array per name; `valid`: {name: bool array} for the columns that have nulls."""
        valid = valid or {}
        n = len(cols[0]) if cols else 0
        vals = np.stack([_bits(c) for c in cols], axis=1) if n else np.zeros((0, len(names)), np.uint64)
        ok = np.stack([np.asarray(valid[c], bool) if c in valid else np.ones(n, bool) for c in names], axis=1) \
            if n else np.zeros((0, len(names)), bool)
        return cls(names, vals, ok)

    def __len__(self):
        return len(self.vals)

    def tuples(self, rows=None):
        idx = range(len(self)) if rows is None else rows
        return [tuple(int(v) if ok else None for v, ok in zip(self.vals[i], self.valid[i])) for i in idx]

    def _sorted(self):
        """Rows as one (n, k + 1) array [values, validity bits] in a canonical order: by a 64-bit fingerprint of the
        row.  Equal rows have equal fingerprints, so two equal multisets sort to equal arrays; the comparison itself is
        on the full rows (a fingerprint collision can only make equal multisets compare unequal)."""
        bits = (self.valid.astype(np.uint64) << np.arange(self.valid.shape[1], dtype=np.uint64)).sum(axis=1, dtype=np.uint64)
        a = np.concatenate([self.vals, bits[:, None]], axis=1)
        h = np.full(len(a), 0xCBF29CE484222325, dtype=np.uint64)
        with np.errstate(over="ignore"):
            for c in range(a.shape[1]):
                h = (h ^ a[:, c]) * np.uint64(0x100000001B3)
                h ^= h >> np.uint64(29)
            h = (h ^ (h >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
            h ^= h >> np.uint64(31)
        return a[np.argsort(h)]


def join_mismatches(want: Rows, got: Rows, limit: int = 10):
    """Differences between two multisets of rows (empty: equal)."""
    if want.names != got.names:
        return [f"columns {got.names}, want {want.names}"]
    a, b = want._sorted(), got._sorted()
    if a.shape == b.shape and np.array_equal(a, b):
        return []
    from collections import Counter
    cw, cg = Counter(want.tuples()), Counter(got.tuples())
    errs = [f"{len(got)} rows, want {len(want)}"]
    errs += [f"missing {r} x{n}" for r, n in (cw - cg).items()][:limit]
    errs += [f"unexpected {r} x{n}" for r, n in (cg - cw).items()][:limit]
    return errs


class _JoinSide:
    """The rows one join input has sent so far: payload bits, timestamps and key values, by arrival number."""

    def __init__(self, on, routing):
        self.on, self.routing = on, tuple(routing)
        self.names = None
        self.chunks, self.ts, self.keys = [], [], []
        self._vals = None

    def add(self, batch):
        cols = _columns(batch)
        names = [c for c in cols if c not in self.routing and c != TIMESTAMP]
        if self.names is None:
            self.names = names
        first = len(self.ts)
        if len(cols[TIMESTAMP]):
            self.chunks.append(np.stack([_bits(cols[c]) for c in names], axis=1))
        self.ts += np.asarray(cols[TIMESTAMP]).astype(np.int64).tolist()
        self.keys += np.asarray(cols[self.on]).tolist()
        self._vals = None
        return range(first, len(self.ts))

    def vals(self):
        if self._vals is None:
            self._vals = np.concatenate(self.chunks) if self.chunks else np.zeros((0, len(self.names or [])), np.uint64)
        return self._vals


def _output(sides, li, ri):
    """Gathers the output rows of the (left row, right row) pairs (-1: that side is null)."""
    lnames = sides[0].names or []
    rnames = sides[1].names or []
    names = list(lnames)
    for c in rnames:
        names.append(c if c not in names else c + "_right")
    names.append(TIMESTAMP)
    li = np.asarray(li, dtype=np.int64)
    ri = np.asarray(ri, dtype=np.int64)
    n = len(li)
    parts, ok = [], []
    lts = np.full(n, np.iinfo(np.int64).min, dtype=np.int64)
    rts = lts.copy()
    for side, idx, tsv in ((sides[0], li, lts), (sides[1], ri, rts)):
        k = len(side.names or [])
        has = idx >= 0
        v = np.zeros((n, k), dtype=np.uint64)
        if has.any():
            v[has] = side.vals()[idx[has]]
            tsv[has] = np.asarray(side.ts, dtype=np.int64)[idx[has]]
        parts.append(v)
        ok.append(np.repeat(has[:, None], k, axis=1))
    parts.append(np.maximum(lts, rts).view(np.uint64)[:, None])  # a null side's timestamp is INT64_MIN
    ok.append(np.ones((n, 1), dtype=bool))
    return Rows(names, np.concatenate(parts, axis=1), np.concatenate(ok, axis=1))


def _cross(pairs_l, pairs_r, ls, rs):
    """Appends every (l, r) pair of two lists of row numbers, l-major."""
    pairs_l.append(np.repeat(np.asarray(ls, dtype=np.int64), len(rs)))
    pairs_r.append(np.tile(np.asarray(rs, dtype=np.int64), len(ls)))


def instant_join(events, join_type, left_on, right_on, left_routing=(), right_routing=()):
    """The windowed join.  `events`: a sequence of (side, batch) with side 0 = left, 1 = right, and ("wm", w).  At
    each watermark w every buffered row with `_timestamp < w` joins the other side's rows with equal (`_timestamp`,
    key); in a left / right / full join a left / right row without a match leaves once with the other side null.
    Rows with `_timestamp >= w` stay buffered.  A batch with a row older than the last watermark raises ValueError
    (the reference panics).  Returns one Rows per watermark, in order."""
    keep = (join_type in ("left", "full"), join_type in ("right", "full"))
    sides = (_JoinSide(left_on, left_routing), _JoinSide(right_on, right_routing))
    buffered = ([], [])
    last_wm = None
    out = []
    for ev, arg in events:
        if ev != "wm":
            rows = sides[ev].add(arg)
            if last_wm is not None and any(sides[ev].ts[r] < last_wm for r in rows):
                raise ValueError("a row older than the watermark")
            buffered[ev].extend(rows)
            continue
        w = min(int(arg), INT64_MAX)
        groups = {}
        for s in (0, 1):
            ts, keys = sides[s].ts, sides[s].keys
            still = []
            for r in buffered[s]:
                if ts[r] < w:
                    groups.setdefault((ts[r], keys[r]), ([], []))[s].append(r)
                else:
                    still.append(r)
            buffered[s][:] = still
        pl, pr = [], []
        for ls, rs in groups.values():
            if ls and rs:
                _cross(pl, pr, ls, rs)
            elif ls and keep[0]:
                _cross(pl, pr, ls, [-1])
            elif rs and keep[1]:
                _cross(pl, pr, [-1], rs)
        cat = lambda p: np.concatenate(p) if p else np.zeros(0, np.int64)  # noqa: E731
        out.append(_output(sides, cat(pl), cat(pr)))
        last_wm = w
    return out


def expiring_join(events, left_on, right_on, left_routing=(), right_routing=()):
    """The join with expiration (inner, append-only inputs, no expiry inside a run).  `events`: a sequence of
    (side, batch).  Each arriving batch joins every earlier row of the other side with an equal key; `_timestamp` =
    max(left, right).  Returns one Rows per batch, in order."""
    sides = (_JoinSide(left_on, left_routing), _JoinSide(right_on, right_routing))
    by_key = ({}, {})
    out = []
    for s, batch in events:
        rows = sides[s].add(batch)
        mine = {}
        for r in rows:
            mine.setdefault(sides[s].keys[r], []).append(r)
        pn, po = [], []
        for k, new in mine.items():
            old = by_key[1 - s].get(k)
            if old:
                _cross(pn, po, new, old)
        for k, new in mine.items():
            by_key[s].setdefault(k, []).extend(new)
        cat = lambda p: np.concatenate(p) if p else np.zeros(0, np.int64)  # noqa: E731
        pn, po = cat(pn), cat(po)
        out.append(_output(sides, pn, po) if s == 0 else _output(sides, po, pn))
    return out


# ---- session windows --------------------------------------------------------------------------------------------
class _SessionAcc:
    """Exact running aggregates of one session: rows, and per value column (exact sum, sum of |x|, min, max)."""
    __slots__ = ("rows", "cols")

    def __init__(self, names):
        self.rows = 0
        self.cols = {c: [0, 0, None, None] for c in names}

    def add(self, cols, lo, hi):
        if hi <= lo:
            return
        self.rows += hi - lo
        for c, st in self.cols.items():
            v = cols[c][lo:hi]
            if len(v) <= 64:
                xs = v.tolist()
                s, a = sum(xs), sum(abs(x) for x in xs)
            else:
                sg, ab = _exact_sums(v, np.zeros(len(v), dtype=np.int64), 1)
                s, a = sg[0], ab[0]
            st[0] += s
            st[1] += a
            mn, mx = int(v.min()), int(v.max())
            st[2] = mn if st[2] is None else min(st[2], mn)
            st[3] = mx if st[3] is None else max(st[3], mx)

    def row(self, aggs):
        out = {}
        for a in aggs:
            if a.kind == "count":
                out[a.name] = self.rows
                continue
            s, ab, mn, mx = self.cols[a.col]
            out[a.name] = {"sum": lambda: _wrap(s), "min": lambda: mn, "max": lambda: mx,
                           "avg": lambda: Mean(Fraction(s, self.rows), ab)}[a.kind]()
        return out


class _SessionKey:
    """One key's state: the active session [ds, de, acc] or None, and the pending runs, a heap of (first ts, insertion
    number, ts, cols)."""
    __slots__ = ("active", "pending")

    def __init__(self):
        self.active, self.pending = None, []


def session_emissions(events, key_name, aggs, gap):
    """The session window aggregate's output, from these rules (session_aggregating_window.rs:60-279, :397-691,
    :802-925):

    Late rows and runs.  Once a watermark w has been seen, a row with ts < w is late; before the first watermark
    nothing is late.  A batch's on-time rows of one key, sorted by ts, form one run.  Each key keeps an optional
    active session (ds, de, rows taken) and pending runs ordered by (first ts, insertion order).

    add(run) under the last watermark w: insert the run; with no watermark yet, stop; if a session is active, fill;
    then advance(w), which must close nothing (the reference bails if it does).

    fill: while the smallest pending start is <= de + gap, pop every run with that start, in insertion order, and
    absorb each one; re-insert any remainder.

    absorb(t[0..n)): (1) if t[n-1] < de + gap, take all rows, de = max(de, t[n-1]), ds = min(ds, t[0]).  (2) Else if
    de + gap < t[0], the whole run is the remainder.  (3) Else ds = min(ds, t[0]) (t[0] < ds - gap is an error), and
    scan from i = 1: v = t[i], i += 1; if v < de continue; if v < de + gap, de = v and continue; otherwise break.  If
    i == n take all rows, else take t[0..i) and the remainder is t[i..n).  On this path the row that breaks the scan is
    taken without extending de, and the first row never extends de.

    advance(w): loop: an active session with de + gap < w closes (window_start = ds, window_end = de + gap,
    _timestamp = de + gap - 1) and the loop goes on; an active session otherwise stops it.  With no active session,
    stop if nothing is pending or w + gap < the smallest start; otherwise open a session with ds = de = that start
    and fill.

    Watermark w: advance only the keys whose next action is < w: de + gap for an active session, else the smallest
    pending start - gap.  So a pending start of exactly w + gap is not opened by the watermark, but by an add under
    the same w.  End of data is w = INT64_MAX.

    Restart.  Each batch's on-time rows are kept in table "s" under the batch's largest ts.  A checkpoint under
    watermark w drops the entries whose largest ts is below w - 100 gap.  On restore, start = the smallest on-time ts
    the operator accepted (table "e"; nothing is restored without one); the entries whose largest ts is
    >= start - 100 gap are replayed in ascending largest ts (ties in insertion order), each filtered to ts >= start
    and added as its own batch under watermark start; then the operator advances to the restored watermark and drops
    what that closes.  Unlike the window operators, a restart can change the results.

    Rows with equal ts inside one run are taken in an unspecified order: streams whose equal-ts rows carry different
    values on both sides of a break have no single answer.

    `events`: ("batch", cols), ("wm", w) or ("restart",); watermarks must not decrease.  Returns (one
    {(key or None, window_start): row} per watermark, the number of late rows, the number of distinct keys the last
    operator lifetime accepted rows for)."""
    names = sorted({a.col for a in aggs if a.kind != "count"})
    keys, table, out = {}, [], []
    st = {"w": None, "late": 0, "min": None, "n": 0, "keys": set()}

    def absorb(k, t, cols):
        a = k.active
        ds, de, acc = a
        n = len(t)
        if t[n - 1] < de + gap:
            a[0], a[1] = min(ds, int(t[0])), max(de, int(t[n - 1]))
            acc.add(cols, 0, n)
            return None
        if de + gap < t[0]:
            return 0
        if t[0] < ds - gap:
            raise ValueError("a run starts before data_start - gap")
        a[0] = min(ds, int(t[0]))
        i = 1
        while i < n:
            v = int(t[i])
            i += 1
            if v < de:
                continue
            if v < de + gap:
                de = v
                continue
            break
        a[1] = de
        acc.add(cols, 0, i)
        return None if i == n else i

    def push(k, t, cols):
        heapq.heappush(k.pending, (int(t[0]), st["n"], t, cols))
        st["n"] += 1

    def fill(k):
        while k.pending and k.pending[0][0] <= k.active[1] + gap:
            first, batch = k.pending[0][0], []
            while k.pending and k.pending[0][0] == first:
                batch.append(heapq.heappop(k.pending))
            for _, _, t, cols in batch:
                i = absorb(k, t, cols)
                if i is not None:
                    push(k, t[i:], {c: v[i:] for c, v in cols.items()})

    def advance(key, k, w, emit):
        while True:
            if k.active is not None:
                ds, de, acc = k.active
                if not de + gap < w:
                    return
                if emit is None:
                    raise ValueError("a session closed while adding a run")
                row = {"window_start": ds, "window_end": de + gap, TIMESTAMP: de + gap - 1, **acc.row(aggs)}
                if key_name:
                    row[key_name] = key
                assert (key, ds) not in emit
                emit[(key, ds)] = row
                k.active = None
                continue
            if not k.pending or w + gap < k.pending[0][0]:
                return
            s0 = k.pending[0][0]
            k.active = [s0, s0, _SessionAcc(names)]
            fill(k)

    def add_batch(cols, w):
        ts = np.asarray(cols[TIMESTAMP]).astype(np.int64)
        if not len(ts):
            return
        key = np.asarray(cols[key_name]) if key_name else np.zeros(len(ts), dtype=np.int64)
        kl = key.tolist()
        order = np.lexsort((ts, key.view(np.int64) if key.dtype == np.uint64 else key.astype(np.int64)))
        vals = {c: np.asarray(cols[c]).astype(np.int64)[order] for c in names}
        ts, kl = ts[order], [kl[i] for i in order.tolist()]
        m = int(ts.min())
        st["min"] = m if st["min"] is None else min(st["min"], m)
        lo = 0
        while lo < len(ts):
            hi = lo + 1
            while hi < len(ts) and kl[hi] == kl[lo]:
                hi += 1
            kv = kl[lo] if key_name else None
            st["keys"].add(kv)
            k = keys.setdefault(kv, _SessionKey())
            push(k, ts[lo:hi], {c: v[lo:hi] for c, v in vals.items()})
            if w is not None:
                if k.active is not None:
                    fill(k)
                advance(kv, k, w, None)
            lo = hi

    def next_action(k):
        if k.active is not None:
            return k.active[1] + gap
        return k.pending[0][0] - gap if k.pending else None

    def watermark(w, emit):
        for kv, k in keys.items():
            na = next_action(k)
            if na is not None and na < w:
                advance(kv, k, w, emit)

    for ev in events:
        if ev[0] == "batch":
            cols = {c: np.asarray(v) for c, v in _columns(ev[1]).items()}
            ts = cols[TIMESTAMP].astype(np.int64)
            keep = np.ones(len(ts), dtype=bool) if st["w"] is None else ts >= st["w"]
            st["late"] += int((~keep).sum())
            if not keep.any():
                continue
            cols = {c: v[keep] for c, v in cols.items()}
            table.append((int(cols[TIMESTAMP].astype(np.int64).max()), len(table), cols))
            add_batch(cols, st["w"])
        elif ev[0] == "wm":
            w = min(int(ev[1]), INT64_MAX)
            if st["w"] is not None and w < st["w"]:
                raise ValueError("watermarks must not decrease")
            st["w"] = w
            emit = {}
            watermark(w, emit)
            out.append(emit)
        else:
            assert ev[0] == "restart", ev
            w, start = st["w"], st["min"]
            if w is not None:
                table = [e for e in table if e[0] >= w - 100 * gap]
            keys.clear()
            st["keys"], st["min"] = set(), None
            if start is None:
                continue
            for _, _, cols in sorted((e for e in table if e[0] >= start - 100 * gap), key=lambda e: (e[0], e[1])):
                keep = cols[TIMESTAMP].astype(np.int64) >= start
                if keep.any():
                    add_batch({c: v[keep] for c, v in cols.items()}, start)
            if w is not None:
                watermark(w, {})
    return out, st["late"], len(st["keys"])


def session_chains(events, key_name, gap):
    """The declarative form of a session, for streams without restarts, with at most one row per key per batch and
    no two rows of a key exactly `gap` apart: every session is a maximal chain of a key's on-time rows whose
    consecutive distances are < gap.  Returns {(key or None, first ts): (last ts + gap, rows)}."""
    w, per_key = None, {}
    for ev in events:
        if ev[0] == "wm":
            w = min(int(ev[1]), INT64_MAX)
            continue
        assert ev[0] == "batch", ev
        cols = _columns(ev[1])
        ts = np.asarray(cols[TIMESTAMP]).astype(np.int64).tolist()
        ks = np.asarray(cols[key_name]).tolist() if key_name else [None] * len(ts)
        for k, t in zip(ks, ts):
            if w is None or t >= w:
                per_key.setdefault(k, []).append(t)
    out = {}
    for k, ts in per_key.items():
        ts.sort()
        first = 0
        for i in range(1, len(ts) + 1):
            if i == len(ts) or ts[i] - ts[i - 1] >= gap:
                out[(k, ts[first])] = (ts[i - 1] + gap, i - first)
                first = i
    return out
