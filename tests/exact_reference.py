"""Exact group-by reference for the window and updating aggregates, computed straight from the raw input rows with
numpy and Python integers.  It shares no code or arithmetic with oracle/, so it can catch mistakes the oracle and
the CUDA operators would make together (an AVG taken over a wrapped integer sum, a float32 or double-rounded mean).

AVG rule (`check_avg`): when the absolute values of a group's inputs sum to less than 2^53, every f64 or exact-integer
AVG path is exact up to its one final division, so the result must be bit-identical to the correctly rounded mean.
Otherwise |got - mean| <= 2u * sum|x| + 2u * |mean| with u = 2^-53: that is n * 2u * sum|x| on the sum, the error
bound of an f64 sum of n terms in any order including the rounding of each input, divided by n, plus the final
division."""
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
    slide = slide or width
    assert width % slide == 0
    cols = _concat(batches)
    ts = cols[TIMESTAMP].astype(np.int64)
    first = ts - ts % np.int64(slide)
    reps = width // slide
    starts = np.concatenate([first - np.int64(k * slide) for k in range(reps)])
    rows = np.tile(np.arange(len(ts)), reps)
    expanded = {c: v[rows] for c, v in cols.items()}
    key = expanded[key_name] if key_name else np.zeros(len(rows), dtype=np.int64)
    uniq, inv, n = _group_keys(key, starts)
    vals = _aggregate(expanded, inv, n, aggs)
    out = {}
    for g in range(n):
        ws = int(uniq[0, g])
        kv = None
        if key_name:
            kv = int(np.int64(uniq[1, g]).view(np.uint64)) if cols[key_name].dtype == np.uint64 else int(uniq[1, g])
        row = {"window_start": ws, "window_end": ws + width, TIMESTAMP: ws + width - 1}
        if key_name:
            row[key_name] = kv
        for a in aggs:
            row[a.name] = vals[a.name][g]
        out[(ws, kv)] = row
    return out


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
