"""Checkpoint and restore of the tumbling, sliding and instant-window aggregates at the value extremes, against the exact
references (tests/exact_reference.window_emissions, where a restart changes nothing), watermark by watermark.

The window aggregate keeps AVG in memory as an exact Int64 sum (shared with a SUM over the same column) until a value
reaches 2^31 or a window 2^32 rows, and then promotes itself to f64 accumulators; table "t" always holds an AVG as
[count] UInt64, [sum] Float64 and a SUM as [sum] Int64.  So a restart is where the two forms meet: a table written after
a promotion holds wrapped Int64 sums next to f64 sums of 2^53 and more, and a table written by the reference may hold
any count or sum.  The streams here restart before the first big value, right after a promotion, while the pane with
the big sums is still open, twice in a row, and after a sliding window has left while its panes are still stored; the
values come from four regimes (R1: |v| < 2^31; R2: INT64_MIN / INT64_MAX, sums of 2^62 that wrap and keys whose only
value is an identity; R3: values of 2^31 and more in one column; cancel: INT64_MAX and INT64_MIN in one group).

Besides the emissions, table "t" is compared with exact per-(pane, key) partials at every checkpoint; checkpoints cross
between the CUDA operator and the numpy oracle both ways; hand-written reference-format tables are restored directly;
and the oracle's own restarts are pinned to the reference on the CPU."""
import ctypes as C
import zlib
from fractions import Fraction

import numpy as np
import pytest

from oracle import arroyo_oracle as O
from tests import exact_reference as X
from tests.test_gpu_agg_plans import PLANS as WIDE

A = O.Agg
TS = O.TIMESTAMP
SEC = 1_000_000_000
ORIGIN = 1_700_000_000 * SEC
INT64_MIN, INT64_MAX = -(1 << 63), (1 << 63) - 1
INTS = [A("count", None, "n"), A("sum", "a", "sa"), A("avg", "a", "ava")]
PLANS = {
    "ints": INTS,                # COUNT, SUM(a), AVG(a): the AVG shares the SUM's accumulator while exact
    "ints_f64": INTS,            # the same with FLAG_AVG_F64: f64 AVG from the start (the control)
    "P2": WIDE["P2"],            # AVG(a) without a SUM over a
    "P5": WIDE["P5"],
    "P6b": WIDE["P6b"],
    "P7": WIDE["P7"],            # two AVGs: starts in f64 mode (no room for promotion)
    "minmax": [A("count", None, "n"), A("min", "a", "mna"), A("max", "a", "mxa"), A("sum", "a", "sa")],
}
# keys: three ordinary ones, then the ones that only get a special value in the big phase of R2: 2^62 (four of them wrap
# the Int64 sum to 0), INT64_MAX (MIN's identity) and INT64_MIN (MAX's identity)
KEYS = {"few": [-1, 0, 1, 5, 6, 7], "u64": [1 << 63, (1 << 64) - 1, 3, (1 << 63) + 5, (1 << 63) + 6, (1 << 63) + 7]}
SPECIAL = {3: 1 << 62, 4: INT64_MAX, 5: INT64_MIN}


# ---- streams ----------------------------------------------------------------------------------------------------------
class Stream:
    """Events ("batch", cols), ("wm", w), ("restart",) over value columns a..d.  Every regime starts calm (R1 values)
    until `big()`; from then on rows take the regime's values."""

    def __init__(self, seed, keys, regime, width, slide=None):
        self.rng = np.random.default_rng(seed)
        self.keys, self.regime, self.width, self.slide = keys, regime, width, slide or width
        self.o = ORIGIN - ORIGIN % self.slide
        self.loud = False
        self.events = []

    def big(self):
        self.loud = self.regime != "R1"

    def _values(self, kid, n):
        rng = self.rng
        cols = {c: rng.integers(-(1 << 31) + 1, 1 << 31, n).astype(np.int64) for c in "abcd"}
        if not self.loud:
            return cols
        if self.regime == "R2":
            pool = np.array([INT64_MIN, INT64_MAX, 1 << 62, (1 << 62) + 3, -(1 << 62), 0, -1, 1], dtype=np.int64)
            for c in "abcd":
                pick = rng.random(n) < 0.75
                cols[c][pick] = rng.choice(pool, int(pick.sum()))
                if kid is not None:
                    for k, v in SPECIAL.items():
                        cols[c][kid == k] = v
        elif self.regime == "R3":
            cols["a"] = rng.integers(1 << 31, 1 << 40, n).astype(np.int64) * rng.choice(np.array([-1, 1]), n)
        elif self.regime == "cancel":
            for c in "abcd":
                pick = rng.random(n) < 0.6
                cols[c][pick] = rng.choice(np.array([INT64_MIN, INT64_MAX], dtype=np.int64), int(pick.sum()))
        return cols

    def batch(self, ts):
        ts = np.asarray(ts, dtype=np.int64)
        n = len(ts)
        cols, kid = {}, None
        if self.keys != "none":
            kid = self.rng.integers(0, 6 if self.loud and self.regime == "R2" else 3, n)
            ks = KEYS[self.keys]
            cols["key"] = np.array([ks[i] for i in kid], dtype=np.uint64 if self.keys == "u64" else np.int64)
        cols.update(self._values(kid, n))
        cols[TS] = ts
        self.events.append(("batch", O.Batch(cols)))

    def rows(self, panes, per=3):
        s = self.slide
        ts = [self.o + p * s + int(x) for p in panes for x in self.rng.integers(0, s, per)]
        self.batch(self.rng.permutation(np.asarray(ts, dtype=np.int64)))

    def wm(self, w):
        self.events.append(("wm", int(w)))

    def restart(self):
        self.events.append(("restart",))

    def end(self):
        self.wm(INT64_MAX)
        return self


def sh_before(st):
    """A restart before the first big value: the restored operator is exact and promotes afterwards."""
    o, s = st.o, st.slide
    st.rows([0, 1, 2])
    st.wm(o + s)
    st.restart()
    st.big()
    st.rows([2, 3], per=6)
    st.rows([3, 4], per=6)
    st.wm(o + 3 * s + 1)
    st.rows([4, 5], per=4)
    return st.end()


def sh_after(st):
    """A restart right after a promotion: the table holds wrapped Int64 sums and f64 sums of 2^53 and 2^63 and more."""
    o, s = st.o, st.slide
    st.rows([0, 1])
    st.big()
    st.rows([1, 2], per=8)
    st.wm(o + s)
    st.restart()
    st.rows([2, 3], per=4)
    st.wm(o + 3 * s)
    st.rows([4])
    return st.end()


def sh_open(st):
    """The pane that holds the big sums is still open at the restart and takes more rows after it."""
    o, s = st.o, st.slide
    st.rows([0])
    st.wm(o)
    st.big()
    st.rows([1], per=8)
    st.rows([1], per=8)
    st.restart()
    st.rows([1, 2], per=8)
    st.wm(o + 2 * s)
    st.rows([2, 3])
    return st.end()


def sh_twice(st):
    """Two restarts in a row, then one more."""
    o, s = st.o, st.slide
    st.big()
    st.rows([0, 1], per=6)
    st.wm(o)
    st.restart()
    st.restart()
    st.rows([1, 2], per=6)
    st.restart()
    st.wm(o + 2 * s)
    st.rows([2, 3])
    return st.end()


def sh_left(st):
    """Sliding: windows have left, the panes they shared with open windows are still stored at the restart."""
    o, s = st.o, st.slide
    st.rows([0])
    st.big()
    st.rows([0, 1, 2], per=6)
    st.wm(o + 3 * s + 1)
    st.restart()
    st.rows([3, 4], per=6)
    st.wm(o + 5 * s)
    st.restart()
    st.rows([5])
    return st.end()


SHAPES = {"before": sh_before, "after": sh_after, "open": sh_open, "twice": sh_twice, "left": sh_left}


def make_stream(shape, kind, keys, regime):
    w, s = (4 * SEC, SEC) if kind != "tumbling" else (SEC, None)
    seed = zlib.crc32(f"{shape}/{kind}/{keys}/{regime}".encode()) % 10_000
    return SHAPES[shape](Stream(seed, keys, regime, w, s))


def config(st, kind, plan):
    key_names = [] if st.keys == "none" else ["key"]
    return O.WindowAggConfig(width=st.width, slide=st.slide if kind != "tumbling" else 0, key_names=key_names,
                             aggs=PLANS[plan], window_index=len(key_names))


def reference(st, cfg):
    return X.window_emissions(st.events, cfg.key_names[0] if cfg.key_names else None, cfg.aggs, cfg.width,
                              cfg.slide or None)


# ---- exact partials of table "t" -----------------------------------------------------------------------------------
class Partials:
    """Exact per-(pane, key) partial states of the on-time rows so far (exact_reference._Panes), with the same lateness
    rule as window_emissions."""

    def __init__(self, cfg):
        self.key = cfg.key_names[0] if cfg.key_names else None
        self.aggs, self.width, self.slide = list(cfg.aggs), cfg.width, cfg.slide or cfg.width
        self.panes = X._Panes(self.key, self.aggs, self.slide)
        self.last_wm = None

    def batch(self, b):
        cols = {c: np.asarray(v) for c, v in b.cols.items()}
        ts = cols[TS].astype(np.int64)
        keep = np.ones(len(ts), dtype=bool)
        if self.last_wm is not None:
            keep = (ts - ts % np.int64(self.slide)) >= self.last_wm - self.last_wm % self.slide
        self.panes.add({c: v[keep] for c, v in cols.items()}, ts[keep])

    def wm(self, w):
        self.last_wm = min(int(w), INT64_MAX)

    def live(self):
        """Panes whose windows have not all been emitted."""
        if self.last_wm is None:
            return set(self.panes.by_pane)
        bound = self.last_wm - self.last_wm % self.slide
        return {p for p in self.panes.by_pane if p + self.width > bound}


def merged_table(table, key):
    """[(pane, O.Batch)] -> {pane: {key (Int64 view): {column: value}}}: counts and sums added (Int64 sums wrapping, f64
    sums as f64), MIN / MAX folded."""
    out = {}
    for t, b in table:
        names = [c for c in b.cols if c not in (key, TS)]
        for i in range(b.num_rows):
            assert int(b[TS][i]) == t
            k = int(np.asarray(b[key])[i:i + 1].view(np.int64)[0]) if key else 0
            row = out.setdefault(t, {}).setdefault(k, {})
            for c in names:
                v = b[c][i]
                if c not in row:
                    row[c] = float(v) if b[c].dtype.kind == "f" else int(v)
                elif c.endswith("[min]"):
                    row[c] = min(row[c], int(v))
                elif c.endswith("[max]"):
                    row[c] = max(row[c], int(v))
                elif b[c].dtype.kind == "f":
                    row[c] = row[c] + float(v)
                else:
                    row[c] = X._wrap(row[c] + int(v)) if b[c].dtype == np.int64 else row[c] + int(v)
    return out


def check_table(table, part, who):
    """Every live pane's merged state equals the exact partials: [count], Int64 [sum] (wrapping), [min] and [max]
    exactly, the Float64 [sum] bit for bit while the group's sum of |x| is below 2^53, else within the f64 summation
    bound 2u * n * sum|x|."""
    got = merged_table(table, part.key)
    live = part.live()
    for pane in sorted(live):
        want = part.panes.by_pane[pane]
        g = got.get(pane, {})
        assert sorted(g) == sorted(want), (who, "pane", pane, sorted(set(g) ^ set(want))[:6])
        for k, st in want.items():
            rows, cols = st[0], g[k]
            for i, a in enumerate(part.aggs, 1):
                if a.kind == "count":
                    assert cols[f"{a.name}[count]"] == rows, (who, pane, k, a.name)
                elif a.kind == "sum":
                    assert cols[f"{a.name}[sum]"] == X._wrap(st[i]), (who, pane, k, a.name, cols, st[i])
                elif a.kind in ("min", "max"):
                    assert cols[f"{a.name}[{a.kind}]"] == st[i], (who, pane, k, a.name)
                else:
                    exact, abs_sum = st[i]
                    assert cols[f"{a.name}[count]"] == rows, (who, pane, k, a.name)
                    f = cols[f"{a.name}[sum]"]
                    if abs_sum < 2 ** 53:
                        assert f == float(exact), (who, pane, k, a.name, f, exact)
                    else:
                        err = abs(Fraction(f) - exact)
                        assert err <= Fraction(2 * X.U) * rows * abs_sum, (who, pane, k, a.name, f, exact)


# ---- drivers ----------------------------------------------------------------------------------------------------------
class _Ptr:
    def __init__(self, ptr, n, typestr):
        self.__cuda_array_interface__ = {"shape": (n,), "typestr": typestr, "data": (ptr, False), "version": 2}


class GpuSegment:
    """One CUDA operator between two restarts, fed through `entry`."""

    def __init__(self, st, kind, cfg, entry, flags, table, last_wm, expected_keys=64):
        import arroyo_b200 as ab
        from arroyo_b200 import ffi, operators as native
        from tests.gpu_ops import to_arrow
        self.ab, self.ffi, self.st, self.cfg, self.entry = ab, ffi, st, cfg, entry
        fl = flags | {"remerge": ffi.FLAG_REMERGE_ONLY}.get(kind, 0)
        fl |= {"two_pass": ffi.FLAG_TWO_PASS_ALWAYS, "one_pass": ffi.FLAG_NO_TWO_PASS}.get(entry, 0)
        cls = native.TumblingAggregatingWindowFunc if kind == "tumbling" else native.SlidingAggregatingWindowFunc
        first = next(ev[1] for ev in st.events if ev[0] == "batch")
        self.names = list(first.cols)
        self.op = cls(cfg, input_schema=to_arrow(first).schema, flags=fl, expected_keys=expected_keys)
        self.ctx = ab.OperatorContext(1)
        if last_wm is not None:
            self.ctx.watermarks.set(0, last_wm)
        t = self.ctx.table("t", cfg.width)
        for ts, b in table:
            t.insert(ts, to_arrow(b))
        self.op.on_start(self.ctx)
        self.keep, self.pending = [], []

    def _host_rows(self, batches):
        from tests.gpu_ops import from_arrow
        return [r for b in batches for r in from_arrow(b).rows()]

    def _dev_rows(self, wins):
        import torch
        names = list(self.cfg.key_names) + ["window_start", "window_end"] + [a.name for a in self.cfg.aggs] + [TS]
        rows = []
        for n, ptrs in wins:
            host = {c: torch.as_tensor(_Ptr(p, n, "<f8" if c.startswith("av") else "<i8"), device="cuda").cpu().numpy()
                    for c, p in zip(names, ptrs)}
            if self.st.keys == "u64":
                host["key"] = host["key"].view(np.uint64)
            rows += O.Batch(host).rows()
        return rows

    def _run_pending(self, wm):
        from arroyo_b200 import operators as native
        from tests.gpu_ops import to_arrow
        if not self.pending:
            return []
        ex = native.ExportedBatches([to_arrow(b) for b in self.pending])
        wms = (C.c_int64 * len(self.pending))(*([self.ffi.NO_WATERMARK] * (len(self.pending) - 1) + [wm]))
        col = self.ab.Collector()
        self.op.run_batches(ex, wms, col)
        self.op.handle_watermark_poll(col, block=True)
        self.pending.clear()
        return col.batches

    def batch(self, b):
        import torch
        from tests.gpu_ops import to_arrow
        e = self.entry
        if e == "run_batches":
            self.pending.append(b)
        elif e == "sliced":
            rb, s, i = to_arrow(b), 0, 0
            while s < b.num_rows:
                z = min((1, 7, 1023, 2)[i % 4], b.num_rows - s)
                self.op.process_batch(rb.slice(s, z), self.ctx, None)
                s, i = s + z, i + 1
        elif e in ("device", "poll"):
            dev = [torch.from_numpy(np.ascontiguousarray(b[c]).view(np.int64)).cuda() for c in self.names]
            self.keep.append(dev)
            self.op.process_device_batch([t.data_ptr() for t in dev], b.num_rows)
        else:
            self.op.process_batch(to_arrow(b), self.ctx, None)

    def wm(self, w):
        from arroyo_b200.context import clamp_watermark
        self.ctx.watermarks.set(0, w)
        if self.entry == "run_batches" and self.pending:
            return self._host_rows(self._run_pending(clamp_watermark(w)))
        if self.entry == "device":
            return self._dev_rows(self.op.handle_watermark_device(w))
        if self.entry == "poll":
            self.op.handle_watermark_device_begin(w)
            return self._dev_rows(self.op.handle_watermark_device_poll())
        col = self.ab.Collector()
        self.op.handle_watermark(w, self.ctx, col)
        return self._host_rows(col.batches)

    def checkpoint(self):
        """Checkpoints; returns table "t" as [(pane, O.Batch)] (every batch written so far)."""
        from tests.gpu_ops import from_arrow
        if self.pending:
            assert not self._run_pending(self.ffi.NO_WATERMARK)
        self.op.handle_checkpoint(None, self.ctx, None)
        t = self.ctx.table("t", self.cfg.width)
        return [(ts, from_arrow(b)) for ts in sorted(t.batches) for b in t.batches[ts]]

    def close(self):
        s = self.op.stats()
        self.op.close()
        return s


class OracleSegment:
    """The numpy oracle between two restarts."""

    def __init__(self, st, kind, cfg, table, last_wm):
        cls = O.TumblingAggregatingWindowFunc if kind == "tumbling" else O.SlidingAggregatingWindowFunc
        self.cfg, self.op, self.ctx = cfg, cls(cfg), O.OperatorContext(1)
        if last_wm is not None:
            self.ctx.watermarks.set(0, last_wm)
        t = self.ctx.table("t", cfg.width)
        for ts, b in table:
            t.flushed.setdefault(ts, []).append(b)
        self.op.on_start(self.ctx)

    def batch(self, b):
        self.op.process_batch(b, self.ctx, O.Collector())

    def wm(self, w):
        self.ctx.watermarks.set(0, w)
        col = O.Collector()
        self.op.handle_watermark(w, self.ctx, col)
        return [r for b in col.batches for r in b.rows()]

    def checkpoint(self):
        self.op.handle_checkpoint(self.ctx)
        t = self.ctx.table("t", self.cfg.width)
        return [(ts, b) for d in (t.flushed, t.to_flush) for ts in sorted(d) for b in d[ts]]

    def close(self):
        return None


def run(st, kind, cfg, impls, entry="host", flags=0, tables=True):
    """Runs the events with one operator per segment between restarts, `impls[i]` ("gpu" or "oracle") for segment i;
    at a restart the table crosses to the next one.  With `tables`, table "t" is checked against the exact partials
    at every checkpoint.  Returns (one list of output rows per watermark, rows_in, rows_late) (the counts over the GPU
    segments)."""
    part = Partials(cfg)
    table, last_wm, outs, totals = [], None, [], [0, 0]

    def start(i):
        if impls[i] == "gpu":
            return GpuSegment(st, kind, cfg, entry, flags, table, last_wm)
        return OracleSegment(st, kind, cfg, table, last_wm)

    seg, i = start(0), 0
    for ev in st.events:
        if ev[0] == "batch":
            part.batch(ev[1])
            seg.batch(ev[1])
        elif ev[0] == "wm":
            part.wm(ev[1])
            last_wm = ev[1]
            outs.append(seg.wm(ev[1]))
        else:
            table = seg.checkpoint()
            if tables:
                check_table(table, part, f"{impls[i]} checkpoint {i}")
            s = seg.close()
            if s:
                totals[0] += s["rows_in"]
                totals[1] += s["rows_late"]
            i += 1
            seg = start(i)
    s = seg.close()
    if s:
        totals[0] += s["rows_in"]
        totals[1] += s["rows_late"]
    return outs, totals[0], totals[1]


def check_emissions(want, got, cfg, who):
    key = cfg.key_names[0] if cfg.key_names else None
    assert len(got) == len(want), (who, len(got), len(want))
    for i, (w, g) in enumerate(zip(want, got)):
        starts = [int(r["window_start"]) for r in g]
        assert starts == sorted(starts), (who, i, "windows out of order")
        errs = X.mismatches(w, g, lambda r: (int(r["window_start"]), int(r[key]) if key else None))
        assert not errs, (who, "watermark", i, errs[:8])


def n_segments(st):
    return 1 + sum(ev[0] == "restart" for ev in st.events)


# ---- the window aggregates across restarts ---------------------------------------------------------------------------
# (shape, window kind, keys, plan, regime, entry): a cross section, not the product
CASES = [
    ("before", "tumbling", "few", "ints", "R3", "host"),
    ("before", "running", "few", "ints", "R2", "two_pass"),
    ("before", "remerge", "u64", "P5", "R3", "sliced"),
    ("before", "running", "none", "P6b", "R2", "device"),
    ("before", "tumbling", "few", "P2", "cancel", "one_pass"),
    ("before", "tumbling", "u64", "ints", "cancel", "host"),
    ("after", "tumbling", "few", "ints", "R2", "host"),
    ("after", "running", "few", "ints", "R2", "one_pass"),
    ("after", "remerge", "few", "ints", "R3", "two_pass"),
    ("after", "running", "few", "ints", "R1", "two_pass"),
    ("after", "tumbling", "u64", "P2", "R2", "host"),
    ("after", "running", "few", "P2", "R3", "poll"),
    ("after", "remerge", "none", "P5", "R2", "run_batches"),
    ("after", "tumbling", "few", "P6b", "cancel", "sliced"),
    ("after", "remerge", "u64", "P6b", "R3", "poll"),
    ("after", "running", "u64", "P7", "R2", "host"),
    ("after", "tumbling", "few", "minmax", "R2", "device"),
    ("after", "running", "few", "ints_f64", "R2", "host"),
    ("open", "tumbling", "few", "ints", "R2", "host"),
    ("open", "running", "few", "ints", "R2", "two_pass"),
    ("open", "running", "none", "ints", "R3", "device"),
    ("open", "remerge", "few", "P2", "R2", "device"),
    ("open", "tumbling", "u64", "P6b", "R3", "run_batches"),
    ("open", "running", "few", "P5", "cancel", "host"),
    ("open", "running", "few", "P7", "R3", "host"),
    ("open", "tumbling", "few", "ints_f64", "cancel", "poll"),
    ("open", "remerge", "few", "minmax", "R2", "sliced"),
    ("twice", "tumbling", "few", "ints", "R3", "one_pass"),
    ("twice", "running", "u64", "ints", "R2", "host"),
    ("twice", "remerge", "few", "P2", "cancel", "host"),
    ("twice", "tumbling", "none", "P7", "R2", "device"),
    ("twice", "running", "few", "P6b", "R2", "poll"),
    ("twice", "tumbling", "few", "minmax", "R2", "run_batches"),
    ("twice", "remerge", "few", "minmax", "R1", "host"),
    ("left", "running", "few", "ints", "R2", "host"),
    ("left", "remerge", "few", "ints", "R2", "host"),
    ("left", "running", "u64", "P2", "R2", "two_pass"),
    ("left", "remerge", "few", "P5", "R3", "device"),
    ("left", "running", "few", "P6b", "cancel", "sliced"),
    ("left", "remerge", "none", "P7", "R3", "host"),
    ("left", "running", "few", "ints_f64", "R2", "run_batches"),
]


def _flags(plan):
    from arroyo_b200 import ffi
    return ffi.FLAG_AVG_F64 if plan == "ints_f64" else 0


@pytest.mark.gpu
@pytest.mark.parametrize("shape,kind,keys,plan,regime,entry", CASES, ids=["-".join(c) for c in CASES])
def test_window_restart_at_extremes(shape, kind, keys, plan, regime, entry):
    st = make_stream(shape, kind, keys, regime)
    cfg = config(st, kind, plan)
    want, late = reference(st, cfg)
    got, rows_in, rows_late = run(st, kind, cfg, ["gpu"] * n_segments(st), entry, _flags(plan))
    check_emissions(want, got, cfg, "gpu")
    assert rows_in == sum(ev[1].num_rows for ev in st.events if ev[0] == "batch")
    assert rows_late == late


# ---- interchange with the oracle at the extremes ----------------------------------------------------------------------
INTERCHANGE = [("after", "tumbling", "ints", "R2"), ("open", "running", "P2", "R3"), ("after", "remerge", "P6b", "R2"),
               ("left", "running", "ints", "R3"), ("open", "tumbling", "P5", "cancel")]


@pytest.mark.gpu
@pytest.mark.parametrize("first", ["oracle", "gpu"])
@pytest.mark.parametrize("shape,kind,plan,regime", INTERCHANGE, ids=["-".join(c) for c in INTERCHANGE])
def test_interchange_with_oracle_at_extremes(shape, kind, plan, regime, first):
    """An oracle-written table "t" restores into the CUDA operator and a GPU-written one into the oracle; each run goes
    on to the uninterrupted result."""
    st = make_stream(shape, kind, "few", regime)
    cfg = config(st, kind, plan)
    want, _ = reference(st, cfg)
    other = {"oracle": "gpu", "gpu": "oracle"}[first]
    impls = [first if i % 2 == 0 else other for i in range(n_segments(st))]
    got, _, _ = run(st, kind, cfg, impls)
    check_emissions(want, got, cfg, "/".join(impls))


# ---- CPU: the oracle's restarts at the extremes ------------------------------------------------------------------------
ORACLE_CASES = [("after", "tumbling", "few", "ints", "R2"), ("open", "running", "few", "ints", "R2"),
                ("left", "running", "u64", "P2", "R3"), ("twice", "tumbling", "none", "P5", "cancel"),
                ("open", "tumbling", "few", "P6b", "R3"), ("after", "running", "few", "P7", "cancel"),
                ("left", "running", "few", "minmax", "R2"), ("before", "tumbling", "u64", "P2", "R2")]


@pytest.mark.parametrize("shape,kind,keys,plan,regime", ORACLE_CASES, ids=["-".join(c) for c in ORACLE_CASES])
def test_oracle_restart_at_extremes(shape, kind, keys, plan, regime):
    """The numpy oracle restarting at every restart of the stream gives window_emissions, and its table "t" holds the
    exact partials: the half of the interchange tests that relies on the oracle is itself pinned."""
    st = make_stream(shape, kind, keys, regime)
    cfg = config(st, kind, plan)
    want, _ = reference(st, cfg)
    got, _, _ = run(st, kind, cfg, ["oracle"] * n_segments(st))
    check_emissions(want, got, cfg, "oracle")


# ---- hand-written reference-format tables ----------------------------------------------------------------------------
def _state_batch(cfg, pane, parts):
    """Table "t" batch of one pane in partial_schema order.  parts: {key: (count, int64 sum, f64 sum)}: the counts
    and the sums of column a; a SUM over another column holds 7, every MIN -5 and every MAX 9."""
    keys = sorted(parts)
    cols = {"key": np.array(keys, dtype=np.int64)}
    for a in cfg.aggs:
        cnt = [parts[k][0] for k in keys]
        if a.kind == "count":
            cols[f"{a.name}[count]"] = np.array(cnt, dtype=np.int64)
        elif a.kind == "sum":
            cols[f"{a.name}[sum]"] = np.array([parts[k][1] if a.col == "a" else 7 for k in keys], dtype=np.int64)
        elif a.kind == "avg":
            cols[f"{a.name}[count]"] = np.array(cnt, dtype=np.uint64)
            cols[f"{a.name}[sum]"] = np.array([parts[k][2] for k in keys], dtype=np.float64)
        else:
            cols[f"{a.name}[{a.kind}]"] = np.array([-5 if a.kind == "min" else 9 for _ in keys], dtype=np.int64)
    cols[TS] = np.full(len(keys), pane, dtype=np.int64)
    return O.Batch(cols)


def _restored_panes(cfg, table):
    """The exact reference's per-(pane, key) partials of a hand-written table: AVG from the f64 [sum] (the reference's
    AVG state), SUM from the Int64 [sum], as exact_reference._Panes holds them."""
    panes = X._Panes("key", cfg.aggs, cfg.slide or cfg.width)
    for pane, b in table:
        for i in range(b.num_rows):
            k = int(b["key"][i])
            st = [None]
            for a in cfg.aggs:
                if a.kind == "count":
                    st.append(int(b[f"{a.name}[count]"][i]))
                    st[0] = st[-1]
                elif a.kind == "sum":
                    st.append(int(b[f"{a.name}[sum]"][i]))
                elif a.kind == "avg":
                    f = float(b[f"{a.name}[sum]"][i])
                    st[0] = int(b[f"{a.name}[count]"][i])
                    st.append((int(f), abs(int(f))))
                else:
                    st.append(int(b[f"{a.name}[{a.kind}]"][i]))
            keys = panes.by_pane.setdefault(pane, {})
            keys[k] = st if k not in keys else panes._merge(keys[k], st)
    return panes


P = 1 << 53
HAND = {
    # name: (plan, window kind, {pane index: {key: (count, int64 sum, f64 sum)}})
    "f64_1.8e19": ("ints", "tumbling", {0: {1: (3, X._wrap(18 * 10 ** 18), 1.8e19), 2: (2, X._wrap(-18 * 10 ** 18),
                                                                                        -1.8e19)}}),
    "f64_1.8e19_avg_only": ("P2", "tumbling", {0: {1: (3, 0, 1.8e19), 2: (2, 0, -1.8e19)}}),
    "f64_2^53+1": ("ints", "tumbling", {0: {1: (4, P + 1, float(P + 1))}, 1: {1: (1, P + 1, float(P + 1))}}),
    "f64_2^53+2_avg_only": ("P2", "running", {0: {1: (4, 0, float(P + 2))}, 1: {1: (1, 0, float(P + 2))}}),
    "int_disagrees": ("ints", "tumbling", {0: {1: (3, 1, 0.0), 2: (3, 5, 5.0)}}),
    "int_disagrees_sliding": ("ints", "running", {0: {1: (3, 1, 0.0)}, 1: {1: (2, -7, -6.0)}}),
    "count_2^32": ("ints", "tumbling", {0: {1: ((1 << 32) + 3, 5 * 10 ** 9, 5e9)}}),
    "count_2^32_avg_only": ("P2", "running", {0: {1: ((1 << 32) + 3, 0, 5e9)}}),
    "near_int64_max": ("ints", "tumbling", {0: {1: (5, INT64_MAX - (1 << 30), float(INT64_MAX - (1 << 30)))}}),
    "near_int64_max_sliding": ("ints", "running", {0: {1: (5, INT64_MAX - (1 << 30), float(INT64_MAX - (1 << 30)))}}),
}


def _hand_rows(cfg, kind, name):
    """Rows after the restore: guarded values (|v| < 2^31) in the restored panes and the next one; for the near-max
    tables they push the Int64 sum past INT64_MAX."""
    rng = np.random.default_rng(zlib.crc32(name.encode()))
    s = cfg.slide or cfg.width
    o = ORIGIN - ORIGIN % s
    n = 24
    a = rng.integers((1 << 31) - 1000, 1 << 31, n) if "near" in name else rng.integers(-(1 << 31) + 1, 1 << 31, n)
    cols = {"key": rng.choice(np.array([1, 2, 3], dtype=np.int64), n)}
    for c in "abcd":
        cols[c] = a.astype(np.int64) if c == "a" else rng.integers(-1000, 1000, n).astype(np.int64)
    cols[TS] = o + rng.integers(0, 2, n) * s + rng.integers(0, s, n)
    return O.Batch(cols)


def _check_hand(cfg, kind, table, batch, flags=0, expected_keys=64, entry="host"):
    """Restores `table` into the CUDA operator, sends `batch` and the end-of-data watermark, and checks every window
    against the restored state merged with the new rows (Fraction sums, check_avg)."""
    width, s = cfg.width, cfg.slide or cfg.width
    o = ORIGIN - ORIGIN % s
    panes = _restored_panes(cfg, table)
    ts = np.asarray(batch[TS], dtype=np.int64)
    panes.add({c: np.asarray(v) for c, v in batch.cols.items()}, ts)
    lo, hi = min(panes.by_pane), max(panes.by_pane)
    want = {(r["window_start"], r["key"]): r for r in panes.windows(range(lo - width + s, hi + 1, s), width, int)}
    st = Stream(0, "few", "R1", cfg.width, cfg.slide or None)
    st.events = [("batch", batch), ("wm", INT64_MAX)]
    seg = GpuSegment(st, kind, cfg, entry, flags, table, o, expected_keys)
    seg.batch(batch)
    got = seg.wm(INT64_MAX)
    s_ = seg.close()
    assert s_["rows_late"] == 0
    errs = X.mismatches(want, got, lambda r: (int(r["window_start"]), int(r["key"])))
    assert not errs, errs[:8]
    return got


def _hand_cfg(plan, kind, width_slides=4):
    w, sl = (width_slides * SEC, SEC) if kind != "tumbling" else (SEC, 0)
    return O.WindowAggConfig(width=w, slide=sl, key_names=["key"], aggs=PLANS[plan], window_index=1)


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(HAND))
def test_restore_reference_format_table(name):
    """Reference-format tables with states a promoted operator or the reference writes: f64 sums of +-1.8e19 and of
    2^53 + 1 (as f64: 2^53) or 2^53 + 2, an Int64 [sum] that is not the f64 [sum] (the reference sums AVG in f64 and
    SUM wrapping), a count of 2^32 and more in one row, an Int64 sum within 2^30 of INT64_MAX that new rows push past."""
    plan, kind, parts = HAND[name]
    cfg = _hand_cfg(plan, kind)
    s = cfg.slide or cfg.width
    o = ORIGIN - ORIGIN % s
    table = [(o + p * s, _state_batch(cfg, o + p * s, kp)) for p, kp in sorted(parts.items())]
    _check_hand(cfg, kind, table, _hand_rows(cfg, kind, name))


@pytest.mark.gpu
def test_restored_rows_count_toward_the_window_row_bound():
    """1040 restored panes of a 2048-slide window, each with 2^31 - 1 rows and an exact sum of 2^53 - 1: every pane
    alone keeps exact AVG valid, but a window of three panes holds 2^32 rows and the windows of more than 1024 panes
    sum past INT64_MAX.  The restored rows must count toward the window's row bound, or the exact Int64 sum wraps."""
    cfg = _hand_cfg("ints", "running", width_slides=2048)
    s = cfg.slide
    o = ORIGIN - ORIGIN % s
    c, v = (1 << 31) - 1, (1 << 53) - 1
    table = [(o + p * s, _state_batch(cfg, o + p * s, {1: (c, v, float(v))})) for p in range(1040)]
    batch = O.Batch({"key": np.array([1, 2], dtype=np.int64), **{x: np.array([3, 4], dtype=np.int64) for x in "abcd"},
                     TS: np.array([o + 1039 * s + 5, o + 1040 * s], dtype=np.int64)})
    got = _check_hand(cfg, "running", table, batch)
    assert len(got) > 3000


# ---- the exact/f64 choice on restore keeps the two-pass ingest -------------------------------------------------------
def _two_pass_kernels(table, last_wm, regime_batch):
    """Ingest launches and the kernels they took, with the two-pass ingest forced on and forced off, on operators
    restored from `table`: the difference is one kernel per two-pass launch."""
    from arroyo_b200 import ffi
    cfg = config(Stream(0, "few", "R1", 4 * SEC, SEC), "running", "ints")
    st = Stream(0, "few", "R1", 4 * SEC, SEC)
    st.events = [("batch", regime_batch)]
    out = {}
    for mode, fl in (("two", ffi.FLAG_TWO_PASS_ALWAYS), ("one", ffi.FLAG_NO_TWO_PASS)):
        seg = GpuSegment(st, "running", cfg, "host", fl, table, last_wm)
        s0 = seg.op.stats()
        seg.batch(regime_batch)
        seg.op.flush()
        s1 = seg.op.stats()
        out[mode] = (s1["ingest_launches"] - s0["ingest_launches"], s1["kernel_launches"] - s0["kernel_launches"])
        seg.close()
    return out


def _checkpoint_of(regime):
    st = Stream(3, "few", regime, 4 * SEC, SEC)
    st.rows([0, 1, 2], per=20)
    st.big()
    st.rows([2], per=20)
    st.wm(st.o + SEC)
    st.restart()
    st.rows([2])
    st.end()
    cfg = config(st, "running", "ints")
    seg = GpuSegment(st, "running", cfg, "host", 0, [], None)
    for ev in st.events[:2]:
        seg.batch(ev[1])
    seg.wm(st.o + SEC)
    table = seg.checkpoint()
    seg.close()
    return table, st.o + SEC, st.events[-2][1]


@pytest.mark.gpu
def test_restore_of_exact_state_keeps_the_two_pass_ingest():
    """After a restart from R1 state (every sum exact) the COUNT / SUM / AVG plan stays in exact mode, whose
    {rows, Int64 sum} accumulators the two-pass ingest takes: each forced two-pass launch runs part_kernel and
    agg_kernel, one kernel more than the one-pass launch.  After a restart from a promoted operator's table (R2) the
    plan has an f64 accumulator and both modes run the one-pass kernel."""
    table, wm, more = _checkpoint_of("R1")
    k = _two_pass_kernels(table, wm, more)
    assert k["two"][0] == k["one"][0] >= 1
    assert k["two"][1] - k["one"][1] == k["two"][0], k
    table, wm, more = _checkpoint_of("R2")
    k = _two_pass_kernels(table, wm, more)
    assert k["two"][0] == k["one"][0] >= 1 and k["two"][1] == k["one"][1], k


# ---- the instant aggregate -------------------------------------------------------------------------------------------
def _instant_stream(keys, regime):
    from tests.test_gpu_instant_window import Stream as IStream

    class S(IStream):
        def __init__(self, seed):
            super().__init__(seed, keys)
            self.vals = Stream(seed, keys if keys != "none" else "none", regime, SEC)

        def batch(self, ts):
            ts = np.asarray(ts, dtype=np.int64)
            self.vals.batch(self.rng.permutation(ts))
            self.events.append(self.vals.events.pop())

    st, o = S(zlib.crc32(f"instant/{keys}/{regime}".encode()) % 1000), ORIGIN
    st.at([o + k * SEC for k in range(4)])
    st.vals.big()
    st.at([o + k * SEC for k in range(3, 8)], per=6)
    st.restart()
    st.wm(o + 3 * SEC)
    st.restart()
    st.restart()
    st.at([o + 2 * SEC, o + 3 * SEC, o + 7 * SEC, o + 12 * SEC], per=4)
    st.wm(o + 5 * SEC)
    st.at([o + 6 * SEC, o + 9 * SEC], per=4)
    st.restart()
    st.wm(o + 8 * SEC)
    st.restart()
    st.at([o + 8 * SEC, o + 7 * SEC, o + 20 * SEC])
    return st.end()


def _instant_means(events, key_name):
    """{(instant, key): Mean of a} over the on-time rows (late: ts < the last watermark)."""
    acc, last = {}, None
    for ev in events:
        if ev[0] == "wm":
            last = ev[1]
        elif ev[0] == "batch":
            b = ev[1]
            for r in range(b.num_rows):
                t = int(b[TS][r])
                if last is not None and t < last:
                    continue
                k = int(b[key_name][r]) if key_name else None
                v = int(b["a"][r])
                s = acc.setdefault((t, k), [0, 0, 0])
                s[0], s[1], s[2] = s[0] + v, s[1] + abs(v), s[2] + 1
    return {g: X.Mean(Fraction(s[0], s[2]), s[1]) for g, s in acc.items()}


INSTANT = [("few", "ints", "R2", "host"), ("few", "ints", "R3", "device"), ("u64", "ints", "R3", "host"), ("none", "ints", "cancel", "sliced"),
           ("few", "minmax", "R2", "run_batches"), ("few", "ints", "cancel", "run_batches"),
           ("u64", "minmax", "R2", "host")]


@pytest.mark.gpu
@pytest.mark.parametrize("keys,plan,regime,entry", INSTANT, ids=["-".join(c) for c in INSTANT])
def test_instant_restart_at_extremes(keys, plan, regime, entry):
    """The instant aggregate keeps f64 AVG from the start; its restarts at the extremes give instant_emissions, the
    integers exactly and AVG by check_avg."""
    from tests.test_gpu_instant_window import PLANS as IPLANS, gpu_config, instant_emissions, run_gpu as irun
    st = _instant_stream(keys, regime)
    key = None if keys == "none" else "key"
    want, late = instant_emissions(st.events, key, IPLANS[plan])
    means = _instant_means(st.events, key)
    got, rows_in, rows_late, _ = irun(st, gpu_config(keys, plan), entry)
    assert len(got) == len(want)
    for i, (w, g) in enumerate(zip(want, got)):
        exp = {(t, k): row for t, rows in w for k, row in rows.items()}
        seen = {(int(r[TS]), int(r[key]) if key else None): r for r in g}
        assert len(seen) == len(g) and sorted(seen, key=str) == sorted(exp, key=str), (i, sorted(set(seen) ^ set(exp), key=str)[:6])
        assert [int(r[TS]) for r in g] == sorted(int(r[TS]) for r in g)
        for gk, row in exp.items():
            for c, v in row.items():
                if c == "ava":
                    assert X.check_avg(float(seen[gk][c]), means[gk]), (i, gk, seen[gk][c], means[gk])
                else:
                    assert int(seen[gk][c]) == v, (i, gk, c, seen[gk][c], v)
    assert rows_in == sum(ev[1].num_rows for ev in st.events if ev[0] == "batch")
    assert rows_late == late
