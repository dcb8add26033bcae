"""Event time of the tumbling and sliding window aggregates against tests/exact_reference.window_emissions, watermark
by watermark: which rows are late, which windows exist, which watermark emits each of them and in what order.

Every stream is an explicit list of ("batch", cols), ("wm", w) and ("restart",) events (a restart is handle_checkpoint,
a new operator and on_start).  The shapes go where the host state of window_agg.cu has edges: watermarks on and next to
bin edges, late rows at every distance, one watermark releasing hundreds of windows, gaps in event time of up to 10^6
slides, panes exactly r * 4096 slides apart, rows far ahead of the watermark, hops of up to 4097 slides, timestamps at
0 and near 2^62, negative watermarks, and restarts at awkward points.  They run over a cross section of window kinds
(tumbling, sliding with a running window, sliding re-merged), key sets and entry points (host batches, sliced batches,
device batches, the device begin/poll pair, run_batches, and the two-pass / one-pass ingest forced)."""
import ctypes as C
import zlib

import numpy as np
import pytest

from oracle import arroyo_oracle as O
from tests import exact_reference as X

pytestmark = pytest.mark.gpu

A = O.Agg
TS = O.TIMESTAMP
INT64_MAX = (1 << 63) - 1
SEC = 1_000_000_000
ORIGIN = 1_700_000_000 * SEC
PLANS = {
    # COUNT / SUM / AVG: invertible, so a sliding window keeps a running block (and the two-pass ingest applies)
    "ints": [A("count", None, "n"), A("sum", "a", "sa"), A("avg", "a", "ava")],
    # MIN / MAX: every window re-merges its panes
    "minmax": [A("count", None, "n"), A("min", "a", "mna"), A("max", "a", "mxa"), A("sum", "a", "sa")],
}


class Stream:
    def __init__(self, seed, keys, width, slide=None):
        self.rng = np.random.default_rng(seed)
        self.keys, self.width, self.slide = keys, width, slide or width
        self.events = []

    def batch(self, ts):
        ts = np.asarray(ts, dtype=np.int64)
        n = len(ts)
        cols = {}
        if self.keys != "none":
            cols["key"] = self.rng.integers(0, 3 if self.keys == "few" else 3000, n).astype(np.int64) - 1
        cols["a"] = self.rng.integers(-1000, 1000, n).astype(np.int64)
        cols[TS] = ts
        self.events.append(("batch", O.Batch(cols)))

    def rows_in(self, panes, per_pane=3, origin=0):
        """Rows at random instants of the given panes (pane numbers relative to `origin`)."""
        s = self.slide
        ts = [origin + p * s + int(x) for p in panes for x in self.rng.integers(0, s, per_pane)]
        self.batch(self.rng.permutation(np.asarray(ts, dtype=np.int64)))

    def wm(self, w):
        self.events.append(("wm", int(w)))

    def restart(self):
        self.events.append(("restart",))

    def end(self):
        self.wm(INT64_MAX)
        return self


def _o(s):
    return ORIGIN - ORIGIN % s


# ---- stream shapes: f(seed, keys, width, slide) -> Stream --------------------------------------------------------------
def t1_edges(seed, keys, w, s):
    st, o = Stream(seed, keys, w, s), _o(s)
    st.wm(o - 1000 * s)  # before any row
    st.rows_in(range(6), origin=o)
    st.wm(o - 500 * s)  # far behind the data
    for k in range(1, 7):
        st.wm(o + k * s - 1)
        st.wm(o + k * s - 1)  # the same watermark twice
        st.rows_in([k + 5], origin=o)
        st.wm(o + k * s)
        st.wm(o + k * s + 1)
    return st.end()


def t2_late(seed, keys, w, s):
    st, o = Stream(seed, keys, w, s), _o(s)
    st.rows_in(range(4), origin=o)
    w1 = o + 4 * s + s // 2
    st.wm(w1)
    lb = o + 4 * s  # bin(w1)
    mixed = [lb - 1, lb - s, lb, w1 - 1, w1, w1, lb - 50 * s, o + 5 * s + 1, o + 6 * s]
    st.batch(st.rng.permutation(np.asarray(mixed * 3, dtype=np.int64)))
    st.batch(lb - 1 - st.rng.integers(0, 3 * s, 40))  # a whole late batch
    st.wm(o + 7 * s + 1)
    st.rows_in([7, 8, 3, 1], origin=o)  # panes 3 and 1 are late now
    st.batch(np.asarray([o + 7 * s, o + 7 * s + 1, o + 7 * s - 1], dtype=np.int64))
    return st.end()


def t3_backlog(seed, keys, w, s):
    st, o = Stream(seed, keys, w, s), _o(s)
    st.wm(o - 1)
    for chunk in range(5):  # 250 panes three slides apart, then one watermark
        st.rows_in(range(chunk * 150, chunk * 150 + 150, 3), per_pane=2, origin=o)
    st.wm(o + 800 * s)
    st.rows_in([800, 801], origin=o)
    return st.end()


def t4_gap(seed, keys, w, s, g):
    st, o = Stream(seed, keys, w, s), _o(s)
    st.rows_in(range(3), origin=o)
    st.wm(o + s)
    # the first rows after the gap arrive before the watermark that empties the window store
    st.rows_in([2 + g, 3 + g], origin=o)
    st.wm(o + (2 + g) * s - s)
    st.rows_in([3 + g, 4 + g], origin=o)
    st.wm(o + (4 + g) * s + 1)
    st.rows_in([5 + g, 6 + g + w // s], origin=o)
    st.wm(o + (6 + g + w // s) * s)
    return st.end()


def t5_alias(seed, keys, w, s):
    st, o = Stream(seed, keys, w, s), _o(s)
    rs = [1 << e for e in range(4, 13)]  # 16 .. 4096
    for _ in range(3):  # every pane live and receiving rows
        st.rows_in([0] + rs + [r + 1 for r in rs], per_pane=2, origin=o)
    st.wm(o + 2 * s)
    st.rows_in([2] + rs, origin=o)
    st.wm(o + 20 * s)
    st.rows_in([20] + rs[2:], origin=o)
    return st.end()


def t5_wide(seed, keys, w, s):
    """80 live panes 4096 slides apart: they all alias one slot of the largest ring, in one batch."""
    st, o = Stream(seed, keys, w, s), _o(s)
    panes = [4096 * j for j in range(80)]
    st.rows_in(panes, per_pane=2, origin=o)
    st.rows_in(panes[::-1], per_pane=1, origin=o)
    st.wm(o + 2 * s)
    st.rows_in([2, 4096, 4097, 79 * 4096], origin=o)
    st.wm(o + 4096 * 40 * s)
    return st.end()


def t6_far(seed, keys, w, s, k):
    st, o = Stream(seed, keys, w, s), _o(s)
    st.rows_in(range(4), origin=o)
    st.wm(o + 2 * s)
    st.rows_in([2 + k, 3 + k], per_pane=2, origin=o)  # k slides ahead of the watermark
    # advance past the pane that shares the far pane's ring slot (k - 4096 slides on), then through its windows
    last = min(max(k - 4096 + 12, 12), 1000)
    for p in range(4, last, 8):
        st.rows_in(range(p, p + 8), per_pane=1, origin=o)
        st.wm(o + p * s)
    st.rows_in([k + 2, k + 5], origin=o)
    st.wm(o + (k + 3) * s + 1)
    return st.end()


def t7_hop(seed, keys, w, s, dense=False):
    st, o = Stream(seed, keys, w, s), _o(s)
    n = w // s
    panes = list(range(n + 1)) if dense else [0, 1, 5, n - 1, n, n + 3]
    half = len(panes) // 2
    for i in range(0, half, 512):
        st.rows_in(panes[i:min(i + 512, half)], per_pane=1, origin=o)
    st.wm(o + 2 * s)
    st.restart()
    for i in range(half, len(panes), 512):
        st.rows_in(panes[i:i + 512], per_pane=1, origin=o)
    st.wm(o + (n + 1) * s)
    st.rows_in([2 * n, 2 * n + 1], origin=o)
    st.restart()
    st.wm(o + 2 * n * s)
    return st.end()


def t8_zero(seed, keys, w, s):
    st = Stream(seed, keys, w, s)
    st.batch(np.asarray([0, 0, 1, s - 1, s, 3 * s], dtype=np.int64))  # pane 0 is the max_q == 0 sentinel
    st.wm(-10 * s)
    st.wm(-1)
    st.batch(np.asarray([0, 2, s + 1, 2 * s], dtype=np.int64))
    st.wm(s)
    st.batch(np.asarray([0, s, 4 * s + 1], dtype=np.int64))
    st.wm(2 * s + 1)
    return st.end()


def t8_negative_wm(seed, keys, w, s):
    """First timestamps below the watermark delay: the watermarks min(ts) - delay are negative."""
    st = Stream(seed, keys, w, s)
    d = 10 * s
    for p in range(0, 6, 2):
        st.rows_in([p, p + 1], origin=0)
        st.wm(p * s - d)
    st.rows_in([12, 13], origin=0)
    st.wm(12 * s - d)
    st.wm(14 * s - d)
    return st.end()


def t8_big(seed, keys, w, s):
    st = Stream(seed, keys, w, s)
    o = (1 << 62) - (1 << 62) % s
    st.rows_in(range(3), origin=o)
    st.wm(o + s + 1)
    st.rows_in([0, 1, 3, 4], origin=o)
    st.wm(o + 3 * s)
    return st.end()


def t9_restarts(seed, keys, w, s):
    st, o = Stream(seed, keys, w, s), _o(s)
    n = w // s
    st.rows_in(range(3), origin=o)
    st.wm(o + (3 + n) * s)  # empties the window store
    st.restart()
    st.rows_in([4 + n, 5 + n], origin=o)
    st.rows_in([5000 + n], origin=o)  # far ahead, pending across the restart
    st.wm(o + (5 + n) * s + 1)
    st.restart()
    st.rows_in([2 + n, 4 + n, 5 + n, 6 + n], origin=o)  # late against the restored watermark, then on time
    st.wm(o + (8 + n) * s)
    st.restart()
    st.rows_in([8 + n, 5000 + n], origin=o)
    return st.end()


def _shape(name, kind):
    """(stream, width, slide) of a named shape; `kind` = tumbling / running / remerge."""
    hop = kind != "tumbling"
    w, s = (4 * SEC, SEC) if hop else (SEC, None)
    base, _, arg = name.partition(":")
    seed = zlib.crc32(f"{name}/{kind}".encode()) % 1000
    if base == "T1":
        return lambda k: t1_edges(seed, k, w, s or w)
    if base == "T2":
        return lambda k: t2_late(seed, k, w, s or w)
    if base == "T3":
        return lambda k: t3_backlog(seed, k, w, s or w)
    if base == "T4":
        named = {"n-1": w // (s or w) - 1, "n": w // (s or w), "n+1": w // (s or w) + 1}
        g = named[arg] if arg in named else int(arg)
        return lambda k: t4_gap(seed, k, w, s or w, g)
    if base == "T5":
        f = t5_wide if arg == "wide" else t5_alias
        return lambda k: f(seed, k, w, s or w)
    if base == "T6":
        return lambda k: t6_far(seed, k, w, s or w, int(arg))
    if base == "T7":
        n, dense = int(arg.rstrip("d")), arg.endswith("d")
        return lambda k: t7_hop(seed, k, n * SEC, SEC, dense)
    if base == "T8":
        sl = {"2": 2, "3": 3, "p": SEC + 7, "2^32-1": (1 << 32) - 1, "2^32+1": (1 << 32) + 1, "30d": 30 * 86400 * SEC}
        sub, _, slide = arg.partition("@")
        sl = sl.get(slide, SEC)
        ww, ss = (4 * sl, sl) if hop else (sl, None)
        f = {"zero": t8_zero, "neg": t8_negative_wm, "big": t8_big}[sub]
        return lambda k: f(seed, k, ww, ss or ww)
    if base == "T9":
        return lambda k: t9_restarts(seed, k, w, s or w)
    raise KeyError(name)


# ---- drivers ----------------------------------------------------------------------------------------------------------
def config(st, kind, plan):
    key_names = [] if st.keys == "none" else ["key"]
    slide = st.slide if kind != "tumbling" else 0
    return O.WindowAggConfig(width=st.width, slide=slide, key_names=key_names, aggs=PLANS[plan],
                             window_index=len(key_names))


def reference(st, cfg):
    return X.window_emissions(st.events, cfg.key_names[0] if cfg.key_names else None, cfg.aggs, cfg.width,
                              cfg.slide or None)


def run_oracle(st, kind, cfg):
    """The numpy oracle on the same events: one list of output rows per watermark."""
    cls = O.TumblingAggregatingWindowFunc if kind == "tumbling" else O.SlidingAggregatingWindowFunc
    ctx, op, outs = O.OperatorContext(1), cls(cfg), []
    for ev in st.events:
        if ev[0] == "batch":
            op.process_batch(ev[1], ctx, O.Collector())
        elif ev[0] == "wm":
            ctx.watermarks.set(0, ev[1])
            col = O.Collector()
            op.handle_watermark(ev[1], ctx, col)
            outs.append([r for b in col.batches for r in b.rows()])
        else:
            op.handle_checkpoint(ctx)
            op = cls(cfg)
            op.on_start(ctx)
    return outs


class _Ptr:
    def __init__(self, ptr, n, typestr):
        self.__cuda_array_interface__ = {"shape": (n,), "typestr": typestr, "data": (ptr, False), "version": 2}


def device_names(cfg):
    """Columns of a device-resident window: [key,] window_start, window_end, aggregates, _timestamp."""
    return list(cfg.key_names) + ["window_start", "window_end"] + [a.name for a in cfg.aggs] + [TS]


def device_rows(wins, names):
    """Rows of device-resident windows, [(n_rows, [column pointers])], copied to the host."""
    import torch
    rows = []
    for n, ptrs in wins:
        assert len(ptrs) == len(names)
        host = {c: torch.as_tensor(_Ptr(p, n, "<f8" if c.startswith("av") else "<i8"), device="cuda").cpu().numpy()
                for c, p in zip(names, ptrs)}
        rows += O.Batch(host).rows()
    return rows


def run_gpu(st, kind, cfg, entry, expected_keys=0, flags=0):
    """The CUDA operator on the same events, with operator flags `flags` added to those of `kind` and `entry`.  Returns
    (one list of output rows per watermark, rows_in, rows_late, n_keys of the last operator).
    `poll_host` feeds device batches and alternates the watermarks between the host call (even ones) and the device
    begin / poll pair (odd ones), so host emissions and checkpoints follow device emissions of any size."""
    import torch

    import arroyo_b200 as ab
    from arroyo_b200 import ffi, operators as native
    from arroyo_b200.context import clamp_watermark
    from tests.gpu_ops import from_arrow, to_arrow
    flags |= {"running": 0, "remerge": ffi.FLAG_REMERGE_ONLY, "tumbling": 0}[kind]
    flags |= {"two_pass": ffi.FLAG_TWO_PASS_ALWAYS, "one_pass": ffi.FLAG_NO_TWO_PASS}.get(entry, 0)
    cls = native.TumblingAggregatingWindowFunc if kind == "tumbling" else native.SlidingAggregatingWindowFunc
    first = next(ev[1] for ev in st.events if ev[0] == "batch")
    schema = to_arrow(first).schema
    names = list(schema.names)
    dev_names = device_names(cfg)

    def make():
        return cls(cfg, input_schema=schema, flags=flags, expected_keys=expected_keys)

    op, ctx, outs, keep, pending = make(), ab.OperatorContext(1), [], [], []
    totals = [0, 0]

    def host_rows(batches):
        return [r for b in batches for r in from_arrow(b).rows()]

    def dev_rows(wins):
        return device_rows(wins, dev_names)

    def run_pending(wm):
        if not pending:
            return []
        ex = native.ExportedBatches([to_arrow(b) for b in pending])
        wms = (C.c_int64 * len(pending))(*([ffi.NO_WATERMARK] * (len(pending) - 1) + [wm]))
        col = ab.Collector()
        op.run_batches(ex, wms, col)
        op.handle_watermark_poll(col, block=True)
        pending.clear()
        return col.batches

    for ev in st.events:
        if ev[0] == "batch":
            b = ev[1]
            if entry == "run_batches":
                pending.append(b)
            elif entry == "sliced":
                rb, s, i = to_arrow(b), 0, 0
                while s < b.num_rows:
                    z = min((1, 7, 1023, 2)[i % 4], b.num_rows - s)
                    op.process_batch(rb.slice(s, z), ctx, None)
                    s, i = s + z, i + 1
            elif entry in ("device", "poll", "poll_host"):
                dev = [torch.from_numpy(np.ascontiguousarray(b[c])).cuda() for c in names]
                keep.append(dev)
                op.process_device_batch([t.data_ptr() for t in dev], b.num_rows)
            else:
                op.process_batch(to_arrow(b), ctx, None)
        elif ev[0] == "wm":
            w = ev[1]
            ctx.watermarks.set(0, w)
            if entry == "run_batches" and pending:
                outs.append(host_rows(run_pending(clamp_watermark(w))))
            elif entry == "device":
                outs.append(dev_rows(op.handle_watermark_device(w)))
            elif entry == "poll" or (entry == "poll_host" and len(outs) % 2 == 1):
                op.handle_watermark_device_begin(w)
                outs.append(dev_rows(op.handle_watermark_device_poll()))
            else:
                col = ab.Collector()
                op.handle_watermark(w, ctx, col)
                outs.append(host_rows(col.batches))
        else:
            if entry == "run_batches" and pending:
                assert not run_pending(ffi.NO_WATERMARK)
            s = op.stats()
            totals[0] += s["rows_in"]
            totals[1] += s["rows_late"]
            op.handle_checkpoint(None, ctx, None)
            op.close()
            op = make()
            op.on_start(ctx)
    s = op.stats()
    totals[0] += s["rows_in"]
    totals[1] += s["rows_late"]
    op.close()
    return outs, totals[0], totals[1], s["n_keys"]


def check_emissions(want, got, cfg, who):
    key = cfg.key_names[0] if cfg.key_names else None
    assert len(got) == len(want), (who, len(got), len(want))
    for i, (w, g) in enumerate(zip(want, got)):
        starts = [int(r["window_start"]) for r in g]
        assert starts == sorted(starts), (who, i, "windows out of order")
        errs = X.mismatches(w, g, lambda r: (int(r["window_start"]), int(r[key]) if key else None))
        assert not errs, (who, "watermark", i, errs[:8])


# (shape, window kind, keys, plan, entry): a cross section, not the product
CASES = [
    ("T1", "tumbling", "few", "ints", "host"),
    ("T1", "running", "many", "ints", "sliced"),
    ("T1", "remerge", "none", "minmax", "device"),
    ("T2", "tumbling", "many", "ints", "two_pass"),
    ("T2", "running", "few", "ints", "one_pass"),
    ("T2", "remerge", "few", "minmax", "sliced"),
    ("T2", "running", "many", "ints", "two_pass"),
    ("T2", "tumbling", "none", "minmax", "run_batches"),
    ("T3", "tumbling", "few", "ints", "device"),
    ("T3", "running", "few", "ints", "poll"),
    ("T3", "remerge", "many", "minmax", "host"),
    ("T3", "running", "none", "ints", "run_batches"),
    ("T4:1", "running", "few", "ints", "host"),
    ("T4:n-1", "remerge", "few", "minmax", "host"),
    ("T4:n", "running", "many", "ints", "two_pass"),
    ("T4:n+1", "running", "none", "ints", "device"),
    ("T4:4095", "tumbling", "few", "ints", "host"),
    ("T4:4096", "remerge", "few", "minmax", "sliced"),
    ("T4:4097", "running", "few", "ints", "poll"),
    ("T4:1000000", "tumbling", "many", "ints", "one_pass"),
    ("T4:1000000", "running", "few", "ints", "host"),
    ("T5", "tumbling", "few", "ints", "host"),
    ("T5", "running", "many", "ints", "two_pass"),
    ("T5", "remerge", "none", "minmax", "one_pass"),
    ("T5:wide", "tumbling", "few", "ints", "host"),
    ("T5:wide", "running", "none", "ints", "one_pass"),
    ("T5:wide", "remerge", "few", "minmax", "device"),
    ("T6:1", "running", "few", "ints", "host"),
    ("T6:2", "tumbling", "few", "ints", "device"),
    ("T6:3", "remerge", "few", "minmax", "host"),
    ("T6:4", "running", "none", "ints", "sliced"),
    ("T6:4095", "tumbling", "few", "ints", "host"),
    ("T6:4096", "running", "few", "ints", "two_pass"),
    ("T6:4097", "remerge", "few", "minmax", "host"),
    ("T6:5000", "running", "many", "ints", "one_pass"),
    ("T6:5000", "tumbling", "none", "minmax", "poll"),
    ("T6:1000000", "running", "few", "ints", "host"),
    ("T6:1000000", "tumbling", "few", "minmax", "run_batches"),
    ("T7:16", "running", "few", "ints", "host"),
    ("T7:16", "remerge", "few", "minmax", "host"),
    ("T7:17", "running", "few", "ints", "device"),
    ("T7:17", "remerge", "none", "ints", "host"),
    ("T7:600", "running", "few", "ints", "host"),
    ("T7:600", "remerge", "few", "minmax", "poll"),
    ("T7:600", "remerge", "few", "minmax", "poll_host"),
    ("T7:600", "running", "few", "ints", "poll_host"),
    ("T3", "running", "few", "ints", "poll_host"),
    ("T3", "remerge", "many", "minmax", "poll_host"),
    ("T9", "remerge", "few", "minmax", "poll_host"),
    ("T7:3600", "running", "few", "ints", "host"),
    ("T7:3600d", "remerge", "none", "minmax", "host"),
    ("T7:4096", "running", "none", "ints", "host"),
    ("T7:4096", "remerge", "few", "minmax", "host"),
    ("T7:4097d", "running", "none", "ints", "host"),
    ("T7:4097", "remerge", "few", "minmax", "device"),
    ("T8:zero", "tumbling", "few", "ints", "host"),
    ("T8:zero", "running", "few", "ints", "one_pass"),
    ("T8:zero", "remerge", "none", "minmax", "host"),
    ("T8:neg", "tumbling", "few", "ints", "host"),
    ("T8:neg", "running", "many", "ints", "two_pass"),
    ("T8:neg", "remerge", "few", "minmax", "device"),
    ("T8:big@30d", "running", "few", "ints", "host"),
    ("T8:big@30d", "tumbling", "none", "minmax", "host"),
    ("T8:zero@2", "running", "few", "ints", "host"),
    ("T8:zero@3", "tumbling", "few", "minmax", "sliced"),
    ("T8:big@p", "remerge", "few", "minmax", "host"),
    ("T8:big@2^32-1", "running", "few", "ints", "host"),
    ("T8:big@2^32+1", "tumbling", "few", "ints", "device"),
    ("T8:neg@p", "running", "none", "ints", "host"),
    ("T9", "tumbling", "few", "ints", "host"),
    ("T9", "running", "few", "ints", "host"),
    ("T9", "remerge", "many", "minmax", "sliced"),
    ("T9", "running", "none", "ints", "device"),
]


@pytest.mark.parametrize("shape,kind,keys,plan,entry", CASES, ids=["-".join(c) for c in CASES])
def test_window_event_time(shape, kind, keys, plan, entry):
    st = _shape(shape, kind)(keys)
    cfg = config(st, kind, plan)
    want, late = reference(st, cfg)
    # small dictionaries keep thousands of live pane blocks cheap
    got, rows_in, rows_late, _ = run_gpu(st, kind, cfg, entry, expected_keys=0 if keys == "many" else 64)
    check_emissions(want, got, cfg, "gpu")
    assert rows_in == sum(ev[1].num_rows for ev in st.events if ev[0] == "batch")
    assert rows_late == late


def test_device_emission_larger_than_max_out():
    """One watermark releases 250 windows.  The device entry hands out at most max_out = 8 per call and queues the
    rest; while windows are queued a new emission is refused; the polls return the rest in order, and every window
    equals the reference."""
    import arroyo_b200 as ab
    from arroyo_b200 import ffi, operators as native
    from tests.gpu_ops import to_arrow
    st = t3_backlog(5, "few", SEC, SEC)
    cfg = config(st, "tumbling", "ints")
    want, _ = reference(st, cfg)
    names = device_names(cfg)
    op = native.TumblingAggregatingWindowFunc(cfg, input_schema=to_arrow(st.events[1][1]).schema, expected_keys=64)
    lib, outb, n = op._lib, (ffi.DeviceBatch * 8)(), C.c_int64(0)
    got, i = [], 0
    for ev in st.events:
        if ev[0] == "batch":
            op.process_batch(to_arrow(ev[1]), ab.OperatorContext(1), None)
            continue
        if ev[1] != ORIGIN + 800 * SEC:
            got.append(device_rows(op.handle_watermark_device(ev[1], max_out=8), names))
            continue
        wins, calls = [], 0
        assert lib.arroyo_b200_op_handle_watermark_device(op._h, ev[1], outb, 8, C.byref(n)) == ffi.OK
        while True:
            calls += 1
            k = n.value
            wins += [(outb[j].n_rows, [outb[j].cols[c] for c in range(outb[j].n_cols)]) for j in range(k)]
            if calls == 1:
                assert k == 8
                later, m = ORIGIN + 900 * SEC, C.c_int64(0)
                assert lib.arroyo_b200_op_handle_watermark_device_begin(op._h, later) == ffi.INVALID_ARGUMENT
                assert lib.arroyo_b200_op_handle_watermark_device(op._h, later, outb, 8, C.byref(m)) == ffi.INVALID_ARGUMENT
            if k < 8:
                break
            assert lib.arroyo_b200_op_handle_watermark_device_poll(op._h, outb, 8, C.byref(n)) == ffi.OK
        assert len(wins) == 250 and calls == 32
        got.append(device_rows(wins, names))
    check_emissions(want, got, cfg, "gpu")
    op.close()


def test_session_device_windows_stay_queued():
    """The same rule on an operator without its own begin / poll: a session emission left queued by max_out = 0 blocks
    the next device emission until it is polled, and it comes back whole."""
    import arroyo_b200 as ab
    from arroyo_b200 import ffi, operators as native
    from tests.gpu_ops import from_arrow, to_arrow
    from tests.test_gpu_parity import S, session_stream
    batches = session_stream(np.random.default_rng(9), n_keys=50, n_bursts=4, gap=2 * S, batch=200)
    cfg = O.SessionConfig(gap=2 * S, key_names=["key"], aggs=[A("count", None, "rows"), A("sum", "value", "sum")],
                          window_index=0)
    ops = [native.SessionAggregatingWindowFunc(cfg) for _ in range(2)]
    for op in ops:
        ctx = ab.OperatorContext(1)
        for b in batches:
            op.process_batch(to_arrow(b), ctx, None)
    host = ab.Collector()
    ctx = ab.OperatorContext(1)
    ctx.watermarks.set(0, ab.FINAL_WATERMARK)
    ops[0].handle_watermark(ab.FINAL_WATERMARK, ctx, host)
    cols = ("key", "window_start", "window_end", "rows", "sum", TS)
    want = sorted(tuple(int(r[c]) for c in cols) for b in host.batches for r in from_arrow(b).rows())
    op, lib = ops[1], ops[1]._lib
    outb, n = (ffi.DeviceBatch * 4)(), C.c_int64(0)
    end = (1 << 63) - 1
    assert lib.arroyo_b200_op_handle_watermark_device(op._h, end, outb, 0, C.byref(n)) == ffi.OK and n.value == 0
    assert lib.arroyo_b200_op_handle_watermark_device_begin(op._h, end) == ffi.INVALID_ARGUMENT
    assert lib.arroyo_b200_op_handle_watermark_device(op._h, end, outb, 4, C.byref(n)) == ffi.INVALID_ARGUMENT
    assert lib.arroyo_b200_op_handle_watermark_device_poll(op._h, outb, 4, C.byref(n)) == ffi.OK and n.value >= 1
    wins = [(outb[j].n_rows, [outb[j].cols[c] for c in range(outb[j].n_cols)]) for j in range(n.value)]
    rows = device_rows(wins, ["window_start", "window_end", "key", "rows", "sum", TS])
    got = sorted(tuple(int(r[c]) for c in cols) for r in rows)
    assert len(want) > 50 and got == want
    assert lib.arroyo_b200_op_handle_watermark_device_begin(op._h, end) == ffi.OK
    for o in ops:
        o.close()
