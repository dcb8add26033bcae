"""The CUDA instant join (csrc/join.cu = InstantJoin) and join with expiration (csrc/ttl_join.cu = JoinWithExpiration)
against the exact reference joins of tests/exact_reference.py, at the shapes where a hash join goes wrong.

InstantJoin, every shape under inner, left, right and full joins: either build orientation (the side with fewer
eligible rows builds, equal counts build on the right), a side with nothing eligible or nothing at all, build counts
around the table's 1024-slot minimum and its power-of-two steps, arenas that grow and compact while they hold rows,
edge, UInt64 >= 2^63 and timestamp-typed keys, hundreds of instants per watermark, instants equal in their low 32 bits,
rows at the watermark, a hot key next to cold ones, routing columns, payload types that must pass bit-exact, and the
host, sliced, 4-input, device and mixed entry points.  Outer-join validity bitmaps are read bit by bit.
JoinWithExpiration: the same key edges, a multimap that rehashes while its chains are live, one key per batch, a long
chain, zero-row batches, one side alone.  Both: the refused plans and inputs, and correct output after a refusal."""
import ctypes as C
import zlib

import numpy as np
import pyarrow as pa
import pytest

from tests import exact_reference as X

pytestmark = pytest.mark.gpu

TS = X.TIMESTAMP
I64_MIN, I64_MAX = -(1 << 63), (1 << 63) - 1
EDGE_KEYS = [0, 1, -1, I64_MIN, I64_MAX]
T0 = 1_700_000_000 * 10 ** 9
W = 10 ** 9
ARROW = {"l": pa.int64(), "L": pa.uint64(), "g": pa.float64(), "tDn": pa.duration("ns"), "tsn:": pa.timestamp("ns")}
NP = {"l": np.int64, "L": np.uint64, "g": np.float64, "tDn": np.int64, "tsn:": np.int64}
JOIN_TYPES = ["inner", "left", "right", "full"]
LEFT = [("id", "l"), ("a", "l"), (TS, "tsn:")]
RIGHT = [("id", "l"), ("b", "l"), (TS, "tsn:")]
# every payload type, names that clash between the sides (`_right`), the key in the middle
WIDE_L = [("u", "L"), ("id", "l"), ("f", "g"), ("d", "tDn"), (TS, "tsn:"), ("t", "tsn:")]
WIDE_R = [("f", "g"), ("t", "tsn:"), ("id", "l"), (TS, "tsn:"), ("u", "L"), ("d", "tDn")]


class Stream:
    """A join input stream: each side's schema [(name, type code)], the join and routing columns, and the events
    (side, {name: numpy array}) / ("wm", watermark).  Routing columns `_key_*` lead the schema and copy the key."""

    def __init__(self, rng, left=LEFT, right=RIGHT, left_on="id", right_on="id", n_routing=0, key_type="l"):
        self.rng = rng
        self.on = (left_on, right_on)
        self.routing = tuple(tuple(f"_key_{i}" for i in range(n_routing)) for _ in range(2))
        self.key_type = key_type
        self.schemas = []
        for sch, on, routing in ((left, left_on, self.routing[0]), (right, right_on, self.routing[1])):
            sch = [(n, key_type if n == on else t) for n, t in sch]
            self.schemas.append([(r, key_type) for r in routing] + sch)
        self.events = []

    def key_array(self, keys):
        u = np.asarray([int(k) % (1 << 64) for k in keys], dtype=np.uint64)
        return u if self.key_type == "L" else u.view(np.int64)

    def payload(self, code, n):
        raw = self.rng.integers(0, 1 << 63, n, dtype=np.uint64) | (self.rng.integers(0, 2, n, dtype=np.uint64) << np.uint64(63))
        if code == "g":
            raw[::7] = np.uint64(0x7FF8000000000123)  # NaN with a payload
            raw[3::7] = np.uint64(0x8000000000000000)  # -0.0
            raw[5::11] = np.uint64(0xFFF0000000000001)  # negative signalling NaN
        return raw.view(NP[code]) if code != "L" else raw

    def send(self, side, keys, ts):
        keys = self.key_array(keys)
        ts = np.asarray(ts, dtype=np.int64)
        assert len(keys) == len(ts)
        cols = {}
        for name, code in self.schemas[side]:
            if name == TS:
                cols[name] = ts
            elif name == self.on[side] or name in self.routing[side]:
                cols[name] = keys.copy()
            else:
                cols[name] = self.payload(code, len(ts))
        self.events.append((side, cols))

    def wm(self, w):
        self.events.append(("wm", w))

    def reference_instant(self, join_type):
        return X.instant_join(self.events, join_type, self.on[0], self.on[1], self.routing[0], self.routing[1])

    def reference_expiring(self):
        return X.expiring_join(self.events, self.on[0], self.on[1], self.routing[0], self.routing[1])


def to_arrow(schema, cols) -> pa.RecordBatch:
    n = len(cols[TS])
    arrays = [pa.Array.from_buffers(ARROW[code], n, [None, pa.py_buffer(np.ascontiguousarray(cols[name]))])
              for name, code in schema]
    return pa.RecordBatch.from_arrays(arrays, names=[name for name, _ in schema])


def rows_of(batches, names):
    """Output batches as X.Rows, read from the Arrow buffers themselves: values as 64-bit patterns, validity bit by
    bit.  Checks each column's null_count against its bitmap, and that a column without nulls has no bitmap."""
    vals, valid = [], []
    for rb in batches:
        assert rb.schema.names == names, (rb.schema.names, names)
        n = rb.num_rows
        v = np.zeros((n, len(names)), dtype=np.uint64)
        ok = np.ones((n, len(names)), dtype=bool)
        for i, arr in enumerate(rb.columns):
            bufs = arr.buffers()
            v[:, i] = np.frombuffer(bufs[1], dtype=np.uint64, count=arr.offset + n)[arr.offset:]
            if bufs[0] is None:
                assert arr.null_count == 0, names[i]
                continue
            bits = np.unpackbits(np.frombuffer(bufs[0], dtype=np.uint8), bitorder="little")[arr.offset:arr.offset + n]
            assert len(bits) == n
            ok[:, i] = bits.astype(bool)
            assert arr.null_count == n - int(bits.sum()) and arr.null_count > 0, (names[i], arr.null_count)
        vals.append(v)
        valid.append(ok)
    k = len(names)
    return X.Rows(names, np.concatenate(vals) if vals else np.zeros((0, k), np.uint64),
                  np.concatenate(valid) if valid else np.zeros((0, k), bool))


def check(want: X.Rows, got: X.Rows, what):
    errs = X.join_mismatches(want, got)
    assert not errs, (what, errs)


def _slices(rb, rng):
    """Odd-length slices of one batch (non-zero offsets)."""
    s = 0
    while s < rb.num_rows:
        z = min(int(rng.integers(0, 600)) * 2 + 1, rb.num_rows - s)
        yield rb.slice(s, z)
        s += z


class _Ptr:
    def __init__(self, ptr, n):
        self.__cuda_array_interface__ = {"shape": (n,), "typestr": "<i8", "data": (ptr, False), "version": 2}


# ---------------------------------------------------------------------------------------------------------------
# InstantJoin shapes
# ---------------------------------------------------------------------------------------------------------------
def _instants(st, n_l, n_r, n_keys, n_instants, key_fn=None, hold=1):
    """n_instants instants, each side's rows of an instant in one batch; after each instant a watermark that releases
    all but the newest `hold` instants, then the end-of-data watermark."""
    rng = st.rng
    key_fn = key_fn or (lambda n: rng.integers(0, n_keys, n))
    for i in range(n_instants):
        t = T0 + i * W
        st.send(0, key_fn(n_l), np.full(n_l, t))
        st.send(1, key_fn(n_r), np.full(n_r, t))
        st.wm(T0 + (i + 1 - hold) * W)
    st.wm(1 << 64)
    return st


def _edge_keys(rng, n, n_keys, frac=0.3):
    k = rng.integers(0, n_keys, n).astype(object)
    pick = rng.random(n) < frac
    k[pick] = rng.choice(np.array(EDGE_KEYS, dtype=object), int(pick.sum()))
    return k


def shape_left_smaller(rng):
    return _instants(Stream(rng), 300, 900, 400, 4)


def shape_right_smaller(rng):
    return _instants(Stream(rng), 900, 300, 400, 4)


def shape_equal(rng):
    return _instants(Stream(rng), 500, 500, 300, 3)


def shape_zero_eligible(rng):
    """At the first watermark the left side buffers rows at the watermark but has none eligible; at the second the
    right side."""
    st = Stream(rng)
    k = lambda n: rng.integers(0, 200, n)  # noqa: E731
    st.send(1, k(500), np.full(500, T0))
    st.send(0, k(400), np.full(400, T0 + W))
    st.wm(T0 + W)
    st.send(0, k(300), np.full(300, T0 + W))
    st.send(1, k(200), np.full(200, T0 + 2 * W))
    st.wm(T0 + 2 * W)
    st.wm(1 << 64)
    return st


def _one_side(rng, side):
    st = Stream(rng)
    for i in range(3):
        st.send(side, rng.integers(0, 100, 250), np.full(250, T0 + i * W))
        st.wm(T0 + i * W + 1)
    st.wm(1 << 64)
    return st


def shape_left_only(rng):
    return _one_side(rng, 0)


def shape_right_only(rng):
    return _one_side(rng, 1)


def _build(n):
    def f(rng):
        """One instant: the left side builds from exactly n eligible rows (the right has n + 700)."""
        st = Stream(rng)
        st.send(0, rng.integers(0, n // 2 + 2, n), np.full(n, T0))
        st.send(1, rng.integers(0, n // 2 + 40, n + 700), np.full(n + 700, T0))
        st.send(1, rng.integers(0, 10, 50), np.full(50, T0 + W))  # stays buffered
        st.wm(T0 + W)
        st.wm(1 << 64)
        return st
    return f


def shape_buffered_70k(rng):
    """35 k rows per side and instant, two instants buffered at every watermark: the arenas grow past 2^16 rows and
    compact while holding rows."""
    return _instants(Stream(rng), 35_000, 35_000, 50_000, 4, hold=2)


def shape_edge_keys(rng):
    return _instants(Stream(rng), 700, 600, 300, 3, key_fn=lambda n: _edge_keys(rng, n, 300))


def shape_u64_keys(rng):
    st = Stream(rng, key_type="L")
    big = lambda n: [(1 << 63) + int(x) if x % 3 else int(x) for x in rng.integers(0, 200, n)]  # noqa: E731
    return _instants(st, 600, 700, 0, 3, key_fn=big)


def shape_ts_keys(rng):
    """Timestamp-typed keys: a join on window_start, as the windowed joins of the goldens."""
    left = [("window_start", "tsn:"), ("a", "l"), (TS, "tsn:")]
    right = [("window_start", "tsn:"), ("b", "g"), (TS, "tsn:")]
    st = Stream(rng, left=left, right=right, left_on="window_start", right_on="window_start", key_type="tsn:")
    return _instants(st, 400, 500, 0, 3, key_fn=lambda n: T0 - W * rng.integers(0, 6, n))


def shape_many_instants(rng):
    """300 instants in one batch per side, the same keys in every instant, all released by one watermark."""
    st = Stream(rng)
    for side, n in ((0, 6000), (1, 7000)):
        st.send(side, rng.integers(0, 20, n), T0 + 1000 * rng.integers(0, 300, n))
    st.wm(T0 + 1000 * 300)
    st.wm(1 << 64)
    return st


def shape_ts_2p32(rng):
    """Instants 2^32 ns apart (equal low 32 bits), the same keys in each: only the full timestamp separates them."""
    st = Stream(rng)
    for side, n in ((0, 900), (1, 1100)):
        st.send(side, rng.integers(0, 30, n), T0 + (1 << 32) * rng.integers(0, 5, n))
    st.wm(T0 + 4 * (1 << 32))
    st.wm(1 << 64)
    return st


def shape_ts_eq_wm(rng):
    """Rows at the watermark wait for the next one; rows one ns below it leave."""
    st = Stream(rng)
    for side, n in ((0, 600), (1, 500)):
        st.send(side, rng.integers(0, 50, n), T0 + W - rng.integers(0, 2, n))
    st.wm(T0 + W)
    st.send(0, rng.integers(0, 50, 100), np.full(100, T0 + W))
    st.wm(T0 + W + 1)
    st.wm(1 << 64)
    return st


def shape_hot_key(rng):
    """One instant: key 7 has 2000 left x 3000 right rows; cold keys match once or not at all."""
    st = Stream(rng)
    lk = np.concatenate([np.full(2000, 7), np.arange(1000, 1500)])
    rk = np.concatenate([np.full(3000, 7), np.arange(1250, 1750)])
    st.send(0, rng.permutation(lk), np.full(len(lk), T0))
    st.send(1, rng.permutation(rk), np.full(len(rk), T0))
    st.wm(1 << 64)
    return st


def _routing(n):
    def f(rng):
        return _instants(Stream(rng, left=WIDE_L, right=WIDE_R, n_routing=n), 333, 401, 150, 3)
    return f


SHAPES = {
    "left_smaller": shape_left_smaller, "right_smaller": shape_right_smaller, "equal": shape_equal,
    "zero_eligible": shape_zero_eligible, "left_only": shape_left_only, "right_only": shape_right_only,
    "build_1": _build(1), "build_511": _build(511), "build_512": _build(512), "build_513": _build(513),
    "buffered_70k": shape_buffered_70k, "edge_keys": shape_edge_keys, "u64_keys": shape_u64_keys,
    "ts_keys": shape_ts_keys, "many_instants": shape_many_instants, "ts_2p32": shape_ts_2p32,
    "ts_eq_wm": shape_ts_eq_wm, "hot_key": shape_hot_key, "routing0": _routing(0), "routing1": _routing(1),
    "routing2": _routing(2),
}
# (shape, entry point): host batches for every shape, the other entry points on a cross section
INSTANT_CASES = [(s, "host") for s in SHAPES] + [
    ("left_smaller", "parts4"), ("routing2", "parts4"), ("edge_keys", "sliced"), ("routing1", "sliced"),
    ("buffered_70k", "device"), ("u64_keys", "device"), ("routing2", "device"), ("ts_2p32", "mixed"),
    ("routing1", "mixed"), ("zero_eligible", "mixed")]


def run_instant(st: Stream, join_type, entry, seed=0):
    """Drives the CUDA InstantJoin through arroyo_b200.operators; returns the output of each watermark as X.Rows."""
    import torch

    import arroyo_b200 as ab
    from arroyo_b200 import ffi, operators as native
    from arroyo_b200.context import clamp_watermark
    rng = np.random.default_rng(seed)
    parts = 4 if entry == "parts4" else 2
    dev_sides = {"device": (0, 1), "mixed": (1,)}.get(entry, ())
    cfg = ab.JoinConfig(left_on=[st.on[0]], right_on=[st.on[1]], join_type=join_type,
                        left_routing_keys=list(st.routing[0]), right_routing_keys=list(st.routing[1]))
    kw = {}
    if dev_sides:  # device input goes straight to the handle: the layouts must be known up front
        kw = {"left_schema": arrow_schema(st.schemas[0]), "right_schema": arrow_schema(st.schemas[1])}
    op = native.InstantJoin(cfg, **kw)
    ctx = ab.OperatorContext(parts)
    lib = op._lib
    keep, outs, sent = [], [], [0, 0]
    dev_out = entry == "device" and join_type == "inner"
    for ev, arg in st.events:
        if ev == "wm":
            for i in range(parts):
                ctx.watermarks.set(i, arg)
            if dev_out:
                outb = (ffi.DeviceBatch * 4)()
                n = C.c_int64(0)
                native._check(lib, op._h, lib.arroyo_b200_op_handle_watermark_device(op._h, clamp_watermark(arg), outb, 4,
                                                                                     C.byref(n)))
                names = op.output_names()
                vals = []
                for b in range(n.value):
                    assert outb[b].n_cols == len(names)
                    cols = [torch.as_tensor(_Ptr(outb[b].cols[c], outb[b].n_rows), device="cuda").cpu().numpy()
                            for c in range(outb[b].n_cols)]
                    vals.append(np.stack(cols, axis=1).view(np.uint64))
                v = np.concatenate(vals) if vals else np.zeros((0, len(names)), np.uint64)
                outs.append(X.Rows(names, v, np.ones(v.shape, bool)))
            else:
                col = ab.Collector()
                op.handle_watermark(arg, ctx, col)
                outs.append(col.batches)
            continue
        side, cols = ev, arg
        index = side * (parts // 2) + sent[side] % (parts // 2)
        sent[side] += 1
        if side in dev_sides:
            dev = [torch.from_numpy(np.ascontiguousarray(cols[name]).view(np.int64)).cuda() for name, _ in st.schemas[side]]
            torch.cuda.synchronize()
            keep.append(dev)
            arr = (C.c_uint64 * len(dev))(*[t.data_ptr() for t in dev])
            native._check(lib, op._h, lib.arroyo_b200_op_process_device_batch(op._h, index, parts, arr, len(dev),
                                                                              len(cols[TS])))
        elif entry == "sliced":
            for piece in _slices(to_arrow(st.schemas[side], cols), rng):
                op.process_batch_index(index, parts, piece, ctx, None)
        else:
            op.process_batch_index(index, parts, to_arrow(st.schemas[side], cols), ctx, None)
    stats = op.stats() if op.created else None
    op.close()
    return outs, stats, dev_sides


def arrow_schema(schema):
    return pa.schema([(name, ARROW[code]) for name, code in schema])


def _types_ok(st, rb, dev_sides):
    """Every output column keeps its input column's Arrow type (host-fed sides: the device path carries none)."""
    want = []
    for side in (0, 1):
        for name, code in st.schemas[side]:
            if name != TS and name not in st.routing[side]:
                want.append(None if side in dev_sides else ARROW[code])
    want.append(pa.timestamp("ns"))
    for f, t in zip(rb.schema, want):
        if t is not None:
            assert f.type == t, (f.name, f.type, t)


@pytest.mark.parametrize("join_type", JOIN_TYPES)
@pytest.mark.parametrize("shape,entry", INSTANT_CASES, ids=[f"{s}-{e}" for s, e in INSTANT_CASES])
def test_instant_join(shape, entry, join_type):
    st = SHAPES[shape](np.random.default_rng(zlib.crc32(shape.encode())))
    want = st.reference_instant(join_type)
    got, stats, dev_sides = run_instant(st, join_type, entry)
    assert len(got) == len(want)
    total = 0
    for i, (w, g) in enumerate(zip(want, got)):
        if not isinstance(g, X.Rows):
            assert len(g) <= 1  # one batch per watermark at most
            names = g[0].schema.names if g else w.names
            if g and "__none" not in names:
                _types_ok(st, g[0], dev_sides)
            g = rows_of(g, names)
            if "__none" in names:  # the side that never sent a row: its stand-in column is all null
                c = names.index("__none")
                assert not g.valid[:, c].any()
                keep = [j for j in range(len(names)) if j != c]
                g = X.Rows([names[j] for j in keep], g.vals[:, keep], g.valid[:, keep])
        check(w, g, (shape, entry, join_type, "watermark", i))
        total += len(w)
    if stats is not None:
        assert stats["rows_out"] == total
    # only these cases may emit nothing: no eligible rows of one side meet the other's, or one side sends nothing
    if shape not in ("zero_eligible", "left_only", "right_only") or join_type == "full":
        assert total > 0


def test_instant_join_hot_key_counts():
    """The hot-key instant emits 2000 x 3000 pairs plus one row per matched cold key."""
    st = shape_hot_key(np.random.default_rng(1))
    want = st.reference_instant("inner")
    assert len(want[-1]) == 2000 * 3000 + 250


def test_instant_join_late_rows():
    """A row older than the previous watermark panics at the next watermark; a row at that watermark is accepted."""
    import arroyo_b200 as ab
    from arroyo_b200 import ffi
    st = Stream(np.random.default_rng(5))
    st.send(0, [1, 2, 3], [T0] * 3)
    st.send(1, [1, 2, 4], [T0] * 3)
    st.wm(T0 + W)
    st.send(0, [5, 6], [T0 + W] * 2)  # == the previous watermark: accepted
    st.send(1, [5, 7], [T0 + W, T0 + 2 * W])
    st.wm(T0 + 2 * W)
    want = st.reference_instant("full")
    got, _, _ = run_instant(st, "full", "host")
    for w, g in zip(want, got):
        check(w, rows_of(g, w.names), "late")
    assert len(want[1]) == 2  # 5 matched, 6 alone; the right row at T0 + 2 W waits
    # one row of the next batch is older than T0 + 2 W
    st.send(1, [8, 9], [T0 + 2 * W, T0 + 2 * W - 1])
    with pytest.raises(ValueError):
        st.reference_instant("full")
    from arroyo_b200 import operators as native
    op = native.InstantJoin(ab.JoinConfig(left_on=["id"], right_on=["id"], join_type="full"))
    ctx = ab.OperatorContext(2)
    for ev, arg in st.events:
        if ev == "wm":
            ctx.watermarks.set(0, arg)
            ctx.watermarks.set(1, arg)
            op.handle_watermark(arg, ctx, ab.Collector())
        else:
            op.process_batch_index(ev, 2, to_arrow(st.schemas[ev], arg), ctx, None)
    ctx.watermarks.set(0, T0 + 3 * W)
    ctx.watermarks.set(1, T0 + 3 * W)
    with pytest.raises(ffi.ArroyoB200Error) as e:
        op.handle_watermark(T0 + 3 * W, ctx, ab.Collector())
    assert e.value.status == ffi.PANIC
    op.close()


# ---------------------------------------------------------------------------------------------------------------
# JoinWithExpiration shapes
# ---------------------------------------------------------------------------------------------------------------
def _alternating(st, n_batches, n_max, key_fn):
    rng = st.rng
    t = T0
    for i in range(n_batches):
        side = int(rng.integers(0, 2)) if i > 1 else i
        n = int(rng.integers(1, n_max))
        st.send(side, key_fn(n), t + np.arange(n))
        t += n
    return st


def tshape_edge_keys(rng):
    return _alternating(Stream(rng), 16, 3000, lambda n: _edge_keys(rng, n, 400, 0.04))


def tshape_u64_keys(rng):
    st = Stream(rng, key_type="L")
    return _alternating(st, 12, 2000, lambda n: [(1 << 63) + int(x) if x % 2 else int(x) for x in rng.integers(0, 300, n)])


def tshape_ts_keys(rng):
    left = [("window_start", "tsn:"), ("a", "l"), (TS, "tsn:")]
    right = [("window_start", "tsn:"), ("b", "g"), (TS, "tsn:")]
    st = Stream(rng, left=left, right=right, left_on="window_start", right_on="window_start", key_type="tsn:")
    return _alternating(st, 10, 1500, lambda n: T0 - W * rng.integers(0, 200, n))


def tshape_rehash(rng):
    """320 k left rows in 16 batches (the multimap grows from 2^16 to 2^20 slots, four rehashes while chains are
    live), a right batch probing after each."""
    st = Stream(rng)
    t = T0
    for i in range(16):
        st.send(0, rng.integers(0, 100_000, 20_000), t + np.arange(20_000))
        t += 20_000
        st.send(1, rng.integers(0, 100_000, 1_000), t + np.arange(1_000))
        t += 1_000
    return st


def tshape_one_key_batch(rng):
    """Every row of a batch on one key (one head for all threads), probed from the other side, then grown."""
    st = Stream(rng)
    st.send(0, np.full(8_000, 42), T0 + np.arange(8_000))
    st.send(1, np.concatenate([np.full(3, 42), rng.integers(0, 50, 100)]), T0 + 10_000 + np.arange(103))
    st.send(0, np.full(4_000, 42), T0 + 20_000 + np.arange(4_000))
    return st


def tshape_long_chain(rng):
    """A 50 k-row chain probed by 20 rows of a later batch: 10^6 pairs."""
    st = Stream(rng)
    st.send(0, np.full(50_000, 5), T0 + np.arange(50_000))
    st.send(1, np.concatenate([np.full(20, 5), np.arange(100, 130)]), T0 + 60_000 + np.arange(50))
    return st


def tshape_zero_rows(rng):
    st = Stream(rng)
    st.send(0, [], [])
    st.send(1, [], [])
    st.send(0, rng.integers(0, 20, 300), T0 + np.arange(300))
    st.send(1, [], [])
    st.send(1, rng.integers(0, 20, 200), T0 + 1000 + np.arange(200))
    st.send(0, [], [])
    st.send(0, rng.integers(0, 20, 100), T0 + 2000 + np.arange(100))
    return st


def tshape_one_side_first(rng):
    st = Stream(rng)
    for i in range(6):
        st.send(0, rng.integers(0, 500, 1500), T0 + i * 2000 + np.arange(1500))
    for i in range(6):
        st.send(1, rng.integers(0, 500, 700), T0 + 20_000 + i * 1000 + np.arange(700))
    st.send(0, rng.integers(0, 500, 900), T0 + 40_000 + np.arange(900))
    return st


def _trouting(n):
    def f(rng):
        return _alternating(Stream(rng, left=WIDE_L, right=WIDE_R, n_routing=n), 12, 1500, lambda m: rng.integers(0, 200, m))
    return f


TSHAPES = {
    "edge_keys": tshape_edge_keys, "u64_keys": tshape_u64_keys, "ts_keys": tshape_ts_keys, "rehash": tshape_rehash,
    "one_key_batch": tshape_one_key_batch, "long_chain": tshape_long_chain, "zero_rows": tshape_zero_rows,
    "one_side_first": tshape_one_side_first, "routing0": _trouting(0), "routing1": _trouting(1),
    "routing2": _trouting(2),
}
EXPIRING_CASES = [(s, "host") for s in TSHAPES] + [
    ("edge_keys", "parts4"), ("routing2", "parts4"), ("routing1", "sliced"), ("rehash", "sliced"),
    ("u64_keys", "sliced")]


def run_expiring(st: Stream, entry, seed=0):
    """Drives the CUDA JoinWithExpiration; returns the output of each batch event as X.Rows."""
    import arroyo_b200 as ab
    from arroyo_b200 import operators as native
    rng = np.random.default_rng(seed)
    parts = 4 if entry == "parts4" else 2
    cfg = ab.JoinConfig(left_on=[st.on[0]], right_on=[st.on[1]], join_type="inner",
                        left_routing_keys=list(st.routing[0]), right_routing_keys=list(st.routing[1]))
    op = native.JoinWithExpiration(cfg)
    ctx = ab.OperatorContext(parts)
    outs, sent = [], [0, 0]
    for side, cols in st.events:
        index = side * (parts // 2) + sent[side] % (parts // 2)
        sent[side] += 1
        col = ab.Collector()
        rb = to_arrow(st.schemas[side], cols)
        for piece in (_slices(rb, rng) if entry == "sliced" and rb.num_rows else [rb]):
            op.process_batch_index(index, parts, piece, ctx, col)
        outs.append(col.batches)
    stats = op.stats() if op.created else None
    op.close()
    return outs, stats


@pytest.mark.parametrize("shape,entry", EXPIRING_CASES, ids=[f"{s}-{e}" for s, e in EXPIRING_CASES])
def test_expiring_join(shape, entry):
    st = TSHAPES[shape](np.random.default_rng(zlib.crc32(shape.encode()) + 1))
    want = st.reference_expiring()
    got, stats = run_expiring(st, entry)
    assert len(got) == len(want)
    total = 0
    for i, (w, g) in enumerate(zip(want, got)):
        for rb in g:
            _types_ok(st, rb, ())
        check(w, rows_of(g, w.names), (shape, entry, "batch", i))
        total += len(w)
    assert total > 0 and stats["rows_out"] == total


# ---------------------------------------------------------------------------------------------------------------
# refusals
# ---------------------------------------------------------------------------------------------------------------
def _make(kind, st, join_type="inner"):
    import arroyo_b200 as ab
    from arroyo_b200 import operators as native
    cfg = ab.JoinConfig(left_on=[st.on[0]], right_on=[st.on[1]], join_type=join_type,
                        left_routing_keys=list(st.routing[0]), right_routing_keys=list(st.routing[1]))
    cls = native.InstantJoin if kind == "instant" else native.JoinWithExpiration
    return cls(cfg, left_schema=arrow_schema(st.schemas[0]), right_schema=arrow_schema(st.schemas[1]))


def _bad_batch(st, what, rng):
    """A right-side batch the join must refuse: a Float64 key, or a UInt64 key against Int64 keys."""
    n = 40
    schema = [(name, ("g" if what == "f64_key" else "L") if name == st.on[1] else code) for name, code in st.schemas[1]]
    cols = {name: (rng.integers(0, 30, n).astype(NP[code]) if name != TS else np.full(n, T0, dtype=np.int64))
            for name, code in schema}
    return to_arrow(schema, cols)


@pytest.mark.parametrize("kind", ["instant", "expiring"])
@pytest.mark.parametrize("what,where", [("f64_key", "first"), ("f64_key", "mid"), ("u64_vs_i64_key", "first"),
                                        ("u64_vs_i64_key", "mid")])
def test_refused_key_types_leave_the_join_intact(kind, what, where):
    """A Float64 key, or keys whose types differ between the sides, are refused (UNSUPPORTED) before any state
    changes; the valid batches around the refused one join exactly as if it had never been sent."""
    import arroyo_b200 as ab
    from arroyo_b200 import ffi
    rng = np.random.default_rng(11)
    st = Stream(rng)
    for i in range(4):
        st.send(0, rng.integers(0, 30, 200), np.full(200, T0 + i))
        st.send(1, rng.integers(0, 30, 150), np.full(150, T0 + i))
    st.wm(1 << 64)
    op = _make(kind, st, "full" if kind == "instant" else "inner")
    ctx = ab.OperatorContext(2)
    bad_at = 1 if where == "first" else 4  # the right side's first batch, or one in the middle of the stream
    got = []
    for i, (ev, arg) in enumerate(st.events):
        if i == bad_at:
            with pytest.raises(ffi.UnsupportedPlan):
                op.process_batch_index(1, 2, _bad_batch(st, what, rng), ctx, ab.Collector())
        col = ab.Collector()
        if ev == "wm":
            if kind == "instant":
                ctx.watermarks.set(0, arg)
                ctx.watermarks.set(1, arg)
                op.handle_watermark(arg, ctx, col)
                got.append(col.batches)
        else:
            op.process_batch_index(ev, 2, to_arrow(st.schemas[ev], arg), ctx, col)
            if kind == "expiring":
                got.append(col.batches)
    if kind == "instant":
        want = st.reference_instant("full")
    else:
        st.events = [e for e in st.events if e[0] != "wm"]
        want = st.reference_expiring()
    assert len(got) == len(want)
    for w, g in zip(want, got):
        check(w, rows_of(g, w.names), (kind, what, where))
    assert sum(len(w) for w in want) > 0
    op.close()


@pytest.mark.parametrize("kind", ["instant", "expiring"])
@pytest.mark.parametrize("col", ["key", "timestamp"])
def test_key_or_timestamp_among_routing_columns_is_refused(kind, col):
    """The routing copies never reach the device, so a join on one of them, or a timestamp among them, is refused when
    the operator is created."""
    from arroyo_b200 import ffi
    st = Stream(np.random.default_rng(0), n_routing=1)
    if col == "key":
        st.on = ("_key_0", "id")
    else:
        st.routing = ((TS,), ())
        st.schemas[0] = [(TS, "tsn:")] + [(n, c) for n, c in st.schemas[0] if n not in (TS, "_key_0")]
        st.schemas[1] = [(n, c) for n, c in st.schemas[1] if n != "_key_0"]
    with pytest.raises(ffi.ArroyoB200Error) as e:
        _make(kind, st)
    assert e.value.status in (ffi.INVALID_ARGUMENT, ffi.UNSUPPORTED)


@pytest.mark.parametrize("kind", ["instant", "expiring"])
def test_device_input_index_out_of_range_is_refused(kind):
    """process_device_batch with an input index >= in_partitions is refused; the join goes on correctly after it."""
    import torch

    import arroyo_b200 as ab
    from arroyo_b200 import ffi, operators as native
    rng = np.random.default_rng(12)
    st = Stream(rng)
    st.send(0, rng.integers(0, 30, 300), np.full(300, T0))
    st.send(1, rng.integers(0, 30, 200), np.full(200, T0))
    st.wm(T0 + 1)
    op = _make(kind, st)
    dev = [torch.from_numpy(np.ascontiguousarray(st.events[0][1][n]).view(np.int64)).cuda() for n, _ in st.schemas[0]]
    torch.cuda.synchronize()
    arr = (C.c_uint64 * len(dev))(*[t.data_ptr() for t in dev])
    for index, parts in ((2, 2), (3, 2), (4, 4), (9, 4)):
        st_code = op._lib.arroyo_b200_op_process_device_batch(op._h, index, parts, arr, len(dev), 300)
        assert st_code in (ffi.INVALID_ARGUMENT, ffi.UNSUPPORTED), (index, parts, st_code)
    if kind == "expiring":
        assert st_code == ffi.UNSUPPORTED  # no device input at all
        op.close()
        return
    ctx = ab.OperatorContext(2)
    native._check(op._lib, op._h, op._lib.arroyo_b200_op_process_device_batch(op._h, 0, 2, arr, len(dev), 300))
    op.process_batch_index(1, 2, to_arrow(st.schemas[1], st.events[1][1]), ctx, None)
    ctx.watermarks.set(0, T0 + 1)
    ctx.watermarks.set(1, T0 + 1)
    col = ab.Collector()
    op.handle_watermark(T0 + 1, ctx, col)
    want = st.reference_instant("inner")[0]
    assert len(want) > 0
    check(want, rows_of(col.batches, want.names), "after refusal")
    op.close()


def test_device_output_wider_than_a_device_batch_is_refused():
    """Device-resident output carries at most ARROYO_B200_MAX_COLS columns: a wider join refuses it (UNSUPPORTED)
    without losing rows, and the host output of the same watermark is complete."""
    import arroyo_b200 as ab
    from arroyo_b200 import ffi
    rng = np.random.default_rng(13)
    left = [("id", "l")] + [(f"a{i}", "l") for i in range(8)] + [(TS, "tsn:")]
    right = [("id", "l")] + [(f"b{i}", "l") for i in range(8)] + [(TS, "tsn:")]
    st = Stream(rng, left=left, right=right)
    st.send(0, rng.integers(0, 20, 100), np.full(100, T0))
    st.send(1, rng.integers(0, 20, 100), np.full(100, T0))
    st.wm(T0 + 1)
    op = _make("instant", st)
    ctx = ab.OperatorContext(2)
    for ev, arg in st.events[:2]:
        op.process_batch_index(ev, 2, to_arrow(st.schemas[ev], arg), ctx, None)
    outb = (ffi.DeviceBatch * 4)()
    n = C.c_int64(0)
    code = op._lib.arroyo_b200_op_handle_watermark_device(op._h, T0 + 1, outb, 4, C.byref(n))
    assert code == ffi.UNSUPPORTED
    ctx.watermarks.set(0, T0 + 1)
    ctx.watermarks.set(1, T0 + 1)
    col = ab.Collector()
    op.handle_watermark(T0 + 1, ctx, col)
    want = st.reference_instant("inner")[0]
    assert len(want) > 0
    check(want, rows_of(col.batches, want.names), "host output after the refusal")
    op.close()
