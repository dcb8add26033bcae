"""The CUDA updating aggregate (csrc/updating_agg.cu) against tests/exact_reference.updating_changes, flush by flush:
which keys each flush retracts and appends, what a retraction carries, and when a change is suppressed.

Every stream is an explicit list of ("batch", cols) and ("flush",) events.  The shapes go where the operator has edges:
every aggregate kind held unchanged while its key is touched, a flush that suppresses every key, a key suppressed at
one flush and changed at the next, timestamps that go backwards, flush cadences, empty and one-row batches, edge keys
(0, +-1, INT64_MIN, INT64_MAX), UInt64 and timestamp keys, the unkeyed operator, dictionary growth from one expected
key to 10^6 keys while touched keys wait for their flush, INT64_MIN / INT64_MAX values, one hot key with 2^22 rows,
and keys built to crowd one dictionary bucket at two sizes.  They run over a cross section of plans and entry points
(host batches, Arrow slices, device batches, runs of device batches, host and device mixed); the flushes go through
handle_tick, handle_checkpoint and on_close(end_of_data) in turn.  The crowded keys also run through the tumbling and
sliding window aggregates, against exact_reference.window_emissions."""
import ctypes as C
import zlib

import numpy as np
import pyarrow as pa
import pytest

from oracle import arroyo_oracle as O
from oracle import updating_oracle as U
from tests import exact_reference as X
from tests.test_gpu_agg_plans import PLANS as AGG_PLANS
from tests.test_gpu_agg_plans import SIZES

pytestmark = pytest.mark.gpu

A = O.Agg
TS = O.TIMESTAMP
I64_MIN, I64_MAX = -(1 << 63), (1 << 63) - 1
T0 = 1_700_000_000_000_000_000
VALS = ("a", "b", "c", "d")
PLANS = dict(AGG_PLANS,
             COUNT=[A("count", None, "n")],
             AMM=[A("avg", "a", "ava"), A("min", "a", "mna"), A("max", "a", "mxa")],
             MM=[A("min", "a", "mna"), A("max", "b", "mxb")])

# A restatement of the key dictionary's bucket function, bdict.cuh: bd_hash = (k ^ (k >> 32)) * 0x9E3779B97F4A7C15,
# bd_bucket = ((h >> 32) * n_buckets) >> 32.  A bucket holds BD_CAPB = 1280 ids; the operator sizes the dictionary at
# BD_MEAN = 1024 keys per bucket (expected_keys 65536 -> 64 buckets).
BD_MULT, BD_CAPB, BD_MEAN = 0x9E3779B97F4A7C15, 1280, 1024


def bd_bucket(keys, n_buckets):
    k = np.asarray(keys, dtype=np.int64).view(np.uint64)
    with np.errstate(over="ignore"):
        h = (k ^ (k >> np.uint64(32))) * np.uint64(BD_MULT)
    return ((h >> np.uint64(32)) * np.uint64(n_buckets)) >> np.uint64(32)


def crowded_keys(n, n_buckets=64):
    """`n` keys that all land in bucket 0 at `n_buckets` and at 2 * n_buckets (a bucket at 2b buckets is one of the
    two halves of a bucket at b), so one doubling does not split them."""
    cand = np.arange(1, 2_000_000, dtype=np.int64)
    keys = cand[bd_bucket(cand, 2 * n_buckets) == 0][:n]
    assert len(keys) == n and (bd_bucket(keys, n_buckets) == 0).all()
    return keys


class Stream:
    """Events for one operator: batches of [key?, a, b, c, d, _timestamp] and flushes."""

    def __init__(self, seed, key_type="i64", expected_keys=0):
        self.rng = np.random.default_rng(seed)
        self.key_type, self.expected_keys = key_type, expected_keys  # key_type None: unkeyed
        self.events = []
        self.t = T0

    def batch(self, keys=None, n=None, vals=None, ts=None):
        n = len(keys) if keys is not None else n
        cols = {}
        if self.key_type is not None:
            k = np.asarray(keys if keys is not None else self.rng.integers(0, 50, n))
            if k.dtype == object:  # Python ints, UInt64 keys up to 2^64 - 1
                k = np.array([int(x) % (1 << 64) for x in k], dtype=np.uint64)
            # UInt64 keys: a negative Int64 stands for its two's complement (>= 2^63)
            k = k.astype(np.uint64 if k.dtype == np.uint64 else np.int64)
            cols["k"] = k.view(np.uint64) if self.key_type == "u64" else k.view(np.int64)
        for i, c in enumerate(VALS):
            v = vals[c] if vals is not None and c in vals else self.rng.integers(-10**6, 10**6, n)
            cols[c] = np.asarray(v, dtype=np.int64).reshape(n)
        if ts is None:
            ts = self.t + self.rng.integers(0, 1000, n)
            self.t += 1000
        cols[TS] = np.asarray(ts, dtype=np.int64).reshape(n)
        self.events.append(("batch", cols))

    def flush(self):
        self.events.append(("flush",))

    def schema(self):
        kt = {"i64": pa.int64(), "u64": pa.uint64(), "ts": pa.timestamp("ns")}
        f = [("k", kt[self.key_type])] if self.key_type else []
        return pa.schema(f + [(c, pa.int64()) for c in VALS] + [(TS, pa.timestamp("ns"))])

    def key_name(self):
        return "k" if self.key_type else None


def to_arrow(cols, schema):
    arrays = []
    for f in schema:
        v = np.ascontiguousarray(cols[f.name])
        arrays.append(pa.array(v.view(np.int64), type=pa.int64()).cast(f.type) if f.type != pa.uint64()
                      else pa.array(v, type=pa.uint64()))
    return pa.RecordBatch.from_arrays(arrays, names=schema.names)


# ---- shapes --------------------------------------------------------------------------------------------------------
def s_random(seed, key_type="i64", every=2, n_batches=12):
    """Random rows over 300 keys, flushed every `every` batches (0: only at the end)."""
    st = Stream(seed, key_type)
    for i in range(n_batches):
        st.batch(keys=st.rng.integers(0, 300, int(st.rng.integers(1, 1500))) * 7919 - 500)
        if every and (i + 1) % every == 0:
            st.flush()
    st.flush()
    return st


class _Quiet:
    """Per-key state of a plan's value columns, to build rows that leave every aggregate of the plan unchanged."""

    def __init__(self, plan):
        self.plan, self.s = plan, {}

    def change(self, st, k, n):
        """n random rows for key k; for AMM the last row makes the key's mean an integer."""
        v = {c: st.rng.integers(-1000, 1000, n) for c in VALS}
        s = self.s.setdefault(k, {"n": 0, "sa": 0, "mna": None, "mxa": None, "mnb": None, "mxb": None})
        if self.plan == "AMM":
            m = int(st.rng.integers(-500, 500))
            v["a"][-1] = m * (s["n"] + n) - s["sa"] - int(v["a"][:-1].sum())
        self._add(s, v, n)
        return v

    def _add(self, s, v, n):
        s["n"] += n
        s["sa"] += int(v["a"].sum())
        for c, lo, hi in (("a", "mna", "mxa"), ("b", "mnb", "mxb")):
            s[lo] = int(v[c].min()) if s[lo] is None else min(s[lo], int(v[c].min()))
            s[hi] = int(v[c].max()) if s[hi] is None else max(s[hi], int(v[c].max()))

    def quiet(self, st, k, n):
        """n rows for key k that change no output of the plan (only _timestamp moves)."""
        s = self.s[k]
        v = {c: st.rng.integers(-1000, 1000, n) for c in VALS}
        if self.plan == "P1":  # sum a: zeros or +x, -x; min b: values above the minimum
            x = st.rng.integers(1, 10**6, n)
            pairs = n % 2 == 0 and st.rng.random() < 0.5
            v["a"] = np.where(np.arange(n) % 2 == 0, x, -np.roll(x, 1)) if pairs else np.zeros(n, np.int64)
            v["b"] = s["mnb"] + st.rng.integers(0, 10**6, n)
        elif self.plan == "MM":  # min a fed larger values, max b fed smaller ones
            v["a"] = s["mna"] + st.rng.integers(0, 10**6, n)
            v["b"] = s["mxb"] - st.rng.integers(0, 10**6, n)
        elif self.plan == "AMM":  # the current mean: AVG, MIN and MAX all stay
            assert s["sa"] % s["n"] == 0
            v["a"] = np.full(n, s["sa"] // s["n"])
        else:
            raise ValueError(self.plan)
        self._add(s, v, n)
        return v


def s_quiet(seed, plan, key_type="i64", whole_flush=False):
    """Keys that are touched but unchanged.  Period 0 creates keys 0..39; in later periods each touched key gets quiet
    rows or random rows at random.  Key 7 is quiet in period 1 and changed in period 2 (its retraction carries the
    _timestamp that moved in period 1).  With `whole_flush`, period 3 holds quiet rows only (for a plan without COUNT:
    its flush emits nothing)."""
    st, q = Stream(seed, key_type), _Quiet(plan)
    keys = list(range(40))

    def send(rows):
        ks = np.concatenate([np.full(len(v["a"]), k) for k, v in rows])
        st.batch(keys=ks, vals={c: np.concatenate([v[c] for _, v in rows]) for c in VALS})

    send([(k, q.change(st, k, int(st.rng.integers(1, 4)))) for k in keys])
    st.flush()
    for period in range(1, 6):
        for _ in range(2):
            rows = []
            for k in st.rng.choice(keys, 15, replace=False).tolist() + [7]:
                n = int(st.rng.integers(1, 4)) * 2
                if k == 7 and period in (1, 2):
                    quiet = period == 1
                else:
                    quiet = (whole_flush and period == 3) or st.rng.random() < 0.6
                rows.append((k, q.quiet(st, k, n) if quiet else q.change(st, k, n)))
            send(rows)
        st.flush()
    return st


def s_ts_backwards(seed, plan_quiet="P1"):
    """Timestamps of later batches below earlier ones, and quiet rows whose timestamps are lower (max unchanged)."""
    st, q = Stream(seed), _Quiet(plan_quiet)
    for i in range(6):
        keys = np.arange(30)
        rows = [(k, q.change(st, k, 2) if i % 2 == 0 else q.quiet(st, k, 2)) for k in keys]
        ts = T0 + 10**9 - i * 10**6 + st.rng.integers(-5000, 5000, 60)
        st.batch(keys=np.repeat(keys, 2), vals={c: np.concatenate([v[c] for _, v in rows]) for c in VALS}, ts=ts)
        st.flush()
    return st


def s_cadence(seed, how):
    st = Stream(seed)
    if how == "tick_first":
        st.flush()
    for i in range(9):
        if how == "empty_and_one":
            st.batch(keys=[] if i % 3 == 0 else st.rng.integers(0, 5, 1 if i % 3 == 1 else 40))
        else:
            st.batch(keys=st.rng.integers(0, 100, 200))
        if how == "every" or (how == "every3" and i % 3 == 2) or how == "empty_and_one":
            st.flush()
        if how == "double" and i % 4 == 1:
            st.flush()
            st.flush()
    st.flush()
    return st


def s_edge_keys(seed, key_type="i64"):
    st = Stream(seed, key_type)
    if key_type == "u64":
        edge = [0, 1, (1 << 63) - 1, 1 << 63, (1 << 63) + 1, (1 << 64) - 2, (1 << 64) - 1]
    else:
        edge = [0, 1, -1, I64_MIN, I64_MAX, I64_MIN + 1, I64_MAX - 1]
    edge = np.array(edge, dtype=np.uint64 if key_type == "u64" else np.int64)
    for i in range(8):
        st.batch(keys=st.rng.choice(edge, 50))
        if i % 2:
            st.flush()
    st.flush()
    return st


def s_unkeyed(seed):
    st = Stream(seed, None)
    for i in range(7):
        st.batch(n=[0, 1, 500, 3, 4097, 1, 20][i])
        if i in (0, 1, 3, 4, 6):
            st.flush()
    st.flush()
    return st


def s_growth(seed, n_keys, batches=8):
    """Keys spread from a dictionary sized for one key to `n_keys` keys; the first flush comes after half the
    batches, so the dictionary doubles several times while the touched list and the previous-flush values are live.
    INT64_MIN is one of the keys."""
    st = Stream(seed, "i64", expected_keys=1)
    universe = np.unique(st.rng.integers(-(1 << 62), 1 << 62, n_keys + n_keys // 10))[:n_keys]
    universe[0] = I64_MIN
    per = len(universe) // (batches // 2)
    for i in range(batches):
        if i < batches // 2:
            ks = universe[i * per:(i + 1) * per] if i < batches // 2 - 1 else universe[i * per:]
            ks = np.concatenate([ks, universe[:1]])
        else:
            ks = st.rng.choice(universe, len(universe) // 3)
        st.batch(keys=st.rng.permutation(ks))
        if i == batches // 2 - 1 or i == batches - 2:
            st.flush()
    st.flush()
    return st


def s_edge_values(seed):
    """INT64_MIN and INT64_MAX in SUM (wrapping), MIN, MAX and AVG (sum of |x| far past 2^53: the plan has COUNT)."""
    st = Stream(seed)
    edge = np.array([I64_MIN, I64_MAX, I64_MIN + 1, I64_MAX - 1, -1, 0, 1], dtype=np.int64)
    for i in range(6):
        n = 300
        vals = {c: st.rng.choice(edge, n) for c in VALS}
        st.batch(keys=st.rng.integers(0, 20, n), vals=vals)
        if i % 2:
            st.flush()
    st.flush()
    return st


def s_hot(seed):
    """One hot key with 2^22 rows in one batch, next to a few cold keys."""
    st = Stream(seed)
    n = 1 << 22
    keys = np.full(n, 99, dtype=np.int64)
    keys[::4096] = np.arange(n // 4096)
    st.batch(keys=[5, 99], vals={c: np.array([1, 2]) for c in VALS})
    st.flush()
    vals = {c: st.rng.integers(-(1 << 30), 1 << 30, n) for c in VALS}
    st.batch(keys=keys, vals=vals, ts=T0 + st.rng.integers(0, 10**12, n))
    st.flush()
    return st


def s_crowded(seed, n, spread=False):
    """Keys that share bucket 0 of a 64- and a 128-bucket dictionary: `n` of them in one batch (more than a bucket
    holds, far fewer than the dictionary's size), or spread over batches with flushes in between."""
    st = Stream(seed, "i64", expected_keys=1 << 16)
    keys = crowded_keys(n)
    if not spread:
        st.batch(keys=st.rng.permutation(np.concatenate([keys, keys[: n // 3]])))
        st.flush()
        st.batch(keys=st.rng.choice(keys, 500))
    else:
        cut = [0, 1000, 1200, 1300, n]
        for i in range(4):
            ks = keys[cut[i]:cut[i + 1]]
            st.batch(keys=st.rng.permutation(np.concatenate([ks, st.rng.choice(keys[:cut[i + 1]], 200)])))
            st.flush()
    st.flush()
    return st


SHAPES = {
    "random": lambda s: s_random(s),
    "random_u64": lambda s: s_random(s, "u64", every=3),
    "random_ts": lambda s: s_random(s, "ts", every=1),
    "quiet_P1": lambda s: s_quiet(s, "P1"),
    "quiet_MM": lambda s: s_quiet(s, "MM"),
    "quiet_AMM": lambda s: s_quiet(s, "AMM"),
    "quiet_flush_P1": lambda s: s_quiet(s, "P1", whole_flush=True),
    "quiet_flush_AMM": lambda s: s_quiet(s, "AMM", "u64", whole_flush=True),
    "ts_backwards": lambda s: s_ts_backwards(s),
    "every": lambda s: s_cadence(s, "every"),
    "every3": lambda s: s_cadence(s, "every3"),
    "at_end": lambda s: s_cadence(s, "end"),
    "double_tick": lambda s: s_cadence(s, "double"),
    "tick_first": lambda s: s_cadence(s, "tick_first"),
    "empty_and_one": lambda s: s_cadence(s, "empty_and_one"),
    "edge_keys": lambda s: s_edge_keys(s),
    "edge_keys_u64": lambda s: s_edge_keys(s, "u64"),
    "edge_keys_ts": lambda s: s_edge_keys(s, "ts"),
    "unkeyed": lambda s: s_unkeyed(s),
    "growth_1e5": lambda s: s_growth(s, 100_000),
    "growth_1e6": lambda s: s_growth(s, 1_000_000),
    "edge_values": lambda s: s_edge_values(s),
    "hot": lambda s: s_hot(s),
    "crowded_1300": lambda s: s_crowded(s, 1300),
    "crowded_3000": lambda s: s_crowded(s, 3000),
    "crowded_spread": lambda s: s_crowded(s, 2000, spread=True),
}


# ---- driver and checks ---------------------------------------------------------------------------------------------
def reference(st, aggs):
    return X.updating_changes(st.events, st.key_name(), aggs)


def run_gpu(st, aggs, entry):
    """Returns (one RecordBatch or None per flush, stats).  Flushes go through handle_tick, handle_checkpoint and
    on_close(end_of_data) in turn (the last flush is always on_close)."""
    import torch

    import arroyo_b200 as ab
    from arroyo_b200 import operators as native
    schema = st.schema()
    cfg = U.UpdatingAggConfig([st.key_name()] if st.key_type else [], aggs)
    op = native.UpdatingAggregatingFunc(cfg, input_schema=schema, expected_keys=st.expected_keys)
    ctx = ab.OperatorContext(1)
    outs, pending, keep = [], [], []
    n_flushes = sum(1 for ev in st.events if ev[0] == "flush")

    def dev(cols):
        ts = [torch.from_numpy(np.ascontiguousarray(cols[f.name]).view(np.int64)).cuda() for f in schema]
        torch.cuda.synchronize()  # the operator's stream has no ordering against torch's
        keep.append(ts)
        return [t.data_ptr() for t in ts]

    def send_pending():
        if not pending:
            return
        if entry == "sliced":
            allc = {c: np.concatenate([p[c] for p in pending]) for c in schema.names}
            big, s, i = to_arrow(allc, schema), 0, 0
            while s < big.num_rows:
                z = min(SIZES[i % len(SIZES)], big.num_rows - s)
                op.process_batch(big.slice(s, z), ctx, None)
                s, i = s + z, i + 1
        else:  # device_run: one FFI call for every batch since the last flush
            ptrs = [p for cols in pending for p in dev(cols)]
            rows = [len(cols[TS]) for cols in pending]
            op.process_device_batches((C.c_uint64 * len(ptrs))(*ptrs), (C.c_int64 * len(rows))(*rows), len(schema))
        pending.clear()

    n_batch = 0
    for ev in st.events:
        if ev[0] == "batch":
            cols = ev[1]
            if entry in ("sliced", "device_run"):
                pending.append(cols)
            elif entry == "device" or (entry == "mixed" and n_batch % 2 == 1):
                op.process_device_batch(dev(cols), len(cols[TS]))
            else:
                op.process_batch(to_arrow(cols, schema), ctx, None)
            n_batch += 1
            continue
        send_pending()
        col = ab.Collector()
        if len(outs) == n_flushes - 1:
            op.on_close("end_of_data", ctx, col)
        elif len(outs) % 2 == 0:
            op.handle_tick(0, ctx, col)
        else:
            op.handle_checkpoint(None, ctx, col)
        assert len(col.batches) <= 1
        outs.append(col.batches[0] if col.batches else None)
        keep.clear()
    stats = op.stats()
    op.close()
    return outs, stats


def _host(arr):
    if pa.types.is_timestamp(arr.type):
        arr = arr.cast(pa.int64())
    return arr.to_numpy(zero_copy_only=False)


def check(st, aggs, got, stats, want, who=""):
    key = st.key_name()
    names = ([key] if key else []) + [a.name for a in aggs] + [TS, "_is_retract"]
    key_type = st.schema().field(key).type if key else None
    assert len(got) == len(want), (who, len(got), len(want))
    n_out = 0
    merged = []
    for i, (g, (wr, wa)) in enumerate(zip(got, want)):
        if g is None:
            assert not wr and not wa, (who, "flush", i, "emitted nothing", len(wr), len(wa))
            continue
        assert wr or wa, (who, "flush", i, "emitted a batch for no change")
        assert g.schema.names == names, (who, g.schema.names)
        types = {TS: pa.timestamp("ns"), "_is_retract": pa.bool_()}
        if key:
            types[key] = key_type
        for a in aggs:
            types[a.name] = pa.float64() if a.kind == "avg" else pa.int64()
        for f in g.schema:
            assert f.type == types[f.name], (who, f.name, f.type, types[f.name])
        cols = {c: _host(g.column(c)) for c in names}
        r = cols["_is_retract"].astype(bool)
        nr = int(r.sum())
        assert r[:nr].all() and not r[nr:].any(), (who, "flush", i, "a retraction after an append")
        rows = [dict(zip(names, t)) for t in zip(*(cols[c].tolist() for c in names))]
        for part, w in ((rows[:nr], wr), (rows[nr:], wa)):
            errs = X.mismatches(w, part, lambda row: int(row[key]) if key else None)
            assert not errs, (who, "flush", i, errs[:8])
        n_out += len(rows)
        merged.append(O.Batch({**{c: cols[c] for c in names if c != "_is_retract"}, U.IS_RETRACT: r}))
    batches = [O.Batch(ev[1]) for ev in st.events if ev[0] == "batch" and len(ev[1][TS])]
    if batches:
        exact = X.updating_rows(batches, key, aggs)
        final = U.merge_change_stream(merged, [key] if key else [])
        errs = X.mismatches({k: {c: v for c, v in r.items() if c != TS} for k, r in exact.items()}, final,
                            lambda row: int(row[key]) if key else None)
        assert not errs, (who, "merged", errs[:8])
    n_in = sum(len(ev[1][TS]) for ev in st.events if ev[0] == "batch")
    n_keys = len({int(k) for ev in st.events if ev[0] == "batch" for k in ev[1].get("k", [])}) if key else 0
    assert stats["rows_in"] == n_in, (who, stats["rows_in"], n_in)
    assert stats["n_keys"] == n_keys, (who, stats["n_keys"], n_keys)
    assert stats["rows_out"] == n_out, (who, stats["rows_out"], n_out)


# (shape, plan, entry): a cross section of the axes, not their product
CASES = [
    ("random", "P1", "host"), ("random", "P2", "sliced"), ("random", "P3", "device"), ("random", "P4", "mixed"),
    ("random", "P5", "device_run"), ("random", "P6a", "host"), ("random", "P6b", "sliced"), ("random", "P7", "host"),
    ("random", "P8", "device"), ("random", "COUNT", "host"), ("random", "AMM", "mixed"),
    ("random_u64", "P2", "host"), ("random_u64", "P7", "device"), ("random_ts", "P3", "sliced"),
    ("random_ts", "P8", "device_run"),
    ("quiet_P1", "P1", "host"), ("quiet_P1", "P1", "device"), ("quiet_MM", "MM", "sliced"), ("quiet_MM", "MM", "mixed"),
    ("quiet_AMM", "AMM", "host"), ("quiet_AMM", "AMM", "device_run"), ("quiet_flush_P1", "P1", "host"),
    ("quiet_flush_P1", "P1", "device"), ("quiet_flush_AMM", "AMM", "sliced"), ("ts_backwards", "P1", "host"),
    ("ts_backwards", "P1", "mixed"),
    ("every", "P2", "host"), ("every3", "P5", "device"), ("at_end", "P4", "host"), ("double_tick", "P1", "mixed"),
    ("tick_first", "P6b", "host"), ("tick_first", "COUNT", "device"), ("empty_and_one", "P3", "host"),
    ("empty_and_one", "P7", "device"), ("empty_and_one", "P8", "sliced"), ("empty_and_one", "AMM", "device_run"),
    ("edge_keys", "P2", "host"), ("edge_keys", "COUNT", "device"), ("edge_keys", "P6a", "sliced"),
    ("edge_keys_u64", "P3", "host"), ("edge_keys_u64", "P8", "device"), ("edge_keys_ts", "P1", "mixed"),
    ("unkeyed", "P2", "host"), ("unkeyed", "P4", "device"), ("unkeyed", "AMM", "sliced"),
    ("growth_1e5", "P2", "host"), ("growth_1e5", "P1", "device"), ("growth_1e5", "P6b", "sliced"),
    ("growth_1e6", "COUNT", "device_run"),
    ("edge_values", "P3", "host"), ("edge_values", "P5", "device"), ("edge_values", "P7", "mixed"),
    ("hot", "P2", "host"), ("hot", "P4", "device"),
    ("crowded_1300", "P2", "host"), ("crowded_1300", "COUNT", "device"), ("crowded_3000", "P1", "host"),
    ("crowded_3000", "P8", "device_run"), ("crowded_spread", "P3", "host"), ("crowded_spread", "P6a", "device"),
]


@pytest.mark.parametrize("shape,plan,entry", CASES, ids=["-".join(c) for c in CASES])
def test_updating_change_stream(shape, plan, entry):
    st = SHAPES[shape](zlib.crc32(f"{shape}/{plan}/{entry}".encode()))
    aggs = PLANS[plan]
    want = reference(st, aggs)
    got, stats = run_gpu(st, aggs, entry)
    check(st, aggs, got, stats, want, f"{shape}/{plan}/{entry}")
    if shape.startswith("crowded"):
        assert stats["rows_deferred"] > 0, stats
    if shape.startswith("quiet_flush") and not any(a.kind == "count" for a in aggs):
        assert got[3] is None  # the period of quiet rows


def test_on_close_without_end_of_data_emits_nothing():
    import arroyo_b200 as ab
    from arroyo_b200 import operators as native
    st = s_random(3, every=0, n_batches=3)
    aggs = PLANS["P2"]
    schema = st.schema()
    op = native.UpdatingAggregatingFunc(U.UpdatingAggConfig(["k"], aggs), input_schema=schema)
    ctx = ab.OperatorContext(1)
    for ev in st.events[:-1]:
        op.process_batch(to_arrow(ev[1], schema), ctx, None)
    col = ab.Collector()
    op.on_close(None, ctx, col)
    assert not col.batches
    op.on_close("end_of_data", ctx, col)
    assert len(col.batches) == 1
    check(st, aggs, [col.batches[0]], op.stats(), reference(st, aggs))
    op.close()


# ---- the window aggregates on the same crowded keys ---------------------------------------------------------------
WCASES = [(kind, mode, n) for kind in ("tumbling", "sliding") for mode in ("two_pass", "one_pass") for n in (1300, 3000)]


@pytest.mark.parametrize("kind,mode,n", WCASES, ids=[f"{k}-{m}-{n}" for k, m, n in WCASES])
def test_window_crowded_bucket(kind, mode, n):
    import arroyo_b200 as ab
    from arroyo_b200 import ffi, operators as native
    from tests import test_gpu_window_time as W
    sec = 1_000_000_000
    rng = np.random.default_rng(n + len(kind) + len(mode))
    keys = crowded_keys(n)
    events, t = [], W.ORIGIN
    for i in range(6):
        ks = rng.permutation(np.concatenate([keys, rng.choice(keys, n // 2)])) if i in (0, 3) else rng.choice(keys, 400)
        m = len(ks)
        events.append(("batch", O.Batch({"key": ks.astype(np.int64), "a": rng.integers(-1000, 1000, m),
                                         TS: t + rng.integers(0, 2 * sec, m)})))
        t += sec
        if i % 2:
            events.append(("wm", t - 2 * sec))
    events.append(("wm", W.INT64_MAX))
    cfg = O.WindowAggConfig(width=2 * sec, slide=sec if kind == "sliding" else 0, key_names=["key"],
                            aggs=W.PLANS["minmax" if kind == "tumbling" else "ints"], window_index=1)
    want, late = X.window_emissions(events, "key", cfg.aggs, cfg.width, cfg.slide or None)
    flags = ffi.FLAG_TWO_PASS_ALWAYS if mode == "two_pass" else ffi.FLAG_NO_TWO_PASS
    cls = native.TumblingAggregatingWindowFunc if kind == "tumbling" else native.SlidingAggregatingWindowFunc
    from tests.gpu_ops import from_arrow, to_arrow as batch_to_arrow
    op = cls(cfg, input_schema=batch_to_arrow(events[0][1]).schema, flags=flags)
    ctx, got = ab.OperatorContext(1), []
    for ev in events:
        if ev[0] == "batch":
            op.process_batch(batch_to_arrow(ev[1]), ctx, None)
        else:
            ctx.watermarks.set(0, ev[1])
            col = ab.Collector()
            op.handle_watermark(ev[1], ctx, col)
            got.append([r for b in col.batches for r in from_arrow(b).rows()])
    stats = op.stats()
    op.close()
    W.check_emissions(want, got, cfg, f"{kind}/{mode}/{n}")
    assert stats["rows_in"] == sum(ev[1].num_rows for ev in events if ev[0] == "batch")
    assert stats["rows_late"] == late
    assert stats["rows_deferred"] > 0, stats
    assert stats["n_keys"] == n


def test_keys_that_never_split_fail_once_and_leave_the_operator_usable():
    """1500 keys whose hashes agree in their high 32 bits share a bucket at every dictionary size: 220 of them can never
    get an id.  The flush gives up with RUNTIME after the dictionary has doubled without placing any; the next flush
    emits the keys that were placed, and rows of other keys still go through."""
    import arroyo_b200 as ab
    from arroyo_b200 import ffi, operators as native
    inv = pow(BD_MULT, -1, 1 << 64)
    folded = [(j * inv) % (1 << 64) for j in range(1, 1501)]  # bd_hash = folded key * BD_MULT = j: high half 0
    keys = np.array([(f >> 32) << 32 | ((f ^ (f >> 32)) & 0xFFFFFFFF) for f in folded], dtype=np.uint64).view(np.int64)
    assert len({int(b) for b in bd_bucket(keys, 1 << 20)}) == 1
    st = Stream(1)
    st.batch(keys=keys)
    aggs = PLANS["COUNT"]
    schema = st.schema()
    op = native.UpdatingAggregatingFunc(U.UpdatingAggConfig(["k"], aggs), input_schema=schema)
    ctx = ab.OperatorContext(1)
    op.process_batch(to_arrow(st.events[0][1], schema), ctx, None)
    with pytest.raises(ffi.ArroyoB200Error) as e:
        op.handle_tick(0, ctx, ab.Collector())
    assert e.value.status == ffi.RUNTIME
    col = ab.Collector()
    op.handle_tick(0, ctx, col)
    placed = col.batches[0].column("k").to_numpy()
    assert len(placed) == BD_CAPB and set(placed.tolist()) <= set(keys.tolist())
    assert op.stats()["n_keys"] == BD_CAPB and op.stats()["rows_deferred"] > 0
    cand = np.arange(1, 100, dtype=np.int64)
    fresh = cand[bd_bucket(cand, 64) != 0][:10]  # outside bucket 0 at every size from 64 buckets on
    other = {"k": fresh, **{c: np.ones(10, dtype=np.int64) for c in VALS},
             TS: np.full(10, T0, dtype=np.int64)}
    op.process_batch(to_arrow(other, schema), ctx, None)
    col = ab.Collector()
    op.on_close("end_of_data", ctx, col)
    assert sorted(col.batches[0].column("k").to_pylist()) == fresh.tolist()
    op.close()
