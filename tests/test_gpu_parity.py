"""GPU parity: the CUDA operators (through the C ABI) against the oracle on seeded synthetic inputs.
Bit-exact for keys, counts, window bounds, i64 SUM/MIN/MAX; 1e-6 relative for f64 AVG (north star)."""
import numpy as np
import pytest

from oracle import arroyo_oracle as O
from tests.golden_cases import multiset

pytestmark = pytest.mark.gpu

S = 1_000_000_000
T0 = 1_700_000_000 * S


@pytest.fixture(scope="module")
def G():
    from tests import gpu_ops as g
    return g


def gen_stream(rng, n_rows, n_keys, rate_per_s, disorder=50, key_dist="uniform", batch=4096, vmax=10**8):
    """Nexmark-bid shaped rows: event time advances by 1/rate, permuted inside groups of `disorder`
    events (nexmark/operator.rs:515-521); keys uniform or 75 % on a hot id."""
    idx = np.arange(n_rows, dtype=np.int64)
    if disorder > 1:
        g = (idx // disorder) * disorder
        perm = np.concatenate([rng.permutation(min(disorder, n_rows - s)) + s for s in range(0, n_rows, disorder)])
        idx = perm
        del g
    ts = T0 + (idx * (S // rate_per_s)).astype(np.int64)
    if key_dist == "uniform":
        keys = rng.integers(0, n_keys, n_rows, dtype=np.int64) * 7919 - 13
    else:
        hot = rng.random(n_rows) < 0.75
        keys = np.where(hot, 42, rng.integers(0, n_keys, n_rows, dtype=np.int64))
    vals = rng.integers(-vmax, vmax, n_rows, dtype=np.int64)
    cols = {"key": keys, "value": vals, O.TIMESTAMP: ts}
    return O.source_batches(cols, batch)


I64MIN, I64MAX = -(1 << 63), (1 << 63) - 1


def gen_multi_stream(rng, n_rows, n_keys, rate_per_s, key_dist="uniform", regime="R1", batch=4096, disorder=50):
    """Rows with the value columns a, b, c, d, in arrival order like `gen_stream` (no row is late for a 1 s
    watermark delay at these rates).

    key_dist: uniform | hot (75 % on one key) | u64 (UInt64 keys >= 2^63).
    regime R1: every value |v| < 2^31, so every AVG path is exact.
    regime R2: R1 plus INT64_MIN / INT64_MAX in every column (the MIN / MAX identities), keys whose only value in a
               column is one of them, and values near 2^62 that make SUMs wrap.
    regime R3: R1 until the middle of the stream, then values >= 2^31 in column d only (value slot 3 of a plan that
               reads a, b, c, d in that order), and from three quarters on in b as well."""
    idx = np.arange(n_rows, dtype=np.int64)
    if disorder > 1:
        idx = np.concatenate([rng.permutation(min(disorder, n_rows - s)) + s for s in range(0, n_rows, disorder)])
    ts = T0 + (idx * (S // rate_per_s)).astype(np.int64)
    if key_dist == "hot":
        keys = np.where(rng.random(n_rows) < 0.75, 42, rng.integers(0, n_keys, n_rows, dtype=np.int64))
    else:
        keys = rng.integers(0, n_keys, n_rows, dtype=np.int64) * 7919 - 13
    lim = (1 << 31) - 1
    vals = {c: rng.integers(-lim, lim + 1, n_rows, dtype=np.int64) for c in "abcd"}
    if regime == "R2":
        for c in "abcd":
            v = vals[c]
            v[rng.random(n_rows) < 0.01] = I64MIN
            v[rng.random(n_rows) < 0.01] = I64MAX
            big = rng.random(n_rows) < 0.02
            v[big] = (1 << 62) + rng.integers(0, 1 << 20, int(big.sum()), dtype=np.int64)
        # keys with a single row each: their only value of a column is an identity value
        lone = rng.choice(n_rows, 40, replace=False)
        keys[lone] = 10_000_000 + np.arange(40)
        for j, r in enumerate(lone):
            for c in "abcd":
                vals[c][r] = I64MAX if (j + "abcd".index(c)) % 2 else I64MIN
    elif regime == "R3":
        half, late = n_rows // 2, 3 * n_rows // 4
        d = vals["d"]
        d[half::97] = (1 << 40) + 12345
        d[half + 5::389] = -(1 << 61)
        vals["b"][late::151] = (1 << 35) - 7
    if key_dist == "u64":
        keys = (keys.view(np.uint64) & np.uint64(0xFFFFFFFF)) | np.uint64(1 << 63)
    cols = {"key": keys, **vals, O.TIMESTAMP: ts}
    return O.source_batches(cols, batch)


def run_both(G, make_oracle, make_gpu, batches, delay_ns=S):
    want = O.run_single_input(make_oracle(), batches, delay_ns).batches
    gop = make_gpu()
    got = G.run_single_input(gop, batches, delay_ns).batches
    return want, got, gop


def rows_of(batches, float_cols=()):
    rows = []
    for b in batches:
        for r in b.rows():
            rows.append(r)
    return rows


def assert_same(want, got, float_cols=(), ordered=True):
    """Exact multiset equality on the non-float columns; floats compared at 1e-6 relative after
    aligning rows by the exact columns."""
    def split(rows):
        ex, fl = [], []
        for r in rows:
            ex.append(tuple(sorted((k, v) for k, v in r.items() if k not in float_cols)))
            fl.append(tuple(r[c] for c in float_cols))
        return ex, fl
    we, wf = split(rows_of(want))
    ge, gf = split(rows_of(got))
    assert len(we) == len(ge)
    wo = sorted(range(len(we)), key=lambda i: we[i])
    go = sorted(range(len(ge)), key=lambda i: ge[i])
    assert [we[i] for i in wo] == [ge[i] for i in go]
    if float_cols:
        a = np.array([wf[i] for i in wo], dtype=np.float64)
        b = np.array([gf[i] for i in go], dtype=np.float64)
        np.testing.assert_allclose(b, a, rtol=1e-6, atol=0)
    # windows are emitted in ascending order (tumbling / sliding; session batches hold many windows)
    if ordered:
        starts = [int(b["window_start"][0]) for b in got if "window_start" in b.cols]
        assert starts == sorted(starts)


SUM_AVG = [O.Agg("sum", "value", "sum"), O.Agg("avg", "value", "avg"), O.Agg("count", None, "count")]


def test_tumbling_count_10k_keys(G):
    """BASELINE config 2 shape: tumbling 1 s COUNT(*) GROUP BY key, 10 K keys."""
    rng = np.random.default_rng(42)
    batches = gen_stream(rng, 200_000, 10_000, rate_per_s=40_000)
    cfg = O.WindowAggConfig(width=S, key_names=["key"], aggs=[O.Agg("count", None, "count")], window_index=1)
    want, got, _ = run_both(G, lambda: O.TumblingAggregatingWindowFunc(cfg),
                            lambda: G.TumblingAggregatingWindowFunc(cfg), batches)
    assert len(want) >= 4
    assert_same(want, got)


@pytest.mark.parametrize("flags_name", ["running", "remerge"])
@pytest.mark.parametrize("dist", ["uniform", "hot"])
def test_sliding_sum_avg(G, flags_name, dist):
    """BASELINE config 3 shape (reduced): hop(1 s, 10 s) SUM/AVG GROUP BY key."""
    from arroyo_b200 import ffi
    rng = np.random.default_rng(7)
    batches = gen_stream(rng, 300_000, 5_000, rate_per_s=20_000, key_dist=dist)
    cfg = O.WindowAggConfig(width=10 * S, slide=S, key_names=["key"], aggs=SUM_AVG, window_index=1)
    flags = ffi.FLAG_REMERGE_ONLY if flags_name == "remerge" else 0
    want, got, gop = run_both(G, lambda: O.SlidingAggregatingWindowFunc(cfg),
                              lambda: G.SlidingAggregatingWindowFunc(cfg, flags=flags), batches)
    assert len(want) >= 20
    assert_same(want, got, float_cols=("avg",))
    st = gop.stats()
    assert st["rows_in"] == 300_000 and st["kernel_launches"] > 0


def test_sliding_min_max_unkeyed_and_keyed(G):
    rng = np.random.default_rng(11)
    batches = gen_stream(rng, 50_000, 300, rate_per_s=5_000, batch=1000)
    aggs = [O.Agg("min", "value", "mn"), O.Agg("max", "value", "mx"), O.Agg("count", None, "n")]
    for keys in ([], ["key"]):
        cfg = O.WindowAggConfig(width=6 * S, slide=2 * S, key_names=keys, aggs=aggs, window_index=len(keys))
        want, got, _ = run_both(G, lambda: O.SlidingAggregatingWindowFunc(cfg),
                                lambda: G.SlidingAggregatingWindowFunc(cfg), batches)
        assert_same(want, got)


def test_late_rows_are_dropped_like_the_reference(G):
    """Stragglers several seconds behind a tight watermark: whole late bins are dropped
    (tumbling :282-291), rows late inside the watermark's own bin are kept."""
    rng = np.random.default_rng(5)
    batches = gen_stream(rng, 120_000, 1_000, rate_per_s=10_000, disorder=3_000, batch=2048)
    for i, b in enumerate(batches):
        ts = b[O.TIMESTAMP].copy()
        ts[::17] -= (i % 5) * S + 300_000_000  # 0.3 .. 4.3 s late
        b.cols[O.TIMESTAMP] = np.maximum(ts, T0)
    cfg = O.WindowAggConfig(width=S, key_names=["key"], aggs=SUM_AVG, window_index=1)
    want, got, gop = run_both(G, lambda: O.TumblingAggregatingWindowFunc(cfg),
                              lambda: G.TumblingAggregatingWindowFunc(cfg), batches, delay_ns=0)
    assert_same(want, got, float_cols=("avg",))
    n_in = sum(b.num_rows for b in batches)
    n_counted = sum(int(b["count"].sum()) for b in got)
    assert gop.stats()["rows_late"] == n_in - n_counted > 0


def test_edge_cases_empty_ragged_offsets_sentinel_wraparound(G):
    """Empty batches, 1-row batches, odd sizes (vector tail path), sliced batches (non-zero Arrow
    offset), the key equal to the dictionary's empty sentinel, i64 SUM wrap-around."""
    import pyarrow as pa
    rng = np.random.default_rng(1)
    I64MIN, I64MAX = -(1 << 63), (1 << 63) - 1
    n = 10_007
    keys = rng.integers(0, 50, n, dtype=np.int64)
    keys[::97] = I64MIN
    keys[5::89] = I64MAX
    vals = rng.integers(-10, 10, n, dtype=np.int64)
    vals[:40] = I64MAX  # forces wrapping sums
    ts = T0 + np.sort(rng.integers(0, 5 * S, n)).astype(np.int64)
    cols = {"key": keys, "value": vals, O.TIMESTAMP: ts}
    sizes = [0, 1, 1, 2, 3, 1023, 1024, 1025, 0, 4097, 1, 2048]
    batches, s = [], 0
    for z in sizes:
        batches.append(O.Batch({k: v[s:s + z] for k, v in cols.items()}))
        s += z
    batches.append(O.Batch({k: v[s:] for k, v in cols.items()}))
    batches = [b for b in batches]
    cfg = O.WindowAggConfig(width=S, key_names=["key"], aggs=[O.Agg("sum", "value", "sum"), O.Agg("count", None, "n")],
                            window_index=0)
    # oracle: empty batches are legal no-ops
    oop = O.TumblingAggregatingWindowFunc(cfg)
    want = O.run_single_input(oop, [b for b in batches if b.num_rows], S).batches
    gop = G.TumblingAggregatingWindowFunc(cfg)
    # feed the GPU operator sliced views of one big batch: every slice has a non-zero offset
    big = G.to_arrow(O.Batch(cols))
    ctx, out = O.OperatorContext(1), O.Collector()
    gen = O.WatermarkGenerator(S)
    s = 0
    from tests.gpu_ops import _CollectAdapter
    for b in batches:
        z = b.num_rows
        gop.op.process_batch(big.slice(s, z), ctx, _CollectAdapter(out))
        s += z
        if z:
            wm = gen.process_batch(b[O.TIMESTAMP])
            if wm is not None:
                ctx.watermarks.set(0, wm)
                gop.handle_watermark(wm, ctx, out)
    ctx.watermarks.set(0, O.FINAL_WATERMARK)
    gop.handle_watermark(O.FINAL_WATERMARK, ctx, out)
    assert_same(want, out.batches)
    assert any((b["key"] == I64MIN).any() for b in out.batches)


def test_dictionary_growth_and_far_future_rows(G):
    """expected_keys far too small (forces id-space growth + rehash) and rows far ahead of the pane ring
    (forces the deferred path and ring growth)."""
    rng = np.random.default_rng(9)
    batches = gen_stream(rng, 150_000, 60_000, rate_per_s=50_000, batch=8192)
    # 100 rows 500 panes in the future, delivered early inside an ordinary batch (so the batch's min
    # timestamp, hence the watermark, stays current)
    b3 = batches[3]
    batches[3] = O.Batch({"key": np.concatenate([b3["key"], np.arange(100, dtype=np.int64)]),
                          "value": np.concatenate([b3["value"], np.ones(100, dtype=np.int64)]),
                          O.TIMESTAMP: np.concatenate([b3[O.TIMESTAMP], np.full(100, T0 + 500 * S, dtype=np.int64)])})
    cfg = O.WindowAggConfig(width=4 * S, slide=S, key_names=["key"], aggs=SUM_AVG, window_index=1)
    want, got, gop = run_both(G, lambda: O.SlidingAggregatingWindowFunc(cfg),
                              lambda: G.SlidingAggregatingWindowFunc(cfg, expected_keys=256), batches)
    assert_same(want, got, float_cols=("avg",))
    st = gop.stats()
    assert st["rows_deferred"] > 0 and st["n_keys"] >= 50_000


@pytest.mark.parametrize("direct", [True, False])
def test_dense_key_range_is_direct_mapped_and_outsiders_still_hash(G, direct):
    """Nexmark-shaped dense ids (1000 + n) next to keys far outside that range -- just below, just above, far away,
    the dictionary's empty sentinel.  (Round 1 mapped the dense range straight onto ids; since the bucketed
    dictionary every key is hashed, and FLAG_NO_DIRECT is accepted and ignored.)"""
    from arroyo_b200 import ffi
    rng = np.random.default_rng(77)
    batches = gen_stream(rng, 120_000, 10, rate_per_s=20_000, batch=4096)
    out = []
    outsiders = np.array([999, 2024, 2100, -5, 10**15, -2**63, 2**63 - 1], dtype=np.int64)
    for i, b in enumerate(batches):
        n = b.num_rows
        key = 1000 + rng.integers(0, 1000, n, dtype=np.int64)
        key[0], key[1] = 1000, 1999  # every batch spans the whole dense range
        if i >= 2:
            key[:: 11] = outsiders[rng.integers(0, len(outsiders), len(key[:: 11]))]
            key[1:: 97] = 2023  # inside the rounded-up direct range, never seen in the first rows
        out.append(O.Batch({"key": key, "value": b["value"], O.TIMESTAMP: b[O.TIMESTAMP]}))
    flags = 0 if direct else ffi.FLAG_NO_DIRECT
    for cfg, mk_o, mk_g, fc in (
            (O.WindowAggConfig(width=4 * S, slide=S, key_names=["key"], aggs=SUM_AVG, window_index=1),
             O.SlidingAggregatingWindowFunc, G.SlidingAggregatingWindowFunc, ("avg",)),
            (O.WindowAggConfig(width=2 * S, key_names=["key"], window_index=1,
                               aggs=[O.Agg("min", "value", "mn"), O.Agg("max", "value", "mx"), O.Agg("count", None, "n")]),
             O.TumblingAggregatingWindowFunc, G.TumblingAggregatingWindowFunc, ())):
        want, got, gop = run_both(G, lambda: mk_o(cfg), lambda: mk_g(cfg, flags=flags), out)
        assert_same(want, got, float_cols=fc)
        n_ids = gop.stats()["n_keys"]
        # 1000 dense keys + 2023 + 7 outsiders, one of which is the empty sentinel (it owns id 0, outside the dictionary)
        assert n_ids == 1007, n_ids


def test_unsupported_inputs_fail_loudly(G):
    import pyarrow as pa
    from arroyo_b200 import ffi, operators as native
    import arroyo_b200 as ab
    cfg = ab.WindowAggConfig(width=S, key_names=["key"], aggs=[ab.Agg("sum", "value", "sum")])
    op = native.TumblingAggregatingWindowFunc(cfg)
    ts = pa.array(np.array([T0, T0 + 1], dtype=np.int64)).cast(pa.timestamp("ns"))
    ctx, col = ab.OperatorContext(1), ab.Collector()
    with pytest.raises(ffi.UnsupportedPlan):  # NULL value
        op.process_batch(pa.RecordBatch.from_arrays([pa.array([1, 2]), pa.array([1, None], type=pa.int64()), ts],
                                                    names=["key", "value", "_timestamp"]), ctx, col)
    with pytest.raises(ffi.UnsupportedPlan):  # string key
        op.process_batch(pa.RecordBatch.from_arrays([pa.array(["a", "b"]), pa.array([1, 2]), ts],
                                                    names=["key", "value", "_timestamp"]), ctx, col)
    with pytest.raises(ffi.UnsupportedPlan):  # instant window
        native.TumblingAggregatingWindowFunc(ab.WindowAggConfig(width=0, aggs=[ab.Agg("count", None, "n")]),
                                             input_schema=pa.schema([("_timestamp", pa.timestamp("ns"))]))


def test_checkpoint_restore_round_trip(G):
    """handle_checkpoint -> partial-state batches (partial_schema) -> on_start of a fresh operator
    continues to the same final output as an uninterrupted oracle run (sliding :693-737, :556-595)."""
    import arroyo_b200 as ab
    from arroyo_b200 import operators as native
    from tests.gpu_ops import from_arrow, to_arrow
    rng = np.random.default_rng(21)
    batches = gen_stream(rng, 80_000, 2_000, rate_per_s=10_000, batch=4000)
    cfg = O.WindowAggConfig(width=4 * S, slide=S, key_names=["key"], aggs=SUM_AVG, window_index=1)
    want = O.run_single_input(O.SlidingAggregatingWindowFunc(cfg), batches, S).batches

    schema = to_arrow(batches[0]).schema
    ctx = ab.OperatorContext(1)
    out = ab.Collector()
    gen = ab.WatermarkGenerator(S)
    op = native.SlidingAggregatingWindowFunc(cfg, input_schema=schema)
    half = len(batches) // 2
    for i, b in enumerate(batches):
        if i == half:
            # checkpoint twice (the second must only carry rows since the first), then restart
            op.handle_checkpoint(None, ctx, out)
            op.process_batch(to_arrow(b), ctx, out)
            op.handle_checkpoint(None, ctx, out)
            op.close()
            op = native.SlidingAggregatingWindowFunc(cfg, input_schema=schema)
            op.on_start(ctx)
        else:
            op.process_batch(to_arrow(b), ctx, out)
        wm = gen.on_batch(int(b[O.TIMESTAMP].min()), int(b[O.TIMESTAMP].max()))
        if wm is not None:
            ctx.watermarks.set(0, wm)
            op.handle_watermark(wm, ctx, out)
    ctx.watermarks.set(0, ab.FINAL_WATERMARK)
    op.handle_watermark(ab.FINAL_WATERMARK, ctx, out)
    got = [from_arrow(b) for b in out.batches]
    assert_same(want, got, float_cols=("avg",))


@pytest.mark.parametrize("split", [False, True])
def test_device_resident_batches_and_device_output(G, split):
    """process_device_batch / handle_watermark_device (the chaining + benchmark path) give the same
    windows as the host path -- with the blocking call, and with the begin / poll pair (row counts read one
    emission late, the next batches handed over and submitted in between; the final watermark emits several
    windows in one emission)."""
    import torch
    import arroyo_b200 as ab
    from arroyo_b200 import operators as native
    rng = np.random.default_rng(3)
    batches = gen_stream(rng, 100_000, 3_000, rate_per_s=10_000, batch=65_536)
    cfg = O.WindowAggConfig(width=3 * S, slide=S, key_names=["key"], aggs=SUM_AVG, window_index=1)
    want = O.run_single_input(O.SlidingAggregatingWindowFunc(cfg), batches, S).batches
    import pyarrow as pa
    schema = pa.schema([("key", pa.int64()), ("value", pa.int64()), ("_timestamp", pa.timestamp("ns"))])
    op = native.SlidingAggregatingWindowFunc(cfg, input_schema=schema)
    gen = ab.WatermarkGenerator(S)
    keep = []
    got = []

    class _Ptr:
        def __init__(self, ptr, n, typestr):
            self.__cuda_array_interface__ = {"shape": (n,), "typestr": typestr, "data": (ptr, False), "version": 2}

    def collect(wins):
        names = ["key", "window_start", "window_end", "sum", "avg", "count", O.TIMESTAMP]
        for n, cols in wins:
            host = {}
            for name, ptr in zip(names, cols):
                t = torch.as_tensor(_Ptr(ptr, n, "<f8" if name == "avg" else "<i8"), device="cuda")
                host[name] = t.cpu().numpy().copy()
            got.append(O.Batch(host))

    for b in batches:
        dev = [torch.from_numpy(np.ascontiguousarray(b[c])).cuda() for c in ("key", "value", O.TIMESTAMP)]
        keep.append(dev)
        op.process_device_batch([t.data_ptr() for t in dev], b.num_rows)
        wm = gen.on_batch(int(b[O.TIMESTAMP].min()), int(b[O.TIMESTAMP].max()))
        if wm is not None:
            if split:
                op.submit()
                collect(op.handle_watermark_device_poll())  # the previous emission (nothing the first time)
                op.handle_watermark_device_begin(wm)
            else:
                collect(op.handle_watermark_device(wm))
    if split:
        collect(op.handle_watermark_device_poll())
        op.handle_watermark_device_begin(ab.FINAL_WATERMARK)
        st = op.stats()  # settles the outstanding emission without consuming it
        collect(op.handle_watermark_device_poll())
        assert collect(op.handle_watermark_device_poll()) is None and st["rows_out"] >= 0
    else:
        collect(op.handle_watermark_device(ab.FINAL_WATERMARK))
    assert_same(want, got, float_cols=("avg",))
    assert op.stats()["rows_out"] == sum(b.num_rows for b in got)


@pytest.mark.parametrize("join_type", ["inner", "left", "right", "full"])
def test_instant_join_matches_oracle(G, join_type):
    """q8-shaped windowed join: persons x auctions per 30 s tumbling window, key = person id = seller,
    duplicates on both sides, unmatched rows on both sides, several instants per watermark, rows that stay
    buffered across watermarks."""
    rng = np.random.default_rng(17)
    W30 = 30 * S
    left_b, right_b = [], []
    for w in range(6):
        ts = T0 + (w + 1) * W30 - 1
        n_p, n_a = 400 + 37 * w, 1200 + 91 * w
        pid = rng.integers(0, 500, n_p, dtype=np.int64)
        left_b.append(O.Batch({"id": pid, "name_code": rng.integers(0, 10**6, n_p, dtype=np.int64),
                               O.TIMESTAMP: np.full(n_p, ts, dtype=np.int64)}))
        seller = rng.integers(250, 750, n_a, dtype=np.int64)
        right_b.append(O.Batch({"seller": seller, "auction": np.arange(n_a, dtype=np.int64) + 1000 * w,
                                "reserve": rng.integers(1, 10**5, n_a, dtype=np.int64),
                                O.TIMESTAMP: np.full(n_a, ts, dtype=np.int64)}))
    # one batch that mixes two instants (general path of process_side, instant_join.rs:149-171)
    mixed = O.Batch.concat([right_b[4], right_b[5]])
    right_b = right_b[:4] + [mixed]
    cfg = O.JoinConfig(left_on=["id"], right_on=["seller"], join_type=join_type)

    def drive(join):
        ctx, out = O.OperatorContext(2), O.Collector()
        for step in range(3):  # 2 windows of each side, then a watermark that releases only part of them
            for b in left_b[2 * step:2 * step + 2]:
                join.process_batch_index(0, 2, b, ctx, out)
            for b in right_b[2 * step:2 * step + 2]:
                join.process_batch_index(1, 2, b, ctx, out)
            wm = T0 + (2 * step + 1) * W30 + 5  # releases the first of the two windows just sent... and older
            for side in (0, 1):
                ctx.watermarks.set(side, wm)
            join.handle_watermark(wm, ctx, out)
        for side in (0, 1):
            ctx.watermarks.set(side, O.FINAL_WATERMARK)
        join.handle_watermark(O.FINAL_WATERMARK, ctx, out)
        rows = []
        for b in out.batches:
            rows += b.rows()
        return rows

    want = drive(O.InstantJoin(cfg))
    got = drive(G.InstantJoin(cfg))
    assert len(want) > 1000
    assert multiset(got) == multiset(want)


def test_avg_exact_sum_promotes_to_f64_on_large_values(G):
    """AVG is derived from the exact integer sum while every value is < 2^31 in magnitude; the first larger
    value parks its row, promotes the operator to f64 AVG accumulators (seeded from the integer sums) and
    re-ingests it.  Results must match the oracle across the switch, and FLAG_AVG_F64 (f64 from the start)
    must match too."""
    from arroyo_b200 import ffi
    rng = np.random.default_rng(33)
    batches = gen_stream(rng, 120_000, 700, rate_per_s=10_000, batch=5000)
    # from the middle of the stream on, sprinkle huge values (some would overflow an i64 sum quickly)
    for b in batches[len(batches) // 2:]:
        v = b["value"].copy()
        v[::211] = (1 << 40) + 12345
        v[5::499] = -(1 << 61)
        b.cols["value"] = v
    cfg = O.WindowAggConfig(width=5 * S, slide=S, key_names=["key"], aggs=SUM_AVG, window_index=1)
    want = O.run_single_input(O.SlidingAggregatingWindowFunc(cfg), batches, S).batches
    for flags in (0, ffi.FLAG_AVG_F64, ffi.FLAG_REMERGE_ONLY):
        gop = G.SlidingAggregatingWindowFunc(cfg, flags=flags)
        got = G.run_single_input(gop, batches, S).batches
        assert_same(want, got, float_cols=("avg",))
        if flags == 0:
            assert gop.stats()["rows_deferred"] > 0  # the parked rows


def test_avg_only_and_avg_with_min_max(G):
    rng = np.random.default_rng(34)
    batches = gen_stream(rng, 60_000, 300, rate_per_s=6_000, batch=3000)
    for aggs in ([O.Agg("avg", "value", "avg")],
                 [O.Agg("min", "value", "mn"), O.Agg("avg", "value", "avg"), O.Agg("max", "value", "mx")]):
        cfg = O.WindowAggConfig(width=3 * S, slide=S, key_names=["key"], aggs=aggs, window_index=1)
        want, got, _ = run_both(G, lambda: O.SlidingAggregatingWindowFunc(cfg),
                                lambda: G.SlidingAggregatingWindowFunc(cfg), batches)
        assert_same(want, got, float_cols=("avg",))


def test_zero_copy_flag_is_accepted_with_the_same_results(G):
    """FLAG_ZERO_COPY is accepted and ignored: Arrow buffers in page-locked memory are staged like any other host
    batch, and the results are the oracle's."""
    import pyarrow as pa
    import torch
    import arroyo_b200 as ab
    from arroyo_b200 import operators as native
    from tests.gpu_ops import from_arrow
    rng = np.random.default_rng(8)
    batches = gen_stream(rng, 150_000, 4_000, rate_per_s=20_000, batch=10_000)
    cfg = O.WindowAggConfig(width=3 * S, slide=S, key_names=["key"], aggs=SUM_AVG, window_index=1)
    want = O.run_single_input(O.SlidingAggregatingWindowFunc(cfg), batches, S).batches
    keep = []

    def pinned_batch(b):
        arrs = []
        for name in ("key", "value", O.TIMESTAMP):
            h = torch.empty(b.num_rows, dtype=torch.int64, pin_memory=True)
            h.numpy()[:] = b[name]
            keep.append(h)
            typ = pa.timestamp("ns") if name == O.TIMESTAMP else pa.int64()
            arrs.append(pa.Array.from_buffers(typ, b.num_rows, [None, pa.py_buffer(h.numpy())]))
        return pa.RecordBatch.from_arrays(arrs, names=["key", "value", O.TIMESTAMP])

    from arroyo_b200 import ffi
    op = native.SlidingAggregatingWindowFunc(cfg, flags=ffi.FLAG_ZERO_COPY)
    ctx, out, gen = ab.OperatorContext(1), ab.Collector(), ab.WatermarkGenerator(S)
    for b in batches:
        op.process_batch(pinned_batch(b), ctx, out)
        wm = gen.on_batch(int(b[O.TIMESTAMP].min()), int(b[O.TIMESTAMP].max()))
        if wm is not None:
            ctx.watermarks.set(0, wm)
            op.handle_watermark(wm, ctx, out)
    ctx.watermarks.set(0, ab.FINAL_WATERMARK)
    op.handle_watermark(ab.FINAL_WATERMARK, ctx, out)
    assert_same(want, [from_arrow(b) for b in out.batches], float_cols=("avg",))
    assert op.stats()["h2d_bytes"] == 150_000 * 24


def test_begin_poll_emission_matches_blocking_handle_watermark(G):
    """handle_watermark_begin / _poll (windows copied back on a second stream while the next batches arrive):
    the same batches, in the same order, as the blocking call; a second `begin` before the first emission was
    collected is refused; checkpoints and the blocking call may be mixed in."""
    import arroyo_b200 as ab
    from arroyo_b200 import ffi, operators as native
    from tests.gpu_ops import from_arrow, to_arrow
    rng = np.random.default_rng(21)
    batches = gen_stream(rng, 200_000, 6_000, rate_per_s=25_000, batch=5_000)
    cfg = O.WindowAggConfig(width=3 * S, slide=S, key_names=["key"], aggs=SUM_AVG, window_index=1)
    want = O.run_single_input(O.SlidingAggregatingWindowFunc(cfg), batches, S).batches
    op = native.SlidingAggregatingWindowFunc(cfg)
    ctx, out, gen = ab.OperatorContext(1), ab.Collector(), ab.WatermarkGenerator(S)
    outstanding, polls, refused = False, 0, 0
    for i, b in enumerate(batches):
        op.process_batch(to_arrow(b), ctx, out)
        if outstanding and op.handle_watermark_poll(out, block=False):
            outstanding = False
        polls += 1
        wm = gen.on_batch(int(b[O.TIMESTAMP].min()), int(b[O.TIMESTAMP].max()))
        if wm is None:
            continue
        ctx.watermarks.set(0, wm)
        if outstanding and refused == 0:
            with pytest.raises(ffi.ArroyoB200Error):
                op.handle_watermark_begin(wm, ctx)
            refused += 1
        if outstanding:
            assert op.handle_watermark_poll(out, block=True)
            outstanding = False
        if i % 7 == 3:
            op.handle_watermark(wm, ctx, out)  # the blocking form in between
        else:
            outstanding = op.handle_watermark_begin(wm, ctx)
    if outstanding:
        assert op.handle_watermark_poll(out, block=True)
    assert op.handle_watermark_poll(out, block=False)  # nothing outstanding: ready, empty
    ctx.watermarks.set(0, ab.FINAL_WATERMARK)
    assert op.handle_watermark_begin(ab.FINAL_WATERMARK, ctx)
    assert op.handle_watermark_poll(out, block=True)
    got = [from_arrow(b) for b in out.batches]
    assert_same(want, got, float_cols=("avg",))
    assert [int(b["window_start"][0]) for b in got] == [int(b["window_start"][0]) for b in want]


@pytest.mark.parametrize("async_emit", [True, False])
def test_run_batches_loop_matches_per_batch_calls(G, async_emit):
    """arroyo_b200_op_run_batches (the subtask run loop inside the library) over runs of queued batches with the
    watermark that follows each: the same windows, in the same order, as one call per batch."""
    import ctypes as C
    import arroyo_b200 as ab
    from arroyo_b200 import ffi, operators as native
    from tests.gpu_ops import from_arrow, to_arrow
    rng = np.random.default_rng(33)
    batches = gen_stream(rng, 150_000, 2_000, rate_per_s=15_000, batch=3_000)
    cfg = O.WindowAggConfig(width=4 * S, slide=S, key_names=["key"], aggs=SUM_AVG, window_index=1)
    want = O.run_single_input(O.SlidingAggregatingWindowFunc(cfg), batches, S).batches
    gen = ab.WatermarkGenerator(S)
    wms = [gen.on_batch(int(b[O.TIMESTAMP].min()), int(b[O.TIMESTAMP].max())) for b in batches]
    op = native.SlidingAggregatingWindowFunc(cfg)
    out = ab.Collector()
    run = 13  # batches per call: emissions fall in the middle and at the end of runs
    for s in range(0, len(batches), run):
        chunk = batches[s:s + run]
        ex = native.ExportedBatches([to_arrow(b) for b in chunk])
        w = (C.c_int64 * len(chunk))(*[ffi.NO_WATERMARK if x is None else x for x in wms[s:s + run]])
        op.run_batches(ex, w, out, async_emit=async_emit)
        assert not any(ex.arrays[i].release for i in range(ex.n))  # every batch was taken
    ctx = ab.OperatorContext(1)
    ctx.watermarks.set(0, ab.FINAL_WATERMARK)
    op.handle_watermark_poll(out, block=True)
    op.handle_watermark(ab.FINAL_WATERMARK, ctx, out)
    got = [from_arrow(b) for b in out.batches]
    assert_same(want, got, float_cols=("avg",))
    assert [int(b["window_start"][0]) for b in got] == [int(b["window_start"][0]) for b in want]


def test_partial_then_final_equals_direct(G):
    """partial -> (shuffle) -> final: a per-pane tumbling stage emits (key, sum, count) partial rows; a
    sliding operator declared with `partial_count_col` merges them.  The windows must equal the direct
    sliding aggregate of the raw rows (the plan shape the N>1 benchmark uses)."""
    import arroyo_b200 as ab
    rng = np.random.default_rng(77)
    batches = gen_stream(rng, 160_000, 3_000, rate_per_s=16_000, batch=8000, key_dist="hot")
    direct = O.WindowAggConfig(width=4 * S, slide=S, key_names=["key"], aggs=SUM_AVG, window_index=1)
    want = O.run_single_input(O.SlidingAggregatingWindowFunc(direct), batches, S).batches

    local = G.TumblingAggregatingWindowFunc(
        ab.WindowAggConfig(width=S, key_names=["key"], aggs=[ab.Agg("sum", "value", "psum"), ab.Agg("count", None, "pcount")],
                           final_projection=False))
    final = G.SlidingAggregatingWindowFunc(
        ab.WindowAggConfig(width=4 * S, slide=S, key_names=["key"],
                           aggs=[ab.Agg("sum", "psum", "sum"), ab.Agg("avg", "psum", "avg"), ab.Agg("count", None, "count")],
                           window_index=1, partial_count_col="pcount"))
    ctx = O.OperatorContext(1)
    out = O.Collector()
    gen = O.WatermarkGenerator(S)

    def forward(wm):
        mid = O.Collector()
        local.handle_watermark(wm, ctx, mid)
        for b in mid.batches:
            final.process_batch(b, ctx, out)
        final.handle_watermark(wm, ctx, out)

    for b in batches:
        local.process_batch(b, ctx, out)
        wm = gen.process_batch(b[O.TIMESTAMP])
        if wm is not None:
            ctx.watermarks.set(0, wm)
            forward(wm)
    ctx.watermarks.set(0, O.FINAL_WATERMARK)
    forward(O.FINAL_WATERMARK)
    assert_same(want, out.batches, float_cols=("avg",))


def test_watermark_generator_device_reductions(G):
    """K7: the WatermarkGenerator's per-batch min / max on the device equals the oracle's generator."""
    import torch
    import arroyo_b200 as ab
    rng = np.random.default_rng(2)
    batches = gen_stream(rng, 50_000, 10, rate_per_s=5_000, disorder=2_000, batch=777)
    og, gg = O.WatermarkGenerator(S), ab.WatermarkGenerator(S)
    for b in batches:
        t = torch.from_numpy(np.ascontiguousarray(b[O.TIMESTAMP])).cuda()
        assert gg.process_device_batch(t.data_ptr(), b.num_rows) == og.process_batch(b[O.TIMESTAMP])


@pytest.mark.parametrize("n_dest", [1, 2, 3, 8])
def test_device_partitioner_matches_repartition(G, n_dest):
    """K6: hash -> dest = (h / (u64::MAX / n)) % n -> per-destination segments, against the oracle's
    restatement of ArrowCollector::repartition (context.rs:506-541): same rows in every segment."""
    import torch
    from arroyo_b200.multi_gpu import DevicePartitioner
    rng = np.random.default_rng(n_dest)
    # the partitioner works on the stream that produces its inputs (stream-ordering contract, arroyo_b200.h)
    torch.cuda.set_stream(torch.cuda.Stream())
    for n in (0, 1, 2047, 2048, 100_003):
        key = rng.integers(-2**63, 2**63 - 1, n, dtype=np.int64)
        val = rng.integers(0, 10**9, n, dtype=np.int64)
        ts = T0 + np.arange(n, dtype=np.int64)
        want = {d: b for d, b in O.repartition(O.Batch({"key": key, "value": val, O.TIMESTAMP: ts}), ["key"], n_dest)}
        part = DevicePartitioner(torch, n_dest, 3, 0, max(n, 1), 0, torch.cuda.current_stream().cuda_stream)
        cols = [torch.from_numpy(x).cuda() for x in (key, val, ts)]
        out, counts = part(cols, n)
        torch.cuda.synchronize()
        counts = counts.cpu().numpy()
        assert counts.sum() == n
        off = 0
        for d in range(n_dest):
            c = int(counts[d])
            got = sorted(zip(*(o[off:off + c].cpu().numpy().tolist() for o in out)))
            exp = sorted(zip(want[d]["key"].tolist(), want[d]["value"].tolist(), want[d][O.TIMESTAMP].tolist())) if d in want else []
            assert got == exp
            off += c
        # packed layout: destination d's block = its three columns back to back
        packed, counts2 = part.pack([c.data_ptr() for c in cols], n)
        torch.cuda.synchronize()
        assert counts2.cpu().numpy().tolist() == counts.tolist()
        flat = packed.cpu().numpy()
        off = 0
        for d in range(n_dest):
            c = int(counts[d])
            blk = flat[3 * off:3 * (off + c)].reshape(3, c)
            got = sorted(zip(*(blk[j].tolist() for j in range(3))))
            exp = sorted(zip(want[d]["key"].tolist(), want[d]["value"].tolist(), want[d][O.TIMESTAMP].tolist())) if d in want else []
            assert got == exp
            off += c
        part.close()


def session_stream(rng, n_keys, n_bursts, gap, batch, jitter=0):
    """Per key: bursts of 1..6 events less than `gap` apart, bursts more than `gap` apart; events of all keys
    are merged in (roughly) time order and cut into batches.  Some gaps are exactly `gap` (the strict `<`)."""
    rows = []
    for k in range(n_keys):
        t = T0 + int(rng.integers(0, 3 * gap))
        for _ in range(n_bursts):
            for _ in range(int(rng.integers(1, 7))):
                rows.append((t, k * 31 + 5, int(rng.integers(-1000, 1000))))
                t += int(rng.integers(1, gap)) if rng.random() > 0.05 else gap
            t += gap + int(rng.integers(1, 4 * gap))
    rows.sort(key=lambda r: r[0] + (int(rng.integers(-jitter, jitter + 1)) if jitter else 0))
    ts = np.array([r[0] for r in rows], dtype=np.int64)
    key = np.array([r[1] for r in rows], dtype=np.int64)
    val = np.array([r[2] for r in rows], dtype=np.int64)
    return O.source_batches({"key": key, "value": val, O.TIMESTAMP: ts}, batch)


SESSION_AGGS = [O.Agg("count", None, "rows"), O.Agg("sum", "value", "sum"), O.Agg("min", "value", "mn"),
                O.Agg("max", "value", "mx"), O.Agg("avg", "value", "avg")]


@pytest.mark.parametrize("case", ["in_order", "small_batches", "multi_row_runs", "disorder", "no_watermark_until_end"])
def test_session_windows_match_oracle(G, case):
    """Per-key session state machines against the oracle's statement-by-statement restatement of the reference
    (including the rows its scan assigns to the 'wrong' session when one batch holds a key's session boundary)."""
    rng = np.random.default_rng({"in_order": 1, "small_batches": 2, "multi_row_runs": 3, "disorder": 4,
                                 "no_watermark_until_end": 5}[case])
    gap = 5 * S
    kw = dict(n_keys=300, n_bursts=6, gap=gap, batch=500)
    delay = S
    if case == "small_batches":
        kw.update(batch=37)
    if case == "multi_row_runs":  # few keys, big batches: one batch spans several bursts of a key
        kw.update(n_keys=12, n_bursts=25, batch=400)
    if case == "disorder":
        kw.update(jitter=2 * S)
        delay = 3 * S
    batches = session_stream(rng, **kw)
    cfg = O.SessionConfig(gap=gap, key_names=["key"], aggs=SESSION_AGGS, window_index=0)
    if case == "no_watermark_until_end":
        def run(op, runner_ctx):
            ctx, out = runner_ctx(1), O.Collector()
            for b in batches:
                op.process_batch(b, ctx, out)
            ctx.watermarks.set(0, O.FINAL_WATERMARK)
            op.handle_watermark(O.FINAL_WATERMARK, ctx, out)
            return out.batches
        want = run(O.SessionAggregatingWindowFunc(cfg), O.OperatorContext)
        got = run(G.SessionAggregatingWindowFunc(cfg), O.OperatorContext)
    else:
        want = O.run_single_input(O.SessionAggregatingWindowFunc(cfg), batches, delay).batches
        got = G.run_single_input(G.SessionAggregatingWindowFunc(cfg), batches, delay).batches
    assert sum(b.num_rows for b in want) > 250
    assert_same(want, got, float_cols=("avg",), ordered=False)


def test_session_unkeyed_and_device_batches(G):
    import torch
    import arroyo_b200 as ab
    from arroyo_b200 import operators as native
    rng = np.random.default_rng(4)
    batches = session_stream(rng, n_keys=1, n_bursts=40, gap=2 * S, batch=64)
    ub = [O.Batch({"value": b["value"], O.TIMESTAMP: b[O.TIMESTAMP]}) for b in batches]
    cfg = O.SessionConfig(gap=2 * S, key_names=[], aggs=[O.Agg("count", None, "rows"), O.Agg("sum", "value", "sum")],
                          window_index=0)
    want = O.run_single_input(O.SessionAggregatingWindowFunc(cfg), ub, S).batches
    got = G.run_single_input(G.SessionAggregatingWindowFunc(cfg), ub, S).batches
    assert_same(want, got, ordered=False)


def test_session_pool_compaction(G, monkeypatch):
    """Long stream with a tiny compaction threshold: the run / row pools are rebuilt from the per-key lists many
    times without changing any result."""
    monkeypatch.setenv("ARROYO_B200_SESSION_COMPACT_MIN", "64")
    rng = np.random.default_rng(12)
    batches = session_stream(rng, n_keys=200, n_bursts=12, gap=3 * S, batch=300, jitter=S)
    cfg = O.SessionConfig(gap=3 * S, key_names=["key"], aggs=SESSION_AGGS, window_index=1)
    want = O.run_single_input(O.SessionAggregatingWindowFunc(cfg), batches, 2 * S).batches
    got = G.run_single_input(G.SessionAggregatingWindowFunc(cfg), batches, 2 * S).batches
    assert_same(want, got, float_cols=("avg",), ordered=False)
