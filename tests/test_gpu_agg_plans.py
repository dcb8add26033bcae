"""Multi-column and wide aggregate plans on the CUDA window, session and updating aggregates.

Every other parity test aggregates one value column.  These plans read up to four value columns (the generic
`ingest_kernel<NV>` paths), need up to nine accumulators, share accumulators between aggregates and list the same
output twice.  Window and updating results are checked against the oracle and against the exact group-by in
tests/exact_reference.py (integers exact, AVG bit-exact while a group's sum of |x| stays below 2^53, else within
the f64 summation bound); sessions against the oracle, whose scan reproduces the reference's boundary handling."""
import numpy as np
import pyarrow as pa
import pytest

from oracle import arroyo_oracle as O
from oracle import updating_oracle as U
from tests import exact_reference as X
from tests.golden_cases import multiset
from tests.test_gpu_parity import S, T0, assert_same, gen_multi_stream

pytestmark = pytest.mark.gpu

A = O.Agg
PLANS = {
    "P1": [A("sum", "a", "sa"), A("min", "b", "mnb")],
    "P2": [A("avg", "a", "ava"), A("max", "b", "mxb"), A("sum", "c", "sc"), A("count", None, "n")],
    "P3": [A("min", "a", "mna"), A("max", "b", "mxb"), A("sum", "c", "sc"), A("avg", "d", "avd"), A("count", None, "n")],
    "P4": [A("avg", "a", "ava"), A("min", "a", "mna"), A("max", "a", "mxa"), A("sum", "b", "sb"), A("min", "b", "mnb"),
           A("max", "b", "mxb"), A("sum", "c", "sc"), A("avg", "d", "avd")],
    "P5": [A("sum", "a", "sa"), A("avg", "a", "ava"), A("min", "a", "mna"), A("min", "a", "mna2"), A("count", None, "n"),
           A("count", None, "n2")],
    "P6a": [A("min", "a", "mna")],
    "P6b": [A("max", "a", "mxa"), A("sum", "a", "sa"), A("avg", "a", "ava")],
    "P7": [A("avg", "a", "ava"), A("avg", "b", "avb"), A("min", "a", "mna"), A("max", "a", "mxa"), A("min", "b", "mnb"),
           A("max", "b", "mxb"), A("sum", "c", "sc"), A("count", None, "n")],
    "P8": [A("sum", "a", "sa"), A("avg", "b", "avb"), A("sum", "c", "sc"), A("count", None, "n")],
}
SIZES = [1, 1023, 1024, 4097]  # host batch sizes of the "sizes" entry point, cut from one batch (non-zero offsets)


def avg_names(aggs):
    return tuple(a.name for a in aggs if a.kind == "avg")


@pytest.fixture(scope="module")
def G():
    from tests import gpu_ops as g
    return g


def stream(keys, regime, n_rows=24_000, batch=3_000, seed=0):
    rng = np.random.default_rng(1000 + seed)
    return gen_multi_stream(rng, n_rows, 1_500, rate_per_s=4_000, key_dist="uniform" if keys == "none" else keys,
                            regime=regime, batch=batch)


def drive_sized(G, op, batches, delay_ns=S):
    """Like gpu_ops.run_single_input, but the rows arrive as slices of one Arrow batch cut to SIZES in turn."""
    from tests.gpu_ops import _CollectAdapter
    allb = O.Batch.concat(batches)
    big = G.to_arrow(allb)
    ctx, out, gen = O.OperatorContext(1), O.Collector(), O.WatermarkGenerator(delay_ns)
    s, i = 0, 0
    while s < allb.num_rows:
        z = min(SIZES[i % len(SIZES)], allb.num_rows - s)
        op.op.process_batch(big.slice(s, z), ctx, _CollectAdapter(out))
        wm = gen.process_batch(allb[O.TIMESTAMP][s:s + z])
        if wm is not None:
            ctx.watermarks.set(0, wm)
            op.handle_watermark(wm, ctx, out)
        s, i = s + z, i + 1
    ctx.watermarks.set(0, O.FINAL_WATERMARK)
    op.handle_watermark(O.FINAL_WATERMARK, ctx, out)
    return out.batches


def without(batches, names):
    return [O.Batch({c: v for c, v in b.cols.items() if c not in names}) for b in batches]


def check_windows(want, got, batches, cfg):
    """Oracle parity on every integer column and on the order of the windows; the operator's and the oracle's
    rows both equal to the exact reference, AVG by its rule.  (Two f64 sums of the same inputs in different orders
    need not agree to any relative tolerance once INT64_MIN and INT64_MAX cancel in them: only the bound holds.)"""
    assert_same(without(want, avg_names(cfg.aggs)), without(got, avg_names(cfg.aggs)))
    key = cfg.key_names[0] if cfg.key_names else None
    exact = X.window_rows(batches, key, cfg.aggs, cfg.width, cfg.slide or None)
    for name, out in (("gpu", got), ("oracle", want)):
        rows = [r for b in out for r in b.rows()]
        errs = X.mismatches(exact, rows, lambda r: (int(r["window_start"]), int(r[key]) if key else None))
        assert not errs, (name, errs[:10])
    if key:
        want_type = batches[0][key].dtype
        assert all(b[key].dtype == want_type for b in got if b.num_rows)


# (window kind, flags, plan, keys, regime, entry point): a cross section of the axes, not their product
WINDOW_CASES = [
    ("tumbling", "default", "P1", "uniform", "R1", "batches"),
    ("tumbling", "default", "P2", "hot", "R2", "batches"),
    ("tumbling", "default", "P3", "u64", "R3", "batches"),
    ("tumbling", "default", "P4", "uniform", "R2", "sizes"),
    ("tumbling", "default", "P5", "none", "R1", "sizes"),
    ("tumbling", "default", "P6a", "hot", "R1", "batches"),
    ("tumbling", "default", "P6b", "uniform", "R2", "batches"),
    ("tumbling", "default", "P7", "uniform", "R3", "batches"),
    ("tumbling", "default", "P8", "u64", "R1", "batches"),
    ("sliding", "default", "P1", "hot", "R2", "sizes"),
    ("sliding", "default", "P2", "uniform", "R1", "batches"),
    ("sliding", "default", "P3", "uniform", "R3", "batches"),
    ("sliding", "default", "P4", "hot", "R3", "batches"),
    ("sliding", "default", "P5", "u64", "R2", "batches"),
    ("sliding", "default", "P6a", "none", "R2", "batches"),
    ("sliding", "default", "P6b", "hot", "R1", "sizes"),
    ("sliding", "default", "P7", "hot", "R3", "batches"),
    ("sliding", "default", "P7", "uniform", "R1", "batches"),
    ("sliding", "default", "P8", "uniform", "R1", "batches"),
    ("sliding", "default", "P8", "hot", "R2", "batches"),
    ("sliding", "remerge", "P3", "hot", "R2", "batches"),
    ("sliding", "remerge", "P7", "u64", "R3", "batches"),
    ("sliding", "remerge", "P8", "u64", "R3", "batches"),
    ("sliding", "avg_f64", "P2", "uniform", "R3", "batches"),
    ("sliding", "avg_f64", "P4", "none", "R1", "batches"),
    ("tumbling", "avg_f64", "P5", "hot", "R2", "batches"),
    ("sliding", "no_combine", "P2", "hot", "R1", "batches"),
    ("sliding", "no_combine", "P3", "hot", "R3", "batches"),
    ("tumbling", "no_combine", "P6a", "hot", "R2", "batches"),
]


@pytest.mark.parametrize("kind,flags,plan,keys,regime,entry", WINDOW_CASES,
                         ids=["-".join(c) for c in WINDOW_CASES])
def test_window_plans(G, kind, flags, plan, keys, regime, entry):
    from arroyo_b200 import ffi
    aggs = PLANS[plan]
    key_names = [] if keys == "none" else ["key"]
    if kind == "sliding":
        cfg = O.WindowAggConfig(width=4 * S, slide=S, key_names=key_names, aggs=aggs, window_index=len(key_names))
        ocls, gcls = O.SlidingAggregatingWindowFunc, G.SlidingAggregatingWindowFunc
    else:
        cfg = O.WindowAggConfig(width=S, key_names=key_names, aggs=aggs, window_index=len(key_names))
        ocls, gcls = O.TumblingAggregatingWindowFunc, G.TumblingAggregatingWindowFunc
    fl = {"default": 0, "remerge": ffi.FLAG_REMERGE_ONLY, "avg_f64": ffi.FLAG_AVG_F64,
          "no_combine": ffi.FLAG_NO_COMBINE}[flags]
    batches = stream(keys, regime, seed=len(plan) + 7 * WINDOW_CASES.index((kind, flags, plan, keys, regime, entry)))
    want = O.run_single_input(ocls(cfg), batches, S).batches
    gop = gcls(cfg, flags=fl)
    got = drive_sized(G, gop, batches) if entry == "sizes" else G.run_single_input(gop, batches, S).batches
    st = gop.stats()
    assert st["rows_late"] == 0 and st["rows_in"] == sum(b.num_rows for b in batches)
    check_windows(want, got, batches, cfg)
    gop.close()


SESSION_CASES = [("P1", "uniform", "R1"), ("P2", "uniform", "R1"), ("P3", "hot", "R3"), ("P4", "u64", "R2"),
                 ("P5", "none", "R1"), ("P6b", "hot", "R2"), ("P7", "uniform", "R3"), ("P8", "uniform", "R2")]


@pytest.mark.parametrize("plan,keys,regime", SESSION_CASES)
def test_session_plans(G, plan, keys, regime):
    """Sessions against the oracle; AVG bit-exact while every key's inputs stay below 2^31 (R1), else within the
    f64 summation bound taken over all of the key's rows (an upper bound of any one session's)."""
    aggs = PLANS[plan]
    key_names = [] if keys == "none" else ["key"]
    rng = np.random.default_rng(500 + SESSION_CASES.index((plan, keys, regime)))
    # about one row per key and second against a 1.5 s gap: sessions of one to many rows, split at random
    n_keys, rate = (20, 20) if keys == "none" else (2_000, 2_000)
    batches = gen_multi_stream(rng, 12_000, n_keys, rate_per_s=rate, key_dist="uniform" if keys == "none" else keys,
                               regime=regime, batch=1_000, disorder=10)
    if keys == "none":  # the rows of one key, without the key column
        batches = [O.Batch({c: v[b["key"] == -13] for c, v in b.cols.items() if c != "key"}) for b in batches]
    cfg = O.SessionConfig(gap=3 * S // 2, key_names=key_names, aggs=aggs, window_index=len(key_names))
    want = O.run_single_input(O.SessionAggregatingWindowFunc(cfg), batches, S).batches
    gop = G.SessionAggregatingWindowFunc(cfg)
    got = G.run_single_input(gop, batches, S).batches
    assert sum(b.num_rows for b in want) > 100
    fc = avg_names(aggs)
    assert_same(without(want, fc), without(got, fc), ordered=False)
    # AVG: align by the exact columns, then the rule
    key = key_names[0] if key_names else None
    allb = O.Batch.concat(batches)
    kcol = allb[key] if key else np.zeros(allb.num_rows, dtype=np.int64)
    bound = {}
    for a in aggs:
        if a.kind == "avg":
            tot = {}
            for k, v in zip(kcol.tolist(), allb[a.col].tolist()):
                tot[k] = tot.get(k, 0) + abs(v)
            bound[a.name] = tot

    def index(bs):
        out = {}
        for b in bs:
            for r in b.rows():
                ex = tuple(sorted((k, int(v)) for k, v in r.items() if k not in fc))
                out.setdefault(ex, []).append(r)
        return out
    wi, gi = index(want), index(got)
    for ex, ws in wi.items():
        for w, g in zip(ws, gi[ex]):
            k = int(w[key]) if key else 0
            for c in fc:
                s = bound[c][k]
                if s < 2 ** 53:
                    assert float(g[c]) == float(w[c]), (ex, c, g[c], w[c])
                else:
                    assert abs(float(g[c]) - float(w[c])) <= 4 * X.U * s + 4 * X.U * abs(float(w[c])), (ex, c)


class _Updating:
    def __init__(self, cfg, **kw):
        import arroyo_b200 as ab
        from arroyo_b200 import operators as native
        self.ab = ab
        self.op = native.UpdatingAggregatingFunc(cfg, **kw)
        self.ctx = ab.OperatorContext(1)

    def process_batch(self, batch):
        from tests.gpu_ops import to_arrow
        self.op.process_batch(to_arrow(batch), self.ctx, None)

    def flush(self):
        from tests.gpu_ops import from_arrow
        col = self.ab.Collector()
        self.op.handle_tick(0, self.ctx, col)
        if not col.batches:
            return None
        cols = dict(from_arrow(col.batches[0]).cols)
        cols[U.IS_RETRACT] = cols.pop("_is_retract").astype(bool)
        return O.Batch(cols)


def run_updating(op, batches, flush_every):
    out = []
    for i, b in enumerate(batches):
        op.process_batch(b)
        if flush_every and (i + 1) % flush_every == 0:
            out.append(op.flush())
    out.append(op.flush())
    return out


def _exact_part(rows, fc):
    return [{k: (bool(v) if k == U.IS_RETRACT else int(v)) for k, v in r.items() if k not in fc} for r in rows]


def check_updating(cfg, batches, got, want):
    fc = avg_names(cfg.aggs)
    key = cfg.key_names[0] if cfg.key_names else None
    assert len(got) == len(want)
    for g, w in zip(got, want):  # flush by flush: the same keys retracted and appended, same integer columns
        gr = [] if g is None else g.rows()
        wr = [] if w is None else w.rows()
        assert multiset(_exact_part(gr, fc)) == multiset(_exact_part(wr, fc))
    exact = X.updating_rows(batches, key, cfg.aggs)
    for name, stream_ in (("gpu", got), ("oracle", want)):
        final = U.merge_change_stream(stream_, cfg.key_names)
        errs = X.mismatches({k: {c: v for c, v in r.items() if c != X.TIMESTAMP} for k, r in exact.items()}, final,
                            lambda r: int(r[key]) if key else None)
        assert not errs, (name, errs[:10])


@pytest.mark.parametrize("plan,keys,regime,flush_every", [
    ("P1", "uniform", "R1", 1), ("P2", "hot", "R2", 3), ("P3", "uniform", "R3", 0), ("P4", "u64", "R1", 3),
    ("P5", "none", "R2", 1), ("P6b", "uniform", "R1", 0), ("P7", "hot", "R3", 0), ("P8", "uniform", "R2", 3)])
def test_updating_plans(G, plan, keys, regime, flush_every):
    aggs = PLANS[plan]
    key_names = [] if keys == "none" else ["key"]
    batches = stream(keys, regime, n_rows=6_000, batch=500, seed=len(plan) + flush_every)
    cfg = U.UpdatingAggConfig(key_names, aggs)
    want = run_updating(U.IncrementalAggregatingFunc(cfg), batches, flush_every)
    got = run_updating(_Updating(cfg), batches, flush_every)
    check_updating(cfg, batches, got, want)


def test_updating_avg_does_not_wrap(G):
    """Four rows of 2^62 on one key: the wrapping i64 sum is 0, the AVG is 2^62 (the inputs are summed as f64)."""
    aggs = [A("avg", "a", "ava"), A("sum", "a", "sa"), A("count", None, "n")]
    cfg = U.UpdatingAggConfig(["key"], aggs)
    a = np.array([1 << 62] * 4 + [3, -4], dtype=np.int64)
    batches = [O.Batch({"key": np.array([7, 7, 7, 7, 8, 8], dtype=np.int64), "a": a,
                        O.TIMESTAMP: T0 + np.arange(6, dtype=np.int64)})]
    got = run_updating(_Updating(cfg), batches, 0)
    final = {r["key"]: r for r in U.merge_change_stream(got, ["key"])}
    assert final[7]["ava"] == float(1 << 62) and final[7]["sa"] == 0 and final[7]["n"] == 4
    assert final[8]["ava"] == -0.5
    check_updating(cfg, batches, got, run_updating(U.IncrementalAggregatingFunc(cfg), batches, 0))


def test_device_batches_four_value_columns(G):
    """P3 through process_device_batch / handle_watermark_device: the device output columns are
    [key, window_start, window_end, min(a), max(b), sum(c), avg(d) as f64, count, _timestamp]."""
    import torch
    import arroyo_b200 as ab
    from arroyo_b200 import operators as native
    aggs = PLANS["P3"]
    batches = stream("hot", "R3", n_rows=40_000, batch=8_000, seed=3)
    cfg = O.WindowAggConfig(width=3 * S, slide=S, key_names=["key"], aggs=aggs, window_index=1)
    want = O.run_single_input(O.SlidingAggregatingWindowFunc(cfg), batches, S).batches
    names = ["key", "a", "b", "c", "d", O.TIMESTAMP]
    schema = pa.schema([(n, pa.timestamp("ns") if n == O.TIMESTAMP else pa.int64()) for n in names])
    op = native.SlidingAggregatingWindowFunc(cfg, input_schema=schema)
    out_names = ["key", "window_start", "window_end"] + [a.name for a in aggs] + [O.TIMESTAMP]
    gen = ab.WatermarkGenerator(S)
    keep, got = [], []

    class _Ptr:
        def __init__(self, ptr, n, typestr):
            self.__cuda_array_interface__ = {"shape": (n,), "typestr": typestr, "data": (ptr, False), "version": 2}

    def collect(wins):
        for n, cols in wins:
            assert len(cols) == len(out_names)
            host = {}
            for name, ptr in zip(out_names, cols):
                t = torch.as_tensor(_Ptr(ptr, n, "<f8" if name == "avd" else "<i8"), device="cuda")
                host[name] = t.cpu().numpy().copy()
            got.append(O.Batch(host))

    for b in batches:
        dev = [torch.from_numpy(np.ascontiguousarray(b[c])).cuda() for c in names]
        keep.append(dev)
        op.process_device_batch([t.data_ptr() for t in dev], b.num_rows)
        wm = gen.on_batch(int(b[O.TIMESTAMP].min()), int(b[O.TIMESTAMP].max()))
        if wm is not None:
            collect(op.handle_watermark_device(wm))
    collect(op.handle_watermark_device(ab.FINAL_WATERMARK))
    check_windows(want, got, batches, cfg)
    op.close()


def _refusal_cases():
    n = 4
    ts = pa.array(T0 + np.arange(n, dtype=np.int64)).cast(pa.timestamp("ns"))
    i64 = pa.array(np.arange(n, dtype=np.int64))
    f64 = pa.array(np.linspace(-2.5, 2.5, n))
    u64 = pa.array(np.array([1, 2, 3, (1 << 63) + 5], dtype=np.uint64))
    cases = []
    for kind in ("avg", "sum", "min", "max"):
        cases.append((f"{kind}_of_f64", ["key"], [A(kind, "v", "x")], [i64, f64, ts]))
        cases.append((f"{kind}_of_u64", ["key"], [A(kind, "v", "x")], [i64, u64, ts]))
    cases.append(("f64_key", ["key"], [A("count", None, "n"), A("sum", "v", "s")], [f64, i64, ts]))
    return cases


@pytest.mark.parametrize("operator", ["tumbling", "session", "updating"])
@pytest.mark.parametrize("case", _refusal_cases(), ids=lambda c: c[0])
def test_unsupported_input_types_are_refused(G, operator, case):
    """Aggregates over Float64 or UInt64 columns and Float64 keys are outside the supported subset (Int64
    aggregate inputs; Int64, UInt64 or timestamp keys): process_batch refuses them, the plan stays on the
    stock operator."""
    import arroyo_b200 as ab
    from arroyo_b200 import ffi, operators as native
    _, key_names, aggs, arrays = case
    rb = pa.RecordBatch.from_arrays(arrays, names=["key", "v", O.TIMESTAMP])
    if operator == "tumbling":
        op = native.TumblingAggregatingWindowFunc(ab.WindowAggConfig(width=S, key_names=key_names, aggs=aggs))
    elif operator == "session":
        op = native.SessionAggregatingWindowFunc(O.SessionConfig(gap=S, key_names=key_names, aggs=aggs))
    else:
        op = native.UpdatingAggregatingFunc(U.UpdatingAggConfig(key_names, aggs))
    with pytest.raises(ffi.UnsupportedPlan):
        op.process_batch(rb, ab.OperatorContext(1), ab.Collector())
    op.close()
