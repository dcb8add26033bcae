"""The window aggregate's one-pass ingest (`ingest_kernel<NV, SIG>` in csrc/window_agg.cu) and its warp-combine
(`combine_accumulate` / `group_reduce`) against the exact group-by.

A. The combine's group key at the pane-number edges: panes numbered 2^32 - 1 modulo 2^32, their neighbours 2^32 - 2 and
   0 modulo 2^32 (the carry into bit 32) and the windows across them, at slides of 1 s, 1 ms and 2 ns.  Every warp
   holds one hot key (or, unkeyed, the single group) on neighbouring lanes next to lanes the kernel does not take on
   its fast path: late rows, keys seen for the first time, rows far ahead of the pane ring, values beyond the exact-AVG
   guard and the idle lanes of a batch's last warp.  Keyed streams hold at most 31 keys, so every dictionary id is
   below 32: the ids of bdict.cuh are BD_ID_BASE (2) + bucket * BD_CAPB + arrival index, one bucket here, and id 0 is
   the key equal to the empty sentinel (INT64_MIN).  Each case runs with the combine on and with FLAG_NO_COMBINE, watermark
   by watermark against tests/exact_reference.window_emissions, with the same rows_in and rows_late.
B. Every one-pass kernel instantiation (the nine AB_LAUNCH branches) in one large device-resident launch: 2^24 rows
   tumbling, 2^22 rows sliding with four panes per window, over 2^20 uniform keys, one key taking 75 % of the rows,
   8 keys, no key and UInt64 keys >= 2^63, with values in the regimes R1 and R2 of gen_multi_stream.
C. Rows deferred at scale: a four-column plan whose dictionary has to grow from 256 to 2^20 keys inside one launch,
   and one value >= 2^31 in the middle of a 2^24-row AVG launch (the operator promotes itself to f64 and re-ingests).

B and C compare every output row with an exact group-by computed with torch on the same device (`group_by`): the
numpy reference is too slow at these sizes.  COUNT, SUM (wrapping), MIN and MAX must be equal; AVG follows
exact_reference.check_avg, evaluated on the device where the group's sum of |x| is below 2^53 (there the exact mean
is one f64 division of exact integers) and by check_avg itself elsewhere."""
from fractions import Fraction

import numpy as np
import pytest

from oracle import arroyo_oracle as O
from tests import exact_reference as X
from tests.test_gpu_parity import S, gen_multi_stream
from tests.test_gpu_window_time import ORIGIN, SEC, Stream, _Ptr, check_emissions, device_names, reference, run_gpu

pytestmark = pytest.mark.gpu

A = O.Agg
TS = O.TIMESTAMP
I64MIN = -(1 << 63)

# ---- A. the combine key at the pane-number edges ---------------------------------------------------------------------
EDGE_PLANS = {
    "count": [A("count", None, "n")],                                   # NV = 0
    "sum": [A("sum", "a", "sa"), A("count", None, "n")],
    "minmax": [A("min", "a", "mna"), A("max", "a", "mxa")],
    "avg": [A("avg", "a", "ava"), A("count", None, "n")],              # exact AVG: the guard applies
    "gen2": [A("sum", "a", "sa"), A("min", "b", "mnb"), A("avg", "a", "ava")],
    "gen4": [A("avg", "a", "ava"), A("min", "a", "mna"), A("max", "b", "mxb"), A("sum", "c", "sc"),
             A("avg", "d", "avd"), A("count", None, "n")],
}
# (width, slide, the pane number q0 with q0 = 2^32 - 1 modulo 2^32)
EDGE_CONFIGS = {
    "tumbling_1s": (SEC, None, (1 << 32) - 1),
    "hop_1ms_4ms": (4_000_000, 1_000_000, 397 * (1 << 32) - 1),        # present-day timestamps
    "hop_2ns_8ns": (8, 2, ((ORIGIN // 2 >> 32) << 32) + (1 << 32) - 1),  # the smallest slide the operator accepts
}
HOT = 42
# 31 keys: INT64_MIN takes id 0, the other 30 ids 2..31 in arrival order
EDGE_KEYS = [HOT, I64MIN] + [1000 + 7 * j for j in range(29)]
LENGTHS = [1, 31, 33, 1000 + 7, 4096]


def _rows(st, n, o, panes, keys, big=False):
    """`n` rows at random instants of `panes` (numbers relative to the edge pane) with keys drawn from `keys`."""
    rng, s = st.rng, st.slide
    ts = o + np.asarray(panes, dtype=np.int64) * s + rng.integers(0, s, n)
    cols = {}
    if st.keys != "none":
        cols["key"] = np.asarray(keys, dtype=np.int64)
    for c in "abcd":
        cols[c] = rng.integers(-1000, 1001, n).astype(np.int64)
    if big:  # beyond the exact-AVG guard (|v| >= 2^31) in value slots 0 and 3
        at = rng.choice(n, max(1, n // 50), replace=False)
        cols["a"][at] = (1 << 31) + rng.integers(0, 1000, len(at))
        cols["d"][at[::2]] = -(1 << 40)
    cols[TS] = ts.astype(np.int64)
    return cols


def _mixed(st, n, o, main, late_below, fresh, far, big):
    """One batch around pane `main`: hot key rows on neighbouring lanes, other seen keys, rows in the neighbour
    panes, and the rows the kernel handles off its fast path (late, first sight of a key, far ahead, big values)."""
    rng = st.rng
    kind = rng.choice(6, n, p=[0.5, 0.14, 0.12, 0.08, 0.08, 0.08])
    panes = np.full(n, main, dtype=np.int64)
    panes[kind == 2] = main + rng.choice([-1, 1], int((kind == 2).sum()))
    panes[kind == 3] = late_below - 1 - rng.integers(0, 3, int((kind == 3).sum()))
    panes[kind == 4] = far
    keys = np.full(n, HOT, dtype=np.int64)
    seen = st.seen
    keys[kind == 1] = rng.choice(seen, int((kind == 1).sum()))
    keys[kind == 2] = rng.choice(seen, int((kind == 2).sum()))
    new = np.flatnonzero(kind == 5)
    for i, k in zip(new, fresh):  # the first sight of a key
        keys[i] = k
    keys[new[len(fresh):]] = HOT
    st.seen = seen + list(fresh[:len(new)])
    cols = _rows(st, n, o, panes, keys, big)
    return O.Batch(cols)


def edge_stream(seed, keyed, width, slide, q0):
    st = Stream(seed, "few" if keyed else "none", width, slide)
    s = st.slide
    o = q0 * s
    st.seen = [HOT, I64MIN] + EDGE_KEYS[2:6]
    fresh = list(EDGE_KEYS[6:])
    warm = _rows(st, 4 * len(st.seen), o, np.repeat(np.arange(-2, 2), len(st.seen)), np.tile(st.seen, 4))
    st.events.append(("batch", O.Batch(warm)))
    st.wm(o - s)  # pane q0 - 1 is the oldest on-time pane
    far = 5000
    for j, n in enumerate(LENGTHS):
        take, fresh = fresh[:3], fresh[3:]
        st.events.append(("batch", _mixed(st, n, o, 0, -1, take, far + 1000 * j, big=j == 3)))
    st.wm(o + s + 1)  # emits the windows that end at the carry; pane q0 is late from here on
    for j, n in enumerate(LENGTHS):
        take, fresh = fresh[:3], fresh[3:]
        st.events.append(("batch", _mixed(st, n, o, 2, 1, take, far + 7000 + 1000 * j, big=False)))
    st.wm(o + 3 * s)
    return st.end()


ENTRIES = ["host", "sliced", "device"]
EDGE_CASES = [(c, k, p, ENTRIES[i % 3]) for i, (c, k, p) in enumerate(
    (c, k, p) for c in EDGE_CONFIGS for k in ("none", "keyed") for p in EDGE_PLANS)]


@pytest.mark.parametrize("combine", ["combine", "no_combine"])
@pytest.mark.parametrize("config,keys,plan,entry", EDGE_CASES, ids=["-".join(c) for c in EDGE_CASES])
def test_combine_key_at_pane_number_edges(config, keys, plan, entry, combine):
    from arroyo_b200 import ffi
    width, slide, q0 = EDGE_CONFIGS[config]
    keyed = keys == "keyed"
    st = edge_stream(EDGE_CASES.index((config, keys, plan, entry)), keyed, width, slide, q0)
    assert set(st.seen) <= set(EDGE_KEYS) and len(EDGE_KEYS) == 31
    cfg = O.WindowAggConfig(width=width, slide=slide or 0, key_names=["key"] if keyed else [], aggs=EDGE_PLANS[plan],
                            window_index=1 if keyed else 0)
    kind = "tumbling" if slide is None else "running" if plan in ("count", "sum", "avg") else "remerge"
    want, late = reference(st, cfg)
    flags = ffi.FLAG_NO_COMBINE if combine == "no_combine" else 0
    got, rows_in, rows_late, n_keys = run_gpu(st, kind, cfg, entry, expected_keys=64, flags=flags)
    check_emissions(want, got, cfg, combine)
    assert rows_in == sum(ev[1].num_rows for ev in st.events if ev[0] == "batch")
    assert rows_late == late and late > 0
    # the statistic counts the keys the dictionary stores: INT64_MIN has the reserved id 0 outside them
    assert n_keys == (len(st.seen) - 1 if keyed else 0)
    # the edge pane and both of its neighbours hold rows
    starts = {k[0] for w in want for k in w}
    s = slide or width
    assert {q0 * s - s, q0 * s, q0 * s + s} <= starts


# ---- B / C. large device-resident launches against a group-by on the device -------------------------------------------
def group_by(cols, key, aggs, width, slide):
    """The exact expected output of a window aggregate over rows that are never late, on the device:
    (window_start, key or None, {aggregate name: values}, the AVG parts {name: (sum hi, sum lo, |x| hi, |x| lo)}),
    sorted by (window_start, key)."""
    import torch
    ts = cols[TS]
    s = slide or width
    bins = ts - ts % s
    starts = torch.cat([bins - k * s for k in range(width // s)])
    rep = width // s
    k = cols[key].repeat(rep) if key else torch.zeros_like(starts)
    uniq, inv = torch.unique(torch.stack([starts, k]), dim=1, return_inverse=True)
    g = uniq.shape[1]
    n = torch.zeros(g, dtype=torch.int64, device=ts.device).index_add_(0, inv, torch.ones_like(starts))
    out, parts = {}, {}
    for a in aggs:
        if a.kind == "count":
            out[a.name] = n
            continue
        v = cols[a.col].repeat(rep)
        if a.kind == "sum":
            out[a.name] = torch.zeros(g, dtype=torch.int64, device=ts.device).index_add_(0, inv, v)
        elif a.kind in ("min", "max"):
            out[a.name] = torch.zeros(g, dtype=torch.int64, device=ts.device).scatter_reduce_(
                0, inv, v, "amin" if a.kind == "min" else "amax", include_self=False)
        else:
            absv = torch.where(v < 0, -v, v)  # INT64_MIN stays INT64_MIN: its bits are 2^63
            halves = (v >> 32, v & 0xFFFFFFFF, (absv >> 32) & 0xFFFFFFFF, absv & 0xFFFFFFFF)
            parts[a.name] = [torch.zeros(g, dtype=torch.int64, device=ts.device).index_add_(0, inv, h) for h in halves]
    return uniq[0], (uniq[1] if key else None), n, out, parts


def check_group_by(got, want, aggs):
    """Every output row equals the group-by: the same (window_start, key) set, integers equal, AVG by its rule."""
    import torch
    ws, key, n, out, parts = want
    gws, gkey = got["window_start"], got.get("key")
    order = torch.argsort(gkey, stable=True) if gkey is not None else torch.arange(len(gws), device=gws.device)
    order = order[torch.argsort(gws[order], stable=True)]
    assert len(gws) == len(ws), (len(gws), len(ws))
    assert torch.equal(gws[order], ws)
    if key is not None:
        assert torch.equal(gkey[order], key)
    for a in aggs:
        g = got[a.name][order]
        if a.kind != "avg":
            bad = torch.nonzero(g != out[a.name]).flatten()
            assert bad.numel() == 0, (a.name, int(bad.numel()), int(bad[0]), int(g[bad[0]]), int(out[a.name][bad[0]]))
            continue
        hi, lo, ahi, alo = parts[a.name]
        abs_sum = torch.clamp(ahi, max=1 << 22) * (1 << 32) + alo
        small = abs_sum < (1 << 53)
        exact = (hi * (1 << 32) + lo).double() / n.double()  # exact integers below 2^53: one rounding
        bad = torch.nonzero(small & (g != exact)).flatten()
        assert bad.numel() == 0, (a.name, int(bad.numel()), float(g[bad[0]]), float(exact[bad[0]]))
        rest = torch.nonzero(~small).flatten()
        cols = [t[rest].cpu().tolist() for t in (g, hi, lo, ahi, alo, n)]
        for gv, h, l, ah, al, c in zip(*cols):
            assert X.check_avg(gv, X.Mean(Fraction((h << 32) + l, c), (ah << 32) + al)), (a.name, gv, h, l, c)


def run_device(cfg, batch, flags, expected_keys, primer):
    """One operator fed device-resident columns: with `primer`, first the first row of every key and of every pane
    (so the pane ring and the dictionary hold them), then every other row in one launch; otherwise every row in one
    launch.  Returns ({column: device tensor} of the output, the operator's statistics at the end and before the
    launch of the rest, the device columns)."""
    import torch

    from arroyo_b200 import operators as native
    from tests.gpu_ops import to_arrow
    names = list(batch.cols)
    key = cfg.key_names[0] if cfg.key_names else None
    n = batch.num_rows
    order = np.arange(n)
    m = 0
    if primer:
        bins = batch[TS] - batch[TS] % (cfg.slide or cfg.width)
        first = np.unique(bins, return_index=True)[1]
        if key:
            first = np.union1d(first, np.unique(batch[key], return_index=True)[1])
        rest = np.setdiff1d(order, first, assume_unique=True)
        order, m = np.concatenate([first, rest]), len(first)
    dev = {c: torch.from_numpy(np.ascontiguousarray(batch[c][order]).view(np.int64)).cuda() for c in names}
    cls = native.TumblingAggregatingWindowFunc if not cfg.slide else native.SlidingAggregatingWindowFunc
    op = cls(cfg, input_schema=to_arrow(O.Batch({c: batch[c][:1] for c in names})).schema, flags=flags,
             expected_keys=expected_keys)
    if m:
        op.process_device_batch([dev[c].data_ptr() for c in names], m)
        op.flush()
        op.flush()  # the second one re-ingests what the first launch deferred
    primed = op.stats()
    op.process_device_batch([dev[c].data_ptr() + 8 * m for c in names], n - m)
    op.flush()
    out_names = device_names(cfg)
    got = {c: [] for c in out_names}
    for rows, ptrs in op.handle_watermark_device(O.FINAL_WATERMARK):
        for c, p in zip(out_names, ptrs):
            got[c].append(torch.as_tensor(_Ptr(p, rows, "<f8" if c.startswith("av") else "<i8"), device="cuda").clone())
    st = op.stats()
    op.close()
    torch.cuda.synchronize()
    got = {c: torch.cat(v) if v else torch.zeros(0, device="cuda") for c, v in got.items()}
    return got, st, primed, dev


def large_stream(n, keys, regime, tumbling, seed):
    """`n` rows from gen_multi_stream over about 2.1 s (tumbling, 1 s windows) or 4.2 s (hop(1 s, 4 s)) of event time,
    in arrival order, rows of neighbouring panes interleaved within 32 rows of each boundary."""
    rng = np.random.default_rng(seed)
    n_keys = {"uniform": 1 << 20, "hot": 1 << 20, "warm8": 8, "none": 1 << 20, "u64": 1 << 20}[keys]
    rate = (n // 2 if tumbling else n // 4) // 1000 * 1000
    b = gen_multi_stream(rng, n, n_keys, rate_per_s=rate, key_dist={"warm8": "uniform", "none": "uniform"}.get(keys, keys),
                         regime=regime, batch=n, disorder=32)[0]
    if keys == "none":
        b = O.Batch({c: v for c, v in b.cols.items() if c != "key"})
    return b


def _cfg(aggs, keyed, tumbling):
    kn = ["key"] if keyed else []
    if tumbling:
        return O.WindowAggConfig(width=S, key_names=kn, aggs=aggs, window_index=len(kn))
    return O.WindowAggConfig(width=4 * S, slide=S, key_names=kn, aggs=aggs, window_index=len(kn))


# branch of `ingest_kernel<NV, SIG>` -> (plan, extra flag); every case runs with FLAG_NO_TWO_PASS
BRANCHES = {
    "nv0": ([A("count", None, "n")], 0),
    "nv1_sum_i64": ([A("sum", "a", "sa"), A("count", None, "n")], 0),
    "nv1_sum_f64": ([A("avg", "a", "ava"), A("count", None, "n")], "avg_f64"),
    "nv1_sum_i64_sum_f64": ([A("sum", "a", "sa"), A("avg", "a", "ava"), A("count", None, "n")], "avg_f64"),
    "nv1_min_max": ([A("min", "a", "mna"), A("max", "a", "mxa"), A("count", None, "n")], 0),
    "nv1_generic": ([A("min", "a", "mna"), A("max", "a", "mxa"), A("sum", "a", "sa"), A("avg", "a", "ava"),
                     A("count", None, "n")], 0),
    "nv2_generic": ([A("sum", "a", "sa"), A("min", "b", "mnb"), A("avg", "a", "ava"), A("count", None, "n")], 0),
    "nv3_generic": ([A("max", "a", "mxa"), A("sum", "b", "sb"), A("avg", "c", "avc"), A("count", None, "n")], 0),
    "nv4_generic": ([A("avg", "a", "ava"), A("min", "a", "mna"), A("max", "b", "mxb"), A("sum", "c", "sc"),
                     A("avg", "d", "avd"), A("count", None, "n")], 0),
}
KEY_SETS = ["uniform", "hot", "warm8", "none", "u64"]
LARGE_CASES = []
for _i, _b in enumerate(BRANCHES):
    LARGE_CASES.append((_b, "tumbling", KEY_SETS[_i % 5], "R1" if _i % 2 else "R2"))
    LARGE_CASES.append((_b, "sliding", KEY_SETS[(_i + 2) % 5], "R2" if _i % 2 else "R1"))


@pytest.mark.parametrize("branch,window,keys,regime", LARGE_CASES, ids=["-".join(c) for c in LARGE_CASES])
def test_every_one_pass_kernel_in_a_large_launch(branch, window, keys, regime):
    from arroyo_b200 import ffi
    aggs, extra = BRANCHES[branch]
    tumbling = window == "tumbling"
    n = 1 << 24 if tumbling else 1 << 22
    b = large_stream(n, keys, regime, tumbling, seed=LARGE_CASES.index((branch, window, keys, regime)))
    cfg = _cfg(aggs, keys != "none", tumbling)
    flags = ffi.FLAG_NO_TWO_PASS | (ffi.FLAG_AVG_F64 if extra == "avg_f64" else 0)
    got, st, primed, dev = run_device(cfg, b, flags, expected_keys=1 << 20 if keys != "warm8" else 64, primer=True)
    assert st["rows_in"] == n and st["rows_late"] == 0
    # with every key and pane known, the launch defers nothing but values beyond the exact-AVG guard
    guarded = regime == "R2" and extra != "avg_f64" and any(a.kind == "avg" for a in aggs)
    assert st["rows_deferred"] == primed["rows_deferred"] or guarded
    key = "key" if keys != "none" else None
    check_group_by(got, group_by(dev, key, aggs, cfg.width, cfg.slide or None), aggs)


def test_deferred_rows_carry_four_columns_while_the_dictionary_grows():
    """P4 over 2^20 keys in one 2^22-row launch on a dictionary sized for 256 keys: rows of unknown keys and of panes
    not yet in the ring are deferred with all four value columns and re-ingested after the dictionary grows."""
    from arroyo_b200 import ffi
    aggs = BRANCHES["nv4_generic"][0]
    b = large_stream(1 << 22, "uniform", "R1", False, seed=101)
    cfg = _cfg(aggs, True, False)
    got, st, _, dev = run_device(cfg, b, ffi.FLAG_NO_TWO_PASS, expected_keys=256, primer=False)
    assert st["rows_deferred"] > 0 and st["rows_in"] == 1 << 22 and st["rows_late"] == 0
    assert st["n_keys"] == len(np.unique(b["key"]))
    check_group_by(got, group_by(dev, "key", aggs, cfg.width, cfg.slide), aggs)


def test_one_big_value_promotes_avg_in_a_large_launch():
    """One value >= 2^31 in the middle of a 2^24-row exact-AVG launch: the row is deferred, the operator promotes AVG to
    f64 accumulators and re-ingests it; no row is lost and every AVG follows the rule."""
    from arroyo_b200 import ffi
    aggs = [A("avg", "a", "ava"), A("sum", "a", "sa"), A("count", None, "n")]
    b = large_stream(1 << 24, "uniform", "R1", True, seed=102)
    b["a"][len(b["a"]) // 2] = (1 << 40) + 3
    cfg = _cfg(aggs, True, True)
    got, st, primed, dev = run_device(cfg, b, ffi.FLAG_NO_TWO_PASS, expected_keys=1 << 20, primer=True)
    assert st["rows_deferred"] > primed["rows_deferred"] and st["rows_in"] == 1 << 24 and st["rows_late"] == 0
    check_group_by(got, group_by(dev, "key", aggs, cfg.width, None), aggs)
