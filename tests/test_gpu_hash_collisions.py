"""Every GPU hash table of the library fed keys that collide and wrap (tests/collide.py), against the exact references.

Random keys at the load factors these tables run at (about 0.25 to 0.5) give probe chains of a few slots, so the code
that only runs on long chains -- the walk past a full home group, the wrap from a table's last slot to slot 0, many
warps inserting first-seen keys into one chain, the rehash and rebuild kernels re-placing long chains, every probe
bound -- never runs under the random-key suites.  Here every key of a case shares one home slot, and that slot is the
table's last one at every size the operator reaches:

* the tumbling and sliding window aggregates (bucketed dictionary, two-pass ingest lookup table), one-pass and
  two-pass, with a restart (restored keys placed by bd_place_kernel), growth that splits a long chain, device input,
  and one 2^20-row launch in which every key is first seen;
* the updating aggregate (the same bucketed dictionary), flush by flush and across a restart;
* the session aggregate (dict.cuh): chains of 1000 to 6000 keys, dictionary growth while the chain is live, restarts;
* the instant-window aggregate: 4000 (instant, key) groups in one chain, a watermark that releases half of it, a
  batch that doubles the group blocks and rebuilds the table while the chain is open;
* the instant join's build table, all four join types, and the join with expiration's multimap through its rehash
  and across restarts;
* the shuffle partitioner with every row routed to one destination, and to the last one;
* structured key families (shifted counters, nanosecond timestamps, equal halves) through the window and session
  aggregates.

The CPU tests check the key sets' properties against the restated home functions, that the restatement still
matches the sources it cites, and that mix64 matches the library's."""
import os

import numpy as np
import pytest

from oracle import arroyo_oracle as O
from tests import collide as K
from tests import exact_reference as X

A = O.Agg
TS = O.TIMESTAMP
SEC = 1_000_000_000
ORIGIN = 1_700_000_000 * SEC
INT64_MAX = (1 << 63) - 1


# ---- CPU: the key sets and the restatement --------------------------------------------------------------------------
def test_restated_hashes_match_the_sources():
    for name, text in K.SOURCES:
        with open(os.path.join(K.CSRC, name)) as f:
            assert text in f.read(), (name, text)


def test_mix64_inverse_and_library():
    from arroyo_b200 import ffi
    rng = np.random.default_rng(1)
    x = np.concatenate([rng.integers(-(1 << 63), INT64_MAX, 2000, dtype=np.int64),
                        np.array([0, 1, -1, -(1 << 63), INT64_MAX], dtype=np.int64)])
    h = K.mix64(x)
    assert (K.mix64_inv(h).view(np.int64) == x).all()
    assert (h == O.mix64(x.view(np.uint64))).all()
    lib = ffi.load()
    for k, hv in zip(x[:300].tolist(), h[:300].tolist()):
        assert lib.arroyo_b200_hash_key(k) == hv


def test_key_sets_have_their_properties():
    for tag in ("one", "distinct"):
        k = K.bucketed_chain(K.BD_CAPB, seed=3, tag=tag)
        assert len(np.unique(k)) == K.BD_CAPB
        assert (K.bd_slot0(k) == K.BD_KS - K.BD_GROUP).all()
        assert (K.p2_group(k) == K.P2_HS - K.P2_HG).all()
        tags = len(set(K.p2_tag(k).tolist()))
        assert tags == 1 if tag == "one" else tags >= 240, tags  # about five keys per tag
        for nb in list(range(1, 65)) + [1000, 1024, 2047, 4095, 4096]:
            assert (K.bd_bucket(k, nb) == nb - 1).all(), nb
    for b in (1, 64):
        k = K.bucketed_chain(1800, seed=4, split_at=b)
        assert (K.bd_bucket(k, b) == b - 1).all() and (K.bd_slot0(k) == K.BD_KS - K.BD_GROUP).all()
        assert np.bincount(K.bd_bucket(k, 2 * b) - (2 * b - 2)).tolist() == [900, 900]
    k = K.session_chain(6000, seed=5)
    assert len(np.unique(k)) == 6000
    for cap in (1024, 3584, 7168, 28679, 1 << 20, (1 << 31) - 3):
        assert (K.dict_home(k, cap) == cap - 1).all(), cap
    k = K.ttl_chain(3000, seed=6)
    assert len(np.unique(k)) == 3000
    for bits in range(10, 33):
        assert (K.tj_home(k, (1 << bits) - 1) == (1 << bits) - 1).all()
    times = ORIGIN + np.arange(50) * SEC
    ts, k = K.instant_chain(times, 80, seed=7)
    assert len({(int(a), int(b)) for a, b in zip(ts, k)}) == 4000
    for bits in range(8, 33):
        m = (1 << bits) - 1
        assert (K.instant_home(ts, k, m) == m).all() and (K.pair_home(k, ts, m) == m).all()
    for where in ("first", "last"):
        k = K.routed(500, where, seed=8)
        for n in (2, 3, 8):
            assert (K.dest(k, n) == (0 if where == "first" else n - 1)).all()
            assert (K.dest(k, n) == O.server_for_hash_array(O.mix64(k.view(np.uint64)), n).astype(np.int64)).all()
    fams = K.families()
    assert len(fams) == 10 and all(len(np.unique(v)) == len(v) for v in fams.values())


# ---- the window aggregates -------------------------------------------------------------------------------------------
KEYSETS = {
    "one_tag": lambda: K.bucketed_chain(K.BD_CAPB, seed=11, tag="one"),
    "tags": lambda: K.bucketed_chain(K.BD_CAPB, seed=12, tag="distinct"),
    # 1800 keys in the one bucket of a dictionary sized for 1024: the bucket runs out of ids, the dictionary doubles,
    # and bd_rehash_kernel splits the chain 900 / 900
    "split": lambda: K.bucketed_chain(1800, seed=13, split_at=1),
}
_KEYS = {}


def keyset(name):
    if name not in _KEYS:
        _KEYS[name] = KEYSETS[name]() if name in KEYSETS else K.families()[name]
    return _KEYS[name]


def window_events(keys, rng, n_per_key=8, restart=True):
    """A few keys to open the stream's pane, then every key first seen in one launch, then a watermark, a restart
    (restored keys go through bd_place_kernel), more rows of every key, and the end."""
    events, n = [], len(keys)

    def batch(ks, t0):
        m = len(ks)
        events.append(("batch", O.Batch({"key": np.asarray(ks, dtype=np.int64), "a": rng.integers(-1000, 1000, m),
                                         TS: t0 + rng.integers(0, SEC, m)})))
    batch(keys[:3], ORIGIN)
    batch(rng.permutation(np.repeat(keys, n_per_key)), ORIGIN)
    batch(rng.permutation(np.repeat(keys, 2)), ORIGIN + SEC)
    events.append(("wm", ORIGIN + SEC))
    if restart:
        events.append(("restart",))
    batch(rng.permutation(np.repeat(keys, 3)), ORIGIN + SEC)
    batch(rng.permutation(keys), ORIGIN + 2 * SEC)
    events.append(("wm", ORIGIN + 2 * SEC + 1))
    events.append(("wm", INT64_MAX))
    return events


WPLANS = {"count": [A("count", None, "n")],
          "sum_avg": [A("sum", "a", "sa"), A("avg", "a", "ava")],
          "minmax": [A("min", "a", "mna"), A("max", "a", "mxa")]}
WCASES = [
    ("tumbling", "one_tag", "sum_avg", "two_pass"), ("tumbling", "one_tag", "count", "one_pass"),
    ("sliding", "one_tag", "count", "two_pass"), ("sliding", "one_tag", "sum_avg", "one_pass"),
    ("tumbling", "tags", "count", "two_pass"), ("sliding", "tags", "sum_avg", "two_pass"),
    ("sliding", "tags", "minmax", "one_pass"), ("tumbling", "tags", "minmax", "device"),
    ("tumbling", "split", "sum_avg", "two_pass"), ("sliding", "split", "count", "two_pass"),
    ("sliding", "split", "minmax", "one_pass"), ("sliding", "one_tag", "sum_avg", "device"),
]


def run_window(keys, kind, plan, entry, seed, restart=True):
    from tests import test_gpu_window_time as W
    rng = np.random.default_rng(seed)
    st = W.Stream(seed, "few", 2 * SEC if kind == "sliding" else SEC, SEC if kind == "sliding" else None)
    st.events = window_events(keys, rng, restart=restart and entry != "device")
    cfg = O.WindowAggConfig(width=st.width, slide=st.slide if kind == "sliding" else 0, key_names=["key"],
                            aggs=WPLANS[plan], window_index=1)
    want, late = X.window_emissions(st.events, "key", cfg.aggs, cfg.width, cfg.slide or None)
    # expected_keys = 1024: one bucket, so the two-pass regions take every row of the launch
    got, rows_in, rows_late, n_keys = W.run_gpu(st, "running" if kind == "sliding" else "tumbling", cfg, entry,
                                                expected_keys=1024)
    W.check_emissions(want, got, cfg, f"{kind}/{plan}/{entry}")
    assert rows_in == sum(ev[1].num_rows for ev in st.events if ev[0] == "batch")
    assert rows_late == late
    assert n_keys == len(np.unique(keys[keys != -(1 << 63)]))  # the INT64_MIN key has a reserved id, not a slot


@pytest.mark.gpu
@pytest.mark.parametrize("kind,keys,plan,entry", WCASES, ids=["-".join(c) for c in WCASES])
def test_window_colliding_keys(kind, keys, plan, entry):
    run_window(keyset(keys), kind, plan, entry, seed=len(kind) * 7 + len(keys) * 3 + len(plan) + len(entry))


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["two_pass", "one_pass"])
@pytest.mark.parametrize("keys", ["one_tag", "tags"])
def test_window_one_launch_of_2_20_rows(mode, keys):
    """Every key first seen inside one 2^20-row launch: many warps insert into the same chain at once.  The window
    is checked against an independent torch group-by of the rows."""
    import torch

    import arroyo_b200 as ab
    from arroyo_b200 import ffi, operators as native
    from tests.gpu_ops import from_arrow, to_arrow
    ks = keyset(keys)
    rng = np.random.default_rng(len(mode) + len(keys))
    n = 1 << 20
    key = ks[rng.integers(0, len(ks), n)]
    key[: len(ks)] = ks
    a = rng.integers(-(1 << 40), 1 << 40, n)
    first = O.Batch({"key": ks[:2].copy(), "a": np.array([5, -7]), TS: np.array([ORIGIN, ORIGIN + 1])})
    big = O.Batch({"key": key, "a": a, TS: ORIGIN + rng.integers(0, SEC, n)})
    aggs = [A("count", None, "n"), A("sum", "a", "sa")]
    cfg = O.WindowAggConfig(width=SEC, slide=0, key_names=["key"], aggs=aggs, window_index=1)
    flags = ffi.FLAG_TWO_PASS_ALWAYS if mode == "two_pass" else ffi.FLAG_NO_TWO_PASS
    op = native.TumblingAggregatingWindowFunc(cfg, input_schema=to_arrow(first).schema, flags=flags,
                                              expected_keys=1024)
    ctx = ab.OperatorContext(1)
    op.process_batch(to_arrow(first), ctx, None)
    op.process_batch(to_arrow(big), ctx, None)
    ctx.watermarks.set(0, INT64_MAX)
    col = ab.Collector()
    op.handle_watermark(INT64_MAX, ctx, col)
    stats = op.stats()
    op.close()
    rows = [r for b in col.batches for r in from_arrow(b).rows()]
    allk = torch.from_numpy(np.concatenate([first["key"], key]))
    alla = torch.from_numpy(np.concatenate([first["a"], a]))
    uk, inv = torch.unique(allk, return_inverse=True)
    cnt = torch.zeros(len(uk), dtype=torch.int64).index_add_(0, inv, torch.ones_like(alla))
    sm = torch.zeros(len(uk), dtype=torch.int64).index_add_(0, inv, alla)
    want = {int(k): (int(c), int(s)) for k, c, s in zip(uk.tolist(), cnt.tolist(), sm.tolist())}
    got = {int(r["key"]): (int(r["n"]), int(r["sa"])) for r in rows}
    assert len(rows) == len(got) == len(ks)
    assert got == want
    assert all(int(r["window_start"]) == ORIGIN - ORIGIN % SEC for r in rows)
    assert stats["rows_in"] == n + 2 and stats["rows_deferred"] == 0 and stats["n_keys"] == len(ks)


# ---- the updating aggregate ------------------------------------------------------------------------------------------
UCASES = [("one_tag", "P2", "host", 1024), ("tags", "COUNT", "device", 1 << 16), ("split", "AMM", "mixed", 1024),
          ("tags", "P1", "sliced", 1024)]


def updating_stream(keys, seed, expected):
    from tests import test_gpu_updating_changes as UC
    st = UC.Stream(seed, "i64", expected_keys=expected)
    st.batch(keys=st.rng.permutation(np.concatenate([keys, keys[: len(keys) // 3]])))
    st.flush()
    st.batch(keys=st.rng.choice(keys, 3000))
    st.batch(keys=st.rng.permutation(keys))
    st.flush()
    st.batch(keys=st.rng.choice(keys, 500))
    st.flush()
    st.batch(keys=st.rng.permutation(keys))
    st.flush()
    return st


@pytest.mark.gpu
@pytest.mark.parametrize("keys,plan,entry,expected", UCASES, ids=["-".join(map(str, c)) for c in UCASES])
def test_updating_colliding_keys(keys, plan, entry, expected):
    from tests import test_gpu_updating_changes as UC
    st = updating_stream(keyset(keys), len(keys) + len(plan), expected)
    aggs = UC.PLANS[plan]
    want = UC.reference(st, aggs)
    got, stats = UC.run_gpu(st, aggs, entry)
    UC.check(st, aggs, got, stats, want, f"{keys}/{plan}/{entry}")


URCASES = [("one_tag", "P2", "host"), ("tags", "COUNT", "device"), ("split", "AMM", "host")]


@pytest.mark.gpu
@pytest.mark.parametrize("keys,plan,entry", URCASES, ids=["-".join(c) for c in URCASES])
def test_updating_colliding_keys_across_a_restart(keys, plan, entry):
    """A restart at the second flush: the new operator, sized for 256 keys (one bucket), places every restored key of
    table "a" through bd_place_kernel into the one colliding chain (for "split": the bucket runs out of ids, the
    dictionary doubles and the chain splits) before the rest of the stream."""
    from tests import test_gpu_updating_changes as UC
    from tests import test_gpu_updating_restore as UR
    st = updating_stream(keyset(keys), len(keys) + len(plan) + 1, 1024)
    aggs = UC.PLANS[plan]
    want = X.updating_changes(st.events, st.key_name(), aggs)
    outs, _, stats, rows_since = UR.run(st, aggs, entry, restarts={1}, seed=len(keys))
    n_out = UR.check_changes(st, aggs, outs, want, f"{keys}/{plan}/{entry}")
    assert stats["rows_in"] == rows_since
    assert stats["n_keys"] == len(keyset(keys))
    assert stats["rows_out"] == sum(n_out[2:])


# ---- the session aggregate -------------------------------------------------------------------------------------------
def session_stream(keys, seed, gap=5 * SEC, restart=False, waves=1):
    from tests import test_gpu_session_time as S
    st, o = S.Stream(seed, "few", gap), ORIGIN
    st.wm(o - 10 * gap)
    for part in np.array_split(keys, waves):  # waves > 1: the dictionary grows while earlier keys' sessions are open
        st.batch(o + st.rng.integers(0, gap // 2, 2 * len(part)), np.tile(part, 2))
        st.wm(o - 5 * gap)
    st.batch(o + gap // 2 + st.rng.integers(0, gap // 2, len(keys)), keys)
    st.wm(o + 2 * gap)  # closes every session opened so far
    if restart:
        st.restart()
    st.batch(o + 3 * gap + st.rng.integers(0, gap, len(keys)), keys[::-1].copy())
    st.batch(o + 5 * gap + st.rng.integers(0, gap, len(keys[::2])), keys[::2].copy())
    st.wm(o + 4 * gap)
    if restart:
        st.restart()
    return st.end()


def check_session_counts(st, cfg, late, n_keys, rows_in, rows_late, n_keys_got):
    """The operator's rows_in, rows_late and n_keys statistics against the stream and the reference."""
    assert rows_in == sum(ev[1].num_rows for ev in st.events if ev[0] == "batch")
    assert rows_late == late
    if cfg.key_names:
        assert n_keys_got == n_keys


SCASES = [(1000, "host", 1, False), (4000, "device", 1, False), (4097, "host", 1, False), (4097, "device", 1, False),
          (6000, "host", 1, True), (6000, "poll_host", 1, False), (4000, "host", 8, False)]


@pytest.mark.gpu
@pytest.mark.parametrize("n,entry,waves,restart", SCASES, ids=[f"{n}-{e}-w{w}{'-restart' if r else ''}"
                                                               for n, e, w, r in SCASES])
def test_session_colliding_keys(n, entry, waves, restart):
    """n keys in one chain that starts at the dictionary's last slot and wraps.  Chains longer than 4096 slots used to
    hit the insert's probe bound: their rows were dropped and the batch failed as a pool overflow."""
    from tests import test_gpu_session_time as S
    st = session_stream(K.session_chain(n, seed=n + waves), n + waves, restart=restart, waves=waves)
    cfg = S.config(st, "mix2")
    want, late, n_keys = S.reference(st, cfg)
    # waves > 1: sized for one key, the id space and the dictionary grow (dict_rebuild_kernel) under the live chain
    got, rows_in, rows_late, nk = S.run_gpu(st, cfg, entry, expected_keys=1 if waves > 1 else 64)
    S.check_emissions(want, got, cfg, f"session {n}")
    check_session_counts(st, cfg, late, n_keys, rows_in, rows_late, nk)
    assert n_keys == n


# ---- the instant-window aggregate ------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("entry", ["host", "device"])
def test_instant_window_colliding_groups(entry):
    """4000 (instant, key) groups in one chain across 50 instants; a watermark releases the first 25 instants, then
    rows arrive for the groups that stay (they must find their groups, not open second ones); one batch of more than
    2^16 rows -- the groups that stay and 4000 new colliding groups, repeated -- makes the operator double its group
    blocks and rebuild its table under a new mask while the chain is open; with host input, a restart."""
    from tests import test_gpu_instant_window as IW
    rng = np.random.default_rng(21)
    times = ORIGIN + np.arange(100, dtype=np.int64) * SEC
    ts, keys = K.instant_chain(times, 80, seed=22)
    first, second = slice(0, 4000), slice(4000, 8000)
    events = []

    def batch(t, k):
        order = rng.permutation(len(t))
        events.append(("batch", O.Batch({"key": k[order], "a": rng.integers(-1000, 1000, len(t)), TS: t[order]})))
    batch(np.repeat(ts[first], 2), np.repeat(keys[first], 2))
    events.append(("wm", int(times[25])))
    stay = slice(25 * 80, 4000)
    batch(ts[stay], keys[stay])
    # 72000 rows in one batch: the operator reserves a group per row handed over, and its first group blocks hold
    # 2^16 groups (instant_agg.cu), so the blocks double and the table is rebuilt (twice the slots, a new mask) from
    # the 2000 open groups of the chain before this batch's rows look their groups up
    big_t = np.concatenate([np.repeat(ts[stay], 18), np.repeat(ts[second], 9)])
    assert len(big_t) > 1 << 16
    batch(big_t, np.concatenate([np.repeat(keys[stay], 18), np.repeat(keys[second], 9)]))
    if entry == "host":
        events.append(("restart",))
    batch(ts[stay], keys[stay])
    events.append(("wm", int(times[60])))
    batch(ts[second], keys[second])
    events.append(("wm", INT64_MAX))
    st = IW.Stream(0, "many")
    st.events = events
    cfg = IW.gpu_config("many", "minmax")
    want, late = IW.instant_emissions(events, "key", IW.PLANS["minmax"])
    got, rows_in, rows_late, _ = IW.run_gpu(st, cfg, entry)
    IW.check_emissions(want, got, "key", f"instant {entry}")
    assert rows_in == sum(ev[1].num_rows for ev in events if ev[0] == "batch") and rows_late == late
    assert sum(len(rows) for w in want for _, rows in w) == 8000


# ---- the joins -------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("join_type", ["inner", "left", "right", "full"])
def test_instant_join_colliding_pairs(join_type):
    """4000 (key, ts) pairs per side that share the build table's last slot, duplicates of the same pair included,
    and a watermark that releases several instants whose pairs all share the slot."""
    from tests import test_gpu_joins as J
    rng = np.random.default_rng(31)
    st = J.Stream(rng)
    times = ORIGIN + np.arange(40, dtype=np.int64) * SEC
    ts, keys = K.pair_chain(times, 100, seed=32)
    left = rng.permutation(4000)
    st.send(0, keys[left].tolist() + keys[left[:500]].tolist(), np.concatenate([ts[left], ts[left[:500]]]))
    right = rng.choice(4000, 3000, replace=False)
    st.send(1, keys[right].tolist() + keys[right[:300]].tolist(), np.concatenate([ts[right], ts[right[:300]]]))
    st.wm(int(times[10]))
    again = left[ts[left] >= times[10]][:800]  # the reference join takes no late rows
    st.send(1, keys[again].tolist(), ts[again])
    st.wm(int(times[30]))
    st.wm(INT64_MAX)
    want = st.reference_instant(join_type)
    got, stats, _ = J.run_instant(st, join_type, "host")
    assert len(got) == len(want)
    total = 0
    for i, (w, g) in enumerate(zip(want, got)):
        J.check(w, J.rows_of(g, g[0].schema.names if g else w.names), ("colliding", join_type, "watermark", i))
        total += len(w)
    assert total > 0 and stats["rows_out"] == total


def expiring_stream(seed, rounds=12, random_left=20_000):
    from tests import test_gpu_joins as J
    rng = np.random.default_rng(seed)
    chain = K.ttl_chain(3000, seed=seed + 1)
    st = J.Stream(rng)
    t = ORIGIN
    for i in range(rounds):
        ks = np.concatenate([rng.choice(chain, 2000), rng.integers(0, 1 << 40, random_left)])
        st.send(0, rng.permutation(ks).tolist(), t + np.arange(len(ks)))
        t += len(ks)
        ks = np.concatenate([rng.choice(chain, 500), rng.integers(0, 1 << 40, 200)])
        st.send(1, ks.tolist(), t + np.arange(len(ks)))
        t += len(ks)
    return st


@pytest.mark.gpu
def test_expiring_join_colliding_keys():
    """3000 keys in one multimap chain on both sides, next to enough random keys that the multimap rehashes four
    times while the chain is live; every batch's output against the exact reference."""
    from tests import test_gpu_joins as J
    st = expiring_stream(41)
    want = st.reference_expiring()
    got, stats = J.run_expiring(st, "host")
    total = 0
    for i, (w, g) in enumerate(zip(want, got)):
        J.check(w, J.rows_of(g, w.names), ("colliding expiring", "batch", i))
        total += len(w)
    assert total > 0 and stats["rows_out"] == total


@pytest.mark.gpu
@pytest.mark.parametrize("at", [[2], [5, 9]])
def test_expiring_join_colliding_keys_across_restarts(at):
    """Restarts with the colliding chain in both tables: restore_side links every restored row into the one chain
    (tj_link_kernel), then the next batches probe it and grow it through rehashes; against the exact restart
    reference."""
    from tests import test_gpu_ttl_join_restore as TR
    st = expiring_stream(43, rounds=6, random_left=12_000)
    events = TR.with_watermarks(st.events)
    want, ops, _ = TR.check_run(st, TR.with_restarts(events, at), 0, what=("colliding restarts", at))
    assert sum(len(w) for w in want) > 0 and len(ops) == len(at) + 1


# ---- the shuffle partitioner -----------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("where", ["first", "last"])
@pytest.mark.parametrize("world", [2, 3, 8])
def test_partition_all_rows_to_one_destination(world, where):
    import torch

    from arroyo_b200.multi_gpu import DevicePartitioner
    n = 50_000
    keys = K.routed(n, where, seed=world)
    rng = np.random.default_rng(world)
    cols = {"key": keys, "v": rng.integers(-(1 << 62), 1 << 62, n), TS: ORIGIN + np.arange(n, dtype=np.int64)}
    want = dict(O.repartition(O.Batch(cols), ["key"], world))
    dst = 0 if where == "first" else world - 1
    assert list(want) == [dst]
    stream = torch.cuda.Stream()
    with torch.cuda.stream(stream):
        dev = [torch.from_numpy(cols[c]).cuda() for c in ("key", "v", TS)]
        part = DevicePartitioner(torch, world, 3, 0, n, 0, stream.cuda_stream)
        try:
            out, counts = part(dev, n)
            stream.synchronize()
            assert counts.cpu().tolist() == [n if d == dst else 0 for d in range(world)]
            got = np.stack([o.cpu().numpy() for o in out], 1)
            packed, counts2 = part.pack([t.data_ptr() for t in dev], n)
            stream.synchronize()
            assert counts2.cpu().tolist() == counts.cpu().tolist()
            pk = packed.cpu().numpy().reshape(3, n).T  # one destination's block: its 3 columns back to back
        finally:
            part.close()
    exp = np.stack([want[dst][c] for c in ("key", "v", TS)], 1)
    for g in (got, pk):
        assert (g[np.lexsort(g.T[::-1])] == exp[np.lexsort(exp.T[::-1])]).all()


# ---- structured key families -----------------------------------------------------------------------------------------
FAMILIES = ["shift0", "shift8", "shift16", "shift32", "shift48", "shift53", "shift56", "shift60", "origin_ns", "halves"]


@pytest.mark.gpu
@pytest.mark.parametrize("family", FAMILIES)
def test_key_families(family):
    """Shifted counters, nanosecond timestamps and equal-halves keys through the two-pass window aggregate and the
    session aggregate."""
    from tests import test_gpu_session_time as S
    keys = keyset(family)
    run_window(keys, "sliding", "sum_avg", "two_pass", seed=len(family), restart=False)
    st = session_stream(keys, len(family))
    cfg = S.config(st, "mix3")
    want, late, n_keys = S.reference(st, cfg)
    got, rows_in, rows_late, nk = S.run_gpu(st, cfg, "host", expected_keys=64)
    S.check_emissions(want, got, cfg, f"session {family}")
    check_session_counts(st, cfg, late, n_keys, rows_in, rows_late, nk)
