"""The join with expiration's key-time tables and lazy restore in the state oracle (tests/ttl_join_state_oracle.py)
against the exact restart reference (`expiring_join_restarts`, built on exact_reference.expiring_join): restarts at
every batch boundary of random two-sided streams, two restarts in a row, empty and one-sided tables, the cutoff at
watermark - ttl and its edges, and the golden `updating_inner_join` across a restart."""
import numpy as np
import pytest

from oracle import arroyo_oracle as O
from tests import exact_reference as X
from tests import ttl_join_state_oracle as S

TS = O.TIMESTAMP
T0 = 1_700_000_000 * 10 ** 9


def random_stream(rng, n_batches=12, n_keys=40, delay=2_000):
    """Two sides with duplicate keys inside and across batches, timestamps rising, a watermark `delay` behind the
    newest row after every other batch."""
    events, t = [], T0
    for i in range(n_batches):
        side = int(rng.integers(0, 2)) if i > 1 else i
        n = int(rng.integers(0, 60)) if i > 1 else 30
        ts = t + np.sort(rng.integers(0, 1_000, n))
        t += 1_000
        cols = {"k": rng.integers(0, n_keys, n).astype(np.int64), ("a" if side == 0 else "b"): rng.integers(-9, 9, n),
                TS: ts.astype(np.int64)}
        events.append((side, cols))
        if i % 2:
            events.append(("wm", t - delay))
    return events


def with_restarts(events, at):
    """`events` with a restart before the batch events numbered in `at` (len(batches): at the end)."""
    out, b = [], 0
    for ev in events:
        if ev[0] in (0, 1):
            out += [("restart", None)] * at.count(b)
            b += 1
        out.append(ev)
    return out + [("restart", None)] * at.count(b)


def check(events, ttl, on="k"):
    want = S.expiring_join_restarts(events, ttl, on, on)
    got, _ = S.run_oracle(events, ttl, on, on)
    assert len(got) == len(want)
    for i, (w, g) in enumerate(zip(want, got)):
        assert not X.join_mismatches(w, g), (i, X.join_mismatches(w, g))
    return want


@pytest.mark.parametrize("ttl", [0, 2_500, 6_000])
@pytest.mark.parametrize("seed", [0, 1, 2])
def test_restart_at_every_batch_boundary(seed, ttl):
    events = random_stream(np.random.default_rng(seed))
    n = sum(1 for e in events if e[0] in (0, 1))
    plain = check(events, ttl)
    dropped = 0
    for k in range(n + 1):
        want = check(with_restarts(events, [k]), ttl)
        dropped += sum(len(a) for a in plain) - sum(len(a) for a in want)
    assert sum(len(a) for a in plain) > 0
    if ttl:  # a small ttl drops batches at some restarts, so some pairs are lost to the cutoff
        assert dropped > 0


@pytest.mark.parametrize("seed", [3, 4])
def test_two_restarts(seed):
    events = random_stream(np.random.default_rng(seed))
    n = sum(1 for e in events if e[0] in (0, 1))
    for at in ([3, 3], [2, 7], [0, 0], [n, n], [4, n]):
        for ttl in (0, 3_000):
            check(with_restarts(events, at), ttl)


def test_restart_with_empty_tables_and_one_sided_tables():
    rng = np.random.default_rng(5)
    events = random_stream(rng)
    check(with_restarts(events, [0]), 0)  # nothing inserted yet

    def batch(name, t):
        return {"k": rng.integers(0, 10, 50), name: rng.integers(0, 9, 50), TS: t + np.arange(50)}
    left = [(0, batch("a", T0 + 100 * i)) for i in range(4)]
    right = [(1, batch("b", T0 + 1_000 + 100 * i)) for i in range(3)]
    want = check(left + [("restart", None)] + right + [("restart", None)] + left, 0)
    assert sum(len(w) for w in want) > 0  # the right side's later batches pair with the restored left rows


def _edge(ts_left, wm, ttl, restart_wm=None):
    """Left batches with newest timestamps `ts_left` (one row each, key 1), a checkpoint at watermark `wm`, a restart,
    optionally a watermark `restart_wm` before the first batch, then one right row with key 1.  Returns the newest
    timestamps of the left batches the right row pairs with."""
    events = [(0, {"k": np.array([1]), "a": np.array([i]), TS: np.array([t])}) for i, t in enumerate(ts_left)]
    if wm is not None:
        events.append(("wm", wm))
    events.append(("restart", None))
    if restart_wm is not None:
        events.append(("wm", restart_wm))
    events.append((1, {"k": np.array([1]), "b": np.array([0]), TS: np.array([max(ts_left) + 1])}))
    want = check(events, ttl)[-1]
    a = want.names.index("a")
    return sorted(ts_left[int(i)] for i in want.vals[:, a])


def test_cutoff_is_inclusive():
    """A batch whose newest timestamp equals watermark - ttl is kept; one at watermark - ttl - 1 is dropped."""
    ttl = 1_000
    assert _edge([T0 - 1, T0, T0 + 5], T0 + ttl, ttl) == [T0, T0 + 5]


def test_a_watermark_after_the_restart_moves_the_cutoff():
    """The tables are loaded at the first batch, with the watermark of that moment."""
    ttl = 1_000
    assert _edge([T0, T0 + 10, T0 + 20], T0 + ttl, ttl) == [T0, T0 + 10, T0 + 20]
    assert _edge([T0, T0 + 10, T0 + 20], T0 + ttl, ttl, restart_wm=T0 + ttl + 10) == [T0 + 10, T0 + 20]


def test_without_a_watermark_the_cutoff_is_the_epoch():
    assert _edge([-1, 0, 5], None, 1_000) == [0, 5]


def test_ttl_zero_means_a_day():
    day = S.DAY_NS
    assert _edge([T0 - day - 1, T0 - day, T0], T0, 0) == [T0 - day, T0]
    assert _edge([T0 - day - 1, T0 - day, T0], T0, day) == [T0 - day, T0]
    assert _edge([T0 - day - 1, T0 - day, T0], T0, 1) == [T0]


def golden_feed(golden, order, batch=32):
    counter, ts = golden[0]["impulse_counter"], golden[0]["impulse_ts"]
    odd = counter % 2 == 1
    left = [(0, b) for b in O.source_batches({"counter": counter, TS: ts}, batch)]
    right = [(1, b) for b in O.source_batches({"counter": counter[odd], TS: ts[odd]}, batch)]
    return {"left_first": left + right, "right_first": right + left,
            "alternating": [x for pair in zip(left, right + [None] * len(left)) for x in pair if x]}[order]


def golden_rows(rows: X.Rows):
    li, ri = rows.names.index("counter"), rows.names.index("counter_right")
    return [{"left_count": int(v[li]), "right_count": int(v[ri])} for v in rows.vals]


@pytest.mark.parametrize("order", ["left_first", "right_first", "alternating"])
def test_updating_inner_join_golden_across_a_restart(golden, accumulator_golden, order):
    from tests.golden_cases import multiset
    feed = golden_feed(golden, order)
    for k in range(len(feed) + 1):
        events = with_restarts(feed, [k])
        got, _ = S.run_oracle(events, 0, "counter", "counter")
        rows = [r for g in got for r in golden_rows(g)]
        assert multiset(rows) == multiset(accumulator_golden["updating_inner_join"]), k
        check(events, 0, "counter")
