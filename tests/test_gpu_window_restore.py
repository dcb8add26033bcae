"""Restores of the tumbling and sliding window aggregates whose panes hold more keys of one dictionary bucket than the
bucket has ids (BD_CAPB = 1280), against tests/exact_reference.window_emissions.

A running window takes such keys by deferring their rows and growing the dictionary (test_gpu_updating_changes.py::
test_window_crowded_bucket).  A checkpoint it writes then holds them in one partial-state batch, and a fresh operator
with the same config (64 buckets) must restore it: every key gets its id first, the dictionary doubling until the
crowded bucket splits, and only then is the batch merged."""
import zlib

import numpy as np
import pytest

from oracle import arroyo_oracle as O
from tests import test_gpu_window_time as W
from tests.test_gpu_updating_changes import BD_CAPB, crowded_keys

pytestmark = pytest.mark.gpu


def crowded_restarts(seed, keys, kind):
    """Two restarts, each while one pane holds every key in `keys`, then more rows of those keys."""
    st = W.Stream(seed, "many", 2 * W.SEC, W.SEC if kind != "tumbling" else None)
    o, s, rng, n = W._o(st.slide), st.slide, st.rng, len(keys)

    def batch(ks, panes):
        ks = np.asarray(ks, dtype=np.int64)
        ts = o + rng.choice(panes, len(ks)) * s + rng.integers(0, s, len(ks))
        st.events.append(("batch", O.Batch({"key": ks, "a": rng.integers(-1000, 1000, len(ks)), W.TS: ts})))

    batch(rng.permutation(keys), [0])
    batch(rng.choice(keys, n // 2), [0, 1])
    st.restart()
    # far enough that table "t" has expired panes 0 and 1 by the next checkpoint: a restore from it would bring them
    # back, a case the exact reference does not model (a restart there changes nothing)
    st.wm(o + 4 * s)
    batch(rng.permutation(keys), [5])
    batch(rng.choice(keys, n // 2), range(7))  # panes 0-3 are late by now
    st.wm(o + 5 * s)  # stats count a launch once a sync point took it back: the late rows above, before the restart
    st.restart()
    st.wm(o + 6 * s)
    batch(rng.choice(keys, 400), [6, 7])
    return st.end()


# (window kind, plan): tumbling, sliding with a running window, sliding re-merged
KINDS = [("tumbling", "minmax"), ("running", "ints"), ("remerge", "minmax")]
CASES = [(kind, plan, entry, n) for kind, plan in KINDS for entry in ("two_pass", "one_pass") for n in (1300, 3000)]


@pytest.mark.parametrize("kind,plan,entry,n", CASES, ids=[f"{k}-{e}-{n}" for k, _, e, n in CASES])
def test_restore_crowded_bucket(kind, plan, entry, n):
    keys = crowded_keys(n)
    assert n > BD_CAPB
    st = crowded_restarts(zlib.crc32(f"{kind}/{entry}/{n}".encode()), keys, kind)
    cfg = W.config(st, kind, plan)
    want, late = W.reference(st, cfg)
    got, rows_in, rows_late, n_keys = W.run_gpu(st, kind, cfg, entry)
    W.check_emissions(want, got, cfg, f"{kind}/{entry}/{n}")
    assert rows_in == sum(ev[1].num_rows for ev in st.events if ev[0] == "batch")
    assert rows_late == late
    assert n_keys == n
