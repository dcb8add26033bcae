"""Host-side pieces of `bench.py --workload join | session` (bench_workloads.py) that need no GPU: the column checksum
both sides of the verification use, the identity Shuffle edge of a one-subtask job, and the CPU baselines (the C
restatements of the join / session operators on key-partitioned subtasks) at toy sizes.  The GPU plans themselves run
through `python bench.py --workload join` and `--workload session` on a GPU."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import bench_workloads as BW  # noqa: E402


def test_numpy_checksum_is_the_wrapping_i64_sum_the_device_side_computes():
    rng = np.random.default_rng(0)
    cols = [rng.integers(-2**63, 2**63 - 1, 1000, dtype=np.int64) for _ in range(9)]
    want = 0
    for c, col in enumerate(cols):
        for v in col.tolist():
            want += v * BW.MULT[c % len(BW.MULT)]
    assert BW._np_checksum(np, cols) == BW._i64(want)
    # torch multiplies and sums int64 with the same wrap-around
    import torch
    acc = torch.zeros((), dtype=torch.int64)
    for c, col in enumerate(cols):
        acc = acc + (torch.from_numpy(col) * BW._i64(BW.MULT[c % len(BW.MULT)])).sum()
    assert int(acc.item()) == BW._i64(want)


def test_one_subtask_edge_forwards_rows_and_reports_each_new_watermark_once():
    e = BW.Edge(None, None, 0, 1, 0, 0, 3, 0, 1 << 10)
    assert e.round([1, 2, 3], 5, 100) == ([([1, 2, 3], 5)], 100)
    assert e.round([1, 2, 3], 5, 100) == ([([1, 2, 3], 5)], None)
    assert e.round(None, 0, 200) == ([], 200)
    assert e.round([4, 5, 6], 1, None) == ([([4, 5, 6], 1)], None)
    e.close()


def test_cpu_baselines_of_the_join_and_session_workloads_run_at_toy_sizes():
    v, threads, sample = BW.cpu_join(1 << 10, 1 << 12, 2, budget_s=30.0)
    assert v > 0 and threads >= 1 and "persons" in sample
    v, threads, sample = BW.cpu_session(2000, 1 << 12, 2, budget_s=30.0)
    assert v > 0 and threads >= 1 and "keys" in sample
