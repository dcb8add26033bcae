"""Restore cost of the join with expiration (arroyo_b200_op_restore_side) on two table shapes, timed on one GPU:

  uniform  2^24 rows per side, keys uniform over 2^20 values   (both tables restored, then a left batch probes)
  hot      2^22 rows on one key, table "left" only            (one chain: every row's link is an atomicExch on one
                                                                head; a right batch with one hot row probes it)

Per shape, three figures (medians over --reps fresh operators):
  device   the restore's host->device copies and `tj_link_kernel`, summed from a torch.profiler trace of a separate
           repetition (device time; CUDA activities only)
  call     host clock of the restore_side calls (export, checks, copies, link, the closing synchronisation)
  probe    host clock of the first 2^16-row batch that probes the restored side (process_batch_emit, pairs on the host)
Prints one JSON line per shape plus the card's name and power limit.

    python tools/ttl_join_restore_rates.py [--scale S] [--reps R]

--scale S divides every row and key count by 2^S (a quick rehearsal of the script)."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

T0 = 1_700_000_000 * 10 ** 9


def card():
    import torch
    try:
        limit = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader"],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        limit = "unknown"
    return {"gpu": torch.cuda.get_device_name(0), "power_limit": limit}


def table(rng, keys, name, n_batches):
    """The batches of one key-time table: [id, name, _timestamp], `len(keys)` rows in `n_batches` batches."""
    import pyarrow as pa
    out = []
    for i, part in enumerate(np.array_split(keys, n_batches)):
        n = len(part)
        out.append(pa.RecordBatch.from_arrays(
            [pa.array(part.astype(np.int64)), pa.array(rng.integers(0, 1 << 40, n)),
             pa.array(np.full(n, T0 + i, np.int64)).cast(pa.timestamp("ns"))], names=["id", name, "_timestamp"]))
    return out


def shapes(scale):
    rng = np.random.default_rng(1)
    n24, n22, n20, n16 = (1 << (b - scale) for b in (24, 22, 20, 16))
    left = table(rng, rng.integers(0, n20, n24), "a", 16)
    right = table(rng, rng.integers(0, n20, n24), "b", 16)
    probe = table(rng, rng.integers(0, n20, n16), "a", 1)[0]
    yield "uniform", {0: left, 1: right}, (0, probe)
    hot = table(rng, np.full(n22, 7), "a", 4)
    probe = table(rng, np.concatenate([[7], rng.integers(100, 100 + n20, n16 - 1)]), "b", 1)[0]
    yield "hot", {0: hot}, (1, probe)


def one(tables, probe, profile):
    import torch

    import arroyo_b200 as ab
    from arroyo_b200 import operators as native
    schema = [tables[0][0].schema, (tables.get(1) or [probe[1]])[0].schema]
    op = native.JoinWithExpiration(ab.JoinConfig(left_on=["id"], right_on=["id"]), left_schema=schema[0],
                                   right_schema=schema[1])
    res = {}
    if profile:
        from torch.profiler import ProfilerActivity, profile as prof
        with prof(activities=[ProfilerActivity.CUDA]) as p:
            for side, batches in tables.items():
                op._restore_side(side, batches)
            torch.cuda.synchronize()
        dev = 0.0
        for e in p.key_averages():
            if "tj_link" in e.key or "Memcpy HtoD" in e.key:
                dev += e.device_time_total
        res["device_ms"] = dev / 1000
    else:
        t = time.perf_counter()
        for side, batches in tables.items():
            op._restore_side(side, batches)
        res["call_ms"] = (time.perf_counter() - t) * 1000
        ctx, col = ab.OperatorContext(2), ab.Collector()
        t = time.perf_counter()
        op.process_batch_index(probe[0], 2, probe[1], ctx, col)
        res["probe_ms"] = (time.perf_counter() - t) * 1000
        res["pairs"] = sum(b.num_rows for b in col.batches)
    st = op.stats()
    assert st["rows_in"] == (0 if profile else probe[1].num_rows)
    op.close()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scale", type=int, default=0)
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    print(json.dumps(card()), flush=True)
    for name, tables, probe in shapes(a.scale):
        one(tables, probe, False)  # warm-up: module load, pinned pool, allocator
        runs = [one(tables, probe, False) for _ in range(a.reps)]
        dev = [one(tables, probe, True)["device_ms"] for _ in range(a.reps)]
        rows = sum(b.num_rows for bs in tables.values() for b in bs)
        print(json.dumps({"shape": name, "rows_restored": rows, "device_ms": round(float(np.median(dev)), 3),
                          "call_ms": round(float(np.median([r["call_ms"] for r in runs])), 3),
                          "probe_ms": round(float(np.median([r["probe_ms"] for r in runs])), 3),
                          "probe_pairs": runs[0]["pairs"]}), flush=True)


if __name__ == "__main__":
    main()
