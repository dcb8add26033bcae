"""Ingest rate and emission time of the instant-window aggregate (InstantAggregatingWindowFunc) on three input shapes,
timed on one GPU:

  q5       2^24 rows, 2^20 keys in one instant    (MAX(num) GROUP BY key of one upstream window)
  hot      2^24 rows in one unkeyed instant       (q5's MaxBids: every row of the window in one group)
  session  2^22 rows in 2^22 distinct instants    (behind a session window: every session ends at its own time)

The rows are device-resident (process_device_batch, the path a GPU upstream window feeds).  Ingest is timed with CUDA
events on the operator's stream; the emission is the wall time of one handle_watermark that releases everything,
host output included.  Prints one JSON line per shape plus the card's name and power limit.

    python tools/instant_rates.py [--scale S] [--reps R]

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

SEC = 1_000_000_000
T0 = 1_700_000_000 * SEC


def card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        limit = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader"],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        limit = "unknown"
    return {"gpu": name, "power_limit": limit}


def shapes(scale):
    rng = np.random.default_rng(1)
    n24, n22, n20 = 1 << (24 - scale), 1 << (22 - scale), 1 << (20 - scale)
    t = T0 + 10 * SEC - 1
    yield "q5", True, {"key": rng.integers(0, n20, n24).astype(np.int64),
                       "num": rng.integers(0, 1000, n24).astype(np.int64), "_timestamp": np.full(n24, t, np.int64)}
    yield "hot", False, {"num": rng.integers(0, 1000, n24).astype(np.int64), "_timestamp": np.full(n24, t, np.int64)}
    yield "session", False, {"num": rng.integers(0, 1000, n22).astype(np.int64),
                             "_timestamp": T0 + rng.permutation(n22).astype(np.int64) * 1000}


def run(name, keyed, cols, reps):
    import pyarrow as pa
    import torch

    import arroyo_b200 as ab
    from arroyo_b200 import config, operators as native
    stream = torch.cuda.Stream()
    names = list(cols)
    dev = [torch.from_numpy(cols[c]).cuda() for c in names]
    schema = pa.schema([(c, pa.timestamp("ns") if c == "_timestamp" else pa.int64()) for c in names])
    cfg = config.WindowAggConfig(width=0, key_names=["key"] if keyed else [], aggs=[config.Agg("max", "num", "m")],
                                 final_projection=False)
    n = len(cols["_timestamp"])
    wm = int(cols["_timestamp"].max()) + 1
    ingest_ms, emit_ms = [], []
    for r in range(reps + 1):  # the first run warms up
        op = native.InstantAggregatingWindowFunc(cfg, input_schema=schema, stream=stream.cuda_stream)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        with torch.cuda.stream(stream):
            e0.record(stream)
            op.process_device_batch([t.data_ptr() for t in dev], n)
            e1.record(stream)
        e1.synchronize()
        ctx, col = ab.OperatorContext(1), ab.Collector()
        ctx.watermarks.set(0, wm)
        t0 = time.perf_counter()
        op.handle_watermark(wm, ctx, col)
        t1 = time.perf_counter()
        out = sum(b.num_rows for b in col.batches)
        s = op.stats()
        op.close()
        if r:
            ingest_ms.append(e0.elapsed_time(e1))
            emit_ms.append((t1 - t0) * 1e3)
    med_i, med_e = float(np.median(ingest_ms)), float(np.median(emit_ms))
    return {"shape": name, "rows": n, "groups_out": out, "instants_out": s["windows_out"], "reps": reps,
            "ingest_ms": round(med_i, 3), "ingest_rows_per_s": round(n / (med_i / 1e3)),
            "emit_ms_per_watermark": round(med_e, 3)}


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--scale", type=int, default=0, help="divide row and key counts by 2^S (0..16)")
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    if not 0 <= a.scale <= 16 or a.reps < 1:
        ap.error("--scale must be in [0, 16] and --reps >= 1")
    print(json.dumps(card()))
    for name, keyed, cols in shapes(a.scale):
        print(json.dumps(run(name, keyed, cols, a.reps)), flush=True)


if __name__ == "__main__":
    main()
