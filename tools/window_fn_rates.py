"""Emission time of the window function (WindowFunction) behind the sliding aggregate, timed on one GPU.

The sliding aggregate has the benchmark's sliding shape (SUM and AVG of an Int64 value over 2^20 keys, 10 s window,
1 s slide, one row per key per slide).  Each slide's window goes device-resident (handle_watermark_device) into two
window functions, ROW_NUMBER() OVER (PARTITION BY window ORDER BY sum DESC, key DESC) with top_n = 1 and with
top_n = 0 (every row leaves).  Per slide, after warm-up:

  sliding_emit_ms   the sliding aggregate's device-resident emission of the slide
  wf_top1_ms        the window function's process_device_batch + handle_watermark with top_n = 1, host output included
  wf_all_ms         the same with top_n = 0 (2^20 rows leave to the host)

With --function F [G ...] more window functions take the same windows in the same slides, every row leaving to the
host.  An aggregate F (sum, count, avg, min or max) adds F(s) OVER (PARTITION BY window) and the running F(s) OVER
(PARTITION BY window ORDER BY s DESC):

  wf_F_window_ms    F over the whole window
  wf_F_running_ms   F over the default frame of ORDER BY s DESC

A value function F (lag, lead, first_value, last_value or nth_value) adds F(s) OVER (PARTITION BY window ORDER BY s
DESC, key DESC), with lag / lead's offset 1 and nth_value's n 2, and percent_rank or cume_dist adds F() over the same:

  wf_F_ms           F over the ordered window

With --frame the same slides also take explicit frames, beside the default-frame SUM and MIN above (added when not
asked for):

  wf_sum_rows_ms    SUM(s) OVER (PARTITION BY window ORDER BY s DESC ROWS BETWEEN 100 PRECEDING AND 100 FOLLOWING)
  wf_min_rows_ms    MIN(s) over the same frame
  wf_sum_range_ms   SUM(s) OVER (... ORDER BY s DESC RANGE BETWEEN 1000 PRECEDING AND 1000 FOLLOWING)
  wf_sum_range_ts_ms  SUM(s) OVER (... ORDER BY _timestamp RANGE BETWEEN 1 s PRECEDING AND CURRENT ROW), which
                    holds the whole window, as every row of a window carries its one _timestamp
  wf_sum_groups_ms  SUM(s) OVER (... ORDER BY s DESC GROUPS BETWEEN 5 PRECEDING AND 5 FOLLOWING)

and --instant-rows N times every window function once more on one instant of N rows (s uniform in [-2^20, 2^20),
one device batch, then the watermark past it): instant_W_ms.

Each is timed with CUDA events on the operators' stream around the calls (every handle_watermark ends in a stream
synchronise); the medians are reported, with the sorted rows per second of each window function.  Prints one JSON
line with the card's name and power limit.

    python tools/window_fn_rates.py [--scale S] [--slides K] [--function F [G ...]] [--frame] [--instant-rows N]

--scale S divides the key count by 2^S (a quick rehearsal of the script)."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SEC = 1_000_000_000
T0 = 1_700_000_000 * SEC
TS = "_timestamp"
AGGREGATES = ["sum", "count", "avg", "min", "max"]
ORDERED = ["lag", "lead", "first_value", "last_value", "nth_value", "percent_rank", "cume_dist"]


def card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        limit = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader"],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        limit = "unknown"
    return {"gpu": name, "power_limit": limit}


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--scale", type=int, default=0, help="divide the key count by 2^S (0..16)")
    ap.add_argument("--slides", type=int, default=20, help="timed slides after the 12 warm-up slides")
    ap.add_argument("--function", nargs="+", default=["row_number"], choices=["row_number", *AGGREGATES, *ORDERED],
                    help="also time F(s) OVER (PARTITION BY window [ORDER BY s DESC]) for an aggregate, or F over "
                         "(PARTITION BY window ORDER BY s DESC, key DESC) for the other functions")
    ap.add_argument("--frame", action="store_true", help="also time ROWS / RANGE / GROUPS frames")
    ap.add_argument("--instant-rows", type=int, default=0, help="also time one instant of N rows")
    a = ap.parse_args()
    if not 0 <= a.scale <= 16 or a.slides < 1:
        ap.error("--scale must be in [0, 16] and --slides >= 1")
    import pyarrow as pa
    import torch

    import arroyo_b200 as ab
    from arroyo_b200 import config, operators as native
    if not torch.cuda.is_available():
        raise SystemExit("window_fn_rates needs a CUDA device")
    keys = 1 << (20 - a.scale)
    stream = torch.cuda.Stream()
    ts_t = pa.timestamp("ns")
    s_cfg = config.WindowAggConfig(width=10 * SEC, slide=SEC, key_names=["key"],
                                   aggs=[config.Agg("sum", "v", "s"), config.Agg("avg", "v", "av")], window_index=1)
    sliding = native.SlidingAggregatingWindowFunc(
        s_cfg, input_schema=pa.schema([("key", pa.int64()), ("v", pa.int64()), (TS, ts_t)]), expected_keys=keys,
        stream=stream.cuda_stream)
    w_schema = pa.schema([("key", pa.int64()), ("window_start", ts_t), ("window_end", ts_t), ("s", pa.int64()),
                          ("av", pa.float64()), (TS, ts_t)])
    cfgs = {what: config.WindowFunctionConfig("row_number", None, [("s", True), ("key", True)], "rn", top_n)
            for what, top_n in (("top1", 1), ("all", 0))}
    if a.frame:
        a.function += [f for f in ("sum", "min") if f not in a.function]
    for f in a.function:
        if f in AGGREGATES:
            for what, order_by in (("window", []), ("running", [("s", True)])):
                cfgs[f"{f}_{what}"] = config.WindowFunctionConfig(f, None, order_by, "f", argument="s")
        elif f in ORDERED:
            cfgs[f] = config.WindowFunctionConfig(f, None, [("s", True), ("key", True)], "f",
                                                  argument=None if f in ("percent_rank", "cume_dist") else "s",
                                                  offset=2 if f == "nth_value" else 1)
    if a.frame:
        s_desc = [("s", True)]
        for what, f, order_by, frame in (
                ("sum_rows", "sum", s_desc, ("rows", ("preceding", 100), ("following", 100))),
                ("min_rows", "min", s_desc, ("rows", ("preceding", 100), ("following", 100))),
                ("sum_range", "sum", s_desc, ("range", ("preceding", 1000), ("following", 1000))),
                ("sum_range_ts", "sum", [(TS, False)], ("range", ("preceding", SEC), "current_row")),
                ("sum_groups", "sum", s_desc, ("groups", ("preceding", 5), ("following", 5)))):
            cfgs[what] = config.WindowFunctionConfig(f, None, order_by, "f", argument="s",
                                                     frame=config.WindowFrame(*frame))
    fns = {what: native.WindowFunction(c, input_schema=w_schema, stream=stream.cuda_stream) for what, c in cfgs.items()}
    ctxs = {w: ab.OperatorContext(1) for w in fns}
    rng = np.random.default_rng(7)
    warm = 12
    times = {"sliding_emit_ms": [], **{f"wf_{w}_ms": [] for w in fns}}
    rows_out = {w: 0 for w in fns}
    window_rows = []

    def timed(f):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        r = f()
        e1.record(stream)
        e1.synchronize()
        return r, e0.elapsed_time(e1)

    with torch.cuda.stream(stream):
        for step in range(warm + a.slides):
            k = torch.from_numpy(rng.permutation(keys).astype(np.int64)).cuda()
            v = torch.from_numpy(rng.integers(-1000, 1000, keys).astype(np.int64)).cuda()
            ts = torch.from_numpy(T0 + step * SEC + rng.integers(0, SEC, keys).astype(np.int64)).cuda()
            stream.synchronize()
            sliding.process_device_batch([k.data_ptr(), v.data_ptr(), ts.data_ptr()], keys)
            wm = T0 + step * SEC
            wins, t_s = timed(lambda: sliding.handle_watermark_device(wm))
            n_rows = sum(n for n, _ in wins)
            for what, op in fns.items():
                def call():
                    for n, ptrs in wins:
                        op.process_device_batch(ptrs, n)
                    col = ab.Collector()
                    ctxs[what].watermarks.set(0, wm)
                    op.handle_watermark(wm, ctxs[what], col)
                    return sum(b.num_rows for b in col.batches)
                out, t_w = timed(call)
                if step >= warm:
                    times[f"wf_{what}_ms"].append(t_w)
                    rows_out[what] += out
            if step >= warm:
                times["sliding_emit_ms"].append(t_s)
                window_rows.append(n_rows)
    if a.instant_rows:
        n = a.instant_rows
        cols = [torch.arange(n, dtype=torch.int64, device="cuda"), torch.zeros(n, dtype=torch.int64, device="cuda"),
                torch.zeros(n, dtype=torch.int64, device="cuda"),
                torch.from_numpy(rng.integers(-(1 << 20), 1 << 20, n).astype(np.int64)).cuda(),
                torch.zeros(n, dtype=torch.int64, device="cuda"), torch.zeros(n, dtype=torch.int64, device="cuda")]
        with torch.cuda.stream(stream):
            for what, op in fns.items():
                for rep in range(6):
                    wm = T0 + (warm + a.slides + rep) * SEC
                    cols[5].fill_(wm - 1)
                    stream.synchronize()

                    def call():
                        op.process_device_batch([c.data_ptr() for c in cols], n)
                        col = ab.Collector()
                        ctxs[what].watermarks.set(0, wm)
                        op.handle_watermark(wm, ctxs[what], col)
                        return sum(b.num_rows for b in col.batches)
                    _, t = timed(call)
                    if rep >= 2:
                        times.setdefault(f"instant_{what}_ms", []).append(t)
    med = {k: float(np.median(v)) for k, v in times.items()}
    rows = float(np.median(window_rows))
    res = {**card(), "keys": keys, "slides": a.slides, "window_rows": int(rows), "instant_rows": a.instant_rows,
           **{k: round(v, 3) for k, v in med.items()},
           **{f"wf_{w}_sorted_rows_per_s": round(rows / (med[f"wf_{w}_ms"] / 1e3)) for w in fns},
           **{f"rows_out_{w}": rows_out[w] for w in fns}}
    print(json.dumps(res), flush=True)
    sliding.close()
    for op in fns.values():
        op.close()


if __name__ == "__main__":
    main()
