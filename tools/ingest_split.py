#!/usr/bin/env python
"""tools/ingest_split.py -- where a step of bench.py's headline workload goes, kernel by kernel.

Drives the operator exactly as bench.py's device-resident loop does (same generator, batch lists, warm-up rule and
FLAG_PROFILE; the helpers are bench.py's own) under torch.profiler with CUDA activities, and prints one JSON line:

  per step (median over the timed steps): part_kernel (pass 1 of the two-pass ingest), agg_kernel (pass 2),
  emit_kernel (the window emission) and everything else on the operator's stream;
  each pass's algorithmic bytes per row (pass 1: 24 read + 16 written; pass 2: 16 read back) and the GB/s they imply;
  the idle gap per step between the end of the ingest and the start of the emission (the host's wait on the ingest
  at the watermark);
  the card's name, power limit and maximum SM clock (nvidia-smi, read only).

Takes bench.py's options (--steps, --warmup, --dist, --keyspace, ...).  A step starts with its first ingest launch.
Writes nothing into the tree (the trace goes to a temporary directory).
"""
import json
import os
import statistics
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench as B  # noqa: E402

BYTES_PER_ROW = {"part_kernel": {"read": 24, "written": 16}, "agg_kernel": {"read": 16, "written": 0}}
KERNELS = ("part_kernel", "agg_kernel", "emit_kernel")


def card(index):
    try:
        out = subprocess.run(["nvidia-smi", f"--id={index}", "--query-gpu=name,power.limit,clocks.max.sm",
                              "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
        name, power, clock = [x.strip() for x in out.split(",")]
        return {"name": name, "power_limit": power, "clocks_max_sm": clock}
    except Exception as e:  # noqa: BLE001
        return {"name": None, "error": f"{type(e).__name__}: {e}"}


def kind(name):
    for k in KERNELS:
        if k + "<" in name:
            return k
    return "other"


def split(trace, W, K):
    """Per-step medians from a chrome trace of W warm-up + K timed steps."""
    ev = [e for e in trace["traceEvents"] if e.get("ph") == "X" and e.get("cat") in ("kernel", "gpu_memcpy", "gpu_memset")]
    parts = sorted((e for e in ev if kind(e["name"]) == "part_kernel"), key=lambda e: e["ts"])
    if not parts:
        raise RuntimeError("no part_kernel in the trace: the two-pass ingest did not run")
    stream = parts[0]["args"].get("stream")
    ev = sorted((e for e in ev if e["args"].get("stream") == stream), key=lambda e: e["ts"])
    per_step = max(1, len(parts) // (W + K))  # ingest launches per step
    starts = [e["ts"] for e in parts[-K * per_step::per_step]]
    bounds = starts + [float("inf")]
    steps = [{"part_kernel": 0.0, "agg_kernel": 0.0, "emit_kernel": 0.0, "other": 0.0, "gap": None} for _ in starts]
    last_agg_end = None
    for e in ev:
        if e["ts"] < starts[0]:
            continue
        i = max(j for j in range(len(starts)) if bounds[j] <= e["ts"])
        k = kind(e["name"])
        steps[i][k] += e["dur"]
        if k == "agg_kernel":
            last_agg_end = e["ts"] + e["dur"]
        elif k == "emit_kernel" and last_agg_end is not None:
            steps[i]["gap"] = (steps[i]["gap"] or 0.0) + max(0.0, e["ts"] - last_agg_end)
            last_agg_end = None  # the emission's later kernels are not a new gap
    med = {k: statistics.median(s[k] for s in steps) / 1e3 for k in ("part_kernel", "agg_kernel", "emit_kernel", "other")}
    gaps = [s["gap"] for s in steps if s["gap"] is not None]
    med["ingest_to_emit_gap"] = statistics.median(gaps) / 1e3 if gaps else None
    return med, per_step, len(steps)


def main():
    args = B.parse()
    import torch
    from torch.profiler import ProfilerActivity, profile

    from arroyo_b200 import ffi, operators as native

    if ffi.load().arroyo_b200_device_count() < 1:
        raise RuntimeError("ingest_split.py needs a CUDA device")
    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    device = torch.device("cuda", local)
    torch.cuda.set_stream(torch.cuda.Stream(device=device, priority=-1))  # as bench.py's run_ours
    W, K = B.steady_warmup(args.warmup), args.steps
    rows = args.rows_per_pane
    gen_pane = B.make_generator(torch, device, rows, args.keys, args.dist, 42, args.keyspace)
    panes = [gen_pane(p) for p in range(W + K)]
    torch.cuda.synchronize()
    with tempfile.TemporaryDirectory() as tmp:
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            ms, d, _, _, _ = B.device_resident(args, torch, native, ffi, local, panes, W, K, rows)
        path = os.path.join(tmp, "trace.json")
        prof.export_chrome_trace(path)
        with open(path) as f:
            trace = json.load(f)
    med, per_step, n_steps = split(trace, W, K)
    rows_per_step = d["ingest_rows_timed"] / K
    kernels = {}
    for k in KERNELS + ("other",):
        kernels[k] = {"ms_per_step": round(med[k], 4)}
        if k in BYTES_PER_ROW:
            b = BYTES_PER_ROW[k]
            kernels[k].update({"bytes_per_row": b, "gbs": round((b["read"] + b["written"]) * rows_per_step / (med[k] * 1e-3)
                                                                / 1e9, 1) if med[k] else None})
    out = {"card": card(local), "steps": K, "warmup": W, "rows_per_step": rows_per_step, "dist": args.dist,
           "keyspace": args.keyspace, "ingest_launches_per_step": per_step, "steps_split": n_steps,
           "kernels": kernels,
           "ingest_to_emit_gap_ms_per_step": round(med["ingest_to_emit_gap"], 4) if med["ingest_to_emit_gap"] else None,
           "ms_per_step_profiled": round(ms / K, 4),
           "note": "medians over the timed steps; times from torch.profiler (CUPTI), so the step time is not bench.py's"}
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
