"""Times of the updating aggregate's time-to-idle path on one GPU (csrc/updating_agg.cu), for DESIGN.md section 6.

* upd_ingest_kernel at 2^24 rows without a ttl (the TTL = false instance) and with one (the stamping instance),
  alternated in one run, over 2^20 uniform keys and with one hot key taking 75 % of the rows;
* the expiry pass (upd_expire_kernel) over 2^20 and 2^24 ids with 0 %, 50 % and 100 % of them expiring;
* one compaction of a 2^24-id dictionary whose keys all expired: checkpoint_state, which writes the tombstones and
  then rebuilds the dictionary (upd_keep_kernel, bd_gather_kernel, bd_place_kernel, bd_map_kernel,
  upd_permute_kernel).

Kernel times come from torch.profiler (CUDA activities), call times from a host clock around calls that end in a
device synchronise.  Prints one JSON object with the GPU's name and power limit.

    python tools/updating_ttl_rates.py > updating_ttl_rates.json
"""
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

T0 = 1_700_000_000_000_000_000
TTL = 10 ** 9


def gpu_info():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    return out[0] if out else "unknown"


def main():
    import numpy as np
    import pyarrow as pa
    import torch
    from torch.profiler import ProfilerActivity, profile

    import arroyo_b200 as ab
    from arroyo_b200 import operators as native
    from oracle import arroyo_oracle as O
    from oracle import updating_oracle as U

    A = O.Agg
    aggs = [A("count", None, "n"), A("sum", "a", "s"), A("min", "a", "mn"), A("max", "a", "mx")]
    cfg = U.UpdatingAggConfig(["k"], aggs)
    schema = pa.schema([("k", pa.int64()), ("a", pa.int64()), ("_timestamp", pa.timestamp("ns"))])
    clock = [0]

    def make(ttl, expected_keys):
        return native.UpdatingAggregatingFunc(cfg, input_schema=schema, expected_keys=expected_keys, ttl=ttl,
                                              clock=lambda: clock[0])

    def feed(op, c):
        op.process_device_batch([t.data_ptr() for t in c], c[0].numel())

    def cols(k, seed):
        g = torch.Generator(device="cuda").manual_seed(seed)
        a = torch.randint(-10**6, 10**6, (k.numel(),), device="cuda", generator=g, dtype=torch.int64)
        ts = torch.full((k.numel(),), T0 + seed, device="cuda", dtype=torch.int64)
        torch.cuda.synchronize()
        return [k, a, ts]

    def kernel_ms(prof, name):
        ev = sorted([e for e in prof.events() if e.device_type.name == "CUDA" and name in e.name],
                    key=lambda e: e.time_range.start)
        return [e.device_time / 1000.0 for e in ev]

    out = {"gpu": gpu_info(), "torch": torch.__version__}
    ctx = ab.OperatorContext(1)
    g = torch.Generator(device="cuda").manual_seed(1)

    # ---- ingest: no ttl against the stamping path, alternated ----
    n, nk, reps = 1 << 24, 1 << 20, 10
    uniform = torch.randint(0, nk, (n,), device="cuda", generator=g, dtype=torch.int64) * 7919 + 11
    hot = torch.where(torch.rand(n, device="cuda", generator=g) < 0.75, torch.full_like(uniform, 5), uniform)
    for name, keys in (("uniform_2^20", uniform), ("hot_75pct", hot)):
        data = cols(keys, 3)
        ops = [make(None, nk), make(TTL, nk)]
        for op in ops:  # warm-up: every key exists
            feed(op, data)
            op.handle_tick(0, ctx, ab.Collector())
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for r in range(reps):
                for op in ops:
                    clock[0] += 1  # the stamping path stores on every id's first row of a call
                    feed(op, data)
                    torch.cuda.synchronize()
        t = kernel_ms(prof, "upd_ingest_kernel")
        assert len(t) == 2 * reps, len(t)
        out[f"ingest_2^24_{name}"] = {"no_ttl_ms": float(np.median(t[0::2])), "ttl_ms": float(np.median(t[1::2])),
                                      "no_ttl_all": t[0::2], "ttl_all": t[1::2]}
        for op in ops:
            op.close()
    del uniform, hot

    # ---- the expiry pass: half the keys stamped at 0, half at TTL / 2 ----
    for log2 in (20, 24):
        n = 1 << log2
        keys = torch.randperm(n, device="cuda", generator=g).to(torch.int64) * 7919 + 11
        for pct, at in ((0, TTL // 2 + TTL // 4), (50, TTL), (100, 2 * TTL)):
            clock[0] = 0
            op = make(TTL, n)
            feed(op, cols(keys[: n // 2].contiguous(), 1))
            clock[0] = TTL // 2
            feed(op, cols(keys[n // 2:].contiguous(), 2))
            op.handle_tick(0, ctx, ab.Collector())  # every key flushed, none idle for a ttl yet
            clock[0] = at
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                t0 = time.perf_counter()
                col = ab.Collector()
                op.handle_tick(0, ctx, col)
                call = (time.perf_counter() - t0) * 1000
            assert sum(b.num_rows for b in col.batches) == n * pct // 100
            rec = {"expire_kernel_ms": sum(kernel_ms(prof, "upd_expire_kernel")), "tick_call_ms": call}
            if log2 == 24 and pct == 100:  # ---- one compaction of 2^24 ids ----
                table = ab.context.KeyValueTable()
                torch.cuda.synchronize()
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    t0 = time.perf_counter()
                    op.checkpoint_state(table)
                    call = (time.perf_counter() - t0) * 1000
                assert sum(b.num_rows for b in table.batches) == n and op.stats()["n_keys"] == 0
                names = ("upd_export_kernel", "upd_keep_kernel", "bd_gather_kernel", "bd_place_kernel",
                         "bd_map_kernel", "bd_fill_keys_kernel", "bd_init_kernel", "upd_init_kernel",
                         "upd_permute_kernel")
                out["compaction_2^24"] = {"checkpoint_state_call_ms": call,
                                          "kernels_ms": {k: sum(kernel_ms(prof, k)) for k in names}}
            op.close()
            out[f"expire_2^{log2}_{pct}pct"] = rec
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
