"""Times of the updating aggregate's state path on one GPU (csrc/updating_agg.cu), for DESIGN.md section 6.

* flush of 2^20 touched keys, with and without the per-key "flushed since the last export" store, alternated in one
  run: the library without the store is linked into a temporary directory from the in-tree objects and
  updating_agg.cu compiled with -DAB_UPDATING_NO_FLUSH_MARK (run build() first);
* export (arroyo_b200_op_checkpoint_state) of 2^20 and 2^24 keys with a five-aggregate plan (COUNT, SUM, AVG, MIN, MAX);
* restore (on_start) of the same tables into an operator created with expected_keys = 256.

Kernel times come from torch.profiler (CUDA activities), call times from a host clock around calls that end in a
device synchronise.  Prints one JSON object with the GPU's name and power limit.

    python tools/updating_state_rates.py > updating_state_rates.json
"""
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

T0 = 1_700_000_000_000_000_000


def gpu_info():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    return out[0] if out else "unknown"


def variant_library(tmp):
    """libarroyo_b200 with the flush kernel built without its marking store."""
    from arroyo_b200 import build, ffi
    objs = [os.path.join(build.HERE, "build", s.replace(".cu", ".o")) for s in build.SOURCES if s != "updating_agg.cu"]
    for o in objs:
        if not os.path.exists(o):
            raise SystemExit(f"{o} is missing: run build() first")
    o = os.path.join(tmp, "updating_agg_nomark.o")
    flags = [*build.GENCODE, "-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC,-Wall,-Wno-unused-function",
             "--expt-relaxed-constexpr", "-DAB_UPDATING_NO_FLUSH_MARK"]
    subprocess.run([build.nvcc_path(), *flags, "-c", os.path.join(build.CSRC, "updating_agg.cu"), "-o", o], check=True)
    lib_path = os.path.join(tmp, "libarroyo_b200_nomark.so")
    subprocess.run([build.nvcc_path(), *build.GENCODE, "-shared", "-o", lib_path, *objs, o, "-lcudart"], check=True)
    lib = C.CDLL(lib_path)
    for name, res, args in ffi.SYMBOLS:
        fn = getattr(lib, name)
        fn.restype, fn.argtypes = res, args
    return lib


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
    aggs = [A("count", None, "n"), A("sum", "a", "s"), A("avg", "a", "av"), A("min", "a", "mn"), A("max", "a", "mx")]
    cfg = U.UpdatingAggConfig(["k"], aggs)
    schema = pa.schema([("k", pa.int64()), ("a", pa.int64()), ("_timestamp", pa.timestamp("ns"))])

    def make(lib=None, expected_keys=0):
        op = native.UpdatingAggregatingFunc(cfg, expected_keys=expected_keys)
        if lib is not None:
            op._lib = lib
        op._build(schema.names)
        op._note_key_type(schema)
        return op

    def cols(n, seed):
        g = torch.Generator(device="cuda").manual_seed(seed)
        k = torch.randperm(n, device="cuda", generator=g).to(torch.int64) * 7919 + 11
        a = torch.randint(-10**6, 10**6, (n,), device="cuda", generator=g, dtype=torch.int64)
        ts = torch.full((n,), T0 + seed, device="cuda", dtype=torch.int64)
        torch.cuda.synchronize()
        return [k, a, ts]

    def feed(op, c):
        op.process_device_batch([t.data_ptr() for t in c], c[0].numel())

    def kernel_ms(prof, name):
        ev = sorted([e for e in prof.events() if e.device_type.name == "CUDA" and name in e.name],
                    key=lambda e: e.time_range.start)
        return [e.device_time / 1000.0 for e in ev]

    out = {"gpu": gpu_info(), "torch": torch.__version__}
    ctx = ab.OperatorContext(1)

    # ---- flush with and without the marking store, alternated ----
    n, reps = 1 << 20, 20
    with tempfile.TemporaryDirectory() as tmp:
        nomark = variant_library(tmp)
        ops = [make(None, n), make(nomark, n)]  # 0: with the store, 1: without
        data = [cols(n, s) for s in range(2)]
        for op in ops:  # warm-up: every key exists, the output buffers are sized
            feed(op, data[0])
            op.handle_tick(0, ctx, ab.Collector())
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for r in range(reps):
                for op in ops:
                    feed(op, data[r % 2])
                    op.handle_tick(0, ctx, ab.Collector())
                    torch.cuda.synchronize()
        t = kernel_ms(prof, "upd_flush_kernel")
        assert len(t) == 2 * reps, len(t)
        with_store, without = t[0::2], t[1::2]
        out["flush_2^20"] = {"with_store_ms": float(np.median(with_store)), "without_store_ms": float(np.median(without)),
                             "with_store_all": with_store, "without_store_all": without}
        for op in ops:
            op.close()

    # ---- export and restore ----
    for log2 in (20, 24):
        n = 1 << log2
        op = make(None, n)
        feed(op, cols(n, 5))
        op.handle_tick(0, ctx, ab.Collector())
        table = ab.context.KeyValueTable()
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            t0 = time.perf_counter()
            op.checkpoint_state(table)
            export_call = (time.perf_counter() - t0) * 1000
        export_kernel = kernel_ms(prof, "upd_export_kernel")
        assert sum(b.num_rows for b in table.batches) == n
        op.close()
        rctx = ab.OperatorContext(1)
        for b in table.batches:
            rctx.key_value_table("a").insert_batch(b)
        op = make(None, 256)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            t0 = time.perf_counter()
            op.on_start(rctx)
            restore_call = (time.perf_counter() - t0) * 1000
        restore_kernels = {k: sum(kernel_ms(prof, k)) for k in ("bd_place_kernel", "upd_restore_gen_kernel",
                                                                 "upd_restore_pos_kernel", "upd_restore_seed_kernel")}
        assert op.stats()["n_keys"] == n
        op.close()
        out[f"state_2^{log2}"] = {"export_call_ms": export_call, "export_kernel_ms": sum(export_kernel),
                                  "restore_call_ms": restore_call, "restore_kernels_ms": restore_kernels}
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
