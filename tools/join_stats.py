"""What the instant join and the join with expiration compute for fixed seeded streams, one JSON line per run: digests
of every output (column names, Arrow types, nullability, validity bits and values) and every field of stats().  `out`
sorts the rows of each batch, `order` keeps them as emitted.  Two builds of the library behave alike on these streams
when `out` and the counters of stats() match; `order` and the wall-clock fields (`*_ms`) may differ between two runs
of one build.

The runs are the shapes and entry points of tests/test_gpu_joins.py: every instant join case under inner, left, right
and full joins (host, sliced, 4-input, device and mixed input; device output for inner joins), every expiring join
case, and one expiring join restored from half of its stream that takes the rest through process_batch_emit and,
for its last batches, through process_batch.

    python tools/join_stats.py [--root DIR] > stats.jsonl

`--root DIR` imports arroyo_b200, and so its library, from the checkout at DIR.  Needs a GPU."""
import argparse
import hashlib
import json
import os
import sys
import zlib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def digest(outs, ordered):
    """sha256 over a run's outputs: lists of host RecordBatches or tests.exact_reference.Rows (device output).  Without
    `ordered` the rows of each batch are sorted first: which of a key's matches comes first follows the kernels' atomics
    and so varies from run to run."""
    import numpy as np
    h = hashlib.sha256()
    for out in outs:
        h.update(b"|")
        if hasattr(out, "vals"):
            mats = [(repr(out.names), np.ascontiguousarray(out.vals, np.uint64), np.ones(out.vals.shape, np.uint64))]
        else:
            mats = []
            for rb in out:
                vals, valid = [], []
                head = str(rb.schema) + str(rb.num_rows)
                for f, arr in zip(rb.schema, rb.columns):
                    bits, data = arr.buffers()
                    n, o = len(arr), arr.offset
                    head += f"{f.nullable}/{arr.null_count}/{bits is None}"
                    vals.append(np.frombuffer(data, np.uint64, count=o + n)[o:])
                    valid.append(np.ones(n, np.uint64) if bits is None else
                                 np.unpackbits(np.frombuffer(bits, np.uint8), bitorder="little")[o:o + n].astype(np.uint64))
                mats.append((head, np.stack(vals, axis=1), np.stack(valid, axis=1)))
        for head, vals, valid in mats:
            rows = np.concatenate([vals, valid], axis=1)
            if not ordered and len(rows):
                rows = rows[np.lexsort(rows.T[::-1])]
            h.update(head.encode() + np.ascontiguousarray(rows).tobytes())
    return h.hexdigest()[:16]


def restored_run(J):
    """An expiring join restored from the first half of a stream's batches, then fed the rest."""
    import numpy as np
    import arroyo_b200 as ab
    from arroyo_b200 import operators as native
    st = J.TSHAPES["rehash"](np.random.default_rng(5))
    cfg = ab.JoinConfig(left_on=[st.on[0]], right_on=[st.on[1]], join_type="inner")
    op = native.JoinWithExpiration(cfg, left_schema=J.arrow_schema(st.schemas[0]),
                                   right_schema=J.arrow_schema(st.schemas[1]))
    half = len(st.events) // 2
    for side in (0, 1):
        op._restore_side(side, [J.to_arrow(st.schemas[s], c) for s, c in st.events[:half] if s == side])
    ctx, outs = ab.OperatorContext(2), []
    for i, (side, cols) in enumerate(st.events[half:]):
        rb = J.to_arrow(st.schemas[side], cols)
        if i < len(st.events) - half - 4:
            col = ab.Collector()
            op.process_batch_index(side, 2, rb, ctx, col)
            outs.append(col.batches)
        else:
            op._process_batch(op._lib.arroyo_b200_op_process_batch, side, 2, rb)
    stats = op.stats()
    op.close()
    return outs, stats


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--root", default=ROOT)
    args = ap.parse_args()
    sys.path.insert(0, ROOT)  # the test helpers
    sys.path.insert(0, os.path.abspath(args.root))
    import numpy as np
    from tests import test_gpu_joins as J

    def line(what, outs, stats):
        print(json.dumps({"run": what, "out": digest(outs, False), "order": digest(outs, True), "stats": stats}),
              flush=True)

    for shape, entry in J.INSTANT_CASES:
        for join_type in J.JOIN_TYPES:
            st = J.SHAPES[shape](np.random.default_rng(zlib.crc32(shape.encode())))
            outs, stats, _ = J.run_instant(st, join_type, entry)
            line(f"instant/{shape}/{entry}/{join_type}", outs, stats)
    for shape, entry in J.EXPIRING_CASES:
        st = J.TSHAPES[shape](np.random.default_rng(zlib.crc32(shape.encode()) + 1))
        outs, stats = J.run_expiring(st, entry)
        line(f"expiring/{shape}/{entry}", outs, stats)
    line("expiring/restored", *restored_run(J))


if __name__ == "__main__":
    main()
