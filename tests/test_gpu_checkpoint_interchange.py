"""Checkpoint compatibility with the CPU operators (SURVEY.md 8(f).1): the partial-state batches the CUDA operator
hands to the shim at a checkpoint are the batches the reference operator writes to table "t"
(sliding_aggregating_window.rs:693-737, tumbling :430-467; schema = partial_schema, builder.rs:163-192), so

  * the GPU's table contents equal the oracle's at the same point of the same stream (per pane timestamp, merged by
    key: the reference splits a pane's state over as many batches as it drained, which is not observable after the
    Final merge);
  * a checkpoint written by the oracle operator restores into the GPU operator, and
  * a checkpoint written by the GPU operator restores into the oracle operator,
    each continuing to the output of an uninterrupted run."""
import numpy as np
import pytest

from oracle import arroyo_oracle as O
from tests.test_gpu_agg_plans import PLANS
from tests.test_gpu_parity import S, assert_same, gen_multi_stream, gen_stream

pytestmark = pytest.mark.gpu

AGGS = [O.Agg("sum", "value", "sum"), O.Agg("avg", "value", "avg"), O.Agg("count", None, "count")]
SUM_ONLY = [O.Agg("sum", "value", "sum")]
MINMAX = [O.Agg("min", "value", "lo"), O.Agg("max", "value", "hi")]


def _cfg(kind, aggs):
    if kind == "sliding":
        return O.WindowAggConfig(width=4 * S, slide=S, key_names=["key"], aggs=aggs, window_index=1)
    return O.WindowAggConfig(width=2 * S, slide=2 * S, key_names=["key"], aggs=aggs, window_index=1)


def _oracle_cls(kind):
    return O.SlidingAggregatingWindowFunc if kind == "sliding" else O.TumblingAggregatingWindowFunc


def _native_cls(kind):
    from arroyo_b200 import operators as native
    return native.SlidingAggregatingWindowFunc if kind == "sliding" else native.TumblingAggregatingWindowFunc


def _merged(batches, key="key"):
    """One pane's state batches merged by key -> {key: tuple of state values} (sums add, min / max fold)."""
    out = {}
    for b in batches:
        names = [c for c in b.cols if c not in (key, O.TIMESTAMP)]
        for i in range(b.num_rows):
            k = int(b[key][i])
            vals = [b[c][i] for c in names]
            if k not in out:
                out[k] = dict(zip(names, vals))
                continue
            for c, v in zip(names, vals):
                if c.endswith("[min]"):
                    out[k][c] = min(out[k][c], v)
                elif c.endswith("[max]"):
                    out[k][c] = max(out[k][c], v)
                else:
                    out[k][c] = out[k][c] + v
    return {k: {c: (float(v) if isinstance(v, (float, np.floating)) else int(v)) for c, v in d.items()} for k, d in out.items()}


def _run_prefix(op, ctx, out, gen, batches, adapt=lambda b: b):
    for b in batches:
        op.process_batch(adapt(b), ctx, out)
        wm = gen.on_batch(int(b[O.TIMESTAMP].min()), int(b[O.TIMESTAMP].max())) if hasattr(gen, "on_batch") else \
            gen.process_batch(b[O.TIMESTAMP])
        if wm is not None:
            ctx.watermarks.set(0, wm)
            op.handle_watermark(wm, ctx, out)


@pytest.mark.parametrize("kind", ["sliding", "tumbling"])
@pytest.mark.parametrize("aggs", [AGGS, SUM_ONLY, MINMAX, PLANS["P3"], PLANS["P4"], PLANS["P5"]],
                         ids=["sum_avg_count", "sum_only", "min_max", "P3", "P4", "P5"])
def test_checkpoint_tables_match_and_restore_both_ways(kind, aggs):
    import arroyo_b200 as ab
    from tests.gpu_ops import from_arrow, to_arrow

    rng = np.random.default_rng(77)
    if any(a.col not in (None, "value") for a in aggs):  # the multi-column plans read a, b, c, d
        batches = gen_multi_stream(rng, 60_000, 1_500, rate_per_s=10_000, batch=3000)
    else:
        batches = gen_stream(rng, 60_000, 1_500, rate_per_s=10_000, batch=3000)
    cfg = _cfg(kind, aggs)
    want = O.run_single_input(_oracle_cls(kind)(cfg), batches, S).batches
    half = len(batches) // 2
    schema = to_arrow(batches[0]).schema

    # ---- both operators up to the checkpoint (two checkpoints: the second one carries deltas only) ----
    o_op, o_ctx, o_out, o_gen = _oracle_cls(kind)(cfg), O.OperatorContext(1), O.Collector(), O.WatermarkGenerator(S)
    g_op = _native_cls(kind)(cfg, input_schema=schema)
    g_ctx, g_out, g_gen = ab.OperatorContext(1), ab.Collector(), ab.WatermarkGenerator(S)
    cut1 = half - 3
    _run_prefix(o_op, o_ctx, o_out, o_gen, batches[:cut1])
    _run_prefix(g_op, g_ctx, g_out, g_gen, batches[:cut1], adapt=to_arrow)
    o_op.handle_checkpoint(o_ctx)
    g_op.handle_checkpoint(None, g_ctx, g_out)
    _run_prefix(o_op, o_ctx, o_out, o_gen, batches[cut1:half])
    _run_prefix(g_op, g_ctx, g_out, g_gen, batches[cut1:half], adapt=to_arrow)
    o_op.handle_checkpoint(o_ctx)
    g_op.handle_checkpoint(None, g_ctx, g_out)
    g_op.close()

    # ---- table "t": same pane timestamps, same per-key state ----
    wm = o_ctx.last_present_watermark()
    assert wm == g_ctx.last_present_watermark()
    o_tab = o_ctx.table("t", cfg.width)
    o_state = {t: bs for t, bs in o_tab.all_batches_for_watermark(wm)}
    g_tab = g_ctx.table("t", cfg.width)
    g_state = {}
    for t, rb in g_tab.all_batches_for_watermark(wm):
        g_state.setdefault(t, []).append(from_arrow(rb))
    assert sorted(o_state) == sorted(g_state) and o_state, (sorted(o_state), sorted(g_state))
    for t in o_state:
        assert _merged(o_state[t]) == _merged(g_state[t]), f"pane {t}"
        for b in g_state[t]:
            assert bool((b[O.TIMESTAMP] == t).all())
            assert list(b.cols) == list(o_state[t][0].cols)  # partial_schema column order

    rest = batches[half:]
    fcols = tuple(a.name for a in aggs if a.kind == "avg")

    def finish(op, ctx, out, gen, adapt=lambda b: b):
        _run_prefix(op, ctx, out, gen, rest, adapt=adapt)
        final = O.FINAL_WATERMARK
        ctx.watermarks.set(0, final)
        op.handle_watermark(final, ctx, out)

    # ---- oracle-written checkpoint -> GPU operator ----
    r_ctx = ab.OperatorContext(1)
    r_ctx.watermarks.set(0, wm)
    r_tab = r_ctx.table("t", cfg.width)
    for t, bs in o_state.items():
        for b in bs:
            r_tab.insert(t, to_arrow(b))
    r_op = _native_cls(kind)(cfg, input_schema=schema)
    r_op.on_start(r_ctx)
    r_out = ab.Collector()
    r_gen = ab.WatermarkGenerator(S)
    r_gen.__dict__.update(g_gen.__dict__)
    finish(r_op, r_ctx, r_out, r_gen, adapt=to_arrow)
    r_op.close()
    got = [from_arrow(b) for b in g_out.batches] + [from_arrow(b) for b in r_out.batches]
    assert_same(want, got, float_cols=fcols)

    # ---- GPU-written checkpoint -> oracle operator ----
    c_ctx = O.OperatorContext(1)
    c_ctx.watermarks.set(0, wm)
    c_tab = c_ctx.table("t", cfg.width)
    for t, bs in g_state.items():
        c_tab.flushed[t] = list(bs)
    c_op = _oracle_cls(kind)(cfg)
    c_op.on_start(c_ctx)
    c_out = O.Collector()
    c_gen = O.WatermarkGenerator(S)
    c_gen.__dict__.update(o_gen.__dict__)
    finish(c_op, c_ctx, c_out, c_gen)
    assert_same(want, list(o_out.batches) + list(c_out.batches), float_cols=fcols)
