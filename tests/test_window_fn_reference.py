"""Pins the exact window function reference (tests/exact_window_fn_reference.py) to the reference's own vector:
golden `most_active_driver_last_hour` is hop(1 min, 1 h) count(*) GROUP BY driver_id, then ROW_NUMBER() OVER
(PARTITION BY window ORDER BY count DESC, driver_id DESC) = 1.  The numpy oracle's sliding aggregate feeds the exact
reference watermark by watermark."""
from oracle import arroyo_oracle as O
from tests import golden_cases as GC
from tests.exact_window_fn_reference import TS, rank_rows, window_fn_emissions

ORDER = [("count", True), ("driver_id", True)]


def sliding_events(inputs):
    """The oracle sliding aggregate's output as window function input events: its batches, then each watermark it
    forwards."""
    cfg = O.WindowAggConfig(width=GC.HOUR, slide=GC.MIN, key_names=["driver_id"], aggs=[O.Agg("count", None, "count")],
                            window_index=1)
    op = O.SlidingAggregatingWindowFunc(cfg)
    ctx, gen, events = O.OperatorContext(1), O.WatermarkGenerator(GC.HOUR), []

    def advance(wm):
        out = O.Collector()
        ctx.watermarks.set(0, wm)
        op.handle_watermark(wm, ctx, out)
        events.extend(("batch", dict(b.cols)) for b in out.batches)
        events.append(("wm", wm))

    for b in O.source_batches({"driver_id": inputs["cars_driver_id"], TS: inputs["cars_ts"]}, GC.BATCH):
        op.process_batch(b, ctx, O.Collector())
        wm = gen.process_batch(b[TS])
        if wm is not None:
            advance(wm)
    advance(O.FINAL_WATERMARK)
    return events


def golden_rows(emissions):
    return [{"start": r["window_start"], "end": r["window_end"], "driver_id": r["driver_id"], "count": r["count"],
             "row_number": r["row_number"]} for rows in emissions for r in rows]


def test_most_active_driver_matches_golden(golden):
    inputs, expected = golden
    events = sliding_events(inputs)
    want = GC.multiset(expected["most_active_driver_last_hour"])
    fused, late, _ = window_fn_emissions(events, None, ORDER, "row_number", "row_number", top_n=1)
    assert late == 0
    assert GC.multiset(golden_rows(fused)) == want
    every, _, _ = window_fn_emissions(events, None, ORDER, "row_number", "row_number")
    assert sum(map(len, every)) > sum(map(len, fused))
    filtered = [[r for r in rows if r["row_number"] == 1] for rows in every]
    assert GC.multiset(golden_rows(filtered)) == want


def test_rank_rules_on_ties():
    """RANK leaves gaps after ties, DENSE_RANK does not, ROW_NUMBER breaks ties by arrival; segments restart them."""
    rows = [{TS: 5, "k": 1, "v": v, "seq": i} for i, v in enumerate([3, 1, 3, 2, 3])] + [{TS: 5, "k": 0, "v": 9, "seq": 5}]
    got = {f: [(r["k"], r["v"], r["seq"], r["f"]) for r in rank_rows(rows, "k", [("v", True)], f, "f")]
           for f in ("row_number", "rank", "dense_rank")}
    assert got["row_number"] == [(0, 9, 5, 1), (1, 3, 0, 1), (1, 3, 2, 2), (1, 3, 4, 3), (1, 2, 3, 4), (1, 1, 1, 5)]
    assert [x[3] for x in got["rank"]] == [1, 1, 1, 1, 4, 5]
    assert [x[3] for x in got["dense_rank"]] == [1, 1, 1, 1, 2, 3]
    assert [r["f"] for r in rank_rows(rows, "k", [("v", True)], "rank", "f", top_n=1)] == [1, 1, 1, 1]


def test_late_rows_and_restart_state():
    events = [("batch", {"v": [1, 2, 3], TS: [10, 20, 20]}), ("wm", 15), ("batch", {"v": [4, 5], TS: [14, 15]}),
              ("restart",), ("batch", {"v": [6], TS: [30]}), ("wm", 31)]
    out, late, states = window_fn_emissions(events, None, [("v", False)], "row_number")
    assert late == 1
    assert [[(r[TS], r["v"], r["fn"]) for r in rows] for rows in out] == [[(10, 1, 1)], [(15, 5, 1), (20, 2, 1),
                                                                                        (20, 3, 2), (30, 6, 1)]]
    assert states == [{20: [{"v": 2, TS: 20}, {"v": 3, TS: 20}], 15: [{"v": 5, TS: 15}]}]
