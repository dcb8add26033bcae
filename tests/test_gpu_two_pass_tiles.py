"""The partition pass's input ring (csrc/ingest_two_pass.cuh: part_kernel) on the tile shapes the bulk copies do not
carry by themselves, checked row by row against an independent group-by (torch.unique + index_add):

  segments whose columns are not 16-byte aligned (all three, or only the value column): loaded with ordinary loads
  segments shorter than a tile, and segments of odd length (a ragged last row after the bulk-copied pairs)
  a pane boundary inside a tile (the tile's other-pane rows take the direct path)
"""
import pytest

from tests.test_gpu_parity import S, T0

pytestmark = pytest.mark.gpu


def test_unaligned_short_and_ragged_segments_and_a_pane_boundary_inside_a_tile():
    import pyarrow as pa
    import torch

    import arroyo_b200 as ab
    from arroyo_b200 import ffi, operators as native
    from arroyo_b200.multi_gpu import _Ptr

    device = torch.device("cuda", 0)
    torch.cuda.set_device(0)
    torch.cuda.set_stream(torch.cuda.Stream(device=device))
    g = torch.Generator(device=device)
    g.manual_seed(7)
    n, n_keys = 1 << 21, 50_000
    key = torch.randint(0, n_keys, (n,), generator=g, device=device, dtype=torch.int64) * 0x1E3779B97F4A7C15
    val = torch.randint(-(1 << 30), 1 << 30, (n,), generator=g, device=device, dtype=torch.int64)
    # in order over two panes: the boundary falls inside a tile
    ts = T0 + torch.sort(torch.randint(0, 2 * S, (n,), generator=g, device=device, dtype=torch.int64)).values
    # a copy of the values one row further on: its pointer is 8 bytes off wherever the others are 16-byte aligned
    val_shifted = torch.empty(n + 1, device=device, dtype=torch.int64)
    val_shifted[1:] = val
    cfg = ab.WindowAggConfig(width=S, key_names=["key"], aggs=[ab.Agg("sum", "value", "sum"), ab.Agg("count", None, "n")],
                             window_index=1)
    schema = pa.schema([("key", pa.int64()), ("value", pa.int64()), ("_timestamp", pa.timestamp("ns"))])
    op = native.TumblingAggregatingWindowFunc(cfg, input_schema=schema, device=0,
                                              stream=torch.cuda.current_stream().cuda_stream,
                                              flags=ffi.FLAG_TWO_PASS_ALWAYS, expected_keys=n_keys)
    # a first small batch tells the operator where the stream is (the two passes need a known newest pane)
    op.process_device_batch([key.data_ptr(), val.data_ptr(), ts.data_ptr()], 4096)
    op.flush()
    # (rows, value column shifted): odd starts misalign every column, the shifted copy misaligns the values only
    sizes = [(1, False), (3001, False), (70_001, False), (5, True), (4096 * 3 + 1, True), (4096, False),
             (100_000, True), (2047, False)]
    start = 4096
    i = 0
    while start < n:
        rows, shifted = sizes[i % len(sizes)]
        rows = min(rows, n - start)
        vp = val_shifted.data_ptr() + 8 * (start + 1) if shifted else val.data_ptr() + 8 * start
        op.process_device_batch([key.data_ptr() + 8 * start, vp, ts.data_ptr() + 8 * start], rows)
        start += rows
        i += 1
    got = {}
    for rows, ptrs in op.handle_watermark_device(T0 + 3 * S):
        cols = [torch.as_tensor(_Ptr(c, rows), device=device).clone() for c in ptrs]
        got[int(cols[1][0])] = cols
    st = op.stats()
    op.close()
    assert sorted(got) == [T0, T0 + S]
    for w0, cols in got.items():
        sel = (ts >= w0) & (ts < w0 + S)
        uk, inv = torch.unique(key[sel], return_inverse=True)
        want_sum = torch.zeros(uk.numel(), dtype=torch.int64, device=device).index_add_(0, inv, val[sel])
        want_cnt = torch.zeros(uk.numel(), dtype=torch.int64, device=device).index_add_(0, inv, torch.ones_like(val[sel]))
        k_out, ws, we, s_out, n_out = cols[0], cols[1], cols[2], cols[3], cols[4]
        order = torch.argsort(k_out)
        assert torch.equal(k_out[order], uk)
        assert torch.equal(n_out[order], want_cnt)
        assert torch.equal(s_out[order], want_sum)
        assert bool((ws == w0).all()) and bool((we == w0 + S).all())
    assert st["rows_in"] == n
