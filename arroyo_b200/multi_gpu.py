"""The Shuffle edge across the GPUs of one box: one process per GPU, key-hash partition on the device,
NCCL all-to-all over NVLink, watermark min-merge at the receiver.

Replaces, for edges between GPU-resident operators, `ArrowCollector::collect -> repartition`
(arroyo-operator/src/context.rs:506-616), the queue mesh of a Shuffle edge
(arroyo-worker/src/engine.rs:341-359) and the per-input watermark merge (`WatermarkHolder`,
context.rs:35-86).  Every subtask is both a sender (it ingests its shard of the upstream) and a receiver
(it owns the keys whose hash falls in its range, arroyo-operator/src/lib.rs:30-41).

Per round every rank
  1. buckets its rows by destination (`arroyo_b200_partition`: histogram -> scan -> scatter; the
     per-destination segments are the all-to-all send buffers),
  2. all-gathers one control row {rows for each destination, its watermark or none}: afterwards every
     rank knows its receive counts and every sender's watermark (signals are broadcast to every
     downstream queue in the reference too, context.rs:663-677),
  3. exchanges the column segments with `all_to_all_single` (variable splits),
  4. hands the received rows to its window operator and then applies the min-merged watermark.
No reduction collective is needed: each key lives on exactly one GPU.

`ShuffleExchange` takes the partition function as a parameter so the protocol can be exercised on CPU
tensors with the `gloo` backend (tests/test_shuffle_gloo.py); the product path uses `DevicePartitioner`.
"""
import ctypes as C
from typing import Callable, List, Optional, Sequence, Tuple

from . import ffi
from .context import WatermarkHolder

NO_WM = -(1 << 63)


class DevicePartitioner:
    """arroyo_b200_partition over torch device tensors (the product path)."""

    def __init__(self, torch, world: int, n_cols: int, key_col: int, max_rows: int, device: int, stream: int):
        if not stream:
            # stream 0 would make the library create a private stream with no ordering against the torch stream
            # that produces `cols` and reads `counts` (include/arroyo_b200.h, stream-ordering contract)
            raise ValueError("DevicePartitioner needs the explicit CUDA stream its inputs are produced on")
        self.torch = torch
        self.lib = ffi.load()
        self.h = C.c_void_p()
        st = self.lib.arroyo_b200_partitioner_create(device, stream, world, n_cols, key_col, max_rows, C.byref(self.h))
        if st != ffi.OK:
            raise ffi.ArroyoB200Error(st, "partitioner_create failed")
        dev = torch.device("cuda", device)
        self.out = [torch.empty(max_rows, dtype=torch.int64, device=dev) for _ in range(n_cols)]
        self.counts = torch.zeros(world, dtype=torch.int64, device=dev)
        self.offsets = torch.zeros(world, dtype=torch.int64, device=dev)
        self.n_cols = n_cols
        self.max_rows = max_rows
        self._packed = None
        self._dev = dev

    def __call__(self, cols: Sequence, n_rows: int):
        inp = (C.c_uint64 * self.n_cols)(*[c.data_ptr() for c in cols])
        outp = (C.c_uint64 * self.n_cols)(*[c.data_ptr() for c in self.out])
        st = self.lib.arroyo_b200_partition(self.h, inp, n_rows, outp, self.counts.data_ptr(), self.offsets.data_ptr())
        if st != ffi.OK:
            raise ffi.ArroyoB200Error(st, "partition failed")
        return [o[:n_rows] for o in self.out], self.counts

    def pack(self, col_ptrs: Sequence[int], n_rows: int, counts_out=None):
        """arroyo_b200_partition_packed: `col_ptrs` are raw device pointers; returns (packed buffer,
        counts[world] device tensor).  Destination d's block holds its n_cols columns back to back.
        `counts_out`: device tensor whose first `world` int64 receive the counts (e.g. the exchange's control
        record) instead of the partitioner's own."""
        if self._packed is None:
            self._packed = self.torch.empty(self.max_rows * self.n_cols, dtype=self.torch.int64, device=self._dev)
        inp = (C.c_uint64 * self.n_cols)(*col_ptrs)
        counts = self.counts if counts_out is None else counts_out
        st = self.lib.arroyo_b200_partition_packed(self.h, inp, n_rows, self._packed.data_ptr(), counts.data_ptr(),
                                                   self.offsets.data_ptr())
        if st != ffi.OK:
            raise ffi.ArroyoB200Error(st, "partition_packed failed")
        return self._packed[:n_rows * self.n_cols], counts

    def close(self):
        if self.h:
            self.lib.arroyo_b200_partitioner_destroy(self.h)
            self.h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class ShuffleExchange:
    """One Shuffle edge between `world` subtasks.  `partition_fn(cols, n_rows) -> (cols bucketed by
    destination in destination order, counts[world] tensor)`."""

    def __init__(self, torch, dist, rank: int, world: int, partition_fn: Callable, device, max_recv_rows: int,
                 n_cols: int):
        self.torch, self.dist, self.rank, self.world = torch, dist, rank, world
        self.partition_fn = partition_fn
        self.device = device
        # one control record per sender and round: rows for every destination, the sender's watermark (or none),
        # and whether the sender has more rounds queued behind this one
        self.ctrl = torch.zeros(world + 2, dtype=torch.int64, device=device)
        self.ctrl_all = torch.zeros(world * (world + 2), dtype=torch.int64, device=device)
        # the two host-written words of a control record (watermark, more-rounds flag) go through one pinned
        # staging tensor: one small async copy per round instead of one tensor op per word
        self._ctl_host = torch.zeros(2, dtype=torch.int64)
        if device.type == "cuda":
            self._ctl_host = self._ctl_host.pin_memory()
        self._recv = None
        self._recv_packed = None
        self._flip = 0
        self.n_cols = n_cols
        self.max_recv_rows = max_recv_rows
        self.holder = WatermarkHolder(world)
        self.bytes_sent = 0

    def exchange_watermark(self, watermark: Optional[int]) -> Optional[int]:
        """Broadcasts this sender's watermark (or none) and returns the min-merged effective watermark if it
        advanced (signals go to every downstream queue, context.rs:663-677; merge = WatermarkHolder)."""
        torch, dist, W = self.torch, self.dist, self.world
        self._ctl_host[0] = NO_WM if watermark is None else int(min(watermark, (1 << 63) - 1))
        self._ctl_host[1] = 0
        self.ctrl[W:].copy_(self._ctl_host, non_blocking=True)  # the count words are not read by this exchange
        dist.all_gather_into_tensor(self.ctrl_all, self.ctrl)
        m = self.ctrl_all.view(W, W + 2)[:, W].cpu().tolist()
        before = self.holder.last_present_watermark
        for s, wm in enumerate(m):
            if wm != NO_WM:
                self.holder.set(s, wm)
        after = self.holder.last_present_watermark
        return after if after is not None and after != before else None

    def round(self, cols: Sequence, n_rows: int, watermark: Optional[int]) -> Tuple[List, int, Optional[int]]:
        """Sends this rank's rows, returns (received columns, received rows, effective watermark after
        this round or None if it did not advance)."""
        torch, dist, W = self.torch, self.dist, self.world
        if n_rows > 0:
            send_cols, counts = self.partition_fn(cols, n_rows)
            self.ctrl[:W] = counts
        else:
            send_cols = [c[:0] for c in cols]
            self.ctrl[:W] = 0
        self.ctrl[W] = NO_WM if watermark is None else int(min(watermark, (1 << 63) - 1))
        self.ctrl[W + 1] = 0
        dist.all_gather_into_tensor(self.ctrl_all, self.ctrl)
        m = self.ctrl_all.view(W, W + 2).cpu()  # the one host sync of the round: split sizes
        send_splits = m[self.rank, :W].tolist()
        recv_splits = m[:, self.rank].tolist()
        n_recv = int(sum(recv_splits))
        if n_recv > self.max_recv_rows:
            raise RuntimeError(f"shuffle receive buffer too small: {n_recv} > {self.max_recv_rows}")
        if self._recv is None:
            self._recv = [torch.empty(self.max_recv_rows, dtype=torch.int64, device=self.device)
                          for _ in range(self.n_cols)]
        out = []
        for c, r in zip(send_cols, self._recv):
            o = r[:n_recv]
            dist.all_to_all_single(o, c, recv_splits, send_splits)
            out.append(o)
        self.bytes_sent += 8 * len(send_cols) * (n_rows - send_splits[self.rank])
        before = self.holder.last_present_watermark
        for s in range(W):
            wm = int(m[s, W])
            if wm != NO_WM:
                self.holder.set(s, wm)
        after = self.holder.last_present_watermark
        return out, n_recv, (after if after is not None and after != before else None)

    def round_packed(self, packed, counts, n_rows: int, watermark: Optional[int], more: bool = False):
        """One round over the packed layout of arroyo_b200_partition_packed: a single all-to-all carries every
        column.  Returns (batches, effective watermark or None, any sender has more rounds) where batches =
        [([device pointer per column], rows)] -- one columnar batch per sender that sent rows.  The receive
        buffer alternates between two allocations, so a batch stays valid until the round after next."""
        torch, dist, W, nc = self.torch, self.dist, self.world, self.n_cols
        if n_rows > 0:
            if counts.data_ptr() != self.ctrl.data_ptr():  # DevicePartitioner.pack(counts_out=ctrl) writes in place
                self.ctrl[:W] = counts
        else:
            self.ctrl[:W] = 0
        self._ctl_host[0] = NO_WM if watermark is None else int(min(watermark, (1 << 63) - 1))
        self._ctl_host[1] = 1 if more else 0
        self.ctrl[W:].copy_(self._ctl_host, non_blocking=True)
        dist.all_gather_into_tensor(self.ctrl_all, self.ctrl)
        m = self.ctrl_all.view(W, W + 2).cpu()
        send_rows = m[self.rank, :W].tolist()
        recv_rows = m[:, self.rank].tolist()
        n_recv = int(sum(recv_rows))
        if n_recv > self.max_recv_rows:
            raise RuntimeError(f"shuffle receive buffer too small: {n_recv} > {self.max_recv_rows}")
        if self._recv_packed is None:
            self._recv_packed = [torch.empty(self.max_recv_rows * nc, dtype=torch.int64, device=self.device)
                                 for _ in range(2)]
        buf = self._recv_packed[self._flip]
        self._flip ^= 1
        o = buf[:n_recv * nc]
        src = packed[:n_rows * nc] if n_rows > 0 else buf[:0]
        dist.all_to_all_single(o, src, [nc * int(r) for r in recv_rows], [nc * int(r) for r in send_rows])
        self.bytes_sent += 8 * nc * (n_rows - int(send_rows[self.rank]))
        batches, off, base = [], 0, o.data_ptr()
        for sdr in range(W):
            r = int(recv_rows[sdr])
            if r:
                batches.append(([base + 8 * (off + c * r) for c in range(nc)], r))
            off += nc * r
        before = self.holder.last_present_watermark
        for sdr in range(W):
            wm = int(m[sdr, W])
            if wm != NO_WM:
                self.holder.set(sdr, wm)
        after = self.holder.last_present_watermark
        any_more = bool(m[:, W + 1].any())
        return batches, (after if after is not None and after != before else None), any_more


# ------------------------------------------------------------------------------------------------
# N > 1 benchmark (called from bench.py under torchrun)
# ------------------------------------------------------------------------------------------------
class _Ptr:
    """Wraps a raw device pointer as a torch tensor (__cuda_array_interface__)."""

    def __init__(self, ptr, n):
        self.__cuda_array_interface__ = {"shape": (n,), "typestr": "<i8", "data": (ptr, False), "version": 2}


class PartialsPlan:
    """partial -> shuffle -> final on one rank (SURVEY.md 8(e): the combiner plan).

    local stage  : tumbling pre-aggregate of width = slide over this rank's shard, on its own CUDA stream;
                   when the min-merged watermark passes a pane its partial rows (key, sum, count, _timestamp)
                   leave as one device batch.
    shuffle edge : arroyo_b200_partition_packed -> control all-gather -> one NCCL all-to-all.
    owner stage  : sliding operator over partial rows (`partial_count_col`), on the caller's stream.

    The two stages are separate operators of the dataflow: `close_panes` (local) returns the batches and the
    watermark the owner stage must see, `owner_stage` consumes them in order.  Callers enqueue the local stage's
    next input before running the owner stage, so the exchange and the owner's kernels overlap the local ingest."""

    N_COLS = 4

    def __init__(self, torch, dist, B, ab, native, args, rank, world, local, device, local_flags, owner_flags,
                 raw_schema=None):
        import pyarrow as pa
        self.torch, self.dist, self.world = torch, dist, world
        self.part_rows = 1 << 22
        stream = torch.cuda.current_stream().cuda_stream
        local_cfg = ab.WindowAggConfig(width=B.SLIDE, key_names=["key"],
                                       aggs=[ab.Agg("sum", "value", "sum"), ab.Agg("count", None, "count")],
                                       final_projection=False)
        # stream=0: the operator creates its own non-blocking stream
        self.local_op = native.TumblingAggregatingWindowFunc(local_cfg, input_schema=raw_schema, device=local, stream=0,
                                                             flags=local_flags, expected_keys=args.keys,
                                                             task_index=rank, parallelism=world,
                                                             chunk_log2=getattr(args, "local_chunk_log2", 21))
        owner_cfg = ab.WindowAggConfig(width=B.WIDTH, slide=B.SLIDE, key_names=["key"],
                                       aggs=[ab.Agg("sum", "sum", "sum"), ab.Agg("avg", "sum", "avg"),
                                             ab.Agg("count", None, "count")], window_index=1, partial_count_col="count")
        p_schema = pa.schema([("key", pa.int64()), ("sum", pa.int64()), ("count", pa.int64()),
                              ("_timestamp", pa.timestamp("ns"))])
        self.owner_op = native.SlidingAggregatingWindowFunc(owner_cfg, input_schema=p_schema, device=local, stream=stream,
                                                            flags=owner_flags,
                                                            expected_keys=max(2 * args.keys // world, 1024),
                                                            task_index=rank, parallelism=world)
        self.part = DevicePartitioner(torch, world, self.N_COLS, 0, self.part_rows, local, stream)
        self.ex = ShuffleExchange(torch, dist, rank, world, None, device, max_recv_rows=2 * self.part_rows,
                                  n_cols=self.N_COLS)

    def close_panes(self, watermark: Optional[int]):
        """Local stage at a watermark point.  Every rank calls this the same number of times (ranks without a
        new watermark pass None).  Returns (effective watermark or None, partial-row batches that left)."""
        eff = self.ex.exchange_watermark(watermark)
        if eff is None:
            return None, []
        chunks = []
        for n, cols in self.local_op.handle_watermark_device(eff):
            for o in range(0, n, self.part_rows):
                chunks.append(([c + 8 * o for c in cols], min(self.part_rows, n - o)))
        return eff, chunks

    def owner_stage(self, eff: int, chunks, sink):
        """Shuffle edge + owner stage for what `close_panes` returned; `sink(owner_op, eff)` emits."""
        i = 0
        while True:
            if i < len(chunks):
                cols, m = chunks[i]
                packed, counts = self.part.pack(cols, m, counts_out=self.ex.ctrl)
            else:
                packed, counts, m = None, None, 0
            i += 1
            batches, _, any_more = self.ex.round_packed(packed, counts, m, None, more=i < len(chunks))
            if batches:
                flat = (C.c_uint64 * (self.N_COLS * len(batches)))(*[p for cols, _ in batches for p in cols])
                nr = (C.c_int64 * len(batches))(*[r for _, r in batches])
                self.owner_op.process_device_batches(flat, nr, self.N_COLS)
            if not any_more:
                break
            self.owner_op.flush()  # more rounds follow: the receive buffers come round again
        sink(self.owner_op, eff)

    def pipeline(self, sink, lag: int = 2, exchange=None):
        """LaggedCombiner over this plan's operators; `sink(owner_op, eff)` emits.  `exchange`: an object with
        ShuffleExchange's round_packed contract that partitions by itself (native_exchange.NativeExchange)."""
        torch = self.torch
        dev = torch.cuda.current_device()
        stream = torch.cuda.current_stream()

        def thread_init():
            torch.cuda.set_device(dev)
            torch.cuda.set_stream(stream)  # the current stream is per thread

        def local_close(eff):
            chunks = []
            for n, cols in self.local_op.handle_watermark_device(eff):
                for o in range(0, n, self.part_rows):
                    chunks.append(([c + 8 * o for c in cols], min(self.part_rows, n - o)))
            return chunks

        def pack(chunk):
            cols, m = chunk
            if exchange is not None:
                return cols, None, m  # the native exchange partitions inside its round
            packed, counts = self.part.pack(cols, m, counts_out=self.ex.ctrl)
            return packed, counts, m

        def owner_ingest(batches, consume_now):
            flat = (C.c_uint64 * (self.N_COLS * len(batches)))(*[p for cols, _ in batches for p in cols])
            nr = (C.c_int64 * len(batches))(*[r for _, r in batches])
            self.owner_op.process_device_batches(flat, nr, self.N_COLS)
            if consume_now:
                self.owner_op.flush()

        return LaggedCombiner(exchange if exchange is not None else self.ex, local_close, pack, owner_ingest,
                              lambda eff: sink(self.owner_op, eff), lag=lag, thread_init=thread_init)

    def close(self):
        self.owner_op.close()
        self.local_op.close()
        self.part.close()


class LaggedCombiner:
    """The combiner plan as a two-stage software pipeline on one rank.

    The local stage (caller's thread) and the shuffle edge + owner stage (a second host thread) are different
    operators of the dataflow, connected by a queue -- exactly as in the reference, where every operator is its own
    task.  Watermarks ride on the data rounds (they are in-band signals of the edge): round p carries this rank's
    watermark after step p and the partial rows of the panes the local stage closed in step p.  The local stage closes
    panes with the effective watermark that came out of round p - lag, so it never waits for the round in flight;
    every rank uses the same (deterministic) lag, hence the same effective watermark for the same step.

    Callbacks (all on device pointers or host arrays -- the class only sequences them):
      local_close(eff) -> [chunk]            panes the local stage closes at `eff` (its output buffers must stay valid
                                             until the chunk was packed; `local_step` waits for that)
      pack(chunk) -> (packed, counts, rows)  arroyo_b200_partition_packed (or its CPU restatement)
      owner_ingest([(cols, rows)], consume_now)  partial rows received in a round (`consume_now`: the buffers are
                                             about to be reused and no owner_watermark call follows)
      owner_watermark(eff)                   the owner stage's handle_watermark"""

    def __init__(self, ex, local_close, pack, owner_ingest, owner_watermark, lag: int = 2, thread_init=None):
        import queue
        import threading
        self.ex, self.lag = ex, lag
        self.local_close, self.pack = local_close, pack
        self.owner_ingest, self.owner_watermark = owner_ingest, owner_watermark
        self.thread_init = thread_init
        self.q = queue.Queue()
        self.cv = threading.Condition()
        self.eff_after = {}      # step -> effective watermark after that step's rounds
        self.packed_upto = -1    # last step whose chunks have left the local stage's buffers
        self.step = 0
        self.last_closed = None
        self.error = None
        # where the host time of a step goes (seconds, accumulated; reset with reset_times())
        self.times = {"feed": 0.0, "wait_round": 0.0, "wait_packed": 0.0, "local_close": 0.0, "pack": 0.0, "exchange": 0.0,
                      "owner_ingest": 0.0, "owner_watermark": 0.0, "owner_idle": 0.0}
        self.th = threading.Thread(target=self._owner_loop, daemon=True)
        self.th.start()

    # ---- local stage (caller's thread) ----
    def local_step(self, feed, watermark):
        """One step of the local stage: `feed()` enqueues the step's input on the local operator (asynchronously);
        then the panes that the effective watermark of round p - lag closes leave as partial rows.  Feeding first
        keeps the device busy with the ingest while this thread waits for the round and for the emission."""
        import time
        T = self.times
        p = self.step
        self.step += 1
        t0 = time.perf_counter()
        feed()
        t1 = time.perf_counter()
        eff = None
        with self.cv:
            if p - self.lag >= 0:
                self.cv.wait_for(lambda: (p - self.lag) in self.eff_after or self.error is not None)
                self._raise()
                eff = self.eff_after.pop(p - self.lag)
            t2 = time.perf_counter()
            # the previous step's partial rows must have been packed before the local stage overwrites them
            self.cv.wait_for(lambda: self.packed_upto >= p - 1 or self.error is not None)
            self._raise()
        t3 = time.perf_counter()
        chunks, closing = [], None
        if eff is not None and eff != self.last_closed:
            chunks = self.local_close(eff)
            closing = self.last_closed = eff
        t4 = time.perf_counter()
        T["feed"] += t1 - t0
        T["wait_round"] += t2 - t1
        T["wait_packed"] += t3 - t2
        T["local_close"] += t4 - t3
        self.q.put((p, closing, chunks, watermark))

    def reset_times(self):
        for k in self.times:
            self.times[k] = 0.0

    def drain(self):
        """Waits until the owner stage has consumed everything queued so far."""
        with self.cv:
            self.cv.wait_for(lambda: self.packed_upto >= self.step - 1 and self.q.unfinished_tasks == 0
                             or self.error is not None)
            self._raise()

    def close(self):
        self.q.put(None)
        self.th.join()
        self._raise()

    def _raise(self):
        if self.error is not None:
            raise RuntimeError(f"owner stage failed: {self.error!r}")

    # ---- shuffle edge + owner stage (second thread) ----
    def _owner_loop(self):
        try:
            if self.thread_init:
                self.thread_init()
            import time
            T = self.times
            while True:
                t0 = time.perf_counter()
                item = self.q.get()
                T["owner_idle"] += time.perf_counter() - t0
                if item is None:
                    self.q.task_done()
                    return
                p, closing, chunks, wm = item
                i = 0
                while True:
                    t0 = time.perf_counter()
                    if i < len(chunks):
                        packed, counts, m = self.pack(chunks[i])
                    else:
                        packed, counts, m = None, None, 0
                    i += 1
                    t1 = time.perf_counter()
                    batches, _, any_more = self.ex.round_packed(packed, counts, m, wm if i == 1 else None,
                                                                more=i < len(chunks))
                    t2 = time.perf_counter()
                    if batches:
                        # the receive buffers come round again two rounds later: rows that no watermark is about to
                        # push through the owner must be consumed now
                        self.owner_ingest(batches, consume_now=any_more or closing is None)
                    T["pack"] += t1 - t0
                    T["exchange"] += t2 - t1
                    T["owner_ingest"] += time.perf_counter() - t2
                    if not any_more:
                        break
                with self.cv:
                    self.packed_upto = p
                    self.eff_after[p] = self.ex.holder.last_present_watermark
                    self.cv.notify_all()
                if closing is not None:
                    t0 = time.perf_counter()
                    self.owner_watermark(closing)
                    T["owner_watermark"] += time.perf_counter() - t0
                self.q.task_done()
                with self.cv:
                    self.cv.notify_all()
        except BaseException as e:  # noqa: BLE001
            with self.cv:
                self.error = e
                self.cv.notify_all()


def _wm_point(wms, p, nb):
    """(batch index inside pane p after which this rank reports to the watermark exchange, watermark or None):
    the batch whose arrival made the WatermarkGenerator emit, else the pane's last batch."""
    found = [(b, wms[p * nb + b]) for b in range(nb) if wms[p * nb + b] is not None]
    if not found:
        return nb - 1, None
    return found[0][0], found[-1][1]


def _e2e_partials(args, torch, dist, B, ab, native, rank, world, local, device, gen_pane, feed=None):
    """End to end at N GPUs: every rank feeds its shard as pinned host Arrow batches through
    arroyo_b200_op_process_batch (host -> device copies inside the timed region), partial aggregates cross the
    all-to-all, and each rank reads the windows of its keys back as host Arrow batches."""
    import time

    rows = args.rows_per_pane
    nb = rows // B.BATCH_ROWS
    K = args.e2e_steps or min(args.steps, 6)
    W = 13
    batches, wms, _keep = feed if feed is not None else B.host_feed(torch, gen_pane, range(W + K), rows)
    plan = PartialsPlan(torch, dist, B, ab, native, args, rank, world, local, device, B.op_flags(args), B.op_flags(args))
    lctx, octx, col = ab.OperatorContext(1), ab.OperatorContext(1), ab.Collector()
    d2h = 0

    def sink(owner_op, eff):
        nonlocal d2h
        octx.watermarks.set(0, eff)
        owner_op.handle_watermark(eff, octx, col)
        for rb in col.batches:
            d2h += rb.num_rows * 48
        col.batches.clear()

    def step(p):
        b0, wm = _wm_point(wms, p, nb)
        for b in range(b0 + 1):
            plan.local_op.process_batch(batches[p][b], lctx, col)
        eff, chunks = plan.close_panes(wm)
        for b in range(b0 + 1, nb):
            plan.local_op.process_batch(batches[p][b], lctx, col)
        if eff is not None:
            plan.owner_stage(eff, chunks, sink)

    for p in range(W):
        step(p)
    plan.owner_op.flush()
    plan.local_op.flush()
    torch.cuda.synchronize()
    dist.barrier()
    d2h = 0
    t0 = time.perf_counter()
    for p in range(W, W + K):
        step(p)
    plan.owner_op.flush()
    plan.local_op.flush()
    torch.cuda.synchronize()
    dist.barrier()
    dt = torch.tensor([time.perf_counter() - t0], dtype=torch.float64, device=device)
    dist.all_reduce(dt, op=dist.ReduceOp.MAX)
    tot = torch.tensor([d2h], dtype=torch.int64, device=device)
    dist.all_reduce(tot)
    plan.close()
    dt = float(dt.item())
    return {"value": world * K * rows / dt, "unit": "rows/s", "h2d_bytes_per_step": world * rows * 24,
            "d2h_bytes_per_step": int(tot.item()) // max(K, 1), "steps": K, "ms_per_step": 1e3 * dt / K,
            "path": "per GPU: pinned host Arrow batches -> arroyo_b200_op_process_batch -> partials over NCCL all-to-all "
                    "-> host Arrow windows"}


def _run_plan(args, torch, dist, B, ab, native, rank, world, local, device, panes, W, K, collect=False, sampler=None):
    """One pass of the N-GPU plan over this rank's `panes`: W warm-up steps, K timed steps (CUDA events, max over
    ranks).  With `collect` every window this rank emits is reduced to checksums on the device (a verification pass;
    its time means nothing).  Returns a dict."""
    import pyarrow as pa

    dog = _Watchdog(rank, f"the {world}-GPU plan (--shuffle {args.shuffle})")
    rows = panes[0][0].numel()
    nb = rows // B.BATCH_ROWS
    mins, maxs = [], []
    for (_, _, t) in panes:
        tb = t.view(nb, B.BATCH_ROWS)
        mins.append(tb.amin(dim=1))
        maxs.append(tb.amax(dim=1))
    mins = torch.stack(mins).cpu().numpy().reshape(-1).tolist()
    maxs = torch.stack(maxs).cpu().numpy().reshape(-1).tolist()
    wms = B.watermark_schedule(list(zip(mins, maxs)))  # this rank's own WatermarkGenerator
    torch.cuda.synchronize()

    stream = torch.cuda.current_stream().cuda_stream
    mode = args.shuffle
    flags = ffi.FLAG_PROFILE | B.op_flags(args)
    raw_schema = pa.schema([("key", pa.int64()), ("value", pa.int64()), ("_timestamp", pa.timestamp("ns"))])
    plan = part = ex = None
    if mode == "partials":
        plan = PartialsPlan(torch, dist, B, ab, native, args, rank, world, local, device, flags, flags,
                            raw_schema=raw_schema)
        local_op, owner_op, ex = plan.local_op, plan.owner_op, plan.ex
    else:
        part_rows = 64 * B.BATCH_ROWS
        local_op = None
        owner_op = native.SlidingAggregatingWindowFunc(B.window_config(), input_schema=raw_schema, device=local,
                                                       stream=stream, flags=flags,
                                                       expected_keys=max(2 * args.keys // world, 1024), task_index=rank,
                                                       parallelism=world)
        part = DevicePartitioner(torch, world, 3, 0, part_rows, local, stream)
        ex = ShuffleExchange(torch, dist, rank, world, part, device, max_recv_rows=2 * part_rows, n_cols=3)
    rows_out = 0
    sums = {}

    outstanding = False

    def gather():
        # the owner stage's outstanding emission (arroyo_b200_op_handle_watermark_device_poll)
        nonlocal rows_out, outstanding
        if not outstanding:
            return
        outstanding = False
        emitted = owner_op.handle_watermark_device_poll()
        for n, _ in emitted:
            rows_out += n
        if collect:
            for ws, we, n, cnt, sm, av in B.window_checksums(torch, device, emitted):
                sums[ws] = (we, n, cnt, sm, av)

    def emit(eff):
        # begin / poll: the owner's emission is enqueued and its row counts are read one emission late, so the thread
        # that runs the shuffle edge goes straight on to the next round
        nonlocal outstanding
        gather()
        owner_op.handle_watermark_device_begin(eff)
        outstanding = True
        dog.beat(f"owner stage emitted at watermark {eff}")

    native_ex = None
    if plan is not None and not args.sync_plan and getattr(args, "native_exchange", False):
        from .native_exchange import NativeExchange
        native_ex = NativeExchange(torch, dist, rank, world, local, stream, plan.N_COLS, 0, plan.part_rows,
                                   2 * plan.part_rows)
    pipe = plan.pipeline(lambda op, w: emit(w), exchange=native_ex) if (plan is not None and not args.sync_plan) else None

    def step_partials(p):
        k, v, t = panes[p]
        b0, wm = _wm_point(wms, p, nb)
        e = (b0 + 1) * B.BATCH_ROWS

        def feed_first():
            local_op.process_device_batch([k.data_ptr(), v.data_ptr(), t.data_ptr()], e)

        def feed_rest():
            if e < rows:
                local_op.process_device_batch([k.data_ptr() + 8 * e, v.data_ptr() + 8 * e, t.data_ptr() + 8 * e], rows - e)
                local_op.submit()

        if pipe is not None:
            # two-stage pipeline: the shuffle edge and the owner stage run on a second host thread, one or two
            # rounds behind the local stage (LaggedCombiner)
            pipe.local_step(lambda: (feed_first(), feed_rest()), wm)
            return
        feed_first()
        eff, chunks = plan.close_panes(wm)
        feed_rest()  # enqueued before the owner stage runs, so the exchange and the owner's kernels overlap it
        if eff is not None:
            plan.owner_stage(eff, chunks, lambda op, w: emit(w))

    def step_rows(p):
        k, v, t = panes[p]
        rb = part_rows // B.BATCH_ROWS
        for r0 in range(0, nb, rb):
            r1 = min(r0 + rb, nb)
            s, e = r0 * B.BATCH_ROWS, r1 * B.BATCH_ROWS
            wm = None
            for b in range(r0, r1):
                if wms[p * nb + b] is not None:
                    wm = wms[p * nb + b]
            cols, n_recv, eff = ex.round([k[s:e], v[s:e], t[s:e]], e - s, wm)
            if n_recv:
                owner_op.process_device_batch([c.data_ptr() for c in cols], n_recv)
            if eff is not None:
                emit(eff)
            else:
                owner_op.flush()  # the receive buffers are reused by the next round

    step_inner = step_partials if mode == "partials" else step_rows

    def step(p):
        step_inner(p)
        dog.beat(f"local stage fed pane {p}")

    timed_op = local_op if mode == "partials" else owner_op
    if sampler is None:
        sampler = B.ClockSampler(local)
        if rank == 0 and not collect:
            sampler.start()
    for p in range(W):
        step(p)
    if pipe is not None:
        pipe.drain()
    gather()
    owner_op.flush()
    torch.cuda.synchronize()
    dist.barrier()
    st0 = timed_op.stats()
    so0 = owner_op.stats()
    if pipe is not None:
        pipe.reset_times()
    rows_out_warm = rows_out
    rows_out = 0
    ex_used = native_ex if native_ex is not None else ex
    sent0 = ex_used.bytes_sent
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    sampler.begin()
    e0.record()
    for p in range(W, W + K):
        step(p)
    if pipe is not None:
        pipe.drain()
    gather()
    owner_op.flush()
    if local_op is not None:
        local_op.flush()
    e1.record()
    torch.cuda.synchronize()
    sampler.end()
    dist.barrier()
    ms = torch.tensor([e0.elapsed_time(e1)], dtype=torch.float64, device=device)
    dist.all_reduce(ms, op=dist.ReduceOp.MAX)
    ms = float(ms.item())
    clocks = sampler.stop() if (rank == 0 and not collect) else None
    st1 = timed_op.stats()
    so1 = owner_op.stats()
    d = {k: st1[k] - st0[k] for k in st1}
    launches = d["kernel_launches"] + (so1["kernel_launches"] - so0["kernel_launches"] if local_op is not None else 0)
    tot = torch.tensor([launches, rows_out, d["rows_in"]], dtype=torch.int64, device=device)
    dist.all_reduce(tot)
    sent = ex_used.bytes_sent - sent0
    host_ms = {k: round(1e3 * v / max(K, 1), 4) for k, v in pipe.times.items()} if pipe is not None else None
    if pipe is not None:
        pipe.close()
    if native_ex is not None:
        native_ex.close()
    if plan is not None:
        plan.close()
    else:
        owner_op.close()
        part.close()
    torch.cuda.empty_cache()
    dog.close()
    return {"ms": ms, "d": d, "launches": int(tot[0].item()), "rows_out": int(tot[1].item()), "sent": sent,
            "clocks": clocks, "sums": sums, "pipelined": pipe is not None, "rows_out_warm": rows_out_warm,
            "host_ms_per_step": host_ms,
            "owner_ms": {"ingest_ms": (so1["ingest_ms"] - so0["ingest_ms"]) / max(K, 1),
                         "emit_ms": (so1["emit_ms"] - so0["emit_ms"]) / max(K, 1)} if local_op is not None else None}


class _Watchdog:
    """Fail fast instead of hanging: a collective whose peer never arrives blocks for ever (and takes the other ranks
    with it).  `beat()` is called from the step loop and the owner stage; if nothing beats for `limit_s` the process
    says where it stood and exits -- the launcher then tears the job down."""

    def __init__(self, rank, what, limit_s=240.0):
        import threading
        import time
        self.rank, self.what, self.limit_s = rank, what, limit_s
        self.last = time.monotonic()
        self.note = "start"
        self.stop = False
        self.t = threading.Thread(target=self._run, daemon=True)
        self.t.start()

    def beat(self, note):
        import time
        self.last = time.monotonic()
        self.note = note

    def _run(self):
        import os
        import sys
        import time
        while not self.stop:
            time.sleep(1.0)
            if time.monotonic() - self.last > self.limit_s:
                print(f"[arroyo_b200] rank {self.rank}: no progress for {self.limit_s:.0f} s in {self.what} "
                      f"(last: {self.note}); giving up.  Python stacks of every thread:", file=sys.stderr, flush=True)
                try:
                    import faulthandler
                    faulthandler.dump_traceback(file=sys.stderr, all_threads=True)  # which call each thread sits in
                except Exception:
                    pass
                sys.stderr.flush()
                os._exit(124)

    def close(self):
        self.stop = True


def _gather_window_sums(torch, dist, device, sums):
    """Sums the per-window checksums over the ranks (keys are disjoint across owners, so a window's global
    checksum is the sum of the owners').  Every rank emits the same windows (same effective watermarks)."""
    ws_sorted = sorted(sums)
    n = torch.tensor([len(ws_sorted)], dtype=torch.int64, device=device)
    nmax = n.clone()
    dist.all_reduce(nmax, op=dist.ReduceOp.MAX)
    nmin = n.clone()
    dist.all_reduce(nmin, op=dist.ReduceOp.MIN)
    if int(nmax.item()) != int(nmin.item()):
        return None, f"ranks emitted different numbers of windows ({int(nmin.item())}..{int(nmax.item())})"
    if not ws_sorted:
        return {}, None
    ints = torch.tensor([[ws, sums[ws][0], sums[ws][1], sums[ws][2], (sums[ws][3] + (1 << 63)) % (1 << 64) - (1 << 63)]
                         for ws in ws_sorted], dtype=torch.int64, device=device)
    flt = torch.tensor([sums[ws][4] for ws in ws_sorted], dtype=torch.float64, device=device)
    first = ints[:, :2].clone()
    dist.broadcast(first, src=0)
    same = torch.tensor([int(torch.equal(first, ints[:, :2]))], dtype=torch.int64, device=device)
    dist.all_reduce(same, op=dist.ReduceOp.MIN)
    if int(same.item()) != 1:
        return None, "ranks emitted different windows"
    acc = ints[:, 2:].clone()
    dist.all_reduce(acc)  # int64 adds wrap: the sum checksum stays a wrapping sum
    dist.all_reduce(flt)
    out = {}
    for i, ws in enumerate(ws_sorted):
        out[ws] = (sums[ws][0], int(acc[i, 0].item()), int(acc[i, 1].item()), int(acc[i, 2].item()) & ((1 << 64) - 1),
                   float(flt[i].item()))
    return out, None


def bench(args, torch, dist, rank, world, local, all_cpus=None):
    """Weak scaling: every GPU ingests its own 16 Mi-row/pane shard of the stream.

    --shuffle partials (default): partial -> shuffle -> final.  Each GPU pre-aggregates its shard per pane
        (the same ingest kernel), and when a pane can no longer receive rows its partial rows
        (key, sum, count) are hash-partitioned on the device and exchanged with an NCCL all-to-all; the
        owner of a key merges the partials into its sliding-window state and emits.  Same results as
        shuffling raw rows (SURVEY.md 8(e): combiner), 1/16 of the bytes over NVLink.
    --shuffle rows: the reference's plan shape -- raw rows are partitioned and exchanged, each GPU
        aggregates only the keys it owns."""
    import json
    import os
    import sys

    import arroyo_b200 as ab
    import bench as B
    from . import operators as native

    device = torch.device("cuda", local)
    # torch, NCCL's ordering, the partitioner and the owner stage share the explicit stream bench.py installed
    # (passing the legacy default stream's handle, 0, would make every native handle create a private stream)
    assert torch.cuda.current_stream().cuda_stream != 0
    # the combiner pipeline closes panes `lag` rounds late: that many more warm-up panes reach the steady state
    W, K = B.steady_warmup(args.warmup, extra=2), args.steps
    rows = args.rows_per_pane
    mode = args.shuffle
    gen_pane = B.make_generator(torch, device, rows, args.keys, args.dist, 42 + rank, args.keyspace)
    panes = [gen_pane(p) for p in range(W + K)]
    job = getattr(args, "_dog", None)
    beat = job.beat if job is not None else (lambda note: None)
    beat("input generated; timed plan")
    res = _run_plan(args, torch, dist, B, ab, native, rank, world, local, device, panes, W, K)
    beat("timed plan done")
    del panes
    ms, d = res["ms"], res["d"]

    e2e = None
    if mode == "partials" and not args.skip_e2e:
        # repeated like the single-GPU pass (the host links are shared with the box's other tenants): median reported
        Ke = args.e2e_steps or min(args.steps, 6)
        feed = B.host_feed(torch, gen_pane, range(13 + Ke), rows)
        trials = []
        for i in range(max(1, args.e2e_trials)):
            beat(f"end-to-end pass {i}")
            trials.append(_e2e_partials(args, torch, dist, B, ab, native, rank, world, local, device, gen_pane, feed=feed))
        trials.sort(key=lambda r: r["value"])
        e2e = dict(trials[len(trials) // 2])
        e2e["trials"] = [round(r["value"]) for r in trials]
        e2e["host_buffers"] = "pinned"
        del feed

    # ---- verify: the same N-GPU plan over the panes the oracle consumes on rank 0 (union of the shards) ----
    verify = cpu = None
    if not args.skip_cpu:
        VP = B.WIDTH // B.SLIDE + 6
        beat("CPU baseline on rank 0 (the other ranks wait for its sample size)")
        n_rows = torch.zeros(1, dtype=torch.int64, device=device)
        if rank == 0:
            if all_cpus:
                os.sched_setaffinity(0, all_cpus)
            cpu = B.run_cpu(torch, args, device, budget_s=40.0, warm_panes=VP - 2, timed_panes=2,
                            seeds=tuple(42 + r for r in range(world)))
            n_rows[0] = cpu["rows_per_step"]
        dist.broadcast(n_rows, src=0)
        vrows = int(n_rows.item())
        beat("verification pass")
        vp = [B.sample_pane(torch, device, gen_pane(p), vrows) for p in range(VP)]
        vres = _run_plan(args, torch, dist, B, ab, native, rank, world, local, device, vp, VP, 0, collect=True)
        del vp
        merged, err = _gather_window_sums(torch, dist, device, vres["sums"])
        if rank == 0:
            if err:
                verify = {"verified": False, "mismatches": [err]}
            else:
                verify = B.compare_windows(merged, cpu["windows"], min_windows=VP - 7)
            verify["rows_per_pane_per_gpu"] = vrows
            verify["panes"] = VP
            verify["plan"] = f"{world} GPUs, --shuffle {mode}: window checksums summed over the owners (all-reduce)"

    if rank == 0:
        peak, peak_kind = B.measured_peak()
        ingest_gbs = 24.0 * d["ingest_rows_timed"] / (d["ingest_ms"] * 1e-3) / 1e9 if d["ingest_ms"] else None
        out = {"metric": "rows/sec sliding-window SUM (1M keys)", "value": world * K * rows / (ms * 1e-3),
               "unit": "rows/s", "n_gpus": world, "steps": K, "warmup": W, "warmup_requested": args.warmup,
               "ms_per_step": ms / K,
               "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "int64", "data": "synthetic",
               "config": B.workload_config(args, world),
               "impl": {"shuffle": ("partial aggregates per pane (partial -> shuffle -> final)" if mode == "partials"
                                    else "raw rows (reference plan shape)"),
                        "exchange": (None if mode != "partials" or args.sync_plan else
                                     "one C call per round: device partition + ncclAllGather of the control records + grouped "
                                     "ncclSend / ncclRecv (csrc/exchange.cu)" if getattr(args, "native_exchange", False) else
                                     "torch.distributed all_gather + all_to_all_single"),
                        "numa": getattr(args, "numa", None),
                        "warmup_note": "warm-up = max(--warmup, width/slide + 5) panes: the timed steps see the steady state"},
               "plan": (None if mode != "partials" else
                        "local stage and shuffle+owner stage on two host threads, watermarks ride on the data rounds, "
                        "local stage closes panes 2 rounds behind (LaggedCombiner)" if res["pipelined"] else
                        "synchronous: watermark exchange, local close, shuffle, owner stage in sequence"),
               "rows_out_per_step": res["rows_out"] / max(K, 1), "gpu_launches": res["launches"],
               "roofline": {"bound": "hbm", "kernel": "ingest",
                            "achieved": round(ingest_gbs, 1) if ingest_gbs else None, "peak": peak,
                            "peak_kind": peak_kind, "unit": "GB/s",
                            "frac": round(ingest_gbs / peak, 4) if ingest_gbs else None,
                            "traffic": None,
                            "algorithmic_bytes_per_launch": 24.0 * d["ingest_rows_timed"] / max(d["ingest_launches"], 1),
                            "note": "rank 0's raw-row ingest kernel"},
               "host_ms_per_step": res["host_ms_per_step"], "owner_stage_kernel_ms_per_step": res["owner_ms"],
               "local_stage_kernel_ms_per_step": {"ingest_ms": d["ingest_ms"] / max(K, 1), "emit_ms": d["emit_ms"] / max(K, 1)},
               "e2e": e2e, "clocks": res["clocks"],
               "shuffle_bytes_sent_per_step_per_gpu": res["sent"] // max(K, 1)}
        if cpu is not None:
            out["cpu_baseline"] = {"value": cpu["rows_per_s"], "unit": "rows/s", "cores": cpu["threads"], "kind": "port",
                                   "sample": cpu["sample"]}
            out["verify"] = verify
            out["verified"] = verify["verified"]
        print(json.dumps(out), flush=True)
    beat("done; final barrier")
    dist.barrier()
    dist.destroy_process_group()
    if job is not None:
        job.close()
    if rank == 0 and verify is not None and not verify["verified"]:
        sys.exit("bench.py: GPU windows differ from the oracle's -- see the verify block of the line above")
