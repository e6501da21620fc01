"""Row-range sharding of one batch across the GPUs of a box (SURVEY.md §8e).

Rows are independent, so a Projector needs no exchange at all and a Filter needs exactly one:
reassembling the SelectionVector.  Each rank filters its contiguous row range and emits GLOBAL
row numbers (`index_base` = first row of the range); because ranges are contiguous and each
run is ascending, concatenating the runs in rank order gives the global ascending vector.
`torch.distributed` is plumbing only (NCCL on GPUs, gloo in the CPU tests)."""
from __future__ import annotations

from typing import Optional, Tuple

import torch
import torch.distributed as dist


def shard_range(num_rows: int, world: int, rank: int, align: int = 64) -> Tuple[int, int]:
    """[first, last) rows of `rank`.  Range starts are multiples of `align` rows so that no two
    shards share a validity-bitmap word and value loads stay 128-byte aligned."""
    per = (num_rows + world - 1) // world
    per = (per + align - 1) // align * align
    first = min(rank * per, num_rows)
    return first, min(first + per, num_rows)


def shard_rows_with_root(total_rows: int, world: int, selectivity: float, bytes_per_row: float, index_bytes: int = 8,
                         write_cost: float = 2.0, align: int = 64) -> list:
    """Row counts per rank (contiguous ranges, in rank order, summing to total_rows) for a Filter whose
    SelectionVector is reassembled on rank 0.  The root streams its own rows AND absorbs the other ranks'
    runs — (world-1) x selectivity x index_bytes per row of a shard, each incoming byte costing the memory
    system about `write_cost` streamed bytes (2.0 by default, DESIGN.md §4) — so with equal ranges every
    step waits for it.  The root's range is shortened until all ranks finish together.  Every range but the
    last is a multiple of `align` rows (no two shards share a validity-bitmap word)."""
    if world <= 1:
        return [total_rows]
    per = total_rows / world
    delta = write_cost * index_bytes * selectivity * (world - 1) / bytes_per_row
    r_root = max(align, int(per * (1.0 - delta * (world - 1) / world)) // align * align)
    r_other = ((total_rows - r_root) // (world - 1)) // align * align
    return [r_root] + [r_other] * (world - 2) + [total_rows - r_root - r_other * (world - 2)]


def wave_layout(shard_rows: list, waves: int, align: int = 1024):
    """Row slices for a batch that is filtered in `waves` waves (PeerSelection(waves=...)).
    Rank r's shard of shard_rows[r] rows is cut into `waves` slices (all but the last a multiple of `align`
    rows); the GLOBAL row order is wave-major — every rank's slice 0 in rank order, then every rank's
    slice 1, ... — so that the runs of one wave are contiguous in the SelectionVector and a wave can be
    pushed as soon as it is filtered.  Returns (rows, first): rows[r][j] = size of rank r's slice j,
    first[r][j] = its first global row (the Filter call's index_base)."""
    world = len(shard_rows)
    rows = []
    for n in shard_rows:
        per = (n // waves) // align * align
        if per == 0:
            rows.append([n] + [0] * (waves - 1))
        else:
            rows.append([per] * (waves - 1) + [n - per * (waves - 1)])
    first = [[0] * waves for _ in range(world)]
    g = 0
    for j in range(waves):
        for r in range(world):
            first[r][j] = g
            g += rows[r][j]
    return rows, first


def gather_selection(local_indices: torch.Tensor, count: int, dst: int = 0,
                     group: Optional[dist.ProcessGroup] = None,
                     out: Optional[torch.Tensor] = None) -> Tuple[Optional[torch.Tensor], int]:
    """Gather every rank's first `count` entries of `local_indices` onto rank `dst`, in rank
    order.  One all-gather of the counts, then variable-length point-to-point transfers of the
    index runs straight into their final position (no padding to the maximum count).
    Returns (global vector on dst | None elsewhere, total count)."""
    world = dist.get_world_size(group)
    rank = dist.get_rank(group)
    dev = local_indices.device
    counts = torch.zeros(world, dtype=torch.int64, device=dev)
    mine = torch.tensor([count], dtype=torch.int64, device=dev)
    dist.all_gather_into_tensor(counts, mine, group=group)
    c = [int(x) for x in counts.tolist()]
    total = sum(c)
    if rank == dst:
        if out is None or out.numel() < total:
            out = torch.empty(max(total, 1), dtype=local_indices.dtype, device=dev)
        ops, off = [], 0
        for r in range(world):
            if r == dst:
                out[off: off + c[r]].copy_(local_indices[: c[r]])
            elif c[r] > 0:
                ops.append(dist.P2POp(dist.irecv, out[off: off + c[r]], r, group))
            off += c[r]
        if ops:
            for w in dist.batch_isend_irecv(ops):
                w.wait()
        return out[:total], total
    if count > 0:
        for w in dist.batch_isend_irecv([dist.P2POp(dist.isend, local_indices[:count].contiguous(), dst, group)]):
            w.wait()
    return None, total


class PeerGather:
    """SelectionVector gather without SMs: every rank writes its index run straight into rank
    `dst`'s buffer over NVLink with the copy engines (peer memory mapped through CUDA IPC), so
    the transfer runs underneath the persistent filter kernel of the next batch -- an NCCL
    send/recv kernel cannot (it finds no free CTA slot until the filter kernel ends).
    Counts travel host-side over a gloo group; the data never touches the host.

    Protocol per batch: `start(local, count)` -> all-gather of counts (gloo), then one async
    device-to-peer copy at this rank's prefix offset on `copy_stream`; `finish()` -> every rank
    waits for its own copy, then a gloo barrier tells `dst` that the vector is complete."""

    def __init__(self, capacity: int, dtype: torch.dtype, device: torch.device, dst: int = 0):
        from torch.multiprocessing.reductions import reduce_tensor
        self.rank, self.world, self.dst = dist.get_rank(), dist.get_world_size(), dst
        self.device = device
        self.cpu_group = dist.new_group(backend="gloo")
        self.copy_stream = torch.cuda.Stream(device)
        self.done = torch.cuda.Event()
        self.buf = None
        payload = [None]
        if self.rank == dst:
            self.buf = torch.empty(capacity, dtype=dtype, device=device)
            fn, args = reduce_tensor(self.buf)
            payload = [(fn, args)]
        dist.broadcast_object_list(payload, src=dst, group=self.cpu_group)
        if self.rank != dst:
            fn, args = payload[0]
            self.buf = fn(*args)          # rank dst's memory, mapped into this process
        self.total = 0
        self._pending = False

    def start(self, local: torch.Tensor, count: int, after: Optional[torch.cuda.Event] = None) -> int:
        # plain CPU tensors over gloo (the *_object collectives pickle and take milliseconds)
        mine = torch.tensor([int(count)], dtype=torch.int64)
        gathered = [torch.zeros(1, dtype=torch.int64) for _ in range(self.world)]
        dist.all_gather(gathered, mine, group=self.cpu_group)
        counts = [int(t[0]) for t in gathered]
        off = sum(counts[: self.rank])
        self.total = sum(counts)
        if self.total > self.buf.numel():
            raise RuntimeError("PeerGather capacity %d < %d selected rows" % (self.buf.numel(), self.total))
        with torch.cuda.stream(self.copy_stream):
            if after is not None:
                self.copy_stream.wait_event(after)
            if count > 0:
                self.buf[off: off + count].copy_(local[:count], non_blocking=True)
            self.done.record(self.copy_stream)
        self._pending = True
        return self.total

    def finish(self) -> Optional[torch.Tensor]:
        """Blocks the host until every rank's run has landed; returns the vector on `dst`."""
        if self._pending:
            self.done.synchronize()
            flag = torch.ones(1, dtype=torch.int32)
            dist.all_reduce(flag, group=self.cpu_group)   # acts as the barrier
            self._pending = False
        return self.buf[: self.total] if self.rank == self.dst else None


class PeerSelection:
    """SelectionVector reassembly with no host in the loop (C-ABI `gdv_selection_push`).

    Rank 0 (the root) owns a ring of `slots` SelectionVector buffers and a small "board" of
    64-bit words; both are mapped into every other rank through CUDA IPC (`gdv_ipc_export` /
    `gdv_ipc_open`: opened with the rank's own device current, which also enables NVLink peer
    access to the root GPU).  Per step:

      * every rank runs its Filter on its row range (`index_base` = first row).  The root writes
        straight into the step's vector (its run starts at offset 0, bounded by the vector's
        capacity: GDV_SEL_BOUNDED); the other ranks write a local run;
      * on a side stream, ordered after the filter kernel by an event, `gdv_selection_push`
        publishes the rank's count on the board, reads the lower ranks' counts from it and stores
        the run at its final offset in the root's vector over NVLink.  The filter is built with
        `sm_reserve` so this copy kernel finds free SMs while the NEXT batch's filter kernel runs;
      * the root's push call waits (on the device) for every rank's `done` word and writes the
        total count next to the vector.

    Nothing is synchronised through the host; `torch.distributed` (gloo) is used once, at
    construction, to hand the IPC handles around.

    `waves` > 1: a step's batch is filtered in `waves` row slices (wave-major global row order: all
    ranks' slice 0, then all ranks' slice 1, ...; `wave_rows`) and each slice's run is pushed while the
    next slice is being filtered, so only the LAST slice's transfer is not hidden.  Every rank, the root
    included, then writes local runs (two buffers, alternating) and the push kernel carries the vector's
    fill level from wave to wave in a device word (`gdv_selection_push`'s d_base)."""

    def __init__(self, capacity: int, local_rows: int, mode: str, device: torch.device,
                 slots: int = 2, ctas: int = 8, root: int = 0, waves: int = 1):
        import ctypes as C
        import gandiva_b200 as gandiva
        assert root == 0, "the root is rank 0 (its run has offset 0 and is written in place)"
        self.g = gandiva
        self.rank, self.world = dist.get_rank(), dist.get_world_size()
        assert self.world <= gandiva.GDV_BOARD_MAX_WORLD and 1 <= slots <= gandiva.GDV_BOARD_SLOTS
        self.device, self.slots, self.ctas = device, slots, ctas
        self.waves = int(waves)
        assert self.waves >= 1
        self.mode = mode
        self.dtype = {"UINT16": torch.int16, "UINT32": torch.int32, "UINT64": torch.int64}[mode]
        self.capacity = int(capacity)
        self.cpu_group = dist.new_group(backend="gloo")
        payload = [None]
        self._opened = []
        if self.rank == 0:
            self.vectors = [torch.empty(self.capacity, dtype=self.dtype, device=device) for _ in range(slots)]
            self.board = torch.zeros(gandiva.GDV_BOARD_BYTES // 8, dtype=torch.int64, device=device)
            torch.cuda.synchronize(device)
            handles = []
            for t in self.vectors + [self.board]:
                h = C.create_string_buffer(64)
                off = C.c_int64()
                gandiva._check(gandiva.lib.gdv_ipc_export(device.index, t.data_ptr(), h, C.byref(off)))
                handles.append((h.raw, off.value))
            payload = [handles]
            self.vector_ptrs = [t.data_ptr() for t in self.vectors]
            self.board_ptr = self.board.data_ptr()
        dist.broadcast_object_list(payload, src=0, group=self.cpu_group)
        if self.rank != 0:
            ptrs = []
            seen = {}
            for raw, off in payload[0]:   # several tensors may live in one exported allocation
                if raw not in seen:
                    p = C.c_void_p()
                    gandiva._check(gandiva.lib.gdv_ipc_open(device.index, raw, 0, C.byref(p)))
                    seen[raw] = p.value
                    self._opened.append(p.value)
                ptrs.append(seen[raw] + off)
            self.vector_ptrs, self.board_ptr = ptrs[:-1], ptrs[-1]
        if self.waves > 1:      # local_rows = the largest slice; runs alternate between two buffers
            self.local = [torch.empty(local_rows, dtype=self.dtype, device=device) for _ in range(2)]
            self.ev_wave = [torch.cuda.Event() for _ in range(2)]
            self.wave_counts = [torch.zeros(1, dtype=torch.int64, device=device) for _ in range(2)]
            self.base = torch.zeros(1, dtype=torch.int64, device=device)
        elif self.rank != 0:
            self.local = [torch.empty(local_rows, dtype=self.dtype, device=device) for _ in range(slots)]
        self.counts = [torch.zeros(1, dtype=torch.int64, device=device) for _ in range(slots)]
        self.totals = [torch.zeros(1, dtype=torch.int64, device=device) for _ in range(slots)]
        self.local_ctr = torch.zeros(1, dtype=torch.int64, device=device)
        self.side = torch.cuda.Stream(device)
        self.ev_filter = [torch.cuda.Event() for _ in range(slots)]
        self.ev_pushed = [torch.cuda.Event() for _ in range(slots)]
        self.local_rows = int(local_rows)
        self.ctas_issued = 0
        torch.cuda.synchronize(device)
        dist.barrier(group=self.cpu_group)

    def close(self) -> None:
        torch.cuda.synchronize(self.device)
        dist.barrier(group=self.cpu_group)
        for p in self._opened:
            self.g.lib.gdv_ipc_close(self.device.index, p, 0)
        self._opened = []
        dist.barrier(group=self.cpu_group)

    def filter_target(self, step: int, wave: int = 0):
        """(device pointer, max_slots, mode string, count pointer) for the Filter call of this step (and wave)."""
        if self.waves > 1:
            lb = (step * self.waves + wave) % 2
            return self.local[lb].data_ptr(), self.local_rows, self.mode, self.wave_counts[lb].data_ptr()
        b = step % self.slots
        if self.rank == 0:
            return self.vector_ptrs[b], self.capacity, self.mode + "|BOUNDED", self.counts[b].data_ptr()
        return self.local[b].data_ptr(), self.local_rows, self.mode, self.counts[b].data_ptr()

    def before_filter(self, step: int, stream: torch.cuda.Stream, wave: int = 0) -> None:
        """The buffers the Filter is about to write are free again once the push that last read them has finished."""
        if self.waves > 1:
            w = step * self.waves + wave
            if w >= 2:
                stream.wait_event(self.ev_wave[w % 2])
            return
        if step >= self.slots:
            stream.wait_event(self.ev_pushed[step % self.slots])

    def after_filter(self, step: int, stream: torch.cuda.Stream, ctas: int = 0, wave: int = 0) -> None:
        """Enqueue the push of this step's (wave's) run (and, on the root, the wait for all runs).
        `ctas` overrides the copy kernel's grid for this call (e.g. the whole GPU for the last
        push of a job, when no filter kernel follows)."""
        g, b = self.g, step % self.slots
        ctas = ctas or self.ctas
        self.ctas_issued += ctas
        if self.waves > 1:
            w = step * self.waves + wave
            lb, seq = w % 2, w + 1
            first, last = wave == 0, wave == self.waves - 1
            self.ev_wave[lb].record(stream)
            self.side.wait_event(self.ev_wave[lb])
            need = step + 1 - self.slots if (first and self.rank != 0 and step >= self.slots) else 0
            g._check(g.lib.gdv_selection_push(
                self.device.index, self.local[lb].data_ptr(), self.wave_counts[lb].data_ptr(), self.vector_ptrs[b],
                self.capacity, self.board_ptr, seq % g.GDV_BOARD_SLOTS, self.rank, self.world, seq, need,
                g._SEL_MODE[self.mode], ctas, self.local_ctr.data_ptr(), self.ctas_issued, self.totals[b].data_ptr(),
                self.base.data_ptr(), (g.GDV_WAVE_FIRST if first else 0) | (g.GDV_WAVE_LAST if last else 0), b,
                g._stream_handle(self.side.cuda_stream)))
            if self.rank == 0 and last:
                g._check(g.lib.gdv_selection_release(self.device.index, self.board_ptr, b, step + 1,
                                                     g._stream_handle(self.side.cuda_stream)))
            self.ev_wave[lb].record(self.side)
            if last:
                self.ev_pushed[b].record(self.side)
            return
        seq = step + 1
        self.ev_filter[b].record(stream)
        self.side.wait_event(self.ev_filter[b])
        need = seq - self.slots if (self.rank != 0 and seq > self.slots) else 0
        src = self.vector_ptrs[b] if self.rank == 0 else self.local[b].data_ptr()
        g._check(g.lib.gdv_selection_push(
            self.device.index, src, self.counts[b].data_ptr(), self.vector_ptrs[b], self.capacity,
            self.board_ptr, b, self.rank, self.world, seq, need, g._SEL_MODE[self.mode], ctas,
            self.local_ctr.data_ptr(), self.ctas_issued, self.totals[b].data_ptr(), None, 0, 0,
            g._stream_handle(self.side.cuda_stream)))
        if self.rank == 0:
            # bench / tests have no consumer: the vector is released as soon as it is complete
            g._check(g.lib.gdv_selection_release(self.device.index, self.board_ptr, b, seq,
                                                 g._stream_handle(self.side.cuda_stream)))
        self.ev_pushed[b].record(self.side)

    def finish(self, stream: torch.cuda.Stream) -> None:
        """Make `stream` wait for every push issued so far."""
        for e in self.ev_pushed + (self.ev_wave if self.waves > 1 else []):
            stream.wait_event(e)

    def result(self, step: int):
        """Root only, after synchronisation: (vector, total) of `step`."""
        b = step % self.slots
        total = int(self.totals[b].item())
        return self.vectors[b][:min(total, self.capacity)], total

    def overflowed(self) -> bool:
        """Root only: some step's runs did not fit the vector's capacity."""
        g = self.g
        return bool(self.board[2 * g.GDV_BOARD_SLOTS * g.GDV_BOARD_MAX_WORLD + g.GDV_BOARD_SLOTS].item() != 0)
