"""The device-side protocol of gdv_selection_push (SURVEY.md §8(e): the one exchange a sharded Filter needs),
exercised on ONE GPU: `world` virtual ranks, each with its own stream, local run buffers, counter and base
word, share a board and a root vector in the same HBM.  The kernels are the ones the multi-GPU path
launches (there the board and the vector are CUDA-IPC mappings of the root's memory and the stores cross
NVLink; tests/peer_push_worker.py covers that on boxes with >= 2 GPUs).  Checked element-wise against an
independent torch evaluation of the Q6 predicate in the layout's global row order."""
import numpy as np
import pytest

import cases
import devmem
from gandiva_b200.sharding import shard_rows_with_root, wave_layout

pytestmark = pytest.mark.gpu


class _Stream:
    """A torch CUDA stream on a GPU box; the simulator has one (synchronous) stream."""

    def __init__(self):
        if devmem.EMU:
            self.t, self.handle = None, 0
        else:
            import torch
            self.t = torch.cuda.Stream(torch.device("cuda", 0))
            self.handle = self.t.cuda_stream

    def wait(self, ev):
        if self.t is not None and ev[0] is not None:
            self.t.wait_event(ev[0])

    def record(self, ev):
        if self.t is not None:
            import torch
            ev[0] = torch.cuda.Event()
            ev[0].record(self.t)


def _run(gandiva, world, waves, steps, shard_rows, ctas=2, slots=2):
    g = gandiva
    total_rows = sum(shard_rows)
    rows, first = wave_layout(shard_rows, waves) if waves > 1 else ([[n] for n in shard_rows],
                                                                    [[sum(shard_rows[:r])] for r in range(world)])
    b = g.TreeExprBuilder()
    filt = [g.make_filter(cases.Q6_SCHEMA, b.make_condition(cases.q6_condition(b)), g.Configuration(device=0, sm_reserve=4))
            for _ in range(world)]
    # Everything a rank will launch is launched once and waited for BEFORE any rank waits for another on the
    # device: the first launch of a kernel loads its module (CUDA loads lazily), and a module load that has to
    # wait for the device would wait forever behind a push kernel that is itself waiting for that rank.
    warm = [devmem.DevBuf(4096, np.int32), devmem.DevBuf(4096, np.float64), devmem.DevBuf(4096, np.float64),
            devmem.DevBuf(4096, np.int64), devmem.DevBuf(1, np.int64, fill=0)]
    for kind, t in ((0, warm[0]), (1, warm[1]), (2, warm[2])):
        g.generate_lineitem(0, kind, 1, 0, 4096, t.ptr, 0, 0, 0)
    for f in filt:
        f.evaluate_device(4096, [(0, warm[0].ptr, 0, 0), (0, warm[1].ptr, 0, 0), (0, warm[2].ptr, 0, 0)], warm[3].ptr,
                          4096, "UINT64", 0, warm[4].ptr, sync=True)
    wb = devmem.DevBuf(g.GDV_BOARD_BYTES // 8, np.int64, fill=0)
    wc = devmem.DevBuf(1, np.int64, fill=0)
    g._check(g.lib.gdv_selection_push(0, warm[3].ptr, warm[4].ptr, warm[3].ptr, 4096, wb.ptr, 0, 0, 1, 1, 0,
                                      g.GDV_SEL_UINT64, 1, wc.ptr, 1, None, None, 0, 0, None))
    g._check(g.lib.gdv_selection_release(0, wb.ptr, 0, 1, None))
    devmem.synchronize()
    cap = int(total_rows * 0.05) + 1024
    vectors = [devmem.DevBuf(cap, np.int64, fill=-1) for _ in range(slots)]
    board = devmem.DevBuf(g.GDV_BOARD_BYTES // 8, np.int64, fill=0)
    streams = [_Stream() for _ in range(world)]
    sides = [_Stream() for _ in range(world)]
    max_slice = max(max(r) for r in rows)
    ship = [devmem.DevBuf(shard_rows[r], np.int32) for r in range(world)]
    disc = [devmem.DevBuf(shard_rows[r], np.float64) for r in range(world)]
    qty = [devmem.DevBuf(shard_rows[r], np.float64) for r in range(world)]
    local = [[devmem.DevBuf(max_slice, np.int64) for _ in range(2)] for _ in range(world)]
    counts = [[devmem.DevBuf(1, np.int64, fill=0) for _ in range(2)] for _ in range(world)]
    totals = [devmem.DevBuf(1, np.int64, fill=0) for _ in range(slots)]
    ctr = [devmem.DevBuf(1, np.int64, fill=0) for _ in range(world)]
    base = [devmem.DevBuf(1, np.int64, fill=0) for _ in range(world)]
    issued = [0] * world
    ev = [[[None], [None]] for _ in range(world)]
    for step in range(steps):
        seed = 42 + step
        vslot = step % slots
        for j in range(waves):
            for r in range(world):      # one rank after the other ENQUEUES; the kernels of different ranks overlap
                st = streams[r].handle
                w = step * waves + j
                lb = w % 2
                n, f0 = rows[r][j], first[r][j]
                lo = sum(rows[r][:j])
                streams[r].wait(ev[r][lb])          # the push that last read local[lb] is done
                for kind, t, sz in ((0, ship[r], 4), (1, disc[r], 8), (2, qty[r], 8)):
                    g.generate_lineitem(0, kind, seed, f0, n, t.ptr + lo * sz, 0, 0, st)
                cols = [(0, ship[r].ptr + 4 * lo, 0, 0), (0, disc[r].ptr + 8 * lo, 0, 0), (0, qty[r].ptr + 8 * lo, 0, 0)]
                in_place = waves == 1 and r == 0
                if in_place:
                    filt[r].evaluate_device(n, cols, vectors[vslot].ptr, cap, "UINT64|BOUNDED", st,
                                            counts[r][lb].ptr, sync=False, index_base=f0)
                else:
                    filt[r].evaluate_device(n, cols, local[r][lb].ptr, max_slice, "UINT64", st,
                                            counts[r][lb].ptr, sync=False, index_base=f0)
                streams[r].record(ev[r][lb])
                sides[r].wait(ev[r][lb])
                issued[r] += ctas
                seq = w + 1
                src = vectors[vslot].ptr if in_place else local[r][lb].ptr
                flags = (g.GDV_WAVE_FIRST if j == 0 else 0) | (g.GDV_WAVE_LAST if j == waves - 1 else 0)
                need = step + 1 - slots if (j == 0 and r != 0 and step >= slots) else 0
                g._check(g.lib.gdv_selection_push(
                    0, src, counts[r][lb].ptr, vectors[vslot].ptr, cap, board.ptr,
                    (seq % g.GDV_BOARD_SLOTS) if waves > 1 else vslot, r, world, seq, need, g.GDV_SEL_UINT64, ctas,
                    ctr[r].ptr, issued[r], totals[vslot].ptr,
                    base[r].ptr if waves > 1 else None, flags if waves > 1 else 0, vslot,
                    g._stream_handle(sides[r].handle)))
                if r == 0 and j == waves - 1:
                    g._check(g.lib.gdv_selection_release(0, board.ptr, vslot, step + 1, g._stream_handle(sides[r].handle)))
                sides[r].record(ev[r][lb])
        devmem.synchronize()
        # the columns now hold this step's rows: the expected vector in the layout's global row order
        want = []
        cols_h = [(ship[r].numpy(), disc[r].numpy(), qty[r].numpy()) for r in range(world)]
        for j in range(waves):
            for r in range(world):
                lo, n = sum(rows[r][:j]), rows[r][j]
                sh, di, qt = (c[lo:lo + n] for c in cols_h[r])
                m = (sh >= 8766) & (sh < 9131) & (di >= 0.05) & (di <= 0.07) & (qt < 24)
                want.append(np.nonzero(m)[0].astype(np.int64) + first[r][j])
        expect = np.concatenate(want)
        total = int(totals[vslot].numpy()[0])
        assert total == len(expect), (step, total, len(expect))
        assert np.array_equal(vectors[vslot].numpy()[:total], expect), "step %d" % step
        if waves > 1:
            assert all(int(x.numpy()[0]) == total for x in base)
    err = int(board.numpy()[2 * g.GDV_BOARD_SLOTS * g.GDV_BOARD_MAX_WORLD + g.GDV_BOARD_SLOTS])
    assert err == 0
    for f in filt:
        f.sync(0)


import os  # noqa: E402

# Several virtual ranks on ONE device wait for each other inside kernels: that needs the kernels of several
# streams to be resident at the same time, which CUDA does not promise (and the CPU simulator runs one kernel
# at a time).  A test that could hang a GPU is therefore opt-in; the real multi-GPU path is
# tests/peer_push_worker.py.
needs_concurrency = pytest.mark.skipif(devmem.EMU or os.environ.get("GDV_TEST_VIRTUAL_RANKS") != "1",
                                       reason="opt-in: GDV_TEST_VIRTUAL_RANKS=1 (ranks wait for each other on one device)")


@needs_concurrency
@pytest.mark.timeout(60)
@pytest.mark.parametrize("world,waves", [(2, 1), (3, 1), (2, 4), (3, 3), (4, 2)])
def test_virtual_ranks_on_one_gpu(world, waves, gandiva):
    shard_rows = shard_rows_with_root(1_500_000 * world + 12_345, world, 0.0127, 20.0)
    _run(gandiva, world, waves, steps=5, shard_rows=shard_rows)


@pytest.mark.parametrize("waves", [1, 2, 5])
def test_single_rank_waves(waves, gandiva):
    """world = 1 (no waiting between ranks, so this one also runs under the simulator): the root's own waves
    land back to back and the base word carries the fill level."""
    _run(gandiva, 1, waves, steps=3, shard_rows=[700_003])
