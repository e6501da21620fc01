"""gdv_sel_push on ONE GPU: a single rank in wave mode copies its own run into the vector (HBM -> HBM), which is the
kernel's copy loop without the link.  Timed with CUDA events for 8 and 264 CTAs (two per H100 SM); run under
`ncu -k gdv_sel_push --set full` for the instruction / memory profile of that loop.
The NVLink side of the same loop is tools/p2p_store_bench.cu."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

import gandiva_b200 as g  # noqa: E402

n = int(sys.argv[1]) if len(sys.argv) > 1 else 64 * 1024 * 1024
dev = torch.device("cuda", 0)
src = torch.arange(n, dtype=torch.int64, device=dev)
dst = torch.empty(n + 16, dtype=torch.int64, device=dev)
cnt = torch.tensor([n], dtype=torch.int64, device=dev)
board = torch.zeros(g.GDV_BOARD_BYTES // 8, dtype=torch.int64, device=dev)
ctr = torch.zeros(1, dtype=torch.int64, device=dev)
base = torch.zeros(1, dtype=torch.int64, device=dev)
total = torch.zeros(1, dtype=torch.int64, device=dev)
stream = torch.cuda.current_stream().cuda_stream
issued, seq = 0, 0
for ctas in (8, 8, 264, 264):
    issued += ctas
    seq += 1
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    g._check(g.lib.gdv_selection_push(0, src.data_ptr(), cnt.data_ptr(), dst.data_ptr(), n + 16, board.data_ptr(),
                                      seq % g.GDV_BOARD_SLOTS, 0, 1, seq, 0, g.GDV_SEL_UINT64, ctas, ctr.data_ptr(), issued,
                                      total.data_ptr(), base.data_ptr(), g.GDV_WAVE_FIRST | g.GDV_WAVE_LAST, 0,
                                      g._stream_handle(stream)))
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1)
    ok = bool(torch.equal(dst[:n], src)) and int(total.item()) == n
    print("ctas %3d: %.3f ms, %.0f GB/s read + %.0f GB/s written, copy %s" % (ctas, ms, n * 8 / ms / 1e6, n * 8 / ms / 1e6,
                                                                           "ok" if ok else "WRONG"), flush=True)
    dst.zero_()
