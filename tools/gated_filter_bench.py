"""Gated loads of the fixed-width Filter, on and off (Configuration.filter_gating = 0 / 1), over the
synthetic lineitem columns resident in HBM (1e9 rows by default, generated on the device from seed 42 as
bench.py does).

    python tools/gated_filter_bench.py [--rows 1000000000] [--rounds 7] [--reps 3]

Workloads: Q6; Q6 with 1 % nulls in every column (bench configs q6_nulls); a dense-first Q6 whose
shipdate range [8035, 10562) keeps every row in the first stage (the worst case for gating); Q6 with
its conjuncts reversed (quantity first); and a conjunct that reads two columns,
`l_discount * 100 < l_quantity AND l_shipdate in [8766, 9131)`.

The two arms alternate, `--rounds` times each; a round times `--reps` launches with CUDA events around
each enqueued evaluate and keeps their median.  Prints one JSON line per workload with the median and the
spread (min, max over rounds) of each arm's kernel time, rows/s, the SelectionVectors' equality
(torch.equal), and the effective bytes per row of the gated kernel: its time times the bandwidth the
ungated kernel reached in the same run over its algorithmic bytes (20 B/row + 3 validity bits/row where
there are nulls + 4 B per selected row).  The card's name and power limit are read in the same run."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import pyarrow as pa
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import cases  # noqa: E402
import gandiva_b200 as gandiva  # noqa: E402


def card():
    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # the number is still reported, without the limit
        out = "power limit unavailable (%s)" % e
    return name, out


def condition(b, kind):
    sd, f, B = pa.date32(), pa.float64(), pa.bool_()
    ship, disc, qty = (cases.F(b, "l_shipdate", sd), cases.F(b, "l_discount", f), cases.F(b, "l_quantity", f))
    fn = b.make_function

    def ship_range(lo, hi):
        return [fn("greater_than_or_equal_to", [ship, b.make_literal(lo, sd)], B),
                fn("less_than", [ship, b.make_literal(hi, sd)], B)]
    disc_range = [fn("greater_than_or_equal_to", [disc, b.make_literal(0.05, f)], B),
                  fn("less_than_or_equal_to", [disc, b.make_literal(0.07, f)], B)]
    qty_lt = [fn("less_than", [qty, b.make_literal(24.0, f)], B)]
    if kind in ("q6", "q6_nulls"):
        return b.make_and(ship_range(8766, 9131) + disc_range + qty_lt)
    if kind == "dense_first":
        return b.make_and(ship_range(8035, 10562) + disc_range + qty_lt)
    if kind == "reversed":
        return b.make_and(qty_lt + disc_range[::-1] + ship_range(8766, 9131)[::-1])
    if kind == "two_column":
        scaled = fn("multiply", [disc, b.make_literal(100.0, f)], f)
        return b.make_and([fn("less_than", [scaled, qty], B)] + ship_range(8766, 9131))
    raise ValueError(kind)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1_000_000_000)
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    n = a.rows
    name, smi = card()
    dev = torch.device("cuda", 0)
    st = torch.cuda.current_stream().cuda_stream
    ship = torch.empty(n, dtype=torch.int32, device=dev)
    disc = torch.empty(n, dtype=torch.float64, device=dev)
    qty = torch.empty(n, dtype=torch.float64, device=dev)
    W = (n + 31) // 32
    vl = [torch.empty(W, dtype=torch.int32, device=dev) for _ in range(3)]
    outs = [torch.empty(n, dtype=torch.int32, device=dev) for _ in range(2)]
    cnts = [torch.zeros(1, dtype=torch.int64, device=dev) for _ in range(2)]
    b = gandiva.TreeExprBuilder()
    for kind in ("q6", "q6_nulls", "dense_first", "reversed", "two_column"):
        nulls = kind == "q6_nulls"
        for k, t, v in ((0, ship, vl[0]), (1, disc, vl[1]), (2, qty, vl[2])):
            gandiva.generate_lineitem(0, k, 42, 0, n, t.data_ptr(), v.data_ptr() if nulls else 0, 10 if nulls else 0, st)
        cols = [((v.data_ptr() if nulls else 0), t.data_ptr(), 0, 0) for t, v in zip((ship, disc, qty), vl)]
        cond = condition(b, kind)
        arms = [gandiva.make_filter(cases.Q6_SCHEMA, b.make_condition(cond), gandiva.Configuration(filter_gating=g))
                for g in (0, 1)]
        counts = [0, 0]

        def launch(i):
            arms[i].evaluate_device(n, cols, outs[i].data_ptr(), n, "UINT32", st, cnts[i].data_ptr(), sync=False)

        per_round = [[], []]
        for i in (0, 1):  # module load, first launch
            launch(i)
            counts[i] = arms[i].sync(st)
        for _ in range(a.rounds):
            for i in (0, 1):
                ms = []
                for _ in range(a.reps):
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    launch(i)
                    e1.record()
                    counts[i] = arms[i].sync(st)
                    ms.append(e0.elapsed_time(e1))
                per_round[i].append(float(np.median(ms)))
        same = counts[0] == counts[1] and bool(torch.equal(outs[0][:counts[0]], outs[1][:counts[1]]))
        med = [float(np.median(r)) for r in per_round]
        algo_per_row = 20.0 + (3 / 8.0 if nulls else 0.0) + 4.0 * counts[1] / n
        off_bw = algo_per_row * n / (med[1] * 1e-3)
        info = arms[0].kernel_info
        print(json.dumps({
            "workload": kind, "rows": n, "selected": counts[0], "gated_stages": info.get("gated_stages"),
            "regs_gated": info["regs"], "regs_off": arms[1].kernel_info["regs"],
            "ms_gated": round(med[0], 4), "ms_gated_spread": [round(min(per_round[0]), 4), round(max(per_round[0]), 4)],
            "ms_off": round(med[1], 4), "ms_off_spread": [round(min(per_round[1]), 4), round(max(per_round[1]), 4)],
            "speedup": round(med[1] / med[0], 3),
            "rows_per_s_gated": n / (med[0] * 1e-3), "rows_per_s_off": n / (med[1] * 1e-3),
            "off_gbs": round(off_bw / 1e9, 1),
            "effective_bytes_per_row_gated": round(off_bw * med[0] * 1e-3 / n, 2),
            "selection_vectors_equal": same, "device": name, "nvidia_smi": smi}), flush=True)
        del arms
    torch.cuda.synchronize()


if __name__ == "__main__":
    main()
