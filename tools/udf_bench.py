"""Q6 with its range tests written as user functions (DESIGN.md §3.8) against the built-in condition, over the
synthetic lineitem columns resident in HBM (1e9 rows by default, generated on the device from seed 42 as
bench.py does).

    python tools/udf_bench.py [--rows 1000000000] [--rounds 7] [--reps 3]

Arm 0 is cases.q6_condition; arm 1 is in_1994(l_shipdate) AND between_f64(l_discount, 0.05, 0.07) AND
lt24(l_quantity), three functions registered as CUDA text.  The two arms alternate, `--rounds` times each; a
round times `--reps` launches with CUDA events around each enqueued evaluate and keeps their median.  Prints
one JSON line with the median and the spread (min, max over rounds) of each arm's kernel time, rows/s, and
the SelectionVectors' equality (torch.equal, every index).  The card's name and power limit are read in the
same run."""
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


def user_condition(b, reg):
    sd, f, B = pa.date32(), pa.float64(), pa.bool_()
    reg.register("in_1994", [sd], B, "return a0 >= 8766 && a0 < 9131;")
    reg.register("between_f64", [f, f, f], B, "return a0 >= a1 && a0 <= a2;")
    reg.register("lt24", [f], B, "return a0 < 24.0;")
    ship, disc, qty = (cases.F(b, "l_shipdate", sd), cases.F(b, "l_discount", f), cases.F(b, "l_quantity", f))
    fn = b.make_function
    return b.make_and([fn("in_1994", [ship], B),
                       fn("between_f64", [disc, b.make_literal(0.05, f), b.make_literal(0.07, f)], B),
                       fn("lt24", [qty], B)])


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
    outs = [torch.empty(n, dtype=torch.int32, device=dev) for _ in range(2)]
    cnts = [torch.zeros(1, dtype=torch.int64, device=dev) for _ in range(2)]
    b = gandiva.TreeExprBuilder()
    for k, t in ((0, ship), (1, disc), (2, qty)):
        gandiva.generate_lineitem(0, k, 42, 0, n, t.data_ptr(), 0, 0, st)
    cols = [(0, t.data_ptr(), 0, 0) for t in (ship, disc, qty)]
    reg = gandiva.FunctionRegistry()
    user = user_condition(b, reg)
    arms = [gandiva.make_filter(cases.Q6_SCHEMA, b.make_condition(cases.q6_condition(b))),
            gandiva.make_filter(cases.Q6_SCHEMA, b.make_condition(user), gandiva.Configuration(function_registry=reg))]
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
    info = [arm.kernel_info for arm in arms]
    print(json.dumps({
        "workload": "q6", "rows": n, "selected": counts[0],
        "gated_stages": [i.get("gated_stages") for i in info], "regs": [i["regs"] for i in info],
        "ms_builtin": round(med[0], 4), "ms_builtin_spread": [round(min(per_round[0]), 4), round(max(per_round[0]), 4)],
        "ms_user": round(med[1], 4), "ms_user_spread": [round(min(per_round[1]), 4), round(max(per_round[1]), 4)],
        "user_over_builtin": round(med[1] / med[0], 4),
        "rows_per_s_builtin": n / (med[0] * 1e-3), "rows_per_s_user": n / (med[1] * 1e-3),
        "selection_vectors_equal": same, "device": name, "nvidia_smi": smi}), flush=True)
    torch.cuda.synchronize()


if __name__ == "__main__":
    main()
