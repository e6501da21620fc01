"""Filter -> Projector with a utf8 output, resident in HBM: the count kept on the device against today's
host round trips.

    python tools/chain_strings_bench.py [--rows 100000000] [--steps 20] [--warmup 3] [--out FILE]

Batch: the Q6 columns from the lineitem generator (l_shipdate date32, l_discount f64, l_quantity f64) plus an
l_comment-like utf8 column (texts of tests/cases.py comment_batch cut to 1..32 bytes, so the column fits int32
offsets).  Filter: TPC-H Q6.  Projector over its SelectionVector (UINT32): upper(substr(l_comment, 1, 32))
and l_quantity * l_discount.
  A (device count): filter enqueued; projector enqueued with d_num_slots = the filter's d_count and a data
    buffer whose capacity is an upper bound (the l_comment column's bytes); then sync both.
  B (host count, today's path): filter, sync (the count comes back); output_var_size over the count (sizing
    pass + scan + sync); evaluate over the count (sizing pass + scan + write); sync.
Each step runs both arms, alternating which goes first; each arm's time is host wall clock from a
synchronised device to the end of its last synchronise.  Prints one JSON line with the median and the
spread (min / max) of each arm, the saving, and whether the outputs of the two arms are byte-identical
(offsets 0..c, bytes, validity words, the fixed-width output).  The card name and power limit are read in the
same run."""
import argparse
import json
import os
import subprocess
import sys
import time

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


def comment_column(n, seed=7):
    """(offsets int32 [n + 1], bytes, total) of n rows drawn from a pool of comment texts cut to 1..32 bytes
    (about 16.5 on average, so 1e8 rows fit int32 offsets)."""
    texts = cases.comment_batch(4096, seed=42, null_prob=0.0).column(0).unique().to_pylist()
    pool = [s.encode()[: 1 + i % 32] for i, s in enumerate(texts)]
    plen = torch.tensor([len(p) for p in pool], dtype=torch.int64, device="cuda")
    pstart = torch.tensor(np.concatenate([[0], np.cumsum([len(p) for p in pool])[:-1]]), dtype=torch.int64, device="cuda")
    pdata = torch.tensor(np.frombuffer(b"".join(pool) + b"\0" * 16, np.uint8).copy(), device="cuda")
    g = torch.Generator(device="cuda").manual_seed(seed)
    idx = torch.randint(0, len(pool), (n,), generator=g, device="cuda", dtype=torch.int64)
    lens = plen[idx]
    offs = torch.zeros(n + 1, dtype=torch.int64, device="cuda")
    torch.cumsum(lens, 0, out=offs[1:])
    total = int(offs[-1])
    assert total < 2**31 - 1, "l_comment column must fit int32 offsets"
    data = torch.zeros(total + 16, dtype=torch.uint8, device="cuda")
    step = 1 << 23
    for lo in range(0, n, step):
        hi = min(lo + step, n)
        ln = lens[lo:hi]
        rel = torch.arange(int(ln.sum()), device="cuda") - torch.repeat_interleave(torch.cumsum(ln, 0) - ln, ln)
        data[torch.repeat_interleave(offs[lo:hi], ln) + rel] = pdata[torch.repeat_interleave(pstart[idx[lo:hi]], ln) + rel]
    return offs.to(torch.int32), data, total


class Outputs:
    def __init__(self, n, capacity):
        self.capacity = capacity
        self.offs = torch.zeros(n + 1 + 8, dtype=torch.int32, device="cuda")
        self.data = torch.zeros(capacity + 16, dtype=torch.uint8, device="cuda")
        self.vld = torch.zeros((n + 31) // 32 + 2, dtype=torch.int32, device="cuda")
        self.val = torch.zeros(n + 8, dtype=torch.float64, device="cuda")
        self.val_vld = torch.zeros((n + 31) // 32 + 2, dtype=torch.int32, device="cuda")

    def args(self, capacity=None):
        return [(self.vld.data_ptr(), self.offs.data_ptr(), self.data.data_ptr(), capacity or self.capacity),
                (self.val_vld.data_ptr(), self.val.data_ptr())]

    def result(self, c):
        total = int(self.offs[c])
        w = (c + 31) // 32
        return (self.offs[: c + 1].clone(), self.data[:total].clone(), self.vld[:w].clone(), self.val[:c].clone(),
                self.val_vld[:w].clone())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=100_000_000)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None, help="also append the JSON line to this file")
    a = ap.parse_args()
    if not gandiva.cuda_available():
        raise SystemExit("chain_strings_bench needs a CUDA device")
    n = a.rows
    name, smi = card()
    st = torch.cuda.current_stream().cuda_stream
    # ---- the batch, resident in HBM
    ship = torch.empty(n + 4, dtype=torch.int32, device="cuda")
    disc = torch.empty(n + 2, dtype=torch.float64, device="cuda")
    qty = torch.empty(n + 2, dtype=torch.float64, device="cuda")
    for kind, t in ((0, ship), (1, disc), (2, qty)):
        gandiva.generate_lineitem(0, kind, 42, 0, n, t.data_ptr(), 0, 0, st)
    coffs, cdata, cbytes = comment_column(n)
    torch.cuda.synchronize()
    schema = pa.schema(list(cases.Q6_SCHEMA) + [pa.field("l_comment", pa.string())])
    cols = [(0, ship.data_ptr(), 0, 0), (0, disc.data_ptr(), 0, 0), (0, qty.data_ptr(), 0, 0),
            (0, coffs.data_ptr(), cdata.data_ptr(), 0)]
    b = gandiva.TreeExprBuilder()
    f = {x.name: b.make_field(x) for x in schema}
    I64, F64 = pa.int64(), pa.float64()
    filt = gandiva.make_filter(schema, b.make_condition(cases.q6_condition(b)))
    up = b.make_function("upper", [b.make_function("substr", [f["l_comment"], b.make_literal(1, I64), b.make_literal(32, I64)],
                                                   pa.string())], pa.string())
    mul = b.make_function("multiply", [f["l_quantity"], f["l_discount"]], F64)
    proj = gandiva.make_projector(schema, [b.make_expression(up, pa.field("c", pa.string())),
                                           b.make_expression(mul, pa.field("r", F64))], None, "UINT32")
    sel = torch.zeros(n + 8, dtype=torch.int32, device="cuda")
    cnt = torch.zeros(1, dtype=torch.int64, device="cuda")
    out_a, out_b = Outputs(n, cbytes), Outputs(n, cbytes)

    def arm_a():
        filt.evaluate_device(n, cols, sel.data_ptr(), n, "UINT32", st, cnt.data_ptr(), sync=False)
        proj.evaluate_device(n, cols, out_a.args(), st, selection=(sel.data_ptr(), n, cnt.data_ptr()))
        proj.sync(st)
        return filt.sync(st)

    def arm_b():
        filt.evaluate_device(n, cols, sel.data_ptr(), n, "UINT32", st, cnt.data_ptr(), sync=False)
        c = filt.sync(st)
        need = proj.output_var_size_device(n, cols, 0, st, selection=(sel.data_ptr(), c))
        proj.evaluate_device(n, cols, out_b.args(need), st, selection=(sel.data_ptr(), c))
        proj.sync(st)
        return c

    times = {"A": [], "B": []}
    counts = {}
    for i in range(a.warmup + a.steps):
        order = (("A", arm_a), ("B", arm_b)) if i % 2 == 0 else (("B", arm_b), ("A", arm_a))
        for arm, fn in order:
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            counts[arm] = fn()
            dt = time.perf_counter() - t0
            if i >= a.warmup:
                times[arm].append(dt * 1e3)
    c = counts["A"]
    same = counts["A"] == counts["B"] and all(torch.equal(x, y) for x, y in zip(out_a.result(c), out_b.result(c)))
    med = {k: float(np.median(v)) for k, v in times.items()}
    line = {"workload": "q6 filter -> upper(substr(l_comment, 1, 32)) + l_quantity * l_discount", "rows": n, "selected": c,
            "out_bytes": int(out_a.offs[c]), "steps": a.steps,
            "device_count_ms": {"median": round(med["A"], 4), "min": round(min(times["A"]), 4), "max": round(max(times["A"]), 4)},
            "host_count_ms": {"median": round(med["B"], 4), "min": round(min(times["B"]), 4), "max": round(max(times["B"]), 4)},
            "saving_ms": round(med["B"] - med["A"], 4), "speedup": round(med["B"] / med["A"], 3),
            "outputs_identical": bool(same), "device": name, "nvidia_smi": smi}
    print(json.dumps(line), flush=True)
    if a.out:
        with open(a.out, "a") as fh:
            fh.write(json.dumps(line) + "\n")
    if not same:
        raise SystemExit("the two arms' outputs differ")


if __name__ == "__main__":
    main()
