"""large_string columns resident in HBM against their utf8 twin.

    python tools/large_string_bench.py [--rows 100000000] [--steps 10] [--warmup 3] [--rounds 3]

Workload: the l_comment-like text of bench configs[3] (tests/cases.py comment_batch's strings, ~27 B per
row, 1 % nulls), `--rows` rows as ONE large_string batch (about 2.7 GB of bytes behind int64 offsets),
and its utf8 twin: the 7.0e7-row prefix, the longest one whose bytes fit int32 offsets.  Three runs:
  like      : Filter LIKE '%special%requests%' (the key-driven kernel);
  config4   : Filter like(upper(substr(c, 1, 32)), '%SPECIAL%REQUESTS%');
  upper     : Projector upper(c) into a large_string output (utf8 output for the twin).
Arms are alternated step by step and timed with CUDA events around the enqueued Evaluate; each round
prints the median, the JSON line the medians and min-max over rounds.  Rates are rows/s and effective
bytes per row: the algorithmic bytes (offset + the row's bytes + 1 validity bit in, 4 B per selected row
or offset + bytes + validity bit out) over the rows.  Every result is compared in full: filters with the
pool-level decision of the CPU oracle expanded over the rows, the large arm's prefix with the twin, the
projection's offsets and bytes with the upper-cased pool gathered over the rows.  The card name and power
limit are read in the same run."""
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
import oracle  # noqa: E402

TWIN_ROWS = 70_000_000


def card():
    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # the number is still reported, without the limit
        out = "power limit unavailable (%s)" % e
    return name, out


def gather(idx, vstart, vdata, lens, out_offsets, out):
    """out[out_offsets[r] + i] = byte i of pool entry idx[r], in row chunks."""
    step = 1 << 23
    for lo in range(0, len(idx), step):
        hi = min(lo + step, len(idx))
        ln = lens[lo:hi]
        n = int(ln.sum())
        if n == 0:
            continue
        src = torch.repeat_interleave(vstart[idx[lo:hi]], ln)
        dst = torch.repeat_interleave(out_offsets[lo:hi], ln)
        within = torch.arange(n, device="cuda") - torch.repeat_interleave(torch.cumsum(ln, 0) - ln, ln)
        out[dst + within] = vdata[src + within]


def pool_tensors(values):
    enc = [b"" if v is None else v.encode() for v in values]
    lens = torch.tensor([len(e) for e in enc], dtype=torch.int64, device="cuda")
    start = torch.tensor(np.concatenate([[0], np.cumsum([len(e) for e in enc])[:-1]]), dtype=torch.int64, device="cuda")
    data = torch.tensor(np.frombuffer(b"".join(enc) + b"\0" * 16, np.uint8).copy(), device="cuda")
    return lens, start, data


def bits(mask):
    """Little-endian validity bitmap of a bool tensor (padded to whole 64-bit words)."""
    n = len(mask)
    m = torch.zeros((n + 63) // 64 * 64, dtype=torch.uint8, device="cuda")
    m[:n] = mask.to(torch.uint8)
    w = torch.tensor([1, 2, 4, 8, 16, 32, 64, 128], dtype=torch.uint8, device="cuda")
    return (m.view(-1, 8) * w).sum(1, dtype=torch.uint8)


def timed(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    fn()
    e1.record()
    return e0, e1


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=100_000_000)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    n = args.rows
    name, limit = card()
    pool = cases.comment_batch(1 << 16, seed=42)
    values = pool.column(0).to_pylist()
    plens, pstart, pdata = pool_tensors(values)
    pvalid = torch.tensor([v is not None for v in values], device="cuda")
    g = torch.Generator(device="cuda").manual_seed(7)
    idx = torch.randint(0, len(values), (n,), device="cuda", generator=g)
    lens = plens[idx]
    offs = torch.zeros(n + 1, dtype=torch.int64, device="cuda")
    torch.cumsum(lens, 0, out=offs[1:])
    data = torch.zeros(int(offs[-1]) + 16, dtype=torch.uint8, device="cuda")
    gather(idx, pstart, pdata, lens, offs[:-1], data)
    valid = pvalid[idx]
    vbits = bits(valid)
    nt = min(n, TWIN_ROWS)
    assert int(offs[nt]) < 2**31, "the twin's bytes must fit int32 offsets"
    offs32 = offs[:nt + 1].to(torch.int32)
    large_cols = [(vbits.data_ptr(), offs.data_ptr(), data.data_ptr(), 0)]
    twin_cols = [(vbits.data_ptr(), offs32.data_ptr(), data.data_ptr(), 0)]
    large_schema = pa.schema([("c", pa.large_string())])
    b = gandiva.TreeExprBuilder()
    st = torch.cuda.current_stream().cuda_stream

    def like(c):
        return b.make_function("like", [c, b.make_literal("%special%requests%", pa.string())], pa.bool_())

    def config4(c):
        sub = b.make_function("substr", [c, b.make_literal(1, pa.int64()), b.make_literal(32, pa.int64())], pa.string())
        return b.make_function("like", [b.make_function("upper", [sub], pa.string()),
                                        b.make_literal("%SPECIAL%REQUESTS%", pa.string())], pa.bool_())

    results = []
    in_bytes = {"large": (8 * (n + 1) + int(offs[-1]) + n / 8) / n, "utf8": (4 * (nt + 1) + int(offs[nt]) + nt / 8) / nt}
    for run, cond in (("like", like), ("config4", config4)):
        fl = gandiva.make_filter(large_schema, b.make_condition(cond(b.make_field(large_schema.field(0)))))
        ft = gandiva.make_filter(cases.COMMENT_SCHEMA, b.make_condition(cond(b.make_field(cases.COMMENT_SCHEMA.field(0)))))
        # the pool-level decision of the CPU oracle, expanded over the rows
        hit = torch.zeros(len(values), dtype=torch.bool, device="cuda")
        pidx = oracle.filter_indices(cond(b.make_field(cases.COMMENT_SCHEMA.field(0))), pool)
        hit[torch.from_numpy(pidx.astype(np.int64)).cuda()] = True
        want = torch.nonzero(hit[idx] & valid).flatten()
        arms = {"large": (fl, n, large_cols), "utf8": (ft, nt, twin_cols)}
        outs = {k: (torch.zeros(r + 8, dtype=torch.int32, device="cuda"), torch.zeros(1, dtype=torch.int64, device="cuda"))
                for k, (_, r, _) in arms.items()}
        rounds = {k: [] for k in arms}
        for _ in range(args.rounds):
            ms = {k: [] for k in arms}
            for i in range(args.warmup + args.steps):
                for k, (f, rows, cols) in arms.items():
                    o, c = outs[k]
                    e0, e1 = timed(lambda: f.evaluate_device(rows, cols, o.data_ptr(), rows, "UINT32", st, c.data_ptr(), sync=False))
                    count = f.sync(st)
                    if i >= args.warmup:
                        ms[k].append(e0.elapsed_time(e1))
            for k in arms:
                rounds[k].append(float(np.median(ms[k])))
        for k, (f, rows, _) in arms.items():
            o, c = outs[k]
            count = int(c.item())
            w = want[want < rows]
            assert count == len(w) and torch.equal(o[:count].to(torch.int64), w), (run, k)
            med = float(np.median(rounds[k]))
            results.append({"run": run, "arm": k, "rows": rows, "kernel": f.kernel_info["name"][:16], "ms": med,
                            "ms_min": min(rounds[k]), "ms_max": max(rounds[k]), "rows_per_s": rows / med * 1e3,
                            "eff_bytes_per_row": in_bytes[k] + 4.0 * count / rows, "selected": count})
    # upper(c): large_string output over the large batch, utf8 output over the twin
    upper_pool = [None if v is None else v.upper() for v in values]
    ulens, ustart, udata = pool_tensors(upper_pool)
    want_bytes = torch.zeros(int(offs[-1]) + 16, dtype=torch.uint8, device="cuda")
    out_lens = torch.where(valid, ulens[idx], 0)
    want_offs = torch.zeros(n + 1, dtype=torch.int64, device="cuda")
    torch.cumsum(out_lens, 0, out=want_offs[1:])
    gather(idx, ustart, udata, out_lens, want_offs[:-1], want_bytes)
    arms = {}
    for k, schema, cols, rows, out_t, ot in (("large", large_schema, large_cols, n, pa.large_string(), torch.int64),
                                            ("utf8", cases.COMMENT_SCHEMA, twin_cols, nt, pa.string(), torch.int32)):
        up = b.make_function("upper", [b.make_field(schema.field(0))], pa.string())
        p = gandiva.make_projector(schema, [b.make_expression(up, pa.field("u", out_t))])
        cap = int(want_offs[rows])
        bufs = (torch.zeros((rows + 31) // 32 + 2, dtype=torch.int32, device="cuda"),
                torch.zeros(rows + 1, dtype=ot, device="cuda"), torch.zeros(cap + 16, dtype=torch.uint8, device="cuda"))
        arms[k] = (p, rows, cols, bufs, cap)
    rounds = {k: [] for k in arms}
    for _ in range(args.rounds):
        ms = {k: [] for k in arms}
        for i in range(args.warmup + args.steps):
            for k, (p, rows, cols, (ov, oo, od), cap) in arms.items():
                e0, e1 = timed(lambda: p.evaluate_device(rows, cols, [(ov.data_ptr(), oo.data_ptr(), od.data_ptr(), cap)], st))
                p.sync(st)
                if i >= args.warmup:
                    ms[k].append(e0.elapsed_time(e1))
        for k in arms:
            rounds[k].append(float(np.median(ms[k])))
    for k, (p, rows, cols, (ov, oo, od), cap) in arms.items():
        assert torch.equal(oo.to(torch.int64), want_offs[:rows + 1]), ("upper offsets", k)
        assert torch.equal(od[:cap], want_bytes[:cap]), ("upper bytes", k)
        med = float(np.median(rounds[k]))
        out_b = (8 if k == "large" else 4) * (rows + 1) + cap + rows / 8
        results.append({"run": "upper", "arm": k, "rows": rows, "ms": med, "ms_min": min(rounds[k]),
                        "ms_max": max(rounds[k]), "rows_per_s": rows / med * 1e3,
                        "eff_bytes_per_row": in_bytes[k] + out_b / rows})
    for r in results:
        print(json.dumps(r))
    by = {(r["run"], r["arm"]): r for r in results}
    print(json.dumps({"card": name, "power": limit, "rows": n, "twin_rows": nt,
                      "large_over_utf8_rows_per_s": {run: by[(run, "large")]["rows_per_s"] / by[(run, "utf8")]["rows_per_s"]
                                                     for run in ("like", "config4", "upper")}}))


if __name__ == "__main__":
    main()
