"""timestamp[us] / [ns] columns resident in HBM against their timestamp[ms] twin.

    python tools/time_unit_bench.py [--rows 1000000000] [--text-rows 100000000] [--steps 5] [--warmup 2]

One set of instants (1992..1998, 1 % nulls) is held three times, in ms, us and ns, next to an int32 column x.
Three runs, each with the arms (ms, us, ns) alternated step by step and timed with CUDA events around the
enqueued Evaluate:
  filter   : Filter ts >= lo AND ts < hi AND x < 24 over --rows rows;
  project  : Projector extractYear(ts), date_trunc_Day(ts) over --rows rows;
  varchar  : Projector castVARCHAR(ts, 32) into a large_string field over --text-rows rows (no nulls).
Every result is compared in full: the ms filter with the rows torch selects, the other arms' selections
with the ms one; extractYear equal, date_trunc_Day equal to the ms result times the unit factor; the text
of each row equal to the ms text plus the extra fraction zeros.  Prints one JSON line with the median
time per arm, rows/s and the ratio to ms; the card name and power limit are read in the same run."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import pyarrow as pa  # noqa: E402
import gandiva_b200 as gandiva  # noqa: E402

UNITS = {"ms": 1, "us": 1000, "ns": 1000 ** 2}   # factor over ms
LO, HI = 757382400000, 788918400000              # [1994-01-01, 1995-01-01) in ms


def card():
    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # the number is still reported, without the limit
        out = "power limit unavailable (%s)" % e
    return name, out


def timed(arms, steps, warmup):
    """arms: name -> callable that enqueues one Evaluate on the current stream.  Returns median ms per arm."""
    times = {k: [] for k in arms}
    for step in range(warmup + steps):
        for k, fn in arms.items():
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            fn()
            b.record()
            b.synchronize()
            if hasattr(fn, "settle"):
                fn.settle()
            if step >= warmup:
                times[k].append(a.elapsed_time(b))
    return {k: float(np.median(v)) for k, v in times.items()}


def equal_where(valid, a, b, scale=1, step=1 << 26):
    """a[valid] == b[valid] * scale over every row, a chunk at a time (no full-size temporaries)."""
    for lo in range(0, valid.numel(), step):
        v = valid[lo:lo + step]
        if not torch.equal(a[lo:lo + step][v], b[lo:lo + step][v] * scale):
            return False
    return True


def bitmap(valid):
    """Arrow validity bits (LSB first) of a bool tensor, as a uint8 tensor."""
    n = valid.numel()
    pad = torch.zeros((n + 63) // 64 * 64, dtype=torch.bool, device="cuda")
    pad[:n] = valid
    w = pad.view(-1, 8).to(torch.uint8) << torch.arange(8, device="cuda", dtype=torch.uint8)
    return w.sum(1, dtype=torch.uint8)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1_000_000_000)
    ap.add_argument("--text-rows", type=int, default=100_000_000)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    n = args.rows
    st = torch.cuda.current_stream().cuda_stream
    g = torch.Generator(device="cuda").manual_seed(1)
    ms = torch.randint(694224000000, 915148800000, (n,), device="cuda", generator=g, dtype=torch.int64)
    x = torch.randint(0, 50, (n,), device="cuda", generator=g, dtype=torch.int32)
    valid = torch.rand(n, device="cuda", generator=g) >= 0.01
    vbits = bitmap(valid)
    ts = {u: ms if f == 1 else ms * f for u, f in UNITS.items()}
    b = gandiva.TreeExprBuilder()
    result = {"card": card(), "rows": n, "text_rows": args.text_rows, "steps": args.steps}

    # ---- filter ----
    filters, sels, cnts = {}, {}, {}
    for u, f in UNITS.items():
        t = pa.timestamp(u)
        schema = pa.schema([pa.field("ts", t), pa.field("x", pa.int32())])
        c = b.make_and([
            b.make_function("greater_than_or_equal_to", [b.make_field(schema.field("ts")), b.make_literal(LO * f, t)], pa.bool_()),
            b.make_function("less_than", [b.make_field(schema.field("ts")), b.make_literal(HI * f, t)], pa.bool_()),
            b.make_function("less_than", [b.make_field(schema.field("x")), b.make_literal(24, pa.int32())], pa.bool_())])
        filters[u] = gandiva.make_filter(schema, b.make_condition(c))
        sels[u] = torch.zeros(n + 8, dtype=torch.int32, device="cuda")
        cnts[u] = torch.zeros(1, dtype=torch.int64, device="cuda")

    def run_filter(u):
        cols = [(vbits.data_ptr(), ts[u].data_ptr(), 0, 0), (0, x.data_ptr(), 0, 0)]

        def go():
            filters[u].evaluate_device(n, cols, sels[u].data_ptr(), n, "UINT32", st, cnts[u].data_ptr())
        go.settle = lambda: filters[u].sync(st)
        return go
    med = timed({u: run_filter(u) for u in UNITS}, args.steps, args.warmup)
    want = torch.nonzero(valid & (ms >= LO) & (ms < HI) & (x < 24)).flatten().to(torch.int32)
    for u in UNITS:
        k = int(cnts[u].item())
        assert k == want.numel() and torch.equal(sels[u][:k], want), "filter %s" % u
    result["filter"] = {u: {"ms": med[u], "rows_per_s": n / (med[u] * 1e-3), "vs_ms": med["ms"] / med[u],
                            "gated_stages": filters[u].kernel_info.get("gated_stages")} for u in UNITS}
    del sels, want, x
    torch.cuda.empty_cache()

    # ---- extractYear, date_trunc_Day ----
    projs = {}
    for u in UNITS:
        t = pa.timestamp(u)
        schema = pa.schema([pa.field("ts", t)])
        f0 = b.make_field(schema.field("ts"))
        projs[u] = gandiva.make_projector(schema, [
            b.make_expression(b.make_function("extractYear", [f0], pa.int64()), pa.field("y", pa.int64())),
            b.make_expression(b.make_function("date_trunc_Day", [f0], t), pa.field("d", t))], None)
    year = torch.empty(n, dtype=torch.int64, device="cuda")
    day = torch.empty(n, dtype=torch.int64, device="cuda")
    ovy = torch.zeros((n + 63) // 8, dtype=torch.uint8, device="cuda")
    ovd = torch.zeros((n + 63) // 8, dtype=torch.uint8, device="cuda")

    def run_project(u):
        cols = [(vbits.data_ptr(), ts[u].data_ptr(), 0, 0)]
        o = [(ovy.data_ptr(), year.data_ptr()), (ovd.data_ptr(), day.data_ptr())]

        def go():
            projs[u].evaluate_device(n, cols, o, st)
        go.settle = lambda: projs[u].sync(st)
        return go
    med = timed({u: run_project(u) for u in UNITS}, args.steps, args.warmup)
    # full comparison: every arm once more, against the ms results
    run_project("ms")()
    projs["ms"].sync(st)
    ref_year, ref_day, ref_v = year.clone(), day.clone(), ovy.clone()
    for u, f in UNITS.items():
        run_project(u)()
        projs[u].sync(st)
        assert torch.equal(ovy, ref_v) and torch.equal(ovd, ref_v), "project validity %s" % u
        assert equal_where(valid, year, ref_year), "extractYear %s" % u
        assert equal_where(valid, day, ref_day, f), "date_trunc_Day %s" % u
    want_day = torch.div(ms, 86400000, rounding_mode="floor")
    assert equal_where(valid, ref_day, want_day, 86400000)
    result["project"] = {u: {"ms": med[u], "rows_per_s": n / (med[u] * 1e-3), "vs_ms": med["ms"] / med[u]} for u in UNITS}
    del year, day, ref_year, ref_day, want_day, projs, ovy, ovd
    torch.cuda.empty_cache()

    # ---- castVARCHAR(ts, 32) ----
    m = args.text_rows
    width = {"ms": 23, "us": 26, "ns": 29}   # "YYYY-MM-DD hh:mm:ss.fff..." for years 1000..9999
    vproj, bufs = {}, {}
    for u in UNITS:
        t = pa.timestamp(u)
        schema = pa.schema([pa.field("ts", t)])
        node = b.make_function("castVARCHAR", [b.make_field(schema.field("ts")), b.make_literal(32, pa.int64())], pa.string())
        # more than 2^31 bytes of text: a large_string result field (int64 offsets)
        vproj[u] = gandiva.make_projector(schema, [b.make_expression(node, pa.field("s", pa.large_string()))], None)
        bufs[u] = (torch.zeros((m + 63) // 8, dtype=torch.uint8, device="cuda"),
                   torch.zeros(m + 1, dtype=torch.int64, device="cuda"),
                   torch.zeros(m * width[u] + 64, dtype=torch.uint8, device="cuda"))

    def run_varchar(u):
        cols = [(0, ts[u].data_ptr(), 0, 0)]
        vb, off, data = bufs[u]
        o = [(vb.data_ptr(), off.data_ptr(), data.data_ptr(), data.numel())]

        def go():
            vproj[u].evaluate_device(m, cols, o, st)
        go.settle = lambda: vproj[u].sync(st)
        return go
    med = timed({u: run_varchar(u) for u in UNITS}, args.steps, args.warmup)
    torch.cuda.synchronize()
    ref = bufs["ms"][2][:m * 23].view(m, 23)
    first = bytes(ref[0].cpu().numpy())
    assert first[:2] == b"19" and len(first) == 23, first
    for u in UNITS:
        off, data = bufs[u][1], bufs[u][2]
        w = width[u]
        bad = torch.nonzero(off != torch.arange(m + 1, device="cuda", dtype=torch.int64) * w).flatten()
        assert bad.numel() == 0, "offsets %s: %d rows differ, first %s: %s" % (
            u, bad.numel(), bad[:4].tolist(), off[bad[:4]].tolist())
        txt = data[:m * w].view(m, w)
        assert torch.equal(txt[:, :23], ref), "text %s" % u
        assert bool((txt[:, 23:] == ord("0")).all()), "fraction %s" % u
    result["varchar"] = {u: {"ms": med[u], "rows_per_s": m / (med[u] * 1e-3), "vs_ms": med["ms"] / med[u],
                             "out_bytes_per_row": width[u] + 8} for u in UNITS}
    print(json.dumps(result))


if __name__ == "__main__":
    main()
