"""string_view columns resident in HBM: Filters with the inline / prefix shortcut on and off, the same
predicates over the utf8 twin, and the identity projection string_view -> utf8 (the conversion a caller
pays when an engine only reads utf8).

    python tools/view_bench.py [--rows 100000000] [--steps 10] [--warmup 3]

Two columns: an l_shipmode-like one (7 distinct values, every row inline) filtered by IN ('MAIL', 'SHIP')
and by = 'MAIL', and the l_comment-like text of bench configs[3] (tests/cases.py comment_batch's strings,
mostly out of line) filtered by LIKE '%special%requests%'.  The view column is laid out as a producer
writes one: the out-of-line bytes of every row are its own, in data buffers of at most 1 GiB each.
Prints one JSON line per (column, form) with rows/s, kernel ms (CUDA events around the enqueued
Evaluate, median of the steps) and the fraction of the H100 data-sheet bandwidth (3.35 TB/s) that the
algorithmic bytes reach:
  view filter      : 16 B view + 1 validity bit per row, + the out-of-line bytes the predicate must read
                     (all of a row's bytes for a substring LIKE, none for the shortcut's inline rows),
                     + 4 B per selected row;
  utf8 twin filter : 4 B offset + the row's bytes + 1 validity bit per row + 4 B per selected row (the
                     longest prefix of the rows whose bytes fit int32 offsets);
  view -> utf8     : the view filter's input bytes + 4 B offset + the row's bytes + 1 validity bit out.
Every result is checked against an independent evaluation (the predicate decided per distinct value in
Python, expanded over the rows with torch; the projection against the utf8 twin) and, on the first
million rows, against the CPU oracle.  The card name and power limit are read in the same run."""
import argparse
import ctypes as C
import json
import os
import re
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

PEAK = 3.35e12
CHUNK = 1 << 30  # bytes per data buffer at most


def card():
    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # the number is still reported, without the limit
        out = "power limit unavailable (%s)" % e
    return name, out


def gather_bytes(idx, vstart, vdata, lens, starts, out):
    """out[starts[r] + i] = value idx[r]'s byte i, in row chunks."""
    step = 1 << 23
    for lo in range(0, len(idx), step):
        hi = min(lo + step, len(idx))
        ln = lens[lo:hi]
        shift = torch.repeat_interleave(vstart[idx[lo:hi]] - starts[lo:hi], ln)
        dst = torch.repeat_interleave(starts[lo:hi], ln) + (
            torch.arange(int(ln.sum()), device="cuda") - torch.repeat_interleave(torch.cumsum(ln, 0) - ln, ln))
        out[dst] = vdata[dst + shift]


def view_column(values, idx):
    """The string_view column of rows values[idx]: (views [n, 16] uint8, [data buffers], sizes)."""
    enc = [v.encode() for v in values]
    vlen = torch.tensor([len(e) for e in enc], dtype=torch.int64, device="cuda")
    vstart = torch.tensor(np.concatenate([[0], np.cumsum([len(e) for e in enc])[:-1]]), dtype=torch.int64, device="cuda")
    vdata = torch.tensor(np.frombuffer(b"".join(enc) + b"\0" * 16, np.uint8).copy(), device="cuda")
    head = np.zeros((len(values), 16), np.uint8)  # len + inline bytes / prefix
    for i, e in enumerate(enc):
        head[i, 0:4] = np.frombuffer(np.int32(len(e)).tobytes(), np.uint8)
        body = e if len(e) <= 12 else e[:4]  # inline bytes, or the prefix
        head[i, 4:4 + len(body)] = np.frombuffer(body, np.uint8)
    views = torch.from_numpy(head).cuda()[idx]
    lens = vlen[idx]
    out_of_line = lens > 12
    ool = torch.where(out_of_line, lens, 0)
    ends = torch.cumsum(ool, 0)
    buf_of = torch.div(ends - ool, CHUNK, rounding_mode="floor")  # the buffer a row's bytes start in
    bufs, sizes = [], []
    n_buf = int(buf_of[-1].item()) + 1 if len(idx) else 0
    v32 = views.view(torch.int32)
    for k in range(n_buf):
        rows = (buf_of == k)
        lo = int(torch.nonzero(rows)[0].item())
        hi = int(torch.nonzero(rows)[-1].item()) + 1
        base = int((ends[lo] - ool[lo]).item())
        starts = ends[lo:hi] - ool[lo:hi] - base
        size = int(ends[hi - 1].item()) - base
        data = torch.zeros(size + 16, dtype=torch.uint8, device="cuda")
        gather_bytes(idx[lo:hi], vstart, vdata, ool[lo:hi], starts, data)
        bufs.append(data)
        sizes.append(size)
        m = out_of_line[lo:hi]
        v32[lo:hi, 2] = torch.where(m, torch.full_like(starts, k), v32[lo:hi, 2].long()).to(torch.int32)
        v32[lo:hi, 3] = torch.where(m, starts, v32[lo:hi, 3].long()).to(torch.int32)
    return views, bufs, sizes, lens


def utf8_twin(values, idx, lens):
    """The plain utf8 twin of the longest prefix of the rows whose bytes fit int32 offsets."""
    nd = int(torch.searchsorted(torch.cumsum(lens, 0), torch.tensor([2**31 - 1], device="cuda")).item())
    nd = min(len(idx), nd)
    enc = [v.encode() for v in values]
    vstart = torch.tensor(np.concatenate([[0], np.cumsum([len(e) for e in enc])[:-1]]), dtype=torch.int64, device="cuda")
    vdata = torch.tensor(np.frombuffer(b"".join(enc) + b"\0" * 16, np.uint8).copy(), device="cuda")
    offsets = torch.zeros(nd + 1, dtype=torch.int64, device="cuda")
    torch.cumsum(lens[:nd], 0, out=offsets[1:])
    data = torch.zeros(int(offsets[-1]) + 16, dtype=torch.uint8, device="cuda")
    gather_bytes(idx[:nd], vstart, vdata, lens[:nd], offsets[:nd], data)
    return nd, offsets.to(torch.int32), data


def time_filter(f, rows, cols, steps, warmup):
    out = torch.zeros(rows + 8, dtype=torch.int32, device="cuda")
    cnt = torch.zeros(1, dtype=torch.int64, device="cuda")
    st = torch.cuda.current_stream().cuda_stream
    ms = []
    for i in range(warmup + steps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        f.evaluate_device(rows, cols, out.data_ptr(), rows, "UINT32", st, cnt.data_ptr(), sync=False)
        e1.record()
        count = f.sync(st)
        if i >= warmup:
            ms.append(e0.elapsed_time(e1))
    return float(np.median(ms)), count, out[:count].to(torch.int64)


def time_identity(p, rows, cols, need, steps, warmup):
    """The projection's utf8 output (validity, offsets, bytes) through the C-ABI's device path."""
    vld = torch.zeros((rows + 63) // 8 + 8, dtype=torch.uint8, device="cuda")
    offs = torch.zeros(rows + 8, dtype=torch.int32, device="cuda")
    data = torch.zeros(need + 16, dtype=torch.uint8, device="cuda")
    cc = (gandiva.gdv_column_t * len(cols))()
    for i, (v, val, var, off) in enumerate(cols):
        cc[i].validity, cc[i].values, cc[i].var_data, cc[i].offset = (v or None), val, gandiva._var_ptr(var), off
    cb = gandiva.gdv_batch_t(rows, len(cols), gandiva.GDV_MEM_DEVICE, cc)
    out = (gandiva.gdv_out_column_t * 1)()
    out[0].validity, out[0].values, out[0].var_data, out[0].var_capacity = vld.data_ptr(), offs.data_ptr(), data.data_ptr(), need
    st = torch.cuda.current_stream().cuda_stream
    ms = []
    for i in range(warmup + steps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        gandiva._check(gandiva.lib.gdv_projector_evaluate(p._h, C.byref(cb), None, out, 1, C.c_void_p(st), 1))
        e1.record()
        p.sync(st)
        if i >= warmup:
            ms.append(e0.elapsed_time(e1))
    return float(np.median(ms)), vld, offs[: rows + 1], data


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=100_000_000)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    n = a.rows
    name, smi = card()
    comments = cases.comment_batch(4096 * 8, seed=42, null_prob=0.0).column(0).unique().to_pylist()
    ship = ["REG AIR", "AIR", "RAIL", "SHIP", "TRUCK", "MAIL", "FOB"]
    columns = [
        ("shipmode", ship, [
            ("in", lambda b, v: b.make_in_expression(v, ["MAIL", "SHIP"], pa.string()), lambda s: s in ("MAIL", "SHIP")),
            ("equal", lambda b, v: b.make_function("equal", [v, b.make_literal("MAIL", pa.string())], pa.bool_()),
             lambda s: s == "MAIL")]),
        ("comment", comments, [
            ("like_substring", lambda b, v: b.make_function("like", [v, b.make_literal("%special%requests%", pa.string())],
                                                            pa.bool_()),
             lambda s: re.search("special.*requests", s, re.S) is not None)]),
    ]
    vschema = pa.schema([("v", pa.string_view())])
    pschema = pa.schema([("v", pa.string())])
    for cname, values, preds in columns:
        g = torch.Generator(device="cuda").manual_seed(7)
        idx = torch.randint(0, len(values), (n,), generator=g, device="cuda", dtype=torch.int64)
        valid = torch.ones(n, dtype=torch.bool, device="cuda")
        valid[::97] = False  # null rows: every 97th
        vbits = torch.from_numpy(np.packbits(valid.cpu().numpy(), bitorder="little")).cuda()
        views, bufs, sizes, lens = view_column(values, idx)
        dsizes = torch.tensor(sizes or [0], dtype=torch.int64, device="cuda")
        vb = gandiva.view_buffers([t.data_ptr() for t in bufs], dsizes.data_ptr())
        vcols = [(vbits.data_ptr(), views.data_ptr(), vb, 0)]
        nd, offs32, pdata = utf8_twin(values, idx, lens)
        pcols = [(vbits.data_ptr(), offs32.data_ptr(), pdata.data_ptr(), 0)]
        ool_bytes = float(torch.where(lens > 12, lens, 0).sum())
        b = gandiva.TreeExprBuilder()
        m = min(n, 1_000_000)
        twin_cpu = pa.RecordBatch.from_arrays(
            [pa.array([values[i] for i in idx[:m].cpu().tolist()], pa.string(), mask=~valid[:m].cpu().numpy())],
            schema=pschema)
        for pname, pred, py_pred in preds:
            keep = torch.tensor([py_pred(v) for v in values], dtype=torch.bool, device="cuda")
            want = torch.nonzero(keep[idx] & valid).flatten()
            want_cpu = oracle.filter_indices(pred(b, b.make_field(pschema.field("v"))), twin_cpu, threads=8)
            substring = pname == "like_substring"
            forms = [("view", 0, vschema, vcols, n, 16 * n + n / 8 + (ool_bytes if substring else 0)),
                     ("view_no_shortcut", 8, vschema, vcols, n, 16 * n + n / 8 + (ool_bytes if substring else 0)),
                     ("utf8", 0, pschema, pcols, nd, 4 * nd + float(lens[:nd].sum()) + nd / 8)]
            for form, scan, schema, cols, rows, in_bytes in forms:
                if substring and form == "view_no_shortcut":
                    continue  # no literal prefix: nothing to turn off
                f = gandiva.make_filter(schema, b.make_condition(pred(b, b.make_field(schema.field("v")))),
                                        gandiva.Configuration(string_scan=scan))
                ms, count, got = time_filter(f, rows, cols, a.steps, a.warmup)
                w_rows = want[want < rows]
                ok = count == len(w_rows) and torch.equal(got, w_rows) and \
                    np.array_equal(got[got < m].cpu().numpy().astype(np.uint64), want_cpu)
                algo = in_bytes + 4 * len(w_rows)
                print(json.dumps({"column": cname, "predicate": pname, "form": form, "rows": rows, "selected": int(count),
                                  "view_shortcuts": f.kernel_info["view_shortcuts"],
                                  "kernel_ms": round(ms, 4), "rows_per_s": rows / (ms * 1e-3),
                                  "algorithmic_bytes": int(algo), "frac_of_3.35TBps": round(algo / (ms * 1e-3) / PEAK, 3),
                                  "check": "ok" if ok else "MISMATCH", "device": name, "nvidia_smi": smi}), flush=True)
        # identity view -> utf8 over the rows the utf8 twin holds (its output needs int32 offsets too)
        p = gandiva.make_projector(vschema, [b.make_expression(b.make_field(vschema.field("v")), pa.field("o", pa.string()))])
        need = int(torch.where(valid[:nd], lens[:nd], 0).sum())
        ms, ovld, ooffs, odata = time_identity(p, nd, vcols, need, a.steps, a.warmup)
        want_lens = torch.where(valid[:nd], lens[:nd], 0)
        got_lens = (ooffs[1:] - ooffs[:-1]).long()
        vmask = torch.from_numpy(np.unpackbits(ovld.cpu().numpy(), bitorder="little")[:nd].astype(bool)).cuda()
        ok = torch.equal(got_lens, want_lens) and torch.equal(vmask, valid[:nd])
        if ok:  # the bytes of the valid rows equal the twin's
            twin_valid = torch.repeat_interleave(valid[:nd], lens[:nd])
            ok = torch.equal(odata[:need], pdata[: int(lens[:nd].sum())][twin_valid])
        ool_nd = float(torch.where(lens[:nd] > 12, lens[:nd], 0).sum())
        algo = 16 * nd + nd / 8 + ool_nd + 4 * nd + need + nd / 8
        print(json.dumps({"column": cname, "predicate": "identity", "form": "view_to_utf8", "rows": nd,
                          "kernel_ms": round(ms, 4), "rows_per_s": nd / (ms * 1e-3), "algorithmic_bytes": int(algo),
                          "frac_of_3.35TBps": round(algo / (ms * 1e-3) / PEAK, 3), "check": "ok" if ok else "MISMATCH",
                          "device": name, "nvidia_smi": smi}), flush=True)
        del idx, views, bufs, offs32, pdata, ovld, ooffs, odata
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
