"""Dictionary-encoded string columns resident in HBM: the dictionary-first Filter against the general row
kernel on the same dictionary batch and against the same predicate over the decoded (plain utf8) column.

    python tools/dict_bench.py [--rows 100000000] [--steps 10] [--warmup 3]

Two columns: a low-cardinality one (7 distinct values, like TPC-H l_shipmode; int8 indices) filtered by
IN ('MAIL', 'SHIP'), and the l_comment-like text of bench configs[3] (tests/cases.py comment_batch's 4 096
distinct strings; int16 indices) filtered by LIKE '%special%requests%'.  Prints one JSON line per
(column, path) with rows/s, kernel ms (CUDA events around the enqueued Evaluate, median of the steps) and
the fraction of the H100 data-sheet bandwidth (3.35 TB/s) that the algorithmic bytes reach:
  dictionary paths: index bytes + 1 validity bit per row + 4 B per selected row (the dictionary is small);
  decoded column : 4 B offset + the row's bytes + 1 validity bit per row + 4 B per selected row (the
                   longest prefix of the rows whose bytes fit int32 offsets: ~70 M rows of the text column).
Every result is checked against an independent evaluation (the predicate decided per distinct value in
Python, expanded over the indices with torch) and, on the first million rows, against the CPU oracle.
The card name and power limit are read in the same run."""
import argparse
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


def card():
    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # the number is still reported, without the limit
        out = "power limit unavailable (%s)" % e
    return name, out


def dev_bytes(a: np.ndarray) -> torch.Tensor:
    return torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).copy()).cuda()


def make_column(values, rows, index_dtype, seed):
    """Device dictionary column: (indices tensor, dictionary arrow array, device dictionary buffers)."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    idx = torch.randint(0, len(values), (rows,), generator=g, device="cuda", dtype=torch.int64).to(index_dtype)
    dictionary = pa.array(values, pa.string())
    bufs = dictionary.buffers()
    offs = dev_bytes(np.frombuffer(bufs[1], dtype=np.int32)[: len(values) + 1])
    data = dev_bytes(np.frombuffer(bufs[2], dtype=np.uint8)[: max(bufs[2].size, 1)])
    return idx, dictionary, (offs, data)


def decoded_column(idx, dictionary):
    """The plain utf8 twin on the device: int32 offsets + bytes, built in row chunks."""
    bufs = dictionary.buffers()
    doff = torch.from_numpy(np.frombuffer(bufs[1], dtype=np.int32)[: len(dictionary) + 1].astype(np.int64)).cuda()
    ddat = torch.from_numpy(np.frombuffer(bufs[2], dtype=np.uint8).copy()).cuda()
    lens = (doff[1:] - doff[:-1])[idx.long()]
    offsets = torch.zeros(len(idx) + 1, dtype=torch.int64, device="cuda")
    torch.cumsum(lens, 0, out=offsets[1:])
    data = torch.empty(int(offsets[-1]) + 16, dtype=torch.uint8, device="cuda")
    step = 1 << 24
    for lo in range(0, len(idx), step):
        hi = min(lo + step, len(idx))
        # byte p of the output comes from dictionary byte p + (entry start - row start)
        shift = torch.repeat_interleave(doff[idx[lo:hi].long()] - offsets[lo:hi], lens[lo:hi])
        dst = torch.arange(int(offsets[lo]), int(offsets[hi]), device="cuda")
        data[dst] = ddat[dst + shift]
    return offsets.to(torch.int32), data, lens


def time_filter(f, rows, cols, steps, warmup, mode="UINT32"):
    out = torch.zeros(rows + 8, dtype=torch.int32, device="cuda")
    cnt = torch.zeros(1, dtype=torch.int64, device="cuda")
    st = torch.cuda.current_stream().cuda_stream
    ms = []
    for i in range(warmup + steps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        f.evaluate_device(rows, cols, out.data_ptr(), rows, mode, st, cnt.data_ptr(), sync=False)
        e1.record()
        count = f.sync(st)
        if i >= warmup:
            ms.append(e0.elapsed_time(e1))
    return float(np.median(ms)), count, out[:count].to(torch.int64)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=100_000_000)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    n = a.rows
    name, smi = card()
    comments = cases.comment_batch(4096 * 8, seed=42, null_prob=0.0).column(0).unique().to_pylist()
    columns = [
        ("shipmode", ["REG AIR", "AIR", "RAIL", "SHIP", "TRUCK", "MAIL", "FOB"], torch.int8,
         lambda b, d: b.make_in_expression(d, ["MAIL", "SHIP"], pa.string()), lambda s: s in ("MAIL", "SHIP")),
        ("comment", comments, torch.int16,
         lambda b, d: b.make_function("like", [d, b.make_literal("%special%requests%", pa.string())], pa.bool_()),
         lambda s: re.search("special.*requests", s, re.S) is not None),
    ]
    for cname, values, idt, pred, py_pred in columns:
        idx, dictionary, (doffs, ddata) = make_column(values, n, idt, seed=7)
        # null indices: every 97th row
        valid = torch.ones(n, dtype=torch.bool, device="cuda")
        valid[::97] = False
        vbits = torch.from_numpy(np.packbits(valid.cpu().numpy(), bitorder="little")).cuda()
        dd = gandiva.gdv_dictionary_t()
        dd.offsets, dd.data, dd.offset, dd.length = doffs.data_ptr(), ddata.data_ptr(), 0, len(values)
        dschema = pa.schema([("d", pa.dictionary({torch.int8: pa.int8(), torch.int16: pa.int16()}[idt], pa.string())),
                             ("s", pa.string())])
        pschema = pa.schema([("d", pa.string())])
        b = gandiva.TreeExprBuilder()
        dfield, sfield = b.make_field(dschema.field("d")), b.make_field(dschema.field("s"))
        always = b.make_or([b.make_function("isnull", [sfield], pa.bool_()), b.make_function("isnotnull", [sfield], pa.bool_())])
        first = gandiva.make_filter(dschema, b.make_condition(pred(b, dfield)))
        general = gandiva.make_filter(dschema, b.make_condition(b.make_and([pred(b, b.make_field(dschema.field("d"))), always])))
        plain = gandiva.make_filter(pschema, b.make_condition(pred(b, b.make_field(pschema.field("d")))))
        # the plain column s of the dictionary batch: one empty string per row (read by the general path only)
        s_offs = torch.zeros(n + 1, dtype=torch.int32, device="cuda")
        dcols = [(vbits.data_ptr(), idx.data_ptr(), dd, 0), (0, s_offs.data_ptr(), s_offs.data_ptr(), 0)]
        # independent answer: the predicate per distinct value, expanded over the indices
        keep = torch.tensor([py_pred(v) for v in values], dtype=torch.bool, device="cuda")
        want = torch.nonzero(keep[idx.long()] & valid).flatten()
        w = torch.empty(0, dtype=idt).element_size()
        results = []
        for path, f, cols, in_bytes in (("dictionary_first", first, dcols, n * w + n / 8),
                                        ("general", general, dcols, n * w + n / 8 + 4 * (n + 1))):
            ms, count, got = time_filter(f, n, cols, a.steps, a.warmup)
            assert f.kernel_info["dictionary_first"] == (1 if path == "dictionary_first" else 0)
            results.append((path, ms, count, got, in_bytes, n))
        # the decoded twin: the longest prefix whose bytes fit int32 offsets (utf8, not large_utf8)
        lens_all = (torch.from_numpy(np.diff(np.frombuffer(dictionary.buffers()[1], dtype=np.int32)[: len(values) + 1]))
                    .cuda().long()[idx.long()])
        nd = int(torch.searchsorted(torch.cumsum(lens_all, 0), torch.tensor([2**31 - 1], device="cuda")).item())
        nd = min(n, nd)
        del lens_all
        offs32, data, lens = decoded_column(idx[:nd], dictionary)
        pcols = [(vbits.data_ptr(), offs32.data_ptr(), data.data_ptr(), 0)]
        ms, count, got = time_filter(plain, nd, pcols, a.steps, a.warmup)
        results.append(("decoded", ms, count, got, 4 * nd + float(lens.sum()) + nd / 8, nd))
        # the CPU oracle on the first million rows of the decoded twin
        m = min(n, 1_000_000)
        rows_py = [values[i] for i in idx[:m].long().cpu().tolist()]
        vmask = valid[:m].cpu().numpy()
        twin = pa.RecordBatch.from_arrays([pa.array(rows_py, pa.string(), mask=~vmask)], schema=pschema)
        want_cpu = oracle.filter_indices(pred(b, b.make_field(pschema.field("d"))), twin, threads=8)
        for path, ms, count, got, in_bytes, rows in results:
            w_rows = want[want < rows]
            ok = count == len(w_rows) and torch.equal(got, w_rows) and \
                np.array_equal(got[got < m].cpu().numpy().astype(np.uint64), want_cpu)
            algo = in_bytes + 4 * len(w_rows)
            print(json.dumps({"column": cname, "path": path, "rows": rows, "selected": int(count), "distinct": len(values),
                              "kernel_ms": round(ms, 4), "rows_per_s": rows / (ms * 1e-3),
                              "algorithmic_bytes": int(algo), "frac_of_3.35TBps": round(algo / (ms * 1e-3) / PEAK, 3),
                              "check": "ok" if ok else "MISMATCH", "device": name, "nvidia_smi": smi}))
        del idx, offs32, data, lens, want
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
