"""Gated loads of the fixed-width Filter (Configuration.filter_gating = 0, the default): a conjunct's
columns are loaded only in the rows the earlier conjuncts kept.  Bit-exact against the CPU oracle and
against the ungated kernel (filter_gating = 1) on every shape the gated group must get right: selective,
empty and full first stages, nulls in every column (hoisted validity), slices, tail groups, every index
width, bounded vectors with an index base, two-column and repeated-column conjuncts, decimal128 and int8
columns, the W = 4 walk of big batches and a Filter -> Projector chain."""
import decimal

import numpy as np
import pyarrow as pa
import pytest

import cases
import devmem

pytestmark = pytest.mark.gpu

SD, F64, B = pa.date32(), pa.float64(), pa.bool_()


def q6_like(b, lo=8766, hi=9131, extra=()):
    fn = b.make_function
    ship, disc, qty = (cases.F(b, "l_shipdate", SD), cases.F(b, "l_discount", F64), cases.F(b, "l_quantity", F64))
    return b.make_and([fn("greater_than_or_equal_to", [ship, b.make_literal(lo, SD)], B),
                       fn("less_than", [ship, b.make_literal(hi, SD)], B),
                       fn("greater_than_or_equal_to", [disc, b.make_literal(0.05, F64)], B),
                       fn("less_than_or_equal_to", [disc, b.make_literal(0.07, F64)], B),
                       fn("less_than", [qty, b.make_literal(24.0, F64)], B)] + [e(b, ship, disc, qty) for e in extra])


def pair(gandiva, schema, b, cond, cfg=None):
    cfg = dict(cfg or {})
    on = gandiva.make_filter(schema, b.make_condition(cond), gandiva.Configuration(filter_gating=0, **cfg))
    off = gandiva.make_filter(schema, b.make_condition(cond), gandiva.Configuration(filter_gating=1, **cfg))
    return on, off


def check(on, off, cond, batch, oracle, dtypes=("int32",)):
    want = oracle.filter_indices(cond, batch, threads=4)
    for dtype in dtypes:
        got = on.evaluate(batch, None, dtype).to_array().to_numpy().astype(np.uint64)
        ref = off.evaluate(batch, None, dtype).to_array().to_numpy().astype(np.uint64)
        assert np.array_equal(got, want), (batch.num_rows, dtype, len(got), len(want))
        assert np.array_equal(ref, want), (batch.num_rows, dtype)
    return want


def without_validity(batch, keep):
    """The batch with validity bitmaps only in the columns listed in `keep`."""
    cols = []
    for j, col in enumerate(batch.columns):
        if j in keep:
            cols.append(col)
        else:
            cols.append(pa.Array.from_buffers(col.type, len(col), [None, col.buffers()[1]], offset=col.offset))
    return pa.RecordBatch.from_arrays(cols, schema=batch.schema)


def test_q6_gated_matches_oracle_and_ungated(gandiva, oracle):
    b = gandiva.TreeExprBuilder()
    cond = cases.q6_condition(b)
    on, off = pair(gandiva, cases.Q6_SCHEMA, b, cond)
    assert on.kernel_info["gated_stages"] == 3 and off.kernel_info["gated_stages"] == 0
    assert "gated loads: 3 stages" in on.llvm_ir and "gated loads" not in off.llvm_ir
    n = 200_003 if devmem.EMU else 1_000_003
    want = check(on, off, cond, cases.q6_batch(n, seed=42), oracle, ("int32", "int64"))
    assert len(want) > 0
    for n in (1, 31, 127, 128, 129, 1000, 4095, 8192 + 77):  # tail groups (not a multiple of 32 R)
        check(on, off, cond, cases.q6_batch(n, seed=n), oracle)
    check(on, off, cond, cases.q6_batch(60_001, seed=9), oracle, ("int16",))


@pytest.mark.parametrize("lo,hi", [(20000, 20001), (8035, 10562), (8766, 9131)], ids=["none", "all", "q6"])
def test_first_stage_keeps_nothing_everything_or_some(lo, hi, gandiva, oracle):
    b = gandiva.TreeExprBuilder()
    cond = q6_like(b, lo, hi)
    on, off = pair(gandiva, cases.Q6_SCHEMA, b, cond)
    assert on.kernel_info["gated_stages"] == 3
    for walk in (1, 4):
        on_w, off_w = pair(gandiva, cases.Q6_SCHEMA, b, cond, {"stages": walk})
        want = check(on_w, off_w, cond, cases.q6_batch(70_001, seed=3), oracle)
        assert (len(want) == 0) == (lo == 20000)


@pytest.mark.parametrize("cols", [(0,), (1,), (2,), (0, 1, 2)], ids=["ship", "disc", "qty", "all"])
def test_nulls_in_each_column(cols, gandiva, oracle):
    b = gandiva.TreeExprBuilder()
    cond = cases.q6_condition(b)
    on, off = pair(gandiva, cases.Q6_SCHEMA, b, cond)
    full = without_validity(cases.q6_batch(70_000, seed=5, null_permille=150), cols)
    for off_, n in ((0, 70_000), (13, 40_000), (45, 1025), (7, 33)):  # offsets that are not multiples of 32
        check(on, off, cond, full.slice(off_, n), oracle)


def test_bounded_vector_with_index_base(gandiva, oracle):
    n = 200_003 if devmem.EMU else 1_000_003
    st = devmem.stream()
    bufs = [devmem.DevBuf(n, np.int32), devmem.DevBuf(n, np.float64), devmem.DevBuf(n, np.float64)]
    for kind, t in enumerate(bufs):
        gandiva.generate_lineitem(0, kind, 42, 0, n, t.ptr, 0, 0, st)
    b = gandiva.TreeExprBuilder()
    cond = cases.q6_condition(b)
    on, off = pair(gandiva, cases.Q6_SCHEMA, b, cond)
    want = oracle.filter_indices(cond, cases.q6_batch(n, seed=42), threads=4)
    cols = [(0, t.ptr, 0, 0) for t in bufs]
    for f in (on, off):
        for mode, cap in (("UINT32", n), ("UINT64|BOUNDED", len(want) // 2)):
            out = devmem.DevBuf(n, np.int64 if "64" in mode else np.int32, fill=-1)
            cnt = devmem.DevBuf(1, np.int64, fill=0)
            f.evaluate_device(n, cols, out.ptr, cap, mode, st, cnt.ptr, index_base=5)
            assert f.sync(st) == len(want)
            k = min(cap, len(want))
            assert np.array_equal(out.numpy()[:k].astype(np.uint64), want[:k] + 5), mode


def test_large_batch_walk(gandiva, oracle):
    """>= 32 M rows: the big-tile variant (W = 4 chunks per warp); the simulator reaches it through
    Configuration(stages=4) on a batch it finishes in seconds."""
    n = 300_007 if devmem.EMU else (32 << 20) + 3
    st = devmem.stream()
    bufs = [devmem.DevBuf(n, np.int32), devmem.DevBuf(n, np.float64), devmem.DevBuf(n, np.float64)]
    for kind, t in enumerate(bufs):
        gandiva.generate_lineitem(0, kind, 42, 0, n, t.ptr, 0, 0, st)
    b = gandiva.TreeExprBuilder()
    cond = cases.q6_condition(b)
    on, off = pair(gandiva, cases.Q6_SCHEMA, b, cond, {"stages": 4} if devmem.EMU else None)
    cols = [(0, t.ptr, 0, 0) for t in bufs]
    res = []
    for f in (on, off):
        out = devmem.DevBuf(n, np.int32, fill=-1)
        cnt = devmem.DevBuf(1, np.int64, fill=0)
        f.evaluate_device(n, cols, out.ptr, n, "UINT32", st, cnt.ptr)
        c = f.sync(st)
        res.append(out.numpy()[:c].astype(np.int64))
    info = on.kernel_info  # the variant the evaluate above ran
    assert info["gated_stages"] == 3 and info["tile_rows"] == 8 * 1024 * 4
    assert np.array_equal(res[0], res[1])
    # the CPU oracle over the whole batch, in chunks of rows from the same generator
    chunk = 1 << 23
    want = []
    for lo in range(0, n, chunk):
        rows = min(chunk, n - lo)
        part = []
        for kind, t in ((0, SD), (1, F64), (2, F64)):
            vals, _ = oracle.generate_lineitem(kind, 42, lo, rows, 0, threads=8)
            part.append(pa.Array.from_buffers(t, rows, [None, pa.py_buffer(vals)]))
        want.append(oracle.filter_indices(cond, pa.RecordBatch.from_arrays(part, schema=cases.Q6_SCHEMA), threads=8) + lo)
    assert np.array_equal(res[0].astype(np.uint64), np.concatenate(want))


def test_two_column_and_repeated_column_conjuncts(gandiva, oracle):
    b = gandiva.TreeExprBuilder()
    fn = b.make_function
    disc, qty, ship = (cases.F(b, "l_discount", F64), cases.F(b, "l_quantity", F64), cases.F(b, "l_shipdate", SD))
    two = b.make_and([fn("less_than", [fn("multiply", [disc, b.make_literal(100.0, F64)], F64), qty], B),
                      fn("greater_than_or_equal_to", [ship, b.make_literal(8766, SD)], B),
                      fn("less_than", [ship, b.make_literal(9131, SD)], B)])
    on, off = pair(gandiva, cases.Q6_SCHEMA, b, two)
    assert on.kernel_info["gated_stages"] == 0  # stage 0 would read 16 of the row's 20 B: not gated
    assert on.llvm_ir == off.llvm_ir
    batch = cases.q6_batch(50_001, seed=8, null_permille=30)
    check(on, off, two, batch, oracle)
    # the same conjuncts with the date range first: the two-column conjunct is stage 1
    two_last = b.make_and([fn("greater_than_or_equal_to", [ship, b.make_literal(8766, SD)], B),
                           fn("less_than", [ship, b.make_literal(9131, SD)], B),
                           fn("less_than", [fn("multiply", [disc, b.make_literal(100.0, F64)], F64), qty], B)])
    on, off = pair(gandiva, cases.Q6_SCHEMA, b, two_last)
    assert on.kernel_info["gated_stages"] == 2
    check(on, off, two_last, batch, oracle)
    # shipdate again at the end: that conjunct joins stage 0
    again = q6_like(b, extra=[lambda b, s, d, q: fn("less_than", [s, b.make_literal(9000, SD)], B)])
    on, off = pair(gandiva, cases.Q6_SCHEMA, b, again)
    assert on.kernel_info["gated_stages"] == 3
    check(on, off, again, batch, oracle)


def test_decimal128_and_int8_columns(gandiva, oracle):
    D = pa.decimal128(12, 2)
    schema = pa.schema([("a", pa.int8()), ("d", D), ("x", pa.int32())])
    b = gandiva.TreeExprBuilder()
    fn = b.make_function
    a, d, x = cases.F(b, "a", pa.int8()), cases.F(b, "d", D), cases.F(b, "x", pa.int32())
    cond = b.make_and([fn("greater_than", [a, b.make_literal(-20, pa.int8())], B),
                       fn("less_than", [d, b.make_literal(decimal.Decimal("0.00"), D)], B),
                       fn("not_equal", [x, b.make_literal(0, pa.int32())], B)])
    on, off = pair(gandiva, schema, b, cond)
    assert on.kernel_info["gated_stages"] == 3
    for n, offset in ((40_007, 0), (5000, 11)):
        check(on, off, cond, cases.random_batch(schema, n, seed=n, null_prob=0.1, offset=offset), oracle)


def test_filter_then_projector(gandiva, oracle):
    b = gandiva.TreeExprBuilder()
    cond = cases.q6_condition(b)
    on, off = pair(gandiva, cases.Q6_SCHEMA, b, cond)
    batch = cases.q6_batch(100_003, seed=12, null_permille=20)
    qty = cases.F(b, "l_quantity", F64)
    root = b.make_function("multiply", [qty, cases.F(b, "l_discount", F64)], F64)
    p = gandiva.make_projector(cases.Q6_SCHEMA, [b.make_expression(root, pa.field("rev", F64))], None, "UINT32")
    sel = on.evaluate(batch)
    want_idx = oracle.filter_indices(cond, batch, threads=4)
    assert np.array_equal(sel.to_array().to_numpy().astype(np.uint64), want_idx)
    got, = p.evaluate(batch, sel)
    want, = oracle.project([root], [F64], batch, selection=want_idx.astype(np.int64), threads=4)
    assert got.equals(want)
    assert off.evaluate(batch).to_array().equals(sel.to_array())
