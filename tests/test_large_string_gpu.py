"""large_string / large_binary columns and outputs (DESIGN.md §2, §3.4, §5): every Filter and Projector result
over a large batch equals the CPU oracle's over the utf8 / binary twin (`cast(pa.string())`), validity
included, with every string path on and off (string_scan 0 / 1 / 4).  Also rows at offsets past 2^31,
a row too long for a string (it reads as null), and a large output of more than 2^31 bytes."""
import os

import numpy as np
import pyarrow as pa
import pytest

import devmem
from helpers import assert_arrays_match
from test_string_view_gpu import WORDS

pytestmark = pytest.mark.gpu

LS, LB, S = pa.large_string(), pa.large_binary(), pa.string()
# above 32 M rows the filters take their large-tile configuration
LARGE = 300_007 if devmem.EMU else (32 << 20) + 3
TEXT = WORDS + ["special", "requests", "carefully final special requests", "special pinto requests sleep",
                "spark fire", "blithely ironic deposits " * 4 + "special final requests"]


def words(n, seed=0, nulls=0.1):
    rng = np.random.default_rng(seed)
    idx = rng.integers(0, len(TEXT), n)
    mask = rng.random(n) < nulls
    return [None if m else TEXT[i] for i, m in zip(idx, mask)]


def batches(vals, large=LS, plain=S, seed=1):
    """(large batch, utf8 twin): column v is `large`, column s a plain utf8 column next to it."""
    rng = np.random.default_rng(seed)
    n = len(vals)
    twin = pa.array(vals, plain)
    other = pa.array(["s%d" % (i % 97) if rng.random() > 0.1 else None for i in range(n)], S)
    return (pa.RecordBatch.from_arrays([twin.cast(large), other], names=["v", "s"]),
            pa.RecordBatch.from_arrays([twin, other], names=["v", "s"]))


def field(b, batch, name="v"):
    return b.make_field(batch.schema.field(name))


def _like(b, v, pat):
    return b.make_function("like", [v, b.make_literal(pat, S)], pa.bool_())


def _config4(b, v):
    """configs[3]: like(upper(substr(c, 1, 32)), '%SPECIAL%REQUESTS%')"""
    sub = b.make_function("substr", [v, b.make_literal(1, pa.int64()), b.make_literal(32, pa.int64())], S)
    return _like(b, b.make_function("upper", [sub], S), "%SPECIAL%REQUESTS%")


PREDICATES = {
    "equal": lambda b, v: b.make_function("equal", [v, b.make_literal("special requests", S)], pa.bool_()),
    "in": lambda b, v: b.make_in_expression(v, ["MAIL", "SHIP", "", "héllo wörld", "spark fire"], S),
    "starts_with": lambda b, v: b.make_function("starts_with", [v, b.make_literal("spe", S)], pa.bool_()),
    "config4": _config4,
    "like_substring": lambda b, v: _like(b, v, "%special%requests%"),
    "like_key": lambda b, v: _like(b, v, "%final%"),
}


def check_filter(gandiva, oracle, batch, plain, pred, dtype="int32", scans=(0, 1, 4)):
    """Every string path on and off selects exactly the oracle's rows; returns the indices."""
    b = gandiva.TreeExprBuilder()
    want = oracle.filter_indices(pred(b, field(b, plain)), plain, threads=4)
    for scan in scans:
        f = gandiva.make_filter(batch.schema, b.make_condition(pred(b, field(b, batch))), gandiva.Configuration(string_scan=scan))
        got = f.evaluate(batch, None, dtype).to_array().to_numpy().astype(np.uint64)
        assert np.array_equal(got, want), "string_scan=%d: %d rows selected, oracle %d" % (scan, len(got), len(want))
    return want


@pytest.mark.parametrize("pred", sorted(PREDICATES))
def test_filters_match_oracle(pred, gandiva, oracle):
    check_filter(gandiva, oracle, *batches(words(6007, seed=len(pred))), PREDICATES[pred])


def test_key_driven_filter_over_long_rows(gandiva, oracle):
    """Rows longer than the string stage, and a warp's run of many anchors (the fallback evaluates every row)."""
    vals = [("special requests " * (1 + i % 40)) if i % 3 else ("x" * (i % 700)) for i in range(9000)]
    for pred in ("like_substring", "config4", "like_key"):
        check_filter(gandiva, oracle, *batches(vals, seed=2), PREDICATES[pred])


def test_binary_filters_and_projections(gandiva, oracle):
    vals = [None if v is None else v.encode() for v in words(4001, seed=9)]
    batch, plain = batches(vals, LB, pa.binary())
    b = gandiva.TreeExprBuilder()
    eq = lambda b, v: b.make_function("equal", [v, b.make_literal(b"MAIL", pa.binary())], pa.bool_())
    inn = lambda b, v: b.make_in_expression(v, [b"SHIP", b"", "héllo wörld".encode()], pa.binary())
    for pred in (eq, inn):
        check_filter(gandiva, oracle, batch, plain, pred)
    want = oracle.project([field(b, plain), b.make_function("octet_length", [field(b, plain)], pa.int32())],
                          [pa.binary(), pa.int32()], plain)
    for out_t in (pa.binary(), LB):
        p = gandiva.make_projector(batch.schema, [b.make_expression(field(b, batch), pa.field("o", out_t)),
                                                  b.make_expression(b.make_function("octet_length", [field(b, batch)], pa.int32()),
                                                                    pa.field("n", pa.int32()))])
        got = p.evaluate(batch)
        assert got[0].type == out_t
        assert_arrays_match(got[0].cast(pa.binary()), want[0], "identity into %s" % out_t)
        assert_arrays_match(got[1], want[1], "octet_length")


def _roots(b, bt):
    v, s = field(b, bt), field(b, bt, "s")
    fn, L = b.make_function, (lambda x: b.make_literal(x, pa.int64()))
    return [v, fn("upper", [v], S), fn("substr", [v, L(2), L(5)], S), fn("concat", [v, s], S),
            fn("castVARCHAR", [v, L(7)], S), fn("char_length", [v], pa.int32())]


def check_projections(gandiva, oracle, batch, plain):
    """Each root into a utf8 output and, when it yields a string, into a large_string output too."""
    b = gandiva.TreeExprBuilder()
    roots = _roots(b, plain)
    types = [S] * (len(roots) - 1) + [pa.int32()]
    want = oracle.project(roots, types, plain, threads=4)
    for scan in (0, 1):
        mine = _roots(b, batch)
        exprs, expect = [], []
        for i, (r, t, w) in enumerate(zip(mine, types, want)):
            for out_t in ((S, LS) if t == S else (t,)):
                exprs.append(b.make_expression(r, pa.field("o%d_%s" % (i, out_t), out_t)))
                expect.append((out_t, w))
        p = gandiva.make_projector(batch.schema, exprs, configuration=gandiva.Configuration(string_scan=scan))
        for k, (g, (out_t, w)) in enumerate(zip(p.evaluate(batch), expect)):
            assert g.type == out_t
            assert_arrays_match(g.cast(w.type), w, "output %d (%s), string_scan=%d" % (k, out_t, scan))


@pytest.mark.parametrize("offset", [0, 5, 33])
def test_projections_match_oracle(offset, gandiva, oracle):
    batch, plain = batches(words(3001 + offset, seed=7))
    check_projections(gandiva, oracle, batch.slice(offset), plain.slice(offset))


def test_sliced_filter(gandiva, oracle):
    batch, plain = batches(words(5000, seed=8))
    for pred in ("config4", "in", "like_substring"):
        check_filter(gandiva, oracle, batch.slice(37, 4000), plain.slice(37, 4000), PREDICATES[pred])


@pytest.mark.parametrize("n", [1, LARGE])
def test_filter_batch_sizes(n, gandiva, oracle):
    rng = np.random.default_rng(n)
    pool = np.array(TEXT, dtype=object)
    twin = pa.array(pool[rng.integers(0, len(TEXT), n)], S, mask=rng.random(n) < 0.1)
    batch = pa.RecordBatch.from_arrays([twin.cast(LS)], names=["v"])
    plain = pa.RecordBatch.from_arrays([twin], names=["v"])
    for pred in ("in", "like_substring"):
        check_filter(gandiva, oracle, batch, plain, PREDICATES[pred], dtype="int64", scans=(0, 4))


def _to_device(keep, data, n_bytes):
    """A device copy of the first n_bytes of `data`, zero padded.  The zero fill runs on torch's stream and the
    copy on the engine's own one: the fill is waited for first, so it cannot land after the copy."""
    buf = devmem.DevBuf(max(n_bytes, 1) + 64, np.uint8, fill=0)
    devmem.synchronize()
    if n_bytes:
        import gandiva_b200
        gandiva_b200.memcpy_htod(0, buf.ptr, np.frombuffer(data, dtype=np.uint8)[:n_bytes].copy())
    keep.append(buf)
    return buf.ptr


def _device_columns(batch, keep):
    """The batch's buffers copied to the device whole (offsets kept, so `offset` still applies)."""
    cols = []
    for c in batch.columns:
        bb = c.buffers()
        vld = _to_device(keep, bb[0], bb[0].size) if bb[0] is not None and c.null_count else 0
        cols.append((vld, _to_device(keep, bb[1], bb[1].size), _to_device(keep, bb[2], bb[2].size), c.offset))
    return cols


def _large_out(n, cap):
    """Device buffers of a large_string output: validity words, n + 1 int64 offsets, `cap` bytes."""
    return (devmem.DevBuf((n + 31) // 32 + 2, np.int32, fill=0), devmem.DevBuf(n + 1, np.int64, fill=0),
            devmem.DevBuf(max(cap, 1) + 16, np.uint8, fill=0))


def _large_array(n, vld, offs, data, t=LS):
    o = offs.numpy()[: n + 1].copy()
    return pa.Array.from_buffers(t, n, [pa.py_buffer(vld.numpy().view(np.uint8)), pa.py_buffer(o),
                                        pa.py_buffer(data.numpy()[: max(int(o[-1]), 1)].copy())])


@pytest.mark.parametrize("pred", ["in", "config4"])
def test_device_batch_filter_then_projector(pred, gandiva, oracle):
    """Device-resident large batch: the Filter writes selection + count on the device, a Projector reads
    both on the same stream and writes a large_string output (offsets[c] is the byte total)."""
    n = 20_011
    batch, plain = batches(words(n + 9, seed=11))
    batch, plain = batch.slice(9), plain.slice(9)
    keep = []
    cols = _device_columns(batch, keep)
    b = gandiva.TreeExprBuilder()
    want_idx = oracle.filter_indices(PREDICATES[pred](b, field(b, plain)), plain, threads=4)
    f = gandiva.make_filter(batch.schema, b.make_condition(PREDICATES[pred](b, field(b, batch))))
    up = lambda bt: b.make_function("upper", [field(b, bt)], S)
    proj = gandiva.make_projector(batch.schema, [b.make_expression(up(batch), pa.field("u", LS))], None, "UINT32")
    want, = oracle.project([up(plain)], [S], plain, selection=want_idx.astype(np.int64))
    st = devmem.stream()
    sel = devmem.DevBuf(n + 8, np.uint32, fill=0)
    cnt = devmem.DevBuf(1, np.int64, fill=0)
    cap = 64 * n
    vld, offs, data = _large_out(n, cap)
    f.evaluate_device(n, cols, sel.ptr, n, "UINT32", st, cnt.ptr, sync=False)
    proj.evaluate_device(n, cols, [(vld.ptr, offs.ptr, data.ptr, cap)], st, selection=(sel.ptr, n, cnt.ptr))
    proj.sync(st)
    count = f.sync(st)
    assert count == len(want_idx)
    assert np.array_equal(sel.numpy()[:count].astype(np.uint64), want_idx)
    assert_arrays_match(_large_array(count, vld, offs, data).cast(S), want, "chained upper into large_string")


def test_row_range_shard_is_a_slice_of_the_offsets(gandiva, oracle):
    """A shard of a large batch = the same bytes + a slice of the offsets; index_base makes the selection
    global (what sharding.py does for every column)."""
    n = 10_000
    batch, plain = batches(words(n, seed=4))
    b = gandiva.TreeExprBuilder()
    want = oracle.filter_indices(PREDICATES["like_substring"](b, field(b, plain)), plain)
    f = gandiva.make_filter(batch.schema, b.make_condition(PREDICATES["like_substring"](b, field(b, batch))))
    keep = []
    cols = _device_columns(batch, keep)
    got = []
    for lo, hi in ((0, 4096), (4096, 10_000)):
        shard = [(v, i, d, off + lo) for v, i, d, off in cols]
        sel = devmem.DevBuf(hi - lo + 8, np.uint64, fill=0)
        cnt = f.evaluate_device(hi - lo, shard, sel.ptr, hi - lo, "UINT64", devmem.stream(), sync=True, index_base=lo)
        got.append(sel.numpy()[:cnt])
    assert np.array_equal(np.concatenate(got).astype(np.uint64), want)


def test_user_function_reads_a_large_column(gandiva):
    """A large column passed to a utf8 parameter reads as the same gdv_str."""
    reg = gandiva.FunctionRegistry()
    reg.register("large_count_a", [S], pa.int32(), "i32 n = 0;\nfor (i32 i = 0; i < a0.len; ++i) n += gdv_ch(a0, i) == 'a';\n"
                                                  "return n;")
    vals = words(5003, seed=5)
    batch, _ = batches(vals)
    b = gandiva.TreeExprBuilder()
    p = gandiva.make_projector(batch.schema, [b.make_expression(b.make_function("large_count_a", [field(b, batch)], pa.int32()),
                                                                pa.field("o", pa.int32()))],
                               configuration=gandiva.Configuration(function_registry=reg))
    got, = p.evaluate(batch.slice(3))
    assert_arrays_match(got, pa.array([None if v is None else v.encode().count(b"a") for v in vals[3:]], pa.int32()))


def test_cpp_layer_matches_the_mirror(gandiva):
    """The C++ namespace-gandiva layer (through the stock pyarrow binding, when it is built) reads a host
    large_string batch and allocates a LargeStringArray output like the Python mirror does."""
    here = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "conformance", "stock")
    if not os.path.isdir(here) or not any(f.startswith("gandiva.") and f.endswith(".so") for f in os.listdir(here)):
        pytest.skip("the stock pyarrow binding over the C++ layer is not built")
    from conformance.run_stock_tests import load_stock_module
    stock = load_stock_module()
    batch, _ = batches(words(5000, seed=12))
    outs = []
    for mod in (stock, gandiva):
        b = mod.TreeExprBuilder()
        v = b.make_field(batch.schema.field("v"))
        up = b.make_function("upper", [v], S)
        p = mod.make_projector(batch.schema, [b.make_expression(up, pa.field("u", LS))], pa.default_memory_pool())
        f = mod.make_filter(batch.schema, b.make_condition(b.make_in_expression(v, ["MAIL", "SHIP"], S)))
        outs.append((p.evaluate(batch)[0], f.evaluate(batch, pa.default_memory_pool()).to_array()))
    assert outs[0][0].type == LS
    assert_arrays_match(outs[0][0], outs[1][0], "C++ layer: upper into large_string")
    assert np.array_equal(outs[0][1].to_numpy(), outs[1][1].to_numpy())


# ---- offsets past 2^31 ------------------------------------------------------------------------------
BIG = 1 << 31


def _after_a_huge_row(gandiva, vals, keep):
    """A device large_string column whose row 0 is 2^31 bytes long (never written: under the simulator
    the "device" buffer is an untouched np.empty) followed by `vals`, whose bytes sit at offsets > 2^31."""
    raw = [b"" if v is None else v.encode() for v in vals]
    offs = np.zeros(len(vals) + 2, np.int64)
    offs[1] = BIG
    offs[2:] = BIG + np.cumsum([len(r) for r in raw])
    tail = b"".join(raw)
    data = devmem.DevBuf(BIG + len(tail) + 64, np.uint8)
    keep.append(data)
    if tail:
        gandiva.memcpy_htod(0, data.ptr + BIG, np.frombuffer(tail, np.uint8).copy())
    valid = np.array([True] + [v is not None for v in vals])
    vbits = np.packbits(valid, bitorder="little").tobytes()
    col = (_to_device(keep, vbits, len(vbits)), _to_device(keep, offs.tobytes(), offs.nbytes), data.ptr)
    return col, len(vals) + 1


def test_rows_past_2gib_and_a_row_too_long_for_a_string(gandiva, oracle):
    vals = words(3001, seed=13)
    keep = []
    (vld, offs, data), n = _after_a_huge_row(gandiva, vals, keep)
    schema = pa.schema([("v", LS)])
    plain = pa.RecordBatch.from_arrays([pa.array(vals, S)], names=["v"])
    b = gandiva.TreeExprBuilder()
    # sliced past row 0: only the rows at offsets > 2^31 are read
    for pred in ("in", "config4", "like_substring"):
        want = oracle.filter_indices(PREDICATES[pred](b, field(b, plain)), plain)
        for scan in (0, 1, 4):
            f = gandiva.make_filter(schema, b.make_condition(PREDICATES[pred](b, b.make_field(schema.field(0)))),
                                    gandiva.Configuration(string_scan=scan))
            sel = devmem.DevBuf(n + 8, np.uint32, fill=0)
            cnt = f.evaluate_device(n - 1, [(vld, offs, data, 1)], sel.ptr, n, "UINT32", devmem.stream(), sync=True)
            assert np.array_equal(sel.numpy()[:cnt].astype(np.uint64), want), (pred, scan)
    up = lambda v: b.make_function("upper", [v], S)
    want, = oracle.project([up(field(b, plain))], [S], plain)
    p = gandiva.make_projector(schema, [b.make_expression(up(b.make_field(schema.field(0))), pa.field("u", LS))])
    cap = 64 * n
    ovld, ooffs, odata = _large_out(n, cap)
    p.evaluate_device(n - 1, [(vld, offs, data, 1)], [(ovld.ptr, ooffs.ptr, odata.ptr, cap)], devmem.stream(), sync=True)
    assert_arrays_match(_large_array(n - 1, ovld, ooffs, odata).cast(S), want, "upper past 2^31")
    # unsliced: row 0's length does not fit a string, so it reads as null and is never dereferenced
    twin = pa.RecordBatch.from_arrays([pa.array([None] + vals, S)], names=["v"])
    scans = (4,) if devmem.EMU else (0, 4)  # the key-driven kernel would stream row 0's 2 GiB under the simulator
    for pred in ("in", "like_substring"):
        want = oracle.filter_indices(PREDICATES[pred](b, field(b, twin)), twin)
        for scan in scans:
            f = gandiva.make_filter(schema, b.make_condition(PREDICATES[pred](b, b.make_field(schema.field(0)))),
                                    gandiva.Configuration(string_scan=scan))
            sel = devmem.DevBuf(n + 8, np.uint32, fill=0)
            cnt = f.evaluate_device(n, [(vld, offs, data, 0)], sel.ptr, n, "UINT32", devmem.stream(), sync=True)
            assert np.array_equal(sel.numpy()[:cnt].astype(np.uint64), want), (pred, scan)
    v = b.make_field(schema.field(0))
    p = gandiva.make_projector(schema, [b.make_expression(v, pa.field("o", S)),
                                        b.make_expression(b.make_function("isnull", [v], pa.bool_()), pa.field("z", pa.bool_()))])
    ovld, ooffs, odata = devmem.DevBuf((n + 31) // 32 + 2, np.int32, fill=0), devmem.DevBuf(n + 1, np.int32, fill=0), \
        devmem.DevBuf(cap + 16, np.uint8, fill=0)
    zvld, zval = devmem.DevBuf((n + 31) // 32 + 2, np.int32, fill=0), devmem.DevBuf((n + 63) // 64 + 2, np.uint64, fill=0)
    p.evaluate_device(n, [(vld, offs, data, 0)], [(ovld.ptr, ooffs.ptr, odata.ptr, cap), (zvld.ptr, zval.ptr)],
                      devmem.stream(), sync=True)
    got = _large_array(n, ovld, ooffs, odata, S)
    assert_arrays_match(got, twin.column(0), "identity with row 0 too long")
    isnull = np.unpackbits(zval.numpy().view(np.uint8), bitorder="little")[:n].astype(bool)
    assert np.array_equal(isnull, ~np.asarray(twin.column(0).is_valid()))


@pytest.mark.skipif(devmem.EMU, reason="more than 2^31 bytes of strings: on the GPU only")
def test_identity_of_more_than_2gib_into_a_large_output(gandiva):
    import torch
    n = 24_000_000
    g = torch.Generator(device="cuda").manual_seed(5)
    lens = torch.randint(0, 180, (n,), device="cuda", generator=g, dtype=torch.int64)
    offs = torch.zeros(n + 1, dtype=torch.int64, device="cuda")
    offs[1:] = torch.cumsum(lens, 0)
    offs += 1000  # rebased output offsets start at 0
    total = int(offs[-1] - offs[0])
    assert total > BIG
    data = torch.randint(0, 256, (int(offs[-1]) + 16,), device="cuda", generator=g, dtype=torch.uint8)
    schema = pa.schema([("v", LS)])
    b = gandiva.TreeExprBuilder()
    cols = [(0, offs.data_ptr(), data.data_ptr(), 0)]
    p = gandiva.make_projector(schema, [b.make_expression(b.make_field(schema.field(0)), pa.field("o", LS))])
    assert p.output_var_size_device(n, cols, 0) == total
    ooffs = torch.zeros(n + 1, dtype=torch.int64, device="cuda")
    odata = torch.zeros(total + 16, dtype=torch.uint8, device="cuda")
    ovld = torch.zeros((n + 31) // 32 + 2, dtype=torch.int32, device="cuda")
    sizes = p.evaluate_device(n, cols, [(ovld.data_ptr(), ooffs.data_ptr(), odata.data_ptr(), total)], sync=True)
    assert sizes == [total]
    assert torch.equal(ooffs, offs - offs[0])
    rows = torch.randint(0, n, (4096,), device="cuda", generator=g)
    for r in rows.tolist()[:256] + [n - 1]:
        a, e = int(offs[r]), int(offs[r + 1])
        assert torch.equal(odata[a - 1000:e - 1000], data[a:e])
    assert torch.equal(odata[total - 4096:total], data[int(offs[-1]) - 4096:int(offs[-1])])
    del odata
    q = gandiva.make_projector(schema, [b.make_expression(b.make_field(schema.field(0)), pa.field("o", S))])
    with pytest.raises(pa.ArrowException, match="2\\^31 - 1"):
        q.output_var_size_device(n, cols, 0)
