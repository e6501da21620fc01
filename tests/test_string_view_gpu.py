"""string_view / binary_view input columns (DESIGN.md §2, §3.7): every Projector and Filter result over a
view batch equals the CPU oracle's over the utf8 / binary twin (`cast(pa.string())`, the plain column
path), validity included, with the inline / prefix shortcut on and off (string_scan bit 3)."""
import ctypes as C
import os

import numpy as np
import pyarrow as pa
import pytest

import devmem
from helpers import assert_arrays_match

pytestmark = pytest.mark.gpu

# above 32 M rows the filters take their large-tile configuration
LARGE = 300_007 if devmem.EMU else (32 << 20) + 3
# lengths 0, 4, 12 and 13 (the inline limit and one past it), non-ASCII text, shared prefixes
WORDS = ["MAIL", "SHIP", "AIR", "REG AIR", "FOB", "", "TWELVE BYTES", "THIRTEEN BYTE", "MAILBOX",
         "héllo wörld", "PROMO BRUSHED BRASS", "PROMO ANODIZED TIN", "STANDARD POLISHED BRASS",
         "MAIL carefully final special requests", "MAIL4", "SHIP SHAPE AND BRISTOL FASHION"]
SHORT = [w for w in WORDS if len(w.encode()) <= 12]
LONG = [w for w in WORDS if len(w.encode()) > 12]


def views(values, nbuf=3, seed=0, invalid=(), binary=False):
    """A string_view (binary_view) array built with from_buffers: rows of more than 12 bytes live in
    `nbuf` data buffers, picked at random per row (so out of order, with gaps between strings); null
    rows' views are random bytes.  `invalid` rows get a view that is invalid Arrow input (a buffer index
    past the last buffer, an offset past the buffer's size, a negative length) while their validity bit
    stays set.  Returns (view array, the twin with those rows null)."""
    rng = np.random.default_rng(seed)
    n = len(values)
    bufs = [bytearray(rng.integers(0, 256, 3).astype(np.uint8).tobytes()) for _ in range(nbuf)]
    vw = np.zeros((max(n, 1), 16), np.uint8)
    valid = np.array([v is not None for v in values], dtype=bool)
    for i, v in enumerate(values):
        if v is None:
            vw[i] = rng.integers(0, 256, 16)
            continue
        b = v.encode() if isinstance(v, str) else v
        vw[i, 0:4] = np.frombuffer(np.int32(len(b)).tobytes(), np.uint8)
        if len(b) <= 12:
            vw[i, 4:4 + len(b)] = np.frombuffer(b, np.uint8)
        else:
            k = int(rng.integers(nbuf))
            bufs[k] += rng.integers(0, 256, int(rng.integers(0, 5))).astype(np.uint8).tobytes()
            vw[i, 4:8] = np.frombuffer(b[:4], np.uint8)
            vw[i, 8:12] = np.frombuffer(np.int32(k).tobytes(), np.uint8)
            vw[i, 12:16] = np.frombuffer(np.int32(len(bufs[k])).tobytes(), np.uint8)
            bufs[k] += b
    bad = set()
    for j, i in enumerate(invalid):
        if values[i] is None:
            continue
        bad.add(i)
        kind = j % 3
        if kind == 0:    # buffer index past the last buffer
            vw[i, 0:4] = np.frombuffer(np.int32(20).tobytes(), np.uint8)
            vw[i, 8:12] = np.frombuffer(np.int32(nbuf + 2).tobytes(), np.uint8)
            vw[i, 12:16] = 0
        elif kind == 1:  # offset + length past the buffer's size
            vw[i, 0:4] = np.frombuffer(np.int32(20).tobytes(), np.uint8)
            vw[i, 8:12] = 0
            vw[i, 12:16] = np.frombuffer(np.int32(len(bufs[0]) - 10).tobytes(), np.uint8)
        else:            # negative length
            vw[i, 0:4] = np.frombuffer(np.int32(-5).tobytes(), np.uint8)
    vtype, ptype = (pa.binary_view(), pa.binary()) if binary else (pa.string_view(), pa.string())
    validity = pa.py_buffer(np.packbits(valid, bitorder="little").tobytes()) if not valid.all() else None
    arr = pa.Array.from_buffers(vtype, n, [validity, pa.py_buffer(vw.tobytes())] + [pa.py_buffer(bytes(b)) for b in bufs],
                                null_count=int((~valid).sum()))
    twin = pa.array([None if (v is None or i in bad) else v for i, v in enumerate(values)], ptype)
    if not bad:
        arr.validate(full=True)
    return arr, twin


def words(n, pool=WORDS, seed=0, nulls=0.1):
    rng = np.random.default_rng(seed)
    idx = rng.integers(0, len(pool), n)
    mask = rng.random(n) < nulls
    return [None if m else pool[i] for i, m in zip(idx, mask)]


def batches(col, twin, seed=1):
    n = len(col)
    rng = np.random.default_rng(seed)
    plain = pa.array(["s%d" % (i % 97) if rng.random() > 0.1 else None for i in range(n)], pa.string())
    return (pa.RecordBatch.from_arrays([col, plain], names=["v", "s"]),
            pa.RecordBatch.from_arrays([twin, plain], names=["v", "s"]))


def field(b, batch, name):
    return b.make_field(batch.schema.field(name))


def lit(b, s, t):
    return b.make_literal(s if t == pa.string() else s.encode(), t)


PREDICATES = {
    "equal": lambda b, v, t: b.make_function("equal", [v, lit(b, "MAIL", t)], pa.bool_()),
    "equal_12": lambda b, v, t: b.make_function("equal", [v, lit(b, "TWELVE BYTES", t)], pa.bool_()),
    "equal_long": lambda b, v, t: b.make_function("equal", [lit(b, "PROMO BRUSHED BRASS", t), v], pa.bool_()),
    "not_equal": lambda b, v, t: b.make_function("not_equal", [v, lit(b, "THIRTEEN BYTE", t)], pa.bool_()),
    "in": lambda b, v, t: b.make_in_expression(v, ["MAIL", "SHIP", "", "héllo wörld"] if t == pa.string()
                                               else [b"MAIL", b"SHIP", b"", "héllo wörld".encode()], t),
    "starts_with": lambda b, v, t: b.make_function("starts_with", [v, lit(b, "MAIL", t)], pa.bool_()),
    "starts_with_long": lambda b, v, t: b.make_function("starts_with", [v, lit(b, "PROMO BRUSHED", t)], pa.bool_()),
    "like_prefix": lambda b, v, t: b.make_function("like", [v, b.make_literal("MAIL%", pa.string())], pa.bool_()),
    "like_prefix_mid": lambda b, v, t: b.make_function("like", [v, b.make_literal("PROMO%BRASS", pa.string())], pa.bool_()),
    "like_one": lambda b, v, t: b.make_function("like", [v, b.make_literal("SH_P%", pa.string())], pa.bool_()),
    "like_substring": lambda b, v, t: b.make_function("like", [v, b.make_literal("%special%requests%", pa.string())],
                                                      pa.bool_()),
    "and_or": lambda b, v, t: b.make_or([
        b.make_and([b.make_function("like", [v, b.make_literal("%A%", pa.string())], pa.bool_()),
                    b.make_function("not_equal", [v, lit(b, "AIR", t)], pa.bool_())]),
        b.make_function("equal", [v, lit(b, "FOB", t)], pa.bool_())]),
}
STRING_ONLY = {"starts_with", "starts_with_long", "like_prefix", "like_prefix_mid", "like_one", "like_substring", "and_or"}


def check_filter(gandiva, oracle, batch, plain, pred, t=pa.string(), dtype="int32"):
    """Both forms (shortcut on / off) select exactly the oracle's rows; returns the indices."""
    b = gandiva.TreeExprBuilder()
    want = oracle.filter_indices(pred(b, field(b, plain, "v"), t), plain, threads=4)
    for scan in (0, 8):
        f = gandiva.make_filter(batch.schema, b.make_condition(pred(b, field(b, batch, "v"), t)),
                                gandiva.Configuration(string_scan=scan))
        got = f.evaluate(batch, None, dtype).to_array().to_numpy().astype(np.uint64)
        assert np.array_equal(got, want), "string_scan=%d: %d rows selected, oracle %d" % (scan, len(got), len(want))
    return want


@pytest.mark.parametrize("kind", ["inline", "out_of_line", "mixed"])
@pytest.mark.parametrize("pred", sorted(PREDICATES))
def test_filters_match_oracle(kind, pred, gandiva, oracle):
    pool = {"inline": SHORT, "out_of_line": LONG, "mixed": WORDS}[kind]
    col, twin = views(words(4099, pool, seed=len(pred)), seed=len(kind))
    check_filter(gandiva, oracle, *batches(col, twin), PREDICATES[pred])


@pytest.mark.parametrize("pred", sorted(set(PREDICATES) - STRING_ONLY))
def test_binary_view_filters(pred, gandiva, oracle):
    col, twin = views(words(3001, seed=9), seed=3, binary=True)
    check_filter(gandiva, oracle, *batches(col, twin), PREDICATES[pred], pa.binary())


def test_shortcut_does_not_trust_inline_padding(gandiva, oracle):
    """Bytes after a short string inside its view are not read as part of it, whatever they hold."""
    vals = words(2000, SHORT, seed=5)
    col, twin = views(vals, seed=5)
    bufs = col.buffers()
    vw = np.frombuffer(bufs[1], np.uint8).reshape(-1, 16).copy()
    for i, v in enumerate(vals):
        if v is not None:
            n = len(v.encode())
            vw[i, 4 + n:] = 0x41   # 'A': "MAIL" + padding would read as "MAILA..."
    col = pa.Array.from_buffers(pa.string_view(), len(vals), [bufs[0], pa.py_buffer(vw.tobytes())] + bufs[2:],
                                null_count=col.null_count)
    for pred in ("equal", "in", "starts_with", "like_prefix", "equal_12"):
        check_filter(gandiva, oracle, *batches(col, twin), PREDICATES[pred])


def test_invalid_views_read_as_null(gandiva, oracle):
    """A view with a bad buffer index, an offset past its buffer or a negative length is invalid Arrow
    input: its row reads as null (never bytes of another row, never memory outside the buffers)."""
    vals = words(3000, seed=6, nulls=0.05)
    col, twin = views(vals, seed=6, invalid=list(range(3, 3000, 7)))
    batch, plain = batches(col, twin)
    for pred in ("equal_long", "in", "like_substring", "not_equal"):
        check_filter(gandiva, oracle, batch, plain, PREDICATES[pred])
    b = gandiva.TreeExprBuilder()
    p = gandiva.make_projector(batch.schema, [b.make_expression(field(b, batch, "v"), pa.field("o", pa.string())),
                                              b.make_expression(b.make_function("isnull", [field(b, batch, "v")], pa.bool_()),
                                                                pa.field("z", pa.bool_()))])
    got_v, got_z = p.evaluate(batch)
    assert_arrays_match(got_v, twin, "invalid views: identity")
    assert np.array_equal(got_z.to_numpy(zero_copy_only=False), ~np.asarray(twin.is_valid()))


@pytest.mark.parametrize("n", [1, 4099, LARGE])
def test_filter_batch_sizes(n, gandiva, oracle):
    rng = np.random.default_rng(n)
    pool = np.array(WORDS, dtype=object)
    twin = pa.array(pool[rng.integers(0, len(WORDS), n)], pa.string(), mask=rng.random(n) < 0.1)
    col = twin.cast(pa.string_view())
    batch, plain = batches(col, twin) if n < 100_000 else (
        pa.RecordBatch.from_arrays([col], names=["v"]), pa.RecordBatch.from_arrays([twin], names=["v"]))
    for pred in ("in", "equal_long"):
        check_filter(gandiva, oracle, batch, plain, PREDICATES[pred], dtype="int64")


def _projections(b, bt):
    v, s = field(b, bt, "v"), field(b, bt, "s")
    fn = b.make_function
    return [(v, pa.string()),
            (fn("upper", [v], pa.string()), pa.string()),
            (fn("substr", [v, b.make_literal(2, pa.int64()), b.make_literal(3, pa.int64())], pa.string()), pa.string()),
            (fn("char_length", [v], pa.int32()), pa.int32()),
            (fn("concat", [v, s], pa.string()), pa.string()),
            (fn("equal", [v, b.make_literal("MAIL", pa.string())], pa.bool_()), pa.bool_()),
            (fn("starts_with", [v, b.make_literal("PROMO B", pa.string())], pa.bool_()), pa.bool_()),
            (b.make_if(fn("equal", [v, b.make_literal("SHIP", pa.string())], pa.bool_()), s, v, pa.string()), pa.string())]


def check_projections(gandiva, oracle, batch, plain):
    b = gandiva.TreeExprBuilder()
    want_roots = _projections(b, plain)
    want = oracle.project([r for r, _ in want_roots], [t for _, t in want_roots], plain, threads=4)
    for scan in (0, 8):
        outs = _projections(b, batch)
        p = gandiva.make_projector(batch.schema, [b.make_expression(r, pa.field("o%d" % i, t))
                                                  for i, (r, t) in enumerate(outs)],
                                   configuration=gandiva.Configuration(string_scan=scan))
        for i, (g, w) in enumerate(zip(p.evaluate(batch), want)):
            assert_arrays_match(g, w, "projection %d, string_scan=%d" % (i, scan))


@pytest.mark.parametrize("offset", [0, 5, 33])
def test_projections_match_oracle(offset, gandiva, oracle):
    col, twin = views(words(3001 + offset, seed=7), seed=7)
    batch, plain = batches(col, twin)
    check_projections(gandiva, oracle, batch.slice(offset), plain.slice(offset))


def test_sliced_filter(gandiva, oracle):
    col, twin = views(words(5000, seed=8), seed=8)
    batch, plain = batches(col, twin)
    for pred in ("equal_long", "like_prefix_mid"):
        check_filter(gandiva, oracle, batch.slice(37, 4000), plain.slice(37, 4000), PREDICATES[pred])


def _to_device(keep, data, n_bytes):
    buf = devmem.DevBuf(max(n_bytes, 1) + 64, np.uint8, fill=0)
    if n_bytes:
        import gandiva_b200
        gandiva_b200.memcpy_htod(0, buf.ptr, np.frombuffer(data, dtype=np.uint8)[:n_bytes].copy())
    keep.append(buf)
    return buf.ptr


def _device_columns(gandiva, batch, keep):
    """The batch's buffers copied to the device whole (offsets kept); a view column gets a
    gdv_view_buffers_t of device pointers with its sizes in device memory."""
    cols = []
    for c in batch.columns:
        bb = c.buffers()
        vld = _to_device(keep, bb[0], bb[0].size) if bb[0] is not None and c.null_count else 0
        val = _to_device(keep, bb[1], bb[1].size)
        if pa.types.is_string_view(c.type) or pa.types.is_binary_view(c.type):
            data = [_to_device(keep, x, x.size) for x in bb[2:]]
            sizes = np.array([x.size for x in bb[2:]] or [0], np.int64)
            vb = gandiva.view_buffers(data, _to_device(keep, sizes.tobytes(), sizes.nbytes))
            keep.append(vb)
            cols.append((vld, val, vb, c.offset))
        else:
            cols.append((vld, val, _to_device(keep, bb[2], bb[2].size), c.offset))
    return cols


@pytest.mark.parametrize("pred", ["in", "like_substring"])
def test_device_batch_filter_then_projector(pred, gandiva, oracle):
    """Device-resident view batch: the Filter writes selection + count on the device, a Projector reads
    both on the same stream (tests/test_chain_gpu.py's shape)."""
    n = 20_011
    col, twin = views(words(n + 9, seed=11), seed=11)
    batch, plain = batches(col, twin)
    batch, plain = batch.slice(9), plain.slice(9)
    keep = []
    cols = _device_columns(gandiva, batch, keep)
    b = gandiva.TreeExprBuilder()
    want_idx = oracle.filter_indices(PREDICATES[pred](b, field(b, plain, "v"), pa.string()), plain, threads=4)
    f = gandiva.make_filter(batch.schema, b.make_condition(PREDICATES[pred](b, field(b, batch, "v"), pa.string())))
    proj = gandiva.make_projector(batch.schema, [b.make_expression(b.make_function("char_length", [field(b, batch, "v")], pa.int32()),
                                                                   pa.field("len", pa.int32()))], None, "UINT32")
    want_len, = oracle.project([b.make_function("char_length", [field(b, plain, "v")], pa.int32())], [pa.int32()], plain,
                               selection=want_idx.astype(np.int64))
    st = devmem.stream()
    sel = devmem.DevBuf(n + 8, np.uint32, fill=0)
    cnt = devmem.DevBuf(1, np.int64, fill=0)
    out = devmem.DevBuf(n + 8, np.int32, fill=0)
    ovl = devmem.DevBuf((n + 31) // 32 + 2, np.int32, fill=0)
    f.evaluate_device(n, cols, sel.ptr, n, "UINT32", st, cnt.ptr, sync=False)
    proj.evaluate_device(n, cols, [(ovl.ptr, out.ptr)], st, selection=(sel.ptr, n, cnt.ptr))
    proj.sync(st)
    count = f.sync(st)
    assert count == len(want_idx)
    assert np.array_equal(sel.numpy()[:count].astype(np.uint64), want_idx)
    got = pa.Array.from_buffers(pa.int32(), count, [pa.py_buffer(ovl.numpy().view(np.uint8)),
                                                    pa.py_buffer(out.numpy()[: max(count, 1)].copy())])
    assert_arrays_match(got, want_len, "chained char_length")


def test_row_range_shard_is_a_slice_of_the_views(gandiva, oracle):
    """A shard of a view batch = the same data buffers + a slice of the views; index_base makes the
    selection global (what sharding.py does for every column)."""
    n = 10_000
    col, twin = views(words(n, seed=4), seed=4)
    batch, plain = batches(col, twin)
    b = gandiva.TreeExprBuilder()
    want = oracle.filter_indices(PREDICATES["like_prefix_mid"](b, field(b, plain, "v"), pa.string()), plain)
    f = gandiva.make_filter(batch.schema, b.make_condition(PREDICATES["like_prefix_mid"](b, field(b, batch, "v"), pa.string())))
    keep = []
    cols = _device_columns(gandiva, batch, keep)
    got = []
    for lo, hi in ((0, 4096), (4096, 10_000)):
        shard = [(v, i, d, off + lo) for v, i, d, off in cols]
        sel = devmem.DevBuf(hi - lo + 8, np.uint64, fill=0)
        cnt = f.evaluate_device(hi - lo, shard, sel.ptr, hi - lo, "UINT64", devmem.stream(), sync=True, index_base=lo)
        got.append(sel.numpy()[:cnt])
    assert np.array_equal(np.concatenate(got).astype(np.uint64), want)


def test_arrow_c_device_import_of_a_view_child(gandiva, oracle):
    """pyarrow's C Device exporter -> the engine's import (views, data buffers and sizes read in place)."""
    col, twin = views(words(12_345 + 17, seed=8), seed=8)
    batch, plain = batches(col, twin)
    batch, plain = batch.slice(17), plain.slice(17)
    b = gandiva.TreeExprBuilder()
    want = oracle.filter_indices(PREDICATES["and_or"](b, field(b, plain, "v"), pa.string()), plain, threads=4)
    f = gandiva.make_filter(batch.schema, b.make_condition(PREDICATES["and_or"](b, field(b, batch, "v"), pa.string())))
    imported = gandiva.ArrowDeviceBatch.from_record_batch(batch)
    res = f.evaluate_arrow(imported, "UINT32")
    ts = gandiva.ArrowSchemaC()
    pa.uint32()._export_to_c(C.addressof(ts))
    got = pa.Array._import_from_c_device(res.address, C.addressof(ts))
    assert np.array_equal(got.to_numpy().astype(np.uint64), want)
    imported.release()
    p = gandiva.make_projector(batch.schema, [b.make_expression(b.make_function("upper", [field(b, batch, "v")], pa.string()),
                                                                pa.field("u", pa.string()))])
    imported = gandiva.ArrowDeviceBatch.from_record_batch(batch)
    got = p.evaluate_arrow(imported).to_record_batch()
    w, = oracle.project([b.make_function("upper", [field(b, plain, "v")], pa.string())], [pa.string()], plain)
    assert_arrays_match(got.column(0), w, "upper through the Arrow C Device import")
    imported.release()


def test_cpp_layer_matches_the_mirror(gandiva):
    """The C++ namespace-gandiva layer (through the stock pyarrow binding, when it is built) reads a
    host string_view batch like the Python mirror does."""
    here = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "conformance", "stock")
    if not os.path.isdir(here) or not any(f.startswith("gandiva.") and f.endswith(".so") for f in os.listdir(here)):
        pytest.skip("the stock pyarrow binding over the C++ layer is not built")
    from conformance.run_stock_tests import load_stock_module
    stock = load_stock_module()
    col, twin = views(words(5000, seed=12), seed=12)
    batch, _ = batches(col, twin)
    outs = []
    for mod in (stock, gandiva):
        b = mod.TreeExprBuilder()
        v = b.make_field(batch.schema.field("v"))
        up = b.make_function("upper", [v], pa.string())
        p = mod.make_projector(batch.schema, [b.make_expression(up, pa.field("u", pa.string()))], pa.default_memory_pool())
        cond = b.make_condition(b.make_in_expression(v, ["MAIL", "SHIP"], pa.string()))
        f = mod.make_filter(batch.schema, cond)
        outs.append((p.evaluate(batch)[0], f.evaluate(batch, pa.default_memory_pool()).to_array()))
    assert_arrays_match(outs[0][0], outs[1][0], "C++ layer: upper")
    assert np.array_equal(outs[0][1].to_numpy(), outs[1][1].to_numpy())
