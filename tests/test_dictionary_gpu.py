"""Dictionary-encoded utf8 / binary input columns (DESIGN.md §2, §3.6): every Projector and Filter result
over a dictionary batch equals the CPU oracle's over the decoded twin (`dictionary_decode()`, the plain
column path), validity included, on both filter paths: the dictionary-first kernel (a condition over
the one dictionary column, evaluated once per entry) and the general row kernel (the same condition
with a conjunct over a plain column added, which is always true)."""
import ctypes as C

import numpy as np
import pyarrow as pa
import pytest

import devmem
from helpers import assert_arrays_match

pytestmark = pytest.mark.gpu

# above 32 M rows the filters take their large-tile configuration
LARGE = 300_007 if devmem.EMU else (32 << 20) + 3
WORDS = ["MAIL", "SHIP", "AIR", "REG AIR", "FOB", "TRUCK", "RAIL", "MAIL", "héllo wörld", "",
         "STANDARD POLISHED BRASS", "ECONOMY ANODIZED STEEL"]
INDEX_TYPES = [pa.int8(), pa.int16(), pa.int32(), pa.int64()]


def dict_column(n, index_type=pa.int32(), seed=0, card=12, null_idx=0.1, null_entry=True, idx_offset=0,
                dict_offset=0, value_type=pa.string()):
    """A DictionaryArray of n rows over `card` entries (duplicates included, unused ones too when n is
    small), optionally with null indices / entries and sliced indices / dictionary."""
    rng = np.random.default_rng(seed)
    entries = [WORDS[i % len(WORDS)] for i in range(card + dict_offset)]
    dvalid = [not (null_entry and i % 5 == 3) for i in range(card + dict_offset)]
    dictionary = pa.array([e if v else None for e, v in zip(entries, dvalid)], type=pa.string())
    if value_type == pa.binary():
        dictionary = dictionary.cast(pa.binary())
    dictionary = dictionary.slice(dict_offset)
    m = n + idx_offset
    idx = rng.integers(0, max(card, 1), m) if card > 0 else np.zeros(m, dtype=np.int64)
    mask = rng.random(m) < null_idx if card > 0 else np.ones(m, dtype=bool)
    indices = pa.array(idx.astype(index_type.to_pandas_dtype()), type=index_type, mask=mask)
    return pa.DictionaryArray.from_arrays(indices, dictionary).slice(idx_offset)


def dict_batch(col, seed=1):
    n = len(col)
    rng = np.random.default_rng(seed)
    plain = pa.array(["s%d" % (i % 97) if rng.random() > 0.1 else None for i in range(min(n, 5000))] *
                     (n // 5000 + 1), type=pa.string()).slice(0, n) if n else pa.array([], pa.string())
    return pa.RecordBatch.from_arrays([col, plain], names=["d", "s"])


def decoded(batch):
    cols = [c.dictionary_decode() if pa.types.is_dictionary(c.type) else c for c in batch.columns]
    return pa.RecordBatch.from_arrays(cols, names=batch.schema.names)


def field(b, batch, name):
    return b.make_field(batch.schema.field(name))


PREDICATES = {
    "like": lambda b, d, t: b.make_function("like", [d, b.make_literal("%AI%", t)], pa.bool_()),
    "in": lambda b, d, t: b.make_in_expression(d, ["MAIL", "SHIP"] if t == pa.string() else [b"MAIL", b"SHIP"], t),
    "regexp": lambda b, d, t: b.make_function("regexp_matches", [d, b.make_literal("^(M|T)", pa.string())], pa.bool_()),
    "equal": lambda b, d, t: b.make_function("equal", [d, b.make_literal("SHIP", t)], pa.bool_()),
    "and_or": lambda b, d, t: b.make_or([
        b.make_and([b.make_function("like", [d, b.make_literal("%A%", t)], pa.bool_()),
                    b.make_function("not_equal", [d, b.make_literal("RAIL", t)], pa.bool_())]),
        b.make_function("equal", [d, b.make_literal("FOB", t)], pa.bool_())]),
}


def _always_true(b, s):
    return b.make_or([b.make_function("isnull", [s], pa.bool_()), b.make_function("isnotnull", [s], pa.bool_())])


def _filters(gandiva, batch, pred, value_type=pa.string(), plain=None):
    """(dictionary-first filter, general-path filter, oracle condition over the decoded batch)."""
    plain = decoded(batch) if plain is None else plain
    b = gandiva.TreeExprBuilder()
    cond = pred(b, field(b, batch, "d"), value_type)
    general = b.make_and([pred(b, field(b, batch, "d"), value_type), _always_true(b, field(b, batch, "s"))])
    want = pred(b, field(b, plain, "d"), value_type)
    return (gandiva.make_filter(batch.schema, b.make_condition(cond)),
            gandiva.make_filter(batch.schema, b.make_condition(general)), want, plain)


def _check_filter(gandiva, oracle, batch, pred, value_type=pa.string(), dtype="int32"):
    first, general, want_cond, plain = _filters(gandiva, batch, pred, value_type)
    want = oracle.filter_indices(want_cond, plain, threads=4)
    got1 = first.evaluate(batch, None, dtype)
    assert first.kernel_info["dictionary_first"] == 1
    got2 = general.evaluate(batch, None, dtype)
    assert general.kernel_info["dictionary_first"] == 0
    for what, got in (("dictionary-first", got1), ("general", got2)):
        g = got.to_array().to_numpy().astype(np.uint64)
        assert np.array_equal(g, want), "%s path: %d rows selected, oracle %d" % (what, len(g), len(want))
    return want


@pytest.mark.parametrize("index_type", INDEX_TYPES, ids=str)
@pytest.mark.parametrize("pred", sorted(PREDICATES))
def test_filter_paths_match_oracle(index_type, pred, gandiva, oracle):
    col = dict_column(4099, index_type, seed=len(pred), idx_offset=5, dict_offset=2)
    _check_filter(gandiva, oracle, dict_batch(col), PREDICATES[pred])


@pytest.mark.parametrize("n", [1, 4099, LARGE])
def test_filter_batch_sizes(n, gandiva, oracle):
    col = dict_column(n, pa.int16(), seed=n, card=7)
    for mode in (("int64",) if n == LARGE else ("int16", "int32", "int64")):
        if mode == "int16" and n > 65536:
            continue
        _check_filter(gandiva, oracle, dict_batch(col), PREDICATES["in"], dtype=mode)


def test_filter_binary_dictionary(gandiva, oracle):
    col = dict_column(3001, pa.int32(), seed=9, value_type=pa.binary())
    _check_filter(gandiva, oracle, dict_batch(col), PREDICATES["in"], value_type=pa.binary())


def test_condition_satisfied_by_null_takes_the_general_path(gandiva, oracle):
    """isnull(d) OR d = 'MAIL' keeps null rows: no per-entry bit can say that, so the row kernel runs."""
    batch = dict_batch(dict_column(5000, pa.int8(), seed=3))
    plain = decoded(batch)
    b = gandiva.TreeExprBuilder()
    mk = lambda bt: b.make_or([b.make_function("isnull", [field(b, bt, "d")], pa.bool_()),
                               b.make_function("equal", [field(b, bt, "d"), b.make_literal("MAIL", pa.string())], pa.bool_())])
    f = gandiva.make_filter(batch.schema, b.make_condition(mk(batch)))
    got = f.evaluate(batch).to_array().to_numpy().astype(np.uint64)
    assert f.kernel_info["dictionary_first"] == 0
    assert np.array_equal(got, oracle.filter_indices(mk(plain), plain))


def _projections(b, bt):
    d, s = field(b, bt, "d"), field(b, bt, "s")
    fn = b.make_function
    return [(d, pa.string()),
            (fn("upper", [d], pa.string()), pa.string()),
            (fn("substr", [d, b.make_literal(2, pa.int64()), b.make_literal(3, pa.int64())], pa.string()), pa.string()),
            (fn("char_length", [d], pa.int32()), pa.int32()),
            (fn("concat", [d, s], pa.string()), pa.string()),
            (fn("hash32", [d], pa.int32()), pa.int32()),
            (fn("hashSHA256", [d], pa.string()), pa.string()),
            (b.make_if(fn("equal", [d, b.make_literal("MAIL", pa.string())], pa.bool_()), s, d, pa.string()), pa.string()),
            (fn("like", [fn("concat", [d, s], pa.string()), b.make_literal("%AIs1%", pa.string())], pa.bool_()), pa.bool_())]


def _check_projections(gandiva, oracle, batch):
    plain = decoded(batch)
    b = gandiva.TreeExprBuilder()
    outs = _projections(b, batch)
    p = gandiva.make_projector(batch.schema, [b.make_expression(r, pa.field("o%d" % i, t)) for i, (r, t) in enumerate(outs)])
    got = p.evaluate(batch)
    want_roots = _projections(b, plain)
    want = oracle.project([r for r, _ in want_roots], [t for _, t in want_roots], plain, threads=4)
    for i, (g, w) in enumerate(zip(got, want)):
        assert_arrays_match(g, w, "projection %d over %s" % (i, batch.schema.field("d").type))


@pytest.mark.parametrize("index_type", INDEX_TYPES, ids=str)
def test_projections_match_oracle(index_type, gandiva, oracle):
    _check_projections(gandiva, oracle, dict_batch(dict_column(3001, index_type, seed=7, idx_offset=3, dict_offset=4)))


@pytest.mark.parametrize("case", ["no_nulls", "duplicates_unused", "all_null_indices", "empty_dictionary", "one_row"])
def test_edge_dictionaries(case, gandiva, oracle):
    col = {"no_nulls": lambda: dict_column(2000, pa.int32(), null_idx=0.0, null_entry=False),
           "duplicates_unused": lambda: dict_column(40, pa.int8(), card=12, seed=2),
           "all_null_indices": lambda: dict_column(1000, pa.int16(), null_idx=1.0),
           "empty_dictionary": lambda: dict_column(777, pa.int64(), card=0),
           "one_row": lambda: dict_column(1, pa.int32(), null_idx=0.0)}[case]()
    batch = dict_batch(col)
    _check_projections(gandiva, oracle, batch)
    _check_filter(gandiva, oracle, batch, PREDICATES["like"])


def test_out_of_range_indices_read_as_null(gandiva, oracle):
    """An index outside [0, dictionary length) is invalid Arrow input: the row reads as null (never the
    bytes of another entry, never memory past the dictionary) in projections and on both filter paths."""
    n = 3000
    rng = np.random.default_rng(5)
    idx = rng.integers(0, 7, n).astype(np.int8)
    bad = np.zeros(n, dtype=bool)
    bad[::7] = True
    idx[::7] = np.array([-1, 7, 100, 127, -128], dtype=np.int8)[np.arange(len(idx[::7])) % 5]
    dictionary = pa.array(WORDS[:7], pa.string())
    col = pa.DictionaryArray.from_arrays(pa.array(idx, pa.int8()), dictionary, safe=False)
    batch = dict_batch(col)
    # the expectation: the same rows with the bad indices null
    sane = pa.DictionaryArray.from_arrays(pa.array(np.where(bad, 0, idx), pa.int8(), mask=bad), dictionary)
    plain = decoded(dict_batch(sane))
    b = gandiva.TreeExprBuilder()
    p = gandiva.make_projector(batch.schema, [b.make_expression(field(b, batch, "d"), pa.field("o", pa.string())),
                                              b.make_expression(b.make_function("isnull", [field(b, batch, "d")], pa.bool_()),
                                                                pa.field("z", pa.bool_()))])
    got_s, got_z = p.evaluate(batch)
    assert_arrays_match(got_s, plain.column(0), "out-of-range identity")
    assert np.array_equal(got_z.to_numpy(zero_copy_only=False), bad | ~np.asarray(plain.column(0).is_valid()))
    first, general, want_cond, _ = _filters(gandiva, batch, PREDICATES["like"], plain=plain)
    want = oracle.filter_indices(want_cond, plain)
    for f in (first, general):
        assert np.array_equal(f.evaluate(batch).to_array().to_numpy().astype(np.uint64), want)


def _to_device(keep, arr_bytes, n_bytes):
    buf = devmem.DevBuf(max(n_bytes, 1) + 64, np.uint8, fill=0)
    if n_bytes:
        import gandiva_b200
        gandiva_b200.memcpy_htod(0, buf.ptr, np.frombuffer(arr_bytes, dtype=np.uint8)[:n_bytes].copy())
    keep.append(buf)
    return buf.ptr


def _device_columns(gandiva, batch, keep):
    """The batch's buffers copied to the device whole (offsets kept), dictionary columns with a
    gdv_dictionary_t of device pointers."""
    cols = []
    for c in batch.columns:
        if pa.types.is_dictionary(c.type):
            ib = c.buffers()
            w = c.type.index_type.bit_width // 8
            vld = _to_device(keep, ib[0], ib[0].size) if ib[0] is not None and c.null_count else 0
            idx = _to_device(keep, ib[1], ib[1].size)
            d = c.dictionary
            db = d.buffers()
            dd = gandiva.gdv_dictionary_t()
            dd.validity = _to_device(keep, db[0], db[0].size) if db[0] is not None and d.null_count else None
            dd.offsets = _to_device(keep, db[1], db[1].size) if db[1] is not None else None
            dd.data = _to_device(keep, db[2], db[2].size) if db[2] is not None else None
            dd.offset, dd.length = d.offset, len(d)
            keep.append(dd)
            cols.append((vld, idx, dd, c.offset))
            assert w in (1, 2, 4, 8)
        else:
            bb = c.buffers()
            vld = _to_device(keep, bb[0], bb[0].size) if bb[0] is not None and c.null_count else 0
            cols.append((vld, _to_device(keep, bb[1], bb[1].size), _to_device(keep, bb[2], bb[2].size), c.offset))
    return cols


@pytest.mark.parametrize("pred", ["in", "regexp"])
def test_device_batch_filter_then_projector(pred, gandiva, oracle):
    """Device-resident dictionary batch: Filter (both paths) writes selection + count on the device,
    a Projector reads both on the same stream (tests/test_chain_gpu.py's shape)."""
    n = 20_011
    batch = dict_batch(dict_column(n, pa.int32(), seed=11, idx_offset=9, dict_offset=3))
    plain = decoded(batch)
    keep = []
    cols = _device_columns(gandiva, batch, keep)
    first, general, want_cond, _ = _filters(gandiva, batch, PREDICATES[pred])
    want_idx = oracle.filter_indices(want_cond, plain, threads=4)
    b = gandiva.TreeExprBuilder()
    proj = gandiva.make_projector(batch.schema, [b.make_expression(b.make_function("char_length", [field(b, batch, "d")], pa.int32()),
                                                                   pa.field("len", pa.int32()))], None, "UINT32")
    want_len, = oracle.project([b.make_function("char_length", [field(b, plain, "d")], pa.int32())], [pa.int32()], plain,
                               selection=want_idx.astype(np.int64))
    st = devmem.stream()
    for f, path in ((first, 1), (general, 0)):
        sel = devmem.DevBuf(n + 8, np.uint32, fill=0)
        cnt = devmem.DevBuf(1, np.int64, fill=0)
        out = devmem.DevBuf(n + 8, np.int32, fill=0)
        ovl = devmem.DevBuf((n + 31) // 32 + 2, np.int32, fill=0)
        f.evaluate_device(n, cols, sel.ptr, n, "UINT32", st, cnt.ptr, sync=False)
        proj.evaluate_device(n, cols, [(ovl.ptr, out.ptr)], st, selection=(sel.ptr, n, cnt.ptr))
        proj.sync(st)
        count = f.sync(st)
        assert f.kernel_info["dictionary_first"] == path
        assert count == len(want_idx)
        assert np.array_equal(sel.numpy()[:count].astype(np.uint64), want_idx)
        got = pa.Array.from_buffers(pa.int32(), count, [pa.py_buffer(ovl.numpy().view(np.uint8)),
                                                        pa.py_buffer(out.numpy()[: max(count, 1)].copy())])
        assert_arrays_match(got, want_len, "chained char_length, path %d" % path)


def test_row_range_shard_is_a_slice_of_the_indices(gandiva, oracle):
    """A shard of a dictionary batch = the same dictionary + a slice of the indices; index_base makes the
    selection global (what sharding.py does for every column)."""
    n = 10_000
    batch = dict_batch(dict_column(n, pa.int16(), seed=4))
    first, _, want_cond, plain = _filters(gandiva, batch, PREDICATES["like"])
    want = oracle.filter_indices(want_cond, plain)
    keep = []
    cols = _device_columns(gandiva, batch, keep)
    got = []
    for lo, hi in ((0, 4096), (4096, 10_000)):
        shard = [(v, i, d, off + lo) for v, i, d, off in cols]
        sel = devmem.DevBuf(hi - lo + 8, np.uint64, fill=0)
        cnt = first.evaluate_device(hi - lo, shard, sel.ptr, hi - lo, "UINT64", devmem.stream(), sync=True, index_base=lo)
        got.append(sel.numpy()[:cnt])
    assert np.array_equal(np.concatenate(got).astype(np.uint64), want)


def test_arrow_c_device_import_of_a_dictionary_child(gandiva, oracle):
    """pyarrow's C Device exporter -> the engine's import (dictionary child read in place) -> results."""
    batch = dict_batch(dict_column(12_345, pa.int64(), seed=8, idx_offset=17, dict_offset=1))
    plain = decoded(batch)
    first, general, want_cond, _ = _filters(gandiva, batch, PREDICATES["and_or"])
    want = oracle.filter_indices(want_cond, plain, threads=4)
    for f in (first, general):
        imported = gandiva.ArrowDeviceBatch.from_record_batch(batch)
        res = f.evaluate_arrow(imported, "UINT32")
        ts = gandiva.ArrowSchemaC()
        pa.uint32()._export_to_c(C.addressof(ts))
        got = pa.Array._import_from_c_device(res.address, C.addressof(ts))
        assert np.array_equal(got.to_numpy().astype(np.uint64), want)
        imported.release()
    b = gandiva.TreeExprBuilder()
    p = gandiva.make_projector(batch.schema, [b.make_expression(b.make_function("upper", [field(b, batch, "d")], pa.string()),
                                                                pa.field("u", pa.string()))])
    imported = gandiva.ArrowDeviceBatch.from_record_batch(batch)
    got = p.evaluate_arrow(imported).to_record_batch()
    w, = oracle.project([b.make_function("upper", [field(b, plain, "d")], pa.string())], [pa.string()], plain)
    assert_arrays_match(got.column(0), w, "upper through the Arrow C Device import")
    imported.release()
