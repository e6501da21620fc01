"""The evaluation runtime's contract at its edges: the refusals a caller meets before any launch (exact
type and message), how many launches each kind of evaluation makes, what one stream's pending state
does between an asynchronous Evaluate and its Sync, and the device pool's trim.  Every case is refused
on the host before a launch or is an ExecutionError the kernels raise by design."""
import ctypes as C

import numpy as np
import pyarrow as pa
import pytest

import cases
import devmem

pytestmark = pytest.mark.gpu

I32, I64, S, B = pa.int32(), pa.int64(), pa.string(), pa.bool_()


def _raises(exc, msg, fn, *args, **kw):
    with pytest.raises(exc) as e:
        fn(*args, **kw)
    assert str(e.value) == msg


def _to_device(keep, data, pad=64):
    a = np.frombuffer(bytes(data), dtype=np.uint8)
    d = devmem.DevBuf(a.size + pad, np.uint8, fill=0)
    if a.size:
        import gandiva_b200
        gandiva_b200.memcpy_htod(0, d.ptr, a.copy())
    keep.append(d)
    return d.ptr


def _fixed_device_columns(batch, keep):
    """(validity|0, values, 0, offset) per fixed-width column of `batch`, copied to the device whole."""
    cols = []
    for c in batch.columns:
        bb = c.buffers()
        vld = _to_device(keep, bb[0]) if bb[0] is not None and c.null_count else 0
        cols.append((vld, _to_device(keep, bb[1]), 0, c.offset))
    return cols


def _device_dictionary(gandiva, keep, dictionary):
    db = dictionary.buffers()
    dd = gandiva.gdv_dictionary_t()
    dd.validity = None
    dd.offsets, dd.data = _to_device(keep, db[1]), _to_device(keep, db[2])
    dd.offset, dd.length, dd.data_size = dictionary.offset, len(dictionary), db[2].size
    keep.append(dd)
    return dd


def _dict_batch(n):
    idx = pa.array((np.arange(n) % 3).astype(np.int32), I32)
    return pa.RecordBatch.from_arrays([pa.DictionaryArray.from_arrays(idx, pa.array(["MAIL", "SHIP", "AIR"], S))],
                                      names=["d"])


def _project(gandiva, schema, root, t, mode="NONE"):
    b = gandiva.TreeExprBuilder()
    return gandiva.make_projector(schema, [b.make_expression(root(b, [b.make_field(f) for f in schema]), pa.field("o", t))],
                                  None, mode)


def _filter(gandiva, schema, cond):
    b = gandiva.TreeExprBuilder()
    return gandiva.make_filter(schema, b.make_condition(cond(b, [b.make_field(f) for f in schema])))


def _dict_filter(gandiva, schema):
    """A condition over the one dictionary column that no null satisfies: the dictionary-first plan."""
    return _filter(gandiva, schema, lambda b, fs: b.make_in_expression(fs[0], ["MAIL", "AIR"], S))


# ---- 1. refusals ------------------------------------------------------------------------------------------
def test_misaligned_device_buffers_are_refused(gandiva):
    n, keep = 1000, []
    st = devmem.stream()
    out = devmem.DevBuf(n + 8, np.int32, fill=0)
    # a fixed-width column two bytes past its element alignment
    schema = pa.schema([("a", I32)])
    p = _project(gandiva, schema, lambda b, fs: b.make_function("negative", [fs[0]], I32), I32)
    vals = _to_device(keep, np.arange(n + 4, dtype=np.int32).tobytes())
    _raises(pa.ArrowInvalid, "device values buffer of column 0 is not aligned to its element width",
            p.evaluate_device, n, [(0, vals + 2, 0, 0)], [(0, out.ptr)], st, sync=True)
    # dictionary indices, through the row kernel and through the dictionary-first filter
    batch = _dict_batch(n)
    col = batch.column(0)
    dd = _device_dictionary(gandiva, keep, col.dictionary)
    idx = _to_device(keep, col.indices.buffers()[1])
    pd = _project(gandiva, batch.schema, lambda b, fs: b.make_function("octet_length", [fs[0]], I32), I32)
    _raises(pa.ArrowInvalid, "device indices buffer of column 0 is not aligned to its element width",
            pd.evaluate_device, n, [(0, idx + 2, dd, 0)], [(0, out.ptr)], st, sync=True)
    fd = _dict_filter(gandiva, batch.schema)
    sel = devmem.DevBuf(n + 8, np.uint32, fill=0)
    _raises(pa.ArrowInvalid, "device indices buffer of column 0 is not aligned to its element width",
            fd.evaluate_device, n, [(0, idx + 2, dd, 0)], sel.ptr, n, "UINT32", st, sync=True)
    # 16-byte views eight bytes off
    view = pa.array(["a short one", "a string longer than twelve bytes", None] * (n // 3 + 1), S).slice(0, n)
    view = view.cast(pa.string_view())
    vb = view.buffers()
    sizes = np.array([x.size for x in vb[2:]] or [0], np.int64)
    tbl = gandiva.view_buffers([_to_device(keep, x) for x in vb[2:]], _to_device(keep, sizes.tobytes()))
    keep.append(tbl)
    pv = _project(gandiva, pa.schema([("v", pa.string_view())]),
                  lambda b, fs: b.make_function("octet_length", [fs[0]], I32), I32)
    views = _to_device(keep, vb[1])
    _raises(pa.ArrowInvalid, "device views buffer of column 0 is not 16-byte aligned",
            pv.evaluate_device, n, [(0, views + 8, tbl, 0)], [(0, out.ptr)], st, sync=True)


def test_missing_buffers_are_refused(gandiva):
    n, keep = 1000, []
    st = devmem.stream()
    out = devmem.DevBuf(n + 8, np.int32, fill=0)
    p = _project(gandiva, pa.schema([("a", I32)]), lambda b, fs: b.make_function("negative", [fs[0]], I32), I32)
    _raises(pa.ArrowInvalid, "column 0 has no values buffer", p.evaluate_device, n, [(0, 0, 0, 0)], [(0, out.ptr)], st,
            sync=True)
    batch = _dict_batch(n)
    idx = _to_device(keep, batch.column(0).indices.buffers()[1])
    pd = _project(gandiva, batch.schema, lambda b, fs: b.make_function("octet_length", [fs[0]], I32), I32)
    _raises(pa.ArrowInvalid, "dictionary column 0 has no dictionary (var_data must point at a gdv_dictionary_t)",
            pd.evaluate_device, n, [(0, idx, 0, 0)], [(0, out.ptr)], st, sync=True)


def _host_selection(gandiva, idx, n, mode, d_num_slots=None):
    return gandiva.gdv_selection_t(idx.ctypes.data_as(C.c_void_p), len(idx), n, mode, gandiva.GDV_MEM_HOST, 0,
                                   d_num_slots)


def test_device_slot_count_needs_device_buffers(gandiva):
    """d_num_slots over a host batch is refused by a fixed-width-only projector as by a utf8 one."""
    n = 1000
    batch = pa.record_batch([pa.array(np.arange(n, dtype=np.int64))], names=["a"])
    cnt = devmem.DevBuf(1, np.int64, fill=n)
    idx = np.arange(n, dtype=np.uint32)
    sel = _host_selection(gandiva, idx, n, gandiva.GDV_SEL_UINT32, C.c_void_p(cnt.ptr))
    cb, _keep = gandiva._batch_to_c(batch)
    fixed = _project(gandiva, batch.schema, lambda b, fs: b.make_function("negative", [fs[0]], I64), I64, "UINT32")
    vals, vld = np.zeros(n + 8, np.int64), np.zeros(n // 8 + 16, np.uint8)
    outs = (gandiva.gdv_out_column_t * 1)()
    outs[0].validity, outs[0].values = vld.ctypes.data_as(C.c_void_p), vals.ctypes.data_as(C.c_void_p)
    _raises(pa.ArrowInvalid, "d_num_slots needs device buffers",
            gandiva._check, gandiva.lib.gdv_projector_evaluate(fixed._h, C.byref(cb), C.byref(sel), outs, 1, None, 0))
    text = _project(gandiva, batch.schema, lambda b, fs: b.make_function("castVARCHAR", [fs[0], b.make_literal(10, I64)], S),
                    S, "UINT32")
    offs, data = np.zeros(n + 1, np.int32), np.zeros(1 << 16, np.uint8)
    outs[0].values = offs.ctypes.data_as(C.c_void_p)
    outs[0].var_data, outs[0].var_capacity = data.ctypes.data_as(C.c_void_p), data.size
    _raises(pa.ArrowInvalid, "d_num_slots needs device buffers",
            gandiva._check, gandiva.lib.gdv_projector_evaluate(text._h, C.byref(cb), C.byref(sel), outs, 1, None, 0))


def test_selection_argument_refusals(gandiva):
    n = 1000
    batch = pa.record_batch([pa.array(np.arange(n, dtype=np.int32))], names=["a"])
    cb, _keep = gandiva._batch_to_c(batch)
    dev_idx = devmem.DevBuf(n + 8, np.uint32, fill=0)
    # projector: a device selection vector over a host batch
    p = _project(gandiva, batch.schema, lambda b, fs: b.make_function("negative", [fs[0]], I32), I32, "UINT32")
    dsel = gandiva.gdv_selection_t(dev_idx.ptr, n, n, gandiva.GDV_SEL_UINT32, gandiva.GDV_MEM_DEVICE)
    vals = np.zeros(n + 8, np.int32)
    outs = (gandiva.gdv_out_column_t * 1)()
    outs[0].values = vals.ctypes.data_as(C.c_void_p)
    _raises(pa.ArrowInvalid, "selection vector and batch must share a memory space",
            gandiva._check, gandiva.lib.gdv_projector_evaluate(p._h, C.byref(cb), C.byref(dsel), outs, 1, None, 0))
    # filter
    f = _filter(gandiva, batch.schema, lambda b, fs: b.make_function("less_than", [fs[0], b.make_literal(500, I32)], B))

    def run(sel):
        gandiva._check(gandiva.lib.gdv_filter_evaluate(f._h, C.byref(cb), C.byref(sel), None, 0, None))

    _raises(pa.ArrowInvalid, "selection vector and batch must share a memory space", run, dsel)
    idx = np.zeros(n + 8, np.uint32)
    bounded = _host_selection(gandiva, idx, 0, gandiva.GDV_SEL_UINT32 | gandiva.GDV_SEL_BOUNDED)
    _raises(pa.ArrowInvalid, "a bounded selection vector needs device buffers", run, bounded)
    short = gandiva.gdv_selection_t(idx.ctypes.data_as(C.c_void_p), n - 1, 0, gandiva.GDV_SEL_UINT32, gandiva.GDV_MEM_HOST)
    _raises(pa.ArrowInvalid, "Selection vector max_slots %d is less than the number of rows %d" % (n - 1, n), run, short)
    big = pa.record_batch([pa.array(np.arange(65537, dtype=np.int32))], names=["a"])
    _raises(pa.ArrowInvalid, "batch too large for a uint16 selection vector", f.evaluate, big, None, "int16")


def test_host_utf8_output_one_byte_short(gandiva):
    n = 1000
    batch = pa.record_batch([pa.array(np.arange(n, dtype=np.int64))], names=["a"])
    cb, _keep = gandiva._batch_to_c(batch)
    p = _project(gandiva, batch.schema, lambda b, fs: b.make_function("castVARCHAR", [fs[0], b.make_literal(10, I64)], S), S)
    need = C.c_int64(0)
    gandiva._check(gandiva.lib.gdv_projector_output_var_size(p._h, C.byref(cb), None, 0, None, C.byref(need)))
    total = sum(len(str(i)) for i in range(n))
    assert need.value == total
    offs, vld, data = np.zeros(n + 1, np.int32), np.zeros(n // 8 + 16, np.uint8), np.zeros(total, np.uint8)
    outs = (gandiva.gdv_out_column_t * 1)()
    outs[0].validity, outs[0].values = vld.ctypes.data_as(C.c_void_p), offs.ctypes.data_as(C.c_void_p)
    outs[0].var_data, outs[0].var_capacity = data.ctypes.data_as(C.c_void_p), total - 1
    _raises(pa.ArrowInvalid, "var_data capacity %d is smaller than the %d bytes the output needs (see var_size)"
            % (total - 1, total), gandiva._check, gandiva.lib.gdv_projector_evaluate(p._h, C.byref(cb), None, outs, 1, None, 0))
    assert outs[0].var_size == total


# ---- 2. launches per call ---------------------------------------------------------------------------------
def _launches(gandiva, fn, *args, **kw):
    before = gandiva.launch_count()
    fn(*args, **kw)
    return gandiva.launch_count() - before


def test_launches_per_call(gandiva):
    n = 5000
    batch = pa.record_batch([pa.array(np.arange(n, dtype=np.int64))], names=["a"])
    fixed = _project(gandiva, batch.schema, lambda b, fs: b.make_function("negative", [fs[0]], I64), I64)
    fixed.evaluate(batch)   # the first call may compile the no-null variant
    assert _launches(gandiva, fixed.evaluate, batch) == 1
    text = _project(gandiva, batch.schema, lambda b, fs: b.make_function("castVARCHAR", [fs[0], b.make_literal(10, I64)], S), S)
    text.evaluate(batch)
    before = gandiva.launch_count()
    cb, _keep = gandiva._batch_to_c(batch)
    offs, data = np.zeros(n + 1, np.int32), np.zeros(8 * n, np.uint8)
    outs = (gandiva.gdv_out_column_t * 1)()
    outs[0].values = offs.ctypes.data_as(C.c_void_p)
    outs[0].var_data, outs[0].var_capacity = data.ctypes.data_as(C.c_void_p), data.size
    gandiva._check(gandiva.lib.gdv_projector_evaluate(text._h, C.byref(cb), None, outs, 1, None, 0))
    assert gandiva.launch_count() - before == 3   # sizing pass, tile scan, write pass
    assert outs[0].var_size == sum(len(str(i)) for i in range(n))
    fused = _filter(gandiva, batch.schema, lambda b, fs: b.make_function("less_than", [fs[0], b.make_literal(500, I64)], B))
    fused.evaluate(batch)
    assert _launches(gandiva, fused.evaluate, batch) == 1
    dbatch = _dict_batch(n)
    dfirst = _dict_filter(gandiva, dbatch.schema)
    dfirst.evaluate(dbatch)
    assert _launches(gandiva, dfirst.evaluate, dbatch) == 2   # the entries, then the rows
    assert dfirst.kernel_info["dictionary_first"] == 1
    # a fixed-width projector over an empty selection launches nothing
    pe = _project(gandiva, batch.schema, lambda b, fs: b.make_function("negative", [fs[0]], I64), I64, "UINT32")
    pe.evaluate(batch, gandiva.SelectionVector(np.arange(4, dtype=np.uint32), 4, gandiva.GDV_SEL_UINT32))
    empty = gandiva.SelectionVector(np.zeros(8, np.uint32), 0, gandiva.GDV_SEL_UINT32)
    assert _launches(gandiva, pe.evaluate, batch, empty) == 0


# ---- 3. pending state on one stream ------------------------------------------------------------------------
def test_two_async_filters_then_one_sync(gandiva, oracle):
    """The second batch has more row tiles, so the stream's look-back state block grows between the two
    launches; the first block stays alive until Sync, which returns the second count."""
    b = gandiva.TreeExprBuilder()
    cond = cases.q6_condition(b)
    f = gandiva.make_filter(cases.Q6_SCHEMA, b.make_condition(cond))
    small = cases.q6_batch(3000, seed=5, null_permille=10)
    keep = []
    st = devmem.stream()
    n1 = small.num_rows
    c1 = _fixed_device_columns(small, keep)
    s1, k1 = devmem.DevBuf(n1 + 8, np.uint32, fill=0), devmem.DevBuf(1, np.int64, fill=0)
    f.evaluate_device(n1, c1, s1.ptr, n1, "UINT32", st, k1.ptr, sync=True)   # compiles and loads the kernel
    tile_rows = f.kernel_info["tile_rows"]
    n2 = 3 * tile_rows + 17
    assert (n2 + tile_rows - 1) // tile_rows > (n1 + tile_rows - 1) // tile_rows
    large = cases.q6_batch(n2, seed=6, null_permille=10)
    c2 = _fixed_device_columns(large, keep)
    s2, k2 = devmem.DevBuf(n2 + 8, np.uint32, fill=0), devmem.DevBuf(1, np.int64, fill=0)
    assert f.evaluate_device(n1, c1, s1.ptr, n1, "UINT32", st, k1.ptr, sync=False) == -1
    assert f.evaluate_device(n2, c2, s2.ptr, n2, "UINT32", st, k2.ptr, sync=False) == -1
    count = f.sync(st)
    w1 = oracle.filter_indices(cond, small, threads=4)
    w2 = oracle.filter_indices(cond, large, threads=4)
    assert count == len(w2) > 0
    assert int(k1.numpy()[0]) == len(w1) > 0
    assert np.array_equal(s1.numpy()[:len(w1)].astype(np.uint64), w1)
    assert np.array_equal(s2.numpy()[:len(w2)].astype(np.uint64), w2)


def test_async_projector_error_then_clean_call(gandiva):
    n, keep = 4096, []
    schema = pa.schema([("a", I32), ("b", I32)])
    p = _project(gandiva, schema, lambda b, fs: b.make_function("divide", fs, I32), I32)
    st = devmem.stream()
    a = np.arange(n, dtype=np.int32)
    d = np.full(n, 7, dtype=np.int32)
    d[n - 3] = 0
    out = devmem.DevBuf(n + 8, np.int32, fill=0)
    bad = [(0, _to_device(keep, a.tobytes()), 0, 0), (0, _to_device(keep, d.tobytes()), 0, 0)]
    assert p.evaluate_device(n, bad, [(0, out.ptr)], st, sync=False) is None
    _raises(gandiva.GandivaError, "ExecutionError: divide by zero error", p.sync, st)
    d[n - 3] = 7
    good = [(0, _to_device(keep, a.tobytes()), 0, 0), (0, _to_device(keep, d.tobytes()), 0, 0)]
    p.evaluate_device(n, good, [(0, out.ptr)], st, sync=True)
    assert np.array_equal(out.numpy()[:n], a // 7)


# ---- 4. pool -----------------------------------------------------------------------------------------------
def test_trim_releases_the_idle_pool(gandiva):
    b = gandiva.TreeExprBuilder()
    f = gandiva.make_filter(cases.Q6_SCHEMA, b.make_condition(cases.q6_condition(b)))
    for n in (1000, 70_000):
        f.evaluate(cases.q6_batch(n, seed=n))
    released = C.c_size_t(0)
    gandiva._check(gandiva.lib.gdv_device_trim(0, 0, C.byref(released)))
    assert released.value > 0
    again = C.c_size_t(1)
    gandiva._check(gandiva.lib.gdv_device_trim(0, 0, C.byref(again)))
    assert again.value == 0
