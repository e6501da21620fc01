"""Filter -> Projector kept on the device with utf8 / binary outputs: the Projector reads the slot count the
Filter left in device memory (gdv_selection_t.d_num_slots) in its sizing pass, the tile scan and its write
pass, and checks the byte total against the caller's var_capacity on the device.  Nothing returns to the
host between the two enqueues.  Bit-exact against oracle.filter_indices + oracle.project(selection=...):
offsets 0..c, bytes and validity; buffers past the count keep their sentinel."""
import numpy as np
import pyarrow as pa
import pytest

import devmem
from helpers import assert_arrays_match

pytestmark = pytest.mark.gpu

S, BIN, I32, I64, F64, B = pa.string(), pa.binary(), pa.int32(), pa.int64(), pa.float64(), pa.bool_()
OFFSET = 5   # every column is a slice: bitmaps and values start past the buffers' first rows
WORDS = ["carefully", "final", "deposits", "sleep", "quickly", "regular", "requests", "haggle", "blithely",
         "ironic", "accounts", "furiously", "pending", "packages", "Tiresias", "héllo", "wörld", "日本"]
MODES = ["MAIL", "SHIP", "AIR", "REG AIR", "FOB", "TRUCK", "RAIL", ""]
OFFS_FILL, DATA_FILL, VLD_FILL = 0x7EEEEEEE, 0xEE, np.int32(-0x11111112)   # VLD_FILL = 0xEEEEEEEE
N_STRING_OUTPUTS = 5


def make_batch(n, seed=3):
    """A lineitem-like batch of n rows (as slices at OFFSET): the Q6 columns, an l_comment-like utf8
    column, a binary column, a dictionary-encoded utf8 column and a string_view column, with nulls.
    Returns (batch, its plain twin: dictionary decoded, views cast to utf8)."""
    rng = np.random.default_rng(seed)
    m = n + OFFSET
    comments = [" ".join(rng.choice(WORDS, size=int(rng.integers(1, 7)))) for _ in range(257)]
    blobs = [rng.integers(0, 256, int(rng.integers(0, 20))).astype(np.uint8).tobytes() for _ in range(61)]
    mask = lambda p: rng.random(m) < p
    ship = pa.array((8035 + rng.integers(0, 2527, m)).astype(np.int32), pa.int32()).cast(pa.date32())
    disc = pa.array(rng.integers(0, 11, m) / 100.0, F64, mask=mask(0.02))
    qty = pa.array(rng.integers(1, 51, m).astype(np.int64), I64, mask=mask(0.02))
    ci, cm = rng.integers(0, len(comments), m), mask(0.05)
    comment = pa.array([None if k else comments[i] for i, k in zip(ci, cm)], S)
    bi, bm = rng.integers(0, len(blobs), m), mask(0.05)
    blob = pa.array([None if k else blobs[i] for i, k in zip(bi, bm)], BIN)
    mode = pa.DictionaryArray.from_arrays(pa.array(rng.integers(0, len(MODES), m).astype(np.int32), I32, mask=mask(0.05)),
                                          pa.array(MODES + [None], S))
    vi, vm = rng.integers(0, len(comments), m), mask(0.05)
    view = pa.array([None if k else comments[i][:int(i % 30)] for i, k in zip(vi, vm)], S).cast(pa.string_view())
    names = ["l_shipdate", "l_discount", "l_quantity", "l_comment", "l_bin", "l_mode", "l_view"]
    cols = [ship, disc, qty, comment, blob, mode, view]
    batch = pa.RecordBatch.from_arrays(cols, names=names).slice(OFFSET)
    plain_cols = [c.dictionary_decode() if pa.types.is_dictionary(c.type) else
                  c.cast(S) if pa.types.is_string_view(c.type) else c for c in batch.columns]
    return batch, pa.RecordBatch.from_arrays(plain_cols, names=names)


def condition(b, batch, kind):
    f = {x.name: b.make_field(x) for x in batch.schema}
    fn, SD = b.make_function, pa.date32()
    if kind == "all":
        return fn("greater_than_or_equal_to", [f["l_shipdate"], b.make_literal(0, SD)], B)
    if kind == "none":
        return fn("less_than", [f["l_shipdate"], b.make_literal(0, SD)], B)
    return b.make_and([fn("greater_than_or_equal_to", [f["l_shipdate"], b.make_literal(8766, SD)], B),
                       fn("less_than", [f["l_shipdate"], b.make_literal(9131, SD)], B),
                       fn("greater_than_or_equal_to", [f["l_discount"], b.make_literal(0.05, F64)], B),
                       fn("less_than_or_equal_to", [f["l_discount"], b.make_literal(0.07, F64)], B),
                       fn("less_than", [f["l_quantity"], b.make_literal(24, I64)], B)])


def outputs(b, batch):
    """Five utf8 / binary outputs, then one fixed-width output."""
    f = {x.name: b.make_field(x) for x in batch.schema}
    fn = b.make_function
    return [(fn("upper", [fn("substr", [f["l_comment"], b.make_literal(1, I64), b.make_literal(12, I64)], S)], S), S),
            (fn("concat", [f["l_comment"], b.make_literal("|", S), f["l_mode"]], S), S),   # a projected rope
            (fn("castVARCHAR", [f["l_quantity"], b.make_literal(10, I64)], S), S),
            (fn("byte_substr", [f["l_bin"], b.make_literal(2, I32), b.make_literal(5, I32)], BIN), BIN),
            (fn("lower", [f["l_view"]], S), S),
            (fn("char_length", [f["l_view"]], I32), I32)]


def _to_device(keep, buf, n_bytes):
    d = devmem.DevBuf(max(n_bytes, 1) + 64, np.uint8, fill=0)
    if n_bytes:
        import gandiva_b200
        gandiva_b200.memcpy_htod(0, d.ptr, np.frombuffer(buf, dtype=np.uint8)[:n_bytes].copy())
    keep.append(d)
    return d.ptr


def device_columns(gandiva, batch, keep):
    """The batch's buffers copied to the device whole (array offsets kept); a dictionary column with a
    gdv_dictionary_t, a view column with a gdv_view_buffers_t of device pointers."""
    cols = []
    for c in batch.columns:
        bb = c.buffers()
        vld = _to_device(keep, bb[0], bb[0].size) if bb[0] is not None and c.null_count else 0
        if pa.types.is_dictionary(c.type):
            d = c.dictionary
            db = d.buffers()
            dd = gandiva.gdv_dictionary_t()
            dd.validity = _to_device(keep, db[0], db[0].size) if db[0] is not None and d.null_count else None
            dd.offsets, dd.data = _to_device(keep, db[1], db[1].size), _to_device(keep, db[2], db[2].size)
            dd.offset, dd.length = d.offset, len(d)
            keep.append(dd)
            cols.append((vld, _to_device(keep, bb[1], bb[1].size), dd, c.offset))
        elif pa.types.is_string_view(c.type):
            data = [_to_device(keep, x, x.size) for x in bb[2:]]
            sizes = np.array([x.size for x in bb[2:]] or [0], np.int64)
            vb = gandiva.view_buffers(data, _to_device(keep, sizes.tobytes(), sizes.nbytes))
            keep.append(vb)
            cols.append((vld, _to_device(keep, bb[1], bb[1].size), vb, c.offset))
        else:
            var = _to_device(keep, bb[2], bb[2].size) if len(bb) > 2 else 0
            cols.append((vld, _to_device(keep, bb[1], bb[1].size), var, c.offset))
    return cols


class StringOut:
    """Device buffers of one utf8 / binary output, filled with sentinels."""

    def __init__(self, n, capacity, slack=64):
        self.capacity = capacity
        self.offs = devmem.DevBuf(n + 1 + 8, np.int32, fill=OFFS_FILL)
        self.data = devmem.DevBuf(capacity + slack, np.uint8, fill=DATA_FILL)
        self.vld = devmem.DevBuf((n + 31) // 32 + 2, np.int32, fill=VLD_FILL)

    def arg(self):
        return (self.vld.ptr, self.offs.ptr, self.data.ptr, self.capacity)


def expected_offsets(want):
    lens = np.array([0 if x is None else len(x.encode() if isinstance(x, str) else x) for x in want.to_pylist()], np.int64)
    return np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)


def check_string_output(got, want, count, what):
    """Offsets 0..count, bytes and validity against the oracle; nothing past the count written."""
    offs, data, vld = got.offs.numpy(), got.data.numpy(), got.vld.numpy()
    exp = expected_offsets(want) if count else np.zeros(1, np.int64)
    assert np.array_equal(offs[: count + 1].astype(np.int64), exp), what + ": offsets"
    assert (offs[count + 1:] == OFFS_FILL).all(), what + ": offsets written past the count"
    total = int(exp[-1])
    want_bytes = b""
    if count:
        want_bytes = b"".join(x.encode() if isinstance(x, str) else x for x in want.to_pylist() if x is not None)
    assert data[:total].tobytes() == want_bytes, what + ": bytes"
    assert (data[total:] == DATA_FILL).all(), what + ": bytes written past offsets[count]"
    words = (count + 31) // 32
    if count:
        bits = np.packbits(np.asarray(want.is_valid().to_numpy(zero_copy_only=False), bool), bitorder="little")
        exp_vld = np.zeros(words * 4, np.uint8)
        exp_vld[: len(bits)] = bits
        assert np.array_equal(vld[:words].view(np.uint8), exp_vld), what + ": validity"
        arr = pa.Array.from_buffers(want.type, count, [pa.py_buffer(vld[:words].tobytes()), pa.py_buffer(offs[: count + 1].tobytes()),
                                                       pa.py_buffer(data[: max(total, 1)].tobytes())])
        assert_arrays_match(arr, want, what)
    assert (vld[words:] == VLD_FILL).all(), what + ": validity words past the count written"
    return total


def run_chain(gandiva, oracle, n, mode, kind, capacity_slack=100, sync_projector=False):
    """Filter + Projector over one device batch, chained through the device count.  Returns a dict with
    the count, the string outputs' totals and what the launches / the output_var_size path saw."""
    npt = {"UINT16": np.uint16, "UINT32": np.uint32, "UINT64": np.uint64}[mode]
    batch, plain = make_batch(n)
    b = gandiva.TreeExprBuilder()
    filt = gandiva.make_filter(batch.schema, b.make_condition(condition(b, batch, kind)))
    outs = outputs(b, batch)
    proj = gandiva.make_projector(batch.schema, [b.make_expression(r, pa.field("o%d" % i, t)) for i, (r, t) in enumerate(outs)],
                                  None, mode)
    want_idx = oracle.filter_indices(condition(b, plain, kind), plain, threads=4)
    want_roots = outputs(b, plain)
    want = (oracle.project([r for r, _ in want_roots], [t for _, t in want_roots], plain,
                           selection=want_idx.astype(np.int64), threads=4) if len(want_idx) else None)
    keep = []
    cols = device_columns(gandiva, batch, keep)
    st = devmem.stream()
    sel = devmem.DevBuf(n * np.dtype(npt).itemsize + 16, np.uint8, fill=0)
    cnt = devmem.DevBuf(1, np.int64, fill=0)
    totals = [0 if want is None else int(expected_offsets(want[k])[-1]) for k in range(N_STRING_OUTPUTS)]
    souts = [StringOut(n, t + capacity_slack) for t in totals]
    fixed = devmem.DevBuf(n + 8, np.int32, fill=-0x11111112)
    fixed_vld = devmem.DevBuf((n + 31) // 32 + 2, np.int32, fill=0)
    launches = gandiva.launch_count()
    # ---- the chain: two enqueues, no synchronisation and no count on the host in between
    filt.evaluate_device(n, cols, sel.ptr, n, mode, st, cnt.ptr, sync=False)
    var_sizes = proj.evaluate_device(n, cols, [o.arg() for o in souts] + [(fixed_vld.ptr, fixed.ptr)], st,
                                     selection=(sel.ptr, n, cnt.ptr), sync=sync_projector)
    enqueued = gandiva.launch_count() - launches
    if not sync_projector:
        proj.sync(st)
    count = filt.sync(st)
    assert count == len(want_idx) == int(cnt.numpy()[0])
    assert np.array_equal(sel.numpy().view(npt)[:count].astype(np.uint64), want_idx)
    got_totals = [check_string_output(souts[k], want[k] if want is not None else None, count,
                                      "output %d (n=%d, %s, %s)" % (k, n, mode, kind)) for k in range(N_STRING_OUTPUTS)]
    fv = fixed.numpy()
    if count:
        arr = pa.Array.from_buffers(I32, count, [pa.py_buffer(fixed_vld.numpy().tobytes()), pa.py_buffer(fv[:count].tobytes())])
        assert_arrays_match(arr, want[N_STRING_OUTPUTS], "fixed-width output (n=%d, %s, %s)" % (n, mode, kind))
    assert (fv[count:n] == -0x11111112).all(), "fixed-width output written past the count"
    # the opt-in exact size: sizing pass + scan over the device count, one round trip
    exact = [proj.output_var_size_device(n, cols, k, st, selection=(sel.ptr, n, cnt.ptr)) for k in range(N_STRING_OUTPUTS)]
    return dict(count=count, totals=got_totals, exact=exact, enqueued=enqueued, var_sizes=var_sizes, proj=proj)


CASES = [(n, mode) for n in (1, 4097, 300_011) for mode in ("UINT16", "UINT32", "UINT64") if mode != "UINT16" or n < 65536]


@pytest.mark.parametrize("n,mode", CASES)
def test_chain_with_string_outputs_matches_oracle(n, mode, gandiva, oracle):
    r = run_chain(gandiva, oracle, n, mode, "q6")
    assert r["enqueued"] == 1 + 1 + 3 * N_STRING_OUTPUTS
    assert r["exact"] == r["totals"]
    assert r["var_sizes"] is None


@pytest.mark.parametrize("kind", ["none", "all"])
@pytest.mark.parametrize("n", [1, 4097, 300_011])
def test_chain_keeping_no_row_or_every_row(kind, n, gandiva, oracle):
    r = run_chain(gandiva, oracle, n, "UINT32", kind)
    assert r["count"] == (0 if kind == "none" else n)
    assert r["exact"] == r["totals"]


def test_synchronous_call_returns_var_size(gandiva, oracle):
    r = run_chain(gandiva, oracle, 4097, "UINT64", "q6", sync_projector=True)
    assert r["var_sizes"] == r["totals"] + [None]


@pytest.mark.parametrize("sync_projector", [False, True])
def test_capacity_one_byte_short(sync_projector, gandiva, oracle):
    """var_capacity one byte below the total: ExecutionError naming the capacity; the bytes from
    var_capacity on keep their sentinel.  Exactly the total succeeds."""
    n = 4097
    batch, plain = make_batch(n)
    b = gandiva.TreeExprBuilder()
    filt = gandiva.make_filter(batch.schema, b.make_condition(condition(b, batch, "q6")))
    root, t = outputs(b, batch)[1]
    proj = gandiva.make_projector(batch.schema, [b.make_expression(root, pa.field("o", t))], None, "UINT32")
    want_idx = oracle.filter_indices(condition(b, plain, "q6"), plain, threads=4)
    want, = oracle.project([outputs(b, plain)[1][0]], [t], plain, selection=want_idx.astype(np.int64), threads=4)
    total = int(expected_offsets(want)[-1])
    assert total > 0
    keep = []
    cols = device_columns(gandiva, batch, keep)
    st = devmem.stream()
    for cap, ok in ((total - 1, False), (total, True)):
        sel = devmem.DevBuf(n + 8, np.uint32, fill=0)
        cnt = devmem.DevBuf(1, np.int64, fill=0)
        out = StringOut(n, cap)
        filt.evaluate_device(n, cols, sel.ptr, n, "UINT32", st, cnt.ptr, sync=False)
        call = lambda: proj.evaluate_device(n, cols, [out.arg()], st, selection=(sel.ptr, n, cnt.ptr), sync=sync_projector)
        if ok:
            sizes = call()
            if not sync_projector:
                proj.sync(st)
            else:
                assert sizes == [total]
            assert filt.sync(st) == len(want_idx)
            check_string_output(out, want, len(want_idx), "capacity == total")
        else:
            with pytest.raises(gandiva.GandivaError, match="ExecutionError: var_data capacity of a utf8/binary output is too "
                                                           "small: output 0 needs %d bytes, its var_capacity is %d" % (total, cap)):
                call()
                proj.sync(st)
            filt.sync(st)
            assert (out.data.numpy()[cap:] == DATA_FILL).all(), "a byte stored at or past var_capacity"


def test_refusals(gandiva, oracle):
    """A host batch with d_num_slots is Invalid; a utf8 output that needs a rope temporary is NotImplemented
    (its temporaries are sized on the host), while a fixed-width output of such a projector still chains."""
    import ctypes as C
    n = 4097
    batch, plain = make_batch(n)
    b = gandiva.TreeExprBuilder()
    f = {x.name: b.make_field(x) for x in batch.schema}
    fn = b.make_function
    cnt = devmem.DevBuf(1, np.int64, fill=0)
    # host batch
    proj = gandiva.make_projector(batch.schema, [b.make_expression(outputs(b, batch)[0][0], pa.field("o", S))], None, "UINT32")
    cb, _keep = gandiva._batch_to_c(batch)
    idx = np.arange(n, dtype=np.uint32)
    hsel = gandiva.gdv_selection_t(idx.ctypes.data_as(C.c_void_p), n, n, gandiva.GDV_SEL_UINT32, gandiva.GDV_MEM_HOST, 0,
                                   C.c_void_p(cnt.ptr))
    offs, vld, data = np.zeros(n + 1, np.int32), np.zeros(n // 8 + 16, np.uint8), np.zeros(1 << 16, np.uint8)
    outs = (gandiva.gdv_out_column_t * 1)()
    outs[0].validity, outs[0].values = vld.ctypes.data_as(C.c_void_p), offs.ctypes.data_as(C.c_void_p)
    outs[0].var_data, outs[0].var_capacity = data.ctypes.data_as(C.c_void_p), data.size
    with pytest.raises(pa.ArrowInvalid, match="d_num_slots needs device buffers"):
        gandiva._check(gandiva.lib.gdv_projector_evaluate(proj._h, C.byref(cb), C.byref(hsel), outs, 1, None, 0))
    # the two-stage rope plan
    keep = []
    cols = device_columns(gandiva, batch, keep)
    st = devmem.stream()
    sel = devmem.DevBuf(n + 8, np.uint32, fill=0)
    filt = gandiva.make_filter(batch.schema, b.make_condition(condition(b, batch, "q6")))
    padded = fn("substr", [fn("lpad", [f["l_comment"], b.make_literal(20, I32), b.make_literal("*", S)], S),
                           b.make_literal(2, I64), b.make_literal(5, I64)], S)
    rope = gandiva.make_projector(batch.schema, [b.make_expression(padded, pa.field("p", S))], None, "UINT32")
    out = StringOut(n, 8 * n)
    filt.evaluate_device(n, cols, sel.ptr, n, "UINT32", st, cnt.ptr, sync=False)
    filt.sync(st)
    with pytest.raises(pa.ArrowNotImplementedError, match="two-stage rope plan"):
        rope.evaluate_device(n, cols, [out.arg()], st, selection=(sel.ptr, n, cnt.ptr))
    with pytest.raises(pa.ArrowNotImplementedError, match="two-stage rope plan"):
        rope.output_var_size_device(n, cols, 0, st, selection=(sel.ptr, n, cnt.ptr))
    assert (out.offs.numpy() == OFFS_FILL).all()
    # a fixed-width output over a rope temporary keeps accepting the device count
    like = fn("like", [fn("concat", [f["l_comment"], b.make_literal(" ", S), f["l_mode"]], S), b.make_literal("%y r%", S)], B)
    pl = gandiva.make_projector(batch.schema, [b.make_expression(like, pa.field("l", B))], None, "UINT32")
    bits = devmem.DevBuf((n + 31) // 32 + 2, np.int32, fill=0)
    bvld = devmem.DevBuf((n + 31) // 32 + 2, np.int32, fill=0)
    pl.evaluate_device(n, cols, [(bvld.ptr, bits.ptr)], st, selection=(sel.ptr, n, cnt.ptr), sync=True)
    count = int(cnt.numpy()[0])
    pf = {x.name: b.make_field(x) for x in plain.schema}
    want_like = fn("like", [fn("concat", [pf["l_comment"], b.make_literal(" ", S), pf["l_mode"]], S), b.make_literal("%y r%", S)], B)
    want_idx = oracle.filter_indices(condition(b, plain, "q6"), plain, threads=4)
    assert count == len(want_idx) > 0
    want, = oracle.project([want_like], [B], plain, selection=want_idx.astype(np.int64), threads=4)
    got = pa.Array.from_buffers(B, count, [pa.py_buffer(bvld.numpy().tobytes()), pa.py_buffer(bits.numpy().tobytes())])
    assert_arrays_match(got, want, "like over a rope temporary, chained")
