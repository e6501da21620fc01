"""User-defined functions on the device (DESIGN.md §3.8): every result is compared bit for bit with numpy and,
where one exists, with the same expression built from built-ins.  The bodies stay within what both NVRTC and
the simulator's host compiler accept (plain C++ over the library's types and accessors)."""
import os

import numpy as np
import pyarrow as pa
import pyarrow.compute as pc
import pytest

import cases
import devmem
from helpers import assert_arrays_match
from test_dictionary_gpu import dict_batch, dict_column
from test_string_view_gpu import LARGE, views, words

pytestmark = pytest.mark.gpu

B, I32, I64, F32, F64, S = pa.bool_(), pa.int32(), pa.int64(), pa.float32(), pa.float64(), pa.string()
D32, TS = pa.date32(), pa.timestamp("ms")
FNV = ("u32 h = 2166136261u;\nfor (i32 i = 0; i < a0.len; ++i) { h ^= (u32)gdv_ch(a0, i); h *= 16777619u; }\n"
       "return (i32)h;")


@pytest.fixture(scope="module")
def reg(gandiva):
    r = _PerWorker(gandiva.FunctionRegistry())
    r.register("fahrenheit", [F64], F64, "return a0 * 1.8 + 32.0;")
    r.register("halve", [F32], F32, "return a0 * 0.5f;")
    r.register("is_even", [I64], B, "return (a0 & 1) == 0;")
    r.register("negate", [B], B, "return !a0;")
    r.register("next_day", [D32], D32, "return a0 + 1;")
    r.register("hour_later", [TS], TS, "return a0 + 3600000;")
    r.register("or_else", [I32, I32], I32, "return v0 ? a0 : (v1 ? a1 : -1);", null_mode="never")
    r.register("non_negative", [I32], I32, "*out_valid = v0 && a0 >= 0;\nreturn a0;", null_mode="internal")
    r.register("checked", [I32], I32, 'if (a0 == 7) gdv_raise(ctx, "seven is not allowed here");\nreturn a0 + 1;',
               can_raise=True)
    r.register("count_byte", [S, I32], I32,
               "i32 n = 0;\nfor (i32 i = 0; i < a0.len; ++i) n += gdv_ch(a0, i) == (u8)a1;\nreturn n;")
    r.register("fnv1a", [S], I32, FNV)
    r.register("between_f64", [F64, F64, F64], B, "return a0 >= a1 && a0 <= a2;")
    r.register("lt24", [F64], B, "return a0 < 24.0;")
    r.register("in_1994", [D32], B, "return a0 >= 8766 && a0 < 9131;")
    return r.reg


class _PerWorker:
    """Under the simulator every pytest-xdist worker registers these functions at the same moment, and its
    compile cache does not expect two processes to build the same new source at once: there, a comment naming
    the worker keeps their sources apart."""

    def __init__(self, reg):
        self.reg = reg

    def register(self, name, params, ret, body, **kw):
        if devmem.EMU:
            body += "  // %s" % os.environ.get("PYTEST_XDIST_WORKER", "main")
        self.reg.register(name, params, ret, body, **kw)


def _project(gandiva, reg, batch, roots, selection=None):
    b, exprs = roots[0], [roots[0].make_expression(r, pa.field("o%d" % i, t)) for i, (r, t) in enumerate(roots[1])]
    mode = "NONE" if selection is None else "UINT32"
    p = gandiva.make_projector(batch.schema, exprs, None, mode, gandiva.Configuration(function_registry=reg))
    return p.evaluate(batch) if selection is None else p.evaluate(batch, selection)


def _nullable(values, t, seed, nulls=0.15):
    rng = np.random.default_rng(seed)
    return pa.array(values, t, mask=rng.random(len(values)) < nulls)


def _fnv(s, upper=False):
    h = 2166136261
    for c in (s.upper() if upper else s).encode():
        h = ((h ^ c) * 16777619) & 0xffffffff
    return h - (1 << 32) if h >= (1 << 31) else h


def test_fixed_width_types_and_null_modes(gandiva, reg):
    n = 10_007
    rng = np.random.default_rng(3)
    x = rng.normal(10, 40, n)
    batch = pa.RecordBatch.from_arrays(
        [_nullable(x, F64, 1), _nullable(x.astype(np.float32), F32, 2), _nullable(rng.integers(-9, 9, n), I64, 3),
         _nullable(rng.integers(-5, 12, n).astype(np.int32), I32, 4), _nullable(rng.integers(-5, 12, n).astype(np.int32), I32, 5),
         _nullable(rng.integers(8000, 9500, n).astype(np.int32), D32, 6), _nullable(rng.integers(0, 1 << 40, n), TS, 7),
         _nullable(rng.random(n) < 0.5, B, 8)], names=["d", "f", "l", "a", "c", "day", "ts", "flag"])
    b = gandiva.TreeExprBuilder()
    f = {x.name: b.make_field(x) for x in batch.schema}
    fn = b.make_function
    roots = [(fn("fahrenheit", [f["d"]], F64), F64), (fn("halve", [f["f"]], F32), F32), (fn("is_even", [f["l"]], B), B),
             (fn("negate", [f["flag"]], B), B), (fn("next_day", [f["day"]], D32), D32), (fn("hour_later", [f["ts"]], TS), TS),
             (fn("or_else", [f["a"], f["c"]], I32), I32), (fn("non_negative", [f["a"]], I32), I32),
             # nested in each other and in built-ins
             (fn("add", [fn("or_else", [fn("non_negative", [f["a"]], I32), f["c"]], I32), fn("non_negative", [f["c"]], I32)], I32), I32),
             # the same from built-ins
             (fn("add", [fn("multiply", [f["d"], b.make_literal(1.8, F64)], F64), b.make_literal(32.0, F64)], F64), F64)]
    got = _project(gandiva, reg, batch, (b, roots))
    col = {k: batch.column(i) for i, k in enumerate(batch.schema.names)}
    npv = lambda a, fill=0: a.fill_null(fill).to_numpy(zero_copy_only=False)
    mask = lambda a: ~np.asarray(a.is_valid())
    assert_arrays_match(got[0], pa.array(npv(col["d"]) * 1.8 + 32.0, F64, mask=mask(col["d"])), "fahrenheit")
    assert_arrays_match(got[0], got[9], "fahrenheit against multiply / add")
    assert_arrays_match(got[1], pa.array(npv(col["f"]) * np.float32(0.5), F32, mask=mask(col["f"])), "halve")
    assert_arrays_match(got[2], pa.array(npv(col["l"]) % 2 == 0, B, mask=mask(col["l"])), "is_even")
    assert_arrays_match(got[3], pc.invert(col["flag"]), "negate")
    assert_arrays_match(got[4], pa.array(npv(col["day"].cast(I32)) + 1, I32, mask=mask(col["day"])).cast(D32), "next_day")
    assert_arrays_match(got[5], pa.array(npv(col["ts"].cast(I64)) + 3600000, I64, mask=mask(col["ts"])).cast(TS), "hour_later")
    a, c = col["a"], col["c"]
    assert_arrays_match(got[6], pc.coalesce(a, c, pa.scalar(-1, I32)), "or_else")
    nn = lambda v: pc.if_else(pc.greater_equal(v, 0), v, pa.scalar(None, I32))
    assert_arrays_match(got[7], nn(a), "non_negative")
    assert_arrays_match(got[8], pc.add(pc.coalesce(nn(a), c, pa.scalar(-1, I32)), nn(c)), "nested")


def _string_roots(b, s):
    fn = b.make_function
    cut = fn("upper", [fn("substr", [s, b.make_literal(1, I64), b.make_literal(8, I64)], S)], S)
    return [(fn("count_byte", [s, b.make_literal(ord("A"), I32)], I32), I32), (fn("fnv1a", [s], I32), I32),
            (fn("fnv1a", [cut], I32), I32), (fn("count_byte", [cut, b.make_literal(ord("A"), I32)], I32), I32)]


def _check_strings(gandiva, reg, batch, name, values):
    b = gandiva.TreeExprBuilder()
    got = _project(gandiva, reg, batch, (b, _string_roots(b, b.make_field(batch.schema.field(name)))))
    want = [[None if v is None else v.encode().count(b"A") for v in values], [None if v is None else _fnv(v) for v in values],
            [None if v is None else _fnv(v[:8], upper=True) for v in values],
            [None if v is None else v[:8].upper().encode().count(b"A") for v in values]]
    for i, w in enumerate(want):
        assert_arrays_match(got[i], pa.array(w, I32), "%s output %d" % (name, i))


def test_string_parameters_over_every_layout(gandiva, reg):
    vals = words(5_003, seed=5)
    vals = [None if v is None else v.encode("ascii", "replace").decode() for v in vals]   # v[:8] is then 8 bytes
    plain = pa.array(vals, S)
    _check_strings(gandiva, reg, pa.RecordBatch.from_arrays([plain], names=["s"]), "s", vals)
    _check_strings(gandiva, reg, pa.RecordBatch.from_arrays([plain.slice(11, 4000)], names=["s"]), "s", vals[11:4011])
    vw, twin = views(vals, seed=6)
    _check_strings(gandiva, reg, pa.RecordBatch.from_arrays([vw], names=["v"]), "v", twin.to_pylist())
    enc = plain.dictionary_encode()
    _check_strings(gandiva, reg, pa.RecordBatch.from_arrays([enc], names=["d"]), "d", vals)


def test_function_over_concat_reads_a_temporary(gandiva, reg):
    vals = words(2_001, seed=9, nulls=0.0)
    batch = pa.RecordBatch.from_arrays([pa.array(vals, S)], names=["s"])
    b = gandiva.TreeExprBuilder()
    s = b.make_field(batch.schema.field("s"))
    root = b.make_function("fnv1a", [b.make_function("concat", [s, b.make_literal("/", S), s], S)], I32)
    got = _project(gandiva, reg, batch, (b, [(root, I32)]))
    assert_arrays_match(got[0], pa.array([_fnv(v + "/" + v) for v in vals], I32), "fnv1a(concat)")


def test_raising_is_lazy_and_only_from_valid_rows(gandiva, reg):
    n = 4_099
    a = np.arange(n, dtype=np.int32) % 11
    b = gandiva.TreeExprBuilder()
    batch = pa.RecordBatch.from_arrays([pa.array(a, I32)], names=["a"])
    fa = b.make_field(batch.schema.field("a"))
    chk = b.make_function("checked", [fa], I32)
    with pytest.raises(gandiva.GandivaError, match="seven is not allowed here") as e:
        _project(gandiva, reg, batch, (b, [(chk, I32)]))
    assert e.value.code == gandiva.GDV_EXECUTION_ERROR
    # the sevens are null: nothing is raised
    masked = pa.RecordBatch.from_arrays([pa.array(a, I32, mask=a == 7)], names=["a"])
    got = _project(gandiva, reg, masked, (b, [(chk, I32)]))
    assert_arrays_match(got[0], pa.array(a + 1, I32, mask=a == 7), "checked over nulls")
    # the untaken branch of an if and the short-circuited side of an and
    ne7 = b.make_function("not_equal", [fa, b.make_literal(7, I32)], B)
    guarded = b.make_if(ne7, chk, b.make_literal(-1, I32), I32)
    both = b.make_and([ne7, b.make_function("greater_than", [chk, b.make_literal(5, I32)], B)])
    got = _project(gandiva, reg, batch, (b, [(guarded, I32), (both, B)]))
    assert_arrays_match(got[0], pa.array(np.where(a != 7, a + 1, -1).astype(np.int32), I32), "if")
    assert_arrays_match(got[1], pa.array((a != 7) & (a + 1 > 5), B), "and")
    f = gandiva.make_filter(batch.schema, b.make_condition(both), gandiva.Configuration(function_registry=reg))
    assert np.array_equal(f.evaluate(batch).to_array().to_numpy(), np.flatnonzero((a != 7) & (a + 1 > 5)))


def _q6_user(b):
    ship, disc, qty = (cases.F(b, n, t) for n, t in (("l_shipdate", D32), ("l_discount", F64), ("l_quantity", F64)))
    fn = b.make_function
    return b.make_and([fn("in_1994", [ship], B), fn("between_f64", [disc, b.make_literal(0.05, F64), b.make_literal(0.07, F64)], B),
                       fn("lt24", [qty], B)])


@pytest.mark.parametrize("n,nulls", [(1, 0), (70_003, 0), (70_003, 30), (LARGE, 10)])
def test_q6_filter_with_user_functions(n, nulls, gandiva, reg, oracle):
    """On the AND spine of a fixed-width Filter: gated and ungated kernels and the built-in condition select the
    same rows, with nullable columns (hoisted validity) and above 32 M rows."""
    batch = cases.q6_batch(n, seed=n % 1000, null_permille=nulls)
    b = gandiva.TreeExprBuilder()
    want = oracle.filter_indices(cases.q6_condition(b), batch, threads=4)
    for gating in (0, 1):
        f = gandiva.make_filter(cases.Q6_SCHEMA, b.make_condition(_q6_user(b)),
                                gandiva.Configuration(function_registry=reg, filter_gating=gating))
        got = f.evaluate(batch).to_array().to_numpy().astype(np.uint64)
        assert np.array_equal(got, want), "gating %d" % gating
        assert f.kernel_info["gated_stages"] == (3 if gating == 0 else 0)


def test_dictionary_first_filter_and_chained_projector(gandiva, reg):
    col = dict_column(20_011, seed=4)
    batch = dict_batch(col)
    name = batch.schema.names[0]
    b = gandiva.TreeExprBuilder()
    d = b.make_field(batch.schema.field(name))
    cond = b.make_function("greater_than", [b.make_function("count_byte", [d, b.make_literal(ord("A"), I32)], I32),
                                            b.make_literal(0, I32)], B)
    cfg = gandiva.Configuration(function_registry=reg)
    f = gandiva.make_filter(batch.schema, b.make_condition(cond), cfg)
    sel = f.evaluate(batch)
    assert f.kernel_info["dictionary_first"] == 1
    vals = batch.column(0).cast(S).to_pylist()
    want = np.array([i for i, v in enumerate(vals) if v is not None and "A" in v], dtype=np.int64)
    assert np.array_equal(sel.to_array().to_numpy().astype(np.int64), want)
    got = _project(gandiva, reg, batch, (b, [(b.make_function("fnv1a", [d], I32), I32)]), selection=sel)
    assert_arrays_match(got[0], pa.array([_fnv(vals[i]) for i in want], I32), "fnv1a over the selection")
