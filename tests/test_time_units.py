"""timestamp[s|ms|us|ns], time32[s|ms] and time64[us|ns] without a GPU: how the types are spelled, what Make()
accepts and refuses, which device function each unit resolves to, that every division by a unit reaches
PTX as a division by a constant, and that the function listing keeps its millisecond entries first
(tests/test_time_units_gpu.py runs the kernels)."""
import os
import re

import pyarrow as pa
import pytest

UNITS = ["s", "ms", "us", "ns"]
TS = {u: pa.timestamp(u) for u in UNITS}
TT = {"s": pa.time32("s"), "ms": pa.time32("ms"), "us": pa.time64("us"), "ns": pa.time64("ns")}
ALL = list(TS.values()) + list(TT.values())
MS_TEMPORAL = {pa.timestamp("ms"), pa.time32("ms")}
NON_MS = {t for t in ALL if t not in MS_TEMPORAL}
PARENT_SIGNATURES = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "signatures_818.txt")


def _project(gandiva, schema, node, rt, **cfg):
    b = gandiva.TreeExprBuilder()
    conf = gandiva.Configuration(**cfg) if cfg else None
    return gandiva.make_projector(schema, [b.make_expression(node, pa.field("o", rt))], None, configuration=conf)


def _fn(gandiva, name, t, rt, extra=()):
    """A projector name(column of type t, *extra literals) -> rt."""
    b = gandiva.TreeExprBuilder()
    f = pa.field("c", t)
    node = b.make_function(name, [b.make_field(f)] + [b.make_literal(v, vt) for v, vt in extra], rt)
    return _project(gandiva, pa.schema([f]), node, rt)


@pytest.mark.parametrize("t", ALL, ids=str)
def test_types_round_trip(gandiva, t):
    c = gandiva._to_c_type(t)
    assert gandiva._from_c_type(c) == t
    b = gandiva.TreeExprBuilder()
    f = b.make_field(pa.field("c", t))
    assert str(f) == "(%s) c" % t
    assert f.return_type() == t


@pytest.mark.parametrize("t", ALL, ids=str)
def test_fields_literals_and_in_lists_are_accepted(gandiva, t):
    b = gandiva.TreeExprBuilder()
    f = pa.field("c", t)
    schema = pa.schema([f])
    lit = b.make_literal(12345, t)
    assert lit.return_type() == t
    cmp = b.make_function("less_than", [b.make_field(f), lit], pa.bool_())
    ir = gandiva.make_filter(schema, b.make_condition(cmp)).llvm_ir
    assert "gdv_filter_expr_" in ir
    inn = b.make_in_expression(b.make_field(f), [1, 2, -3], t)
    gandiva.make_filter(schema, b.make_condition(inn))
    # identity projection, if/else and nvl keep the type
    cond = b.make_function("isnotnull", [b.make_field(f)], pa.bool_())
    iff = b.make_if(cond, b.make_field(f), b.make_literal(7, t), t)
    nvl = b.make_function("nvl", [b.make_field(f), b.make_literal(7, t)], t)
    p = gandiva.make_projector(schema, [b.make_expression(b.make_field(f), pa.field("a", t)),
                                        b.make_expression(iff, pa.field("b", t)),
                                        b.make_expression(nvl, pa.field("c2", t))], None)
    assert "gdv_project_expr_" in p.llvm_ir


def test_time_zone_columns_read_as_utc_instants(gandiva):
    t = pa.timestamp("us", tz="UTC")
    b = gandiva.TreeExprBuilder()
    f = pa.field("c", t)
    node = b.make_function("extractYear", [b.make_field(f)], pa.int64())
    p = _project(gandiva, pa.schema([f]), node, pa.int64())
    assert "extractYear_timestamp_us(" in p.llvm_ir


def test_mixed_units_are_refused(gandiva):
    b = gandiva.TreeExprBuilder()
    a, c = pa.field("a", TS["us"]), pa.field("c", TS["ms"])
    node = b.make_function("less_than", [b.make_field(a), b.make_field(c)], pa.bool_())
    with pytest.raises(gandiva.GandivaError, match="not supported yet"):
        gandiva.make_filter(pa.schema([a, c]), b.make_condition(node))
    inn = b.make_in_expression(b.make_field(a), [1], TS["ms"])
    with pytest.raises(gandiva.GandivaError):
        gandiva.make_filter(pa.schema([a, c]), b.make_condition(inn))


@pytest.mark.parametrize("name", ["date_trunc_Day", "timestampaddDay", "add_months", "castTIME"])
def test_unit_preserving_functions_refuse_another_declared_unit(gandiva, name):
    extra = [] if name in ("date_trunc_Day", "castTIME") else [(1, pa.int32())]
    wrong = pa.time64("ns") if name == "castTIME" else TS["ns"]
    with pytest.raises(gandiva.GandivaError, match="does not match"):
        _fn(gandiva, name, TS["us"], wrong, extra)
    right = pa.time64("us") if name == "castTIME" else TS["us"]
    assert "%s_timestamp_us" % name in _fn(gandiva, name, TS["us"], right, extra).llvm_ir


@pytest.mark.parametrize("u", UNITS)
def test_constructors_take_the_declared_unit(gandiva, u):
    suffix = "" if u == "ms" else "_" + u
    assert ("castTIMESTAMP%s_int64(" % suffix) in _fn(gandiva, "castTIMESTAMP", pa.int64(), TS[u]).llvm_ir
    assert ("castTIMESTAMP%s_date64(" % suffix) in _fn(gandiva, "castTIMESTAMP", pa.date64(), TS[u]).llvm_ir
    assert ("castTIMESTAMP%s_utf8(" % suffix) in _fn(gandiva, "castTIMESTAMP", pa.string(), TS[u]).llvm_ir
    assert ("to_timestamp%s_float64(" % suffix) in _fn(gandiva, "to_timestamp", pa.float64(), TS[u]).llvm_ir
    assert ("to_time%s_int32(" % suffix) in _fn(gandiva, "to_time", pa.int32(), TT[u]).llvm_ir
    for v in UNITS:
        if v != u:
            ir = _fn(gandiva, "castTIMESTAMP", TS[v], TS[u]).llvm_ir
            assert "castTIMESTAMP_%s_%s(" % (u, "timestamp" if v == "ms" else "timestamp_" + v) in ir
    # castTIMESTAMP(timestamp[ms]) -> timestamp[ms] is no signature (a no-op, and only old types)
    if u == "ms":
        with pytest.raises(gandiva.GandivaError):
            _fn(gandiva, "castTIMESTAMP", TS["ms"], TS["ms"])


def test_user_functions_stay_millisecond_only(gandiva):
    reg = gandiva.FunctionRegistry()
    with pytest.raises(pa.ArrowInvalid, match="unsupported parameter type"):
        reg.register("f_us", [TS["us"]], pa.int64(), "return 0;")


def _div64(ir):
    return len(re.findall(r"\b(?:div|rem)\.[su]64\b", ir))


@pytest.mark.parametrize("name", ["extractYear", "date_trunc_Day"])
def test_divisions_by_a_unit_are_by_constants(gandiva, name):
    def ptx(u):
        rt = pa.int64() if name.startswith("extract") else TS[u]
        b = gandiva.TreeExprBuilder()
        f = pa.field("c", TS[u])
        node = b.make_function(name, [b.make_field(f)], rt)
        return _project(gandiva, pa.schema([f]), node, rt, dump_ir=True).llvm_ir
    ms = _div64(ptx("ms"))
    for u in ("us", "ns"):
        assert _div64(ptx(u)) <= ms, u
    # the count finds a division by a run-time value
    b = gandiva.TreeExprBuilder()
    x, y = pa.field("x", pa.int64()), pa.field("y", pa.int64())
    node = b.make_function("divide", [b.make_field(x), b.make_field(y)], pa.int64())
    assert _div64(_project(gandiva, pa.schema([x, y]), node, pa.int64(), dump_ir=True).llvm_ir) > 0


def test_signature_listing_keeps_the_millisecond_entries_first(gandiva):
    with open(PARENT_SIGNATURES) as f:
        parent = f.read().splitlines()
    assert len(parent) == 818
    sigs = gandiva.get_registered_function_signatures()
    assert [str(s) for s in sigs[:len(parent)]] == parent
    new = sigs[len(parent):]
    assert new
    for s in new:
        assert any(t in NON_MS for t in s.param_types() + [s.return_type()]), str(s)
    names = {s.name() for s in new}
    for n in ("extractYear", "date_trunc_Day", "castTIMESTAMP", "castVARCHAR", "months_between", "castTIME",
              "to_timestamp", "to_time", "hash64", "nvl", "is_distinct_from"):
        assert n in names
