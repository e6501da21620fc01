"""Where the fixed-width Filter gates its loads (kernel attribute `gated_stages`), checked without a GPU:
the kernel is generated and compiled with NVRTC at Make().  Conditions that gating does not apply to keep
exactly the kernel they had before it existed: the source with Configuration.filter_gating = 0 equals
the source with it off."""
import pyarrow as pa
import pytest

import cases

B, I32 = pa.bool_(), pa.int32()


def _filters(gandiva, schema, cond):
    b = cond[0]
    return [gandiva.make_filter(schema, b.make_condition(cond[1]), gandiva.Configuration(filter_gating=g)) for g in (0, 1)]


def _lt(b, x, v, t=I32):
    return b.make_function("less_than", [x, b.make_literal(v, t)], B)


def test_q6_has_three_stages(gandiva):
    b = gandiva.TreeExprBuilder()
    on, off = _filters(gandiva, cases.Q6_SCHEMA, (b, cases.q6_condition(b)))
    assert on.kernel_info["gated_stages"] == 3 and off.kernel_info["gated_stages"] == 0
    assert on.llvm_ir != off.llvm_ir


def _single_column(b):
    a = cases.F(b, "a", I32)
    return pa.schema([("a", I32), ("c", I32)]), b.make_and([_lt(b, a, 5), b.make_function("greater_than", [a, b.make_literal(-5, I32)], B)])


def _top_level_or(b):
    a, c = cases.F(b, "a", I32), cases.F(b, "c", I32)
    return pa.schema([("a", I32), ("c", I32)]), b.make_or([_lt(b, a, 5), _lt(b, c, 5)])


def _can_raise(b):
    a, c = cases.F(b, "a", I32), cases.F(b, "c", I32)
    return pa.schema([("a", I32), ("c", I32)]), b.make_and([_lt(b, a, 5), _lt(b, b.make_function("divide", [a, c], I32), 2)])


def _string(b):
    s, a = cases.F(b, "s", pa.string()), cases.F(b, "a", I32)
    return pa.schema([("a", I32), ("s", pa.string())]), b.make_and(
        [_lt(b, a, 5), b.make_function("equal", [s, b.make_literal("ab", pa.string())], B)])


def _dictionary(b):
    DT = pa.dictionary(pa.int32(), pa.string())
    d, a = cases.F(b, "d", DT), cases.F(b, "a", I32)
    return pa.schema([("a", I32), ("d", DT)]), b.make_and(
        [_lt(b, a, 5), b.make_function("equal", [d, b.make_literal("ab", pa.string())], B)])


def _view(b):
    v, a = cases.F(b, "v", pa.string_view()), cases.F(b, "a", I32)
    return pa.schema([("a", I32), ("v", pa.string_view())]), b.make_and(
        [_lt(b, a, 5), b.make_function("equal", [v, b.make_literal("ab", pa.string())], B)])


def _dense_first_stage(b):
    """Stage 0 would read 16 of the row's 20 bytes: too little is left to gate."""
    d, q, t = cases.F(b, "l_discount", pa.float64()), cases.F(b, "l_quantity", pa.float64()), cases.F(b, "l_shipdate", pa.date32())
    scaled = b.make_function("multiply", [d, b.make_literal(100.0, pa.float64())], pa.float64())
    return cases.Q6_SCHEMA, b.make_and([b.make_function("less_than", [scaled, q], B), _lt(b, t, 9131, pa.date32())])


@pytest.mark.parametrize("make", [_single_column, _top_level_or, _can_raise, _string, _dictionary, _view, _dense_first_stage],
                         ids=lambda f: f.__name__.strip("_"))
def test_not_gated(make, gandiva):
    b = gandiva.TreeExprBuilder()
    schema, cond = make(b)
    on, off = _filters(gandiva, schema, (b, cond))
    assert on.kernel_info["gated_stages"] == 0
    assert on.llvm_ir == off.llvm_ir


@pytest.mark.parametrize("case", cases.all_filter_cases(), ids=[c.__name__ for c in cases.all_filter_cases()])
def test_ungated_source_unchanged(case, gandiva):
    b = gandiva.TreeExprBuilder()
    schema, outs, _ = case(b)
    on, off = _filters(gandiva, schema, (b, outs[0][0]))
    if on.kernel_info["gated_stages"] == 0:
        assert on.llvm_ir == off.llvm_ir
    else:
        assert on.llvm_ir != off.llvm_ir and off.kernel_info["gated_stages"] == 0
