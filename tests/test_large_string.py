"""large_string / large_binary columns and outputs without a GPU: how the types are spelled, what Make()
refuses, and which kernels a Filter or Projector over a large column generates
(tests/test_large_string_gpu.py runs them)."""
import ctypes as C

import pyarrow as pa
import pytest

LS, LB, S = pa.large_string(), pa.large_binary(), pa.string()


def _field(b, schema, name="s"):
    return b.make_field(schema.field(name))


def _lit(b, s):
    return b.make_literal(s, S)


def test_large_types_are_spelled_as_arrow_spells_them(gandiva):
    schema = pa.schema([pa.field("s", LS), pa.field("z", LB)])
    b = gandiva.TreeExprBuilder()
    s = _field(b, schema)
    assert str(s) == "(large_string) s"
    assert s.return_type() == LS
    assert _field(b, schema, "z").return_type() == LB
    for t in (LS, LB):
        c = gandiva._to_c_type(t)
        assert (c.id, c.precision, c.scale) == ({LS: 34, LB: 35}[t], 0, 0)
        assert gandiva._from_c_type(c) == t
    cond = b.make_condition(b.make_function("like", [s, _lit(b, "%x")], pa.bool_()))
    assert "like((large_string) s" in str(cond)


def test_large_result_fields_are_accepted(gandiva):
    """An expression's result field may be large when its root yields utf8 / binary; the write pass then
    stores int64 offsets."""
    schema = pa.schema([pa.field("s", LS), pa.field("u", S)])
    b = gandiva.TreeExprBuilder()
    up = b.make_function("upper", [_field(b, schema, "u")], S)
    p = gandiva.make_projector(schema, [b.make_expression(up, pa.field("o", LS)),
                                        b.make_expression(_field(b, schema), pa.field("i", LS)),
                                        b.make_expression(_field(b, schema), pa.field("n", S))])
    ir = p.llvm_ir
    assert "i64* offs = reinterpret_cast<i64*>(A.out_val[0]);" in ir
    assert "i32* offs = reinterpret_cast<i32*>(A.out_val[0]);" in ir  # the utf8 output keeps int32 offsets


def test_large_node_return_types_are_refused(gandiva):
    schema = pa.schema([pa.field("s", LS)])
    b = gandiva.TreeExprBuilder()
    up = b.make_function("upper", [_field(b, schema)], LS)
    with pytest.raises(pa.ArrowNotImplementedError, match="'upper' has a large_string return type"):
        gandiva.make_projector(schema, [b.make_expression(up, pa.field("o", LS))])
    cond = b.make_function("isnull", [_field(b, schema)], pa.bool_())
    sel = b.make_if(cond, _field(b, schema), _field(b, schema), LS)
    with pytest.raises(pa.ArrowNotImplementedError, match="'if' has a large_string return type"):
        gandiva.make_projector(schema, [b.make_expression(sel, pa.field("o", LS))])
    lit = b.make_literal(b"x", LB)
    with pytest.raises(pa.ArrowNotImplementedError, match="'literal' has a large_binary return type"):
        gandiva.make_projector(schema, [b.make_expression(lit, pa.field("o", LB))])


def test_field_type_must_match_the_schema_layout(gandiva):
    schema = pa.schema([pa.field("s", LS)])
    b = gandiva.TreeExprBuilder()
    plain = b.make_field(pa.field("s", S))
    with pytest.raises(pa.ArrowException, match="large_string different from field"):
        gandiva.make_projector(schema, [b.make_expression(b.make_function("upper", [plain], S), pa.field("o", S))])


def test_row_kernels_read_int64_offsets(gandiva):
    schema = pa.schema([pa.field("s", LS)])
    b = gandiva.TreeExprBuilder()
    n = b.make_function("char_length", [_field(b, schema)], pa.int32())
    p = gandiva.make_projector(schema, [b.make_expression(n, pa.field("n", pa.int32()))])
    ir = p.llvm_ir
    assert "const i64* in_val0 = reinterpret_cast<const i64*>(A.in_val[0]);" in ir
    assert "gdv_large_str(" in ir
    assert p.kernel_info["nullable"] == 1  # a row whose length does not fit a string reads as null


def _filter_ir(gandiva, t, pat, scan):
    schema = pa.schema([pa.field("s", t)])
    b = gandiva.TreeExprBuilder()
    cond = b.make_condition(b.make_function("like", [_field(b, schema), _lit(b, pat)], pa.bool_()))
    return gandiva.make_filter(schema, cond, gandiva.Configuration(string_scan=scan)).llvm_ir


def test_filter_keeps_the_key_driven_kernel(gandiva):
    """A Filter over a large column gets the key-driven kernel, like its utf8 twin; its anchors are
    relative to the warp's run."""
    for t in (S, LS):
        assert "gdv_key_mask" in _filter_ir(gandiva, t, "%special%requests%", 0)
    ir = _filter_ir(gandiva, LS, "%special%requests%", 0)
    assert "const i64* const offs = in_val0;" in ir
    assert "wanch[ix] = (u32)(pos - b0);" in ir
    assert "lost = b1 - b0 > 0xffffffffll" in ir


def test_filter_keeps_the_string_stage_and_the_cooperative_scan(gandiva):
    """string_scan bit 2: the row-driven kernel, with the shared-memory stage and the warp-cooperative LIKE
    scan over a large column as over its utf8 twin; bit 0 takes the per-lane matcher."""
    for t in (S, LS):
        ir = _filter_ir(gandiva, t, "%special%requests%", 4)
        assert "gdv_key_mask" not in ir and "hctr0" in ir and "gdv_cp_async16" in ir
        assert "hctr0" not in _filter_ir(gandiva, t, "%special%requests%", 5)
    ir = _filter_ir(gandiva, LS, "%special%requests%", 4)
    assert "const i64 gn64 = in_val0[" in ir


def test_arrow_c_device_interface_refuses_large_outputs(gandiva):
    schema = pa.schema([pa.field("s", LS)])
    b = gandiva.TreeExprBuilder()
    p = gandiva.make_projector(schema, [b.make_expression(_field(b, schema), pa.field("o", LS))])
    out = gandiva.ArrowSchemaC()
    rc = gandiva.lib.gdv_projector_output_schema_arrow(p._h, C.byref(out))
    assert rc == 10  # GDV_NOT_IMPLEMENTED
    assert b"Arrow C Device interface" in gandiva.lib.gdv_last_error()


def test_user_function_parameters_stay_utf8(gandiva):
    reg = gandiva.FunctionRegistry()
    with pytest.raises(pa.ArrowException):
        reg.register("large_len", [LS], pa.int32(), "return a0.len;")
