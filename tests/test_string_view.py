"""string_view / binary_view input columns without a GPU: how the types are spelled, what Make() and the
Arrow C import refuse, and which call sites the inline / prefix shortcut lowers (tests/test_string_view_gpu.py
runs the columns)."""
import ctypes as C

import pyarrow as pa
import pytest

SV = pa.string_view()


def _field(b, schema, name="s"):
    return b.make_field(schema.field(name))


def _lit(b, s):
    return b.make_literal(s, pa.string())


def test_view_types_are_spelled_as_arrow_spells_them(gandiva):
    schema = pa.schema([pa.field("s", SV), pa.field("z", pa.binary_view())])
    b = gandiva.TreeExprBuilder()
    s = _field(b, schema)
    assert str(s) == "(string_view) s"
    assert s.return_type() == SV
    assert _field(b, schema, "z").return_type() == pa.binary_view()
    for t in (SV, pa.binary_view()):
        assert gandiva._from_c_type(gandiva._to_c_type(t)) == t
    cond = b.make_condition(b.make_function("like", [s, _lit(b, "%x")], pa.bool_()))
    assert "like((string_view) s" in str(cond)


def test_view_outputs_are_refused(gandiva):
    schema = pa.schema([pa.field("s", SV)])
    b = gandiva.TreeExprBuilder()
    with pytest.raises(pa.ArrowNotImplementedError, match="string_view outputs are not supported"):
        gandiva.make_projector(schema, [b.make_expression(_field(b, schema), pa.field("o", SV))])
    up = b.make_function("upper", [_field(b, schema)], SV)
    with pytest.raises(pa.ArrowNotImplementedError, match="string_view outputs are not supported"):
        gandiva.make_projector(schema, [b.make_expression(up, pa.field("o", pa.string()))])
    cond = b.make_function("isnull", [_field(b, schema)], pa.bool_())
    sel = b.make_if(cond, _field(b, schema), _field(b, schema), SV)
    with pytest.raises(pa.ArrowNotImplementedError, match="string_view outputs are not supported"):
        gandiva.make_projector(schema, [b.make_expression(sel, pa.field("o", pa.string()))])


def test_projector_over_a_view_column_builds_the_row_view(gandiva):
    schema = pa.schema([pa.field("s", SV)])
    b = gandiva.TreeExprBuilder()
    # functions resolve against utf8; the identity is a utf8 result
    up = b.make_function("upper", [_field(b, schema)], pa.string())
    p = gandiva.make_projector(schema, [b.make_expression(up, pa.field("u", pa.string())),
                                        b.make_expression(_field(b, schema), pa.field("o", pa.string()))])
    assert "gdv_sv_view" in p.llvm_ir


def test_field_type_must_match_the_schema_layout(gandiva):
    schema = pa.schema([pa.field("s", SV)])
    b = gandiva.TreeExprBuilder()
    plain = b.make_field(pa.field("s", pa.string()))
    with pytest.raises(Exception, match="different from field in expression"):
        gandiva.make_filter(schema, b.make_condition(b.make_function("isnull", [plain], pa.bool_())))


def _shortcuts(gandiva, schema, node, string_scan=0):
    b = gandiva.TreeExprBuilder()
    f = gandiva.make_filter(schema, b.make_condition(node), gandiva.Configuration(string_scan=string_scan))
    return f.kernel_info["view_shortcuts"]


def test_view_shortcuts_count_the_lowered_call_sites(gandiva):
    schema = pa.schema([pa.field("s", SV), pa.field("p", pa.string())])
    b = gandiva.TreeExprBuilder()
    s = _field(b, schema)
    eq = b.make_function("equal", [s, _lit(b, "MAIL")], pa.bool_())
    inl = b.make_in_expression(s, ["MAIL", "SHIP"], pa.string())
    sw = b.make_function("starts_with", [s, _lit(b, "PROMO BRUSHED")], pa.bool_())
    lk = b.make_function("like", [s, _lit(b, "MAIL%")], pa.bool_())
    lk2 = b.make_function("like", [s, _lit(b, "PROMO%BRASS")], pa.bool_())
    ne = b.make_function("not_equal", [_lit(b, "a longer literal"), s], pa.bool_())
    assert _shortcuts(gandiva, schema, eq) == 1
    assert _shortcuts(gandiva, schema, inl) == 1
    assert _shortcuts(gandiva, schema, sw) == 1
    assert _shortcuts(gandiva, schema, lk) == 1
    both = b.make_or([b.make_and([eq, sw]), lk, lk2, ne, inl])
    assert _shortcuts(gandiva, schema, both) == 6
    # off switch: the same filters read the bytes through the view
    for node in (eq, inl, sw, lk, both):
        assert _shortcuts(gandiva, schema, node, string_scan=8) == 0
    # not a bare view column, not a literal prefix, or not a view column at all
    up = b.make_function("equal", [b.make_function("upper", [s], pa.string()), _lit(b, "X")], pa.bool_())
    assert _shortcuts(gandiva, schema, up) == 0
    assert _shortcuts(gandiva, schema, b.make_function("like", [s, _lit(b, "%MAIL")], pa.bool_())) == 0
    plain = b.make_function("equal", [_field(b, schema, "p"), _lit(b, "X")], pa.bool_())
    assert _shortcuts(gandiva, schema, plain) == 0


def test_kernels_without_view_columns_keep_their_layout(gandiva):
    schema = pa.schema([pa.field("p", pa.string())])
    b = gandiva.TreeExprBuilder()
    eq = b.make_function("equal", [_field(b, schema, "p"), _lit(b, "MAIL")], pa.bool_())
    ir = gandiva.make_filter(schema, b.make_condition(eq)).llvm_ir
    assert "in_vbf" not in ir and "gdv_sv_" not in ir.split("extern \"C\"")[-1]


def _export(batch, gandiva):
    arr, sch = gandiva.ArrowDeviceArrayC(), gandiva.ArrowSchemaC()
    batch._export_to_c_device(C.addressof(arr), C.addressof(sch))
    return arr, sch


def test_arrow_schema_import_of_view_fields(gandiva):
    lib = gandiva.lib
    good = pa.schema([pa.field("s", SV), pa.field("z", pa.binary_view())])
    c = gandiva.ArrowSchemaC()
    good._export_to_c(C.addressof(c))
    h = C.c_void_p()
    gandiva._check(lib.gdv_schema_from_arrow(C.addressof(c), C.byref(h)))
    lib.gdv_schema_release(h)
    gandiva._RELEASE_SCHEMA(c.release)(C.byref(c))
    # a dictionary whose values are views: not implemented; the utf8 / binary message is unchanged
    for bad, msg in ((pa.dictionary(pa.int32(), SV), "string_view are not supported"),
                     (pa.dictionary(pa.int32(), pa.int64()), "dictionaries need utf8 or binary values")):
        c = gandiva.ArrowSchemaC()
        pa.schema([pa.field("d", bad)])._export_to_c(C.addressof(c))
        assert lib.gdv_schema_from_arrow(C.addressof(c), C.byref(h)) == gandiva.GDV_NOT_IMPLEMENTED
        assert msg in lib.gdv_last_error().decode()
        gandiva._RELEASE_SCHEMA(c.release)(C.byref(c))


def test_arrow_import_rejects_a_malformed_view_child(gandiva):
    col = pa.array(["short", "a string longer than twelve bytes", None]).cast(SV)
    batch = pa.RecordBatch.from_arrays([col], names=["s"])
    arr, sch = _export(batch, gandiva)
    gandiva._RELEASE_SCHEMA(sch.release)(C.byref(sch))
    child = arr.array.children[0].contents
    saved = child.n_buffers
    assert saved == 4   # validity, views, one data buffer, the sizes
    child.n_buffers = 2
    with pytest.raises(pa.ArrowInvalid, match="malformed string_view"):
        gandiva.ArrowDeviceBatch(C.addressof(arr), batch.schema)
    child.n_buffers = saved
    assert arr.array.release   # not moved: still the producer's
    # the schema says plain utf8 but the array is a view array
    with pytest.raises(pa.ArrowInvalid, match="expected 3 buffers, got 4"):
        gandiva.ArrowDeviceBatch(C.addressof(arr), pa.schema([pa.field("s", pa.string())]))
    imported = gandiva.ArrowDeviceBatch(C.addressof(arr), batch.schema)
    assert imported.num_rows == 3
    imported.release()
