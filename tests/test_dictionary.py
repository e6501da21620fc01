"""Dictionary-encoded input columns without a GPU: what Make() and the Arrow C import refuse, and how the
type is spelled (tests/test_dictionary_gpu.py runs the columns)."""
import ctypes as C

import pyarrow as pa
import pytest

DT = pa.dictionary(pa.int32(), pa.string())


def _field(b, schema, name="d"):
    return b.make_field(schema.field(name))


@pytest.mark.parametrize("bad", [pa.dictionary(pa.uint8(), pa.string()), pa.dictionary(pa.uint32(), pa.binary()),
                                 pa.dictionary(pa.int8(), pa.int32()), pa.dictionary(pa.int16(), pa.float64()),
                                 pa.dictionary(pa.int32(), pa.large_string())], ids=str)
def test_unsupported_dictionary_types_are_refused_at_make(bad, gandiva):
    schema = pa.schema([pa.field("d", bad)])
    b = gandiva.TreeExprBuilder()
    cond = b.make_condition(b.make_function("isnull", [_field(b, schema)], pa.bool_()))
    with pytest.raises(pa.ArrowNotImplementedError, match="dictionary columns need utf8 or binary values"):
        gandiva.make_filter(schema, cond)


def test_dictionary_outputs_are_refused(gandiva):
    schema = pa.schema([pa.field("d", DT)])
    b = gandiva.TreeExprBuilder()
    with pytest.raises(pa.ArrowNotImplementedError, match="dictionary-encoded outputs are not supported"):
        gandiva.make_projector(schema, [b.make_expression(_field(b, schema), pa.field("o", DT))])
    # a plain utf8 result of the same column is fine, and functions resolve against the value type
    up = b.make_function("upper", [_field(b, schema)], pa.string())
    p = gandiva.make_projector(schema, [b.make_expression(up, pa.field("u", pa.string())),
                                        b.make_expression(_field(b, schema), pa.field("o", pa.string()))])
    assert "gdv_dict_view" in p.llvm_ir


def test_field_type_must_match_the_schema_encoding(gandiva):
    schema = pa.schema([pa.field("d", DT)])
    b = gandiva.TreeExprBuilder()
    plain = b.make_field(pa.field("d", pa.string()))
    with pytest.raises(Exception, match="different from field in expression"):
        gandiva.make_filter(schema, b.make_condition(b.make_function("isnull", [plain], pa.bool_())))


def test_to_string_spells_the_dictionary_type(gandiva):
    schema = pa.schema([pa.field("d", DT), pa.field("o", pa.dictionary(pa.int8(), pa.binary(), ordered=True))])
    b = gandiva.TreeExprBuilder()
    d = _field(b, schema)
    assert str(d) == "(dictionary<values=string, indices=int32, ordered=0>) d"
    assert d.return_type() == DT
    assert _field(b, schema, "o").return_type() == pa.dictionary(pa.int8(), pa.binary(), ordered=True)
    cond = b.make_condition(b.make_function("like", [d, b.make_literal("%x", pa.string())], pa.bool_()))
    assert "like((dictionary<values=string, indices=int32, ordered=0>) d" in str(cond)


def _export(batch, gandiva):
    arr, sch = gandiva.ArrowDeviceArrayC(), gandiva.ArrowSchemaC()
    batch._export_to_c_device(C.addressof(arr), C.addressof(sch))
    return arr, sch


def test_arrow_schema_import_of_dictionary_fields(gandiva):
    lib = gandiva.lib
    good = pa.schema([pa.field("d", DT), pa.field("z", pa.dictionary(pa.int64(), pa.binary()))])
    c = gandiva.ArrowSchemaC()
    good._export_to_c(C.addressof(c))
    h = C.c_void_p()
    gandiva._check(lib.gdv_schema_from_arrow(C.addressof(c), C.byref(h)))
    lib.gdv_schema_release(h)
    gandiva._RELEASE_SCHEMA(c.release)(C.byref(c))
    for bad in (pa.dictionary(pa.uint16(), pa.string()), pa.dictionary(pa.int32(), pa.int64())):
        c = gandiva.ArrowSchemaC()
        pa.schema([pa.field("d", bad)])._export_to_c(C.addressof(c))
        assert lib.gdv_schema_from_arrow(C.addressof(c), C.byref(h)) == gandiva.GDV_NOT_IMPLEMENTED
        gandiva._RELEASE_SCHEMA(c.release)(C.byref(c))


def test_arrow_import_rejects_a_malformed_dictionary_child(gandiva):
    col = pa.DictionaryArray.from_arrays(pa.array([0, 1, None, 0], pa.int32()), pa.array(["a", "b"]))
    batch = pa.RecordBatch.from_arrays([col], names=["d"])
    arr, sch = _export(batch, gandiva)
    gandiva._RELEASE_SCHEMA(sch.release)(C.byref(sch))
    child = arr.array.children[0].contents
    dictionary = child.dictionary.contents
    saved = dictionary.n_buffers
    dictionary.n_buffers = 2   # a utf8 dictionary needs validity, offsets and data
    with pytest.raises(pa.ArrowInvalid, match="malformed dictionary"):
        gandiva.ArrowDeviceBatch(C.addressof(arr), batch.schema)
    dictionary.n_buffers = saved
    assert arr.array.release   # not moved: still the producer's
    # the schema says plain utf8 but the array is dictionary-encoded (and the other way round)
    with pytest.raises(pa.ArrowNotImplementedError, match="dictionary-encoded"):
        gandiva.ArrowDeviceBatch(C.addressof(arr), pa.schema([pa.field("d", pa.string())]))
    imported = gandiva.ArrowDeviceBatch(C.addressof(arr), batch.schema)
    assert imported.num_rows == 4
    imported.release()
    plain = pa.RecordBatch.from_arrays([pa.array(["a", "b"])], names=["d"])
    arr, sch = _export(plain, gandiva)
    gandiva._RELEASE_SCHEMA(sch.release)(C.byref(sch))
    with pytest.raises(pa.ArrowInvalid, match="is not dictionary-encoded"):
        gandiva.ArrowDeviceBatch(C.addressof(arr), batch.schema)
    gandiva._RELEASE_ARRAY(arr.array.release)(C.byref(arr.array))
