"""User-defined functions (DESIGN.md §3.8), the part that needs no GPU: registration and its errors, what the
fuser writes into a kernel, which cubins are shared, and that a registry changes nothing for trees that call
no user function.  tests/test_udf_gpu.py runs the functions."""
import os
import re
import shutil
import subprocess

import pyarrow as pa
import pytest

import cases

B, I32, I64, F64, S = pa.bool_(), pa.int32(), pa.int64(), pa.float64(), pa.string()


def _populated(gandiva):
    reg = gandiva.FunctionRegistry()
    reg.register("lt24", [F64], B, "return a0 < 24.0;")
    reg.register("count_byte", [S, I32], I32,
                 "i32 n = 0;\nfor (i32 i = 0; i < a0.len; ++i) n += gdv_ch(a0, i) == (u8)a1;\nreturn n;")
    reg.register("checked_inc", [I32], I32, 'if (a0 == 7) gdv_raise(ctx, "seven");\nreturn a0 + 1;', can_raise=True)
    return reg


def test_register_and_enumerate(gandiva):
    before = [str(s) for s in gandiva.get_registered_function_signatures()]
    reg = _populated(gandiva)
    assert [str(s) for s in reg.signatures()] == ["bool lt24(double)", "int32 count_byte(string, int32)",
                                                  "int32 checked_inc(int32)"]
    assert [str(s) for s in gandiva.get_registered_function_signatures()] == before
    assert gandiva.FunctionRegistry().signatures() == []


def test_registration_errors(gandiva):
    reg = gandiva.FunctionRegistry()
    reg.register("twice", [I32], I32, "return 2 * a0;")
    with pytest.raises(pa.ArrowInvalid, match="already registered"):
        reg.register("twice", [I32], I32, "return a0 + a0;")
    reg.register("twice", [I64], I64, "return 2 * a0;")   # another parameter list is another function
    with pytest.raises(pa.ArrowInvalid, match="built-in"):
        reg.register("add", [I32, I32], I32, "return a0 + a1;")
    with pytest.raises(pa.ArrowInvalid, match="built-in"):   # the fuser knows built-ins by name: no overloads
        reg.register("nvl", [S, I32], I32, "return a1;")
    with pytest.raises(pa.ArrowInvalid, match="identifier"):
        reg.register("not an identifier", [I32], I32, "return a0;")
    with pytest.raises(pa.ArrowInvalid, match="unsupported parameter type"):
        reg.register("f", [pa.list_(I32)], I32, "return 0;")
    with pytest.raises(pa.ArrowInvalid, match="unsupported parameter type"):
        reg.register("f", [pa.timestamp("ns")], I64, "return a0;")
    with pytest.raises(pa.ArrowNotImplementedError, match="decimal128 parameters"):
        reg.register("f", [pa.decimal128(12, 2)], I32, "return 0;")
    for t in (S, pa.binary(), pa.decimal128(12, 2)):
        with pytest.raises(pa.ArrowNotImplementedError, match="return types are not supported"):
            reg.register("f", [I32], t, "return 0;")
    with pytest.raises(ValueError, match="null_mode"):
        reg.register("f", [I32], I32, "return 0;", null_mode="sometimes")
    assert len(reg.signatures()) == 2


def test_body_that_does_not_compile_is_refused_at_registration(gandiva):
    reg = gandiva.FunctionRegistry()
    with pytest.raises(gandiva.GandivaError) as e:
        reg.register("broken", [I32], I32, "return a0 +;")
    assert e.value.code == gandiva.GDV_CODEGEN_ERROR
    assert "int32 broken(int32)" in str(e.value) and "return a0 +;" in str(e.value) and "error" in str(e.value)
    with pytest.raises(gandiva.GandivaError, match="gdv_raise"):   # ctx only exists with can_raise
        reg.register("raises", [I32], I32, 'gdv_raise(ctx, "no"); return a0;')
    assert reg.signatures() == []


def test_unknown_function_message_is_unchanged(gandiva):
    b = gandiva.TreeExprBuilder()
    schema = pa.schema([("a", I32)])
    e = b.make_expression(b.make_function("lt24", [cases.F(b, "a", I32)], B), pa.field("r", B))
    msgs = []
    for cfg in (None, gandiva.Configuration(function_registry=_populated(gandiva))):   # lt24(double) only
        with pytest.raises(gandiva.GandivaError) as err:
            gandiva.make_projector(schema, [e], None, "NONE", cfg)
        msgs.append(str(err.value))
    assert msgs[0] == msgs[1] and "Function bool lt24(int32) not supported yet" in msgs[0]


def test_registry_is_read_only_once_used(gandiva):
    reg = _populated(gandiva)
    b = gandiva.TreeExprBuilder()
    schema, outs, _ = cases.case_q6_filter(b)
    gandiva.make_filter(schema, b.make_condition(outs[0][0]), gandiva.Configuration(function_registry=reg))
    with pytest.raises(pa.ArrowInvalid, match="already in use"):
        reg.register("late", [I32], I32, "return a0;")


def _source(gandiva, case, cfg):
    b = gandiva.TreeExprBuilder()
    schema, outs, kind = case(b)
    if kind == "project":
        exprs = [b.make_expression(r, pa.field("o%d" % i, t)) for i, (r, t) in enumerate(outs)]
        return gandiva.make_projector(schema, exprs, None, "NONE", cfg).llvm_ir
    return gandiva.make_filter(schema, b.make_condition(outs[0][0]), cfg).llvm_ir


ALL_CASES = cases.all_project_cases() + cases.all_filter_cases()


def test_trees_without_user_functions_generate_the_same_source(gandiva):
    """Every expression of tests/cases.py: byte-identical kernels with no registry, an empty one and a
    populated one (and therefore the same cubin-cache entries)."""
    empty = gandiva.Configuration(function_registry=gandiva.FunctionRegistry())
    full = gandiva.Configuration(function_registry=_populated(gandiva))
    for case in ALL_CASES:
        plain = _source(gandiva, case, None)
        assert _source(gandiva, case, empty) == plain, case.__name__
        assert _source(gandiva, case, full) == plain, case.__name__


def _f_of_double(gandiva, body):
    reg = gandiva.FunctionRegistry()
    reg.register("f", [F64], F64, body)
    b = gandiva.TreeExprBuilder()
    e = b.make_expression(b.make_function("f", [cases.F(b, "x", F64)], F64), pa.field("r", F64))
    return gandiva.make_projector(pa.schema([("x", F64)]), [e], None, "NONE", gandiva.Configuration(function_registry=reg))


def test_source_shows_the_function_and_cubins_are_keyed_on_it(gandiva, monkeypatch):
    monkeypatch.delenv("GDV_CUBIN_CACHE_DIR", raising=False)
    body = "return a0 * 1.8 + 32.0;  /* %d */" % os.getpid()
    c0 = gandiva.compile_count()
    one = _f_of_double(gandiva, body)
    assert gandiva.compile_count() == c0 + 1
    ir = one.llvm_ir
    symbol = re.search(r"gdv_udf_[0-9a-f]{16}", ir).group(0)
    assert body in ir and "// user function: double f(double) [if_null]" in ir
    assert ir.count("__forceinline__ f64 " + symbol) == 1 and ir.index(symbol) > ir.index('#include "gdv_device_lib.cuh"')
    again = _f_of_double(gandiva, body)   # another registry object, the same definition: the same kernel
    assert gandiva.compile_count() == c0 + 1 and again.llvm_ir == ir
    other = _f_of_double(gandiva, body.replace("1.8", "1.75"))
    assert gandiva.compile_count() == c0 + 2
    assert symbol not in other.llvm_ir and other.kernel_info["name"] != one.kernel_info["name"]


def test_prelude_and_helper_are_written_once(gandiva):
    reg = gandiva.FunctionRegistry()
    prelude = "__device__ const i32 udf_weights[4] = {1, 3, 7, 9};"
    reg.register("w", [I32], I32, "return udf_weights[a0 & 3];", prelude=prelude)
    reg.register("w2", [I32], I32, 'if (a0 < 0) gdv_raise(ctx, "negative");\nreturn 2 * udf_weights[a0 & 3];',
                 prelude=prelude, can_raise=True)
    reg.register("unused", [I32], I32, "return -a0;")
    b = gandiva.TreeExprBuilder()
    a = cases.F(b, "a", I32)
    w = lambda name, x: b.make_function(name, [x], I32)
    exprs = [b.make_expression(b.make_function("add", [w("w", a), w("w2", w("w", a))], I32), pa.field("r", I32)),
             b.make_expression(w("w2", a), pa.field("r2", I32))]
    ir = gandiva.make_projector(pa.schema([("a", I32)]), exprs, None, "NONE", gandiva.Configuration(function_registry=reg)).llvm_ir
    assert ir.count(prelude) == 1 and ir.count("void gdv_raise(") == 1
    assert ir.count("// user function: int32 w(int32)") == 1 and ir.count("// user function: int32 w2(int32)") == 1
    assert "unused" not in ir


def _q6_with_lt24(b, raising=False):
    sd, f = pa.date32(), F64
    ship, disc, qty = cases.F(b, "l_shipdate", sd), cases.F(b, "l_discount", f), cases.F(b, "l_quantity", f)
    fn = b.make_function
    return b.make_and([fn("greater_than_or_equal_to", [ship, b.make_literal(8766, sd)], B),
                       fn("less_than", [ship, b.make_literal(9131, sd)], B),
                       fn("greater_than_or_equal_to", [disc, b.make_literal(0.05, f)], B),
                       fn("less_than_or_equal_to", [disc, b.make_literal(0.07, f)], B),
                       fn("lt24_raising" if raising else "lt24", [qty], B)])


def _resources(gandiva, monkeypatch, tmp_path, make):
    """(registers, stack bytes) of the Filter's kernel, read from the cubin NVRTC produced."""
    tmp_path.mkdir()
    monkeypatch.setenv("GDV_DUMP_DIR", str(tmp_path))
    monkeypatch.delenv("GDV_CUBIN_CACHE_DIR", raising=False)
    f = make()
    out = subprocess.run([CUOBJDUMP, "-res-usage", str(tmp_path / (f.kernel_info["name"] + ".cubin"))],
                         capture_output=True, text=True, check=True).stdout
    m = re.search(r"REG:(\d+) STACK:(\d+)", out[out.index(f.kernel_info["name"]):])
    return f, int(m.group(1)), int(m.group(2))


CUOBJDUMP = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"


@pytest.mark.skipif(not os.path.exists(CUOBJDUMP), reason="cuobjdump not installed")
def test_q6_with_a_user_function_keeps_its_kernel_shape(gandiva, monkeypatch, tmp_path):
    """`l_quantity < 24` as lt24(double): still three gated stages, and after inlining the registers and
    the (empty) stack of the built-in kernel."""
    reg = gandiva.FunctionRegistry()
    reg.register("lt24", [F64], B, "return a0 < 24.0;")
    reg.register("lt24_raising", [F64], B, 'if (a0 < 0.0) gdv_raise(ctx, "negative quantity");\nreturn a0 < 24.0;', can_raise=True)
    cfg = gandiva.Configuration(function_registry=reg)
    b = gandiva.TreeExprBuilder()
    builtin, regs0, stack0 = _resources(gandiva, monkeypatch, tmp_path / "a", lambda: gandiva.make_filter(
        cases.Q6_SCHEMA, b.make_condition(cases.q6_condition(b)), cfg))
    user, regs1, stack1 = _resources(gandiva, monkeypatch, tmp_path / "b", lambda: gandiva.make_filter(
        cases.Q6_SCHEMA, b.make_condition(_q6_with_lt24(b)), cfg))
    assert builtin.kernel_info["gated_stages"] == 3 and user.kernel_info["gated_stages"] == 3
    assert "gdv_udf_" in user.llvm_ir and "gdv_udf_" not in builtin.llvm_ir
    assert (regs1, stack1) == (regs0, stack0) and stack0 == 0
    # a function that can raise must see exactly the rows a row-at-a-time evaluation would: no gating
    raising = gandiva.make_filter(cases.Q6_SCHEMA, b.make_condition(_q6_with_lt24(b, raising=True)), cfg)
    assert raising.kernel_info["gated_stages"] == 0


def test_loaders_still_apply(gandiva):
    """A user function is function code, not a loader: the Q1-width projector keeps the TMA loader."""
    reg = _populated(gandiva)
    cfg = gandiva.Configuration(function_registry=reg)
    b = gandiva.TreeExprBuilder()
    schema, outs, _ = cases.case_q1_projector(b)
    qty = cases.F(b, "l_discount_f", F64)
    exprs = [b.make_expression(r, pa.field("o%d" % i, t)) for i, (r, t) in enumerate(outs)]
    plain = gandiva.make_projector(schema, exprs, None)
    exprs.append(b.make_expression(b.make_function("lt24", [qty], B), pa.field("cheap", B)))
    with_udf = gandiva.make_projector(schema, exprs, None, "NONE", cfg)
    assert plain.kernel_info["staged"] == 1 and with_udf.kernel_info["staged"] == 1
    assert "gdv_udf_" in with_udf.llvm_ir
