"""Host-side behaviour of the mirrored interface (no GPU needed): builder, validation errors,
registry, and that every catalogue expression lowers to CUDA and compiles with NVRTC for
sm_90a at Make() time.  Mirrors site-packages/pyarrow/tests/test_gandiva.py:255-434."""
import pyarrow as pa
import pytest

import cases


def test_literals(gandiva):
    builder = gandiva.TreeExprBuilder()
    builder.make_literal(True, pa.bool_())
    builder.make_literal(0, pa.uint8())
    builder.make_literal(1, pa.uint16())
    builder.make_literal(2, pa.uint32())
    builder.make_literal(3, pa.uint64())
    builder.make_literal(4, pa.int8())
    builder.make_literal(5, pa.int16())
    builder.make_literal(6, pa.int32())
    builder.make_literal(7, pa.int64())
    builder.make_literal(8.0, pa.float32())
    builder.make_literal(9.0, pa.float64())
    builder.make_literal("hello", pa.string())
    builder.make_literal(b"world", pa.binary())
    builder.make_literal(True, "bool")
    builder.make_literal(0, "uint8")
    builder.make_literal(7, "int64")
    builder.make_literal(8.0, "float32")
    builder.make_literal("hello", "string")
    builder.make_literal(b"world", "binary")
    with pytest.raises(TypeError):
        builder.make_literal("hello", pa.int64())
    with pytest.raises(TypeError):
        builder.make_literal(True, None)


def test_rejects_none(gandiva):
    builder = gandiva.TreeExprBuilder()
    field_x = pa.field('x', pa.int32())
    schema = pa.schema([field_x])
    literal_true = builder.make_literal(True, pa.bool_())
    with pytest.raises(TypeError):
        builder.make_field(None)
    with pytest.raises(TypeError):
        builder.make_if(literal_true, None, None, None)
    with pytest.raises(TypeError):
        builder.make_and([literal_true, None])
    with pytest.raises(TypeError):
        builder.make_or([None, literal_true])
    with pytest.raises(TypeError):
        builder.make_in_expression(None, [1, 2, 3], pa.int32())
    with pytest.raises(TypeError):
        builder.make_expression(None, field_x)
    with pytest.raises(TypeError):
        builder.make_condition(None)
    with pytest.raises(TypeError):
        builder.make_function('less_than', [literal_true, None], pa.bool_())
    with pytest.raises(TypeError):
        gandiva.make_projector(schema, [None])
    with pytest.raises(TypeError):
        gandiva.make_filter(schema, None)


def test_get_registered_function_signatures(gandiva):
    signatures = gandiva.get_registered_function_signatures()
    assert isinstance(signatures[0].return_type(), pa.DataType)
    assert type(signatures[0].param_types()) is list
    assert hasattr(signatures[0], "name")
    names = {s.name() for s in signatures}
    for n in ["add", "subtract", "multiply", "divide", "less_than", "greater_than", "like", "not",
              "substr", "upper", "isnull", "castBIGINT", "extractYear"]:
        assert n in names


def test_return_type_and_condition(gandiva):
    b = gandiva.TreeExprBuilder()
    fa = pa.field('a', pa.int32())
    na = b.make_field(fa)
    assert na.return_type() == fa.type
    cond = b.make_condition(b.make_function("greater_than", [na, na], pa.bool_()))
    assert cond.result().type == pa.bool_()
    expr = b.make_expression(na, pa.field('r', pa.int32()))
    assert expr.result().type == pa.int32()


def test_validation_errors(gandiva):
    b = gandiva.TreeExprBuilder()
    fa = pa.field('a', pa.int32())
    schema = pa.schema([fa])
    na = b.make_field(fa)
    # unknown field
    e = b.make_expression(b.make_field(pa.field('zz', pa.int32())), pa.field('r', pa.int32()))
    with pytest.raises(gandiva.GandivaError, match="ExpressionValidationError.*not in schema"):
        gandiva.make_projector(schema, [e])
    # unknown function signature
    e = b.make_expression(b.make_function("add", [na, b.make_literal(1.0, pa.float64())], pa.int32()),
                          pa.field('r', pa.int32()))
    with pytest.raises(gandiva.GandivaError, match="not supported yet"):
        gandiva.make_projector(schema, [e])
    # root type != result type
    e = b.make_expression(na, pa.field('r', pa.int64()))
    with pytest.raises(gandiva.GandivaError, match="ExpressionValidationError"):
        gandiva.make_projector(schema, [e])
    # if branches disagree
    bad_if = b.make_if(b.make_literal(True, pa.bool_()), na, b.make_literal(1, pa.int64()), pa.int32())
    with pytest.raises(gandiva.GandivaError, match="not matching"):
        gandiva.make_projector(schema, [b.make_expression(bad_if, pa.field('r', pa.int32()))])
    # non-boolean condition in a filter
    with pytest.raises(gandiva.GandivaError, match="ExpressionValidationError"):
        gandiva.make_filter(schema, b.make_condition(na))
    # IN value type mismatch
    with pytest.raises(gandiva.GandivaError, match="IN clause"):
        gandiva.make_filter(schema, b.make_condition(b.make_in_expression(na, [1, 2], pa.int64())))
    # like needs a literal pattern
    fs = pa.field('s', pa.string())
    ns = b.make_field(fs)
    with pytest.raises(gandiva.GandivaError, match="literal"):
        gandiva.make_filter(pa.schema([fs]),
                            b.make_condition(b.make_function("like", [ns, ns], pa.bool_())))


def test_dump_ir_is_cuda_source(gandiva):
    """DumpIR returns the fused CUDA kernel (the reference returns LLVM IR with @expr_N
    functions; here the kernel symbol carries expr_ too)."""
    b = gandiva.TreeExprBuilder()
    fa, fb = pa.field('a', pa.int32()), pa.field('b', pa.int32())
    na, nb = b.make_field(fa), b.make_field(fb)
    e = b.make_expression(b.make_function("add", [na, nb], pa.int32()), pa.field('r', pa.int32()))
    p = gandiva.make_projector(pa.schema([fa, fb]), [e], None, "NONE",
                               gandiva.Configuration(dump_ir=True))
    ir = p.llvm_ir
    assert "__global__" in ir and "add_int32_int32" in ir and "__ballot_sync" in ir
    assert "expr_" in ir
    assert ".target sm_90a" in ir  # PTX for H100 appended when dump_ir is set
    info = p.kernel_info
    assert info["name"].startswith("gdv_project_expr_") and info["rows_per_thread"] >= 1


# the arithmetic / comparison type matrix at the head of the list differs only in a type name:
# every third one is enough for the compile gate (the GPU parity suite still runs them all)
_PROJECT = cases.all_project_cases()
_MATRIX = [c for c in _PROJECT if c.__name__.startswith(("add_", "subtract_", "multiply_", "equal_", "not_equal_", "less_than_",
                                                          "greater_than_", "less_than_or_equal_to_", "greater_than_or_equal_to_"))]
ALL_CASES = [c for c in _PROJECT if c not in _MATRIX] + _MATRIX[::3] + cases.all_filter_cases()


@pytest.mark.parametrize("case", ALL_CASES, ids=[c.__name__ for c in ALL_CASES])
def test_make_compiles_for_sm100a(case, gandiva):
    """Make() lowers the tree to one fused kernel and NVRTC compiles it for sm_90a -- the
    'does every generated kernel build' gate that needs no GPU."""
    b = gandiva.TreeExprBuilder()
    schema, outs, kind = case(b)
    if kind == "project":
        exprs = [b.make_expression(r, pa.field("o%d" % i, t)) for i, (r, t) in enumerate(outs)]
        p = gandiva.make_projector(schema, exprs, None)
        assert "__global__" in p.llvm_ir
    else:
        f = gandiva.make_filter(schema, b.make_condition(outs[0][0]))
        assert "gdv_tile_exclusive_prefix" in f.llvm_ir


NONULL_CASES = ALL_CASES[::6] + [cases.case_string_outputs, cases.case_binary_output, cases.case_q1_projector,
                                 cases.case_filter_string]


@pytest.mark.parametrize("case", NONULL_CASES, ids=[c.__name__ for c in NONULL_CASES])
def test_nonull_variants_compile(case, gandiva, monkeypatch):
    """The kernel variants specialised for batches without validity bitmaps are built lazily at
    the first Evaluate; GDV_EAGER_NONULL builds them at Make() so that they are compile-checked
    here, without a GPU (fixed-width, string-size / string-write and filter variants)."""
    monkeypatch.setenv("GDV_EAGER_NONULL", "1")
    b = gandiva.TreeExprBuilder()
    schema, outs, kind = case(b)
    if kind == "project":
        exprs = [b.make_expression(r, pa.field("o%d" % i, t)) for i, (r, t) in enumerate(outs)]
        assert "__global__" in gandiva.make_projector(schema, exprs, None).llvm_ir
    else:
        assert "__global__" in gandiva.make_filter(schema, b.make_condition(outs[0][0])).llvm_ir


def test_like_scan_kernels_compile(gandiva):
    """LIKE over view chains lowers to the warp-cooperative scan (hit list + per-row chain);
    string_scan=1 keeps the per-lane matcher only.  Both variants compile for sm_90a."""
    for case in cases.all_like_scan_cases()[::5] + [cases.case_like_scan("%special%requests%", "upper_substr32", "filter")]:
        b = gandiva.TreeExprBuilder()
        schema, outs, kind = case(b)
        for scan in (0, 1):
            cfg = gandiva.Configuration(string_scan=scan | 4)   # bit 2: the row-driven filter kernel
            if kind == "project":
                src = gandiva.make_projector(schema, [b.make_expression(outs[0][0], pa.field("o", pa.bool_()))],
                                             None, "NONE", cfg).llvm_ir
            else:
                src = gandiva.make_filter(schema, b.make_condition(outs[0][0]), cfg).llvm_ir
            assert ("gdv_likeh_" in src) == (scan == 0), case.__name__
            assert ("gdv_eqhalf_msb(" in src) == (scan == 0)
    # patterns that do not qualify (a middle segment shorter than 3 bytes, '_' wildcards) stay per lane
    for pat in ["%a%b%c%", "s_ark%", "spark%", "%ss"]:
        b = gandiva.TreeExprBuilder()
        schema, outs, _ = cases.case_like(pat)(b)
        src = gandiva.make_projector(schema, [b.make_expression(outs[0][0], pa.field("o", pa.bool_()))], None).llvm_ir
        assert "gdv_likeh_" not in src


def test_rope_consumers_build_a_two_stage_plan(gandiva):
    """concat() / repeat / pad / reverse results are ropes of views: projected, concatenated again or chosen by
    if/else directly; any other consumer makes Make() build a two-stage plan (the rope is materialised into a
    temporary column first, csrc/gdv_rope_temps.h) instead of failing.  (Results: tests/test_rope_consumers_gpu.py.)"""
    b = gandiva.TreeExprBuilder()
    t = pa.string()
    schema = pa.schema([("s", t), ("u", t)])
    cfg = gandiva.Configuration(dump_ir=True)
    cc = b.make_function("concat", [cases.F(b, "s", t), cases.F(b, "u", t)], t)
    p = gandiva.make_projector(schema, [b.make_expression(b.make_function("hash32", [cc], pa.int32()), pa.field("r", pa.int32()))],
                               None, configuration=cfg)
    assert "__gdv_rope_0" in p.llvm_ir
    # the length functions and the ASCII case maps distribute over the pieces instead: no temporary
    for ok_fn, rt in (("octet_length", pa.int32()), ("char_length", pa.int32()), ("upper", t)):
        q = gandiva.make_projector(schema, [b.make_expression(b.make_function(ok_fn, [cc], rt), pa.field("r", rt))], None,
                                   configuration=cfg)
        assert "__gdv_rope_" not in q.llvm_ir
    like = b.make_function("like", [cc, b.make_literal("%ab%", t)], pa.bool_())
    f = gandiva.make_filter(schema, b.make_condition(like), cfg)
    assert "__gdv_rope_0" in f.llvm_ir
    # replace() needs literal from / to
    with pytest.raises(pa.ArrowNotImplementedError, match="literal"):
        gandiva.make_projector(schema, [b.make_expression(
            b.make_function("replace", [cases.F(b, "s", t), cases.F(b, "u", t), b.make_literal("x", t)], t), pa.field("r", t))], None)
    # the virtual pieces of repeat / space / lpad / rpad / reverse go the same way
    for inner in (b.make_function("repeat", [cases.F(b, "s", t), b.make_literal(2, pa.int32())], t),
                  b.make_function("reverse", [cases.F(b, "s", t)], t),
                  b.make_function("lpad", [cases.F(b, "s", t), b.make_literal(9, pa.int32())], t)):
        q = gandiva.make_projector(schema, [b.make_expression(b.make_function("upper", [inner], t), pa.field("r", t))], None,
                                   configuration=cfg)
        assert "__gdv_rope_0" in q.llvm_ir


def test_cubin_cache(gandiva):
    """Two Make() calls that lower to the same kernel share one NVRTC compilation (the reference
    caches built projectors / filters); a different expression or configuration compiles anew."""
    def make(lit, cfg=None):
        b = gandiva.TreeExprBuilder()
        t = pa.int32()
        schema = pa.schema([("cache_a", t), ("cache_b", t)])
        root = b.make_function("add", [b.make_function("multiply", [cases.F(b, "cache_a", t), b.make_literal(lit, t)], t),
                                       cases.F(b, "cache_b", t)], t)
        return gandiva.make_projector(schema, [b.make_expression(root, pa.field("r", t))], None, "NONE", cfg)
    c0 = gandiva.compile_count()
    p1 = make(12345)
    c1 = gandiva.compile_count()
    assert c1 == c0 + 1
    p2 = make(12345)
    assert gandiva.compile_count() == c1
    assert p1.kernel_info["name"] == p2.kernel_info["name"]
    p3 = make(54321)
    assert gandiva.compile_count() == c1 + 1 and p3.kernel_info["name"] != p1.kernel_info["name"]
    make(12345, gandiva.Configuration(rows_per_thread=4))
    assert gandiva.compile_count() == c1 + 2


def test_selection_mode_names(gandiva):
    b = gandiva.TreeExprBuilder()
    fa = pa.field('a', pa.int32())
    e = b.make_expression(b.make_field(fa), pa.field('r', pa.int32()))
    for mode in ["NONE", "UINT16", "UINT32", "UINT64", "uint32"]:
        gandiva.make_projector(pa.schema([fa]), [e], None, mode)
    with pytest.raises(ValueError):
        gandiva.make_projector(pa.schema([fa]), [e], None, "UINT8")


def test_evaluate_without_gpu_fails_loudly(gandiva):
    """No CPU fallback: on a box without a CUDA device Evaluate raises."""
    if gandiva.cuda_available():
        pytest.skip("CUDA device present")
    b = gandiva.TreeExprBuilder()
    fa = pa.field('a', pa.int32())
    e = b.make_expression(b.make_field(fa), pa.field('r', pa.int32()))
    p = gandiva.make_projector(pa.schema([fa]), [e], None)
    batch = pa.RecordBatch.from_arrays([pa.array([1, 2, 3], pa.int32())], names=['a'])
    with pytest.raises(gandiva.GandivaError, match="CUDA"):
        p.evaluate(batch)


def test_disk_cubin_cache(tmp_path):
    import os
    """GDV_CUBIN_CACHE_DIR: a second process that lowers to the same kernel compiles nothing."""
    import subprocess
    import sys
    prog = ("import sys; sys.path.insert(0, %r); sys.path.insert(0, %r)\n"
            "import gandiva_b200 as g, cases\n"
            "b = g.TreeExprBuilder()\n"
            "f = g.make_filter(cases.Q6_SCHEMA, b.make_condition(cases.q6_condition(b)))\n"
            "print('COMPILED', g.compile_count())\n") % (os.path.dirname(os.path.dirname(os.path.abspath(__file__))),
                                                          os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ, GDV_CUBIN_CACHE_DIR=str(tmp_path))
    first = subprocess.run([sys.executable, "-c", prog], env=env, capture_output=True, text=True)
    second = subprocess.run([sys.executable, "-c", prog], env=env, capture_output=True, text=True)
    assert "COMPILED 1" in first.stdout, first.stdout + first.stderr
    assert "COMPILED 0" in second.stdout, second.stdout + second.stderr
    assert len([p for p in os.listdir(tmp_path) if p.endswith(".cubin")]) == 1
