"""gandiva_b200 — host-side mirror of the reference's Python interface over the C-ABI.

The public names, argument meaning and error behaviour follow `pyarrow.gandiva`
(P/gandiva.pyx:179-706, P = site-packages/pyarrow): `TreeExprBuilder`,
`make_projector`, `make_filter`, `Projector.evaluate`, `Filter.evaluate`,
`SelectionVector`, `Configuration`, `get_registered_function_signatures`.
A test written for `pyarrow.gandiva` runs here after `import gandiva_b200 as gandiva`.

Every call goes through `libgandiva_b200.so` (include/gandiva_b200.h) with ctypes; there
is no Python or CPU fallback: if the library or the GPU is missing the call raises.
Device-resident entry points (`evaluate_device`) take raw device pointers (e.g.
`torch.Tensor.data_ptr()`) and a CUDA stream handle; PyTorch is only used by callers for
device memory, streams and torch.distributed.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Any, Iterable, Sequence

import numpy as np
import pyarrow as pa

__all__ = [
    "TreeExprBuilder", "Node", "Expression", "Condition", "Configuration", "SelectionVector",
    "Projector", "Filter", "FunctionSignature", "FunctionRegistry", "make_projector", "make_filter",
    "get_registered_function_signatures", "GandivaError", "cuda_available", "lib",
]

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "libgandiva_b200.so")

# ---- status codes (include/gandiva_b200.h) --------------------------------------------------
GDV_OK = 0
GDV_OUT_OF_MEMORY = 1
GDV_INVALID = 4
GDV_NOT_IMPLEMENTED = 10
GDV_CODEGEN_ERROR = 40
GDV_EXPRESSION_VALIDATION_ERROR = 41
GDV_EXECUTION_ERROR = 42
GDV_CUDA_ERROR = 100

GDV_SEL_NONE, GDV_SEL_UINT16, GDV_SEL_UINT32, GDV_SEL_UINT64 = 0, 1, 2, 3
GDV_SEL_BOUNDED = 0x100
GDV_BOARD_MAX_WORLD, GDV_BOARD_SLOTS = 16, 4
GDV_BOARD_BYTES = (2 * GDV_BOARD_SLOTS * GDV_BOARD_MAX_WORLD + GDV_BOARD_SLOTS + 1) * 8
GDV_MEM_HOST, GDV_MEM_DEVICE = 0, 1


class GandivaError(pa.ArrowException):
    """Raised for Gandiva status codes 40/41/42 and CUDA failures."""

    def __init__(self, code: int, message: str):
        prefix = {GDV_CODEGEN_ERROR: "CodeGenError", GDV_EXPRESSION_VALIDATION_ERROR:
                  "ExpressionValidationError", GDV_EXECUTION_ERROR: "ExecutionError",
                  GDV_CUDA_ERROR: "CudaError"}.get(code, "Error(%d)" % code)
        super().__init__("%s: %s" % (prefix, message))
        self.code = code


class gdv_type_t(C.Structure):
    _fields_ = [("id", C.c_int32), ("precision", C.c_int32), ("scale", C.c_int32)]


class gdv_config_t(C.Structure):
    _fields_ = [("optimize", C.c_int32), ("dump_ir", C.c_int32), ("device", C.c_int32),
                ("rows_per_thread", C.c_int32), ("block_threads", C.c_int32),
                ("loader", C.c_int32), ("sm_reserve", C.c_int32), ("stages", C.c_int32),
                ("string_scan", C.c_int32), ("filter_gating", C.c_int32), ("function_registry", C.c_void_p)]


class gdv_function_def_t(C.Structure):
    _fields_ = [("name", C.c_char_p), ("params", C.POINTER(gdv_type_t)), ("n_params", C.c_int32),
                ("ret", gdv_type_t), ("null_mode", C.c_int32), ("can_raise", C.c_int32),
                ("body", C.c_char_p), ("prelude", C.c_char_p)]


class gdv_column_t(C.Structure):
    _fields_ = [("validity", C.c_void_p), ("values", C.c_void_p), ("var_data", C.c_void_p),
                ("offset", C.c_int64), ("var_data_size", C.c_int64)]


class gdv_dictionary_t(C.Structure):
    """The dictionary of a dictionary-encoded column (include/gandiva_b200.h): the column's
    gdv_column_t holds validity + indices, and its var_data points at one of these."""
    _fields_ = [("validity", C.c_void_p), ("offsets", C.c_void_p), ("data", C.c_void_p),
                ("offset", C.c_int64), ("length", C.c_int64), ("data_size", C.c_int64)]


class gdv_view_buffers_t(C.Structure):
    """The data buffers of a string_view / binary_view column (include/gandiva_b200.h): the column's
    gdv_column_t holds validity + 16-byte views, and its var_data points at one of these.  `data` is
    a host array of `n` buffer pointers and `sizes` their n int64 sizes, both in the batch's memory
    space (device pointers and a device sizes array for evaluate_device)."""
    _fields_ = [("data", C.POINTER(C.c_void_p)), ("sizes", C.c_void_p), ("n", C.c_int32)]


class gdv_batch_t(C.Structure):
    _fields_ = [("num_rows", C.c_int64), ("num_columns", C.c_int32), ("mem_space", C.c_int32),
                ("columns", C.POINTER(gdv_column_t))]


class gdv_out_column_t(C.Structure):
    _fields_ = [("validity", C.c_void_p), ("values", C.c_void_p), ("var_data", C.c_void_p),
                ("var_capacity", C.c_int64), ("var_size", C.c_int64)]


class gdv_selection_t(C.Structure):
    _fields_ = [("indices", C.c_void_p), ("max_slots", C.c_int64), ("num_slots", C.c_int64),
                ("mode", C.c_int32), ("mem_space", C.c_int32), ("index_base", C.c_int64),
                ("d_num_slots", C.c_void_p)]


def _load() -> C.CDLL:
    if not os.path.exists(_LIB_PATH):
        raise ImportError(
            "gandiva_b200: %s is missing; build it with `python -m gandiva_b200.build` "
            "(there is no CPU fallback)" % _LIB_PATH)
    L = C.CDLL(_LIB_PATH)
    vp, i32, i64 = C.c_void_p, C.c_int32, C.c_int64
    P = C.POINTER
    sig = {
        "gdv_config_default": (None, [P(gdv_config_t)]),
        "gdv_version": (C.c_char_p, []),
        "gdv_last_error": (C.c_char_p, []),
        "gdv_cuda_available": (i32, []),
        "gdv_device_count": (i32, []),
        "gdv_node_field": (i32, [C.c_char_p, gdv_type_t, P(vp)]),
        "gdv_node_literal": (i32, [gdv_type_t, vp, i64, i32, P(vp)]),
        "gdv_node_function": (i32, [C.c_char_p, P(vp), i32, gdv_type_t, P(vp)]),
        "gdv_node_if": (i32, [vp, vp, vp, gdv_type_t, P(vp)]),
        "gdv_node_and": (i32, [P(vp), i32, P(vp)]),
        "gdv_node_or": (i32, [P(vp), i32, P(vp)]),
        "gdv_node_in": (i32, [vp, gdv_type_t, vp, P(i32), i32, P(vp)]),
        "gdv_node_return_type": (i32, [vp, P(gdv_type_t)]),
        "gdv_node_to_string": (i64, [vp, C.c_char_p, i64]),
        "gdv_node_release": (None, [vp]),
        "gdv_expression_make": (i32, [vp, C.c_char_p, gdv_type_t, P(vp)]),
        "gdv_expression_to_string": (i64, [vp, C.c_char_p, i64]),
        "gdv_expression_release": (None, [vp]),
        "gdv_condition_make": (i32, [vp, P(vp)]),
        "gdv_condition_to_string": (i64, [vp, C.c_char_p, i64]),
        "gdv_condition_release": (None, [vp]),
        "gdv_schema_make": (i32, [P(C.c_char_p), P(gdv_type_t), i32, P(vp)]),
        "gdv_schema_release": (None, [vp]),
        "gdv_projector_make": (i32, [vp, P(vp), i32, i32, P(gdv_config_t), P(vp)]),
        "gdv_projector_evaluate": (i32, [vp, P(gdv_batch_t), P(gdv_selection_t),
                                         P(gdv_out_column_t), i32, vp, i32]),
        "gdv_projector_sync": (i32, [vp, vp]),
        "gdv_device_alloc": (i32, [i32, C.c_size_t, P(vp)]),
        "gdv_device_free": (i32, [i32, vp]),
        "gdv_device_trim": (i32, [i32, C.c_size_t, P(C.c_size_t)]),
        "gdv_staged_bytes": (C.c_int64, []),
        "gdv_projector_output_var_size": (i32, [vp, P(gdv_batch_t), P(gdv_selection_t), i32, vp,
                                                P(i64)]),
        "gdv_projector_dump_ir": (i64, [vp, C.c_char_p, i64]),
        "gdv_projector_kernel_info": (i32, [vp, C.c_char_p, i64, P(i32), P(i32), P(i32), P(i32)]),
        "gdv_projector_release": (None, [vp]),
        "gdv_filter_make": (i32, [vp, vp, P(gdv_config_t), P(vp)]),
        "gdv_filter_evaluate": (i32, [vp, P(gdv_batch_t), P(gdv_selection_t), vp, i32, vp]),
        "gdv_filter_sync": (i32, [vp, vp, P(i64)]),
        "gdv_filter_dump_ir": (i64, [vp, C.c_char_p, i64]),
        "gdv_filter_kernel_info": (i32, [vp, C.c_char_p, i64, P(i32), P(i32), P(i32), P(i32)]),
        "gdv_selection_push": (i32, [i32, vp, vp, vp, i64, vp, i32, i32, i32, C.c_uint64, C.c_uint64, i32,
                                     i32, vp, C.c_uint64, vp, vp, i32, i32, vp]),
        "gdv_selection_release": (i32, [i32, vp, i32, C.c_uint64, vp]),
        "gdv_enable_peer_access": (i32, [i32, i32]),
        "gdv_ipc_export": (i32, [i32, vp, C.c_char_p, P(i64)]),
        "gdv_ipc_open": (i32, [i32, C.c_char_p, i64, P(vp)]),
        "gdv_ipc_close": (i32, [i32, vp, i64]),
        "gdv_projector_kernel_attr": (i32, [vp, C.c_char_p, P(i64)]),
        "gdv_filter_kernel_attr": (i32, [vp, C.c_char_p, P(i64)]),
        "gdv_filter_release": (None, [vp]),
        "gdv_registry_size": (i32, []),
        "gdv_registry_get": (i32, [i32, P(C.c_char_p), P(gdv_type_t), P(gdv_type_t), i32, P(i32)]),
        "gdv_function_registry_create": (i32, [P(vp)]),
        "gdv_function_registry_release": (None, [vp]),
        "gdv_function_registry_add": (i32, [vp, P(gdv_function_def_t)]),
        "gdv_function_registry_signatures": (i32, [vp]),
        "gdv_function_registry_get": (i32, [vp, i32, P(C.c_char_p), P(gdv_type_t), P(gdv_type_t), i32, P(i32)]),
        "gdv_host_alloc": (i32, [C.c_size_t, P(vp)]),
        "gdv_host_free": (i32, [vp]),
        "gdv_generate_lineitem": (i32, [i32, i32, C.c_uint64, i64, i64, vp, vp, i32, vp]),
        "gdv_launch_count": (i64, []),
        "gdv_compile_count": (i64, []),
        # include/gandiva_b200_arrow.h
        "gdv_schema_from_arrow": (i32, [vp, P(vp)]),
        "gdv_arrow_batch_import": (i32, [vp, vp, P(vp)]),
        "gdv_arrow_batch_view": (P(gdv_batch_t), [vp]),
        "gdv_arrow_batch_wait": (i32, [vp, vp]),
        "gdv_arrow_batch_release": (None, [vp]),
        "gdv_projector_output_schema_arrow": (i32, [vp, vp]),
        "gdv_projector_evaluate_arrow": (i32, [vp, vp, vp, vp]),
        "gdv_filter_evaluate_arrow": (i32, [vp, vp, i32, vp, vp]),
        "gdv_memcpy": (i32, [i32, vp, vp, C.c_size_t, i32]),
    }
    for name, (res, args) in sig.items():
        fn = getattr(L, name)
        fn.restype = res
        fn.argtypes = args
    return L


lib = _load()
C_ABI_SYMBOLS = None  # filled lazily by tests from include/gandiva_b200.h


def _check(status: int) -> None:
    if status == GDV_OK:
        return
    msg = (lib.gdv_last_error() or b"").decode("utf-8", "replace")
    if status == GDV_INVALID:
        raise pa.ArrowInvalid(msg)
    if status == GDV_NOT_IMPLEMENTED:
        raise pa.ArrowNotImplementedError(msg)
    if status == GDV_OUT_OF_MEMORY:
        raise pa.ArrowMemoryError(msg)
    raise GandivaError(status, msg)


def cuda_available() -> bool:
    return bool(lib.gdv_cuda_available())


def compile_count() -> int:
    """NVRTC compilations so far (Make() calls served from the cubin cache do not count)."""
    return int(lib.gdv_compile_count())


def launch_count() -> int:
    return int(lib.gdv_launch_count())


# ---- type mapping ------------------------------------------------------------------------
_UNIT = {"s": 0, "ms": 1, "us": 2, "ns": 3}


GDV_TYPE_DICTIONARY = 29
GDV_DICT_ORDERED = 0x100
GDV_TYPE_STRING_VIEW = 39
GDV_TYPE_BINARY_VIEW = 40
GDV_TYPE_LARGE_STRING = 34
GDV_TYPE_LARGE_BINARY = 35


def _to_c_type(t: pa.DataType) -> gdv_type_t:
    if pa.types.is_dictionary(t):
        return gdv_type_t(GDV_TYPE_DICTIONARY, int(t.index_type.id) | (GDV_DICT_ORDERED if t.ordered else 0),
                          int(t.value_type.id))
    if pa.types.is_decimal128(t):
        return gdv_type_t(int(t.id), t.precision, t.scale)
    if pa.types.is_timestamp(t) or pa.types.is_time32(t) or pa.types.is_time64(t):
        return gdv_type_t(int(t.id), _UNIT[t.unit], 0)
    return gdv_type_t(int(t.id), 0, 0)


def _from_c_type(t: gdv_type_t) -> pa.DataType:
    tid = t.id
    simple = {1: pa.bool_(), 2: pa.uint8(), 3: pa.int8(), 4: pa.uint16(), 5: pa.int16(),
              6: pa.uint32(), 7: pa.int32(), 8: pa.uint64(), 9: pa.int64(), 11: pa.float32(),
              12: pa.float64(), 13: pa.string(), 14: pa.binary(), 16: pa.date32(),
              17: pa.date64(), GDV_TYPE_STRING_VIEW: pa.string_view(), GDV_TYPE_BINARY_VIEW: pa.binary_view(),
              GDV_TYPE_LARGE_STRING: pa.large_string(), GDV_TYPE_LARGE_BINARY: pa.large_binary()}
    if tid in simple:
        return simple[tid]
    if tid == GDV_TYPE_DICTIONARY:
        return pa.dictionary(simple[t.precision & 0xff], simple[t.scale], bool(t.precision & GDV_DICT_ORDERED))
    unit = {0: "s", 1: "ms", 2: "us", 3: "ns"}.get(t.precision, "ms")
    if tid == 18:
        return pa.timestamp(unit)
    if tid == 19:
        return pa.time32(unit if unit in ("s", "ms") else "ms")
    if tid == 20:
        return pa.time64(unit if unit in ("us", "ns") else "us")
    if tid == 23:
        return pa.decimal128(max(t.precision, 1), t.scale)
    raise pa.ArrowNotImplementedError("unsupported type id %d" % tid)


def _ensure_type(t: Any) -> pa.DataType:
    if t is None:
        raise TypeError("DataType expected, got None")
    if isinstance(t, pa.DataType):
        return t
    if isinstance(t, str):
        return pa.type_for_alias(t)
    raise TypeError("DataType expected, got %r" % type(t))


def _to_string(fn, handle) -> str:
    n = fn(handle, None, 0)
    buf = C.create_string_buffer(int(n) + 1)
    fn(handle, buf, int(n) + 1)
    return buf.value.decode("utf-8", "replace")


# ---- nodes -------------------------------------------------------------------------------
class Node:
    """Expression-tree node (gandiva::Node, P/includes/libgandiva.pxd:29-31).

    Besides the native handle the Python object keeps the tree structure (`kind`, `children`,
    `payload`) so tests can hand the same tree to the CPU oracle."""

    def __init__(self, handle: int, kind: str, dtype: pa.DataType, children: Sequence["Node"] = (),
                 payload: Any = None):
        self._h = C.c_void_p(handle)
        self.kind = kind
        self.dtype = dtype
        self.children = list(children)
        self.payload = payload

    def __del__(self):
        try:
            if self._h:
                lib.gdv_node_release(self._h)
        except Exception:
            pass

    def __str__(self) -> str:
        return _to_string(lib.gdv_node_to_string, self._h)

    def return_type(self) -> pa.DataType:
        return self.dtype


class Expression:
    def __init__(self, handle: int, root: Node, field: pa.Field):
        self._h = C.c_void_p(handle)
        self._root = root
        self._field = field

    def __del__(self):
        try:
            lib.gdv_expression_release(self._h)
        except Exception:
            pass

    def __str__(self) -> str:
        return _to_string(lib.gdv_expression_to_string, self._h)

    def root(self) -> Node:
        return self._root

    def result(self) -> pa.Field:
        return self._field


class Condition:
    def __init__(self, handle: int, root: Node):
        self._h = C.c_void_p(handle)
        self._root = root

    def __del__(self):
        try:
            lib.gdv_condition_release(self._h)
        except Exception:
            pass

    def __str__(self) -> str:
        return _to_string(lib.gdv_condition_to_string, self._h)

    def root(self) -> Node:
        return self._root

    def result(self) -> pa.Field:
        return pa.field("cond", pa.bool_())


_INT_RANGE = {
    pa.int8(): (np.int8, -2**7, 2**7 - 1), pa.int16(): (np.int16, -2**15, 2**15 - 1),
    pa.int32(): (np.int32, -2**31, 2**31 - 1), pa.int64(): (np.int64, -2**63, 2**63 - 1),
    pa.uint8(): (np.uint8, 0, 2**8 - 1), pa.uint16(): (np.uint16, 0, 2**16 - 1),
    pa.uint32(): (np.uint32, 0, 2**32 - 1), pa.uint64(): (np.uint64, 0, 2**64 - 1),
}


def _node_arr(nodes: Iterable[Node]):
    nodes = list(nodes)
    for n in nodes:
        if not isinstance(n, Node):
            raise TypeError("Node expected, got %r" % type(n))
    arr = (C.c_void_p * max(len(nodes), 1))(*[n._h for n in nodes])
    return arr, len(nodes)


class TreeExprBuilder:
    """gandiva::TreeExprBuilder (P/gandiva.pyx:283-589)."""

    def make_literal(self, value: Any, dtype: Any) -> Node:
        t = _ensure_type(dtype)
        out = C.c_void_p()
        if value is None:
            _check(lib.gdv_node_literal(_to_c_type(t), None, 0, 1, C.byref(out)))
            return Node(out.value, "literal", t, payload=None)
        if pa.types.is_boolean(t):
            if not isinstance(value, (bool, np.bool_)):
                raise TypeError("bool literal expected")
            raw = np.array([1 if value else 0], dtype=np.uint8).tobytes()
        elif t in _INT_RANGE:
            if isinstance(value, (bool, str, bytes, float)) or not isinstance(value, (int, np.integer)):
                raise TypeError("integer literal expected for %s" % t)
            npt, lo, hi = _INT_RANGE[t]
            if not lo <= int(value) <= hi:
                raise OverflowError("literal %r out of range for %s" % (value, t))
            raw = np.array([value], dtype=npt).tobytes()
        elif pa.types.is_float32(t) or pa.types.is_float64(t):
            if isinstance(value, (str, bytes)):
                raise TypeError("float literal expected")
            raw = np.array([value], dtype=np.float32 if pa.types.is_float32(t) else np.float64).tobytes()
        elif _is_varlen(t):
            if isinstance(value, str):
                raw = value.encode("utf-8")
            elif isinstance(value, (bytes, bytearray)):
                raw = bytes(value)
            else:
                raise TypeError("str/bytes literal expected")
            buf = C.create_string_buffer(raw, len(raw)) if raw else None
            _check(lib.gdv_node_literal(_to_c_type(t), C.cast(buf, C.c_void_p) if buf else None,
                                        len(raw), 0, C.byref(out)))
            return Node(out.value, "literal", t, payload=raw)
        elif pa.types.is_decimal128(t):
            import decimal
            d = decimal.Decimal(value) if not isinstance(value, int) else None
            unscaled = int(value) if d is None else int(d.scaleb(t.scale).to_integral_value())
            raw = (unscaled & ((1 << 128) - 1)).to_bytes(16, "little")
            value = unscaled
        elif pa.types.is_date32(t) or pa.types.is_time32(t):
            raw = np.array([int(value)], dtype=np.int32).tobytes()
        elif pa.types.is_date64(t) or pa.types.is_timestamp(t) or pa.types.is_time64(t):
            raw = np.array([int(value)], dtype=np.int64).tobytes()
        else:
            raise TypeError("Didn't recognize dtype " + str(t))
        buf = C.create_string_buffer(raw, len(raw))
        _check(lib.gdv_node_literal(_to_c_type(t), C.cast(buf, C.c_void_p), len(raw), 0, C.byref(out)))
        return Node(out.value, "literal", t, payload=value)

    def make_expression(self, root_node: Node, return_field: pa.Field) -> Expression:
        if not isinstance(root_node, Node):
            raise TypeError("Node expected")
        if not isinstance(return_field, pa.Field):
            raise TypeError("Field expected")
        out = C.c_void_p()
        _check(lib.gdv_expression_make(root_node._h, return_field.name.encode(),
                                       _to_c_type(return_field.type), C.byref(out)))
        return Expression(out.value, root_node, return_field)

    def make_function(self, name: str, children: Sequence[Node], return_type: Any) -> Node:
        t = _ensure_type(return_type)
        arr, n = _node_arr(children)
        out = C.c_void_p()
        _check(lib.gdv_node_function(name.encode(), arr, n, _to_c_type(t), C.byref(out)))
        return Node(out.value, "function", t, children, payload=name)

    def make_field(self, field: pa.Field) -> Node:
        if not isinstance(field, pa.Field):
            raise TypeError("Field expected")
        out = C.c_void_p()
        _check(lib.gdv_node_field(field.name.encode(), _to_c_type(field.type), C.byref(out)))
        return Node(out.value, "field", field.type, payload=field.name)

    def make_if(self, condition: Node, this_node: Node, else_node: Node, return_type: Any) -> Node:
        for n in (condition, this_node, else_node):
            if not isinstance(n, Node):
                raise TypeError("Node expected")
        t = _ensure_type(return_type)
        out = C.c_void_p()
        _check(lib.gdv_node_if(condition._h, this_node._h, else_node._h, _to_c_type(t), C.byref(out)))
        return Node(out.value, "if", t, [condition, this_node, else_node])

    def make_and(self, children: Sequence[Node]) -> Node:
        arr, n = _node_arr(children)
        out = C.c_void_p()
        _check(lib.gdv_node_and(arr, n, C.byref(out)))
        return Node(out.value, "and", pa.bool_(), children)

    def make_or(self, children: Sequence[Node]) -> Node:
        arr, n = _node_arr(children)
        out = C.c_void_p()
        _check(lib.gdv_node_or(arr, n, C.byref(out)))
        return Node(out.value, "or", pa.bool_(), children)

    def make_in_expression(self, node: Node, values: Iterable[Any], dtype: Any) -> Node:
        if not isinstance(node, Node):
            raise TypeError("Node expected")
        t = _ensure_type(dtype)
        values = list(values)
        out = C.c_void_p()
        if _is_varlen(t):
            raws = [v.encode("utf-8") if isinstance(v, str) else bytes(v) for v in values]
            blob = b"".join(raws)
            lens = (C.c_int32 * max(len(raws), 1))(*[len(r) for r in raws])
            buf = C.create_string_buffer(blob, max(len(blob), 1))
            _check(lib.gdv_node_in(node._h, _to_c_type(t), C.cast(buf, C.c_void_p), lens, len(raws),
                                   C.byref(out)))
            return Node(out.value, "in", pa.bool_(), [node], payload=(t, raws))
        if pa.types.is_floating(t) and t.bit_width in (32, 64):
            # C++ MakeInExpressionFloat / Double: the constants travel as bit patterns
            ft, it = (np.float32, np.int32) if t.bit_width == 32 else (np.float64, np.int64)
            arr = np.ascontiguousarray(np.array(values, dtype=ft)).view(it)
            _check(lib.gdv_node_in(node._h, _to_c_type(t), arr.ctypes.data_as(C.c_void_p), None, len(arr), C.byref(out)))
            return Node(out.value, "in", pa.bool_(), [node], payload=(t, [float(x) for x in np.array(values, dtype=ft)]))
        if t.bit_width == 32:
            arr = np.array(pa.array(values, type=t).cast(pa.int32()).to_numpy(), dtype=np.int32) \
                if values else np.zeros(0, np.int32)
        elif t.bit_width == 64:
            arr = np.array(pa.array(values, type=t).cast(pa.int64()).to_numpy(), dtype=np.int64) \
                if values else np.zeros(0, np.int64)
        else:
            raise TypeError("Data type " + str(t) + " not supported")
        arr = np.ascontiguousarray(arr)
        _check(lib.gdv_node_in(node._h, _to_c_type(t), arr.ctypes.data_as(C.c_void_p), None,
                               len(arr), C.byref(out)))
        return Node(out.value, "in", pa.bool_(), [node], payload=(t, [int(x) for x in arr]))

    def make_condition(self, condition: Node) -> Condition:
        if not isinstance(condition, Node):
            raise TypeError("Node expected")
        out = C.c_void_p()
        _check(lib.gdv_condition_make(condition._h, C.byref(out)))
        return Condition(out.value, condition)


# ---- configuration -----------------------------------------------------------------------
class Configuration:
    """gandiva::Configuration (optimize, dump_ir) plus device placement / tuning knobs."""

    def __init__(self, optimize: bool = True, dump_ir: bool = False, device: int = 0,
                 rows_per_thread: int = 0, block_threads: int = 0, loader: int = 0,
                 sm_reserve: int = 0, stages: int = 0, string_scan: int = 0, filter_gating: int = 0,
                 function_registry: "FunctionRegistry | None" = None):
        self.function_registry = function_registry
        self.stages = int(stages)
        self.string_scan = int(string_scan)
        self.filter_gating = int(filter_gating)
        self.optimize = bool(optimize)
        self.dump_ir = bool(dump_ir)
        self.device = int(device)
        self.rows_per_thread = int(rows_per_thread)
        self.block_threads = int(block_threads)
        self.loader = int(loader)
        self.sm_reserve = int(sm_reserve)

    def _c(self) -> gdv_config_t:
        c = gdv_config_t()
        lib.gdv_config_default(C.byref(c))
        c.optimize = int(self.optimize)
        c.dump_ir = int(self.dump_ir)
        c.device = self.device
        c.rows_per_thread = self.rows_per_thread
        c.block_threads = self.block_threads
        c.loader = self.loader
        c.sm_reserve = self.sm_reserve
        c.stages = self.stages
        c.string_scan = self.string_scan
        c.filter_gating = self.filter_gating
        if self.function_registry is not None:
            c.function_registry = self.function_registry._h
        return c


# ---- selection vector --------------------------------------------------------------------
GDV_WAVE_FIRST, GDV_WAVE_LAST = 1, 2
_SEL_MODE = {"NONE": GDV_SEL_NONE, "UINT16": GDV_SEL_UINT16, "UINT32": GDV_SEL_UINT32,
             "UINT64": GDV_SEL_UINT64}
_SEL_NP = {GDV_SEL_UINT16: np.uint16, GDV_SEL_UINT32: np.uint32, GDV_SEL_UINT64: np.uint64}


def _ensure_selection_mode(name: str) -> int:
    try:
        name = name.upper()
        if name.endswith("|BOUNDED"):   # device-resident Filter only (GDV_SEL_BOUNDED)
            return _SEL_MODE[name[:-8]] | GDV_SEL_BOUNDED
        return _SEL_MODE[name]
    except KeyError:
        raise ValueError("Invalid value for Selection Mode: %r" % (name,))


class SelectionVector:
    """gandiva::SelectionVector: ascending row indices (P/includes/libgandiva.pxd:43-71)."""

    def __init__(self, indices: np.ndarray, num_slots: int, mode: int):
        self._indices = indices
        self.num_slots = int(num_slots)
        self.mode = mode

    def to_array(self) -> pa.Array:
        return pa.array(self._indices[: self.num_slots])

    def _c(self) -> gdv_selection_t:
        return gdv_selection_t(self._indices.ctypes.data_as(C.c_void_p), len(self._indices),
                               self.num_slots, self.mode, GDV_MEM_HOST)


# ---- batch marshalling -------------------------------------------------------------------
def _dictionary_to_c(d: pa.Array) -> gdv_dictionary_t:
    """A utf8 / binary dictionary -> gdv_dictionary_t over its own buffers (no copies).  The
    struct keeps the arrays it points into alive."""
    bufs = d.buffers()
    if len(bufs) != 3:
        raise pa.ArrowNotImplementedError("dictionary of type %s: only utf8 and binary dictionaries are supported"
                                          % d.type)
    c = gdv_dictionary_t()
    c.validity = bufs[0].address if bufs[0] is not None and d.null_count > 0 else None
    c.offsets = bufs[1].address if bufs[1] is not None else None
    c.data = bufs[2].address if bufs[2] is not None else None
    c.offset = d.offset
    c.length = len(d)
    c.data_size = bufs[2].size if bufs[2] is not None else 0
    c._keep = (d, bufs)
    return c


def view_buffers(data: Sequence[int], sizes: int) -> gdv_view_buffers_t:
    """gdv_view_buffers_t over `data` (buffer addresses) and `sizes` (address of len(data) int64
    sizes), e.g. device pointers for Projector / Filter evaluate_device."""
    c = gdv_view_buffers_t()
    table = (C.c_void_p * max(len(data), 1))(*[int(p) or None for p in data])
    c.data = C.cast(table, C.POINTER(C.c_void_p))
    c.sizes = sizes or None
    c.n = len(data)
    c._keep = table
    return c


def _view_buffers_to_c(arr: pa.Array) -> gdv_view_buffers_t:
    """The data buffers of a string_view / binary_view array (sliced ones included: a slice keeps
    every buffer of its parent) -> gdv_view_buffers_t with host pointers.  pyarrow lists them as
    buffers()[2:], without the variadic sizes buffer: the sizes are the buffers' own sizes."""
    data = [b for b in arr.buffers()[2:]]
    sizes = np.array([b.size if b is not None else 0 for b in data] or [0], dtype=np.int64)
    c = view_buffers([b.address if b is not None else 0 for b in data], sizes.ctypes.data)
    c._keep = (c._keep, data, sizes)
    return c


def _is_varlen(t: pa.DataType) -> bool:
    """utf8 / binary with contiguous bytes behind int32 or int64 offsets."""
    return pa.types.is_string(t) or pa.types.is_binary(t) or pa.types.is_large_string(t) or pa.types.is_large_binary(t)


def _batch_to_c(batch: pa.RecordBatch):
    """RecordBatch -> gdv_batch_t over the batch's own buffers (no copies)."""
    cols = (gdv_column_t * max(batch.num_columns, 1))()
    keep = []
    for i in range(batch.num_columns):
        arr = batch.column(i)
        bufs = arr.buffers()
        keep.append(bufs)
        c = cols[i]
        # a bitmap without any cleared bit is passed as "no validity" (selects the no-null kernel)
        c.validity = bufs[0].address if bufs[0] is not None and arr.null_count > 0 else None
        t = arr.type
        if pa.types.is_dictionary(t):
            # indices like a fixed-width column; var_data -> the dictionary (zero copy)
            c.values = bufs[1].address if bufs[1] is not None else None
            d = _dictionary_to_c(arr.dictionary)
            keep.append(d)
            c.var_data = C.addressof(d)
        elif pa.types.is_string_view(t) or pa.types.is_binary_view(t):
            # views like a fixed-width column; var_data -> the data buffers (zero copy)
            c.values = bufs[1].address if bufs[1] is not None else None
            v = _view_buffers_to_c(arr)
            keep.append(v)
            c.var_data = C.addressof(v)
        elif _is_varlen(t):
            # int32 offsets, or int64 for large_string / large_binary; var_data -> the bytes
            c.values = bufs[1].address if bufs[1] is not None else None
            c.var_data = bufs[2].address if len(bufs) > 2 and bufs[2] is not None else None
            c.var_data_size = bufs[2].size if len(bufs) > 2 and bufs[2] is not None else 0
        else:
            c.values = bufs[1].address if len(bufs) > 1 and bufs[1] is not None else None
        c.offset = arr.offset
    b = gdv_batch_t(batch.num_rows, batch.num_columns, GDV_MEM_HOST, cols)
    return b, (cols, keep)


def _var_ptr(var):
    """var_data of a device column: the bytes of a utf8 / binary column, a gdv_dictionary_t (with
    device pointers) for a dictionary-encoded one, or a gdv_view_buffers_t for a view column."""
    if isinstance(var, (gdv_dictionary_t, gdv_view_buffers_t)):
        return C.addressof(var)
    return var or None


class _SchemaHandle:
    def __init__(self, schema: pa.Schema):
        if not isinstance(schema, pa.Schema):
            raise TypeError("Schema expected")
        n = len(schema)
        names = (C.c_char_p * max(n, 1))(*[f.name.encode() for f in schema])
        types = (gdv_type_t * max(n, 1))(*[_to_c_type(f.type) for f in schema])
        self._h = C.c_void_p()
        _check(lib.gdv_schema_make(names, types, n, C.byref(self._h)))

    def __del__(self):
        try:
            lib.gdv_schema_release(self._h)
        except Exception:
            pass


def _stream_handle(stream: int) -> C.c_void_p:
    """cudaStream_t value -> handle for the C-ABI.  The C-ABI reads NULL as "the engine's own
    stream"; a caller that passes 0 here means CUDA's legacy default stream (torch's default
    stream), whose explicit handle is CU_STREAM_LEGACY (0x1)."""
    return C.c_void_p(stream if stream else 1)


def _kernel_info(fn, handle, attr_fn=None) -> dict:
    name = C.create_string_buffer(256)
    regs, smem, rpt, bt = C.c_int32(), C.c_int32(), C.c_int32(), C.c_int32()
    _check(fn(handle, name, 256, C.byref(regs), C.byref(smem), C.byref(rpt), C.byref(bt)))
    info = {"name": name.value.decode(), "regs": regs.value, "smem_bytes": smem.value,
            "rows_per_thread": rpt.value, "block_threads": bt.value}
    if attr_fn is not None:
        keys = ["staged", "stages", "dynamic_smem", "cta_tile_rows", "tile_rows", "nullable"]
        keys.append("view_shortcuts")
        if attr_fn is lib.gdv_filter_kernel_attr:
            keys += ["dictionary_first", "gated_stages"]
        if regs.value >= 0:
            keys.append("blocks_per_sm")
        for key in keys:
            v = C.c_int64()
            if attr_fn(handle, key.encode(), C.byref(v)) == 0:
                info[key] = v.value
    return info


# ---- Projector ---------------------------------------------------------------------------
class Projector:
    """gandiva::Projector (P/gandiva.pyx:179-226)."""

    def __init__(self, handle: int, schema: pa.Schema, exprs: Sequence[Expression], mode: int,
                 schema_handle: _SchemaHandle):
        self._h = C.c_void_p(handle)
        self._schema = schema
        self._exprs = list(exprs)
        self._mode = mode
        self._schema_handle = schema_handle

    def __del__(self):
        try:
            lib.gdv_projector_release(self._h)
        except Exception:
            pass

    @property
    def llvm_ir(self) -> str:
        """The generated CUDA source (+PTX with dump_ir); the reference returns LLVM IR here."""
        return _to_string(lib.gdv_projector_dump_ir, self._h)

    @property
    def kernel_info(self) -> dict:
        return _kernel_info(lib.gdv_projector_kernel_info, self._h, lib.gdv_projector_kernel_attr)

    def evaluate(self, batch: pa.RecordBatch, selection: SelectionVector | None = None) -> list:
        if not isinstance(batch, pa.RecordBatch):
            raise TypeError("RecordBatch expected")
        cb, keep = _batch_to_c(batch)
        n = batch.num_rows if selection is None else selection.num_slots
        outs = (gdv_out_column_t * len(self._exprs))()
        holders = []
        csel = None
        if selection is not None:
            s = selection._c()
            csel = C.byref(s)
        for i, e in enumerate(self._exprs):
            t = e.result().type
            vbytes = (n + 7) // 8
            vbuf = np.zeros((vbytes + 7) // 8 * 8, dtype=np.uint8)
            var = None
            if _is_varlen(t):
                # utf8/binary: size the data buffer with the sizing pass, as the C++ layer does
                need = C.c_int64(0)
                _check(lib.gdv_projector_output_var_size(self._h, C.byref(cb), csel, i, None, C.byref(need)))
                large = pa.types.is_large_string(t) or pa.types.is_large_binary(t)
                dbuf = np.zeros(n + 1, dtype=np.int64 if large else np.int32)
                var = np.zeros(max(need.value, 8), dtype=np.uint8)
                outs[i].var_data = var.ctypes.data_as(C.c_void_p)
                outs[i].var_capacity = need.value
            elif pa.types.is_boolean(t):
                dbuf = np.zeros((vbytes + 7) // 8 * 8, dtype=np.uint8)
            else:
                dbuf = np.zeros(max(n * (t.bit_width // 8), 8), dtype=np.uint8)
            holders.append((vbuf, dbuf, var))
            outs[i].validity = vbuf.ctypes.data_as(C.c_void_p)
            outs[i].values = dbuf.ctypes.data_as(C.c_void_p)
        _check(lib.gdv_projector_evaluate(self._h, C.byref(cb), csel, outs, len(self._exprs), None, 0))
        result = []
        for (vbuf, dbuf, var), e in zip(holders, self._exprs):
            t = e.result().type
            bufs = [pa.py_buffer(vbuf), pa.py_buffer(dbuf)]
            if var is not None:
                bufs.append(pa.py_buffer(var))
            result.append(pa.Array.from_buffers(t, n, bufs))
        return result

    # -- device-resident path (bench / multi-GPU): raw pointers in HBM, caller-owned stream ----
    def evaluate_device(self, num_rows: int, columns: Sequence[tuple], outputs: Sequence[tuple],
                        stream: int = 0, selection: tuple | None = None, sync: bool = False) -> list | None:
        """columns: per schema field (validity_ptr|0, values_ptr, var_data_ptr|0, offset), where a
        dictionary-encoded column passes its indices as values and a gdv_dictionary_t as var_data, and
        a string_view / binary_view column its 16-byte views and a gdv_view_buffers_t (view_buffers());
        a large_string / large_binary column passes its int64 offsets as values and its bytes as var_data;
        outputs: per expression (validity_ptr|0, values_ptr), or for a utf8 / binary output
        (validity_ptr|0, offsets_ptr, var_data_ptr, var_capacity) with room for num_slots + 1 int32
        offsets (int64 for a large_string / large_binary output); selection: (ptr, num_slots) or (ptr, max_slots, d_count_ptr): the slot count is read
        from device memory (the d_count a Filter.evaluate_device(..., sync=False) wrote on the same
        stream), no host round trip.  A utf8 / binary output whose bytes exceed its var_capacity raises
        ExecutionError here (sync=True) or from sync().  With sync=True returns each output's var_size
        (bytes written; None for fixed-width outputs)."""
        cb, _keep = self._device_batch(num_rows, columns)
        outs = (gdv_out_column_t * max(len(outputs), 1))()
        for i, o in enumerate(outputs):
            outs[i].validity, outs[i].values = (o[0] or None), (o[1] or None)
            if len(o) > 2:
                outs[i].var_data, outs[i].var_capacity = (o[2] or None), o[3]
        s = self._device_selection(selection)
        _check(lib.gdv_projector_evaluate(self._h, C.byref(cb), None if s is None else C.byref(s), outs, len(outputs),
                                          _stream_handle(stream), 0 if sync else 1))
        if sync:
            return [outs[i].var_size if len(o) > 2 else None for i, o in enumerate(outputs)]
        return None

    def output_var_size_device(self, num_rows: int, columns: Sequence[tuple], index: int, stream: int = 0,
                               selection: tuple | None = None) -> int:
        """Exact var_data bytes of utf8 / binary output `index` over a device batch (columns and selection as
        in evaluate_device; with a d_count_ptr the count is read on the device).  Runs the sizing pass and
        the scan and synchronises the stream: one round trip, for callers who want an exact buffer rather
        than an upper bound."""
        cb, _keep = self._device_batch(num_rows, columns)
        s = self._device_selection(selection)
        need = C.c_int64(0)
        _check(lib.gdv_projector_output_var_size(self._h, C.byref(cb), None if s is None else C.byref(s), index,
                                                 _stream_handle(stream), C.byref(need)))
        return need.value

    @staticmethod
    def _device_batch(num_rows: int, columns: Sequence[tuple]):
        cols = (gdv_column_t * max(len(columns), 1))()
        for i, (vld, val, var, off) in enumerate(columns):
            cols[i].validity, cols[i].values, cols[i].var_data, cols[i].offset = \
                (vld or None), (val or None), _var_ptr(var), off
        return gdv_batch_t(num_rows, len(columns), GDV_MEM_DEVICE, cols), cols

    def _device_selection(self, selection: tuple | None):
        if selection is None:
            return None
        return gdv_selection_t(selection[0], selection[1], selection[1], self._mode, GDV_MEM_DEVICE, 0,
                               selection[2] if len(selection) > 2 else None)

    def sync(self, stream: int = 0) -> None:
        _check(lib.gdv_projector_sync(self._h, _stream_handle(stream)))


# ---- Filter ------------------------------------------------------------------------------
class Filter:
    """gandiva::Filter (P/gandiva.pyx:229-280)."""

    def __init__(self, handle: int, schema: pa.Schema, condition: Condition,
                 schema_handle: _SchemaHandle):
        self._h = C.c_void_p(handle)
        self._schema = schema
        self._condition = condition
        self._schema_handle = schema_handle

    def __del__(self):
        try:
            lib.gdv_filter_release(self._h)
        except Exception:
            pass

    @property
    def llvm_ir(self) -> str:
        return _to_string(lib.gdv_filter_dump_ir, self._h)

    @property
    def kernel_info(self) -> dict:
        return _kernel_info(lib.gdv_filter_kernel_info, self._h, lib.gdv_filter_kernel_attr)

    def evaluate(self, batch: pa.RecordBatch, pool: Any = None, dtype: Any = "int32") -> SelectionVector:
        if not isinstance(batch, pa.RecordBatch):
            raise TypeError("RecordBatch expected")
        t = _ensure_type(dtype)
        if t in (pa.int16(), pa.uint16()):
            mode = GDV_SEL_UINT16
        elif t in (pa.int32(), pa.uint32()):
            mode = GDV_SEL_UINT32
        elif t in (pa.int64(), pa.uint64()):
            mode = GDV_SEL_UINT64
        else:
            raise ValueError("'dtype' of the selection vector should be one of 'int16', 'int32' and 'int64'.")
        idx = np.zeros(max(batch.num_rows, 1), dtype=_SEL_NP[mode])
        sel = gdv_selection_t(idx.ctypes.data_as(C.c_void_p), batch.num_rows, 0, mode, GDV_MEM_HOST)
        cb, keep = _batch_to_c(batch)
        _check(lib.gdv_filter_evaluate(self._h, C.byref(cb), C.byref(sel), None, 0, None))
        return SelectionVector(idx, sel.num_slots, mode)

    def evaluate_device(self, num_rows: int, columns: Sequence[tuple], out_indices: int,
                        max_slots: int, mode: str = "UINT32", stream: int = 0, d_count: int = 0,
                        sync: bool = False, index_base: int = 0) -> int:
        """Device-resident filter: writes indices at `out_indices` (device pointer).  With
        sync=False only enqueues; the count lands in `d_count` (device uint64) and is returned
        by sync()."""
        cols = (gdv_column_t * max(len(columns), 1))()
        for i, (vld, val, var, off) in enumerate(columns):
            cols[i].validity, cols[i].values, cols[i].var_data, cols[i].offset = \
                (vld or None), (val or None), _var_ptr(var), off
        cb = gdv_batch_t(num_rows, len(columns), GDV_MEM_DEVICE, cols)
        sel = gdv_selection_t(out_indices, max_slots, 0, _ensure_selection_mode(mode), GDV_MEM_DEVICE,
                              index_base)
        _check(lib.gdv_filter_evaluate(self._h, C.byref(cb), C.byref(sel), _stream_handle(stream),
                                       0 if sync else 1, C.c_void_p(d_count) if d_count else None))
        return int(sel.num_slots)

    def sync(self, stream: int = 0) -> int:
        n = C.c_int64(-1)
        _check(lib.gdv_filter_sync(self._h, _stream_handle(stream), C.byref(n)))
        return int(n.value)


# ---- Arrow C Device Data interface (include/gandiva_b200_arrow.h) -----------------------------
class ArrowSchemaC(C.Structure):
    pass


ArrowSchemaC._fields_ = [("format", C.c_char_p), ("name", C.c_char_p), ("metadata", C.c_char_p),
                         ("flags", C.c_int64), ("n_children", C.c_int64),
                         ("children", C.POINTER(C.POINTER(ArrowSchemaC))), ("dictionary", C.POINTER(ArrowSchemaC)),
                         ("release", C.c_void_p), ("private_data", C.c_void_p)]


class ArrowArrayC(C.Structure):
    pass


ArrowArrayC._fields_ = [("length", C.c_int64), ("null_count", C.c_int64), ("offset", C.c_int64),
                        ("n_buffers", C.c_int64), ("n_children", C.c_int64),
                        ("buffers", C.POINTER(C.c_void_p)), ("children", C.POINTER(C.POINTER(ArrowArrayC))),
                        ("dictionary", C.POINTER(ArrowArrayC)), ("release", C.c_void_p),
                        ("private_data", C.c_void_p)]

ARROW_DEVICE_CPU, ARROW_DEVICE_CUDA, ARROW_DEVICE_CUDA_HOST = 1, 2, 3


class ArrowDeviceArrayC(C.Structure):
    _fields_ = [("array", ArrowArrayC), ("device_id", C.c_int64), ("device_type", C.c_int32),
                ("sync_event", C.c_void_p), ("reserved", C.c_int64 * 3)]


_RELEASE_ARRAY = C.CFUNCTYPE(None, C.POINTER(ArrowArrayC))
_RELEASE_SCHEMA = C.CFUNCTYPE(None, C.POINTER(ArrowSchemaC))


class ArrowDeviceBatch:
    """A record batch imported from a struct-typed ArrowDeviceArray (zero copy; device buffers
    stay in HBM).  `address` is the address of the producer's `struct ArrowDeviceArray`, which is
    MOVED (marked released) by the import."""

    def __init__(self, address: int, schema: pa.Schema):
        self._schema_handle = _SchemaHandle(schema)
        self._h = C.c_void_p()
        _check(lib.gdv_arrow_batch_import(C.c_void_p(address), self._schema_handle._h, C.byref(self._h)))

    @classmethod
    def from_record_batch(cls, batch: pa.RecordBatch) -> "ArrowDeviceBatch":
        """Host batch through pyarrow's own exporter (device type ARROW_DEVICE_CPU)."""
        arr = ArrowDeviceArrayC()
        sch = ArrowSchemaC()
        batch._export_to_c_device(C.addressof(arr), C.addressof(sch))
        try:
            return cls(C.addressof(arr), batch.schema)
        finally:
            if sch.release:
                _RELEASE_SCHEMA(sch.release)(C.byref(sch))
            if arr.array.release:  # import failed: the array was not moved
                _RELEASE_ARRAY(arr.array.release)(C.byref(arr.array))

    @property
    def num_rows(self) -> int:
        return int(lib.gdv_arrow_batch_view(self._h).contents.num_rows)

    @property
    def mem_space(self) -> int:
        return int(lib.gdv_arrow_batch_view(self._h).contents.mem_space)

    def release(self) -> None:
        if self._h:
            lib.gdv_arrow_batch_release(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.release()
        except Exception:
            pass


class ArrowDeviceResult:
    """An ArrowDeviceArray exported by the engine (+ its ArrowSchema for projector results);
    the buffers go back to the engine's pool on release()."""

    def __init__(self):
        self.array = ArrowDeviceArrayC()
        self.schema = None

    @property
    def address(self) -> int:
        return C.addressof(self.array)

    def to_record_batch(self) -> pa.RecordBatch:
        """Host results only: hands array + schema to pyarrow's importer (which takes ownership)."""
        if self.array.device_type != ARROW_DEVICE_CPU:
            raise pa.ArrowNotImplementedError("pyarrow in this image cannot import CUDA device arrays")
        rb = pa.RecordBatch._import_from_c_device(C.addressof(self.array), C.addressof(self.schema))
        return rb

    def release(self) -> None:
        if self.array.array.release:
            _RELEASE_ARRAY(self.array.array.release)(C.byref(self.array.array))
        if self.schema is not None and self.schema.release:
            _RELEASE_SCHEMA(self.schema.release)(C.byref(self.schema))

    def __del__(self):
        try:
            self.release()
        except Exception:
            pass


def _projector_evaluate_arrow(self, batch: ArrowDeviceBatch, stream: int = 0) -> ArrowDeviceResult:
    res = ArrowDeviceResult()
    res.schema = ArrowSchemaC()
    _check(lib.gdv_projector_output_schema_arrow(self._h, C.addressof(res.schema)))
    _check(lib.gdv_projector_evaluate_arrow(self._h, batch._h, _stream_handle(stream) if stream else None,
                                            C.addressof(res.array)))
    return res


def _filter_evaluate_arrow(self, batch: ArrowDeviceBatch, mode: str = "UINT32", stream: int = 0) -> ArrowDeviceResult:
    res = ArrowDeviceResult()
    _check(lib.gdv_filter_evaluate_arrow(self._h, batch._h, _ensure_selection_mode(mode),
                                         _stream_handle(stream) if stream else None, C.addressof(res.array)))
    return res


Projector.evaluate_arrow = _projector_evaluate_arrow
Filter.evaluate_arrow = _filter_evaluate_arrow


def memcpy_dtoh(device: int, dst: np.ndarray, src_ptr: int) -> None:
    _check(lib.gdv_memcpy(device, dst.ctypes.data_as(C.c_void_p), C.c_void_p(src_ptr), dst.nbytes, 2))


def memcpy_htod(device: int, dst_ptr: int, src: np.ndarray) -> None:
    _check(lib.gdv_memcpy(device, C.c_void_p(dst_ptr), src.ctypes.data_as(C.c_void_p), src.nbytes, 1))


# ---- factories ---------------------------------------------------------------------------
def make_projector(schema: pa.Schema, children: Sequence[Expression], pool: Any = None,
                   selection_mode: str = "NONE", configuration: Configuration | None = None) -> Projector:
    """gandiva.make_projector (P/gandiva.pyx:629-673)."""
    if not isinstance(schema, pa.Schema):
        raise TypeError("Schema expected")
    children = list(children)
    for c in children:
        if not isinstance(c, Expression):
            raise TypeError("Expressions must not be None")
    if configuration is None:
        configuration = Configuration()
    if not isinstance(configuration, Configuration):
        raise TypeError("Configuration must be specified.")
    mode = _ensure_selection_mode(selection_mode)
    sh = _SchemaHandle(schema)
    arr = (C.c_void_p * max(len(children), 1))(*[c._h for c in children])
    cfg = configuration._c()
    out = C.c_void_p()
    _check(lib.gdv_projector_make(sh._h, arr, len(children), mode, C.byref(cfg), C.byref(out)))
    return Projector(out.value, schema, children, mode, sh)


def make_filter(schema: pa.Schema, condition: Condition,
                configuration: Configuration | None = None) -> Filter:
    """gandiva.make_filter (P/gandiva.pyx:676-706)."""
    if not isinstance(schema, pa.Schema):
        raise TypeError("Schema expected")
    if condition is None or not isinstance(condition, Condition):
        raise TypeError("Condition must not be None")
    if configuration is None:
        configuration = Configuration()
    if not isinstance(configuration, Configuration):
        raise TypeError("Configuration must be specified.")
    sh = _SchemaHandle(schema)
    cfg = configuration._c()
    out = C.c_void_p()
    _check(lib.gdv_filter_make(sh._h, condition._h, C.byref(cfg), C.byref(out)))
    return Filter(out.value, schema, condition, sh)


class FunctionSignature:
    """gandiva::FunctionSignature (P/gandiva.pyx:709-741)."""

    def __init__(self, name: str, ret: pa.DataType, params: list):
        self._name, self._ret, self._params = name, ret, params

    def return_type(self) -> pa.DataType:
        return self._ret

    def param_types(self) -> list:
        return list(self._params)

    def name(self) -> str:
        return self._name

    def __repr__(self) -> str:
        return "FunctionSignature(%s)" % self

    def __str__(self) -> str:
        return "%s %s(%s)" % (self._ret, self._name, ", ".join(str(p) for p in self._params))


_NULL_MODES = {"if_null": 0, "never": 1, "internal": 2}


class FunctionRegistry:
    """Functions the caller adds to the engine as CUDA text (include/gandiva_b200.h, "user-defined
    functions", has the calling convention).  `Configuration(function_registry=reg)` makes a Projector or
    Filter resolve names against the built-ins first and `reg` second; the fuser writes each user function
    a kernel calls into that kernel.  Functions can be registered until the registry is first used by
    make_projector / make_filter."""

    def __init__(self):
        h = C.c_void_p()
        _check(lib.gdv_function_registry_create(C.byref(h)))
        self._h = h.value

    def __del__(self):
        if getattr(self, "_h", None) and lib is not None:
            lib.gdv_function_registry_release(self._h)
            self._h = None

    def register(self, name: str, param_types: list, return_type: pa.DataType, body: str, *,
                 null_mode: str = "if_null", can_raise: bool = False, prelude: str = "") -> None:
        """`body`: the statements of the device function; parameters are a0, a1, ... (plus v0, v1, ... with
        null_mode "never" / "internal", `out_valid` with "internal", `ctx` with can_raise)."""
        if null_mode not in _NULL_MODES:
            raise ValueError("null_mode must be one of %s, not %r" % (sorted(_NULL_MODES), null_mode))
        params = (gdv_type_t * max(1, len(param_types)))(*[_to_c_type(t) for t in param_types])
        d = gdv_function_def_t(name.encode(), params, len(param_types), _to_c_type(return_type),
                               _NULL_MODES[null_mode], int(bool(can_raise)), body.encode(), prelude.encode())
        _check(lib.gdv_function_registry_add(self._h, C.byref(d)))

    def signatures(self) -> list:
        """The signatures of this registry only (get_registered_function_signatures() lists the built-ins)."""
        out = []
        for i in range(lib.gdv_function_registry_signatures(self._h)):
            name = C.c_char_p()
            ret = gdv_type_t()
            params = (gdv_type_t * 16)()
            n = C.c_int32()
            _check(lib.gdv_function_registry_get(self._h, i, C.byref(name), C.byref(ret), params, 16, C.byref(n)))
            out.append(FunctionSignature(name.value.decode(), _from_c_type(ret),
                                         [_from_c_type(params[k]) for k in range(min(n.value, 16))]))
        return out


def generate_lineitem(device: int, kind: int, seed: int, first_row: int, num_rows: int,
                      values_ptr: int, validity_ptr: int = 0, null_permille: int = 0,
                      stream: int = 0) -> None:
    """Synthetic TPC-H lineitem column written straight into device memory (harness helper;
    column kinds in csrc/device/static_kernels.cu).  `stream` as in evaluate_device."""
    _check(lib.gdv_generate_lineitem(device, kind, seed, first_row, num_rows, values_ptr,
                                     validity_ptr or None, null_permille, _stream_handle(stream)))


def get_registered_function_signatures() -> list:
    out = []
    for i in range(lib.gdv_registry_size()):
        name = C.c_char_p()
        ret = gdv_type_t()
        params = (gdv_type_t * 16)()
        n = C.c_int32()
        _check(lib.gdv_registry_get(i, C.byref(name), C.byref(ret), params, 16, C.byref(n)))
        out.append(FunctionSignature(name.value.decode(), _from_c_type(ret),
                                     [_from_c_type(params[k]) for k in range(n.value)]))
    return out
