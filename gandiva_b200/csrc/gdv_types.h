// Data types of the expression engine.  Type ids are arrow::Type::type values
// (P/include/arrow/type_fwd.h:330-473) so the C++ drop-in layer converts with a cast.
#pragma once
#include <cstdint>
#include <string>

#include "gandiva_b200.h"

namespace gdv {

// A dictionary-encoded column (arrow::DictionaryType) is its value type plus the index type:
// `id` is the value type's id, `index` the signed integer id of the indices (0 = plain column).
// Everything that reads values -- function resolution, if/else and IN type checks -- sees the
// value type; operator== compares value types, same() also the encoding.  At the C-ABI it is
// GDV_TYPE_DICTIONARY (include/gandiva_b200.h).
// A string_view / binary_view column (arrow::StringViewType / BinaryViewType) works the same way:
// `id` is GDV_TYPE_STRING / BINARY and `view` is set, so everything that reads values sees utf8 /
// binary and only same() and the kernels' row loaders see the 16-byte views.  is_varlen() holds
// for all three layouts; HasByteRun (gdv_codegen.cc) is what "contiguous offsets + bytes" means.
// A large_string / large_binary column (arrow::LargeStringType / LargeBinaryType) is utf8 / binary
// with `large` set: the same contiguous bytes behind int64 offsets.  Unlike the two encodings above
// it may also be an expression's result type (an output with int64 offsets).
struct DataType {
  int32_t id = GDV_TYPE_NA;
  int32_t precision = 0;  // decimal precision, or time unit for timestamp/time
  int32_t scale = 0;
  int32_t index = 0;      // dictionary columns: GDV_TYPE_INT8..INT64 (or what the caller sent)
  bool ordered = false;   // dictionary columns: DictionaryType::ordered
  bool view = false;      // string_view / binary_view columns
  bool large = false;     // large_string / large_binary columns and results (int64 offsets)

  DataType() = default;
  DataType(int32_t i, int32_t p = 0, int32_t s = 0) : id(i), precision(p), scale(s) {}
  explicit DataType(const gdv_type_t& t) : id(t.id), precision(t.precision), scale(t.scale) {
    if (t.id == GDV_TYPE_DICTIONARY) {
      id = t.scale;
      index = t.precision & 0xff;
      ordered = (t.precision & GDV_DICT_ORDERED) != 0;
      precision = scale = 0;
    } else if (t.id == GDV_TYPE_STRING_VIEW || t.id == GDV_TYPE_BINARY_VIEW) {
      id = t.id == GDV_TYPE_STRING_VIEW ? GDV_TYPE_STRING : GDV_TYPE_BINARY;
      view = true;
      precision = scale = 0;
    } else if (t.id == GDV_TYPE_LARGE_STRING || t.id == GDV_TYPE_LARGE_BINARY) {
      id = t.id == GDV_TYPE_LARGE_STRING ? GDV_TYPE_STRING : GDV_TYPE_BINARY;
      large = true;
      precision = scale = 0;
    }
  }
  gdv_type_t c() const {
    if (view) return gdv_type_t{id == GDV_TYPE_BINARY ? GDV_TYPE_BINARY_VIEW : GDV_TYPE_STRING_VIEW, 0, 0};
    if (large) return gdv_type_t{id == GDV_TYPE_BINARY ? GDV_TYPE_LARGE_BINARY : GDV_TYPE_LARGE_STRING, 0, 0};
    if (index != 0) return gdv_type_t{GDV_TYPE_DICTIONARY, index | (ordered ? GDV_DICT_ORDERED : 0), id};
    return gdv_type_t{id, precision, scale};
  }
  bool is_dict() const { return index != 0; }
  bool is_view() const { return view; }
  bool is_large() const { return large; }
  // The type of the values (the dictionary's type for a dictionary column, utf8 / binary for a view
  // or a large column).
  DataType value_type() const { return DataType(id, precision, scale); }
  bool same(const DataType& o) const {
    return *this == o && index == o.index && ordered == o.ordered && view == o.view && large == o.large;
  }

  bool operator==(const DataType& o) const {
    if (id != o.id) return false;
    if (id == GDV_TYPE_DECIMAL128) return precision == o.precision && scale == o.scale;
    if (id == GDV_TYPE_TIMESTAMP || id == GDV_TYPE_TIME32 || id == GDV_TYPE_TIME64)
      return precision == o.precision;
    return true;
  }
  bool operator!=(const DataType& o) const { return !(*this == o); }

  bool is_varlen() const { return id == GDV_TYPE_STRING || id == GDV_TYPE_BINARY; }
  bool is_bool() const { return id == GDV_TYPE_BOOL; }
  bool is_decimal() const { return id == GDV_TYPE_DECIMAL128; }
  bool is_float() const { return id == GDV_TYPE_FLOAT || id == GDV_TYPE_DOUBLE; }
  bool is_integer() const { return id >= GDV_TYPE_UINT8 && id <= GDV_TYPE_INT64; }
  bool is_signed_integer() const {
    return id == GDV_TYPE_INT8 || id == GDV_TYPE_INT16 || id == GDV_TYPE_INT32 ||
           id == GDV_TYPE_INT64;
  }

  // Width in bytes of one value in the Arrow values buffer (0 for bool = bit-packed,
  // 4 for the offsets buffer of utf8/binary, 8 for large_string / large_binary).
  int width() const;
  // arrow::DataType::ToString() spelling ("int32", "double", "decimal128(12, 2)", ...).
  std::string ToString() const;
  // C type used for a value of this type inside generated device code.
  const char* ctype() const;
  // Suffix used in precompiled function names ("int32", "float64", "utf8", ...), the
  // naming scheme of the reference's function library (add_int32_int32, ...).
  const char* fn_suffix() const;
};

inline DataType boolean() { return DataType(GDV_TYPE_BOOL); }
inline DataType int32() { return DataType(GDV_TYPE_INT32); }
inline DataType int64() { return DataType(GDV_TYPE_INT64); }
inline DataType float32() { return DataType(GDV_TYPE_FLOAT); }
inline DataType float64() { return DataType(GDV_TYPE_DOUBLE); }
inline DataType utf8() { return DataType(GDV_TYPE_STRING); }
inline DataType binary() { return DataType(GDV_TYPE_BINARY); }
inline DataType date32() { return DataType(GDV_TYPE_DATE32); }
inline DataType date64() { return DataType(GDV_TYPE_DATE64); }
inline DataType timestamp_ms() { return DataType(GDV_TYPE_TIMESTAMP, 1); }
inline DataType time32_ms() { return DataType(GDV_TYPE_TIME32, 1); }
inline DataType decimal128(int p, int s) { return DataType(GDV_TYPE_DECIMAL128, p, s); }

}  // namespace gdv
