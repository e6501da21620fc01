#include "gdv_node.h"

#include <cstdio>
#include <sstream>

namespace gdv {

int DataType::width() const {
  if (large) return 8;
  switch (id) {
    case GDV_TYPE_BOOL: return 0;
    case GDV_TYPE_UINT8: case GDV_TYPE_INT8: return 1;
    case GDV_TYPE_UINT16: case GDV_TYPE_INT16: return 2;
    case GDV_TYPE_UINT32: case GDV_TYPE_INT32: case GDV_TYPE_FLOAT:
    case GDV_TYPE_DATE32: case GDV_TYPE_TIME32: return 4;
    case GDV_TYPE_UINT64: case GDV_TYPE_INT64: case GDV_TYPE_DOUBLE:
    case GDV_TYPE_DATE64: case GDV_TYPE_TIMESTAMP: case GDV_TYPE_TIME64: return 8;
    case GDV_TYPE_DECIMAL128: return 16;
    case GDV_TYPE_STRING: case GDV_TYPE_BINARY: return 4;
    default: return 0;
  }
}

static const char* unit_name(int u) {
  switch (u) {
    case 0: return "s";
    case 1: return "ms";
    case 2: return "us";
    default: return "ns";
  }
}

std::string DataType::ToString() const {
  if (view) return id == GDV_TYPE_BINARY ? "binary_view" : "string_view";
  if (large) return id == GDV_TYPE_BINARY ? "large_binary" : "large_string";
  if (index != 0)
    return "dictionary<values=" + value_type().ToString() + ", indices=" + DataType(index).ToString() +
           ", ordered=" + (ordered ? "1" : "0") + ">";
  switch (id) {
    case GDV_TYPE_NA: return "null";
    case GDV_TYPE_BOOL: return "bool";
    case GDV_TYPE_UINT8: return "uint8";
    case GDV_TYPE_INT8: return "int8";
    case GDV_TYPE_UINT16: return "uint16";
    case GDV_TYPE_INT16: return "int16";
    case GDV_TYPE_UINT32: return "uint32";
    case GDV_TYPE_INT32: return "int32";
    case GDV_TYPE_UINT64: return "uint64";
    case GDV_TYPE_INT64: return "int64";
    case GDV_TYPE_FLOAT: return "float";
    case GDV_TYPE_DOUBLE: return "double";
    case GDV_TYPE_STRING: return "string";
    case GDV_TYPE_BINARY: return "binary";
    case GDV_TYPE_DATE32: return "date32[day]";
    case GDV_TYPE_DATE64: return "date64[ms]";
    case GDV_TYPE_TIMESTAMP: return std::string("timestamp[") + unit_name(precision) + "]";
    case GDV_TYPE_TIME32: return std::string("time32[") + unit_name(precision) + "]";
    case GDV_TYPE_TIME64: return std::string("time64[") + unit_name(precision) + "]";
    case GDV_TYPE_DECIMAL128:
      return "decimal128(" + std::to_string(precision) + ", " + std::to_string(scale) + ")";
    default: return "type(" + std::to_string(id) + ")";
  }
}

const char* DataType::ctype() const {
  switch (id) {
    case GDV_TYPE_BOOL: return "bool";
    case GDV_TYPE_UINT8: return "u8";
    case GDV_TYPE_INT8: return "i8";
    case GDV_TYPE_UINT16: return "u16";
    case GDV_TYPE_INT16: return "i16";
    case GDV_TYPE_UINT32: return "u32";
    case GDV_TYPE_INT32: case GDV_TYPE_DATE32: case GDV_TYPE_TIME32: return "i32";
    case GDV_TYPE_UINT64: return "u64";
    case GDV_TYPE_INT64: case GDV_TYPE_DATE64: case GDV_TYPE_TIMESTAMP: case GDV_TYPE_TIME64:
      return "i64";
    case GDV_TYPE_FLOAT: return "f32";
    case GDV_TYPE_DOUBLE: return "f64";
    case GDV_TYPE_DECIMAL128: return "i128";
    case GDV_TYPE_STRING: case GDV_TYPE_BINARY: return "gdv_str";
    default: return "void";
  }
}

const char* DataType::fn_suffix() const {
  switch (id) {
    case GDV_TYPE_BOOL: return "boolean";
    case GDV_TYPE_UINT8: return "uint8";
    case GDV_TYPE_INT8: return "int8";
    case GDV_TYPE_UINT16: return "uint16";
    case GDV_TYPE_INT16: return "int16";
    case GDV_TYPE_UINT32: return "uint32";
    case GDV_TYPE_INT32: return "int32";
    case GDV_TYPE_UINT64: return "uint64";
    case GDV_TYPE_INT64: return "int64";
    case GDV_TYPE_FLOAT: return "float32";
    case GDV_TYPE_DOUBLE: return "float64";
    case GDV_TYPE_STRING: return "utf8";
    case GDV_TYPE_BINARY: return "binary";
    case GDV_TYPE_DATE32: return "date32";
    case GDV_TYPE_DATE64: return "date64";
    // milliseconds keep the plain names; the other units name theirs (extractYear_timestamp_us, ...)
    case GDV_TYPE_TIMESTAMP:
      return precision == 0 ? "timestamp_s" : precision == 2 ? "timestamp_us" : precision == 3 ? "timestamp_ns" : "timestamp";
    case GDV_TYPE_TIME32: return precision == 0 ? "time32_s" : "time32";
    case GDV_TYPE_TIME64: return precision == 3 ? "time64_ns" : "time64_us";
    case GDV_TYPE_DECIMAL128: return "decimal128";
    default: return "unknown";
  }
}

std::string FieldNode::ToString() const {
  return "(" + return_type().ToString() + ") " + name_;
}

LiteralNode::LiteralNode(DataType t, const void* value, int64_t len, bool is_null)
    : Node(NodeKind::kLiteral, t), is_null_(is_null) {
  std::memset(raw_, 0, sizeof(raw_));
  if (is_null || value == nullptr) return;
  if (t.is_varlen()) {
    bytes_.assign(static_cast<const char*>(value), static_cast<size_t>(len));
  } else {
    int w = t.is_bool() ? 1 : t.width();
    std::memcpy(raw_, value, static_cast<size_t>(w));
  }
}

// Signed 128-bit little-endian -> decimal digits.
static std::string Int128ToString(const uint8_t* raw) {
  unsigned __int128 u;
  std::memcpy(&u, raw, 16);
  __int128 v = static_cast<__int128>(u);
  bool neg = v < 0;
  unsigned __int128 m = neg ? (~u + 1) : u;
  if (m == 0) return "0";
  std::string s;
  while (m != 0) {
    s.push_back(static_cast<char>('0' + static_cast<int>(m % 10)));
    m /= 10;
  }
  if (neg) s.push_back('-');
  return std::string(s.rbegin(), s.rend());
}

std::string LiteralNode::ToString() const {
  std::stringstream ss;
  const DataType& t = return_type();
  ss << "(const " << t.ToString() << ") ";
  if (is_null_) {
    ss << "null";
    return ss.str();
  }
  switch (t.id) {
    case GDV_TYPE_BOOL: ss << (raw_[0] ? 1 : 0); break;
    case GDV_TYPE_UINT8: ss << static_cast<unsigned>(as<uint8_t>()); break;
    case GDV_TYPE_INT8: ss << static_cast<int>(as<int8_t>()); break;
    case GDV_TYPE_UINT16: ss << as<uint16_t>(); break;
    case GDV_TYPE_INT16: ss << as<int16_t>(); break;
    case GDV_TYPE_UINT32: ss << as<uint32_t>(); break;
    case GDV_TYPE_INT32: case GDV_TYPE_DATE32: case GDV_TYPE_TIME32: ss << as<int32_t>(); break;
    case GDV_TYPE_UINT64: ss << as<uint64_t>(); break;
    case GDV_TYPE_INT64: case GDV_TYPE_DATE64: case GDV_TYPE_TIMESTAMP: case GDV_TYPE_TIME64:
      ss << as<int64_t>();
      break;
    case GDV_TYPE_FLOAT: {
      char hex[32];
      std::snprintf(hex, sizeof(hex), "%08X", as<uint32_t>());
      ss << as<float>() << " raw(" << hex << ")";
      break;
    }
    case GDV_TYPE_DOUBLE: {
      char hex[32];
      std::snprintf(hex, sizeof(hex), "%016llX", static_cast<unsigned long long>(as<uint64_t>()));
      ss << as<double>() << " raw(" << hex << ")";
      break;
    }
    case GDV_TYPE_DECIMAL128:
      ss << Int128ToString(raw_) << "," << t.precision << "," << t.scale;
      break;
    case GDV_TYPE_STRING: case GDV_TYPE_BINARY: ss << "'" << bytes_ << "'"; break;
    default: ss << "?"; break;
  }
  return ss.str();
}

std::string FunctionNode::ToString() const {
  std::stringstream ss;
  ss << return_type().ToString() << " " << name_ << "(";
  bool first = true;
  for (const auto& c : children_) {
    if (!first) ss << ", ";
    ss << c->ToString();
    first = false;
  }
  ss << ")";
  return ss.str();
}

std::string IfNode::ToString() const {
  return "if (" + cond_->ToString() + ") { " + then_->ToString() + " } else { " +
         else_->ToString() + " }";
}

std::string BooleanNode::ToString() const {
  std::stringstream ss;
  bool first = true;
  for (const auto& c : children_) {
    if (!first) ss << (op_ == kAnd ? " && " : " || ");
    ss << c->ToString();
    first = false;
  }
  return ss.str();
}

std::string InNode::ToString() const {
  std::stringstream ss;
  ss << child_->ToString() << " IN (";
  bool first = true;
  if (value_type_.is_varlen()) {
    for (const auto& s : strs_) {
      if (!first) ss << ", ";
      ss << s;
      first = false;
    }
  } else {
    for (auto v : ints_) {
      if (!first) ss << ", ";
      ss << v;
      first = false;
    }
  }
  ss << ")";
  return ss.str();
}

NodeVector Children(const Node& node) {
  switch (node.kind()) {
    case NodeKind::kFunction: return static_cast<const FunctionNode&>(node).children();
    case NodeKind::kIf: {
      const auto& n = static_cast<const IfNode&>(node);
      return {n.condition(), n.then_node(), n.else_node()};
    }
    case NodeKind::kBoolean: return static_cast<const BooleanNode&>(node).children();
    case NodeKind::kIn: return {static_cast<const InNode&>(node).child()};
    default: return {};
  }
}

NodePtr WithChildren(const NodePtr& node, NodeVector children) {
  if (children == Children(*node)) return node;
  switch (node->kind()) {
    case NodeKind::kFunction: {
      const auto& fn = static_cast<const FunctionNode&>(*node);
      return std::make_shared<FunctionNode>(fn.name(), std::move(children), fn.return_type());
    }
    case NodeKind::kIf:
      return std::make_shared<IfNode>(children[0], children[1], children[2], node->return_type());
    case NodeKind::kBoolean:
      return std::make_shared<BooleanNode>(static_cast<const BooleanNode&>(*node).op(), std::move(children));
    case NodeKind::kIn: {
      const auto& n = static_cast<const InNode&>(*node);
      return std::make_shared<InNode>(children[0], n.value_type(), n.ints(), n.strs());
    }
    default: return node;
  }
}

}  // namespace gdv
