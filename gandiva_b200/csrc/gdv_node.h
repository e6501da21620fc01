// Expression tree: the nodes TreeExprBuilder makes (P/includes/libgandiva.pxd:110-212).
// ToString() formats are the ones the descendant's tests pin
// (P/tests/test_gandiva.py:376-393).
#pragma once
#include <cstdint>
#include <cstring>
#include <memory>
#include <string>
#include <vector>

#include "gdv_types.h"

namespace gdv {

enum class NodeKind { kField, kLiteral, kFunction, kIf, kBoolean, kIn };

class Node;
using NodePtr = std::shared_ptr<Node>;
using NodeVector = std::vector<NodePtr>;

class Node {
 public:
  Node(NodeKind k, DataType t) : kind_(k), type_(t) {}
  virtual ~Node() = default;
  NodeKind kind() const { return kind_; }
  const DataType& return_type() const { return type_; }
  virtual std::string ToString() const = 0;

 private:
  NodeKind kind_;
  DataType type_;
};

class FieldNode : public Node {
 public:
  FieldNode(std::string name, DataType t) : Node(NodeKind::kField, t), name_(std::move(name)) {}
  const std::string& name() const { return name_; }
  std::string ToString() const override;

 private:
  std::string name_;
};

// A literal holds up to 16 bytes of fixed-width storage (little-endian, the Arrow
// in-buffer representation) or a byte string.
class LiteralNode : public Node {
 public:
  LiteralNode(DataType t, const void* value, int64_t len, bool is_null);
  bool is_null() const { return is_null_; }
  const uint8_t* raw() const { return raw_; }
  const std::string& bytes() const { return bytes_; }
  template <typename T>
  T as() const {
    T v;
    std::memcpy(&v, raw_, sizeof(T));
    return v;
  }
  std::string ToString() const override;

 private:
  bool is_null_;
  uint8_t raw_[16];
  std::string bytes_;
};

class FunctionNode : public Node {
 public:
  FunctionNode(std::string name, NodeVector children, DataType ret)
      : Node(NodeKind::kFunction, ret), name_(std::move(name)), children_(std::move(children)) {}
  const std::string& name() const { return name_; }
  const NodeVector& children() const { return children_; }
  std::string ToString() const override;

 private:
  std::string name_;
  NodeVector children_;
};

class IfNode : public Node {
 public:
  IfNode(NodePtr c, NodePtr t, NodePtr e, DataType ret)
      : Node(NodeKind::kIf, ret), cond_(std::move(c)), then_(std::move(t)), else_(std::move(e)) {}
  const NodePtr& condition() const { return cond_; }
  const NodePtr& then_node() const { return then_; }
  const NodePtr& else_node() const { return else_; }
  std::string ToString() const override;

 private:
  NodePtr cond_, then_, else_;
};

class BooleanNode : public Node {
 public:
  enum Op { kAnd, kOr };
  BooleanNode(Op op, NodeVector children)
      : Node(NodeKind::kBoolean, boolean()), op_(op), children_(std::move(children)) {}
  Op op() const { return op_; }
  const NodeVector& children() const { return children_; }
  std::string ToString() const override;

 private:
  Op op_;
  NodeVector children_;
};

// IN (v1, v2, ...) over a fixed-width or string/binary child.
class InNode : public Node {
 public:
  InNode(NodePtr child, DataType value_type, std::vector<int64_t> ints,
         std::vector<std::string> strs)
      : Node(NodeKind::kIn, boolean()),
        child_(std::move(child)),
        value_type_(value_type),
        ints_(std::move(ints)),
        strs_(std::move(strs)) {}
  const NodePtr& child() const { return child_; }
  const DataType& value_type() const { return value_type_; }
  const std::vector<int64_t>& ints() const { return ints_; }
  const std::vector<std::string>& strs() const { return strs_; }
  std::string ToString() const override;

 private:
  NodePtr child_;
  DataType value_type_;
  std::vector<int64_t> ints_;  // all fixed-width integer-like values, sign-extended
  std::vector<std::string> strs_;
};

// The children of a node in evaluation order (an If's condition, then, else); none for fields and
// literals.  Walks that treat every kind of node alike go through these two instead of a switch.
NodeVector Children(const Node& node);
// The same node over `children` (as many as Children(*node) returns).  Returns `node` itself when no
// child pointer changed.
NodePtr WithChildren(const NodePtr& node, NodeVector children);

struct Field {
  std::string name;
  DataType type;
};

class Schema {
 public:
  explicit Schema(std::vector<Field> f) : fields_(std::move(f)) {}
  const std::vector<Field>& fields() const { return fields_; }
  int index_of(const std::string& name) const {
    for (size_t i = 0; i < fields_.size(); ++i)
      if (fields_[i].name == name) return static_cast<int>(i);
    return -1;
  }

 private:
  std::vector<Field> fields_;
};
using SchemaPtr = std::shared_ptr<Schema>;

class Expression {
 public:
  Expression(NodePtr root, Field result) : root_(std::move(root)), result_(std::move(result)) {}
  const NodePtr& root() const { return root_; }
  const Field& result() const { return result_; }
  std::string ToString() const { return root_->ToString(); }

 private:
  NodePtr root_;
  Field result_;
};
using ExpressionPtr = std::shared_ptr<Expression>;

// A Condition is an Expression whose result is the boolean field "cond".
class Condition : public Expression {
 public:
  explicit Condition(NodePtr root) : Expression(std::move(root), Field{"cond", boolean()}) {}
};
using ConditionPtr = std::shared_ptr<Condition>;

}  // namespace gdv
