#include "gdv_codegen.h"
#include "gdv_datefmt.h"
#include "gdv_regex.h"

#include <algorithm>
#include <cctype>
#include <cstdio>
#include <map>
#include <sstream>

#include "gdv_registry.h"

namespace gdv {

// ======================================================================================
// Validation (replaces the reference's expression validator, SURVEY.md §2 / §8a row a3)
// ======================================================================================
namespace {

Status VErr(const std::string& m) { return Status::Make(GDV_EXPRESSION_VALIDATION_ERROR, m); }

// Dictionary-encoded columns are inputs only: results are plain utf8 / binary, as Gandiva's are.
Status DictionaryResult(const std::string& what) {
  return Status::Make(GDV_NOT_IMPLEMENTED, "'" + what + "' has a dictionary result type: dictionary-encoded "
                                           "outputs are not supported (results are plain utf8 / binary)");
}

// string_view / binary_view columns are inputs only, like dictionary-encoded ones.
Status ViewResult(const std::string& what, const DataType& t) {
  return Status::Make(GDV_NOT_IMPLEMENTED, "'" + what + "' has a " + t.ToString() + " result type: " + t.ToString() +
                                           " outputs are not supported (results are plain utf8 / binary)");
}

// large_string / large_binary is a layout of a column or of an expression's result field; a node that
// computes a value yields plain utf8 / binary (the output's offsets are widened when it is written).
Status LargeResult(const std::string& what, const DataType& t) {
  return Status::Make(GDV_NOT_IMPLEMENTED, "'" + what + "' has a " + t.ToString() + " return type: only a field or an "
                                           "expression's result may be " + t.ToString() + " (nodes yield utf8 / binary)");
}

bool IsSupportedType(const DataType& t) {
  switch (t.id) {
    case GDV_TYPE_BOOL: case GDV_TYPE_UINT8: case GDV_TYPE_INT8: case GDV_TYPE_UINT16:
    case GDV_TYPE_INT16: case GDV_TYPE_UINT32: case GDV_TYPE_INT32: case GDV_TYPE_UINT64:
    case GDV_TYPE_INT64: case GDV_TYPE_FLOAT: case GDV_TYPE_DOUBLE: case GDV_TYPE_STRING:
    case GDV_TYPE_BINARY: case GDV_TYPE_DATE32: case GDV_TYPE_DATE64: case GDV_TYPE_DECIMAL128:
      return true;
    // every Arrow unit: timestamp[s|ms|us|ns], time32[s|ms], time64[us|ns]
    case GDV_TYPE_TIMESTAMP: return t.precision >= 0 && t.precision <= 3;
    case GDV_TYPE_TIME32: return t.precision == 0 || t.precision == 1;
    case GDV_TYPE_TIME64: return t.precision == 2 || t.precision == 3;
    default: return false;
  }
}

// True when the string this node yields carries the initcap case map: initcap itself, or a function that
// hands its argument through with the start of the view untouched.
static bool EndsInInitcap(const Node& node) {
  if (node.kind() == NodeKind::kIf) {
    const auto& n = static_cast<const IfNode&>(node);
    return EndsInInitcap(*n.then_node()) || EndsInInitcap(*n.else_node());
  }
  if (node.kind() != NodeKind::kFunction) return false;
  const auto& fn = static_cast<const FunctionNode&>(node);
  if (fn.name() == "initcap") return true;
  if (fn.name() == "rtrim" || fn.name() == "nvl")
    for (const auto& c : fn.children())
      if (c->return_type().id == GDV_TYPE_STRING && EndsInInitcap(*c)) return true;
  return false;
}

Status ValidateNode(const Schema& schema, const Node& node) {
  switch (node.kind()) {
    case NodeKind::kField: {
      const auto& f = static_cast<const FieldNode&>(node);
      const int idx = schema.index_of(f.name());
      if (idx < 0) return VErr("Field " + f.name() + " not in schema");
      if (!schema.fields()[idx].type.same(f.return_type()))
        return VErr("Field definition in schema " + schema.fields()[idx].name + ": " +
                    schema.fields()[idx].type.ToString() +
                    " different from field in expression " + f.ToString());
      if (f.return_type().is_dict()) {
        const DataType& t = f.return_type();
        if (!t.is_varlen() || !DataType(t.index).is_signed_integer())
          return Status::Make(GDV_NOT_IMPLEMENTED,
                              "Field " + f.name() + " has unsupported data type " + t.ToString() +
                                  ": dictionary columns need utf8 or binary values and int8, int16, "
                                  "int32 or int64 indices");
        return Status::OK();
      }
      if (!IsSupportedType(f.return_type()))
        return VErr("Field " + f.name() + " has unsupported data type " +
                    f.return_type().ToString());
      return Status::OK();
    }
    case NodeKind::kLiteral: {
      if (!IsSupportedType(node.return_type()) || node.return_type().is_dict() || node.return_type().is_view())
        return VErr("Value " + node.ToString() + " has unsupported data type " +
                    node.return_type().ToString());
      if (node.return_type().is_large()) return LargeResult("literal", node.return_type());
      return Status::OK();
    }
    case NodeKind::kFunction: {
      const auto& fn = static_cast<const FunctionNode&>(node);
      if (fn.return_type().is_dict()) return DictionaryResult(fn.name());
      if (fn.return_type().is_view()) return ViewResult(fn.name(), fn.return_type());
      if (fn.return_type().is_large()) return LargeResult(fn.name(), fn.return_type());
      std::vector<DataType> params;
      for (const auto& c : fn.children()) {
        Status s = ValidateNode(schema, *c);
        if (!s.ok()) return s;
        params.push_back(c->return_type());
      }
      const FunctionDef* def = LookupFunction(fn.name(), params, fn.return_type());
      if (def == nullptr) {
        std::string sig = fn.return_type().ToString() + " " + fn.name() + "(";
        for (size_t i = 0; i < params.size(); ++i)
          sig += (i ? ", " : "") + params[i].ToString();
        sig += ")";
        return VErr("Function " + sig + " not supported yet. ");
      }
      if (def->ret.id != fn.return_type().id ||
          (def->ret.id != GDV_TYPE_DECIMAL128 && def->ret != fn.return_type()))
        return VErr("Function " + def->signature() + " not supported yet: return type " +
                    fn.return_type().ToString() + " does not match");
      // initcap is a lazy case map that looks one byte back (csrc/device/gdv_device_lib.cuh, gdv_ch): a
      // function that then moves the START of the view (substr, ltrim, right, ...) or re-orders its bytes
      // would make the first byte of its result depend on a byte it no longer has.
      if ((def->ret.id == GDV_TYPE_STRING || def->ret.id == GDV_TYPE_BINARY) && fn.name() != "upper" &&
          fn.name() != "lower" && fn.name() != "initcap" && fn.name() != "rtrim" && fn.name() != "nvl" &&
          fn.name() != "concat" && fn.name() != "concatOperator") {
        for (const auto& c : fn.children())
          if (c->return_type().id == GDV_TYPE_STRING && EndsInInitcap(*c))
            return Status::Make(GDV_NOT_IMPLEMENTED, "'" + fn.name() + "' over the result of initcap is not supported: "
                                                      "apply initcap last (initcap(" + fn.name() + "(...)))");
      }
      if (def->flags & kDateFormat) {
        for (size_t i = 1; i < fn.children().size(); ++i) {
          const Node& c = *fn.children()[i];
          if (c.kind() != NodeKind::kLiteral || static_cast<const LiteralNode&>(c).is_null())
            return VErr(i == 1 ? "'to_date' function requires a literal as the second parameter"
                               : "The third parameter of 'to_date' (suppress errors) must be a literal 0 or 1");
        }
        std::vector<uint8_t> prog;
        std::string why;
        const int rc = CompileDateFormat(static_cast<const LiteralNode&>(*fn.children()[1]).bytes(), &prog, &why);
        if (rc == 1) return VErr(why);
        if (rc != 0) return Status::Make(GDV_NOT_IMPLEMENTED, why);
      }
      if (def->flags & kRegexHolder) {
        const Node& c = *fn.children()[1];
        if (c.kind() != NodeKind::kLiteral || static_cast<const LiteralNode&>(c).is_null())
          return VErr("'" + fn.name() + "' function requires a literal as the second parameter");
        RegexProgram prog;
        std::string why;
        const int rc = CompileRegex(static_cast<const LiteralNode&>(c).bytes(), &prog, &why);
        if (rc == 1) return VErr(why);
        if (rc != 0) return Status::Make(GDV_NOT_IMPLEMENTED, why);
      }
      if (def->flags & kLikeHolder) {
        for (size_t i = 1; i < fn.children().size(); ++i) {
          const Node& c = *fn.children()[i];
          if (c.kind() != NodeKind::kLiteral || static_cast<const LiteralNode&>(c).is_null())
            return VErr("'like' function requires a literal as the second parameter");
        }
        if (fn.children().size() == 3 &&
            static_cast<const LiteralNode&>(*fn.children()[2]).bytes().size() != 1)
          return VErr("The length of escape char in 'like' function must be 1");
        if (fn.children().size() == 3 && (fn.name() == "like" || fn.name() == "ilike")) {
          // the reference's pattern translation accepts the escape character only in front of
          // '_', '%' or itself, and never as the last character of the pattern
          const std::string& pat = static_cast<const LiteralNode&>(*fn.children()[1]).bytes();
          const char esc = static_cast<const LiteralNode&>(*fn.children()[2]).bytes()[0];
          for (size_t i = 0; i < pat.size(); ++i) {
            if (pat[i] != esc) continue;
            if (i + 1 == pat.size()) return VErr("Unexpected escape char at the end of pattern " + pat);
            const char nx = pat[++i];
            if (nx != '_' && nx != '%' && nx != esc)
              return VErr("Invalid escape sequence in pattern " + pat + " at offset " + std::to_string(i));
          }
        }
      }
      return Status::OK();
    }
    case NodeKind::kIf: {
      const auto& n = static_cast<const IfNode&>(node);
      if (n.return_type().is_dict()) return DictionaryResult("if");
      if (n.return_type().is_view()) return ViewResult("if", n.return_type());
      if (n.return_type().is_large()) return LargeResult("if", n.return_type());
      for (const NodePtr* c : {&n.condition(), &n.then_node(), &n.else_node()}) {
        Status s = ValidateNode(schema, **c);
        if (!s.ok()) return s;
      }
      if (n.condition()->return_type() != boolean())
        return VErr("condition must be of boolean type, found type " +
                    n.condition()->return_type().ToString());
      if (n.then_node()->return_type() != n.return_type())
        return VErr("return type of if " + n.return_type().ToString() + " and then " +
                    n.then_node()->return_type().ToString() + " not matching.");
      if (n.else_node()->return_type() != n.return_type())
        return VErr("return type of if " + n.return_type().ToString() + " and else " +
                    n.else_node()->return_type().ToString() + " not matching.");
      return Status::OK();
    }
    case NodeKind::kBoolean: {
      const auto& n = static_cast<const BooleanNode&>(node);
      if (n.children().size() < 2)
        return VErr("Boolean expression has " + std::to_string(n.children().size()) +
                    " children, expected at least two");
      for (const auto& c : n.children()) {
        Status s = ValidateNode(schema, *c);
        if (!s.ok()) return s;
        if (c->return_type() != boolean())
          return VErr("Boolean expression has a child with return type " +
                      c->return_type().ToString() + ", expected return type boolean");
      }
      return Status::OK();
    }
    case NodeKind::kIn: {
      const auto& n = static_cast<const InNode&>(node);
      Status s = ValidateNode(schema, *n.child());
      if (!s.ok()) return s;
      if (n.child()->return_type() != n.value_type())
        return VErr("Evaluation expression for IN clause returns " +
                    n.child()->return_type().ToString() + " values are of type" +
                    n.value_type().ToString());
      const int id = n.value_type().id;
      const bool ok = n.value_type().is_varlen() || id == GDV_TYPE_INT32 ||
                      id == GDV_TYPE_INT64 || id == GDV_TYPE_DATE32 || id == GDV_TYPE_DATE64 ||
                      id == GDV_TYPE_TIMESTAMP || id == GDV_TYPE_TIME32 || id == GDV_TYPE_TIME64 ||
                      id == GDV_TYPE_FLOAT || id == GDV_TYPE_DOUBLE;
      if (!ok) return VErr("IN expression over " + n.value_type().ToString() + " not supported");
      return Status::OK();
    }
  }
  return VErr("unknown node kind");
}

}  // namespace

Status ValidateExpression(const Schema& schema, const Expression& expr) {
  if (expr.root() == nullptr) return VErr("Expression has no root node");
  if (expr.result().type.is_dict()) return DictionaryResult(expr.result().name);
  if (expr.result().type.is_view()) return ViewResult(expr.result().name, expr.result().type);
  Status s = ValidateNode(schema, *expr.root());
  if (!s.ok()) return s;
  if (expr.root()->return_type() != expr.result().type)
    return VErr("Return type of root node " + expr.root()->return_type().ToString() +
                " does not match that of expression " + expr.result().type.ToString());
  return Status::OK();
}

// ======================================================================================
// Args layout
// ======================================================================================
ArgsLayout::ArgsLayout(int n_inputs, int n_outputs, bool dictionary, bool views)
    : ni(std::max(n_inputs, 1)), no(std::max(n_outputs, 1)), dict(dictionary), view(views) {
  size_t o = 80;
  off_in_val = o; o += 8u * ni;
  off_in_vld = o; o += 8u * ni;
  off_in_var = o; o += 8u * ni;
  off_out_val = o; o += 8u * no;
  off_out_vld = o; o += 8u * no;
  off_out_var = o; o += 8u * no;
  off_in_vsh = o; o += 4u * ni;
  off_in_dsh = o; o += 4u * ni;
  if (dict) {
    o = (o + 7u) & ~size_t(7);
    off_in_dof = o; o += 8u * ni;
    off_in_dvl = o; o += 8u * ni;
    off_in_dln = o; o += 8u * ni;
    off_in_dvs = o; o += 4u * ni;
  }
  if (view) {
    o = (o + 7u) & ~size_t(7);
    off_in_vbf = o; o += 8u * ni;
    off_in_vsz = o; o += 8u * ni;
    off_in_vbn = o; o += 8u * ni;
  }
  size = (o + 7u) & ~size_t(7);
}

bool HasDictionary(const std::vector<ColumnSlot>& slots) {
  for (const auto& s : slots)
    if (s.type.is_dict()) return true;
  return false;
}

bool HasView(const std::vector<ColumnSlot>& slots) {
  for (const auto& s : slots)
    if (s.type.is_view()) return true;
  return false;
}

// ======================================================================================
// Body generation
// ======================================================================================
namespace {

struct Val {
  std::string v;   // C expression (usually a local variable name)
  std::string ok;  // C expression of type bool; "true"/"false" when statically known
  DataType type;
  // concat() results are ropes: the C expressions (type gdv_str) of the pieces, in order.  Only
  // a string output, another concat or an if/else may consume one; `v` is unused then.
  std::vector<std::string> parts;
};

// Text that is safe inside a `//` comment of the generated source: bytes outside printable ASCII
// (a binary literal's 0xff made NVRTC drop the rest of the translation unit) and backslashes (a
// trailing one would splice the next line into the comment) are written as \\xNN.
std::string CommentSafe(const std::string& s) {
  std::string o;
  for (unsigned char c : s) {
    if (c < 0x20 || c >= 0x7f || c == '\\') {
      char b[8];
      std::snprintf(b, sizeof(b), "<%02x>", static_cast<unsigned>(c));
      o += b;
    } else {
      o.push_back(static_cast<char>(c));
    }
  }
  return o;
}

std::string HexLit(uint64_t bits) {
  char b[40];
  std::snprintf(b, sizeof(b), "0x%016llxull", static_cast<unsigned long long>(bits));
  return b;
}

// One '%'-delimited middle segment of a LIKE pattern that the cooperative scan of column `slot`
// looks for: occurrences are recorded as (id << 24 | stage byte offset) in the warp's hit list.
struct CoopSeg {
  int slot = 0;
  unsigned xf = 0;     // case map of the view the pattern is matched against
  std::string bytes;
  int id = 0;          // unique per slot
  int like = 0;        // which LIKE node of the slot the segment belongs to
  bool is_key = false; // the segment of its LIKE the scan looks for (rarest digram)
  int digram = 0;      // key: index of the first byte of the adjacent pair the scan tests
};
constexpr int kHitCap = 64;  // hits per warp and group; more -> the group falls back per lane
constexpr int kKeyAnchorCap = 256;  // key-driven filter: anchors a warp queues between two drains

// Plan of the key-driven string filter (EmitKeyFilter): the condition holds only in rows whose
// string column `slot` contains `key` (a literal segment of a LIKE / is_substr / starts_with /
// ends_with / equal conjunct on the condition's AND spine), compared through the ASCII case map
// `xf` of the view chain.
struct KeyPlan {
  int slot = -1;
  unsigned xf = 0u;
  std::string key;
};

class BodyGen {
 public:
  BodyGen(const Schema& schema, std::vector<ColumnSlot>* slots, bool nullable, bool coop, bool view_sc = true)
      : schema_(schema), slots_(slots), nullable_(nullable), coop_(coop), view_sc_(view_sc) {}

  // Device-scope definitions the body needs; GDV_NS = call sites that write text into scratch slots.
  std::string globals() const {
    std::string g = n_scratch_ > 0 ? "#define GDV_NS " + std::to_string(n_scratch_) + "\n" + globals_ : globals_;
    if (!repl_sites_.empty()) {
      // replace() call sites: one switch each for the output length and the copy
      std::string len = "__device__ __forceinline__ i32 gdv_repl_len(const gdv_str& v) {\n  switch ((v.xf >> 12) & 0xffu) {\n";
      std::string cpy = "__device__ __forceinline__ void gdv_repl_copy(u8* dst, const gdv_str& v) {\n  switch ((v.xf >> 12) & 0xffu) {\n";
      for (size_t i = 0; i < repl_sites_.size(); ++i) {
        const ReplSite& r = repl_sites_[i];
        len += "    case " + std::to_string(i) + ": return gdv_replace_len(v, " + r.from + ", " + std::to_string(r.fl) +
               ", " + std::to_string(r.tl) + ");\n";
        cpy += "    case " + std::to_string(i) + ": gdv_replace_copy(dst, v, " + r.from + ", " + std::to_string(r.fl) +
               ", " + r.to + ", " + std::to_string(r.tl) + "); return;\n";
      }
      g += len + "  }\n  return v.len;\n}\n" + cpy + "  }\n}\n";
    }
    return g;
  }
  bool has_replace() const { return !repl_sites_.empty(); }
  int scratch_sites() const { return n_scratch_; }
  // Declaration of the thread-private scratch slots of a kernel that evaluates R rows per group.
  std::string ScratchDecl(int R) const {
    if (n_scratch_ == 0) return std::string();
    return "  u8 gdv_scr[" + std::to_string(R) + " * GDV_NS * GDV_SCRATCH_SLOT];  // text written by castVARCHAR(number)\n";
  }
  const std::vector<CoopSeg>& coop_segs() const { return coop_segs_; }
  bool uses_ctx() const { return uses_ctx_; }
  const std::string& error() const { return error_; }
  int view_shortcuts() const { return view_shortcuts_; }

  // Emit the statements that evaluate `node` for the row held in slot arrays at [k].
  Val Gen(const Node& node, std::string* out, int indent) {
    switch (node.kind()) {
      case NodeKind::kField: return GenField(static_cast<const FieldNode&>(node));
      case NodeKind::kLiteral: return GenLiteral(static_cast<const LiteralNode&>(node));
      case NodeKind::kFunction:
        return GenFunction(static_cast<const FunctionNode&>(node), out, indent);
      case NodeKind::kIf: return GenIf(static_cast<const IfNode&>(node), out, indent);
      case NodeKind::kBoolean:
        return GenBoolean(static_cast<const BooleanNode&>(node), out, indent);
      case NodeKind::kIn: return GenIn(static_cast<const InNode&>(node), out, indent);
    }
    return Val{"0", "false", node.return_type()};
  }

  // "valid and true" of a boolean expression, for consumers that need nothing else (a Filter
  // keeps a row iff its condition is valid and true).  Under SQL three-valued logic
  //   truth(a AND b) = truth(a) && truth(b),   truth(a OR b) = truth(a) || truth(b),
  // so the Kleene bookkeeping (decided / all-valid flags per child) of GenBoolean is not needed
  // on this path: a nullable Q6 predicate drops from ~6 to ~2 instructions per comparison.
  // Children that can raise keep the general, lazily evaluated form.
  Val GenTruth(const Node& node, std::string* out, int indent) {
    if (node.kind() == NodeKind::kBoolean && !CanFail(node)) {
      const auto& n = static_cast<const BooleanNode&>(node);
      const bool is_and = n.op() == BooleanNode::kAnd;
      std::string e;
      for (const auto& c : n.children()) {
        const Val cv = GenTruth(*c, out, indent);
        e += (e.empty() ? "" : (is_and ? " && " : " || ")) + std::string("(") + cv.v + ")";
      }
      const std::string v = NewVar("v");
      *out += Ind(indent) + "const bool " + v + " = " + e + ";\n";
      return Val{v, "true", boolean(), {}};
    }
    const Val r = Gen(node, out, indent);
    if (r.ok == "true") return r;
    const std::string v = NewVar("v");
    *out += Ind(indent) + "const bool " + v + " = (" + r.ok + ") && (" + r.v + ");\n";
    return Val{v, "true", boolean(), {}};
  }

  int SlotFor(const FieldNode& f) {
    const int idx = schema_.index_of(f.name());
    for (size_t j = 0; j < slots_->size(); ++j)
      if ((*slots_)[j].schema_index == idx) return static_cast<int>(j);
    slots_->push_back(ColumnSlot{idx, f.return_type()});
    return static_cast<int>(slots_->size()) - 1;
  }

  // Finds, on the AND spine of a filter condition, a conjunct that can only be true in rows whose
  // string column contains a literal of >= 3 bytes (a '%'-free segment of a LIKE pattern, or the
  // literal of is_substr / starts_with / ends_with / equal) seen through a view chain: the filter is
  // then driven by the occurrences of that literal in the column's bytes (EmitKeyFilter).  The
  // longest literal wins (>= 7 bytes allows the aligned-word test), ties go to the rarer digrams.
  bool PlanKey(const Node& cond, KeyPlan* plan) {
    std::vector<const Node*> conj;
    std::vector<const Node*> todo = {&cond};
    while (!todo.empty()) {
      const Node* n = todo.back();
      todo.pop_back();
      if (n->kind() == NodeKind::kBoolean &&
          static_cast<const BooleanNode*>(n)->op() == BooleanNode::kAnd) {
        for (const auto& c : static_cast<const BooleanNode*>(n)->children()) todo.push_back(c.get());
      } else {
        conj.push_back(n);
      }
    }
    double best = -1.0;
    auto offer = [&](const std::string& sg, int slot, unsigned xf) {
      if (sg.size() < 3 || sg.size() > 64) return;
      double rare = 1e300;
      for (unsigned char c : sg)
        if ((xf == 1u && c >= 'a' && c <= 'z') || (xf == 2u && c >= 'A' && c <= 'Z')) return;  // can never match
      for (size_t i = 0; i + 1 < sg.size(); ++i)
        rare = std::min(rare, DigramScore(static_cast<unsigned char>(sg[i]), static_cast<unsigned char>(sg[i + 1]), xf));
      const double score = static_cast<double>(std::min<size_t>(sg.size(), 16)) * 100.0 - std::min(rare, 50.0);
      if (score > best) {
        best = score;
        plan->slot = slot;
        plan->xf = xf;
        plan->key = sg;
      }
    };
    for (const Node* n : conj) {
      if (n->kind() != NodeKind::kFunction) continue;
      const auto& fn = *static_cast<const FunctionNode*>(n);
      if (fn.children().size() < 2 || fn.children()[1]->kind() != NodeKind::kLiteral) continue;
      int slot = -1;
      unsigned xf = 0u;
      if (fn.name() == "is_substr" || fn.name() == "starts_with" || fn.name() == "ends_with" ||
          fn.name() == "equal" || fn.name() == "eq" || fn.name() == "same") {
        // s contains / starts with / ends with / equals a literal: the literal itself is the key
        // (comparisons see the view through its case map, like LIKE does)
        const auto& lit = static_cast<const LiteralNode&>(*fn.children()[1]);
        if (lit.is_null() || !lit.return_type().is_varlen()) continue;
        if (!ViewChain(*fn.children()[0], &slot, &xf)) continue;
        offer(lit.bytes(), slot, xf);
        continue;
      }
      if (fn.name() != "like") continue;
      const auto& pat = static_cast<const LiteralNode&>(*fn.children()[1]);
      if (pat.is_null()) continue;
      const bool has_esc = fn.children().size() == 3;
      const char esc = has_esc ? static_cast<const LiteralNode&>(*fn.children()[2]).bytes()[0] : 0;
      const std::vector<unsigned> toks = LikeTokens(pat.bytes(), has_esc, esc);
      if (!ViewChain(*fn.children()[0], &slot, &xf)) continue;
      // literal runs between wildcards ('%' and '_' both end a run)
      std::string cur;
      for (unsigned t : toks) {
        if ((t >> 8) == 0u) {
          cur.push_back(static_cast<char>(t & 0xffu));
        } else {
          offer(cur, slot, xf);
          cur.clear();
        }
      }
      offer(cur, slot, xf);
    }
    return plan->slot >= 0;
  }

  // Schema columns whose NULL makes `node` not-true (truth context: a Filter keeps a row iff its
  // condition is valid and true).  AND needs every child true (union), OR one of them
  // (intersection); everything else is true only if valid, and a function with the default null
  // rule is null as soon as one argument is.
  void TruthStrict(const Node& node, std::vector<int>* cols) const {
    if (node.kind() == NodeKind::kBoolean && !CanFail(node)) {
      const auto& n = static_cast<const BooleanNode&>(node);
      const bool is_and = n.op() == BooleanNode::kAnd;
      bool first = true;
      for (const auto& c : n.children()) {
        std::vector<int> cc;
        TruthStrict(*c, &cc);
        if (is_and) {
          for (int x : cc)
            if (std::find(cols->begin(), cols->end(), x) == cols->end()) cols->push_back(x);
        } else if (first) {
          *cols = cc;
        } else {
          std::vector<int> both;
          for (int x : *cols)
            if (std::find(cc.begin(), cc.end(), x) != cc.end()) both.push_back(x);
          *cols = both;
        }
        first = false;
      }
      return;
    }
    ValueStrict(node, cols);
  }
  void ValueStrict(const Node& node, std::vector<int>* cols) const {
    auto add = [&](int x) {
      if (std::find(cols->begin(), cols->end(), x) == cols->end()) cols->push_back(x);
    };
    switch (node.kind()) {
      case NodeKind::kField: add(schema_.index_of(static_cast<const FieldNode&>(node).name())); return;
      case NodeKind::kIn: ValueStrict(*static_cast<const InNode&>(node).child(), cols); return;
      case NodeKind::kFunction: {
        const auto& fn = static_cast<const FunctionNode&>(node);
        std::vector<DataType> params;
        for (const auto& c : fn.children()) params.push_back(c->return_type());
        const FunctionDef* def = LookupFunction(fn.name(), params, fn.return_type());
        if (def == nullptr || def->nulls != NullMode::kIfNull || (def->flags & (kConcat | kVirtual)) || fn.name() == "nvl")
          return;
        for (const auto& c : fn.children()) ValueStrict(*c, cols);
        return;
      }
      default: return;  // literals, if/else, Kleene and/or as values: no column is strict
    }
  }

  static double PairScore(unsigned char a, unsigned char b, unsigned xf) { return DigramScore(a, b, xf); }

  // castVARCHAR(x, n) raises on n < 0 ("Output buffer length can't be negative"), locate(sub, s, start)
  // on start < 1 ("Start position must be greater than 0"), as the reference's functions do.  Returns
  // the index of the argument a can-fail helper must check, or -1 (literals that can never raise).
  static int ArgGuard(const FunctionNode& fn) {
    int arg = -1;
    int64_t least = 0;
    if (fn.name() == "castVARCHAR" && fn.children().size() == 2) arg = 1;
    if ((fn.name() == "locate" || fn.name() == "position") && fn.children().size() == 3) {
      arg = 2;
      least = 1;
    }
    if (arg < 0) return -1;
    const Node& c = *fn.children()[static_cast<size_t>(arg)];
    if (c.kind() == NodeKind::kLiteral) {
      const auto& lit = static_cast<const LiteralNode&>(c);
      if (lit.is_null()) return -1;  // a null argument makes the row null: nothing is called
      const int64_t v = c.return_type().id == GDV_TYPE_INT32 ? static_cast<int64_t>(lit.as<int32_t>()) : lit.as<int64_t>();
      if (v >= least) return -1;
    }
    return arg;
  }

  static bool CanFail(const Node& node) {
    if (node.kind() == NodeKind::kFunction) {
      const auto& fn = static_cast<const FunctionNode&>(node);
      std::vector<DataType> params;
      for (const auto& c : fn.children()) params.push_back(c->return_type());
      const FunctionDef* def = LookupFunction(fn.name(), params, fn.return_type());
      if (def != nullptr && (def->flags & kCanFail)) return true;
      if (ArgGuard(fn) >= 0) return true;
    }
    for (const auto& c : Children(node))
      if (CanFail(*c)) return true;
    return false;
  }

 private:
  std::string NewVar(const char* prefix) { return std::string(prefix) + std::to_string(next_id_++); }
  static std::string Ind(int n) { return std::string(static_cast<size_t>(n) * 2, ' '); }

  static std::string AndOk(const std::vector<std::string>& oks) {
    std::string r;
    for (const auto& o : oks) {
      if (o == "false") return "false";
      if (o == "true") continue;
      r += (r.empty() ? "" : " && ") + o;
    }
    return r.empty() ? "true" : r;
  }

  static std::string ZeroOf(const DataType& t) {
    if (t.is_varlen()) return "gdv_make_str(nullptr, 0)";
    if (t.is_bool()) return "false";
    return std::string("(") + t.ctype() + ")0";
  }

  Val GenField(const FieldNode& f) {
    const int j = SlotFor(f);
    return Val{"f" + std::to_string(j) + "[k]",
               nullable_ ? "k" + std::to_string(j) + "[k]" : std::string("true"), f.return_type().value_type()};
  }

  std::string BytesArray(const std::string& bytes, const char* prefix) {
    const std::string name = NewVar(prefix);
    std::string s = "__device__ const u8 " + name + "[" +
                    std::to_string(std::max<size_t>(bytes.size(), 1)) + "] = {";
    if (bytes.empty()) s += "0";
    for (size_t i = 0; i < bytes.size(); ++i) {
      if (i) s += ",";
      s += std::to_string(static_cast<unsigned>(static_cast<uint8_t>(bytes[i])));
    }
    s += "};\n";
    globals_ += s;
    return name;
  }

  Val GenLiteral(const LiteralNode& lit) {
    const DataType& t = lit.return_type();
    if (lit.is_null()) return Val{ZeroOf(t), "false", t};
    std::string v;
    switch (t.id) {
      case GDV_TYPE_BOOL: v = lit.raw()[0] ? "true" : "false"; break;
      case GDV_TYPE_INT8: v = "(i8)" + std::to_string(static_cast<int>(lit.as<int8_t>())); break;
      case GDV_TYPE_INT16: v = "(i16)" + std::to_string(lit.as<int16_t>()); break;
      case GDV_TYPE_UINT8:
        v = "(u8)" + std::to_string(static_cast<unsigned>(lit.as<uint8_t>()));
        break;
      case GDV_TYPE_UINT16: v = "(u16)" + std::to_string(lit.as<uint16_t>()); break;
      case GDV_TYPE_UINT32: v = std::to_string(lit.as<uint32_t>()) + "u"; break;
      case GDV_TYPE_INT32: case GDV_TYPE_DATE32: case GDV_TYPE_TIME32:
        v = "(i32)" + HexLit(static_cast<uint64_t>(lit.as<uint32_t>()));
        break;
      case GDV_TYPE_UINT64: v = HexLit(lit.as<uint64_t>()); break;
      case GDV_TYPE_INT64: case GDV_TYPE_DATE64: case GDV_TYPE_TIMESTAMP: case GDV_TYPE_TIME64:
        v = "(i64)" + HexLit(lit.as<uint64_t>());
        break;
      case GDV_TYPE_FLOAT:
        v = "__uint_as_float(" + std::to_string(lit.as<uint32_t>()) + "u)";
        break;
      case GDV_TYPE_DOUBLE: v = "__longlong_as_double((i64)" + HexLit(lit.as<uint64_t>()) + ")"; break;
      case GDV_TYPE_DECIMAL128: {
        uint64_t lo, hi;
        std::memcpy(&lo, lit.raw(), 8);
        std::memcpy(&hi, lit.raw() + 8, 8);
        v = "(i128)(((u128)" + HexLit(hi) + " << 64) | (u128)" + HexLit(lo) + ")";
        break;
      }
      case GDV_TYPE_STRING: case GDV_TYPE_BINARY: {
        const std::string arr = BytesArray(lit.bytes(), "gdv_lit_");
        v = "gdv_make_str(" + arr + ", " + std::to_string(lit.bytes().size()) + ")";
        break;
      }
      default: v = "0"; break;
    }
    return Val{v, "true", t};
  }

  // Tokenise a SQL LIKE pattern: '%' any run, '_' one glyph, escape char quotes the next byte.
  // Token = (kind << 8) | byte with kind 0 literal, 1 '_', 2 '%'.
  static std::vector<unsigned> LikeTokens(const std::string& pat, bool has_escape, char esc) {
    std::vector<unsigned> toks;
    for (size_t i = 0; i < pat.size(); ++i) {
      const unsigned char c = static_cast<unsigned char>(pat[i]);
      if (has_escape && pat[i] == esc && i + 1 < pat.size()) {
        toks.push_back(static_cast<unsigned char>(pat[++i]));
      } else if (c == '%') {
        if (toks.empty() || (toks.back() >> 8) != 2u) toks.push_back(2u << 8);
      } else if (c == '_') {
        toks.push_back(1u << 8);
      } else {
        toks.push_back(c);
      }
    }
    return toks;
  }

  // Generic matcher: tokens in a __device__ table, interpreted by gdv_like_match().
  std::string LikePatternTable(const std::vector<unsigned>& toks) {
    const std::string name = NewVar("gdv_pat_");
    std::string s = "__device__ const u16 " + name + "[" +
                    std::to_string(std::max<size_t>(toks.size(), 1)) + "] = {";
    if (toks.empty()) s += "0";
    for (size_t i = 0; i < toks.size(); ++i) s += (i ? "," : "") + std::to_string(toks[i]);
    s += "};\n";
    globals_ += s;
    return name;
  }

  // Patterns made of literal runs and '%' only (no '_') compile to straight code: the pattern
  // bytes become immediates, the first segment is anchored at the start unless the pattern
  // begins with '%', the last at the end unless it ends with '%', the ones in between are
  // found leftmost-first.  Returns the name of the emitted device function.
  static void LikeSegments(const std::vector<unsigned>& toks, std::vector<std::string>* segs,
                           bool* lead_any, bool* trail_any) {
    std::string cur;
    *lead_any = !toks.empty() && (toks.front() >> 8) == 2u;
    *trail_any = !toks.empty() && (toks.back() >> 8) == 2u;
    for (unsigned t : toks) {
      if ((t >> 8) == 2u) {
        if (!cur.empty()) segs->push_back(cur);
        cur.clear();
      } else {
        cur.push_back(static_cast<char>(t & 0xffu));
      }
    }
    if (!cur.empty()) segs->push_back(cur);
  }

  // A "view chain": upper/lower/substr/trim applied (in any order) to a string column.  The
  // result is a sub-range of the row's stored bytes under a statically known ASCII case map,
  // which is what the cooperative LIKE scan needs.
  bool ViewChain(const Node& node, int* slot, unsigned* xf) {
    if (node.kind() == NodeKind::kField) {
      // a dictionary or view column's rows are not one contiguous run of bytes
      const DataType& t = node.return_type();
      if (!t.is_varlen() || t.is_dict() || t.is_view()) return false;
      *slot = SlotFor(static_cast<const FieldNode&>(node));
      *xf = 0u;
      return true;
    }
    if (node.kind() != NodeKind::kFunction) return false;
    const auto& fn = static_cast<const FunctionNode&>(node);
    const std::string& n = fn.name();
    const bool is_case = n == "upper" || n == "lower";
    const bool is_view = n == "substr" || n == "substring" || n == "ltrim" || n == "rtrim" ||
                         n == "btrim" || n == "trim" || n == "left" || n == "right";
    if (!is_case && !is_view) return false;
    if (fn.children().empty() || !fn.children()[0]->return_type().is_varlen()) return false;
    if (!ViewChain(*fn.children()[0], slot, xf)) return false;
    if (n == "upper") *xf = 1u;
    if (n == "lower") *xf = 2u;
    return true;
  }

  // Static byte-rarity score (English text; lower = rarer) used to pick the byte of a segment
  // the cooperative scan looks for.
  static double ByteScore(unsigned char c, unsigned xf) {
    static const double letter[26] = {8.2, 1.5, 2.8, 4.3, 12.7, 2.2, 2.0, 6.1, 7.0, 0.15, 0.77,
                                      4.0, 2.4, 6.7, 7.5, 1.9, 0.095, 6.0, 6.3, 9.1, 2.8, 0.98,
                                      2.4, 0.15, 2.0, 0.074};
    if (c >= 'a' && c <= 'z') return letter[c - 'a'];
    if (c >= 'A' && c <= 'Z') return xf != 0u ? letter[c - 'A'] : letter[c - 'A'] * 0.05;
    if (c == ' ') return 15.0;
    if (c >= 0x80) return 0.3;
    if (c >= '0' && c <= '9') return 1.0;
    return 0.5;
  }

  // Frequency estimate (percent) of the adjacent pair (a, b): independent letters, floored by a
  // table of the digrams English text is known to repeat (or that are perfectly correlated,
  // like "qu"), so that the scan does not pick a pair that looks rare but is not.
  static double DigramScore(unsigned char a, unsigned char b, unsigned xf) {
    double sc = ByteScore(a, xf) * ByteScore(b, xf) / 100.0;
    auto low = [&](unsigned char c) -> char {
      if (c >= 'A' && c <= 'Z') return static_cast<char>(c + 32);
      return static_cast<char>(c);
    };
    const bool letters = ((a | 0x20) >= 'a' && (a | 0x20) <= 'z') && ((b | 0x20) >= 'a' && (b | 0x20) <= 'z');
    const bool lower_ctx = xf != 0u || ((a >= 'a' && a <= 'z') && (b >= 'a' && b <= 'z'));
    if (letters && lower_ctx) {
      static const struct { const char* d; double f; } known[] = {
          {"th", 3.56}, {"he", 3.07}, {"in", 2.43}, {"er", 2.05}, {"an", 1.99}, {"re", 1.85}, {"on", 1.76},
          {"at", 1.49}, {"en", 1.45}, {"nd", 1.35}, {"ti", 1.34}, {"es", 1.34}, {"or", 1.28}, {"te", 1.20},
          {"of", 1.17}, {"ed", 1.17}, {"is", 1.13}, {"it", 1.12}, {"al", 1.09}, {"ar", 1.07}, {"st", 1.05},
          {"to", 1.05}, {"nt", 1.04}, {"ng", 0.95}, {"se", 0.93}, {"ha", 0.93}, {"as", 0.87}, {"ou", 0.87},
          {"io", 0.83}, {"le", 0.83}, {"ve", 0.83}, {"co", 0.79}, {"me", 0.79}, {"de", 0.76}, {"hi", 0.76},
          {"ri", 0.73}, {"ro", 0.73}, {"ic", 0.70}, {"ne", 0.69}, {"ea", 0.69}, {"ra", 0.69}, {"ce", 0.65},
          {"li", 0.62}, {"ch", 0.60}, {"ll", 0.58}, {"be", 0.58}, {"ma", 0.57}, {"si", 0.55}, {"om", 0.55},
          {"ur", 0.54}, {"qu", 0.095}, {"ly", 0.43}, {"ck", 0.12}, {"ss", 0.41}, {"ee", 0.38}, {"oo", 0.21}};
      for (const auto& kd : known)
        if (kd.d[0] == low(a) && kd.d[1] == low(b)) sc = std::max(sc, kd.f);
    }
    return sc;
  }


  // LIKE over a view chain of column `slot` whose '%'-separated middle segments are all >= 3
  // bytes: the warp scans the staged bytes of a whole group for segment occurrences once
  // (EmitGroup, "cooperative scan") and leaves the verified hits in shared memory; this emits the
  // per-row function that chains those hits leftmost-first inside the row's view instead of
  // walking the row's bytes.  Returns "" when the pattern does not qualify.
  std::string LikeFromHits(const std::vector<unsigned>& toks, int slot, unsigned xf) {
    std::vector<std::string> segs;
    bool lead_any, trail_any;
    LikeSegments(toks, &segs, &lead_any, &trail_any);
    size_t first_mid = lead_any ? 0 : 1;
    size_t last_mid = trail_any ? segs.size() : (segs.empty() ? 0 : segs.size() - 1);
    if (segs.empty() || first_mid >= last_mid) return "";
    size_t total = 0;
    for (const auto& sg : segs) {
      total += sg.size();
      for (unsigned char c : sg) {
        // a literal the case map can never produce: the per-lane matcher already answers false
        if ((xf == 1u && c >= 'a' && c <= 'z') || (xf == 2u && c >= 'A' && c <= 'Z')) return "";
      }
    }
    for (size_t k = first_mid; k < last_mid; ++k)
      if (segs[k].size() < 3) return "";
    int n_slot_segs = 0;
    for (const auto& cs : coop_segs_) n_slot_segs += cs.slot == slot ? 1 : 0;
    if (n_slot_segs + static_cast<int>(last_mid - first_mid) > 8) return "";

    const std::string name = NewVar("gdv_likeh_");
    std::string f = "__device__ __forceinline__ bool " + name +
                    "(const gdv_str& s, const u8* stage, const u32* hits, u32 nh) {\n";
    f += "  if (s.len < " + std::to_string(total) + ") return false;\n";
    f += "  i32 cur = (i32)(s.p - stage);\n";
    f += "  i32 lim = cur + s.len;\n";
    auto match_at = [&](const std::string& seg, const std::string& at) {
      std::string e;
      for (size_t i = 0; i < seg.size(); ++i)
        e += (i ? " && " : "") + std::string("gdv_ch_eq(s, ") + at + " + " + std::to_string(i) + ", " +
             std::to_string(static_cast<unsigned>(static_cast<unsigned char>(seg[i]))) + "u)";
      return e;
    };
    if (!lead_any) {
      f += "  if (!(" + match_at(segs[0], "0") + ")) return false;\n";
      f += "  cur += " + std::to_string(segs[0].size()) + ";\n";
    }
    if (!trail_any) {
      const std::string L = std::to_string(segs.back().size());
      f += "  if (!(" + match_at(segs.back(), "(s.len - " + L + ")") + ")) return false;\n";
      f += "  lim -= " + L + ";\n";
    }
    // ids are unique per slot; the key of this LIKE is the middle segment with the rarest digram
    int like_idx = 0;
    for (const auto& cs : coop_segs_)
      if (cs.slot == slot) like_idx = std::max(like_idx, cs.like + 1);
    size_t key_k = first_mid;
    int key_d = 0;
    double key_score = 1e300;
    for (size_t k = first_mid; k < last_mid; ++k) {
      if (segs[k].size() > 32) continue;  // lane i verifies byte i of the key
      for (size_t i = 0; i + 1 < segs[k].size(); ++i) {
        const double sc = DigramScore(static_cast<unsigned char>(segs[k][i]),
                                      static_cast<unsigned char>(segs[k][i + 1]), xf);
        if (sc < key_score) {
          key_score = sc;
          key_k = k;
          key_d = static_cast<int>(i);
        }
      }
    }
    if (key_score == 1e300) return "";
    for (size_t k = first_mid; k < last_mid; ++k) {
      CoopSeg cs;
      cs.slot = slot;
      cs.xf = xf;
      cs.bytes = segs[k];
      cs.id = n_slot_segs++;
      cs.like = like_idx;
      cs.is_key = k == key_k;
      cs.digram = cs.is_key ? key_d : 0;
      coop_segs_.push_back(cs);
      const std::string L = std::to_string(segs[k].size());
      f += "  {\n    i32 best = 0x7fffffff;\n";
      f += "    for (u32 h = 0u; h < nh; ++h) {\n";
      f += "      const u32 e = hits[h];\n";
      f += "      const i32 p = (i32)(e & 0xffffffu);\n";
      f += "      if ((e >> 24) == " + std::to_string(cs.id) + "u && p >= cur && p + " + L +
           " <= lim && p < best) best = p;\n";
      f += "    }\n";
      f += "    if (best == 0x7fffffff) return false;\n";
      f += "    cur = best + " + L + ";\n  }\n";
    }
    f += "  return true;\n}\n";
    globals_ += f;
    return name;
  }

  std::string LikeSpecialised(const std::vector<unsigned>& toks) {
    std::vector<std::string> segs;
    bool lead_any, trail_any;
    LikeSegments(toks, &segs, &lead_any, &trail_any);
    const std::string name = NewVar("gdv_like_");
    std::string f = "__device__ __forceinline__ bool " + name + "(const gdv_str& s) {\n";
    f += "  const i32 n = s.len;\n";
    auto match_at = [&](const std::string& seg, const std::string& at) {
      std::string e;
      for (size_t i = 0; i < seg.size(); ++i)
        e += (i ? " && " : "") + std::string("gdv_ch_eq(s, ") + at + " + " + std::to_string(i) + ", " +
             std::to_string(static_cast<unsigned>(static_cast<unsigned char>(seg[i]))) + "u)";
      return e;
    };
    size_t total = 0;
    for (const auto& sg : segs) total += sg.size();
    if (segs.empty()) {
      // "" matches only the empty string; "%" (or "%%") matches everything
      f += toks.empty() ? "  return n == 0;\n}\n" : "  return true;\n}\n";
      globals_ += f;
      return name;
    }
    if (!lead_any && !trail_any && segs.size() == 1) {
      f += "  return n == " + std::to_string(segs[0].size()) + " && " + match_at(segs[0], "0") + ";\n}\n";
      globals_ += f;
      return name;
    }
    f += "  if (n < " + std::to_string(total) + ") return false;\n";
    f += "  i32 pos = 0;\n";
    size_t first_mid = 0, last_mid = segs.size();
    if (!lead_any) {
      f += "  if (!(" + match_at(segs[0], "0") + ")) return false;\n";
      f += "  pos = " + std::to_string(segs[0].size()) + ";\n";
      first_mid = 1;
    }
    if (!trail_any) last_mid = segs.size() - 1;
    for (size_t k = first_mid; k < last_mid; ++k) {
      const std::string L = std::to_string(segs[k].size());
      // Byte-at-a-time leftmost search (the fallback of the cooperative scan).
      f += "  {\n    bool found = false;\n";
      f += "    for (; pos + " + L + " <= n; ++pos) {\n";
      f += "      if (" + match_at(segs[k], "pos") + ") { found = true; break; }\n";
      f += "    }\n    if (!found) return false;\n    pos += " + L + ";\n  }\n";
    }
    if (!trail_any) {
      const std::string L = std::to_string(segs.back().size());
      f += "  if (n - " + L + " < pos) return false;\n";
      f += "  return " + match_at(segs.back(), "(n - " + L + ")") + ";\n";
    } else {
      f += "  return true;\n";
    }
    f += "}\n";
    globals_ += f;
    return name;
  }

  // A user function's prelude and definition go into the kernel's file scope at its first call site, each once
  // (two functions of one registry may share a prelude).
  void EmitUserFunction(const FunctionDef& def) {
    auto once = [&](const std::string& text) {
      if (text.empty() || std::find(user_text_.begin(), user_text_.end(), text) != user_text_.end()) return;
      user_text_.push_back(text);
      globals_ += text;
    };
    if (def.flags & kCanFail) once(kUserRaiseHelper);
    once(def.prelude);
    once(def.source);
  }

  Val GenFunction(const FunctionNode& fn, std::string* out, int indent) {
    std::vector<DataType> ptypes;
    for (const auto& c : fn.children()) ptypes.push_back(c->return_type());
    const FunctionDef* def = LookupFunction(fn.name(), ptypes, fn.return_type());
    const DataType& rt = fn.return_type();

    if (def->is_user()) EmitUserFunction(*def);
    else if (Val r; ViewShortcut(fn, out, indent, &r)) return r;

    if (def->flags & kDateFormat) {
      Val s = Gen(*fn.children()[0], out, indent);
      if (!s.parts.empty() && error_.empty()) error_ = fn.name() + "(concat(...)) is not supported yet";
      std::vector<uint8_t> prog;
      std::string why;
      if (CompileDateFormat(static_cast<const LiteralNode&>(*fn.children()[1]).bytes(), &prog, &why) != 0 && error_.empty())
        error_ = why;
      bool suppress = false;
      if (fn.children().size() == 3) {
        const auto& lit = static_cast<const LiteralNode&>(*fn.children()[2]);
        suppress = lit.as<int32_t>() != 0;
      }
      const std::string arr = NewVar("gdv_datefmt_");
      std::string t = "__device__ const u8 " + arr + "[" + std::to_string(prog.size() + 1) + "] = {";
      for (uint8_t b : prog) t += std::to_string(static_cast<unsigned>(b)) + ",";
      t += "0};\n";
      globals_ += t;
      const std::string v = NewVar("v"), okv = NewVar("ok");
      uses_ctx_ = true;
      *out += Ind(indent) + "i64 " + v + " = 0;\n";
      *out += Ind(indent) + "bool " + okv + " = false;\n";
      *out += Ind(indent) + "if (in && (" + s.ok + ")) " + v + " = gdv_to_date_fmt(&ctx, " + s.v + ", " + arr + ", " +
              std::to_string(prog.size()) + ", " + (suppress ? "true" : "false") + ", &" + okv + ");\n";
      return Val{v, okv, rt};
    }

    if (def->flags & kRegexHolder) {
      Val s = Gen(*fn.children()[0], out, indent);
      if (!s.parts.empty() && error_.empty()) error_ = fn.name() + "(concat(...)) is not supported yet";
      RegexProgram prog;
      std::string why;
      if (CompileRegex(static_cast<const LiteralNode&>(*fn.children()[1]).bytes(), &prog, &why) != 0 && error_.empty())
        error_ = why;
      // program block: first, last, flags, follow, byte classes -- one u64 per set for <= 64 positions
      // (gdv_regex_match), two for up to 128 (gdv_regex_match2)
      const bool wide = prog.positions > 64;
      const int W = wide ? 2 : 1, NP = wide ? 128 : 64;
      const std::string arr = NewVar("gdv_re_");
      auto hex = [](uint64_t v) {
        char buf[32];
        std::snprintf(buf, sizeof buf, "0x%llxull", static_cast<unsigned long long>(v));
        return std::string(buf);
      };
      std::string t = "__device__ const u64 " + arr + "[" + std::to_string(2 * W + 1 + NP * W + 256 * W) + "] = {";
      for (int w = 0; w < W; ++w) t += hex(prog.first[w]) + ",";
      for (int w = 0; w < W; ++w) t += hex(prog.last[w]) + ",";
      t += hex((prog.nullable ? 1u : 0u) | (prog.anchor_start ? 2u : 0u) | (prog.anchor_end ? 4u : 0u));
      for (int k = 0; k < NP; ++k)
        for (int w = 0; w < W; ++w) t += "," + hex(prog.follow[k][w]);
      for (int k = 0; k < 256; ++k)
        for (int w = 0; w < W; ++w) t += ((k % 16 == 0 && w == 0) ? ",\n    " : ",") + hex(prog.cls[k][w]);
      t += "};\n";
      globals_ += t;
      const std::string v = NewVar("v");
      *out += Ind(indent) + "const bool " + v + " = " + (wide ? "gdv_regex_match2(" : "gdv_regex_match(") + s.v + ", " + arr + ");\n";
      return Val{v, s.ok, rt};
    }

    if (def->flags & kLikeHolder) {
      Val s = Gen(*fn.children()[0], out, indent);
      if (!s.parts.empty() && error_.empty()) error_ = "like(concat(...)) is not supported yet";
      const auto& pat = static_cast<const LiteralNode&>(*fn.children()[1]);
      bool has_esc = fn.children().size() == 3;
      char esc = has_esc ? static_cast<const LiteralNode&>(*fn.children()[2]).bytes()[0] : 0;
      const std::vector<unsigned> toks = LikeTokens(pat.bytes(), has_esc, esc);
      bool has_one = false;
      for (unsigned t : toks) has_one = has_one || (t >> 8) == 1u;
      const std::string v = NewVar("v");
      if (!has_one) {
        const std::string fn_name = LikeSpecialised(toks);
        int slot = -1;
        unsigned xf = 0u;
        std::string hits_fn;
        if (coop_ && ViewChain(*fn.children()[0], &slot, &xf)) hits_fn = LikeFromHits(toks, slot, xf);
        if (!hits_fn.empty()) {
          const std::string J = std::to_string(slot);
          *out += Ind(indent) + "const bool " + v + " = coop" + J + " ? " + hits_fn + "(" + s.v +
                  ", stage" + J + ", hits" + J + ", nh" + J + ") : " + fn_name + "(" + s.v + ");\n";
        } else {
          *out += Ind(indent) + "const bool " + v + " = " + fn_name + "(" + s.v + ");\n";
        }
      } else {
        const std::string arr = LikePatternTable(toks);
        *out += Ind(indent) + "const bool " + v + " = gdv_like_match(" + s.v + ", " + arr + ", " +
                std::to_string(toks.size()) + ");\n";
      }
      return Val{v, s.ok, rt};
    }

    std::vector<Val> args;
    for (const auto& c : fn.children()) args.push_back(Gen(*c, out, indent));

    if (def->flags & kConcat) {
      // concat: a null argument counts as the empty string, the result is never null;
      // concatOperator: null if any argument is null.  Either way no byte moves here: the
      // result is the list of its arguments' views, copied piece by piece by the write pass.
      const bool null_as_empty = fn.name() == "concat";
      Val r;
      r.type = rt;
      std::vector<std::string> oks;
      for (const auto& a : args) {
        oks.push_back(a.ok);
        if (!a.parts.empty()) {
          // a rope argument that is null (a null concatOperator result) contributes nothing
          for (const auto& p : a.parts) {
            if (null_as_empty && a.ok != "true") {
              const std::string pv = NewVar("v");
              *out += Ind(indent) + "const gdv_str " + pv + " = (" + a.ok + ") ? " + p +
                      " : gdv_make_str(nullptr, 0);\n";
              r.parts.push_back(pv);
            } else {
              r.parts.push_back(p);
            }
          }
        } else if (null_as_empty && a.ok != "true") {
          const std::string pv = NewVar("v");
          *out += Ind(indent) + "const gdv_str " + pv + " = (" + a.ok + ") ? " + a.v +
                  " : gdv_make_str(nullptr, 0);\n";
          r.parts.push_back(pv);
        } else {
          r.parts.push_back(a.v);
        }
      }
      if (r.parts.size() > 8 && error_.empty())
        error_ = "concat of more than 8 pieces is not supported";
      r.ok = null_as_empty ? std::string("true") : AndOk(oks);
      if (r.ok != "true" && r.ok != "false" && r.ok.find("&&") != std::string::npos) {
        const std::string okv = NewVar("ok");
        *out += Ind(indent) + "const bool " + okv + " = " + r.ok + ";\n";
        r.ok = okv;
      }
      r.v = "gdv_make_str(nullptr, 0)";
      return r;
    }
    for (const auto& a : args)
      if (!a.parts.empty() && error_.empty())
        error_ = "the result of concat / repeat / space / lpad / rpad / reverse can only be projected, "
                 "concatenated again or chosen by if/else; " + fn.name() + "(...) over it is not supported yet";

    if (def->flags & kVirtual) {
      // repeat / space / reverse: one virtual piece; lpad / rpad: the padding piece and the text
      // piece.  Pieces are plain gdv_str values whose xf marks them periodic / reversed; only the
      // string write pass knows how to read those, so the result is a rope like concat's.
      std::vector<std::string> oks;
      for (const auto& a : args) oks.push_back(a.ok);
      Val r;
      r.type = rt;
      r.ok = AndOk(oks);
      if (r.ok != "true" && r.ok != "false" && r.ok.find("&&") != std::string::npos) {
        const std::string okv = NewVar("ok");
        *out += Ind(indent) + "const bool " + okv + " = " + r.ok + ";\n";
        r.ok = okv;
      }
      r.v = "gdv_make_str(nullptr, 0)";
      auto piece = [&](const std::string& expr) {
        const std::string pv = NewVar("v");
        *out += Ind(indent) + "const gdv_str " + pv + " = " + expr + ";\n";
        r.parts.push_back(pv);
      };
      const std::string& nm = fn.name();
      if (nm == "replace") {
        const Node& fnode = *fn.children()[1];
        const Node& tnode = *fn.children()[2];
        if (fnode.kind() != NodeKind::kLiteral || tnode.kind() != NodeKind::kLiteral ||
            static_cast<const LiteralNode&>(fnode).is_null() || static_cast<const LiteralNode&>(tnode).is_null()) {
          if (error_.empty()) error_ = "replace(s, from, to) needs literal, non-null from / to strings";
          return r;
        }
        if (repl_sites_.size() >= 256 && error_.empty()) error_ = "more than 256 replace() calls in one kernel";
        const std::string& fb = static_cast<const LiteralNode&>(fnode).bytes();
        const std::string& tb = static_cast<const LiteralNode&>(tnode).bytes();
        ReplSite site{BytesArray(fb, "gdv_rfrom_"), BytesArray(tb, "gdv_rto_"), static_cast<int>(fb.size()),
                      static_cast<int>(tb.size())};
        piece("gdv_repl_view(" + args[0].v + ", " + std::to_string(repl_sites_.size()) + "u)");
        repl_sites_.push_back(site);
      } else if (nm == "lpad" || nm == "rpad") {
        const std::string fill = args.size() == 3 ? args[2].v : std::string("gdv_make_str(gdv_one_space, 1)");
        const std::string pad = "gdv_pad_fill(" + args[0].v + ", " + args[1].v + ", " + fill + ")";
        const std::string text = "gdv_pad_text(" + args[0].v + ", " + args[1].v + ")";
        if (nm == "lpad") { piece(pad); piece(text); }
        else { piece(text); piece(pad); }
      } else {
        std::string call = def->device_name() + "(";
        for (size_t i = 0; i < args.size(); ++i) call += (i ? ", " : "") + args[i].v;
        piece(call + ")");
      }
      return r;
    }

    if (const int ga = ArgGuard(fn); ga >= 0) {
      std::vector<std::string> goks;
      for (const auto& a : args) goks.push_back(a.ok);
      const std::string gok = AndOk(goks);
      const std::string gv = NewVar("v");
      Val& g = args[static_cast<size_t>(ga)];
      *out += Ind(indent) + g.type.ctype() + " " + gv + " = " + (ga == 1 ? "0" : "1") + ";\n";
      *out += Ind(indent) + "if (in && (" + gok + ")) " + gv + " = " + (ga == 1 ? "gdv_check_len" : "gdv_check_start") +
              "(&ctx, " + g.v + ");\n";
      g.v = gv;
      uses_ctx_ = true;
    }

    if (fn.name() == "nvl") {
      // nvl(a, b) = a where a is valid, else b: a select on a's validity, no device function
      const Val& a = args[0];
      const Val& b = args[1];
      if (a.ok == "true") return a;
      const std::string v = NewVar("v");
      *out += Ind(indent) + "const " + rt.ctype() + " " + v + " = (" + a.ok + ") ? " + a.v + " : " + b.v + ";\n";
      if (b.ok == "true") return Val{v, "true", rt};
      const std::string okv = NewVar("ok");
      *out += Ind(indent) + "const bool " + okv + " = (" + a.ok + ") || (" + b.ok + ");\n";
      return Val{v, okv, rt};
    }

    std::string call = def->device_name() + "(";
    bool first = true;
    auto add = [&](const std::string& a) {
      if (!first) call += ", ";
      call += a;
      first = false;
    };
    if (def->flags & kCanFail) {
      add("&ctx");
      uses_ctx_ = true;
    }
    for (size_t i = 0; i < args.size(); ++i) {
      add(args[i].v);
      if (def->nulls != NullMode::kIfNull) add(args[i].ok);
      if ((def->flags & kDecimalArgs) && args[i].type.is_decimal()) {
        add(std::to_string(args[i].type.precision));
        add(std::to_string(args[i].type.scale));
      }
    }
    if ((def->flags & kDecimalArgs) && rt.is_decimal()) {
      add(std::to_string(rt.precision));
      add(std::to_string(rt.scale));
    }
    if (def->flags & kScratch)
      add("gdv_scr + ((size_t)k * GDV_NS + " + std::to_string(n_scratch_++) + ") * GDV_SCRATCH_SLOT");
    call += ")";

    const std::string v = NewVar("v");
    if (def->nulls != NullMode::kIfNull && (def->flags & kCanFail)) {
      // sees nulls and can raise: called for every row of the batch (never for the padding of a tail)
      std::string okv = "true";
      if (def->nulls == NullMode::kInternal) {
        okv = NewVar("ok");
        *out += Ind(indent) + "bool " + okv + " = false;\n";
        call.insert(call.size() - 1, ", &" + okv);
      }
      *out += Ind(indent) + rt.ctype() + " " + v + " = " + ZeroOf(rt) + ";\n";
      *out += Ind(indent) + "if (in) " + v + " = " + call + ";\n";
      return Val{v, okv, rt};
    }
    if (def->nulls == NullMode::kNever) {
      *out += Ind(indent) + "const " + rt.ctype() + " " + v + " = " + call + ";\n";
      return Val{v, "true", rt};
    }
    if (def->nulls == NullMode::kInternal) {
      // the function decides validity itself: it receives (value, valid) pairs and writes *out_valid
      const std::string okv = NewVar("ok");
      call.insert(call.size() - 1, ", &" + okv);
      *out += Ind(indent) + "bool " + okv + " = false;\n";
      *out += Ind(indent) + "const " + rt.ctype() + " " + v + " = " + call + ";\n";
      return Val{v, okv, rt};
    }
    std::vector<std::string> oks;
    for (const auto& a : args) oks.push_back(a.ok);
    std::string ok = AndOk(oks);
    if (ok != "true" && ok != "false" && ok.find("&&") != std::string::npos) {
      const std::string okv = NewVar("ok");
      *out += Ind(indent) + "const bool " + okv + " = " + ok + ";\n";
      ok = okv;
    }
    if (def->flags & kCanFail) {
      // functions that can raise are only called on valid rows (and on rows in range)
      *out += Ind(indent) + rt.ctype() + " " + v + " = " + ZeroOf(rt) + ";\n";
      *out += Ind(indent) + "if (in && (" + ok + ")) " + v + " = " + call + ";\n";
    } else {
      *out += Ind(indent) + "const " + rt.ctype() + " " + v + " = " + call + ";\n";
    }
    return Val{v, ok, rt};
  }

  Val GenIf(const IfNode& n, std::string* out, int indent) {
    const DataType& rt = n.return_type();
    Val c = Gen(*n.condition(), out, indent);
    const std::string v = NewVar("v"), ok = NewVar("ok");
    // Branches are generated into side buffers first: when one of them is a concat rope the
    // result needs one variable per piece, and the number of pieces is only known afterwards.
    std::string tb, eb;
    Val t = Gen(*n.then_node(), &tb, indent + 1);
    Val e = Gen(*n.else_node(), &eb, indent + 1);
    const size_t np = std::max(t.parts.size(), e.parts.size());
    if (np == 0) {
      *out += Ind(indent) + rt.ctype() + " " + v + ";\n";
    } else {
      for (size_t i = 0; i < np; ++i)
        *out += Ind(indent) + "gdv_str " + v + "_" + std::to_string(i) + " = gdv_make_str(nullptr, 0);\n";
    }
    *out += Ind(indent) + "bool " + ok + ";\n";
    *out += Ind(indent) + "if ((" + c.ok + ") && (" + c.v + ")) {\n";
    auto assign = [&](const Val& b, const std::string& code) {
      *out += code;
      if (np == 0) {
        *out += Ind(indent + 1) + v + " = " + b.v + ";\n";
      } else if (b.parts.empty()) {
        *out += Ind(indent + 1) + v + "_0 = " + b.v + ";\n";
      } else {
        for (size_t i = 0; i < b.parts.size(); ++i)
          *out += Ind(indent + 1) + v + "_" + std::to_string(i) + " = " + b.parts[i] + ";\n";
      }
      *out += Ind(indent + 1) + ok + " = " + b.ok + ";\n";
    };
    assign(t, tb);
    *out += Ind(indent) + "} else {\n";
    assign(e, eb);
    *out += Ind(indent) + "}\n";
    Val r{v, ok, rt, {}};
    for (size_t i = 0; i < np; ++i) r.parts.push_back(v + "_" + std::to_string(i));
    if (np != 0) r.v = "gdv_make_str(nullptr, 0)";
    return r;
  }

  // SQL three-valued AND/OR.  AND: false if any child is (valid, false); else null if any
  // child is null; else true.  OR is the dual.  Children after the first are evaluated
  // lazily (only while the result is still undecided) when they contain a function that
  // can raise, which is the reference's short-circuit behaviour.
  Val GenBoolean(const BooleanNode& n, std::string* out, int indent) {
    const bool is_and = n.op() == BooleanNode::kAnd;
    const std::string dec = NewVar("dec");    // some child decided the result
    const std::string allok = NewVar("aok");  // every child so far was valid
    *out += Ind(indent) + "bool " + dec + " = false;\n";
    *out += Ind(indent) + "bool " + allok + " = true;\n";
    int opened = 0;
    int ind = indent;
    for (size_t i = 0; i < n.children().size(); ++i) {
      const Node& c = *n.children()[i];
      if (i > 0 && CanFail(c)) {
        *out += Ind(ind) + "if (!" + dec + ") {\n";
        ++opened;
        ++ind;
      }
      Val cv = Gen(c, out, ind);
      const std::string deciding = is_and ? ("!(" + cv.v + ")") : ("(" + cv.v + ")");
      *out += Ind(ind) + dec + " = " + dec + " || ((" + cv.ok + ") && " + deciding + ");\n";
      *out += Ind(ind) + allok + " = " + allok + " && (" + cv.ok + ");\n";
    }
    while (opened-- > 0) {
      --ind;
      *out += Ind(ind) + "}\n";
    }
    const std::string v = NewVar("v"), ok = NewVar("ok");
    *out += Ind(indent) + "const bool " + v + " = " + (is_and ? "!" : "") + dec + ";\n";
    *out += Ind(indent) + "const bool " + ok + " = " + dec + " || " + allok + ";\n";
    return Val{v, ok, boolean()};
  }

  Val GenIn(const InNode& n, std::string* out, int indent) {
    Val c = Gen(*n.child(), out, indent);
    if (!c.parts.empty() && error_.empty()) error_ = "IN over concat(...) is not supported yet";
    const std::string v = NewVar("v");
    const DataType& t = n.value_type();
    if (const int j = ViewSlot(*n.child()); j >= 0 && t.is_varlen()) {
      std::string e;
      for (const auto& s : n.strs()) e += (e.empty() ? "" : " || ") + ViewTest(true, j, s);
      if (e.empty()) e = "false";
      ++view_shortcuts_;
      *out += Ind(indent) + "const bool " + v + " = " + e + ";\n";
    } else if (t.is_varlen()) {
      std::string e;
      std::vector<std::string> sorted = n.strs();
      std::sort(sorted.begin(), sorted.end());
      for (const auto& s : sorted) {
        const std::string arr = BytesArray(s, "gdv_lit_");
        e += (e.empty() ? "" : " || ") + std::string("equal_utf8_utf8(") + c.v +
             ", gdv_make_str(" + arr + ", " + std::to_string(s.size()) + "))";
      }
      if (e.empty()) e = "false";
      *out += Ind(indent) + "const bool " + v + " = " + e + ";\n";
    } else if (t.id == GDV_TYPE_FLOAT || t.id == GDV_TYPE_DOUBLE) {
      // the constants arrive as bit patterns; membership is IEEE equality (-0.0 is in {0.0}, NaN is in nothing)
      std::vector<int64_t> vals = n.ints();
      std::sort(vals.begin(), vals.end());
      vals.erase(std::unique(vals.begin(), vals.end()), vals.end());
      std::string e;
      for (auto x : vals) {
        const std::string lit = t.id == GDV_TYPE_DOUBLE
                                    ? "gdv_f64_from_bits(" + HexLit(static_cast<uint64_t>(x)) + ")"
                                    : "__int_as_float((int)" + HexLit(static_cast<uint64_t>(x) & 0xffffffffull) + ")";
        e += (e.empty() ? "" : " || ") + std::string("(") + c.v + " == " + lit + ")";
      }
      if (e.empty()) e = "false";
      *out += Ind(indent) + "const bool " + v + " = " + e + ";\n";
    } else {
      std::vector<int64_t> vals = n.ints();
      std::sort(vals.begin(), vals.end());
      vals.erase(std::unique(vals.begin(), vals.end()), vals.end());
      const char* ct = t.ctype();
      if (vals.size() <= 8) {
        std::string e;
        for (auto x : vals)
          e += (e.empty() ? "" : " || ") + std::string("(") + c.v + " == (" + ct + ")" +
               HexLit(static_cast<uint64_t>(x)) + ")";
        if (e.empty()) e = "false";
        *out += Ind(indent) + "const bool " + v + " = " + e + ";\n";
      } else {
        const std::string arr = NewVar("gdv_in_");
        std::string g = std::string("__device__ const ") + ct + " " + arr + "[" +
                        std::to_string(vals.size()) + "] = {";
        for (size_t i = 0; i < vals.size(); ++i)
          g += (i ? "," : "") + std::string("(") + ct + ")" + HexLit(static_cast<uint64_t>(vals[i]));
        g += "};\n";
        globals_ += g;
        // branch-free binary search over the sorted constants
        *out += Ind(indent) + "bool " + v + ";\n";
        *out += Ind(indent) + "{\n";
        *out += Ind(indent + 1) + "int lo = 0, hi = " + std::to_string(vals.size()) + ";\n";
        *out += Ind(indent + 1) + "while (lo < hi) { const int mid = (lo + hi) >> 1; if (" +
                arr + "[mid] < " + c.v + ") lo = mid + 1; else hi = mid; }\n";
        *out += Ind(indent + 1) + v + " = lo < " + std::to_string(vals.size()) + " && " + arr +
                "[lo] == " + c.v + ";\n";
        *out += Ind(indent) + "}\n";
      }
    }
    return Val{v, c.ok, boolean()};
  }

  // ---- inline / prefix shortcut over string_view / binary_view columns (DESIGN.md §3.7) ----
  // The slot of `node` when it is a bare view column and the shortcut is on, else -1.
  int ViewSlot(const Node& node) {
    if (!view_sc_ || node.kind() != NodeKind::kField || !node.return_type().is_view()) return -1;
    return SlotFor(static_cast<const FieldNode&>(node));
  }

  // The test "the row of view slot j equals (equal) / starts with (!equal) the bytes b", decided from
  // the raw view w<j>[k] in registers: the length first, then the inline bytes or the 4-byte prefix
  // word; only out-of-line rows whose prefix agrees read their bytes, through the row's gdv_str.
  std::string ViewTest(bool equal, int j, const std::string& b) {
    uint32_t w[3] = {0u, 0u, 0u};
    for (size_t i = 0; i < b.size() && i < 12; ++i)
      w[i / 4] |= static_cast<uint32_t>(static_cast<uint8_t>(b[i])) << (8 * (i % 4));
    const bool reads = equal ? b.size() > 12 : b.size() > 4;
    const std::string arr = reads ? BytesArray(b, "gdv_lit_") : std::string("nullptr");
    char words[64];
    std::snprintf(words, sizeof(words), "0x%08xu, 0x%08xu, 0x%08xu", w[0], w[1], w[2]);
    const std::string J = std::to_string(j);
    return std::string(equal ? "gdv_sv_equal(" : "gdv_sv_starts(") + "w" + J + "[k], f" + J + "[k], " +
           std::to_string(b.size()) + ", " + words + ", " + arr + ")";
  }

  // equal / not_equal / starts_with of a bare view column and a literal, and LIKE whose pattern
  // starts with a literal run, lowered against the raw view (ViewTest).  string_scan bit 3 turns
  // this off: the same calls then read the row's bytes through its gdv_str like any other function.
  bool ViewShortcut(const FunctionNode& fn, std::string* out, int indent, Val* r) {
    if (!view_sc_ || fn.children().size() < 2) return false;
    const std::string& nm = fn.name();
    const bool eq = nm == "equal" || nm == "not_equal";
    if (!eq && nm != "starts_with" && nm != "like") return false;
    const Node* col = fn.children()[0].get();
    const Node* lit = fn.children()[1].get();
    if (eq && col->kind() == NodeKind::kLiteral) std::swap(col, lit);
    if (lit->kind() != NodeKind::kLiteral) return false;
    const auto& l = static_cast<const LiteralNode&>(*lit);
    if (l.is_null() || !l.return_type().is_varlen()) return false;
    const int j = ViewSlot(*col);
    if (j < 0) return false;
    const Val c = Gen(*col, out, indent);
    std::string test;
    if (eq) {
      test = (nm == "not_equal" ? "!" : "") + ViewTest(true, j, l.bytes());
    } else if (nm == "starts_with") {
      if (l.bytes().empty()) return false;
      test = ViewTest(false, j, l.bytes());
    } else {
      const bool has_esc = fn.children().size() == 3;
      const char esc = has_esc ? static_cast<const LiteralNode&>(*fn.children()[2]).bytes()[0] : 0;
      const std::vector<unsigned> toks = LikeTokens(l.bytes(), has_esc, esc);
      std::string head;
      size_t i = 0;
      for (; i < toks.size() && (toks[i] >> 8) == 0u; ++i) head.push_back(static_cast<char>(toks[i] & 0xffu));
      if (head.empty()) return false;
      if (i == toks.size()) {
        test = ViewTest(true, j, head);  // no wildcard: the pattern is one string
      } else if (i + 1 == toks.size() && (toks[i] >> 8) == 2u) {
        test = ViewTest(false, j, head);  // 'lit%'
      } else {
        bool has_one = false;
        for (unsigned t : toks) has_one = has_one || (t >> 8) == 1u;
        const std::string match = has_one ? "gdv_like_match(" + c.v + ", " + LikePatternTable(toks) + ", " +
                                                std::to_string(toks.size()) + ")"
                                          : LikeSpecialised(toks) + "(" + c.v + ")";
        test = ViewTest(false, j, head) + " && " + match;
      }
    }
    ++view_shortcuts_;
    const std::string v = NewVar("v");
    *out += Ind(indent) + "const bool " + v + " = " + test + ";\n";
    *r = Val{v, c.ok, boolean(), {}};
    return true;
  }

  const Schema& schema_;
  std::vector<ColumnSlot>* slots_;
  bool nullable_;
  bool coop_;
  bool view_sc_;
  int view_shortcuts_ = 0;
  std::string error_;  // first construct the fuser cannot lower (reported by GenerateKernel)
  std::vector<CoopSeg> coop_segs_;
  std::string globals_;
  std::vector<std::string> user_text_;  // preludes and user functions already in globals_
  struct ReplSite {
    std::string from, to;  // names of the literal byte arrays
    int fl, tl;
  };
  std::vector<ReplSite> repl_sites_;
  int n_scratch_ = 0;
  int next_id_ = 0;
  bool uses_ctx_ = false;
};

std::string EmitArgsStruct(const ArgsLayout& L) {
  std::stringstream s;
  s << "struct gdv_args {\n"
    << "  i64 n;            // rows (or selection slots) to process\n"
    << "  i64 row_base;     // added to every index a filter emits (row-range sharding)\n"
    << "  const void* sel;  // project: input selection vector (or null)\n"
    << "  void* out_idx;    // filter: output selection vector\n"
    << "  u64* out_count;   // filter: number of indices written\n"
    << "  u64* tile_state;  // filter: look-back descriptors, one per CTA tile\n"
    << "  u64* ticket;      // filter: dynamic tile counter\n"
    << "  int* err;         // first ExecutionError code raised by a device function\n"
    << "  i64 out_cap;      // filter: capacity of out_idx; selected rows past it are counted, not stored\n"
    << "  const u64* n_ptr; // project with a selection vector: slot count in device memory (or null: n)\n"
    << "  const void* in_val[" << L.ni << "];\n"
    << "  const u8* in_vld[" << L.ni << "];\n"
    << "  const u8* in_var[" << L.ni << "];\n"
    << "  void* out_val[" << L.no << "];\n"
    << "  u32* out_vld[" << L.no << "];\n"
    << "  u8* out_var[" << L.no << "];\n"
    << "  u32 in_vsh[" << L.ni << "];\n"
    << "  u32 in_dsh[" << L.ni << "];\n";
  if (L.dict)
    s << "  const i32* in_dof[" << L.ni << "];  // dictionary columns: the dictionary's offsets,\n"
      << "  const u32* in_dvl[" << L.ni << "];  // validity words (or null),\n"
      << "  i64 in_dln[" << L.ni << "];         // length\n"
      << "  u32 in_dvs[" << L.ni << "];         // and validity bit shift; in_var = its bytes\n";
  if (L.view)
    s << "  const u8* const* in_vbf[" << L.ni << "];  // view columns: the data buffers' device pointers,\n"
      << "  const i64* in_vsz[" << L.ni << "];        // their sizes\n"
      << "  i64 in_vbn[" << L.ni << "];               // and count\n";
  s << "};\n";
  return s.str();
}

const char* SelCType(int mode) {
  switch (mode) {
    case GDV_SEL_UINT16: return "u16";
    case GDV_SEL_UINT64: return "u64";
    default: return "u32";
  }
}

// ---- kernel skeleton pieces ------------------------------------------------------------
// Hoisted, typed views of the argument block (read once per thread, live in registers /
// uniform registers for the whole kernel), and `sel` when the kernel reads its rows through a
// selection vector (`has_sel`).
void EmitPrologue(const std::vector<ColumnSlot>& slots, const KernelSpec& spec, bool has_sel, std::string* o) {
  for (size_t j = 0; j < slots.size(); ++j) {
    const DataType& t = slots[j].type;
    const std::string J = std::to_string(j);
    if (t.is_bool()) {
      *o += "  const u32* in_dat" + J + " = reinterpret_cast<const u32*>(A.in_val[" + J + "]);\n";
      *o += "  const u32 in_dsh" + J + " = A.in_dsh[" + J + "];\n";
    } else if (t.is_dict()) {
      const std::string it = DataType(t.index).ctype();
      *o += "  const " + it + "* in_val" + J + " = reinterpret_cast<const " + it + "*>(A.in_val[" + J + "]);\n";
      *o += "  const u8* in_var" + J + " = A.in_var[" + J + "];\n";
      *o += "  const i32* in_dof" + J + " = A.in_dof[" + J + "];\n";
      *o += "  const u32* in_dvl" + J + " = A.in_dvl[" + J + "];\n";
      *o += "  const i64 in_dln" + J + " = A.in_dln[" + J + "];\n";
      *o += "  const u32 in_dvs" + J + " = A.in_dvs[" + J + "];\n";
    } else if (t.is_view()) {
      *o += "  const uint4* in_val" + J + " = reinterpret_cast<const uint4*>(A.in_val[" + J + "]);\n";
      *o += "  const u8* const* in_vbf" + J + " = A.in_vbf[" + J + "];\n";
      *o += "  const i64* in_vsz" + J + " = A.in_vsz[" + J + "];\n";
      *o += "  const i64 in_vbn" + J + " = A.in_vbn[" + J + "];\n";
    } else if (t.is_varlen()) {
      const std::string ot = t.is_large() ? "i64" : "i32";
      *o += "  const " + ot + "* in_val" + J + " = reinterpret_cast<const " + ot + "*>(A.in_val[" + J + "]);\n";
      *o += "  const u8* in_var" + J + " = A.in_var[" + J + "];\n";
    } else {
      *o += "  const " + std::string(t.ctype()) + "* in_val" + J + " = reinterpret_cast<const " +
            t.ctype() + "*>(A.in_val[" + J + "]);\n";
    }
    if (spec.nullable) {
      *o += "  const u32* in_vld" + J + " = reinterpret_cast<const u32*>(A.in_vld[" + J + "]);\n";
      *o += "  const u32 in_vsh" + J + " = A.in_vsh[" + J + "];\n";
      *o += "  const bool in_hv" + J + " = in_vld" + J + " != nullptr;\n";
      // branch-free validity windows on the fast path: a column without a bitmap reads an all-ones
      // word at index 0, so the window loads of all columns issue back to back with the value
      // loads instead of sitting behind one uniform branch (and one load latency) each
      *o += "  const u32* const in_vp" + J + " = in_hv" + J + " ? in_vld" + J + " : gdv_all_ones;\n";
      *o += "  const i64 in_vm" + J + " = in_hv" + J + " ? -1ll : 0ll;\n";
    }
  }
  if (has_sel)
    *o += "  const " + std::string(SelCType(spec.selection_mode)) +
          "* sel = reinterpret_cast<const " + SelCType(spec.selection_mode) + "*>(A.sel);\n";
}

// One group of R steps (32 rows each) starting at row `base` (a multiple of 32):
// declarations, load phase, then the compute loop whose per-step tail is `step_tail`
// (stores / ballots; may use `s`, `in`, `k`).  `has_sel`: row s of the group is row sel[s] of the
// batch (a projector given a selection vector).  `fast` = every row of the group is in range
// and rows are contiguous (no selection vector): loads are unconditional, back to back, with
// immediate offsets from one pointer per column; validity arrives as one 32-bit window per
// step (a warp-uniform load) instead of one byte load per row.
// Group modes: kPred = per-row range predicates (tail group / selection vector), kFast = whole
// group in range, direct global loads, kStaged = whole CTA tile already in shared memory (TMA).
enum GroupMode { kPred = 0, kFast = 1, kStaged = 2 };

// Cooperative LIKE scan of the staged bytes of column J (BodyGen::LikeFromHits registers the
// segments).  Level 1: every lane takes 16-byte chunks of the group's byte run and tests all 16
// byte positions for the rarest adjacent byte pair (digram) of each LIKE's key segment with two
// halfword zero tests per word; the (rare) candidates go to a list.  Level 2, per candidate and
// warp-uniform: lane i verifies byte i of the key segment, the row that holds the occurrence is
// found with a ballot over the lanes' row ranges, and the row's bytes are searched for the
// LIKE's other segments, 32 positions at a time.  Verified occurrences are appended to the hit
// list as (segment id << 24 | stage offset); the per-row function chains them.  More than
// kHitCap candidates or hits: the group falls back to the per-lane matcher.
bool ScanFolds(const CoopSeg& cs, unsigned char c) {
  return (cs.xf == 1u && c >= 'A' && c <= 'Z') || (cs.xf == 2u && c >= 'a' && c <= 'z');
}

std::string SegVerifyExpr(const CoopSeg& cs, const std::string& stage, const std::string& at) {
  std::string e;
  for (size_t i = 0; i < cs.bytes.size(); ++i) {
    const unsigned char lit = static_cast<unsigned char>(cs.bytes[i]);
    const std::string ld = "(u32)" + stage + "[" + at + " + " + std::to_string(i) + "]";
    if (!e.empty()) e += " && ";
    if (ScanFolds(cs, lit))
      e += "((" + ld + " | 0x20u) == " + std::to_string(static_cast<unsigned>(lit | 0x20u)) + "u)";
    else
      e += "(" + ld + " == " + std::to_string(static_cast<unsigned>(lit)) + "u)";
  }
  return e;
}

std::string EmitCoopScan(int j, const std::vector<CoopSeg>& segs, int R, const std::string& I,
                         bool accumulate_hibits = false) {
  const std::string J = std::to_string(j);
  const std::string CAP = std::to_string(kHitCap) + "u";
  std::string o;
  std::vector<const CoopSeg*> keys;
  for (const auto& cs : segs)
    if (cs.slot == j && cs.is_key) keys.push_back(&cs);
  o += I + "if (lane < 2u) hctr" + J + "[lane] = 0u;\n";
  o += I + "__syncwarp();\n";
  o += I + "const i32 lo = (i32)mis, hi = (i32)mis + gn;\n";
  // ---- level 1: digram candidates
  o += I + "for (i32 c = (i32)lane; c < nchunks; c += 32) {\n";
  o += I + "  const uint4 v = reinterpret_cast<const uint4*>(stage" + J + ")[c];\n";
  o += I + "  const u32 vn = reinterpret_cast<const u32*>(stage" + J + ")[4 * c + 4];\n";
  if (accumulate_hibits) o += I + "  hibits |= v.x | v.y | v.z | v.w;\n";
  std::string any;
  for (const CoopSeg* k : keys) {
    const std::string S = std::to_string(k->id);
    const unsigned char c1 = static_cast<unsigned char>(k->bytes[k->digram]);
    const unsigned char c2 = static_cast<unsigned char>(k->bytes[k->digram + 1]);
    const bool f1 = ScanFolds(*k, c1), f2 = ScanFolds(*k, c2);
    const unsigned b1 = f1 ? (c1 | 0x20u) : c1, b2 = f2 ? (c2 | 0x20u) : c2;
    const unsigned fold = (f1 ? 0x20u : 0u) | (f2 ? 0x2000u : 0u);
    char pat[16], fm[16];
    std::snprintf(pat, sizeof(pat), "0x%08xu", (b1 | (b2 << 8)) * 0x00010001u);
    std::snprintf(fm, sizeof(fm), "0x%08xu", fold * 0x00010001u);
    // the odd-offset test sees the bytes rotated by one: the fold mask and pattern stay aligned
    // with (first, second) because the word is shifted, not the pattern
    const char* w[5] = {"v.x", "v.y", "v.z", "v.w", "vn"};
    // Both bytes fold (or neither): fold the words once, before the byte shift of the odd test.
    // Mixed: the fold mask must line up with (first, second) byte, so it is applied after it.
    const bool uniform = f1 == f2;
    const std::string orfm = fold != 0u ? std::string(" | ") + fm : std::string();
    for (int q = 0; q < 5; ++q)
      o += I + "  const u32 x" + S + "_" + std::to_string(q) + " = " + w[q] + (uniform ? orfm : std::string()) +
           ";\n";
    for (int q = 0; q < 4; ++q) {
      const std::string Q = std::to_string(q), Qn = std::to_string(q + 1);
      o += I + "  const u32 e" + S + "_" + Q + " = gdv_eqhalf_msb(x" + S + "_" + Q + (uniform ? std::string() : orfm) +
           ", " + pat + ");\n";
      o += I + "  const u32 o" + S + "_" + Q + " = gdv_eqhalf_msb(__funnelshift_r(x" + S + "_" + Q + ", x" +
           S + "_" + Qn + ", 8)" + (uniform ? std::string() : orfm) + ", " + pat + ");\n";
      any += (any.empty() ? "" : " | ") + std::string("e") + S + "_" + Q + " | o" + S + "_" + Q;
    }
  }
  o += I + "  if ((" + any + ") != 0u) {\n";
  for (const CoopSeg* k : keys) {
    const std::string S = std::to_string(k->id);
    o += I + "    {\n";
    o += I + "      u32 mk = gdv_mask16_half(e" + S + "_0, o" + S + "_0, e" + S + "_1, o" + S + "_1, e" + S +
         "_2, o" + S + "_2, e" + S + "_3, o" + S + "_3);\n";
    o += I + "      while (mk != 0u) {\n";
    o += I + "        const i32 st = 16 * c + (__ffs((int)mk) - 1) - " + std::to_string(k->digram) + ";\n";
    o += I + "        mk &= mk - 1u;\n";
    o += I + "        if (st >= lo && st + " + std::to_string(k->bytes.size()) + " <= hi && " +
         SegVerifyExpr(*k, "stage" + J, "st") + ") {\n";
    o += I + "          const u32 cx = atomicAdd(hctr" + J + " + 1, 1u);\n";
    o += I + "          if (cx < " + CAP + ") cand" + J + "[cx] = (" + std::to_string(k->like) +
         "u << 24) | (u32)st;\n";
    o += I + "        }\n";
    o += I + "      }\n";
    o += I + "    }\n";
  }
  o += I + "  }\n";
  o += I + "}\n";
  o += I + "__syncwarp();\n";
  // ---- level 2: verify candidates, find their rows, search the rows for the other segments
  o += I + "const u32 ncand = hctr" + J + "[1];\n";
  o += I + "if (ncand != 0u && ncand <= " + CAP + ") {\n";
  o += I + "  for (u32 h = 0u; h < ncand; ++h) {\n";
  o += I + "    const u32 ce = cand" + J + "[h];\n";
  o += I + "    const i32 p = (i32)(ce & 0xffffffu);\n";
  for (const CoopSeg* k : keys) {
    const std::string KL = std::to_string(k->bytes.size());
    // per-lane byte of the key: immediate select chain would be long; use a packed table
    o += I + "    if ((ce >> 24) == " + std::to_string(k->like) + "u) {\n";
    o += I + "      {\n";
    o += I + "        i32 rs = 0, re = -1;\n";
    o += I + "        #pragma unroll\n";
    o += I + "        for (int k = 0; k < " + std::to_string(R) + "; ++k) {\n";
    // (large column: ptr and gb are i64; the group's bytes fit the stage, so the difference fits i32)
    o += I + "          const i32 a = ptr" + J + "[32 * k] - gb + (i32)mis;\n";
    o += I + "          const i32 b = ptr" + J + "[32 * k + 1] - gb + (i32)mis;\n";
    o += I + "          const u32 own = __ballot_sync(GDV_FULL, a <= p && p + " + KL + " <= b);\n";
    o += I + "          if (own != 0u) {\n";
    o += I + "            const int src = __ffs((int)own) - 1;\n";
    o += I + "            rs = __shfl_sync(GDV_FULL, a, src);\n";
    o += I + "            re = __shfl_sync(GDV_FULL, b, src);\n";
    o += I + "          }\n";
    o += I + "        }\n";
    o += I + "        if (re >= 0) {\n";
    o += I + "          if (lane == 0u) {\n";
    o += I + "            const u32 hx = atomicAdd(hctr" + J + ", 1u);\n";
    o += I + "            if (hx < " + CAP + ") hits" + J + "[hx] = (" + std::to_string(k->id) + "u << 24) | (u32)p;\n";
    o += I + "          }\n";
    for (const auto& os : segs) {
      if (os.slot != j || os.like != k->like || os.id == k->id) continue;
      const std::string L = std::to_string(os.bytes.size());
      o += I + "          for (i32 q = rs + (i32)lane; q + " + L + " <= re; q += 32) {\n";
      o += I + "            if (" + SegVerifyExpr(os, "stage" + J, "q") + ") {\n";
      o += I + "              const u32 hx = atomicAdd(hctr" + J + ", 1u);\n";
      o += I + "              if (hx < " + CAP + ") hits" + J + "[hx] = (" + std::to_string(os.id) + "u << 24) | (u32)q;\n";
      o += I + "            }\n";
      o += I + "          }\n";
    }
    o += I + "        }\n";
    o += I + "      }\n";
    o += I + "    }\n";
  }
  o += I + "  }\n";
  o += I + "  __syncwarp();\n";
  o += I + "}\n";
  o += I + "nh" + J + " = hctr" + J + "[0];\n";
  o += I + "coop" + J + " = ncand <= " + CAP + " && nh" + J + " <= " + CAP + ";\n";
  return o;
}

// Row view of dictionary column J for the index expression `ix` (gdv_dict_view); the entry's
// validity lands in d<J>[k].
std::string DictView(const std::string& J, const std::string& ix) {
  return "gdv_dict_view(in_dof" + J + ", in_var" + J + ", in_dvl" + J + ", in_dvs" + J + ", in_dln" + J + ", " + ix +
         ", &d" + J + "[k])";
}

// Row view of string_view / binary_view column J from its 16-byte view w<J>[k], loaded from `at`
// (gdv_sv_view); the view's validity lands in d<J>[k].
std::string SvView(const std::string& J, const std::string& at) {
  return "gdv_sv_view(w" + J + "[k], " + at + ", in_vbf" + J + ", in_vsz" + J + ", in_vbn" + J + ", &d" + J + "[k])";
}

// A utf8 / binary column whose group of rows is one contiguous run of the data buffer (what the
// shared-memory string stage copies); a dictionary or view column's rows are not.
bool HasByteRun(const ColumnSlot& s) { return s.type.is_varlen() && !s.type.is_dict() && !s.type.is_view(); }

bool SlotHasCoop(const std::vector<CoopSeg>& segs, int j) {
  for (const auto& cs : segs)
    if (cs.slot == j) return true;
  return false;
}

void EmitGroup(const std::vector<ColumnSlot>& slots, const KernelSpec& spec, bool has_sel, int R, int mode,
               const std::string& body, const std::string& step_tail, std::string* o, int indent,
               int stage_bytes = 0, const std::string& after_loads = std::string(),
               const std::vector<CoopSeg>& coop = std::vector<CoopSeg>(), bool prefetched = false) {
  const bool fast = mode != kPred;
  const std::string I(static_cast<size_t>(indent) * 2, ' ');
  const std::string sR = std::to_string(R);
  for (size_t j = 0; j < slots.size(); ++j) {
    const DataType& t = slots[j].type;
    *o += I + t.ctype() + " f" + std::to_string(j) + "[" + sR + "];\n";
    if (spec.nullable) *o += I + "bool k" + std::to_string(j) + "[" + sR + "];\n";
    if (t.is_dict()) {
      // dictionary column: the entry behind the row's index is valid (and the index in range)
      *o += I + "bool d" + std::to_string(j) + "[" + sR + "];\n";
    } else if (t.is_view()) {
      // view column: the raw 16-byte views (the inline / prefix shortcut reads them) and whether
      // each view is valid
      *o += I + "uint4 w" + std::to_string(j) + "[" + sR + "];\n";
      *o += I + "bool d" + std::to_string(j) + "[" + sR + "];\n";
    } else if (t.is_varlen()) {
      // group state of the string stage: rows known to be ASCII, cooperative-scan hit list usable;
      // large column: whether each row's length fits a gdv_str (gdv_large_str)
      if (t.is_large()) *o += I + "bool d" + std::to_string(j) + "[" + sR + "];\n";
      *o += I + "u32 ascii" + std::to_string(j) + " = 0u;\n";
      if (SlotHasCoop(coop, static_cast<int>(j))) {
        *o += I + "bool coop" + std::to_string(j) + " = false;\n";
        *o += I + "u32 nh" + std::to_string(j) + " = 0u;\n";
      }
    }
  }
  if (mode == kStaged) {
    *o += I + "#pragma unroll\n";
    *o += I + "for (int k = 0; k < " + sR + "; ++k) {\n";
    for (size_t j = 0; j < slots.size(); ++j) {
      const std::string J = std::to_string(j);
      *o += I + "  f" + J + "[k] = gdv_lds(sp" + J + " + 32 * k);\n";
      if (spec.nullable && slots[j].hoist)
        *o += I + "  k" + J + "[k] = true;\n";
      else if (spec.nullable)
        *o += I + "  k" + J + "[k] = !in_hv" + J + " || ((gdv_ldwin_s(sv" + J + ", wid * " + sR +
              "u + (u32)k, in_vsh" + J + ") >> lane) & 1u) != 0u;\n";
    }
    *o += I + "}\n";
    *o += after_loads;
  } else if (fast) {
    bool staged_any = false;
    for (size_t j = 0; j < slots.size(); ++j) {
      const DataType& t = slots[j].type;
      const std::string J = std::to_string(j);
      if (!t.is_bool())
        *o += I + "const " +
              (t.is_dict()   ? std::string(DataType(t.index).ctype())
               : t.is_view() ? std::string("uint4")
               : t.is_large() ? std::string("i64")
               : t.is_varlen() ? std::string("i32") : std::string(t.ctype())) +
              "* ptr" + J + " = in_val" + J + " + base + (i64)lane;\n";
      if (HasByteRun(slots[j]) && stage_bytes > 0) {
        // The bytes of the group's 32*R strings are one contiguous run: copy it into this
        // warp's shared-memory stage with coalesced 16-byte loads, then every lane walks its
        // own string out of shared memory instead of issuing one global load per byte.
        staged_any = true;
        *o += I + "const u8* sbase" + J + " = in_var" + J + ";\n";
        *o += I + "{\n";
        if (t.is_large()) {
          // int64 offsets: the run is measured in i64 and narrowed once it is known to fit the stage
          *o += I + "  const i64 gb = in_val" + J + "[base];\n";
          *o += I + "  const i64 gn64 = in_val" + J + "[base + " + std::to_string(32 * R) + "] - gb;\n";
          *o += I + "  const u8* src = in_var" + J + " + gb;\n";
          *o += I + "  const u32 mis = (u32)((unsigned long long)src & 15ull);\n";
          *o += I + "  if (gn64 + (i64)mis <= " + std::to_string(stage_bytes) + ") {\n";
          *o += I + "    const i32 gn = (i32)gn64;\n";
        } else {
          *o += I + "  const i32 gb = in_val" + J + "[base];\n";
          *o += I + "  const i32 gn = in_val" + J + "[base + " + std::to_string(32 * R) + "] - gb;\n";
          *o += I + "  const u8* src = in_var" + J + " + gb;\n";
          *o += I + "  const u32 mis = (u32)((unsigned long long)src & 15ull);\n";
          *o += I + "  if (gn + (i32)mis <= " + std::to_string(stage_bytes) + ") {\n";
        }
        *o += I + "    const i32 nchunks = (gn + (i32)mis + 15) >> 4;\n";
        *o += I + "    u32 hibits = 0u;\n";
        if (!prefetched) {
          // four 16-byte loads in flight per lane, then the stores; the OR of all words tells
          // whether the whole run is ASCII
          *o += I + "    const uint4* s4 = reinterpret_cast<const uint4*>(src - mis);\n";
          *o += I + "    for (i32 c0 = (i32)lane; c0 < nchunks; c0 += 128) {\n";
          *o += I + "      uint4 t4[4];\n";
          *o += I + "      #pragma unroll\n";
          *o += I + "      for (int u = 0; u < 4; ++u)\n";
          *o += I + "        if (c0 + 32 * u < nchunks) t4[u] = __ldcs(s4 + c0 + 32 * u);\n";
          *o += I + "      #pragma unroll\n";
          *o += I + "      for (int u = 0; u < 4; ++u)\n";
          *o += I + "        if (c0 + 32 * u < nchunks) {\n";
          *o += I + "          reinterpret_cast<uint4*>(stage" + J + ")[c0 + 32 * u] = t4[u];\n";
          *o += I + "          hibits |= t4[u].x | t4[u].y | t4[u].z | t4[u].w;\n";
          *o += I + "        }\n";
          *o += I + "    }\n";
        }
        // prefetched: the bytes were copied by cp.async one group ahead (filter kernel) and the
        // caller has waited for them; the ASCII test rides on the scan's pass over the stage
        *o += I + "    sbase" + J + " = stage" + J + " + mis - gb;\n";
        if (SlotHasCoop(coop, static_cast<int>(j))) {
          *o += EmitCoopScan(static_cast<int>(j), coop, R, I + "    ", prefetched);
        } else if (prefetched) {
          *o += I + "    for (i32 c = (i32)lane; c < nchunks; c += 32) {\n";
          *o += I + "      const uint4 v = reinterpret_cast<const uint4*>(stage" + J + ")[c];\n";
          *o += I + "      hibits |= v.x | v.y | v.z | v.w;\n";
          *o += I + "    }\n";
        } else {
          *o += I + "    __syncwarp();\n";
        }
        *o += I + "    ascii" + J + " = __any_sync(GDV_FULL, (hibits & 0x80808080u) != 0u) ? 0u : GDV_XF_ASCII;\n";
        *o += I + "  }\n";
        *o += I + "}\n";
      }
    }
    (void)staged_any;
    *o += I + "#pragma unroll\n";
    *o += I + "for (int k = 0; k < " + sR + "; ++k) {\n";
    for (size_t j = 0; j < slots.size(); ++j) {
      const DataType& t = slots[j].type;
      const std::string J = std::to_string(j);
      if (t.is_bool()) {
        *o += I + "  f" + J + "[k] = ((gdv_ldwin(in_dat" + J + ", (base >> 5) + k, in_dsh" + J +
              ") >> lane) & 1u) != 0u;\n";
      } else if (t.is_dict()) {
        *o += I + "  f" + J + "[k] = " + DictView(J, "(i64)gdv_ldp(ptr" + J + " + 32 * k)") + ";\n";
      } else if (t.is_view()) {
        *o += I + "  w" + J + "[k] = gdv_ldview(ptr" + J + " + 32 * k);\n";
        *o += I + "  f" + J + "[k] = " + SvView(J, "ptr" + J + " + 32 * k") + ";\n";
      } else if (t.is_large()) {
        *o += I + "  { f" + J + "[k] = gdv_large_str(" + (stage_bytes > 0 ? "sbase" : "in_var") + J + ", ptr" + J +
              "[32 * k], ptr" + J + "[32 * k + 1], &d" + J + "[k]); f" + J + "[k].xf = ascii" + J + "; }\n";
      } else if (t.is_varlen()) {
        *o += I + "  { const i32 sb = ptr" + J + "[32 * k]; const i32 se = ptr" + J +
              "[32 * k + 1]; f" + J + "[k] = gdv_make_str(" +
              (stage_bytes > 0 ? "sbase" : "in_var") + J + " + sb, se - sb); f" + J +
              "[k].xf = ascii" + J + "; }\n";
      } else {
        *o += I + "  f" + J + "[k] = gdv_ldp(ptr" + J + " + 32 * k);\n";
      }
    }
    *o += I + "}\n";
    if (spec.nullable) {
      *o += I + "#pragma unroll\n";
      *o += I + "for (int k = 0; k < " + sR + "; ++k) {\n";
      for (size_t j = 0; j < slots.size(); ++j) {
        const std::string J = std::to_string(j);
        if (slots[j].hoist)  // validity ANDed into the keep-mask after the row loop (EmitHoistedValidity)
          *o += I + "  k" + J + "[k] = true;\n";
        else
          *o += I + "  k" + J + "[k] = ((gdv_ldwin(in_vp" + J + ", ((base >> 5) + k) & in_vm" + J + ", in_vsh" +
                J + ") >> lane) & 1u) != 0u" +
                (slots[j].type.is_dict() || slots[j].type.is_view() || slots[j].type.is_large() ? " && d" + J + "[k]" : "") +
                ";\n";
      }
      *o += I + "}\n";
    }
  } else {
    *o += I + "#pragma unroll\n";
    *o += I + "for (int k = 0; k < " + sR + "; ++k) {\n";
    *o += I + "  const i64 s = base + 32 * k + (i64)lane;\n";
    *o += I + "  const bool in = s < A.n;\n";
    *o += I + std::string("  const i64 r = in ? ") + (has_sel ? "(i64)sel[s]" : "s") + " : 0;\n";
    for (size_t j = 0; j < slots.size(); ++j) {
      const DataType& t = slots[j].type;
      const std::string J = std::to_string(j);
      if (t.is_bool()) {
        *o += I + "  f" + J + "[k] = in && gdv_ldbit(reinterpret_cast<const u8*>(in_dat" + J + "), in_dsh" +
              J + ", r);\n";
      } else if (t.is_dict()) {
        *o += I + "  f" + J + "[k] = " + DictView(J, "in ? (i64)gdv_ldp(in_val" + J + " + r) : -1ll") + ";\n";
      } else if (t.is_view()) {
        *o += I + "  w" + J + "[k] = in ? gdv_ldview(in_val" + J + " + r) : make_uint4(0u, 0u, 0u, 0u);\n";
        *o += I + "  f" + J + "[k] = " + SvView(J, "in_val" + J + " + r") + ";\n";
      } else if (t.is_large()) {
        *o += I + "  f" + J + "[k] = gdv_large_str(in_var" + J + ", in ? in_val" + J + "[r] : 0ll, in ? in_val" + J +
              "[r + 1] : 0ll, &d" + J + "[k]);\n";
      } else if (t.is_varlen()) {
        *o += I + "  { const i32 sb = in ? in_val" + J + "[r] : 0; const i32 se = in ? in_val" + J +
              "[r + 1] : 0; f" + J + "[k] = gdv_make_str(in_var" + J + " + sb, se - sb); }\n";
      } else {
        *o += I + "  f" + J + "[k] = in ? gdv_ldp(in_val" + J + " + r) : (" + t.ctype() + ")0;\n";
      }
      if (spec.nullable && slots[j].hoist)
        *o += I + "  k" + J + "[k] = in;\n";
      else if (spec.nullable)
        *o += I + "  k" + J + "[k] = in && (!in_hv" + J + " || gdv_ldbit(reinterpret_cast<const u8*>(in_vld" +
              J + "), in_vsh" + J + ", r))" + (t.is_dict() || t.is_view() || t.is_large() ? " && d" + J + "[k]" : "") +
              ";\n";
    }
    *o += I + "}\n";
  }
  *o += I + "#pragma unroll\n";
  *o += I + "for (int k = 0; k < " + sR + "; ++k) {\n";
  *o += I + "  const i64 s = base + 32 * k + (i64)lane;\n";
  *o += I + (fast ? "  const bool in = true;\n" : "  const bool in = s < A.n;\n");
  *o += body;
  *o += step_tail;
  *o += I + "}\n";
  if (fast && stage_bytes > 0) {
    bool any = false;
    for (const auto& sl : slots) any = any || (sl.type.is_varlen() && !sl.type.is_view());
    if (any) *o += I + "__syncwarp();  // all lanes are done with the stage before it is refilled\n";
  }
}

// Gated loads of a fixed-width Filter (DESIGN.md §3.3): the conjuncts of the condition's AND spine
// are evaluated in stages, and stage s loads its columns only in the rows every earlier stage kept.
// Stage s loads slots [first_slot[s], first_slot[s + 1]) (slots are numbered by first appearance on
// the spine) and ANDs in the conjuncts whose last column is among them (PlanGate).
struct GatePlan {
  std::vector<int> first_slot;                      // one per stage, plus slots.size() at the end
  std::vector<std::vector<const Node*>> conjuncts;  // per stage, in spine order
  int stages() const { return static_cast<int>(conjuncts.size()); }
};

// One group of R steps of a gated fixed-width Filter (GatePlan; mode kFast or kPred).  Stage 0 loads
// like EmitGroup; the loads of a later stage are issued, all R of them, only in the lanes whose row
// is still alive, so a row that an earlier conjunct dropped reads none of the later columns' bytes.
// A group in which stage 0 kept every row loads all later columns at once instead.
// seg[s] evaluates stage s's conjuncts for row [k] and ANDs them into alive[k]; validity (per-row or
// hoisted) is read as EmitGroup reads it, whatever the stage.
void EmitGatedGroup(const std::vector<ColumnSlot>& slots, const KernelSpec& spec, int R, int mode,
                    const GatePlan& plan, const std::vector<std::string>& seg, const std::string& step_tail,
                    std::string* o, int indent) {
  const bool fast = mode == kFast;
  const std::string I(static_cast<size_t>(indent) * 2, ' ');
  const std::string sR = std::to_string(R);
  for (size_t j = 0; j < slots.size(); ++j) {
    *o += I + slots[j].type.ctype() + " f" + std::to_string(j) + "[" + sR + "];\n";
    if (spec.nullable) *o += I + "bool k" + std::to_string(j) + "[" + sR + "];\n";
  }
  *o += I + "bool alive[" + sR + "];\n";
  if (fast)
    for (size_t j = 0; j < slots.size(); ++j)
      *o += I + "const " + slots[j].type.ctype() + "* ptr" + std::to_string(j) + " = in_val" + std::to_string(j) +
            " + base + (i64)lane;\n";
  const std::string row = I + "  const i64 s = base + 32 * k + (i64)lane;\n" +
                          I + (fast ? "  const bool in = true;\n" : "  const bool in = s < A.n;\n");
  // stage st: its loads (stage 0: the validity of every column too; `dense`: unpredicated), then its conjuncts
  auto stage = [&](int st, bool load, bool dense, const std::string& J2) {
    if (load) {
      *o += J2 + "#pragma unroll\n";
      *o += J2 + "for (int k = 0; k < " + sR + "; ++k) {\n";
      if (!fast || (st == 0 && spec.nullable)) *o += row;
      const std::string on = st == 0 ? std::string("in") : std::string("alive[k]");
      const int last = dense ? static_cast<int>(slots.size()) : plan.first_slot[st + 1];
      for (int j = plan.first_slot[st]; j < last; ++j) {
        const std::string J = std::to_string(j);
        const std::string zero = std::string("(") + slots[j].type.ctype() + ")0";
        if (fast && (st == 0 || dense))
          *o += J2 + "  f" + J + "[k] = gdv_ldp(ptr" + J + " + 32 * k);\n";
        else if (fast)
          *o += J2 + "  f" + J + "[k] = alive[k] ? gdv_ldp(ptr" + J + " + 32 * k) : " + zero + ";\n";
        else
          *o += J2 + "  f" + J + "[k] = " + on + " ? gdv_ldp(in_val" + J + " + s) : " + zero + ";\n";
      }
      if (st == 0 && spec.nullable) {
        for (size_t j = 0; j < slots.size(); ++j) {
          const std::string J = std::to_string(j);
          if (slots[j].hoist)  // validity ANDed into the keep-mask after the row loop (EmitFilterEpilogue)
            *o += J2 + "  k" + J + "[k] = in;\n";
          else if (fast)
            *o += J2 + "  k" + J + "[k] = ((gdv_ldwin(in_vp" + J + ", ((base >> 5) + k) & in_vm" + J + ", in_vsh" + J +
                  ") >> lane) & 1u) != 0u;\n";
          else
            *o += J2 + "  k" + J + "[k] = in && (!in_hv" + J + " || gdv_ldbit(reinterpret_cast<const u8*>(in_vld" + J +
                  "), in_vsh" + J + ", s));\n";
        }
      }
      *o += J2 + "}\n";
    }
    *o += J2 + "#pragma unroll\n";
    *o += J2 + "for (int k = 0; k < " + sR + "; ++k) {\n";
    *o += row;
    if (st == 0) *o += J2 + "  alive[k] = in;\n";
    *o += seg[static_cast<size_t>(st)];
    *o += J2 + "}\n";
  };
  stage(0, true, false, I);
  if (fast && plan.stages() > 2) {
    // Every row of the group survived stage 0 (a condition whose first conjuncts keep most rows):
    // gating could skip no sector, so the later columns are loaded together, one round trip instead
    // of one per stage.
    *o += I + "bool all_alive = true;\n";
    *o += I + "#pragma unroll\n";
    *o += I + "for (int k = 0; k < " + sR + "; ++k) all_alive = all_alive && alive[k];\n";
    *o += I + "if (__all_sync(GDV_FULL, all_alive)) {\n";
    for (int st = 1; st < plan.stages(); ++st) stage(st, st == 1, true, I + "  ");
    *o += I + "} else {\n";
    for (int st = 1; st < plan.stages(); ++st) stage(st, true, false, I + "  ");
    *o += I + "}\n";
  } else {
    for (int st = 1; st < plan.stages(); ++st) stage(st, true, false, I);
  }
  *o += I + "#pragma unroll\n";
  *o += I + "for (int k = 0; k < " + sR + "; ++k) {\n";
  *o += row;
  *o += step_tail;
  *o += I + "}\n";
}

void ReplaceAll(std::string* s, const std::string& from, const std::string& to) {
  for (size_t pos = 0; (pos = s->find(from, pos)) != std::string::npos; pos += to.size())
    s->replace(pos, from.size(), to);
}

// After the row loops of a filter tile: lane k of the warp holds, in mymask[w], the keep-mask of
// step k of its w-th 1024-row chunk (first row of chunk 0: wbase0).  ANDs in the validity words of
// the hoisted columns (ColumnSlot::hoist: one coalesced word load per lane and chunk instead of one
// warp-uniform window load per step and column inside the row loop), then positions the kept rows —
// scan over chunks and steps inside the warp, over warps inside the CTA, decoupled look-back over
// tiles — and writes the ascending indices.
void EmitFilterEpilogue(const std::vector<ColumnSlot>& slots, const KernelSpec& spec, int NW, int W,
                        const std::string& IDX, std::string* o) {
  const std::string sW = std::to_string(W), sNW = std::to_string(NW);
  std::string& src = *o;
  if (spec.nullable) {
    bool any = false;
    for (const auto& sl : slots) any = any || sl.hoist;
    if (any) {
      src += "    #pragma unroll\n";
      src += "    for (int w = 0; w < " + sW + "; ++w) {\n";
      src += "      const i64 rb = wbase0 + 1024 * w + 32 * (i64)lane;  // first row of the step whose mask this lane holds\n";
      for (size_t j = 0; j < slots.size(); ++j) {
        if (!slots[j].hoist) continue;
        const std::string J = std::to_string(j);
        src += "      if (in_hv" + J + " && rb < A.n) mymask[w] &= gdv_ldwin_rows(in_vld" + J + ", in_vsh" + J + ", rb, A.n);\n";
      }
      src += "    }\n";
    }
  }
  // per chunk: exclusive positions run over chunks, then steps
  src += "    u32 step_excl[" + sW + "];\n";
  src += "    u32 run = 0u;\n";
  src += "    #pragma unroll\n";
  src += "    for (int w = 0; w < " + sW + "; ++w) {\n";
  src += "      const u32 c = (u32)__popc(mymask[w]);\n";
  src += "      u32 incl = c;\n";
  src += "      #pragma unroll\n";
  src += "      for (int o = 1; o < 32; o <<= 1) {\n";
  src += "        const u32 t = __shfl_up_sync(GDV_FULL, incl, o);\n";
  src += "        if (lane >= (u32)o) incl += t;\n";
  src += "      }\n";
  src += "      step_excl[w] = run + incl - c;\n";
  src += "      run += __shfl_sync(GDV_FULL, incl, 31);\n";
  src += "    }\n";
  src += "    if (lane == 0u) s_wcount[wid] = run;\n";
  src += "    __syncthreads();\n";
  src += "    if (wid == 0u) {\n";
  src += "      const u32 wc = lane < " + sNW + "u ? s_wcount[lane] : 0u;\n";
  src += "      u32 winc = wc;\n";
  src += "      #pragma unroll\n";
  src += "      for (int o = 1; o < 32; o <<= 1) {\n";
  src += "        const u32 t = __shfl_up_sync(GDV_FULL, winc, o);\n";
  src += "        if (lane >= (u32)o) winc += t;\n";
  src += "      }\n";
  src += "      const u32 total = __shfl_sync(GDV_FULL, winc, 31);\n";
  src += "      if (lane < " + sNW + "u) s_wcount[lane] = winc - wc;\n";
  src += "      const u64 excl = gdv_tile_exclusive_prefix(A.tile_state, tile, (u64)total, lane);\n";
  src += "      if (lane == 0u) {\n";
  src += "        s_excl = excl;\n";
  src += "        if (tile == n_tiles - 1) *A.out_count = excl + (u64)total;\n";
  src += "      }\n";
  src += "    }\n";
  src += "    __syncthreads();\n";
  src += "    const u64 wpos = s_excl + (u64)s_wcount[wid];\n";
  // The whole run of this warp fits the vector (always, unless GDV_SEL_BOUNDED): 32-bit offsets
  // from one 64-bit base and no per-row capacity test.
  src += "    if (run != 0u && wpos + (u64)run <= (u64)A.out_cap) {\n";
  src += "      " + IDX + "* const wout = out_idx + wpos;\n";
  src += "      #pragma unroll\n";
  src += "      for (int w = 0; w < " + sW + "; ++w) {\n";
  src += "        if (__ballot_sync(GDV_FULL, mymask[w] != 0u) == 0u) continue;\n";
  src += "        #pragma unroll 4\n";
  src += "        for (int k = 0; k < 32; ++k) {\n";
  src += "          const u32 m = __shfl_sync(GDV_FULL, mymask[w], k);\n";
  src += "          if (m == 0u) continue;  // warp-uniform: most steps of a selective filter keep nothing\n";
  src += "          const u32 off = __shfl_sync(GDV_FULL, step_excl[w], k);\n";
  src += "          if ((m >> lane) & 1u)\n";
  src += "            wout[off + (u32)__popc(m & lt)] = (" + IDX + ")(A.row_base + wbase0 + 1024 * w + 32 * k + (i64)lane);\n";
  src += "        }\n";
  src += "      }\n";
  src += "    } else if (run != 0u) {\n";
  src += "      #pragma unroll\n";
  src += "      for (int w = 0; w < " + sW + "; ++w) {\n";
  src += "        #pragma unroll 1\n";
  src += "        for (int k = 0; k < 32; ++k) {\n";
  src += "          const u32 m = __shfl_sync(GDV_FULL, mymask[w], k);\n";
  src += "          if (m == 0u) continue;\n";
  src += "          const u32 off = __shfl_sync(GDV_FULL, step_excl[w], k);\n";
  src += "          const u64 pos = wpos + (u64)off + (u64)__popc(m & lt);\n";
  src += "          if (((m >> lane) & 1u) && pos < (u64)A.out_cap)\n";
  src += "            out_idx[pos] = (" + IDX + ")(A.row_base + wbase0 + 1024 * w + 32 * k + (i64)lane);\n";
  src += "        }\n";
  src += "      }\n";
  src += "    }\n";
}

// ---- key-driven string filter ---------------------------------------------------------------------
// A filter whose condition implies "column J contains KEY" (BodyGen::PlanKey) does not have to look
// at rows: every warp streams the BYTES of its 1024 rows (one contiguous run of the Arrow data
// buffer) straight from global memory, 4 x 16 bytes per lane in flight, and tests aligned machine
// words against the key's bytes:
//   * KEY of >= 7 bytes: wherever it starts, one of its aligned 4-byte words is key[o .. o+4) for
//     o = start phase 0..3: four compares per loaded word, nothing else (no case-fold arithmetic
//     beyond one OR, no cross-word shifts);
//   * KEY of 3..6 bytes: the same with aligned halfwords (key[o .. o+2), o = 0, 1), verified against
//     the whole key before it counts (two bytes alone are too common).
// A match is only an *anchor*: its byte position goes to a small per-warp list; when the list fills
// or the run ends, the lanes take one anchor each, bisect the row it lies in (int32 offsets of the
// warp's 1024 rows), and evaluate the FULL condition for that row with the ordinary per-row body
// (substr, upper, the exact LIKE matcher, other conjuncts, validity).  Rows without an anchor cost
// no instruction and their offsets are never read.  Bytes that share a 16-byte chunk with memory
// outside the column (first / last chunk of the batch) are not loaded as chunks: every such byte is
// an anchor.  More anchors than the list holds between two drains: the warp evaluates all its rows.
std::string EmitKeyFilter(const std::vector<ColumnSlot>& slots, const KernelSpec& spec,
                          const KeyPlan& plan, const std::string& body, const Val& result, int BT, int W,
                          const std::string& scratch_decl) {
  const int NW = BT / 32;
  const int L = static_cast<int>(plan.key.size());
  const bool words = L >= 7;
  const int unit = words ? 4 : 2;  // bytes per tested unit = start phases that need their own pattern
  auto is_letter = [](unsigned char c) { return (c >= 'a' && c <= 'z') || (c >= 'A' && c <= 'Z'); };
  // pattern of phase o: the rarest unit among key[o + unit * j ..) (they share the alignment)
  std::vector<unsigned> pats, folds;
  std::vector<int> pat_at;
  for (int o = 0; o < unit; ++o) {
    int best_at = o;
    double best = 1e300;
    for (int at = o; at + unit <= L; at += unit) {
      double sc = 0.0;
      for (int i = 0; i + 1 < unit; ++i)
        sc += BodyGen::PairScore(static_cast<unsigned char>(plan.key[static_cast<size_t>(at + i)]),
                                   static_cast<unsigned char>(plan.key[static_cast<size_t>(at + i + 1)]), plan.xf);
      if (sc < best) {
        best = sc;
        best_at = at;
      }
    }
    unsigned pat = 0u, fold = 0u;
    for (int i = 0; i < unit; ++i) {
      const unsigned char c = static_cast<unsigned char>(plan.key[static_cast<size_t>(best_at + i)]);
      const unsigned f = (plan.xf != 0u && is_letter(c)) ? 0x20u : 0u;
      pat |= static_cast<unsigned>(c | f) << (8 * i);
      fold |= f << (8 * i);
    }
    pats.push_back(pat);
    folds.push_back(fold);
    pat_at.push_back(best_at);
  }
  auto hex = [](unsigned v) {
    char b[16];
    std::snprintf(b, sizeof(b), "0x%08xu", v);
    return std::string(b);
  };
  // mask function: bit i = unit i of a 16-byte chunk equals some phase pattern.  Branch-free: four
  // compares per word into one predicate (the compiler must not turn them into a decision tree: the
  // lanes of a warp would take different paths through it), one test of the four predicates.
  std::string mk = "// units of a 16-byte chunk (bit i = unit i) that equal a phase pattern of the key '" +
                   CommentSafe(plan.key) + "'\n";
  const char* comp[4] = {"v.x", "v.y", "v.z", "v.w"};
  if (words) {
    mk += "__device__ __forceinline__ u32 gdv_key_word(u32 x) {\n";
    std::string e;
    for (int o = 0; o < unit; ++o)
      e += (o ? " | " : "") + std::string("(u32)((x") + (folds[o] ? " | " + hex(folds[o]) : "") + ") == " + hex(pats[o]) + ")";
    mk += "  return " + e + ";\n}\n";
    mk += "__device__ __forceinline__ u32 gdv_key_mask(const uint4& v) {\n";
    mk += "  const u32 a = gdv_key_word(v.x), b = gdv_key_word(v.y), c = gdv_key_word(v.z), d = gdv_key_word(v.w);\n";
    mk += "  return a | (b << 1) | (c << 2) | (d << 3);\n}\n";
    // the streaming loop only needs "some unit of the chunk matches": 16 compares chained into ONE predicate
    std::string eb;
    for (int o = 0; o < unit; ++o)
      eb += (o ? " | " : "") + std::string("((x") + (folds[o] ? " | " + hex(folds[o]) : "") + ") == " + hex(pats[o]) + ")";
    mk += "__device__ __forceinline__ bool gdv_key_wordb(u32 x) {\n  return " + eb + ";\n}\n";
    mk += "__device__ __forceinline__ bool gdv_key_any(const uint4& v) {\n";
    mk += "  return gdv_key_wordb(v.x) | gdv_key_wordb(v.y) | gdv_key_wordb(v.z) | gdv_key_wordb(v.w);\n}\n";
  } else {
    mk += "__device__ __forceinline__ u32 gdv_key_mask(const uint4& v) {\n";
    mk += "  u32 h[4];\n";
    for (int wi = 0; wi < 4; ++wi) {
      std::string e;
      for (int o = 0; o < unit; ++o) {
        const unsigned p2 = pats[o] | (pats[o] << 16), f2 = folds[o] | (folds[o] << 16);
        e += (o ? " | " : "") + std::string("gdv_eqhalf_msb(") + comp[wi] + (f2 ? " | " + hex(f2) : "") + ", " + hex(p2) + ")";
      }
      mk += "  h[" + std::to_string(wi) + "] = " + e + ";\n";
    }
    // 0x8000 flags halfword 0, 0x80000000 halfword 1 (the upper one may be flagged falsely: anchors are verified)
    mk += "  if ((h[0] | h[1] | h[2] | h[3]) == 0u) return 0u;\n";
    mk += "  u32 m = 0u;\n";
    mk += "  #pragma unroll\n";
    mk += "  for (int i = 0; i < 4; ++i) m |= (((h[i] >> 15) & 1u) | ((h[i] >> 30) & 2u)) << (2 * i);\n";
    mk += "  return m;\n}\n";
    mk += "__device__ __forceinline__ bool gdv_key_any(const uint4& v) {\n";
    std::string eh;
    for (int wi = 0; wi < 4; ++wi)
      for (int o = 0; o < unit; ++o) {
        const unsigned p2 = pats[o] | (pats[o] << 16), f2 = folds[o] | (folds[o] << 16);
        eh += (eh.empty() ? "" : " | ") + std::string("gdv_eqhalf_msb(") + comp[wi] + (f2 ? " | " + hex(f2) : "") + ", " + hex(p2) + ")";
      }
    mk += "  return (" + eh + ") != 0u;\n}\n";
  }

  // the condition of ONE row per lane: EmitGroup's per-row path with `base` chosen so that row s is
  // the anchor's row (lanes without one get s = A.n, i.e. out of range)
  std::string pred;
  EmitGroup(slots, spec, false, 1, kPred, body,
            "              { keep = in && (" + result.ok + ") && (" + result.v + "); }\n", &pred, 7);
  std::string k = mk + R"K(extern "C" __global__ void __launch_bounds__(@BT@, @MINB@) @NAME@(const __grid_constant__ gdv_args A) {
  const u32 lane = threadIdx.x & 31u;
  const u32 wid = threadIdx.x >> 5;
  gdv_ctx ctx;
  ctx.err = A.err;
@PROLOGUE@  extern __shared__ uint4 gdv_smem[];
  u32* const wmask = reinterpret_cast<u32*>(gdv_smem) + (size_t)wid * (@CAP@ + 32 * @W@ + 4);  // keep-mask of step k of this warp's rows
  u32* const wctr = wmask + 32 * @W@;      // [0] anchors queued since the last drain
  u32* const wanch = wmask + 32 * @W@ + 4; // their byte positions in the column's data buffer
  __shared__ u32 s_wcount[@NW@];
  __shared__ i64 s_tile;
  __shared__ u64 s_excl;
  const @OFFT@* const offs = in_val@J@;
  const u8* const data = in_var@J@;
  const i64 n_tiles = (A.n + @TILE@ - 1) / @TILE@;
  const i64 B0 = (i64)offs[0], B1 = (i64)offs[A.n];
  // chunk c holds the bytes [16 c - mis, 16 c - mis + 16) of the data buffer
  const i64 mis = (i64)((unsigned long long)data & 15ull);
  const uint4* const abase = reinterpret_cast<const uint4*>(data - mis);
  const i64 c_safe_lo = (B0 + mis + 15) >> 4;  // chunks that lie entirely inside the column's bytes
  const i64 c_safe_hi = (B1 + mis) >> 4;
  @IDX@* out_idx = reinterpret_cast<@IDX@*>(A.out_idx);
  const u32 lt = gdv_lanemask_lt();
  while (true) {
    if (threadIdx.x == 0) s_tile = (i64)atomicAdd(A.ticket, 1ull);
    __syncthreads();
    const i64 tile = s_tile;
    if (tile >= n_tiles) break;
    // every warp owns @W@ consecutive 1024-row chunks: one run of bytes, one anchor list, one drain
    const i64 wbase0 = tile * @TILE@ + (i64)wid * (1024 * @W@);
    #pragma unroll
    for (int w = 0; w < @W@; ++w) wmask[32 * w + lane] = 0u;
    if (lane == 0u) wctr[0] = 0u;
    __syncwarp();
    if (wbase0 < A.n) {
      const i64 r0 = wbase0;
      const i64 r1 = r0 + 1024 * @W@ < A.n ? r0 + 1024 * @W@ : A.n;
      const i64 b0 = (i64)offs[r0], b1 = (i64)offs[r1];
      auto push = [&](i64 pos) {
        const u32 ix = atomicAdd(wctr, 1u);
        if (ix < @CAP@u) wanch[ix] = (u32)@ANCHOR@;
      };
      // bytes of this run that share a chunk with memory outside the column: every one is an anchor
      i64 c_lo = (b0 + mis) >> 4, c_hi = (b1 + mis + 15) >> 4;
      if (c_lo < c_safe_lo) {
        const i64 e = b1 < (c_safe_lo << 4) - mis ? b1 : (c_safe_lo << 4) - mis;
        for (i64 q = b0 + (i64)lane; q < e; q += 32) push(q);
        c_lo = c_safe_lo;
      }
      if (c_hi > c_safe_hi) {
        const i64 s = b0 > (c_safe_hi << 4) - mis ? b0 : (c_safe_hi << 4) - mis;
        for (i64 q = s + (i64)lane; q < b1; q += 32) push(q);
        c_hi = c_safe_hi;
      }
      // Blocks of 128 chunks (2 KB): 4 x 16 bytes in flight per lane; 32-bit chunk indices relative to
      // the run's first chunk, positions are only formed for the (rare) matches.  After every block
      // the queued anchors are drained if the list is half full (or the run is over): one anchor per
      // lane, row of the anchor, then the full condition for that row — the only copy of the per-row
      // body in this kernel.  Should a block ever queue more anchors than the list holds (every word
      // of it a match), the warp goes over its rows a second time, 128 rows per step, with the first
      // byte of every non-empty row as its anchor.
      const uint4* const cp = abase + c_lo + (i64)lane;
      const i32 nch = @NCH@;
      i32 ci = 0;
      i64 redo_row = r0;
      bool redo = false, lost = @LOST@;
      while (true) {
        bool last;
        if (!redo) {
          // four blocks (8 KB) between two looks at the anchor list: the warp-wide hand-shake below
          // costs as much as a quarter of a block's compares
          #pragma unroll 1
          for (int rep = 0; rep < 4 && ci < nch; ++rep, ci += 128) {
            bool any[4];
            if (ci + 128 <= nch) {
              uint4 v[4];
              #pragma unroll
              for (int u = 0; u < 4; ++u) v[u] = __ldcs(cp + ci + 32 * u);
              #pragma unroll
              for (int u = 0; u < 4; ++u) any[u] = gdv_key_any(v[u]);
            } else {
              #pragma unroll
              for (int u = 0; u < 4; ++u) {
                any[u] = false;
                if (ci + 32 * u + (i32)lane < nch) any[u] = gdv_key_any(__ldcs(cp + ci + 32 * u));
              }
            }
            if (any[0] | any[1] | any[2] | any[3]) {
              #pragma unroll 1
              for (int u = 0; u < 4; ++u) {
                if (!any[u]) continue;
                // the chunk is read again (it is in L2 / L1): keeping 64 loaded bytes per lane alive for
                // this rare path would cost the streaming loop 16 registers
                u32 mm = gdv_key_mask(__ldg(cp + ci + 32 * u));
                while (mm != 0u) {
                  const int bit = __ffs((int)mm) - 1;
                  mm &= mm - 1u;
                  const i64 pos = ((c_lo + (i64)(ci + 32 * u) + (i64)lane) << 4) - mis + @UNIT@ * bit;
@VERIFY@                  push(pos);
                }
              }
            }
          }
          last = ci >= nch;
        } else {
          #pragma unroll
          for (int u = 0; u < 4; ++u) {
            const i64 row = redo_row + 32 * u + (i64)lane;
            if (row < r1) {
@REDO_PUSH@            }
          }
          redo_row += 128;
          last = redo_row >= r1;
        }
        __syncwarp();
        // one lane reads the count and broadcasts it: a lane that read it on its own could see the
        // pushes faster lanes already make for the next block
        const u32 queued = __shfl_sync(GDV_FULL, wctr[0], 0);
        if (queued >= @CAP@u / 2u || (last && queued != 0u)) {
          if (queued > @CAP@u) lost = true;
          const u32 nc = queued < @CAP@u ? queued : @CAP@u;
          for (u32 i0 = 0u; i0 < nc; i0 += 32u) {
            const bool has = i0 + lane < nc;
@DRAIN_ROW@            bool keep = false;
            {
              const i64 base = (cand ? lo : A.n) - (i64)lane;
@PRED@            }
            if (keep) atomicOr(&wmask[rr >> 5], 1u << (rr & 31u));
          }
          __syncwarp();
          if (lane == 0u) wctr[0] = 0u;
          __syncwarp();
        }
        if (last) {
          if (redo || !lost) break;
          redo = true;
        }
      }
    }
    u32 mymask[@W@];
    #pragma unroll
    for (int w = 0; w < @W@; ++w) mymask[w] = wmask[32 * w + lane];
    __syncwarp();
@EPILOGUE@  }
}
)K";
  // halfword mode: an anchor counts only if the whole key is there (two bytes alone are too common):
  // the matched halfword is key[at .. at+2) for the phase pattern it equals, so the key would start
  // at pos - at for one of the (at most two) pattern offsets
  std::string verify;
  if (!words) {
    std::string e;
    for (int i = 0; i < L; ++i)
      e += (i ? " && " : "") + std::string("gdv_ch_eq(kv, ") + std::to_string(i) + ", " +
           std::to_string(static_cast<unsigned>(static_cast<unsigned char>(plan.key[static_cast<size_t>(i)]))) + "u)";
    verify += "            {\n";
    verify += "              bool hit = false;\n";
    for (int o = 0; o < unit; ++o) {
      if (o == 1 && pat_at[1] == pat_at[0]) continue;
      verify += "              {\n";
      verify += "                const i64 st = pos - " + std::to_string(pat_at[static_cast<size_t>(o)]) + ";\n";
      verify += "                if (st >= B0 && st + " + std::to_string(L) + " <= B1) {\n";
      verify += "                  gdv_str kv = gdv_make_str(data + st, " + std::to_string(L) + ");\n";
      verify += "                  kv.xf = " + std::to_string(plan.xf) + "u;\n";
      verify += "                  if (" + e + ") hit = true;\n";
      verify += "                }\n";
      verify += "              }\n";
    }
    verify += "              if (!hit) continue;\n";
    verify += "            }\n";
  }
  std::string prologue, epilogue;
  EmitPrologue(slots, spec, false, &prologue);
  prologue += scratch_decl;
  EmitFilterEpilogue(slots, spec, NW, W, SelCType(spec.selection_mode), &epilogue);
  ReplaceAll(&k, "@PROLOGUE@", prologue);
  ReplaceAll(&k, "@EPILOGUE@", epilogue);
  ReplaceAll(&k, "@PRED@", pred);
  ReplaceAll(&k, "@VERIFY@", verify);
  ReplaceAll(&k, "@BT@", std::to_string(BT));
  // the streaming loop needs ~40 registers; the per-row body (rare) may spill: ask for 48 warps per SM
  ReplaceAll(&k, "@MINB@", std::to_string(std::max(1, 1536 / BT)));
  ReplaceAll(&k, "@NW@", std::to_string(NW));
  ReplaceAll(&k, "@NAME@", spec.name);
  ReplaceAll(&k, "@CAP@", std::to_string(kKeyAnchorCap));
  ReplaceAll(&k, "@J@", std::to_string(plan.slot));
  ReplaceAll(&k, "@TILE@", std::to_string(static_cast<long long>(NW) * 1024 * W) + "ll");
  ReplaceAll(&k, "@W@", std::to_string(W));
  ReplaceAll(&k, "@IDX@", SelCType(spec.selection_mode));
  ReplaceAll(&k, "@UNIT@", std::to_string(unit));
  // Anchor positions are u32.  A utf8 / binary column's are absolute; a large column's are relative to
  // the warp's run base b0, and in the fallback (redo) the list holds rows relative to r0 instead of
  // first bytes, so no position past the u32 range is ever stored.  A run longer than a u32 position
  // can address skips the streaming loop and goes to the fallback: every row of the run is evaluated.
  const bool large = slots[static_cast<size_t>(plan.slot)].type.is_large();
  ReplaceAll(&k, "@OFFT@", large ? "i64" : "i32");
  ReplaceAll(&k, "@ANCHOR@", large ? "(pos - b0)" : "pos");
  ReplaceAll(&k, "@NCH@", large ? "c_hi > c_lo && b1 - b0 <= 0xffffffffll ? (i32)(c_hi - c_lo) : 0"
                                : "c_hi > c_lo ? (i32)(c_hi - c_lo) : 0");
  ReplaceAll(&k, "@LOST@", large ? "b1 - b0 > 0xffffffffll" : "false");
  if (large) {
    ReplaceAll(&k, "@REDO_PUSH@",
               "              if (__ldg(offs + row + 1) > __ldg(offs + row)) push(b0 + (row - r0));  // stores row - r0\n");
    ReplaceAll(&k, "@DRAIN_ROW@",
               "            const i64 pos = has ? b0 + (i64)wanch[i0 + lane] : b0;\n"
               "            // fallback: the list holds rows; else the last row r in [r0, r1) with offs[r] <= pos\n"
               "            // (offsets are non-decreasing; empty rows are skipped)\n"
               "            i64 lo = r0, hi = r1;\n"
               "            if (redo) {\n"
               "              lo = r0 + (pos - b0);\n"
               "            } else {\n"
               "              while (hi - lo > 1) {\n"
               "                const i64 mid = (lo + hi) >> 1;\n"
               "                if (__ldg(offs + mid) <= pos) lo = mid;\n"
               "                else hi = mid;\n"
               "              }\n"
               "            }\n"
               "            const u32 rr = (u32)(lo - r0);\n"
               "            const bool cand = has && (redo ? lo < r1 : pos >= b0 && pos < b1) &&\n"
               "                              ((wmask[rr >> 5] >> (rr & 31u)) & 1u) == 0u;\n");
  } else {
    ReplaceAll(&k, "@REDO_PUSH@", R"K(              const i32 a = __ldg(offs + row);
              if (__ldg(offs + row + 1) > a) push((i64)a);
)K");
    ReplaceAll(&k, "@DRAIN_ROW@", R"K(            const i64 pos = has ? (i64)wanch[i0 + lane] : b0;
            // last row r in [r0, r1) with offs[r] <= pos (offsets are non-decreasing; empty rows are skipped)
            i64 lo = r0, hi = r1;
            while (hi - lo > 1) {
              const i64 mid = (lo + hi) >> 1;
              if ((i64)__ldg(offs + mid) <= pos) lo = mid;
              else hi = mid;
            }
            const u32 rr = (u32)(lo - r0);
            const bool cand = has && pos >= b0 && pos < b1 && ((wmask[rr >> 5] >> (rr & 31u)) & 1u) == 0u;
)K");
  }
  return k;
}

// Projector kernels that read their rows through a selection vector may get the slot count from
// device memory (gdv_selection_t.d_num_slots: the count a Filter left there, so that a Filter ->
// Projector chain never returns to the host): every use of A.n in the kernel body becomes gdv_n, the
// smaller of *A.n_ptr and A.n (the host-side upper bound the grid was sized with).
void ApplyDeviceCount(std::string* src) {
  const std::string sig = "(const __grid_constant__ gdv_args A) {\n";
  const size_t at = src->find(sig);
  if (at == std::string::npos) return;
  const size_t body = at + sig.size();
  std::string tail = src->substr(body);
  std::string out;
  out.reserve(tail.size() + 64);
  for (size_t i = 0; i < tail.size();) {
    if (tail.compare(i, 3, "A.n") == 0 && (i + 3 >= tail.size() || !(std::isalnum(static_cast<unsigned char>(tail[i + 3])) || tail[i + 3] == '_'))) {
      out += "gdv_n";
      i += 3;
    } else {
      out.push_back(tail[i++]);
    }
  }
  *src = src->substr(0, body) +
         "  const i64 gdv_n = A.n_ptr != nullptr ? ((i64)*A.n_ptr < A.n ? (i64)*A.n_ptr : A.n) : A.n;\n" + out;
}

// Filter kernels: columns whose NULL makes the condition not-true (BodyGen::TruthStrict) have their
// validity ANDed into the keep-mask one 32-row word at a time after the row loop; inside the loop
// they count as valid (no function of the kernel can raise, so a null slot's value is harmless).
void MarkHoisted(const BodyGen& gen, const Node& cond, std::vector<ColumnSlot>* slots) {
  std::vector<int> strict;
  gen.TruthStrict(cond, &strict);
  for (auto& sl : *slots)  // a dictionary / view / large row's validity also depends on its entry / view / length
    if (!sl.type.is_dict() && !sl.type.is_view() && !sl.type.is_large() && std::find(strict.begin(), strict.end(), sl.schema_index) != strict.end())
      sl.hoist = true;
}

// The schema columns a tree reads, each once, in the order of their first use.
void CollectColumns(const Schema& schema, const Node& node, std::vector<int>* cols) {
  if (node.kind() == NodeKind::kField) {
    const int i = schema.index_of(static_cast<const FieldNode&>(node).name());
    if (std::find(cols->begin(), cols->end(), i) == cols->end()) cols->push_back(i);
  }
  for (const auto& c : Children(node)) CollectColumns(schema, *c, cols);
}

void SpineConjuncts(const Node& node, std::vector<const Node*>* out) {
  if (node.kind() == NodeKind::kBoolean && static_cast<const BooleanNode&>(node).op() == BooleanNode::kAnd) {
    for (const auto& c : static_cast<const BooleanNode&>(node).children()) SpineConjuncts(*c, out);
    return;
  }
  out->push_back(&node);
}

// Stage plan of a Filter condition over `slots`, or false when gating does not apply: some column
// is not a plain fixed-width value (string, dictionary, view, bit-packed bool), the condition can
// raise (errors must come from every row that holds the value), it has a single stage, or its first
// stage reads more than half of the row's bytes.
bool PlanGate(const Schema& schema, const Node& cond, const std::vector<ColumnSlot>& slots, GatePlan* plan) {
  if (BodyGen::CanFail(cond)) return false;
  for (const auto& sl : slots)
    if (sl.type.is_varlen() || sl.type.is_bool()) return false;  // dictionaries and views are varlen
  std::vector<const Node*> conj;
  SpineConjuncts(cond, &conj);
  // a conjunct waits for the last of its columns
  std::vector<int> level(conj.size(), 0);
  for (size_t c = 0; c < conj.size(); ++c) {
    std::vector<int> cols;
    CollectColumns(schema, *conj[c], &cols);
    for (int col : cols) {
      int j = -1;
      for (size_t s = 0; s < slots.size(); ++s)
        if (slots[s].schema_index == col) j = static_cast<int>(s);
      if (j < 0) return false;
      level[c] = std::max(level[c], j);
    }
  }
  std::vector<int> ends(level);
  std::sort(ends.begin(), ends.end());
  ends.erase(std::unique(ends.begin(), ends.end()), ends.end());
  if (ends.size() < 2 || ends.back() != static_cast<int>(slots.size()) - 1) return false;
  // The gated stages must carry most of the row: when stage 0 already reads more than half of the
  // row's bytes, the most gating can save is less than the dependent round trip each later stage
  // adds (`d * 100 < q AND date in range`: 16 of 20 B in stage 0, 7 % slower gated on an H100).
  int row_bytes = 0, first_bytes = 0;
  for (size_t s = 0; s < slots.size(); ++s) {
    row_bytes += std::max(slots[s].type.width(), 1);
    if (static_cast<int>(s) <= ends[0]) first_bytes += std::max(slots[s].type.width(), 1);
  }
  if (2 * first_bytes > row_bytes) return false;
  plan->first_slot.assign(1, 0);
  plan->conjuncts.assign(ends.size(), {});
  for (size_t s = 0; s < ends.size(); ++s) {
    plan->first_slot.push_back(ends[s] + 1);
    for (size_t c = 0; c < conj.size(); ++c)
      if (level[c] == ends[s]) plan->conjuncts[s].push_back(conj[c]);
  }
  return true;
}

int PickRowsPerThread(int in_bytes, int out_bytes, KernelKind kind) {
  // The map kernels want ~160-190 bytes of loads in flight per thread to cover HBM latency
  // (add int32: R=16, Q6 predicate: R=8); the filter, whose tile is large
  // and whose compaction tail needs registers, is best at R=2..4.
  (void)out_bytes;
  const int bytes = std::max(in_bytes, 1);
  int r = kind == KernelKind::kFilter ? 96 / bytes : 192 / bytes;
  r = std::max(kind == KernelKind::kFilter ? 2 : 1, std::min(r, kind == KernelKind::kFilter ? 8 : 16));
  int p = 1;
  while (p * 2 <= r) p *= 2;
  return p;
}

// ---- pieces every kernel generator shares -------------------------------------------------------
// A BodyGen over `slots` as `spec` configures it: string_scan bit 0 turns the cooperative LIKE scan
// off, bit 3 the inline / prefix shortcut over string_view / binary_view views.
BodyGen SpecBodyGen(const Schema& schema, std::vector<ColumnSlot>* slots, const KernelSpec& spec) {
  return BodyGen(schema, slots, spec.nullable, (spec.string_scan & 1) == 0, (spec.string_scan & 8) == 0);
}

// Algorithmic bytes (values only) a kernel over `slots` reads per row.
int InBytesPerRow(const std::vector<ColumnSlot>& slots) {
  int bytes = 0;
  for (const auto& s : slots)
    bytes += s.type.is_dict() ? DataType(s.type.index).width()  // the index; the dictionary is cached
             : s.type.is_view()   ? 16                               // the view; out-of-line bytes on demand
             : s.type.is_large()  ? 36                               // 8 B offset + ~28 B data
             : s.type.is_varlen() ? 32 : std::max(s.type.width(), 1);  // 4 B offset + ~28 B data
  return bytes;
}

// The fields of `out` that follow from the spec and the kernel's input slots, among them the layout
// of the argument block the kernel is emitted with and the host packs.
void DescribeKernel(const KernelSpec& spec, const std::vector<ColumnSlot>& slots, int n_out, GeneratedKernel* out) {
  out->name = spec.name;
  out->kind = spec.kind;
  out->selection_mode = spec.selection_mode;
  out->nullable = spec.nullable;
  out->inputs = slots;
  out->in_bytes_per_row = InBytesPerRow(slots);
  out->args = ArgsLayout(static_cast<int>(slots.size()), n_out, HasDictionary(slots), HasView(slots));
}

// The comment lines a kernel's source starts with.
std::string HeaderLines(const std::string& shape, const KernelSpec& spec, const std::vector<ExpressionPtr>& exprs) {
  std::string h = "// generated by gandiva_b200 kernel fuser; " + shape;
  h += spec.nullable ? " (inputs may carry validity bitmaps)\n" : " (no input has nulls)\n";
  for (size_t i = 0; i < exprs.size(); ++i)
    h += "// expr_" + std::to_string(i) + ": " + CommentSafe(exprs[i]->ToString()) + "\n";
  return h;
}

// A kernel's text up to its loops: the `header` lines, the device library, the argument block of
// `out`, the globals of `gen`, the signature with launch bounds `bounds`, lane / wid / ctx, the
// prologue and the scratch of `gen` for out.rows_per_thread rows per group.
std::string EmitKernelFrame(const KernelSpec& spec, bool has_sel, const GeneratedKernel& out, const BodyGen& gen,
                            const std::string& header, const std::string& bounds) {
  std::string src = header;
  src += "#include \"gdv_device_lib.cuh\"\n";
  src += EmitArgsStruct(out.args);
  src += gen.globals();
  src += "extern \"C\" __global__ void __launch_bounds__(" + bounds + ") " + spec.name +
         "(const __grid_constant__ gdv_args A) {\n";
  src += "  const u32 lane = threadIdx.x & 31u;\n";
  src += "  const u32 wid = threadIdx.x >> 5;\n";
  src += "  gdv_ctx ctx;\n  ctx.err = A.err;\n";
  EmitPrologue(out.inputs, spec, has_sel, &src);
  src += gen.ScratchDecl(out.rows_per_thread);
  return src;
}

// Shared memory of the string columns (HasByteRun), per warp and column: `stages` stages of 48 B
// per row of a group, then the hit list and counters of the cooperative scan.
struct StringStages {
  int columns = 0;
  int stages = 1;
  int stage_bytes = 0;
  int hit_bytes = 0;  // candidates, hits, two counters
  int block() const { return stages * stage_bytes + hit_bytes; }
  int dynamic_smem(int BT) const { return block() * (BT / 32) * columns; }
};

// Block size and string stages of a row-driven kernel over `slots` with R rows per thread.  Many
// string columns (e.g. a schema extended by materialised ropes, gdv_rope_temps.h): the per-warp stages
// of all of them must fit the CTA's shared memory — fewer rows per thread first, then fewer warps per CTA.
Status FitStages(const KernelSpec& spec, const BodyGen& gen, const std::vector<ColumnSlot>& slots, int n_stages,
                 int* R, int* BT, StringStages* st) {
  int n_varlen = 0;
  for (const auto& s : slots) n_varlen += HasByteRun(s) ? 1 : 0;
  // String predicates are instruction-bound and stage bytes per warp in shared memory: they run
  // 512 threads on big batches; everything else runs 256.
  *BT = spec.block_threads > 0 ? spec.block_threads
                               : (spec.kind == KernelKind::kFilter && n_varlen > 0 && spec.large_batch ? 512 : 256);
  if (*BT % 32 != 0 || *BT > 1024)
    return Status::Make(GDV_INVALID, "block_threads must be a multiple of 32 and <= 1024");
  const int hit = gen.coop_segs().empty() ? 0 : 8 * kHitCap + 16;
  auto need = [&](int r, int bt) { return (n_stages * 48 * 32 * r + hit) * (bt / 32) * n_varlen; };
  const int kMaxStage = 200 * 1024;
  while (need(*R, *BT) > kMaxStage && *R > 1) *R /= 2;
  while (need(*R, *BT) > kMaxStage && *BT > 64 && spec.block_threads == 0) *BT /= 2;
  if (need(*R, *BT) > kMaxStage)
    return Status::Make(GDV_NOT_IMPLEMENTED, "too many utf8/binary columns for one kernel (" + std::to_string(n_varlen) + ")");
  st->columns = n_varlen;
  st->stages = n_stages;
  st->stage_bytes = n_varlen > 0 ? 48 * 32 * *R : 0;
  st->hit_bytes = hit;
  return Status::OK();
}

// Warp `wid`'s stage of every string column (`decl` stage<j><suffix>) and, for the columns the
// cooperative scan reads, its hit list and counters (hctr<j> ... `hctr_end`).
std::string EmitStageDecls(const std::vector<ColumnSlot>& slots, const std::vector<CoopSeg>& coop,
                           const StringStages& st, const std::string& decl, const std::string& suffix,
                           const std::string& hctr_end) {
  std::string o = "  extern __shared__ uint4 gdv_smem[];\n";
  int vi = 0;
  for (size_t j = 0; j < slots.size(); ++j) {
    if (!HasByteRun(slots[j])) continue;
    const std::string J = std::to_string(j), SJ = "stage" + J + suffix;
    o += "  " + decl + SJ + " = reinterpret_cast<u8*>(gdv_smem) + ((size_t)wid * " + std::to_string(st.columns) +
         " + " + std::to_string(vi) + ") * " + std::to_string(st.block()) + ";\n";
    if (SlotHasCoop(coop, static_cast<int>(j))) {
      o += "  u32* cand" + J + " = reinterpret_cast<u32*>(" + SJ + " + " + std::to_string(st.stages * st.stage_bytes) + ");\n";
      o += "  u32* hits" + J + " = cand" + J + " + " + std::to_string(kHitCap) + ";\n";
      o += "  u32* hctr" + J + " = hits" + J + " + " + std::to_string(kHitCap) + hctr_end;
    }
    ++vi;
  }
  return o;
}

// ---- string-producing projections ---------------------------------------------------------------
// One utf8/binary output expression = two kernels around a tile scan (DESIGN.md "String outputs"):
//   gdv_strsize_*  : bytes produced by every CTA tile -> tile_state[tile]
//   gdv_scan_tiles : (static kernel) exclusive scan of tile_state, total -> out_count
//   gdv_strwrite_* : re-evaluates the rows (the values are views, so this is cheap), scans the
//                    row lengths inside the tile, writes the int32 offsets and copies the bytes
//                    (through the view's case map) warp-cooperatively, row by row.
// No CTA waits on another one; the host may read the total between the scan and the write to
// size the data buffer (Projector::Evaluate with host batches does).
Status GenerateStringKernel(const Schema& schema, const ExpressionPtr& expr, const KernelSpec& spec,
                            GeneratedKernel* out) {
  const bool is_size = spec.kind == KernelKind::kStringSize;
  std::vector<ColumnSlot> slots;
  BodyGen gen = SpecBodyGen(schema, &slots, spec);
  std::string body;
  const Val res = gen.Gen(*expr->root(), &body, 4);
  if (!gen.error().empty()) return Status::Make(GDV_NOT_IMPLEMENTED, gen.error());
  int R = spec.rows_per_thread > 0 ? std::min(spec.rows_per_thread, 8) : 2;
  int BT = 0;
  StringStages st;
  const Status fit = FitStages(spec, gen, slots, 1, &R, &BT, &st);
  if (!fit.ok()) return fit;
  const int NW = BT / 32;
  const int T = BT * R;
  const bool has_sel = spec.selection_mode != GDV_SEL_NONE;
  DescribeKernel(spec, slots, 1, out);
  out->rows_per_thread = R;
  out->block_threads = BT;
  const std::string sR = std::to_string(R), s32R = std::to_string(32 * R), sT = std::to_string(T);
  // large_string / large_binary output: int64 offsets, and the running byte counts inside a thread and
  // a warp are u64 (the totals across warps and tiles already are)
  const bool large_out = expr->result().type.is_large();
  const std::string OFF = large_out ? "i64" : "i32", RUN = large_out ? "u64" : "u32";

  std::string header = HeaderLines(is_size ? "string projection, sizing pass" : "string projection, write pass", spec, {expr});
  if (gen.has_replace()) header += "#define GDV_HAS_REPL 1\n";
  std::string src = EmitKernelFrame(spec, has_sel, *out, gen, header, std::to_string(BT));
  if (st.stage_bytes > 0) src += EmitStageDecls(slots, gen.coop_segs(), st, "u8* ", "", ";\n");
  src += "  __shared__ u64 s_part[" + std::to_string(NW) + "];\n";
  if (has_sel && !is_size)  // a device count of 0 leaves no tile to write offsets[0]
    src += "  if (A.n == 0 && blockIdx.x == 0 && threadIdx.x == 0) reinterpret_cast<" + OFF + "*>(A.out_val[0])[0] = 0;\n";
  src += "  const i64 n_tiles = (A.n + " + std::to_string(T - 1) + ") / " + sT + ";\n";
  src += "  for (i64 tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {\n";
  src += "    const i64 base = tile * " + sT + " + (i64)wid * " + s32R + ";\n";
  // a plain string value is a rope of one piece
  std::vector<std::string> parts = res.parts;
  if (parts.empty()) parts.push_back(res.v);
  const int K = static_cast<int>(parts.size());
  const std::string sK = std::to_string(K);
  std::string total_len;
  for (int i = 0; i < K; ++i) total_len += (i ? " + " : "") + std::string("gdv_piece_len(") + parts[i] + ")";
  std::string tail;
  if (is_size) {
    src += "    " + RUN + " tsum = 0u;\n";
    tail = "        tsum += (in && (" + res.ok + ")) ? " + (large_out ? "(u64)(" : "(") + total_len + ") : 0u;\n";
  } else {
    src += "    u32 slen[" + sR + "];\n    gdv_str sv[" + sR + "][" + sK + "];\n    u32 vw0 = 0u;\n";
    tail = "        { const bool okk = in && (" + res.ok + "); slen[k] = okk ? (" + total_len + ") : 0u;\n";
    for (int i = 0; i < K; ++i)
      tail += "          sv[k][" + std::to_string(i) + "] = " + parts[i] + ";\n";
    tail += "          const u32 m = __ballot_sync(GDV_FULL, okk); if (lane == (u32)k) vw0 = m; }\n";
  }
  if (!has_sel) {
    src += "    if (base + " + s32R + " <= A.n) {\n";
    EmitGroup(slots, spec, has_sel, R, kFast, body, tail, &src, 3, st.stage_bytes, std::string(), gen.coop_segs());
    src += "    } else {\n";
    EmitGroup(slots, spec, has_sel, R, kPred, body, tail, &src, 3, 0, std::string(), gen.coop_segs());
    src += "    }\n";
  } else {
    src += "    {\n";
    EmitGroup(slots, spec, has_sel, R, kPred, body, tail, &src, 3, 0, std::string(), gen.coop_segs());
    src += "    }\n";
  }
  if (is_size) {
    src += "    u64 ws = (u64)tsum;\n";
    src += "    for (int o = 16; o > 0; o >>= 1) ws += __shfl_xor_sync(GDV_FULL, ws, o);\n";
    src += "    if (lane == 0u) s_part[wid] = ws;\n";
    src += "    __syncthreads();\n";
    src += "    if (threadIdx.x == 0) {\n";
    src += "      u64 t = 0ull;\n";
    src += "      for (int w = 0; w < " + std::to_string(NW) + "; ++w) t += s_part[w];\n";
    src += "      A.tile_state[tile] = t;\n";
    src += "    }\n";
    src += "    __syncthreads();\n";
  } else {
    // lengths -> inclusive offsets inside the warp (row order: step k, then lane), then across warps
    src += "    " + RUN + " incl[" + sR + "];\n";
    src += "    " + RUN + " run = 0u;\n";
    src += "    #pragma unroll\n";
    src += "    for (int k = 0; k < " + sR + "; ++k) {\n";
    src += "      " + RUN + " x = slen[k];\n";
    src += "      #pragma unroll\n";
    src += "      for (int o = 1; o < 32; o <<= 1) {\n";
    src += "        const " + RUN + " t = __shfl_up_sync(GDV_FULL, x, o);\n";
    src += "        if (lane >= (u32)o) x += t;\n";
    src += "      }\n";
    src += "      incl[k] = run + x;\n";
    src += "      run += __shfl_sync(GDV_FULL, x, 31);\n";
    src += "    }\n";
    src += "    if (lane == 0u) s_part[wid] = (u64)run;\n";
    src += "    __syncthreads();\n";
    src += "    u64 wbase = A.tile_state[tile];\n";
    src += "    for (u32 w = 0u; w < wid; ++w) wbase += s_part[w];\n";
    src += "    __syncthreads();\n";
    src += "    " + OFF + "* offs = reinterpret_cast<" + OFF + "*>(A.out_val[0]);\n";
    src += "    u8* data = A.out_var[0];\n";
    src += "    #pragma unroll\n";
    src += "    for (int k = 0; k < " + sR + "; ++k) {\n";
    src += "      const i64 s = base + 32 * k + (i64)lane;\n";
    src += "      if (s < A.n) offs[s + 1] = (" + OFF + ")(wbase + (u64)incl[k]);\n";
    src += "    }\n";
    src += "    if (tile == 0 && threadIdx.x == 0) offs[0] = 0;\n";
    src += "    #pragma unroll\n";
    src += "    for (int k = 0; k < " + sR + "; ++k) {\n";
    src += "      u64 dst0 = wbase + (u64)(incl[k] - slen[k]);\n";
    src += "      const bool rowok = slen[k] != 0u;\n";
    src += "      #pragma unroll\n";
    src += "      for (int piece = 0; piece < " + sK + "; ++piece) {\n";
    src += "        const u32 plen = rowok ? gdv_piece_len(sv[k][piece]) : 0u;\n";
    src += "        // text in a thread-private scratch slot is copied by its owner, everything else by the warp\n";
    src += "        const bool mine_only = (sv[k][piece].xf & (GDV_XF_LOCAL | GDV_XF_REV | GDV_XF_REPL)) != 0u;\n";
    src += "        if (plen != 0u && mine_only) {\n";
    src += "          if (dst0 + (u64)plen <= (u64)A.out_cap) {\n";
    src += "            if ((sv[k][piece].xf & GDV_XF_REPL) != 0u) gdv_repl_copy(data + dst0, sv[k][piece]);\n";
    src += "            else if ((sv[k][piece].xf & GDV_XF_REV) != 0u) gdv_copy_reversed(data + dst0, sv[k][piece]);\n";
    src += "            else for (u32 i = 0u; i < plen; ++i) data[dst0 + (u64)i] = gdv_piece_byte(sv[k][piece], (i32)i);\n";
    src += "          } else {\n";
    src += "            gdv_set_error(&ctx, GDV_ERR_VAR_CAPACITY);\n";
    src += "          }\n";
    src += "        }\n";
    src += "        const u32 nonempty = __ballot_sync(GDV_FULL, plen != 0u && !mine_only);\n";
    src += "        for (u32 rest = nonempty; rest != 0u; rest &= rest - 1u) {\n";
    src += "          const int j = __ffs((int)rest) - 1;\n";
    src += "          gdv_str v;\n";
    src += "          v.p = reinterpret_cast<const u8*>(__shfl_sync(GDV_FULL, (u64)sv[k][piece].p, j));\n";
    src += "          v.len = (i32)__shfl_sync(GDV_FULL, plen, j);\n";
    src += "          v.xf = __shfl_sync(GDV_FULL, sv[k][piece].xf, j);\n";
    src += "          const u64 d = __shfl_sync(GDV_FULL, dst0, j);\n";
    src += "          if (d + (u64)v.len <= (u64)A.out_cap) {\n";
    src += "            for (i32 i = (i32)lane; i < v.len; i += 32) data[d + (u64)i] = gdv_piece_byte(v, i);\n";
    src += "          } else if (lane == 0u) {\n";
    src += "            gdv_set_error(&ctx, GDV_ERR_VAR_CAPACITY);\n";
    src += "          }\n";
    src += "        }\n";
    src += "        dst0 += (u64)plen;\n";
    src += "      }\n";
    src += "    }\n";
    src += "    if (lane < " + sR + "u && base + 32 * (i64)lane < A.n && A.out_vld[0] != nullptr)\n";
    src += "      A.out_vld[0][(base >> 5) + (i64)lane] = vw0;\n";
    src += "    __syncwarp();  // the views may point into this warp's stage: done before it is refilled\n";
  }
  src += "  }\n";
  src += "}\n";
  // selection-vector projectors may read the slot count from device memory: both passes then cover
  // the device count's tiles and rows only (the scan stops at the same tile, gdv_scan_tiles)
  if (has_sel) ApplyDeviceCount(&src);

  out->source = std::move(src);
  out->outputs = {expr->result().type};
  out->uses_ctx = gen.uses_ctx() || !is_size;
  out->out_bytes_per_row = large_out ? 8 : 4;
  out->dynamic_smem = st.dynamic_smem(BT);
  out->tile_rows = T;
  out->cta_tile_rows = T;
  out->view_shortcuts = gen.view_shortcuts();
  return Status::OK();
}

// ---- key-driven string Filter -------------------------------------------------------------------
// Default wherever it applies (string_scan bit 2 keeps the row-driven kernel): driven by the
// occurrences of a literal of the condition in the column's bytes.  Conditions that can raise keep
// the row-driven kernel so that errors come from the same rows.  False, with `out` untouched, where
// it does not apply.
bool GenerateKeyFilter(const Schema& schema, const std::vector<ExpressionPtr>& exprs, const KernelSpec& spec,
                       GeneratedKernel* out) {
  if ((spec.string_scan & 4) != 0 || exprs.size() != 1 || BodyGen::CanFail(*exprs[0]->root())) return false;
  std::vector<ColumnSlot> kslots;
  BodyGen kgen(schema, &kslots, spec.nullable, /*coop=*/false);
  KeyPlan plan;
  const int kBT = spec.block_threads > 0 ? spec.block_threads : 256;
  // chunks of 1024 rows per warp and tile: more rows per anchor drain and per tile-end barrier on
  // big batches (Configuration.stages overrides), one on small ones (enough tiles for 132 SMs)
  const int kW = (spec.stages == 1 || spec.stages == 2 || spec.stages == 4) ? spec.stages : (spec.large_batch ? 2 : 1);
  if (kBT % 32 != 0 || kBT > 1024 || !kgen.PlanKey(*exprs[0]->root(), &plan)) return false;
  std::string kbody;
  const Val kres = kgen.GenTruth(*exprs[0]->root(), &kbody, 6);
  // the anchor drain loads rows one by one from plain columns only
  if (!kgen.error().empty() || kgen.uses_ctx() || HasDictionary(kslots) || HasView(kslots)) return false;
  if (spec.nullable) MarkHoisted(kgen, *exprs[0]->root(), &kslots);
  DescribeKernel(spec, kslots, 0, out);
  std::string src = HeaderLines("key-driven string Filter", spec, exprs);
  src += "// key: '" + CommentSafe(plan.key) + "' in column slot " + std::to_string(plan.slot) +
         ", case map " + std::to_string(plan.xf) + "\n";
  src += "#include \"gdv_device_lib.cuh\"\n";
  src += EmitArgsStruct(out->args);
  src += kgen.globals();
  src += EmitKeyFilter(kslots, spec, plan, kbody, kres, kBT, kW, kgen.ScratchDecl(1));
  out->source = std::move(src);
  out->rows_per_thread = 1;
  out->block_threads = kBT;
  out->dynamic_smem = (kBT / 32) * (kKeyAnchorCap + 32 * kW + 4) * 4;
  out->tile_rows = static_cast<int64_t>(kBT / 32) * 1024 * kW;
  out->key_driven = true;
  return true;
}

// ---- row-driven Filter --------------------------------------------------------------------------
// Fixed-width columns.  Every warp walks W consecutive 1024-row chunks per tile, so a 32K-row tile
// needs 256 threads at W = 4 and eight small CTAs share an SM: while one sits in its tile-end
// barriers and look-back, seven keep streaming.  Gated loads (EmitGatedGroup) where `gate_seg` is
// not empty.
void EmitChunkLoop(const std::vector<ColumnSlot>& slots, const KernelSpec& spec, int R, int W, const std::string& body,
                   const std::string& step_tail, const std::vector<CoopSeg>& coop, const GatePlan& gate,
                   const std::vector<std::string>& gate_seg, std::string* o) {
  std::string& src = *o;
  const std::string sR = std::to_string(R), s32R = std::to_string(32 * R);
  const bool gated = !gate_seg.empty();
  src += "    #pragma unroll\n";
  src += "    for (int w = 0; w < " + std::to_string(W) + "; ++w) {\n";
  src += "      const i64 wbase = wbase0 + 1024 * w;\n";
  src += "      u32 cur = 0u;\n";
  src += "      #pragma unroll 1\n";
  src += "      for (int g = 0; g < 32; g += " + sR + ") {\n";
  src += "        const i64 base = wbase + 32 * g;\n";
  src += "        if (base >= A.n) break;\n";
  src += "        if (base + " + s32R + " <= A.n) {\n";
  const std::string gated_tail =
      "          { const u32 m = __ballot_sync(GDV_FULL, in && alive[k]); if (lane == (u32)(g + k)) cur = m; }\n";
  if (gated)
    EmitGatedGroup(slots, spec, R, kFast, gate, gate_seg, gated_tail, &src, 5);
  else
    EmitGroup(slots, spec, false, R, kFast, body, step_tail, &src, 5, 0, std::string(), coop);
  src += "        } else {\n";
  if (gated)
    EmitGatedGroup(slots, spec, R, kPred, gate, gate_seg, gated_tail, &src, 5);
  else
    EmitGroup(slots, spec, false, R, kPred, body, step_tail, &src, 5, 0, std::string(), coop);
  src += "        }\n";
  src += "      }\n";
  src += "      mymask[w] = cur;\n";
  src += "    }\n";
}

// String columns: one 1024-row chunk per warp; the bytes of the NEXT group are copied into a
// second shared-memory stage with cp.async while the current group is scanned.
void EmitPrefetchLoop(const std::vector<ColumnSlot>& slots, const KernelSpec& spec, int R, int stage_bytes,
                      const std::string& body, const std::string& step_tail, const std::vector<CoopSeg>& coop,
                      std::string* o) {
  std::string& src = *o;
  const std::string sR = std::to_string(R), s32R = std::to_string(32 * R);
  src += "    const i64 wbase = wbase0;\n";
  src += "    u32 cur = 0u;\n";
  // issue(b, par): cp.async the bytes of the full group that starts at row b into stage `par`
  src += "    auto issue = [&](i64 b, u32 par) {\n";
  for (size_t j = 0; j < slots.size(); ++j) {
    if (!HasByteRun(slots[j])) continue;
    const std::string J = std::to_string(j);
    src += "      {\n";
    if (slots[j].type.is_large()) {  // as in EmitGroup: i64 run, narrowed once it fits the stage
      src += "        const i64 gb = in_val" + J + "[b];\n";
      src += "        const i64 gn64 = in_val" + J + "[b + " + s32R + "] - gb;\n";
      src += "        const u8* src = in_var" + J + " + gb;\n";
      src += "        const u32 mis = (u32)((unsigned long long)src & 15ull);\n";
      src += "        if (gn64 + (i64)mis <= " + std::to_string(stage_bytes) + ") {\n";
      src += "          const i32 gn = (i32)gn64;\n";
    } else {
      src += "        const i32 gb = in_val" + J + "[b];\n";
      src += "        const i32 gn = in_val" + J + "[b + " + s32R + "] - gb;\n";
      src += "        const u8* src = in_var" + J + " + gb;\n";
      src += "        const u32 mis = (u32)((unsigned long long)src & 15ull);\n";
      src += "        if (gn + (i32)mis <= " + std::to_string(stage_bytes) + ") {\n";
    }
    src += "          const i32 nchunks = (gn + (i32)mis + 15) >> 4;\n";
    src += "          u8* dst = stage" + J + "_0 + (size_t)par * " + std::to_string(stage_bytes) + "u;\n";
    src += "          for (i32 c = (i32)lane; c < nchunks; c += 32)\n";
    src += "            gdv_cp_async16(dst + 16 * c, src - mis + 16 * c);\n";
    src += "        }\n";
    src += "      }\n";
  }
  src += "      gdv_cp_async_commit();\n";
  src += "    };\n";
  src += "    u32 par = 0u;\n";
  src += "    if (wbase + " + s32R + " <= A.n) issue(wbase, 0u);\n";
  src += "    #pragma unroll 1\n";
  src += "    for (int g = 0; g < 32; g += " + sR + ") {\n";
  src += "      const i64 base = wbase + 32 * g;\n";
  src += "      if (base >= A.n) break;\n";
  for (size_t j = 0; j < slots.size(); ++j)
    if (HasByteRun(slots[j]))
      src += "      u8* const stage" + std::to_string(j) + " = stage" + std::to_string(j) +
             "_0 + (size_t)par * " + std::to_string(stage_bytes) + "u;\n";
  src += "      if (base + " + s32R + " <= A.n) {\n";
  src += "        if (g + " + sR + " < 32 && base + " + std::to_string(64 * R) + " <= A.n) {\n";
  src += "          issue(base + " + s32R + ", par ^ 1u);\n";
  src += "          gdv_cp_async_wait<1>();\n";
  src += "        } else {\n";
  src += "          gdv_cp_async_wait<0>();\n";
  src += "        }\n";
  src += "        __syncwarp();\n";
  src += "        par ^= 1u;\n";
  EmitGroup(slots, spec, false, R, kFast, body, step_tail, &src, 4, stage_bytes, std::string(), coop, true);
  src += "      } else {\n";
  EmitGroup(slots, spec, false, R, kPred, body, step_tail, &src, 4, 0, std::string(), coop);
  src += "      }\n";
  src += "    }\n";
  src += "    mymask[0] = cur;\n";
}

// Filter: every warp owns 1024 consecutive rows per chunk (32 steps of 32 rows).  Step k's
// keep-mask is one ballot word, parked in lane k, so a chunk costs one register per thread
// regardless of its size; loads are issued R steps at a time for memory-level parallelism.
// Large tiles keep the number of look-back descriptors per launch small, which is what bounds
// ordered compaction at HBM bandwidth (DESIGN.md "Filter kernel").
Status GenerateFilter(const Schema& schema, const std::vector<ExpressionPtr>& exprs, const KernelSpec& spec,
                      GeneratedKernel* out) {
  std::vector<ColumnSlot> slots;
  BodyGen gen = SpecBodyGen(schema, &slots, spec);
  // Per-row body (uses f<j>[k] / k<j>[k]); generated first so we know the slots.
  std::string body;
  std::vector<Val> results;
  for (const auto& e : exprs) results.push_back(gen.GenTruth(*e->root(), &body, 4));
  if (!gen.error().empty()) return Status::Make(GDV_NOT_IMPLEMENTED, gen.error());
  if (spec.nullable && !gen.uses_ctx() && exprs.size() == 1) MarkHoisted(gen, *exprs[0]->root(), &slots);
  // Fixed-width Filter: gated loads (EmitGatedGroup) wherever PlanGate finds a plan.  gate_seg[s] ANDs
  // stage s's conjuncts into alive[k]; the segments come from a BodyGen of their own (over the same
  // slots), whose globals replace those of `body`, which a gated kernel does not emit.
  GatePlan gate;
  std::vector<std::string> gate_seg;
  std::vector<ColumnSlot> gate_slots = slots;
  BodyGen sgen = SpecBodyGen(schema, &gate_slots, spec);
  if (spec.filter_gating == 0 && exprs.size() == 1 && PlanGate(schema, *exprs[0]->root(), slots, &gate)) {
    for (const auto& cj : gate.conjuncts) {
      std::string seg, all;
      for (const Node* c : cj) all += " && (" + sgen.GenTruth(*c, &seg, 6).v + ")";
      gate_seg.push_back(seg + "            alive[k] = alive[k]" + all + ";\n");
    }
  }
  const bool gated = !gate_seg.empty();
  DescribeKernel(spec, slots, 0, out);
  int R = spec.rows_per_thread > 0 ? spec.rows_per_thread : PickRowsPerThread(out->in_bytes_per_row, 0, spec.kind);
  if (R > 32) R = 32;
  // the filter walks 32 steps per warp in groups of R: R must divide 32
  int p = 1;
  while (p * 2 <= R) p *= 2;
  R = p;
  // Filters copy the string bytes of the NEXT group into a second stage with cp.async while the
  // current group is scanned (per-warp double buffering): the copy costs no registers and its
  // latency is hidden behind the scan instead of behind other warps.
  int BT = 0;
  StringStages st;
  const Status fit = FitStages(spec, gen, slots, 2, &R, &BT, &st);
  if (!fit.ok()) return fit;
  const int n_varlen = st.columns;
  // 1024-row chunks every warp walks per tile (Configuration.stages; 1 unless asked)
  const int W = n_varlen != 0 ? 1
                : (spec.stages == 1 || spec.stages == 2 || spec.stages == 4 || spec.stages == 8) ? spec.stages
                : (spec.large_batch ? 4 : 1);
  out->rows_per_thread = R;
  out->block_threads = BT;

  std::string header = HeaderLines("one fused kernel per Filter", spec, exprs);
  if (gated) header += "// gated loads: " + std::to_string(gate.stages()) + " stages\n";
  // Fixed-width filters are bandwidth-bound and want every warp slot of the SM: ask for
  // 2048 / BT resident CTAs, which caps the kernel at 32 registers per thread (what it needs).
  std::string bounds = std::to_string(BT);
  bool light = n_varlen == 0 && BT >= 256 && 2048 % BT == 0 && !gen.uses_ctx() && body.size() < 6000;
  for (const auto& sl : slots)  // 128-bit math and string functions over dictionary views want registers
    light = light && !sl.type.is_decimal() && !sl.type.is_dict() && !sl.type.is_view();
  if (light && W > 1 && gated) {
    // the stage chain keeps more values live than the ungated group: hold the 48 warps per SM that
    // the ungated kernel reaches at W > 1 (40 registers)
    bounds += ", " + std::to_string(1536 / BT);
    light = false;
  }
  if (W > 1) light = false;  // W chunks keep 2 W more registers
  if (light) bounds += ", " + std::to_string(2048 / BT);
  std::string src = EmitKernelFrame(spec, false, *out, gated ? sgen : gen, header, bounds);
  if (st.stage_bytes > 0)
    src += EmitStageDecls(slots, gen.coop_segs(), st, "u8* const ", "_0", ";  // [0] hits, [1] candidates\n");

  const std::string IDX = SelCType(spec.selection_mode);
  const int NW = BT / 32;
  const int WT = NW * 1024 * W;
  src += "  __shared__ u32 s_wcount[" + std::to_string(NW) + "];\n";
  src += "  __shared__ i64 s_tile;\n";
  src += "  __shared__ u64 s_excl;\n";
  src += "  const i64 n_tiles = (A.n + " + std::to_string(WT - 1) + ") / " + std::to_string(WT) + ";\n";
  src += "  " + IDX + "* out_idx = reinterpret_cast<" + IDX + "*>(A.out_idx);\n";
  src += "  const u32 lt = gdv_lanemask_lt();\n";
  src += "  while (true) {\n";
  src += "    if (threadIdx.x == 0) s_tile = (i64)atomicAdd(A.ticket, 1ull);\n";
  src += "    __syncthreads();\n";
  src += "    const i64 tile = s_tile;\n";
  src += "    if (tile >= n_tiles) break;\n";
  src += "    const i64 wbase0 = tile * " + std::to_string(WT) + " + (i64)wid * " + std::to_string(1024 * W) + ";\n";
  src += "    u32 mymask[" + std::to_string(W) + "];\n";
  const std::string step_tail =
      "          { const u32 m = __ballot_sync(GDV_FULL, in && (" + results[0].ok + ") && (" +
      results[0].v + ")); if (lane == (u32)(g + k)) cur = m; }\n";
  if (n_varlen == 0)
    EmitChunkLoop(slots, spec, R, W, body, step_tail, gen.coop_segs(), gate, gate_seg, &src);
  else
    EmitPrefetchLoop(slots, spec, R, st.stage_bytes, body, step_tail, gen.coop_segs(), &src);
  EmitFilterEpilogue(slots, spec, NW, W, IDX, &src);
  src += "  }\n";
  src += "}\n";

  out->source = std::move(src);
  out->uses_ctx = gen.uses_ctx();
  out->dynamic_smem = st.dynamic_smem(BT);
  out->tile_rows = static_cast<int64_t>(NW) * 1024 * W;
  out->cta_tile_rows = static_cast<int64_t>(BT) * R;
  out->view_shortcuts = gen.view_shortcuts();
  out->gated_stages = gated ? gate.stages() : 0;
  return Status::OK();
}

// ---- Projector ----------------------------------------------------------------------------------
// Per-step tail of a projector group: the stores (`fast`: every row of the group is in range) and the
// validity / boolean-data ballots into lane k's words.
std::string ProjectStepTail(const std::vector<ExpressionPtr>& exprs, const std::vector<Val>& results, bool fast) {
  std::string t5;
  for (size_t o = 0; o < exprs.size(); ++o) {
    const DataType& t = exprs[o]->result().type;
    const std::string O = std::to_string(o);
    if (t.is_bool()) {
      t5 += "        { const u32 m = __ballot_sync(GDV_FULL, in && (" + results[o].v +
            ")); if (lane == (u32)k) dw" + O + " = m; }\n";
    } else if (fast) {
      t5 += "        gdv_stp(out" + O + " + s, (" + std::string(t.ctype()) + ")(" + results[o].v +
            "));\n";
    } else {
      t5 += "        if (in) gdv_stp(out" + O + " + s, (" + std::string(t.ctype()) + ")(" +
            results[o].v + "));\n";
    }
    t5 += "        { const u32 m = __ballot_sync(GDV_FULL, in && (" + results[o].ok +
          ")); if (lane == (u32)k) vw" + O + " = m; }\n";
  }
  return t5;
}

// A warp tile's output words, one per 32 rows and held by lane k for step k: validity vw<o> and,
// for a boolean output, its bit-packed data dw<o>.
std::string EmitOutWordDecls(const std::vector<ExpressionPtr>& exprs) {
  std::string o;
  for (size_t i = 0; i < exprs.size(); ++i) {
    o += "    u32 vw" + std::to_string(i) + " = 0u;\n";
    if (exprs[i]->result().type.is_bool()) o += "    u32 dw" + std::to_string(i) + " = 0u;\n";
  }
  return o;
}

// Their write-back: lanes k < R (and `guard`) store word k of the warp tile that starts at `base`.
std::string EmitOutWordStores(const std::vector<ExpressionPtr>& exprs, int R, const std::string& guard) {
  std::string o = "    if (lane < " + std::to_string(R) + "u" + guard + ") {\n";
  o += "      const i64 w = (base >> 5) + (i64)lane;\n";
  for (size_t i = 0; i < exprs.size(); ++i) {
    const std::string O = std::to_string(i);
    o += "      if (A.out_vld[" + O + "] != nullptr) A.out_vld[" + O + "][w] = vw" + O + ";\n";
    if (exprs[i]->result().type.is_bool()) o += "      reinterpret_cast<u32*>(A.out_val[" + O + "])[w] = dw" + O + ";\n";
  }
  return o + "    }\n";
}

// TMA loader (fixed-width inputs, no selection vector): each CTA tile (BT * R rows) of every input
// column is copied into a shared-memory stage by one cp.async.bulk; S stages per CTA keep (S - 1)
// tiles in flight per CTA while one computes.  Emits the loop over the staged tiles of the kernel
// `out` describes and sets its staged / stages / dynamic_smem; false, with nothing emitted, when two
// stages do not fit.
bool EmitStagedTiles(const KernelSpec& spec, const std::vector<ExpressionPtr>& exprs, const std::string& body,
                     const std::vector<Val>& results, const std::vector<CoopSeg>& coop, std::string* o,
                     GeneratedKernel* out) {
  const std::vector<ColumnSlot>& slots = out->inputs;
  const int R = out->rows_per_thread, BT = out->block_threads;
  std::vector<int> val_off(slots.size(), 0), vld_off(slots.size(), 0);
  int stage_total = 0, val_tx = 0, S = 0;
  const int vld_copy = BT * R / 8 + 32;
  int off = 0;
  for (size_t j = 0; j < slots.size(); ++j) {
    val_off[j] = off;
    off += BT * R * slots[j].type.width() + 16;
    val_tx += BT * R * slots[j].type.width() + 16;
  }
  if (spec.nullable)
    for (size_t j = 0; j < slots.size(); ++j) {
      vld_off[j] = off;
      off += vld_copy;
    }
  stage_total = (off + 127) / 128 * 128;
  S = spec.stages > 0 ? spec.stages : 4;
  while (S > 2 && S * stage_total > 220 * 1024) --S;
  if (S < 2 || S * stage_total > 220 * 1024) return false;
  out->dynamic_smem = S * stage_total;
  out->staged = true;
  out->stages = S;

  std::string& src = *o;
  const int T = BT * R;  // rows per CTA tile
  const std::string sS = std::to_string(S), sT = std::to_string(T), s32R = std::to_string(32 * R);
  src += "  extern __shared__ uint4 gdv_smem[];\n";
  src += "  __shared__ u64 gdv_full[" + sS + "];\n";
  src += "  u8* const stage0 = reinterpret_cast<u8*>(gdv_smem);\n";
  std::string tx = std::to_string(val_tx) + "u";
  for (size_t j = 0; j < slots.size(); ++j) {
    const std::string J = std::to_string(j);
    src += "  const u32 mis" + J + " = (u32)((unsigned long long)in_val" + J + " & 15ull);\n";
    if (spec.nullable) {
      src += "  const u32 vmis" + J + " = (u32)((unsigned long long)in_vld" + J + " & 15ull);\n";
      tx += " + (in_hv" + J + " ? " + std::to_string(vld_copy) + "u : 0u)";
    }
  }
  src += "  const u32 tx_bytes = " + tx + ";\n";
  src += "  const u64 pol = gdv_policy_evict_first();\n";
  // a bulk copy may read up to 32 bytes past its tile: the last 256 rows are never staged
  src += "  const i64 n_st = A.n > 256 ? (A.n - 256) / " + sT + " : 0;\n";
  src += "  if (threadIdx.x == 0) {\n";
  src += "    for (u32 s = 0; s < " + sS + "u; ++s) gdv_mbar_init(&gdv_full[s], 1u);\n";
  src += "    gdv_fence_mbar_init();\n";
  src += "  }\n";
  src += "  __syncthreads();\n";
  src += "  auto issue = [&](i64 t, u32 s) {\n";
  src += "    u8* sb = stage0 + (size_t)s * " + std::to_string(stage_total) + "u;\n";
  src += "    gdv_mbar_expect_tx(&gdv_full[s], tx_bytes);\n";
  for (size_t j = 0; j < slots.size(); ++j) {
    const std::string J = std::to_string(j);
    const int w = slots[j].type.width();
    src += "    gdv_bulk_g2s(sb + " + std::to_string(val_off[j]) + ", reinterpret_cast<const u8*>(in_val" +
           J + ") - mis" + J + " + t * " + std::to_string(static_cast<long long>(T) * w) + "ll, " +
           std::to_string(T * w + 16) + "u, &gdv_full[s], pol);\n";
    if (spec.nullable)
      src += "    if (in_hv" + J + ") gdv_bulk_g2s(sb + " + std::to_string(vld_off[j]) +
             ", reinterpret_cast<const u8*>(in_vld" + J + ") - vmis" + J + " + t * " +
             std::to_string(T / 8) + "ll, " + std::to_string(vld_copy) + "u, &gdv_full[s], pol);\n";
  }
  src += "  };\n";
  src += "  if (threadIdx.x == 0) {\n";
  src += "    for (u32 s = 0; s < " + sS + "u; ++s) {\n";
  src += "      const i64 t = (i64)blockIdx.x + (i64)s * gridDim.x;\n";
  src += "      if (t < n_st) issue(t, s);\n";
  src += "    }\n";
  src += "  }\n";
  src += "  u32 it = 0u;\n";
  src += "  for (i64 t = blockIdx.x; t < n_st; t += gridDim.x, ++it) {\n";
  src += "    const u32 s = it % " + sS + "u;\n";
  src += "    const u32 par = (it / " + sS + "u) & 1u;\n";
  src += "    const u8* sb = stage0 + (size_t)s * " + std::to_string(stage_total) + "u;\n";
  src += "    const i64 base = t * " + sT + " + (i64)wid * " + s32R + ";\n";
  for (size_t j = 0; j < slots.size(); ++j) {
    const std::string J = std::to_string(j);
    const std::string ct = slots[j].type.ctype();
    src += "    const " + ct + "* sp" + J + " = reinterpret_cast<const " + ct + "*>(sb + " +
           std::to_string(val_off[j]) + " + mis" + J + ") + wid * " + s32R + "u + lane;\n";
    if (spec.nullable)
      src += "    const u32* sv" + J + " = reinterpret_cast<const u32*>(sb + " +
             std::to_string(vld_off[j]) + " + vmis" + J + ");\n";
  }
  src += EmitOutWordDecls(exprs);
  src += "    gdv_mbar_wait(&gdv_full[s], par);\n";
  src += "    {\n";
  std::string after;
  after += "      __syncthreads();  // every thread holds its rows: the stage can be refilled\n";
  after += "      if (threadIdx.x == 0) {\n";
  after += "        const i64 tn = t + (i64)" + sS + " * gridDim.x;\n";
  after += "        if (tn < n_st) issue(tn, s);\n";
  after += "      }\n";
  EmitGroup(slots, spec, false, R, kStaged, body, ProjectStepTail(exprs, results, true), &src, 3, 0, after, coop);
  src += "    }\n";
  src += EmitOutWordStores(exprs, R, "");
  src += "  }\n";
  return true;
}

// Direct loads: warp tiles of 32 R rows, from warp tile `wt_first` on (the rows after the staged tiles).
void EmitDirectTiles(const KernelSpec& spec, bool has_sel, const std::vector<ExpressionPtr>& exprs,
                     const std::string& body, const std::vector<Val>& results, const std::vector<CoopSeg>& coop,
                     int stage_bytes, const std::string& wt_first, const GeneratedKernel& out, std::string* o) {
  std::string& src = *o;
  const std::vector<ColumnSlot>& slots = out.inputs;
  const int R = out.rows_per_thread, NWP = out.block_threads / 32;
  const std::string s32R = std::to_string(32 * R);
  src += "  const i64 n_wtiles = (A.n + " + std::to_string(32 * R - 1) + ") / " + s32R + ";\n";
  src += "  const i64 wstride = (i64)gridDim.x * " + std::to_string(NWP) + ";\n";
  src += "  for (i64 wt = " + wt_first + " + (i64)blockIdx.x * " + std::to_string(NWP) +
         " + wid; wt < n_wtiles; wt += wstride) {\n";
  src += "    const i64 base = wt * " + s32R + ";\n";
  src += EmitOutWordDecls(exprs);
  if (!has_sel) {
    src += "    if (base + " + s32R + " <= A.n) {\n";
    EmitGroup(slots, spec, false, R, kFast, body, ProjectStepTail(exprs, results, true), &src, 3, stage_bytes, std::string(), coop);
    src += "    } else {\n";
    EmitGroup(slots, spec, false, R, kPred, body, ProjectStepTail(exprs, results, false), &src, 3, 0, std::string(), coop);
    src += "    }\n";
  } else {
    src += "    {\n";
    EmitGroup(slots, spec, true, R, kPred, body, ProjectStepTail(exprs, results, false), &src, 3, 0, std::string(), coop);
    src += "    }\n";
  }
  src += EmitOutWordStores(exprs, R, " && base + 32 * (i64)lane < A.n");
  src += "  }\n";
}

Status GenerateProjector(const Schema& schema, const std::vector<ExpressionPtr>& exprs, const KernelSpec& spec,
                         GeneratedKernel* out) {
  std::vector<ColumnSlot> slots;
  BodyGen gen = SpecBodyGen(schema, &slots, spec);
  // Per-row body (uses f<j>[k] / k<j>[k]); generated first so we know the slots.
  std::string body;
  std::vector<Val> results;
  for (const auto& e : exprs) {
    if (e->result().type.is_varlen())
      return Status::Make(GDV_NOT_IMPLEMENTED,
                          "variable-length projection outputs are handled by the two-pass "
                          "string projector, not by GenerateKernel");
    results.push_back(gen.Gen(*e->root(), &body, 4));
  }
  if (!gen.error().empty()) return Status::Make(GDV_NOT_IMPLEMENTED, gen.error());
  DescribeKernel(spec, slots, static_cast<int>(exprs.size()), out);
  for (const auto& e : exprs) {
    out->outputs.push_back(e->result().type);
    out->out_bytes_per_row += std::max(e->result().type.width(), 1);
  }
  // The TMA loader is the default for wide-row projectors (the Q1 projector, 166 B/row): bulk copies
  // keep a whole tile per column in flight without spending registers on it, where the direct path
  // runs out of registers before it has enough loads in flight.
  bool want_staged = spec.selection_mode == GDV_SEL_NONE && spec.loader != 1 && !slots.empty() &&
                     (spec.loader == 2 || out->in_bytes_per_row >= 48);
  for (const auto& sl : slots)
    if (sl.type.is_varlen() || sl.type.is_bool()) want_staged = false;
  int R = spec.rows_per_thread > 0
              ? spec.rows_per_thread
              : (want_staged ? 2 : PickRowsPerThread(out->in_bytes_per_row, out->out_bytes_per_row, spec.kind));
  if (R > 32) R = 32;
  int BT = 0;
  StringStages st;
  const Status fit = FitStages(spec, gen, slots, 1, &R, &BT, &st);
  if (!fit.ok()) return fit;
  out->rows_per_thread = R;
  out->block_threads = BT;
  out->dynamic_smem = st.dynamic_smem(BT);
  const bool has_sel = spec.selection_mode != GDV_SEL_NONE;

  std::string src = EmitKernelFrame(spec, has_sel, *out, gen, HeaderLines("one fused kernel per Projector", spec, exprs),
                                    std::to_string(BT));
  if (st.stage_bytes > 0) src += EmitStageDecls(slots, gen.coop_segs(), st, "u8* const ", "", ";  // [0] hits, [1] candidates\n");
  for (size_t o = 0; o < exprs.size(); ++o) {
    const DataType& t = exprs[o]->result().type;
    const std::string O = std::to_string(o);
    if (!t.is_bool())
      src += "  " + std::string(t.ctype()) + "* out" + O + " = reinterpret_cast<" + t.ctype() +
             "*>(A.out_val[" + O + "]);\n";
  }
  std::string wt_first = "0";
  if (want_staged && (BT * R) % 128 == 0 && EmitStagedTiles(spec, exprs, body, results, gen.coop_segs(), &src, out))
    wt_first = "n_st * " + std::to_string(BT / 32);  // rows after the staged tiles take the direct path
  EmitDirectTiles(spec, has_sel, exprs, body, results, gen.coop_segs(), st.stage_bytes, wt_first, *out, &src);
  src += "}\n";
  if (has_sel) ApplyDeviceCount(&src);

  out->source = std::move(src);
  out->uses_ctx = gen.uses_ctx();
  out->cta_tile_rows = static_cast<int64_t>(BT) * R;
  out->view_shortcuts = gen.view_shortcuts();
  return Status::OK();
}

}  // namespace

namespace {

// Functions that are spelled in terms of others are rewritten before lowering:
//   ilike(s, 'pattern') -> like(lower(s), 'lower-cased pattern')   (ASCII case folding)
// Returns the node itself when nothing below it changes.
NodePtr RewriteAliases(const NodePtr& node) {
  NodeVector kids;
  for (const auto& c : Children(*node)) kids.push_back(RewriteAliases(c));
  if (node->kind() == NodeKind::kFunction) {
    const auto& fn = static_cast<const FunctionNode&>(*node);
    if (fn.name() == "ilike" && kids.size() == 2 && kids[1]->kind() == NodeKind::kLiteral) {
      const auto& pat = static_cast<const LiteralNode&>(*kids[1]);
      std::string low = pat.bytes();
      for (auto& ch : low)
        if (ch >= 'A' && ch <= 'Z') ch = static_cast<char>(ch + 32);
      NodePtr text = std::make_shared<FunctionNode>("lower", NodeVector{kids[0]}, utf8());
      NodePtr lit = std::make_shared<LiteralNode>(utf8(), low.data(), static_cast<int64_t>(low.size()),
                                                  pat.is_null());
      return std::make_shared<FunctionNode>("like", NodeVector{text, lit}, boolean());
    }
    // A concat result is a rope that only projection / concat / if-else can read.  Two consumers
    // distribute over its pieces instead: the ASCII case maps, and the length functions.
    if (kids.size() == 1 && kids[0]->kind() == NodeKind::kFunction) {
      const auto& inner = static_cast<const FunctionNode&>(*kids[0]);
      const bool is_concat = inner.name() == "concat" || inner.name() == "concatOperator";
      if (is_concat && (fn.name() == "upper" || fn.name() == "lower")) {
        NodeVector parts;
        for (const auto& c : inner.children())
          parts.push_back(RewriteAliases(std::make_shared<FunctionNode>(fn.name(), NodeVector{c}, c->return_type())));
        return std::make_shared<FunctionNode>(inner.name(), std::move(parts), inner.return_type());
      }
      const bool is_len = fn.name() == "char_length" || fn.name() == "length" || fn.name() == "lengthUtf8" ||
                          fn.name() == "octet_length" || fn.name() == "bit_length";
      if (is_concat && is_len && !inner.children().empty()) {
        // concat counts a NULL argument as the empty string; concatOperator is NULL if any argument is
        NodePtr sum;
        const int32_t zero = 0;
        for (const auto& c : inner.children()) {
          NodePtr len = RewriteAliases(std::make_shared<FunctionNode>(fn.name(), NodeVector{c}, fn.return_type()));
          if (inner.name() == "concat")
            len = std::make_shared<FunctionNode>(
                "nvl", NodeVector{len, std::make_shared<LiteralNode>(fn.return_type(), &zero, 4, false)}, fn.return_type());
          sum = sum == nullptr ? len : std::make_shared<FunctionNode>("add", NodeVector{sum, len}, fn.return_type());
        }
        return sum;
      }
    }
  }
  return WithChildren(node, std::move(kids));
}

}  // namespace

int DictionaryFirstColumn(const Schema& schema, const Node& cond) {
  std::vector<int> cols;
  CollectColumns(schema, cond, &cols);
  if (cols.size() != 1 || cols[0] < 0 || !schema.fields()[cols[0]].type.is_dict()) return -1;
  if (BodyGen::CanFail(cond)) return -1;  // errors must come from the rows that hold the value
  std::vector<ColumnSlot> slots;
  const BodyGen gen(schema, &slots, true, false);
  std::vector<int> strict;
  gen.TruthStrict(cond, &strict);
  return std::find(strict.begin(), strict.end(), cols[0]) != strict.end() ? cols[0] : -1;
}

NodePtr WithValueTypes(const NodePtr& node) {
  if (node->kind() == NodeKind::kField && node->return_type().is_dict())
    return std::make_shared<FieldNode>(static_cast<const FieldNode&>(*node).name(), node->return_type().value_type());
  NodeVector kids;
  for (const auto& c : Children(*node)) kids.push_back(WithValueTypes(c));
  return WithChildren(node, std::move(kids));
}

static bool ReadsRowCheckedColumn(const Node& node) {
  if (node.kind() == NodeKind::kField)
    return node.return_type().is_dict() || node.return_type().is_view() || node.return_type().is_large();
  for (const auto& c : Children(node))
    if (ReadsRowCheckedColumn(*c)) return true;
  return false;
}

Status GenerateKernel(const Schema& schema, const std::vector<ExpressionPtr>& exprs,
                      const KernelSpec& spec, GeneratedKernel* out) {
  std::vector<ExpressionPtr> lowered;
  KernelSpec s = spec;
  for (const auto& e : exprs) {
    NodePtr r = RewriteAliases(e->root());
    lowered.push_back(r == e->root() ? e : std::make_shared<Expression>(r, e->result()));
    // a dictionary row is null when its entry is, or when its index is out of range, a view row
    // when its view is invalid, and a large row when its length does not fit a gdv_str: such kernels
    // always keep the validity plumbing
    if (ReadsRowCheckedColumn(*r)) s.nullable = true;
  }
  if (s.kind == KernelKind::kStringSize || s.kind == KernelKind::kStringWrite) {
    if (lowered.size() != 1 || !lowered[0]->result().type.is_varlen())
      return Status::Make(GDV_INVALID, "a string kernel takes exactly one utf8/binary expression");
    return GenerateStringKernel(schema, lowered[0], s, out);
  }
  if (s.kind == KernelKind::kProject) return GenerateProjector(schema, lowered, s, out);
  if (GenerateKeyFilter(schema, lowered, s, out)) return Status::OK();
  return GenerateFilter(schema, lowered, s, out);
}

}  // namespace gdv
