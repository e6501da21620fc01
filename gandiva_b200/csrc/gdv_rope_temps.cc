#include "gdv_rope_temps.h"

#include <algorithm>

namespace gdv {

bool IsRopeConsumerError(const Status& s) {
  if (s.code != GDV_NOT_IMPLEMENTED) return false;
  return s.msg.find("concat of more than 8 pieces") != std::string::npos ||
         s.msg.find("over it is not supported yet") != std::string::npos ||
         s.msg.find("(concat(...)) is not supported yet") != std::string::npos ||
         s.msg.find("over concat(...) is not supported yet") != std::string::npos;
}

namespace {

bool IsRopeFunction(const std::string& n) {
  return n == "concat" || n == "concatOperator" || n == "repeat" || n == "space" || n == "reverse" || n == "lpad" ||
         n == "rpad" || n == "replace";
}

// A node whose value is a rope: one of the functions above, or an if/else that may yield one.
bool IsRope(const Node& node) {
  if (!node.return_type().is_varlen()) return false;
  if (node.kind() == NodeKind::kFunction) return IsRopeFunction(static_cast<const FunctionNode&>(node).name());
  if (node.kind() == NodeKind::kIf) {
    const auto& n = static_cast<const IfNode&>(node);
    return IsRope(*n.then_node()) || IsRope(*n.else_node());
  }
  return false;
}

// Pieces a rope brings into the concat that reads it (lpad / rpad: padding + text; an if/else: the wider branch).
int Pieces(const Node& node) {
  if (node.kind() == NodeKind::kIf) {
    const auto& n = static_cast<const IfNode&>(node);
    return std::max(Pieces(*n.then_node()), Pieces(*n.else_node()));
  }
  if (node.kind() != NodeKind::kFunction || !node.return_type().is_varlen()) return 1;
  const auto& fn = static_cast<const FunctionNode&>(node);
  if (fn.name() == "concat" || fn.name() == "concatOperator") {
    int n = 0;
    for (const auto& c : fn.children()) n += Pieces(*c);
    return n;
  }
  return (fn.name() == "lpad" || fn.name() == "rpad") ? 2 : 1;
}

struct Extractor {
  RopeTemps* out;
  bool in_temp = false;  // walking the expression of a temp

  NodePtr Temp(const NodePtr& inner, const DataType& type) {
    const std::string text = inner->ToString();
    for (size_t k = 0; k < out->temps.size(); ++k)
      if (out->temps[k]->ToString() == text && out->fields[k].type == type)
        return std::make_shared<FieldNode>(out->fields[k].name, out->fields[k].type);
    Field f{"__gdv_rope_" + std::to_string(out->temps.size()), type};
    out->temps.push_back(std::make_shared<Expression>(inner, f));
    out->fields.push_back(f);
    return std::make_shared<FieldNode>(f.name, f.type);
  }

  // `rope_ok`: the parent can read a rope (it is the output root, a concat, or an if/else in such a position)
  NodePtr Walk(const NodePtr& node, bool rope_ok) {
    if (IsRope(*node) && !rope_ok) {
      // a consumer inside the arguments of a rope that is itself being materialised stays where it is: the
      // internal Projector that evaluates the temp is built the same way and takes care of it (next level)
      if (in_temp) return node;
      in_temp = true;
      const NodePtr inner = Walk(node, true);
      in_temp = false;
      return Temp(inner, node->return_type());
    }
    switch (node->kind()) {
      case NodeKind::kFunction: {
        const auto& fn = static_cast<const FunctionNode&>(*node);
        const bool is_concat = fn.name() == "concat" || fn.name() == "concatOperator";  // its arguments may be ropes
        // A concat the fuser cannot hold in one rope (more than 8 pieces) keeps its scalar arguments and reads
        // its widest rope arguments through temporaries (one piece each) until it fits; a concat with more than
        // 8 arguments is folded from the left, 8 at a time.  Not inside a temp: its own Projector does that.
        if (is_concat && !in_temp && Pieces(*node) > 8) {
          NodeVector args = fn.children();
          NodeVector orig = fn.children();  // what each argument stands for, over the ORIGINAL schema: the
                                            // expression of a temp may not name another temp's field
          auto total = [&] {
            int n = 0;
            for (const auto& a : args) n += Pieces(*a);
            return n;
          };
          while (total() > 8) {
            size_t widest = 0;
            for (size_t i = 1; i < args.size(); ++i)
              if (Pieces(*args[i]) > Pieces(*args[widest])) widest = i;
            if (Pieces(*args[widest]) > 1) {
              in_temp = true;
              const NodePtr inner = Walk(orig[widest], true);
              in_temp = false;
              args[widest] = Temp(inner, orig[widest]->return_type());
            } else {  // every argument is one piece: fold the first eight into one
              NodeVector head(orig.begin(), orig.begin() + 8);
              const NodePtr folded = std::make_shared<FunctionNode>(fn.name(), std::move(head), fn.return_type());
              in_temp = true;
              const NodePtr inner = Walk(folded, true);
              in_temp = false;
              args.erase(args.begin(), args.begin() + 8);
              args.insert(args.begin(), Temp(inner, fn.return_type()));
              orig.erase(orig.begin(), orig.begin() + 8);
              orig.insert(orig.begin(), folded);
            }
          }
          NodeVector kids;
          for (const auto& c : args) kids.push_back(Walk(c, true));
          return std::make_shared<FunctionNode>(fn.name(), std::move(kids), fn.return_type());
        }
        NodeVector kids;
        for (const auto& c : fn.children()) kids.push_back(Walk(c, is_concat));
        return WithChildren(node, std::move(kids));
      }
      case NodeKind::kIf: {
        const auto& n = static_cast<const IfNode&>(*node);
        return WithChildren(node, {Walk(n.condition(), false), Walk(n.then_node(), rope_ok), Walk(n.else_node(), rope_ok)});
      }
      default: {  // and / or / IN read no rope
        NodeVector kids;
        for (const auto& c : Children(*node)) kids.push_back(Walk(c, false));
        return WithChildren(node, std::move(kids));
      }
    }
  }
};

}  // namespace

bool ExtractRopes(const NodePtr& root, bool root_is_output, RopeTemps* out, NodePtr* rewritten) {
  Extractor x{out};
  *rewritten = x.Walk(root, root_is_output);
  return true;
}

}  // namespace gdv
