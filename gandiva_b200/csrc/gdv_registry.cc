#include "gdv_registry.h"

#include <cctype>
#include <cstdio>

#include "gdv_cuda.h"

namespace gdv {

std::string FunctionDef::device_name() const {
  if (is_user()) return device_base;
  std::string s = device_base;
  for (const auto& p : params) {
    s += "_";
    s += p.fn_suffix();
  }
  return s;
}

std::string FunctionDef::signature() const {
  std::string s = ret.ToString() + " " + name + "(";
  for (size_t i = 0; i < params.size(); ++i) {
    if (i) s += ", ";
    s += params[i].ToString();
  }
  return s + ")";
}

void Registry::Add(const std::string& name, std::vector<DataType> params, DataType ret,
                   NullMode nulls, uint32_t flags, const std::vector<std::string>& aliases) {
  FunctionDef d;
  d.name = name;
  d.device_base = name;
  d.params = std::move(params);
  d.ret = ret;
  d.nulls = nulls;
  d.flags = flags;
  defs_.push_back(d);
  for (const auto& a : aliases) {
    FunctionDef e = d;
    e.name = a;
    defs_.push_back(e);
  }
}

static bool ParamMatches(const DataType& want, const DataType& got) {
  if (want.id != got.id) return false;
  if (want.id == GDV_TYPE_DECIMAL128) return true;  // any precision/scale
  if (want.id == GDV_TYPE_TIMESTAMP || want.id == GDV_TYPE_TIME32 || want.id == GDV_TYPE_TIME64)
    return want.precision == got.precision;
  return true;
}

const FunctionDef* Registry::Lookup(const std::string& name, const std::vector<DataType>& params,
                                    const DataType& ret) const {
  const FunctionDef* first = nullptr;
  for (const auto& d : defs_) {
    if (d.name != name || d.params.size() != params.size()) continue;
    bool ok = true;
    for (size_t i = 0; i < params.size() && ok; ++i) ok = ParamMatches(d.params[i], params[i]);
    if (!ok) continue;
    if (d.ret == ret) return &d;
    if (first == nullptr) first = &d;
  }
  return first;
}

const Registry& Registry::Get() {
  static const Registry r;
  return r;
}

// ======================================================================================
// User functions
// ======================================================================================
namespace {

thread_local const FunctionRegistry* tl_user_functions = nullptr;

bool IsUserValueType(const DataType& t, bool allow_varlen) {
  if (t.is_dict() || t.is_view() || t.is_large()) return false;
  switch (t.id) {
    case GDV_TYPE_BOOL: case GDV_TYPE_UINT8: case GDV_TYPE_INT8: case GDV_TYPE_UINT16: case GDV_TYPE_INT16:
    case GDV_TYPE_UINT32: case GDV_TYPE_INT32: case GDV_TYPE_UINT64: case GDV_TYPE_INT64: case GDV_TYPE_FLOAT:
    case GDV_TYPE_DOUBLE: case GDV_TYPE_DATE32: case GDV_TYPE_DATE64:
      return true;
    case GDV_TYPE_TIMESTAMP: case GDV_TYPE_TIME32: return t.precision == 1;  // milliseconds, as everywhere
    case GDV_TYPE_STRING: case GDV_TYPE_BINARY: return allow_varlen;
    default: return false;
  }
}

const char* NullModeName(NullMode m) {
  return m == NullMode::kIfNull ? "if_null" : m == NullMode::kNever ? "never" : "internal";
}

// The device function the fuser calls: the engine writes the signature in the convention built-ins of
// the same null mode use (GenFunction), the caller supplies the statements.
std::string UserFunctionText(const UserFunction& fn, const std::string& symbol, const std::string& signature) {
  const bool pairs = fn.nulls != NullMode::kIfNull;
  std::string t = "// user function: " + signature + " [" + NullModeName(fn.nulls) + (fn.can_raise ? ", can raise" : "") + "]\n";
  t += std::string("__device__ __forceinline__ ") + fn.ret.ctype() + " " + symbol + "(";
  bool first = true;
  auto add = [&](const std::string& p) {
    t += (first ? "" : ", ") + p;
    first = false;
  };
  if (fn.can_raise) add("gdv_ctx* ctx");
  for (size_t i = 0; i < fn.params.size(); ++i) {
    const std::string n = std::to_string(i);
    add(fn.params[i].is_varlen() ? "const gdv_str& a" + n : std::string(fn.params[i].ctype()) + " a" + n);
    if (pairs) add("bool v" + n);
  }
  if (fn.nulls == NullMode::kInternal) add("bool* out_valid");
  t += ") {\n" + fn.body;
  if (fn.body.empty() || fn.body.back() != '\n') t += "\n";
  return t + "}\n";
}

uint64_t Fnv1a64(const std::string& s) {
  uint64_t h = 1469598103934665603ull;
  for (unsigned char c : s) {
    h ^= c;
    h *= 1099511628211ull;
  }
  return h;
}

}  // namespace

// ExecutionErrors with a caller's text: the lane that raises first writes the message behind the error
// word (the engine's error block is 256 bytes) and the host reads it back with the code.  Written into a
// kernel before its first user function that can raise.
const char kUserRaiseHelper[] =
    "#define GDV_ERR_USER 1000\n"
    "__device__ __noinline__ void gdv_raise(gdv_ctx* c, const char* msg) {\n"
    "  if (c->err == nullptr || atomicCAS(c->err, 0, GDV_ERR_USER) != 0) return;\n"
    "  char* d = reinterpret_cast<char*>(c->err) + 8;\n"
    "  int i = 0;\n"
    "  for (; i < 239 && msg[i] != 0; ++i) d[i] = msg[i];\n"
    "  d[i] = 0;\n"
    "}\n";

Status FunctionRegistry::Register(const UserFunction& fn) {
  auto invalid = [](const std::string& m) { return Status::Make(GDV_INVALID, m); };
  if (fn.name.empty() || !(std::isalpha(static_cast<unsigned char>(fn.name[0])) || fn.name[0] == '_'))
    return invalid("user function name '" + fn.name + "' is not an identifier");
  for (unsigned char c : fn.name)
    if (!(std::isalnum(c) || c == '_')) return invalid("user function name '" + fn.name + "' is not an identifier");
  FunctionDef d;
  d.name = fn.name;
  d.params = fn.params;
  d.ret = fn.ret;
  d.nulls = fn.nulls;
  d.flags = fn.can_raise ? static_cast<uint32_t>(kCanFail) : 0u;
  const std::string sig = d.signature();
  for (const auto& p : fn.params) {
    if (p.id == GDV_TYPE_DECIMAL128)
      return Status::Make(GDV_NOT_IMPLEMENTED, "user function " + sig + ": decimal128 parameters are not supported");
    if (!IsUserValueType(p, true)) return invalid("user function " + sig + ": unsupported parameter type " + p.ToString());
  }
  if (fn.ret.is_varlen() || fn.ret.id == GDV_TYPE_DECIMAL128)
    return Status::Make(GDV_NOT_IMPLEMENTED, "user function " + sig + ": " + fn.ret.ToString() +
                                                 " return types are not supported (fixed-width results only)");
  if (!IsUserValueType(fn.ret, false)) return invalid("user function " + sig + ": unsupported return type " + fn.ret.ToString());
  // The fuser recognises many built-ins by name (nvl, like, locate, equal over views, ...), so a built-in's
  // name is taken for every parameter list, not only the ones it is defined for.
  for (const auto& b : Registry::Get().all())
    if (b.name == fn.name)
      return invalid("user function " + sig + " clashes with the built-in function '" + fn.name +
                     "': built-ins cannot be shadowed or overloaded");
  if (fn.body.empty()) return invalid("user function " + sig + " has an empty body");

  std::string hashed = sig + "|" + NullModeName(fn.nulls) + "|" + (fn.can_raise ? "1" : "0") + "|" + fn.prelude;
  hashed.push_back('\0');
  hashed += fn.body;
  char hex[24];
  std::snprintf(hex, sizeof(hex), "%016llx", static_cast<unsigned long long>(Fnv1a64(hashed)));
  d.device_base = std::string("gdv_udf_") + hex;
  d.prelude = fn.prelude;
  if (!d.prelude.empty() && d.prelude.back() != '\n') d.prelude += "\n";
  d.source = UserFunctionText(fn, d.device_base, sig);

  std::lock_guard<std::mutex> lock(mu_);
  if (frozen_)
    return invalid("this function registry is already in use by a Projector or Filter: register every function "
                   "before the first Make()");
  if (Lookup(fn.name, fn.params) != nullptr) return invalid("user function " + sig + " is already registered");

  // Probe: the prelude, the function and one kernel that calls it, with the options every kernel gets.
  std::string probe = "#include \"gdv_device_lib.cuh\"\n";
  if (fn.can_raise) probe += kUserRaiseHelper;
  probe += d.prelude + d.source;
  probe += "extern \"C\" __global__ void gdv_udf_probe(" + std::string(fn.ret.ctype()) + "* out, int* err) {\n";
  if (fn.can_raise) probe += "  gdv_ctx ctx;\n  ctx.err = err;\n";
  if (fn.nulls == NullMode::kInternal) probe += "  bool ov = false;\n";
  probe += "  *out = " + d.device_base + "(";
  bool first = true;
  auto add = [&](const std::string& a) {
    probe += (first ? "" : ", ") + a;
    first = false;
  };
  if (fn.can_raise) add("&ctx");
  for (const auto& p : fn.params) {
    add(p.is_varlen() ? std::string("gdv_make_str(nullptr, 0)") : std::string("(") + p.ctype() + ")0");
    if (fn.nulls != NullMode::kIfNull) add("true");
  }
  if (fn.nulls == NullMode::kInternal) add("&ov");
  probe += ");\n}\n";
  std::vector<char> cubin;
  std::string log;
  Status st = CompileToCubin(probe, "sm_90a", true, false, &cubin, nullptr, &log);
  if (!st.ok()) {
    if (st.code != GDV_CODEGEN_ERROR) return st;
    return Status::Make(GDV_CODEGEN_ERROR, "user function " + sig + " does not compile:\n" + st.msg);
  }
  defs_.push_back(std::move(d));
  return Status::OK();
}

void FunctionRegistry::Freeze() {
  std::lock_guard<std::mutex> lock(mu_);
  frozen_ = true;
}

const FunctionDef* FunctionRegistry::Lookup(const std::string& name, const std::vector<DataType>& params) const {
  for (const auto& d : defs_) {
    if (d.name != name || d.params.size() != params.size()) continue;
    bool ok = true;
    for (size_t i = 0; i < params.size() && ok; ++i) ok = ParamMatches(d.params[i], params[i]);
    if (ok) return &d;
  }
  return nullptr;
}

FunctionRegistry::Scope::Scope(const FunctionRegistry* reg) : prev_(tl_user_functions) { tl_user_functions = reg; }
FunctionRegistry::Scope::~Scope() { tl_user_functions = prev_; }

const FunctionDef* LookupFunction(const std::string& name, const std::vector<DataType>& params, const DataType& ret) {
  if (const FunctionDef* d = Registry::Get().Lookup(name, params, ret)) return d;
  return tl_user_functions != nullptr ? tl_user_functions->Lookup(name, params) : nullptr;
}

Registry::Registry() {
  const DataType B = boolean();
  const DataType I8(GDV_TYPE_INT8), I16(GDV_TYPE_INT16), I32 = int32(), I64 = int64();
  const DataType U8(GDV_TYPE_UINT8), U16(GDV_TYPE_UINT16), U32(GDV_TYPE_UINT32),
      U64(GDV_TYPE_UINT64);
  const DataType F32 = float32(), F64 = float64();
  const DataType S = utf8(), BIN = binary();
  const DataType D32 = date32(), D64 = date64(), TS = timestamp_ms(), T32 = time32_ms();
  const DataType DEC = decimal128(0, 0);
  const std::vector<DataType> numeric = {I8, I16, I32, I64, U8, U16, U32, U64, F32, F64};
  const std::vector<DataType> dates = {D32, D64, TS, T32};

  // ---- arithmetic -------------------------------------------------------------------
  for (const auto& t : numeric) {
    Add("add", {t, t}, t);
    Add("subtract", {t, t}, t);
    Add("multiply", {t, t}, t);
    Add("divide", {t, t}, t, NullMode::kIfNull, kCanFail);
  }
  Add("mod", {I64, I32}, I32, NullMode::kIfNull, 0, {"modulo"});
  Add("mod", {I64, I64}, I64, NullMode::kIfNull, 0, {"modulo"});
  Add("mod", {I32, I32}, I32, NullMode::kIfNull, 0, {"modulo"});
  Add("mod", {F64, F64}, F64, NullMode::kIfNull, kCanFail, {"modulo"});
  for (const auto& t : {I32, I64, F32, F64}) {
    Add("abs", {t}, t);
    Add("negative", {t}, t);
  }
  for (const auto& t : {I32, I64}) {
    Add("bitwise_and", {t, t}, t);
    Add("bitwise_or", {t, t}, t);
    Add("bitwise_xor", {t, t}, t);
    Add("bitwise_not", {t}, t);
  }
  Add("sqrt", {F64}, F64);
  Add("exp", {F64}, F64);
  Add("log", {F64}, F64, NullMode::kIfNull, 0, {"ln"});
  Add("log10", {F64}, F64);
  Add("log", {F64, F64}, F64, NullMode::kIfNull, kCanFail);
  Add("cbrt", {F64}, F64);
  for (const auto& t : {I32, I64, F32, F64})
    for (const char* f : {"sin", "cos", "tan", "cot"}) Add(f, {t}, F64);
  Add("power", {F64, F64}, F64, NullMode::kIfNull, 0, {"pow"});
  for (const char* f : {"sinh", "cosh", "tanh", "asin", "acos", "atan"}) Add(f, {F64}, F64);
  Add("atan2", {F64, F64}, F64);
  Add("degrees", {F64}, F64);
  Add("radians", {F64}, F64);
  for (const auto& t : {I32, I64}) {
    Add("div", {t, t}, t, NullMode::kIfNull, kCanFail);
    Add("pmod", {t, t}, t);
    Add("factorial", {t}, I64, NullMode::kIfNull, kCanFail);
  }
  Add("bround", {F64}, F64);
  for (const auto& t : {I32, I64, F32, F64}) {
    Add("sign", {t}, t);
    for (size_t n = 2; n <= 4; ++n) {
      Add("greatest", std::vector<DataType>(n, t), t);
      Add("least", std::vector<DataType>(n, t), t);
    }
  }

  // ---- comparisons ------------------------------------------------------------------
  std::vector<DataType> relop_types = numeric;
  relop_types.insert(relop_types.end(), dates.begin(), dates.end());
  relop_types.push_back(S);
  relop_types.push_back(BIN);
  for (const auto& t : relop_types) {
    Add("equal", {t, t}, B, NullMode::kIfNull, 0, {"eq", "same"});
    Add("not_equal", {t, t}, B);
    Add("less_than", {t, t}, B);
    Add("less_than_or_equal_to", {t, t}, B);
    Add("greater_than", {t, t}, B);
    Add("greater_than_or_equal_to", {t, t}, B);
  }
  Add("equal", {B, B}, B, NullMode::kIfNull, 0, {"eq", "same"});
  Add("not_equal", {B, B}, B);
  for (const char* op : {"equal", "not_equal", "less_than", "less_than_or_equal_to",
                         "greater_than", "greater_than_or_equal_to"})
    Add(op, {DEC, DEC}, B, NullMode::kIfNull, kDecimalArgs);

  // ---- boolean / null tests ---------------------------------------------------------
  Add("not", {B}, B);
  std::vector<DataType> all_types = relop_types;
  all_types.push_back(B);
  all_types.push_back(DEC);
  for (const auto& t : all_types) {
    Add("isnull", {t}, B, NullMode::kNever);
    Add("isnotnull", {t}, B, NullMode::kNever);
  }
  Add("istrue", {B}, B, NullMode::kNever);
  Add("isfalse", {B}, B, NullMode::kNever);
  Add("isnottrue", {B}, B, NullMode::kNever);
  Add("isnotfalse", {B}, B, NullMode::kNever);
  std::vector<DataType> distinct_types = numeric;
  distinct_types.insert(distinct_types.end(), dates.begin(), dates.end());
  distinct_types.push_back(B);
  for (const auto& t : distinct_types) {
    Add("is_distinct_from", {t, t}, B, NullMode::kNever);
    Add("is_not_distinct_from", {t, t}, B, NullMode::kNever);
  }

  // ---- casts --------------------------------------------------------------------------
  Add("castBIGINT", {I32}, I64);
  Add("castINT", {I64}, I32);
  Add("castFLOAT4", {I32}, F32);
  Add("castFLOAT4", {I64}, F32);
  Add("castFLOAT4", {F64}, F32);
  Add("castFLOAT8", {I32}, F64);
  Add("castFLOAT8", {I64}, F64);
  Add("castFLOAT8", {F32}, F64);
  Add("castDATE", {I64}, D64);
  Add("castTIMESTAMP", {I64}, TS);
  Add("castTIMESTAMP", {D64}, TS);
  Add("castDATE", {TS}, D64);
  Add("castBIGINT", {D64}, I64);
  Add("castBIGINT", {TS}, I64);
  Add("castINT", {D32}, I32);
  Add("castDATE", {I32}, D32);

  // ---- date / time extraction (date64 and timestamp are milliseconds since epoch) ----
  // SQL-style short names are aliases of the extract* functions (same device function, same signature)
  static const std::pair<const char*, std::vector<std::string>> kExtract[] = {
      {"extractYear", {"year"}},       {"extractMonth", {"month"}},     {"extractDay", {"day", "dayofmonth"}},
      {"extractHour", {"hour"}},       {"extractMinute", {"minute"}},   {"extractSecond", {"second"}},
      {"extractDoy", {"dayofyear"}},   {"extractDow", {"dayofweek"}},   {"extractQuarter", {"quarter"}},
      {"extractEpoch", {}}};
  for (const auto& t : {D64, TS}) {
    for (const auto& e : kExtract) Add(e.first, {t}, I64, NullMode::kIfNull, 0, e.second);
  }
  Add("extractYear", {D32}, I64, NullMode::kIfNull, 0, {"year"});
  Add("extractMonth", {D32}, I64, NullMode::kIfNull, 0, {"month"});
  Add("extractDay", {D32}, I64, NullMode::kIfNull, 0, {"day", "dayofmonth"});

  // ---- rounding ------------------------------------------------------------------------
  Add("round", {F64}, F64);
  Add("round", {F32}, F32);
  Add("round", {I32}, I32);
  Add("round", {I64}, I64);
  Add("round", {F64, I32}, F64);
  Add("ceil", {F64}, F64);
  Add("floor", {F64}, F64);
  Add("truncate", {F64}, F64, NullMode::kIfNull, 0, {"trunc"});
  Add("truncate", {F64, I32}, F64, NullMode::kIfNull, 0, {"trunc"});
  Add("round", {I32, I32}, I32);
  Add("round", {I64, I32}, I64);
  Add("truncate", {I32, I32}, I32, NullMode::kIfNull, 0, {"trunc"});
  Add("truncate", {I64, I32}, I64, NullMode::kIfNull, 0, {"trunc"});

  // ---- date / time arithmetic -------------------------------------------------------------
  // every unit in both argument orders (count, timestamp) / (timestamp, count) and with int32 / int64 counts
  for (const char* f : {"timestampaddSecond", "timestampaddMinute", "timestampaddHour", "timestampaddDay",
                        "timestampaddWeek", "timestampaddMonth", "timestampaddQuarter", "timestampaddYear"}) {
    Add(f, {I32, TS}, TS);
    Add(f, {I64, TS}, TS);
    Add(f, {TS, I32}, TS);
    Add(f, {TS, I64}, TS);
  }
  for (const auto& t : {D64, TS}) {
    Add("add_months", {t, I32}, t);
    Add("add_months", {t, I64}, t);
  }
  Add("date_add", {D64, I32}, D64);
  Add("date_sub", {D64, I32}, D64);
  Add("date_add", {TS, I32}, TS);
  Add("date_sub", {TS, I32}, TS);
  for (const char* f : {"timestampdiffSecond", "timestampdiffMinute", "timestampdiffHour", "timestampdiffDay",
                        "timestampdiffWeek"})
    Add(f, {TS, TS}, I32);

  // ---- calendar fields, truncation, time of day ----------------------------------------------
  for (const auto& t : {D64, TS}) {
    Add("extractWeek", {t}, I64, NullMode::kIfNull, 0, {"weekofyear", "yearweek"});
    for (const char* f : {"extractDecade", "extractCentury", "extractMillennium"}) Add(f, {t}, I64);
    for (const char* u : {"Second", "Minute", "Hour", "Day", "Week", "Month", "Quarter", "Year", "Decade",
                          "Century", "Millennium"})
      Add(std::string("date_trunc_") + u, {t}, t);
    Add("last_day", {t}, D64);
  }
  for (const char* f : {"timestampdiffMonth", "timestampdiffQuarter", "timestampdiffYear"}) Add(f, {TS, TS}, I32);
  Add("months_between", {TS, TS}, F64);
  Add("months_between", {D64, D64}, F64);
  Add("datediff", {TS, TS}, I32);
  Add("datediff", {D64, D64}, I32);
  Add("castTIME", {TS}, T32);
  Add("extractHour", {T32}, I64, NullMode::kIfNull, 0, {"hour"});
  Add("extractMinute", {T32}, I64, NullMode::kIfNull, 0, {"minute"});
  Add("extractSecond", {T32}, I64, NullMode::kIfNull, 0, {"second"});

  // ---- decimal128 ---------------------------------------------------------------------
  Add("add", {DEC, DEC}, DEC, NullMode::kIfNull, kDecimalArgs);
  Add("subtract", {DEC, DEC}, DEC, NullMode::kIfNull, kDecimalArgs);
  Add("multiply", {DEC, DEC}, DEC, NullMode::kIfNull, kDecimalArgs);
  Add("divide", {DEC, DEC}, DEC, NullMode::kIfNull, kDecimalArgs | kCanFail);
  Add("mod", {DEC, DEC}, DEC, NullMode::kIfNull, kDecimalArgs | kCanFail, {"modulo"});
  Add("round", {DEC}, DEC, NullMode::kIfNull, kDecimalArgs);
  Add("round", {DEC, I32}, DEC, NullMode::kIfNull, kDecimalArgs);
  Add("truncate", {DEC}, DEC, NullMode::kIfNull, kDecimalArgs, {"trunc"});
  Add("truncate", {DEC, I32}, DEC, NullMode::kIfNull, kDecimalArgs, {"trunc"});
  Add("ceil", {DEC}, DEC, NullMode::kIfNull, kDecimalArgs);
  Add("floor", {DEC}, DEC, NullMode::kIfNull, kDecimalArgs);
  Add("abs", {DEC}, DEC, NullMode::kIfNull, kDecimalArgs);
  Add("negative", {DEC}, DEC, NullMode::kIfNull, kDecimalArgs);
  Add("castDECIMAL", {I32}, DEC, NullMode::kIfNull, kDecimalArgs);
  Add("castDECIMAL", {I64}, DEC, NullMode::kIfNull, kDecimalArgs);
  Add("castDECIMAL", {F64}, DEC, NullMode::kIfNull, kDecimalArgs);
  Add("castDECIMAL", {F32}, DEC, NullMode::kIfNull, kDecimalArgs);
  Add("castDECIMAL", {DEC}, DEC, NullMode::kIfNull, kDecimalArgs);
  Add("castDECIMAL", {S}, DEC, NullMode::kIfNull, kDecimalArgs | kCanFail);
  Add("castVARCHAR", {DEC, I64}, S, NullMode::kIfNull, kDecimalArgs | kScratch);
  Add("castBIGINT", {DEC}, I64, NullMode::kIfNull, kDecimalArgs);
  Add("castFLOAT8", {DEC}, F64, NullMode::kIfNull, kDecimalArgs);

  // ---- hashes (never null: a null input yields the seed) --------------------------------
  std::vector<DataType> hash_types = numeric;
  hash_types.insert(hash_types.end(), dates.begin(), dates.end());
  hash_types.push_back(B);
  hash_types.push_back(S);
  hash_types.push_back(BIN);
  for (const auto& t : hash_types) {
    const bool num = !t.is_varlen();
    Add("hash32", {t}, I32, NullMode::kNever, 0,
        num ? std::vector<std::string>{"hash", "hash32AsDouble"} : std::vector<std::string>{"hash"});
    Add("hash32", {t, I32}, I32, NullMode::kNever, 0,
        num ? std::vector<std::string>{"hash32AsDouble"} : std::vector<std::string>{});
    Add("hash64", {t}, I64, NullMode::kNever, 0,
        num ? std::vector<std::string>{"hash64AsDouble"} : std::vector<std::string>{});
    Add("hash64", {t, I64}, I64, NullMode::kNever, 0,
        num ? std::vector<std::string>{"hash64AsDouble"} : std::vector<std::string>{});
  }

  // ---- strings ------------------------------------------------------------------------
  Add("regexp_matches", {S, S}, B, NullMode::kIfNull, kRegexHolder, {"regexp_like"});
  Add("like", {S, S}, B, NullMode::kIfNull, kLikeHolder);
  Add("like", {S, S, S}, B, NullMode::kIfNull, kLikeHolder);
  Add("substr", {S, I64, I64}, S, NullMode::kIfNull, kStringView, {"substring"});
  Add("substr", {S, I64}, S, NullMode::kIfNull, kStringView, {"substring"});
  Add("upper", {S}, S, NullMode::kIfNull, kStringView);
  Add("lower", {S}, S, NullMode::kIfNull, kStringView);
  Add("initcap", {S}, S, NullMode::kIfNull, kStringView);
  Add("to_date", {S, S}, D64, NullMode::kInternal, kDateFormat | kCanFail);
  Add("to_date", {S, S, I32}, D64, NullMode::kInternal, kDateFormat | kCanFail);
  Add("char_length", {S}, I32, NullMode::kIfNull, 0, {"length", "lengthUtf8"});
  Add("octet_length", {S}, I32);
  Add("octet_length", {BIN}, I32);
  Add("bit_length", {S}, I32);
  Add("bit_length", {BIN}, I32);
  Add("starts_with", {S, S}, B);
  Add("ends_with", {S, S}, B);
  Add("is_substr", {S, S}, B);
  Add("ltrim", {S}, S, NullMode::kIfNull, kStringView);
  Add("rtrim", {S}, S, NullMode::kIfNull, kStringView);
  Add("btrim", {S}, S, NullMode::kIfNull, kStringView, {"trim"});
  Add("castVARCHAR", {S, I64}, S, NullMode::kIfNull, kStringView);
  // numbers / dates as text: the digits are written into a thread-private scratch slot
  Add("castVARCHAR", {F32, I64}, S, NullMode::kIfNull, kScratch);
  Add("castVARCHAR", {F64, I64}, S, NullMode::kIfNull, kScratch);
  Add("castVARCHAR", {I32, I64}, S, NullMode::kIfNull, kScratch);
  Add("castVARCHAR", {I64, I64}, S, NullMode::kIfNull, kScratch);
  Add("castVARCHAR", {D64, I64}, S, NullMode::kIfNull, kScratch);
  Add("castVARCHAR", {TS, I64}, S, NullMode::kIfNull, kScratch);
  Add("castVARCHAR", {B, I64}, S);
  // new bytes without a bound: virtual pieces (periodic / reversed views) read by the write pass only
  Add("replace", {S, S, S}, S, NullMode::kIfNull, kVirtual);   // from / to must be literals
  Add("repeat", {S, I32}, S, NullMode::kIfNull, kVirtual);
  Add("space", {I32}, S, NullMode::kIfNull, kVirtual);
  Add("reverse", {S}, S, NullMode::kIfNull, kVirtual);
  Add("lpad", {S, I32, S}, S, NullMode::kIfNull, kVirtual);
  Add("rpad", {S, I32, S}, S, NullMode::kIfNull, kVirtual);
  Add("lpad", {S, I32}, S, NullMode::kIfNull, kVirtual);
  Add("rpad", {S, I32}, S, NullMode::kIfNull, kVirtual);
  Add("ascii", {S}, I32);
  Add("left", {S, I32}, S, NullMode::kIfNull, kStringView);
  Add("right", {S, I32}, S, NullMode::kIfNull, kStringView);
  Add("locate", {S, S}, I32, NullMode::kIfNull, 0, {"position"});
  Add("locate", {S, S, I32}, I32);
  Add("strpos", {S, S}, I32, NullMode::kIfNull, 0, {"instr"});
  Add("byte_substr", {BIN, I32, I32}, BIN, NullMode::kIfNull, kStringView, {"bytesubstring"});
  Add("ltrim", {S, S}, S, NullMode::kIfNull, kStringView);
  Add("rtrim", {S, S}, S, NullMode::kIfNull, kStringView);
  Add("btrim", {S, S}, S, NullMode::kIfNull, kStringView, {"trim"});
  Add("split_part", {S, S, I32}, S, NullMode::kIfNull, kStringView | kCanFail);
  for (const auto& t : {S, BIN}) {   // digests as lower-case hex text
    Add("hashSHA256", {t}, S, NullMode::kIfNull, kScratch, {"sha256"});
    Add("hashSHA1", {t}, S, NullMode::kIfNull, kScratch, {"sha1"});
    Add("hashMD5", {t}, S, NullMode::kIfNull, kScratch, {"md5"});
  }
  Add("crc32", {S}, I64);
  Add("crc32", {BIN}, I64);
  Add("to_hex", {I64}, S, NullMode::kIfNull, kScratch);
  Add("to_hex", {I32}, S, NullMode::kIfNull, kScratch);
  Add("castBIT", {S}, B, NullMode::kIfNull, kCanFail, {"castBOOLEAN"});
  Add("find_in_set", {S, S}, I32);
  for (const auto& t : {F32, F64}) {
    Add("castBIGINT", {t}, I64);
    Add("castINT", {t}, I32);
  }
  for (const auto& t : {I32, I64, F32, F64}) {
    Add("to_timestamp", {t}, TS);
    Add("to_time", {t}, T32);
  }
  Add("castBIGINT", {S}, I64, NullMode::kIfNull, kCanFail);
  Add("castINT", {S}, I32, NullMode::kIfNull, kCanFail);
  Add("castFLOAT8", {S}, F64, NullMode::kIfNull, kCanFail);
  Add("castFLOAT4", {S}, F32, NullMode::kIfNull, kCanFail);
  Add("castDATE", {S}, D64, NullMode::kIfNull, kCanFail);
  Add("castTIMESTAMP", {S}, TS, NullMode::kIfNull, kCanFail);
  // ilike(s, pattern): like() over lower-cased text and pattern (ASCII case folding); rewritten
  // at Make() (RewriteAliases), never called as a device function
  Add("ilike", {S, S}, B, NullMode::kIfNull, kLikeHolder);
  // nvl(a, b): a when a is valid, else b; lowered by the fuser itself
  {
    std::vector<DataType> nvl_types = numeric;
    nvl_types.insert(nvl_types.end(), dates.begin(), dates.end());
    nvl_types.push_back(B);
    nvl_types.push_back(S);
    nvl_types.push_back(BIN);
    for (const auto& t : nvl_types) Add("nvl", {t, t}, t, NullMode::kInternal);
  }
  // concat: null arguments are empty strings, never null; concatOperator: null if any is null.  2..10 arguments
  // like the reference; a rope holds 8 pieces, wider concats are folded through temporaries (gdv_rope_temps.h)
  for (int n = 2; n <= 10; ++n) {
    Add("concat", std::vector<DataType>(static_cast<size_t>(n), S), S, NullMode::kNever, kConcat);
    Add("concatOperator", std::vector<DataType>(static_cast<size_t>(n), S), S, NullMode::kIfNull, kConcat);
  }
  AddTimeUnits();
}

// The twins of every timestamp[ms] / time32[ms] signature at the other units: timestamp[s|us|ns] with the
// time of day in time32[s], time64[us], time64[ns].  They come after every millisecond signature, so the
// enumeration keeps its earlier entries and order, and each of them mentions a non-millisecond type.
// Constructors (castTIMESTAMP, to_timestamp, to_time) take the declared return type's unit: Lookup
// prefers the def whose return type matches, and their device functions carry the unit in the name
// (castTIMESTAMP_us_int64, ...).
void Registry::AddTimeUnits() {
  const DataType B = boolean(), I32 = int32(), I64 = int64(), F32 = float32(), F64 = float64(), S = utf8();
  const DataType D64 = date64();
  static const char* const kUnitName[4] = {"s", "ms", "us", "ns"};
  auto ts = [](int u) { return DataType(GDV_TYPE_TIMESTAMP, u); };
  auto tt = [](int u) { return u <= 1 ? DataType(GDV_TYPE_TIME32, u) : DataType(GDV_TYPE_TIME64, u); };
  auto ctor = [&](const char* name, std::vector<DataType> params, const DataType& ret, int unit, uint32_t flags = 0) {
    Add(name, std::move(params), ret, NullMode::kIfNull, flags);
    defs_.back().device_base = std::string(name) + "_" + kUnitName[unit];
  };
  static const std::pair<const char*, std::vector<std::string>> kExtract[] = {
      {"extractYear", {"year"}},       {"extractMonth", {"month"}},     {"extractDay", {"day", "dayofmonth"}},
      {"extractHour", {"hour"}},       {"extractMinute", {"minute"}},   {"extractSecond", {"second"}},
      {"extractDoy", {"dayofyear"}},   {"extractDow", {"dayofweek"}},   {"extractQuarter", {"quarter"}},
      {"extractEpoch", {}}};
  for (int u : {0, 2, 3}) {
    const DataType TS = ts(u), TT = tt(u);
    for (const auto& t : {TS, TT}) {
      Add("equal", {t, t}, B, NullMode::kIfNull, 0, {"eq", "same"});
      Add("not_equal", {t, t}, B);
      Add("less_than", {t, t}, B);
      Add("less_than_or_equal_to", {t, t}, B);
      Add("greater_than", {t, t}, B);
      Add("greater_than_or_equal_to", {t, t}, B);
      Add("isnull", {t}, B, NullMode::kNever);
      Add("isnotnull", {t}, B, NullMode::kNever);
      Add("is_distinct_from", {t, t}, B, NullMode::kNever);
      Add("is_not_distinct_from", {t, t}, B, NullMode::kNever);
      Add("hash32", {t}, I32, NullMode::kNever, 0, {"hash", "hash32AsDouble"});
      Add("hash32", {t, I32}, I32, NullMode::kNever, 0, {"hash32AsDouble"});
      Add("hash64", {t}, I64, NullMode::kNever, 0, {"hash64AsDouble"});
      Add("hash64", {t, I64}, I64, NullMode::kNever, 0, {"hash64AsDouble"});
      Add("nvl", {t, t}, t, NullMode::kInternal);
    }
    Add("castBIGINT", {TS}, I64);
    Add("castDATE", {TS}, D64);
    for (const auto& e : kExtract) Add(e.first, {TS}, I64, NullMode::kIfNull, 0, e.second);
    Add("extractWeek", {TS}, I64, NullMode::kIfNull, 0, {"weekofyear", "yearweek"});
    for (const char* f : {"extractDecade", "extractCentury", "extractMillennium"}) Add(f, {TS}, I64);
    for (const char* un : {"Second", "Minute", "Hour", "Day", "Week", "Month", "Quarter", "Year", "Decade",
                           "Century", "Millennium"})
      Add(std::string("date_trunc_") + un, {TS}, TS);
    Add("last_day", {TS}, D64);
    for (const char* f : {"timestampaddSecond", "timestampaddMinute", "timestampaddHour", "timestampaddDay",
                          "timestampaddWeek", "timestampaddMonth", "timestampaddQuarter", "timestampaddYear"}) {
      Add(f, {I32, TS}, TS);
      Add(f, {I64, TS}, TS);
      Add(f, {TS, I32}, TS);
      Add(f, {TS, I64}, TS);
    }
    Add("add_months", {TS, I32}, TS);
    Add("add_months", {TS, I64}, TS);
    Add("date_add", {TS, I32}, TS);
    Add("date_sub", {TS, I32}, TS);
    for (const char* f : {"timestampdiffSecond", "timestampdiffMinute", "timestampdiffHour", "timestampdiffDay",
                          "timestampdiffWeek", "timestampdiffMonth", "timestampdiffQuarter", "timestampdiffYear"})
      Add(f, {TS, TS}, I32);
    Add("months_between", {TS, TS}, F64);
    Add("datediff", {TS, TS}, I32);
    Add("castTIME", {TS}, TT);
    Add("extractHour", {TT}, I64, NullMode::kIfNull, 0, {"hour"});
    Add("extractMinute", {TT}, I64, NullMode::kIfNull, 0, {"minute"});
    Add("extractSecond", {TT}, I64, NullMode::kIfNull, 0, {"second"});
    Add("castVARCHAR", {TS, I64}, S, NullMode::kIfNull, kScratch);
    // constructors in this unit
    ctor("castTIMESTAMP", {I64}, TS, u);
    ctor("castTIMESTAMP", {D64}, TS, u);
    ctor("castTIMESTAMP", {S}, TS, u, kCanFail);
    for (const auto& t : {I32, I64, F32, F64}) {
      ctor("to_timestamp", {t}, TS, u);
      ctor("to_time", {t}, TT, u);
    }
  }
  // unit conversions between any two different units
  for (int to = 0; to < 4; ++to)
    for (int from = 0; from < 4; ++from)
      if (from != to) ctor("castTIMESTAMP", {ts(from)}, ts(to), to);
}

}  // namespace gdv
