// Function registry: name + parameter types + return type -> device function and its
// null behaviour.  Replaces the reference's precompiled-bitcode function_registry
// (named in BASELINE.json north_star; enumeration API P/includes/libgandiva.pxd:258-277).
// Device functions live in device/gdv_device_lib.cuh and are named
// <base>_<suffix of each param>, the reference library's naming scheme.
#pragma once
#include <deque>
#include <mutex>
#include <string>
#include <vector>

#include "gdv_types.h"

namespace gdv {

enum class NullMode {
  kIfNull,    // result is null iff any input is null; function sees values only
  kNever,     // result is never null; function receives (value, valid) pairs
  kInternal,  // function computes validity: receives (value, valid) pairs + bool* out_valid
};

enum FnFlags : uint32_t {
  kCanFail = 1u << 0,      // may raise an ExecutionError -> takes gdv_ctx*, only called on valid rows
  kLikeHolder = 1u << 1,   // second (third) arg must be a literal pattern, compiled at Make()
  kDecimalArgs = 1u << 2,  // decimal params are followed by (precision, scale); out (p, s) appended
  kStringView = 1u << 3,   // returns a view/transform of its first argument (no new bytes)
  kConcat = 1u << 4,       // result = the pieces of its arguments in order (a rope, see the fuser)
  kScratch = 1u << 5,      // writes its result bytes into a per-row scratch slot passed as last argument
  kRegexHolder = 1u << 7,  // second arg is a literal regular expression, compiled at Make() (gdv_regex.h)
  kDateFormat = 1u << 8,   // second arg is a literal date format, compiled at Make() (gdv_datefmt.h); a third
                           // (int32 literal) argument suppresses parse errors: the row is NULL instead
  kVirtual = 1u << 6,      // result is a rope of "virtual" pieces (repeated / reversed bytes) that only the
                           // string write pass can read: projectable, concat-able, if/else-able, nothing else
};

struct FunctionDef {
  std::string name;               // name as written by the user (alias or canonical)
  std::string device_base;        // canonical base used for the device symbol
  std::vector<DataType> params;   // decimal params match any precision/scale
  DataType ret;                   // decimal: precision/scale come from the call site
  NullMode nulls = NullMode::kIfNull;
  uint32_t flags = 0;
  // User functions (FunctionRegistry) only: the file-scope text the caller supplied and the complete
  // definition of the device function, written into every kernel that calls it.  device_base is then
  // the whole symbol (gdv_udf_<hash>).
  std::string prelude;
  std::string source;
  bool is_user() const { return !source.empty(); }
  std::string device_name() const;  // e.g. add_int32_int32
  std::string signature() const;    // "int32 add(int32, int32)"
};

class Registry {
 public:
  static const Registry& Get();
  // Exact match on name and parameter types (decimal: id only; timestamp/time: unit too).  Among the
  // defs that match, the one whose return type equals `ret` (the type the call site declares) wins,
  // else the first: constructors such as castTIMESTAMP(int64) exist once per result unit.
  const FunctionDef* Lookup(const std::string& name, const std::vector<DataType>& params, const DataType& ret) const;
  const std::vector<FunctionDef>& all() const { return defs_; }

 private:
  Registry();
  void Add(const std::string& name, std::vector<DataType> params, DataType ret,
           NullMode nulls = NullMode::kIfNull, uint32_t flags = 0,
           const std::vector<std::string>& aliases = {});
  void AddTimeUnits();
  std::vector<FunctionDef> defs_;
};

struct Status;

// What a caller hands to FunctionRegistry::Register: a signature plus the statements of the device
// function (see include/gandiva_b200.h, gdv_function_def_t, for the calling convention).
struct UserFunction {
  std::string name;
  std::vector<DataType> params;
  DataType ret;
  NullMode nulls = NullMode::kIfNull;
  bool can_raise = false;
  std::string body;
  std::string prelude;
};

// Functions a caller adds to the engine: CUDA text that the fuser writes into the kernels that call it
// (DESIGN.md §3.8).  A registry is scoped by the Config handed to Make(); the built-in table
// (Registry::Get()) and its enumeration never change.
//
// Lifetime rule: Register() may be called until the first Make() that is given the registry; that Make()
// freezes it (later Register() calls fail with GDV_INVALID).  A frozen registry is read without locks, so
// any number of threads may Make() against it, and Projectors / Filters keep it alive.
class FunctionRegistry {
 public:
  // Validates the definition and compiles it once with NVRTC for sm_90a (no GPU needed): a body that does
  // not compile is refused here with GDV_CODEGEN_ERROR and NVRTC's log.
  Status Register(const UserFunction& fn);
  void Freeze();
  const FunctionDef* Lookup(const std::string& name, const std::vector<DataType>& params) const;
  const std::deque<FunctionDef>& all() const { return defs_; }

  // Makes `reg` (may be null) the registry that LookupFunction() consults on this thread after the
  // built-ins, for the lifetime of the object: validation and kernel generation run inside one.
  class Scope {
   public:
    explicit Scope(const FunctionRegistry* reg);
    ~Scope();
    Scope(const Scope&) = delete;
    Scope& operator=(const Scope&) = delete;

   private:
    const FunctionRegistry* prev_;
  };

 private:
  mutable std::mutex mu_;
  bool frozen_ = false;
  std::deque<FunctionDef> defs_;  // a deque: definitions never move once a kernel plan points at them
};

// Text of gdv_raise(ctx, "message"), written into a kernel before its first user function that can raise.
extern const char kUserRaiseHelper[];

// Built-ins first, then the registry of the enclosing FunctionRegistry::Scope.  `ret` is the return type
// the call site declares (see Registry::Lookup).
const FunctionDef* LookupFunction(const std::string& name, const std::vector<DataType>& params, const DataType& ret);

}  // namespace gdv
