// gandiva/function_registry.h — user-defined functions (the counterpart of Arrow Gandiva's external
// FunctionRegistry handed over through Configuration).  A function arrives as CUDA text and is fused
// into every Projector / Filter kernel that calls it; include/gandiva_b200.h ("user-defined functions")
// states the calling convention of `body` per NullMode.
#pragma once
#include <memory>
#include <string>
#include <vector>

#include "gandiva/arrow.h"
#include "gandiva/function_signature.h"

namespace gandiva {

class GANDIVA_EXPORT FunctionRegistry {
 public:
  enum class NullMode {
    kIfNull = 0,    // T f(a0, a1, ...): null iff an argument is null
    kNever = 1,     // T f(a0, bool v0, ...): never null
    kInternal = 2,  // T f(a0, bool v0, ..., bool* out_valid)
  };

  FunctionRegistry();
  ~FunctionRegistry();
  FunctionRegistry(const FunctionRegistry&) = delete;
  FunctionRegistry& operator=(const FunctionRegistry&) = delete;

  /// Validates the function and compiles it once for sm_90a (no GPU needed).  Fails with CodeGenError and
  /// NVRTC's log when `body` does not compile, with Invalid once a Projector or Filter uses the registry.
  Status Register(const FunctionSignature& signature, const std::string& body,
                  NullMode null_mode = NullMode::kIfNull, bool can_raise = false,
                  const std::string& prelude = "");
  /// The signatures of this registry only (ExpressionRegistry lists the built-ins).
  std::vector<FunctionSignature> GetSignatures() const;

  void* handle() const { return handle_; }

 private:
  void* handle_ = nullptr;
};

}  // namespace gandiva
