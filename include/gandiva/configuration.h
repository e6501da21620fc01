// gandiva/configuration.h (P/includes/libgandiva.pxd:279-298).
#pragma once
#include <memory>

#include "gandiva/arrow.h"
#include "gandiva/function_registry.h"

namespace gandiva {

class GANDIVA_EXPORT Configuration {
 public:
  Configuration() = default;
  Configuration(bool optimize, bool dump_ir) : optimize_(optimize), dump_ir_(dump_ir) {}
  bool optimize() const { return optimize_; }
  bool dump_ir() const { return dump_ir_; }
  int device() const { return device_; }
  void set_optimize(bool optimize) { optimize_ = optimize; }
  void set_dump_ir(bool dump_ir) { dump_ir_ = dump_ir; }
  /// CUDA device ordinal the Projector / Filter is placed on (extension; default 0).
  void set_device(int device) { device_ = device; }
  /// User functions looked up after the built-ins (null = none).
  const std::shared_ptr<FunctionRegistry>& function_registry() const { return function_registry_; }
  void set_function_registry(std::shared_ptr<FunctionRegistry> r) { function_registry_ = std::move(r); }
  /// Two configurations are equal when they build the same kernels: same options, same registry object.
  bool operator==(const Configuration& o) const {
    return optimize_ == o.optimize_ && dump_ir_ == o.dump_ir_ && device_ == o.device_ &&
           function_registry_ == o.function_registry_;
  }
  bool operator!=(const Configuration& o) const { return !(*this == o); }

 private:
  bool optimize_ = true;
  bool dump_ir_ = false;
  int device_ = 0;
  std::shared_ptr<FunctionRegistry> function_registry_;
};

class GANDIVA_EXPORT ConfigurationBuilder {
 public:
  std::shared_ptr<Configuration> build() { return std::make_shared<Configuration>(); }
  std::shared_ptr<Configuration> build(bool dump_ir) {
    return std::make_shared<Configuration>(true, dump_ir);
  }
  std::shared_ptr<Configuration> build(std::shared_ptr<FunctionRegistry> function_registry) {
    auto c = std::make_shared<Configuration>();
    c->set_function_registry(std::move(function_registry));
    return c;
  }
  static std::shared_ptr<Configuration> DefaultConfiguration() {
    static std::shared_ptr<Configuration> c = std::make_shared<Configuration>();
    return c;
  }
};

}  // namespace gandiva
