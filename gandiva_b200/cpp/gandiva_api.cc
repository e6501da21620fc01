// namespace gandiva — the reference's public C++ API (P/includes/libgandiva.pxd:27-298)
// implemented as a thin layer over the C-ABI of libgandiva_b200.so.  Links libarrow only for
// the Arrow types that appear in the signatures (RecordBatch, Array, MemoryPool, Status).
#include <cstring>
#include <memory>

#include "arrow/array/util.h"
#include "arrow/buffer.h"
#include "arrow/device.h"
#include "arrow/util/bit_util.h"
#include "gandiva/condition.h"
#include "gandiva/device.h"
#include "gandiva/configuration.h"
#include "gandiva/expression.h"
#include "gandiva/expression_registry.h"
#include "gandiva/filter.h"
#include "gandiva/function_registry.h"
#include "gandiva/function_signature.h"
#include "gandiva/node.h"
#include "gandiva/projector.h"
#include "gandiva/selection_vector.h"
#include "gandiva/tree_expr_builder.h"
#include "gandiva_b200.h"

namespace gandiva {

namespace {

gdv_type_t ToC(const arrow::DataType& t) {
  gdv_type_t c{static_cast<int32_t>(t.id()), 0, 0};
  switch (t.id()) {
    case arrow::Type::DECIMAL128: {
      const auto& d = static_cast<const arrow::Decimal128Type&>(t);
      c.precision = d.precision();
      c.scale = d.scale();
      break;
    }
    case arrow::Type::TIMESTAMP:
      c.precision = static_cast<int32_t>(static_cast<const arrow::TimestampType&>(t).unit());
      break;
    case arrow::Type::TIME32:
      c.precision = static_cast<int32_t>(static_cast<const arrow::Time32Type&>(t).unit());
      break;
    case arrow::Type::TIME64:
      c.precision = static_cast<int32_t>(static_cast<const arrow::Time64Type&>(t).unit());
      break;
    default: break;
  }
  return c;
}

DataTypePtr FromC(const gdv_type_t& t) {
  switch (t.id) {
    case GDV_TYPE_BOOL: return arrow::boolean();
    case GDV_TYPE_UINT8: return arrow::uint8();
    case GDV_TYPE_INT8: return arrow::int8();
    case GDV_TYPE_UINT16: return arrow::uint16();
    case GDV_TYPE_INT16: return arrow::int16();
    case GDV_TYPE_UINT32: return arrow::uint32();
    case GDV_TYPE_INT32: return arrow::int32();
    case GDV_TYPE_UINT64: return arrow::uint64();
    case GDV_TYPE_INT64: return arrow::int64();
    case GDV_TYPE_FLOAT: return arrow::float32();
    case GDV_TYPE_DOUBLE: return arrow::float64();
    case GDV_TYPE_STRING: return arrow::utf8();
    case GDV_TYPE_BINARY: return arrow::binary();
    case GDV_TYPE_STRING_VIEW: return arrow::utf8_view();
    case GDV_TYPE_BINARY_VIEW: return arrow::binary_view();
    case GDV_TYPE_LARGE_STRING: return arrow::large_utf8();
    case GDV_TYPE_LARGE_BINARY: return arrow::large_binary();
    case GDV_TYPE_DATE32: return arrow::date32();
    case GDV_TYPE_DATE64: return arrow::date64();
    case GDV_TYPE_TIMESTAMP: return arrow::timestamp(static_cast<arrow::TimeUnit::type>(t.precision));
    case GDV_TYPE_TIME32: return arrow::time32(static_cast<arrow::TimeUnit::type>(t.precision));
    case GDV_TYPE_TIME64: return arrow::time64(static_cast<arrow::TimeUnit::type>(t.precision));
    case GDV_TYPE_DECIMAL128: return arrow::decimal128(t.precision > 0 ? t.precision : 38, t.scale);
    default: return arrow::null();
  }
}

// gdv_status values are arrow::StatusCode values (40/41/42 included); CUDA failures map to
// ExecutionError so callers that only know Gandiva's codes still see an error.
Status ToStatus(gdv_status st) {
  if (st == GDV_OK) return Status::OK();
  const std::string msg = gdv_last_error();
  switch (st) {
    case GDV_OUT_OF_MEMORY: return Status::OutOfMemory(msg);
    case GDV_INVALID: return Status::Invalid(msg);
    case GDV_NOT_IMPLEMENTED: return Status::NotImplemented(msg);
    case GDV_CODEGEN_ERROR: return Status::CodeGenError(msg);
    case GDV_EXPRESSION_VALIDATION_ERROR: return Status::ExpressionValidationError(msg);
    case GDV_EXECUTION_ERROR: return Status::ExecutionError(msg);
    default: return Status::ExecutionError("CUDA: ", msg);
  }
}

std::string HandleToString(int64_t (*fn)(void*, char*, int64_t), void* h) {
  const int64_t n = fn(h, nullptr, 0);
  if (n < 0) return "";
  std::string s(static_cast<size_t>(n) + 1, '\0');
  fn(h, &s[0], n + 1);
  s.resize(static_cast<size_t>(n));
  return s;
}

template <typename T>
NodePtr MakeFixedLiteral(DataTypePtr type, T value) {
  gdv_node_t h = nullptr;
  if (gdv_node_literal(ToC(*type), &value, sizeof(T), 0, &h) != GDV_OK) return nullptr;
  return std::make_shared<Node>(std::move(type), h);
}

NodePtr MakeBytesLiteral(DataTypePtr type, const std::string& value) {
  gdv_node_t h = nullptr;
  if (gdv_node_literal(ToC(*type), value.data(), static_cast<int64_t>(value.size()), 0, &h) != GDV_OK)
    return nullptr;
  return std::make_shared<Node>(std::move(type), h);
}

std::vector<gdv_node_t> Handles(const NodeVector& nodes, bool* ok) {
  std::vector<gdv_node_t> hs;
  *ok = true;
  for (const auto& n : nodes) {
    if (n == nullptr) {
      *ok = false;
      break;
    }
    hs.push_back(static_cast<gdv_node_t>(n->handle()));
  }
  return hs;
}

template <typename T>
NodePtr MakeIn(NodePtr node, DataTypePtr type, const std::unordered_set<T>& constants) {
  if (node == nullptr) return nullptr;
  std::vector<T> vals(constants.begin(), constants.end());
  gdv_node_t h = nullptr;
  if (gdv_node_in(static_cast<gdv_node_t>(node->handle()), ToC(*type), vals.data(), nullptr,
                  static_cast<int32_t>(vals.size()), &h) != GDV_OK)
    return nullptr;
  return std::make_shared<Node>(arrow::boolean(), h);
}

NodePtr MakeInBytes(NodePtr node, DataTypePtr type, const std::unordered_set<std::string>& constants) {
  if (node == nullptr) return nullptr;
  std::string blob;
  std::vector<int32_t> lens;
  for (const auto& s : constants) {
    blob += s;
    lens.push_back(static_cast<int32_t>(s.size()));
  }
  gdv_node_t h = nullptr;
  const char dummy = 0;
  if (gdv_node_in(static_cast<gdv_node_t>(node->handle()), ToC(*type), blob.empty() ? &dummy : blob.data(),
                  lens.data(), static_cast<int32_t>(lens.size()), &h) != GDV_OK)
    return nullptr;
  return std::make_shared<Node>(arrow::boolean(), h);
}

gdv_schema_t MakeSchemaHandle(const arrow::Schema& schema) {
  std::vector<const char*> names;
  std::vector<gdv_type_t> types;
  for (const auto& f : schema.fields()) {
    names.push_back(f->name().c_str());
    types.push_back(ToC(*f->type()));
  }
  gdv_schema_t h = nullptr;
  gdv_schema_make(names.data(), types.data(), static_cast<int32_t>(names.size()), &h);
  return h;
}

gdv_config_t ConfigToC(const std::shared_ptr<Configuration>& c) {
  gdv_config_t cfg;
  gdv_config_default(&cfg);
  if (c != nullptr) {
    cfg.optimize = c->optimize() ? 1 : 0;
    cfg.dump_ir = c->dump_ir() ? 1 : 0;
    cfg.device = c->device();
    if (c->function_registry() != nullptr)
      cfg.function_registry = static_cast<gdv_function_registry_t>(c->function_registry()->handle());
  }
  return cfg;
}

// The data buffers of a string_view / binary_view column (buffers[2..] of its ArrayData), held for
// one Evaluate call: the pointer table, the sizes (copied into device memory for a device batch) and
// the gdv_view_buffers_t the column's var_data points at.
struct ViewBuffers {
  std::vector<const void*> data;
  std::vector<int64_t> sizes;
  std::shared_ptr<arrow::Buffer> device_sizes;
  std::shared_ptr<arrow::MemoryManager> mm;
  gdv_view_buffers_t c{};
};

// RecordBatch -> raw buffer addresses (arrow::ArrayData, P/include/arrow/array/data.h:468-474).
// All buffers of a batch must live in one memory space: CPU (GDV_MEM_HOST, staged by the engine) or the
// HBM of one GPU (GDV_MEM_DEVICE: kernels read them in place).  *mm = the MemoryManager of the first
// device buffer, from which device outputs are allocated.  View columns' descriptors go to *views.
Status ToColumns(const arrow::RecordBatch& batch, std::vector<gdv_column_t>* cols, int* mem_space,
                 std::shared_ptr<arrow::MemoryManager>* mm, std::vector<std::unique_ptr<ViewBuffers>>* views) {
  int n_cpu = 0, n_dev = 0;
  for (int i = 0; i < batch.num_columns(); ++i) {
    const arrow::ArrayData& a = *batch.column_data(i);
    gdv_column_t c;
    std::memset(&c, 0, sizeof(c));
    for (const auto& b : a.buffers) {
      if (b == nullptr) continue;
      if (b->is_cpu()) {
        ++n_cpu;
      } else {
        if (b->device_type() != arrow::DeviceAllocationType::kCUDA &&
            b->device_type() != arrow::DeviceAllocationType::kCUDA_MANAGED)
          return Status::NotImplemented("buffers of device type ", static_cast<int>(b->device_type()),
                                        " (only CPU and CUDA memory can be evaluated)");
        ++n_dev;
        if (mm != nullptr && *mm == nullptr) *mm = b->memory_manager();
      }
    }
    // address() is valid for both spaces (data() is null for non-CPU buffers).  null_count is read as
    // stored: computing it would walk a bitmap that may live in HBM.
    if (a.buffers.size() > 0 && a.buffers[0] != nullptr && a.null_count.load() != 0)
      c.validity = reinterpret_cast<const void*>(a.buffers[0]->address());
    if (a.buffers.size() > 1 && a.buffers[1] != nullptr) c.values = reinterpret_cast<const void*>(a.buffers[1]->address());
    const auto tid = a.type->id();
    if (tid == arrow::Type::STRING_VIEW || tid == arrow::Type::BINARY_VIEW) {
      auto v = std::make_unique<ViewBuffers>();
      for (size_t k = 2; k < a.buffers.size(); ++k) {
        const auto& b = a.buffers[k];
        v->data.push_back(b != nullptr ? reinterpret_cast<const void*>(b->address()) : nullptr);
        v->sizes.push_back(b != nullptr ? b->size() : 0);
        if (b != nullptr && !b->is_cpu() && v->mm == nullptr) v->mm = b->memory_manager();
      }
      v->c.data = v->data.data();
      v->c.sizes = v->sizes.data();
      v->c.n = static_cast<int32_t>(v->data.size());
      c.var_data = &v->c;
      views->push_back(std::move(v));
    } else if (a.buffers.size() > 2 && a.buffers[2] != nullptr) {
      c.var_data = reinterpret_cast<const void*>(a.buffers[2]->address());
      c.var_data_size = a.buffers[2]->size();
    }
    c.offset = a.offset;
    cols->push_back(c);
  }
  if (n_cpu > 0 && n_dev > 0)
    return Status::Invalid("the buffers of a RecordBatch must all be in host memory or all in device memory");
  *mem_space = n_dev > 0 ? GDV_MEM_DEVICE : GDV_MEM_HOST;
  if (*mem_space == GDV_MEM_DEVICE) {
    // the engine reads a device batch's view sizes on the device
    for (auto& v : *views) {
      if (v->sizes.empty()) continue;
      if (v->mm == nullptr) return Status::Invalid("a device string_view column has no device data buffer");
      auto host = std::make_shared<arrow::Buffer>(reinterpret_cast<const uint8_t*>(v->sizes.data()),
                                                  static_cast<int64_t>(v->sizes.size() * 8));
      ARROW_ASSIGN_OR_RAISE(v->device_sizes, arrow::MemoryManager::CopyBuffer(host, v->mm));
      v->c.sizes = reinterpret_cast<const int64_t*>(v->device_sizes->address());
    }
  }
  return Status::OK();
}

int SelModeToC(SelectionVector::Mode m) {
  switch (m) {
    case SelectionVector::MODE_UINT16: return GDV_SEL_UINT16;
    case SelectionVector::MODE_UINT32: return GDV_SEL_UINT32;
    case SelectionVector::MODE_UINT64: return GDV_SEL_UINT64;
    default: return GDV_SEL_NONE;
  }
}

int64_t NodeToStringFn(void* h, char* b, int64_t n) { return gdv_node_to_string(static_cast<gdv_node_t>(h), b, n); }
int64_t ProjDumpFn(void* h, char* b, int64_t n) { return gdv_projector_dump_ir(static_cast<gdv_projector_t>(h), b, n); }
int64_t FiltDumpFn(void* h, char* b, int64_t n) { return gdv_filter_dump_ir(static_cast<gdv_filter_t>(h), b, n); }

}  // namespace

// ---- Node / Expression / Condition ---------------------------------------------------------
Node::Node(DataTypePtr return_type, void* handle)
    : return_type_(std::move(return_type)), handle_(handle) {}
Node::~Node() { gdv_node_release(static_cast<gdv_node_t>(handle_)); }
std::string Node::ToString() const { return HandleToString(NodeToStringFn, handle_); }

Expression::Expression(NodePtr root, FieldPtr result)
    : root_(std::move(root)), result_(std::move(result)) {
  gdv_expression_t h = nullptr;
  if (root_ != nullptr && result_ != nullptr)
    gdv_expression_make(static_cast<gdv_node_t>(root_->handle()), result_->name().c_str(),
                        ToC(*result_->type()), &h);
  handle_ = h;
}
Expression::~Expression() {
  if (handle_ != nullptr) gdv_expression_release(static_cast<gdv_expression_t>(handle_));
}
std::string Expression::ToString() const { return root_ ? root_->ToString() : ""; }

Condition::Condition(NodePtr root)
    : Expression(std::move(root), arrow::field("cond", arrow::boolean())) {
  gdv_condition_t h = nullptr;
  if (root_ != nullptr) gdv_condition_make(static_cast<gdv_node_t>(root_->handle()), &h);
  cond_handle_ = h;
}
Condition::~Condition() {
  if (cond_handle_ != nullptr) gdv_condition_release(static_cast<gdv_condition_t>(cond_handle_));
}

// ---- TreeExprBuilder -------------------------------------------------------------------------
NodePtr TreeExprBuilder::MakeLiteral(bool value) {
  return MakeFixedLiteral<uint8_t>(arrow::boolean(), value ? 1 : 0);
}
NodePtr TreeExprBuilder::MakeLiteral(uint8_t value) { return MakeFixedLiteral(arrow::uint8(), value); }
NodePtr TreeExprBuilder::MakeLiteral(uint16_t value) { return MakeFixedLiteral(arrow::uint16(), value); }
NodePtr TreeExprBuilder::MakeLiteral(uint32_t value) { return MakeFixedLiteral(arrow::uint32(), value); }
NodePtr TreeExprBuilder::MakeLiteral(uint64_t value) { return MakeFixedLiteral(arrow::uint64(), value); }
NodePtr TreeExprBuilder::MakeLiteral(int8_t value) { return MakeFixedLiteral(arrow::int8(), value); }
NodePtr TreeExprBuilder::MakeLiteral(int16_t value) { return MakeFixedLiteral(arrow::int16(), value); }
NodePtr TreeExprBuilder::MakeLiteral(int32_t value) { return MakeFixedLiteral(arrow::int32(), value); }
NodePtr TreeExprBuilder::MakeLiteral(int64_t value) { return MakeFixedLiteral(arrow::int64(), value); }
NodePtr TreeExprBuilder::MakeLiteral(float value) { return MakeFixedLiteral(arrow::float32(), value); }
NodePtr TreeExprBuilder::MakeLiteral(double value) { return MakeFixedLiteral(arrow::float64(), value); }
NodePtr TreeExprBuilder::MakeStringLiteral(const std::string& value) {
  return MakeBytesLiteral(arrow::utf8(), value);
}
NodePtr TreeExprBuilder::MakeBinaryLiteral(const std::string& value) {
  return MakeBytesLiteral(arrow::binary(), value);
}
NodePtr TreeExprBuilder::MakeDecimalLiteral(const uint8_t unscaled_le[16], int32_t precision,
                                            int32_t scale) {
  DataTypePtr t = arrow::decimal128(precision, scale);
  gdv_node_t h = nullptr;
  if (gdv_node_literal(ToC(*t), unscaled_le, 16, 0, &h) != GDV_OK) return nullptr;
  return std::make_shared<Node>(std::move(t), h);
}
NodePtr TreeExprBuilder::MakeNull(DataTypePtr data_type) {
  if (data_type == nullptr) return nullptr;
  gdv_node_t h = nullptr;
  if (gdv_node_literal(ToC(*data_type), nullptr, 0, 1, &h) != GDV_OK) return nullptr;
  return std::make_shared<Node>(std::move(data_type), h);
}

NodePtr TreeExprBuilder::MakeField(FieldPtr field) {
  if (field == nullptr) return nullptr;
  gdv_node_t h = nullptr;
  if (gdv_node_field(field->name().c_str(), ToC(*field->type()), &h) != GDV_OK) return nullptr;
  return std::make_shared<Node>(field->type(), h);
}

NodePtr TreeExprBuilder::MakeFunction(const std::string& name, const NodeVector& params,
                                      DataTypePtr return_type) {
  if (return_type == nullptr) return nullptr;
  bool ok;
  std::vector<gdv_node_t> hs = Handles(params, &ok);
  if (!ok) return nullptr;
  gdv_node_t h = nullptr;
  if (gdv_node_function(name.c_str(), hs.data(), static_cast<int32_t>(hs.size()), ToC(*return_type),
                        &h) != GDV_OK)
    return nullptr;
  return std::make_shared<Node>(std::move(return_type), h);
}

NodePtr TreeExprBuilder::MakeIf(NodePtr condition, NodePtr then_node, NodePtr else_node,
                                DataTypePtr result_type) {
  if (!condition || !then_node || !else_node || !result_type) return nullptr;
  gdv_node_t h = nullptr;
  if (gdv_node_if(static_cast<gdv_node_t>(condition->handle()),
                  static_cast<gdv_node_t>(then_node->handle()),
                  static_cast<gdv_node_t>(else_node->handle()), ToC(*result_type), &h) != GDV_OK)
    return nullptr;
  return std::make_shared<Node>(std::move(result_type), h);
}

NodePtr TreeExprBuilder::MakeAnd(const NodeVector& children) {
  bool ok;
  std::vector<gdv_node_t> hs = Handles(children, &ok);
  if (!ok) return nullptr;
  gdv_node_t h = nullptr;
  if (gdv_node_and(hs.data(), static_cast<int32_t>(hs.size()), &h) != GDV_OK) return nullptr;
  return std::make_shared<Node>(arrow::boolean(), h);
}

NodePtr TreeExprBuilder::MakeOr(const NodeVector& children) {
  bool ok;
  std::vector<gdv_node_t> hs = Handles(children, &ok);
  if (!ok) return nullptr;
  gdv_node_t h = nullptr;
  if (gdv_node_or(hs.data(), static_cast<int32_t>(hs.size()), &h) != GDV_OK) return nullptr;
  return std::make_shared<Node>(arrow::boolean(), h);
}

ExpressionPtr TreeExprBuilder::MakeExpression(NodePtr root_node, FieldPtr result_field) {
  if (result_field == nullptr) return nullptr;
  return std::make_shared<Expression>(std::move(root_node), std::move(result_field));
}

ExpressionPtr TreeExprBuilder::MakeExpression(const std::string& function,
                                              const FieldVector& in_fields, FieldPtr out_field) {
  if (out_field == nullptr) return nullptr;
  NodeVector kids;
  for (const auto& f : in_fields) kids.push_back(MakeField(f));
  return MakeExpression(MakeFunction(function, kids, out_field->type()), out_field);
}

ConditionPtr TreeExprBuilder::MakeCondition(NodePtr root_node) {
  if (root_node == nullptr) return nullptr;
  return std::make_shared<Condition>(std::move(root_node));
}

ConditionPtr TreeExprBuilder::MakeCondition(const std::string& function,
                                            const FieldVector& in_fields) {
  NodeVector kids;
  for (const auto& f : in_fields) kids.push_back(MakeField(f));
  return MakeCondition(MakeFunction(function, kids, arrow::boolean()));
}

NodePtr TreeExprBuilder::MakeInExpressionInt32(NodePtr node, const std::unordered_set<int32_t>& c) {
  return MakeIn(std::move(node), arrow::int32(), c);
}
NodePtr TreeExprBuilder::MakeInExpressionInt64(NodePtr node, const std::unordered_set<int64_t>& c) {
  return MakeIn(std::move(node), arrow::int64(), c);
}
NodePtr TreeExprBuilder::MakeInExpressionFloat(NodePtr node, const std::unordered_set<float>& c) {
  return MakeIn(std::move(node), arrow::float32(), c);
}
NodePtr TreeExprBuilder::MakeInExpressionDouble(NodePtr node, const std::unordered_set<double>& c) {
  return MakeIn(std::move(node), arrow::float64(), c);
}
NodePtr TreeExprBuilder::MakeInExpressionString(NodePtr node, const std::unordered_set<std::string>& c) {
  return MakeInBytes(std::move(node), arrow::utf8(), c);
}
NodePtr TreeExprBuilder::MakeInExpressionBinary(NodePtr node, const std::unordered_set<std::string>& c) {
  return MakeInBytes(std::move(node), arrow::binary(), c);
}
NodePtr TreeExprBuilder::MakeInExpressionDate32(NodePtr node, const std::unordered_set<int32_t>& c) {
  return MakeIn(std::move(node), arrow::date32(), c);
}
NodePtr TreeExprBuilder::MakeInExpressionDate64(NodePtr node, const std::unordered_set<int64_t>& c) {
  return MakeIn(std::move(node), arrow::date64(), c);
}
NodePtr TreeExprBuilder::MakeInExpressionTime32(NodePtr node, const std::unordered_set<int32_t>& c) {
  return MakeIn(std::move(node), arrow::time32(arrow::TimeUnit::MILLI), c);
}
NodePtr TreeExprBuilder::MakeInExpressionTime64(NodePtr node, const std::unordered_set<int64_t>& c) {
  return MakeIn(std::move(node), arrow::time64(arrow::TimeUnit::MICRO), c);
}
NodePtr TreeExprBuilder::MakeInExpressionTimeStamp(NodePtr node, const std::unordered_set<int64_t>& c) {
  return MakeIn(std::move(node), arrow::timestamp(arrow::TimeUnit::MILLI), c);
}

// ---- SelectionVector -------------------------------------------------------------------------
static int ModeWidth(SelectionVector::Mode m) {
  return m == SelectionVector::MODE_UINT16 ? 2 : (m == SelectionVector::MODE_UINT32 ? 4 : 8);
}

uint64_t SelectionVector::GetIndex(int64_t index) const {
  uint64_t host_copy = 0;
  const uint8_t* p = buffer_->data();
  if (!buffer_->is_cpu()) {  // a vector in HBM: one element over PCIe (debugging aid, not a hot path)
    const int w = mode_ == MODE_UINT16 ? 2 : (mode_ == MODE_UINT32 ? 4 : 8);
    if (arrow::MemoryManager::CopyBufferSliceToCPU(buffer_, index * w, w, reinterpret_cast<uint8_t*>(&host_copy)).ok())
      return host_copy;
    return 0;
  }
  switch (mode_) {
    case MODE_UINT16: return reinterpret_cast<const uint16_t*>(p)[index];
    case MODE_UINT32: return reinterpret_cast<const uint32_t*>(p)[index];
    default: return reinterpret_cast<const uint64_t*>(p)[index];
  }
}

void SelectionVector::SetIndex(int64_t index, uint64_t value) {
  uint8_t* p = buffer_->mutable_data();
  switch (mode_) {
    case MODE_UINT16: reinterpret_cast<uint16_t*>(p)[index] = static_cast<uint16_t>(value); break;
    case MODE_UINT32: reinterpret_cast<uint32_t*>(p)[index] = static_cast<uint32_t>(value); break;
    default: reinterpret_cast<uint64_t*>(p)[index] = value; break;
  }
}

uint64_t SelectionVector::GetMaxSupportedValue() const {
  return mode_ == MODE_UINT16 ? UINT16_MAX : (mode_ == MODE_UINT32 ? UINT32_MAX : UINT64_MAX);
}

ArrayPtr SelectionVector::ToArray() const {
  DataTypePtr t = mode_ == MODE_UINT16 ? arrow::uint16()
                                       : (mode_ == MODE_UINT32 ? arrow::uint32() : arrow::uint64());
  auto data = arrow::ArrayData::Make(t, num_slots_, {nullptr, buffer_}, 0);
  return arrow::MakeArray(data);
}

Status SelectionVector::Make(Mode mode, int64_t max_slots, arrow::MemoryPool* pool,
                             std::shared_ptr<SelectionVector>* out) {
  ARROW_ASSIGN_OR_RAISE(std::unique_ptr<arrow::Buffer> buf,
                        arrow::AllocateBuffer(std::max<int64_t>(max_slots, 1) * ModeWidth(mode), pool));
  *out = std::make_shared<SelectionVector>(mode, max_slots, std::shared_ptr<arrow::Buffer>(std::move(buf)));
  return Status::OK();
}
Status SelectionVector::MakeInt16(int64_t n, arrow::MemoryPool* p, std::shared_ptr<SelectionVector>* o) {
  return Make(MODE_UINT16, n, p, o);
}
Status SelectionVector::MakeInt32(int64_t n, arrow::MemoryPool* p, std::shared_ptr<SelectionVector>* o) {
  return Make(MODE_UINT32, n, p, o);
}
Status SelectionVector::MakeInt64(int64_t n, arrow::MemoryPool* p, std::shared_ptr<SelectionVector>* o) {
  return Make(MODE_UINT64, n, p, o);
}
static Status MakeFromBuffer(SelectionVector::Mode mode, int64_t max_slots,
                             std::shared_ptr<arrow::Buffer> buffer,
                             std::shared_ptr<SelectionVector>* out) {
  if (buffer == nullptr || buffer->size() < max_slots * ModeWidth(mode))
    return Status::Invalid("buffer too small for a selection vector of ", max_slots, " slots");
  *out = std::make_shared<SelectionVector>(mode, max_slots, std::move(buffer));
  return Status::OK();
}
Status SelectionVector::MakeInt16(int64_t n, std::shared_ptr<arrow::Buffer> b, std::shared_ptr<SelectionVector>* o) {
  return MakeFromBuffer(MODE_UINT16, n, std::move(b), o);
}
Status SelectionVector::MakeInt32(int64_t n, std::shared_ptr<arrow::Buffer> b, std::shared_ptr<SelectionVector>* o) {
  return MakeFromBuffer(MODE_UINT32, n, std::move(b), o);
}
Status SelectionVector::MakeInt64(int64_t n, std::shared_ptr<arrow::Buffer> b, std::shared_ptr<SelectionVector>* o) {
  return MakeFromBuffer(MODE_UINT64, n, std::move(b), o);
}

// ---- Projector -------------------------------------------------------------------------------
Projector::~Projector() {
  if (handle_ != nullptr) gdv_projector_release(static_cast<gdv_projector_t>(handle_));
  if (schema_handle_ != nullptr) gdv_schema_release(static_cast<gdv_schema_t>(schema_handle_));
}

Status Projector::Make(SchemaPtr schema, const ExpressionVector& exprs,
                       std::shared_ptr<Projector>* projector) {
  return Make(std::move(schema), exprs, SelectionVector::MODE_NONE,
              ConfigurationBuilder::DefaultConfiguration(), projector);
}
Status Projector::Make(SchemaPtr schema, const ExpressionVector& exprs,
                       std::shared_ptr<Configuration> configuration,
                       std::shared_ptr<Projector>* projector) {
  return Make(std::move(schema), exprs, SelectionVector::MODE_NONE, std::move(configuration),
              projector);
}
Status Projector::Make(SchemaPtr schema, const ExpressionVector& exprs,
                       SelectionVector::Mode selection_vector_mode,
                       std::shared_ptr<Configuration> configuration,
                       std::shared_ptr<Projector>* projector) {
  if (schema == nullptr) return Status::Invalid("Schema cannot be null");
  if (exprs.empty()) return Status::Invalid("Expressions cannot be empty");
  if (configuration == nullptr) return Status::Invalid("Configuration cannot be null");
  std::vector<gdv_expression_t> hs;
  FieldVector outs;
  for (const auto& e : exprs) {
    if (e == nullptr || e->handle() == nullptr) return Status::Invalid("Expression cannot be null");
    hs.push_back(static_cast<gdv_expression_t>(e->handle()));
    outs.push_back(e->result());
  }
  std::shared_ptr<Projector> p(new Projector());
  p->schema_ = schema;
  p->output_fields_ = std::move(outs);
  p->exprs_ = exprs;
  p->mode_ = selection_vector_mode;
  p->schema_handle_ = MakeSchemaHandle(*schema);
  gdv_config_t cfg = ConfigToC(configuration);
  gdv_projector_t h = nullptr;
  ARROW_RETURN_NOT_OK(ToStatus(gdv_projector_make(static_cast<gdv_schema_t>(p->schema_handle_), hs.data(),
                                                  static_cast<int32_t>(hs.size()),
                                                  SelModeToC(selection_vector_mode), &cfg, &h)));
  p->handle_ = h;
  *projector = std::move(p);
  return Status::OK();
}

Status Projector::Evaluate(const arrow::RecordBatch& batch, arrow::MemoryPool* pool,
                           arrow::ArrayVector* output) const {
  return Evaluate(batch, nullptr, pool, output);
}

Status Projector::Evaluate(const arrow::RecordBatch& batch, const SelectionVector* selection_vector,
                           arrow::MemoryPool* pool, arrow::ArrayVector* output) const {
  if (output == nullptr) return Status::Invalid("Output must be non-null.");
  if (pool == nullptr) return Status::Invalid("Memory pool must be non-null.");
  if (!batch.schema()->Equals(*schema_))
    return Status::Invalid("RecordBatch schema must expected schema: ", schema_->ToString());
  if (batch.num_rows() == 0) return Status::Invalid("RecordBatch must be non-empty.");
  if (mode_ != SelectionVector::MODE_NONE && selection_vector == nullptr)
    return Status::Invalid("Selection vector must be non-null.");
  std::vector<gdv_column_t> cols;
  int space = GDV_MEM_HOST;
  std::shared_ptr<arrow::MemoryManager> mm;
  std::vector<std::unique_ptr<ViewBuffers>> views;
  ARROW_RETURN_NOT_OK(ToColumns(batch, &cols, &space, &mm, &views));
  const bool on_device = space == GDV_MEM_DEVICE;
  gdv_batch_t b{batch.num_rows(), batch.num_columns(), space, cols.data()};
  const int64_t n = selection_vector != nullptr && mode_ != SelectionVector::MODE_NONE
                        ? selection_vector->GetNumSlots()
                        : batch.num_rows();
  gdv_selection_t sel;
  std::memset(&sel, 0, sizeof(sel));
  const gdv_selection_t* psel = nullptr;
  if (mode_ != SelectionVector::MODE_NONE) {
    if (selection_vector->GetBuffer().is_cpu() == on_device)
      return Status::Invalid("the selection vector and the RecordBatch must live in the same memory space");
    sel.indices = reinterpret_cast<void*>(selection_vector->GetBuffer().address());
    sel.max_slots = selection_vector->GetMaxSlots();
    sel.num_slots = selection_vector->GetNumSlots();
    sel.mode = SelModeToC(selection_vector->GetMode());
    sel.mem_space = space;
    psel = &sel;
  }
  // Outputs: from the caller's pool for host batches (as the reference does); for device batches from
  // the MemoryManager of the batch's buffers, so that results stay next to their inputs in HBM.
  auto alloc = [&](int64_t bytes, bool zero) -> arrow::Result<std::shared_ptr<arrow::Buffer>> {
    if (on_device) {
      ARROW_ASSIGN_OR_RAISE(std::unique_ptr<arrow::Buffer> buf, mm->AllocateBuffer(bytes));
      return std::shared_ptr<arrow::Buffer>(std::move(buf));
    }
    ARROW_ASSIGN_OR_RAISE(std::unique_ptr<arrow::Buffer> buf, arrow::AllocateBuffer(bytes, pool));
    if (zero) std::memset(buf->mutable_data(), 0, static_cast<size_t>(bytes));
    return std::shared_ptr<arrow::Buffer>(std::move(buf));
  };
  std::vector<gdv_out_column_t> outs(output_fields_.size());
  std::vector<ArrayDataPtr> datas;
  for (size_t i = 0; i < outs.size(); ++i) {
    std::memset(&outs[i], 0, sizeof(outs[i]));
    const DataTypePtr& t = output_fields_[i]->type();
    const int64_t bitmap_bytes = arrow::bit_util::RoundUpToMultipleOf8(arrow::bit_util::BytesForBits(n)) + 8;
    ARROW_ASSIGN_OR_RAISE(std::shared_ptr<arrow::Buffer> validity, alloc(bitmap_bytes, true));
    outs[i].validity = reinterpret_cast<void*>(validity->address());
    const bool large = t->id() == arrow::Type::LARGE_STRING || t->id() == arrow::Type::LARGE_BINARY;
    if (t->id() == arrow::Type::STRING || t->id() == arrow::Type::BINARY || large) {
      // utf8/binary: the sizing pass says how many bytes the data buffer needs, then the
      // offsets (n + 1 int32, or int64 for large_string / large_binary) and the bytes are allocated
      int64_t need = 0;
      ARROW_RETURN_NOT_OK(ToStatus(gdv_projector_output_var_size(
          static_cast<gdv_projector_t>(handle_), &b, psel, static_cast<int32_t>(i), nullptr, &need)));
      ARROW_ASSIGN_OR_RAISE(std::shared_ptr<arrow::Buffer> offsets, alloc((n + 1) * (large ? 8 : 4) + 8, false));
      ARROW_ASSIGN_OR_RAISE(std::shared_ptr<arrow::Buffer> bytes, alloc(need + 8, false));
      outs[i].values = reinterpret_cast<void*>(offsets->address());
      outs[i].var_data = reinterpret_cast<void*>(bytes->address());
      outs[i].var_capacity = need;
      datas.push_back(arrow::ArrayData::Make(t, n, {validity, offsets, bytes}));
      continue;
    }
    const int64_t value_bytes = t->id() == arrow::Type::BOOL ? bitmap_bytes : n * (t->bit_width() / 8) + 8;
    ARROW_ASSIGN_OR_RAISE(std::shared_ptr<arrow::Buffer> values, alloc(value_bytes, t->id() == arrow::Type::BOOL));
    outs[i].values = reinterpret_cast<void*>(values->address());
    datas.push_back(arrow::ArrayData::Make(t, n, {validity, values}));
  }
  ARROW_RETURN_NOT_OK(ToStatus(gdv_projector_evaluate(static_cast<gdv_projector_t>(handle_), &b, psel,
                                                      outs.data(), static_cast<int32_t>(outs.size()),
                                                      nullptr, 0)));
  for (auto& d : datas) output->push_back(arrow::MakeArray(d));
  return Status::OK();
}

std::string Projector::DumpIR() { return HandleToString(ProjDumpFn, handle_); }

// ---- Filter -----------------------------------------------------------------------------------
Filter::~Filter() {
  if (handle_ != nullptr) gdv_filter_release(static_cast<gdv_filter_t>(handle_));
  if (schema_handle_ != nullptr) gdv_schema_release(static_cast<gdv_schema_t>(schema_handle_));
}

Status Filter::Make(SchemaPtr schema, ConditionPtr condition, std::shared_ptr<Filter>* filter) {
  return Make(std::move(schema), std::move(condition), ConfigurationBuilder::DefaultConfiguration(), filter);
}

Status Filter::Make(SchemaPtr schema, ConditionPtr condition,
                    std::shared_ptr<Configuration> configuration, std::shared_ptr<Filter>* filter) {
  if (schema == nullptr) return Status::Invalid("Schema cannot be null");
  if (condition == nullptr || condition->condition_handle() == nullptr)
    return Status::Invalid("Condition cannot be null");
  if (configuration == nullptr) return Status::Invalid("Configuration cannot be null");
  std::shared_ptr<Filter> f(new Filter());
  f->schema_ = schema;
  f->condition_ = condition;
  f->schema_handle_ = MakeSchemaHandle(*schema);
  gdv_config_t cfg = ConfigToC(configuration);
  gdv_filter_t h = nullptr;
  ARROW_RETURN_NOT_OK(ToStatus(gdv_filter_make(static_cast<gdv_schema_t>(f->schema_handle_),
                                               static_cast<gdv_condition_t>(condition->condition_handle()),
                                               &cfg, &h)));
  f->handle_ = h;
  *filter = std::move(f);
  return Status::OK();
}

Status Filter::Evaluate(const arrow::RecordBatch& batch, std::shared_ptr<SelectionVector> out_selection) {
  if (out_selection == nullptr) return Status::Invalid("out_selection must be non-null.");
  if (!batch.schema()->Equals(*schema_))
    return Status::Invalid("RecordBatch schema must expected schema: ", schema_->ToString());
  if (batch.num_rows() == 0) return Status::Invalid("RecordBatch must be non-empty.");
  if (out_selection->GetMaxSlots() < batch.num_rows())
    return Status::Invalid("Output selection vector capacity too small");
  std::vector<gdv_column_t> cols;
  int space = GDV_MEM_HOST;
  std::vector<std::unique_ptr<ViewBuffers>> views;
  ARROW_RETURN_NOT_OK(ToColumns(batch, &cols, &space, nullptr, &views));
  if (out_selection->GetBuffer().is_cpu() == (space == GDV_MEM_DEVICE))
    return Status::Invalid("the selection vector and the RecordBatch must live in the same memory space "
                           "(SelectionVector::MakeInt32(max_slots, <device buffer>, &out) for device batches)");
  gdv_batch_t b{batch.num_rows(), batch.num_columns(), space, cols.data()};
  gdv_selection_t sel;
  std::memset(&sel, 0, sizeof(sel));
  sel.indices = reinterpret_cast<void*>(out_selection->GetBuffer().address());
  sel.max_slots = out_selection->GetMaxSlots();
  sel.mode = SelModeToC(out_selection->GetMode());
  sel.mem_space = space;
  ARROW_RETURN_NOT_OK(
      ToStatus(gdv_filter_evaluate(static_cast<gdv_filter_t>(handle_), &b, &sel, nullptr, 0, nullptr)));
  out_selection->SetNumSlots(sel.num_slots);
  return Status::OK();
}

std::string Filter::DumpIR() { return HandleToString(FiltDumpFn, handle_); }

// ---- registry ---------------------------------------------------------------------------------
std::string FunctionSignature::ToString() const {
  std::string s = ret_type_->ToString() + " " + base_name_ + "(";
  for (size_t i = 0; i < param_types_.size(); ++i) {
    if (i) s += ", ";
    s += param_types_[i]->ToString();
  }
  return s + ")";
}

std::vector<std::shared_ptr<FunctionSignature>> GetRegisteredFunctionSignatures() {
  std::vector<std::shared_ptr<FunctionSignature>> out;
  const int32_t n = gdv_registry_size();
  for (int32_t i = 0; i < n; ++i) {
    const char* name = nullptr;
    gdv_type_t ret;
    gdv_type_t params[16];
    int32_t np = 0;
    if (gdv_registry_get(i, &name, &ret, params, 16, &np) != GDV_OK) continue;
    DataTypeVector pts;
    for (int32_t k = 0; k < np && k < 16; ++k) pts.push_back(FromC(params[k]));
    out.push_back(std::make_shared<FunctionSignature>(name, std::move(pts), FromC(ret)));
  }
  return out;
}

// ---- user-defined functions ----------------------------------------------------------------------
FunctionRegistry::FunctionRegistry() {
  gdv_function_registry_t h = nullptr;
  gdv_function_registry_create(&h);
  handle_ = h;
}

FunctionRegistry::~FunctionRegistry() { gdv_function_registry_release(static_cast<gdv_function_registry_t>(handle_)); }

Status FunctionRegistry::Register(const FunctionSignature& signature, const std::string& body, NullMode null_mode,
                                  bool can_raise, const std::string& prelude) {
  std::vector<gdv_type_t> params;
  for (const auto& t : signature.param_types()) {
    if (t == nullptr) return Status::Invalid("parameter type cannot be null");
    params.push_back(ToC(*t));
  }
  if (signature.ret_type() == nullptr) return Status::Invalid("return type cannot be null");
  gdv_function_def_t def;
  std::memset(&def, 0, sizeof(def));
  def.name = signature.base_name().c_str();
  def.params = params.data();
  def.n_params = static_cast<int32_t>(params.size());
  def.ret = ToC(*signature.ret_type());
  def.null_mode = static_cast<int32_t>(null_mode);
  def.can_raise = can_raise ? 1 : 0;
  def.body = body.c_str();
  def.prelude = prelude.c_str();
  return ToStatus(gdv_function_registry_add(static_cast<gdv_function_registry_t>(handle_), &def));
}

std::vector<FunctionSignature> FunctionRegistry::GetSignatures() const {
  std::vector<FunctionSignature> out;
  auto reg = static_cast<gdv_function_registry_t>(handle_);
  const int32_t n = gdv_function_registry_signatures(reg);
  for (int32_t i = 0; i < n; ++i) {
    const char* name = nullptr;
    gdv_type_t ret;
    gdv_type_t params[16];
    int32_t np = 0;
    if (gdv_function_registry_get(reg, i, &name, &ret, params, 16, &np) != GDV_OK) continue;
    DataTypeVector pts;
    for (int32_t k = 0; k < np && k < 16; ++k) pts.push_back(FromC(params[k]));
    out.emplace_back(name, std::move(pts), FromC(ret));
  }
  return out;
}

// ---- HBM as an arrow::MemoryManager ------------------------------------------------------------
namespace {

class HbmDevice : public arrow::Device {
 public:
  explicit HbmDevice(int ordinal) : arrow::Device(false), ordinal_(ordinal) {}
  const char* type_name() const override { return "gandiva_b200::HbmDevice"; }
  std::string ToString() const override { return "gandiva_b200 CUDA device " + std::to_string(ordinal_); }
  bool Equals(const arrow::Device& other) const override {
    return other.device_type() == device_type() && other.device_id() == device_id();
  }
  int64_t device_id() const override { return ordinal_; }
  arrow::DeviceAllocationType device_type() const override { return arrow::DeviceAllocationType::kCUDA; }
  std::shared_ptr<arrow::MemoryManager> default_memory_manager() override;

 private:
  int ordinal_;
};

// A block of the engine's pooled allocator; goes back to the pool with the buffer.
class HbmBuffer : public arrow::MutableBuffer {
 public:
  HbmBuffer(int ordinal, void* p, int64_t size, std::shared_ptr<arrow::MemoryManager> mm)
      : arrow::MutableBuffer(static_cast<uint8_t*>(p), size, std::move(mm)), ordinal_(ordinal), p_(p) {}
  ~HbmBuffer() override { gdv_device_free(ordinal_, p_); }

 private:
  int ordinal_;
  void* p_;
};

class HbmMemoryManager : public arrow::MemoryManager {
 public:
  HbmMemoryManager(const std::shared_ptr<arrow::Device>& dev, int ordinal) : arrow::MemoryManager(dev), ordinal_(ordinal) {}
  arrow::Result<std::shared_ptr<arrow::io::RandomAccessFile>> GetBufferReader(std::shared_ptr<arrow::Buffer>) override {
    return Status::NotImplemented("no file interface over HBM buffers: copy them to the host first");
  }
  arrow::Result<std::shared_ptr<arrow::io::OutputStream>> GetBufferWriter(std::shared_ptr<arrow::Buffer>) override {
    return Status::NotImplemented("no file interface over HBM buffers");
  }
  arrow::Result<std::unique_ptr<arrow::Buffer>> AllocateBuffer(int64_t size) override {
    void* p = nullptr;
    ARROW_RETURN_NOT_OK(ToStatus(gdv_device_alloc(ordinal_, static_cast<size_t>(size > 0 ? size : 1), &p)));
    return std::unique_ptr<arrow::Buffer>(new HbmBuffer(ordinal_, p, size, shared_from_this()));
  }

 protected:
  arrow::Result<std::shared_ptr<arrow::Buffer>> CopyBufferFrom(const std::shared_ptr<arrow::Buffer>& buf,
                                                              const std::shared_ptr<arrow::MemoryManager>& from) override {
    ARROW_ASSIGN_OR_RAISE(std::unique_ptr<arrow::Buffer> out, CopyNonOwnedFrom(*buf, from));
    return std::shared_ptr<arrow::Buffer>(std::move(out));
  }
  arrow::Result<std::unique_ptr<arrow::Buffer>> CopyNonOwnedFrom(const arrow::Buffer& buf,
                                                               const std::shared_ptr<arrow::MemoryManager>& from) override {
    if (!from->is_cpu()) return std::unique_ptr<arrow::Buffer>();  // unsupported here: let the other side try
    ARROW_ASSIGN_OR_RAISE(std::unique_ptr<arrow::Buffer> out, AllocateBuffer(buf.size()));
    ARROW_RETURN_NOT_OK(ToStatus(gdv_memcpy(ordinal_, reinterpret_cast<void*>(out->address()), buf.data(),
                                            static_cast<size_t>(buf.size()), 1)));
    return out;
  }
  arrow::Result<std::shared_ptr<arrow::Buffer>> CopyBufferTo(const std::shared_ptr<arrow::Buffer>& buf,
                                                            const std::shared_ptr<arrow::MemoryManager>& to) override {
    ARROW_ASSIGN_OR_RAISE(std::unique_ptr<arrow::Buffer> out, CopyNonOwnedTo(*buf, to));
    return std::shared_ptr<arrow::Buffer>(std::move(out));
  }
  arrow::Result<std::unique_ptr<arrow::Buffer>> CopyNonOwnedTo(const arrow::Buffer& buf,
                                                             const std::shared_ptr<arrow::MemoryManager>& to) override {
    if (!to->is_cpu()) return std::unique_ptr<arrow::Buffer>();
    ARROW_ASSIGN_OR_RAISE(std::unique_ptr<arrow::Buffer> out, to->AllocateBuffer(buf.size()));
    ARROW_RETURN_NOT_OK(ToStatus(gdv_memcpy(ordinal_, out->mutable_data(), reinterpret_cast<const void*>(buf.address()),
                                            static_cast<size_t>(buf.size()), 2)));
    return out;
  }

 private:
  int ordinal_;
};

std::shared_ptr<arrow::MemoryManager> HbmDevice::default_memory_manager() {
  return std::make_shared<HbmMemoryManager>(shared_from_this(), ordinal_);
}

}  // namespace

arrow::Result<std::shared_ptr<arrow::MemoryManager>> DeviceMemoryManager(int device) {
  if (!gdv_cuda_available()) return Status::ExecutionError("CUDA: no usable device (", gdv_last_error(), ")");
  if (device < 0 || device >= gdv_device_count()) return Status::Invalid("no CUDA device ", device);
  auto dev = std::make_shared<HbmDevice>(device);
  return dev->default_memory_manager();
}

arrow::Result<std::shared_ptr<arrow::RecordBatch>> CopyToDevice(const arrow::RecordBatch& batch, int device) {
  ARROW_ASSIGN_OR_RAISE(std::shared_ptr<arrow::MemoryManager> mm, DeviceMemoryManager(device));
  return batch.CopyTo(mm);
}
arrow::Result<std::shared_ptr<arrow::RecordBatch>> CopyToHost(const arrow::RecordBatch& batch) {
  return batch.CopyTo(arrow::default_cpu_memory_manager());
}
arrow::Result<std::shared_ptr<arrow::Array>> CopyToHost(const arrow::Array& array) {
  return array.CopyTo(arrow::default_cpu_memory_manager());
}

}  // namespace gandiva
