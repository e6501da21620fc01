// extern "C" entry points declared in include/gandiva_b200.h.
#include <cstring>
#include <string>
#include <vector>

#include "gandiva_b200.h"
#include "gdv_capi_internal.h"
#include "gdv_node.h"
#include "gdv_registry.h"
#include "gdv_runtime.h"
#include "gdv_staging.h"

using namespace gdv;
using namespace gdv::capi;

namespace {
thread_local std::string tl_error;
}

namespace gdv {
namespace capi {
gdv_status Fail(const Status& s) {
  tl_error = s.msg;
  return s.code;
}
gdv_status Fail(int code, const std::string& msg) {
  tl_error = msg;
  return code;
}
}  // namespace capi
}  // namespace gdv

namespace {

NodeH* N(gdv_node_t h) { return reinterpret_cast<NodeH*>(h); }

int64_t CopyOut(const std::string& s, char* buf, int64_t len) {
  if (buf != nullptr && len > 0) {
    const size_t n = std::min(static_cast<size_t>(len - 1), s.size());
    std::memcpy(buf, s.data(), n);
    buf[n] = '\0';
  }
  return static_cast<int64_t>(s.size());
}

Config FromC(const gdv_config_t* c) {
  Config cfg;
  if (c != nullptr) {
    cfg.optimize = c->optimize != 0;
    cfg.dump_ir = c->dump_ir != 0;
    cfg.device = c->device;
    cfg.rows_per_thread = c->rows_per_thread;
    cfg.block_threads = c->block_threads;
    cfg.loader = c->loader;
    cfg.stages = c->stages;
    cfg.string_scan = c->string_scan;
    cfg.sm_reserve = c->sm_reserve;
  }
  return cfg;
}

}  // namespace

extern "C" {

void gdv_config_default(gdv_config_t* cfg) {
  if (cfg == nullptr) return;
  std::memset(cfg, 0, sizeof(*cfg));
  cfg->optimize = 1;
}

const char* gdv_version(void) { return "gandiva_b200 0.1 (sm_90a)"; }
const char* gdv_last_error(void) { return tl_error.c_str(); }

int32_t gdv_cuda_available(void) {
  const DriverApi& d = Driver();
  if (!d.loaded) return 0;
  int n = 0;
  if (d.DeviceGetCount(&n) != CUDA_SUCCESS) return 0;
  return n > 0 ? 1 : 0;
}

int32_t gdv_device_count(void) {
  const DriverApi& d = Driver();
  if (!d.loaded) return 0;
  int n = 0;
  if (d.DeviceGetCount(&n) != CUDA_SUCCESS) return 0;
  return n;
}

// ---- TreeExprBuilder ----------------------------------------------------------------------
gdv_status gdv_node_field(const char* name, gdv_type_t type, gdv_node_t* out) {
  if (name == nullptr || out == nullptr) return Fail(GDV_INVALID, "null argument");
  *out = reinterpret_cast<gdv_node_t>(
      new NodeH{std::make_shared<FieldNode>(std::string(name), DataType(type))});
  return GDV_OK;
}

gdv_status gdv_node_literal(gdv_type_t type, const void* value, int64_t len, int32_t is_null,
                            gdv_node_t* out) {
  if (out == nullptr) return Fail(GDV_INVALID, "null argument");
  if (!is_null && value == nullptr && !(DataType(type).is_varlen() && len == 0))
    return Fail(GDV_INVALID, "literal value is null");
  *out = reinterpret_cast<gdv_node_t>(
      new NodeH{std::make_shared<LiteralNode>(DataType(type), value, len, is_null != 0)});
  return GDV_OK;
}

static bool CollectChildren(const gdv_node_t* children, int32_t n, NodeVector* out) {
  for (int32_t i = 0; i < n; ++i) {
    if (children == nullptr || children[i] == nullptr) return false;
    out->push_back(N(children[i])->p);
  }
  return true;
}

gdv_status gdv_node_function(const char* name, const gdv_node_t* children, int32_t n_children,
                             gdv_type_t return_type, gdv_node_t* out) {
  if (name == nullptr || out == nullptr) return Fail(GDV_INVALID, "null argument");
  NodeVector kids;
  if (!CollectChildren(children, n_children, &kids)) return Fail(GDV_INVALID, "null child node");
  *out = reinterpret_cast<gdv_node_t>(new NodeH{
      std::make_shared<FunctionNode>(std::string(name), std::move(kids), DataType(return_type))});
  return GDV_OK;
}

gdv_status gdv_node_if(gdv_node_t condition, gdv_node_t then_node, gdv_node_t else_node,
                       gdv_type_t return_type, gdv_node_t* out) {
  if (!condition || !then_node || !else_node || !out) return Fail(GDV_INVALID, "null argument");
  *out = reinterpret_cast<gdv_node_t>(new NodeH{std::make_shared<IfNode>(
      N(condition)->p, N(then_node)->p, N(else_node)->p, DataType(return_type))});
  return GDV_OK;
}

gdv_status gdv_node_and(const gdv_node_t* children, int32_t n_children, gdv_node_t* out) {
  if (out == nullptr) return Fail(GDV_INVALID, "null argument");
  NodeVector kids;
  if (!CollectChildren(children, n_children, &kids)) return Fail(GDV_INVALID, "null child node");
  *out = reinterpret_cast<gdv_node_t>(
      new NodeH{std::make_shared<BooleanNode>(BooleanNode::kAnd, std::move(kids))});
  return GDV_OK;
}

gdv_status gdv_node_or(const gdv_node_t* children, int32_t n_children, gdv_node_t* out) {
  if (out == nullptr) return Fail(GDV_INVALID, "null argument");
  NodeVector kids;
  if (!CollectChildren(children, n_children, &kids)) return Fail(GDV_INVALID, "null child node");
  *out = reinterpret_cast<gdv_node_t>(
      new NodeH{std::make_shared<BooleanNode>(BooleanNode::kOr, std::move(kids))});
  return GDV_OK;
}

gdv_status gdv_node_in(gdv_node_t child, gdv_type_t type, const void* values,
                       const int32_t* lengths, int32_t n_values, gdv_node_t* out) {
  if (child == nullptr || out == nullptr) return Fail(GDV_INVALID, "null argument");
  if (n_values > 0 && values == nullptr) return Fail(GDV_INVALID, "null values");
  DataType t(type);
  std::vector<int64_t> ints;
  std::vector<std::string> strs;
  if (t.is_varlen()) {
    if (n_values > 0 && lengths == nullptr) return Fail(GDV_INVALID, "null lengths");
    const char* p = static_cast<const char*>(values);
    for (int32_t i = 0; i < n_values; ++i) {
      strs.emplace_back(p, static_cast<size_t>(lengths[i]));
      p += lengths[i];
    }
  } else {
    const int w = t.width();
    if (w != 4 && w != 8) return Fail(GDV_INVALID, "IN expression supports 4- and 8-byte values");
    const uint8_t* p = static_cast<const uint8_t*>(values);
    for (int32_t i = 0; i < n_values; ++i) {
      if (w == 4) {
        int32_t v;
        std::memcpy(&v, p + 4 * i, 4);
        ints.push_back(v);
      } else {
        int64_t v;
        std::memcpy(&v, p + 8 * i, 8);
        ints.push_back(v);
      }
    }
  }
  *out = reinterpret_cast<gdv_node_t>(
      new NodeH{std::make_shared<InNode>(N(child)->p, t, std::move(ints), std::move(strs))});
  return GDV_OK;
}

gdv_status gdv_node_return_type(gdv_node_t node, gdv_type_t* out) {
  if (node == nullptr || out == nullptr) return Fail(GDV_INVALID, "null argument");
  *out = N(node)->p->return_type().c();
  return GDV_OK;
}

int64_t gdv_node_to_string(gdv_node_t node, char* buf, int64_t buf_len) {
  if (node == nullptr) return -1;
  return CopyOut(N(node)->p->ToString(), buf, buf_len);
}

void gdv_node_release(gdv_node_t node) { delete N(node); }

gdv_status gdv_expression_make(gdv_node_t root, const char* result_name, gdv_type_t result_type,
                               gdv_expression_t* out) {
  if (root == nullptr || result_name == nullptr || out == nullptr)
    return Fail(GDV_INVALID, "null argument");
  *out = reinterpret_cast<gdv_expression_t>(new ExprH{std::make_shared<Expression>(
      N(root)->p, Field{std::string(result_name), DataType(result_type)})});
  return GDV_OK;
}
int64_t gdv_expression_to_string(gdv_expression_t e, char* buf, int64_t buf_len) {
  if (e == nullptr) return -1;
  return CopyOut(reinterpret_cast<ExprH*>(e)->p->ToString(), buf, buf_len);
}
void gdv_expression_release(gdv_expression_t e) { delete reinterpret_cast<ExprH*>(e); }

gdv_status gdv_condition_make(gdv_node_t root, gdv_condition_t* out) {
  if (root == nullptr || out == nullptr) return Fail(GDV_INVALID, "null argument");
  *out = reinterpret_cast<gdv_condition_t>(new CondH{std::make_shared<Condition>(N(root)->p)});
  return GDV_OK;
}
int64_t gdv_condition_to_string(gdv_condition_t c, char* buf, int64_t buf_len) {
  if (c == nullptr) return -1;
  return CopyOut(reinterpret_cast<CondH*>(c)->p->ToString(), buf, buf_len);
}
void gdv_condition_release(gdv_condition_t c) { delete reinterpret_cast<CondH*>(c); }

gdv_status gdv_schema_make(const char* const* names, const gdv_type_t* types, int32_t n_fields,
                           gdv_schema_t* out) {
  if (out == nullptr || (n_fields > 0 && (names == nullptr || types == nullptr)))
    return Fail(GDV_INVALID, "null argument");
  std::vector<Field> fields;
  for (int32_t i = 0; i < n_fields; ++i)
    fields.push_back(Field{std::string(names[i]), DataType(types[i])});
  *out = reinterpret_cast<gdv_schema_t>(new SchemaH{std::make_shared<Schema>(std::move(fields))});
  return GDV_OK;
}
void gdv_schema_release(gdv_schema_t s) { delete reinterpret_cast<SchemaH*>(s); }

// ---- Projector ----------------------------------------------------------------------------
gdv_status gdv_projector_make(gdv_schema_t schema, const gdv_expression_t* exprs, int32_t n_exprs,
                              int32_t selection_mode, const gdv_config_t* cfg,
                              gdv_projector_t* out) {
  if (schema == nullptr || out == nullptr || (n_exprs > 0 && exprs == nullptr))
    return Fail(GDV_INVALID, "null argument");
  std::vector<ExpressionPtr> ev;
  for (int32_t i = 0; i < n_exprs; ++i) {
    if (exprs[i] == nullptr) return Fail(GDV_INVALID, "Expression cannot be null");
    ev.push_back(reinterpret_cast<ExprH*>(exprs[i])->p);
  }
  std::shared_ptr<Projector> p;
  Status s = Projector::Make(reinterpret_cast<SchemaH*>(schema)->p, std::move(ev), selection_mode,
                             FromC(cfg), &p);
  if (!s.ok()) return Fail(s);
  *out = reinterpret_cast<gdv_projector_t>(new ProjH{std::move(p)});
  return GDV_OK;
}

gdv_status gdv_projector_evaluate(gdv_projector_t p, const gdv_batch_t* batch,
                                  const gdv_selection_t* selection, gdv_out_column_t* outs,
                                  int32_t n_outs, void* stream, int32_t async) {
  if (p == nullptr) return Fail(GDV_INVALID, "null projector");
  Status s = reinterpret_cast<ProjH*>(p)->p->Evaluate(batch, selection, outs, n_outs, stream,
                                                      async != 0);
  return s.ok() ? GDV_OK : Fail(s);
}

gdv_status gdv_projector_sync(gdv_projector_t p, void* stream) {
  if (p == nullptr) return Fail(GDV_INVALID, "null projector");
  Status s = reinterpret_cast<ProjH*>(p)->p->Sync(stream);
  return s.ok() ? GDV_OK : Fail(s);
}

gdv_status gdv_projector_output_var_size(gdv_projector_t p, const gdv_batch_t* batch,
                                         const gdv_selection_t* selection, int32_t out_index,
                                         void* stream, int64_t* out) {
  if (p == nullptr) return Fail(GDV_INVALID, "null projector");
  Status s = reinterpret_cast<ProjH*>(p)->p->OutputVarSize(batch, selection, out_index, stream, out);
  return s.ok() ? GDV_OK : Fail(s);
}

int64_t gdv_projector_dump_ir(gdv_projector_t p, char* buf, int64_t buf_len) {
  if (p == nullptr) return -1;
  return CopyOut(reinterpret_cast<ProjH*>(p)->p->DumpIR(), buf, buf_len);
}

static gdv_status KernelInfo(CompiledKernel& k, const Config& cfg, char* name_buf, int64_t name_len,
                             int32_t* regs, int32_t* smem, int32_t* rpt, int32_t* bt) {
  CopyOut(k.gen.name, name_buf, name_len);
  if (rpt) *rpt = k.gen.rows_per_thread;
  if (bt) *bt = k.gen.block_threads;
  if (regs) *regs = -1;
  if (smem) *smem = -1;
  Device* dev = nullptr;
  if (Driver().loaded && Device::Get(cfg.device, &dev).ok()) {
    CompiledKernel::Loaded l;
    Status s = k.Load(dev, &l);
    if (!s.ok()) return Fail(s);
    if (regs) *regs = l.regs;
    if (smem) *smem = l.smem;
  }
  return GDV_OK;
}

gdv_status gdv_projector_kernel_info(gdv_projector_t p, char* name_buf, int64_t name_len,
                                     int32_t* regs, int32_t* smem_bytes, int32_t* rows_per_thread,
                                     int32_t* block_threads) {
  if (p == nullptr) return Fail(GDV_INVALID, "null projector");
  auto& pr = *reinterpret_cast<ProjH*>(p)->p;
  return KernelInfo(pr.kernel(), pr.config(), name_buf, name_len, regs, smem_bytes, rows_per_thread,
                    block_threads);
}

static gdv_status KernelAttr(CompiledKernel& k, const Config& cfg, const char* key, int64_t* out) {
  if (key == nullptr || out == nullptr) return Fail(GDV_INVALID, "null argument");
  const std::string kk(key);
  if (kk == "staged") { *out = k.gen.staged ? 1 : 0; return GDV_OK; }
  if (kk == "stages") { *out = k.gen.stages; return GDV_OK; }
  if (kk == "dynamic_smem") { *out = k.gen.dynamic_smem; return GDV_OK; }
  if (kk == "cta_tile_rows") { *out = k.gen.cta_tile_rows; return GDV_OK; }
  if (kk == "tile_rows") { *out = k.gen.tile_rows; return GDV_OK; }
  if (kk == "nullable") { *out = k.gen.nullable ? 1 : 0; return GDV_OK; }
  if (kk == "in_bytes_per_row") { *out = k.gen.in_bytes_per_row; return GDV_OK; }
  if (kk == "blocks_per_sm") {
    Device* dev = nullptr;
    Status s = Device::Get(cfg.device, &dev);
    if (!s.ok()) return Fail(s);
    CompiledKernel::Loaded l;
    s = k.Load(dev, &l);
    if (!s.ok()) return Fail(s);
    *out = l.blocks_per_sm;
    return GDV_OK;
  }
  return Fail(GDV_INVALID, "unknown kernel attribute " + kk);
}

gdv_status gdv_projector_kernel_attr(gdv_projector_t p, const char* key, int64_t* out) {
  if (p == nullptr) return Fail(GDV_INVALID, "null projector");
  auto& pr = *reinterpret_cast<ProjH*>(p)->p;
  return KernelAttr(pr.kernel(), pr.config(), key, out);
}

void gdv_projector_release(gdv_projector_t p) { delete reinterpret_cast<ProjH*>(p); }

// ---- Filter -------------------------------------------------------------------------------
gdv_status gdv_filter_make(gdv_schema_t schema, gdv_condition_t condition, const gdv_config_t* cfg,
                           gdv_filter_t* out) {
  if (schema == nullptr || out == nullptr) return Fail(GDV_INVALID, "null argument");
  if (condition == nullptr) return Fail(GDV_INVALID, "Condition cannot be null");
  std::shared_ptr<Filter> f;
  Status s = Filter::Make(reinterpret_cast<SchemaH*>(schema)->p,
                          reinterpret_cast<CondH*>(condition)->p, FromC(cfg), &f);
  if (!s.ok()) return Fail(s);
  *out = reinterpret_cast<gdv_filter_t>(new FiltH{std::move(f)});
  return GDV_OK;
}

gdv_status gdv_filter_evaluate(gdv_filter_t f, const gdv_batch_t* batch,
                               gdv_selection_t* out_selection, void* stream, int32_t async,
                               void* d_count) {
  if (f == nullptr) return Fail(GDV_INVALID, "null filter");
  Status s =
      reinterpret_cast<FiltH*>(f)->p->Evaluate(batch, out_selection, stream, async != 0, d_count);
  return s.ok() ? GDV_OK : Fail(s);
}

gdv_status gdv_filter_sync(gdv_filter_t f, void* stream, int64_t* num_slots) {
  if (f == nullptr) return Fail(GDV_INVALID, "null filter");
  Status s = reinterpret_cast<FiltH*>(f)->p->Sync(stream, num_slots);
  return s.ok() ? GDV_OK : Fail(s);
}

int64_t gdv_filter_dump_ir(gdv_filter_t f, char* buf, int64_t buf_len) {
  if (f == nullptr) return -1;
  return CopyOut(reinterpret_cast<FiltH*>(f)->p->DumpIR(), buf, buf_len);
}

gdv_status gdv_filter_kernel_info(gdv_filter_t f, char* name_buf, int64_t name_len, int32_t* regs,
                                  int32_t* smem_bytes, int32_t* rows_per_thread,
                                  int32_t* block_threads) {
  if (f == nullptr) return Fail(GDV_INVALID, "null filter");
  auto& fl = *reinterpret_cast<FiltH*>(f)->p;
  CompiledKernel* k = fl.last_used();
  if (k == nullptr) {
    Status s = fl.KernelFor(GDV_SEL_UINT32, true, false, &k);
    if (!s.ok()) return Fail(s);
  }
  return KernelInfo(*k, fl.config(), name_buf, name_len, regs, smem_bytes, rows_per_thread,
                    block_threads);
}

gdv_status gdv_filter_kernel_attr(gdv_filter_t f, const char* key, int64_t* out) {
  if (f == nullptr) return Fail(GDV_INVALID, "null filter");
  auto& fl = *reinterpret_cast<FiltH*>(f)->p;
  CompiledKernel* k = fl.last_used();
  if (k == nullptr) {
    Status s = fl.KernelFor(GDV_SEL_UINT32, true, false, &k);
    if (!s.ok()) return Fail(s);
  }
  return KernelAttr(*k, fl.config(), key, out);
}

void gdv_filter_release(gdv_filter_t f) { delete reinterpret_cast<FiltH*>(f); }

// ---- registry -----------------------------------------------------------------------------
int32_t gdv_registry_size(void) { return static_cast<int32_t>(Registry::Get().all().size()); }

gdv_status gdv_registry_get(int32_t i, const char** name, gdv_type_t* ret, gdv_type_t* params,
                            int32_t max_params, int32_t* n_params) {
  const auto& all = Registry::Get().all();
  if (i < 0 || i >= static_cast<int32_t>(all.size())) return Fail(GDV_INVALID, "index out of range");
  const FunctionDef& d = all[i];
  if (name) *name = d.name.c_str();
  if (ret) *ret = d.ret.c();
  if (n_params) *n_params = static_cast<int32_t>(d.params.size());
  for (int32_t k = 0; params != nullptr && k < max_params && k < static_cast<int32_t>(d.params.size()); ++k)
    params[k] = d.params[k].c();
  return GDV_OK;
}

// ---- harness helpers ----------------------------------------------------------------------
gdv_status gdv_device_alloc(int32_t device, size_t bytes, void** out) {
  if (out == nullptr) return Fail(GDV_INVALID, "null argument");
  *out = nullptr;
  Device* dev = nullptr;
  Status s = Device::Get(device, &dev);
  if (!s.ok()) return Fail(s);
  CUdeviceptr p = 0;
  s = dev->Alloc(bytes > 0 ? bytes : 1, &p);
  if (!s.ok()) return Fail(s);
  *out = reinterpret_cast<void*>(p);
  return GDV_OK;
}

gdv_status gdv_device_free(int32_t device, void* p) {
  if (p == nullptr) return GDV_OK;
  Device* dev = nullptr;
  Status s = Device::Get(device, &dev);
  if (!s.ok()) return Fail(s);
  dev->Free(reinterpret_cast<CUdeviceptr>(p));
  return GDV_OK;
}

gdv_status gdv_device_trim(int32_t device, size_t keep_bytes, size_t* released) {
  Device* dev = nullptr;
  Status s = Device::Get(device, &dev);
  if (!s.ok()) return Fail(s);
  const size_t r = dev->Trim(keep_bytes);
  if (released != nullptr) *released = r;
  return GDV_OK;
}

int64_t gdv_staged_bytes(void) { return static_cast<int64_t>(StagedBytes()); }

gdv_status gdv_host_alloc(size_t bytes, void** out) {
  if (out == nullptr) return Fail(GDV_INVALID, "null argument");
  Device* dev = nullptr;
  Status s = Device::Get(0, &dev);
  if (!s.ok()) return Fail(s);
  s = CuCheck(Driver().MemHostAlloc(out, bytes, CU_MEMHOSTALLOC_PORTABLE), "cuMemHostAlloc");
  return s.ok() ? GDV_OK : Fail(s);
}

gdv_status gdv_host_free(void* p) {
  if (p == nullptr) return GDV_OK;
  const DriverApi& d = Driver();
  if (!d.loaded) return Fail(GDV_CUDA_ERROR, d.load_error);
  Status s = CuCheck(d.MemFreeHost(p), "cuMemFreeHost");
  return s.ok() ? GDV_OK : Fail(s);
}

gdv_status gdv_generate_lineitem(int32_t device, int32_t column_kind, uint64_t seed,
                                 int64_t first_row, int64_t num_rows, void* d_values,
                                 void* d_validity, int32_t null_permille, void* stream) {
  Device* dev = nullptr;
  Status s = Device::Get(device, &dev);
  if (!s.ok()) return Fail(s);
  CUfunction fn = nullptr;
  s = dev->StaticFunction("gdv_gen_lineitem", &fn);
  if (!s.ok()) return Fail(s);
  if (num_rows <= 0) return GDV_OK;
  CUstream st = stream != nullptr ? static_cast<CUstream>(stream) : dev->stream();
  void* params[] = {&column_kind, &seed, &first_row, &num_rows, &d_values, &d_validity,
                    &null_permille};
  const int64_t warps = (num_rows + 31) / 32;
  const int64_t blocks = (warps + 7) / 8;
  const unsigned grid = static_cast<unsigned>(std::min<int64_t>(blocks, int64_t(dev->sm_count()) * 32));
  g_launch_count.fetch_add(1);
  s = CuCheck(Driver().LaunchKernel(fn, grid, 1, 1, 256, 1, 1, 0, st, params, nullptr),
              "cuLaunchKernel(gdv_gen_lineitem)");
  return s.ok() ? GDV_OK : Fail(s);
}

gdv_status gdv_enable_peer_access(int32_t device, int32_t peer_device) {
  if (device == peer_device) return GDV_OK;
  const DriverApi& d = Driver();
  if (!d.loaded) return Fail(GDV_CUDA_ERROR, d.load_error);
  Device* dev = nullptr;
  Status s = Device::Get(device, &dev);
  if (!s.ok()) return Fail(s);
  CUdevice cu_dev = 0, cu_peer = 0;
  s = CuCheck(d.DeviceGet(&cu_dev, device), "cuDeviceGet");
  if (s.ok()) s = CuCheck(d.DeviceGet(&cu_peer, peer_device), "cuDeviceGet(peer)");
  if (!s.ok()) return Fail(s);
  int can = 0;
  s = CuCheck(d.DeviceCanAccessPeer(&can, cu_dev, cu_peer), "cuDeviceCanAccessPeer");
  if (!s.ok()) return Fail(s);
  if (!can)
    return Fail(GDV_CUDA_ERROR, "device " + std::to_string(device) + " cannot access device " +
                                    std::to_string(peer_device) + " (no NVLink / PCIe P2P path)");
  CUcontext peer_ctx = nullptr;
  s = CuCheck(d.DevicePrimaryCtxRetain(&peer_ctx, cu_peer), "cuDevicePrimaryCtxRetain(peer)");
  if (!s.ok()) return Fail(s);
  s = dev->MakeCurrent();
  if (!s.ok()) return Fail(s);
  const CUresult r = d.CtxEnablePeerAccess(peer_ctx, 0);
  if (r != CUDA_SUCCESS && r != CUDA_ERROR_PEER_ACCESS_ALREADY_ENABLED)
    return Fail(CuCheck(r, "cuCtxEnablePeerAccess"));
  return GDV_OK;
}

// CUDA IPC: the root exports the allocation behind its SelectionVector / board, every other rank
// opens it with ITS OWN device context current and CU_IPC_MEM_LAZY_ENABLE_PEER_ACCESS, which maps
// the memory into that device's address space and enables NVLink peer access to the root GPU.
gdv_status gdv_ipc_export(int32_t device, const void* d_ptr, uint8_t* handle64, int64_t* offset) {
  static_assert(sizeof(CUipcMemHandle) == 64, "CUipcMemHandle is 64 bytes");
  if (d_ptr == nullptr || handle64 == nullptr || offset == nullptr)
    return Fail(GDV_INVALID, "gdv_ipc_export: null argument");
  Device* dev = nullptr;
  Status s = Device::Get(device, &dev);
  if (!s.ok()) return Fail(s);
  const DriverApi& d = Driver();
  CUdeviceptr base = 0;
  size_t size = 0;
  s = CuCheck(d.MemGetAddressRange(&base, &size, reinterpret_cast<CUdeviceptr>(d_ptr)),
              "cuMemGetAddressRange");
  if (!s.ok()) return Fail(s);
  CUipcMemHandle h;
  s = CuCheck(d.IpcGetMemHandle(&h, base), "cuIpcGetMemHandle");
  if (!s.ok()) return Fail(s);
  std::memcpy(handle64, &h, 64);
  *offset = static_cast<int64_t>(reinterpret_cast<CUdeviceptr>(d_ptr) - base);
  return GDV_OK;
}

gdv_status gdv_ipc_open(int32_t device, const uint8_t* handle64, int64_t offset, void** out_ptr) {
  if (handle64 == nullptr || out_ptr == nullptr) return Fail(GDV_INVALID, "gdv_ipc_open: null argument");
  Device* dev = nullptr;
  Status s = Device::Get(device, &dev);  // makes the context of `device` current
  if (!s.ok()) return Fail(s);
  CUipcMemHandle h;
  std::memcpy(&h, handle64, 64);
  CUdeviceptr base = 0;
  s = CuCheck(Driver().IpcOpenMemHandle(&base, h, CU_IPC_MEM_LAZY_ENABLE_PEER_ACCESS),
              "cuIpcOpenMemHandle");
  if (!s.ok()) return Fail(s);
  *out_ptr = reinterpret_cast<void*>(base + static_cast<CUdeviceptr>(offset));
  return GDV_OK;
}

gdv_status gdv_ipc_close(int32_t device, void* d_ptr, int64_t offset) {
  if (d_ptr == nullptr) return GDV_OK;
  Device* dev = nullptr;
  Status s = Device::Get(device, &dev);
  if (!s.ok()) return Fail(s);
  s = CuCheck(Driver().IpcCloseMemHandle(reinterpret_cast<CUdeviceptr>(d_ptr) -
                                          static_cast<CUdeviceptr>(offset)),
              "cuIpcCloseMemHandle");
  return s.ok() ? GDV_OK : Fail(s);
}

gdv_status gdv_selection_push(int32_t device, const void* d_src, const void* d_count, void* d_dst,
                              int64_t dst_capacity, void* board, int32_t board_slot, int32_t rank,
                              int32_t world, uint64_t seq, uint64_t need_consumed, int32_t mode,
                              int32_t ctas, void* d_local_counter, uint64_t done_target,
                              void* d_total_out, void* d_base, int32_t wave_flags,
                              int32_t consumed_slot, void* stream) {
  if (d_base != nullptr && (consumed_slot < 0 || consumed_slot >= GDV_BOARD_SLOTS))
    return Fail(GDV_INVALID, "gdv_selection_push: bad consumed_slot");
  if (world < 1 || world > GDV_BOARD_MAX_WORLD || rank < 0 || rank >= world || board == nullptr ||
      d_count == nullptr || board_slot < 0 || board_slot >= GDV_BOARD_SLOTS)
    return Fail(GDV_INVALID, "gdv_selection_push: bad arguments");
  const int sel = mode & ~GDV_SEL_BOUNDED;
  const int elem = sel == GDV_SEL_UINT16 ? 2 : sel == GDV_SEL_UINT32 ? 4 : sel == GDV_SEL_UINT64 ? 8 : 0;
  if (elem == 0) return Fail(GDV_INVALID, "gdv_selection_push: invalid selection vector mode");
  Device* dev = nullptr;
  Status s = Device::Get(device, &dev);
  if (!s.ok()) return Fail(s);
  CUfunction fn = nullptr;
  s = dev->StaticFunction("gdv_sel_push", &fn);
  if (!s.ok()) return Fail(s);
  CUstream st = stream != nullptr ? static_cast<CUstream>(stream) : dev->stream();
  uint64_t* b = static_cast<uint64_t*>(board);
  uint64_t* b_count = b + static_cast<size_t>(board_slot) * GDV_BOARD_MAX_WORLD;
  uint64_t* b_done = b + static_cast<size_t>(GDV_BOARD_SLOTS + board_slot) * GDV_BOARD_MAX_WORLD;
  uint64_t* b_cons = b + static_cast<size_t>(2 * GDV_BOARD_SLOTS) * GDV_BOARD_MAX_WORLD +
                     (d_base != nullptr ? consumed_slot : board_slot);
  uint64_t* b_err = b + static_cast<size_t>(2 * GDV_BOARD_SLOTS) * GDV_BOARD_MAX_WORLD + GDV_BOARD_SLOTS;
  int elem_bytes = elem;
  void* params[] = {&d_src, &d_count, &d_dst, &dst_capacity, &b_count, &b_done, &b_cons, &b_err,
                    &rank, &world, &seq, &need_consumed, &elem_bytes, &d_local_counter, &done_target,
                    &d_total_out, &d_base, &wave_flags};
  const bool one_thread = rank == 0 && d_base == nullptr;  // the root of a one-run-per-rank vector only waits
  const unsigned grid = one_thread ? 1u : static_cast<unsigned>(std::max(1, ctas));
  const unsigned threads = one_thread ? 32u : 256u;  // fits the slots a 256-thread persistent filter leaves free
  g_launch_count.fetch_add(1);
  s = CuCheck(Driver().LaunchKernel(fn, grid, 1, 1, threads, 1, 1, 0, st, params, nullptr),
              "cuLaunchKernel(gdv_sel_push)");
  return s.ok() ? GDV_OK : Fail(s);
}

gdv_status gdv_selection_release(int32_t device, void* board, int32_t board_slot, uint64_t seq,
                                 void* stream) {
  if (board == nullptr || board_slot < 0 || board_slot >= GDV_BOARD_SLOTS)
    return Fail(GDV_INVALID, "gdv_selection_release: bad arguments");
  Device* dev = nullptr;
  Status s = Device::Get(device, &dev);
  if (!s.ok()) return Fail(s);
  CUfunction fn = nullptr;
  s = dev->StaticFunction("gdv_sel_release", &fn);
  if (!s.ok()) return Fail(s);
  CUstream st = stream != nullptr ? static_cast<CUstream>(stream) : dev->stream();
  uint64_t* b_cons = static_cast<uint64_t*>(board) +
                     static_cast<size_t>(2 * GDV_BOARD_SLOTS) * GDV_BOARD_MAX_WORLD + board_slot;
  void* params[] = {&b_cons, &seq};
  g_launch_count.fetch_add(1);
  s = CuCheck(Driver().LaunchKernel(fn, 1, 1, 1, 32, 1, 1, 0, st, params, nullptr),
              "cuLaunchKernel(gdv_sel_release)");
  return s.ok() ? GDV_OK : Fail(s);
}

int64_t gdv_launch_count(void) { return g_launch_count.load(); }
int64_t gdv_compile_count(void) { return g_compile_count.load(); }

}  // extern "C"
