#include "gdv_runtime.h"
#include "gdv_rope_temps.h"

#include "gdv_staging.h"

#include <unistd.h>

#include <algorithm>
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstring>

namespace gdv {

std::atomic<long long> g_launch_count{0};
std::atomic<long long> g_compile_count{0};

const char* ExecutionErrorMessage(int code) {
  switch (code) {
    case 1: return "divide by zero error";
    case 2: return "a utf8/binary output needs more than 2^31 - 1 bytes (int32 offsets)";
    case 3: return "var_data capacity of a utf8/binary output is too small";
    case 4: return "Failed to cast the string to an integer of the requested type";
    case 5: return "Failed to cast the string to a date / timestamp (not a valid date / timestamp)";
    case 6: return "Index in split_part must be positive";
    case 7: return "Failed to cast the string to a decimal (not a decimal number)";
    case 8: return "Failed to cast the string to a float (not a number)";
    case 9: return "Invalid value for boolean";
    case 10: return "Output buffer length can't be negative";
    case 11: return "Start position must be greater than 0";
    case 12: return "Factorial of negative number not exist!";
    case 13: return "Factorial of number greater than 20 not supported!";
    case 14: return "Error parsing value for given format (to_date)";
    default: return "execution error in device function";
  }
}

// A user function raised (gdv_raise, kUserRaiseHelper): its message sits behind the error word of the
// 256-byte error block.
constexpr int kUserError = 1000;
static std::string UserErrorText(CUdeviceptr d_err, CUstream stream) {
  char text[248] = {0};
  const DriverApi& d = Driver();
  if (d.MemcpyDtoHAsync(text, d_err + 8, 240, stream) != CUDA_SUCCESS || d.StreamSynchronize(stream) != CUDA_SUCCESS ||
      text[0] == 0)
    return "error raised by a user function";
  return text;
}

// ======================================================================================
// Device
// ======================================================================================
namespace {
std::mutex g_dev_mu;
Device* g_devices[64] = {nullptr};

#define GDV_RETURN_NOT_OK(expr)      \
  do {                               \
    ::gdv::Status _s = (expr);       \
    if (!_s.ok()) return _s;         \
  } while (0)

// GDV_TRACE=1: phase timings of host-batch evaluations on stderr (where a call's microseconds go).
bool TraceOn() {
  static const bool on = std::getenv("GDV_TRACE") != nullptr;
  return on;
}
double NowUs() {
  return std::chrono::duration<double, std::micro>(std::chrono::steady_clock::now().time_since_epoch()).count();
}

size_t RoundPool(size_t bytes) {
  if (bytes < 512) return 512;
  if (bytes <= (1u << 20)) {
    size_t p = 512;
    while (p < bytes) p <<= 1;
    return p;
  }
  const size_t g = size_t(2) << 20;
  return (bytes + g - 1) / g * g;
}
}  // namespace

Status Device::Get(int ordinal, Device** out) {
  const DriverApi& d = Driver();
  if (!d.loaded)
    return Status::Make(GDV_CUDA_ERROR, "CUDA driver unavailable: " + d.load_error);
  if (ordinal < 0 || ordinal >= 64) return Status::Make(GDV_INVALID, "bad device ordinal");
  std::lock_guard<std::mutex> lock(g_dev_mu);
  if (g_devices[ordinal] == nullptr) {
    int count = 0;
    GDV_RETURN_NOT_OK(CuCheck(d.DeviceGetCount(&count), "cuDeviceGetCount"));
    if (ordinal >= count)
      return Status::Make(GDV_CUDA_ERROR, "device " + std::to_string(ordinal) +
                                              " not present (" + std::to_string(count) +
                                              " devices)");
    std::unique_ptr<Device> dev(new Device());
    dev->ordinal_ = ordinal;
    GDV_RETURN_NOT_OK(CuCheck(d.DeviceGet(&dev->dev_, ordinal), "cuDeviceGet"));
    GDV_RETURN_NOT_OK(
        CuCheck(d.DevicePrimaryCtxRetain(&dev->ctx_, dev->dev_), "cuDevicePrimaryCtxRetain"));
    GDV_RETURN_NOT_OK(CuCheck(d.CtxSetCurrent(dev->ctx_), "cuCtxSetCurrent"));
    d.DeviceGetAttribute(&dev->sm_count_, CU_DEVICE_ATTRIBUTE_MULTIPROCESSOR_COUNT, dev->dev_);
    d.DeviceGetAttribute(&dev->cc_major_, CU_DEVICE_ATTRIBUTE_COMPUTE_CAPABILITY_MAJOR, dev->dev_);
    d.DeviceGetAttribute(&dev->cc_minor_, CU_DEVICE_ATTRIBUTE_COMPUTE_CAPABILITY_MINOR, dev->dev_);
    GDV_RETURN_NOT_OK(
        CuCheck(d.StreamCreate(&dev->stream_, CU_STREAM_NON_BLOCKING), "cuStreamCreate"));
    dev->owner_thread_ = std::this_thread::get_id();
    if (const char* lim = std::getenv("GDV_POOL_LIMIT_MB")) dev->pool_limit_ = static_cast<size_t>(std::atoll(lim)) << 20;
    g_devices[ordinal] = dev.release();
  }
  *out = g_devices[ordinal];
  return (*out)->MakeCurrent();
}

namespace {
// Streams of the threads that did not create the Device; released at thread exit.
struct ThreadStreams {
  CUstream by_device[64] = {nullptr};
  ~ThreadStreams() {
    const DriverApi& d = Driver();
    if (!d.loaded) return;
    for (CUstream s : by_device)
      if (s != nullptr) d.StreamDestroy(s);  // fails harmlessly once the context is gone
  }
};
thread_local ThreadStreams tl_streams;
}  // namespace

CUstream Device::stream() const {
  if (std::this_thread::get_id() == owner_thread_) return stream_;
  CUstream& s = tl_streams.by_device[ordinal_];
  if (s == nullptr) {
    if (!MakeCurrent().ok() ||
        Driver().StreamCreate(&s, CU_STREAM_NON_BLOCKING) != CUDA_SUCCESS)
      return stream_;  // out of streams: fall back to the shared one
  }
  return s;
}

Status Device::MakeCurrent() const {
  return CuCheck(Driver().CtxSetCurrent(ctx_), "cuCtxSetCurrent");
}

std::string Device::arch() const {
  // This engine targets H100 only: sm_90a.  Other parts get their plain sm_XY so the
  // test-suite can still run on whatever GPU a developer has, without arch-specific code.
  if (cc_major_ == 9 && cc_minor_ == 0) return "sm_90a";
  return "sm_" + std::to_string(cc_major_) + std::to_string(cc_minor_);
}

Status Device::Alloc(size_t bytes, CUdeviceptr* out) {
  const size_t want = RoundPool(bytes);
  {
    std::lock_guard<std::mutex> lock(mu_);
    auto it = free_.lower_bound(want);
    if (it != free_.end() && it->first <= want * 2) {
      *out = it->second;
      idle_bytes_ -= it->first;
      free_.erase(it);
      return Status::OK();
    }
  }
  GDV_RETURN_NOT_OK(MakeCurrent());
  CUdeviceptr p = 0;
  CUresult r = Driver().MemAlloc(&p, want);
  if (r == CUDA_ERROR_OUT_OF_MEMORY) {
    // drop the cache and retry once
    Trim(0);
    r = Driver().MemAlloc(&p, want);
  }
  if (r != CUDA_SUCCESS) {
    Status s = CuCheck(r, "cuMemAlloc");
    if (r == CUDA_ERROR_OUT_OF_MEMORY) s.code = GDV_OUT_OF_MEMORY;
    return s;
  }
  {
    std::lock_guard<std::mutex> lock(mu_);
    sizes_[p] = want;
  }
  *out = p;
  return Status::OK();
}

void Device::Free(CUdeviceptr p) {
  if (p == 0) return;
  {
    std::lock_guard<std::mutex> lock(mu_);
    auto it = sizes_.find(p);
    if (it == sizes_.end()) return;
    free_.emplace(it->second, p);
    idle_bytes_ += it->second;
    if (idle_bytes_ <= pool_limit_) return;
  }
  // over the limit: the largest idle blocks go back to the driver (cuMemFree waits for work that
  // still uses a block, so releasing one that a queued kernel reads is safe, only slow)
  Trim(pool_limit_);
}

size_t Device::Trim(size_t keep_bytes) {
  std::vector<CUdeviceptr> drop;
  size_t released = 0;
  {
    std::lock_guard<std::mutex> lock(mu_);
    while (idle_bytes_ > keep_bytes && !free_.empty()) {
      auto big = std::prev(free_.end());
      idle_bytes_ -= big->first;
      released += big->first;
      sizes_.erase(big->second);
      drop.push_back(big->second);
      free_.erase(big);
    }
  }
  if (!drop.empty() && MakeCurrent().ok())
    for (auto q : drop) Driver().MemFree(q);
  return released;
}

Status Device::StaticFunction(const char* name, CUfunction* out) {
  std::lock_guard<std::mutex> lock(mu_);
  GDV_RETURN_NOT_OK(MakeCurrent());
  if (static_mod_ == nullptr) {
    GDV_RETURN_NOT_OK(CuCheck(Driver().ModuleLoadData(&static_mod_, gdv_static_kernels_cubin),
                              "cuModuleLoadData(static kernels)"));
  }
  auto it = static_fns_.find(name);
  if (it == static_fns_.end()) {
    CUfunction fn = nullptr;
    GDV_RETURN_NOT_OK(
        CuCheck(Driver().ModuleGetFunction(&fn, static_mod_, name), "cuModuleGetFunction"));
    it = static_fns_.emplace(name, fn).first;
  }
  *out = it->second;
  return Status::OK();
}

// ======================================================================================
// CompiledKernel
// ======================================================================================
Status CompiledKernel::Load(Device* dev, Loaded* out) {
  std::lock_guard<std::mutex> lock(mu_);
  auto it = loaded_.find(dev->ordinal());
  if (it != loaded_.end()) {
    *out = it->second;
    return Status::OK();
  }
  GDV_RETURN_NOT_OK(dev->MakeCurrent());
  const DriverApi& d = Driver();
  Loaded l;
  GDV_RETURN_NOT_OK(CuCheck(d.ModuleLoadData(&l.mod, cubin.data()), "cuModuleLoadData"));
  GDV_RETURN_NOT_OK(
      CuCheck(d.ModuleGetFunction(&l.fn, l.mod, gen.name.c_str()), "cuModuleGetFunction"));
  d.FuncGetAttribute(&l.regs, CU_FUNC_ATTRIBUTE_NUM_REGS, l.fn);
  d.FuncGetAttribute(&l.smem, CU_FUNC_ATTRIBUTE_SHARED_SIZE_BYTES, l.fn);
  if (gen.dynamic_smem > 32 * 1024)  // static + dynamic may pass the default 48 KB window
    GDV_RETURN_NOT_OK(CuCheck(d.FuncSetAttribute(l.fn, CU_FUNC_ATTRIBUTE_MAX_DYNAMIC_SHARED_SIZE_BYTES,
                                                 gen.dynamic_smem),
                              "cuFuncSetAttribute(max dynamic shared)"));
  int b = 0;
  if (d.OccupancyMaxActiveBlocksPerMultiprocessor(&b, l.fn, gen.block_threads,
                                                  static_cast<size_t>(gen.dynamic_smem)) ==
          CUDA_SUCCESS &&
      b > 0)
    l.blocks_per_sm = b;
  loaded_[dev->ordinal()] = l;
  *out = l;
  return Status::OK();
}

namespace {

// Compiled-kernel cache (the reference keeps an LRU of built projectors / filters keyed on schema +
// expressions + configuration, SURVEY.md §2): here the key is the generated translation unit
// itself plus the compile options, so two Make() calls that lower to the same kernel share one
// NVRTC compilation whatever objects they came from.  Kernel symbols are named after the hash of
// the source, which keeps the source text (and so the key) independent of creation order.
struct CachedCubin {
  std::vector<char> cubin;
  std::string ptx, log;
};
std::mutex g_cache_mu;
std::unordered_map<std::string, std::shared_ptr<const CachedCubin>> g_cubin_cache;
constexpr size_t kCubinCacheEntries = 512;

uint64_t Fnv1a(const std::string& s, uint64_t h = 1469598103934665603ull) {
  for (unsigned char c : s) {
    h ^= c;
    h *= 1099511628211ull;
  }
  return h;
}

const char* KernelPrefix(KernelKind kind) {
  switch (kind) {
    case KernelKind::kProject: return "gdv_project_expr_";
    case KernelKind::kFilter: return "gdv_filter_expr_";
    case KernelKind::kStringSize: return "gdv_strsize_expr_";
    default: return "gdv_strwrite_expr_";
  }
}

std::string Hex64(uint64_t h) {
  char hex[24];
  std::snprintf(hex, sizeof(hex), "%016llx", static_cast<unsigned long long>(h));
  return hex;
}

// The device function library is part of every translation unit: its text is part of the key, so a
// persisted cubin can never outlive the library it was compiled against.
std::string CubinKey(const std::string& arch, const Config& cfg, const std::string& source) {
  static const std::string lib_hex =
      Hex64(Fnv1a(std::string(gdv_device_lib_text, static_cast<size_t>(gdv_device_lib_text_len))));
  return arch + (cfg.optimize ? "|O3|" : "|O0|") + (cfg.dump_ir ? "ptx|" : "|") + lib_hex + "|" + source;
}

void RememberCubin(const std::string& key, std::shared_ptr<const CachedCubin> entry) {
  std::lock_guard<std::mutex> lock(g_cache_mu);
  if (g_cubin_cache.size() >= kCubinCacheEntries) g_cubin_cache.clear();
  g_cubin_cache.emplace(key, std::move(entry));
}

// GDV_CUBIN_CACHE_DIR=<dir>: cubins also persist across processes (the counterpart of the
// reference's object-code cache): <dir>/<fnv64 of arch|options|source>.cubin, written atomically.
// Empty when off, and with dump_ir: DumpIR wants the PTX too, so that always compiles.
std::string DiskCachePath(const std::string& key, const Config& cfg) {
  const char* cdir = std::getenv("GDV_CUBIN_CACHE_DIR");
  if (cdir == nullptr || cfg.dump_ir) return "";
  return std::string(cdir) + "/" + Hex64(Fnv1a(key)) + ".cubin";
}

bool IsElf(const std::vector<char>& b) {
  return b.size() > 4 && b[0] == 0x7f && b[1] == 'E' && b[2] == 'L' && b[3] == 'F';
}

// The persisted cubin at `path` when it is an ELF image that holds kernel `name`, else null.
std::shared_ptr<const CachedCubin> ReadDiskCubin(const std::string& path, const std::string& name) {
  FILE* f = std::fopen(path.c_str(), "rb");
  if (f == nullptr) return nullptr;
  std::vector<char> blob;
  char buf[65536];
  size_t got;
  while ((got = std::fread(buf, 1, sizeof(buf), f)) > 0) blob.insert(blob.end(), buf, buf + got);
  std::fclose(f);
  if (!IsElf(blob) || std::search(blob.begin(), blob.end(), name.begin(), name.end()) == blob.end()) return nullptr;
  auto entry = std::make_shared<CachedCubin>();
  entry->cubin = std::move(blob);
  return entry;
}

// Written to a per-process temporary and renamed, so that a reader never sees half a file.
void WriteDiskCubin(const std::string& path, const std::vector<char>& cubin) {
  if (!IsElf(cubin)) return;
  const std::string tmp = path + ".tmp" + std::to_string(static_cast<long long>(::getpid()));
  FILE* f = std::fopen(tmp.c_str(), "wb");
  if (f == nullptr) return;
  const bool ok = std::fwrite(cubin.data(), 1, cubin.size(), f) == cubin.size();
  std::fclose(f);
  if (ok) std::rename(tmp.c_str(), path.c_str());
  else std::remove(tmp.c_str());
}

// GDV_DUMP_DIR=<dir>: write <kernel>.cu / <kernel>.cubin for offline SASS inspection
// (cuobjdump -sass) and so that ncu's source page can find the generated code, and <kernel>.info
// with the launch fields the fuser chose (one key=value per line), so that two versions of the
// fuser can be compared kernel by kernel.
void DumpKernel(const char* dir, const CompiledKernel& k) {
  const std::string base = std::string(dir) + "/" + k.gen.name;
  if (FILE* f = std::fopen((base + ".cu").c_str(), "w")) {
    std::fwrite(k.gen.source.data(), 1, k.gen.source.size(), f);
    std::fclose(f);
  }
  if (FILE* f = std::fopen((base + ".info").c_str(), "w")) {
    const GeneratedKernel& g = k.gen;
    std::fprintf(f, "rows_per_thread=%d\nblock_threads=%d\nselection_mode=%d\nnullable=%d\n", g.rows_per_thread,
                 g.block_threads, g.selection_mode, g.nullable ? 1 : 0);
    for (size_t j = 0; j < g.inputs.size(); ++j) {
      const gdv_type_t t = g.inputs[j].type.c();
      std::fprintf(f, "input%zu=col %d type %d/%d/%d hoist %d\n", j, g.inputs[j].schema_index, t.id, t.precision,
                   t.scale, g.inputs[j].hoist ? 1 : 0);
    }
    for (size_t o = 0; o < g.outputs.size(); ++o) {
      const gdv_type_t t = g.outputs[o].c();
      std::fprintf(f, "output%zu=type %d/%d/%d\n", o, t.id, t.precision, t.scale);
    }
    std::fprintf(f, "uses_ctx=%d\nin_bytes_per_row=%d\nout_bytes_per_row=%d\nargs_size=%zu\ndynamic_smem=%d\n",
                 g.uses_ctx ? 1 : 0, g.in_bytes_per_row, g.out_bytes_per_row, g.args.size, g.dynamic_smem);
    std::fprintf(f, "tile_rows=%lld\nkey_driven=%d\nstaged=%d\nstages=%d\ncta_tile_rows=%lld\n",
                 static_cast<long long>(g.tile_rows), g.key_driven ? 1 : 0, g.staged ? 1 : 0, g.stages,
                 static_cast<long long>(g.cta_tile_rows));
    std::fprintf(f, "view_shortcuts=%d\ngated_stages=%d\n", g.view_shortcuts, g.gated_stages);
    std::fclose(f);
  }
  if (FILE* f = std::fopen((base + ".cubin").c_str(), "wb")) {
    std::fwrite(k.cubin.data(), 1, k.cubin.size(), f);
    std::fclose(f);
  }
}

Status BuildKernel(const Schema& schema, const std::vector<ExpressionPtr>& exprs,
                   KernelKind kind, int selection_mode, bool nullable, const Config& cfg,
                   std::unique_ptr<CompiledKernel>* out) {
  KernelSpec spec;
  spec.kind = kind;
  spec.nullable = nullable;
  spec.selection_mode = selection_mode;
  spec.rows_per_thread = cfg.rows_per_thread;
  spec.block_threads = cfg.block_threads;  // 0: the fuser picks per kernel shape
  spec.loader = cfg.loader;
  spec.stages = cfg.stages;
  spec.string_scan = cfg.string_scan;
  spec.filter_gating = cfg.filter_gating;
  spec.large_batch = cfg.large_batch;
  const std::string placeholder = std::string(KernelPrefix(kind)) + "PLACEHOLDER";
  spec.name = placeholder;
  std::unique_ptr<CompiledKernel> k(new CompiledKernel());
  const FunctionRegistry::Scope user_functions(cfg.functions.get());
  GDV_RETURN_NOT_OK(GenerateKernel(schema, exprs, spec, &k->gen));
  // Compile for the device we will run on when one is visible, else for H100.
  std::string arch = "sm_90a";
  Device* dev = nullptr;
  if (Driver().loaded && Device::Get(cfg.device, &dev).ok()) arch = dev->arch();
  // name the kernel after its own text
  const std::string name = std::string(KernelPrefix(kind)) + Hex64(Fnv1a(arch, Fnv1a(k->gen.source)));
  for (size_t pos = 0; (pos = k->gen.source.find(placeholder, pos)) != std::string::npos;)
    k->gen.source.replace(pos, placeholder.size(), name);
  k->gen.name = name;
  const std::string key = CubinKey(arch, cfg, k->gen.source);
  std::shared_ptr<const CachedCubin> hit;
  {
    std::lock_guard<std::mutex> lock(g_cache_mu);
    auto it = g_cubin_cache.find(key);
    if (it != g_cubin_cache.end()) hit = it->second;
  }
  const std::string disk_path = DiskCachePath(key, cfg);
  if (hit == nullptr && !disk_path.empty()) {
    hit = ReadDiskCubin(disk_path, name);
    if (hit != nullptr) RememberCubin(key, hit);
  }
  if (hit != nullptr) {
    k->cubin = hit->cubin;
    k->ptx = hit->ptx;
    k->compile_log = hit->log;
  } else {
    g_compile_count.fetch_add(1);
    GDV_RETURN_NOT_OK(CompileToCubin(k->gen.source, arch, cfg.optimize, cfg.dump_ir, &k->cubin,
                                     &k->ptx, &k->compile_log));
    if (!disk_path.empty()) WriteDiskCubin(disk_path, k->cubin);
    // a translation unit can compile "successfully" without the kernel in it (e.g. when the
    // front end stops at a stray byte): make that a code-generation error here, not a missing
    // symbol at the first Evaluate on a GPU
    if (std::search(k->cubin.begin(), k->cubin.end(), name.begin(), name.end()) == k->cubin.end())
      return Status::Make(GDV_CODEGEN_ERROR, "NVRTC produced a module without the kernel " + name);
    auto entry = std::make_shared<CachedCubin>();
    entry->cubin = k->cubin;
    entry->ptx = k->ptx;
    entry->log = k->compile_log;
    RememberCubin(key, std::move(entry));
  }
  if (const char* dir = std::getenv("GDV_DUMP_DIR")) DumpKernel(dir, *k);
  *out = std::move(k);
  return Status::OK();
}

// One kernel input after staging: device addresses + bit shifts.  Dictionary columns: val / vld /
// vsh are the indices', var the dictionary's bytes, and dof / dvl / dvs / dln the dictionary's
// offsets, validity words, bit shift and length.  View columns: val is the views, and vbf / vsz /
// vbn the device pointer table of the data buffers, their sizes and their count.
struct ResolvedIn {
  CUdeviceptr val = 0, vld = 0, var = 0;
  uint32_t vsh = 0, dsh = 0;
  CUdeviceptr dof = 0, dvl = 0;
  uint32_t dvs = 0;
  int64_t dln = 0;
  CUdeviceptr vbf = 0, vsz = 0;
  int64_t vbn = 0;
};

inline int64_t BitBytes(int64_t bit_begin, int64_t nbits) {
  // bytes that cover bits [bit_begin, bit_begin + nbits) counted from the byte of bit_begin
  return ((bit_begin & 7) + nbits + 7) / 8;
}

constexpr const char* kValuesMisaligned = "device values buffer of column %d is not aligned to its element width";
constexpr const char* kIndicesMisaligned = "device indices buffer of column %d is not aligned to its element width";

// A contiguous array of `bytes` bytes as the kernels read it.  A host array is staged into pooled scratch
// with `pad` bytes to spare; a device array is read in place and must be aligned to `align` bytes, or the
// call fails with `what` (a format that takes the column `col`).
Status ResolveArray(Device* dev, const void* p, size_t bytes, size_t pad, size_t align, bool host, CUstream stream,
                    ScratchScope* scratch, const char* what, int col, CUdeviceptr* out) {
  if (host) {
    GDV_RETURN_NOT_OK(scratch->Alloc(bytes + pad, out));
    return bytes > 0 ? StagedHtoD(dev, *out, p, bytes, stream) : Status::OK();
  }
  if (reinterpret_cast<uintptr_t>(p) % align != 0) {
    char msg[128];
    std::snprintf(msg, sizeof(msg), what, col);
    return Status::Make(GDV_INVALID, msg);
  }
  *out = reinterpret_cast<CUdeviceptr>(p);
  return Status::OK();
}

// A bitmap of `nbits` bits from bit `off` on as the kernels read it: a 4-byte aligned word pointer
// plus a bit shift in [0, 31] (host bitmaps are staged into pooled device memory first).
Status ResolveBitmap(Device* dev, const void* bits, int64_t off, int64_t nbits, bool host, CUstream stream,
                     ScratchScope* scratch, CUdeviceptr* ptr, uint32_t* sh) {
  const uint8_t* p = static_cast<const uint8_t*>(bits) + (off >> 3);
  *sh = static_cast<uint32_t>(off & 7);
  if (host) return ResolveArray(dev, p, static_cast<size_t>(BitBytes(off, nbits)), 8, 1, host, stream, scratch, nullptr, 0, ptr);
  const uintptr_t mis = reinterpret_cast<uintptr_t>(p) & 3u;
  *ptr = reinterpret_cast<CUdeviceptr>(p - mis);
  *sh += static_cast<uint32_t>(8 * mis);
  return Status::OK();
}

// The dictionary of a dictionary-encoded column (gdv_dictionary_t, reached through var_data).
Status ResolveDictionary(Device* dev, int col, const gdv_column_t& c, bool host, CUstream stream,
                         ScratchScope* scratch, ResolvedIn* r) {
  const auto* dict = static_cast<const gdv_dictionary_t*>(c.var_data);
  const std::string what = "dictionary column " + std::to_string(col);
  if (dict == nullptr) return Status::Make(GDV_INVALID, what + " has no dictionary (var_data must point at a gdv_dictionary_t)");
  if (dict->length < 0 || dict->offset < 0) return Status::Make(GDV_INVALID, what + ": negative dictionary length or offset");
  r->dln = dict->length;
  if (dict->length == 0) return Status::OK();  // every index is out of range: no row reads it
  if (dict->offsets == nullptr) return Status::Make(GDV_INVALID, what + ": the dictionary has no offsets buffer");
  const int32_t* offs = static_cast<const int32_t*>(dict->offsets) + dict->offset;
  if (dict->validity != nullptr)
    GDV_RETURN_NOT_OK(ResolveBitmap(dev, dict->validity, dict->offset, dict->length, host, stream, scratch, &r->dvl, &r->dvs));
  GDV_RETURN_NOT_OK(ResolveArray(dev, offs, static_cast<size_t>(dict->length + 1) * 4, 0, 1, host, stream, scratch,
                                 nullptr, col, &r->dof));
  if (!host) {
    r->var = reinterpret_cast<CUdeviceptr>(dict->data);
    return Status::OK();
  }
  const int64_t first = offs[0], last = offs[dict->length];
  if (first < 0 || last < first || (last > first && (dict->data == nullptr || last > dict->data_size)))
    return Status::Make(GDV_INVALID, what + ": the dictionary's offsets reach past its data buffer");
  GDV_RETURN_NOT_OK(ResolveArray(dev, static_cast<const uint8_t*>(dict->data) + first, static_cast<size_t>(last - first),
                                 16, 1, host, stream, scratch, nullptr, col, &r->var));
  r->var -= static_cast<CUdeviceptr>(first);  // kernel addresses bytes as var + offs[i]
  return Status::OK();
}

// The data buffers of a string_view / binary_view column (gdv_view_buffers_t, reached through
// var_data).  Device batches: the buffers and their sizes are read in place; only the host array of
// buffer pointers is copied, asynchronously on `stream`, into pooled scratch.  Host batches: every
// buffer is staged whole (a sliced batch may carry bytes no row of the slice uses), and the table of
// their device copies and the sizes next to them.  Only what is cheap is checked here; a view that
// reaches outside its buffer is caught per row by the kernel (gdv_sv_view).
Status ResolveViewBuffers(Device* dev, int col, const gdv_column_t& c, bool host, CUstream stream,
                          ScratchScope* scratch, ResolvedIn* r) {
  const auto* vb = static_cast<const gdv_view_buffers_t*>(c.var_data);
  const std::string what = "view column " + std::to_string(col);
  if (vb == nullptr)
    return Status::Make(GDV_INVALID, what + " has no data buffers (var_data must point at a gdv_view_buffers_t)");
  if (vb->n < 0) return Status::Make(GDV_INVALID, what + ": negative data buffer count");
  r->vbn = vb->n;
  if (vb->n == 0) return Status::OK();  // every valid view is inline
  if (vb->data == nullptr || vb->sizes == nullptr)
    return Status::Make(GDV_INVALID, what + ": null data buffer table or sizes");
  const size_t tbytes = static_cast<size_t>(vb->n) * 8;
  GDV_RETURN_NOT_OK(scratch->Alloc(tbytes, &r->vbf));
  if (!host) {
    GDV_RETURN_NOT_OK(StagedHtoD(dev, r->vbf, vb->data, tbytes, stream));
    r->vsz = reinterpret_cast<CUdeviceptr>(vb->sizes);
    return Status::OK();
  }
  std::vector<CUdeviceptr> table(static_cast<size_t>(vb->n), 0);
  for (int32_t i = 0; i < vb->n; ++i) {
    const int64_t sz = vb->sizes[i];
    if (sz < 0) return Status::Make(GDV_INVALID, what + ": negative size of data buffer " + std::to_string(i));
    if (sz == 0) continue;
    if (vb->data[i] == nullptr) return Status::Make(GDV_INVALID, what + ": data buffer " + std::to_string(i) + " is null");
    GDV_RETURN_NOT_OK(ResolveArray(dev, vb->data[i], static_cast<size_t>(sz), 16, 1, host, stream, scratch, nullptr, col,
                                   &table[static_cast<size_t>(i)]));
  }
  GDV_RETURN_NOT_OK(StagedHtoD(dev, r->vbf, table.data(), tbytes, stream));
  return ResolveArray(dev, vb->sizes, tbytes, 0, 1, host, stream, scratch, nullptr, col, &r->vsz);
}

Status ResolveInputs(Device* dev, const GeneratedKernel& gen, const gdv_batch_t* batch,
                     CUstream stream, ScratchScope* scratch, std::vector<ResolvedIn>* out) {
  const bool host = batch->mem_space == GDV_MEM_HOST;
  const int64_t n = batch->num_rows;
  out->resize(gen.inputs.size());
  for (size_t j = 0; j < gen.inputs.size(); ++j) {
    const ColumnSlot& slot = gen.inputs[j];
    if (slot.schema_index < 0 || slot.schema_index >= batch->num_columns)
      return Status::Make(GDV_INVALID, "batch has fewer columns than the schema");
    const int col = slot.schema_index;
    const gdv_column_t& c = batch->columns[col];
    ResolvedIn r;
    const int64_t off = c.offset;
    const DataType& t = slot.type;
    if (c.values == nullptr && n > 0)
      return Status::Make(GDV_INVALID, "column " + std::to_string(col) + " has no values buffer");
    if (c.validity != nullptr)
      GDV_RETURN_NOT_OK(ResolveBitmap(dev, c.validity, off, n, host, stream, scratch, &r.vld, &r.vsh));
    const uint8_t* values = static_cast<const uint8_t*>(c.values);
    if (t.is_bool()) {
      GDV_RETURN_NOT_OK(ResolveBitmap(dev, c.values, off, n, host, stream, scratch, &r.val, &r.dsh));
    } else if (t.is_dict()) {
      // the indices like a fixed-width column of the index type, then the dictionary
      const int w = DataType(t.index).width();
      GDV_RETURN_NOT_OK(ResolveArray(dev, values + off * w, static_cast<size_t>(n) * w, 16, w, host, stream, scratch, kIndicesMisaligned, col,
                                     &r.val));
      GDV_RETURN_NOT_OK(ResolveDictionary(dev, col, c, host, stream, scratch, &r));
    } else if (t.is_view()) {
      // the 16-byte views like a fixed-width column, then the data buffers
      GDV_RETURN_NOT_OK(ResolveArray(dev, values + off * 16, static_cast<size_t>(n) * 16, 16, 16, host, stream, scratch,
                                     "device views buffer of column %d is not 16-byte aligned", col, &r.val));
      GDV_RETURN_NOT_OK(ResolveViewBuffers(dev, col, c, host, stream, scratch, &r));
    } else if (t.is_varlen()) {
      // n + 1 offsets of t.width() bytes (int32, or int64 for a large column)
      const int w = t.width();
      const uint8_t* offs = values + off * w;
      auto at = [&](int64_t i) -> int64_t {
        return t.is_large() ? reinterpret_cast<const int64_t*>(offs)[i] : reinterpret_cast<const int32_t*>(offs)[i];
      };
      GDV_RETURN_NOT_OK(ResolveArray(dev, offs, static_cast<size_t>(n + 1) * w, 0, 1, host, stream, scratch, nullptr, col,
                                     &r.val));
      if (host) {
        const int64_t first = n > 0 ? at(0) : 0, last = n > 0 ? at(n) : 0;
        GDV_RETURN_NOT_OK(ResolveArray(dev, static_cast<const uint8_t*>(c.var_data) + first,
                                       static_cast<size_t>(last - first), 16, 1, host, stream, scratch, nullptr, col,
                                       &r.var));
        // kernel addresses bytes as var + offs[r]; rebase so offs[0] lands on the staged bytes
        r.var -= static_cast<CUdeviceptr>(first);
      } else {
        r.var = reinterpret_cast<CUdeviceptr>(c.var_data);
      }
    } else {
      const int w = t.width();
      GDV_RETURN_NOT_OK(ResolveArray(dev, values + off * w, static_cast<size_t>(n) * w, 16, w, host, stream, scratch, kValuesMisaligned, col,
                                     &r.val));
    }
    (*out)[j] = r;
  }
  return Status::OK();
}

template <typename T>
void Put(std::vector<uint8_t>& buf, size_t off, T v) {
  std::memcpy(buf.data() + off, &v, sizeof(T));
}

void PutInputs(std::vector<uint8_t>& args, const ArgsLayout& L, const std::vector<ResolvedIn>& ins) {
  for (size_t j = 0; j < ins.size(); ++j) {
    Put<CUdeviceptr>(args, L.off_in_val + 8 * j, ins[j].val);
    Put<CUdeviceptr>(args, L.off_in_vld + 8 * j, ins[j].vld);
    Put<CUdeviceptr>(args, L.off_in_var + 8 * j, ins[j].var);
    Put<uint32_t>(args, L.off_in_vsh + 4 * j, ins[j].vsh);
    Put<uint32_t>(args, L.off_in_dsh + 4 * j, ins[j].dsh);
    if (L.dict) {
      Put<CUdeviceptr>(args, L.off_in_dof + 8 * j, ins[j].dof);
      Put<CUdeviceptr>(args, L.off_in_dvl + 8 * j, ins[j].dvl);
      Put<int64_t>(args, L.off_in_dln + 8 * j, ins[j].dln);
      Put<uint32_t>(args, L.off_in_dvs + 4 * j, ins[j].dvs);
    }
    if (L.view) {
      Put<CUdeviceptr>(args, L.off_in_vbf + 8 * j, ins[j].vbf);
      Put<CUdeviceptr>(args, L.off_in_vsz + 8 * j, ins[j].vsz);
      Put<int64_t>(args, L.off_in_vbn + 8 * j, ins[j].vbn);
    }
  }
}

Status LaunchKernel(Device* dev, const CompiledKernel::Loaded& l, const GeneratedKernel& gen,
                    std::vector<uint8_t>& args, unsigned grid, CUstream stream) {
  void* params[] = {args.data()};
  if (grid == 0) return Status::OK();
  g_launch_count.fetch_add(1);
  return CuCheck(Driver().LaunchKernel(l.fn, grid, 1, 1, static_cast<unsigned>(gen.block_threads),
                                       1, 1, static_cast<unsigned>(gen.dynamic_smem), stream,
                                       params, nullptr),
                 "cuLaunchKernel");
}

int SelWidth(int mode) {
  switch (mode) {
    case GDV_SEL_UINT16: return 2;
    case GDV_SEL_UINT32: return 4;
    case GDV_SEL_UINT64: return 8;
    default: return 0;
  }
}

// Blocks for a grid-stride kernel: as many as the work needs, at most `blocks_per_sm` on each SM the
// configuration leaves to the engine.
unsigned GridFor(const Device* dev, const Config& cfg, int blocks_per_sm, int64_t blocks_needed) {
  const int64_t cap = static_cast<int64_t>(std::max(1, dev->sm_count() - cfg.sm_reserve)) * blocks_per_sm;
  return static_cast<unsigned>(std::min(blocks_needed, cap));
}

// The selection vector's `n` slots into `args` (host indices are staged into scratch), and where the
// kernel reads the slot count when it stays on the device.
Status PutSelection(Device* dev, const gdv_selection_t* sel, int64_t n, bool host, CUstream stream,
                    ScratchScope* scratch, const ArgsLayout& L, std::vector<uint8_t>& args) {
  CUdeviceptr dsel = 0;
  GDV_RETURN_NOT_OK(ResolveArray(dev, sel->indices, static_cast<size_t>(n) * SelWidth(sel->mode), 16, 1, host, stream,
                                 scratch, nullptr, 0, &dsel));
  Put<CUdeviceptr>(args, L.off_sel, dsel);
  if (sel->d_num_slots != nullptr) Put<CUdeviceptr>(args, L.off_n_ptr, reinterpret_cast<CUdeviceptr>(sel->d_num_slots));
  return Status::OK();
}

}  // namespace

// ======================================================================================
// PendingTable
// ======================================================================================
Status PendingTable::Entry::ErrorBlock(Device* dev, CUstream stream, CUdeviceptr* out) {
  if (d_err == 0) {
    GDV_RETURN_NOT_OK(dev->Alloc(256, &d_err));
    GDV_RETURN_NOT_OK(CuCheck(Driver().MemsetD8Async(d_err, 0, 256, stream), "memset err"));
  }
  *out = d_err;
  return Status::OK();
}

Status PendingTable::Settle(Device* dev, CUstream stream, int64_t* num_slots) {
  const DriverApi& d = Driver();
  Entry pend;
  bool have = false;
  {
    std::lock_guard<std::mutex> lock(mu_);
    auto it = entries_.find(stream);
    if (it != entries_.end()) {
      pend = std::move(it->second);
      entries_.erase(it);
      have = true;
    }
  }
  int err = 0;
  uint64_t count = 0;
  Status copy = Status::OK();
  if (pend.d_err != 0) copy = CuCheck(d.MemcpyDtoHAsync(&err, pend.d_err, sizeof(int), stream), "D2H err");
  if (copy.ok() && pend.d_count != 0)
    copy = CuCheck(d.MemcpyDtoHAsync(&count, pend.d_count, sizeof(count), stream), "D2H count");
  Status s = CuCheck(d.StreamSynchronize(stream), "cuStreamSynchronize");
  std::string detail;  // a capacity error of a device-count string output: which output, how many bytes
  if (copy.ok() && s.ok() && err == 3) {
    for (const auto& vc : pend.var_checks) {
      uint64_t total = 0;
      if (d.MemcpyDtoHAsync(&total, vc.d_total, 8, stream) != CUDA_SUCCESS || d.StreamSynchronize(stream) != CUDA_SUCCESS) break;
      if (total > static_cast<uint64_t>(vc.capacity)) {
        detail = ": output " + std::to_string(vc.out_index) + " needs " + std::to_string(total) +
                 " bytes, its var_capacity is " + std::to_string(vc.capacity);
        break;
      }
    }
  }
  std::string user_text;
  if (copy.ok() && s.ok() && err == kUserError) user_text = UserErrorText(pend.d_err, stream);
  // on every path: the pending blocks go back to the pool once the stream is idle
  if (pend.d_err != 0) dev->Free(pend.d_err);
  for (auto p : pend.scratch) dev->Free(p);
  GDV_RETURN_NOT_OK(copy);
  GDV_RETURN_NOT_OK(s);
  if (err != 0) return Status::Make(GDV_EXECUTION_ERROR, (err == kUserError ? user_text : ExecutionErrorMessage(err)) + detail);
  if (num_slots != nullptr) *num_slots = have ? static_cast<int64_t>(count) : -1;
  return Status::OK();
}

// ======================================================================================
// Projector
// ======================================================================================
Status Projector::Make(SchemaPtr schema, std::vector<ExpressionPtr> exprs, int selection_mode,
                       const Config& cfg, std::shared_ptr<Projector>* out) {
  if (schema == nullptr) return Status::Make(GDV_INVALID, "Schema cannot be null");
  if (exprs.empty()) return Status::Make(GDV_INVALID, "Expressions cannot be empty");
  const FunctionRegistry::Scope user_functions(cfg.functions.get());
  for (const auto& e : exprs) {
    if (e == nullptr) return Status::Make(GDV_INVALID, "Expression cannot be null");
    GDV_RETURN_NOT_OK(ValidateExpression(*schema, *e));
  }
  std::shared_ptr<Projector> p(new Projector());
  p->schema_ = schema;
  p->exprs_ = std::move(exprs);
  p->selection_mode_ = selection_mode;
  p->cfg_ = cfg;
  Status st = p->BuildKernels();
  if (!st.ok()) {
    // something other than projection / concat / if-else reads a rope: materialise the ropes first
    if (!IsRopeConsumerError(st)) return st;
    const Status two_stage = MakeWithRopeTemps(schema, p->exprs_, selection_mode, cfg, p.get());
    // the plan can still hit another limit of the fuser (e.g. a concat of more than 8 pieces): say that one
    if (!two_stage.ok()) return IsRopeConsumerError(two_stage) ? st : two_stage;
  }
  *out = std::move(p);
  return Status::OK();
}

Status Projector::BuildKernels() {
  Projector* p = this;
  const SchemaPtr& schema = schema_;
  const int selection_mode = selection_mode_;
  const Config& cfg = cfg_;
  p->strings_.clear();
  p->fixed_exprs_.clear();
  p->fixed_idx_.clear();
  // Fixed-width outputs share ONE fused kernel; every utf8/binary output gets its own
  // sizing + write kernel pair (its bytes cannot be placed before all lengths are known).
  for (size_t i = 0; i < p->exprs_.size(); ++i) {
    if (p->exprs_[i]->result().type.is_varlen()) {
      StringKernels sk;
      sk.out_index = static_cast<int>(i);
      p->strings_.push_back(std::move(sk));
    } else {
      p->fixed_exprs_.push_back(p->exprs_[i]);
      p->fixed_idx_.push_back(static_cast<int>(i));
    }
  }
  if (!p->fixed_exprs_.empty())
    GDV_RETURN_NOT_OK(BuildKernel(*schema, p->fixed_exprs_, KernelKind::kProject, selection_mode, true,
                                  cfg, &p->kernel_));
  for (auto& sk : p->strings_) {
    CompiledKernel *a = nullptr, *b = nullptr;
    GDV_RETURN_NOT_OK(p->StringKernelsFor(&sk, true, &a, &b));
    if (std::getenv("GDV_EAGER_NONULL") != nullptr) GDV_RETURN_NOT_OK(p->StringKernelsFor(&sk, false, &a, &b));
  }
  if (std::getenv("GDV_EAGER_NONULL") != nullptr && p->kernel_ != nullptr) {
    CompiledKernel* k = nullptr;
    GDV_RETURN_NOT_OK(p->KernelFor(false, &k));
  }
  return Status::OK();
}

// ---- consumers of a rope: temps first (gdv_rope_temps.h) ---------------------------------------------------
namespace {
// The first stage of the two-stage plan: the ropes that `exprs` consume become the expressions of `rt`,
// `rewritten` reads them as columns of the returned schema, `schema` plus one column per temporary.
SchemaPtr ExtractRopeTemps(const SchemaPtr& schema, const std::vector<ExpressionPtr>& exprs, RopeTemps* rt,
                           std::vector<ExpressionPtr>* rewritten) {
  for (const auto& e : exprs) {
    NodePtr r;
    ExtractRopes(e->root(), e->result().type.is_varlen(), rt, &r);
    rewritten->push_back(std::make_shared<Expression>(r, e->result()));
  }
  std::vector<Field> fields = schema->fields();
  fields.insert(fields.end(), rt->fields.begin(), rt->fields.end());
  return std::make_shared<Schema>(std::move(fields));
}

// Runs `eval` over `batch` extended by the temporaries `pre` materialises.  The temporaries of a device
// batch go back to the pool when this returns: not before the work that reads them.
template <typename Eval>
Status EvaluateOverTemps(Projector* pre, const gdv_batch_t* batch, void* stream_v, Eval eval) {
  TempColumns tc;
  GDV_RETURN_NOT_OK(tc.Build(pre, batch, stream_v));
  Status st = eval(&tc.batch);
  if (batch->mem_space != GDV_MEM_HOST) {
    Device* dev = nullptr;
    Status w = Device::Get(pre->config().device, &dev);
    if (w.ok()) {
      CUstream stream = stream_v != nullptr ? static_cast<CUstream>(stream_v) : dev->stream();
      w = CuCheck(Driver().StreamSynchronize(stream), "cuStreamSynchronize");
    }
    if (st.ok()) st = w;
  }
  return st;
}
}  // namespace

Status Projector::MakeWithRopeTemps(const SchemaPtr& schema, const std::vector<ExpressionPtr>& exprs,
                                    int selection_mode, const Config& cfg, Projector* into) {
  RopeTemps rt;
  std::vector<ExpressionPtr> rewritten;
  const SchemaPtr extended = ExtractRopeTemps(schema, exprs, &rt, &rewritten);
  if (rt.temps.empty()) return Status::Make(GDV_NOT_IMPLEMENTED, "no rope to materialise");
  // nesting: the temps' own Projector may need temporaries of its own (a consumer inside a rope's arguments)
  static thread_local int depth = 0;
  if (depth >= 8) return Status::Make(GDV_NOT_IMPLEMENTED, "rope consumers nested more than 8 levels deep");
  struct Level {
    int& d;
    explicit Level(int& x) : d(x) { ++d; }
    ~Level() { --d; }
  } level(depth);
  std::shared_ptr<Projector> pre, main;
  GDV_RETURN_NOT_OK(Projector::Make(schema, rt.temps, GDV_SEL_NONE, cfg, &pre));
  GDV_RETURN_NOT_OK(Projector::Make(extended, rewritten, selection_mode, cfg, &main));
  if (main->rope_main_ != nullptr) return Status::Make(GDV_NOT_IMPLEMENTED, "rope consumer left after materialisation");
  into->rope_pre_ = std::move(pre);
  into->rope_main_ = std::move(main);
  return Status::OK();
}

TempColumns::~TempColumns() {
  if (dev != nullptr)
    for (CUdeviceptr p : device) dev->Free(p);
}

// Runs the pre-projector over `in` (all rows, no selection vector) and appends its utf8 outputs to the batch's
// columns: in host vectors for a host batch, in pooled device memory for a device batch.  Synchronous.
Status TempColumns::Build(Projector* pre, const gdv_batch_t* in, void* stream) {
  if (pre->rope_main() != nullptr) {
    lower.reset(new TempColumns());
    GDV_RETURN_NOT_OK(lower->Build(pre->rope_pre(), in, stream));
    return Run(pre->rope_main(), &lower->batch, in, stream);
  }
  return Run(pre, in, in, stream);
}

// `pre` evaluated over `eval` (which may carry lower-level temporaries); its outputs appended to the columns of `in`.
Status TempColumns::Run(Projector* pre, const gdv_batch_t* eval, const gdv_batch_t* in, void* stream) {
  const int n_temps = pre->num_outputs();
  const int64_t n = in->num_rows;
  const bool on_host = in->mem_space == GDV_MEM_HOST;
  cols.assign(in->columns, in->columns + in->num_columns);
  std::vector<gdv_out_column_t> outs(static_cast<size_t>(n_temps));
  const size_t off_bytes = static_cast<size_t>(n + 1) * 4 + 16, vld_bytes = static_cast<size_t>((n + 63) / 64) * 8 + 8;
  if (!on_host) GDV_RETURN_NOT_OK(Device::Get(pre->config().device, &dev));
  for (int k = 0; k < n_temps; ++k) {
    int64_t bytes = 0;
    GDV_RETURN_NOT_OK(pre->OutputVarSize(eval, nullptr, k, stream, &bytes));
    gdv_out_column_t& o = outs[static_cast<size_t>(k)];
    std::memset(&o, 0, sizeof(o));
    const size_t data_bytes = static_cast<size_t>(bytes) + 16;
    if (on_host) {
      host.emplace_back(off_bytes);
      o.values = host.back().data();
      host.emplace_back(vld_bytes);
      o.validity = host.back().data();
      host.emplace_back(data_bytes);
      o.var_data = host.back().data();
    } else {
      CUdeviceptr p = 0;
      GDV_RETURN_NOT_OK(dev->Alloc(off_bytes, &p));
      device.push_back(p);
      o.values = reinterpret_cast<void*>(p);
      GDV_RETURN_NOT_OK(dev->Alloc(vld_bytes, &p));
      device.push_back(p);
      o.validity = reinterpret_cast<void*>(p);
      GDV_RETURN_NOT_OK(dev->Alloc(data_bytes, &p));
      device.push_back(p);
      o.var_data = reinterpret_cast<void*>(p);
    }
    o.var_capacity = bytes;
  }
  GDV_RETURN_NOT_OK(pre->Evaluate(eval, nullptr, outs.data(), n_temps, stream, /*async=*/false));
  for (int k = 0; k < n_temps; ++k) {
    gdv_column_t c;
    std::memset(&c, 0, sizeof(c));
    c.validity = outs[static_cast<size_t>(k)].validity;
    c.values = outs[static_cast<size_t>(k)].values;
    c.var_data = outs[static_cast<size_t>(k)].var_data;
    c.offset = 0;
    c.var_data_size = outs[static_cast<size_t>(k)].var_capacity;
    cols.push_back(c);
  }
  batch = *in;
  batch.num_columns = static_cast<int32_t>(cols.size());
  batch.columns = cols.data();
  return Status::OK();
}

CompiledKernel& Projector::kernel() {
  if (rope_main_ != nullptr) return rope_main_->kernel();
  if (last_used_ != nullptr) return *last_used_;
  if (kernel_ != nullptr) return *kernel_;
  return *strings_.front().write[0];
}

Status Projector::StringKernelsFor(StringKernels* sk, bool nullable, CompiledKernel** size,
                                   CompiledKernel** write) {
  std::lock_guard<std::mutex> lock(mu_);
  const int v = nullable ? 0 : 1;
  if (sk->size[v] == nullptr) {
    std::vector<ExpressionPtr> one = {exprs_[static_cast<size_t>(sk->out_index)]};
    Config cfg = cfg_;
    cfg.loader = 1;
    GDV_RETURN_NOT_OK(BuildKernel(*schema_, one, KernelKind::kStringSize, selection_mode_, nullable, cfg,
                                  &sk->size[v]));
    GDV_RETURN_NOT_OK(BuildKernel(*schema_, one, KernelKind::kStringWrite, selection_mode_, nullable, cfg,
                                  &sk->write[v]));
  }
  *size = sk->size[v].get();
  *write = sk->write[v].get();
  return Status::OK();
}

Status Projector::KernelFor(bool nullable, CompiledKernel** out) {
  if (rope_main_ != nullptr) return rope_main_->KernelFor(nullable, out);
  if (kernel_ == nullptr) return Status::Make(GDV_INVALID, "projector has no fixed-width output");
  if (nullable) {
    *out = kernel_.get();
    return Status::OK();
  }
  std::lock_guard<std::mutex> lock(mu_);
  if (kernel_nonull_ == nullptr)
    GDV_RETURN_NOT_OK(BuildKernel(*schema_, fixed_exprs_, KernelKind::kProject, selection_mode_, false,
                                  cfg_, &kernel_nonull_));
  *out = kernel_nonull_.get();
  return Status::OK();
}

// True when some column the kernel reads carries a validity bitmap, or is dictionary-encoded, a view
// column or a large column (a row is also null where its dictionary entry is, where its view is
// invalid, or where its length does not fit a gdv_str).
static bool AnyValidity(const GeneratedKernel& gen, const gdv_batch_t* batch) {
  for (const auto& slot : gen.inputs)
    if (slot.type.is_dict() || slot.type.is_view() || slot.type.is_large() || (slot.schema_index >= 0 && slot.schema_index < batch->num_columns &&
                                batch->columns[slot.schema_index].validity != nullptr))
      return true;
  return false;
}

namespace {
// Source + PTX of one kernel.  NVRTC's PTX text ends with a NUL: dropped, or a char* reader would stop there and
// lose every kernel after the first one.
std::string KernelText(const CompiledKernel& k) {
  std::string ptx = k.ptx;
  while (!ptx.empty() && ptx.back() == '\0') ptx.pop_back();
  return k.gen.source + (ptx.empty() ? "" : "\n// ---- PTX ----\n" + ptx);
}
}  // namespace

std::string Projector::DumpIR() const {
  if (rope_main_ != nullptr) return rope_pre_->DumpIR() + "\n" + rope_main_->DumpIR();
  std::string ir;
  if (kernel_ != nullptr) ir += KernelText(*kernel_);
  for (const auto& sk : strings_)
    for (const auto* k : {sk.size[0].get(), sk.write[0].get()})
      if (k != nullptr) ir += "\n" + KernelText(*k);
  return ir;
}

Status Projector::CheckEvaluateArgs(const gdv_batch_t* batch, const gdv_selection_t* sel,
                                    int64_t* n) const {
  if (batch == nullptr) return Status::Make(GDV_INVALID, "null argument");
  if (batch->num_columns != static_cast<int>(schema_->fields().size()))
    return Status::Make(GDV_INVALID, "RecordBatch schema must match the schema of Make()");
  if (batch->num_rows <= 0) return Status::Make(GDV_INVALID, "RecordBatch must be non-empty.");
  if (selection_mode_ != GDV_SEL_NONE) {
    if (sel == nullptr) return Status::Make(GDV_INVALID, "selection vector required by Make()");
    if (sel->mode != selection_mode_)
      return Status::Make(GDV_INVALID, "selection vector mode differs from the mode given to Make()");
    if (sel->mem_space != batch->mem_space)
      return Status::Make(GDV_INVALID, "selection vector and batch must share a memory space");
  } else if (sel != nullptr && sel->mode != GDV_SEL_NONE) {
    return Status::Make(GDV_INVALID, "projector was built without a selection vector mode");
  }
  *n = selection_mode_ != GDV_SEL_NONE ? sel->num_slots : batch->num_rows;
  if (*n < 0) return Status::Make(GDV_INVALID, "negative slot count");
  if (selection_mode_ != GDV_SEL_NONE && sel->d_num_slots != nullptr && batch->mem_space == GDV_MEM_HOST)
    return Status::Make(GDV_INVALID, "d_num_slots needs device buffers");
  return Status::OK();
}

namespace {
Status CheckFilterArgs(const gdv_batch_t* batch, const gdv_selection_t* out_sel) {
  if (batch->num_rows <= 0) return Status::Make(GDV_INVALID, "RecordBatch must be non-empty.");
  // GDV_SEL_BOUNDED: the caller sized the index buffer for the rows it expects to be selected
  // (row-range shards writing into a shared SelectionVector); rows past max_slots are counted
  // but not stored, so count > max_slots tells the caller that the vector overflowed.
  const bool bounded = (out_sel->mode & GDV_SEL_BOUNDED) != 0;
  const int sel_mode = out_sel->mode & ~GDV_SEL_BOUNDED;
  if (sel_mode < GDV_SEL_UINT16 || sel_mode > GDV_SEL_UINT64)
    return Status::Make(GDV_INVALID, "invalid selection vector mode");
  if (bounded && (batch->mem_space != GDV_MEM_DEVICE || out_sel->max_slots < 0))
    return Status::Make(GDV_INVALID, "a bounded selection vector needs device buffers");
  if (!bounded && out_sel->max_slots < batch->num_rows)
    return Status::Make(GDV_INVALID, "Selection vector max_slots " + std::to_string(out_sel->max_slots) +
                                         " is less than the number of rows " + std::to_string(batch->num_rows));
  if (out_sel->mem_space != batch->mem_space)
    return Status::Make(GDV_INVALID, "selection vector and batch must share a memory space");
  if (sel_mode == GDV_SEL_UINT16 && batch->num_rows > 65536)
    return Status::Make(GDV_INVALID, "batch too large for a uint16 selection vector");
  if (sel_mode == GDV_SEL_UINT32 && batch->num_rows > (int64_t(1) << 32))
    return Status::Make(GDV_INVALID, "batch too large for a uint32 selection vector");
  return Status::OK();
}
}  // namespace

// The two-stage rope plan sizes its temporaries on the host, synchronously, so it cannot take part in
// a chain that keeps the slot count on the device: its utf8/binary outputs refuse d_num_slots.  (Its
// fixed-width outputs have always accepted it, and still do.)  Host batches fall through to the
// "d_num_slots needs device buffers" of the evaluation itself.
Status Projector::RefuseDeviceCountWithRopeTemps(const gdv_batch_t* batch, const gdv_selection_t* sel) const {
  if (sel == nullptr || sel->mode == GDV_SEL_NONE || sel->d_num_slots == nullptr || batch->mem_space == GDV_MEM_HOST)
    return Status::OK();
  return Status::Make(GDV_NOT_IMPLEMENTED,
                      "d_num_slots: a utf8/binary output of a projector that materialises rope temporaries (the "
                      "two-stage rope plan) needs the slot count on the host; its temporaries are sized there");
}

Status Projector::OutputVarSize(const gdv_batch_t* batch, const gdv_selection_t* sel, int out_index,
                                void* stream, int64_t* bytes) {
  if (bytes == nullptr) return Status::Make(GDV_INVALID, "null argument");
  *bytes = 0;
  if (out_index < 0 || out_index >= num_outputs())
    return Status::Make(GDV_INVALID, "output index out of range");
  if (rope_main_ != nullptr) {
    if (batch == nullptr) return Status::Make(GDV_INVALID, "null argument");
    for (const auto& sk : rope_main_->strings_)
      if (sk.out_index == out_index) GDV_RETURN_NOT_OK(RefuseDeviceCountWithRopeTemps(batch, sel));
    return EvaluateOverTemps(rope_pre_.get(), batch, stream, [&](const gdv_batch_t* with_temps) {
      return rope_main_->OutputVarSize(with_temps, sel, out_index, stream, bytes);
    });
  }
  for (auto& sk : strings_)
    if (sk.out_index == out_index)
      return EvaluateString(&sk, batch, sel, nullptr, stream, false, true, bytes);
  return Status::OK();  // fixed-width output
}

// One utf8/binary output: sizing kernel -> tile scan -> (host: read the total, size the staging
// buffers) -> write kernel.  size_only stops after the scan and returns the total.
Status Projector::EvaluateString(StringKernels* sk, const gdv_batch_t* batch,
                                 const gdv_selection_t* sel, gdv_out_column_t* out, void* stream_v,
                                 bool async, bool size_only, int64_t* total_out) {
  int64_t n = 0;
  GDV_RETURN_NOT_OK(CheckEvaluateArgs(batch, sel, &n));
  const bool host = batch->mem_space == GDV_MEM_HOST;
  // Device slot count: n is only the upper bound the grids and the tile array are sized with; both
  // passes and the scan read the count on the device, and the scan checks the total against the
  // caller's var_capacity (the host never sees the total before the write pass).
  const bool dev_count = selection_mode_ != GDV_SEL_NONE && sel->d_num_slots != nullptr;
  Device* dev = nullptr;
  GDV_RETURN_NOT_OK(Device::Get(cfg_.device, &dev));
  CompiledKernel *ksize = nullptr, *kwrite = nullptr;
  GDV_RETURN_NOT_OK(StringKernelsFor(sk, AnyValidity(sk->size[0]->gen, batch), &ksize, &kwrite));
  CompiledKernel::Loaded lsize, lwrite;
  GDV_RETURN_NOT_OK(ksize->Load(dev, &lsize));
  GDV_RETURN_NOT_OK(kwrite->Load(dev, &lwrite));
  last_used_ = kwrite;
  const DriverApi& d = Driver();
  CUstream stream = stream_v != nullptr ? static_cast<CUstream>(stream_v) : dev->stream();
  const GeneratedKernel& gen = ksize->gen;  // both kernels read the same input slots
  // a large_string / large_binary output has int64 offsets and no 2^31 - 1 byte limit (code 2)
  const bool large_out = kwrite->gen.outputs.at(0).is_large();
  const size_t off_w = large_out ? 8 : 4;

  ScratchScope scratch(dev);
  scratch.Guard(stream);
  std::vector<ResolvedIn> ins;
  GDV_RETURN_NOT_OK(ResolveInputs(dev, gen, batch, stream, &scratch, &ins));
  const ArgsLayout& L = gen.args;
  std::vector<uint8_t> args(L.size, 0);
  Put<int64_t>(args, L.off_n, n);
  PutInputs(args, L, ins);
  if (selection_mode_ != GDV_SEL_NONE) GDV_RETURN_NOT_OK(PutSelection(dev, sel, n, host, stream, &scratch, L, args));
  if (dev_count && !size_only) {
    if (out == nullptr || out->values == nullptr) return Status::Make(GDV_INVALID, "output offsets buffer is null");
    if (out->var_capacity < 0) return Status::Make(GDV_INVALID, "negative var_capacity");
  }
  // [total u64][pad u64][one u64 per CTA tile]; lives until the stream is synchronised
  const int64_t T = gen.tile_rows;
  const int64_t n_tiles = (n + T - 1) / T;
  CUdeviceptr d_state = 0, d_err = 0;
  {
    auto pend = pending_.At(stream);
    GDV_RETURN_NOT_OK(dev->Alloc(16 + static_cast<size_t>(n_tiles) * 8, &d_state));
    pend->scratch.push_back(d_state);
    GDV_RETURN_NOT_OK(pend->ErrorBlock(dev, stream, &d_err));
    if (dev_count && !size_only) pend->var_checks.push_back({d_state, out->var_capacity, sk->out_index});
  }
  Put<CUdeviceptr>(args, L.off_err, d_err);
  Put<CUdeviceptr>(args, L.off_tile_state, d_state + 16);
  Put<CUdeviceptr>(args, L.off_out_count, d_state);
  const int64_t blocks_needed = std::max<int64_t>(1, n_tiles);
  GDV_RETURN_NOT_OK(LaunchKernel(dev, lsize, ksize->gen, args, GridFor(dev, cfg_, lsize.blocks_per_sm, blocks_needed),
                                 stream));
  {
    CUfunction scan = nullptr;
    GDV_RETURN_NOT_OK(dev->StaticFunction("gdv_scan_tiles", &scan));
    CUdeviceptr tiles = d_state + 16, total = d_state, errp = d_err;
    CUdeviceptr n_ptr = dev_count ? reinterpret_cast<CUdeviceptr>(sel->d_num_slots) : 0;
    int64_t nt = n_tiles, tile_rows = T;
    uint64_t offset_limit = large_out ? ~0ull : 0x7fffffffull;  // the largest total the output's offsets hold
    uint64_t limit = offset_limit;
    if (dev_count && !size_only) limit = std::min<uint64_t>(limit, static_cast<uint64_t>(out->var_capacity));
    void* params[] = {&tiles, &nt, &total, &errp, &limit, &n_ptr, &tile_rows, &offset_limit};
    g_launch_count.fetch_add(1);
    GDV_RETURN_NOT_OK(CuCheck(d.LaunchKernel(scan, 1, 1, 1, 1024, 1, 1, 0, stream, params, nullptr),
                              "cuLaunchKernel(gdv_scan_tiles)"));
  }
  uint64_t total = 0;
  if (size_only || host || !async) {
    GDV_RETURN_NOT_OK(CuCheck(d.MemcpyDtoHAsync(&total, d_state, 8, stream), "D2H total"));
    GDV_RETURN_NOT_OK(CuCheck(d.StreamSynchronize(stream), "cuStreamSynchronize"));
    if (!large_out && total > 0x7fffffffull) {
      Sync(stream);  // releases the pending blocks; reports the overflow below
      return Status::Make(GDV_EXECUTION_ERROR, ExecutionErrorMessage(2));
    }
    if (total_out != nullptr) *total_out = static_cast<int64_t>(total);
  }
  if (size_only) return Sync(stream);

  if (out == nullptr || out->values == nullptr)
    return Status::Make(GDV_INVALID, "output offsets buffer is null");
  const size_t words = static_cast<size_t>((n + 31) / 32);
  CUdeviceptr d_offs = reinterpret_cast<CUdeviceptr>(out->values);
  CUdeviceptr d_data = reinterpret_cast<CUdeviceptr>(out->var_data);
  CUdeviceptr d_vld = reinterpret_cast<CUdeviceptr>(out->validity);
  int64_t out_cap = out->var_capacity;
  if (host) {
    out->var_size = static_cast<int64_t>(total);
    if (static_cast<int64_t>(total) > out->var_capacity || (total > 0 && out->var_data == nullptr)) {
      Sync(stream);
      return Status::Make(GDV_INVALID, "var_data capacity " + std::to_string(out->var_capacity) +
                                           " is smaller than the " + std::to_string(total) +
                                           " bytes the output needs (see var_size)");
    }
    GDV_RETURN_NOT_OK(scratch.Alloc(static_cast<size_t>(n + 1) * off_w + 16, &d_offs));
    GDV_RETURN_NOT_OK(scratch.Alloc(static_cast<size_t>(total) + 16, &d_data));
    if (out->validity != nullptr) GDV_RETURN_NOT_OK(scratch.Alloc(words * 4 + 8, &d_vld));
    out_cap = static_cast<int64_t>(total);
  } else {
    out->var_size = async ? -1 : static_cast<int64_t>(total);
    if (out->var_data == nullptr && out->var_capacity > 0)
      return Status::Make(GDV_INVALID, "output var_data buffer is null");
  }
  Put<CUdeviceptr>(args, L.off_out_val, d_offs);
  Put<CUdeviceptr>(args, L.off_out_vld, d_vld);
  Put<CUdeviceptr>(args, L.off_out_var, d_data);
  Put<int64_t>(args, L.off_out_cap, out_cap);
  GDV_RETURN_NOT_OK(LaunchKernel(dev, lwrite, kwrite->gen, args, GridFor(dev, cfg_, lwrite.blocks_per_sm, blocks_needed),
                                 stream));
  if (host) {
    GDV_RETURN_NOT_OK(StagedDtoH(dev, out->values, d_offs, static_cast<size_t>(n + 1) * off_w, stream));
    if (total > 0) GDV_RETURN_NOT_OK(StagedDtoH(dev, out->var_data, d_data, static_cast<size_t>(total), stream));
    if (out->validity != nullptr)
      GDV_RETURN_NOT_OK(StagedDtoH(dev, out->validity, d_vld, static_cast<size_t>((n + 7) / 8), stream));
    // the staging blocks go back to the pool when `scratch` dies: wait for the copies first
    GDV_RETURN_NOT_OK(CuCheck(d.StreamSynchronize(stream), "cuStreamSynchronize"));
  }
  return Status::OK();
}

Status Projector::Evaluate(const gdv_batch_t* batch, const gdv_selection_t* sel,
                           gdv_out_column_t* all_outs, int n_all_outs, void* stream_v, bool async) {
  if (batch == nullptr || all_outs == nullptr) return Status::Make(GDV_INVALID, "null argument");
  if (n_all_outs != num_outputs())
    return Status::Make(GDV_INVALID, "expected " + std::to_string(num_outputs()) +
                                         " output columns, got " + std::to_string(n_all_outs));
  if (rope_main_ != nullptr) {
    if (batch->num_columns != static_cast<int>(schema_->fields().size()))
      return Status::Make(GDV_INVALID, "RecordBatch schema must match the schema of Make()");
    if (!rope_main_->strings_.empty()) GDV_RETURN_NOT_OK(RefuseDeviceCountWithRopeTemps(batch, sel));
    return EvaluateOverTemps(rope_pre_.get(), batch, stream_v, [&](const gdv_batch_t* with_temps) {
      return rope_main_->Evaluate(with_temps, sel, all_outs, n_all_outs, stream_v, async);
    });
  }
  int64_t n = 0;
  GDV_RETURN_NOT_OK(CheckEvaluateArgs(batch, sel, &n));
  const bool host = batch->mem_space == GDV_MEM_HOST;
  // utf8/binary outputs first (each runs its own kernel pair), then the fused fixed-width kernel
  for (auto& sk : strings_) {
    int64_t total = 0;
    GDV_RETURN_NOT_OK(EvaluateString(&sk, batch, sel, &all_outs[sk.out_index], stream_v, async, false,
                                     &total));
  }
  if (fixed_exprs_.empty()) {
    if (host || !async) return Sync(stream_v);
    return Status::OK();
  }
  std::vector<gdv_out_column_t> fixed_outs;
  for (int idx : fixed_idx_) fixed_outs.push_back(all_outs[idx]);
  gdv_out_column_t* outs = fixed_outs.data();
  const int n_outs = static_cast<int>(fixed_outs.size());

  Device* dev = nullptr;
  GDV_RETURN_NOT_OK(Device::Get(cfg_.device, &dev));
  CompiledKernel* kernel = nullptr;
  GDV_RETURN_NOT_OK(KernelFor(AnyValidity(kernel_->gen, batch), &kernel));
  last_used_ = kernel;
  CompiledKernel::Loaded l;
  GDV_RETURN_NOT_OK(kernel->Load(dev, &l));
  CUstream stream = stream_v != nullptr ? static_cast<CUstream>(stream_v) : dev->stream();
  const GeneratedKernel& gen = kernel->gen;

  const double t_begin = TraceOn() ? NowUs() : 0.0;
  ScratchScope scratch(dev);
  scratch.Guard(stream);
  std::vector<ResolvedIn> ins;
  GDV_RETURN_NOT_OK(ResolveInputs(dev, gen, batch, stream, &scratch, &ins));
  const double t_inputs = TraceOn() ? NowUs() : 0.0;

  const ArgsLayout& L = gen.args;
  std::vector<uint8_t> args(L.size, 0);
  Put<int64_t>(args, L.off_n, n);
  PutInputs(args, L, ins);
  if (selection_mode_ != GDV_SEL_NONE) GDV_RETURN_NOT_OK(PutSelection(dev, sel, n, host, stream, &scratch, L, args));
  // outputs
  struct OutStage {
    CUdeviceptr val = 0, vld = 0;
    size_t val_bytes = 0, vld_bytes = 0;
  };
  std::vector<OutStage> stage(n_outs);
  const size_t words = static_cast<size_t>((n + 31) / 32);
  for (int o = 0; o < n_outs; ++o) {
    const DataType& t = gen.outputs[o];
    if (outs[o].values == nullptr && n > 0)
      return Status::Make(GDV_INVALID, "output values buffer is null");
    OutStage& st = stage[o];
    st.val_bytes = t.is_bool() ? static_cast<size_t>((n + 7) / 8) : static_cast<size_t>(n) * t.width();
    st.vld_bytes = static_cast<size_t>((n + 7) / 8);
    if (host) {
      GDV_RETURN_NOT_OK(scratch.Alloc(t.is_bool() ? words * 4 + 8 : st.val_bytes + 16, &st.val));
      if (outs[o].validity != nullptr) GDV_RETURN_NOT_OK(scratch.Alloc(words * 4 + 8, &st.vld));
    } else {
      st.val = reinterpret_cast<CUdeviceptr>(outs[o].values);
      st.vld = reinterpret_cast<CUdeviceptr>(outs[o].validity);
    }
    Put<CUdeviceptr>(args, L.off_out_val + 8 * o, st.val);
    Put<CUdeviceptr>(args, L.off_out_vld + 8 * o, st.vld);
  }
  if (gen.uses_ctx) {
    CUdeviceptr d_err = 0;
    GDV_RETURN_NOT_OK(pending_.At(stream)->ErrorBlock(dev, stream, &d_err));
    Put<CUdeviceptr>(args, L.off_err, d_err);
  }

  const int R = gen.rows_per_thread, BT = gen.block_threads;
  const int64_t wtiles = (n + 32 * R - 1) / (32 * R);
  const int64_t blocks_needed = (wtiles + BT / 32 - 1) / (BT / 32);  // none for an empty selection
  GDV_RETURN_NOT_OK(LaunchKernel(dev, l, gen, args, GridFor(dev, cfg_, l.blocks_per_sm, blocks_needed), stream));

  if (host) {
    const double t_launch = TraceOn() ? NowUs() : 0.0;
    for (int o = 0; o < n_outs; ++o) {
      if (stage[o].val_bytes > 0)
        GDV_RETURN_NOT_OK(StagedDtoH(dev, outs[o].values, stage[o].val, stage[o].val_bytes, stream));
      if (outs[o].validity != nullptr && stage[o].vld_bytes > 0)
        GDV_RETURN_NOT_OK(StagedDtoH(dev, outs[o].validity, stage[o].vld, stage[o].vld_bytes, stream));
    }
    const double t_out = TraceOn() ? NowUs() : 0.0;
    Status st = Sync(stream);
    if (TraceOn())
      std::fprintf(stderr, "gdv trace: projector host batch %lld rows: inputs %.0f us, args+launch %.0f us, outputs %.0f us, "
                           "sync %.0f us\n", static_cast<long long>(n), t_inputs - t_begin, t_launch - t_inputs,
                   t_out - t_launch, NowUs() - t_out);
    return st;
  }
  if (!async) return Sync(stream);
  // async with device buffers: inputs were not staged, scratch holds nothing the kernel reads
  return Status::OK();
}

Status Projector::Sync(void* stream_v) {
  if (rope_main_ != nullptr) return rope_main_->Sync(stream_v);
  Device* dev = nullptr;
  GDV_RETURN_NOT_OK(Device::Get(cfg_.device, &dev));
  return pending_.Settle(dev, stream_v != nullptr ? static_cast<CUstream>(stream_v) : dev->stream(), nullptr);
}

// ======================================================================================
// Filter
// ======================================================================================
Status Filter::Make(SchemaPtr schema, ConditionPtr cond, const Config& cfg,
                    std::shared_ptr<Filter>* out) {
  if (schema == nullptr) return Status::Make(GDV_INVALID, "Schema cannot be null");
  if (cond == nullptr) return Status::Make(GDV_INVALID, "Condition cannot be null");
  const FunctionRegistry::Scope user_functions(cfg.functions.get());
  GDV_RETURN_NOT_OK(ValidateExpression(*schema, *cond));
  std::shared_ptr<Filter> f(new Filter());
  f->schema_ = schema;
  f->cond_ = cond;
  f->cfg_ = cfg;
  // The default Python/Cython path uses UINT32 indices: compile that variant eagerly so
  // Make() surfaces code-generation errors, as the reference does.
  CompiledKernel* k = nullptr;
  Status st = f->KernelFor(GDV_SEL_UINT32, true, false, &k);
  if (!st.ok()) {
    if (!IsRopeConsumerError(st)) return st;
    // something in the condition reads a rope: materialise the ropes first (gdv_rope_temps.h)
    RopeTemps rt;
    std::vector<ExpressionPtr> rewritten;
    const SchemaPtr extended = ExtractRopeTemps(schema, {cond}, &rt, &rewritten);
    if (rt.temps.empty()) return st;
    std::shared_ptr<Projector> pre;
    std::shared_ptr<Filter> main;
    Status two_stage = Projector::Make(schema, rt.temps, GDV_SEL_NONE, cfg, &pre);
    if (two_stage.ok())
      two_stage = Filter::Make(extended, std::make_shared<Condition>(rewritten[0]->root()), cfg, &main);
    if (two_stage.ok() && main->rope_main_ != nullptr) two_stage = st;
    if (!two_stage.ok()) return IsRopeConsumerError(two_stage) ? st : two_stage;  // another limit of the fuser: say that one
    f->rope_pre_ = std::move(pre);
    f->rope_main_ = std::move(main);
    *out = std::move(f);
    return Status::OK();
  }
  if (std::getenv("GDV_EAGER_NONULL") != nullptr)
    GDV_RETURN_NOT_OK(f->KernelFor(GDV_SEL_UINT32, false, true, &k));
  // A condition over one dictionary column that no null can satisfy: evaluate it once per entry
  // (a Projector over the dictionary) and keep rows by their index (DESIGN.md §3.6).
  const int dc = DictionaryFirstColumn(*schema, *cond->root());
  if (dc >= 0) {
    const Field& fd = schema->fields()[static_cast<size_t>(dc)];
    auto entries = std::make_shared<Schema>(std::vector<Field>{Field{fd.name, fd.type.value_type()}});
    NodePtr truth = std::make_shared<FunctionNode>("istrue", NodeVector{WithValueTypes(cond->root())}, boolean());
    GDV_RETURN_NOT_OK(Projector::Make(entries, {std::make_shared<Expression>(truth, Field{"keep", boolean()})},
                                      GDV_SEL_NONE, cfg, &f->dict_entries_));
    f->dict_column_ = dc;
  }
  *out = std::move(f);
  return Status::OK();
}

Status Filter::LaunchDictionaryFirst(Device* dev, const gdv_batch_t* batch, CUstream stream, bool async, bool large,
                                     CUdeviceptr d_bits, CUdeviceptr d_idx, int idx_width, CUdeviceptr d_count,
                                     CUdeviceptr d_state, int64_t n_tiles, int64_t row_base, int64_t out_cap,
                                     ScratchScope* scratch) {
  const bool host = batch->mem_space == GDV_MEM_HOST;
  const int64_t n = batch->num_rows;
  const gdv_column_t& c = batch->columns[dict_column_];
  const auto* dict = static_cast<const gdv_dictionary_t*>(c.var_data);
  if (dict == nullptr || dict->length < 0 || dict->offset < 0)
    return Status::Make(GDV_INVALID, "dictionary column " + std::to_string(dict_column_) +
                                         " has no valid dictionary (var_data must point at a gdv_dictionary_t)");
  const int64_t dlen = dict->length;
  const size_t words = static_cast<size_t>((dlen + 31) / 32);
  // 1. the condition over every entry: the dictionary is a one-column batch of its value type
  if (dlen > 0) {
    gdv_column_t dc;
    dc.validity = dict->validity;
    dc.values = dict->offsets;
    dc.var_data = dict->data;
    dc.offset = dict->offset;
    dc.var_data_size = dict->data_size;
    const gdv_batch_t db{dlen, 1, batch->mem_space, &dc};
    gdv_out_column_t out;
    std::memset(&out, 0, sizeof(out));
    std::vector<uint32_t> hbits;
    if (host) {
      hbits.assign(words + 2, 0u);
      out.values = hbits.data();
    } else {
      out.values = reinterpret_cast<void*>(d_bits);
    }
    GDV_RETURN_NOT_OK(dict_entries_->Evaluate(&db, nullptr, &out, 1, stream, !host && async));
    if (host) GDV_RETURN_NOT_OK(StagedHtoD(dev, d_bits, hbits.data(), words * 4, stream));
  }
  // 2. the rows: indices and their validity only
  const DataType it(schema_->fields()[static_cast<size_t>(dict_column_)].type.index);
  const int w = it.width();
  if (c.values == nullptr) return Status::Make(GDV_INVALID, "dictionary column has no indices buffer");
  CUdeviceptr d_in = 0, d_vld = 0;
  uint32_t vsh = 0;
  GDV_RETURN_NOT_OK(ResolveArray(dev, static_cast<const uint8_t*>(c.values) + c.offset * w, static_cast<size_t>(n) * w,
                                 16, w, host, stream, scratch, kIndicesMisaligned, dict_column_, &d_in));
  if (c.validity != nullptr)
    GDV_RETURN_NOT_OK(ResolveBitmap(dev, c.validity, c.offset, n, host, stream, scratch, &d_vld, &vsh));
  const std::string name = std::string("gdv_dict_filter_") + it.ctype() + (large ? "_w4" : "_w1");
  CUfunction fn = nullptr;
  GDV_RETURN_NOT_OK(dev->StaticFunction(name.c_str(), &fn));
  // the entry bitmap lives in shared memory up to 64 K entries (8 KB per CTA, DESIGN.md §3.6)
  int smem_words = dlen <= 65536 ? static_cast<int>(words) : 0;
  const size_t smem = static_cast<size_t>(smem_words) * 4;
  const DriverApi& d = Driver();
  int per_sm = 1;
  if (d.OccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, fn, 256, smem) != CUDA_SUCCESS || per_sm < 1) per_sm = 1;
  const unsigned grid = GridFor(dev, cfg_, per_sm, std::max<int64_t>(1, n_tiles));
  CUdeviceptr tile_state = d_state + 16, ticket = d_state;
  int64_t nn = n, rb = row_base, oc = out_cap, dl = dlen;
  int ow = idx_width;
  void* params[] = {&d_in, &d_vld, &vsh, &d_bits, &dl, &smem_words, &nn, &rb, &d_idx, &ow, &d_count, &tile_state, &ticket, &oc};
  g_launch_count.fetch_add(1);
  return CuCheck(d.LaunchKernel(fn, grid, 1, 1, 256, 1, 1, static_cast<unsigned>(smem), stream, params, nullptr),
                 "cuLaunchKernel(gdv_dict_filter)");
}

Status Filter::KernelFor(int mode, bool nullable, bool large, CompiledKernel** out) {
  if (rope_main_ != nullptr) return rope_main_->KernelFor(mode, nullable, large, out);
  std::lock_guard<std::mutex> lock(mu_);
  const int key = mode * 4 + (nullable ? 1 : 0) + (large ? 2 : 0);
  auto it = kernels_.find(key);
  if (it == kernels_.end()) {
    std::unique_ptr<CompiledKernel> k;
    std::vector<ExpressionPtr> exprs = {cond_};
    // Big batches want big tiles (few look-back descriptors), small ones enough tiles to occupy the
    // 132 SMs: the fuser picks block size and chunks per warp from this flag (GenerateKeyFilter,
    // GenerateFilter and FitStages in gdv_codegen.cc).
    Config cfg = cfg_;
    cfg.large_batch = large;
    GDV_RETURN_NOT_OK(BuildKernel(*schema_, exprs, KernelKind::kFilter, mode, nullable, cfg, &k));
    it = kernels_.emplace(key, std::move(k)).first;
  }
  *out = it->second.get();
  return Status::OK();
}

std::string Filter::DumpIR() const {
  if (rope_main_ != nullptr) return rope_pre_->DumpIR() + "\n" + rope_main_->DumpIR();
  std::lock_guard<std::mutex> lock(mu_);
  auto it = kernels_.find(GDV_SEL_UINT32 * 4 + 1);
  if (it == kernels_.end()) return "";
  return KernelText(*it->second);
}

Status Filter::Evaluate(const gdv_batch_t* batch, gdv_selection_t* out_sel, void* stream_v,
                        bool async, void* d_count_user) {
  if (batch == nullptr || out_sel == nullptr) return Status::Make(GDV_INVALID, "null argument");
  if (batch->num_columns != static_cast<int>(schema_->fields().size()))
    return Status::Make(GDV_INVALID, "RecordBatch schema must match the schema of Make()");
  if (rope_main_ != nullptr) {
    return EvaluateOverTemps(rope_pre_.get(), batch, stream_v, [&](const gdv_batch_t* with_temps) {
      return rope_main_->Evaluate(with_temps, out_sel, stream_v, async, d_count_user);
    });
  }
  GDV_RETURN_NOT_OK(CheckFilterArgs(batch, out_sel));
  const bool bounded = (out_sel->mode & GDV_SEL_BOUNDED) != 0;
  const int sel_mode = out_sel->mode & ~GDV_SEL_BOUNDED;
  const int64_t n = batch->num_rows;
  const bool host = batch->mem_space == GDV_MEM_HOST;

  Device* dev = nullptr;
  GDV_RETURN_NOT_OK(Device::Get(cfg_.device, &dev));
  const bool large = batch->num_rows >= (int64_t(32) << 20);
  const bool dict_first = dict_entries_ != nullptr;
  dict_first_used_ = dict_first;
  CompiledKernel* kernel = nullptr;
  CompiledKernel::Loaded l;
  if (!dict_first) {
    CompiledKernel* general = nullptr;
    GDV_RETURN_NOT_OK(KernelFor(GDV_SEL_UINT32, true, false, &general));
    GDV_RETURN_NOT_OK(KernelFor(sel_mode, AnyValidity(general->gen, batch), large, &kernel));
    last_used_ = kernel;
    GDV_RETURN_NOT_OK(kernel->Load(dev, &l));
  }
  const DriverApi& d = Driver();
  CUstream stream = stream_v != nullptr ? static_cast<CUstream>(stream_v) : dev->stream();

  ScratchScope scratch(dev);
  scratch.Guard(stream);
  std::vector<ResolvedIn> ins;
  if (!dict_first) GDV_RETURN_NOT_OK(ResolveInputs(dev, kernel->gen, batch, stream, &scratch, &ins));

  // Row tiles: ceil(n / tile_rows) look-back descriptors (the dictionary-first kernel: 8 warps x W
  // 1024-row chunks, W = 4 on big batches like the fused filter's).
  const int64_t tile_rows = dict_first ? int64_t(8 * 1024) * (large ? 4 : 1) : kernel->gen.tile_rows;
  const int64_t n_tiles = (n + tile_rows - 1) / tile_rows;

  // Per-stream persistent scratch: [ticket u64][count u64][tile_state n_tiles x u64]
  const size_t state_bytes = 16 + static_cast<size_t>(n_tiles) * 8;
  CUdeviceptr d_state = 0, d_err = 0, d_bits = 0;
  {
    auto pend = pending_.At(stream);
    if (pend->state_cap < state_bytes) {
      // earlier blocks stay alive until Sync(): launches still queued may be using them
      GDV_RETURN_NOT_OK(dev->Alloc(state_bytes, &pend->d_state));
      pend->scratch.push_back(pend->d_state);
      pend->state_cap = state_bytes;
    }
    d_state = pend->d_state;
    if (dict_first) {
      const auto* dict = static_cast<const gdv_dictionary_t*>(batch->columns[dict_column_].var_data);
      const int64_t dlen = dict != nullptr ? dict->length : 0;
      const size_t bits_bytes = static_cast<size_t>(std::max<int64_t>(dlen, 0) + 31) / 32 * 4 + 16;
      if (pend->bits_cap < bits_bytes) {
        GDV_RETURN_NOT_OK(dev->Alloc(bits_bytes, &pend->d_bits));
        pend->scratch.push_back(pend->d_bits);
        pend->bits_cap = bits_bytes;
      }
      d_bits = pend->d_bits;
    }
    if (!dict_first && kernel->gen.uses_ctx) GDV_RETURN_NOT_OK(pend->ErrorBlock(dev, stream, &d_err));
    pend->d_count = d_count_user != nullptr ? reinterpret_cast<CUdeviceptr>(d_count_user) : d_state + 8;
  }
  GDV_RETURN_NOT_OK(CuCheck(d.MemsetD8Async(d_state, 0, state_bytes, stream), "memset tile state"));
  CUdeviceptr d_count = d_state + 8;
  if (d_count_user != nullptr) {
    d_count = reinterpret_cast<CUdeviceptr>(d_count_user);
    GDV_RETURN_NOT_OK(CuCheck(d.MemsetD8Async(d_count, 0, 8, stream), "memset count"));
  }

  CUdeviceptr d_idx = reinterpret_cast<CUdeviceptr>(out_sel->indices);
  const int iw = SelWidth(sel_mode);
  if (host) GDV_RETURN_NOT_OK(scratch.Alloc(static_cast<size_t>(n) * iw + 16, &d_idx));

  if (dict_first) {
    GDV_RETURN_NOT_OK(LaunchDictionaryFirst(dev, batch, stream, async, large, d_bits, d_idx, iw, d_count, d_state, n_tiles,
                                            out_sel->index_base, bounded ? out_sel->max_slots : n, &scratch));
  } else {
    const GeneratedKernel& gen = kernel->gen;
    const ArgsLayout& L = gen.args;
    std::vector<uint8_t> args(L.size, 0);
    Put<int64_t>(args, L.off_n, n);
    Put<int64_t>(args, L.off_row_base, out_sel->index_base);
    Put<CUdeviceptr>(args, L.off_out_idx, d_idx);
    Put<CUdeviceptr>(args, L.off_out_count, d_count);
    Put<CUdeviceptr>(args, L.off_tile_state, d_state + 16);
    Put<CUdeviceptr>(args, L.off_ticket, d_state);
    Put<CUdeviceptr>(args, L.off_err, d_err);
    Put<int64_t>(args, L.off_out_cap, bounded ? out_sel->max_slots : n);
    PutInputs(args, L, ins);
    GDV_RETURN_NOT_OK(LaunchKernel(dev, l, gen, args, GridFor(dev, cfg_, l.blocks_per_sm, std::max<int64_t>(1, n_tiles)),
                                   stream));
  }

  out_sel->num_slots = -1;
  if (host) {
    int64_t count = 0;
    GDV_RETURN_NOT_OK(Sync(stream, &count));
    if (count > 0) {
      GDV_RETURN_NOT_OK(StagedDtoH(dev, out_sel->indices, d_idx, static_cast<size_t>(count) * iw, stream));
      GDV_RETURN_NOT_OK(CuCheck(d.StreamSynchronize(stream), "cuStreamSynchronize"));
    }
    out_sel->num_slots = count;
    return Status::OK();
  }
  if (!async) {
    int64_t count = 0;
    GDV_RETURN_NOT_OK(Sync(stream, &count));
    out_sel->num_slots = count;
  }
  return Status::OK();
}

Status Filter::Sync(void* stream_v, int64_t* num_slots) {
  if (rope_main_ != nullptr) return rope_main_->Sync(stream_v, num_slots);
  Device* dev = nullptr;
  GDV_RETURN_NOT_OK(Device::Get(cfg_.device, &dev));
  return pending_.Settle(dev, stream_v != nullptr ? static_cast<CUstream>(stream_v) : dev->stream(), num_slots);
}

}  // namespace gdv
