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
    GDV_RETURN_NOT_OK(
        CuCheck(d.StreamCreate(&dev->copy_stream_, CU_STREAM_NON_BLOCKING), "cuStreamCreate"));
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
    std::vector<CUdeviceptr> drop;
    {
      std::lock_guard<std::mutex> lock(mu_);
      for (auto& kv : free_) {
        drop.push_back(kv.second);
        sizes_.erase(kv.second);
      }
      free_.clear();
      idle_bytes_ = 0;
    }
    for (auto q : drop) Driver().MemFree(q);
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
  std::vector<CUdeviceptr> drop;
  {
    std::lock_guard<std::mutex> lock(mu_);
    auto it = sizes_.find(p);
    if (it == sizes_.end()) return;
    free_.emplace(it->second, p);
    idle_bytes_ += it->second;
    // over the limit: the largest idle blocks go back to the driver (cuMemFree waits for work that
    // still uses a block, so releasing one that a queued kernel reads is safe, only slow)
    while (idle_bytes_ > pool_limit_ && !free_.empty()) {
      auto big = std::prev(free_.end());
      idle_bytes_ -= big->first;
      sizes_.erase(big->second);
      drop.push_back(big->second);
      free_.erase(big);
    }
  }
  if (!drop.empty() && MakeCurrent().ok())
    for (auto q : drop) Driver().MemFree(q);
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
  spec.large_batch = cfg.large_batch;
  const std::string placeholder = std::string(KernelPrefix(kind)) + "PLACEHOLDER";
  spec.name = placeholder;
  std::unique_ptr<CompiledKernel> k(new CompiledKernel());
  GDV_RETURN_NOT_OK(GenerateKernel(schema, exprs, spec, &k->gen));
  // Compile for the device we will run on when one is visible, else for H100.
  std::string arch = "sm_90a";
  Device* dev = nullptr;
  if (Driver().loaded && Device::Get(cfg.device, &dev).ok()) arch = dev->arch();
  // name the kernel after its own text
  char hex[24];
  std::snprintf(hex, sizeof(hex), "%016llx", static_cast<unsigned long long>(Fnv1a(arch, Fnv1a(k->gen.source))));
  const std::string name = std::string(KernelPrefix(kind)) + hex;
  for (size_t pos = 0; (pos = k->gen.source.find(placeholder, pos)) != std::string::npos;)
    k->gen.source.replace(pos, placeholder.size(), name);
  k->gen.name = name;
  // the device function library is part of every translation unit: its text is part of the key, so a
  // persisted cubin can never outlive the library it was compiled against
  static const uint64_t lib_hash = Fnv1a(std::string(gdv_device_lib_text, static_cast<size_t>(gdv_device_lib_text_len)));
  char lib_hex[24];
  std::snprintf(lib_hex, sizeof(lib_hex), "%016llx", static_cast<unsigned long long>(lib_hash));
  const std::string key = arch + (cfg.optimize ? "|O3|" : "|O0|") + (cfg.dump_ir ? "ptx|" : "|") + lib_hex + "|" + k->gen.source;
  std::shared_ptr<const CachedCubin> hit;
  {
    std::lock_guard<std::mutex> lock(g_cache_mu);
    auto it = g_cubin_cache.find(key);
    if (it != g_cubin_cache.end()) hit = it->second;
  }
  // GDV_CUBIN_CACHE_DIR=<dir>: cubins also persist across processes (the counterpart of the
  // reference's object-code cache): <dir>/<fnv64 of arch|options|source>.cubin, written atomically.
  std::string disk_path;
  if (const char* cdir = std::getenv("GDV_CUBIN_CACHE_DIR")) {
    if (!cfg.dump_ir) {  // DumpIR wants the PTX too: always compile
      char kh[24];
      std::snprintf(kh, sizeof(kh), "%016llx", static_cast<unsigned long long>(Fnv1a(key)));
      disk_path = std::string(cdir) + "/" + kh + ".cubin";
    }
  }
  if (hit == nullptr && !disk_path.empty()) {
    if (FILE* f = std::fopen(disk_path.c_str(), "rb")) {
      std::vector<char> blob;
      char buf[65536];
      size_t got;
      while ((got = std::fread(buf, 1, sizeof(buf), f)) > 0) blob.insert(blob.end(), buf, buf + got);
      std::fclose(f);
      const bool elf = blob.size() > 4 && blob[0] == 0x7f && blob[1] == 'E' && blob[2] == 'L' && blob[3] == 'F';
      if (elf && std::search(blob.begin(), blob.end(), name.begin(), name.end()) != blob.end()) {
        auto entry = std::make_shared<CachedCubin>();
        entry->cubin = std::move(blob);
        hit = entry;
        std::lock_guard<std::mutex> lock(g_cache_mu);
        if (g_cubin_cache.size() >= kCubinCacheEntries) g_cubin_cache.clear();
        g_cubin_cache.emplace(key, entry);
      }
    }
  }
  if (hit != nullptr) {
    k->cubin = hit->cubin;
    k->ptx = hit->ptx;
    k->compile_log = hit->log;
  } else {
    g_compile_count.fetch_add(1);
    GDV_RETURN_NOT_OK(CompileToCubin(k->gen.source, arch, cfg.optimize, cfg.dump_ir, &k->cubin,
                                     &k->ptx, &k->compile_log));
    const bool elf_out = k->cubin.size() > 4 && k->cubin[0] == 0x7f && k->cubin[1] == 'E';
    if (!disk_path.empty() && elf_out) {
      const std::string tmp = disk_path + ".tmp" + std::to_string(static_cast<long long>(::getpid()));
      if (FILE* f = std::fopen(tmp.c_str(), "wb")) {
        const bool ok = std::fwrite(k->cubin.data(), 1, k->cubin.size(), f) == k->cubin.size();
        std::fclose(f);
        if (ok) std::rename(tmp.c_str(), disk_path.c_str());
        else std::remove(tmp.c_str());
      }
    }
    // a translation unit can compile "successfully" without the kernel in it (e.g. when the
    // front end stops at a stray byte): make that a code-generation error here, not a missing
    // symbol at the first Evaluate on a GPU
    if (std::search(k->cubin.begin(), k->cubin.end(), name.begin(), name.end()) == k->cubin.end())
      return Status::Make(GDV_CODEGEN_ERROR, "NVRTC produced a module without the kernel " + name);
    auto entry = std::make_shared<CachedCubin>();
    entry->cubin = k->cubin;
    entry->ptx = k->ptx;
    entry->log = k->compile_log;
    std::lock_guard<std::mutex> lock(g_cache_mu);
    if (g_cubin_cache.size() >= kCubinCacheEntries) g_cubin_cache.clear();
    g_cubin_cache.emplace(key, std::move(entry));
  }
  // GDV_DUMP_DIR=<dir>: write <kernel>.cu / <kernel>.cubin for offline SASS inspection
  // (cuobjdump -sass) and so that ncu's source page can find the generated code.
  if (const char* dir = std::getenv("GDV_DUMP_DIR")) {
    const std::string base = std::string(dir) + "/" + k->gen.name;
    if (FILE* f = std::fopen((base + ".cu").c_str(), "w")) {
      std::fwrite(k->gen.source.data(), 1, k->gen.source.size(), f);
      std::fclose(f);
    }
    if (FILE* f = std::fopen((base + ".cubin").c_str(), "wb")) {
      std::fwrite(k->cubin.data(), 1, k->cubin.size(), f);
      std::fclose(f);
    }
  }
  *out = std::move(k);
  return Status::OK();
}

// One kernel input after staging: device addresses + bit shifts.
struct ResolvedIn {
  CUdeviceptr val = 0, vld = 0, var = 0;
  uint32_t vsh = 0, dsh = 0;
};

inline int64_t BitBytes(int64_t bit_begin, int64_t nbits) {
  // bytes that cover bits [bit_begin, bit_begin + nbits) counted from the byte of bit_begin
  return ((bit_begin & 7) + nbits + 7) / 8;
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
    const gdv_column_t& c = batch->columns[slot.schema_index];
    ResolvedIn r;
    const int64_t off = c.offset;
    const DataType& t = slot.type;
    if (c.values == nullptr && n > 0)
      return Status::Make(GDV_INVALID, "column " + std::to_string(slot.schema_index) +
                                           " has no values buffer");
    // ---- validity
    // Bitmaps reach the kernel as a 4-byte aligned word pointer plus a bit shift in [0, 31].
    if (c.validity != nullptr) {
      const uint8_t* p = static_cast<const uint8_t*>(c.validity) + (off >> 3);
      r.vsh = static_cast<uint32_t>(off & 7);
      if (host) {
        const size_t bytes = static_cast<size_t>(BitBytes(off, n));
        CUdeviceptr dp;
        GDV_RETURN_NOT_OK(scratch->Alloc(bytes + 8, &dp));
        GDV_RETURN_NOT_OK(StagedHtoD(dev, dp, p, bytes, stream));
        r.vld = dp;
      } else {
        const uintptr_t mis = reinterpret_cast<uintptr_t>(p) & 3u;
        r.vld = reinterpret_cast<CUdeviceptr>(p - mis);
        r.vsh += static_cast<uint32_t>(8 * mis);
      }
    }
    // ---- values
    if (t.is_bool()) {
      const uint8_t* p = static_cast<const uint8_t*>(c.values) + (off >> 3);
      r.dsh = static_cast<uint32_t>(off & 7);
      if (host) {
        const size_t bytes = static_cast<size_t>(BitBytes(off, n));
        CUdeviceptr dp;
        GDV_RETURN_NOT_OK(scratch->Alloc(bytes + 8, &dp));
        GDV_RETURN_NOT_OK(StagedHtoD(dev, dp, p, bytes, stream));
        r.val = dp;
      } else {
        const uintptr_t mis = reinterpret_cast<uintptr_t>(p) & 3u;
        r.val = reinterpret_cast<CUdeviceptr>(p - mis);
        r.dsh += static_cast<uint32_t>(8 * mis);
      }
    } else if (t.is_varlen()) {
      const int32_t* offs = static_cast<const int32_t*>(c.values) + off;
      if (host) {
        const size_t obytes = static_cast<size_t>(n + 1) * 4;
        CUdeviceptr dp;
        GDV_RETURN_NOT_OK(scratch->Alloc(obytes, &dp));
        GDV_RETURN_NOT_OK(StagedHtoD(dev, dp, offs, obytes, stream));
        r.val = dp;
        const int64_t first = n > 0 ? offs[0] : 0, last = n > 0 ? offs[n] : 0;
        const size_t vbytes = static_cast<size_t>(last - first);
        CUdeviceptr dv;
        GDV_RETURN_NOT_OK(scratch->Alloc(vbytes + 16, &dv));
        if (vbytes > 0)
          GDV_RETURN_NOT_OK(StagedHtoD(dev, dv, static_cast<const uint8_t*>(c.var_data) + first, vbytes, stream));
        // kernel addresses bytes as var + offs[r]; rebase so offs[0] lands on dv
        r.var = dv - static_cast<CUdeviceptr>(first);
      } else {
        r.val = reinterpret_cast<CUdeviceptr>(offs);
        r.var = reinterpret_cast<CUdeviceptr>(c.var_data);
      }
    } else {
      const int w = t.width();
      const uint8_t* p = static_cast<const uint8_t*>(c.values) + off * w;
      if (host) {
        const size_t bytes = static_cast<size_t>(n) * w;
        CUdeviceptr dp;
        GDV_RETURN_NOT_OK(scratch->Alloc(bytes + 16, &dp));
        if (bytes > 0)
          GDV_RETURN_NOT_OK(StagedHtoD(dev, dp, p, bytes, stream));
        r.val = dp;
      } else {
        if (reinterpret_cast<uintptr_t>(p) % static_cast<uintptr_t>(w) != 0)
          return Status::Make(GDV_INVALID, "device values buffer of column " +
                                               std::to_string(slot.schema_index) +
                                               " is not aligned to its element width");
        r.val = reinterpret_cast<CUdeviceptr>(p);
      }
    }
    (*out)[j] = r;
  }
  return Status::OK();
}

template <typename T>
void Put(std::vector<uint8_t>& buf, size_t off, T v) {
  std::memcpy(buf.data() + off, &v, sizeof(T));
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

}  // namespace

// ======================================================================================
// Projector
// ======================================================================================
Status Projector::Make(SchemaPtr schema, std::vector<ExpressionPtr> exprs, int selection_mode,
                       const Config& cfg, std::shared_ptr<Projector>* out) {
  if (schema == nullptr) return Status::Make(GDV_INVALID, "Schema cannot be null");
  if (exprs.empty()) return Status::Make(GDV_INVALID, "Expressions cannot be empty");
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
SchemaPtr ExtendedSchema(const SchemaPtr& schema, const RopeTemps& rt) {
  std::vector<Field> fields = schema->fields();
  fields.insert(fields.end(), rt.fields.begin(), rt.fields.end());
  return std::make_shared<Schema>(std::move(fields));
}
}  // namespace

Status Projector::MakeWithRopeTemps(const SchemaPtr& schema, const std::vector<ExpressionPtr>& exprs,
                                    int selection_mode, const Config& cfg, Projector* into) {
  RopeTemps rt;
  std::vector<ExpressionPtr> rewritten;
  for (const auto& e : exprs) {
    NodePtr r;
    ExtractRopes(e->root(), e->result().type.is_varlen(), &rt, &r);
    rewritten.push_back(std::make_shared<Expression>(r, e->result()));
  }
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
  GDV_RETURN_NOT_OK(Projector::Make(ExtendedSchema(schema, rt), rewritten, selection_mode, cfg, &main));
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

namespace {
// The temps of a device batch go back to the pool when TempColumns dies: not before the work that reads them.
Status WaitForStream(int device, void* stream_v) {
  Device* dev = nullptr;
  GDV_RETURN_NOT_OK(Device::Get(device, &dev));
  CUstream stream = stream_v != nullptr ? static_cast<CUstream>(stream_v) : dev->stream();
  return CuCheck(Driver().StreamSynchronize(stream), "cuStreamSynchronize");
}
}  // namespace

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

// True when some column the kernel reads carries a validity bitmap.
static bool AnyValidity(const GeneratedKernel& gen, const gdv_batch_t* batch) {
  for (const auto& slot : gen.inputs)
    if (slot.schema_index >= 0 && slot.schema_index < batch->num_columns &&
        batch->columns[slot.schema_index].validity != nullptr)
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
  return Status::OK();
}

Status Projector::OutputVarSize(const gdv_batch_t* batch, const gdv_selection_t* sel, int out_index,
                                void* stream, int64_t* bytes) {
  if (bytes == nullptr) return Status::Make(GDV_INVALID, "null argument");
  *bytes = 0;
  if (out_index < 0 || out_index >= num_outputs())
    return Status::Make(GDV_INVALID, "output index out of range");
  if (rope_main_ != nullptr) {
    if (batch == nullptr) return Status::Make(GDV_INVALID, "null argument");
    TempColumns tc;
    GDV_RETURN_NOT_OK(tc.Build(rope_pre_.get(), batch, stream));
    return rope_main_->OutputVarSize(&tc.batch, sel, out_index, stream, bytes);  // synchronous: reads the total back
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
  if (sel != nullptr && sel->d_num_slots != nullptr)
    return Status::Make(GDV_NOT_IMPLEMENTED, "utf8/binary outputs need the slot count on the host (d_num_slots is for fixed-width outputs)");
  const bool host = batch->mem_space == GDV_MEM_HOST;
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

  ScratchScope scratch(dev);
  scratch.Guard(stream);
  std::vector<ResolvedIn> ins;
  GDV_RETURN_NOT_OK(ResolveInputs(dev, gen, batch, stream, &scratch, &ins));
  ArgsLayout L(static_cast<int>(gen.inputs.size()), 1);
  std::vector<uint8_t> args(L.size, 0);
  Put<int64_t>(args, L.off_n, n);
  for (size_t j = 0; j < ins.size(); ++j) {
    Put<CUdeviceptr>(args, L.off_in_val + 8 * j, ins[j].val);
    Put<CUdeviceptr>(args, L.off_in_vld + 8 * j, ins[j].vld);
    Put<CUdeviceptr>(args, L.off_in_var + 8 * j, ins[j].var);
    Put<uint32_t>(args, L.off_in_vsh + 4 * j, ins[j].vsh);
    Put<uint32_t>(args, L.off_in_dsh + 4 * j, ins[j].dsh);
  }
  if (selection_mode_ != GDV_SEL_NONE) {
    CUdeviceptr dsel = reinterpret_cast<CUdeviceptr>(sel->indices);
    if (host) {
      const size_t bytes = static_cast<size_t>(n) * SelWidth(selection_mode_);
      GDV_RETURN_NOT_OK(scratch.Alloc(bytes + 16, &dsel));
      if (bytes > 0)
        GDV_RETURN_NOT_OK(StagedHtoD(dev, dsel, sel->indices, bytes, stream));
    }
    Put<CUdeviceptr>(args, L.off_sel, dsel);
  }
  // [total u64][pad u64][one u64 per CTA tile]; lives until the stream is synchronised
  const int64_t T = gen.tile_rows;
  const int64_t n_tiles = (n + T - 1) / T;
  CUdeviceptr d_state = 0, d_err = 0;
  {
    std::lock_guard<std::mutex> lock(mu_);
    Pending& pend = pending_[stream];
    pend.dev = dev;
    GDV_RETURN_NOT_OK(dev->Alloc(16 + static_cast<size_t>(n_tiles) * 8, &d_state));
    pend.scratch.push_back(d_state);
    if (pend.d_err == 0) {
      pend.uses_ctx = true;
      GDV_RETURN_NOT_OK(dev->Alloc(256, &pend.d_err));
      GDV_RETURN_NOT_OK(CuCheck(d.MemsetD8Async(pend.d_err, 0, 256, stream), "memset err"));
    }
    d_err = pend.d_err;
  }
  Put<CUdeviceptr>(args, L.off_err, d_err);
  Put<CUdeviceptr>(args, L.off_tile_state, d_state + 16);
  Put<CUdeviceptr>(args, L.off_out_count, d_state);
  const int64_t cap_blocks =
      static_cast<int64_t>(std::max(1, dev->sm_count() - cfg_.sm_reserve)) * lsize.blocks_per_sm;
  unsigned grid = static_cast<unsigned>(std::max<int64_t>(1, std::min<int64_t>(n_tiles, cap_blocks)));
  GDV_RETURN_NOT_OK(LaunchKernel(dev, lsize, ksize->gen, args, grid, stream));
  {
    CUfunction scan = nullptr;
    GDV_RETURN_NOT_OK(dev->StaticFunction("gdv_scan_tiles", &scan));
    CUdeviceptr tiles = d_state + 16, total = d_state, errp = d_err;
    int64_t nt = n_tiles;
    uint64_t limit = 0x7fffffffull;
    void* params[] = {&tiles, &nt, &total, &errp, &limit};
    g_launch_count.fetch_add(1);
    GDV_RETURN_NOT_OK(CuCheck(d.LaunchKernel(scan, 1, 1, 1, 1024, 1, 1, 0, stream, params, nullptr),
                              "cuLaunchKernel(gdv_scan_tiles)"));
  }
  uint64_t total = 0;
  if (size_only || host || !async) {
    GDV_RETURN_NOT_OK(CuCheck(d.MemcpyDtoHAsync(&total, d_state, 8, stream), "D2H total"));
    GDV_RETURN_NOT_OK(CuCheck(d.StreamSynchronize(stream), "cuStreamSynchronize"));
    if (total > 0x7fffffffull) {
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
    GDV_RETURN_NOT_OK(scratch.Alloc(static_cast<size_t>(n + 1) * 4 + 16, &d_offs));
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
  const int64_t cap_w =
      static_cast<int64_t>(std::max(1, dev->sm_count() - cfg_.sm_reserve)) * lwrite.blocks_per_sm;
  grid = static_cast<unsigned>(std::max<int64_t>(1, std::min<int64_t>(n_tiles, cap_w)));
  GDV_RETURN_NOT_OK(LaunchKernel(dev, lwrite, kwrite->gen, args, grid, stream));
  if (host) {
    GDV_RETURN_NOT_OK(StagedDtoH(dev, out->values, d_offs, static_cast<size_t>(n + 1) * 4, stream));
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
    TempColumns tc;
    GDV_RETURN_NOT_OK(tc.Build(rope_pre_.get(), batch, stream_v));
    Status st = rope_main_->Evaluate(&tc.batch, sel, all_outs, n_all_outs, stream_v, async);
    if (batch->mem_space != GDV_MEM_HOST) {
      const Status w = WaitForStream(cfg_.device, stream_v);
      if (st.ok()) st = w;
    }
    return st;
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
  const DriverApi& d = Driver();
  CUstream stream = stream_v != nullptr ? static_cast<CUstream>(stream_v) : dev->stream();
  const GeneratedKernel& gen = kernel->gen;

  const double t_begin = TraceOn() ? NowUs() : 0.0;
  ScratchScope scratch(dev);
  scratch.Guard(stream);
  std::vector<ResolvedIn> ins;
  GDV_RETURN_NOT_OK(ResolveInputs(dev, gen, batch, stream, &scratch, &ins));
  const double t_inputs = TraceOn() ? NowUs() : 0.0;

  ArgsLayout L(static_cast<int>(gen.inputs.size()), n_outs);
  std::vector<uint8_t> args(L.size, 0);
  Put<int64_t>(args, L.off_n, n);
  for (size_t j = 0; j < ins.size(); ++j) {
    Put<CUdeviceptr>(args, L.off_in_val + 8 * j, ins[j].val);
    Put<CUdeviceptr>(args, L.off_in_vld + 8 * j, ins[j].vld);
    Put<CUdeviceptr>(args, L.off_in_var + 8 * j, ins[j].var);
    Put<uint32_t>(args, L.off_in_vsh + 4 * j, ins[j].vsh);
    Put<uint32_t>(args, L.off_in_dsh + 4 * j, ins[j].dsh);
  }
  // selection vector
  if (selection_mode_ != GDV_SEL_NONE) {
    CUdeviceptr dsel = reinterpret_cast<CUdeviceptr>(sel->indices);
    if (host) {
      const size_t bytes = static_cast<size_t>(n) * SelWidth(selection_mode_);
      GDV_RETURN_NOT_OK(scratch.Alloc(bytes + 16, &dsel));
      if (bytes > 0)
        GDV_RETURN_NOT_OK(StagedHtoD(dev, dsel, sel->indices, bytes, stream));
    }
    Put<CUdeviceptr>(args, L.off_sel, dsel);
    if (sel->d_num_slots != nullptr) {
      if (host) return Status::Make(GDV_INVALID, "d_num_slots needs device buffers");
      Put<CUdeviceptr>(args, L.off_n_ptr, reinterpret_cast<CUdeviceptr>(sel->d_num_slots));
    }
  }
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
  // error flag
  CUdeviceptr d_err = 0;
  if (gen.uses_ctx) {
    std::lock_guard<std::mutex> lock(mu_);
    Pending& pend = pending_[stream];
    if (pend.d_err == 0) {
      pend.dev = dev;
      pend.uses_ctx = true;
      GDV_RETURN_NOT_OK(dev->Alloc(256, &pend.d_err));
      GDV_RETURN_NOT_OK(CuCheck(d.MemsetD8Async(pend.d_err, 0, 256, stream), "memset err"));
    }
    d_err = pend.d_err;
    Put<CUdeviceptr>(args, L.off_err, d_err);
  }

  const int R = gen.rows_per_thread, BT = gen.block_threads;
  const int64_t wtiles = (n + 32 * R - 1) / (32 * R);
  const int64_t blocks_needed = (wtiles + BT / 32 - 1) / (BT / 32);
  const int64_t cap =
      static_cast<int64_t>(std::max(1, dev->sm_count() - cfg_.sm_reserve)) * l.blocks_per_sm;
  const unsigned grid = static_cast<unsigned>(std::min<int64_t>(blocks_needed, cap));
  GDV_RETURN_NOT_OK(LaunchKernel(dev, l, gen, args, grid, stream));

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
  CUstream stream = stream_v != nullptr ? static_cast<CUstream>(stream_v) : dev->stream();
  const DriverApi& d = Driver();
  Pending pend;
  bool have = false;
  {
    std::lock_guard<std::mutex> lock(mu_);
    auto it = pending_.find(stream);
    if (it != pending_.end()) {
      pend = it->second;
      pending_.erase(it);
      have = true;
    }
  }
  int err = 0;
  Status copy = Status::OK();
  if (have && pend.d_err != 0) copy = CuCheck(d.MemcpyDtoHAsync(&err, pend.d_err, sizeof(int), stream), "D2H err");
  Status s = CuCheck(d.StreamSynchronize(stream), "cuStreamSynchronize");
  if (have) {  // on every path: the pending blocks go back to the pool once the stream is idle
    if (pend.d_err != 0) dev->Free(pend.d_err);
    for (auto p : pend.scratch) dev->Free(p);
  }
  GDV_RETURN_NOT_OK(copy);
  GDV_RETURN_NOT_OK(s);
  if (err != 0) return Status::Make(GDV_EXECUTION_ERROR, ExecutionErrorMessage(err));
  return Status::OK();
}

// ======================================================================================
// Filter
// ======================================================================================
Status Filter::Make(SchemaPtr schema, ConditionPtr cond, const Config& cfg,
                    std::shared_ptr<Filter>* out) {
  if (schema == nullptr) return Status::Make(GDV_INVALID, "Schema cannot be null");
  if (cond == nullptr) return Status::Make(GDV_INVALID, "Condition cannot be null");
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
    NodePtr r;
    ExtractRopes(cond->root(), false, &rt, &r);
    if (rt.temps.empty()) return st;
    std::shared_ptr<Projector> pre;
    std::shared_ptr<Filter> main;
    Status two_stage = Projector::Make(schema, rt.temps, GDV_SEL_NONE, cfg, &pre);
    if (two_stage.ok()) two_stage = Filter::Make(ExtendedSchema(schema, rt), std::make_shared<Condition>(r), cfg, &main);
    if (two_stage.ok() && main->rope_main_ != nullptr) two_stage = st;
    if (!two_stage.ok()) return IsRopeConsumerError(two_stage) ? st : two_stage;  // another limit of the fuser: say that one
    f->rope_pre_ = std::move(pre);
    f->rope_main_ = std::move(main);
    *out = std::move(f);
    return Status::OK();
  }
  if (std::getenv("GDV_EAGER_NONULL") != nullptr)
    GDV_RETURN_NOT_OK(f->KernelFor(GDV_SEL_UINT32, false, true, &k));
  *out = std::move(f);
  return Status::OK();
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
    // 132 SMs: the fuser picks block size and chunks per warp from this flag (GenerateKernelImpl).
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
    TempColumns tc;
    GDV_RETURN_NOT_OK(tc.Build(rope_pre_.get(), batch, stream_v));
    Status st = rope_main_->Evaluate(&tc.batch, out_sel, stream_v, async, d_count_user);
    if (batch->mem_space != GDV_MEM_HOST) {
      const Status w = WaitForStream(cfg_.device, stream_v);
      if (st.ok()) st = w;
    }
    return st;
  }
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
    return Status::Make(GDV_INVALID, "Selection vector max_slots " +
                                         std::to_string(out_sel->max_slots) +
                                         " is less than the number of rows " +
                                         std::to_string(batch->num_rows));
  if (out_sel->mem_space != batch->mem_space)
    return Status::Make(GDV_INVALID, "selection vector and batch must share a memory space");
  const int64_t n = batch->num_rows;
  if (sel_mode == GDV_SEL_UINT16 && n > 65536)
    return Status::Make(GDV_INVALID, "batch too large for a uint16 selection vector");
  if (sel_mode == GDV_SEL_UINT32 && n > (int64_t(1) << 32))
    return Status::Make(GDV_INVALID, "batch too large for a uint32 selection vector");
  const bool host = batch->mem_space == GDV_MEM_HOST;

  Device* dev = nullptr;
  GDV_RETURN_NOT_OK(Device::Get(cfg_.device, &dev));
  CompiledKernel* general = nullptr;
  GDV_RETURN_NOT_OK(KernelFor(GDV_SEL_UINT32, true, false, &general));
  CompiledKernel* kernel = nullptr;
  const bool large = batch->num_rows >= (int64_t(32) << 20);
  GDV_RETURN_NOT_OK(
      KernelFor(sel_mode, AnyValidity(general->gen, batch), large, &kernel));
  last_used_ = kernel;
  CompiledKernel::Loaded l;
  GDV_RETURN_NOT_OK(kernel->Load(dev, &l));
  const DriverApi& d = Driver();
  CUstream stream = stream_v != nullptr ? static_cast<CUstream>(stream_v) : dev->stream();
  const GeneratedKernel& gen = kernel->gen;

  ScratchScope scratch(dev);
  scratch.Guard(stream);
  std::vector<ResolvedIn> ins;
  GDV_RETURN_NOT_OK(ResolveInputs(dev, gen, batch, stream, &scratch, &ins));

  // Row tiles: ceil(n / tile_rows) look-back descriptors.
  const int64_t tile_rows = gen.tile_rows;
  const int64_t n_tiles = (n + tile_rows - 1) / tile_rows;

  // Per-stream persistent scratch: [ticket u64][count u64][tile_state n_tiles x u64]
  const size_t state_bytes = 16 + static_cast<size_t>(n_tiles) * 8;
  CUdeviceptr d_state = 0, d_err = 0;
  {
    std::lock_guard<std::mutex> lock(mu_);
    Pending& pend = pending_[stream];
    pend.dev = dev;
    if (pend.state_cap < state_bytes) {
      // earlier blocks stay alive until Sync(): launches still queued may be using them
      GDV_RETURN_NOT_OK(dev->Alloc(state_bytes, &pend.d_state));
      pend.scratch.push_back(pend.d_state);
      pend.state_cap = state_bytes;
    }
    d_state = pend.d_state;
    if (gen.uses_ctx) {
      if (pend.d_err == 0) {
        GDV_RETURN_NOT_OK(dev->Alloc(256, &pend.d_err));
        GDV_RETURN_NOT_OK(CuCheck(d.MemsetD8Async(pend.d_err, 0, 256, stream), "memset err"));
        pend.uses_ctx = true;
      }
      d_err = pend.d_err;
    }
    pend.d_count = d_count_user != nullptr ? reinterpret_cast<CUdeviceptr>(d_count_user)
                                           : d_state + 8;
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

  ArgsLayout L(static_cast<int>(gen.inputs.size()), 0);
  std::vector<uint8_t> args(L.size, 0);
  Put<int64_t>(args, L.off_n, n);
  Put<int64_t>(args, L.off_row_base, out_sel->index_base);
  Put<CUdeviceptr>(args, L.off_out_idx, d_idx);
  Put<CUdeviceptr>(args, L.off_out_count, d_count);
  Put<CUdeviceptr>(args, L.off_tile_state, d_state + 16);
  Put<CUdeviceptr>(args, L.off_ticket, d_state);
  Put<CUdeviceptr>(args, L.off_err, d_err);
  Put<int64_t>(args, L.off_out_cap, bounded ? out_sel->max_slots : n);
  for (size_t j = 0; j < ins.size(); ++j) {
    Put<CUdeviceptr>(args, L.off_in_val + 8 * j, ins[j].val);
    Put<CUdeviceptr>(args, L.off_in_vld + 8 * j, ins[j].vld);
    Put<CUdeviceptr>(args, L.off_in_var + 8 * j, ins[j].var);
    Put<uint32_t>(args, L.off_in_vsh + 4 * j, ins[j].vsh);
    Put<uint32_t>(args, L.off_in_dsh + 4 * j, ins[j].dsh);
  }
  const int64_t cap =
      static_cast<int64_t>(std::max(1, dev->sm_count() - cfg_.sm_reserve)) * l.blocks_per_sm;
  const unsigned grid = static_cast<unsigned>(std::max<int64_t>(1, std::min<int64_t>(n_tiles, cap)));
  GDV_RETURN_NOT_OK(LaunchKernel(dev, l, gen, args, grid, stream));

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
  CUstream stream = stream_v != nullptr ? static_cast<CUstream>(stream_v) : dev->stream();
  const DriverApi& d = Driver();
  Pending pend;
  bool have = false;
  {
    std::lock_guard<std::mutex> lock(mu_);
    auto it = pending_.find(stream);
    if (it != pending_.end()) {
      pend = it->second;
      pending_.erase(it);
      have = true;
    }
  }
  int err = 0;
  uint64_t count = 0;
  Status copy = Status::OK();
  if (have && pend.d_err != 0) copy = CuCheck(d.MemcpyDtoHAsync(&err, pend.d_err, sizeof(int), stream), "D2H err");
  if (copy.ok() && have && pend.d_count != 0)
    copy = CuCheck(d.MemcpyDtoHAsync(&count, pend.d_count, sizeof(count), stream), "D2H count");
  Status s = CuCheck(d.StreamSynchronize(stream), "cuStreamSynchronize");
  if (have) {  // on every path: the pending blocks go back to the pool once the stream is idle
    if (pend.d_err != 0) dev->Free(pend.d_err);
    for (auto p : pend.scratch) dev->Free(p);
  }
  GDV_RETURN_NOT_OK(copy);
  GDV_RETURN_NOT_OK(s);
  if (err != 0) return Status::Make(GDV_EXECUTION_ERROR, ExecutionErrorMessage(err));
  if (num_slots != nullptr) *num_slots = have ? static_cast<int64_t>(count) : -1;
  return Status::OK();
}

}  // namespace gdv
