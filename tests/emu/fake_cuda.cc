// fake_cuda.cc — TEST INFRASTRUCTURE: a functional stand-in for libcuda.so.1 so that the whole,
// unmodified product stack (C-ABI -> runtime -> driver calls -> generated kernels) can be
// exercised on a box without a GPU.  Built to tests/emu/lib/libcuda.so.1 and put in front of the
// real driver with LD_LIBRARY_PATH by tests/test_emu.py only; see tests/emu/README.md.
//
// "Device memory" is host memory, streams execute synchronously at enqueue time, and
// cuLaunchKernel runs the grid one CTA at a time with every CUDA thread as a ucontext fiber
// (tests/emu/gdv_emu.h has the device-side half).  A module is either the blob fake_nvrtc.cc
// returns ("GDVEMU1\0<path of a host-compiled .so>") or, for any other image (the embedded
// static-kernel cubin), the host build of device/static_kernels.cu (libgdv_emu_static.so).
#include <cuda.h>
#include <dlfcn.h>
#include <ucontext.h>
#include <unistd.h>

#include <algorithm>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <mutex>
#include <string>
#include <vector>

struct gdv_emu_uint3 {
  unsigned x, y, z;
};
struct gdv_emu_thread {
  gdv_emu_uint3 tid, bid, bdim, gdim;
  void* dyn_smem;
  unsigned lane, warp;
};

extern "C" gdv_emu_thread* gdv_emu_cur;

namespace {

constexpr size_t kStackBytes = 256 * 1024;

struct WarpSync {
  unsigned arrived = 0, gen = 0;
  unsigned long long vals[32];
  unsigned long long snap[32];
};
struct CtaRun;
struct Fiber {
  ucontext_t ctx;
  gdv_emu_thread th;
  CtaRun* cta = nullptr;
  bool done = false;
};
// One resident CTA.  Several may be resident at once (GDV_EMU_CTAS): each runs its own copy of the
// kernel's shared object, because `__shared__` variables are function-local statics there.
struct CtaRun {
  std::vector<Fiber> fibers;
  std::vector<WarpSync> warps;
  std::vector<char*> stacks;
  unsigned live = 0, bar_arrived = 0, bar_gen = 0;
  void (*entry)(void**) = nullptr;
  void** params = nullptr;
  void* dyn_smem = nullptr;
  bool active = false;
};
ucontext_t g_sched;
std::recursive_mutex g_mu;
int g_resident_ctas = 1;   // GDV_EMU_CTAS: CTAs resident at once (> 1 exercises look-back waits)
int g_sched_policy = 0;    // GDV_EMU_SCHED: 0 = lowest CTA first, 1 = highest CTA first, 2 = xorshift

struct Module {
  std::vector<void*> handles;  // [0] the shared object, [i] private copies for concurrently resident CTAs
  std::string path;
};
struct Function {
  std::vector<void (*)(void**)> entries;  // one per copy
  std::string name;
  int max_dyn_smem = 48 * 1024;
};

Fiber* CurFiber() {
  return reinterpret_cast<Fiber*>(reinterpret_cast<char*>(gdv_emu_cur) - offsetof(Fiber, th));
}

}  // namespace

extern "C" {
gdv_emu_thread* gdv_emu_cur = nullptr;

void gdv_emu_yield() {
  Fiber* f = CurFiber();
  swapcontext(&f->ctx, &g_sched);
}

void gdv_emu_syncthreads() {
  CtaRun* c = CurFiber()->cta;
  const unsigned my = c->bar_gen;
  if (++c->bar_arrived >= c->live) {
    c->bar_arrived = 0;
    ++c->bar_gen;
    return;
  }
  while (c->bar_gen == my) gdv_emu_yield();
}

void gdv_emu_warp_gather(unsigned mask, unsigned long long v, unsigned long long* out) {
  CtaRun* c = CurFiber()->cta;
  gdv_emu_thread* t = gdv_emu_cur;
  WarpSync& w = c->warps[t->warp];
  if (((mask >> t->lane) & 1u) == 0u) {
    std::fprintf(stderr, "gdv_emu: lane %u calls a warp collective with mask %08x\n", t->lane, mask);
    std::abort();
  }
  w.vals[t->lane] = v;
  w.arrived |= 1u << t->lane;
  const unsigned my = w.gen;
  if (w.arrived == mask) {
    for (int l = 0; l < 32; ++l) w.snap[l] = ((mask >> l) & 1u) ? w.vals[l] : 0ull;
    w.arrived = 0;
    ++w.gen;
  } else {
    if ((w.arrived & ~mask) != 0u) {
      std::fprintf(stderr, "gdv_emu: warp collective with diverging masks\n");
      std::abort();
    }
    while (w.gen == my) gdv_emu_yield();
  }
  std::memcpy(out, w.snap, sizeof(w.snap));
}
}

namespace {

void FiberEntry() {
  Fiber* f = CurFiber();
  CtaRun* c = f->cta;
  c->entry(c->params);
  f->done = true;
  --c->live;
  // a thread that exits no longer takes part in CTA barriers: release one that is now complete
  if (c->live > 0 && c->bar_arrived >= c->live) {
    c->bar_arrived = 0;
    ++c->bar_gen;
  }
  swapcontext(&f->ctx, &g_sched);
}

void StartCta(CtaRun* cta, void (*entry)(void**), void** params, const gdv_emu_uint3& bid,
              const gdv_emu_uint3& bdim, const gdv_emu_uint3& gdim, size_t smem) {
  const unsigned nthreads = bdim.x * bdim.y * bdim.z;
  cta->fibers.assign(nthreads, Fiber());
  cta->warps.assign((nthreads + 31) / 32, WarpSync());
  cta->live = nthreads;
  cta->bar_arrived = 0;
  cta->bar_gen = 0;
  cta->entry = entry;
  cta->params = params;
  cta->active = true;
  while (cta->stacks.size() < nthreads) cta->stacks.push_back(static_cast<char*>(std::malloc(kStackBytes)));
  std::memset(cta->dyn_smem, 0xA5, smem + 1024);  // shared memory starts undefined
  for (unsigned i = 0; i < nthreads; ++i) {
    Fiber& f = cta->fibers[i];
    f.cta = cta;
    f.th.tid = {i % bdim.x, (i / bdim.x) % bdim.y, i / (bdim.x * bdim.y)};
    f.th.bid = bid;
    f.th.bdim = bdim;
    f.th.gdim = gdim;
    f.th.dyn_smem = cta->dyn_smem;
    f.th.lane = i & 31u;
    f.th.warp = i >> 5;
    getcontext(&f.ctx);
    f.ctx.uc_stack.ss_sp = cta->stacks[i];
    f.ctx.uc_stack.ss_size = kStackBytes;
    f.ctx.uc_link = &g_sched;
    makecontext(&f.ctx, FiberEntry, 0);
  }
}

std::vector<CtaRun*> g_slots;  // reused across launches (stacks are expensive)

// Runs the grid with up to `resident` CTAs at a time; CTA i uses copy (slot index) of the kernel.
bool RunGrid(Function* fn, const gdv_emu_uint3& gdim, const gdv_emu_uint3& bdim, size_t smem, void** params) {
  const unsigned long long total = 1ull * gdim.x * gdim.y * gdim.z;
  const unsigned resident = static_cast<unsigned>(
      std::min<unsigned long long>(total, std::min<size_t>(fn->entries.size(), static_cast<size_t>(g_resident_ctas))));
  while (g_slots.size() < resident) g_slots.push_back(new CtaRun());
  for (unsigned s = 0; s < resident; ++s) {
    std::free(g_slots[s]->dyn_smem);
    g_slots[s]->dyn_smem = nullptr;
    if (posix_memalign(&g_slots[s]->dyn_smem, 1024, smem + 1024) != 0) return false;
    g_slots[s]->active = false;
  }
  unsigned long long next = 0, finished = 0, idle_rounds = 0, rng = 0x9E3779B97F4A7C15ull;
  auto bid_of = [&](unsigned long long i) {
    return gdv_emu_uint3{static_cast<unsigned>(i % gdim.x), static_cast<unsigned>((i / gdim.x) % gdim.y),
                         static_cast<unsigned>(i / (1ull * gdim.x * gdim.y))};
  };
  while (finished < total) {
    for (unsigned s = 0; s < resident; ++s)
      if (!g_slots[s]->active && next < total) {
        StartCta(g_slots[s], fn->entries[s], params, bid_of(next), bdim, gdim, smem);
        ++next;
      }
    bool progressed = false;
    for (unsigned k = 0; k < resident; ++k) {
      unsigned s = k;
      if (g_sched_policy == 1) s = resident - 1 - k;
      else if (g_sched_policy == 2) {
        rng ^= rng << 13; rng ^= rng >> 7; rng ^= rng << 17;
        s = static_cast<unsigned>(rng % resident);
      }
      CtaRun* cta = g_slots[s];
      if (!cta->active) continue;
      const unsigned live_before = cta->live, gen_before = cta->bar_gen;
      for (Fiber& f : cta->fibers) {
        if (f.done) continue;
        gdv_emu_cur = &f.th;
        swapcontext(&g_sched, &f.ctx);
      }
      if (cta->live != live_before || cta->bar_gen != gen_before) progressed = true;
      if (cta->live == 0) {
        cta->active = false;
        ++finished;
        progressed = true;
      }
    }
    // crude hang detector: no thread exits and no CTA barrier completes for a very long time
    if (!progressed) {
      if (++idle_rounds > 200'000ull) {
        std::fprintf(stderr, "gdv_emu: kernel %s appears to hang\n", fn->name.c_str());
        gdv_emu_cur = nullptr;
        return false;
      }
    } else {
      idle_rounds = 0;
    }
  }
  gdv_emu_cur = nullptr;
  return true;
}

int g_device_count = 1;
int g_sm_count = 4;

}  // namespace

#define EMU_OK return CUDA_SUCCESS

extern "C" {

CUresult cuInit(unsigned int) {
  if (const char* e = std::getenv("GDV_EMU_DEVICES")) g_device_count = std::atoi(e);
  if (const char* e = std::getenv("GDV_EMU_SMS")) g_sm_count = std::atoi(e);
  if (const char* e = std::getenv("GDV_EMU_CTAS")) g_resident_ctas = std::max(1, std::atoi(e));
  if (const char* e = std::getenv("GDV_EMU_SCHED")) g_sched_policy = std::atoi(e);
  EMU_OK;
}
CUresult cuDeviceGetCount(int* n) { *n = g_device_count; EMU_OK; }
CUresult cuDeviceGet(CUdevice* d, int ordinal) {
  if (ordinal < 0 || ordinal >= g_device_count) return CUDA_ERROR_INVALID_DEVICE;
  *d = ordinal;
  EMU_OK;
}
CUresult cuDeviceGetAttribute(int* v, CUdevice_attribute a, CUdevice) {
  switch (a) {
    case CU_DEVICE_ATTRIBUTE_MULTIPROCESSOR_COUNT: *v = g_sm_count; break;
    case CU_DEVICE_ATTRIBUTE_COMPUTE_CAPABILITY_MAJOR: *v = 9; break;
    case CU_DEVICE_ATTRIBUTE_COMPUTE_CAPABILITY_MINOR: *v = 0; break;
    case CU_DEVICE_ATTRIBUTE_MAX_SHARED_MEMORY_PER_BLOCK_OPTIN: *v = 227 * 1024; break;
    case CU_DEVICE_ATTRIBUTE_WARP_SIZE: *v = 32; break;
    default: *v = 0; break;
  }
  EMU_OK;
}
CUresult cuDevicePrimaryCtxRetain(CUcontext* c, CUdevice d) {
  *c = reinterpret_cast<CUcontext>(static_cast<uintptr_t>(0x1000 + d));
  EMU_OK;
}
CUresult cuCtxSetCurrent(CUcontext) { EMU_OK; }
CUresult cuCtxGetCurrent(CUcontext* c) { *c = reinterpret_cast<CUcontext>(static_cast<uintptr_t>(0x1000)); EMU_OK; }

// allocations are padded on both sides: the staged loaders legitimately read a few bytes around a
// column (16-byte aligned windows), which is inside the allocation granule on a real device
constexpr size_t kPad = 512;
static std::map<uintptr_t, size_t> g_allocs;
CUresult cuMemAlloc_v2(CUdeviceptr* p, size_t n) {
  std::lock_guard<std::recursive_mutex> lock(g_mu);
  void* raw = nullptr;
  if (posix_memalign(&raw, 512, n + 2 * kPad) != 0) return CUDA_ERROR_OUT_OF_MEMORY;
  std::memset(raw, 0xCD, n + 2 * kPad);  // garbage, like a fresh device allocation
  const uintptr_t user = reinterpret_cast<uintptr_t>(raw) + kPad;
  g_allocs[user] = n;
  *p = static_cast<CUdeviceptr>(user);
  EMU_OK;
}
// Guard bands: the kPad bytes on either side of every allocation keep their 0xCD fill unless a
// kernel (or a copy) wrote out of bounds.  Checked after every launch and at free.
static bool GuardsIntact(const char* when) {
  bool ok = true;
  for (const auto& kv : g_allocs) {
    const unsigned char* lo = reinterpret_cast<const unsigned char*>(kv.first - kPad);
    const unsigned char* hi = reinterpret_cast<const unsigned char*>(kv.first + kv.second);
    for (size_t i = 0; i < kPad; ++i) {
      if (lo[i] != 0xCD || hi[i] != 0xCD) {
        std::fprintf(stderr, "gdv_emu: out-of-bounds WRITE detected %s: allocation of %zu bytes at %p, guard byte %s%zu\n",
                     when, kv.second, reinterpret_cast<void*>(kv.first), lo[i] != 0xCD ? "-" : "+",
                     lo[i] != 0xCD ? kPad - i : i);
        ok = false;
        break;
      }
    }
  }
  return ok;
}
CUresult cuMemFree_v2(CUdeviceptr p) {
  std::lock_guard<std::recursive_mutex> lock(g_mu);
  if (p == 0) EMU_OK;
  auto it = g_allocs.find(static_cast<uintptr_t>(p));
  if (it == g_allocs.end()) return CUDA_ERROR_INVALID_VALUE;
  if (!GuardsIntact("at cuMemFree")) return CUDA_ERROR_ILLEGAL_ADDRESS;
  g_allocs.erase(it);
  std::free(reinterpret_cast<void*>(static_cast<uintptr_t>(p) - kPad));
  EMU_OK;
}
CUresult cuMemGetAddressRange_v2(CUdeviceptr* base, size_t* size, CUdeviceptr p) {
  std::lock_guard<std::recursive_mutex> lock(g_mu);
  auto it = g_allocs.upper_bound(static_cast<uintptr_t>(p));
  if (it == g_allocs.begin()) return CUDA_ERROR_INVALID_VALUE;
  --it;
  if (static_cast<uintptr_t>(p) >= it->first + it->second) return CUDA_ERROR_INVALID_VALUE;
  if (base) *base = static_cast<CUdeviceptr>(it->first);
  if (size) *size = it->second;
  EMU_OK;
}
// pinned ranges, so cuPointerGetAttribute can tell them from pageable memory like the driver does
static std::mutex g_pinned_mu;
static std::map<uintptr_t, size_t> g_pinned;
CUresult cuMemHostAlloc(void** p, size_t n, unsigned int) {
  *p = std::malloc(n ? n : 1);
  if (*p == nullptr) return CUDA_ERROR_OUT_OF_MEMORY;
  std::lock_guard<std::mutex> g(g_pinned_mu);
  g_pinned[reinterpret_cast<uintptr_t>(*p)] = n ? n : 1;
  return CUDA_SUCCESS;
}
CUresult cuMemFreeHost(void* p) {
  {
    std::lock_guard<std::mutex> g(g_pinned_mu);
    g_pinned.erase(reinterpret_cast<uintptr_t>(p));
  }
  std::free(p);
  EMU_OK;
}
CUresult cuMemcpyHtoDAsync_v2(CUdeviceptr d, const void* s, size_t n, CUstream) {
  std::memcpy(reinterpret_cast<void*>(d), s, n);
  EMU_OK;
}
CUresult cuMemcpyDtoHAsync_v2(void* d, CUdeviceptr s, size_t n, CUstream) {
  std::memcpy(d, reinterpret_cast<const void*>(s), n);
  EMU_OK;
}
CUresult cuMemcpyDtoDAsync_v2(CUdeviceptr d, CUdeviceptr s, size_t n, CUstream) {
  std::memmove(reinterpret_cast<void*>(d), reinterpret_cast<const void*>(s), n);
  EMU_OK;
}
CUresult cuMemsetD8Async(CUdeviceptr d, unsigned char v, size_t n, CUstream) {
  std::memset(reinterpret_cast<void*>(d), v, n);
  EMU_OK;
}
CUresult cuStreamCreate(CUstream* s, unsigned int) {
  static uintptr_t next = 0x2000;
  *s = reinterpret_cast<CUstream>(next += 16);
  EMU_OK;
}
CUresult cuStreamSynchronize(CUstream) { EMU_OK; }
CUresult cuStreamDestroy_v2(CUstream) { EMU_OK; }
CUresult cuStreamWaitEvent(CUstream, CUevent, unsigned int) { EMU_OK; }
CUresult cuEventCreate(CUevent* e, unsigned int) {
  static uintptr_t next = 0x3000;
  *e = reinterpret_cast<CUevent>(next += 16);
  EMU_OK;
}
CUresult cuEventRecord(CUevent, CUstream) { EMU_OK; }
CUresult cuEventSynchronize(CUevent) { EMU_OK; }
CUresult cuEventDestroy_v2(CUevent) { EMU_OK; }

// A private copy of the shared object: dlopen of a different path gives different statics.
static void* OpenCopy(const std::string& path, int copy) {
  if (copy == 0) return dlopen(path.c_str(), RTLD_NOW | RTLD_LOCAL);
  const std::string cp = path + ".c" + std::to_string(copy) + ".so";
  if (access(cp.c_str(), R_OK) != 0) {
    const std::string tmp = cp + ".tmp" + std::to_string(getpid());
    FILE* in = std::fopen(path.c_str(), "rb");
    FILE* out = std::fopen(tmp.c_str(), "wb");
    if (in == nullptr || out == nullptr) return nullptr;
    char buf[65536];
    size_t n;
    while ((n = std::fread(buf, 1, sizeof(buf), in)) > 0) std::fwrite(buf, 1, n, out);
    std::fclose(in);
    std::fclose(out);
    std::rename(tmp.c_str(), cp.c_str());
  }
  return dlopen(cp.c_str(), RTLD_NOW | RTLD_LOCAL);
}
CUresult cuModuleLoadData(CUmodule* m, const void* image) {
  std::lock_guard<std::recursive_mutex> lock(g_mu);
  std::string path;
  if (std::memcmp(image, "GDVEMU1", 8) == 0) {
    path = static_cast<const char*>(image) + 8;
  } else {
    const char* s = std::getenv("GDV_EMU_STATIC_LIB");
    if (s == nullptr) return CUDA_ERROR_INVALID_IMAGE;
    path = s;
  }
  Module* mod = new Module();
  mod->path = path;
  for (int c = 0; c < g_resident_ctas; ++c) {
    void* h = OpenCopy(path, c);
    if (h == nullptr) {
      std::fprintf(stderr, "gdv_emu: dlopen(%s, copy %d): %s\n", path.c_str(), c, dlerror());
      delete mod;
      return CUDA_ERROR_INVALID_IMAGE;
    }
    mod->handles.push_back(h);
  }
  *m = reinterpret_cast<CUmodule>(mod);
  EMU_OK;
}
CUresult cuModuleUnload(CUmodule m) {
  delete reinterpret_cast<Module*>(m);  // the objects stay mapped: kernels keep function-local statics
  EMU_OK;
}
CUresult cuModuleGetFunction(CUfunction* f, CUmodule m, const char* name) {
  Module* mod = reinterpret_cast<Module*>(m);
  const std::string tramp = std::string(name) + "__emu";
  Function* fn = new Function();
  for (void* h : mod->handles) {
    void* p = dlsym(h, tramp.c_str());
    if (p == nullptr) {
      delete fn;
      return CUDA_ERROR_NOT_FOUND;
    }
    fn->entries.push_back(reinterpret_cast<void (*)(void**)>(p));
  }
  fn->name = name;
  *f = reinterpret_cast<CUfunction>(fn);
  EMU_OK;
}
CUresult cuFuncGetAttribute(int* v, CUfunction_attribute a, CUfunction) {
  switch (a) {
    case CU_FUNC_ATTRIBUTE_NUM_REGS: *v = 32; break;
    case CU_FUNC_ATTRIBUTE_MAX_THREADS_PER_BLOCK: *v = 1024; break;
    default: *v = 0; break;
  }
  EMU_OK;
}
CUresult cuFuncSetAttribute(CUfunction f, CUfunction_attribute a, int v) {
  if (a == CU_FUNC_ATTRIBUTE_MAX_DYNAMIC_SHARED_SIZE_BYTES) {
    if (v > 227 * 1024) return CUDA_ERROR_INVALID_VALUE;
    reinterpret_cast<Function*>(f)->max_dyn_smem = v;
  }
  EMU_OK;
}
CUresult cuOccupancyMaxActiveBlocksPerMultiprocessor(int* n, CUfunction, int block, size_t smem) {
  int by_threads = 2048 / (block > 0 ? block : 1);
  int by_smem = smem > 0 ? static_cast<int>((227 * 1024) / smem) : 32;
  *n = by_threads < by_smem ? by_threads : by_smem;
  if (*n > 32) *n = 32;
  EMU_OK;
}
CUresult cuLaunchKernel(CUfunction f, unsigned gx, unsigned gy, unsigned gz, unsigned bx, unsigned by,
                        unsigned bz, unsigned smem, CUstream, void** params, void**) {
  std::lock_guard<std::recursive_mutex> lock(g_mu);
  Function* fn = reinterpret_cast<Function*>(f);
  if (bx * by * bz == 0 || bx * by * bz > 1024 || gx * gy * gz == 0) return CUDA_ERROR_INVALID_VALUE;
  if (static_cast<int>(smem) > fn->max_dyn_smem) return CUDA_ERROR_INVALID_VALUE;
  const bool ok = RunGrid(fn, gdv_emu_uint3{gx, gy, gz}, gdv_emu_uint3{bx, by, bz}, smem, params);
  if (ok && !GuardsIntact(("after kernel " + fn->name).c_str())) return CUDA_ERROR_ILLEGAL_ADDRESS;
  return ok ? CUDA_SUCCESS : CUDA_ERROR_LAUNCH_TIMEOUT;
}
CUresult cuGetErrorString(CUresult r, const char** s) {
  *s = r == CUDA_SUCCESS ? "no error" : "emulated driver error";
  EMU_OK;
}
CUresult cuPointerGetAttribute(void* out, CUpointer_attribute, CUdeviceptr ptr) {
  std::lock_guard<std::mutex> g(g_pinned_mu);
  auto it = g_pinned.upper_bound(static_cast<uintptr_t>(ptr));
  if (it == g_pinned.begin()) return CUDA_ERROR_INVALID_VALUE;
  --it;
  if (static_cast<uintptr_t>(ptr) >= it->first + it->second) return CUDA_ERROR_INVALID_VALUE;
  *static_cast<unsigned int*>(out) = 1;  // CU_MEMORYTYPE_HOST
  return CUDA_SUCCESS;
}
CUresult cuCtxEnablePeerAccess(CUcontext, unsigned int) { EMU_OK; }
CUresult cuDeviceCanAccessPeer(int* can, CUdevice, CUdevice) { *can = 0; EMU_OK; }
CUresult cuIpcGetMemHandle(CUipcMemHandle*, CUdeviceptr) { return CUDA_ERROR_NOT_SUPPORTED; }
CUresult cuIpcOpenMemHandle_v2(CUdeviceptr*, CUipcMemHandle, unsigned int) { return CUDA_ERROR_NOT_SUPPORTED; }
CUresult cuIpcCloseMemHandle(CUdeviceptr) { return CUDA_ERROR_NOT_SUPPORTED; }
}
