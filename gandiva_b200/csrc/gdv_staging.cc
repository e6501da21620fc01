#include "gdv_staging.h"

#include <pthread.h>
#include <sched.h>

#include <atomic>
#include <chrono>
#include <condition_variable>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <mutex>
#include <thread>
#include <vector>

#include "gdv_runtime.h"

namespace gdv {

namespace {

constexpr size_t kSlotBytes = size_t(8) << 20;   // one DMA piece: ~150 us at PCIe Gen5 x16
constexpr int kSlots = 6;                        // pieces in flight (memcpy of i+1.. while DMA of i)
constexpr size_t kDirectBelow = size_t(1) << 20; // smaller copies are not worth the hand-offs

std::atomic<long long> g_staged_bytes{0};

// ---- NUMA placement ---------------------------------------------------------------------------------------
// The pinned ring and the copy threads belong on the NUMA node the GPU hangs off: a slot on the other socket
// makes every DMA cross the socket interconnect, and copy threads floating over both sockets make the pageable
// path's rate vary widely from run to run on a two-socket host.

// CPUs of NUMA node `node` that this process may run on ("0-31,64-95" in sysfs); false if unreadable.
bool NodeCpus(int node, cpu_set_t* out) {
  char path[96];
  std::snprintf(path, sizeof(path), "/sys/devices/system/node/node%d/cpulist", node);
  FILE* f = std::fopen(path, "r");
  if (f == nullptr) return false;
  char buf[4096];
  const size_t len = std::fread(buf, 1, sizeof(buf) - 1, f);
  std::fclose(f);
  buf[len] = 0;
  cpu_set_t allowed;
  if (sched_getaffinity(0, sizeof(allowed), &allowed) != 0) return false;
  CPU_ZERO(out);
  int count = 0;
  for (const char* p = buf; *p != 0;) {
    char* end = nullptr;
    const long a = std::strtol(p, &end, 10);
    if (end == p) break;
    long b = a;
    p = end;
    if (*p == '-') {
      b = std::strtol(p + 1, &end, 10);
      p = end;
    }
    for (long c = a; c <= b && c < CPU_SETSIZE; ++c)
      if (CPU_ISSET(c, &allowed)) {
        CPU_SET(c, out);
        ++count;
      }
    while (*p == ',' || *p == '\n' || *p == ' ') ++p;
  }
  return count >= 1;
}

// NUMA node of the GPU (sysfs numa_node of its PCI function), else of the calling thread, else -1.
int StagingNode(Device* dev) {
  if (const char* e = std::getenv("GDV_STAGE_PIN"))
    if (std::atoi(e) == 0) return -1;
  const DriverApi& d = Driver();
  int bus = -1, slot = -1, domain = 0;
  if (d.DeviceGetAttribute(&bus, CU_DEVICE_ATTRIBUTE_PCI_BUS_ID, dev->cu_device()) == CUDA_SUCCESS &&
      d.DeviceGetAttribute(&slot, CU_DEVICE_ATTRIBUTE_PCI_DEVICE_ID, dev->cu_device()) == CUDA_SUCCESS &&
      d.DeviceGetAttribute(&domain, CU_DEVICE_ATTRIBUTE_PCI_DOMAIN_ID, dev->cu_device()) == CUDA_SUCCESS && bus >= 0) {
    char path[128];
    std::snprintf(path, sizeof(path), "/sys/bus/pci/devices/%04x:%02x:%02x.0/numa_node", domain, bus, slot);
    if (FILE* f = std::fopen(path, "r")) {
      int node = -1;
      const int got = std::fscanf(f, "%d", &node);
      std::fclose(f);
      if (got == 1 && node >= 0) return node;
    }
  }
  const int cpu = sched_getcpu();
  if (cpu < 0) return -1;
  for (int node = 0; node < 64; ++node) {
    cpu_set_t set;
    if (!NodeCpus(node, &set)) break;
    if (CPU_ISSET(cpu, &set)) return node;
  }
  return -1;
}

// Runs the calling thread on `node` for the lifetime of the object (memory it allocates and first touches
// lands there), then restores its affinity mask.
class OnNode {
 public:
  explicit OnNode(int node) {
    cpu_set_t set;
    if (node >= 0 && NodeCpus(node, &set) && sched_getaffinity(0, sizeof(saved_), &saved_) == 0)
      moved_ = sched_setaffinity(0, sizeof(set), &set) == 0;
  }
  ~OnNode() {
    if (moved_) sched_setaffinity(0, sizeof(saved_), &saved_);
  }

 private:
  cpu_set_t saved_;
  bool moved_ = false;
};

// A few threads that copy pieces of one transfer in parallel (one memcpy stream does ~10 GB/s, the link wants
// ~55).  Started on first use; they poll for 2 ms after a job and park on a condition variable after that.
class CopyPool {
 public:
  // `node`: where the workers run (the first caller decides; one process drives one GPU).
  static CopyPool& Get(int node) {
    static CopyPool* p = new CopyPool(node);  // never destroyed: threads may outlive static destructors
    return *p;
  }
  // Copies in kChunk pieces that the calling thread and the workers CLAIM one at a time, so the call
  // never waits for a worker to wake up: a worker that is asleep (or descheduled) simply claims nothing
  // and the caller copies those pieces itself: waiting for seven sleeping workers to wake can cost more
  // than the copy of a 1M-row column.
  void Copy(void* dst, const void* src, size_t bytes) {
    if (bytes < 2 * kChunk || workers_ == 0) {
      std::memcpy(dst, src, bytes);
      return;
    }
    std::lock_guard<std::mutex> one_caller(caller_mu_);
    const unsigned long long e = (ticket_.load(std::memory_order_relaxed) >> 32) + 1;
    // Full ring slots (the pieces of a bulk transfer) go in 1 MB pieces: memcpy then takes its streaming
    // (non-temporal store) path and the 8 threads each get one piece.  Smaller copies (one
    // column of a 1M-row batch) go in 256 KB pieces so that every thread has something to claim.
    const size_t chunk = chunk_override_ != 0 ? chunk_override_ : (bytes >= kSlotBytes ? 4 * kChunk : kChunk);
    const unsigned nchunks = static_cast<unsigned>((bytes + chunk - 1) / chunk);
    chunk_.store(chunk, std::memory_order_relaxed);
    dst_.store(static_cast<char*>(dst), std::memory_order_relaxed);
    src_.store(static_cast<const char*>(src), std::memory_order_relaxed);
    bytes_.store(bytes, std::memory_order_relaxed);
    nchunks_.store(nchunks, std::memory_order_relaxed);
    done_.store(0, std::memory_order_relaxed);
    ticket_.store(e << 32, std::memory_order_seq_cst);  // publishes the fields above
    // (seq_cst here and on the sleeper's side: either this load sees the sleeper or its predicate sees the
    // job.  A missed wake-up would only cost parallelism — the caller copies every unclaimed piece.)
    if (sleepers_.load(std::memory_order_seq_cst) > 0) {
      std::lock_guard<std::mutex> g(mu_);
      cv_.notify_one();  // a woken worker wakes the next one: the caller pays for one wake-up, not seven
    }
    Work(e);
    while (done_.load(std::memory_order_acquire) != nchunks) {  // pieces still in a worker's hands
#if defined(__x86_64__)
      __builtin_ia32_pause();
#endif
    }
  }

 private:
  static constexpr size_t kChunk = size_t(256) << 10;

  explicit CopyPool(int node) {
    int want = 8;
    if (const char* e = std::getenv("GDV_STAGE_THREADS")) want = std::atoi(e);
    const int hw = static_cast<int>(std::thread::hardware_concurrency());
    if (hw > 0 && want > hw) want = hw;
    if (const char* e = std::getenv("GDV_STAGE_CHUNK_KB")) chunk_override_ = static_cast<size_t>(std::atoi(e)) << 10;
    cpu_set_t node_cpus;
    const bool pin = node >= 0 && NodeCpus(node, &node_cpus);
    for (int t = 1; t < want; ++t) {
      std::thread th([this] { Loop(); });
      if (pin) pthread_setaffinity_np(th.native_handle(), sizeof(node_cpus), &node_cpus);
      th.detach();
      ++workers_;
    }
  }
  // Claims and copies pieces of job `e` until none is left.  A claim is a CAS on (epoch << 32 | next
  // piece): it can only succeed while job `e` is still the published one, and the caller does not return
  // (so the fields do not change) before every claimed piece is counted in done_.
  void Work(unsigned long long e) {
    for (;;) {
      unsigned long long t = ticket_.load(std::memory_order_acquire);
      if ((t >> 32) != e) return;
      const unsigned idx = static_cast<unsigned>(t & 0xffffffffu);
      if (idx >= nchunks_.load(std::memory_order_relaxed)) return;
      char* d = dst_.load(std::memory_order_relaxed);
      const char* s = src_.load(std::memory_order_relaxed);
      const size_t bytes = bytes_.load(std::memory_order_relaxed);
      const size_t chunk = chunk_.load(std::memory_order_relaxed);
      if (!ticket_.compare_exchange_weak(t, t + 1, std::memory_order_acq_rel)) continue;
      const size_t off = static_cast<size_t>(idx) * chunk;
      std::memcpy(d + off, s + off, std::min(chunk, bytes - off));
      done_.fetch_add(1, std::memory_order_acq_rel);
    }
  }
  bool HasWork(unsigned long long e) const {
    const unsigned long long t = ticket_.load(std::memory_order_acquire);
    return (t >> 32) == e && static_cast<unsigned>(t & 0xffffffffu) < nchunks_.load(std::memory_order_relaxed);
  }
  void Loop() {
    unsigned long long seen = 0;
    for (;;) {
      // A host batch is several copies back to back (one per column, then — a DMA and a kernel later —
      // the results): after a job the worker polls for the next one for 2 ms before it goes to sleep.
      bool got = false;
      const auto t_end = std::chrono::steady_clock::now() + std::chrono::milliseconds(2);
      for (unsigned spin = 0; !got; ++spin) {
        if ((ticket_.load(std::memory_order_acquire) >> 32) != seen) {
          got = true;
        } else if ((spin & 255u) == 255u) {
          if (std::chrono::steady_clock::now() >= t_end) break;
          std::this_thread::yield();
        }
      }
      if (!got) {
        std::unique_lock<std::mutex> g(mu_);
        sleepers_.fetch_add(1, std::memory_order_seq_cst);
        cv_.wait(g, [&] { return (ticket_.load(std::memory_order_seq_cst) >> 32) != seen; });
        sleepers_.fetch_sub(1, std::memory_order_acq_rel);
      }
      seen = ticket_.load(std::memory_order_acquire) >> 32;
      if (!got && sleepers_.load(std::memory_order_acquire) > 0 && HasWork(seen)) {
        std::lock_guard<std::mutex> g(mu_);
        cv_.notify_one();
      }
      Work(seen);
    }
  }
  int workers_ = 0;
  size_t chunk_override_ = 0;
  std::mutex mu_, caller_mu_;
  std::condition_variable cv_;
  std::atomic<char*> dst_{nullptr};
  std::atomic<const char*> src_{nullptr};
  std::atomic<size_t> bytes_{0}, chunk_{0};
  std::atomic<unsigned> nchunks_{0}, done_{0};
  std::atomic<int> sleepers_{0};
  std::atomic<unsigned long long> ticket_{0};  // (job number << 32) | next unclaimed piece
};

// The pinned slots of one device.  One transfer at a time uses the ring (the link is shared anyway).
struct Ring {
  std::mutex mu;
  bool ready = false;
  void* slot[kSlots] = {nullptr};
  CUevent ev[kSlots] = {nullptr};
  bool busy[kSlots] = {false};
  int next = 0;

  int node = -1;

  Status Init(Device* dev) {
    if (ready) return Status::OK();
    const DriverApi& d = Driver();
    node = StagingNode(dev);
    OnNode here(node);  // the slots are allocated (and so placed) from a CPU of the GPU's node
    for (int i = 0; i < kSlots; ++i) {
      Status s = CuCheck(d.MemHostAlloc(&slot[i], kSlotBytes, 0), "cuMemHostAlloc(staging slot)");
      if (!s.ok()) return s;
      s = CuCheck(d.EventCreate(&ev[i], CU_EVENT_DISABLE_TIMING), "cuEventCreate");
      if (!s.ok()) return s;
    }
    ready = true;
    return Status::OK();
  }
};

std::mutex g_rings_mu;
Ring* g_rings[64] = {nullptr};

Ring* RingFor(Device* dev) {
  std::lock_guard<std::mutex> g(g_rings_mu);
  Ring*& r = g_rings[dev->ordinal()];
  if (r == nullptr) r = new Ring();
  return r;
}

}  // namespace

long long StagedBytes() { return g_staged_bytes.load(); }

bool IsPageableHost(const void* p) {
  const DriverApi& d = Driver();
  if (!d.loaded) return false;
  unsigned int type = 0;
  const CUresult r = d.PointerGetAttribute(&type, CU_POINTER_ATTRIBUTE_MEMORY_TYPE,
                                           reinterpret_cast<CUdeviceptr>(p));
  // memory the driver has never seen: cuPointerGetAttribute fails with INVALID_VALUE
  return r != CUDA_SUCCESS;
}

Status StagedHtoD(Device* dev, CUdeviceptr dst, const void* src, size_t bytes, CUstream stream) {
  const DriverApi& d = Driver();
  if (bytes == 0) return Status::OK();
  if (bytes < kDirectBelow || !IsPageableHost(src))
    return CuCheck(d.MemcpyHtoDAsync(dst, src, bytes, stream), "cuMemcpyHtoDAsync");
  Ring* ring = RingFor(dev);
  std::lock_guard<std::mutex> lock(ring->mu);
  Status st = ring->Init(dev);
  if (!st.ok()) return st;
  CopyPool& pool = CopyPool::Get(ring->node);
  const char* s = static_cast<const char*>(src);
  for (size_t off = 0; off < bytes; off += kSlotBytes) {
    const size_t n = std::min(kSlotBytes, bytes - off);
    const int i = ring->next;
    ring->next = (i + 1) % kSlots;
    if (ring->busy[i]) {  // the DMA that last read this slot must be done
      st = CuCheck(d.EventSynchronize(ring->ev[i]), "cuEventSynchronize(staging slot)");
      if (!st.ok()) return st;
      ring->busy[i] = false;
    }
    pool.Copy(ring->slot[i], s + off, n);
    st = CuCheck(d.MemcpyHtoDAsync(dst + off, ring->slot[i], n, stream), "cuMemcpyHtoDAsync(staged)");
    if (!st.ok()) return st;
    st = CuCheck(d.EventRecord(ring->ev[i], stream), "cuEventRecord");
    if (!st.ok()) return st;
    ring->busy[i] = true;
  }
  g_staged_bytes.fetch_add(static_cast<long long>(bytes));
  return Status::OK();
}

Status StagedDtoH(Device* dev, void* dst, CUdeviceptr src, size_t bytes, CUstream stream) {
  const DriverApi& d = Driver();
  if (bytes == 0) return Status::OK();
  if (bytes < kDirectBelow || !IsPageableHost(dst))
    return CuCheck(d.MemcpyDtoHAsync(dst, src, bytes, stream), "cuMemcpyDtoHAsync");
  Ring* ring = RingFor(dev);
  std::lock_guard<std::mutex> lock(ring->mu);
  Status st = ring->Init(dev);
  if (!st.ok()) return st;
  CopyPool& pool = CopyPool::Get(ring->node);
  char* out = static_cast<char*>(dst);
  // every slot may still be read by an earlier H2D: wait for those first
  for (int i = 0; i < kSlots; ++i)
    if (ring->busy[i]) {
      st = CuCheck(d.EventSynchronize(ring->ev[i]), "cuEventSynchronize(staging slot)");
      if (!st.ok()) return st;
      ring->busy[i] = false;
    }
  const size_t pieces = (bytes + kSlotBytes - 1) / kSlotBytes;
  // DMA of piece p + depth is enqueued before piece p is copied out of its slot
  const size_t depth = static_cast<size_t>(kSlots) - 1;
  auto issue = [&](size_t p) -> Status {
    const size_t off = p * kSlotBytes, n = std::min(kSlotBytes, bytes - off);
    const int i = static_cast<int>(p % kSlots);
    Status s2 = CuCheck(d.MemcpyDtoHAsync(ring->slot[i], src + off, n, stream), "cuMemcpyDtoHAsync(staged)");
    if (!s2.ok()) return s2;
    return CuCheck(d.EventRecord(ring->ev[i], stream), "cuEventRecord");
  };
  for (size_t p = 0; p < std::min(depth, pieces); ++p) {
    st = issue(p);
    if (!st.ok()) return st;
  }
  for (size_t p = 0; p < pieces; ++p) {
    const size_t off = p * kSlotBytes, n = std::min(kSlotBytes, bytes - off);
    const int i = static_cast<int>(p % kSlots);
    st = CuCheck(d.EventSynchronize(ring->ev[i]), "cuEventSynchronize(staging slot)");
    if (!st.ok()) return st;
    pool.Copy(out + off, ring->slot[i], n);
    if (p + depth < pieces) {
      st = issue(p + depth);
      if (!st.ok()) return st;
    }
  }
  ring->next = 0;
  g_staged_bytes.fetch_add(static_cast<long long>(bytes));
  return Status::OK();
}

}  // namespace gdv
