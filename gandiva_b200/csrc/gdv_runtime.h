// Runtime behind Projector / Filter: device handles, scratch pool, compiled kernels,
// buffer marshalling and launches.  Replaces the reference's Engine (module ownership,
// compile, function pointers) and the evaluate-time half of its Annotator (RecordBatch ->
// flat pointer block); SURVEY.md §3 call stacks A-D.
#pragma once
#include <atomic>
#include <map>
#include <memory>
#include <mutex>
#include <string>
#include <thread>
#include <unordered_map>
#include <vector>

#include "gdv_codegen.h"
#include "gdv_cuda.h"

namespace gdv {

extern std::atomic<long long> g_launch_count;
extern std::atomic<long long> g_compile_count;  // NVRTC compilations (cache misses)

class Device {
 public:
  static Status Get(int ordinal, Device** out);
  Status MakeCurrent() const;
  int ordinal() const { return ordinal_; }
  int sm_count() const { return sm_count_; }
  CUdevice cu_device() const { return dev_; }
  std::string arch() const;
  // The engine's own stream for calls that pass stream == NULL: one non-blocking stream per
  // (host thread, device), so that concurrent Evaluate calls from different threads never share
  // stream-ordered scratch or error / count read-backs.  The thread that created the Device uses
  // stream_; other threads get theirs on first use (destroyed when the thread exits).
  CUstream stream() const;
  CUstream copy_stream() const { return copy_stream_; }

  // Pooled device scratch: freed blocks are cached and reused (no cuMemFree on the hot path).  The
  // cache is bounded: once the idle blocks hold more than the limit (default 4 GiB, GDV_POOL_LIMIT_MB
  // or SetPoolLimit), the largest idle blocks go back to the driver, so one multi-GB batch does not
  // pin that much HBM for the life of the process.
  Status Alloc(size_t bytes, CUdeviceptr* out);
  void Free(CUdeviceptr p);
  // Returns idle blocks to the driver until at most keep_bytes stay cached; returns the bytes released.
  size_t Trim(size_t keep_bytes);
  void SetPoolLimit(size_t bytes) { pool_limit_ = bytes; }
  size_t idle_bytes() const { return idle_bytes_; }

  // Kernels of device/static_kernels.cu (embedded sm_90a cubin).
  Status StaticFunction(const char* name, CUfunction* out);

 private:
  Device() = default;
  int ordinal_ = 0;
  CUdevice dev_ = 0;
  CUcontext ctx_ = nullptr;
  CUstream stream_ = nullptr;
  CUstream copy_stream_ = nullptr;
  std::thread::id owner_thread_;
  int sm_count_ = 0, cc_major_ = 0, cc_minor_ = 0;
  std::mutex mu_;
  std::multimap<size_t, CUdeviceptr> free_;
  std::unordered_map<CUdeviceptr, size_t> sizes_;
  size_t idle_bytes_ = 0;                  // bytes held by free_
  size_t pool_limit_ = size_t(4) << 30;
  CUmodule static_mod_ = nullptr;
  std::map<std::string, CUfunction> static_fns_;
};

class Projector;
// A batch extended by the temporary columns a rope pre-projector produced (gdv_rope_temps.h); owns them.
struct TempColumns {
  std::vector<gdv_column_t> cols;
  gdv_batch_t batch;
  std::vector<std::vector<uint8_t>> host;
  Device* dev = nullptr;
  std::vector<CUdeviceptr> device;
  std::unique_ptr<TempColumns> lower;  // the temporaries `pre` itself reads, when it is a two-stage plan
  ~TempColumns();
  // batch = `in` + one utf8 column per output of `pre`.  A two-stage `pre` has its own temporaries built ONCE
  // here (not once per sizing pass and once more for the write pass, which would multiply per nesting level).
  Status Build(Projector* pre, const gdv_batch_t* in, void* stream);

 private:
  Status Run(Projector* proj, const gdv_batch_t* eval, const gdv_batch_t* in, void* stream);
};

// RAII list of scratch blocks returned to the pool when the evaluation ends.
class ScratchScope {
 public:
  explicit ScratchScope(Device* d) : dev_(d) {}
  // Work that reads or writes the blocks may still be queued on `stream` when an Evaluate returns
  // early with an error: the destructor then waits for the stream before the blocks go back to the
  // pool (where another thread could be handed them).  Settled() after the call's own final
  // synchronisation skips that wait.
  void Guard(CUstream stream) {
    stream_ = stream;
    guarded_ = true;
  }
  void Settled() { guarded_ = false; }
  ~ScratchScope() {
    if (guarded_ && !blocks_.empty()) Driver().StreamSynchronize(stream_);
    for (auto p : blocks_) dev_->Free(p);
  }
  Status Alloc(size_t bytes, CUdeviceptr* out) {
    Status s = dev_->Alloc(bytes, out);
    if (s.ok()) blocks_.push_back(*out);
    return s;
  }
  std::vector<CUdeviceptr> Release() {
    std::vector<CUdeviceptr> b;
    b.swap(blocks_);
    return b;
  }

 private:
  Device* dev_;
  std::vector<CUdeviceptr> blocks_;
  CUstream stream_ = nullptr;
  bool guarded_ = false;
};

struct Config {
  bool optimize = true;
  bool dump_ir = false;
  int device = 0;
  int rows_per_thread = 0;
  int block_threads = 0;
  int loader = 0;
  int stages = 0;
  int sm_reserve = 0;
  int string_scan = 0;
  bool large_batch = false;  // set per kernel variant by Filter::KernelFor (batches >= 32 M rows)
};

class CompiledKernel {
 public:
  GeneratedKernel gen;
  std::vector<char> cubin;
  std::string ptx;
  std::string compile_log;

  struct Loaded {
    CUmodule mod = nullptr;
    CUfunction fn = nullptr;
    int blocks_per_sm = 1;
    int regs = 0;
    int smem = 0;
  };
  // Lazily loads the cubin into `dev`'s context.
  Status Load(Device* dev, Loaded* out);

 private:
  std::mutex mu_;
  std::map<int, Loaded> loaded_;
};

// Pending asynchronous evaluation state (error flag / count readback) per stream.
struct Pending {
  Device* dev = nullptr;
  std::vector<CUdeviceptr> scratch;  // returned to the pool at sync
  CUdeviceptr d_err = 0;
  CUdeviceptr d_count = 0;
  CUdeviceptr d_state = 0;  // filter look-back state, reused by stream-ordered launches
  size_t state_cap = 0;
  bool uses_ctx = false;
};

class Projector {
 public:
  static Status Make(SchemaPtr schema, std::vector<ExpressionPtr> exprs, int selection_mode,
                     const Config& cfg, std::shared_ptr<Projector>* out);
  Status Evaluate(const gdv_batch_t* batch, const gdv_selection_t* sel, gdv_out_column_t* outs,
                  int n_outs, void* stream, bool async);
  // Bytes output `out_index` (utf8/binary) produces for this batch: runs the sizing pass only.
  Status OutputVarSize(const gdv_batch_t* batch, const gdv_selection_t* sel, int out_index,
                       void* stream, int64_t* bytes);
  Status Sync(void* stream);
  std::string DumpIR() const;
  CompiledKernel& kernel();
  // Variant specialised on whether any referenced input carries a validity bitmap.
  Status KernelFor(bool nullable, CompiledKernel** out);
  const Config& config() const { return cfg_; }
  int num_outputs() const { return static_cast<int>(exprs_.size()); }
  const SchemaPtr& schema() const { return schema_; }
  const std::vector<ExpressionPtr>& expressions() const { return exprs_; }
  Projector* rope_pre() const { return rope_pre_.get(); }
  Projector* rope_main() const { return rope_main_.get(); }

 private:
  // Consumers of a rope (gdv_rope_temps.h): the ropes are materialised by rope_pre_ into temporary utf8
  // columns and rope_main_ evaluates the caller's expressions over the batch plus those columns.
  std::shared_ptr<Projector> rope_pre_, rope_main_;
  Status BuildKernels();
  static Status MakeWithRopeTemps(const SchemaPtr& schema, const std::vector<ExpressionPtr>& exprs,
                                  int selection_mode, const Config& cfg, Projector* into);
  // One utf8/binary output expression: sizing + write kernels, [0] nullable inputs, [1] no nulls.
  struct StringKernels {
    int out_index = 0;
    std::unique_ptr<CompiledKernel> size[2], write[2];
  };
  Status StringKernelsFor(StringKernels* sk, bool nullable, CompiledKernel** size,
                          CompiledKernel** write);
  Status CheckEvaluateArgs(const gdv_batch_t* batch, const gdv_selection_t* sel, int64_t* n) const;
  Status EvaluateString(StringKernels* sk, const gdv_batch_t* batch, const gdv_selection_t* sel,
                        gdv_out_column_t* out, void* stream, bool async, bool size_only,
                        int64_t* total);

  SchemaPtr schema_;
  std::vector<ExpressionPtr> exprs_;
  std::vector<ExpressionPtr> fixed_exprs_;  // fixed-width outputs: one fused kernel
  std::vector<int> fixed_idx_;              // their positions in exprs_
  std::vector<StringKernels> strings_;      // utf8/binary outputs
  int selection_mode_ = GDV_SEL_NONE;
  Config cfg_;
  std::unique_ptr<CompiledKernel> kernel_;          // general (nullable) variant, built at Make()
  std::unique_ptr<CompiledKernel> kernel_nonull_;   // built on first batch without nulls
  std::atomic<CompiledKernel*> last_used_{nullptr};  // variant of the latest Evaluate (kernel_info)
  std::mutex mu_;
  std::map<void*, Pending> pending_;
};

class Filter {
 public:
  static Status Make(SchemaPtr schema, ConditionPtr cond, const Config& cfg,
                     std::shared_ptr<Filter>* out);
  Status Evaluate(const gdv_batch_t* batch, gdv_selection_t* out_sel, void* stream, bool async,
                  void* d_count);
  Status Sync(void* stream, int64_t* num_slots);
  std::string DumpIR() const;
  // One kernel per selection-vector index width, compiled on first use.
  // One kernel per (index width, nullable inputs?, large batch?), compiled on first use.
  Status KernelFor(int mode, bool nullable, bool large, CompiledKernel** out);
  const Config& config() const { return cfg_; }
  const SchemaPtr& schema() const { return schema_; }
  CompiledKernel* last_used() const { return rope_main_ != nullptr ? rope_main_->last_used() : last_used_.load(); }

 private:
  std::shared_ptr<Projector> rope_pre_;  // consumers of a rope (gdv_rope_temps.h): temps first,
  std::shared_ptr<Filter> rope_main_;    // then the condition over the batch plus the temp columns
  std::atomic<CompiledKernel*> last_used_{nullptr};
  SchemaPtr schema_;
  ConditionPtr cond_;
  Config cfg_;
  mutable std::mutex mu_;
  std::map<int, std::unique_ptr<CompiledKernel>> kernels_;
  std::map<void*, Pending> pending_;
};

const char* ExecutionErrorMessage(int code);

}  // namespace gdv
