// Kernel fuser: lowers a set of validated expression trees to ONE CUDA kernel
// (source text) per Projector / Filter.  Replaces the reference's LLVMGenerator +
// Annotator + BitmapAccumulator (named in BASELINE.json north_star; SURVEY.md §2):
//   * Annotator        -> ColumnSlot table (which schema columns the kernel reads) and the
//                         flat gdv_args pointer block the kernel indexes;
//   * LLVMGenerator    -> EmitBody(): straight-line per-row code calling the device library;
//   * BitmapAccumulator-> validity is ANDed in registers and written with one warp ballot
//                         per 32 rows, inside the same kernel.
#pragma once
#include <string>
#include <vector>

#include "gdv_node.h"

namespace gdv {

struct Status {
  int code = GDV_OK;
  std::string msg;
  bool ok() const { return code == GDV_OK; }
  static Status OK() { return Status(); }
  static Status Make(int c, std::string m) {
    Status s;
    s.code = c;
    s.msg = std::move(m);
    return s;
  }
};

// Validate one expression against the schema and the function registry
// (ExpressionValidationError on failure).
Status ValidateExpression(const Schema& schema, const Expression& expr);

enum class KernelKind { kProject, kFilter, kStringSize, kStringWrite };

struct KernelSpec {
  KernelKind kind = KernelKind::kProject;
  int selection_mode = GDV_SEL_NONE;  // project: input selection; filter: output index width
  int rows_per_thread = 0;            // 0 = pick from bytes/row
  int block_threads = 0;              // 0 = pick per kernel shape
  bool large_batch = false;           // filter: the batch has >= 32 M rows (big tiles)
  std::string name;                   // kernel symbol
  bool nullable = true;               // false: specialised for batches where no input has nulls
  int loader = 0;                     // 0 = engine picks, 1 = direct LDG, 2 = TMA bulk -> shared
  int stages = 0;                     // projector, TMA loader: shared-memory stages per CTA (0 = pick);
                                      // fixed-width filter: 1024-row chunks every warp walks per tile (1/2/4/8)
  int string_scan = 0;                // bit 0: LIKE with the per-lane matcher only (no cooperative scan);
                                      // bit 2: row-driven string filter even where the key-driven one applies
                                      // bit 3: no inline / prefix shortcut over string_view / binary_view views
  int filter_gating = 0;              // fixed-width filter: 0 = gated loads wherever they apply, 1 = off
};

struct ColumnSlot {
  int schema_index;
  DataType type;
  // Filter kernels: a null in this column makes the condition not-true whatever the other columns
  // hold, so its validity is ANDed into the tile's keep-mask 32 rows at a time after the row loop
  // instead of being read per row (BodyGen::TruthStrict).
  bool hoist = false;
};

// Byte offsets inside gdv_args; the host packs the same layout (see EmitArgsStruct()).
struct ArgsLayout {
  int ni, no;  // array extents (>= 1)
  size_t off_n = 0, off_row_base = 8, off_sel = 16, off_out_idx = 24, off_out_count = 32,
         off_tile_state = 40, off_ticket = 48, off_err = 56, off_out_cap = 64, off_n_ptr = 72;
  size_t off_in_val, off_in_vld, off_in_var, off_out_val, off_out_vld, off_out_var, off_in_vsh,
      off_in_dsh, size;
  // Kernels that read a dictionary column get one more block per input (HasDictionary): the
  // dictionary's offsets, validity word pointer, length and validity bit shift.  Zero otherwise.
  bool dict = false;
  size_t off_in_dof = 0, off_in_dvl = 0, off_in_dln = 0, off_in_dvs = 0;
  // Kernels that read a string_view / binary_view column get one more block per input (HasView):
  // the device pointer of the data buffers' pointer table, the sizes' device pointer and the buffer
  // count.  Zero otherwise, so every other kernel keeps its layout and source.
  bool view = false;
  size_t off_in_vbf = 0, off_in_vsz = 0, off_in_vbn = 0;
  ArgsLayout(int n_inputs, int n_outputs, bool dictionary = false, bool views = false);
};

// What the fuser generated, and how the runtime launches it.  Fields a kernel shape does not use
// keep their defaults.
struct GeneratedKernel {
  std::string source;   // full translation unit (device library is #include'd by name)
  std::string name;
  KernelKind kind = KernelKind::kProject;
  int rows_per_thread = 0;
  int block_threads = 0;
  int selection_mode = GDV_SEL_NONE;
  bool nullable = true;
  std::vector<ColumnSlot> inputs;   // kernel input slot j reads schema column inputs[j]
  std::vector<DataType> outputs;    // project: one per expression; filter: empty
  bool uses_ctx = false;            // some function can raise an ExecutionError
  int in_bytes_per_row = 0;         // algorithmic bytes (values only) read per row
  int out_bytes_per_row = 0;
  ArgsLayout args{0, 0};            // the gdv_args layout the kernel was emitted with; the host packs it
  int dynamic_smem = 0;             // bytes of dynamic shared memory (string staging)
  int64_t tile_rows = 0;            // filter: rows per CTA tile (one look-back descriptor each)
  bool key_driven = false;          // string filter driven by the occurrences of a literal key in the column's bytes
  bool staged = false;              // project: inputs staged through shared memory by TMA bulk copies
  int stages = 0;                   // staged: shared-memory stages per CTA
  int64_t cta_tile_rows = 0;        // staged: rows per CTA tile (block_threads * rows_per_thread)
  int view_shortcuts = 0;           // call sites decided from the raw 16-byte views (BodyGen::ViewShortcut)
  int gated_stages = 0;             // fixed-width filter: stages of gated loads (GatePlan), 0 = not gated
};

bool HasDictionary(const std::vector<ColumnSlot>& slots);
bool HasView(const std::vector<ColumnSlot>& slots);

Status GenerateKernel(const Schema& schema, const std::vector<ExpressionPtr>& exprs,
                      const KernelSpec& spec, GeneratedKernel* out);

// Filter conditions that can be evaluated once per dictionary entry (DESIGN.md §3.6): the condition
// reads exactly one column, that column is dictionary-encoded, nothing in it can raise, and a null in
// the column makes it not-true (so a null index, a null entry or an index out of range is never kept).
// Returns the column's schema index, or -1.
int DictionaryFirstColumn(const Schema& schema, const Node& cond);
// The same tree with every dictionary-encoded field read as a plain column of its value type.
NodePtr WithValueTypes(const NodePtr& node);

}  // namespace gdv
