/*
 * gandiva_b200.h — C-ABI of the H100-native expression engine.
 *
 * This is the drop-in boundary for the Gandiva hot path (Projector / Filter
 * Make + Evaluate over Arrow buffers).  Everything here is `extern "C"`, plain
 * pointers and sizes; no C++ types, no torch types, no Arrow C++ types.  The
 * C++ API in include/gandiva/ (namespace gandiva, the declarations that
 * pyarrow/includes/libgandiva.pxd binds) is a thin layer over these calls; so
 * is the Python mirror in gandiva_b200/__init__.py (ctypes).
 *
 * Reference interface each group replaces (the reference mount holds no
 * source, see SURVEY.md §0; citations are to the descendant's binding
 * declarations shipped with pyarrow 24.0.0, `P` =
 * site-packages/pyarrow):
 *
 *   gdv_node_*            <- gandiva::TreeExprBuilder::Make*      P/includes/libgandiva.pxd:110-212
 *   gdv_expression_make   <- TreeExprBuilder::MakeExpression      P/includes/libgandiva.pxd:151-153
 *   gdv_condition_make    <- TreeExprBuilder::MakeCondition       P/includes/libgandiva.pxd:172-174
 *   gdv_projector_make    <- gandiva::Projector::Make             P/includes/libgandiva.pxd:230-240
 *   gdv_projector_evaluate<- gandiva::Projector::Evaluate (both)  P/includes/libgandiva.pxd:218-226
 *   gdv_projector_dump_ir <- gandiva::Projector::DumpIR           P/includes/libgandiva.pxd:228
 *   gdv_filter_make       <- gandiva::Filter::Make                P/includes/libgandiva.pxd:252-256
 *   gdv_filter_evaluate   <- gandiva::Filter::Evaluate            P/includes/libgandiva.pxd:246-248
 *   gdv_filter_dump_ir    <- gandiva::Filter::DumpIR              P/includes/libgandiva.pxd:250
 *   gdv_registry_*        <- GetRegisteredFunctionSignatures      P/includes/libgandiva.pxd:258-277
 *   gdv_config_t          <- gandiva::Configuration               P/includes/libgandiva.pxd:279-298
 *   GDV_SEL_*             <- gandiva::SelectionVector::Mode       P/includes/libgandiva.pxd:49-56
 *   status codes          <- arrow::StatusCode (40/41/42)         P/include/arrow/status.h:97-100
 *
 * Ownership: every handle returned through an out-parameter is owned by the
 * caller and released with the matching *_release call.  Nodes are
 * reference-counted inside the library: a parent keeps its children alive, so
 * a caller may release child handles right after building the parent.
 * Threading: Make calls may run concurrently; a built projector/filter may be
 * evaluated from several threads at once (per-call scratch; the engine's own
 * stream -- the one a NULL `stream` argument names -- is per host thread, so
 * stream-ordered scratch and error / count read-backs are never shared).  A
 * caller-provided stream must not be used from two threads at the same time,
 * and an asynchronous Evaluate on the NULL stream is completed by *_sync() on
 * the same thread.
 * Errors: every call returns a gdv_status; gdv_last_error() returns the
 * thread-local message of the last failing call on this thread.
 */
#ifndef GANDIVA_B200_H
#define GANDIVA_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ---- status codes (numerically equal to arrow::StatusCode) ------------- */
typedef int32_t gdv_status;
#define GDV_OK 0
#define GDV_OUT_OF_MEMORY 1
#define GDV_INVALID 4
#define GDV_NOT_IMPLEMENTED 10
#define GDV_CODEGEN_ERROR 40              /* arrow::StatusCode::CodeGenError */
#define GDV_EXPRESSION_VALIDATION_ERROR 41 /* ExpressionValidationError */
#define GDV_EXECUTION_ERROR 42            /* ExecutionError */
#define GDV_CUDA_ERROR 100                /* driver / NVRTC unavailable or failed */

/* ---- data types (ids numerically equal to arrow::Type::type) ----------- */
#define GDV_TYPE_NA 0
#define GDV_TYPE_BOOL 1
#define GDV_TYPE_UINT8 2
#define GDV_TYPE_INT8 3
#define GDV_TYPE_UINT16 4
#define GDV_TYPE_INT16 5
#define GDV_TYPE_UINT32 6
#define GDV_TYPE_INT32 7
#define GDV_TYPE_UINT64 8
#define GDV_TYPE_INT64 9
#define GDV_TYPE_FLOAT 11
#define GDV_TYPE_DOUBLE 12
#define GDV_TYPE_STRING 13
#define GDV_TYPE_BINARY 14
#define GDV_TYPE_DATE32 16
#define GDV_TYPE_DATE64 17
#define GDV_TYPE_TIMESTAMP 18
#define GDV_TYPE_TIME32 19
#define GDV_TYPE_TIME64 20
#define GDV_TYPE_DECIMAL128 23
/* Dictionary-encoded column (arrow::DictionaryType): precision = index type id (GDV_TYPE_INT8,
 * INT16, INT32 or INT64), OR'ed with GDV_DICT_ORDERED for an ordered dictionary; scale = value
 * type id (GDV_TYPE_STRING or GDV_TYPE_BINARY).  Input columns only: functions resolve against
 * the value type, and results are plain utf8 / binary.  Any other value or index type, and a
 * dictionary result type, is refused at Make() with GDV_NOT_IMPLEMENTED. */
#define GDV_TYPE_DICTIONARY 29
#define GDV_DICT_ORDERED 0x100
/* Arrow's 16-byte view layouts of utf8 / binary (arrow::StringViewType, BinaryViewType; C format
 * "vu" / "vz"), described by gdv_view_buffers_t.  Input columns only, like dictionary columns:
 * functions resolve against utf8 / binary, and results are plain utf8 / binary.  A view result
 * type is refused at Make() with GDV_NOT_IMPLEMENTED. */
#define GDV_TYPE_STRING_VIEW 39
#define GDV_TYPE_BINARY_VIEW 40
/* Arrow's int64-offset layouts of utf8 / binary (arrow::LargeStringType, LargeBinaryType; C format
 * "U" / "Z"): the utf8 / binary layout with int64 offsets, so a column may hold more than 2^31 - 1
 * bytes.  Functions, IN and if/else resolve against utf8 / binary.  An expression's result field may
 * be large_string / large_binary when its root yields utf8 / binary; a function, if/else or literal
 * node with a large return type is refused at Make() with GDV_NOT_IMPLEMENTED. */
#define GDV_TYPE_LARGE_STRING 34
#define GDV_TYPE_LARGE_BINARY 35

typedef struct gdv_type {
  int32_t id;        /* GDV_TYPE_* */
  int32_t precision; /* decimal128: precision; timestamp/time: arrow::TimeUnit (0=s,1=ms,2=us,3=ns);
                        dictionary: index type id (| GDV_DICT_ORDERED) */
  int32_t scale;     /* decimal128: scale; dictionary: value type id */
} gdv_type_t;

/* ---- opaque handles ----------------------------------------------------- */
typedef struct gdv_node_s* gdv_node_t;
typedef struct gdv_expression_s* gdv_expression_t;
typedef struct gdv_condition_s* gdv_condition_t;
typedef struct gdv_schema_s* gdv_schema_t;
typedef struct gdv_projector_s* gdv_projector_t;
typedef struct gdv_filter_s* gdv_filter_t;
typedef struct gdv_function_registry_s* gdv_function_registry_t;

/* ---- configuration (gandiva::Configuration + device placement) --------- */
typedef struct gdv_config {
  int32_t optimize;     /* reference option; here: ptxas -O3 (1) or -O0 (0) */
  int32_t dump_ir;      /* keep generated CUDA source + PTX for DumpIR */
  int32_t device;       /* CUDA device ordinal (default 0) */
  int32_t rows_per_thread; /* 0 = engine picks; otherwise unroll factor override */
  int32_t block_threads;   /* 0 = engine picks (256) */
  int32_t loader;          /* Projector: 0 = engine picks; 1 = direct coalesced LDG; 2 = TMA bulk -> shared */
  int32_t sm_reserve;      /* SMs left without CTAs of the persistent kernels, so that a
                              concurrent stream (e.g. the push of the previous batch's
                              SelectionVector) can run; default 0 */
  int32_t stages;          /* Projector, TMA loader: shared-memory stages per CTA (0 = engine picks).
                              Fixed-width Filter: 1 / 2 / 4 / 8 = 1024-row chunks every warp walks per
                              tile (0 = engine picks: 4 on batches >= 32 M rows, else 1) */
  int32_t string_scan;     /* string columns, bit mask; 0 = engine picks (everything on):
                              bit 0: LIKE with the per-lane matcher only (no warp-cooperative scan),
                              bit 2: row-driven string Filter kernel even where the condition implies a
                                     literal and the key-driven kernel (driven by the literal's
                                     occurrences in the column's bytes) would apply,
                              bit 3 (value 8): string_view / binary_view columns: no inline / prefix
                                     shortcut; equal, IN, starts_with and LIKE 'lit%...' read the row's
                                     bytes through the view like any other string function */
  int32_t filter_gating;   /* fixed-width Filter: 0 = engine decides (gated loads wherever they apply: a
                              conjunct's columns are read only in rows the earlier conjuncts kept),
                              1 = off (every column read for every row; the reference kernel) */
  gdv_function_registry_t function_registry; /* user functions looked up after the built-ins (see
                              gdv_function_registry_add); NULL = none.  These 8 bytes at offset 40 were
                              `int32_t reserved[2]`: the struct keeps its size, and a caller that zeroes it or
                              calls gdv_config_default keeps the built-in library only. */
} gdv_config_t;
void gdv_config_default(gdv_config_t* cfg);

/* ---- selection-vector modes -------------------------------------------- */
#define GDV_SEL_NONE 0
#define GDV_SEL_UINT16 1
#define GDV_SEL_UINT32 2
#define GDV_SEL_UINT64 3
/* OR'ed into gdv_selection_t.mode for Filter evaluation with device buffers: max_slots may be
 * smaller than num_rows; selected rows past max_slots are counted but not stored (the caller
 * detects overflow by num_slots > max_slots).  Used by row-range shards that write into one
 * shared SelectionVector. */
#define GDV_SEL_BOUNDED 0x100

/* ---- memory spaces of the buffers handed to Evaluate ------------------- */
#define GDV_MEM_HOST 0   /* pageable or pinned host memory: engine stages H2D/D2H */
#define GDV_MEM_DEVICE 1 /* buffers already live in the HBM of cfg.device */

/* One Arrow array, as its raw buffers (arrow::ArrayData, P/include/arrow/array/data.h:468-474).
 *  fixed width : validity | values                (values = buffers[1])
 *  bool        : validity | bit-packed values
 *  utf8/binary : validity | int32 offsets | bytes (values = offsets, var_data = bytes)
 *  large_string / large_binary : validity | int64 offsets | bytes (values = offsets, var_data = bytes,
 *                var_data_size).  A non-null row whose length offsets[r+1] - offsets[r] is negative
 *                or above INT32_MAX is invalid input here (a row's string is at most 2^31 - 1 bytes):
 *                it reads as null and its bytes are never read.  Offsets are non-decreasing otherwise,
 *                as Arrow requires.
 *  string_view / binary_view : validity | 16-byte views | var_data = gdv_view_buffers_t* (below)
 * `offset` is ArrayData::offset (in elements/bits), applied to every buffer.
 * validity may be NULL (no nulls). */
typedef struct gdv_column {
  const void* validity;
  const void* values;
  const void* var_data;
  int64_t offset;
  int64_t var_data_size; /* bytes in var_data (needed to stage host strings); 0 otherwise */
} gdv_column_t;

/* The dictionary of a dictionary-encoded column (schema type GDV_TYPE_DICTIONARY): a utf8 /
 * binary array in the batch's memory space, described like a gdv_column_t plus its length.
 * The column itself is
 *  dictionary  : validity | signed int8/16/32/64 indices (values) | var_data = const gdv_dictionary_t*
 * with `offset` applying to the indices and this struct's `offset` to the dictionary, so the
 * layout of gdv_column_t / gdv_batch_t is the same for every column kind.  Row r is
 * dictionary[indices[r]]; it is null when the index slot or the dictionary entry is null, and
 * also when the index lies outside [0, length) (invalid Arrow input: never dereferenced).  Host
 * batches stage the three dictionary buffers with the indices; device batches read them in place.
 * The struct is read during the Evaluate call only (host memory). */
typedef struct gdv_dictionary {
  const void* validity;  /* may be NULL (no null entries) */
  const void* offsets;   /* length + 1 int32 offsets, from `offset` on */
  const void* data;      /* the bytes the offsets index */
  int64_t offset;        /* ArrayData::offset of the dictionary */
  int64_t length;        /* entries */
  int64_t data_size;     /* bytes in data (needed to stage host dictionaries) */
} gdv_dictionary_t;

/* The data buffers of a string_view / binary_view column (GDV_TYPE_STRING_VIEW / BINARY_VIEW).
 * The column itself is
 *  view        : validity | 16-byte views (values) | var_data = const gdv_view_buffers_t*
 * with `offset` applying to the validity and the views.  A view is {int32 len, then either the
 * len <= 12 bytes inline (zero padded), or a 4-byte prefix, int32 buffer index and int32 offset into
 * data[buffer index]}.  A non-null view is invalid Arrow input when len < 0, or when len > 12 and the
 * buffer index is outside [0, n), the offset is negative or offset + len > sizes[buffer index]: its
 * row reads as null and nothing is dereferenced for it.  Null slots are never read through.  Host
 * batches stage the validity, the views and every data buffer whole (a sliced batch may carry bytes
 * no row in the slice uses); device batches read them in place.  The struct is read during the
 * Evaluate call only. */
typedef struct gdv_view_buffers {
  const void* const* data; /* host array of n buffer pointers, in the batch's memory space */
  const int64_t* sizes;    /* n byte sizes, in the batch's memory space */
  int32_t n;               /* data buffers (may be 0: every view is inline) */
} gdv_view_buffers_t;

typedef struct gdv_batch {
  int64_t num_rows;
  int32_t num_columns; /* must equal the schema's field count, same order */
  int32_t mem_space;   /* GDV_MEM_* */
  const gdv_column_t* columns;
} gdv_batch_t;

/* Caller-allocated output array (Projector::Evaluate allocates these from the
 * MemoryPool in the C++ layer).  Output offset is always 0.
 *  validity : ceil(n/8) bytes rounded up to 8; may be NULL -> validity not written
 *  values   : n*width bytes (bool: ceil(n/8) rounded up to 8); utf8: (n+1) int32 offsets;
 *             large_string / large_binary: (n+1) int64 offsets (no 2^31 - 1 byte limit)
 *  var_data : utf8/binary outputs only, capacity var_capacity bytes */
typedef struct gdv_out_column {
  void* validity;
  void* values;
  void* var_data;
  int64_t var_capacity;
  int64_t var_size; /* out: bytes produced (utf8/binary) */
} gdv_out_column_t;

/* Selection vector storage (gandiva::SelectionVector): ascending row indices. */
typedef struct gdv_selection {
  void* indices;      /* uint16/uint32/uint64 per mode; host or device per mem_space */
  int64_t max_slots;  /* capacity in indices */
  int64_t num_slots;  /* in: slots to read (projector); out: slots written (filter) */
  int32_t mode;       /* GDV_SEL_* */
  int32_t mem_space;  /* GDV_MEM_* */
  int64_t index_base; /* filter: added to every emitted index (row-range sharding: the
                         shard's first global row); projector: ignored */
  const void* d_num_slots; /* projector, device buffers, may be NULL: device uint64 holding the slot
                         count (e.g. the d_count a Filter wrote on the same stream).  The kernel reads
                         it on the device, so a Filter -> Projector chain needs no host round trip;
                         num_slots is then only an upper bound (grid size, output capacity): the kernels
                         use c = min(*d_num_slots, num_slots) rows.  Rows past c are not written: no
                         value, no offset past offsets[c], no byte past offsets[c], no validity word that
                         lies wholly past c (in the word holding row c-1 the bits past it are 0).
                         utf8/binary outputs: values holds num_slots + 1 int32 offsets (int64 for
                         large_string / large_binary) and var_data
                         var_capacity bytes, an upper bound the caller picks; the byte total is
                         offsets[c].  var_size is the total after a synchronous call, -1 after an async
                         one.  A total above var_capacity is an ExecutionError (from the call when it is
                         synchronous, else from gdv_projector_sync) and no byte past var_capacity is
                         stored.  gdv_projector_output_var_size over a d_num_slots selection returns the
                         exact total (one round trip).  Device buffers only (GDV_INVALID otherwise);
                         utf8/binary outputs of a projector that materialises rope temporaries (the
                         two-stage rope plan) refuse it with GDV_NOT_IMPLEMENTED. */
} gdv_selection_t;

/* ---- library / device ---------------------------------------------------- */
const char* gdv_version(void);
const char* gdv_last_error(void);
/* 1 when libcuda + a device are usable, 0 otherwise (never fails). */
int32_t gdv_cuda_available(void);
int32_t gdv_device_count(void);

/* ---- TreeExprBuilder ---------------------------------------------------- */
gdv_status gdv_node_field(const char* name, gdv_type_t type, gdv_node_t* out);
/* Literals: `value` points at the C value of the type (bool: uint8_t, intN: intN_t,
 * float/double, date/time as their storage int; decimal128: 16 little-endian bytes;
 * string/binary: bytes with `len`).  is_null != 0 makes a typed null literal. */
gdv_status gdv_node_literal(gdv_type_t type, const void* value, int64_t len, int32_t is_null,
                            gdv_node_t* out);
gdv_status gdv_node_function(const char* name, const gdv_node_t* children, int32_t n_children,
                             gdv_type_t return_type, gdv_node_t* out);
gdv_status gdv_node_if(gdv_node_t condition, gdv_node_t then_node, gdv_node_t else_node,
                       gdv_type_t return_type, gdv_node_t* out);
gdv_status gdv_node_and(const gdv_node_t* children, int32_t n_children, gdv_node_t* out);
gdv_status gdv_node_or(const gdv_node_t* children, int32_t n_children, gdv_node_t* out);
/* IN expression.  Fixed-width: `values` is n_values packed values of `type`.
 * string/binary: `values` is the concatenated bytes, `lengths` the n_values lengths. */
gdv_status gdv_node_in(gdv_node_t child, gdv_type_t type, const void* values,
                       const int32_t* lengths, int32_t n_values, gdv_node_t* out);
gdv_status gdv_node_return_type(gdv_node_t node, gdv_type_t* out);
/* Writes a NUL-terminated string; returns the full length needed (excluding NUL). */
int64_t gdv_node_to_string(gdv_node_t node, char* buf, int64_t buf_len);
void gdv_node_release(gdv_node_t node);

gdv_status gdv_expression_make(gdv_node_t root, const char* result_name, gdv_type_t result_type,
                               gdv_expression_t* out);
int64_t gdv_expression_to_string(gdv_expression_t e, char* buf, int64_t buf_len);
void gdv_expression_release(gdv_expression_t e);
gdv_status gdv_condition_make(gdv_node_t root, gdv_condition_t* out);
int64_t gdv_condition_to_string(gdv_condition_t c, char* buf, int64_t buf_len);
void gdv_condition_release(gdv_condition_t c);

/* ---- schema ------------------------------------------------------------- */
gdv_status gdv_schema_make(const char* const* names, const gdv_type_t* types, int32_t n_fields,
                           gdv_schema_t* out);
void gdv_schema_release(gdv_schema_t s);

/* ---- Projector ---------------------------------------------------------- */
gdv_status gdv_projector_make(gdv_schema_t schema, const gdv_expression_t* exprs, int32_t n_exprs,
                              int32_t selection_mode, const gdv_config_t* cfg,
                              gdv_projector_t* out);
/* Evaluate.  `selection` NULL (mode NONE) or a selection vector of the mode given at Make.
 * `stream` is a CUstream/cudaStream_t; NULL = the engine's own non-blocking stream (pass
 * CU_STREAM_LEGACY, (void*)0x1, to name CUDA's default stream explicitly).  With host
 * buffers the call is synchronous.  With device buffers and `async` != 0 it only
 * enqueues work on `stream`; errors raised by device functions are then reported
 * by gdv_projector_sync(). */
gdv_status gdv_projector_evaluate(gdv_projector_t p, const gdv_batch_t* batch,
                                  const gdv_selection_t* selection, gdv_out_column_t* outs,
                                  int32_t n_outs, void* stream, int32_t async);
gdv_status gdv_projector_sync(gdv_projector_t p, void* stream);
/* Bytes needed for output i's var_data given the batch (utf8/binary outputs): runs the
 * sizing pass and the scan, then synchronises the stream.  Fixed-width outputs return 0.  With
 * selection->d_num_slots it sizes the rows of the device count: the opt-in path for a caller of a
 * device-resident Filter -> Projector chain who wants an exact buffer rather than an upper bound,
 * at the cost of one host round trip. */
gdv_status gdv_projector_output_var_size(gdv_projector_t p, const gdv_batch_t* batch,
                                         const gdv_selection_t* selection, int32_t out_index,
                                         void* stream, int64_t* out_bytes);
int64_t gdv_projector_dump_ir(gdv_projector_t p, char* buf, int64_t buf_len);
/* Name of the generated kernel, its registers/thread and static shared memory. */
gdv_status gdv_projector_kernel_info(gdv_projector_t p, char* name_buf, int64_t name_len,
                                     int32_t* regs, int32_t* smem_bytes, int32_t* rows_per_thread,
                                     int32_t* block_threads);
/* Integer attribute of the kernel variant used by the latest Evaluate: "staged" (1 = TMA bulk
 * loader), "stages", "dynamic_smem", "cta_tile_rows", "tile_rows", "nullable",
 * "in_bytes_per_row", "view_shortcuts" (call sites decided from the 16-byte views of string_view /
 * binary_view columns: equal, IN, starts_with, LIKE 'lit%...'), "gated_stages" (fixed-width Filter:
 * stages of gated loads, 0 = not gated), "blocks_per_sm" (needs a device). */
gdv_status gdv_projector_kernel_attr(gdv_projector_t p, const char* key, int64_t* out);
void gdv_projector_release(gdv_projector_t p);

/* ---- Filter --------------------------------------------------------------- */
gdv_status gdv_filter_make(gdv_schema_t schema, gdv_condition_t condition, const gdv_config_t* cfg,
                           gdv_filter_t* out);
/* Fills `out_selection->indices` (capacity max_slots >= batch->num_rows) with the ascending
 * indices of rows whose condition is true and valid; sets num_slots.  With device buffers and
 * async != 0, num_slots is written to `d_count` (device uint64_t*, may be NULL) when the stream
 * reaches that point and out_selection->num_slots is left at -1; gdv_filter_sync() returns it. */
gdv_status gdv_filter_evaluate(gdv_filter_t f, const gdv_batch_t* batch,
                               gdv_selection_t* out_selection, void* stream, int32_t async,
                               void* d_count);
gdv_status gdv_filter_sync(gdv_filter_t f, void* stream, int64_t* num_slots);
int64_t gdv_filter_dump_ir(gdv_filter_t f, char* buf, int64_t buf_len);
gdv_status gdv_filter_kernel_info(gdv_filter_t f, char* name_buf, int64_t name_len, int32_t* regs,
                                  int32_t* smem_bytes, int32_t* rows_per_thread,
                                  int32_t* block_threads);
/* Same keys as gdv_projector_kernel_attr, plus "dictionary_first": 1 when the latest Evaluate kept rows
 * through the dictionary-first kernel (a condition over one dictionary column, evaluated once per entry). */
gdv_status gdv_filter_kernel_attr(gdv_filter_t f, const char* key, int64_t* out);
void gdv_filter_release(gdv_filter_t f);

/* ---- function registry (ExpressionRegistry) ------------------------------ */
int32_t gdv_registry_size(void);
/* Signature i: name, return type, parameter types (up to max_params written; returns count). */
gdv_status gdv_registry_get(int32_t i, const char** name, gdv_type_t* ret, gdv_type_t* params,
                            int32_t max_params, int32_t* n_params);

/* ---- user-defined functions ----------------------------------------------------------------
 * A function registry holds functions the caller adds to the engine as CUDA text.  A Projector or
 * Filter made with gdv_config_t.function_registry set resolves a function name against the built-ins
 * first and the registry second, and the fuser writes every user function a kernel calls into that
 * kernel's source (gdv_*_dump_ir shows it), where NVRTC inlines it like a built-in.  The global
 * enumeration above never changes.  User code runs inside the engine's kernels with the engine's
 * privileges: a registry is for trusted callers, exactly like linking a library.
 *
 * The caller writes the statements of the function; the engine writes the signature.
 *   - parameter i is `a<i>`: bool, i8..i64 / u8..u64, f32, f64 (date32 / time32 are i32; date64 /
 *     timestamp are i64), `const gdv_str&` for utf8 / binary: s.len bytes, byte i is gdv_ch(s, i)
 *     (never s.p[i]: upper / lower / initcap views re-case bytes as they are read).  The same text
 *     serves plain, sliced, dictionary-encoded and string_view / binary_view columns.
 *   - GDV_NULL_IF_NULL  T f(a0, a1, ...)                     result is null iff an argument is null;
 *                                                            arguments of null rows are unspecified
 *   - GDV_NULL_NEVER    T f(a0, bool v0, a1, bool v1, ...)   v<i> = argument i is valid; never null
 *   - GDV_NULL_INTERNAL T f(a0, bool v0, ..., bool* out_valid)   *out_valid (preset to false) = result
 *                                                            is valid
 *   - can_raise: `gdv_ctx* ctx` comes first; gdv_raise(ctx, "message") makes the evaluation fail with
 *     GDV_EXECUTION_ERROR and that message (at most 239 bytes; the first raise wins).  Such a function
 *     is called only for rows of the batch that reach it (not in the untaken branch of an if, not
 *     past a decided and / or), and with GDV_NULL_IF_NULL only where every argument is valid.
 *   - prelude: file-scope text written once before the function (helpers, __constant__ tables).
 * Types: fixed-width parameters and results, utf8 / binary parameters.  utf8 / binary / decimal128
 * results and decimal128 parameters are refused with GDV_NOT_IMPLEMENTED.  A built-in's name cannot
 * be reused, whatever the parameter types.  Everything is compiled with --fmad=false like the
 * engine's own code.
 *
 * gdv_function_registry_add validates and compiles the function once for sm_90a (no GPU needed): text
 * that does not compile is refused there with GDV_CODEGEN_ERROR and NVRTC's log in gdv_last_error().
 * Functions can be added until the first gdv_projector_make / gdv_filter_make that is given the
 * registry; from then on the registry is read-only (add fails with GDV_INVALID) and may be shared by
 * any number of threads.  Projectors and Filters keep what they need: the handle may be released
 * while they live.
 *
 *   gdv_function_registry_t reg;
 *   gdv_function_registry_create(&reg);
 *   gdv_type_t f64 = {GDV_TYPE_DOUBLE, 0, 0};
 *   gdv_function_def_t def = {0};
 *   def.name = "fahrenheit";  def.params = &f64;  def.n_params = 1;  def.ret = f64;
 *   def.null_mode = GDV_NULL_IF_NULL;
 *   def.body = "return a0 * 1.8 + 32.0;";
 *   gdv_function_registry_add(reg, &def);
 *   gdv_config_t cfg;  gdv_config_default(&cfg);  cfg.function_registry = reg;
 *   // gdv_node_function("fahrenheit", &celsius, 1, f64, &node) ... gdv_projector_make(..., &cfg, &p)
 */
#define GDV_NULL_IF_NULL 0
#define GDV_NULL_NEVER 1
#define GDV_NULL_INTERNAL 2
typedef struct gdv_function_def {
  const char* name;
  const gdv_type_t* params;
  int32_t n_params;
  gdv_type_t ret;
  int32_t null_mode; /* GDV_NULL_* */
  int32_t can_raise;
  const char* body;
  const char* prelude; /* may be NULL */
} gdv_function_def_t;
gdv_status gdv_function_registry_create(gdv_function_registry_t* out);
void gdv_function_registry_release(gdv_function_registry_t reg);
gdv_status gdv_function_registry_add(gdv_function_registry_t reg, const gdv_function_def_t* def);
/* Enumeration of this registry only: gdv_function_registry_signatures returns the count; signature i
 * as in gdv_registry_get. */
int32_t gdv_function_registry_signatures(gdv_function_registry_t reg);
gdv_status gdv_function_registry_get(gdv_function_registry_t reg, int32_t i, const char** name, gdv_type_t* ret,
                                     gdv_type_t* params, int32_t max_params, int32_t* n_params);

/* ---- device memory (the engine's pooled allocator; what the C++ layer's arrow::MemoryManager
 *      for HBM, include/gandiva/device.h, allocates from) ---------------------------------- */
gdv_status gdv_device_alloc(int32_t device, size_t bytes, void** out);
gdv_status gdv_device_free(int32_t device, void* p);
/* Returns idle pool blocks to the driver until at most keep_bytes stay cached (the pool also trims
 * itself above GDV_POOL_LIMIT_MB, default 4096); *released (may be NULL) = bytes given back. */
gdv_status gdv_device_trim(int32_t device, size_t keep_bytes, size_t* released);
/* Copy between host and device memory on the engine's stream, synchronously.
 * kind 1 = host -> device, 2 = device -> host. */
gdv_status gdv_memcpy(int32_t device, void* dst, const void* src, size_t bytes, int32_t kind);

/* ---- device helpers used by the harness (bench.py, tests) ---------------- */
/* Pinned host memory (cuMemHostAlloc) so H2D staging runs at PCIe speed. */
gdv_status gdv_host_alloc(size_t bytes, void** out);
gdv_status gdv_host_free(void* p);
/* Bytes that host batches in PAGEABLE memory have moved through the pinned staging ring since the
 * library was loaded (csrc/gdv_staging.cc); pinned and device-resident batches never add to it. */
int64_t gdv_staged_bytes(void);
/* Synthetic TPC-H lineitem columns generated straight into device memory (counter-based
 * hash RNG, identical stream to oracle/lineitem.c):
 *  kind 0: l_shipdate date32  1: l_discount f64  2: l_quantity f64 ... see DESIGN.md */
gdv_status gdv_generate_lineitem(int32_t device, int32_t column_kind, uint64_t seed,
                                 int64_t first_row, int64_t num_rows, void* d_values,
                                 void* d_validity, int32_t null_permille, void* stream);
/* ---- SelectionVector reassembly across row-range shards (one process per GPU) -----------
 * Replaces nothing in the reference (it is single-node CPU); BASELINE.json north_star asks for
 * "row-range-shards a batch across the 8 GPUs of one box, with an optional ... gather over
 * NVLink to reassemble the SelectionVector".  Each rank filters its row range with
 * gdv_filter_evaluate (index_base = first row of the range) into a local run, then calls
 * gdv_selection_push on a side stream: the kernel reads the lower ranks' counts from the board,
 * and stores the run at its final offset of the root's vector `d_dst` (peer-mapped memory of the
 * root GPU, e.g. through CUDA IPC) over NVLink.  No host round trip, no collective library.
 *  board       : GDV_BOARD_BYTES of zero-initialised memory on the root GPU, mapped by every rank
 *  board_slot  : which of the GDV_BOARD_SLOTS in-flight steps this is (step % slots)
 *  seq         : step number + 1 (strictly increasing; board words are never reset)
 *  need_consumed: 0, or the seq the root must have released for this slot before d_dst is
 *                overwritten (seq - GDV_BOARD_SLOTS in a ring of buffers)
 *  rank 0 (root): its filter wrote straight into d_dst (offset 0); the call waits on the device
 *                for every rank's run and writes the total to d_total_out (device uint64).
 *  ctas        : CTAs of the copy kernel on non-root ranks (leave that many SMs free with
 *                gdv_config_t.sm_reserve so it overlaps the next batch's filter kernel)
 *  d_local_counter: zero-initialised device uint64 owned by the calling rank; every CTA of every
 *                push adds one to it.  done_target: the value it reaches when this call's last
 *                CTA has finished (= sum of `ctas` over all pushes issued so far, this one
 *                included), so `ctas` may differ from call to call.
 *  d_base      : NULL = the vector is one run per rank (above).  Otherwise the batch is filtered in
 *                several WAVES (row slices, wave-major global row order) so that the transfer of
 *                wave j hides under the filter kernel of wave j+1 and only the last wave's
 *                transfer is exposed: d_base is a device uint64 owned by the calling rank that
 *                carries the vector's fill level from wave to wave; every rank, the root included
 *                (its filter then writes a local run like everyone else), stores this wave's run
 *                at *d_base + the lower ranks' runs of this wave and then adds the wave's total.
 *                Each wave is one call with its own seq; board_slot = seq % GDV_BOARD_SLOTS;
 *                consumed_slot = which vector of the ring (need_consumed only on the first wave).
 *  wave_flags  : GDV_WAVE_FIRST starts a vector, GDV_WAVE_LAST completes it (the root waits for
 *                every rank and writes d_total_out). */
#define GDV_WAVE_FIRST 1
#define GDV_WAVE_LAST 2
/* Lets kernels running on `device` dereference memory of `peer_device` (cuCtxEnablePeerAccess);
 * required once per process before gdv_selection_push stores into the root's vector. */
gdv_status gdv_enable_peer_access(int32_t device, int32_t peer_device);
/* CUDA IPC plumbing for the above (one process per GPU).  The root exports the allocation that
 * holds `d_ptr` (64-byte handle + byte offset of d_ptr inside it); every other rank opens it with
 * its own device current: the memory is mapped into that device's address space with NVLink peer
 * access to the root GPU enabled (CU_IPC_MEM_LAZY_ENABLE_PEER_ACCESS). */
gdv_status gdv_ipc_export(int32_t device, const void* d_ptr, uint8_t* handle64, int64_t* offset);
gdv_status gdv_ipc_open(int32_t device, const uint8_t* handle64, int64_t offset, void** out_ptr);
gdv_status gdv_ipc_close(int32_t device, void* d_ptr, int64_t offset);
#define GDV_BOARD_MAX_WORLD 16
#define GDV_BOARD_SLOTS 4
#define GDV_BOARD_BYTES ((2 * GDV_BOARD_SLOTS * GDV_BOARD_MAX_WORLD + GDV_BOARD_SLOTS + 1) * 8)
gdv_status gdv_selection_push(int32_t device, const void* d_src, const void* d_count, void* d_dst,
                              int64_t dst_capacity, void* board, int32_t board_slot, int32_t rank,
                              int32_t world, uint64_t seq, uint64_t need_consumed, int32_t mode,
                              int32_t ctas, void* d_local_counter, uint64_t done_target,
                              void* d_total_out, void* d_base, int32_t wave_flags,
                              int32_t consumed_slot, void* stream);
/* root: marks slot `board_slot`'s vector of step `seq` as consumed (its buffer may be reused). */
gdv_status gdv_selection_release(int32_t device, void* board, int32_t board_slot, uint64_t seq,
                                 void* stream);
/* Number of kernels this library has launched since load (gpu_launches in bench.py). */
int64_t gdv_launch_count(void);
/* Number of NVRTC compilations since load.  Make() calls that lower to a kernel already built in
 * this process (same generated source, architecture and options) reuse its cubin: the counterpart
 * of the reference's projector / filter cache. */
int64_t gdv_compile_count(void);

#ifdef __cplusplus
}
#endif
#endif /* GANDIVA_B200_H */
