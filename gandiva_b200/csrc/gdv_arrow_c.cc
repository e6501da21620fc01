// Arrow C Data / C Device Data interface ingestion (include/gandiva_b200_arrow.h).
//
// A struct-typed ArrowDeviceArray is turned into the engine's gdv_batch_t without touching the
// buffers: device buffers stay where the producer put them (GDV_MEM_DEVICE), results are exported
// back as an ArrowDeviceArray whose buffers come from the engine's pooled device allocator.
// Layout facts used here: P/include/arrow/c/abi.h:68-121 (ArrowSchema / ArrowArray),
// :140-287 (ArrowDeviceArray: device_id, device_type, sync_event = cudaEvent_t*).
#include <cstdlib>
#include <cstring>
#include <memory>
#include <string>
#include <vector>

#include "gandiva_b200_arrow.h"
#include "gdv_capi_internal.h"

using namespace gdv;
using namespace gdv::capi;

namespace {

// ---- format strings <-> DataType ---------------------------------------------------------
Status ParseFormat(const char* f, DataType* out) {
  const std::string s(f ? f : "");
  auto unit = [](char c, int* u) {
    switch (c) {
      case 's': *u = 0; return true;
      case 'm': *u = 1; return true;
      case 'u': *u = 2; return true;
      case 'n': *u = 3; return true;
      default: return false;
    }
  };
  if (s == "b") { *out = DataType(GDV_TYPE_BOOL); return Status::OK(); }
  if (s == "c") { *out = DataType(GDV_TYPE_INT8); return Status::OK(); }
  if (s == "C") { *out = DataType(GDV_TYPE_UINT8); return Status::OK(); }
  if (s == "s") { *out = DataType(GDV_TYPE_INT16); return Status::OK(); }
  if (s == "S") { *out = DataType(GDV_TYPE_UINT16); return Status::OK(); }
  if (s == "i") { *out = DataType(GDV_TYPE_INT32); return Status::OK(); }
  if (s == "I") { *out = DataType(GDV_TYPE_UINT32); return Status::OK(); }
  if (s == "l") { *out = DataType(GDV_TYPE_INT64); return Status::OK(); }
  if (s == "L") { *out = DataType(GDV_TYPE_UINT64); return Status::OK(); }
  if (s == "f") { *out = DataType(GDV_TYPE_FLOAT); return Status::OK(); }
  if (s == "g") { *out = DataType(GDV_TYPE_DOUBLE); return Status::OK(); }
  if (s == "u") { *out = DataType(GDV_TYPE_STRING); return Status::OK(); }
  if (s == "z") { *out = DataType(GDV_TYPE_BINARY); return Status::OK(); }
  if (s == "vu") { *out = DataType(gdv_type_t{GDV_TYPE_STRING_VIEW, 0, 0}); return Status::OK(); }
  if (s == "vz") { *out = DataType(gdv_type_t{GDV_TYPE_BINARY_VIEW, 0, 0}); return Status::OK(); }
  if (s == "tdD") { *out = DataType(GDV_TYPE_DATE32); return Status::OK(); }
  if (s == "tdm") { *out = DataType(GDV_TYPE_DATE64); return Status::OK(); }
  int u = 0;
  if (s.size() >= 4 && s.compare(0, 2, "ts") == 0 && unit(s[2], &u) && s[3] == ':') {
    *out = DataType(GDV_TYPE_TIMESTAMP, u);
    return Status::OK();
  }
  if (s.size() == 3 && s.compare(0, 2, "tt") == 0 && unit(s[2], &u)) {
    *out = DataType(u <= 1 ? GDV_TYPE_TIME32 : GDV_TYPE_TIME64, u);
    return Status::OK();
  }
  if (s.size() > 2 && s.compare(0, 2, "d:") == 0) {
    int p = 0, sc = 0, bits = 128;
    const int got = std::sscanf(s.c_str() + 2, "%d,%d,%d", &p, &sc, &bits);
    if (got >= 2 && bits == 128 && p >= 1 && p <= 38) {
      *out = DataType(GDV_TYPE_DECIMAL128, p, sc);
      return Status::OK();
    }
  }
  return Status::Make(GDV_NOT_IMPLEMENTED, "Arrow format string '" + s + "' is not supported");
}

// The Arrow C Device interface speaks int32-offset utf8 / binary only: a projector with a
// large_string / large_binary result is refused there.
Status RefuseLargeOutputs(const std::vector<ExpressionPtr>& exprs) {
  for (const auto& e : exprs)
    if (e->result().type.is_large())
      return Status::Make(GDV_NOT_IMPLEMENTED, "output '" + e->result().name + "' is " + e->result().type.ToString() +
                                                   ": the Arrow C Device interface takes utf8 / binary outputs only");
  return Status::OK();
}

std::string FormatOf(const DataType& t) {
  static const char kUnit[] = {'s', 'm', 'u', 'n'};
  if (t.is_view()) return t.id == GDV_TYPE_BINARY ? "vz" : "vu";
  switch (t.id) {
    case GDV_TYPE_BOOL: return "b";
    case GDV_TYPE_INT8: return "c";
    case GDV_TYPE_UINT8: return "C";
    case GDV_TYPE_INT16: return "s";
    case GDV_TYPE_UINT16: return "S";
    case GDV_TYPE_INT32: return "i";
    case GDV_TYPE_UINT32: return "I";
    case GDV_TYPE_INT64: return "l";
    case GDV_TYPE_UINT64: return "L";
    case GDV_TYPE_FLOAT: return "f";
    case GDV_TYPE_DOUBLE: return "g";
    case GDV_TYPE_STRING: return "u";
    case GDV_TYPE_BINARY: return "z";
    case GDV_TYPE_DATE32: return "tdD";
    case GDV_TYPE_DATE64: return "tdm";
    case GDV_TYPE_TIMESTAMP: return std::string("ts") + kUnit[t.precision & 3] + ":";
    case GDV_TYPE_TIME32:
    case GDV_TYPE_TIME64: return std::string("tt") + kUnit[t.precision & 3];
    case GDV_TYPE_DECIMAL128:
      return "d:" + std::to_string(t.precision) + "," + std::to_string(t.scale);
    default: return "n";
  }
}

// ---- exported ArrowSchema ("+s" with flat children) ------------------------------------
struct SchemaPriv {
  std::vector<std::string> formats, names;
  std::vector<ArrowSchema> children;
  std::vector<ArrowSchema*> child_ptrs;
};
void ReleaseChildSchema(ArrowSchema* s) { s->release = nullptr; }
void ReleaseSchema(ArrowSchema* s) {
  if (s == nullptr || s->release == nullptr) return;
  SchemaPriv* p = static_cast<SchemaPriv*>(s->private_data);
  for (auto& c : p->children)
    if (c.release != nullptr) c.release(&c);
  delete p;
  s->release = nullptr;
}

// ---- imported batch -------------------------------------------------------------------------
}  // namespace

struct gdv_arrow_batch_s {
  ArrowDeviceArray array;  // moved from the producer's struct
  SchemaPtr schema;
  std::vector<gdv_column_t> columns;
  std::vector<gdv_dictionary_t> dictionaries;  // dictionary columns' var_data points here
  std::vector<gdv_view_buffers_t> view_buffers;  // view columns' var_data points here
  gdv_batch_t view;
  int device = -1;  // CUDA ordinal, -1 for host memory
};

namespace {

// ---- exported ArrowDeviceArray ---------------------------------------------------------------
struct ArrayPriv {
  Device* dev = nullptr;               // non-null: buffers are pooled device blocks
  std::vector<CUdeviceptr> dev_blocks;
  std::vector<void*> host_blocks;
  std::vector<ArrowArray> children;
  std::vector<ArrowArray*> child_ptrs;
  std::vector<std::vector<const void*>> buffers;  // [0] = the parent's
};
void ReleaseChildArray(ArrowArray* a) { a->release = nullptr; }
void ReleaseArray(ArrowArray* a) {
  if (a == nullptr || a->release == nullptr) return;
  ArrayPriv* p = static_cast<ArrayPriv*>(a->private_data);
  for (auto& c : p->children)
    if (c.release != nullptr) c.release(&c);
  for (CUdeviceptr b : p->dev_blocks) p->dev->Free(b);
  for (void* b : p->host_blocks) std::free(b);
  delete p;
  a->release = nullptr;
}

// One output buffer in the memory space of the batch.
Status AllocOut(ArrayPriv* priv, bool device, size_t bytes, void** out) {
  bytes = (bytes + 63) / 64 * 64 + 64;
  if (device) {
    CUdeviceptr p = 0;
    Status s = priv->dev->Alloc(bytes, &p);
    if (!s.ok()) return s;
    priv->dev_blocks.push_back(p);
    *out = reinterpret_cast<void*>(p);
  } else {
    void* p = std::aligned_alloc(64, bytes);
    if (p == nullptr) return Status::Make(GDV_OUT_OF_MEMORY, "host allocation failed");
    priv->host_blocks.push_back(p);
    *out = p;
  }
  return Status::OK();
}

void InitDeviceArray(ArrowDeviceArray* out, gdv_arrow_batch_t in) {
  std::memset(out, 0, sizeof(*out));
  out->device_id = in->array.device_id;
  out->device_type = in->array.device_type;
  out->sync_event = nullptr;  // results are complete when the call returns
}

}  // namespace

extern "C" {

gdv_status gdv_schema_from_arrow(const struct ArrowSchema* schema, gdv_schema_t* out) {
  if (schema == nullptr || out == nullptr) return Fail(GDV_INVALID, "null argument");
  if (schema->release == nullptr) return Fail(GDV_INVALID, "ArrowSchema was already released");
  if (schema->format == nullptr || std::strcmp(schema->format, "+s") != 0)
    return Fail(GDV_INVALID, "expected a struct-typed ArrowSchema (format \"+s\")");
  std::vector<Field> fields;
  for (int64_t i = 0; i < schema->n_children; ++i) {
    const ArrowSchema* c = schema->children[i];
    if (c == nullptr) return Fail(GDV_INVALID, "null child schema");
    DataType t;
    Status s = ParseFormat(c->format, &t);
    if (!s.ok()) return Fail(s);
    if (c->dictionary != nullptr) {
      // dictionary-encoded: the child's format is the index type's, the dictionary's the values'
      DataType v;
      s = ParseFormat(c->dictionary->format, &v);
      if (s.ok() && v.is_view())
        s = Status::Make(GDV_NOT_IMPLEMENTED, "column '" + std::string(c->name ? c->name : "") + "': dictionaries whose "
                                                  "values are " + v.ToString() + " are not supported");
      if (s.ok() && (!v.is_varlen() || !t.is_signed_integer()))
        s = Status::Make(GDV_NOT_IMPLEMENTED, "column '" + std::string(c->name ? c->name : "") +
                                                  "': dictionaries need utf8 or binary values and signed int8 / int16 / "
                                                  "int32 / int64 indices");
      if (!s.ok()) return Fail(s);
      v.index = t.id;
      v.ordered = (c->flags & ARROW_FLAG_DICTIONARY_ORDERED) != 0;
      t = v;
    }
    fields.push_back(Field{std::string(c->name ? c->name : ""), t});
  }
  *out = reinterpret_cast<gdv_schema_t>(new SchemaH{std::make_shared<Schema>(std::move(fields))});
  return GDV_OK;
}

gdv_status gdv_arrow_batch_import(struct ArrowDeviceArray* array, gdv_schema_t schema,
                                  gdv_arrow_batch_t* out) {
  if (array == nullptr || schema == nullptr || out == nullptr) return Fail(GDV_INVALID, "null argument");
  const ArrowArray& a = array->array;
  if (a.release == nullptr) return Fail(GDV_INVALID, "ArrowDeviceArray was already released");
  const SchemaPtr& sch = reinterpret_cast<SchemaH*>(schema)->p;
  const auto& fields = sch->fields();
  if (a.n_children != static_cast<int64_t>(fields.size()))
    return Fail(GDV_INVALID, "ArrowDeviceArray has " + std::to_string(a.n_children) +
                                 " children, the schema has " + std::to_string(fields.size()) + " fields");
  if (a.null_count > 0) return Fail(GDV_NOT_IMPLEMENTED, "a record batch with struct-level nulls is not supported");
  int mem = GDV_MEM_HOST;
  switch (array->device_type) {
    case ARROW_DEVICE_CPU:
    case ARROW_DEVICE_CUDA_HOST: mem = GDV_MEM_HOST; break;
    case ARROW_DEVICE_CUDA:
    case ARROW_DEVICE_CUDA_MANAGED: mem = GDV_MEM_DEVICE; break;
    default:
      return Fail(GDV_NOT_IMPLEMENTED, "ArrowDeviceType " + std::to_string(array->device_type) + " is not supported");
  }
  std::unique_ptr<gdv_arrow_batch_s> b(new gdv_arrow_batch_s());
  b->schema = sch;
  b->device = mem == GDV_MEM_DEVICE ? static_cast<int>(array->device_id) : -1;
  b->dictionaries.assign(fields.size(), gdv_dictionary_t{});
  b->view_buffers.assign(fields.size(), gdv_view_buffers_t{});
  for (size_t i = 0; i < fields.size(); ++i) {
    const ArrowArray* c = a.children[i];
    const DataType& t = fields[i].type;
    if (c == nullptr) return Fail(GDV_INVALID, "null child array");
    if (t.is_view() && (c->n_buffers < 3 || c->n_children != 0 || c->dictionary != nullptr))
      return Fail(GDV_INVALID, "column '" + fields[i].name + "': malformed " + t.ToString() + " array (expected "
                               "validity, views, the data buffers and their sizes, and no children or dictionary)");
    if (c->n_children != 0) return Fail(GDV_NOT_IMPLEMENTED, "nested columns are not supported");
    if ((c->dictionary != nullptr) != t.is_dict())
      return Fail(c->dictionary != nullptr ? GDV_NOT_IMPLEMENTED : GDV_INVALID,
                  "column '" + fields[i].name + "': the array " + (c->dictionary != nullptr ? "is" : "is not") +
                      " dictionary-encoded but the schema's type is " + t.ToString());
    const int64_t want = t.is_view() ? c->n_buffers : t.is_varlen() && !t.is_dict() ? 3 : 2;
    if (c->n_buffers != want)
      return Fail(GDV_INVALID, "column '" + fields[i].name + "': expected " + std::to_string(want) +
                                   " buffers, got " + std::to_string(c->n_buffers));
    if (c->length < a.offset + a.length)
      return Fail(GDV_INVALID, "column '" + fields[i].name + "' is shorter than the batch");
    gdv_column_t col;
    std::memset(&col, 0, sizeof(col));
    col.validity = c->null_count == 0 ? nullptr : c->buffers[0];
    col.values = c->buffers[1];
    col.offset = c->offset + a.offset;
    if (t.is_dict()) {
      // zero copy: the dictionary's buffers are read where the producer put them
      const ArrowArray* d = c->dictionary;
      if (d->n_buffers != 3 || d->n_children != 0 || d->dictionary != nullptr || d->length < 0 || d->offset < 0 ||
          (d->length > 0 && d->buffers[1] == nullptr))
        return Fail(GDV_INVALID, "column '" + fields[i].name + "': malformed dictionary (expected a utf8 / binary "
                                 "array of 3 buffers with offsets)");
      gdv_dictionary_t& dict = b->dictionaries[i];
      dict.validity = d->null_count == 0 ? nullptr : d->buffers[0];
      dict.offsets = d->buffers[1];
      dict.data = d->buffers[2];
      dict.offset = d->offset;
      dict.length = d->length;
      if (mem == GDV_MEM_HOST && d->length > 0)
        dict.data_size = static_cast<const int32_t*>(d->buffers[1])[d->offset + d->length];
      col.var_data = &dict;
    } else if (t.is_view()) {
      // zero copy: the producer's buffer array already is the table of data buffers, and its last
      // buffer the int64 sizes (device memory for a CUDA array: read there by the kernel)
      gdv_view_buffers_t& vb = b->view_buffers[i];
      vb.n = static_cast<int32_t>(c->n_buffers - 3);
      vb.data = c->buffers + 2;
      vb.sizes = static_cast<const int64_t*>(c->buffers[c->n_buffers - 1]);
      col.var_data = &vb;
    } else if (t.is_varlen()) {
      col.var_data = c->buffers[2];
      if (mem == GDV_MEM_HOST && c->buffers[1] != nullptr)
        col.var_data_size = static_cast<const int32_t*>(c->buffers[1])[col.offset + a.length];
    }
    if (col.values == nullptr && a.length > 0)
      return Fail(GDV_INVALID, "column '" + fields[i].name + "' has no values buffer");
    b->columns.push_back(col);
  }
  b->view.num_rows = a.length;
  b->view.num_columns = static_cast<int32_t>(b->columns.size());
  b->view.mem_space = mem;
  b->view.columns = b->columns.data();
  // move: the consumer now owns the array, the producer's struct is marked released
  std::memcpy(&b->array, array, sizeof(ArrowDeviceArray));
  array->array.release = nullptr;
  *out = b.release();
  return GDV_OK;
}

const gdv_batch_t* gdv_arrow_batch_view(gdv_arrow_batch_t batch) {
  return batch == nullptr ? nullptr : &batch->view;
}

gdv_status gdv_arrow_batch_wait(gdv_arrow_batch_t batch, void* stream) {
  if (batch == nullptr) return Fail(GDV_INVALID, "null batch");
  if (batch->array.sync_event == nullptr || batch->view.mem_space != GDV_MEM_DEVICE) return GDV_OK;
  const DriverApi& d = Driver();
  if (!d.loaded) return Fail(GDV_CUDA_ERROR, d.load_error);
  Device* dev = nullptr;
  Status s = Device::Get(batch->device, &dev);
  if (s.ok()) s = dev->MakeCurrent();
  if (!s.ok()) return Fail(s);
  CUstream st = stream != nullptr ? static_cast<CUstream>(stream) : dev->stream();
  CUevent ev = *static_cast<CUevent*>(batch->array.sync_event);
  s = CuCheck(d.StreamWaitEvent(st, ev, 0), "cuStreamWaitEvent(sync_event)");
  return s.ok() ? GDV_OK : Fail(s);
}

void gdv_arrow_batch_release(gdv_arrow_batch_t batch) {
  if (batch == nullptr) return;
  if (batch->array.array.release != nullptr) batch->array.array.release(&batch->array.array);
  delete batch;
}

gdv_status gdv_projector_output_schema_arrow(gdv_projector_t p, struct ArrowSchema* out) {
  if (p == nullptr || out == nullptr) return Fail(GDV_INVALID, "null argument");
  const auto& exprs = reinterpret_cast<ProjH*>(p)->p->expressions();
  if (Status s = RefuseLargeOutputs(exprs); !s.ok()) return Fail(s);
  SchemaPriv* priv = new SchemaPriv();
  const size_t n = exprs.size();
  priv->formats.reserve(n);
  priv->names.reserve(n);
  priv->children.resize(n);
  for (size_t i = 0; i < n; ++i) {
    priv->formats.push_back(FormatOf(exprs[i]->result().type));
    priv->names.push_back(exprs[i]->result().name);
  }
  for (size_t i = 0; i < n; ++i) {
    ArrowSchema& c = priv->children[i];
    std::memset(&c, 0, sizeof(c));
    c.format = priv->formats[i].c_str();
    c.name = priv->names[i].c_str();
    c.flags = ARROW_FLAG_NULLABLE;
    c.release = ReleaseChildSchema;
    priv->child_ptrs.push_back(&c);
  }
  std::memset(out, 0, sizeof(*out));
  out->format = "+s";
  out->name = "";
  out->n_children = static_cast<int64_t>(n);
  out->children = priv->child_ptrs.data();
  out->release = ReleaseSchema;
  out->private_data = priv;
  return GDV_OK;
}

gdv_status gdv_projector_evaluate_arrow(gdv_projector_t p, gdv_arrow_batch_t batch, void* stream,
                                        struct ArrowDeviceArray* out) {
  if (p == nullptr || batch == nullptr || out == nullptr) return Fail(GDV_INVALID, "null argument");
  Projector& pr = *reinterpret_cast<ProjH*>(p)->p;
  if (Status s = RefuseLargeOutputs(pr.expressions()); !s.ok()) return Fail(s);
  const bool device = batch->view.mem_space == GDV_MEM_DEVICE;
  if (device && batch->device != pr.config().device)
    return Fail(GDV_INVALID, "the batch lives on device " + std::to_string(batch->device) +
                                 ", the projector was made for device " + std::to_string(pr.config().device));
  gdv_status rc = gdv_arrow_batch_wait(batch, stream);
  if (rc != GDV_OK) return rc;
  const int64_t n = batch->view.num_rows;
  const auto& exprs = pr.expressions();
  const int n_outs = static_cast<int>(exprs.size());
  std::unique_ptr<ArrayPriv> priv(new ArrayPriv());
  if (device) {
    Status s = Device::Get(pr.config().device, &priv->dev);
    if (!s.ok()) return Fail(s);
  }
  // ReleaseArray needs a live struct to run on if anything below fails
  ArrowArray guard;
  std::memset(&guard, 0, sizeof(guard));
  guard.release = ReleaseArray;
  guard.private_data = priv.get();
  ArrayPriv* pv = priv.release();
  auto fail = [&](const Status& s) {
    guard.release(&guard);
    return Fail(s);
  };
  std::vector<gdv_out_column_t> outs(n_outs);
  const size_t vld_bytes = static_cast<size_t>((n + 31) / 32) * 4;
  for (int o = 0; o < n_outs; ++o) {
    const DataType& t = exprs[o]->result().type;
    gdv_out_column_t& oc = outs[o];
    std::memset(&oc, 0, sizeof(oc));
    Status s = AllocOut(pv, device, vld_bytes, &oc.validity);
    if (!s.ok()) return fail(s);
    if (t.is_varlen()) {
      int64_t bytes = 0;
      s = pr.OutputVarSize(&batch->view, nullptr, o, stream, &bytes);
      if (s.ok()) s = AllocOut(pv, device, static_cast<size_t>(n + 1) * 4, &oc.values);
      if (s.ok()) s = AllocOut(pv, device, static_cast<size_t>(bytes), &oc.var_data);
      if (!s.ok()) return fail(s);
      oc.var_capacity = bytes;
    } else {
      const size_t vb = t.is_bool() ? vld_bytes : static_cast<size_t>(n) * t.width();
      s = AllocOut(pv, device, vb, &oc.values);
      if (!s.ok()) return fail(s);
    }
  }
  if (n > 0) {
    Status s = pr.Evaluate(&batch->view, nullptr, outs.data(), n_outs, stream, /*async=*/false);
    if (!s.ok()) return fail(s);
  }
  // export: parent struct + one child per output
  pv->children.resize(n_outs);
  pv->buffers.resize(n_outs + 1);
  pv->buffers[0] = {nullptr};
  for (int o = 0; o < n_outs; ++o) {
    const DataType& t = exprs[o]->result().type;
    ArrowArray& c = pv->children[o];
    std::memset(&c, 0, sizeof(c));
    if (t.is_varlen())
      pv->buffers[o + 1] = {outs[o].validity, outs[o].values, outs[o].var_data};
    else
      pv->buffers[o + 1] = {outs[o].validity, outs[o].values};
    c.length = n;
    c.null_count = -1;
    c.n_buffers = static_cast<int64_t>(pv->buffers[o + 1].size());
    c.buffers = pv->buffers[o + 1].data();
    c.release = ReleaseChildArray;
    pv->child_ptrs.push_back(&c);
  }
  InitDeviceArray(out, batch);
  out->array.length = n;
  out->array.null_count = 0;
  out->array.n_buffers = 1;
  out->array.buffers = pv->buffers[0].data();
  out->array.n_children = n_outs;
  out->array.children = pv->child_ptrs.data();
  out->array.release = ReleaseArray;
  out->array.private_data = pv;
  return GDV_OK;
}

gdv_status gdv_filter_evaluate_arrow(gdv_filter_t f, gdv_arrow_batch_t batch, int32_t mode,
                                     void* stream, struct ArrowDeviceArray* out) {
  if (f == nullptr || batch == nullptr || out == nullptr) return Fail(GDV_INVALID, "null argument");
  Filter& fl = *reinterpret_cast<FiltH*>(f)->p;
  const bool device = batch->view.mem_space == GDV_MEM_DEVICE;
  if (device && batch->device != fl.config().device)
    return Fail(GDV_INVALID, "the batch lives on device " + std::to_string(batch->device) +
                                 ", the filter was made for device " + std::to_string(fl.config().device));
  int width = 0;
  switch (mode) {
    case GDV_SEL_UINT16: width = 2; break;
    case GDV_SEL_UINT32: width = 4; break;
    case GDV_SEL_UINT64: width = 8; break;
    default: return Fail(GDV_INVALID, "selection mode must be UINT16, UINT32 or UINT64");
  }
  gdv_status rc = gdv_arrow_batch_wait(batch, stream);
  if (rc != GDV_OK) return rc;
  const int64_t n = batch->view.num_rows;
  std::unique_ptr<ArrayPriv> priv(new ArrayPriv());
  if (device) {
    Status s = Device::Get(fl.config().device, &priv->dev);
    if (!s.ok()) return Fail(s);
  }
  ArrowArray guard;
  std::memset(&guard, 0, sizeof(guard));
  guard.release = ReleaseArray;
  guard.private_data = priv.get();
  ArrayPriv* pv = priv.release();
  void* idx = nullptr;
  Status s = AllocOut(pv, device, static_cast<size_t>(n) * width, &idx);
  gdv_selection_t sel;
  std::memset(&sel, 0, sizeof(sel));
  sel.indices = idx;
  sel.max_slots = n;
  sel.mode = mode;
  sel.mem_space = batch->view.mem_space;
  if (s.ok() && n > 0) s = fl.Evaluate(&batch->view, &sel, stream, /*async=*/false, nullptr);
  if (!s.ok()) {
    guard.release(&guard);
    return Fail(s);
  }
  pv->buffers.resize(1);
  pv->buffers[0] = {nullptr, idx};
  InitDeviceArray(out, batch);
  out->array.length = n > 0 ? sel.num_slots : 0;
  out->array.null_count = 0;
  out->array.n_buffers = 2;
  out->array.buffers = pv->buffers[0].data();
  out->array.release = ReleaseArray;
  out->array.private_data = pv;
  return GDV_OK;
}

gdv_status gdv_memcpy(int32_t device, void* dst, const void* src, size_t bytes, int32_t kind) {
  const DriverApi& d = Driver();
  if (!d.loaded) return Fail(GDV_CUDA_ERROR, d.load_error);
  Device* dev = nullptr;
  Status s = Device::Get(device, &dev);
  if (s.ok()) s = dev->MakeCurrent();
  if (!s.ok()) return Fail(s);
  if (bytes == 0) return GDV_OK;
  if (kind == 1)
    s = CuCheck(d.MemcpyHtoDAsync(reinterpret_cast<CUdeviceptr>(dst), src, bytes, dev->stream()), "H2D");
  else if (kind == 2)
    s = CuCheck(d.MemcpyDtoHAsync(dst, reinterpret_cast<CUdeviceptr>(src), bytes, dev->stream()), "D2H");
  else
    return Fail(GDV_INVALID, "kind must be 1 (host to device) or 2 (device to host)");
  if (s.ok()) s = CuCheck(d.StreamSynchronize(dev->stream()), "cuStreamSynchronize");
  return s.ok() ? GDV_OK : Fail(s);
}

}  // extern "C"
