// capi.cu — extern "C" entry points declared in include/arkflow_b200.h.
#include <chrono>
#include <map>
#include <mutex>

#include "abi.h"

using namespace ark;

namespace {

template <typename Make>
int create_proc(Make make, const char* config_json, ark_proc_t** out) {
  return guarded([&] {
    if (!out) fail(ARK_ERR_PROCESS, "null output handle");
    *out = nullptr;
    auto p = make(config_json);
    auto* h = new ark_proc();
    h->impl = std::move(p);
    *out = h;
  });
}

// What the four codec processors' entry points differ in (processor/json.rs:42-113, processor/protobuf.rs:98-148).
struct Codec {
  const char* type;
  const std::string& (*value_field)(const Processor&);  // the one column imported; nullptr: every column
  bool none_on_empty;                                    // an empty input is ProcessResult::None (protobuf.rs:101-103)
  bool codec_types;                                      // see import_host
  Batch (*run)(const Processor&, Batch&, cudaStream_t);
};

const Codec kJsonToArrow{"json_to_arrow", json_to_arrow_value_field, false, false, json_to_arrow_device};
const Codec kArrowToJson{"arrow_to_json", nullptr, false, false, arrow_to_json_device};
const Codec kProtobufToArrow{"protobuf_to_arrow", protobuf_to_arrow_value_field, true, false, protobuf_to_arrow_device};
const Codec kArrowToProtobuf{"arrow_to_protobuf", nullptr, true, true, arrow_to_protobuf_device};

std::vector<bool> value_field_mask(const Codec& c, const Processor& p, const ArrowSchema* schema) {
  std::vector<Field> fields = schema_fields(schema);
  std::vector<bool> m(fields.size(), false);
  for (size_t i = 0; i < fields.size(); ++i) if (fields[i].name == c.value_field(p)) m[i] = true;
  return m;
}

int codec_process(const Codec& c, ark_proc_t* p, ArrowArray* in, ArrowSchema* in_schema, ArrowArray* out, ArrowSchema* out_schema) {
  BufferPtr in_owner = adopt_array(in);
  return guarded([&] {
    zero_out(out, out_schema);
    Processor* proc = proc_of(p, c.type);
    const ArrowArray* arr = adopted(in_owner);
    if (c.none_on_empty && arr->length == 0) return;
    std::vector<bool> mask;
    if (c.value_field) mask = value_field_mask(c, *proc, in_schema);
    StreamLease lease;
    Batch b = import_host(arr, in_schema, c.value_field ? &mask : nullptr, lease.s, nullptr, c.codec_types);
    Batch r = c.run(*proc, b, lease.s);
    export_host(r, lease.s, out, out_schema);
  });
}

int codec_process_device(const Codec& c, ark_proc_t* p, ArrowDeviceArray* in, ArrowSchema* in_schema, ArrowDeviceArray* out,
                         ArrowSchema* out_schema) {
  BufferPtr in_owner = adopt_array(&in->array);
  return guarded([&] {
    zero_out(out, out_schema);
    Processor* proc = proc_of(p, c.type);
    ArrowDeviceArray view = device_view(*in, in_owner);
    if (c.none_on_empty && view.array.length == 0) return;
    std::vector<bool> mask;
    if (c.value_field) mask = value_field_mask(c, *proc, in_schema);
    StreamLease lease;
    Batch b = import_device(&view, in_schema, c.value_field ? &mask : nullptr, in_owner, c.codec_types);
    Batch r = c.run(*proc, b, lease.s);
    export_device(r, out, out_schema, lease);
  });
}

}  // namespace

extern "C" {

int ark_b200_init(int device) {
  return guarded([&] {
    if (device >= 0) ARK_CUDA(cudaSetDevice(device));
    ARK_CUDA(cudaFree(0));
    cudaDeviceProp prop;
    int dev = 0;
    ARK_CUDA(cudaGetDevice(&dev));
    ARK_CUDA(cudaGetDeviceProperties(&prop, dev));
    // sm_90a code runs on compute capability 9.0 only (the "a" features do not carry forward)
    if (prop.major != 9 || prop.minor != 0) fail(ARK_ERR_CUDA, std::string("arkflow_b200 is built for sm_90a (H100); found ") + prop.name);
    bind_device(dev);
  });
}

int ark_b200_device_count(int* out_count) {
  return guarded([&] { ARK_CUDA(cudaGetDeviceCount(out_count)); });
}

const char* ark_b200_version(void) { return "arkflow_b200 0.1.0 (sm_90a)"; }
const char* ark_last_error(void) { return last_error_ref().c_str(); }

int ark_sql_create(const char* config_json, ark_proc_t** out) { return create_proc(SqlProcessor::from_config, config_json, out); }

int ark_sql_process(ark_proc_t* p, ArrowArray* in, ArrowSchema* in_schema, ArrowArray* out, ArrowSchema* out_schema) {
  BufferPtr in_owner = adopt_array(in);
  return guarded([&] {
    zero_out(out, out_schema);
    SqlProcessor* sp = as_sql(p);
    const ArrowArray* arr = adopted(in_owner);
    if (arr->length == 0) return;  // ProcessResult::None, sql.rs:211-213
    auto bound = sp->bind(in_schema);
    StreamLease lease;
    Batch b = import_host(arr, in_schema, &bound->mask, lease.s);
    Batch r = sp->execute(*bound->plan, b, lease.s);
    export_host(r, lease.s, out, out_schema);
  });
}

int ark_sql_process_device(ark_proc_t* p, ArrowDeviceArray* in, ArrowSchema* in_schema, ArrowDeviceArray* out,
                           ArrowSchema* out_schema) {
  BufferPtr in_owner = adopt_array(&in->array);
  return guarded([&] {
    zero_out(out, out_schema);
    SqlProcessor* sp = as_sql(p);
    ArrowDeviceArray view = device_view(*in, in_owner);
    if (view.array.length == 0) return;
    const bool trace = trace_enabled();  // per-phase host time of this entry point, to stderr
    auto now = [] { return std::chrono::steady_clock::now(); };
    auto us = [](std::chrono::steady_clock::time_point a, std::chrono::steady_clock::time_point b) {
      return (double)std::chrono::duration_cast<std::chrono::nanoseconds>(b - a).count() / 1e3;
    };
    const auto t0 = now();
    tl_call_trace = CallTrace{t0, t0, t0};  // stays at t0 unless the filter fast path ran
    auto bound = sp->bind(in_schema);
    const auto t1 = now();
    StreamLease lease;
    Batch b = import_device(&view, in_schema, &bound->mask, in_owner, false, &bound->fields);
    const auto t2 = now();
    Batch r = sp->execute(*bound->plan, b, lease.s);
    const auto t3 = now();
    export_device(r, out, out_schema, lease);
    const auto t4 = now();
    // the input's release (an outside callback) runs here, unless an exported column still aliases it
    r = Batch();
    b = Batch();
    in_owner.reset();
    if (trace) {
      const auto t5 = now();
      const CallTrace& ct = tl_call_trace;
      fprintf(stderr,
              "[ark trace] sql_process_device: plan %.1f us, import %.1f us, execute %.1f us (to launch enqueued %.1f us = outputs and "
              "scratch %.1f us + launch %.1f us, gpu wait %.1f us), sync return to export done %.1f us, input release %.1f us, total %.1f us\n",
              us(t0, t1), us(t1, t2), us(t2, t3), us(t2, ct.launched), us(t2, ct.prepared), us(ct.prepared, ct.launched),
              us(ct.launched, ct.synced), us(ct.synced, t4), us(t4, t5), us(t0, t5));
    }
  });
}

int ark_sql_partial_aggregate_device(ark_proc_t* p, ArrowDeviceArray* in, ArrowSchema* in_schema, int n_parts,
                                     ArrowDeviceArray* out, ArrowSchema* out_schema, int64_t* part_rows) {
  BufferPtr in_owner = adopt_array(&in->array);
  return guarded([&] {
    zero_out(out, out_schema);
    SqlProcessor* sp = as_sql(p);
    ArrowDeviceArray view = device_view(*in, in_owner);
    if (n_parts < 1) fail(ARK_ERR_PROCESS, "n_parts must be >= 1");
    auto bound = sp->bind(in_schema);
    if (bound->plan->kind != Plan::Aggregate) fail(ARK_ERR_PROCESS, "partial aggregate requested for a query without aggregation");
    refuse_limit_across_ranks(*bound->plan);
    StreamLease lease;
    Batch b = import_device(&view, in_schema, &bound->mask, in_owner, false, &bound->fields);
    if (!bound->plan->derived.empty()) b = append_json_columns(*bound->plan, b, lease.s);
    std::vector<int64_t> rows;
    ExportAllocScope exported;  // the partial states are published to the other ranks over CUDA IPC
    Batch r = run_partial_aggregate(*bound->plan, b, n_parts, rows, lease.s);
    for (int i = 0; i < n_parts; ++i) part_rows[i] = rows[i];
    export_device(r, out, out_schema, lease);
  });
}

int ark_sql_final_aggregate_device(ark_proc_t* p, ArrowDeviceArray* in, ArrowSchema* in_schema, ArrowDeviceArray* out,
                                   ArrowSchema* out_schema) {
  BufferPtr in_owner = adopt_array(&in->array);
  return guarded([&] {
    zero_out(out, out_schema);
    SqlProcessor* sp = as_sql(p);
    ArrowDeviceArray view = device_view(*in, in_owner);
    auto plan = sp->last_aggregate_plan();
    if (!plan) fail(ARK_ERR_PROCESS, "final aggregate called before any partial aggregate bound the query");
    refuse_limit_across_ranks(*plan);
    StreamLease lease;
    Batch b = import_device(&view, in_schema, nullptr, in_owner);
    Batch r = run_final_aggregate(*plan, b, lease.s);
    export_device(r, out, out_schema, lease);
  });
}

// Runs the processor's query over several named tables (JoinOperation, buffer/join.rs:92-118).
static Batch run_tables(SqlProcessor* sp, std::vector<std::string>& names, std::vector<std::vector<Field>>& schemas,
                        std::vector<Batch>& tables, cudaStream_t stream) {
  auto plan = sp->join_plan_for(names, schemas);
  if (plan->kind == Plan::Join) {
    int li = -1, ri = -1;
    for (size_t i = 0; i < names.size(); ++i) { if (names[i] == plan->left_table) li = (int)i; if (names[i] == plan->right_table) ri = (int)i; }
    if (li < 0 || ri < 0) fail(ARK_ERR_PROCESS, "Failed to execute SQL query: table not found");
    return run_join(*plan, tables[li], tables[ri], stream);
  }
  // a single-table query evaluated through the multi-table entry point
  for (size_t i = 0; i < names.size(); ++i)
    if (names[i] == sp->ast.from.name) return sp->execute(*plan, tables[i], stream);
  fail(ARK_ERR_PROCESS, "Failed to execute SQL query: table '" + sp->ast.from.name + "' not found");
}

int ark_sql_process_tables(ark_proc_t* p, int n_tables, const char* const* names, ArrowArray* ins, ArrowSchema* in_schemas,
                           ArrowArray* out, ArrowSchema* out_schema) {
  std::vector<BufferPtr> owners;
  for (int i = 0; i < n_tables; ++i) owners.push_back(adopt_array(&ins[i]));
  return guarded([&] {
    zero_out(out, out_schema);
    SqlProcessor* sp = as_sql(p);
    StreamLease lease;
    std::vector<std::string> nm;
    std::vector<std::vector<Field>> schemas;
    std::vector<Batch> tables;
    for (int i = 0; i < n_tables; ++i) {
      nm.push_back(names[i]);
      schemas.push_back(schema_fields(&in_schemas[i]));
      tables.push_back(import_host(adopted(owners[i]), &in_schemas[i], nullptr, lease.s));
    }
    Batch r = run_tables(sp, nm, schemas, tables, lease.s);
    export_host(r, lease.s, out, out_schema);
  });
}

int ark_sql_process_tables_device(ark_proc_t* p, int n_tables, const char* const* names, ArrowDeviceArray* ins,
                                  ArrowSchema* in_schemas, ArrowDeviceArray* out, ArrowSchema* out_schema) {
  std::vector<BufferPtr> owners;
  for (int i = 0; i < n_tables; ++i) owners.push_back(adopt_array(&ins[i].array));
  return guarded([&] {
    zero_out(out, out_schema);
    SqlProcessor* sp = as_sql(p);
    StreamLease lease;
    std::vector<std::string> nm;
    std::vector<std::vector<Field>> schemas;
    std::vector<Batch> tables;
    for (int i = 0; i < n_tables; ++i) {
      nm.push_back(names[i]);
      schemas.push_back(schema_fields(&in_schemas[i]));
      ArrowDeviceArray view = device_view(ins[i], owners[i]);
      tables.push_back(import_device(&view, &in_schemas[i], nullptr, owners[i]));
    }
    Batch r = run_tables(sp, nm, schemas, tables, lease.s);
    export_device(r, out, out_schema, lease);
  });
}

int ark_hash_partition_device(ArrowDeviceArray* in, ArrowSchema* in_schema, const char* key_column, int n_parts,
                              ArrowDeviceArray* out, ArrowSchema* out_schema, int64_t* part_rows) {
  BufferPtr in_owner = adopt_array(&in->array);
  return guarded([&] {
    zero_out(out, out_schema);
    ArrowDeviceArray view = device_view(*in, in_owner);
    StreamLease lease;
    Batch b = import_device(&view, in_schema, nullptr, in_owner);
    std::vector<int64_t> rows;
    Batch r = hash_partition(b, key_column ? key_column : "", n_parts, rows, lease.s);
    for (int i = 0; i < n_parts; ++i) part_rows[i] = rows[i];
    export_device(r, out, out_schema, lease);
  });
}

int ark_json_to_arrow_create(const char* config_json, ark_proc_t** out) { return create_proc(make_json_to_arrow, config_json, out); }
int ark_json_to_arrow_process(ark_proc_t* p, ArrowArray* in, ArrowSchema* in_schema, ArrowArray* out, ArrowSchema* out_schema) {
  return codec_process(kJsonToArrow, p, in, in_schema, out, out_schema);
}
int ark_json_to_arrow_process_device(ark_proc_t* p, ArrowDeviceArray* in, ArrowSchema* in_schema, ArrowDeviceArray* out,
                                     ArrowSchema* out_schema) {
  return codec_process_device(kJsonToArrow, p, in, in_schema, out, out_schema);
}

int ark_arrow_to_json_create(const char* config_json, ark_proc_t** out) { return create_proc(make_arrow_to_json, config_json, out); }
int ark_arrow_to_json_process(ark_proc_t* p, ArrowArray* in, ArrowSchema* in_schema, ArrowArray* out, ArrowSchema* out_schema) {
  return codec_process(kArrowToJson, p, in, in_schema, out, out_schema);
}
int ark_arrow_to_json_process_device(ark_proc_t* p, ArrowDeviceArray* in, ArrowSchema* in_schema, ArrowDeviceArray* out,
                                     ArrowSchema* out_schema) {
  return codec_process_device(kArrowToJson, p, in, in_schema, out, out_schema);
}

int ark_protobuf_to_arrow_create(const char* config_json, ark_proc_t** out) { return create_proc(make_protobuf_to_arrow, config_json, out); }
int ark_protobuf_to_arrow_process(ark_proc_t* p, ArrowArray* in, ArrowSchema* in_schema, ArrowArray* out, ArrowSchema* out_schema) {
  return codec_process(kProtobufToArrow, p, in, in_schema, out, out_schema);
}
int ark_protobuf_to_arrow_process_device(ark_proc_t* p, ArrowDeviceArray* in, ArrowSchema* in_schema, ArrowDeviceArray* out,
                                         ArrowSchema* out_schema) {
  return codec_process_device(kProtobufToArrow, p, in, in_schema, out, out_schema);
}

int ark_arrow_to_protobuf_create(const char* config_json, ark_proc_t** out) { return create_proc(make_arrow_to_protobuf, config_json, out); }
int ark_arrow_to_protobuf_process(ark_proc_t* p, ArrowArray* in, ArrowSchema* in_schema, ArrowArray* out, ArrowSchema* out_schema) {
  return codec_process(kArrowToProtobuf, p, in, in_schema, out, out_schema);
}
int ark_arrow_to_protobuf_process_device(ark_proc_t* p, ArrowDeviceArray* in, ArrowSchema* in_schema, ArrowDeviceArray* out,
                                         ArrowSchema* out_schema) {
  return codec_process_device(kArrowToProtobuf, p, in, in_schema, out, out_schema);
}

// ---- expr::evaluate_expr (plugin/expr/mod.rs:92-122) ---------------------------------------------------
namespace {

bool references_column(const Expr& e) {
  if (e.kind == Expr::Column || e.kind == Expr::Star) return true;
  for (auto& a : e.args) if (references_column(*a)) return true;
  return false;
}

struct CachedExpr { std::shared_ptr<SqlProcessor> proc; bool scalar; };

// EXPR_CACHE (expr/mod.rs:27-28): expression text → bound processor (plans are cached per schema inside it)
CachedExpr expr_processor(const char* text) {
  static std::mutex mu;
  static std::map<std::string, CachedExpr> cache;
  {
    std::lock_guard<std::mutex> l(mu);
    auto it = cache.find(text);
    if (it != cache.end()) return it->second;
  }
  ExprPtr e = parse_sql_expr(text);
  CachedExpr ce;
  ce.scalar = !references_column(*e);
  if (e->kind == Expr::Literal && e->lit_type == DType::Utf8) {  // a bare string: the one-argument concat of it
    auto f = std::make_unique<Expr>();
    f->kind = Expr::Func; f->name = "concat"; f->args.push_back(std::move(e));
    e = std::move(f);
  }
  auto p = std::make_shared<SqlProcessor>();
  p->query_text = text;
  p->ast.from.name = p->table_name;
  SelectItem it;
  it.expr = std::move(e);
  it.alias = "value";
  p->ast.select.push_back(std::move(it));
  ce.proc = p;
  std::lock_guard<std::mutex> l(mu);
  if (cache.size() > 256) cache.clear();
  cache[text] = ce;
  return ce;
}

Batch evaluate_expr_on(const CachedExpr& ce, Batch& in, const std::vector<Field>& fields, cudaStream_t stream) {
  auto plan = ce.proc->plan_for(ce.scalar ? std::vector<Field>{} : fields);
  if (plan->kind != Plan::FilterProject)
    fail(ARK_ERR_PROCESS, "Error during planning: aggregate functions are not valid in a scalar expression");
  if (ce.scalar) {
    Batch one;
    one.num_rows = 1;
    return ce.proc->execute(*plan, one, stream);
  }
  if (in.num_rows == 0) {  // an empty array of the expression's type
    Batch out;
    Column c;
    c.field.name = "value"; c.field.nullable = true; c.length = 0;
    c.field.type = (!plan->final_items.empty() && plan->final_items[0].is_concat) ? DType::Utf8 : plan->outputs[0].src.type;
    BufferPtr z = device_alloc(16);
    ARK_CUDA(cudaMemsetAsync(z.get(), 0, 16, stream));
    c.data = (const uint8_t*)z.get(); c.data_bytes = 0;
    if (c.field.type == DType::Utf8 || c.field.type == DType::Binary) { c.offsets = (const int32_t*)z.get(); c.first_offset = 0; }
    c.owners = {z};
    out.cols.push_back(c);
    return out;
  }
  return ce.proc->execute(*plan, in, stream);
}

}  // namespace

int ark_expr_evaluate(const char* expr, ArrowArray* in, ArrowSchema* in_schema, ArrowArray* out, ArrowSchema* out_schema, int* is_scalar) {
  BufferPtr in_owner = adopt_array(in);
  return guarded([&] {
    zero_out(out, out_schema);
    if (!expr || !out) fail(ARK_ERR_PROCESS, "null argument");
    const ArrowArray* arr = adopted(in_owner);
    CachedExpr ce = expr_processor(expr);
    if (is_scalar) *is_scalar = ce.scalar ? 1 : 0;
    std::vector<Field> fields = schema_fields(in_schema);
    auto plan = ce.proc->plan_for(ce.scalar ? std::vector<Field>{} : fields);
    StreamLease lease;
    Batch b;
    if (!ce.scalar) {
      std::vector<bool> mask = needed_mask(*plan, fields.size());
      b = import_host(arr, in_schema, &mask, lease.s);
    }
    Batch r = evaluate_expr_on(ce, b, fields, lease.s);
    export_host(r, lease.s, out, out_schema);
  });
}

int ark_expr_evaluate_device(const char* expr, ArrowDeviceArray* in, ArrowSchema* in_schema, ArrowDeviceArray* out, ArrowSchema* out_schema,
                             int* is_scalar) {
  BufferPtr in_owner = adopt_array(&in->array);
  return guarded([&] {
    zero_out(out, out_schema);
    if (!expr || !out) fail(ARK_ERR_PROCESS, "null argument");
    ArrowDeviceArray view = device_view(*in, in_owner);
    CachedExpr ce = expr_processor(expr);
    if (is_scalar) *is_scalar = ce.scalar ? 1 : 0;
    std::vector<Field> fields = schema_fields(in_schema);
    auto plan = ce.proc->plan_for(ce.scalar ? std::vector<Field>{} : fields);
    StreamLease lease;
    Batch b;
    if (!ce.scalar) {
      std::vector<bool> mask = needed_mask(*plan, fields.size());
      b = import_device(&view, in_schema, &mask, in_owner);
    }
    Batch r = evaluate_expr_on(ce, b, fields, lease.s);
    export_device(r, out, out_schema, lease);
  });
}

int ark_proc_close(ark_proc_t*) { return ARK_OK; }  // Processor::close is a no-op in the reference (sql.rs:222-224)

void ark_proc_destroy(ark_proc_t* p) { delete p; }

int64_t ark_kernel_launch_count(void) { return launch_count(); }
void ark_kernel_timing_enable(int on) { timing_enable(on); }
void ark_kernel_timing_reset(void) { timing_reset(); }
int ark_kernel_timing_get(const char* name, double* total_ms, int64_t* launches) {
  return timing_get(name, total_ms, launches) ? 0 : 1;
}

}  // extern "C"
