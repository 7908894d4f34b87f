// capi.cu — extern "C" entry points declared in include/arkflow_b200.h.
#include <cstring>

#include <chrono>
#include <map>
#include <mutex>

#include "engine.h"

using namespace ark;

struct ark_proc {
  std::unique_ptr<Processor> impl;
};

namespace {

template <typename F>
int guarded(F&& f) {
  try {
    f();
    return ARK_OK;
  } catch (const ArkError& e) {
    set_last_error(e.what());
    return e.code;
  } catch (const std::bad_alloc&) {
    set_last_error("out of host memory");
    return ARK_ERR_PROCESS;
  } catch (const std::exception& e) {
    set_last_error(e.what());
    return ARK_ERR_PROCESS;
  }
}

SqlProcessor* as_sql(ark_proc_t* p) {
  if (!p || !p->impl || strcmp(p->impl->type(), "sql") != 0) fail(ARK_ERR_PROCESS, "handle is not a sql processor");
  return static_cast<SqlProcessor*>(p->impl.get());
}

std::vector<bool> needed_mask(const Plan& plan, size_t n_fields) {
  std::vector<bool> m(n_fields, false);
  if (plan.identity) { std::fill(m.begin(), m.end(), true); return m; }
  for (int c : plan.used_cols) m[c] = true;
  return m;
}

void set_none(ArrowArray* out, ArrowSchema* out_schema) {
  memset(out, 0, sizeof(*out));
  if (out_schema) memset(out_schema, 0, sizeof(*out_schema));
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

int ark_sql_create(const char* config_json, ark_proc_t** out) {
  return guarded([&] {
    if (!out) fail(ARK_ERR_PROCESS, "null output handle");
    *out = nullptr;
    auto p = SqlProcessor::from_config(config_json);
    auto* h = new ark_proc();
    h->impl = std::move(p);
    *out = h;
  });
}

int ark_sql_process(ark_proc_t* p, ArrowArray* in, ArrowSchema* in_schema, ArrowArray* out, ArrowSchema* out_schema) {
  BufferPtr in_owner = adopt_array(in);  // moved in: released on every path
  return guarded([&] {
    SqlProcessor* sp = as_sql(p);
    const ArrowArray* arr = (const ArrowArray*)in_owner.get();
    if (!arr) fail(ARK_ERR_PROCESS, "input array already released");
    if (arr->length == 0) { set_none(out, out_schema); return; }  // ProcessResult::None, sql.rs:211-213
    std::vector<Field> fields = schema_fields(in_schema);
    auto plan = sp->plan_for(fields);
    std::vector<bool> mask = needed_mask(*plan, fields.size());
    StreamLease lease;
    Batch b = import_host(arr, in_schema, &mask, lease.s);
    Batch r = sp->execute(*plan, b, lease.s);
    export_host(r, lease.s, out, out_schema);
  });
}

int ark_sql_process_device(ark_proc_t* p, ArrowDeviceArray* in, ArrowSchema* in_schema, ArrowDeviceArray* out,
                           ArrowSchema* out_schema) {
  BufferPtr in_owner = adopt_array(&in->array);
  return guarded([&] {
    SqlProcessor* sp = as_sql(p);
    if (!in_owner) fail(ARK_ERR_PROCESS, "input array already released");
    ArrowDeviceArray view = *in;
    view.array = *(const ArrowArray*)in_owner.get();
    if (view.array.length == 0) { memset(out, 0, sizeof(*out)); if (out_schema) memset(out_schema, 0, sizeof(*out_schema)); return; }
    static const bool trace = getenv("ARK_TRACE") != nullptr;  // per-phase host time of this entry point, to stderr
    auto now = [] { return std::chrono::steady_clock::now(); };
    auto us = [](std::chrono::steady_clock::time_point a, std::chrono::steady_clock::time_point b) {
      return (double)std::chrono::duration_cast<std::chrono::nanoseconds>(b - a).count() / 1e3;
    };
    const auto t0 = now();
    std::vector<Field> fields = schema_fields(in_schema);
    auto plan = sp->plan_for(fields);
    std::vector<bool> mask = needed_mask(*plan, fields.size());
    const auto t1 = now();
    StreamLease lease;
    Batch b = import_device(&view, in_schema, &mask, in_owner);
    const auto t2 = now();
    Batch r = sp->execute(*plan, b, lease.s);
    const auto t3 = now();
    ARK_CUDA(cudaStreamSynchronize(lease.s));
    export_device(r, out, out_schema);
    if (trace) {
      const auto t4 = now();
      fprintf(stderr, "[ark trace] sql_process_device: plan %.1f us, import %.1f us, execute %.1f us, export %.1f us\n", us(t0, t1), us(t1, t2),
              us(t2, t3), us(t3, t4));
    }
  });
}

int ark_sql_partial_aggregate_device(ark_proc_t* p, ArrowDeviceArray* in, ArrowSchema* in_schema, int n_parts,
                                     ArrowDeviceArray* out, ArrowSchema* out_schema, int64_t* part_rows) {
  BufferPtr in_owner = adopt_array(&in->array);
  return guarded([&] {
    SqlProcessor* sp = as_sql(p);
    if (!in_owner) fail(ARK_ERR_PROCESS, "input array already released");
    if (n_parts < 1) fail(ARK_ERR_PROCESS, "n_parts must be >= 1");
    ArrowDeviceArray view = *in;
    view.array = *(const ArrowArray*)in_owner.get();
    std::vector<Field> fields = schema_fields(in_schema);
    auto plan = sp->plan_for(fields);
    if (plan->kind != Plan::Aggregate) fail(ARK_ERR_PROCESS, "partial aggregate requested for a query without aggregation");
    std::vector<bool> mask = needed_mask(*plan, fields.size());
    StreamLease lease;
    Batch b = import_device(&view, in_schema, &mask, in_owner);
    std::vector<int64_t> rows;
    ExportAllocScope exported;  // the partial states are published to the other ranks over CUDA IPC
    Batch r = run_partial_aggregate(*plan, b, n_parts, rows, lease.s);
    for (int i = 0; i < n_parts; ++i) part_rows[i] = rows[i];
    export_device(r, out, out_schema);
  });
}

int ark_sql_final_aggregate_device(ark_proc_t* p, ArrowDeviceArray* in, ArrowSchema* in_schema, ArrowDeviceArray* out,
                                   ArrowSchema* out_schema) {
  BufferPtr in_owner = adopt_array(&in->array);
  return guarded([&] {
    SqlProcessor* sp = as_sql(p);
    if (!in_owner) fail(ARK_ERR_PROCESS, "input array already released");
    ArrowDeviceArray view = *in;
    view.array = *(const ArrowArray*)in_owner.get();
    auto plan = sp->last_aggregate_plan();
    if (!plan) fail(ARK_ERR_PROCESS, "final aggregate called before any partial aggregate bound the query");
    StreamLease lease;
    Batch b = import_device(&view, in_schema, nullptr, in_owner);
    Batch r = run_final_aggregate(*plan, b, lease.s);
    export_device(r, out, out_schema);
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
    SqlProcessor* sp = as_sql(p);
    StreamLease lease;
    std::vector<std::string> nm;
    std::vector<std::vector<Field>> schemas;
    std::vector<Batch> tables;
    for (int i = 0; i < n_tables; ++i) {
      nm.push_back(names[i]);
      schemas.push_back(schema_fields(&in_schemas[i]));
      tables.push_back(import_host((const ArrowArray*)owners[i].get(), &in_schemas[i], nullptr, lease.s));
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
    SqlProcessor* sp = as_sql(p);
    StreamLease lease;
    std::vector<std::string> nm;
    std::vector<std::vector<Field>> schemas;
    std::vector<Batch> tables;
    for (int i = 0; i < n_tables; ++i) {
      nm.push_back(names[i]);
      schemas.push_back(schema_fields(&in_schemas[i]));
      ArrowDeviceArray view = ins[i];
      view.array = *(const ArrowArray*)owners[i].get();
      tables.push_back(import_device(&view, &in_schemas[i], nullptr, owners[i]));
    }
    Batch r = run_tables(sp, nm, schemas, tables, lease.s);
    export_device(r, out, out_schema);
  });
}

int ark_hash_partition_device(ArrowDeviceArray* in, ArrowSchema* in_schema, const char* key_column, int n_parts,
                              ArrowDeviceArray* out, ArrowSchema* out_schema, int64_t* part_rows) {
  BufferPtr in_owner = adopt_array(&in->array);
  return guarded([&] {
    if (!in_owner) fail(ARK_ERR_PROCESS, "input array already released");
    ArrowDeviceArray view = *in;
    view.array = *(const ArrowArray*)in_owner.get();
    StreamLease lease;
    Batch b = import_device(&view, in_schema, nullptr, in_owner);
    std::vector<int64_t> rows;
    Batch r = hash_partition(b, key_column ? key_column : "", n_parts, rows, lease.s);
    for (int i = 0; i < n_parts; ++i) part_rows[i] = rows[i];
    export_device(r, out, out_schema);
  });
}

int ark_json_to_arrow_create(const char* config_json, ark_proc_t** out) {
  return guarded([&] {
    if (!out) fail(ARK_ERR_PROCESS, "null output handle");
    *out = nullptr;
    auto p = make_json_to_arrow(config_json);
    auto* h = new ark_proc();
    h->impl = std::move(p);
    *out = h;
  });
}

static Processor* as_json(ark_proc_t* p) {
  if (!p || !p->impl || strcmp(p->impl->type(), "json_to_arrow") != 0) fail(ARK_ERR_PROCESS, "handle is not a json_to_arrow processor");
  return p->impl.get();
}

static std::vector<bool> json_mask(const Processor& jp, const std::vector<Field>& fields) {
  std::vector<bool> m(fields.size(), false);
  for (size_t i = 0; i < fields.size(); ++i) if (fields[i].name == json_to_arrow_value_field(jp)) m[i] = true;
  return m;
}

int ark_json_to_arrow_process(ark_proc_t* p, ArrowArray* in, ArrowSchema* in_schema, ArrowArray* out, ArrowSchema* out_schema) {
  BufferPtr in_owner = adopt_array(in);
  return guarded([&] {
    Processor* jp = as_json(p);
    const ArrowArray* arr = (const ArrowArray*)in_owner.get();
    if (!arr) fail(ARK_ERR_PROCESS, "input array already released");
    std::vector<Field> fields = schema_fields(in_schema);
    std::vector<bool> mask = json_mask(*jp, fields);
    StreamLease lease;
    Batch b = import_host(arr, in_schema, &mask, lease.s);
    Batch r = json_to_arrow_device(*jp, b, lease.s);
    export_host(r, lease.s, out, out_schema);
  });
}

int ark_json_to_arrow_process_device(ark_proc_t* p, ArrowDeviceArray* in, ArrowSchema* in_schema, ArrowDeviceArray* out,
                                     ArrowSchema* out_schema) {
  BufferPtr in_owner = adopt_array(&in->array);
  return guarded([&] {
    Processor* jp = as_json(p);
    if (!in_owner) fail(ARK_ERR_PROCESS, "input array already released");
    ArrowDeviceArray view = *in;
    view.array = *(const ArrowArray*)in_owner.get();
    std::vector<Field> fields = schema_fields(in_schema);
    std::vector<bool> mask = json_mask(*jp, fields);
    StreamLease lease;
    Batch b = import_device(&view, in_schema, &mask, in_owner);
    Batch r = json_to_arrow_device(*jp, b, lease.s);
    export_device(r, out, out_schema);
  });
}

int ark_arrow_to_json_create(const char* config_json, ark_proc_t** out) {
  return guarded([&] {
    if (!out) fail(ARK_ERR_PROCESS, "null output handle");
    *out = nullptr;
    auto p = make_arrow_to_json(config_json);
    auto* h = new ark_proc();
    h->impl = std::move(p);
    *out = h;
  });
}

int ark_arrow_to_json_process(ark_proc_t* p, ArrowArray* in, ArrowSchema* in_schema, ArrowArray* out, ArrowSchema* out_schema) {
  BufferPtr in_owner = adopt_array(in);
  return guarded([&] {
    if (!p || !p->impl || strcmp(p->impl->type(), "arrow_to_json") != 0) fail(ARK_ERR_PROCESS, "handle is not an arrow_to_json processor");
    const ArrowArray* arr = (const ArrowArray*)in_owner.get();
    if (!arr) fail(ARK_ERR_PROCESS, "input array already released");
    StreamLease lease;
    Batch b = import_host(arr, in_schema, nullptr, lease.s);
    Batch r = arrow_to_json_device(*p->impl, b, lease.s);
    export_host(r, lease.s, out, out_schema);
  });
}

int ark_arrow_to_json_process_device(ark_proc_t* p, ArrowDeviceArray* in, ArrowSchema* in_schema, ArrowDeviceArray* out,
                                     ArrowSchema* out_schema) {
  BufferPtr in_owner = adopt_array(&in->array);
  return guarded([&] {
    if (!p || !p->impl || strcmp(p->impl->type(), "arrow_to_json") != 0) fail(ARK_ERR_PROCESS, "handle is not an arrow_to_json processor");
    if (!in_owner) fail(ARK_ERR_PROCESS, "input array already released");
    ArrowDeviceArray view = *in;
    view.array = *(const ArrowArray*)in_owner.get();
    StreamLease lease;
    Batch b = import_device(&view, in_schema, nullptr, in_owner);
    std::vector<Column*> all;
    for (auto& c : b.cols) all.push_back(&c);
    resolve_varlen_extents_many(all, lease.s);
    Batch r = arrow_to_json_device(*p->impl, b, lease.s);
    export_device(r, out, out_schema);
  });
}

// ---- protobuf_to_arrow / arrow_to_protobuf (processor/protobuf.rs:98-148) --------------------------------------
static int create_proc(std::unique_ptr<Processor> (*make)(const char*), const char* config_json, ark_proc_t** out) {
  return guarded([&] {
    if (!out) fail(ARK_ERR_PROCESS, "null output handle");
    *out = nullptr;
    auto p = make(config_json);
    auto* h = new ark_proc();
    h->impl = std::move(p);
    *out = h;
  });
}

static Processor* as_type(ark_proc_t* p, const char* type) {
  if (!p || !p->impl || strcmp(p->impl->type(), type) != 0) fail(ARK_ERR_PROCESS, std::string("handle is not a ") + type + " processor");
  return p->impl.get();
}

int ark_protobuf_to_arrow_create(const char* config_json, ark_proc_t** out) { return create_proc(make_protobuf_to_arrow, config_json, out); }

static std::vector<bool> protobuf_mask(const Processor& pp, const std::vector<Field>& fields) {
  std::vector<bool> m(fields.size(), false);
  for (size_t i = 0; i < fields.size(); ++i) if (fields[i].name == protobuf_to_arrow_value_field(pp)) m[i] = true;
  return m;
}

int ark_protobuf_to_arrow_process(ark_proc_t* p, ArrowArray* in, ArrowSchema* in_schema, ArrowArray* out, ArrowSchema* out_schema) {
  BufferPtr in_owner = adopt_array(in);
  return guarded([&] {
    Processor* pp = as_type(p, "protobuf_to_arrow");
    const ArrowArray* arr = (const ArrowArray*)in_owner.get();
    if (!arr) fail(ARK_ERR_PROCESS, "input array already released");
    if (arr->length == 0) { set_none(out, out_schema); return; }  // ProcessResult::None, protobuf.rs:101-103
    std::vector<Field> fields = schema_fields(in_schema);
    std::vector<bool> mask = protobuf_mask(*pp, fields);
    StreamLease lease;
    Batch b = import_host(arr, in_schema, &mask, lease.s);
    Batch r = protobuf_to_arrow_device(*pp, b, lease.s);
    export_host(r, lease.s, out, out_schema);
  });
}

int ark_protobuf_to_arrow_process_device(ark_proc_t* p, ArrowDeviceArray* in, ArrowSchema* in_schema, ArrowDeviceArray* out,
                                         ArrowSchema* out_schema) {
  BufferPtr in_owner = adopt_array(&in->array);
  return guarded([&] {
    Processor* pp = as_type(p, "protobuf_to_arrow");
    if (!in_owner) fail(ARK_ERR_PROCESS, "input array already released");
    ArrowDeviceArray view = *in;
    view.array = *(const ArrowArray*)in_owner.get();
    if (view.array.length == 0) { memset(out, 0, sizeof(*out)); if (out_schema) memset(out_schema, 0, sizeof(*out_schema)); return; }
    std::vector<Field> fields = schema_fields(in_schema);
    std::vector<bool> mask = protobuf_mask(*pp, fields);
    StreamLease lease;
    Batch b = import_device(&view, in_schema, &mask, in_owner);
    Batch r = protobuf_to_arrow_device(*pp, b, lease.s);
    export_device(r, out, out_schema);
  });
}

int ark_arrow_to_protobuf_create(const char* config_json, ark_proc_t** out) { return create_proc(make_arrow_to_protobuf, config_json, out); }

int ark_arrow_to_protobuf_process(ark_proc_t* p, ArrowArray* in, ArrowSchema* in_schema, ArrowArray* out, ArrowSchema* out_schema) {
  BufferPtr in_owner = adopt_array(in);
  return guarded([&] {
    Processor* pp = as_type(p, "arrow_to_protobuf");
    const ArrowArray* arr = (const ArrowArray*)in_owner.get();
    if (!arr) fail(ARK_ERR_PROCESS, "input array already released");
    if (arr->length == 0) { set_none(out, out_schema); return; }  // ProcessResult::None, protobuf.rs:101-103
    StreamLease lease;
    Batch b = import_host(arr, in_schema, nullptr, lease.s, nullptr, true);
    Batch r = arrow_to_protobuf_device(*pp, b, lease.s);
    export_host(r, lease.s, out, out_schema);
  });
}

int ark_arrow_to_protobuf_process_device(ark_proc_t* p, ArrowDeviceArray* in, ArrowSchema* in_schema, ArrowDeviceArray* out,
                                         ArrowSchema* out_schema) {
  BufferPtr in_owner = adopt_array(&in->array);
  return guarded([&] {
    Processor* pp = as_type(p, "arrow_to_protobuf");
    if (!in_owner) fail(ARK_ERR_PROCESS, "input array already released");
    ArrowDeviceArray view = *in;
    view.array = *(const ArrowArray*)in_owner.get();
    if (view.array.length == 0) { memset(out, 0, sizeof(*out)); if (out_schema) memset(out_schema, 0, sizeof(*out_schema)); return; }
    StreamLease lease;
    Batch b = import_device(&view, in_schema, nullptr, in_owner, true);
    std::vector<Column*> all;
    for (auto& c : b.cols) all.push_back(&c);
    resolve_varlen_extents_many(all, lease.s);
    Batch r = arrow_to_protobuf_device(*pp, b, lease.s);
    export_device(r, out, out_schema);
  });
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
    if (!expr || !out) fail(ARK_ERR_PROCESS, "null argument");
    const ArrowArray* arr = (const ArrowArray*)in_owner.get();
    if (!arr) fail(ARK_ERR_PROCESS, "input array already released");
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
    if (!expr || !out) fail(ARK_ERR_PROCESS, "null argument");
    if (!in_owner) fail(ARK_ERR_PROCESS, "input array already released");
    ArrowDeviceArray view = *in;
    view.array = *(const ArrowArray*)in_owner.get();
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
    ARK_CUDA(cudaStreamSynchronize(lease.s));
    export_device(r, out, out_schema);
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
