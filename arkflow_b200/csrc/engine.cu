// engine.cu — SqlProcessor (host side) and the filter/project executor.
#include "engine.h"

#include <algorithm>

#include "bitmap.h"
#include "json_mini.h"

namespace ark {

std::unique_ptr<SqlProcessor> SqlProcessor::from_config(const char* config_json) {
  // reference: sql.rs:235-239 — the message really says "Batch processor" (copy-paste in the reference)
  if (!config_json) fail(ARK_ERR_CONFIG, "Batch processor configuration is missing");
  JsonValue cfg = parse_json(config_json);
  if (cfg.kind == JsonValue::Null) fail(ARK_ERR_CONFIG, "Batch processor configuration is missing");
  if (cfg.kind != JsonValue::Object) fail(ARK_ERR_SERIALIZATION, "invalid type: expected struct SqlProcessorConfig");
  const JsonValue* q = cfg.get("query");
  if (!q) fail(ARK_ERR_SERIALIZATION, "missing field `query`");
  if (q->kind != JsonValue::String) fail(ARK_ERR_SERIALIZATION, "invalid type for `query`: expected a string");
  auto p = std::make_unique<SqlProcessor>();
  p->query_text = q->str;
  p->json_functions = true;  // sql.rs:18-24 registers datafusion-functions-json
  if (const JsonValue* t = cfg.get("table_name")) {
    if (t->kind == JsonValue::String) p->table_name = t->str;
    else if (t->kind != JsonValue::Null) fail(ARK_ERR_SERIALIZATION, "invalid type for `table_name`: expected a string");
  }
  bool resolved = false;  // the shim owns Resource.temporary: it checks the names (sql.rs:70-86) and says so
  if (const JsonValue* r = cfg.get("temporaries_resolved")) resolved = r->kind == JsonValue::Bool && r->b;
  if (const JsonValue* tl = cfg.get("temporary_list")) {
    if (tl->kind == JsonValue::Array && !tl->arr.empty() && !resolved) {
      // sql.rs:70-86: temporaries are looked up in Resource; without the shim's confirmation a configured
      // temporary is by construction "not found".
      const JsonValue* nm = tl->arr[0].get("name");
      fail(ARK_ERR_PROCESS, "Temporary " + (nm && nm->kind == JsonValue::String ? nm->str : std::string("?")) + " not found");
    }
  }
  p->ast = parse_sql(p->query_text);  // throws "SQL query error: …" (sql.rs:92-98)
  return p;
}

std::shared_ptr<const Plan> SqlProcessor::plan_for(const std::vector<Field>& fields) {
  std::string key = schema_fingerprint(fields);
  {
    std::lock_guard<std::mutex> l(mu_);
    auto it = plans_.find(key);
    if (it != plans_.end()) { if (it->second->kind == Plan::Aggregate) last_agg_ = it->second; return it->second; }
  }
  auto plan = std::make_shared<Plan>(bind_query(ast, table_name, fields, json_functions));
  std::lock_guard<std::mutex> l(mu_);
  if (plans_.size() > 64) plans_.clear();
  plans_[key] = plan;
  if (plan->kind == Plan::Aggregate) last_agg_ = plan;
  return plan;
}

std::vector<bool> needed_mask(const Plan& plan, size_t n_fields) {
  std::vector<bool> m(n_fields, false);
  if (plan.identity) { std::fill(m.begin(), m.end(), true); return m; }
  for (int c : plan.used_cols) if ((size_t)c < n_fields) m[c] = true;  // the others are derived columns
  for (auto& d : plan.derived) m[d.doc_col] = true;
  return m;
}

static bool same_schema(const ArrowSchema* s, const std::vector<Field>& f) {
  if (!s || !s->format || strcmp(s->format, "+s") != 0 || s->n_children != (int64_t)f.size()) return false;
  for (size_t i = 0; i < f.size(); ++i) {
    const ArrowSchema* c = s->children[i];
    if (strcmp(c->name ? c->name : "", f[i].name.c_str()) != 0 || strcmp(c->format ? c->format : "", f[i].format.c_str()) != 0 ||
        ((c->flags & ARROW_FLAG_NULLABLE) != 0) != f[i].nullable)
      return false;
  }
  return true;
}

std::shared_ptr<const SqlProcessor::BoundSchema> SqlProcessor::bind(const ArrowSchema* schema) {
  {
    std::lock_guard<std::mutex> l(mu_);
    if (last_bound_ && same_schema(schema, last_bound_->fields)) {
      if (last_bound_->plan->kind == Plan::Aggregate) last_agg_ = last_bound_->plan;  // as plan_for does
      return last_bound_;
    }
  }
  auto b = std::make_shared<BoundSchema>();
  b->fields = schema_fields(schema);
  b->plan = plan_for(b->fields);
  b->mask = needed_mask(*b->plan, b->fields.size());
  std::lock_guard<std::mutex> l(mu_);
  last_bound_ = b;
  return b;
}

std::shared_ptr<const Plan> SqlProcessor::last_aggregate_plan() {
  std::lock_guard<std::mutex> l(mu_);
  return last_agg_;
}

std::shared_ptr<const Plan> SqlProcessor::join_plan_for(const std::vector<std::string>& names,
                                                        const std::vector<std::vector<Field>>& tables) {
  std::string key = "J";
  for (size_t i = 0; i < names.size(); ++i) { key += names[i]; key += '\x1d'; key += schema_fingerprint(tables[i]); key += '\x1c'; }
  {
    std::lock_guard<std::mutex> l(mu_);
    auto it = plans_.find(key);
    if (it != plans_.end()) return it->second;
  }
  auto plan = std::make_shared<Plan>(bind_join(ast, names, tables));
  std::lock_guard<std::mutex> l(mu_);
  if (plans_.size() > 64) plans_.clear();
  plans_[key] = plan;
  return plan;
}

Batch SqlProcessor::execute(const Plan& plan, Batch& batch, cudaStream_t stream) {
  Batch with_json;
  if (!plan.derived.empty()) with_json = append_json_columns(plan, batch, stream);
  Batch& in = plan.derived.empty() ? batch : with_json;
  switch (plan.kind) {
    case Plan::FilterProject: {
      Batch r = run_filter_project(plan, in, stream);
      return plan.concats.empty() ? r : apply_concats(plan, r, stream);
    }
    case Plan::Aggregate: return run_aggregate(plan, in, stream);
    default: fail(ARK_ERR_PROCESS, "internal: join plan executed through the single-table path");
  }
}

// ---- filter / project ---------------------------------------------------------------------------------

namespace {

struct PendingOut {
  int out_index;            // index into plan.outputs
  BufferPtr data, offsets, valid_bytes;
  bool is_bool = false;
};

}  // namespace

const char* vm_error_text(int e) {
  switch (e) {
    case VMERR_DIV_ZERO: return "Arrow error: Divide by zero error";
    case VMERR_OVERFLOW: return "Arrow error: Arithmetic overflow: Overflow happened on: -9223372036854775808 / -1";
    case VMERR_OVERFLOW_MOD: return "Arrow error: Arithmetic overflow: Overflow happened on: -9223372036854775808 % -1";
    case VMERR_CAST: return "Arrow error: Cast error: Can't cast value to type Int64";
    default: return "unknown evaluation error";
  }
}


// ---- fast path: filter_project_tma.cu ------------------------------------------------------------------
int filter_project_tma_tile_rows();
int filter_project_tma_max_fixed_out();
size_t filter_project_tma_desc_words(int64_t n_tiles);
void filter_project_tma_note_avg_len(double avg);
bool launch_filter_project_tma(int64_t n_rows, const void* pred_in, int n_fixed_out, const void* const* fixed_in, void* const* fixed_out,
                               const int32_t* offsets_in, const uint8_t* data_in, int64_t data_bytes, int32_t* offsets_out, uint8_t* data_out,
                               int cmp, int is_f64, uint64_t constant, unsigned long long* desc, unsigned long long* desc_next,
                               long long* totals, cudaStream_t stream);

// SELECT <fixed-width cols…> [, <1 var-len col>] WHERE <fixed col> <cmp> <literal>, no NULLs in the used columns.
static bool try_fast_filter(const Plan& plan, Batch& in, Batch& out, cudaStream_t stream) {
  if (!plan.has_pred || !plan.simple.enabled || plan.outputs.empty()) return false;
  auto src_col = [&](int slot) -> Column& { return in.cols[plan.used_cols[slot]]; };
  for (size_t s = 0; s < plan.used_cols.size(); ++s) if (src_col((int)s).validity) return false;
  const int max_fixed = filter_project_tma_max_fixed_out();
  std::vector<int> fixed_outs;
  int varlen_out = -1;
  for (size_t i = 0; i < plan.outputs.size(); ++i) {
    const OutputCol& oc = plan.outputs[i];
    if (oc.src.kind != ValueSource::PassThrough) return false;
    const DType t = src_col(oc.src.slot).field.type;
    if (t == DType::Int64 || t == DType::Float64) { if ((int)fixed_outs.size() == max_fixed) return false; fixed_outs.push_back((int)i); }
    else if (t == DType::Utf8 || t == DType::Binary) { if (varlen_out >= 0) return false; varlen_out = (int)i; }
    else return false;
  }
  const int64_t n = in.num_rows;
  const int n_tiles = (int)ceil_div(n, filter_project_tma_tile_rows());
  const void* fin[8] = {nullptr};
  void* fout[8] = {nullptr};
  std::vector<BufferPtr> fbuf(fixed_outs.size());
  BufferPtr obuf, dbuf;
  const Column* vs = varlen_out >= 0 ? &src_col(plan.outputs[varlen_out].src.slot) : nullptr;
  {  // every output buffer is cut from one pool block (one allocation and one free per call); each piece is 256-byte aligned
    auto piece = [](size_t bytes) { return (size_t)round_up((int64_t)bytes, 256); };
    const size_t fixed_bytes = piece((size_t)n * 8 + 16), off_bytes = vs ? piece((size_t)(n + 1) * 4 + 16) : 0;
    const size_t data_bytes = vs ? piece((size_t)std::max<int64_t>(varlen_bytes_bound(*vs), 0) + 32) : 0;
    BufferPtr block = device_alloc(fixed_bytes * fixed_outs.size() + off_bytes + data_bytes);
    uint8_t* p = (uint8_t*)block.get();
    for (size_t c = 0; c < fixed_outs.size(); ++c, p += fixed_bytes) {
      fin[c] = src_col(plan.outputs[fixed_outs[c]].src.slot).data;
      fbuf[c] = BufferPtr(block, p);
      fout[c] = p;
    }
    if (vs) { obuf = BufferPtr(block, p); dbuf = BufferPtr(block, p + off_bytes); }
  }
  // Look-back descriptors: the stream's two buffers in turn.  Each launch's tiles zero, in the other buffer, the words the
  // next launch with the same tile count reads; calls on one stream are serialised, so nothing reads that buffer meanwhile.
  // A buffer whose state is unknown or that was zeroed for another tile count is cleared with one memset.
  FilterScratch unleased;  // a stream this thread does not lease: nothing is known about its buffers
  FilterScratch* leased = lease_filter_scratch(stream);
  FilterScratch& fs = leased ? *leased : unleased;
  const size_t desc_bytes = filter_project_tma_desc_words(n_tiles) * 8;
  const int cur = fs.next, other = cur ^ 1;
  for (int k : {cur, other})
    if (fs.desc_bytes[k] < desc_bytes) {
      fs.desc[k] = device_alloc(desc_bytes);
      fs.desc_bytes[k] = desc_bytes;
      fs.zeroed_for[k] = -1;
    }
  if (fs.zeroed_for[cur] != n_tiles) ARK_CUDA(cudaMemsetAsync(fs.desc[cur].get(), 0, desc_bytes, stream));
  // the kernel's last tile stores the two totals straight into pinned host memory (device-accessible under unified
  // addressing): one stream synchronize, no separate device→host copy on the critical path of every call
  if (!fs.totals) fs.totals = pinned_alloc(64);
  long long* totals = (long long*)fs.totals.get();
  fs.zeroed_for[cur] = -1;
  if (trace_enabled()) tl_call_trace.prepared = std::chrono::steady_clock::now();
  if (!launch_filter_project_tma(n, src_col(plan.simple.slot).data, (int)fixed_outs.size(), fin, fout, vs ? vs->offsets : nullptr,
                                 vs ? vs->data : nullptr, vs ? vs->data_bytes : 0 /* -1 = unknown */, vs ? (int32_t*)obuf.get() : nullptr,
                                 vs ? (uint8_t*)dbuf.get() : nullptr, plan.simple.cmp, plan.simple.is_f64, plan.simple.constant,
                                 (unsigned long long*)fs.desc[cur].get(), (unsigned long long*)fs.desc[other].get(), totals, stream))
    return false;
  ARK_CUDA(cudaGetLastError());
  fs.zeroed_for[other] = n_tiles;
  fs.next = other;
  if (trace_enabled()) tl_call_trace.launched = std::chrono::steady_clock::now();
  ARK_CUDA(cudaStreamSynchronize(stream));
  if (trace_enabled()) tl_call_trace.synced = std::chrono::steady_clock::now();
  const int64_t count = totals[0], bytes = totals[1];
  if (vs && count > 0) filter_project_tma_note_avg_len((double)bytes / (double)count);
  out.cols.resize(plan.outputs.size());
  out.num_rows = count;
  for (size_t i = 0; i < plan.outputs.size(); ++i) {
    const OutputCol& oc = plan.outputs[i];
    Column& c = out.cols[i];
    c.field.name = oc.name; c.field.type = oc.src.type; c.field.nullable = oc.src.nullable;
    c.length = count; c.null_count = 0;
    if ((int)i == varlen_out) {
      c.offsets = (const int32_t*)obuf.get(); c.data = (const uint8_t*)dbuf.get(); c.data_bytes = bytes; c.first_offset = 0;
      c.owners = {obuf, dbuf};
    } else {
      size_t k = 0;
      while (fixed_outs[k] != (int)i) ++k;
      c.data = (const uint8_t*)fbuf[k].get(); c.data_bytes = count * 8; c.owners = {fbuf[k]};
    }
  }
  return true;
}

// CAST(Binary AS Utf8) columns: arrow-cast (safe = false) fails the query on invalid UTF-8.
static void validate_utf8_outputs(const Plan& plan, Batch& out, cudaStream_t stream) {
  bool any = false;
  for (auto& oc : plan.outputs) any = any || oc.src.validate_utf8;
  if (!any || out.num_rows == 0) return;
  BufferPtr flag = device_alloc(16), h = pinned_alloc(16);
  ARK_CUDA(cudaMemsetAsync(flag.get(), 0, 16, stream));
  for (size_t i = 0; i < plan.outputs.size(); ++i) {
    if (!plan.outputs[i].src.validate_utf8) continue;
    const Column& c = out.cols[i];
    launch_utf8_validate(c.offsets, c.data, c.validity, c.validity_bit0, c.length, (int*)flag.get(), stream);
  }
  ARK_CUDA(cudaMemcpyAsync(h.get(), flag.get(), 4, cudaMemcpyDeviceToHost, stream));
  ARK_CUDA(cudaStreamSynchronize(stream));
  if (*(int*)h.get()) fail(ARK_ERR_PROCESS, "Collection query results error: Arrow error: Cast error: Cannot cast binary to string: invalid utf-8 sequence");
}

Batch run_filter_project(const Plan& plan, Batch& in, cudaStream_t stream) {
  const int64_t n = in.num_rows;
  Batch out;
  out.input_name = in.input_name;
  auto src_col = [&](int slot) -> Column& { return in.cols[plan.used_cols[slot]]; };

  if (plan.identity) {  // SELECT * FROM flow: the batch itself (zero copy)
    out.cols = in.cols;
    out.num_rows = n;
    return out;
  }

  {  // outputs are allocated worst-case: an upper bound on each var-len source is enough
    std::vector<int> unknown;
    for (auto& oc : plan.outputs)
      if (oc.src.kind == ValueSource::PassThrough) {
        const Column& c = in.cols[plan.used_cols[oc.src.slot]];
        if ((c.field.type == DType::Utf8 || c.field.type == DType::Binary) && varlen_bytes_bound(c) < 0) unknown.push_back(plan.used_cols[oc.src.slot]);
      }
    if (!unknown.empty()) resolve_varlen_extents(in, unknown, stream);
  }

  if (try_fast_filter(plan, in, out, stream)) {
    validate_utf8_outputs(plan, out, stream);
    if (plan.limit >= 0 && out.num_rows > plan.limit) {
      out.num_rows = plan.limit;
      for (auto& c : out.cols) { c.length = plan.limit; if (c.field.type == DType::Utf8 || c.field.type == DType::Binary) c.data_bytes = -1; }
      std::vector<int> all;
      for (size_t i = 0; i < out.cols.size(); ++i) all.push_back((int)i);
      resolve_varlen_extents(out, all, stream);
    }
    return out;
  }

  out.cols.resize(plan.outputs.size());
  std::vector<int> todo;  // outputs that need the kernel
  for (size_t i = 0; i < plan.outputs.size(); ++i) {
    const OutputCol& oc = plan.outputs[i];
    Column& c = out.cols[i];
    c.field.name = oc.name; c.field.type = oc.src.type; c.field.nullable = oc.src.nullable;
    if (!plan.has_pred && oc.src.kind == ValueSource::PassThrough) {
      Column& s = src_col(oc.src.slot);  // no filter: the projected column is the input column
      Field f = c.field;
      c = s; c.field = f;
    } else todo.push_back((int)i);
  }
  out.num_rows = n;

  int64_t count = n;
  if (!todo.empty() || plan.has_pred) {
    const int n_tiles = (int)ceil_div(n, FP_TILE);
    if (n_tiles <= 0) fail(ARK_ERR_PROCESS, "internal: empty batch reached the filter kernel");
    std::vector<PendingOut> pend;
    // scratch: [desc | ticket | totals | error] per launch; results gathered into one pinned block
    const size_t desc_bytes = (size_t)n_tiles * FP_CHANNELS * 8;
    const size_t scratch_bytes = round_up((int64_t)desc_bytes + 64 + FP_CHANNELS * 8, 256);
    size_t pos = 0;
    std::vector<BufferPtr> scratches;
    std::vector<int> launch_n_out;
    BufferPtr host_res = pinned_alloc(4096);
    int launches = 0;
    bool first = true;
    while (first || pos < todo.size()) {
      first = false;
      FpParams P;
      memset(&P, 0, sizeof P);
      P.n_rows = n; P.n_tiles = n_tiles;
      for (size_t s = 0; s < plan.used_cols.size(); ++s) P.cols[s] = src_col((int)s).view();
      int pred_kind = !plan.has_pred ? 0 : (plan.simple.enabled ? 1 : 2);
      if (pred_kind == 1) { P.sp_slot = plan.simple.slot; P.sp_cmp = plan.simple.cmp; P.sp_is_f64 = plan.simple.is_f64; P.sp_const = plan.simple.constant; }
      if (pred_kind == 2) P.pred = plan.pred;
      int n_progs = 0;
      while (pos < todo.size() && P.n_out < FP_MAX_OUT) {
        const int oi = todo[pos];
        const OutputCol& oc = plan.outputs[oi];
        const bool computed = oc.src.kind == ValueSource::Computed;
        const bool varlen = !computed && (oc.src.type == DType::Utf8 || oc.src.type == DType::Binary);
        if (computed && n_progs == FP_MAX_PROGS) break;
        if (varlen && P.n_varlen == FP_MAX_VARLEN) break;
        FpOutput& fo = P.outs[P.n_out];
        PendingOut po; po.out_index = oi;
        const Column* s = computed ? nullptr : &src_col(oc.src.slot);
        bool want_valid = computed ? oc.src.nullable : (s->validity != nullptr);
        if (want_valid) { po.valid_bytes = device_alloc((size_t)n); fo.out_valid = (uint8_t*)po.valid_bytes.get(); fo.write_validity = 1; }
        if (computed) {
          fo.prog = n_progs; P.progs[n_progs++] = oc.src.prog;
          if (oc.src.type == DType::Bool) { fo.kind = FP_OUT_COMPUTED_BOOL; po.is_bool = true; po.data = device_alloc((size_t)n); }
          else { fo.kind = FP_OUT_COMPUTED8; po.data = device_alloc((size_t)n * 8); }
        } else if (varlen) {
          fo.kind = FP_OUT_VARLEN; fo.slot = oc.src.slot; fo.varlen_idx = P.n_varlen;
          P.varlen_slot[P.n_varlen++] = oc.src.slot;
          po.offsets = device_alloc((size_t)(n + 1) * 4);
          po.data = device_alloc((size_t)std::max<int64_t>(varlen_bytes_bound(*s), 0) + 16);
          fo.out_offsets = (int32_t*)po.offsets.get();
        } else if (oc.src.type == DType::Bool) {
          fo.kind = FP_OUT_BOOL; fo.slot = oc.src.slot; po.is_bool = true; po.data = device_alloc((size_t)n);
        } else if (oc.src.type == DType::Int64 || oc.src.type == DType::Float64) {
          fo.kind = FP_OUT_FIXED8; fo.slot = oc.src.slot; po.data = device_alloc((size_t)n * 8);
        } else {
          fail(ARK_ERR_UNSUPPORTED, std::string("projection of a ") + dtype_name(oc.src.type) + " column");
        }
        fo.out_data = po.data.get();
        pend.push_back(std::move(po));
        ++P.n_out; ++pos;
      }
      BufferPtr scratch = device_alloc(scratch_bytes);
      ARK_CUDA(cudaMemsetAsync(scratch.get(), 0, scratch_bytes, stream));
      P.desc = (unsigned long long*)scratch.get();
      P.ticket = (unsigned int*)((char*)scratch.get() + desc_bytes);
      P.totals = (long long*)((char*)scratch.get() + desc_bytes + 16);
      P.error = (int32_t*)((char*)scratch.get() + desc_bytes + 8);
      launch_filter_project(P, pred_kind, stream);
      ARK_CUDA(cudaGetLastError());
      if (launches >= 32) fail(ARK_ERR_UNSUPPORTED, "too many output columns");
      // totals[FP_CHANNELS] + error live contiguously from desc_bytes+8: copy 8 + 8 + 24 bytes
      ARK_CUDA(cudaMemcpyAsync((char*)host_res.get() + launches * 64, (char*)scratch.get() + desc_bytes, 64,
                               cudaMemcpyDeviceToHost, stream));
      scratches.push_back(scratch);
      launch_n_out.push_back(P.n_out);
      ++launches;
    }
    ARK_CUDA(cudaStreamSynchronize(stream));
    for (int l = 0; l < launches; ++l) {
      const char* base = (const char*)host_res.get() + l * 64;
      int32_t err = *(const int32_t*)(base + 8);
      if (err) fail(ARK_ERR_PROCESS, std::string("Collection query results error: ") + vm_error_text(err));
    }
    count = *(const int64_t*)((const char*)host_res.get() + 16);
    // finish the columns produced by the kernel
    size_t pi = 0;
    for (int l = 0; l < launches; ++l) {
      const int64_t* totals = (const int64_t*)((const char*)host_res.get() + l * 64 + 16);
      int vseen = 0;
      const int n_out = launch_n_out[l];
      for (int k = 0; k < n_out; ++k, ++pi) {
        PendingOut& po = pend[pi];
        const OutputCol& oc = plan.outputs[po.out_index];
        Column& c = out.cols[po.out_index];
        c.length = count; c.present = true;
        const bool varlen = po.offsets != nullptr;
        if (varlen) {
          c.offsets = (const int32_t*)po.offsets.get(); c.data = (const uint8_t*)po.data.get();
          c.data_bytes = totals[1 + vseen]; c.first_offset = 0; ++vseen;
          c.owners = {po.offsets, po.data};
        } else if (po.is_bool) {
          set_bool_values(c, po.data, count, stream);
        } else {
          c.data = (const uint8_t*)po.data.get(); c.data_bytes = count * 8; c.owners = {po.data};
        }
        if (po.valid_bytes) set_validity_unknown(c, po.valid_bytes, count, stream);
        else set_validity(c, nullptr, 0);
        (void)oc;
      }
    }
    // zero-copy passthrough columns of a predicate-less projection keep length n (= count)
    out.num_rows = count;
  }

  validate_utf8_outputs(plan, out, stream);
  if (plan.limit >= 0 && out.num_rows > plan.limit) {
    // LIMIT k without ORDER BY on a single-partition scan: the first k surviving rows
    out.num_rows = plan.limit;
    for (auto& c : out.cols) {
      c.length = plan.limit;
      if (c.field.type == DType::Utf8 || c.field.type == DType::Binary) c.data_bytes = -1;
    }
    std::vector<int> all;
    for (size_t i = 0; i < out.cols.size(); ++i) all.push_back((int)i);
    resolve_varlen_extents(out, all, stream);
  }
  return out;
}

void refuse_limit_across_ranks(const Plan& plan) {
  if (plan.kind == Plan::Aggregate && plan.limit >= 0)
    fail(ARK_ERR_UNSUPPORTED, "SQL outside the GPU subset: LIMIT on an aggregate split across ranks (each rank holds only part of the "
                              "groups, so a per-rank LIMIT is not the query's LIMIT)");
}

// HAVING, computed items and LIMIT of an aggregate query: its stage plan over the group frame, on the call's stream.
Batch run_group_stage(const Plan& plan, Batch& frame, cudaStream_t stream) {
  if (!plan.stage) return frame;
  const Plan& stage = *plan.stage;
  if (frame.num_rows > 0) {
    Batch r = run_filter_project(stage, frame, stream);
    return stage.concats.empty() ? r : apply_concats(stage, r, stream);
  }
  // no group (a WHERE that kept no row): the filter kernels need a row, so the empty result is built here
  Batch out;
  out.input_name = frame.input_name;
  BufferPtr z = device_alloc(16);
  ARK_CUDA(cudaMemsetAsync(z.get(), 0, 16, stream));
  auto empty = [&](const std::string& name, DType type, bool nullable) {
    Column c;
    c.field.name = name; c.field.type = type; c.field.nullable = nullable;
    c.length = 0; c.data = (const uint8_t*)z.get(); c.data_bytes = 0;
    if (type == DType::Utf8 || type == DType::Binary) { c.offsets = (const int32_t*)z.get(); c.first_offset = 0; }
    c.owners = {z};
    out.cols.push_back(c);
  };
  if (stage.concats.empty()) {
    for (const OutputCol& oc : stage.outputs) empty(oc.name, oc.src.type, oc.src.nullable);
  } else {
    for (const FinalItem& fi : stage.final_items) {
      if (!fi.is_concat) { const OutputCol& oc = stage.outputs[fi.index]; empty(oc.name, oc.src.type, oc.src.nullable); continue; }
      const ConcatItem& ci = stage.concats[fi.index];
      const bool cast_col = ci.is_cast && !ci.parts.empty() && !ci.parts[0].is_literal;
      empty(ci.name, DType::Utf8, cast_col ? stage.outputs[ci.parts[0].out_index].src.nullable : true);
    }
  }
  ARK_CUDA(cudaStreamSynchronize(stream));
  return out;
}

}  // namespace ark
