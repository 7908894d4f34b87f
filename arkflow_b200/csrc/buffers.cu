// buffers.cu — the buffer stage: memory / session_window / tumbling_window / sliding_window
// (+ JoinOperation) and the count/timeout `batch` processor, with the queued batches resident in HBM and
// concat / json-decode / join running as kernels.
//
//   MemoryBuffer   ← crates/arkflow-plugin/src/buffer/memory.rs:39-237   (drain OLDEST first: push_front / pop_back)
//   BaseWindow     ← crates/arkflow-plugin/src/buffer/window.rs:28-217   (per-input queues, drain NEWEST first: push_front / pop_front)
//   SessionWindow  ← crates/arkflow-plugin/src/buffer/session_window.rs:97-159
//   TumblingWindow ← crates/arkflow-plugin/src/buffer/tumbling_window.rs:90-145
//   JoinOperation  ← crates/arkflow-plugin/src/buffer/join.rs:62-146
//   SlidingWindow  ← crates/arkflow-plugin/src/buffer/sliding_window.rs:52-238 (FIFO of batches; a window = the
//                    first window_size BATCHES in arrival order, then slide_size of them are dropped)
//   BatchProcessor ← crates/arkflow-plugin/src/processor/batch.rs:37-124
// tokio's Notify + timer task become a condition variable + a timer thread; the wake-up rules are the
// reference's (capacity reached, timer tick, flush/close).  Deliberate differences (SURVEY.md app. D):
// row totals are kept incrementally instead of recounted on every write; a reader that is already
// waiting when the window is flushed drains what is left instead of waiting for a tick that never comes;
// a sliding-window reader blocked on a flushed/closed buffer gets None instead of hanging (the
// reference's timer task exits on close, so nothing would ever wake that reader again).
#include <algorithm>
#include <chrono>
#include <condition_variable>
#include <deque>
#include <thread>

#include "abi.h"
#include "json_mini.h"

using namespace ark;

namespace {

using Clock = std::chrono::steady_clock;

// humantime::parse_duration subset: "<int><unit>" terms, units ns us µs ms s sec m min h hr d
std::chrono::nanoseconds parse_duration(const std::string& s) {
  auto bad = [&]() -> std::chrono::nanoseconds {
    fail(ARK_ERR_SERIALIZATION, "invalid value: string \"" + s + "\", expected a duration like '10ms' or '1s'");
  };
  size_t i = 0;
  long double total = 0;
  bool any = false;
  while (i < s.size()) {
    while (i < s.size() && isspace((unsigned char)s[i])) ++i;
    if (i >= s.size()) break;
    size_t j = i;
    while (j < s.size() && isdigit((unsigned char)s[j])) ++j;
    if (j == i) bad();
    const long double v = (long double)strtoull(s.substr(i, j - i).c_str(), nullptr, 10);
    size_t k = j;
    while (k < s.size() && !isdigit((unsigned char)s[k]) && !isspace((unsigned char)s[k])) ++k;
    const std::string u = s.substr(j, k - j);
    long double mul;
    if (u == "ns" || u == "nsec") mul = 1;
    else if (u == "us" || u == "usec" || u == "\xC2\xB5s") mul = 1e3;
    else if (u == "ms" || u == "msec") mul = 1e6;
    else if (u == "s" || u == "sec" || u == "secs" || u == "second" || u == "seconds") mul = 1e9;
    else if (u == "m" || u == "min" || u == "mins" || u == "minute" || u == "minutes") mul = 60e9;
    else if (u == "h" || u == "hr" || u == "hour" || u == "hours") mul = 3600e9;
    else if (u == "d" || u == "day" || u == "days") mul = 86400e9;
    else bad();
    total += v * mul;
    any = true;
    i = k;
  }
  if (!any) bad();
  return std::chrono::nanoseconds((long long)total);
}

std::chrono::nanoseconds duration_field(const JsonValue& cfg, const char* key, const char* struct_name) {
  const JsonValue* v = cfg.get(key);
  if (!v) fail(ARK_ERR_SERIALIZATION, std::string("missing field `") + key + "` (" + struct_name + ")");
  if (v->kind != JsonValue::String) fail(ARK_ERR_SERIALIZATION, std::string("invalid type for `") + key + "`: expected a duration string");
  return parse_duration(v->str);
}

struct Queued {
  Batch batch;
  uint64_t ack;
};

struct JoinOp {  // JoinConfig / JoinOperation, join.rs:29-60
  std::unique_ptr<SqlProcessor> sql;
  std::unique_ptr<Processor> decoder;  // json codec = try_to_arrow(content, None), codec/json.rs:39-47
  std::vector<std::string> input_names;
};

std::unique_ptr<JoinOp> make_join(const JsonValue& j, const char* input_names_json) {
  auto op = std::make_unique<JoinOp>();
  const JsonValue* q = j.get("query");
  if (!q || q->kind != JsonValue::String) fail(ARK_ERR_SERIALIZATION, "missing field `query` (JoinConfig)");
  std::string vf = "__value__";
  if (const JsonValue* v = j.get("value_field")) if (v->kind == JsonValue::String) vf = v->str;
  const JsonValue* codec = j.get("codec");
  if (!codec || codec->kind != JsonValue::Object) fail(ARK_ERR_SERIALIZATION, "missing field `codec` (JoinConfig)");
  const JsonValue* ct = codec->get("type");
  if (!ct || ct->kind != JsonValue::String) fail(ARK_ERR_SERIALIZATION, "missing field `type` (CodecConfig)");
  if (ct->str != "json") fail(ARK_ERR_UNSUPPORTED, "join codec '" + ct->str + "' (only the json codec runs on the GPU)");
  std::string sql_cfg = "{\"query\": ";
  sql_cfg += '"';
  for (char ch : q->str) { if (ch == '"' || ch == '\\') sql_cfg += '\\'; if (ch == '\n') { sql_cfg += "\\n"; continue; } sql_cfg += ch; }
  sql_cfg += "\"}";
  op->sql = SqlProcessor::from_config(sql_cfg.c_str());
  std::string dec_cfg = "{\"value_field\": \"" + vf + "\"}";
  op->decoder = make_json_to_arrow(dec_cfg.c_str());
  if (input_names_json) {
    JsonValue names = parse_json(input_names_json);
    if (names.kind == JsonValue::Array) for (auto& n : names.arr) if (n.kind == JsonValue::String) op->input_names.push_back(n.str);
  }
  return op;
}

}  // namespace

struct ark_buf {
  enum Kind { Memory, Session, Tumbling, Sliding } kind;
  std::mutex mu;
  std::condition_variable cv;
  bool closed = false;
  std::thread timer;
  std::chrono::nanoseconds period{0};
  // memory
  uint32_t capacity = 0;
  std::deque<Queued> queue;  // front = newest
  int64_t queued_rows = 0;
  // sliding window: `queue` is FIFO here (push_back / front = oldest), sliding_window.rs:170-174
  uint32_t window_size = 0, slide_size = 0;
  // windows
  std::vector<std::string> input_order;
  std::vector<std::deque<Queued>> input_queues;  // per input, front = newest
  Clock::time_point last_write = Clock::now();
  std::unique_ptr<JoinOp> join;

  bool windows_empty() const {
    for (auto& q : input_queues) if (!q.empty()) return false;
    return true;
  }
  void start_timer() {
    timer = std::thread([this] {
      std::unique_lock<std::mutex> l(mu);
      while (!closed) {
        cv.wait_for(l, period);  // a notify (capacity / close) restarts the period, like the select! in the reference
        cv.notify_all();
      }
    });
  }
  ~ark_buf() {
    { std::lock_guard<std::mutex> l(mu); closed = true; }
    cv.notify_all();
    if (timer.joinable()) timer.join();
  }
};

namespace {

Batch concat_named(std::vector<Batch>& bs, cudaStream_t s) {
  Batch r = concat_device(bs, s);
  return r;
}

// BaseWindow::process_window (window.rs:99-177).  Caller holds no lock; queues were moved out.
Batch process_window(ark_buf* b, std::vector<std::string>& names, std::vector<std::deque<Queued>>& queues, std::vector<uint64_t>& acks,
                     bool* empty_schema, cudaStream_t stream) {
  std::vector<Batch> per_input;
  std::vector<std::string> per_name;
  for (size_t i = 0; i < queues.size(); ++i) {
    if (queues[i].empty()) continue;
    std::vector<Batch> bs;
    while (!queues[i].empty()) {  // pop_front: newest first (window.rs:121)
      bs.push_back(std::move(queues[i].front().batch));
      acks.push_back(queues[i].front().ack);
      queues[i].pop_front();
    }
    Batch merged = concat_named(bs, stream);
    merged.input_name = names[i];
    per_input.push_back(std::move(merged));
    per_name.push_back(names[i]);
  }
  *empty_schema = false;
  if (!b->join) return concat_named(per_input, stream);  // window.rs:148-166
  // ---- JoinOperation::join_operation (join.rs:62-132) ----
  std::vector<std::string> table_names;
  std::vector<std::vector<Field>> schemas;
  std::vector<Batch> tables;
  for (size_t i = 0; i < per_input.size(); ++i) {
    Batch decoded = json_to_arrow_device(*b->join->decoder, per_input[i], stream);  // decode_batch, join.rs:134-146
    if (per_name[i].empty()) continue;  // join.rs:76-79: batches without an input name are skipped
    std::vector<Field> f;
    for (auto& c : decoded.cols) f.push_back(c.field);
    for (auto& x : f) if (x.format.empty()) x.format = dtype_arrow_format(x.type);
    table_names.push_back(per_name[i]);
    schemas.push_back(f);
    tables.push_back(std::move(decoded));
  }
  for (auto& need : b->join->input_names)  // join.rs:102-109
    if (std::find(table_names.begin(), table_names.end(), need) == table_names.end()) { *empty_schema = true; return Batch(); }
  for (auto& t : tables) for (auto& c : t.cols) if (c.field.format.empty()) c.field.format = dtype_arrow_format(c.field.type);
  auto plan = b->join->sql->join_plan_for(table_names, schemas);
  if (plan->kind == Plan::Join) {
    int li = -1, ri = -1;
    for (size_t i = 0; i < table_names.size(); ++i) { if (table_names[i] == plan->left_table) li = (int)i; if (table_names[i] == plan->right_table) ri = (int)i; }
    if (li < 0 || ri < 0) fail(ARK_ERR_PROCESS, "Failed to execute SQL query: table not found");
    return run_join(*plan, tables[li], tables[ri], stream);
  }
  for (size_t i = 0; i < table_names.size(); ++i)
    if (table_names[i] == b->join->sql->ast.from.name) {
      if (tables[i].num_rows == 0) { *empty_schema = true; return Batch(); }
      return b->join->sql->execute(*plan, tables[i], stream);
    }
  fail(ARK_ERR_PROCESS, "Failed to execute SQL query: table '" + b->join->sql->ast.from.name + "' not found");
}

}  // namespace

extern "C" {

int ark_buffer_create(const char* kind, const char* config_json, const char* input_names_json, ark_buf_t** out) {
  return guarded([&] {
    if (!out || !kind) fail(ARK_ERR_PROCESS, "null argument");
    *out = nullptr;
    const std::string k = kind;
    const char* missing = k == "memory" ? "Memory buffer configuration is missing"          // memory.rs:256-258
                          : k == "session_window" ? "Session window configuration is missing"  // session_window.rs:178-180
                          : k == "tumbling_window" ? "Tumbling window configuration is missing"  // tumbling_window.rs:164-166
                          : k == "sliding_window" ? "Sliding window configuration is missing"    // sliding_window.rs:248-252
                          : nullptr;
    if (!missing) fail(ARK_ERR_CONFIG, "Unknown buffer type: " + k);
    if (!config_json) fail(ARK_ERR_CONFIG, missing);
    JsonValue cfg = parse_json(config_json);
    if (cfg.kind == JsonValue::Null) fail(ARK_ERR_CONFIG, missing);
    if (cfg.kind != JsonValue::Object) fail(ARK_ERR_SERIALIZATION, "invalid type: expected a buffer configuration object");
    auto b = std::make_unique<ark_buf>();
    if (k == "memory") {
      b->kind = ark_buf::Memory;
      const JsonValue* cap = cfg.get("capacity");
      if (!cap) fail(ARK_ERR_SERIALIZATION, "missing field `capacity` (MemoryBufferConfig)");
      if (cap->kind != JsonValue::Number || !cap->is_int || cap->i64 < 0 || cap->i64 > 0xFFFFFFFFll)
        fail(ARK_ERR_SERIALIZATION, "invalid value for `capacity`: expected u32");
      b->capacity = (uint32_t)cap->i64;
      b->period = duration_field(cfg, "timeout", "MemoryBufferConfig");
    } else if (k == "sliding_window") {
      b->kind = ark_buf::Sliding;
      auto u32_field = [&](const char* key) -> uint32_t {
        const JsonValue* v = cfg.get(key);
        if (!v) fail(ARK_ERR_SERIALIZATION, std::string("missing field `") + key + "` (SlidingWindowConfig)");
        if (v->kind != JsonValue::Number || !v->is_int || v->i64 < 0 || v->i64 > 0xFFFFFFFFll)
          fail(ARK_ERR_SERIALIZATION, std::string("invalid value for `") + key + "`: expected u32");
        return (uint32_t)v->i64;
      };
      b->window_size = u32_field("window_size");
      b->period = duration_field(cfg, "interval", "SlidingWindowConfig");
      b->slide_size = u32_field("slide_size");
      if (b->window_size == 0) fail(ARK_ERR_CONFIG, "Sliding window window_size must be greater than 0");            // sliding_window.rs:256-260
      if (b->slide_size == 0) fail(ARK_ERR_CONFIG, "Sliding window slide_size must be greater than 0");              // sliding_window.rs:261-265
      if (b->window_size < b->slide_size) fail(ARK_ERR_CONFIG, "Sliding window window_size must be greater than slide_size");  // :266-270
    } else {
      b->kind = k == "session_window" ? ark_buf::Session : ark_buf::Tumbling;
      b->period = duration_field(cfg, k == "session_window" ? "gap" : "interval", k == "session_window" ? "SessionWindowConfig" : "TumblingWindowConfig");
      if (const JsonValue* j = cfg.get("join")) if (j->kind == JsonValue::Object) b->join = make_join(*j, input_names_json);
    }
    if (b->period.count() <= 0) b->period = std::chrono::nanoseconds(1);
    b->start_timer();
    *out = b.release();
  });
}

static void buffer_enqueue(ark_buf* b, Batch&& batch, const char* input_name, uint64_t ack_token) {
  batch.input_name = input_name ? input_name : "";
  std::lock_guard<std::mutex> l(b->mu);
  if (b->kind == ark_buf::Memory) {
    b->queued_rows += batch.num_rows;
    b->queue.push_front({std::move(batch), ack_token});            // memory.rs:155
    if (b->queued_rows >= (int64_t)b->capacity) b->cv.notify_all();  // memory.rs:164-167
  } else if (b->kind == ark_buf::Sliding) {
    b->queue.push_back({std::move(batch), ack_token});               // sliding_window.rs:170-174
    if (b->queue.size() >= b->window_size) b->cv.notify_all();       // (the reference waits for the next timer tick)
  } else {
    size_t idx = 0;
    for (; idx < b->input_order.size(); ++idx) if (b->input_order[idx] == batch.input_name) break;
    if (idx == b->input_order.size()) { b->input_order.push_back(batch.input_name); b->input_queues.emplace_back(); }
    b->input_queues[idx].push_front({std::move(batch), ack_token});  // window.rs:184-187
    if (b->kind == ark_buf::Session) b->last_write = Clock::now();   // session_window.rs:109
  }
}

int ark_buffer_write(ark_buf_t* b, ArrowArray* in, ArrowSchema* in_schema, const char* input_name, uint64_t ack_token) {
  BufferPtr in_owner = adopt_array(in);
  return guarded([&] {
    if (!b) fail(ARK_ERR_PROCESS, "null buffer");
    const ArrowArray* arr = adopted(in_owner);
    StreamLease lease;
    Batch batch = import_host(arr, in_schema, nullptr, lease.s, nullptr, true);  // the window lives in HBM from here on
    ARK_CUDA(cudaStreamSynchronize(lease.s));
    buffer_enqueue(b, std::move(batch), input_name, ack_token);
  });
}

// The same write for a batch that is already in HBM (an input or processor of this library produced it): the
// buffer keeps the caller's device buffers alive, nothing is copied.
int ark_buffer_write_device(ark_buf_t* b, ArrowDeviceArray* in, ArrowSchema* in_schema, const char* input_name, uint64_t ack_token) {
  BufferPtr in_owner = adopt_array(&in->array);
  return guarded([&] {
    if (!b) fail(ARK_ERR_PROCESS, "null buffer");
    ArrowDeviceArray view = device_view(*in, in_owner);
    Batch batch = import_device(&view, in_schema, nullptr, in_owner, true);
    buffer_enqueue(b, std::move(batch), input_name, ack_token);
  });
}

// out_host XOR out_dev: where the window is exported to
static int buffer_read_impl(ark_buf_t* b, ArrowArray* out_host, ArrowDeviceArray* out_dev, ArrowSchema* out_schema, uint64_t* acks, int64_t acks_cap,
                            int64_t* n_acks) {
  return guarded([&] {
    if (out_host) zero_out(out_host, out_schema); else zero_out(out_dev, out_schema);
    if (!b) fail(ARK_ERR_PROCESS, "null buffer");
    if (n_acks) *n_acks = 0;
    std::vector<uint64_t> got_acks;
    StreamLease lease;
    auto export_window = [&](const Batch& r) {
      if (out_host) export_host(r, lease.s, out_host, out_schema);
      else export_device(r, out_dev, out_schema, lease);
    };
    if (b->kind == ark_buf::Memory) {
      std::vector<Batch> bs;
      {
        std::unique_lock<std::mutex> l(b->mu);
        while (b->queue.empty()) {        // memory.rs:179-195
          if (b->closed) return;          // Ok(None)
          b->cv.wait(l);
        }
        while (!b->queue.empty()) {       // pop_back: oldest first (memory.rs:117-120)
          bs.push_back(std::move(b->queue.back().batch));
          got_acks.push_back(b->queue.back().ack);
          b->queue.pop_back();
        }
        b->queued_rows = 0;
      }
      export_window(concat_device(bs, lease.s));
    } else if (b->kind == ark_buf::Sliding) {
      std::vector<Batch> bs;
      {
        std::unique_lock<std::mutex> l(b->mu);
        if (b->closed) return;                                 // sliding_window.rs:183-185
        while (b->queue.size() < b->window_size) {            // sliding_window.rs:187-201
          if (b->closed) return;
          b->cv.wait(l);
        }
        for (uint32_t i = 0; i < b->window_size; ++i) {       // the first window_size batches, oldest first (:112-131)
          bs.push_back(b->queue[i].batch);                     // shared buffers: the batches stay queued for the next window
          got_acks.push_back(b->queue[i].ack);                 // VecAck of every batch in the window (:140)
        }
        for (uint32_t i = 0; i < b->slide_size && !b->queue.empty(); ++i) b->queue.pop_front();  // :144-148
      }
      export_window(concat_device(bs, lease.s));
    } else {
      std::vector<std::string> names;
      std::vector<std::deque<Queued>> queues;
      {
        std::unique_lock<std::mutex> l(b->mu);
        if (b->closed) return;  // session_window.rs:120-122, tumbling_window.rs:110-112
        while (true) {
          if (!b->windows_empty()) {
            if (b->kind == ark_buf::Tumbling) break;                                  // tumbling_window.rs:115-120
            if (Clock::now() - b->last_write >= b->period || b->closed) break;        // session_window.rs:126-133
          } else if (b->closed) return;
          b->cv.wait(l);
        }
        names.swap(b->input_order);
        queues.swap(b->input_queues);
      }
      bool empty_schema = false;
      Batch r = process_window(b, names, queues, got_acks, &empty_schema, lease.s);
      if (empty_schema) r = Batch();  // RecordBatch::new_empty(Schema::empty()), join.rs:108
      export_window(r);
    }
    if ((int64_t)got_acks.size() > acks_cap) fail(ARK_ERR_PROCESS, "ack array too small: need " + std::to_string(got_acks.size()));
    for (size_t i = 0; i < got_acks.size(); ++i) acks[i] = got_acks[i];
    if (n_acks) *n_acks = (int64_t)got_acks.size();
  });
}

int ark_buffer_read(ark_buf_t* b, ArrowArray* out, ArrowSchema* out_schema, uint64_t* acks, int64_t acks_cap, int64_t* n_acks) {
  return buffer_read_impl(b, out, nullptr, out_schema, acks, acks_cap, n_acks);
}
// The window stays in HBM: out->array.release == NULL ⇒ Ok(None).
int ark_buffer_read_device(ark_buf_t* b, ArrowDeviceArray* out, ArrowSchema* out_schema, uint64_t* acks, int64_t acks_cap, int64_t* n_acks) {
  return buffer_read_impl(b, nullptr, out, out_schema, acks, acks_cap, n_acks);
}

int ark_buffer_flush(ark_buf_t* b) {
  return guarded([&] {
    if (!b) fail(ARK_ERR_PROCESS, "null buffer");
    { std::lock_guard<std::mutex> l(b->mu); b->closed = true; }  // memory.rs:204-215, window.rs:203-211
    b->cv.notify_all();
  });
}

int ark_buffer_close(ark_buf_t* b) {
  return guarded([&] {
    if (!b) fail(ARK_ERR_PROCESS, "null buffer");
    { std::lock_guard<std::mutex> l(b->mu); b->closed = true; }
    b->cv.notify_all();
  });
}

void ark_buffer_destroy(ark_buf_t* b) { delete b; }

// ---- `batch` processor (processor/batch.rs) -----------------------------------------------------------
struct ark_batcher {
  std::mutex mu;
  uint64_t count = 0, timeout_ms = 0;
  std::vector<Batch> held;                 // device-resident
  Clock::time_point last_flush = Clock::now();  // batch.rs:49 (creation), :90-92 (each flush)
};

int ark_batch_create(const char* config_json, ark_batcher_t** out) {
  return guarded([&] {
    if (!out) fail(ARK_ERR_PROCESS, "null output handle");
    *out = nullptr;
    if (!config_json) fail(ARK_ERR_CONFIG, "Batch processor configuration is missing");  // batch.rs:135-139
    JsonValue cfg = parse_json(config_json);
    if (cfg.kind == JsonValue::Null) fail(ARK_ERR_CONFIG, "Batch processor configuration is missing");
    if (cfg.kind != JsonValue::Object) fail(ARK_ERR_SERIALIZATION, "invalid type: expected a batch processor configuration object");
    auto u64_field = [&](const char* key) -> uint64_t {
      const JsonValue* v = cfg.get(key);
      if (!v) fail(ARK_ERR_SERIALIZATION, std::string("missing field `") + key + "` (BatchProcessorConfig)");
      if (v->kind != JsonValue::Number || !v->is_int || v->i64 < 0) fail(ARK_ERR_SERIALIZATION, std::string("invalid value for `") + key + "`: expected an unsigned integer");
      return (uint64_t)v->i64;
    };
    auto b = std::make_unique<ark_batcher>();
    b->count = u64_field("count");
    b->timeout_ms = u64_field("timeout_ms");
    *out = b.release();
  });
}

static void batcher_flush_locked(ark_batcher* b, ArrowArray* out, ArrowSchema* out_schema) {
  if (b->held.empty()) return;  // Ok(vec![]) → ProcessResult::None (batch.rs:77-79, 107-108)
  StreamLease lease;
  Batch r = concat_device(b->held, lease.s);
  export_host(r, lease.s, out, out_schema);
  b->held.clear();
  b->last_flush = Clock::now();
}

int ark_batch_process(ark_batcher_t* b, ArrowArray* in, ArrowSchema* in_schema, ArrowArray* out, ArrowSchema* out_schema) {
  BufferPtr in_owner = adopt_array(in);
  return guarded([&] {
    zero_out(out, out_schema);
    if (!b) fail(ARK_ERR_PROCESS, "null batch processor");
    const ArrowArray* arr = adopted(in_owner);
    Batch batch;
    {
      StreamLease lease;
      batch = import_host(arr, in_schema, nullptr, lease.s, nullptr, true);
      ARK_CUDA(cudaStreamSynchronize(lease.s));
    }
    std::lock_guard<std::mutex> l(b->mu);
    b->held.push_back(std::move(batch));  // batch.rs:98-102
    const bool by_count = b->held.size() >= b->count;  // batch.rs:56-58
    const bool by_time = (uint64_t)std::chrono::duration_cast<std::chrono::milliseconds>(Clock::now() - b->last_flush).count() >= b->timeout_ms;  // :60-65
    if (by_count || by_time) batcher_flush_locked(b, out, out_schema);
  });
}

int ark_batch_flush(ark_batcher_t* b, ArrowArray* out, ArrowSchema* out_schema) {
  return guarded([&] {
    zero_out(out, out_schema);
    if (!b) fail(ARK_ERR_PROCESS, "null batch processor");
    std::lock_guard<std::mutex> l(b->mu);
    batcher_flush_locked(b, out, out_schema);
  });
}

int ark_batch_close(ark_batcher_t* b) {  // batch.rs:118-123
  return guarded([&] {
    if (!b) fail(ARK_ERR_PROCESS, "null batch processor");
    std::lock_guard<std::mutex> l(b->mu);
    b->held.clear();
  });
}

void ark_batch_destroy(ark_batcher_t* b) { delete b; }

}  // extern "C"
