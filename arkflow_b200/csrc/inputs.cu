// inputs.cu — the two inputs that feed the hot path with batches produced ON the device:
//
//   generate  ← crates/arkflow-plugin/src/input/generate.rs:26-96.  `batch_size` clones of the `context` payload per
//               read() as a non-null Binary column `__value__` (core/lib.rs:243-270), paced by `interval` (the first
//               read is immediate), Error::EOF once `count` messages were produced or the next batch would exceed it.
//               The reference allocates a Vec<u8> per message and copies it into the BinaryArray; Arrow buffers are
//               immutable, so here the replicated payload column is built ONCE in HBM (replicate kernel) and every
//               read() hands out another reference to it — BASELINE configs[4]'s "100 M msg/s generate input" costs
//               no memory traffic at all until a processor reads the messages.
//   file      ← crates/arkflow-plugin/src/input/file.rs:395-455 (`input_type: {type: json | csv | avro | arrow, path}`,
//               optional `query`): one driver for every format (file_input.h) uploads the file's bytes to HBM once,
//               cuts reads into `batch_size` rows and runs the optional query through the sql processor.  Line starts
//               are found by a newline-index kernel (LineIndex); NDJSON lines are decoded by the json_to_arrow kernels
//               (csrc/json.cu), CSV rows by csrc/csv.cu, Avro object container files (codecs null and snappy) by
//               csrc/avro.cu, whose block table is built on the host while the upload's chunks pass, Arrow IPC files
//               (uncompressed and LZ4_FRAME bodies) by csrc/arrow_ipc.cu, whose metadata is read before the upload and
//               whose batches are views of the uploaded file where they can be.  Parquet, ZSTD
//               IPC bodies, the Avro codecs deflate / zstandard / bzip2 / xz and remote object stores are not read here
//               (ARK_ERR_UNSUPPORTED).
//               The NDJSON schema is merged over the first 1000 records and fixed for the file, as DataFusion does.
//               NDJSON and CSV lines: `\n` and `\r\n` both end a line, and the last line needs no terminator.  An empty line
//               (nothing but `\r` before its `\n`) is not a record in either format, as in csv-core and arrow-json: it is
//               left out of the line index, so it never counts toward `batch_size`.  Every batch but the last therefore
//               holds exactly `batch_size` rows; an NDJSON line of spaces only is a line that the decoder drops, so such a
//               batch comes out shorter.  CSV's types and errors are described in csv.cu.
//               A missing or unopenable file is reported by connect() before the device is touched.
#include <fcntl.h>
#include <sys/stat.h>
#include <unistd.h>

#include <chrono>
#include <cstdio>
#include <exception>
#include <thread>

#include <thrust/iterator/counting_iterator.h>

#include <cub/device/device_select.cuh>

#include <thrust/count.h>
#include <thrust/execution_policy.h>

#include "abi.h"
#include "file_input.h"
#include "json_mini.h"

using namespace ark;

namespace {

using Clock = std::chrono::steady_clock;

// humantime subset shared with buffers.cu's configs ("1ns", "10ms", "1s", "2m" …)
std::chrono::nanoseconds parse_duration_in(const std::string& s) {
  size_t i = 0;
  long double total = 0;
  bool any = false;
  auto bad = [&]() { fail(ARK_ERR_SERIALIZATION, "invalid value: string \"" + s + "\", expected a duration like '10ms' or '1s'"); };
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
    long double mul = 0;
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

// out[i*len .. (i+1)*len) = payload, offsets[i] = i*len; 16 bytes per thread.  The payload is read through the
// read-only cache: it has any length a Binary array admits, so it is not staged in shared memory.
__global__ void replicate_kernel(const uint8_t* __restrict__ payload, int len, long long n, uint8_t* out, int32_t* offsets) {
  const long long total = n * len;
  for (long long p = ((long long)blockIdx.x * blockDim.x + threadIdx.x) * 16; p < total; p += (long long)gridDim.x * blockDim.x * 16) {
    uint8_t v[16];
    int k = (int)(p % len);
#pragma unroll
    for (int b = 0; b < 16; ++b) { v[b] = __ldg(payload + k); if (++k == len) k = 0; }
    if (p + 16 <= total) *reinterpret_cast<uint4*>(out + p) = *reinterpret_cast<const uint4*>(v);
    else for (int b = 0; p + b < total; ++b) out[p + b] = v[b];
  }
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i <= n; i += (long long)gridDim.x * blockDim.x) offsets[i] = (int32_t)(i * len);
}

// ---- line index --------------------------------------------------------------------------------------------------
// flags[i] = 1 when byte i starts a line (i == 0 or byte i-1 is '\n') that is not empty: it has a byte other than
// '\r' before its '\n' or the end of the file
__global__ void line_start_flags_kernel(const uint8_t* data, long long n, uint8_t* flags) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    uint8_t f = 0;
    if (i == 0 || data[i - 1] == '\n') {
      long long j = i;
      while (j < n && data[j] == '\r') ++j;
      f = j < n && data[j] != '\n';
    }
    flags[i] = f;
  }
}

__global__ void rebase_offsets_kernel(const long long* starts, long long first, long long n, int32_t* out) {
  const long long base = starts[first];
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i <= n; i += (long long)gridDim.x * blockDim.x) out[i] = (int32_t)(starts[first + i] - base);
}

}  // namespace

// ---- host file -----------------------------------------------------------------------------------------------------
HostFile::HostFile(const std::string& p) : path(p) {
  struct stat st;
  if (stat(path.c_str(), &st) != 0) fail(ARK_ERR_PROCESS, "Read input failed: Object at location " + path + " not found");
  size = (int64_t)st.st_size;
  fd = ::open(path.c_str(), O_RDONLY);
  if (fd < 0) fail(ARK_ERR_PROCESS, "Read input failed: cannot open " + path);
}

HostFile::~HostFile() { if (fd >= 0) close(fd); }

size_t HostFile::read_some(int64_t off, void* dst, size_t n) const {
  size_t done = 0;
  while (done < n) {
    const ssize_t got = pread(fd, (char*)dst + done, n - done, (off_t)(off + (int64_t)done));
    if (got <= 0) break;
    done += (size_t)got;
  }
  return done;
}

std::string HostFile::read(int64_t off, int64_t n) const {
  std::string s((size_t)n, '\0');
  if (read_some(off, &s[0], (size_t)n) != (size_t)n) fail(ARK_ERR_PROCESS, "Read input failed: short read");
  return s;
}

// ---- line index ----------------------------------------------------------------------------------------------------
void LineIndex::build(const BufferPtr& file_dev, int64_t file_bytes, cudaStream_t stream) {
  file = file_dev;
  bytes = file_bytes;
  lines = 0;
  starts = nullptr;
  const int64_t n = bytes;
  if (n == 0) return;
  BufferPtr flags = device_alloc((size_t)n);
  {
    KernelTimer t("line_start_flags_kernel", stream);
    line_start_flags_kernel<<<grid_of(n), 256, 0, stream>>>((const uint8_t*)file.get(), n, (uint8_t*)flags.get());
  }
  BufferPtr cnt = device_alloc(16);
  size_t tb = 0;
  thrust::counting_iterator<long long> ids(0);
  // a file of single-byte lines would need n entries: size for that worst case
  starts = device_alloc((size_t)(n + 1) * 8);
  cub::DeviceSelect::Flagged(nullptr, tb, ids, (const uint8_t*)flags.get(), (long long*)starts.get(), (long long*)cnt.get(), n, stream);
  BufferPtr tmp = device_alloc(tb + 16);
  note_launch("cub::DeviceSelect::Flagged");
  cub::DeviceSelect::Flagged(tmp.get(), tb, ids, (const uint8_t*)flags.get(), (long long*)starts.get(), (long long*)cnt.get(), n, stream);
  BufferPtr h = pinned_alloc(16);
  ARK_CUDA(cudaMemcpyAsync(h.get(), cnt.get(), 8, cudaMemcpyDeviceToHost, stream));
  ARK_CUDA(cudaStreamSynchronize(stream));
  lines = *(long long*)h.get();
  ARK_CUDA(cudaMemcpyAsync((long long*)starts.get() + lines, &bytes, 8, cudaMemcpyHostToDevice, stream));  // sentinel: file end
  ARK_CUDA(cudaStreamSynchronize(stream));
}

std::pair<int64_t, int64_t> LineIndex::span(int64_t l0, int64_t n, cudaStream_t stream) const {
  BufferPtr h = pinned_alloc(32);
  ARK_CUDA(cudaMemcpyAsync(h.get(), (const long long*)starts.get() + l0, 8, cudaMemcpyDeviceToHost, stream));
  ARK_CUDA(cudaMemcpyAsync((char*)h.get() + 8, (const long long*)starts.get() + l0 + n, 8, cudaMemcpyDeviceToHost, stream));
  ARK_CUDA(cudaStreamSynchronize(stream));
  const int64_t byte0 = ((long long*)h.get())[0], byte1 = ((long long*)h.get())[1];
  if (byte1 - byte0 > 2147483647ll) fail(ARK_ERR_PROCESS, "file input: a batch of lines exceeds 2 GiB; lower batch_size");
  return {byte0, byte1};
}

BufferPtr LineIndex::rebased(int64_t l0, int64_t n, cudaStream_t stream) const {
  BufferPtr off = device_alloc((size_t)(n + 1) * 4);
  KernelTimer t("rebase_offsets_kernel", stream);
  rebase_offsets_kernel<<<grid_of(n + 1), 256, 0, stream>>>((const long long*)starts.get(), l0, n, (int32_t*)off.get());
  return off;
}

std::vector<std::string> LineIndex::sample(int64_t k, cudaStream_t stream, int64_t* first) const {
  std::vector<long long> at((size_t)k + 1);
  ARK_CUDA(cudaMemcpyAsync(at.data(), starts.get(), (size_t)(k + 1) * 8, cudaMemcpyDeviceToHost, stream));
  ARK_CUDA(cudaStreamSynchronize(stream));
  std::string text((size_t)(at[(size_t)k] - at[0]), '\0');
  ARK_CUDA(cudaMemcpyAsync(&text[0], (const uint8_t*)file.get() + at[0], text.size(), cudaMemcpyDeviceToHost, stream));
  ARK_CUDA(cudaStreamSynchronize(stream));
  std::vector<std::string> out;
  for (int64_t i = 0; i < k; ++i) out.push_back(text.substr((size_t)(at[(size_t)i] - at[0]), (size_t)(at[(size_t)i + 1] - at[(size_t)i])));
  if (first) *first = at[0];
  return out;
}

long long LineIndex::physical_line(long long off, cudaStream_t stream) const {
  const uint8_t* f = (const uint8_t*)file.get();
  note_launch("thrust::count");
  return 1 + (long long)thrust::count(thrust::cuda::par.on(stream), f, f + off, (uint8_t)'\n');
}

namespace {

// ---- NDJSON ----------------------------------------------------------------------------------------------------------
// Every line is one record for the json decoder, whose schema is merged over the file's first ≤ 1000 records
// (DataFusion's schema_infer_max_records) and fixed for every batch.
struct JsonFormat : FileFormat {
  LineIndex lines;
  std::unique_ptr<Processor> decoder;

  int64_t prepare(const BufferPtr& file_dev, int64_t bytes, cudaStream_t stream) override {
    lines.build(file_dev, bytes, stream);
    if (lines.lines > 0) decoder = make_json_to_arrow_for_sample(lines.sample(std::min<int64_t>(lines.lines, 1000), stream));
    return lines.lines;
  }

  // lines [l0, l0 + n) as a Binary column whose rows are the lines (each still ends with its '\n'), then the decoder
  Batch batch(int64_t l0, int64_t n, cudaStream_t stream) override {
    const auto [byte0, byte1] = lines.span(l0, n, stream);
    BufferPtr off = lines.rebased(l0, n, stream);
    Batch b;
    b.num_rows = n;
    Column c;
    c.field.name = "__value__"; c.field.type = DType::Binary; c.field.format = "z"; c.field.nullable = false;
    c.length = n; c.null_count = 0;
    c.offsets = (const int32_t*)off.get(); c.data = (const uint8_t*)lines.file.get() + byte0; c.data_bytes = byte1 - byte0; c.first_offset = 0;
    c.owners = {off, lines.file};
    b.cols.push_back(std::move(c));
    return json_to_arrow_device(*decoder, b, stream);
  }
};

std::unique_ptr<FileFormat> make_file_format(const std::string& type, bool has_header) {
  if (type == "json") return std::make_unique<JsonFormat>();
  if (type == "csv") return make_csv_format(has_header);
  if (type == "avro") return make_avro_format();
  if (type == "arrow") return make_arrow_ipc_format();
  if (type == "parquet") fail(ARK_ERR_UNSUPPORTED, "file input: " + type + " files are not decoded on the GPU (json, csv, avro and arrow are)");
  fail(ARK_ERR_SERIALIZATION, "unknown variant `" + type + "`, expected one of `avro`, `arrow`, `json`, `csv`, `parquet`");
}

// ---- the file driver -------------------------------------------------------------------------------------------------
struct FileDriver {
  std::string path;
  std::unique_ptr<FileFormat> format;
  std::unique_ptr<SqlProcessor> sql;
  int64_t rows = 0, next_row = 0, rows_per_batch = 1 << 22;
  bool connected = false, closed = false;

  void connect() {
    HostFile file(path);
    format->open(file);
    StreamLease lease;
    const cudaStream_t stream = lease.s;
    const int64_t n = file.size;
    BufferPtr file_dev = device_alloc((size_t)std::max<int64_t>(n, 1) + 64);
    // file → pinned chunks → HBM (two chunks in flight); the format sees every chunk in file order
    const size_t CH = 8u << 20;
    BufferPtr stage = pinned_alloc(2 * CH);
    cudaEvent_t ev[2];
    for (auto& e : ev) ARK_CUDA(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
    bool used[2] = {false, false};
    int64_t done = 0;
    int turn = 0;
    bool io_error = false;
    std::exception_ptr scan_error;
    while (done < n) {
      uint8_t* slot = (uint8_t*)stage.get() + (size_t)turn * CH;
      if (used[turn]) ARK_CUDA(cudaEventSynchronize(ev[turn]));
      const size_t got = file.read_some(done, slot, (size_t)std::min<int64_t>((int64_t)CH, n - done));
      if (got == 0) { io_error = true; break; }
      try { format->scan(slot, got, done); } catch (...) { scan_error = std::current_exception(); break; }
      ARK_CUDA(cudaMemcpyAsync((uint8_t*)file_dev.get() + done, slot, got, cudaMemcpyHostToDevice, stream));
      ARK_CUDA(cudaEventRecord(ev[turn], stream));
      used[turn] = true;
      done += (int64_t)got;
      turn ^= 1;
    }
    ARK_CUDA(cudaStreamSynchronize(stream));
    for (auto& e : ev) cudaEventDestroy(e);
    if (io_error) fail(ARK_ERR_PROCESS, "Read input failed: short read on " + path);
    if (scan_error) std::rethrow_exception(scan_error);
    rows = format->prepare(file_dev, n, stream);
    next_row = 0;
    connected = true;
  }

  // The query's planner sees the fixed-width columns other than Int64 and Float64 (Int32, UInt32, UInt64, Float32) as
  // the sql processor's import presents them, so a query that reads one is Unsupported as it is there.
  Batch query(Batch& b, cudaStream_t stream) {
    std::vector<Field> fields;
    for (auto& c : b.cols) {
      if (c.field.format.empty()) c.field.format = dtype_arrow_format(c.field.type);
      Field f = c.field;
      if (fixed_width(f.type) && f.type != DType::Int64 && f.type != DType::Float64) f.type = DType::Null;
      fields.push_back(f);
    }
    auto plan = sql->plan_for(fields);
    return sql->execute(*plan, b, stream);
  }

  // returns false at EOF
  bool next(Batch& out, cudaStream_t stream) {
    if (!connected) fail(ARK_ERR_PROCESS, "Stream is None");  // file.rs:433-435
    while (true) {
      if (closed || next_row >= rows) return false;
      const int64_t r0 = next_row;
      const int64_t n = std::min<int64_t>(rows_per_batch, rows - r0);
      next_row += n;
      Batch b = format->batch(r0, n, stream);
      if (b.num_rows == 0) continue;  // NDJSON lines that hold only spaces
      if (sql) {
        b = query(b, stream);
        if (b.num_rows == 0 && b.cols.empty()) continue;
      }
      ARK_CUDA(cudaStreamSynchronize(stream));
      out = std::move(b);
      return true;
    }
  }
};

}  // namespace

struct ark_input {
  std::mutex mu;
  std::unique_ptr<FileDriver> file;  // the `file` input; nullptr: `generate`
  // generate
  std::string context;
  std::chrono::nanoseconds interval{0};
  bool has_count = false;
  int64_t count_limit = 0, produced = 0, batch_size = 1;
  bool first = true;
  Batch cached;  // the replicated payload column (immutable)
};

namespace {

Batch generate_batch(ark_input* in, cudaStream_t stream) {
  const int64_t n = in->batch_size;
  const int len = (int)in->context.size();
  if ((int64_t)len * n > 2147483647ll) fail(ARK_ERR_PROCESS, "generate: batch_size x context exceeds a Binary array's 2 GiB");
  Batch b;
  b.num_rows = n;
  BufferPtr off = device_alloc((size_t)(n + 1) * 4), data = device_alloc((size_t)std::max<int64_t>((int64_t)len * n, 1) + 16);
  BufferPtr pay = device_alloc((size_t)std::max(len, 1));
  if (len) ARK_CUDA(cudaMemcpyAsync(pay.get(), in->context.data(), (size_t)len, cudaMemcpyHostToDevice, stream));
  {
    KernelTimer t("replicate_kernel", stream);
    replicate_kernel<<<grid_of(std::max<long long>((long long)len * n / 16, n + 1)), 256, 0, stream>>>(
        (const uint8_t*)pay.get(), std::max(len, 0), n, (uint8_t*)data.get(), (int32_t*)off.get());
  }
  ARK_CUDA(cudaGetLastError());
  ARK_CUDA(cudaStreamSynchronize(stream));
  Column c;
  c.field.name = "__value__"; c.field.type = DType::Binary; c.field.format = "z"; c.field.nullable = false;  // core/lib.rs:255-262
  c.length = n; c.null_count = 0;
  c.offsets = (const int32_t*)off.get(); c.data = (const uint8_t*)data.get(); c.data_bytes = (int64_t)len * n; c.first_offset = 0;
  c.owners = {off, data};
  b.cols.push_back(std::move(c));
  return b;
}

// returns false at EOF
bool generate_next(ark_input* in, Batch& out, cudaStream_t stream) {
  bool sleep_first;
  {
    std::lock_guard<std::mutex> l(in->mu);
    sleep_first = !in->first;
    in->first = false;
  }
  if (sleep_first && in->interval.count() > 0) std::this_thread::sleep_for(in->interval);  // generate.rs:67-69
  std::lock_guard<std::mutex> l(in->mu);
  if (in->has_count) {                                                                      // generate.rs:71-80
    if (in->produced >= in->count_limit) return false;
    if (in->produced + in->batch_size > in->count_limit) return false;
  }
  if (in->cached.cols.empty()) in->cached = generate_batch(in, stream);
  in->produced += in->batch_size;
  out = in->cached;  // another reference to the same immutable buffers
  return true;
}

bool input_next(ark_input* in, Batch& out, cudaStream_t stream) {
  if (!in->file) return generate_next(in, out, stream);
  std::lock_guard<std::mutex> l(in->mu);
  return in->file->next(out, stream);
}

}  // namespace

extern "C" {

int ark_input_create(const char* type, const char* config_json, ark_input_t** out) {
  return guarded([&] {
    if (!out || !type) fail(ARK_ERR_PROCESS, "null argument");
    *out = nullptr;
    const std::string k = type;
    if (k != "generate" && k != "file") fail(ARK_ERR_CONFIG, "Unknown input type: " + k + " (this library builds `generate` and `file`)");
    if (!config_json) fail(ARK_ERR_CONFIG, k == "generate" ? "Generate input configuration is missing" : "File input configuration is missing");
    JsonValue cfg = parse_json(config_json);
    if (cfg.kind == JsonValue::Null) fail(ARK_ERR_CONFIG, k == "generate" ? "Generate input configuration is missing" : "File input configuration is missing");
    if (cfg.kind != JsonValue::Object) fail(ARK_ERR_SERIALIZATION, "invalid type: expected an input configuration object");
    auto in = std::make_unique<ark_input>();
    auto opt_u = [&](const char* key, int64_t* dst) -> bool {
      const JsonValue* v = cfg.get(key);
      if (!v || v->kind == JsonValue::Null) return false;
      if (v->kind != JsonValue::Number || !v->is_int || v->i64 < 0) fail(ARK_ERR_SERIALIZATION, std::string("invalid value for `") + key + "`: expected usize");
      *dst = v->i64;
      return true;
    };
    if (k == "generate") {
      const JsonValue* c = cfg.get("context");
      if (!c) fail(ARK_ERR_SERIALIZATION, "missing field `context`");
      if (c->kind != JsonValue::String) fail(ARK_ERR_SERIALIZATION, "invalid type for `context`: expected a string");
      in->context = c->str;
      const JsonValue* iv = cfg.get("interval");
      if (!iv) fail(ARK_ERR_SERIALIZATION, "missing field `interval`");
      if (iv->kind != JsonValue::String) fail(ARK_ERR_SERIALIZATION, "invalid type for `interval`: expected a duration string");
      in->interval = parse_duration_in(iv->str);
      in->has_count = opt_u("count", &in->count_limit);
      if (!opt_u("batch_size", &in->batch_size)) in->batch_size = 1;  // generate.rs:49
    } else {
      in->file = std::make_unique<FileDriver>();
      FileDriver& fd = *in->file;
      const JsonValue* it = cfg.get("input_type");
      if (!it || it->kind != JsonValue::Object) fail(ARK_ERR_SERIALIZATION, "missing field `input_type`");
      const JsonValue* ty = it->get("type");
      if (!ty || ty->kind != JsonValue::String) fail(ARK_ERR_SERIALIZATION, "missing field `type` (InputType)");
      bool has_header = true;
      if (const JsonValue* hh = it->get("has_header")) if (hh->kind == JsonValue::Bool) has_header = hh->b;
      fd.format = make_file_format(ty->str, has_header);
      const JsonValue* p = it->get("path");
      if (!p || p->kind != JsonValue::String) fail(ARK_ERR_SERIALIZATION, "missing field `path`");
      if (const JsonValue* st = it->get("store")) if (st->kind != JsonValue::Null) fail(ARK_ERR_UNSUPPORTED, "file input: remote object stores (network I/O) stay in the reference's input");
      if (const JsonValue* bl = cfg.get("ballista")) if (bl->kind != JsonValue::Null) fail(ARK_ERR_UNSUPPORTED, "file input: ballista");
      fd.path = p->str;
      if (fd.path.rfind("file://", 0) == 0) fd.path = fd.path.substr(7);
      opt_u("batch_size", &fd.rows_per_batch);  // extension: rows per RecordBatch (DataFusion's execution.batch_size)
      if (fd.rows_per_batch <= 0) fd.rows_per_batch = 1 << 22;
      if (const JsonValue* q = cfg.get("query")) {
        if (q->kind == JsonValue::Object) {
          const JsonValue* qs = q->get("query");
          if (!qs || qs->kind != JsonValue::String) fail(ARK_ERR_SERIALIZATION, "missing field `query` (QueryConfig)");
          std::string table = "flow";  // default_table(), file.rs
          if (const JsonValue* t = q->get("table")) if (t->kind == JsonValue::String) table = t->str;
          std::string sc = "{\"query\": \"";
          for (char ch : qs->str) { if (ch == '"' || ch == '\\') sc += '\\'; if (ch == '\n') { sc += "\\n"; continue; } sc += ch; }
          sc += "\", \"table_name\": \"" + table + "\"}";
          fd.sql = SqlProcessor::from_config(sc.c_str());
        } else if (q->kind != JsonValue::Null) fail(ARK_ERR_SERIALIZATION, "invalid type for `query`: expected QueryConfig");
      }
    }
    *out = in.release();
  });
}

int ark_input_connect(ark_input_t* in) {
  return guarded([&] {
    if (!in) fail(ARK_ERR_PROCESS, "null input");
    if (!in->file) return;  // generate.rs:62-64
    std::lock_guard<std::mutex> l(in->mu);
    if (!in->file->connected) in->file->connect();
  });
}

int ark_input_read_device(ark_input_t* in, ArrowDeviceArray* out, ArrowSchema* out_schema) {
  return guarded([&] {
    zero_out(out, out_schema);
    if (!in || !out) fail(ARK_ERR_PROCESS, "null argument");
    StreamLease lease;
    Batch b;
    if (!input_next(in, b, lease.s)) fail(ARK_ERR_EOF, "EOF");
    export_device(b, out, out_schema, lease);
  });
}

int ark_input_read(ark_input_t* in, ArrowArray* out, ArrowSchema* out_schema) {
  return guarded([&] {
    zero_out(out, out_schema);
    if (!in || !out) fail(ARK_ERR_PROCESS, "null argument");
    StreamLease lease;
    Batch b;
    if (!input_next(in, b, lease.s)) fail(ARK_ERR_EOF, "EOF");
    export_host(b, lease.s, out, out_schema);
  });
}

int ark_input_close(ark_input_t* in) {
  return guarded([&] {
    if (!in) fail(ARK_ERR_PROCESS, "null input");
    std::lock_guard<std::mutex> l(in->mu);
    if (in->file) in->file->closed = true;  // file.rs:458-461 cancels the stream; generate.rs:93-95 is a no-op
  });
}

void ark_input_destroy(ark_input_t* in) { delete in; }

}  // extern "C"
