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
//               optional `query`): the file's bytes go to HBM once; line starts are found by a newline-index kernel,
//               NDJSON lines are decoded by the json_to_arrow kernels (csrc/json.cu), CSV rows by csv_parse_kernel,
//               Avro object container files (codecs null and snappy) by the kernels of csrc/avro.cu, whose block table
//               is built on the host while the upload's chunks pass, Arrow IPC files (uncompressed and LZ4_FRAME
//               bodies) by csrc/arrow_ipc.cu, whose metadata is read before the upload and whose batches are views of
//               the uploaded file where they can be; the optional query runs through the sql processor.  Parquet, ZSTD
//               IPC bodies, the Avro codecs deflate / zstandard / bzip2 / xz and remote object stores are not read here
//               (ARK_ERR_UNSUPPORTED).
//               The NDJSON schema is merged over the first 1000 records and fixed for the file, as DataFusion does.
//               Deviations from DataFusion's readers: CSV types come from the first 1000 records with the
//               types Int64 / Float64 / Boolean / Utf8 (dates stay strings), quoted CSV fields may not contain line
//               breaks (oracle/csv_oracle.py lists the smaller ones).  A CSV column is Int64 when its sample values are decimal integers within the i64 range, and
//               Float64 when they are decimals or nan / inf / infinity (any case, optional sign; Arrow's reader
//               accepts these spellings too); Float64 values are correctly rounded.
//               Lines: `\n` and `\r\n` both end a line, and the last line needs no terminator.  An empty line (nothing
//               but `\r` before its `\n`) is not a record in either format, as in csv-core and arrow-json: it is left
//               out of the line index, so it never counts toward `batch_size` and the CSV header is the first line
//               that is not empty.  Every batch but the last therefore holds exactly `batch_size` lines; an NDJSON line
//               of spaces only is a line that the decoder drops, so such a batch comes out shorter.
//               CSV errors: a batch reports the error of its FIRST failing line in file order, and the line number in
//               the message counts physical lines from 1, empty ones included.  Within one line the order is: wrong
//               number of fields (bytes after a closing quote count as such), then a value that does not parse as its
//               column's type (invalid UTF-8 in a numeric or Boolean field is this error), then invalid UTF-8 in a
//               Utf8 field.  tests/test_inputs_edges_gpu.py checks all of this against oracle/csv_oracle.py.
#include <sys/stat.h>

#include <chrono>
#include <cstdio>
#include <exception>
#include <functional>
#include <thread>

#include <thrust/iterator/counting_iterator.h>

#include <cub/device/device_select.cuh>

#include <thrust/count.h>
#include <thrust/execution_policy.h>

#include "bitmap.h"
#include "decimal.cuh"
#include "abi.h"
#include "json_mini.h"
#include "utf8.cuh"
#include "varlen.h"

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

// ---- CSV ---------------------------------------------------------------------------------------------------------
enum CsvType : int32_t { CSV_I64 = 0, CSV_F64 = 1, CSV_BOOL = 2, CSV_STR = 3 };
constexpr int CSV_MAX_COLS = 32;

struct CsvParams {
  const uint8_t* data;
  const int32_t* line_off;  // [n_rows + 1] starts of the data rows (+ end)
  long long n_rows;
  int32_t n_cols;
  int32_t delim;
  int32_t types[CSV_MAX_COLS];
  void* values[CSV_MAX_COLS];        // Int64 / Float64: 8 B per row; Boolean: byte per row
  uint8_t* valid[CSV_MAX_COLS];      // byte per row
  int32_t* str_len[CSV_MAX_COLS];    // Utf8: decoded length per row (n_rows + 1 entries; scanned into offsets)
  long long* str_src[CSV_MAX_COLS];  // Utf8: absolute position of the field body
  int32_t* str_raw[CSV_MAX_COLS];    // Utf8: raw length; negative ⇒ quoted field with "" escapes
  unsigned long long* error;         // min over the failing rows of row << 2 | code (all ones: none); code 1 = bad value,
                                     // 2 = wrong field count, 3 = invalid UTF-8 in a Utf8 field
};

// The host's type inference (csv_infer_type) calls the same two grammar tests as the kernel, so a column inferred
// Int64 / Float64 from its sample rows parses on the device.
__host__ __device__ inline bool csv_parse_i64(const uint8_t* p, int len, long long* out) {
  if (len <= 0) return false;
  int i = 0;
  bool neg = false;
  if (p[0] == '-' || p[0] == '+') { neg = p[0] == '-'; i = 1; }
  if (i >= len) return false;
  unsigned long long v = 0;
  for (; i < len; ++i) {
    const unsigned d = (unsigned)p[i] - '0';
    if (d > 9) return false;
    if (v > (0xFFFFFFFFFFFFFFFFull - d) / 10) return false;
    v = v * 10 + d;
  }
  if (neg) { if (v > 0x8000000000000000ull) return false; *out = (long long)(0 - v); }
  else { if (v > 0x7FFFFFFFFFFFFFFFull) return false; *out = (long long)v; }
  return true;
}

// [+-]? then nan / inf / infinity in any case, as Arrow's CSV reader spells them → the f64 bits.  NaN keeps no sign.
__host__ __device__ inline bool csv_special_f64(const uint8_t* p, int len, unsigned long long* bits) {
  int i = (len > 0 && (p[0] == '-' || p[0] == '+')) ? 1 : 0;
  const bool neg = i == 1 && p[0] == '-';
  auto word = [&](const char* w, int n) {
    if (len - i != n) return false;
    for (int k = 0; k < n; ++k) if ((p[i + k] | 32) != w[k]) return false;
    return true;
  };
  if (word("nan", 3)) { *bits = 0x7FF8000000000000ull; return true; }
  if (word("inf", 3) || word("infinity", 8)) { *bits = neg ? 0xFFF0000000000000ull : 0x7FF0000000000000ull; return true; }
  return false;
}

// decimal → double, correctly rounded (decimal.cuh, the routine the JSON decoder uses), or one of the special spellings
__device__ inline bool csv_parse_f64(const uint8_t* p, int len, double* out) {
  unsigned long long bits;
  if (csv_special_f64(p, len, &bits)) { *out = __longlong_as_double((long long)bits); return true; }
  return decimal_to_f64(p, len, out);
}

// One thread per row: split at the delimiter (quoted fields may hold delimiters and "" escapes), convert per type.
// A failing row folds row << 2 | code into P.error with one atomicMin, so the batch reports its first failing row.
__global__ void csv_parse_kernel(const __grid_constant__ CsvParams P) {
  for (long long row = (long long)blockIdx.x * blockDim.x + threadIdx.x; row < P.n_rows; row += (long long)gridDim.x * blockDim.x) {
    long long pos = P.line_off[row], end = P.line_off[row + 1];
    while (end > pos && (P.data[end - 1] == '\n' || P.data[end - 1] == '\r')) --end;
    int col = 0;
    bool bad = false, bad_utf8 = false, few = false;
    while (col < P.n_cols) {
      long long f0 = pos, f1;
      bool escaped = false;
      if (pos < end && P.data[pos] == '"') {
        f0 = ++pos;
        while (pos < end) {
          if (P.data[pos] == '"') { if (pos + 1 < end && P.data[pos + 1] == '"') { escaped = true; pos += 2; continue; } break; }
          ++pos;
        }
        f1 = pos;
        if (pos < end) ++pos;  // closing quote
      } else {
        while (pos < end && P.data[pos] != (uint8_t)P.delim) ++pos;
        f1 = pos;
      }
      const int len = (int)(f1 - f0);
      const uint8_t* fp = P.data + f0;
      const bool is_null = len == 0;  // arrow-csv: the empty string is NULL for every type (quoted or not)
      P.valid[col][row] = !is_null;
      switch (P.types[col]) {
        case CSV_I64: { long long v = 0; if (!is_null && !csv_parse_i64(fp, len, &v)) bad = true; ((long long*)P.values[col])[row] = v; break; }
        case CSV_F64: { double v = 0; if (!is_null && !csv_parse_f64(fp, len, &v)) bad = true; ((double*)P.values[col])[row] = v; break; }
        case CSV_BOOL: {
          uint8_t v = 0;
          if (!is_null) {
            if (len == 4 && (fp[0] | 32) == 't' && (fp[1] | 32) == 'r' && (fp[2] | 32) == 'u' && (fp[3] | 32) == 'e') v = 1;
            else if (len == 5 && (fp[0] | 32) == 'f' && (fp[1] | 32) == 'a' && (fp[2] | 32) == 'l' && (fp[3] | 32) == 's' && (fp[4] | 32) == 'e') v = 0;
            else bad = true;
          }
          ((uint8_t*)P.values[col])[row] = v;
          break;
        }
        default: {
          int dec = len;
          if (escaped) { dec = 0; for (int i = 0; i < len; ++i) { ++dec; if (fp[i] == '"') ++i; } }
          P.str_len[col][row] = dec;
          P.str_src[col][row] = f0;
          P.str_raw[col][row] = escaped ? -len : len;
          // arrow-csv: an empty unquoted field of a Utf8 column is NULL too (nulls are decided before the type)
          if (!utf8_valid(fp, len)) bad_utf8 = true;  // a Utf8 array holds valid UTF-8 ("" escapes are ASCII)
          break;
        }
      }
      if (++col == P.n_cols) break;  // what is left of the line, a trailing delimiter too, is one field too many
      if (pos < end && P.data[pos] == (uint8_t)P.delim) ++pos;
      else { few = true; for (; col < P.n_cols; ++col) { P.valid[col][row] = 0; if (P.types[col] == CSV_STR) { P.str_len[col][row] = 0; P.str_src[col][row] = 0; P.str_raw[col][row] = 0; } } }
    }
    const int code = (few || pos < end) ? 2 : bad ? 1 : bad_utf8 ? 3 : 0;
    if (code) atomicMin(P.error, ((unsigned long long)row << 2) | (unsigned long long)code);
  }
}

__global__ void csv_strings_kernel(const uint8_t* data, long long n, const int32_t* out_off, const long long* src, const int32_t* raw, uint8_t* out) {
  for (long long row = (long long)blockIdx.x * blockDim.x + threadIdx.x; row < n; row += (long long)gridDim.x * blockDim.x) {
    const uint8_t* s = data + src[row];
    uint8_t* d = out + out_off[row];
    int r = raw[row];
    if (r >= 0) { for (int i = 0; i < r; ++i) d[i] = s[i]; }
    else { r = -r; for (int i = 0; i < r; ++i) { *d++ = s[i]; if (s[i] == '"') ++i; } }
  }
}

unsigned grid_of(long long n, int threads = 256) { return (unsigned)std::max<long long>(1, std::min<long long>((n + threads - 1) / threads, sm_count() * 16)); }

}  // namespace

struct ark_input {
  enum Kind { Generate, FileJson, FileCsv, FileAvro, FileArrow } kind = Generate;
  std::mutex mu;
  // generate
  std::string context;
  std::chrono::nanoseconds interval{0};
  bool has_count = false;
  int64_t count_limit = 0, produced = 0, batch_size = 1;
  bool first = true;
  Batch cached;  // the replicated payload column (immutable)
  // file
  std::string path;
  bool connected = false, closed = false;
  BufferPtr file_dev;       // the file's bytes in HBM
  int64_t file_bytes = 0;
  BufferPtr line_off;       // int64 starts of the lines that are not empty (+ file end) on the device
  int64_t n_lines = 0, next_line = 0, rows_per_batch = 1 << 22;  // Avro: records, not lines
  std::unique_ptr<Processor> decoder;
  std::unique_ptr<SqlProcessor> sql;
  // csv
  std::vector<std::string> csv_names;
  std::vector<int> csv_types;
  int delim = ',';
  bool has_header = true;
  // avro
  std::shared_ptr<AvroFile> avro;  // header, schema and block table
  // arrow
  std::shared_ptr<IpcFile> ipc;    // schema and every record batch's nodes and buffers
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

// `visit`, when given, sees the file's bytes in order as they pass through the pinned chunks: (bytes, count, file offset)
using ChunkVisitor = std::function<void(const uint8_t*, size_t, int64_t)>;

void file_connect(ark_input* in, cudaStream_t stream, const ChunkVisitor* visit = nullptr) {
  struct stat st;
  if (stat(in->path.c_str(), &st) != 0) fail(ARK_ERR_PROCESS, "Read input failed: Object at location " + in->path + " not found");
  const int64_t n = (int64_t)st.st_size;
  FILE* f = fopen(in->path.c_str(), "rb");
  if (!f) fail(ARK_ERR_PROCESS, "Read input failed: cannot open " + in->path);
  in->file_dev = device_alloc((size_t)std::max<int64_t>(n, 1) + 64);
  // file → pinned chunks → HBM (two chunks in flight)
  const size_t CH = 8u << 20;
  BufferPtr stage = pinned_alloc(2 * CH);
  cudaEvent_t ev[2];
  for (auto& e : ev) ARK_CUDA(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
  bool used[2] = {false, false};
  int64_t done = 0;
  int turn = 0;
  bool io_error = false;
  std::exception_ptr visit_error;
  while (done < n) {
    uint8_t* slot = (uint8_t*)stage.get() + (size_t)turn * CH;
    if (used[turn]) ARK_CUDA(cudaEventSynchronize(ev[turn]));
    const size_t want = (size_t)std::min<int64_t>((int64_t)CH, n - done);
    const size_t got = fread(slot, 1, want, f);
    if (got == 0) { io_error = true; break; }
    if (visit) {
      try { (*visit)(slot, got, done); } catch (...) { visit_error = std::current_exception(); break; }
    }
    ARK_CUDA(cudaMemcpyAsync((uint8_t*)in->file_dev.get() + done, slot, got, cudaMemcpyHostToDevice, stream));
    ARK_CUDA(cudaEventRecord(ev[turn], stream));
    used[turn] = true;
    done += (int64_t)got;
    turn ^= 1;
  }
  fclose(f);
  ARK_CUDA(cudaStreamSynchronize(stream));
  for (auto& e : ev) cudaEventDestroy(e);
  if (io_error) fail(ARK_ERR_PROCESS, "Read input failed: short read on " + in->path);
  if (visit_error) std::rethrow_exception(visit_error);
  in->file_bytes = n;
  if (in->kind == ark_input::FileAvro || in->kind == ark_input::FileArrow) return;  // no lines: records come from the block tables
  // line starts
  if (n == 0) { in->n_lines = 0; return; }
  BufferPtr flags = device_alloc((size_t)n);
  {
    KernelTimer t("line_start_flags_kernel", stream);
    line_start_flags_kernel<<<grid_of(n), 256, 0, stream>>>((const uint8_t*)in->file_dev.get(), n, (uint8_t*)flags.get());
  }
  BufferPtr starts;
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
  in->n_lines = *(long long*)h.get();
  ARK_CUDA(cudaMemcpyAsync((long long*)starts.get() + in->n_lines, &in->file_bytes, 8, cudaMemcpyHostToDevice, stream));  // sentinel: file end
  ARK_CUDA(cudaStreamSynchronize(stream));
  in->line_off = starts;
  in->next_line = 0;
}

__global__ void rebase_offsets_kernel(const long long* starts, long long first, long long n, int32_t* out) {
  const long long base = starts[first];
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i <= n; i += (long long)gridDim.x * blockDim.x) out[i] = (int32_t)(starts[first + i] - base);
}

// lines [l0, l0 + n) as a Binary column whose rows are the lines (each still ends with its '\n')
Batch lines_batch(ark_input* in, int64_t l0, int64_t n, int64_t byte0, int64_t byte1, cudaStream_t stream) {
  if (byte1 - byte0 > 2147483647ll) fail(ARK_ERR_PROCESS, "file input: a batch of lines exceeds 2 GiB; lower batch_size");
  BufferPtr off = device_alloc((size_t)(n + 1) * 4);
  {
    KernelTimer t("rebase_offsets_kernel", stream);
    rebase_offsets_kernel<<<grid_of(n + 1), 256, 0, stream>>>((const long long*)in->line_off.get(), l0, n, (int32_t*)off.get());
  }
  Batch b;
  b.num_rows = n;
  Column c;
  c.field.name = "__value__"; c.field.type = DType::Binary; c.field.format = "z"; c.field.nullable = false;
  c.length = n; c.null_count = 0;
  c.offsets = (const int32_t*)off.get(); c.data = (const uint8_t*)in->file_dev.get() + byte0; c.data_bytes = byte1 - byte0; c.first_offset = 0;
  c.owners = {off, in->file_dev};
  b.cols.push_back(std::move(c));
  return b;
}

// the 1-based physical line that holds byte `off` of the file: the line terminators before it, empty lines included
long long physical_line(ark_input* in, long long off, cudaStream_t stream) {
  const uint8_t* file = (const uint8_t*)in->file_dev.get();
  note_launch("thrust::count");
  return 1 + (long long)thrust::count(thrust::cuda::par.on(stream), file, file + off, (uint8_t)'\n');
}

std::vector<std::string> split_csv_line(const std::string& line, char delim) {
  std::vector<std::string> out;
  std::string cur;
  size_t i = 0;
  while (true) {
    cur.clear();
    if (i < line.size() && line[i] == '"') {
      ++i;
      while (i < line.size()) {
        if (line[i] == '"') { if (i + 1 < line.size() && line[i + 1] == '"') { cur += '"'; i += 2; continue; } break; }
        cur += line[i++];
      }
      if (i < line.size()) ++i;
    } else {
      while (i < line.size() && line[i] != delim) cur += line[i++];
    }
    out.push_back(cur);
    if (i < line.size() && line[i] == delim) { ++i; continue; }
    break;
  }
  return out;
}

int csv_infer_type(const std::string& f, int cur) {  // -1 = no evidence yet (only empty fields)
  if (f.empty()) return cur;
  const uint8_t* p = (const uint8_t*)f.data();
  const int n = (int)f.size();
  auto is_int = [&] { long long v; return csv_parse_i64(p, n, &v); };  // digits, and a value that fits i64
  auto is_float = [&] { unsigned long long b; DecimalScan d; return csv_special_f64(p, n, &b) || decimal_scan(p, n, &d); };
  auto is_bool = [&] { std::string l; for (char c : f) l += (char)tolower((unsigned char)c); return l == "true" || l == "false"; };
  int t = is_int() ? CSV_I64 : (is_float() ? CSV_F64 : (is_bool() ? CSV_BOOL : CSV_STR));
  if (cur < 0) return t;
  if (cur == t) return t;
  if ((cur == CSV_I64 && t == CSV_F64) || (cur == CSV_F64 && t == CSV_I64)) return CSV_F64;
  return CSV_STR;
}

void csv_prepare(ark_input* in, cudaStream_t stream) {
  if (in->n_lines == 0) return;
  // the header, when there is one, + up to 1000 rows on the host
  const int64_t sample_lines = std::min<int64_t>(in->n_lines, (in->has_header ? 1 : 0) + 1000);
  std::vector<long long> starts((size_t)sample_lines + 1);
  ARK_CUDA(cudaMemcpyAsync(starts.data(), in->line_off.get(), (size_t)(sample_lines + 1) * 8, cudaMemcpyDeviceToHost, stream));
  ARK_CUDA(cudaStreamSynchronize(stream));
  const int64_t bytes = starts[(size_t)sample_lines] - starts[0];
  std::string text((size_t)bytes, '\0');
  ARK_CUDA(cudaMemcpyAsync(&text[0], (const uint8_t*)in->file_dev.get() + starts[0], (size_t)bytes, cudaMemcpyDeviceToHost, stream));
  ARK_CUDA(cudaStreamSynchronize(stream));
  auto line = [&](int64_t i) {
    std::string s = text.substr((size_t)(starts[(size_t)i] - starts[0]), (size_t)(starts[(size_t)i + 1] - starts[(size_t)i]));
    while (!s.empty() && (s.back() == '\n' || s.back() == '\r')) s.pop_back();
    return s;
  };
  std::vector<std::string> head = split_csv_line(line(0), (char)in->delim);
  if (in->has_header)
    for (auto& h : head)
      if (!utf8_valid((const uint8_t*)h.data(), (long long)h.size())) fail(ARK_ERR_PROCESS, "Read input failed: Arrow error: Csv error: Encountered invalid UTF-8 data for line " + std::to_string(physical_line(in, starts[0], stream)));
  if (in->has_header) in->csv_names = head;
  else for (size_t i = 0; i < head.size(); ++i) in->csv_names.push_back("column_" + std::to_string(i + 1));
  if ((int)in->csv_names.size() > CSV_MAX_COLS) fail(ARK_ERR_UNSUPPORTED, "csv input: more than 32 columns");
  std::vector<int> types(in->csv_names.size(), -1);
  for (int64_t i = in->has_header ? 1 : 0; i < sample_lines; ++i) {
    std::vector<std::string> f = split_csv_line(line(i), (char)in->delim);
    for (size_t c = 0; c < types.size() && c < f.size(); ++c) types[c] = csv_infer_type(f[c], types[c]);
  }
  for (auto& t : types) if (t < 0) t = CSV_STR;
  in->csv_types = types;
  in->next_line = in->has_header ? 1 : 0;
}

Batch csv_batch(ark_input* in, int64_t l0, int64_t n, cudaStream_t stream) {
  const int nc = (int)in->csv_names.size();
  CsvParams P;
  memset(&P, 0, sizeof P);
  P.data = (const uint8_t*)in->file_dev.get();
  // 32-bit line offsets relative to the batch's first byte
  BufferPtr h = pinned_alloc(32);
  ARK_CUDA(cudaMemcpyAsync(h.get(), (const long long*)in->line_off.get() + l0, 8, cudaMemcpyDeviceToHost, stream));
  ARK_CUDA(cudaMemcpyAsync((char*)h.get() + 8, (const long long*)in->line_off.get() + l0 + n, 8, cudaMemcpyDeviceToHost, stream));
  ARK_CUDA(cudaStreamSynchronize(stream));
  const long long byte0 = ((long long*)h.get())[0], byte1 = ((long long*)h.get())[1];
  if (byte1 - byte0 > 2147483647ll) fail(ARK_ERR_PROCESS, "file input: a batch of lines exceeds 2 GiB; lower batch_size");
  BufferPtr loff = device_alloc((size_t)(n + 1) * 4);
  {
    KernelTimer t("rebase_offsets_kernel", stream);
    rebase_offsets_kernel<<<grid_of(n + 1), 256, 0, stream>>>((const long long*)in->line_off.get(), l0, n, (int32_t*)loff.get());
  }
  P.data += byte0; P.line_off = (const int32_t*)loff.get(); P.n_rows = n; P.n_cols = nc; P.delim = in->delim;
  std::vector<BufferPtr> vals(nc), valid(nc), slen(nc), ssrc(nc), sraw(nc);
  BufferPtr err = device_alloc(16);
  ARK_CUDA(cudaMemsetAsync(err.get(), 0xFF, 16, stream));
  P.error = (unsigned long long*)err.get();
  for (int c = 0; c < nc; ++c) {
    P.types[c] = in->csv_types[c];
    valid[c] = device_alloc((size_t)std::max<int64_t>(n, 1));
    P.valid[c] = (uint8_t*)valid[c].get();
    if (in->csv_types[c] == CSV_STR) {
      slen[c] = device_alloc((size_t)(n + 1) * 4); ssrc[c] = device_alloc((size_t)std::max<int64_t>(n, 1) * 8); sraw[c] = device_alloc((size_t)std::max<int64_t>(n, 1) * 4);
      ARK_CUDA(cudaMemsetAsync((int32_t*)slen[c].get() + n, 0, 4, stream));
      P.str_len[c] = (int32_t*)slen[c].get(); P.str_src[c] = (long long*)ssrc[c].get(); P.str_raw[c] = (int32_t*)sraw[c].get();
    } else {
      vals[c] = device_alloc((size_t)std::max<int64_t>(n, 1) * (in->csv_types[c] == CSV_BOOL ? 1 : 8));
      P.values[c] = vals[c].get();
    }
  }
  {
    KernelTimer t("csv_parse_kernel", stream);
    csv_parse_kernel<<<grid_of(n, 128), 128, 0, stream>>>(P);
  }
  ARK_CUDA(cudaGetLastError());
  BufferPtr herr = pinned_alloc(16);
  ARK_CUDA(cudaMemcpyAsync(herr.get(), err.get(), 8, cudaMemcpyDeviceToHost, stream));
  ARK_CUDA(cudaStreamSynchronize(stream));
  const unsigned long long ekey = *(const unsigned long long*)herr.get();
  if (ekey != ~0ull) {
    const int ecode = (int)(ekey & 3);
    ARK_CUDA(cudaMemcpyAsync(herr.get(), (const long long*)in->line_off.get() + l0 + (long long)(ekey >> 2), 8, cudaMemcpyDeviceToHost, stream));
    ARK_CUDA(cudaStreamSynchronize(stream));
    const long long lineno = physical_line(in, *(const long long*)herr.get(), stream);
    fail(ARK_ERR_PROCESS, ecode == 2 ? "Read input failed: Arrow error: Csv error: incorrect number of fields for line " + std::to_string(lineno)
                          : ecode == 3 ? "Read input failed: Arrow error: Csv error: Encountered invalid UTF-8 data for line " + std::to_string(lineno)
                                       : "Read input failed: Arrow error: Parser error: Error while parsing value of line " + std::to_string(lineno));
  }
  Batch b;
  b.num_rows = n;
  for (int c = 0; c < nc; ++c) {
    Column col;
    col.field.name = in->csv_names[c]; col.field.nullable = true; col.length = n;
    switch (in->csv_types[c]) {
      case CSV_I64: col.field.type = DType::Int64; col.field.format = "l"; col.data = (const uint8_t*)vals[c].get(); col.data_bytes = n * 8; col.owners = {vals[c]}; break;
      case CSV_F64: col.field.type = DType::Float64; col.field.format = "g"; col.data = (const uint8_t*)vals[c].get(); col.data_bytes = n * 8; col.owners = {vals[c]}; break;
      case CSV_BOOL: col.field.type = DType::Bool; col.field.format = "b"; set_bool_values(col, vals[c], n, stream); break;
      default: {
        // a field's bytes lie inside its line, so the batch's byte span (at most 2 GiB, checked above) bounds the column
        const Varlen v = varlen_layout((const int32_t*)slen[c].get(), n, nullptr, byte1 - byte0, "file input: column '" + in->csv_names[c] + "'", stream);
        if (n) {
          KernelTimer t("csv_strings_kernel", stream);
          csv_strings_kernel<<<grid_of(n), 256, 0, stream>>>(P.data, n, (const int32_t*)v.offsets.get(), (const long long*)ssrc[c].get(), (const int32_t*)sraw[c].get(), (uint8_t*)v.bytes.get());
        }
        col.field.type = DType::Utf8; col.field.format = "u";
        set_varlen(col, v);
        break;
      }
    }
    set_validity_exact(col, (const uint8_t*)valid[c].get(), n, stream);
    b.cols.push_back(std::move(col));
  }
  return b;
}

// returns false at EOF
bool input_next(ark_input* in, Batch& out, cudaStream_t stream) {
  if (in->kind == ark_input::Generate) {
    {
      std::lock_guard<std::mutex> l(in->mu);
      if (in->closed) return false;
    }
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
  std::lock_guard<std::mutex> l(in->mu);
  if (!in->connected) fail(ARK_ERR_PROCESS, "Stream is None");  // file.rs:433-435
  while (true) {
    if (in->closed || in->next_line >= in->n_lines) return false;
    const int64_t l0 = in->next_line;
    const int64_t n = std::min<int64_t>(in->rows_per_batch, in->n_lines - l0);
    in->next_line += n;
    Batch b;
    if (in->kind == ark_input::FileAvro) {
      b = avro_batch(*in->avro, in->file_dev, l0, n, stream);
    } else if (in->kind == ark_input::FileArrow) {
      b = ipc_batch(*in->ipc, in->file_dev, l0, n, stream);
    } else if (in->kind == ark_input::FileJson) {
      BufferPtr h = pinned_alloc(32);
      ARK_CUDA(cudaMemcpyAsync(h.get(), (const long long*)in->line_off.get() + l0, 8, cudaMemcpyDeviceToHost, stream));
      ARK_CUDA(cudaMemcpyAsync((char*)h.get() + 8, (const long long*)in->line_off.get() + l0 + n, 8, cudaMemcpyDeviceToHost, stream));
      ARK_CUDA(cudaStreamSynchronize(stream));
      Batch lines = lines_batch(in, l0, n, ((long long*)h.get())[0], ((long long*)h.get())[1], stream);
      b = json_to_arrow_device(*in->decoder, lines, stream);
    } else {
      b = csv_batch(in, l0, n, stream);
    }
    if (b.num_rows == 0) continue;  // NDJSON lines that hold only spaces
    if (in->sql) {
      std::vector<Field> fields;
      for (auto& c : b.cols) {
        Field f = c.field;
        if (f.format.empty()) f.format = dtype_arrow_format(f.type);
        // Arrow IPC columns of the types the SQL subset does not compute on (Int32, UInt32, UInt64, Float32) reach the
        // planner as the sql processor's import presents them, so a query that reads one is Unsupported as it is there
        if (in->kind == ark_input::FileArrow && fixed_width(f.type) && f.type != DType::Int64 && f.type != DType::Float64) f.type = DType::Null;
        fields.push_back(f);
      }
      for (auto& c : b.cols) if (c.field.format.empty()) c.field.format = dtype_arrow_format(c.field.type);
      auto plan = in->sql->plan_for(fields);
      b = in->sql->execute(*plan, b, stream);
      if (b.num_rows == 0 && b.cols.empty()) continue;
    }
    ARK_CUDA(cudaStreamSynchronize(stream));
    out = std::move(b);
    return true;
  }
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
      in->kind = ark_input::Generate;
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
      in->connected = true;
    } else {
      const JsonValue* it = cfg.get("input_type");
      if (!it || it->kind != JsonValue::Object) fail(ARK_ERR_SERIALIZATION, "missing field `input_type`");
      const JsonValue* ty = it->get("type");
      if (!ty || ty->kind != JsonValue::String) fail(ARK_ERR_SERIALIZATION, "missing field `type` (InputType)");
      if (ty->str == "json") in->kind = ark_input::FileJson;
      else if (ty->str == "csv") in->kind = ark_input::FileCsv;
      else if (ty->str == "avro") in->kind = ark_input::FileAvro;
      else if (ty->str == "arrow") in->kind = ark_input::FileArrow;
      else if (ty->str == "parquet")
        fail(ARK_ERR_UNSUPPORTED, "file input: " + ty->str + " files are not decoded on the GPU (json, csv, avro and arrow are)");
      else fail(ARK_ERR_SERIALIZATION, "unknown variant `" + ty->str + "`, expected one of `avro`, `arrow`, `json`, `csv`, `parquet`");
      const JsonValue* p = it->get("path");
      if (!p || p->kind != JsonValue::String) fail(ARK_ERR_SERIALIZATION, "missing field `path`");
      if (const JsonValue* st = it->get("store")) if (st->kind != JsonValue::Null) fail(ARK_ERR_UNSUPPORTED, "file input: remote object stores (network I/O) stay in the reference's input");
      if (const JsonValue* bl = cfg.get("ballista")) if (bl->kind != JsonValue::Null) fail(ARK_ERR_UNSUPPORTED, "file input: ballista");
      in->path = p->str;
      if (in->path.rfind("file://", 0) == 0) in->path = in->path.substr(7);
      opt_u("batch_size", &in->rows_per_batch);  // extension: rows per RecordBatch (DataFusion's execution.batch_size)
      if (in->rows_per_batch <= 0) in->rows_per_batch = 1 << 22;
      if (const JsonValue* hh = it->get("has_header")) if (hh->kind == JsonValue::Bool) in->has_header = hh->b;
      if (const JsonValue* q = cfg.get("query")) {
        if (q->kind == JsonValue::Object) {
          const JsonValue* qs = q->get("query");
          if (!qs || qs->kind != JsonValue::String) fail(ARK_ERR_SERIALIZATION, "missing field `query` (QueryConfig)");
          std::string table = "flow";  // default_table(), file.rs
          if (const JsonValue* t = q->get("table")) if (t->kind == JsonValue::String) table = t->str;
          std::string sc = "{\"query\": \"";
          for (char ch : qs->str) { if (ch == '"' || ch == '\\') sc += '\\'; if (ch == '\n') { sc += "\\n"; continue; } sc += ch; }
          sc += "\", \"table_name\": \"" + table + "\"}";
          in->sql = SqlProcessor::from_config(sc.c_str());
        } else if (q->kind != JsonValue::Null) fail(ARK_ERR_SERIALIZATION, "invalid type for `query`: expected QueryConfig");
      }
      if (in->kind == ark_input::FileJson) in->decoder = make_json_to_arrow("{}");
    }
    *out = in.release();
  });
}

int ark_input_connect(ark_input_t* in) {
  return guarded([&] {
    if (!in) fail(ARK_ERR_PROCESS, "null input");
    if (in->kind == ark_input::Generate) return;  // generate.rs:62-64
    std::lock_guard<std::mutex> l(in->mu);
    if (in->connected) return;
    if (in->kind == ark_input::FileAvro) {
      // the header (schema and codec, whose errors need no device) first, then the block table during the upload
      std::shared_ptr<AvroFile> av = avro_open(in->path);
      StreamLease lease;
      if (!av) { file_connect(in, lease.s); fail(ARK_ERR_PROCESS, "Read input failed: cannot open " + in->path); }
      const ChunkVisitor visit = [&](const uint8_t* p, size_t n, int64_t base) { avro_scan(*av, p, n, base); };
      file_connect(in, lease.s, &visit);
      avro_scan_end(*av);
      in->avro = av;
      in->n_lines = avro_rows(*av);
      in->next_line = 0;
      in->connected = true;
      return;
    }
    if (in->kind == ark_input::FileArrow) {
      // every piece of metadata first (its errors need no device), then the upload
      std::shared_ptr<IpcFile> ipc = ipc_open(in->path);
      StreamLease lease;
      file_connect(in, lease.s);
      if (!ipc) fail(ARK_ERR_PROCESS, "Read input failed: cannot open " + in->path);
      in->ipc = ipc;
      in->n_lines = ipc_rows(*ipc);
      in->next_line = 0;
      in->connected = true;
      return;
    }
    StreamLease lease;
    file_connect(in, lease.s);
    if (in->kind == ark_input::FileCsv) csv_prepare(in, lease.s);
    else if (in->n_lines > 0) {
      // schema of the file = merge over its first ≤ 1000 records (DataFusion's schema_infer_max_records), fixed for every batch
      const int64_t sample_lines = std::min<int64_t>(in->n_lines, 1000);
      std::vector<long long> starts((size_t)sample_lines + 1);
      ARK_CUDA(cudaMemcpyAsync(starts.data(), in->line_off.get(), (size_t)(sample_lines + 1) * 8, cudaMemcpyDeviceToHost, lease.s));
      ARK_CUDA(cudaStreamSynchronize(lease.s));
      std::string text((size_t)(starts[(size_t)sample_lines] - starts[0]), '\0');
      ARK_CUDA(cudaMemcpyAsync(&text[0], (const uint8_t*)in->file_dev.get() + starts[0], text.size(), cudaMemcpyDeviceToHost, lease.s));
      ARK_CUDA(cudaStreamSynchronize(lease.s));
      std::vector<std::string> sample;
      for (int64_t i = 0; i < sample_lines; ++i)
        sample.push_back(text.substr((size_t)(starts[(size_t)i] - starts[0]), (size_t)(starts[(size_t)i + 1] - starts[(size_t)i])));
      in->decoder = make_json_to_arrow_for_sample(sample);
    }
    in->connected = true;
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
    if (in->kind != ark_input::Generate) in->closed = true;  // file.rs:458-461 cancels the stream; generate.rs:93-95 is a no-op
  });
}

void ark_input_destroy(ark_input_t* in) { delete in; }

}  // extern "C"
