// csv.cu — the `file` input's `csv` type: records parsed on the device, one thread per record.
//
// Column types come from the first 1000 records, inferred on the host as Int64 / Float64 / Boolean / Utf8 (dates stay
// strings); quoted CSV fields may not contain line breaks (oracle/csv_oracle.py lists the smaller deviations from
// DataFusion's reader).  A CSV column is Int64 when its sample values are decimal integers within the i64 range, and
// Float64 when they are decimals or nan / inf / infinity (any case, optional sign; Arrow's reader accepts these spellings
// too); Float64 values are correctly rounded.  The CSV header is the first line that is not empty (file_input.h's
// LineIndex leaves empty lines out).
// CSV errors: a batch reports the error of its FIRST failing line in file order, and the line number in the message
// counts physical lines from 1, empty ones included.  Within one line the order is: wrong number of fields (bytes after
// a closing quote count as such), then a value that does not parse as its column's type (invalid UTF-8 in a numeric or
// Boolean field is this error), then invalid UTF-8 in a Utf8 field.  tests/test_inputs_edges_gpu.py checks all of this
// against oracle/csv_oracle.py.
#include "decimal.cuh"
#include "decoded.h"
#include "file_input.h"
#include "utf8.cuh"
#include "varlen.h"

using namespace ark;

namespace {
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


struct CsvFormat : FileFormat {
  explicit CsvFormat(bool header) : has_header(header) {}
  bool has_header;
  int delim = ',';
  LineIndex lines;
  std::vector<std::string> names;
  std::vector<int> types;

  int64_t prepare(const BufferPtr& file_dev, int64_t bytes, cudaStream_t stream) override {
    lines.build(file_dev, bytes, stream);
    if (lines.lines == 0) return 0;
    // the header, when there is one, + up to 1000 rows on the host
    int64_t first = 0;
    std::vector<std::string> sample = lines.sample(std::min<int64_t>(lines.lines, (has_header ? 1 : 0) + 1000), stream, &first);
    for (auto& s : sample) while (!s.empty() && (s.back() == '\n' || s.back() == '\r')) s.pop_back();
    std::vector<std::string> head = split_csv_line(sample[0], (char)delim);
    names.clear();
    if (has_header)
      for (auto& h : head)
        if (!utf8_valid((const uint8_t*)h.data(), (long long)h.size())) fail(ARK_ERR_PROCESS, "Read input failed: Arrow error: Csv error: Encountered invalid UTF-8 data for line " + std::to_string(lines.physical_line(first, stream)));
    if (has_header) names = head;
    else for (size_t i = 0; i < head.size(); ++i) names.push_back("column_" + std::to_string(i + 1));
    if ((int)names.size() > CSV_MAX_COLS) fail(ARK_ERR_UNSUPPORTED, "csv input: more than 32 columns");
    types.assign(names.size(), -1);
    for (size_t i = has_header ? 1 : 0; i < sample.size(); ++i) {
      std::vector<std::string> f = split_csv_line(sample[i], (char)delim);
      for (size_t c = 0; c < types.size() && c < f.size(); ++c) types[c] = csv_infer_type(f[c], types[c]);
    }
    for (auto& t : types) if (t < 0) t = CSV_STR;
    return lines.lines - (has_header ? 1 : 0);
  }

  Batch batch(int64_t r0, int64_t n, cudaStream_t stream) override {
    const int64_t l0 = r0 + (has_header ? 1 : 0);
    const int nc = (int)names.size();
    CsvParams P;
    memset(&P, 0, sizeof P);
    // 32-bit line offsets relative to the batch's first byte
    const auto [byte0, byte1] = lines.span(l0, n, stream);
    BufferPtr loff = lines.rebased(l0, n, stream);
    P.data = (const uint8_t*)lines.file.get() + byte0; P.line_off = (const int32_t*)loff.get(); P.n_rows = n; P.n_cols = nc; P.delim = delim;
    BufferPtr err = device_alloc(16);
    ARK_CUDA(cudaMemsetAsync(err.get(), 0xFF, 16, stream));
    P.error = (unsigned long long*)err.get();
    static const DType dtype[] = {DType::Int64, DType::Float64, DType::Bool, DType::Utf8};
    std::vector<StagedColumn> cols;
    for (int c = 0; c < nc; ++c) {
      P.types[c] = types[c];
      cols.push_back(stage_column(dtype[types[c]], n, true, true, stream));
      StagedColumn& s = cols.back();
      P.valid[c] = (uint8_t*)s.valid.get();
      P.values[c] = s.values.get();
      P.str_len[c] = (int32_t*)s.len.get(); P.str_src[c] = (long long*)s.src.get(); P.str_raw[c] = (int32_t*)s.raw.get();
      // a field's bytes lie inside its line, so the batch's byte span (at most 2 GiB, checked above) bounds the column
      s.bound = byte1 - byte0; s.what = "file input: column '" + names[c] + "'";
    }
    {
      KernelTimer t("csv_parse_kernel", stream);
      csv_parse_kernel<<<grid_of(n, 128), 128, 0, stream>>>(P);
    }
    ARK_CUDA(cudaGetLastError());
    settle_columns(cols, err.get(), 8, [&](const void* h) {
      const unsigned long long ekey = *(const unsigned long long*)h;
      if (ekey == ~0ull) return;
      const int ecode = (int)(ekey & 3);
      BufferPtr hstart = pinned_alloc(8);
      ARK_CUDA(cudaMemcpyAsync(hstart.get(), (const long long*)lines.starts.get() + l0 + (long long)(ekey >> 2), 8, cudaMemcpyDeviceToHost, stream));
      ARK_CUDA(cudaStreamSynchronize(stream));
      const long long lineno = lines.physical_line(*(const long long*)hstart.get(), stream);
      fail(ARK_ERR_PROCESS, ecode == 2 ? "Read input failed: Arrow error: Csv error: incorrect number of fields for line " + std::to_string(lineno)
                            : ecode == 3 ? "Read input failed: Arrow error: Csv error: Encountered invalid UTF-8 data for line " + std::to_string(lineno)
                                         : "Read input failed: Arrow error: Parser error: Error while parsing value of line " + std::to_string(lineno));
    }, stream);
    Batch b;
    b.num_rows = n;
    for (int c = 0; c < nc; ++c)
      b.cols.push_back(finish_column(cols[c], Field{names[c], dtype[types[c]], true, dtype_arrow_format(dtype[types[c]])}, [&](const StagedColumn& s, uint8_t* bytes) {
        if (!n) return;
        KernelTimer t("csv_strings_kernel", stream);
        csv_strings_kernel<<<grid_of(n), 256, 0, stream>>>(P.data, n, (const int32_t*)s.offsets.get(), (const long long*)s.src.get(), (const int32_t*)s.raw.get(), bytes);
      }, stream));
    return b;
  }
};

}  // namespace

std::unique_ptr<FileFormat> ark::make_csv_format(bool has_header) { return std::make_unique<CsvFormat>(has_header); }
