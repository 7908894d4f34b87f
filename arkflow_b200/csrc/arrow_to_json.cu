// arrow_to_json.cu — `arrow_to_json`: one JSON object per row, appended as a Binary `__value__` column.
//
// Stands in for ArrowToJsonProcessor::process / arrow_to_json (crates/arkflow-plugin/src/processor/
// json.rs:78-113) + MessageBatch::new_binary_with_origin (crates/arkflow-core/src/lib.rs:280-302), i.e.
// arrow-json 55.2's LineDelimitedWriter (third-party, not under /root/reference) with its defaults:
//   * fields in schema order, NULL fields omitted (explicit_nulls = false), no whitespace;
//   * Int64 as decimal, Boolean as true/false, Utf8 escaped like serde_json (\" \\ \b \f \n \r \t,
//     other control characters as \u00xx, everything else verbatim), Binary as lowercase hex;
//   * Float64 through lexical-core's writer: shortest round-trip digits (Ryu, tables generated and
//     self-checked by scripts/gen_ryu_tables.py), positional with at least ".0" while the scientific
//     exponent is in [-5, 9], d.ddde±x outside; NaN / ±inf → null.
// Two passes, one thread per row: measure → exclusive scan → write.
#include <cub/device/device_scan.cuh>

#include <algorithm>

#include "engine.h"
#include "stage_store.cuh"
#include "json_mini.h"
#include "ryu_tables.h"

namespace ark {

namespace {

constexpr int AJ_MAX_COLS = 16;
constexpr int AJ_KEY_BYTES = 72;

struct AjCol {
  int32_t dtype;
  int32_t key_len;            // bytes of `"name":` (already JSON-escaped)
  char key[AJ_KEY_BYTES];
  ColView view;
};

struct AjParams {
  int64_t n_rows;
  int32_t n_cols;
  AjCol cols[AJ_MAX_COLS];
};

struct Sink {
  uint8_t* p;   // nullptr ⇒ counting only
  int n;
  __device__ __forceinline__ void put(uint8_t c) { if (p) p[n] = c; ++n; }
};

__device__ void put_u64(Sink& s, unsigned long long v) {
  char buf[20];
  int k = 0;
  do { buf[k++] = (char)('0' + v % 10); v /= 10; } while (v);
  while (k) s.put((uint8_t)buf[--k]);
}

__device__ void put_i64(Sink& s, long long v) {
  if (v < 0) { s.put('-'); put_u64(s, 0ull - (unsigned long long)v); }
  else put_u64(s, (unsigned long long)v);
}

// ---- Ryu (transcription of d2d() in scripts/gen_ryu_tables.py) ----
__device__ __forceinline__ int pow5bits(int e) { return (int)(((unsigned)e * 1217359u) >> 19) + 1; }
__device__ __forceinline__ int log10pow2(int e) { return (int)(((unsigned)e * 78913u) >> 18); }
__device__ __forceinline__ int log10pow5(int e) { return (int)(((unsigned)e * 732923u) >> 20); }

__device__ __forceinline__ unsigned long long mulshift64(unsigned long long m, const unsigned long long* mul, int j) {
  // ((m * mul) >> j), mul = {low, high}, 64 <= j < 128+
  const unsigned long long b0_hi = __umul64hi(m, mul[0]);
  const unsigned long long b2_lo = m * mul[1], b2_hi = __umul64hi(m, mul[1]);
  const unsigned long long sum_lo = b0_hi + b2_lo;
  const unsigned long long sum_hi = b2_hi + (sum_lo < b0_hi ? 1ull : 0ull);
  const int sh = j - 64;  // 0 < sh < 64 on every call path
  return (sum_hi << (64 - sh)) | (sum_lo >> sh);
}
__device__ __forceinline__ bool multiple_of_pow5(unsigned long long v, int p) {
  int c = 0;
  while (v && v % 5 == 0) { v /= 5; ++c; }
  return c >= p;
}

__device__ void d2d(unsigned long long bits, unsigned long long* digits, int* exp10) {
  const unsigned long long ieee_m = bits & ((1ull << 52) - 1);
  const int ieee_e = (int)((bits >> 52) & 0x7FF);
  int e2; unsigned long long m2;
  if (ieee_e == 0) { e2 = 1 - 1023 - 52 - 2; m2 = ieee_m; }
  else { e2 = ieee_e - 1023 - 52 - 2; m2 = (1ull << 52) | ieee_m; }
  const bool accept = (m2 & 1) == 0;
  const unsigned long long mv = 4 * m2;
  const int mm_shift = (ieee_m != 0 || ieee_e <= 1) ? 1 : 0;
  unsigned long long vr, vp, vm;
  int e10;
  bool vm_tz = false, vr_tz = false;
  if (e2 >= 0) {
    const int q = log10pow2(e2) - (e2 > 3);
    e10 = q;
    const int k = ARK_RYU_POW5_INV_BITCOUNT + pow5bits(q) - 1;
    const int i = -e2 + q + k;
    vr = mulshift64(4 * m2, kRyuPow5Inv[q], i);
    vp = mulshift64(4 * m2 + 2, kRyuPow5Inv[q], i);
    vm = mulshift64(4 * m2 - 1 - mm_shift, kRyuPow5Inv[q], i);
    if (q <= 21) {
      if (mv % 5 == 0) vr_tz = multiple_of_pow5(mv, q);
      else if (accept) vm_tz = multiple_of_pow5(mv - 1 - mm_shift, q);
      else vp -= multiple_of_pow5(mv + 2, q) ? 1 : 0;
    }
  } else {
    const int q = log10pow5(-e2) - (-e2 > 1);
    e10 = q + e2;
    const int i = -e2 - q;
    const int k = pow5bits(i) - ARK_RYU_POW5_BITCOUNT;
    const int j = q - k;
    vr = mulshift64(4 * m2, kRyuPow5[i], j);
    vp = mulshift64(4 * m2 + 2, kRyuPow5[i], j);
    vm = mulshift64(4 * m2 - 1 - mm_shift, kRyuPow5[i], j);
    if (q <= 1) {
      vr_tz = true;
      if (accept) vm_tz = mm_shift == 1; else --vp;
    } else if (q < 63) {
      vr_tz = (mv & ((1ull << q) - 1)) == 0;
    }
  }
  int removed = 0;
  unsigned last = 0;
  unsigned long long out;
  if (vm_tz || vr_tz) {
    while (vp / 10 > vm / 10) {
      vm_tz = vm_tz && vm % 10 == 0;
      vr_tz = vr_tz && last == 0;
      last = (unsigned)(vr % 10);
      vr /= 10; vp /= 10; vm /= 10; ++removed;
    }
    if (vm_tz) {
      while (vm % 10 == 0) {
        vr_tz = vr_tz && last == 0;
        last = (unsigned)(vr % 10);
        vr /= 10; vp /= 10; vm /= 10; ++removed;
      }
    }
    if (vr_tz && last == 5 && vr % 2 == 0) last = 4;
    out = vr + (((vr == vm && (!accept || !vm_tz)) || last >= 5) ? 1 : 0);
  } else {
    bool round_up = false;
    while (vp / 10 > vm / 10) {
      round_up = vr % 10 >= 5;
      vr /= 10; vp /= 10; vm /= 10; ++removed;
    }
    out = vr + ((vr == vm || round_up) ? 1 : 0);
  }
  *digits = out; *exp10 = e10 + removed;
}

__device__ void put_f64(Sink& s, unsigned long long bits) {
  const unsigned long long mag = bits & 0x7FFFFFFFFFFFFFFFull;
  if ((mag >> 52) == 0x7FF) { s.put('n'); s.put('u'); s.put('l'); s.put('l'); return; }  // NaN / inf
  if (bits >> 63) s.put('-');
  if (mag == 0) { s.put('0'); s.put('.'); s.put('0'); return; }
  unsigned long long digits; int e10;
  d2d(mag, &digits, &e10);
  char ds[20];
  int nd = 0;
  { char rev[20]; unsigned long long v = digits; do { rev[nd++] = (char)('0' + v % 10); v /= 10; } while (v); for (int i = 0; i < nd; ++i) ds[i] = rev[nd - 1 - i]; }
  const int sci = e10 + nd - 1;
  if (sci >= -5 && sci <= 9) {
    if (e10 >= 0) {
      for (int i = 0; i < nd; ++i) s.put(ds[i]);
      for (int i = 0; i < e10; ++i) s.put('0');
      s.put('.'); s.put('0');
    } else if (-e10 < nd) {
      for (int i = 0; i < nd + e10; ++i) s.put(ds[i]);
      s.put('.');
      for (int i = nd + e10; i < nd; ++i) s.put(ds[i]);
    } else {
      s.put('0'); s.put('.');
      for (int i = 0; i < -e10 - nd; ++i) s.put('0');
      for (int i = 0; i < nd; ++i) s.put(ds[i]);
    }
  } else {
    s.put(ds[0]); s.put('.');
    if (nd > 1) { for (int i = 1; i < nd; ++i) s.put(ds[i]); } else s.put('0');
    s.put('e');
    put_i64(s, sci);
  }
}

__device__ void put_json_string(Sink& s, const uint8_t* p, int len) {
  const char* hex = "0123456789abcdef";
  s.put('"');
  for (int i = 0; i < len; ++i) {
    const uint8_t c = p[i];
    if (c == '"') { s.put('\\'); s.put('"'); }
    else if (c == '\\') { s.put('\\'); s.put('\\'); }
    else if (c >= 0x20) s.put(c);
    else if (c == '\b') { s.put('\\'); s.put('b'); }
    else if (c == '\f') { s.put('\\'); s.put('f'); }
    else if (c == '\n') { s.put('\\'); s.put('n'); }
    else if (c == '\r') { s.put('\\'); s.put('r'); }
    else if (c == '\t') { s.put('\\'); s.put('t'); }
    else { s.put('\\'); s.put('u'); s.put('0'); s.put('0'); s.put(hex[c >> 4]); s.put(hex[c & 15]); }
  }
  s.put('"');
}

__device__ void put_hex(Sink& s, const uint8_t* p, int len) {
  const char* hex = "0123456789abcdef";
  s.put('"');
  for (int i = 0; i < len; ++i) { s.put(hex[p[i] >> 4]); s.put(hex[p[i] & 15]); }
  s.put('"');
}

__device__ int emit_row(const AjParams& P, int64_t row, uint8_t* out) {
  Sink s{out, 0};
  s.put('{');
  bool first = true;
  for (int c = 0; c < P.n_cols; ++c) {
    const AjCol& col = P.cols[c];
    if ((DType)col.dtype == DType::Null) continue;
    const ColView& v = col.view;
    if (v.validity && !((v.validity[(row + v.validity_bit0) >> 3] >> ((row + v.validity_bit0) & 7)) & 1)) continue;
    if (!first) s.put(',');
    first = false;
    for (int i = 0; i < col.key_len; ++i) s.put((uint8_t)col.key[i]);
    switch ((DType)col.dtype) {
      case DType::Int64: put_i64(s, ((const long long*)v.data)[row]); break;
      case DType::Float64: put_f64(s, ((const unsigned long long*)v.data)[row]); break;
      case DType::Bool: {
        const int64_t b = row + v.data_bit0;
        const bool t = (((const uint8_t*)v.data)[b >> 3] >> (b & 7)) & 1;
        const char* w = t ? "true" : "false";
        for (int i = 0; w[i]; ++i) s.put((uint8_t)w[i]);
        break;
      }
      case DType::Utf8: put_json_string(s, (const uint8_t*)v.data + v.offsets[row], v.offsets[row + 1] - v.offsets[row]); break;
      default: put_hex(s, (const uint8_t*)v.data + v.offsets[row], v.offsets[row + 1] - v.offsets[row]); break;
    }
  }
  s.put('}');
  return s.n;
}

__global__ void arrow_to_json_measure_kernel(const __grid_constant__ AjParams P, int32_t* lens) {
  const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r < P.n_rows) lens[r] = emit_row(P, r, nullptr);
}
// The lines of one CTA's rows are contiguous in the output: each thread formats its row into a shared-memory
// image of that range, which then leaves with 16-byte stores (byte-wise stores at a ~65-byte stride straight
// to global memory cost an order of magnitude more than the formatting itself).
constexpr int AJ_THREADS = 128;
__global__ void __launch_bounds__(AJ_THREADS) arrow_to_json_write_kernel(const __grid_constant__ AjParams P, const int32_t* offsets, uint8_t* out,
                                                                          int stage_bytes) {
  extern __shared__ __align__(16) uint8_t aj_stage[];
  const int64_t r0 = (int64_t)blockIdx.x * AJ_THREADS;
  const int rows = (int)((P.n_rows - r0) < AJ_THREADS ? (P.n_rows - r0) : AJ_THREADS);
  const int64_t r = r0 + threadIdx.x;
  const int32_t bb = offsets[r0];
  const int tb = offsets[r0 + rows] - bb;
  if (tb + 16 > stage_bytes) {  // long rows: format straight into global memory
    if (r < P.n_rows) emit_row(P, r, out + offsets[r]);
    return;
  }
  const int mis = stage_misalignment(out + bb);
  if (r < P.n_rows) emit_row(P, r, aj_stage + mis + (offsets[r] - bb));
  __syncthreads();
  stage_store(out + bb, aj_stage, mis, tb, threadIdx.x, AJ_THREADS);
}

std::string json_escape_key(const std::string& name) {
  static const char* hex = "0123456789abcdef";
  std::string o = "\"";
  for (unsigned char c : name) {
    if (c == '"') o += "\\\"";
    else if (c == '\\') o += "\\\\";
    else if (c >= 0x20) o += (char)c;
    else if (c == '\b') o += "\\b"; else if (c == '\f') o += "\\f"; else if (c == '\n') o += "\\n";
    else if (c == '\r') o += "\\r"; else if (c == '\t') o += "\\t";
    else { o += "\\u00"; o += hex[c >> 4]; o += hex[c & 15]; }
  }
  return o + "\":";
}

}  // namespace

// zero-column batch → zero lines → length mismatch in new_binary_with_origin
void fail_filtered_to_no_columns() {
  fail(ARK_ERR_PROCESS, "Creating an Arrow record batch failed: Invalid argument error: all columns in a record batch must have the same length");
}

struct ArrowToJsonProcessor : Processor {
  const char* type() const override { return "arrow_to_json"; }
  bool has_include = false;
  std::vector<std::string> include;
};

std::unique_ptr<Processor> make_arrow_to_json(const char* config_json) {
  // reference: json.rs:141-145 — the message really says "JsonToArrow" for both processors
  if (!config_json) fail(ARK_ERR_CONFIG, "JsonToArrow processor configuration is missing");
  JsonValue cfg = parse_json(config_json);
  if (cfg.kind == JsonValue::Null) fail(ARK_ERR_CONFIG, "JsonToArrow processor configuration is missing");
  if (cfg.kind != JsonValue::Object) fail(ARK_ERR_SERIALIZATION, "invalid type: expected struct JsonProcessorConfig");
  auto p = std::make_unique<ArrowToJsonProcessor>();
  if (const JsonValue* v = cfg.get("fields_to_include")) {
    if (v->kind == JsonValue::Array) {
      p->has_include = true;
      for (auto& e : v->arr) {
        if (e.kind != JsonValue::String) fail(ARK_ERR_SERIALIZATION, "invalid type in `fields_to_include`: expected a string");
        p->include.push_back(e.str);
      }
    } else if (v->kind != JsonValue::Null) fail(ARK_ERR_SERIALIZATION, "invalid type for `fields_to_include`: expected a sequence");
  }
  return p;
}

Batch arrow_to_json_device(const Processor& proc, Batch& in, cudaStream_t stream) {
  const auto& ap = static_cast<const ArrowToJsonProcessor&>(proc);
  const int64_t n = in.num_rows;
  AjParams P;
  memset(&P, 0, sizeof P);
  P.n_rows = n;
  for (auto& c : in.cols) {
    if (!c.present && c.field.format != "n") fail(ARK_ERR_UNSUPPORTED, "arrow_to_json: column '" + c.field.name + "' has Arrow type '" + c.field.format + "'");
    if (c.field.format == "n") continue;  // Null-typed column: never emitted
    if (ap.has_include && std::find(ap.include.begin(), ap.include.end(), c.field.name) == ap.include.end()) continue;  // filter_columns, lib.rs:304-328
    if (P.n_cols == AJ_MAX_COLS) fail(ARK_ERR_UNSUPPORTED, "arrow_to_json: more than 16 columns");
    const std::string key = json_escape_key(c.field.name);
    if ((int)key.size() > AJ_KEY_BYTES) fail(ARK_ERR_UNSUPPORTED, "arrow_to_json: column name too long");
    AjCol& a = P.cols[P.n_cols++];
    a.dtype = (int)c.field.type; a.key_len = (int)key.size();
    memcpy(a.key, key.data(), key.size());
    a.view = c.view();
  }
  if (ap.has_include && P.n_cols == 0 && n > 0) fail_filtered_to_no_columns();
  BufferPtr lens = device_alloc((size_t)(n + 1) * 4), offs = device_alloc((size_t)(n + 1) * 4);
  ARK_CUDA(cudaMemsetAsync(lens.get(), 0, (size_t)(n + 1) * 4, stream));
  const unsigned grid = (unsigned)std::max<int64_t>(1, ceil_div(n, 128));
  if (n) {
    KernelTimer t("arrow_to_json_measure_kernel", stream);
    arrow_to_json_measure_kernel<<<grid, 128, 0, stream>>>(P, (int32_t*)lens.get());
  }
  size_t tb = 0;
  cub::DeviceScan::ExclusiveSum(nullptr, tb, (int32_t*)lens.get(), (int32_t*)offs.get(), (int)(n + 1), stream);
  BufferPtr tmp = device_alloc(tb + 16);
  note_launch("cub::DeviceScan::ExclusiveSum");
  cub::DeviceScan::ExclusiveSum(tmp.get(), tb, (int32_t*)lens.get(), (int32_t*)offs.get(), (int)(n + 1), stream);
  BufferPtr h = pinned_alloc(64);
  ARK_CUDA(cudaMemcpyAsync(h.get(), (int32_t*)offs.get() + n, 4, cudaMemcpyDeviceToHost, stream));
  ARK_CUDA(cudaStreamSynchronize(stream));
  const int32_t total = *(int32_t*)h.get();
  if (total < 0) fail(ARK_ERR_PROCESS, "Arrow JSON Serialization error: output exceeds 2 GiB");
  BufferPtr bytes = device_alloc((size_t)total + 16);
  if (n) {
    KernelTimer t("arrow_to_json_write_kernel", stream);
    // staging window: the average CTA's bytes + 50 %; CTAs whose rows are longer take the direct path
    const int stage = (int)std::min<int64_t>(44 * 1024, round_up((int64_t)((double)total / (double)n * AJ_THREADS * 1.5) + 256, 1024));
    arrow_to_json_write_kernel<<<grid, AJ_THREADS, stage, stream>>>(P, (const int32_t*)offs.get(), (uint8_t*)bytes.get(), stage);
  }
  ARK_CUDA(cudaGetLastError());
  Batch out;
  out.num_rows = n; out.input_name = in.input_name;
  out.cols = in.cols;  // new_binary_with_origin: every original column, then __value__
  Column v;
  v.field.name = "__value__"; v.field.type = DType::Binary; v.field.nullable = false; v.field.format = "z";
  v.length = n;
  v.offsets = (const int32_t*)offs.get(); v.data = (const uint8_t*)bytes.get(); v.data_bytes = total; v.first_offset = 0;
  v.owners = {offs, bytes};
  out.cols.push_back(v);
  ARK_CUDA(cudaStreamSynchronize(stream));
  return out;
}

}  // namespace ark
