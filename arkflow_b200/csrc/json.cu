// json.cu — `json_to_arrow`: NDJSON payloads (a Binary column) → typed Arrow columns, on the device.
//
// Stands in for JsonToArrowProcessor::process (crates/arkflow-plugin/src/processor/json.rs:48-61) and
// component::json::try_to_arrow (crates/arkflow-plugin/src/component/json.rs:22-58), i.e. arrow-json
// 55.2's infer_json_schema(.., Some(1)) + tape decoder (third-party, not under /root/reference):
//   * the schema comes from the FIRST record only, fields in first-seen order, all nullable:
//     integer that fits i64 → Int64, other number → Float64, bool → Boolean, string → Utf8, null → Null;
//   * decoding is non-strict: unknown keys are skipped, missing keys → NULL;
//   * Int64 column: a number with fraction/exponent (or beyond i64) is parsed as f64 and truncated;
//     a quoted number is accepted for numeric columns; anything else is a decode error;
//   * Utf8 column: only JSON strings (escapes decoded); Boolean column: only true/false.
// The reference makes two full copies of the payload bytes around the decoder (json.rs:56,
// component/json.rs:54); here the payload bytes are read in place, once per pass.
//
// One thread parses one payload (a payload may hold several whitespace-separated records).
#include <cub/device/device_scan.cuh>

#include <algorithm>
#include <cmath>

#include "bitmap.cuh"
#include "bitmap.h"
#include "decoded.h"
#include "engine.h"
#include "stage_store.cuh"
#include "tma.cuh"
#include "json_mini.h"
#include "json_text.cuh"
#include "decimal.cuh"
#include "utf8.cuh"
#include "varlen.h"

namespace ark {

namespace {

constexpr int JS_MAX_FIELDS = 16;   // fields that travel in the kernel parameter block (constant bank); larger schemas use a table in HBM
constexpr int JS_MAX_NAME = 48;     // name bytes held inline; longer names are read through long_name
constexpr int JS_MAX_FIELDS_EXT = 64;  // the per-record `seen` mask is 64 bits wide
constexpr int JS_QUOTED_NUM_MAX = 128;  // decoded bytes of a quoted number written with escapes (parse_escaped_number)

// JE_STRING: a string that is not well-formed (escape, surrogate pairing or raw UTF-8), see strings_valid
enum JsonErr : int32_t { JE_NONE = 0, JE_SYNTAX = 1, JE_NOT_OBJECT = 2, JE_TYPE = 3, JE_NUMBER = 4, JE_STRING = 5 };

struct JsonField {
  int32_t dtype;     // DType as int
  int32_t name_len;
  char name[JS_MAX_NAME];
  void* values;            // Int64/Float64: 8 B per row; Boolean: byte per row
  uint8_t* valid_bytes;    // byte per row
  int32_t* str_len;        // Utf8: decoded length per row (pass A), later the offsets array
  long long* str_src;      // Utf8: absolute source position of the raw string body (after the quote)
  int32_t* str_raw_len;    // Utf8: raw (escaped) byte length; negative ⇒ contains escapes.  List / Struct: the value's raw span
                           // (str_src / str_raw_len), decoded by a second stage (json_list_* kernels / a nested parse pass)
  const char* long_name;   // name bytes in HBM when name_len > JS_MAX_NAME, else nullptr
};

struct JsonParams {
  const uint8_t* data;      // payload bytes base
  const int32_t* offsets;   // payload i = data[offsets[i] .. offsets[i+1])
  const uint8_t* validity;  // payload validity (NULL payloads are skipped: to_binary flattens them away)
  int32_t validity_bit0;
  int64_t n_payloads;
  int32_t n_fields;
  JsonField fields[JS_MAX_FIELDS];
  const JsonField* fields_ext; // the field table in HBM when n_fields > JS_MAX_FIELDS (else nullptr: `fields` is used)
  // nested pass: payload i is the span data[span_src[i] .. + span_len[i]) (the raw value of a Struct field) instead of
  // a row of the Binary column; a zero-length span (NULL / missing struct) yields a row of NULL children
  const long long* span_src;
  const int32_t* span_len;
  const long long* row_start;  // pass A: first output row of payload i
  int32_t* counts;             // count pass: records in payload i
  int32_t* error;              // [0] = JsonErr, [1] = payload index (first error wins), [2] = some payload does not hold exactly one record,
                               // [3] = some Int64 / Float64 row is a quoted number with escapes (valid_bytes 2, see json_quoted_numbers_kernel)
  int32_t stage_bytes;         // shared-memory staging window per CTA (0 = parse straight from global memory)
};

constexpr int JS_THREADS = 128;


struct Cursor {
  const uint8_t* p;
  const uint8_t* end;
  unsigned need = 0;  // bit 7: some string skip_string passed holds an escape or a byte >= 0x80 (see strings_valid)
};

__device__ __forceinline__ bool is_ws(unsigned ch) {  // ' ' \t \n \r: one range test + one bit test
  return ch <= 0x20u && ((0x100002600ull >> ch) & 1ull);
}
__device__ __forceinline__ void skip_ws(Cursor& c) {
  while (c.p < c.end && is_ws(*c.p)) ++c.p;
}

// Is the string body b[0..len) well-formed: every escape accepted by skip_escape, the raw bytes well-formed UTF-8 (an
// arrow-rs StringArray always holds valid UTF-8)?
__device__ __noinline__ bool body_valid(const uint8_t* b, int len) {
  const uint8_t* end = b + len;
  for (const uint8_t* p = b; p < end;) {
    if (*p != '\\') { ++p; continue; }
    p = skip_escape(p, end);
    if (!p) return false;
  }
  return utf8_valid(b, len);
}

// Cursor on the opening quote; leaves it after the closing quote.  Returns false when the string is unterminated or
// holds a raw control byte.  Every string the decoder reads passes through here — keys, values, skipped values and
// the spans the List / Struct stages decode again.  The scan is the plain one (an escape skips the byte after the
// backslash) and costs ASCII text nothing more: the common branch takes bytes above '\\' as signed chars, so a byte
// >= 0x80 falls through to the rarer branches, where it is noted like an escape.  A string with either sets bit 7 of
// c.need, and json_parse_kernel then checks that payload's strings once (strings_valid), out of line.
__device__ bool skip_string(Cursor& c, const uint8_t** body, int* raw_len, bool* has_escape) {
  ++c.p;
  const uint8_t* start = c.p;
  bool esc = false;
  unsigned other = 0;  // OR of the bytes off the common branch: bit 7 set <=> a byte >= 0x80
  while (c.p < c.end) {
    const uint8_t ch = *c.p;
    if ((int8_t)ch > '\\') { ++c.p; continue; }  // lower-case letters, '_', '{': the common case first
    if (ch == '"') {
      c.need |= other | (esc ? 0x80u : 0u);
      *body = start; *raw_len = (int)(c.p - start); *has_escape = esc; ++c.p;
      return true;
    }
    if (ch == '\\') { esc = true; c.p += 2; continue; }
    if (ch < 0x20) return false;
    other |= ch;
    ++c.p;
  }
  return false;
}

// Are the strings of the payload b[0..end) well-formed (body_valid)?  Called once per payload whose strings set bit 7
// of Cursor::need, after the payload parsed: its strings are terminated and nothing outside them is a quote or a byte
// >= 0x80.  A malformed string is JE_STRING wherever it stands — key, value, skipped value, inside a List or Struct
// span — so the List / Struct stages and json_strings_kernel only ever see well-formed bodies.
__device__ __noinline__ bool strings_valid(const uint8_t* b, const uint8_t* end) {
  while (b < end) {
    if (*b++ != '"') continue;
    const uint8_t* s = b;
    while (b < end && *b != '"') b += *b == '\\' ? 2 : 1;
    if (b > end) b = end;
    if (!body_valid(s, (int)(b - s))) return false;
    ++b;
  }
  return true;
}

__device__ bool skip_value(Cursor& c, int depth);

// Scans one JSON number.  When `fast` is given it also receives the value of a plain integer literal that fits
// i64 (no fraction, no exponent) — the digits are then read once instead of scanned and parsed again.
struct FastInt { bool ok; long long value; };
__device__ bool skip_number(Cursor& c, const uint8_t** start, int* len, FastInt* fast = nullptr) {
  *start = c.p;
  bool neg = false;
  if (c.p < c.end && *c.p == '-') { neg = true; ++c.p; }
  const uint8_t* d0 = c.p;
  unsigned long long acc = 0;
  bool plain = true;
  while (c.p < c.end && *c.p >= '0' && *c.p <= '9') {
    const unsigned d = *c.p - '0';
    if (acc > 922337203685477580ull) plain = false;  // acc * 10 + d could pass 2^63: leave it to parse_i64
    acc = acc * 10 + d;
    ++c.p;
  }
  if (c.p == d0) return false;
  if (c.p < c.end && *c.p == '.') { plain = false; ++c.p; const uint8_t* f0 = c.p; while (c.p < c.end && *c.p >= '0' && *c.p <= '9') ++c.p; if (c.p == f0) return false; }
  if (c.p < c.end && (*c.p == 'e' || *c.p == 'E')) {
    plain = false;
    ++c.p;
    if (c.p < c.end && (*c.p == '+' || *c.p == '-')) ++c.p;
    const uint8_t* e0 = c.p;
    while (c.p < c.end && *c.p >= '0' && *c.p <= '9') ++c.p;
    if (c.p == e0) return false;
  }
  *len = (int)(c.p - *start);
  if (fast) {
    fast->ok = plain && acc <= 0x7FFFFFFFFFFFFFFFull;
    fast->value = neg ? -(long long)acc : (long long)acc;
  }
  return true;
}

__device__ bool match_lit(Cursor& c, const char* lit, int n) {
  if (c.end - c.p < n) return false;
  for (int i = 0; i < n; ++i) if (c.p[i] != (uint8_t)lit[i]) return false;
  c.p += n;
  return true;
}

// iterative skip of any JSON value (nested containers tracked with a depth counter)
__device__ bool skip_value(Cursor& c, int) {
  skip_ws(c);
  if (c.p >= c.end) return false;
  int depth = 0;
  do {
    skip_ws(c);
    if (c.p >= c.end) return false;
    const uint8_t ch = *c.p;
    if (ch == '{' || ch == '[') { ++depth; ++c.p; }
    else if (ch == '}' || ch == ']') { --depth; ++c.p; }
    else if (ch == '"') { const uint8_t* b; int l; bool e; if (!skip_string(c, &b, &l, &e)) return false; }
    else if (ch == ',' || ch == ':') { ++c.p; }
    else if (ch == 't') { if (!match_lit(c, "true", 4)) return false; }
    else if (ch == 'f') { if (!match_lit(c, "false", 5)) return false; }
    else if (ch == 'n') { if (!match_lit(c, "null", 4)) return false; }
    else { const uint8_t* s; int l; if (!skip_number(c, &s, &l)) return false; }
  } while (depth > 0);
  return depth == 0;
}

// JSON number text (or the body of a quoted number) → f64, correctly rounded (decimal.cuh)
__device__ bool parse_f64(const uint8_t* s, int len, double* out) { return decimal_to_f64(s, len, out); }

// JSON number text → i64 as arrow-json's ParseJsonNumber does: integer parse, else f64 then NumCast.
__device__ bool parse_i64(const uint8_t* s, int len, long long* out) {
  int i = 0;
  bool neg = false;
  if (i < len && s[i] == '-') { neg = true; ++i; }
  else if (i < len && s[i] == '+') ++i;
  unsigned long long v = 0;
  bool ok = i < len, overflow = false;
  for (; i < len; ++i) {
    if (s[i] < '0' || s[i] > '9') { ok = false; break; }
    const unsigned d = s[i] - '0';
    // v * 10 + d > u64::MAX  ⇔  v > 1844674407370955161 or (v == 1844674407370955161 and d > 5)
    if (v > 1844674407370955161ull || (v == 1844674407370955161ull && d > 5)) { overflow = true; break; }
    v = v * 10 + d;
  }
  if (ok && !overflow) {
    if (!neg && v <= 0x7FFFFFFFFFFFFFFFull) { *out = (long long)v; return true; }
    if (neg && v <= 0x8000000000000000ull) { *out = (long long)(0 - v); return true; }
  }
  double d;
  if (!parse_f64(s, len, &d)) return false;
  if (!(d > -9223372036854777856.0 && d < 9223372036854775808.0)) return false;  // NumCast::from → None
  *out = (long long)d;
  return true;
}

// A quoted number written with escapes (a digit spelled as a u-escape): decoded, then parsed like any number body, as
// arrow-json decodes the string first.  Out of line: a cold branch the parse kernels' registers do not carry.  A
// decoded text longer than JS_QUOTED_NUM_MAX bytes is no number this decoder reads.
__device__ __noinline__ bool parse_escaped_number(const uint8_t* b, int raw, bool as_i64, void* out) {
  const int n = decoded_len(b, raw);
  if (n > JS_QUOTED_NUM_MAX) return false;
  uint8_t buf[JS_QUOTED_NUM_MAX];
  decode_string(b, raw, buf);
  return as_i64 ? parse_i64(buf, n, (long long*)out) : parse_f64(buf, n, (double*)out);
}

__device__ void raise(const JsonParams& P, int code, int64_t payload) {
  if (atomicCAS(P.error, 0, code) == 0) P.error[1] = (int32_t)payload;
}

// MODE 0: count records per payload.  MODE 1: parse into the columns (row_start from the count pass).
// MODE 2: optimistic single pass — payload i → row i; raises error[2] when a payload does not hold exactly
// one record (the host then reruns the batch through MODE 0 + MODE 1).
//
// The payloads of one CTA are contiguous in the Binary column, so their bytes arrive through ONE 1-D TMA
// bulk copy (cp.async.bulk → mbarrier) of the 16-byte-aligned window around them and every thread parses
// its payload from shared memory: 63-byte messages read byte by byte from global memory touch ~16 cache
// lines per warp instruction; from shared memory an odd stride is conflict-free.
// Nine CTAs per SM keep MODE 1 / 2 at 56 registers: left free, ptxas takes 64 and the SM holds one CTA fewer, which
// made the parse ~12 % slower on 63-byte messages (H100).
template <int MODE>
__global__ void __launch_bounds__(JS_THREADS, 9) json_parse_kernel(const __grid_constant__ JsonParams P) {
  extern __shared__ __align__(16) uint8_t js_stage[];
  __shared__ __align__(8) unsigned long long s_bar;
  __shared__ long long s_stage_off;  // payload-column byte offset of js_stage[0] (may be slightly negative)
  __shared__ int s_staged;
  const int64_t i0 = (int64_t)blockIdx.x * JS_THREADS;
  const int64_t i = i0 + threadIdx.x;
  if (threadIdx.x == 0) {
    s_staged = 0;
    if (P.stage_bytes > 0) {
      const int rows = (int)((P.n_payloads - i0) < JS_THREADS ? (P.n_payloads - i0) : JS_THREADS);
      const int32_t o0 = P.offsets[i0], o1 = P.offsets[i0 + rows];
      const uintptr_t a0 = reinterpret_cast<uintptr_t>(P.data + o0), a1 = reinterpret_cast<uintptr_t>(P.data + o1);
      const uintptr_t lo = a0 & ~(uintptr_t)15, hi = (a1 + 15) & ~(uintptr_t)15;
      if (o1 > o0 && hi - lo <= (uintptr_t)P.stage_bytes) {
        mbar_init(&s_bar, 1);
        mbar_fence_init();
        mbar_expect_tx(&s_bar, (unsigned)(hi - lo));
        tma_load_1d(js_stage, reinterpret_cast<const void*>(lo), (unsigned)(hi - lo), &s_bar);
        s_stage_off = (long long)o0 - (long long)(a0 - lo);
        s_staged = 1;
      }
    }
  }
  __syncthreads();
  const bool staged = s_staged != 0;
  const long long stage_off = staged ? s_stage_off : 0;
  if (staged) mbar_wait(&s_bar, 0);
  if (i >= P.n_payloads) return;
  if (P.validity && !bit_get(P.validity, i + P.validity_bit0)) {
    if (MODE == 0) P.counts[i] = 0;
    if (MODE == 2) P.error[2] = 1;
    return;
  }
  const JsonField* const FT = P.fields_ext ? P.fields_ext : P.fields;
  // `origin` + column byte offset = address of that byte (in the staging window or in global memory)
  const uint8_t* origin = staged ? js_stage - stage_off : P.data;
  Cursor c = P.span_src ? Cursor{P.data + P.span_src[i], P.data + P.span_src[i] + P.span_len[i]} : Cursor{origin + P.offsets[i], origin + P.offsets[i + 1]};
  int records = 0;
  long long row = MODE == 1 ? P.row_start[i] : (MODE == 2 ? (long long)i : 0);
  while (true) {
    skip_ws(c);
    if (c.p >= c.end) break;
    if (MODE == 2 && records == 1) { P.error[2] = 1; return; }  // a second record: not the one-row-per-payload shape
    if (*c.p != '{') { raise(P, *c.p == '[' || *c.p == '"' || (*c.p >= '0' && *c.p <= '9') || *c.p == '-' || *c.p == 't' || *c.p == 'f' || *c.p == 'n' ? JE_NOT_OBJECT : JE_SYNTAX, i); return; }
    if (MODE == 0) {
      if (!skip_value(c, 0)) { raise(P, JE_SYNTAX, i); return; }
      ++records;
      continue;
    }
    // ---- MODE 1: one object → one row ----
    ++c.p;
    unsigned long long seen = 0;
    int next_field = 0;
    skip_ws(c);
    bool first = true;
    while (true) {
      skip_ws(c);
      if (c.p >= c.end) { raise(P, JE_SYNTAX, i); return; }
      if (*c.p == '}') { ++c.p; break; }
      if (!first) { if (*c.p != ',') { raise(P, JE_SYNTAX, i); return; } ++c.p; skip_ws(c); }
      first = false;
      if (c.p >= c.end || *c.p != '"') { raise(P, JE_SYNTAX, i); return; }
      const uint8_t* kb; int kl; bool kesc;
      if (!skip_string(c, &kb, &kl, &kesc)) { raise(P, JE_SYNTAX, i); return; }
      skip_ws(c);
      if (c.p >= c.end || *c.p != ':') { raise(P, JE_SYNTAX, i); return; }
      ++c.p;
      skip_ws(c);
      int f = -1;
      if (!kesc) {
        // records usually list their keys in the order of the first record: try that position first
        for (int t = 0, k = next_field; t < P.n_fields; ++t, k = (k + 1 == P.n_fields ? 0 : k + 1)) {
          if (FT[k].name_len != kl) continue;
          const char* nm = FT[k].long_name ? FT[k].long_name : FT[k].name;
          bool eq = true;
          for (int b = 0; b < kl; ++b) if ((uint8_t)nm[b] != kb[b]) { eq = false; break; }
          if (eq) { f = k; break; }
        }
        if (f >= 0) next_field = f + 1 == P.n_fields ? 0 : f + 1;
      } else {  // a key written with escapes ("val\u0075e"): compared after decoding, as arrow-json's tape decoder does
        for (int k = 0; k < P.n_fields; ++k) {
          const char* nm = FT[k].long_name ? FT[k].long_name : FT[k].name;
          if (decoded_equals(kb, kl, nm, FT[k].name_len)) { f = k; break; }
        }
      }
      if (f < 0) { if (!skip_value(c, 0)) { raise(P, JE_SYNTAX, i); return; } continue; }
      const JsonField& F = FT[f];
      if (c.p >= c.end) { raise(P, JE_SYNTAX, i); return; }
      const uint8_t ch = *c.p;
      if (ch == 'n') {  // null
        if (!match_lit(c, "null", 4)) { raise(P, JE_SYNTAX, i); return; }
        F.valid_bytes[row] = 0; seen |= 1ull << f;
        if (F.dtype == (int)DType::Utf8) { F.str_len[row] = 0; F.str_raw_len[row] = 0; }
        if (F.dtype == (int)DType::List || F.dtype == (int)DType::Struct) F.str_raw_len[row] = 0;
        continue;
      }
      switch ((DType)F.dtype) {
        case DType::Int64: case DType::Float64: {
          const uint8_t* ns; int nl;
          FastInt fi{false, 0};
          bool nesc = false;
          if (ch == '"') { if (!skip_string(c, &ns, &nl, &nesc)) { raise(P, JE_SYNTAX, i); return; } }
          else if (ch == '-' || (ch >= '0' && ch <= '9')) { if (!skip_number(c, &ns, &nl, &fi)) { raise(P, JE_SYNTAX, i); return; } }
          else { raise(P, JE_TYPE, i); return; }
          if (nesc) {  // rare: json_quoted_numbers_kernel decodes and parses it, so this kernel carries no call for it
            if (nl > 0xFFFF) { raise(P, JE_NUMBER, i); return; }  // decodes to far more than JS_QUOTED_NUM_MAX bytes
            ((long long*)F.values)[row] = (long long)(ns - origin) << 16 | nl;
            F.valid_bytes[row] = 2; seen |= 1ull << f; P.error[3] = 1;
            continue;
          }
          if ((DType)F.dtype == DType::Int64) {
            long long v = fi.value;
            if (!fi.ok && !parse_i64(ns, nl, &v)) { raise(P, JE_NUMBER, i); return; }
            ((long long*)F.values)[row] = v;
          } else {
            double v;
            if (!parse_f64(ns, nl, &v)) { raise(P, JE_NUMBER, i); return; }
            ((double*)F.values)[row] = v;
          }
          break;
        }
        case DType::Bool: {
          if (ch == 't') { if (!match_lit(c, "true", 4)) { raise(P, JE_SYNTAX, i); return; } ((uint8_t*)F.values)[row] = 1; }
          else if (ch == 'f') { if (!match_lit(c, "false", 5)) { raise(P, JE_SYNTAX, i); return; } ((uint8_t*)F.values)[row] = 0; }
          else { raise(P, JE_TYPE, i); return; }
          break;
        }
        case DType::Utf8: {
          if (ch != '"') { raise(P, JE_TYPE, i); return; }
          const uint8_t* sb; int sl; bool esc;
          if (!skip_string(c, &sb, &sl, &esc)) { raise(P, JE_SYNTAX, i); return; }
          F.str_len[row] = esc ? decoded_len(sb, sl) : sl; F.str_src[row] = (long long)(sb - origin); F.str_raw_len[row] = esc ? -sl : sl;
          break;
        }
        case DType::List: case DType::Struct: {  // the raw span of the value; its elements / fields are decoded by a second stage
          if (ch != ((DType)F.dtype == DType::List ? '[' : '{')) { raise(P, JE_TYPE, i); return; }
          const uint8_t* v0 = c.p;
          if (!skip_value(c, 0)) { raise(P, JE_SYNTAX, i); return; }
          F.str_src[row] = (long long)(v0 - origin); F.str_raw_len[row] = (int)(c.p - v0);
          break;
        }
        default:  // Null-typed column: any non-null value is a type error in arrow-json's NullArrayDecoder
          raise(P, JE_TYPE, i); return;
      }
      F.valid_bytes[row] = 1; seen |= 1ull << f;
    }
    for (int k = 0; k < P.n_fields; ++k) {
      if (!((seen >> k) & 1)) {  // missing key → NULL
        FT[k].valid_bytes[row] = 0;
        if (FT[k].dtype == (int)DType::Utf8) { FT[k].str_len[row] = 0; FT[k].str_raw_len[row] = 0; }
        if (FT[k].dtype == (int)DType::List || FT[k].dtype == (int)DType::Struct) FT[k].str_raw_len[row] = 0;
      }
    }
    ++row; ++records;
  }
  if (c.need & 0x80) {  // the payload's start is read again rather than kept in a register through the parse
    const uint8_t* c0 = P.span_src ? P.data + P.span_src[i] : origin + P.offsets[i];
    if (!strings_valid(c0, c.end)) { raise(P, JE_STRING, i); return; }
  }
  if (MODE == 0) P.counts[i] = records;
  if (MODE == 2 && records != 1) {
    if (P.span_src && records == 0) {  // nested pass, NULL / missing struct: a row of NULL children
      for (int k = 0; k < P.n_fields; ++k) {
        FT[k].valid_bytes[i] = 0;
        if (FT[k].dtype == (int)DType::Utf8) { FT[k].str_len[i] = 0; FT[k].str_raw_len[i] = 0; }
      }
    } else P.error[2] = 1;  // blank payload: no row
  }
}

// ---- List<primitive> columns: second stage over the raw spans captured by the parse pass -------------------------
// counts[row] = number of elements of the array at data[src[row] .. + raw[row]) (0 for NULL rows)
__global__ void json_list_count_kernel(const uint8_t* data, const long long* src, const int32_t* raw, int64_t n, int32_t* counts, int32_t* error) {
  const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n) return;
  int cnt = 0;
  if (raw[r] > 0) {
    Cursor c{data + src[r] + 1, data + src[r] + raw[r]};  // past '['
    skip_ws(c);
    if (c.p < c.end && *c.p != ']') {
      while (true) {
        if (!skip_value(c, 0)) { if (atomicCAS(error, 0, JE_SYNTAX) == 0) error[1] = (int32_t)r; break; }
        ++cnt;
        skip_ws(c);
        if (c.p < c.end && *c.p == ',') { ++c.p; continue; }
        break;
      }
    }
  }
  counts[r] = cnt;
}

// elements of row r go to child positions offsets[r] ..; same scalar rules as the top-level decoder
__global__ void json_list_fill_kernel(const uint8_t* data, const long long* src, const int32_t* raw, int64_t n, const int32_t* offsets, int elem_dtype,
                                      void* values, uint8_t* valid, int32_t* str_len, long long* str_src, int32_t* str_raw, int32_t* error) {
  const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n || raw[r] <= 0) return;
  Cursor c{data + src[r] + 1, data + src[r] + raw[r]};
  long long e = offsets[r];
  const long long e_end = offsets[r + 1];
  auto bad = [&](int code) { if (atomicCAS(error, 0, code) == 0) error[1] = (int32_t)r; };
  while (e < e_end) {
    skip_ws(c);
    if (c.p >= c.end) { bad(JE_SYNTAX); return; }
    const uint8_t ch = *c.p;
    if (ch == 'n') {
      if (!match_lit(c, "null", 4)) { bad(JE_SYNTAX); return; }
      valid[e] = 0;
      if (elem_dtype == (int)DType::Utf8) { str_len[e] = 0; str_raw[e] = 0; }
    } else {
      switch ((DType)elem_dtype) {
        case DType::Int64: case DType::Float64: {
          const uint8_t* ns; int nl;
          FastInt fi{false, 0};
          bool nesc = false;
          if (ch == '"') { if (!skip_string(c, &ns, &nl, &nesc)) { bad(JE_SYNTAX); return; } }
          else if (ch == '-' || (ch >= '0' && ch <= '9')) { if (!skip_number(c, &ns, &nl, &fi)) { bad(JE_SYNTAX); return; } }
          else { bad(JE_TYPE); return; }
          if (nesc) {
            if (!parse_escaped_number(ns, nl, (DType)elem_dtype == DType::Int64, (uint8_t*)values + e * 8)) { bad(JE_NUMBER); return; }
          } else if ((DType)elem_dtype == DType::Int64) {
            long long v = fi.value;
            if (!fi.ok && !parse_i64(ns, nl, &v)) { bad(JE_NUMBER); return; }
            ((long long*)values)[e] = v;
          } else {
            double v;
            if (!parse_f64(ns, nl, &v)) { bad(JE_NUMBER); return; }
            ((double*)values)[e] = v;
          }
          break;
        }
        case DType::Bool: {
          if (ch == 't') { if (!match_lit(c, "true", 4)) { bad(JE_SYNTAX); return; } ((uint8_t*)values)[e] = 1; }
          else if (ch == 'f') { if (!match_lit(c, "false", 5)) { bad(JE_SYNTAX); return; } ((uint8_t*)values)[e] = 0; }
          else { bad(JE_TYPE); return; }
          break;
        }
        case DType::Utf8: {
          if (ch != '"') { bad(JE_TYPE); return; }
          const uint8_t* sb; int sl; bool esc;
          if (!skip_string(c, &sb, &sl, &esc)) { bad(JE_SYNTAX); return; }
          str_len[e] = esc ? decoded_len(sb, sl) : sl;  // the parse pass checked the span's strings
          str_src[e] = (long long)(sb - data); str_raw[e] = esc ? -sl : sl;
          break;
        }
        default: bad(JE_TYPE); return;  // List<Null>: only nulls
      }
      valid[e] = 1;
    }
    ++e;
    skip_ws(c);
    if (c.p < c.end && *c.p == ',') ++c.p;
  }
}

// Rows of one Int64 / Float64 column whose value was a quoted number with escapes: the parse kernel left valid_bytes 2
// and values = (column byte offset of the body << 16 | raw length).  Decoded and parsed here; thread per row.
__global__ void json_quoted_numbers_kernel(const uint8_t* data, int64_t n, bool as_i64, long long* values, uint8_t* valid, int32_t* error) {
  const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n || valid[r] != 2) return;
  const long long span = values[r];
  if (!parse_escaped_number(data + (span >> 16), (int)(span & 0xFFFF), as_i64, values + r)) {
    if (atomicCAS(error, 0, JE_NUMBER) == 0) error[1] = (int32_t)r;
    return;
  }
  valid[r] = 1;
}

// string bytes of one Utf8 column: thread per row
__global__ void json_strings_kernel(const uint8_t* data, const long long* src, const int32_t* raw_len, const int32_t* offsets,
                                    int64_t n_rows, uint8_t* out) {
  const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n_rows) return;
  const int raw = raw_len[r];
  if (raw == 0) return;
  uint8_t* d = out + offsets[r];
  const uint8_t* s = data + src[r];
  if (raw > 0) { for (int i = 0; i < raw; ++i) d[i] = s[i]; }
  else decode_string(s, -raw, d);
}

__global__ void i32_to_i64_kernel(const int32_t* in, long long* out, int64_t n) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = in[i];
}

}  // namespace

void launch_json_strings(const uint8_t* data, const StagedColumn& s, uint8_t* bytes, cudaStream_t stream) {
  if (!s.rows) return;
  KernelTimer t("json_strings_kernel", stream);
  json_strings_kernel<<<(unsigned)ceil_div(s.rows, 256), 256, 0, stream>>>(data, (const long long*)s.src.get(), (const int32_t*)s.raw.get(),
                                                                           (const int32_t*)s.offsets.get(), s.rows, bytes);
}

// One column of the inferred schema.  List: `elem` is the element type; Struct: `kids` are its (scalar) fields.
// Deeper nesting (arrays of arrays / of objects, objects inside objects) is outside the GPU subset → `supported` false.
struct InferredField {
  std::string name;
  DType type = DType::Null;
  DType elem = DType::Null;
  std::vector<InferredField> kids;
  bool supported = true;
  std::string why;
};

namespace {

// arrow-json's type of one JSON value (infer_json_schema): scalars as documented in SURVEY.md §8(c); an array's element
// type is the coercion of its elements' types (Int64 + Float64 → Float64, X + Null → X, [] → List<Null>).
InferredField infer_value(const std::string& name, const JsonValue& v, int depth) {
  InferredField f;
  f.name = name;
  switch (v.kind) {
    case JsonValue::Null: f.type = DType::Null; break;
    case JsonValue::Bool: f.type = DType::Bool; break;
    case JsonValue::Number: f.type = v.is_int ? DType::Int64 : DType::Float64; break;
    case JsonValue::String: f.type = DType::Utf8; break;
    case JsonValue::Array: {
      f.type = DType::List;
      if (depth > 0) { f.supported = false; f.why = "List inside a nested value"; break; }
      DType t = DType::Null;
      for (auto& e : v.arr) {
        if (e.kind == JsonValue::Array || e.kind == JsonValue::Object) { f.supported = false; f.why = "List of nested values"; break; }
        const DType et = e.kind == JsonValue::Null ? DType::Null : e.kind == JsonValue::Bool ? DType::Bool
                         : e.kind == JsonValue::Number ? (e.is_int ? DType::Int64 : DType::Float64) : DType::Utf8;
        if (t == DType::Null) t = et;
        else if (et == DType::Null || et == t) {}
        else if ((t == DType::Int64 && et == DType::Float64) || (t == DType::Float64 && et == DType::Int64)) t = DType::Float64;
        else { f.supported = false; f.why = "List of mixed types"; break; }
      }
      f.elem = t;
      break;
    }
    case JsonValue::Object: {
      f.type = DType::Struct;
      if (depth > 0) { f.supported = false; f.why = "Struct inside a nested value"; break; }
      for (auto& kv : v.obj) {
        bool dup = false;
        for (auto& k : f.kids) if (k.name == kv.first) dup = true;
        if (dup) continue;
        InferredField k = infer_value(kv.first, kv.second, depth + 1);
        if (!k.supported) { f.supported = false; f.why = k.why; }
        f.kids.push_back(std::move(k));
      }
      break;
    }
  }
  return f;
}

// arrow-json infer_json_schema over the first record (host side; the record is a few dozen bytes)
std::vector<InferredField> infer_schema(const std::string& first_record) {
  JsonValue v;
  try {
    // the first payload may hold several records: parse only the first value
    std::string s = first_record;
    // find the end of the first top-level value by bracket matching
    int depth = 0; bool in_str = false; size_t end = std::string::npos;
    for (size_t i = 0; i < s.size(); ++i) {
      char ch = s[i];
      if (in_str) { if (ch == '\\') ++i; else if (ch == '"') in_str = false; continue; }
      if (ch == '"') in_str = true;
      else if (ch == '{' || ch == '[') ++depth;
      else if (ch == '}' || ch == ']') { if (--depth == 0) { end = i + 1; break; } }
      else if (depth == 0 && !isspace((unsigned char)ch)) break;
    }
    if (end == std::string::npos) fail(ARK_ERR_PROCESS, "Schema inference error: Json error: Expected JSON record to be an object");
    if (!utf8_valid((const uint8_t*)s.data(), (long long)end)) fail(ARK_ERR_PROCESS, "Schema inference error: Json error: invalid UTF-8");
    v = parse_json(s.substr(0, end));
  } catch (const ArkError& e) {
    if (e.code == ARK_ERR_SERIALIZATION) fail(ARK_ERR_PROCESS, std::string("Schema inference error: Json error: ") + e.what());
    throw;
  }
  if (v.kind != JsonValue::Object)
    fail(ARK_ERR_PROCESS, "Schema inference error: Json error: Expected JSON record to be an object, found " +
                              std::string(v.kind == JsonValue::Array ? "Array" : "a scalar"));
  std::vector<InferredField> out;
  for (auto& kv : v.obj) {
    bool dup = false;
    for (auto& f : out) if (f.name == kv.first) dup = true;
    if (dup) continue;
    out.push_back(infer_value(kv.first, kv.second, 0));
  }
  return out;
}

// coerce_data_type of arrow-json's schema inference over several records: X + Null → X, Int64 + Float64 → Float64,
// equal types stay, anything else → Utf8; nested types must agree (their element / child types are merged the same way)
void merge_field(InferredField& into, const InferredField& f) {
  if (!f.supported) { into.supported = false; into.why = f.why; }
  if (f.type == DType::Null) return;
  if (into.type == DType::Null) { const std::string n = into.name; const bool sup = into.supported; const std::string why = into.why; into = f; into.name = n; if (!sup) { into.supported = false; into.why = why; } return; }
  if (into.type == f.type) {
    if (f.type == DType::List) {
      if (into.elem == DType::Null) into.elem = f.elem;
      else if (f.elem == DType::Null || f.elem == into.elem) {}
      else if ((into.elem == DType::Int64 && f.elem == DType::Float64) || (into.elem == DType::Float64 && f.elem == DType::Int64)) into.elem = DType::Float64;
      else into.elem = DType::Utf8;
    } else if (f.type == DType::Struct) {
      for (auto& k : f.kids) {
        bool found = false;
        for (auto& mine : into.kids) if (mine.name == k.name) { merge_field(mine, k); found = true; }
        if (!found) into.kids.push_back(k);
      }
    }
    return;
  }
  if ((into.type == DType::Int64 && f.type == DType::Float64) || (into.type == DType::Float64 && f.type == DType::Int64)) { into.type = DType::Float64; return; }
  if (into.type == DType::List || into.type == DType::Struct || f.type == DType::List || f.type == DType::Struct) { into.supported = false; into.why = "nested and scalar values under one key"; return; }
  into.type = DType::Utf8;
}

const char* json_err_text(int code) {
  switch (code) {
    case JE_NOT_OBJECT: return "Arrow JSON Reader Error: Json error: expected { got a non-object value";
    case JE_TYPE: return "Arrow JSON Reader Error: Json error: whilst decoding field: value does not match the inferred column type";
    case JE_NUMBER: return "Arrow JSON Reader Error: Json error: failed to parse number";
    case JE_STRING: return "Arrow JSON Reader Error: Json error: invalid string: a malformed escape, an unpaired surrogate or invalid UTF-8";
    default: return "Arrow JSON Reader Error: Json error: Encountered unexpected token / truncated record";
  }
}

[[noreturn]] void raise_json(int code, int where, const char* what) {
  fail(ARK_ERR_PROCESS, std::string(json_err_text(code)) + " (" + what + " " + std::to_string(where) + ")");
}

// A column of `rows` rows for the parse or List fill kernel.  `data_bytes`, the bytes of the input Binary column, bounds a
// Utf8 column: a decoded string is never longer than its raw span there.
StagedColumn stage_json(const std::string& name, DType type, int64_t rows, int64_t data_bytes, cudaStream_t stream) {
  StagedColumn s = stage_column(type, rows, true, true, stream);
  s.bound = data_bytes;
  s.what = "json_to_arrow: column '" + name + "'";
  return s;
}

// The Column of a settled scalar or Null column; `data` is the byte base its str_src refers to.
Column json_column(const std::string& name, const StagedColumn& s, const uint8_t* data, cudaStream_t stream) {
  return finish_column(s, Field{name, s.type, true, s.type == DType::Null ? "n" : ""},
                       [&](const StagedColumn& s, uint8_t* bytes) { launch_json_strings(data, s, bytes, stream); }, stream);
}

// List<primitive> column from the raw spans of the rows of the settled `s` (s.src / s.raw)
Column finish_list(const InferredField& f, const StagedColumn& s, const uint8_t* data, int64_t data_bytes, cudaStream_t stream) {
  const int64_t rows = s.rows;
  BufferPtr err = device_alloc(16), h = pinned_alloc(32);
  ARK_CUDA(cudaMemsetAsync(err.get(), 0, 16, stream));
  BufferPtr counts = device_alloc((size_t)(rows + 1) * 4);
  ARK_CUDA(cudaMemsetAsync((int32_t*)counts.get() + rows, 0, 4, stream));
  const unsigned g = (unsigned)std::max<int64_t>(1, ceil_div(rows, 128));
  if (rows) {
    KernelTimer t("json_list_count_kernel", stream);
    json_list_count_kernel<<<g, 128, 0, stream>>>(data, (const long long*)s.src.get(), (const int32_t*)s.raw.get(), rows, (int32_t*)counts.get(), (int32_t*)err.get());
  }
  // every element takes at least one byte of its row's raw span inside the input column
  varlen_guard((const int32_t*)counts.get(), rows, data_bytes, "json_to_arrow: column '" + f.name + "'", stream);
  BufferPtr offs = varlen_scan((const int32_t*)counts.get(), rows, stream);
  ARK_CUDA(cudaMemcpyAsync(h.get(), (int32_t*)offs.get() + rows, 4, cudaMemcpyDeviceToHost, stream));
  ARK_CUDA(cudaMemcpyAsync((char*)h.get() + 8, err.get(), 8, cudaMemcpyDeviceToHost, stream));
  ARK_CUDA(cudaStreamSynchronize(stream));
  if (((int32_t*)((char*)h.get() + 8))[0]) raise_json(((int32_t*)((char*)h.get() + 8))[0], ((int32_t*)((char*)h.get() + 8))[1], "row");
  const int64_t total = *(const int32_t*)h.get();
  std::vector<StagedColumn> item = {stage_json("item", f.elem, total, data_bytes, stream)};  // arrow-rs names a list's field "item"
  const StagedColumn& e = item[0];
  if (rows && total) {
    KernelTimer t("json_list_fill_kernel", stream);
    json_list_fill_kernel<<<g, 128, 0, stream>>>(data, (const long long*)s.src.get(), (const int32_t*)s.raw.get(), rows, (const int32_t*)offs.get(), (int)f.elem,
                                                 e.values.get(), (uint8_t*)e.valid.get(), (int32_t*)e.len.get(), (long long*)e.src.get(), (int32_t*)e.raw.get(),
                                                 (int32_t*)err.get());
  }
  settle_columns(item, err.get(), 8, [](const void* h) {
    const int32_t* e = (const int32_t*)h;
    if (e[0]) raise_json(e[0], e[1], "row");
  }, stream);
  Column c;
  c.field.name = f.name; c.field.type = DType::List; c.field.format = "+l"; c.field.nullable = true; c.length = rows;
  set_validity(c, s.bits, s.null_count);
  c.offsets = (const int32_t*)offs.get(); c.first_offset = 0;
  c.owners.push_back(offs);
  c.children.push_back(json_column("item", e, data, stream));
  return c;
}

}  // namespace

struct JsonToArrowProcessor : Processor {
  const char* type() const override { return "json_to_arrow"; }
  std::string value_field = "__value__";  // DEFAULT_BINARY_VALUE_FIELD, core/lib.rs:46
  bool has_include = false;
  std::vector<std::string> include;
  // the `file` input fixes the schema once per file (DataFusion infers it from the first 1000 records at connect time)
  bool has_fixed_schema = false;
  std::vector<InferredField> fixed_schema;
};

// A decoder whose schema is the merge of `sample` (one JSON record per string): what DataFusion's NDJSON reader does
// with schema_infer_max_records = 1000 (crates/arkflow-plugin/src/input/file.rs:218-228 → ctx.read_json).
std::unique_ptr<Processor> make_json_to_arrow_for_sample(const std::vector<std::string>& sample) {
  auto p = std::make_unique<JsonToArrowProcessor>();
  p->has_fixed_schema = true;
  for (auto& rec : sample) {
    bool blank = true;
    for (char ch : rec) if (!isspace((unsigned char)ch)) blank = false;
    if (blank) continue;
    std::vector<InferredField> one = infer_schema(rec);
    for (auto& f : one) {
      bool found = false;
      for (auto& mine : p->fixed_schema) if (mine.name == f.name) { merge_field(mine, f); found = true; }
      if (!found) p->fixed_schema.push_back(f);
    }
  }
  return p;
}

std::unique_ptr<Processor> make_json_to_arrow(const char* config_json) {
  // reference: json.rs:124-128 (missing configuration)
  if (!config_json) fail(ARK_ERR_CONFIG, "JsonToArrow processor configuration is missing");
  JsonValue cfg = parse_json(config_json);
  if (cfg.kind == JsonValue::Null) fail(ARK_ERR_CONFIG, "JsonToArrow processor configuration is missing");
  if (cfg.kind != JsonValue::Object) fail(ARK_ERR_SERIALIZATION, "invalid type: expected struct JsonProcessorConfig");
  auto p = std::make_unique<JsonToArrowProcessor>();
  if (const JsonValue* v = cfg.get("value_field")) {
    if (v->kind == JsonValue::String) p->value_field = v->str;
    else if (v->kind != JsonValue::Null) fail(ARK_ERR_SERIALIZATION, "invalid type for `value_field`: expected a string");
  }
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

const std::string& json_to_arrow_value_field(const Processor& p) { return static_cast<const JsonToArrowProcessor&>(p).value_field; }

namespace {

// Decodes `specs` into `rows` rows.  The payloads are rows of a Binary column (P.offsets) or raw spans (P.span_src).
// optimistic: payload i → row i in ONE pass; returns false (nothing raised) when the batch is not of that shape or
// holds an error — the caller then takes the two-pass route, which reports errors the canonical way.
bool decode_fields(const std::vector<InferredField>& specs, JsonParams Q, unsigned grid, size_t smem, int64_t rows, bool optimistic,
                   const long long* row_start, const uint8_t* data, int64_t data_bytes, std::vector<Column>& out_cols, cudaStream_t stream) {
  const size_t nf = specs.size();
  std::vector<StagedColumn> cols;
  std::vector<JsonField> table(nf);
  // names longer than the inline slot live in one HBM pool
  std::string pool;
  std::vector<size_t> pool_off(nf, 0);
  for (size_t k = 0; k < nf; ++k) if ((int)specs[k].name.size() > JS_MAX_NAME) { pool_off[k] = pool.size(); pool += specs[k].name; }
  BufferPtr names_dev;
  if (!pool.empty()) {
    names_dev = device_alloc(pool.size());
    ARK_CUDA(cudaMemcpyAsync(names_dev.get(), pool.data(), pool.size(), cudaMemcpyHostToDevice, stream));
  }
  for (size_t k = 0; k < nf; ++k) {
    JsonField& F = table[k];
    memset(&F, 0, sizeof F);
    F.dtype = (int)specs[k].type; F.name_len = (int)specs[k].name.size();
    if ((int)specs[k].name.size() > JS_MAX_NAME) F.long_name = (const char*)names_dev.get() + pool_off[k];
    else memcpy(F.name, specs[k].name.data(), specs[k].name.size());
    cols.push_back(stage_json(specs[k].name, specs[k].type, rows, data_bytes, stream));
    const StagedColumn& s = cols.back();
    F.values = s.values.get(); F.valid_bytes = (uint8_t*)s.valid.get();
    F.str_len = (int32_t*)s.len.get(); F.str_src = (long long*)s.src.get(); F.str_raw_len = (int32_t*)s.raw.get();
  }
  Q.n_fields = (int)nf;
  Q.row_start = row_start;
  BufferPtr table_dev;
  if (nf > (size_t)JS_MAX_FIELDS) {
    table_dev = device_alloc(nf * sizeof(JsonField));
    ARK_CUDA(cudaMemcpyAsync(table_dev.get(), table.data(), nf * sizeof(JsonField), cudaMemcpyHostToDevice, stream));
    ARK_CUDA(cudaStreamSynchronize(stream));  // `table` / `pool` are host temporaries
    Q.fields_ext = (const JsonField*)table_dev.get();
  } else {
    for (size_t k = 0; k < nf; ++k) Q.fields[k] = table[k];
    Q.fields_ext = nullptr;
    if (!pool.empty()) ARK_CUDA(cudaStreamSynchronize(stream));
  }
  BufferPtr err = device_alloc(16), h = pinned_alloc(32);
  Q.error = (int32_t*)err.get();
  ARK_CUDA(cudaMemsetAsync(err.get(), 0, 16, stream));
  {
    KernelTimer t("json_parse_kernel", stream);
    if (optimistic) json_parse_kernel<2><<<grid, JS_THREADS, smem, stream>>>(Q);
    else json_parse_kernel<1><<<grid, JS_THREADS, smem, stream>>>(Q);
  }
  ARK_CUDA(cudaGetLastError());
  ARK_CUDA(cudaMemcpyAsync(h.get(), err.get(), 16, cudaMemcpyDeviceToHost, stream));
  ARK_CUDA(cudaStreamSynchronize(stream));
  const int32_t* e = (const int32_t*)h.get();
  if (optimistic && (e[0] != JE_NONE || e[2])) return false;
  if (e[0] != JE_NONE) raise_json(e[0], e[1], Q.span_src ? "row" : "payload");
  if (e[3]) {  // quoted numbers written with escapes
    ARK_CUDA(cudaMemsetAsync(err.get(), 0, 16, stream));
    for (size_t k = 0; k < nf; ++k) {
      if (specs[k].type != DType::Int64 && specs[k].type != DType::Float64) continue;
      KernelTimer t("json_quoted_numbers_kernel", stream);
      json_quoted_numbers_kernel<<<(unsigned)ceil_div(rows, 256), 256, 0, stream>>>(data, rows, specs[k].type == DType::Int64, (long long*)table[k].values,
                                                                                   table[k].valid_bytes, (int32_t*)err.get());
    }
    ARK_CUDA(cudaMemcpyAsync(h.get(), err.get(), 16, cudaMemcpyDeviceToHost, stream));
    ARK_CUDA(cudaStreamSynchronize(stream));
    if (e[0] != JE_NONE) raise_json(e[0], e[1], "row");
  }
  // every scalar column of the level and the validity of its List / Struct columns come back in one round trip
  settle_columns(cols, nullptr, 0, nullptr, stream);
  out_cols.clear();
  for (size_t k = 0; k < nf; ++k) {
    const InferredField& f = specs[k];
    if (f.type == DType::List) out_cols.push_back(finish_list(f, cols[k], data, data_bytes, stream));
    else if (f.type == DType::Struct) {
      // the struct's children: the same decoder over the captured spans, one row per span
      JsonParams S;
      memset(&S, 0, sizeof S);
      S.data = data; S.n_payloads = rows; S.stage_bytes = 0;
      S.span_src = (const long long*)cols[k].src.get(); S.span_len = (const int32_t*)cols[k].raw.get();
      std::vector<Column> kids;
      if (rows > 0 && !f.kids.empty()) {
        if (!decode_fields(f.kids, S, (unsigned)ceil_div(rows, JS_THREADS), 32, rows, true, nullptr, data, data_bytes, kids, stream))
          decode_fields(f.kids, S, (unsigned)ceil_div(rows, JS_THREADS), 32, rows, false, nullptr, data, data_bytes, kids, stream);  // raises the canonical error
      } else {
        for (auto& kf : f.kids) { Column kc; kc.field.name = kf.name; kc.field.type = kf.type; kc.field.nullable = true; kc.length = rows; if (kf.type == DType::Null) kc.field.format = "n"; kids.push_back(kc); }
      }
      Column c;
      c.field.name = f.name; c.field.type = DType::Struct; c.field.format = "+s"; c.field.nullable = true; c.length = rows;
      set_validity(c, cols[k].bits, cols[k].null_count);
      c.children = std::move(kids);
      out_cols.push_back(std::move(c));
    } else out_cols.push_back(json_column(f.name, cols[k], data, stream));
  }
  ARK_CUDA(cudaGetLastError());
  ARK_CUDA(cudaStreamSynchronize(stream));
  return true;
}

}  // namespace

// `in` holds the payload column (device-resident).
Batch json_to_arrow_device(const Processor& proc, Batch& in, cudaStream_t stream) {
  const auto& jp = static_cast<const JsonToArrowProcessor&>(proc);
  const int ci = in.find(jp.value_field);
  if (ci < 0) fail(ARK_ERR_PROCESS, "not found column");                                  // core/lib.rs:357-359
  Column& col = in.cols[ci];
  if (col.field.format != "z" || !col.present) fail(ARK_ERR_PROCESS, "not support data type");  // core/lib.rs:363-367
  std::vector<int> vl = {ci};
  resolve_varlen_extents(in, vl, stream);
  const int64_t n = col.length;
  Batch out;
  out.input_name = in.input_name;
  if (n == 0 || col.data_bytes == 0) return out;  // empty input → RecordBatch::new_empty(inferred = empty schema)

  // ---- schema from the first non-null, non-blank payload (host side; offsets fetched 256 at a time) ----
  std::string first;
  {
    constexpr int64_t CH = 256;
    BufferPtr hoff = pinned_alloc((size_t)(CH + 1) * 4 + CH / 8 + 16);
    int32_t* ho = (int32_t*)hoff.get();
    for (int64_t base = 0; base < n && first.empty(); base += CH) {
      const int64_t m = std::min<int64_t>(CH, n - base);
      ARK_CUDA(cudaMemcpyAsync(ho, col.offsets + base, (size_t)(m + 1) * 4, cudaMemcpyDeviceToHost, stream));
      ARK_CUDA(cudaStreamSynchronize(stream));
      for (int64_t k = 0; k < m && first.empty(); ++k) {
        const int64_t i = base + k;
        if (col.validity) {
          const int64_t bit = i + col.validity_bit0;
          uint8_t byte = 0;
          ARK_CUDA(cudaMemcpyAsync(&byte, col.validity + (bit >> 3), 1, cudaMemcpyDeviceToHost, stream));
          ARK_CUDA(cudaStreamSynchronize(stream));
          if (!((byte >> (bit & 7)) & 1)) continue;
        }
        const int len = ho[k + 1] - ho[k];
        if (len <= 0) continue;
        std::string s((size_t)len, '\0');
        ARK_CUDA(cudaMemcpyAsync(&s[0], col.data + ho[k], (size_t)len, cudaMemcpyDeviceToHost, stream));
        ARK_CUDA(cudaStreamSynchronize(stream));
        bool blank = true;
        for (char ch : s) if (!isspace((unsigned char)ch)) blank = false;
        if (!blank) first = s;
      }
    }
  }
  if (first.empty()) return out;
  std::vector<InferredField> inferred = jp.has_fixed_schema ? jp.fixed_schema : infer_schema(first);
  std::vector<InferredField> fields;
  if (jp.has_include) {
    for (auto& f : inferred) if (std::find(jp.include.begin(), jp.include.end(), f.name) != jp.include.end()) fields.push_back(f);
  } else fields = inferred;
  for (auto& f : fields)
    if (!f.supported) fail(ARK_ERR_UNSUPPORTED, "json_to_arrow: field '" + f.name + "': " + f.why + " (one level of List<primitive> / Struct<primitives> is decoded)");
  if ((int)fields.size() > JS_MAX_FIELDS_EXT) fail(ARK_ERR_UNSUPPORTED, "json_to_arrow: more than 64 fields in one record");
  for (auto& f : fields) if ((int)f.kids.size() > JS_MAX_FIELDS_EXT) fail(ARK_ERR_UNSUPPORTED, "json_to_arrow: more than 64 fields in one nested object");

  JsonParams P;
  memset(&P, 0, sizeof P);
  P.data = col.data; P.offsets = col.offsets; P.validity = col.validity; P.validity_bit0 = col.validity_bit0;
  P.n_payloads = n;
  static const bool no_stage = getenv("ARK_JSON_NO_STAGE") != nullptr;
  P.stage_bytes = no_stage ? 0 : record_stage_window(col.data_bytes, n, JS_THREADS);
  const size_t smem = (size_t)P.stage_bytes + 32;
  const unsigned grid = (unsigned)ceil_div(n, JS_THREADS);

  // ---- one pass when every payload holds exactly one record (the shape of every shipped example) ----
  static const bool two_pass_only = getenv("ARK_JSON_TWO_PASS") != nullptr;
  if (!two_pass_only && decode_fields(fields, P, grid, smem, n, true, nullptr, col.data, col.data_bytes, out.cols, stream)) { out.num_rows = n; return out; }

  // ---- general route: records per payload → row offsets → parse ----
  BufferPtr err = device_alloc(16), h = pinned_alloc(64);
  BufferPtr counts = device_alloc((size_t)(n + 1) * 4), counts64 = device_alloc((size_t)(n + 1) * 8), row_start = device_alloc((size_t)(n + 1) * 8);
  ARK_CUDA(cudaMemsetAsync(err.get(), 0, 16, stream));
  ARK_CUDA(cudaMemsetAsync(counts.get(), 0, (size_t)(n + 1) * 4, stream));
  P.counts = (int32_t*)counts.get();
  P.error = (int32_t*)err.get();
  {
    KernelTimer t("json_count_kernel", stream);
    json_parse_kernel<0><<<grid, JS_THREADS, smem, stream>>>(P);
  }
  {
    KernelTimer t("i32_to_i64_kernel", stream);
    i32_to_i64_kernel<<<(unsigned)ceil_div(n + 1, 256), 256, 0, stream>>>((const int32_t*)counts.get(), (long long*)counts64.get(), n + 1);
  }
  size_t tmp_bytes = 0;
  cub::DeviceScan::ExclusiveSum(nullptr, tmp_bytes, (long long*)counts64.get(), (long long*)row_start.get(), (int)(n + 1), stream);
  BufferPtr tmp = device_alloc(tmp_bytes + 16);
  note_launch("cub::DeviceScan::ExclusiveSum");
  cub::DeviceScan::ExclusiveSum(tmp.get(), tmp_bytes, (long long*)counts64.get(), (long long*)row_start.get(), (int)(n + 1), stream);
  ARK_CUDA(cudaMemcpyAsync((char*)h.get() + 16, (long long*)row_start.get() + n, 8, cudaMemcpyDeviceToHost, stream));
  ARK_CUDA(cudaMemcpyAsync(h.get(), err.get(), 16, cudaMemcpyDeviceToHost, stream));
  ARK_CUDA(cudaStreamSynchronize(stream));
  if (((const int32_t*)h.get())[0] != JE_NONE) raise_json(((const int32_t*)h.get())[0], ((const int32_t*)h.get())[1], "payload");
  const int64_t rows = *(const long long*)((char*)h.get() + 16);
  decode_fields(fields, P, grid, smem, rows, false, (const long long*)row_start.get(), col.data, col.data_bytes, out.cols, stream);
  out.num_rows = rows;
  return out;
}

}  // namespace ark
