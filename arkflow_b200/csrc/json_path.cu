// json_path.cu — the derived columns of the json_* calls of a query (plan.h DerivedCol), filled from their documents.
//
// Restates datafusion-functions-json 0.47 over jiter 0.9 (third-party; registered by sql.rs:18-24): each call follows
// its path from the document's first value, as jiter_json_find does, and reads the value it lands on.  The walk is lazy
// as jiter is: it reads the document only up to the end of the last value it needs, so bytes after a found value are
// never looked at, while everything before it must be well-formed JSON.  DESIGN.md §6 lists the rules and §9 the
// assumptions that are not verified against the crate.
//
// One thread walks one document and follows up to JSON_MAX_CALLS paths at once, so a query with several calls on one
// column reads each document once.  A container no path leads into is parsed through without consulting the paths.
#include "decoded.h"
#include "engine.h"
#include "decimal.cuh"
#include "json_text.cuh"
#include "varlen.h"

namespace ark {

namespace {

constexpr int JSON_MAX_CALLS = 8;   // paths one launch follows
constexpr int JP_MAX_DEPTH = 256;   // deeper nesting is treated as malformed
constexpr int JP_THREADS = 128;

struct JpCall {
  int32_t fn;                        // JsonFn
  int32_t n_path;
  uint32_t key_mask;                 // bit j: path element j is a key (else an index)
  int32_t key_off[JSON_MAX_PATH], key_len[JSON_MAX_PATH];  // into JpParams::keys
  long long index[JSON_MAX_PATH];
  void* values;                      // Int64 / Float64: 8 bytes per row; Boolean: one byte
  uint8_t* valid;                    // one byte per row (none for json_contains: never NULL)
  int32_t* len;                      // Utf8: result bytes per row
  long long* src;                    // Utf8: position in `data` of the value's bytes (a string's body)
  int32_t* raw;                      // json_get_str / json_as_text: source bytes, negative when they hold escapes
};

struct JpParams {
  const uint8_t* data;               // documents: data[offsets[r] .. offsets[r + 1])
  const int32_t* offsets;
  const uint8_t* validity;
  int32_t validity_bit0;
  int64_t n_rows;
  const uint8_t* keys;
  int32_t n_calls;
  JpCall calls[JSON_MAX_CALLS];
};

enum : uint8_t { K_OBJ = 1, K_ARR, K_STR, K_NUM, K_TRUE, K_FALSE, K_NULL };
enum : uint8_t { S_PENDING, S_FOUND, S_DONE, S_FAILED };  // FOUND: at the value's start; DONE: its end is known too

struct JpState {
  int32_t start, len, count;         // the value's span in the document; json_length: its elements
  int8_t m;                          // path elements matched: the value at nesting level m is on this path
  uint8_t status, kind;
  bool esc;                          // a string value with escapes
  bool is_int;                       // a number without fraction or exponent
};

__device__ __forceinline__ bool jp_ws(unsigned ch) { return ch <= 0x20u && ((0x100002600ull >> ch) & 1ull); }

// The string whose opening quote is b[*pos]: escapes as skip_escape accepts them, no raw control byte.  Leaves *pos
// after the closing quote.
__device__ bool jp_string(const uint8_t* b, int n, int* pos, bool* esc) {
  int p = *pos + 1;
  bool e = false;
  while (true) {
    if (p >= n) return false;
    const uint8_t ch = b[p];
    if (ch == '"') break;
    if (ch == '\\') {
      const uint8_t* q = skip_escape(b + p, b + n);
      if (!q) return false;
      p = (int)(q - b);
      e = true;
      continue;
    }
    if (ch < 0x20) return false;
    ++p;
  }
  *pos = p + 1;
  *esc = e;
  return true;
}

// JSON's number grammar: -?(0|[1-9][0-9]*)(\.[0-9]+)?([eE][+-]?[0-9]+)?.  Stops at the first byte that cannot continue it.
__device__ bool jp_number(const uint8_t* b, int n, int* pos, bool* is_int) {
  int p = *pos;
  auto digit = [&](int i) { return i < n && b[i] >= '0' && b[i] <= '9'; };
  if (p < n && b[p] == '-') ++p;
  if (!digit(p)) return false;
  if (b[p] == '0') { ++p; if (digit(p)) return false; }
  else while (digit(p)) ++p;
  bool in = true;
  if (p < n && b[p] == '.') { in = false; ++p; if (!digit(p)) return false; while (digit(p)) ++p; }
  if (p < n && (b[p] == 'e' || b[p] == 'E')) {
    in = false;
    ++p;
    if (p < n && (b[p] == '+' || b[p] == '-')) ++p;
    if (!digit(p)) return false;
    while (digit(p)) ++p;
  }
  *pos = p;
  *is_int = in;
  return true;
}

__device__ __forceinline__ bool jp_key_equals(const uint8_t* body, int raw, bool esc, const uint8_t* key, int klen) {
  if (esc) return decoded_equals(body, raw, (const char*)key, klen);
  if (raw != klen) return false;
  for (int i = 0; i < raw; ++i) if (body[i] != key[i]) return false;
  return true;
}

// Walks the document b[0, n) until every call is settled.  Returns false at the first malformed byte it reads.
__device__ bool jp_walk(const JpParams& P, const uint8_t* b, int n, JpState* st) {
  const int nc = P.n_calls;
  int open = nc;                       // calls not yet DONE or FAILED
  int pos = 0, depth = 0;
  uint32_t is_obj[JP_MAX_DEPTH / 32];  // bit d: the container at nesting level d is an object
  long long elem[JSON_MAX_PATH + 1];   // index of the current element of the array at level d (d < JSON_MAX_PATH)
  // The child of the container at level `depth - 1` whose key is key[0, klen) or whose index is idx starts here.
  auto enter_child = [&](const uint8_t* key, int klen, bool kesc, long long idx) {
    const int L = depth - 1;
    const bool obj = key != nullptr;
    for (int c = 0; c < nc; ++c) {
      JpState& s = st[c];
      const JpCall& C = P.calls[c];
      if (s.status == S_FOUND && s.m == L) ++s.count;  // an element of a container json_length is counting
      if (s.status != S_PENDING || s.m != L || L >= C.n_path) continue;  // n_path <= JSON_MAX_PATH
      const bool want_key = (C.key_mask >> L) & 1;
      if (want_key != obj) continue;
      if (obj ? jp_key_equals(key, klen, kesc, P.keys + C.key_off[L], C.key_len[L]) : C.index[L] == idx) s.m = (int8_t)depth;
    }
  };
  // A value ends at `pos`: the calls it settles.
  auto value_end = [&]() {
    for (int c = 0; c < nc; ++c) {
      JpState& s = st[c];
      if (s.m != depth) continue;
      if (s.status == S_FOUND) { s.len = pos - s.start; s.status = S_DONE; --open; }
      else if (s.status == S_PENDING) { s.status = S_FAILED; --open; }
    }
  };
  while (true) {
    // ---- a value starts (after whitespace) at nesting level `depth`
    while (pos < n && jp_ws(b[pos])) ++pos;
    if (pos >= n) return false;
    const uint8_t ch = b[pos];
    const uint8_t kind = ch == '{' ? K_OBJ : ch == '[' ? K_ARR : ch == '"' ? K_STR : ch == 't' ? K_TRUE : ch == 'f' ? K_FALSE
                       : ch == 'n' ? K_NULL : K_NUM;
    for (int c = 0; c < nc; ++c) {
      JpState& s = st[c];
      if (s.status != S_PENDING || s.m != depth || depth != P.calls[c].n_path) continue;
      s.start = pos; s.kind = kind;
      s.status = S_FOUND;
      if (P.calls[c].fn == (int)JsonFn::Contains) { s.status = S_DONE; --open; }  // the path resolves: jiter only peeks
    }
    if (open == 0) return true;
    if (kind == K_OBJ || kind == K_ARR) {
      if (depth >= JP_MAX_DEPTH) return false;
      const uint32_t bit = 1u << (depth & 31);
      is_obj[depth >> 5] = kind == K_OBJ ? is_obj[depth >> 5] | bit : is_obj[depth >> 5] & ~bit;
      ++depth;
      ++pos;
      while (pos < n && jp_ws(b[pos])) ++pos;
      if (pos < n && b[pos] == (kind == K_OBJ ? '}' : ']')) { ++pos; --depth; value_end(); }
      else {
        if (kind == K_ARR) {
          if (depth - 1 < JSON_MAX_PATH) elem[depth - 1] = 0;
          enter_child(nullptr, 0, false, 0);
        } else {
          if (pos >= n || b[pos] != '"') return false;
          const int k0 = pos + 1;
          bool kesc;
          if (!jp_string(b, n, &pos, &kesc)) return false;
          const int klen = pos - 1 - k0;
          while (pos < n && jp_ws(b[pos])) ++pos;
          if (pos >= n || b[pos] != ':') return false;
          ++pos;
          enter_child(b + k0, klen, kesc, 0);
        }
        continue;
      }
    } else {
      if (kind == K_STR) {
        bool e;
        if (!jp_string(b, n, &pos, &e)) return false;
        for (int c = 0; c < nc; ++c) if (st[c].status == S_FOUND && st[c].m == depth) st[c].esc = e;
      } else if (kind == K_NUM) {
        bool in;
        if (!jp_number(b, n, &pos, &in)) return false;
        for (int c = 0; c < nc; ++c) if (st[c].status == S_FOUND && st[c].m == depth) st[c].is_int = in;
      } else {
        const char* lit = kind == K_TRUE ? "true" : kind == K_FALSE ? "false" : "null";
        const int ln = kind == K_FALSE ? 5 : 4;
        if (n - pos < ln) return false;
        for (int i = 0; i < ln; ++i) if (b[pos + i] != (uint8_t)lit[i]) return false;
        pos += ln;
      }
      value_end();
    }
    // ---- after a value: the next element of its container, or the container's end
    while (true) {
      if (open == 0 || depth == 0) return true;
      while (pos < n && jp_ws(b[pos])) ++pos;
      if (pos >= n) return false;
      const int L = depth - 1;
      const bool obj = (is_obj[L >> 5] >> (L & 31)) & 1;
      if (b[pos] == (obj ? '}' : ']')) { ++pos; --depth; value_end(); continue; }
      if (b[pos] != ',') return false;
      ++pos;
      if (obj) {
        while (pos < n && jp_ws(b[pos])) ++pos;
        if (pos >= n || b[pos] != '"') return false;
        const int k0 = pos + 1;
        bool kesc;
        if (!jp_string(b, n, &pos, &kesc)) return false;
        const int klen = pos - 1 - k0;
        while (pos < n && jp_ws(b[pos])) ++pos;
        if (pos >= n || b[pos] != ':') return false;
        ++pos;
        enter_child(b + k0, klen, kesc, 0);
      } else {
        while (pos < n && jp_ws(b[pos])) ++pos;
        if (pos < n && b[pos] == ']') return false;  // a trailing comma (jiter's array_step)
        long long i = 0;
        if (L < JSON_MAX_PATH) i = ++elem[L];
        enter_child(nullptr, 0, false, i);
      }
      break;
    }
  }
}

// An integer's text → i64; false beyond i64 (jiter's BigInt).
__device__ bool jp_i64(const uint8_t* s, int len, long long* out) {
  int i = 0;
  const bool neg = s[0] == '-';
  if (neg) ++i;
  unsigned long long v = 0;
  for (; i < len; ++i) {
    const unsigned d = s[i] - '0';
    if (v > (0xFFFFFFFFFFFFFFFFull - d) / 10) return false;
    v = v * 10 + d;
  }
  if (!neg && v > 0x7FFFFFFFFFFFFFFFull) return false;
  if (neg && v > 0x8000000000000000ull) return false;
  *out = neg ? (long long)(0 - v) : (long long)v;
  return true;
}

__global__ void __launch_bounds__(JP_THREADS) json_path_kernel(const __grid_constant__ JpParams P) {
  const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= P.n_rows) return;
  JpState st[JSON_MAX_CALLS];
  const int nc = P.n_calls;
  for (int c = 0; c < nc; ++c) { st[c] = JpState{}; st[c].status = S_FAILED; }
  const int64_t vb = P.validity_bit0 + r;
  const bool present = !P.validity || ((P.validity[vb >> 3] >> (vb & 7)) & 1);
  const int32_t o0 = P.offsets[r];
  const uint8_t* doc = P.data + o0;
  if (present) {
    for (int c = 0; c < nc; ++c) st[c].status = S_PENDING;
    if (!jp_walk(P, doc, P.offsets[r + 1] - o0, st))
      for (int c = 0; c < nc; ++c) if (st[c].status != S_DONE) st[c].status = S_FAILED;
  }
  for (int c = 0; c < nc; ++c) {
    const JpCall& C = P.calls[c];
    const JpState& s = st[c];
    const bool got = s.status == S_DONE;
    const JsonFn fn = (JsonFn)C.fn;
    bool ok = false;
    switch (fn) {
      case JsonFn::Contains: ((uint8_t*)C.values)[r] = got; continue;
      case JsonFn::GetBool:
        ok = got && (s.kind == K_TRUE || s.kind == K_FALSE);
        ((uint8_t*)C.values)[r] = ok && s.kind == K_TRUE;
        break;
      case JsonFn::GetInt: {
        long long v = 0;
        ok = got && s.kind == K_NUM && s.is_int && jp_i64(doc + s.start, s.len, &v);
        ((long long*)C.values)[r] = v;
        break;
      }
      case JsonFn::GetFloat: {
        double v = 0.0;
        // an integer converts as jiter's i64 / BigInt does: "-0" is the integer 0, so +0.0
        ok = got && s.kind == K_NUM && decimal_to_f64(doc + s.start, s.len, &v) && !isinf(v);
        if (s.is_int) v += 0.0;
        ((double*)C.values)[r] = ok ? v : 0.0;
        break;
      }
      case JsonFn::Length:
        ok = got && (s.kind == K_ARR || s.kind == K_OBJ);
        ((long long*)C.values)[r] = ok ? s.count : 0;
        break;
      default: {  // Utf8 results
        int len = 0, raw = 0;
        long long src = 0;
        const bool text = fn == JsonFn::GetStr || (fn == JsonFn::AsText && s.kind == K_STR);
        if (got && text && s.kind == K_STR) {
          ok = true;
          src = o0 + s.start + 1;
          raw = s.len - 2;
          len = s.esc ? decoded_len(doc + s.start + 1, raw) : raw;
          if (s.esc) raw = -raw;
        } else if (got && !text && !(fn == JsonFn::AsText && s.kind == K_NULL)) {
          ok = true;
          src = o0 + s.start;
          len = raw = s.len;
        }
        C.len[r] = len;
        C.src[r] = src;
        if (C.raw) C.raw[r] = raw;
      }
    }
    C.valid[r] = ok;
  }
}

}  // namespace

Batch append_json_columns(const Plan& plan, const Batch& in, cudaStream_t stream) {
  if (in.cols.size() != plan.n_input_fields) fail(ARK_ERR_PROCESS, "internal: batch does not match the plan's input");
  const int64_t n = in.num_rows;
  const size_t nd = plan.derived.size();
  std::vector<StagedColumn> staged(nd);
  std::vector<uint8_t> keys;
  for (size_t k = 0; k < nd; ++k) {
    const DerivedCol& d = plan.derived[k];
    const Field& f = plan.input_fields[plan.n_input_fields + k];
    const bool wants_raw = d.fn == JsonFn::GetStr || d.fn == JsonFn::AsText;
    staged[k] = stage_column(f.type, n, d.fn != JsonFn::Contains, wants_raw, stream);
    // a value's bytes lie inside its document (decoding escapes only shortens them), so the column's bytes bound it
    staged[k].bound = std::max<int64_t>(varlen_bytes_bound(in.cols[d.doc_col]), 0);
    staged[k].what = "column '" + f.name + "'";
    for (auto& e : d.path) keys.insert(keys.end(), e.key.begin(), e.key.end());
  }
  BufferPtr dkeys = device_alloc(keys.size() + 16);
  if (!keys.empty()) ARK_CUDA(cudaMemcpyAsync(dkeys.get(), keys.data(), keys.size(), cudaMemcpyHostToDevice, stream));
  // CAST(<Binary> AS STRING) runs over every row before the function sees it, so invalid UTF-8 fails the query
  BufferPtr bad;
  std::vector<bool> doc_done(plan.n_input_fields, false);
  for (auto& d : plan.derived) {
    if (!d.doc_cast || doc_done[d.doc_col] || n == 0) continue;
    if (!bad) { bad = device_alloc(16); ARK_CUDA(cudaMemsetAsync(bad.get(), 0, 16, stream)); }
    const Column& c = in.cols[d.doc_col];
    launch_utf8_validate(c.offsets, c.data, c.validity, c.validity_bit0, n, (int*)bad.get(), stream);
    doc_done[d.doc_col] = true;
  }
  // one launch per document column and JSON_MAX_CALLS of its calls
  std::vector<bool> launched(nd, false);
  size_t key_pos = 0;
  std::vector<size_t> key_at(nd);
  for (size_t k = 0; k < nd; ++k) { key_at[k] = key_pos; for (auto& e : plan.derived[k].path) key_pos += e.key.size(); }
  for (size_t k0 = 0; k0 < nd && n > 0; ++k0) {
    if (launched[k0]) continue;
    const Column& doc = in.cols[plan.derived[k0].doc_col];
    JpParams P;
    memset(&P, 0, sizeof P);
    P.data = doc.data; P.offsets = doc.offsets; P.validity = doc.validity; P.validity_bit0 = doc.validity_bit0;
    P.n_rows = n; P.keys = (const uint8_t*)dkeys.get();
    for (size_t k = k0; k < nd && P.n_calls < JSON_MAX_CALLS; ++k) {
      const DerivedCol& d = plan.derived[k];
      if (launched[k] || d.doc_col != plan.derived[k0].doc_col) continue;
      launched[k] = true;
      JpCall& C = P.calls[P.n_calls++];
      C.fn = (int32_t)d.fn;
      C.n_path = (int32_t)d.path.size();
      int32_t at = (int32_t)key_at[k];
      for (size_t j = 0; j < d.path.size(); ++j) {
        if (d.path[j].is_key) C.key_mask |= 1u << j;
        C.key_off[j] = at; C.key_len[j] = (int32_t)d.path[j].key.size(); C.index[j] = d.path[j].index;
        at += C.key_len[j];
      }
      StagedColumn& s = staged[k];
      C.values = s.values.get(); C.valid = (uint8_t*)s.valid.get(); C.len = (int32_t*)s.len.get();
      C.src = (long long*)s.src.get(); C.raw = (int32_t*)s.raw.get();
    }
    KernelTimer t("json_path_kernel", stream);
    json_path_kernel<<<(unsigned)ceil_div(n, JP_THREADS), JP_THREADS, 0, stream>>>(P);
  }
  ARK_CUDA(cudaGetLastError());
  settle_columns(staged, bad.get(), bad ? 4 : 0, [](const void* h) {
    if (*(const int*)h) fail(ARK_ERR_PROCESS, "Collection query results error: Arrow error: Cast error: Cannot cast binary to string: invalid utf-8 sequence");
  }, stream);
  Batch out = in;
  for (size_t k = 0; k < nd; ++k) {
    const DerivedCol& d = plan.derived[k];
    const uint8_t* data = in.cols[d.doc_col].data;
    out.cols.push_back(finish_column(staged[k], plan.input_fields[plan.n_input_fields + k], [&](const StagedColumn& s, uint8_t* bytes) {
      if (d.fn == JsonFn::GetJson) launch_span_copy(data, nullptr, (const long long*)s.src.get(), (const int32_t*)s.offsets.get(), s.rows, bytes, stream);
      else launch_json_strings(data, s, bytes, stream);
    }, stream));
  }
  return out;
}

}  // namespace ark
