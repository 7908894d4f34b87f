// json_text.cuh — JSON string bodies on the device: escape checks, decoded lengths, key comparison and decoding.  Shared
// by the JSON decoder (json.cu) and the JSON path functions (json_path.cu).
#pragma once
#include <cstdint>

namespace ark {
namespace {

__device__ __forceinline__ unsigned hex_digit(unsigned h) {  // 16 when h is not a hex digit
  const unsigned l = h | 0x20;
  return h - '0' <= 9u ? h - '0' : l - 'a' <= 5u ? l - 'a' + 10 : 16;
}

// The escape at p (on its backslash) must be one of JSON's nine; \u takes four hex digits, a high surrogate must be
// followed by a \u low surrogate, and a low surrogate may not stand alone.  Returns the position after the escape,
// nullptr when it is malformed.
__device__ __forceinline__ const uint8_t* skip_escape(const uint8_t* p, const uint8_t* end) {
  if (end - p < 2) return nullptr;
  const uint8_t e = p[1];
  if (e != 'u') return e == '"' || e == '\\' || e == '/' || e == 'b' || e == 'f' || e == 'n' || e == 'r' || e == 't' ? p + 2 : nullptr;
  auto hex4 = [&](const uint8_t* q, unsigned* cp) {
    if (end - q < 4) return false;
    unsigned v = 0;
    for (int k = 0; k < 4; ++k) { const unsigned d = hex_digit(q[k]); if (d > 15) return false; v = v * 16 + d; }
    *cp = v;
    return true;
  };
  unsigned hi, lo;
  if (!hex4(p + 2, &hi)) return nullptr;
  p += 6;
  if (hi < 0xD800 || hi > 0xDFFF) return p;
  if (hi >= 0xDC00) return nullptr;  // a low surrogate with no high one before it
  if (end - p < 2 || p[0] != '\\' || p[1] != 'u' || !hex4(p + 2, &lo) || lo < 0xDC00 || lo > 0xDFFF) return nullptr;
  return p + 6;
}

// Decoding.  json_strings_kernel, the List stage and json_quoted_numbers_kernel decode bodies that strings_valid has
// accepted; the parse kernels measure and compare bodies before their payload is checked, so the escape reader stays
// inside b[0..raw) whatever it holds (a malformed body then fails the payload's check).
__device__ __forceinline__ unsigned hex4_unchecked(const uint8_t* q) {
  unsigned v = 0;
  for (int k = 0; k < 4; ++k) v = v * 16 + hex_digit(q[k]);
  return v;
}

// the escape at b[*i] (on its backslash) of the body b[0..raw) → its code point, a surrogate pair combined; *i moves past it
__device__ __forceinline__ unsigned escape_cp(const uint8_t* b, int raw, int* i) {
  const uint8_t e = *i + 1 < raw ? b[*i + 1] : '\\';
  if (e != 'u' || *i + 6 > raw) { *i += 2; return e == 'b' ? '\b' : e == 'f' ? '\f' : e == 'n' ? '\n' : e == 'r' ? '\r' : e == 't' ? '\t' : e; }
  unsigned cp = hex4_unchecked(b + *i + 2);
  *i += 6;
  if (cp >= 0xD800 && cp < 0xDC00 && *i + 6 <= raw) { cp = 0x10000 + ((cp - 0xD800) << 10) + (hex4_unchecked(b + *i + 2) - 0xDC00); *i += 6; }
  return cp;
}

__device__ __forceinline__ int put_utf8(unsigned cp, uint8_t* out) {
  if (cp < 0x80) { out[0] = (uint8_t)cp; return 1; }
  if (cp < 0x800) { out[0] = 0xC0 | (cp >> 6); out[1] = 0x80 | (cp & 0x3F); return 2; }
  if (cp < 0x10000) { out[0] = 0xE0 | (cp >> 12); out[1] = 0x80 | ((cp >> 6) & 0x3F); out[2] = 0x80 | (cp & 0x3F); return 3; }
  out[0] = 0xF0 | (cp >> 18); out[1] = 0x80 | ((cp >> 12) & 0x3F); out[2] = 0x80 | ((cp >> 6) & 0x3F); out[3] = 0x80 | (cp & 0x3F);
  return 4;
}

// length of a JSON string body once escapes are decoded
__device__ int decoded_len(const uint8_t* b, int raw) {
  int n = 0;
  for (int i = 0; i < raw;) {
    if (b[i] != '\\') { ++n; ++i; continue; }
    const unsigned cp = escape_cp(b, raw, &i);
    n += cp < 0x80 ? 1 : cp < 0x800 ? 2 : cp < 0x10000 ? 3 : 4;
  }
  return n;
}

// does the JSON string body b[0..raw) (which contains escapes) decode to exactly nm[0..nlen)?
__device__ bool decoded_equals(const uint8_t* b, int raw, const char* nm, int nlen) {
  int n = 0;
  for (int i = 0; i < raw;) {
    uint8_t out[4];
    int k = 1;
    if (b[i] != '\\') out[0] = b[i++];
    else k = put_utf8(escape_cp(b, raw, &i), out);
    for (int q = 0; q < k; ++q) { if (n >= nlen || (uint8_t)nm[n] != out[q]) return false; ++n; }
  }
  return n == nlen;
}

__device__ void decode_string(const uint8_t* b, int raw, uint8_t* out) {
  for (int i = 0; i < raw;) {
    if (b[i] != '\\') { *out++ = b[i++]; continue; }
    out += put_utf8(escape_cp(b, raw, &i), out);
  }
}

}  // namespace
}  // namespace ark
