// utf8.cuh — well-formed UTF-8 per Unicode table 3-7 (no overlongs, no surrogates, ≤ U+10FFFF): the check
// Rust's str::from_utf8 makes, used by CAST(Binary AS Utf8), the protobuf decoder's `string` fields, the JSON
// decoder's strings and schema inference, and the CSV input's Utf8 fields and header.
#pragma once
#include <cstdint>

namespace ark {

__host__ __device__ __forceinline__ bool utf8_valid(const uint8_t* p, long long len) {
  long long i = 0;
  while (i < len) {
    const uint8_t b0 = p[i];
    if (b0 < 0x80) { ++i; continue; }
    int need; uint8_t lo = 0x80, hi = 0xBF;
    if (b0 >= 0xC2 && b0 <= 0xDF) need = 1;
    else if (b0 == 0xE0) { need = 2; lo = 0xA0; }
    else if ((b0 >= 0xE1 && b0 <= 0xEC) || b0 == 0xEE || b0 == 0xEF) need = 2;
    else if (b0 == 0xED) { need = 2; hi = 0x9F; }
    else if (b0 == 0xF0) { need = 3; lo = 0x90; }
    else if (b0 >= 0xF1 && b0 <= 0xF3) need = 3;
    else if (b0 == 0xF4) { need = 3; hi = 0x8F; }
    else return false;
    if (i + need >= len) return false;  // truncated sequence
    if (p[i + 1] < lo || p[i + 1] > hi) return false;
    for (int k = 2; k <= need; ++k) if ((p[i + k] & 0xC0) != 0x80) return false;
    i += need + 1;
  }
  return true;
}

}  // namespace ark
