// bitmap.cuh — reading an Arrow bitmap (validity or Boolean values) on the device.  bitmap.h builds them.
#pragma once
#include "vm.h"

namespace ark {

// Bit i of a bitmap: bit i & 7 of byte i >> 3, least significant bit first.
__device__ __forceinline__ bool bit_get(const uint8_t* bm, int64_t i) {
  return (bm[i >> 3] >> (i & 7)) & 1;
}

__device__ __forceinline__ bool col_valid(const ColView& c, int64_t row) {
  return c.validity == nullptr || bit_get(c.validity, row + c.validity_bit0);
}

}  // namespace ark
