// stage_store.cuh — write a CTA's contiguous output byte range from shared memory to global memory with
// destination-aligned 16-byte stores.  The staging buffer must start at the destination's misalignment
// (stage_misalignment) so that shared and global addresses agree mod 16.
#pragma once
#include <algorithm>
#include <cstdint>

#include "common.h"

namespace ark {

__device__ __forceinline__ int stage_misalignment(const uint8_t* gdst) { return (int)(reinterpret_cast<uintptr_t>(gdst) & 15); }

// `stage` is 16-byte aligned; the range's bytes sit at stage[mis .. mis + bytes).  Call from every thread
// of the CTA after a __syncthreads().
__device__ __forceinline__ void stage_store(uint8_t* gdst, const uint8_t* stage, int mis, int bytes, int tid, int nthreads) {
  const int head = min((16 - mis) & 15, bytes);
  if (tid < head) gdst[tid] = stage[mis + tid];
  const int body = (bytes - head) >> 4;
  const uint4* sv = reinterpret_cast<const uint4*>(stage + mis + head);  // mis + head ≡ 0 (mod 16) whenever body > 0
  uint4* gv = reinterpret_cast<uint4*>(gdst + head);
  for (int g = tid; g < body; g += nthreads) gv[g] = sv[g];
  const int tail0 = head + body * 16;
  if (tid < bytes - tail0) gdst[tail0 + tid] = stage[mis + tail0 + tid];
}

// Staging window of a kernel whose CTAs write `rows_per_cta` rows of a `total`-byte, `n`-row output through stage_store:
// the average CTA's bytes + 50 %, at most 44 KiB.  CTAs whose rows are longer take the kernel's direct path.
inline int stage_window(int64_t total, int64_t n, int rows_per_cta) {
  return (int)std::min<int64_t>(44 * 1024, round_up((int64_t)((double)total / (double)n * rows_per_cta * 1.5) + 256, 1024));
}

// Staging window of a decode kernel whose CTAs of `threads` threads parse one record each from `bytes` bytes of `n`
// records: the average CTA's bytes + 25 % + alignment slack, or 0 when records average more than 256 bytes (every CTA
// parses in place).
inline int record_stage_window(int64_t bytes, int64_t n, int threads) {
  const double avg = (double)bytes / (double)n;
  return avg <= 256.0 ? (int)round_up((int64_t)(avg * threads * 1.25) + 256, 1024) : 0;
}

}  // namespace ark
