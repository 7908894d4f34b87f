// smem_table.cuh — open-addressing table of Key16 keys in shared memory (the low-cardinality GROUP BY's per-CTA table).
#pragma once
#include "hash_agg.cuh"
#include "hashkey.cuh"

namespace ark {

constexpr unsigned long long KEY_PENDING = 0xFFFFFFFFFFFFFFFEull;  // tag 0xFFFFFFFF is never a key tag

static __device__ __forceinline__ unsigned long long lds_volatile(const unsigned long long* p) { return *reinterpret_cast<const volatile unsigned long long*>(p); }
static __device__ __forceinline__ void sts_volatile(unsigned long long* p, unsigned long long v) { *reinterpret_cast<volatile unsigned long long*>(p) = v; }

// Finds or claims the slot of `mine` in the shared-memory region (linear probing, wraps inside the region).
// Claim protocol without a 128-bit shared-memory CAS: hi EMPTY → PENDING (64-bit CAS), lo stored, then
// hi published; readers re-read while they see PENDING.  The owner never waits on anybody, so the loop
// terminates under any warp scheduling.  Returns -1 when the region is full.
static __device__ __forceinline__ int region_find_or_claim(Key16* K, int S, unsigned int home, Key16 mine, const ColView& kc, unsigned int* claimed) {
  unsigned int s = home;
  int probes = 0;
  while (true) {
    unsigned long long hi = lds_volatile(&K[s].hi);
    if (hi == mine.hi) {  // the common case first: the group exists
      const Key16 stored{lds_volatile(&K[s].lo), hi};
      if (key_equal(mine, stored, kc, kc)) return (int)s;
    } else if (hi == KEY_EMPTY) {
      const unsigned long long old = atomicCAS(&K[s].hi, KEY_EMPTY, KEY_PENDING);
      if (old == KEY_EMPTY) {
        sts_volatile(&K[s].lo, mine.lo);
        __threadfence_block();
        sts_volatile(&K[s].hi, mine.hi);
        ++*claimed;
        return (int)s;
      }
      continue;  // somebody else claimed it: look again
    } else if (hi == KEY_PENDING) {
      continue;
    }
    s = (s + 1) & (unsigned int)(S - 1);
    if (++probes >= S) return -1;
  }
}


}  // namespace ark
