// hash_agg_tile.cu — GROUP BY for low-cardinality keys (table ≤ 2048 slots): the whole hash table of a CTA —
// keys and accumulators — lives in shared memory, and the global table is touched once per CTA and group.
//
// This is the shape of every shipped example (sensor ∈ {temp_1, temp_2, …}).  hash_agg_kernel sends each row to
// the global table (a 128-bit load + two L2 atomics per row, and hot keys serialise on the L2 atomic unit: with two
// keys the kernel is dozens of times slower than with many).  Here a persistent CTA takes 1024-row tiles, each thread
// owns 4 consecutive rows:
//   * the tile's key bytes arrive through ONE 1-D TMA bulk copy (cp.async.bulk → mbarrier) of the
//     16-byte-aligned window around [offsets[t0], offsets[t1]); offsets / predicate / argument values are
//     16-byte vector loads issued up front;
//   * keys are found or claimed in the CTA's shared-memory table (smem_table.cuh) and accumulated there;
//   * tables of ≤ 64 slots (and global aggregates) first reduce each distinct slot of a warp with shuffles, so a
//     hot key costs one shared-memory atomic per warp instead of 32 serialised ones;
//   * at the end each CTA merges its ≤ S groups into the global table (128-bit CAS + global atomics), which
//     keeps the layout every downstream step expects.
// A batch with more distinct keys than slots raises `overflow`; the host retries with 4× the slots.
#include <atomic>

#include "tma.cuh"
#include "agg_acc.cuh"
#include "engine.h"
#include "hash_agg.cuh"
#include "hashkey.cuh"
#include "smem_table.cuh"

namespace ark {

namespace {

constexpr int HT_THREADS = 256;
constexpr int HT_TILE = HT_THREADS * 4;


// Tables of ≤ 64 slots.  For every distinct slot among the warp's 128 rows: each lane first combines its own rows
// of that slot, one shuffle reduction per slot follows, lane 0 applies the result to the WARP'S OWN copy of the
// accumulator with a plain read-modify-write (no atomics, no contention between warps).
// CLS: 0 count, 1 sum i64, 2 sum f64, 3 min i64, 4 min f64 (totalOrder key), 5 max i64, 6 max f64.
template <int CLS>
__device__ __forceinline__ void tiny_accumulate(unsigned long long* acc, const int (&slot)[4], unsigned ok, unsigned valid,
                                                const unsigned long long (&av)[4], int arg_is_f64, int lane) {
  unsigned act0 = __ballot_sync(0xffffffffu, ok & 1), act1 = __ballot_sync(0xffffffffu, (ok >> 1) & 1),
           act2 = __ballot_sync(0xffffffffu, (ok >> 2) & 1), act3 = __ballot_sync(0xffffffffu, (ok >> 3) & 1);
  while (act0 | act1 | act2 | act3) {
    const unsigned am = act0 ? act0 : act1 ? act1 : act2 ? act2 : act3;
    const int pick = act0 ? slot[0] : act1 ? slot[1] : act2 ? slot[2] : slot[3];
    const int s = __shfl_sync(0xffffffffu, pick, __ffs(am) - 1);
    long long li = CLS == 3 || CLS == 4 ? 0x7FFFFFFFFFFFFFFFll : (CLS == 5 || CLS == 6 ? (long long)0x8000000000000000ull : 0);
    double lf = 0.0;
    int lcnt = 0;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const bool in = ((ok >> j) & 1) && slot[j] == s;
      const unsigned m = __ballot_sync(0xffffffffu, in);
      if (j == 0) act0 &= ~m; else if (j == 1) act1 &= ~m; else if (j == 2) act2 &= ~m; else act3 &= ~m;
      if (in && ((valid >> j) & 1)) {
        ++lcnt;
        if (CLS == 1) li += (long long)av[j];
        if (CLS == 2) lf += arg_is_f64 ? __longlong_as_double((long long)av[j]) : (double)(long long)av[j];
        if (CLS == 3 || CLS == 5) { const long long x = (long long)av[j]; li = CLS == 3 ? (x < li ? x : li) : (x > li ? x : li); }
        if (CLS == 4 || CLS == 6) { const long long x = f64_total_key(av[j]); li = CLS == 4 ? (x < li ? x : li) : (x > li ? x : li); }
      }
    }
    unsigned long long* dst = acc + s;
    if (CLS == 0) { const int c = __reduce_add_sync(0xffffffffu, lcnt); if (lane == 0) *dst += (unsigned long long)c; }
    else if (CLS == 1) { const long long v = warp_sum_ll(li); if (lane == 0) *dst += (unsigned long long)v; }
    else if (CLS == 2) {
      const double v = warp_sum_f64(lf);
      const bool any = __any_sync(0xffffffffu, lcnt > 0);
      if (lane == 0 && any) *reinterpret_cast<double*>(dst) += v;
    } else if (CLS == 3 || CLS == 4) { const long long v = warp_min_ll(li); if (lane == 0 && v < *reinterpret_cast<long long*>(dst)) *reinterpret_cast<long long*>(dst) = v; }
    else { const long long v = warp_max_ll(li); if (lane == 0 && v > *reinterpret_cast<long long*>(dst)) *reinterpret_cast<long long*>(dst) = v; }
  }
}

// fold warp copy `src` into copy 0 (same slot, same accumulator)
__device__ __forceinline__ void fold_acc(int kind, unsigned long long* dst, unsigned long long v) {
  switch (kind) {
    case ACC_COUNT_STAR: case ACC_COUNT: case ACC_SUM_I64: *dst += v; break;
    case ACC_SUM_F64: *reinterpret_cast<double*>(dst) += __longlong_as_double((long long)v); break;
    case ACC_MIN_I64: case ACC_MIN_F64: if ((long long)v < *reinterpret_cast<long long*>(dst)) *reinterpret_cast<long long*>(dst) = (long long)v; break;
    default: if ((long long)v > *reinterpret_cast<long long*>(dst)) *reinterpret_cast<long long*>(dst) = (long long)v; break;
  }
}

template <int PRED>
__global__ void __launch_bounds__(HT_THREADS, 3) hash_agg_tile_kernel(const __grid_constant__ AggParams P, const int str_cap, const int log2_slots) {
  extern __shared__ __align__(16) uint8_t smem[];  // [key bytes window: str_cap + 32][Key16 K[S]][u64 ACC[copies][n_acc][S]], copies = 8 warps when S ≤ 64
  __shared__ __align__(8) unsigned long long s_bar;
  __shared__ int s_str_base, s_str_staged, s_stop;
  const int tid = threadIdx.x, lane = tid & 31;
  const int S = 1 << log2_slots;
  uint8_t* in_bytes = smem;
  Key16* K = reinterpret_cast<Key16*>(smem + (str_cap ? str_cap + 32 : 0));
  unsigned long long* ACC = reinterpret_cast<unsigned long long*>(K + S);
  const int64_t n = P.n_rows;
  const int n_tiles = (int)((n + HT_TILE - 1) / HT_TILE);
  const bool bytes_key = P.key_kind == KEY_BYTES;
  const bool tiny = S <= 64;  // hot keys: reduce inside the warp before touching shared memory
  const ColView& kc = P.cols[P.key_kind == KEY_NONE ? 0 : P.key_slot];
  const int32_t* koff = kc.offsets;

  if (tid == 0) {
    mbar_init(&s_bar, 1);
    mbar_fence_init();
    if (P.key_kind == KEY_NONE && blockIdx.x == 0) {  // a global aggregate always yields one row
      Key16 mine; unsigned long long h;
      make_key(KEY_NONE, kc, 0, &mine, &h);
      unsigned int c = 0;
      table_find_or_claim(P.table, P.mask >> 2, P.bucket_stride, h, mine, kc, kc, &c);
      if (c) atomicAdd(P.group_count, c);
    }
  }
  const int copies = tiny ? HT_THREADS / 32 : 1;
  for (int s = tid; s < S; s += HT_THREADS) K[s] = Key16{KEY_EMPTY, KEY_EMPTY};
  for (int i = tid; i < copies * P.n_acc * S; i += HT_THREADS) ACC[i] = acc_identity(P.accs[(i / S) % P.n_acc].kind);
  __syncthreads();

  unsigned int claimed = 0;
  bool full = false;
  unsigned phase = 0;  // mbarrier phases completed so far: advances only for tiles whose bulk copy was issued (CTA-uniform)
  const long long pred_c = P.sp_is_f64 ? f64_total_key(P.sp_const) : (long long)P.sp_const;
  for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    const int64_t row0 = (int64_t)tile * HT_TILE;
    const int rows = (int)((n - row0) < HT_TILE ? (n - row0) : HT_TILE);
    if (tid == 0) s_stop = *reinterpret_cast<volatile int32_t*>(P.overflow);  // table too small: the host retries with 4× the slots
    if (bytes_key && tid == 0 && !s_stop) {
      const int32_t o0 = koff[row0], o1 = koff[row0 + rows];
      const uintptr_t a0 = reinterpret_cast<uintptr_t>((const uint8_t*)kc.data + o0), a1 = reinterpret_cast<uintptr_t>((const uint8_t*)kc.data + o1);
      const uintptr_t lo = a0 & ~(uintptr_t)15, hi = (a1 + 15) & ~(uintptr_t)15;
      int staged = 0;
      if (o1 > o0 && hi - lo <= (uintptr_t)str_cap) {
        staged = 1;
        mbar_expect_tx(&s_bar, (unsigned)(hi - lo));
        tma_load_1d(in_bytes, reinterpret_cast<const void*>(lo), (unsigned)(hi - lo), &s_bar);
      }
      s_str_base = o0 - (int32_t)(a0 - lo); s_str_staged = staged;
    }
    // ---- loads in flight: offsets, predicate column ----
    const int lr0 = 4 * tid;
    const bool full_rows = lr0 + 4 <= rows;
    int off[5] = {0, 0, 0, 0, 0};
    unsigned long long pv[4] = {0, 0, 0, 0};
    if (bytes_key) {
      const int32_t* os = koff + row0 + lr0;
      if (full_rows && (reinterpret_cast<uintptr_t>(os) & 15) == 0) {
        asm volatile("ld.global.cs.v4.s32 {%0, %1, %2, %3}, [%4];" : "=r"(off[0]), "=r"(off[1]), "=r"(off[2]), "=r"(off[3]) : "l"(os));
      } else {
#pragma unroll
        for (int j = 0; j < 4; ++j) off[j] = (lr0 + j <= rows) ? os[j] : 0;
      }
      off[4] = __shfl_down_sync(0xffffffffu, off[0], 1);
      if ((lane == 31 || lr0 + 4 >= rows) && lr0 + 4 <= rows) off[4] = os[4];
    }
    if (PRED == 1) {
      const unsigned long long* src = (const unsigned long long*)P.cols[P.sp_slot].data + row0 + lr0;
      if (full_rows && (reinterpret_cast<uintptr_t>(src) & 15) == 0) {
        asm volatile("ld.global.cs.v2.u64 {%0, %1}, [%2];" : "=l"(pv[0]), "=l"(pv[1]) : "l"(src));
        asm volatile("ld.global.cs.v2.u64 {%0, %1}, [%2];" : "=l"(pv[2]), "=l"(pv[3]) : "l"(src + 2));
      } else {
#pragma unroll
        for (int j = 0; j < 4; ++j) pv[j] = (lr0 + j < rows) ? src[j] : 0;
      }
    }
    __syncthreads();  // s_str_staged / s_str_base / s_stop visible; (it > 0) previous tile's readers are done
    if (s_stop) break;  // CTA-uniform; no bulk copy was issued for this tile
    unsigned ok = 0;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      bool f = lr0 + j < rows;
      if (PRED == 1 && f) {
        const ColView& c = P.cols[P.sp_slot];
        f = cmp_i64(P.sp_cmp, P.sp_is_f64 ? f64_total_key(pv[j]) : (long long)pv[j], pred_c) && col_valid(c, row0 + lr0 + j);
      }
      ok |= (unsigned)f << j;
    }
    const bool staged = bytes_key && s_str_staged;
    if (staged) { mbar_wait(&s_bar, phase & 1); ++phase; }
    // ---- keys → slots of the shared-memory table ----
    int slot[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      slot[j] = -1;
      if (!((ok >> j) & 1)) continue;
      const int64_t row = row0 + lr0 + j;
      Key16 mine;
      unsigned int h32;
      if (bytes_key && staged && col_valid(kc, row)) {
        make_key_smem(in_bytes + (off[j] - s_str_base), off[j + 1] - off[j], row, &mine, &h32);
      } else {
        int llen = 0;
        const uint8_t* lp = make_key_raw(P.key_kind, kc, row, &mine, &llen);
        if (lp) { const unsigned long long h = hash_bytes(lp, llen); h32 = (unsigned)(h >> 32) ^ (unsigned)h; }
        else h32 = hash32_key16(mine);
      }
      slot[j] = region_find_or_claim(K, S, h32 & (unsigned)(S - 1), mine, kc, &claimed);
      if (slot[j] < 0) { full = true; ok &= ~(1u << j); }
    }
    // ---- accumulate ----
    for (int a = 0; a < P.n_acc; ++a) {
      const AccParam& A = P.accs[a];
      unsigned long long av[4] = {0, 0, 0, 0};
      unsigned valid = ok;
      if (A.kind != ACC_COUNT_STAR) {
        const ColView& c = P.cols[A.arg_slot];
        // COUNT(x) reads x's validity only (x may be Utf8 / Binary / Boolean: no 8-byte values to load)
        if (A.kind != ACC_COUNT) {
          const unsigned long long* src = (const unsigned long long*)c.data + row0 + lr0;
          if (full_rows && (reinterpret_cast<uintptr_t>(src) & 15) == 0) {
            asm volatile("ld.global.cs.v2.u64 {%0, %1}, [%2];" : "=l"(av[0]), "=l"(av[1]) : "l"(src));
            asm volatile("ld.global.cs.v2.u64 {%0, %1}, [%2];" : "=l"(av[2]), "=l"(av[3]) : "l"(src + 2));
          } else {
#pragma unroll
            for (int j = 0; j < 4; ++j) av[j] = (lr0 + j < rows) ? src[j] : 0;
          }
        }
        if (c.validity) {
#pragma unroll
          for (int j = 0; j < 4; ++j) if (((valid >> j) & 1) && !col_valid(c, row0 + lr0 + j)) valid &= ~(1u << j);
        }
      }
      unsigned long long* acc = ACC + ((tiny ? (tid >> 5) * P.n_acc : 0) + a) * S;
      if (tiny) {
        const int is_f64 = A.arg_is_f64;
        switch (A.kind) {
          case ACC_COUNT_STAR: case ACC_COUNT: tiny_accumulate<0>(acc, slot, ok, valid, av, is_f64, lane); break;
          case ACC_SUM_I64: tiny_accumulate<1>(acc, slot, ok, valid, av, is_f64, lane); break;
          case ACC_SUM_F64: tiny_accumulate<2>(acc, slot, ok, valid, av, is_f64, lane); break;
          case ACC_MIN_I64: tiny_accumulate<3>(acc, slot, ok, valid, av, is_f64, lane); break;
          case ACC_MIN_F64: tiny_accumulate<4>(acc, slot, ok, valid, av, is_f64, lane); break;
          case ACC_MAX_I64: tiny_accumulate<5>(acc, slot, ok, valid, av, is_f64, lane); break;
          default: tiny_accumulate<6>(acc, slot, ok, valid, av, is_f64, lane); break;
        }
      } else {
#pragma unroll
        for (int j = 0; j < 4; ++j)
          if ((valid >> j) & 1) accumulate(A.kind, A.arg_is_f64, acc + slot[j], av[j]);
      }
    }
    __syncthreads();  // everyone is done with in_bytes before the next tile's bulk copy overwrites it
  }
  if (full) atomicExch(P.overflow, 1);
  __syncthreads();
  if (tiny) {  // fold the warps' copies into copy 0
    for (int i = tid; i < P.n_acc * S; i += HT_THREADS)
      for (int w = 1; w < copies; ++w) fold_acc(P.accs[i / S].kind, ACC + i, ACC[w * P.n_acc * S + i]);
    __syncthreads();
  }
  // ---- merge this CTA's groups into the global table ----
  for (int s = tid; s < S; s += HT_THREADS) {
    const Key16 mine = K[s];
    if (mine.hi == KEY_EMPTY) continue;
    unsigned int c = 0;
    const unsigned long long g = table_find_or_claim(P.table, P.mask >> 2, P.bucket_stride, P.key_kind == KEY_NONE ? 0ull : stored_key_hash(mine, kc),
                                                     mine, kc, kc, &c, 1024);
    if (g == ~0ull) { atomicExch(P.overflow, 1); continue; }
    if (c) {
      const unsigned cnt = atomicAdd(P.group_count, 1u);
      if (cnt >= P.max_groups) atomicExch(P.overflow, 1);
    }
    for (int a = 0; a < P.n_acc; ++a) {
      const unsigned long long v = ACC[a * S + s];
      if (v != acc_identity(P.accs[a].kind)) merge_acc(P.accs[a].kind, tbl_acc(P.table, g, a, P.bucket_stride), v);
    }
  }
}

}  // namespace

// Returns false when the plan/batch shape is not covered (caller uses hash_agg_kernel).
bool launch_hash_agg_tile(const AggParams& P, unsigned long long capacity, unsigned int groups_hint, int64_t key_bytes, cudaStream_t stream) {
  if (P.pred_kind == 2) return false;
  for (int a = 0; a < P.n_acc; ++a) if (P.accs[a].arg_prog >= 0) return false;
  const int64_t n = P.n_rows;
  int cap = 0;
  if (P.key_kind == KEY_BYTES) {
    // hash_pass passes the key column's extent (the batch's own, or the plan's last-seen average × rows)
    const double avg = (n > 0 && key_bytes >= 0) ? (double)key_bytes / (double)n : 12.8;
    cap = (int)round_up((int64_t)(avg * HT_TILE * 1.0625) + 64, 1024);
    cap = std::max(4096, std::min(cap, 48 * 1024));
  }
  if (capacity > 2048 || (capacity & (capacity - 1)) || P.n_acc > 6) return false;
  // shared-memory table: 4× the groups last seen (short probe chains keep the lanes of a warp together), between 16
  // slots (tiny tables reduce inside the warp first) and the global capacity
  int log2_slots = 4;
  const unsigned long long want = groups_hint ? 4ull * groups_hint : capacity;
  while ((1ull << log2_slots) < want && (1ull << log2_slots) < capacity) ++log2_slots;
  const size_t copies = log2_slots <= 6 ? HT_THREADS / 32 : 1;
  const size_t smem = (cap ? cap + 32 : 0) + ((size_t)(16 + 8 * P.n_acc * copies) << log2_slots);
  static bool configured = false;
  if (!configured) {
    ARK_CUDA(cudaFuncSetAttribute(hash_agg_tile_kernel<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    ARK_CUDA(cudaFuncSetAttribute(hash_agg_tile_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    configured = true;
  }
  const int n_tiles = (int)ceil_div(n, HT_TILE);
  const int per_sm = (int)std::max<size_t>(1, std::min<size_t>(6, (200 * 1024) / std::max<size_t>(smem, 1)));
  const int grid = std::max(1, std::min(n_tiles, sm_count() * per_sm));
  KernelTimer t("hash_agg_tile_kernel", stream);
  if (P.pred_kind == 0) hash_agg_tile_kernel<0><<<grid, HT_THREADS, smem, stream>>>(P, cap, log2_slots);
  else hash_agg_tile_kernel<1><<<grid, HT_THREADS, smem, stream>>>(P, cap, log2_slots);
  return true;
}

}  // namespace ark
