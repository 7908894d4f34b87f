// filter_project_tma.cu — the fast path of filter + project + compaction for the common shape
//   SELECT <fixed-width columns…> [, <one Utf8/Binary column>] FROM t WHERE <col> <cmp> <literal>
// (BASELINE config 2: SELECT sensor, value FROM flow WHERE value >= 10), no NULLs in the used columns.
//
// Same single-pass algorithm as filter_project.cu (ticketed tiles, ballot ranking, decoupled
// look-back) with the data movement rebuilt around what each buffer needs:
//   * fixed-width columns never touch shared memory: one coalesced 8-byte load per row into a
//     register, and — because the 32 lanes of a warp hold 32 consecutive rows — the surviving lanes
//     store to CONSECUTIVE output slots, i.e. a warp-contiguous (coalesced) store without staging;
//   * the tile's string bytes form one contiguous, arbitrarily aligned byte range: a single 1-D TMA
//     bulk copy (cp.async.bulk → UBLKCP, completion on an mbarrier) drops the 16-byte-aligned window
//     around it into shared memory while the CTA evaluates the predicate and runs the look-back;
//   * strings are compacted shared→shared at word granularity (aligned source words funnel-shifted
//     into destination words) into a buffer that mirrors the destination's 16-byte alignment, then
//     leave as 16-byte vector stores.
// 1024-row tiles, 256 threads, ~33 KB shared memory per CTA ⇒ 6-7 CTAs per SM: look-back and load
// latency are hidden by CTA-level parallelism.  (A persistent 2-stage warp-specialised variant was
// slower than the generic kernel: with staging for inputs AND outputs only 2 tiles per SM were in
// flight and the look-back latency serialised each CTA.)
// Bulk copies only touch 16-byte blocks that contain at least one valid byte of the source buffer,
// so they never reach into an unmapped page.
#include <atomic>

#include "tma.cuh"
#include "batch.h"
#include "filter_project.cuh"
#include "vm.cuh"

#ifndef ARK_FP_MINBLOCKS
#define ARK_FP_MINBLOCKS 6
#endif

namespace ark {

namespace {

constexpr int T_MAX_FIXED_OUT = 2;

struct TmaParams {
  int64_t n_rows;
  int32_t n_tiles;
  int32_t n_fixed_out;
  int32_t has_varlen;
  int32_t str_cap;                          // bytes of shared memory per string buffer (multiple of 16)
  int32_t desc_stride;                      // u64 words between consecutive tile descriptors
  int32_t sp_is_f64, negate;                // predicate as a range test on the (totalOrder) key
  long long range_lo;
  unsigned long long range_span;            // keep ⇔ ((u64)(key - range_lo) <= range_span) != negate
  uint32_t fixed_is_pred;                   // bit c ⇒ fixed output c is the predicate column (already in registers)
  const unsigned long long* pred_in;        // predicate column
  const unsigned long long* fixed_in[T_MAX_FIXED_OUT];
  unsigned long long* fixed_out[T_MAX_FIXED_OUT];
  const int32_t* offsets_in;
  const uint8_t* data_in;
  int32_t* offsets_out;
  uint8_t* data_out;
  unsigned long long* desc;
  unsigned int* ticket;
  long long* totals;
  int32_t debug;                            // measurement knob (ARK_FP_DEBUG): bit 0 = skip the look-back (results are garbage)
  int32_t lb_windows;                       // tile kernel: 32-tile windows requested per look-back round (≤ 8)
  int32_t lb_mode;                          // tile kernel: 2 = two-level look-back (groups of 32 tiles), 1 = one chain of tiles
  int32_t lb_sleep, lb_delay;               // tile kernel: ns between polls of an unpublished descriptor / before the first poll
};

constexpr unsigned long long DESC_AGG = 1ull << 62;
constexpr unsigned long long DESC_PREFIX = 2ull << 62;

__device__ __forceinline__ unsigned long long ld_stream_u64(const unsigned long long* p) {
  unsigned long long v;
  asm volatile("ld.global.nc.L1::no_allocate.u64 %0, [%1];" : "=l"(v) : "l"(p));
  return v;
}
__device__ __forceinline__ unsigned long long ld_volatile_u64(const unsigned long long* p) {
  unsigned long long v;
  // descriptor traffic stays inside this GPU: relaxed.gpu (LDG.E.64.STRONG.GPU) — ld.volatile compiles to the system-scope form
  asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_volatile_u64(unsigned long long* p, unsigned long long v) {
  asm volatile("st.relaxed.gpu.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}

// Tile descriptor: [status:2 | rows:31 | bytes:31] in ONE 64-bit word, so both running sums travel (and
// change status) atomically.  A batch on this path has < 2^31 rows and < 2^31 string bytes.
__device__ __forceinline__ unsigned long long desc_pack(unsigned long long status, long long cnt, long long bytes) {
  return status | ((unsigned long long)cnt << 31) | (unsigned long long)bytes;
}
constexpr unsigned long long DESC_FIELD = (1ull << 31) - 1;
constexpr int LB_WINDOWS = 2;  // 2 × 32 predecessor tiles fetched per look-back round

// Forward progress without relying on CTA dispatch order.  A tile's look-back may only wait for tiles whose CTAs are
// running; with tile = blockIdx.x that holds when CTAs are dispatched in blockIdx order (what CUB's single-pass scans
// assume), but nothing in the programming model promises it (MPS, time slicing, a debugger, compute-sanitizer).  So a
// warp that has spun `spin_limit` times on an unpublished predecessor HELPS: it computes that tile's aggregate itself
// — the predicate over the tile's 1024 rows, 32 per lane — and publishes it with a CAS if it is still missing.  The
// aggregate is a pure function of the input, so helper and owner can only ever write the same value; the owner still
// publishes its inclusive prefix when it gets to run.  The fast path never executes this (`ARK_FP_DEBUG=4` forces it:
// tests/test_sql_filter_gpu.py).
template <bool VARLEN, int TT>
__device__ __forceinline__ void help_publish_aggregate(const TmaParams& P, int t, int lane) {
  const int64_t row0 = (int64_t)t * TT;
  const int rows = (int)((P.n_rows - row0) < TT ? (P.n_rows - row0) : TT);
  int cnt = 0, bytes = 0;
  for (int r = lane; r < rows; r += 32) {
    const unsigned long long v = P.pred_in[row0 + r];
    const long long key = P.sp_is_f64 ? f64_total_key(v) : (long long)v;
    bool f = (unsigned long long)(key - P.range_lo) <= P.range_span;
    f = f != (bool)P.negate;
    if (f) { ++cnt; if (VARLEN) bytes += P.offsets_in[row0 + r + 1] - P.offsets_in[row0 + r]; }
  }
  cnt = __reduce_add_sync(0xffffffffu, cnt);
  bytes = __reduce_add_sync(0xffffffffu, bytes);
  if (lane == 0) atomicCAS(P.desc + (size_t)t * P.desc_stride, 0ull, desc_pack(t == 0 ? DESC_PREFIX : DESC_AGG, cnt, bytes));
}

// Decoupled look-back, resolve half (warp 0).  The tile's aggregate is already published.
// The sustainable tile rate of a single-pass scan is (tiles inspected per round) / (round latency):
// at ~85 tiles/µs a 32-wide round with shuffle reductions (~0.4 µs) is exactly the limit, so the
// round is kept short — one volatile load per window, REDUX (`__reduce_add_sync`) instead of shuffle
// trees, the prefix tile's sums fetched with one shuffle — and two windows are in flight per round.
// HELP = false (the r1 / pipe kernels, kept for A/B runs): plain spinning, as in round 1.
// WINDOWS: compile-time upper bound of the windows per round; the tile kernel picks P.lb_windows ≤ WINDOWS at run time.
template <bool VARLEN, int TT = 1024, bool HELP = true, int WINDOWS = LB_WINDOWS>
__device__ void lookback_resolve(const TmaParams& P, int tile, long long agg_cnt, long long agg_bytes, int lane,
                                 long long* ex_cnt, long long* ex_bytes) {
  unsigned long long* const desc = P.desc;
  const int stride = P.desc_stride;
  const int spin_limit = (P.debug & 4) ? 2 : 4096;
  const int nw = HELP ? (P.lb_windows < WINDOWS ? P.lb_windows : WINDOWS) : WINDOWS;
  long long run_c = 0, run_b = 0;
  if (HELP && P.lb_delay) __nanosleep(P.lb_delay);
  if (tile > 0) {
    int look = tile - 1;
    bool done = false;
    while (!done) {
      // WINDOWS × 32 predecessor descriptors are requested before any is inspected: one L2 round trip per round
      unsigned long long dwin[WINDOWS];
#pragma unroll
      for (int w = 0; w < WINDOWS; ++w) {
        const int idxw = look - 32 * w - lane;
        dwin[w] = DESC_PREFIX;  // virtual tile -1: prefix 0
        if (w < nw && idxw >= 0) dwin[w] = ld_volatile_u64(desc + (size_t)idxw * stride);
      }
#pragma unroll
      for (int w = 0; w < WINDOWS; ++w) {
        if (!done && w < nw) {  // warp-uniform
          const int idx = look - 32 * w - lane;
          unsigned long long dw = dwin[w];
          int spins = 0;
          while (true) {  // a predecessor has not published yet
            const unsigned pending = __ballot_sync(0xffffffffu, (dw >> 62) == 0);
            if (!pending) break;
            if (HELP && ++spins > spin_limit) {  // not making progress: do the nearest missing tile's counting ourselves
              const int helped = __shfl_sync(0xffffffffu, idx, __ffs(pending) - 1);
              help_publish_aggregate<VARLEN, TT>(P, helped, lane);
              spins = 0;
            }
            if (HELP && P.lb_sleep) __nanosleep(P.lb_sleep);
            if ((dw >> 62) == 0) dw = ld_volatile_u64(desc + (size_t)idx * stride);
          }
          const unsigned pm = __ballot_sync(0xffffffffu, (dw >> 62) == 2);
          const int first = pm ? __ffs(pm) - 1 : 32;
          // aggregates of the tiles nearer than the first prefix tile (small numbers: REDUX on u32)
          const bool is_agg = lane < first;
          run_c += __reduce_add_sync(0xffffffffu, is_agg ? (unsigned)((dw >> 31) & DESC_FIELD) : 0u);
          run_b += __reduce_add_sync(0xffffffffu, is_agg ? (unsigned)(dw & DESC_FIELD) : 0u);
          if (pm) {
            const unsigned long long dp = __shfl_sync(0xffffffffu, dw, first);
            run_c += (long long)((dp >> 31) & DESC_FIELD);
            run_b += (long long)(dp & DESC_FIELD);
            done = true;
          }
        }
      }
      look -= nw * 32;
    }
    if (lane == 0) st_volatile_u64(desc + (size_t)tile * stride, desc_pack(DESC_PREFIX, run_c + agg_cnt, run_b + agg_bytes));
  }
  *ex_cnt = run_c; *ex_bytes = run_b;
}

// ---- two-level look-back -------------------------------------------------------------------------------
// A single chain of tile descriptors moves a prefix forward by one window (64 tiles) per L2 round trip, and the CTAs of
// one wave (every SM × 5-6 CTAs) publish their aggregates at about the same time — so the prefix crawls through every
// wave at a fixed tile rate whatever the byte rate.  Here tiles form groups of 32.  A tile sums the aggregates of the tiles before it in its
// own group (one window) and, at the same time, looks back over GROUP descriptors (one window = 32 groups = 1024 tiles,
// more than a wave), which the last tile of every group publishes: first the group's aggregate, then — after its own
// group-level look-back — the inclusive prefix.  No descriptor waits for a PREFIX that is itself waiting: every tile
// resolves two or three round trips after the aggregates around it exist.
// Group descriptors live behind the tile descriptors (same stride); the trailing partial group is never published.
template <bool VARLEN, int TT>
__device__ __forceinline__ void help_publish_group(const TmaParams& P, unsigned long long* gdesc, int g, int lane) {
  const int t = g * 32 + lane;  // only complete groups are ever waited for
  unsigned long long d = ld_volatile_u64(P.desc + (size_t)t * P.desc_stride);
  unsigned miss = __ballot_sync(0xffffffffu, (d >> 62) == 0);
  while (miss) {
    help_publish_aggregate<VARLEN, TT>(P, g * 32 + __ffs(miss) - 1, lane);
    miss &= miss - 1;
  }
  while ((d >> 62) == 0) d = ld_volatile_u64(P.desc + (size_t)t * P.desc_stride);  // owner or helper has published by now
  const unsigned c = __reduce_add_sync(0xffffffffu, (unsigned)((d >> 31) & DESC_FIELD));
  const unsigned b = __reduce_add_sync(0xffffffffu, (unsigned)(d & DESC_FIELD));
  if (lane == 0) atomicCAS(gdesc + (size_t)g * P.desc_stride, 0ull, desc_pack(g == 0 ? DESC_PREFIX : DESC_AGG, c, b));
}

template <bool VARLEN, int TT, bool HELP = true>
__device__ __forceinline__ void lookback_two_level(const TmaParams& P, int tile, long long agg_cnt, long long agg_bytes, int lane,
                                                   long long* ex_cnt, long long* ex_bytes) {
  unsigned long long* const desc = P.desc;
  const int stride = P.desc_stride;
  unsigned long long* const gdesc = desc + (size_t)P.n_tiles * stride;
  const int spin_limit = (P.debug & 4) ? 2 : 4096;
  const int g = tile >> 5, i = tile & 31;
  // both windows are requested before either is inspected
  if (P.lb_delay) __nanosleep(P.lb_delay);
  const int tidx = tile - 1 - lane;          // lanes < i: the tiles before this one in its group
  unsigned long long dt = DESC_AGG;          // other lanes: an empty aggregate
  if (lane < i) dt = ld_volatile_u64(desc + (size_t)tidx * stride);
  int look = g - 1;
  unsigned long long dg = DESC_PREFIX;       // virtual group -1: prefix 0
  if (look - lane >= 0) dg = ld_volatile_u64(gdesc + (size_t)(look - lane) * stride);
  for (int spins = 0;;) {
    const unsigned pending = __ballot_sync(0xffffffffu, (dt >> 62) == 0);
    if (!pending) break;
    if (HELP && ++spins > spin_limit) { help_publish_aggregate<VARLEN, TT>(P, tile - 1 - (__ffs(pending) - 1), lane); spins = 0; }
    if (P.lb_sleep) __nanosleep(P.lb_sleep);
    if ((dt >> 62) == 0) dt = ld_volatile_u64(desc + (size_t)tidx * stride);
  }
  const long long in_c = __reduce_add_sync(0xffffffffu, lane < i ? (unsigned)((dt >> 31) & DESC_FIELD) : 0u);
  const long long in_b = __reduce_add_sync(0xffffffffu, lane < i ? (unsigned)(dt & DESC_FIELD) : 0u);
  const bool closes_group = i == 31;
  if (closes_group && lane == 0) st_volatile_u64(gdesc + (size_t)g * stride, desc_pack(g == 0 ? DESC_PREFIX : DESC_AGG, in_c + agg_cnt, in_b + agg_bytes));
  long long run_c = 0, run_b = 0;
  if (g > 0) {
    for (;;) {
      const int idx = look - lane;
      for (int spins = 0;;) {
        const unsigned pending = __ballot_sync(0xffffffffu, (dg >> 62) == 0);
        if (!pending) break;
        if (HELP && ++spins > spin_limit) { help_publish_group<VARLEN, TT>(P, gdesc, look - (__ffs(pending) - 1), lane); spins = 0; }
        if (P.lb_sleep) __nanosleep(P.lb_sleep);
        if ((dg >> 62) == 0) dg = ld_volatile_u64(gdesc + (size_t)idx * stride);
      }
      const unsigned pm = __ballot_sync(0xffffffffu, (dg >> 62) == 2);
      const int first = pm ? __ffs(pm) - 1 : 32;
      const bool is_agg = lane < first;
      run_c += __reduce_add_sync(0xffffffffu, is_agg ? (unsigned)((dg >> 31) & DESC_FIELD) : 0u);
      run_b += __reduce_add_sync(0xffffffffu, is_agg ? (unsigned)(dg & DESC_FIELD) : 0u);
      if (pm) {
        const unsigned long long dp = __shfl_sync(0xffffffffu, dg, first);
        run_c += (long long)((dp >> 31) & DESC_FIELD);
        run_b += (long long)(dp & DESC_FIELD);
        break;
      }
      look -= 32;
      dg = DESC_PREFIX;
      if (look - lane >= 0) dg = ld_volatile_u64(gdesc + (size_t)(look - lane) * stride);
    }
    if (closes_group && lane == 0) st_volatile_u64(gdesc + (size_t)g * stride, desc_pack(DESC_PREFIX, run_c + in_c + agg_cnt, run_b + in_b + agg_bytes));
  }
  *ex_cnt = run_c + in_c; *ex_bytes = run_b + in_b;
}

// copy len bytes inside shared memory, word-granular on the destination
__device__ __forceinline__ void smem_copy(uint8_t* dst, const uint8_t* src, int len) {
  const unsigned d0 = smem_addr(dst), s0 = smem_addr(src);
  if (((d0 | s0 | (unsigned)len) & 3) == 0) {  // everything word aligned (fixed-length keys such as "temp_0000123")
    const unsigned* s = reinterpret_cast<const unsigned*>(src);
    unsigned* d = reinterpret_cast<unsigned*>(dst);
    if (len == 12) { const unsigned a = s[0], b = s[1], c = s[2]; d[0] = a; d[1] = b; d[2] = c; return; }
#pragma unroll 4
    for (int i = 0; i < (len >> 2); ++i) d[i] = s[i];
    return;
  }
  int i = 0;
  for (; i < len && ((d0 + i) & 3); ++i) dst[i] = src[i];  // head: up to 3 bytes
  const int words = (len - i) >> 2;
  if (words > 0) {
    const unsigned sa = s0 + i;
    const unsigned sh = (sa & 3) * 8;
    const unsigned* sw = reinterpret_cast<const unsigned*>(src + i - (sa & 3));  // aligned word holding src[i]
    unsigned* d = reinterpret_cast<unsigned*>(dst + i);
    if (sh == 0) {
      for (int w = 0; w < words; ++w) d[w] = sw[w];
    } else {
      unsigned lo = sw[0];
      for (int w = 0; w < words; ++w) {
        const unsigned hi = sw[w + 1];
        d[w] = __funnelshift_r(lo, hi, sh);
        lo = hi;
      }
    }
    i += words * 4;
  }
  for (; i < len; ++i) dst[i] = src[i];  // tail
}

__device__ __forceinline__ int warp_incl_scan(int v, int lane) {
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(0xffffffffu, v, o); if (lane >= o) v += t; }
  return v;
}

// Loads rows 4t..4t+3 of a tile: predicate values and (VARLEN) the 5 bounding offsets.
template <bool VARLEN>
__device__ __forceinline__ void load_rows(const TmaParams& P, int64_t row0, int rows, int lr0, int lane, unsigned long long pv[4], int off[5]) {
  const bool full = lr0 + 4 <= rows;
  const unsigned long long* src = P.pred_in + row0 + lr0;
  if (full && (reinterpret_cast<uintptr_t>(src) & 15) == 0) {
    asm volatile("ld.global.nc.L1::no_allocate.v2.u64 {%0, %1}, [%2];" : "=l"(pv[0]), "=l"(pv[1]) : "l"(src));
    asm volatile("ld.global.nc.L1::no_allocate.v2.u64 {%0, %1}, [%2];" : "=l"(pv[2]), "=l"(pv[3]) : "l"(src + 2));
  } else {
#pragma unroll
    for (int j = 0; j < 4; ++j) pv[j] = (lr0 + j < rows) ? src[j] : 0;
  }
  if (VARLEN) {
    const int32_t* os = P.offsets_in + row0 + lr0;
    if (full && (reinterpret_cast<uintptr_t>(os) & 15) == 0) {
      asm volatile("ld.global.nc.v4.s32 {%0, %1, %2, %3}, [%4];" : "=r"(off[0]), "=r"(off[1]), "=r"(off[2]), "=r"(off[3]) : "l"(os));
    } else {
#pragma unroll
      for (int j = 0; j < 4; ++j) off[j] = (lr0 + j <= rows) ? os[j] : 0;
    }
    off[4] = __shfl_down_sync(0xffffffffu, off[0], 1);
    if ((lane == 31 || lr0 + 4 >= rows) && lr0 + 4 <= rows) off[4] = os[4];
  }
}

template <bool VARLEN>
__device__ __forceinline__ unsigned eval_rows(const TmaParams& P, int rows, int lr0, const unsigned long long pv[4], const int off[5],
                                              int* cnt, int* sel_bytes) {
  unsigned flags = 0;
  int c = 0, sb = 0;
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const long long key = P.sp_is_f64 ? f64_total_key(pv[j]) : (long long)pv[j];
    bool f = (unsigned long long)(key - P.range_lo) <= P.range_span;
    f = (f != (bool)P.negate) && (lr0 + j < rows);
    flags |= (unsigned)f << j;
    c += f;
    if (VARLEN && f) sb += off[j + 1] - off[j];
  }
  *cnt = c; *sel_bytes = sb;
  return flags;
}

// Thread t owns rows 4t..4t+3 of the tile (blocked): two 16-byte loads per 8-byte column, one warp scan
// per quantity, thread-local ranks.
//
// The tile rate of a single-pass scan is bounded by the descriptor traffic, not by HBM: with descriptors
// packed 4 per 32-byte sector every variant of this kernel (with or without strings, look-back before or
// after staging, 32..256-tile rounds, aggregates published one CTA lifetime ahead by "scout" CTAs) ran at
// the same tile rate; one descriptor per sector raised it.  512-thread / 2048-row tiles were not faster.
template <int NF, bool VARLEN, int THREADS>
__global__ void __launch_bounds__(THREADS, THREADS == 256 ? ARK_FP_MINBLOCKS : 3) filter_project_tma_kernel(const __grid_constant__ TmaParams P) {
  constexpr int TT = THREADS * 4;          // rows per tile
  constexpr int T_WARPS = THREADS / 32;
  constexpr int T_THREADS = THREADS;
  extern __shared__ __align__(16) uint8_t smem[];   // [in_bytes: str_cap + 32][out_bytes: str_cap + 32]
  __shared__ __align__(8) unsigned long long s_bar;
  __shared__ int s_str_base, s_str_staged;
  __shared__ int s_cnt[T_WARPS], s_bytes[T_WARPS];
  __shared__ long long s_excl[2];

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  // tile = blockIdx.x relies on CTAs being dispatched in launch order (as CUB's single-pass scans assume); with a ticket
  // (ARK_FP_TICKET=1) a tile is only ever owned by a running CTA, whatever the dispatch order
  __shared__ int s_tile;
  int tile = blockIdx.x;
  if (P.ticket) {
    if (tid == 0) s_tile = (int)atomicAdd(P.ticket, 1u);
    __syncthreads();
    tile = s_tile;
    if (tile >= P.n_tiles) return;
  }
  const int64_t row0 = (int64_t)tile * TT;
  const int rows = (int)((P.n_rows - row0) < TT ? (P.n_rows - row0) : TT);
  uint8_t* in_bytes = smem;
  uint8_t* out_bytes = smem + P.str_cap + 32;

  if (VARLEN && tid == 0) {
    mbar_init(&s_bar, 1);
    mbar_fence_init();
    const int32_t o0 = P.offsets_in[row0], o1 = P.offsets_in[row0 + rows];
    const uintptr_t a0 = reinterpret_cast<uintptr_t>(P.data_in + o0), a1 = reinterpret_cast<uintptr_t>(P.data_in + o1);
    const uintptr_t lo = a0 & ~(uintptr_t)15, hi = (a1 + 15) & ~(uintptr_t)15;
    int staged = 0;
    if (o1 > o0 && hi - lo <= (uintptr_t)P.str_cap) {  // staged ⇒ selected bytes ≤ window ≤ str_cap
      staged = 1;
      mbar_expect_tx(&s_bar, (unsigned)(hi - lo));
      tma_load_1d(in_bytes, reinterpret_cast<const void*>(lo), (unsigned)(hi - lo), &s_bar);
    }
    s_str_base = o0 - (int32_t)(a0 - lo); s_str_staged = staged;
  }

  // ---- A: loads ----
  const int lr0 = 4 * tid;
  unsigned long long pv[4];
  int off[5] = {0, 0, 0, 0, 0};
  load_rows<VARLEN>(P, row0, rows, lr0, lane, pv, off);
  // ---- B: predicate, thread-local and warp-level prefix sums ----
  int cnt, sel_bytes;
  const unsigned flags = eval_rows<VARLEN>(P, rows, lr0, pv, off, &cnt, &sel_bytes);
  const int cnt_incl = warp_incl_scan(cnt, lane);
  int bytes_incl = 0;
  if (VARLEN) bytes_incl = warp_incl_scan(sel_bytes, lane);
  if (lane == 31) { s_cnt[warp] = cnt_incl; if (VARLEN) s_bytes[warp] = bytes_incl; }
  __syncthreads();

  // ---- D: tile scan over the per-warp totals (every warp, redundantly); publish the tile aggregate at once ----
  int w_cnt_excl, w_bytes_excl = 0, tile_cnt, tb = 0;
  {
    const int c = lane < T_WARPS ? s_cnt[lane] : 0;
    int incl = c;
#pragma unroll
    for (int o = 1; o < T_WARPS; o <<= 1) { const int t = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += t; }
    w_cnt_excl = __shfl_sync(0xffffffffu, incl - c, warp);
    tile_cnt = __shfl_sync(0xffffffffu, incl, T_WARPS - 1);
    if (VARLEN) {
      const int b = lane < T_WARPS ? s_bytes[lane] : 0;
      int bi = b;
#pragma unroll
      for (int o = 1; o < T_WARPS; o <<= 1) { const int t = __shfl_up_sync(0xffffffffu, bi, o); if (lane >= o) bi += t; }
      w_bytes_excl = __shfl_sync(0xffffffffu, bi - b, warp);
      tb = __shfl_sync(0xffffffffu, bi, T_WARPS - 1);
    }
  }
  if (warp == 0 && lane == 0) st_volatile_u64(P.desc + (size_t)tile * P.desc_stride, desc_pack(tile == 0 ? DESC_PREFIX : DESC_AGG, tile_cnt, tb));

  // ---- E: compact the strings in shared memory at tile-local positions ----
  const int my_cnt_excl = w_cnt_excl + cnt_incl - cnt;
  int lpos[4];
  bool str_fast = false;
  if (VARLEN) {
    int run = w_bytes_excl + bytes_incl - sel_bytes;
#pragma unroll
    for (int j = 0; j < 4; ++j) { lpos[j] = run; if ((flags >> j) & 1) run += off[j + 1] - off[j]; }
    str_fast = s_str_staged;
    if (str_fast) {
      mbar_wait(&s_bar, 0);  // TMA window landed (issued before phase A)
      const int base = s_str_base;
#pragma unroll
      for (int j = 0; j < 4; ++j)
        if ((flags >> j) & 1) smem_copy(out_bytes + lpos[j], in_bytes + (off[j] - base), off[j + 1] - off[j]);
    }
  }
  // ---- F: decoupled look-back (warp 0) ----
  if (warp == 0) {
    long long ex0, ex1;
    if (P.lb_mode == 2) lookback_two_level<VARLEN, TT, false>(P, tile, tile_cnt, tb, lane, &ex0, &ex1);
    else lookback_resolve<VARLEN, 1024, false>(P, tile, tile_cnt, tb, lane, &ex0, &ex1);
    if (lane == 0) { s_excl[0] = ex0; s_excl[1] = ex1; }
  }
  __syncthreads();
  const long long base_cnt = s_excl[0];
  const long long bb = VARLEN ? s_excl[1] : 0;
  if (tile == P.n_tiles - 1 && tid == 0) { P.totals[0] = base_cnt + tile_cnt; P.totals[1] = bb + tb; }

  // ---- G: stores ----
  {
    long long pos = base_cnt + my_cnt_excl;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      if (!((flags >> j) & 1)) continue;
#pragma unroll
      for (int c = 0; c < NF; ++c)
        P.fixed_out[c][pos] = ((P.fixed_is_pred >> c) & 1) ? pv[j] : ld_stream_u64(P.fixed_in[c] + row0 + lr0 + j);
      if (VARLEN) P.offsets_out[pos] = (int32_t)(bb + lpos[j]);
      ++pos;
    }
  }
  if (VARLEN) {
    if (tile == P.n_tiles - 1 && tid == 0) P.offsets_out[base_cnt + tile_cnt] = (int32_t)(bb + tb);
    if (str_fast) {
      // destination-aligned 16-byte stores; the shared-memory source is misaligned by d = (-bb) mod 16
      uint8_t* gdst = P.data_out + bb;
      const int head = (int)((16 - (bb & 15)) & 15) < tb ? (int)((16 - (bb & 15)) & 15) : tb;
      if (tid < head) gdst[tid] = out_bytes[tid];
      const int body = (tb - head) >> 4;
      const unsigned* sw = reinterpret_cast<const unsigned*>(out_bytes + (head & ~3));
      const unsigned sh = (head & 3) * 8;
      for (int g = tid; g < body; g += T_THREADS) {
        const unsigned* w = sw + g * 4;
        uint4 v;
        if (sh == 0) { v.x = w[0]; v.y = w[1]; v.z = w[2]; v.w = w[3]; }
        else {
          const unsigned a = w[0], b = w[1], c = w[2], d = w[3], e = w[4];
          v.x = __funnelshift_r(a, b, sh); v.y = __funnelshift_r(b, c, sh); v.z = __funnelshift_r(c, d, sh); v.w = __funnelshift_r(d, e, sh);
        }
        *reinterpret_cast<uint4*>(gdst + head + g * 16) = v;
      }
      const int done = head + body * 16;
      if (tid < tb - done) gdst[done + tid] = out_bytes[done + tid];
    } else {  // long strings: straight from global to global
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        if (!((flags >> j) & 1)) continue;
        const uint8_t* src = P.data_in + off[j];
        uint8_t* dst = P.data_out + bb + lpos[j];
        for (int i = 0; i < off[j + 1] - off[j]; ++i) dst[i] = src[i];
      }
    }
  }
}

// ================================================================================================
// filter_project_pipe_kernel — the same tile algorithm as a PERSISTENT, software-pipelined kernel with
// warp-striped rows.
//
// What a profile of filter_project_tma_kernel above shows: the LSU data pipe is the busiest unit and half of its
// shared-memory wavefronts are bank conflicts; L1 hands the crossbar about three times the output's bytes as
// stores; warps spend much of their time at the look-back barrier and waiting for the tile's own loads.  A thread there owns
// four CONSECUTIVE rows (two 16-byte loads per column), so the lanes of a warp touch strings 48 bytes apart in
// shared memory (4-way conflicts) and every store instruction sprays 32 partial sectors.  Here:
//   * rows are WARP-STRIPED: lane l of warp w owns rows 128 w + 32 j + l, j = 0..3.  For a given j the lanes
//     read consecutive 12-byte strings (conflict-free) and the surviving lanes write CONSECUTIVE output slots
//     (whole sectors); ranks come from ballots + popc instead of shuffle scans, and a warp whose 128 strings all
//     have the same length (ids, codes: the benchmark's "temp_%07d") derives byte positions from the ranks;
//   * the kernel is persistent and tiles come from a TICKET, so a tile is only ever owned by a running CTA and the
//     look-back cannot wait on a CTA that was never scheduled (the r1 kernel relied on blockIdx dispatch order);
//   * the loads of the NEXT tile — predicate column and offsets into registers, the string window by TMA into
//     the other half of a two-stage ring — are issued before the current tile is evaluated; a tile's aggregate
//     is published a few hundred cycles after its iteration starts, which keeps its successors' look-back short.
// Producer duties (ticket two tiles ahead, the tile's two bounding offsets one tile ahead, then the bulk copy)
// belong to one thread of the LAST warp, so that warp 0 keeps only the look-back.  The three tickets a CTA holds
// at start-up are claimed one dependent-load latency apart: a CTA must not own ADJACENT tiles, because it
// publishes them one iteration apart and every later tile's look-back would wait for that.
// ================================================================================================
template <bool VARLEN>
__device__ __forceinline__ void load_rows_striped(const TmaParams& P, int64_t row0, int rows, int wrow0, int lane, unsigned long long pv[4], int off[4],
                                                  int* offx) {
  const unsigned long long* src = P.pred_in + row0 + wrow0 + lane;
  const int32_t* os = P.offsets_in + row0 + wrow0 + lane;
  const bool full = wrow0 + 128 <= rows;
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const int r = wrow0 + 32 * j + lane;
    if (full || r < rows) asm volatile("ld.global.nc.L1::no_allocate.u64 %0, [%1];" : "=l"(pv[j]) : "l"(src + 32 * j));
    else pv[j] = 0;
    if (VARLEN) {
      if (full || r <= rows) asm volatile("ld.global.nc.L1::no_allocate.s32 %0, [%1];" : "=r"(off[j]) : "l"(os + 32 * j));
      else off[j] = 0;
    }
  }
  if (VARLEN) {  // offsets[first row of the next warp]: the end of lane 31's last string
    *offx = 0;
    if (lane == 31 && wrow0 + 128 <= rows) asm volatile("ld.global.nc.L1::no_allocate.s32 %0, [%1];" : "=r"(*offx) : "l"(os + 97));
  }
}

template <int NF, bool VARLEN, int MINB>
__global__ void __launch_bounds__(256, MINB) filter_project_pipe_kernel(const __grid_constant__ TmaParams P) {
  constexpr int T_THREADS = 256, TT = T_THREADS * 4, T_WARPS = T_THREADS / 32;
  constexpr int PRODUCER = T_THREADS - 32;  // lane 0 of the last warp
  extern __shared__ __align__(16) uint8_t smem[];   // [in_bytes stage 0][in_bytes stage 1][out_bytes], each str_cap + 32
  __shared__ __align__(8) unsigned long long s_bar[2];
  __shared__ int s_tile[4];
  __shared__ int s_str_base[2], s_str_staged[2];
  __shared__ int s_cnt[T_WARPS], s_bytes[T_WARPS];
  __shared__ long long s_excl[2];

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int wrow0 = warp * 128;
  const unsigned lt_mask = (1u << lane) - 1u;
  const int stage_bytes = P.str_cap + 32;
  uint8_t* const out_bytes = smem + 2 * stage_bytes;
  const int n_tiles = P.n_tiles;
  auto tile_rows = [&](int t) { const int64_t r = P.n_rows - (int64_t)t * TT; return (int)(r < TT ? r : TT); };
  // producer: arm stage `st` for the tile whose bounding offsets are o0, o1
  auto issue_window = [&](int st, int32_t o0, int32_t o1) {
    const uintptr_t a0 = reinterpret_cast<uintptr_t>(P.data_in + o0), a1 = reinterpret_cast<uintptr_t>(P.data_in + o1);
    const uintptr_t lo = a0 & ~(uintptr_t)15, hi = (a1 + 15) & ~(uintptr_t)15;
    int staged = 0;
    if (o1 > o0 && hi - lo <= (uintptr_t)P.str_cap) {  // staged ⇒ selected bytes ≤ window ≤ str_cap
      staged = 1;
      mbar_expect_tx(&s_bar[st], (unsigned)(hi - lo));
      tma_load_1d(smem + st * stage_bytes, reinterpret_cast<const void*>(lo), (unsigned)(hi - lo), &s_bar[st]);
    }
    s_str_base[st] = o0 - (int32_t)(a0 - lo); s_str_staged[st] = staged;
  };

  // ---- prologue: the CTA's first three tickets, each claimed only after the previous one's dependent loads ----
  unsigned tk_next = 0;
  int32_t bo0 = 0, bo1 = 0;  // bounding offsets of the NEXT tile (consumed when its bulk copy is issued)
  if (tid == PRODUCER) {
    if (VARLEN) { mbar_init(&s_bar[0], 1); mbar_init(&s_bar[1], 1); mbar_fence_init(); }
    const unsigned t0 = atomicAdd(P.ticket, 1u);
    s_tile[0] = (int)min(t0, (unsigned)n_tiles);
    unsigned dep = 0;  // makes the next claim wait for this tile's loads (separates the claims in time)
    if ((int)t0 < n_tiles) {
      const int64_t r0 = (int64_t)t0 * TT;
      if (VARLEN) { const int32_t o0 = P.offsets_in[r0], o1 = P.offsets_in[r0 + tile_rows((int)t0)]; issue_window(0, o0, o1); dep = (unsigned)(o0 ^ o1) & 0x80000000u; }
      else dep = (unsigned)(ld_volatile_u64(P.pred_in + r0) >> 63) & 0u;
    }
    const unsigned t1 = atomicAdd(P.ticket, 1u + dep);
    s_tile[1] = (int)min(t1, (unsigned)n_tiles);
    dep = 0;
    if ((int)t1 < n_tiles) {
      const int64_t r1 = (int64_t)t1 * TT;
      if (VARLEN) { bo0 = P.offsets_in[r1]; bo1 = P.offsets_in[r1 + tile_rows((int)t1)]; dep = (unsigned)(bo0 ^ bo1) & 0x80000000u; }
      else dep = (unsigned)(ld_volatile_u64(P.pred_in + r1) >> 63) & 0u;
    }
    tk_next = atomicAdd(P.ticket, 1u + dep);
  }
  __syncthreads();
  int tile = s_tile[0];
  unsigned long long pvn[4] = {0, 0, 0, 0};
  int offn[4] = {0, 0, 0, 0}, offxn = 0;
  if (tile < n_tiles) load_rows_striped<VARLEN>(P, (int64_t)tile * TT, tile_rows(tile), wrow0, lane, pvn, offn, &offxn);
  unsigned ph = 0;  // bit s: parity to wait for on stage s (flips only when a bulk copy was issued for it)

  for (int it = 0; tile < n_tiles; ++it) {
    const int st = it & 1;
    const int64_t row0 = (int64_t)tile * TT;
    const int rows = tile_rows(tile);
    uint8_t* const in_bytes = smem + st * stage_bytes;
    // this tile's registers (loaded one iteration ago)
    unsigned long long pv[4] = {pvn[0], pvn[1], pvn[2], pvn[3]};
    int off[4] = {offn[0], offn[1], offn[2], offn[3]};
    const int offx = offxn;
    // ---- A: everything the NEXT tile needs is put in flight now ----
    const int next = s_tile[(it + 1) & 3];
    if (tid == PRODUCER) {
      if (VARLEN && next < n_tiles) issue_window(st ^ 1, bo0, bo1);
      const int next2 = (int)min(tk_next, (unsigned)n_tiles);
      s_tile[(it + 2) & 3] = next2;
      if (VARLEN && next2 < n_tiles) { const int64_t r2 = (int64_t)next2 * TT; bo0 = P.offsets_in[r2]; bo1 = P.offsets_in[r2 + tile_rows(next2)]; }
      if (next2 < n_tiles) tk_next = atomicAdd(P.ticket, 1u);
    }
    if (next < n_tiles) load_rows_striped<VARLEN>(P, (int64_t)next * TT, tile_rows(next), wrow0, lane, pvn, offn, &offxn);
    // ---- B: predicate; ranks from ballots; byte positions ----
    unsigned flags = 0;
    int len[4] = {0, 0, 0, 0};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const long long key = P.sp_is_f64 ? f64_total_key(pv[j]) : (long long)pv[j];
      bool f = (unsigned long long)(key - P.range_lo) <= P.range_span;
      f = (f != (bool)P.negate) && (wrow0 + 32 * j + lane < rows);
      flags |= (unsigned)f << j;
    }
    if (VARLEN) {
      // end of row (j, lane) = start of row (j, lane + 1); lane 31: row (j + 1, 0), or the next warp's first row
      const int rows_w = rows - wrow0;  // rows of this warp's slice that exist (may be ≤ 0 or < 128 in the last tile)
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        int e = __shfl_down_sync(0xffffffffu, off[j], 1);
        const int nxt = j < 3 ? __shfl_sync(0xffffffffu, off[j < 3 ? j + 1 : 3], 0) : offx;
        if (lane == 31) e = nxt;
        len[j] = (32 * j + lane < rows_w) ? e - off[j] : 0;
      }
    }
    int wpos[4];  // rank of row (j, lane) among the warp's selected rows
    int warp_cnt = 0;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const unsigned m = __ballot_sync(0xffffffffu, (flags >> j) & 1);
      wpos[j] = warp_cnt + __popc(m & lt_mask);
      warp_cnt += __popc(m);
    }
    int bpos[4] = {0, 0, 0, 0};  // byte position of row (j, lane) among the warp's selected bytes
    int warp_bytes = 0;
    if (VARLEN) {
      const int len0 = __shfl_sync(0xffffffffu, len[0], 0);
      const bool same = (len[0] == len0 || wrow0 + lane >= rows) && (len[1] == len0 || wrow0 + 32 + lane >= rows) &&
                        (len[2] == len0 || wrow0 + 64 + lane >= rows) && (len[3] == len0 || wrow0 + 96 + lane >= rows);
      if (__all_sync(0xffffffffu, same)) {  // fixed-width strings: positions follow from the ranks
#pragma unroll
        for (int j = 0; j < 4; ++j) bpos[j] = wpos[j] * len0;
        warp_bytes = warp_cnt * len0;
      } else {
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int sl = ((flags >> j) & 1) ? len[j] : 0;
          const int incl = warp_incl_scan(sl, lane);
          bpos[j] = warp_bytes + incl - sl;
          warp_bytes += __shfl_sync(0xffffffffu, incl, 31);
        }
      }
    }
    if (lane == 0) { s_cnt[warp] = warp_cnt; if (VARLEN) s_bytes[warp] = warp_bytes; }
    // other projected fixed-width columns: requested now, stored after the look-back
    unsigned long long fx[NF > 0 ? NF : 1][4];
#pragma unroll
    for (int c = 0; c < NF; ++c) {
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        fx[c][j] = pv[j];
        if (!((P.fixed_is_pred >> c) & 1) && ((flags >> j) & 1)) fx[c][j] = ld_stream_u64(P.fixed_in[c] + row0 + wrow0 + 32 * j + lane);
      }
    }
    __syncthreads();   // (1)

    // ---- D: tile scan over the per-warp totals (every warp, redundantly); publish the tile aggregate at once ----
    int w_cnt_excl, w_bytes_excl = 0, tile_cnt, tb = 0;
    {
      const int c = lane < T_WARPS ? s_cnt[lane] : 0;
      int incl = c;
#pragma unroll
      for (int o = 1; o < T_WARPS; o <<= 1) { const int t = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += t; }
      w_cnt_excl = __shfl_sync(0xffffffffu, incl - c, warp);
      tile_cnt = __shfl_sync(0xffffffffu, incl, T_WARPS - 1);
      if (VARLEN) {
        const int b = lane < T_WARPS ? s_bytes[lane] : 0;
        int bi = b;
#pragma unroll
        for (int o = 1; o < T_WARPS; o <<= 1) { const int t = __shfl_up_sync(0xffffffffu, bi, o); if (lane >= o) bi += t; }
        w_bytes_excl = __shfl_sync(0xffffffffu, bi - b, warp);
        tb = __shfl_sync(0xffffffffu, bi, T_WARPS - 1);
      }
    }
    if (warp == 0 && lane == 0) st_volatile_u64(P.desc + (size_t)tile * P.desc_stride, desc_pack(tile == 0 ? DESC_PREFIX : DESC_AGG, tile_cnt, tb));
    // ---- F: decoupled look-back (warp 0) runs while the other warps compact the strings ----
    if (warp == 0) {
      long long ex0, ex1;
      if (P.debug & 1) { ex0 = (long long)tile * (TT / 2); ex1 = ex0 * 12; }
      else lookback_resolve<VARLEN, 1024, false>(P, tile, tile_cnt, tb, lane, &ex0, &ex1);
      if (lane == 0) { s_excl[0] = ex0; s_excl[1] = ex1; }
    }
    // ---- E: compact the strings in shared memory at tile-local positions ----
    bool str_fast = false;
    if (VARLEN) {
      str_fast = s_str_staged[st];
      if (str_fast) {
        mbar_wait(&s_bar[st], (ph >> st) & 1);  // this tile's window (issued one iteration ago)
        ph ^= 1u << st;
        const int base = s_str_base[st];
#pragma unroll
        for (int j = 0; j < 4; ++j)
          if ((flags >> j) & 1) smem_copy(out_bytes + w_bytes_excl + bpos[j], in_bytes + (off[j] - base), len[j]);
      }
    }
    __syncthreads();   // (2)
    const long long base_cnt = s_excl[0];
    const long long bb = VARLEN ? s_excl[1] : 0;
    if (tile == n_tiles - 1 && tid == 0) { P.totals[0] = base_cnt + tile_cnt; P.totals[1] = bb + tb; }

    // ---- G: stores — for each j the surviving lanes of a warp write consecutive slots ----
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      if (!((flags >> j) & 1)) continue;
      const long long pos = base_cnt + w_cnt_excl + wpos[j];
#pragma unroll
      for (int c = 0; c < NF; ++c) P.fixed_out[c][pos] = fx[c][j];
      if (VARLEN) P.offsets_out[pos] = (int32_t)(bb + w_bytes_excl + bpos[j]);
    }
    if (VARLEN) {
      if (tile == n_tiles - 1 && tid == 0) P.offsets_out[base_cnt + tile_cnt] = (int32_t)(bb + tb);
      if (str_fast) {
        // destination-aligned 16-byte stores; the shared-memory source is misaligned by d = (-bb) mod 16
        uint8_t* gdst = P.data_out + bb;
        const int head = (int)((16 - (bb & 15)) & 15) < tb ? (int)((16 - (bb & 15)) & 15) : tb;
        if (tid < head) gdst[tid] = out_bytes[tid];
        const int body = (tb - head) >> 4;
        const unsigned* sw = reinterpret_cast<const unsigned*>(out_bytes + (head & ~3));
        const unsigned sh = (head & 3) * 8;
        for (int g = tid; g < body; g += T_THREADS) {
          const unsigned* w = sw + g * 4;
          uint4 v;
          if (sh == 0) { v.x = w[0]; v.y = w[1]; v.z = w[2]; v.w = w[3]; }
          else {
            const unsigned a = w[0], b = w[1], c = w[2], d = w[3], e = w[4];
            v.x = __funnelshift_r(a, b, sh); v.y = __funnelshift_r(b, c, sh); v.z = __funnelshift_r(c, d, sh); v.w = __funnelshift_r(d, e, sh);
          }
          *reinterpret_cast<uint4*>(gdst + head + g * 16) = v;
        }
        const int done = head + body * 16;
        if (tid < tb - done) gdst[done + tid] = out_bytes[done + tid];
      } else {  // long strings: straight from global to global
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          if (!((flags >> j) & 1)) continue;
          const uint8_t* src = P.data_in + off[j];
          uint8_t* dst = P.data_out + bb + w_bytes_excl + bpos[j];
          for (int i = 0; i < len[j]; ++i) dst[i] = src[i];
        }
      }
    }
    tile = next;
    // out_bytes / s_cnt / s_excl are next written after barrier (1) resp. (2) of the following iteration — every
    // thread has finished this iteration's reads before it arrives there.
  }
}

// ================================================================================================
// filter_project_tile_kernel — the default.  Warp-striped rows (lane l of warp w owns rows 128w + 32j + l: coalesced
// 8-byte loads and stores, no shared-memory bank conflicts), ONE tile per CTA, a ninth warp that sets up the bulk copy of
// the tile's string bytes and runs the two-level look-back while the data warps compact the strings.
// On config 2 (2^24 rows):
//   * with the look-back stubbed out the kernel is the data path alone; the look-back adds the time a tile's CTA waits for
//     the aggregates of the tiles before it (their loads were issued at the same time and some always land late), during
//     which it holds its slot on the SM without having loads in flight.  5 CTAs per SM (40 registers x 288 threads) do not
//     cover it, and 7 CTAs at 32 registers spill.  2048-row tiles (DT = 512), a ticket instead of blockIdx, one chain of
//     tile descriptors instead of the two levels and the persistent pipelined kernel above (its CTAs wait for each other
//     in a convoy) were all slower.
//   * tried against that wait and dropped: "scout" CTAs that compute the aggregates of a whole group of 32 tiles ahead of
//     the tiles' own CTAs (one CTA cannot stream a group's inputs fast enough to stay ahead); the look-back warp of every
//     CTA computing the aggregate of the tile 64-2048 tiles ahead from a bulk copy of its predicate column and offsets,
//     before barrier (1) (it makes the CTA late) or after barrier (2) (extra L2 reads and a lingering warp).
//   * forward progress does not depend on CTA dispatch order: see help_publish_aggregate / help_publish_group.
// ================================================================================================
// MAXR: register cap (__maxnreg__): CTAs per SM follow from it — ptxas rounds a 288- / 544-thread CTA up when it derives
// the cap from __launch_bounds__'s minBlocks (544 threads, 3 blocks → 32 registers and spills instead of the 40 that fit)
template <int NF, bool VARLEN, int MAXR, int DT>
__global__ void __launch_bounds__(DT + 32) __maxnreg__(MAXR) filter_project_tile_kernel(const __grid_constant__ TmaParams P) {
  // warps 0..7: the tile's rows; warp 8: producer (tile id, bulk copy) and look-back — nothing but its own few values is
  // live there, so the (rare) call into help_publish_aggregate costs the data warps no registers and no spills
  // DT data threads: 256 (1024-row tiles) or 512 (2048-row tiles: half the descriptors on the look-back chain)
  constexpr int T_THREADS = DT, TT = T_THREADS * 4, T_WARPS = T_THREADS / 32, LB_WARP = T_WARPS;
  extern __shared__ __align__(16) uint8_t smem[];   // [in_bytes][out_bytes], each str_cap + 32
  __shared__ __align__(8) unsigned long long s_bar;
  __shared__ int s_tile;
  __shared__ int s_str_base, s_str_staged;
  __shared__ int s_cnt[T_WARPS], s_bytes[T_WARPS];
  __shared__ long long s_excl[2];

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int wrow0 = warp * 128;
  const unsigned lt_mask = (1u << lane) - 1u;
  uint8_t* const in_bytes = smem;
  uint8_t* const out_bytes = smem + P.str_cap + 32;
  const int n_tiles = P.n_tiles;
  // tile = blockIdx.x: no atomic on the CTA's critical path (a ticket — tiles in START order — makes every CTA wait ~1 µs
  // for its atomicAdd before it can issue a load; ARK_FP_TICKET=1 selects it).  Forward progress does not depend on the
  // dispatch order either way: see help_publish_aggregate.
  int tile = blockIdx.x;
  if (P.ticket) {
    if (tid == LB_WARP * 32) s_tile = (int)atomicAdd(P.ticket, 1u);
    __syncthreads();
    tile = s_tile;
  }
  if (tile >= n_tiles) return;
  // the data warps issue their loads at once; the window of string bytes is set up by the look-back warp meanwhile (its two
  // offset loads used to sit in front of a CTA-wide barrier: every tile started one memory latency late)
  if (VARLEN && tid == LB_WARP * 32) {
    mbar_init(&s_bar, 1); mbar_fence_init();
    const int64_t r0 = (int64_t)tile * TT;
    const int64_t rr = P.n_rows - r0;
    const int32_t o0 = P.offsets_in[r0], o1 = P.offsets_in[r0 + (rr < TT ? rr : TT)];
    const uintptr_t a0 = reinterpret_cast<uintptr_t>(P.data_in + o0), a1 = reinterpret_cast<uintptr_t>(P.data_in + o1);
    const uintptr_t lo = a0 & ~(uintptr_t)15, hi = (a1 + 15) & ~(uintptr_t)15;
    int staged = 0;
    if (o1 > o0 && hi - lo <= (uintptr_t)P.str_cap) {  // staged ⇒ selected bytes ≤ window ≤ str_cap
      staged = 1;
      mbar_expect_tx(&s_bar, (unsigned)(hi - lo));
      tma_load_1d(in_bytes, reinterpret_cast<const void*>(lo), (unsigned)(hi - lo), &s_bar);
    }
    s_str_base = o0 - (int32_t)(a0 - lo); s_str_staged = staged;   // read by the data warps after barrier (1)
  }
  if (warp == LB_WARP) {
    __syncthreads();   // (1): the data warps' totals are in shared memory
    int tile_cnt = lane < T_WARPS ? s_cnt[lane] : 0, tb = (VARLEN && lane < T_WARPS) ? s_bytes[lane] : 0;
    tile_cnt = __reduce_add_sync(0xffffffffu, tile_cnt);
    tb = __reduce_add_sync(0xffffffffu, tb);
    if ((P.debug & 4) && (tile % 37) == 5) __nanosleep(40000);  // test knob: a late tile, so that successors have to help
    if (lane == 0) st_volatile_u64(P.desc + (size_t)tile * P.desc_stride, desc_pack(tile == 0 ? DESC_PREFIX : DESC_AGG, tile_cnt, tb));
    long long ex0, ex1;
    if (P.debug & 1) { ex0 = (long long)tile * (TT / 2) + ((P.debug & 8) ? 3 : 0); ex1 = ex0 * 12 + ((P.debug & 8) ? 5 : 0); }  // bit 3: misaligned fake positions
    else if (P.lb_mode == 2) lookback_two_level<VARLEN, TT>(P, tile, tile_cnt, tb, lane, &ex0, &ex1);
    else lookback_resolve<VARLEN, TT, true, 2>(P, tile, tile_cnt, tb, lane, &ex0, &ex1);
    if (lane == 0) { s_excl[0] = ex0; s_excl[1] = ex1; }
    __syncthreads();   // (2)
    return;
  }
  const int64_t row0 = (int64_t)tile * TT;
  const int rows = (int)((P.n_rows - row0) < TT ? (P.n_rows - row0) : TT);
  unsigned long long pv[4];
  int off[4] = {0, 0, 0, 0}, offx = 0;
  load_rows_striped<VARLEN>(P, row0, rows, wrow0, lane, pv, off, &offx);
  // ---- B: predicate; ranks from ballots; byte positions ----
  unsigned flags = 0;
  int len[4] = {0, 0, 0, 0};
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const long long key = P.sp_is_f64 ? f64_total_key(pv[j]) : (long long)pv[j];
    bool f = (unsigned long long)(key - P.range_lo) <= P.range_span;
    f = (f != (bool)P.negate) && (wrow0 + 32 * j + lane < rows);
    flags |= (unsigned)f << j;
  }
  if (VARLEN) {
    // end of row (j, lane) = start of row (j, lane + 1); lane 31: row (j + 1, 0), or the next warp's first row
    const int rows_w = rows - wrow0;  // rows of this warp's slice that exist (may be ≤ 0 or < 128 in the last tile)
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      int e = __shfl_down_sync(0xffffffffu, off[j], 1);
      const int nxt = j < 3 ? __shfl_sync(0xffffffffu, off[j < 3 ? j + 1 : 3], 0) : offx;
      if (lane == 31) e = nxt;
      len[j] = (32 * j + lane < rows_w) ? e - off[j] : 0;
    }
  }
  int wpos[4];  // rank of row (j, lane) among the warp's selected rows
  int warp_cnt = 0;
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const unsigned m = __ballot_sync(0xffffffffu, (flags >> j) & 1);
    wpos[j] = warp_cnt + __popc(m & lt_mask);
    warp_cnt += __popc(m);
  }
  int bpos[4] = {0, 0, 0, 0};  // byte position of row (j, lane) among the warp's selected bytes
  int warp_bytes = 0;
  if (VARLEN) {
    const int len0 = __shfl_sync(0xffffffffu, len[0], 0);
    const bool same = (len[0] == len0 || wrow0 + lane >= rows) && (len[1] == len0 || wrow0 + 32 + lane >= rows) &&
                      (len[2] == len0 || wrow0 + 64 + lane >= rows) && (len[3] == len0 || wrow0 + 96 + lane >= rows);
    if (__all_sync(0xffffffffu, same)) {  // fixed-width strings: positions follow from the ranks
#pragma unroll
      for (int j = 0; j < 4; ++j) bpos[j] = wpos[j] * len0;
      warp_bytes = warp_cnt * len0;
    } else {
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int sl = ((flags >> j) & 1) ? len[j] : 0;
        const int incl = warp_incl_scan(sl, lane);
        bpos[j] = warp_bytes + incl - sl;
        warp_bytes += __shfl_sync(0xffffffffu, incl, 31);
      }
    }
  }
  if (lane == 0) { s_cnt[warp] = warp_cnt; if (VARLEN) s_bytes[warp] = warp_bytes; }
  // other projected fixed-width columns: requested now, stored after the look-back
  unsigned long long fx[NF > 0 ? NF : 1][4];
#pragma unroll
  for (int c = 0; c < NF; ++c) {
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      fx[c][j] = pv[j];
      if (!((P.fixed_is_pred >> c) & 1) && ((flags >> j) & 1)) fx[c][j] = ld_stream_u64(P.fixed_in[c] + row0 + wrow0 + 32 * j + lane);
    }
  }
  __syncthreads();

  // ---- D: tile scan over the per-warp totals (every warp, redundantly); publish the tile aggregate at once ----
  int w_cnt_excl, w_bytes_excl = 0, tile_cnt, tb = 0;
  {
    const int c = lane < T_WARPS ? s_cnt[lane] : 0;
    int incl = c;
#pragma unroll
    for (int o = 1; o < T_WARPS; o <<= 1) { const int t = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += t; }
    w_cnt_excl = __shfl_sync(0xffffffffu, incl - c, warp);
    tile_cnt = __shfl_sync(0xffffffffu, incl, T_WARPS - 1);
    if (VARLEN) {
      const int b = lane < T_WARPS ? s_bytes[lane] : 0;
      int bi = b;
#pragma unroll
      for (int o = 1; o < T_WARPS; o <<= 1) { const int t = __shfl_up_sync(0xffffffffu, bi, o); if (lane >= o) bi += t; }
      w_bytes_excl = __shfl_sync(0xffffffffu, bi - b, warp);
      tb = __shfl_sync(0xffffffffu, bi, T_WARPS - 1);
    }
  }
  // ---- E: compact the strings in shared memory at tile-local positions ----
  bool str_fast = false;
  if (VARLEN) {
    str_fast = s_str_staged;
    if (str_fast) {
      mbar_wait(&s_bar, 0);  // this tile's window
      const int base = s_str_base;
#pragma unroll
      for (int j = 0; j < 4; ++j)
        if ((flags >> j) & 1) smem_copy(out_bytes + w_bytes_excl + bpos[j], in_bytes + (off[j] - base), len[j]);
    }
  }
  __syncthreads();
  const long long base_cnt = s_excl[0];
  const long long bb = VARLEN ? s_excl[1] : 0;
  if (tile == n_tiles - 1 && tid == 0) { P.totals[0] = base_cnt + tile_cnt; P.totals[1] = bb + tb; }

  // ---- G: stores — for each j the surviving lanes of a warp write consecutive slots ----
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    if (!((flags >> j) & 1)) continue;
    const long long pos = base_cnt + w_cnt_excl + wpos[j];
#pragma unroll
    for (int c = 0; c < NF; ++c) P.fixed_out[c][pos] = fx[c][j];
    if (VARLEN) P.offsets_out[pos] = (int32_t)(bb + w_bytes_excl + bpos[j]);
  }
  if (VARLEN) {
    if (tile == n_tiles - 1 && tid == 0) P.offsets_out[base_cnt + tile_cnt] = (int32_t)(bb + tb);
    if (str_fast) {
      // destination-aligned 16-byte stores; the shared-memory source is misaligned by d = (-bb) mod 16
      uint8_t* gdst = P.data_out + bb;
      const int head = (int)((16 - (bb & 15)) & 15) < tb ? (int)((16 - (bb & 15)) & 15) : tb;
      if (tid < head) gdst[tid] = out_bytes[tid];
      const int body = (tb - head) >> 4;
      const unsigned* sw = reinterpret_cast<const unsigned*>(out_bytes + (head & ~3));
      const unsigned sh = (head & 3) * 8;
      for (int g = tid; g < body; g += T_THREADS) {
        const unsigned* w = sw + g * 4;
        uint4 v;
        if (sh == 0) { v.x = w[0]; v.y = w[1]; v.z = w[2]; v.w = w[3]; }
        else {
          const unsigned a = w[0], b = w[1], c = w[2], d = w[3], e = w[4];
          v.x = __funnelshift_r(a, b, sh); v.y = __funnelshift_r(b, c, sh); v.z = __funnelshift_r(c, d, sh); v.w = __funnelshift_r(d, e, sh);
        }
        *reinterpret_cast<uint4*>(gdst + head + g * 16) = v;
      }
      const int done = head + body * 16;
      if (tid < tb - done) gdst[done + tid] = out_bytes[done + tid];
    } else {  // long strings: straight from global to global
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        if (!((flags >> j) & 1)) continue;
        const uint8_t* src = P.data_in + off[j];
        uint8_t* dst = P.data_out + bb + w_bytes_excl + bpos[j];
        for (int i = 0; i < len[j]; ++i) dst[i] = src[i];
      }
    }
  }
}


// ================================================================================================
// filter_project_ring_kernel — persistent CTAs, every input of a tile by TMA, the store of tile k AFTER the count of tile k+1.
//
// One tile per CTA (above) leaves a CTA idle on its SM while the tiles before it publish their aggregates.  Here a CTA
// keeps two input stages and two output stages in shared memory:
//   * the producer (thread 0) issues the bulk copies of tile it+2 — predicate column, key offsets, string bytes — as soon
//     as every warp has consumed the stage of tile it: two tiles per CTA are always in flight, no registers involved;
//   * the data warps evaluate tile it from shared memory and compact the surviving values, tile-local offsets and
//     string bytes into OUTPUT stage it&1; warp 0 publishes the tile's aggregate at once;
//   * a ninth warp runs the two-level look-back of the tiles one after the other;
//   * the data warps store output stage (it-1)&1 — whose prefix the ninth warp has resolved meanwhile — with coalesced
//     stores, then go on to tile it+1.  The look-back latency of a tile overlaps the count phase of the next one.
// On config 2 (ARK_FP_IMPL=3) the look-back wait is hidden, but with two CTAs of nine warps per SM the serial chain of a
// tile (wait for the stage, LDS, ballots, barrier, STS, barrier, stores, barrier) is exposed and the data path itself is
// slower than the one-tile-per-CTA kernel's.  512-row tiles and four CTAs per SM: same data path, more descriptors.  Kept
// selectable, not the default: it is slower with two fixed-width outputs.
// ================================================================================================
constexpr int ring_pred_bytes(int tt) { return tt * 8 + 32; }
constexpr int ring_offs_bytes(int tt) { return ((tt + 1) * 4 + 32 + 15) / 16 * 16; }   // (tt + 1) offsets + alignment hull
// DT data threads, DT * 4 rows per tile: 256 (two CTAs per SM) or 128 (four: more independent tile chains per SM)
template <int NF, int NFX, int DT>
__global__ void __launch_bounds__(DT + 32) filter_project_ring_kernel(const __grid_constant__ TmaParams P) {
  constexpr int TT = DT * 4, T_THREADS = DT, T_WARPS = DT / 32, LB_WARP = T_WARPS;
  constexpr int RING_PRED_BYTES = ring_pred_bytes(TT), RING_OFFS_BYTES = ring_offs_bytes(TT);
  extern __shared__ __align__(16) uint8_t smem[];
  // Two input and two output stages.  Measured alternative: three input stages and ONE output stage (the store of tile k-1
  // between the count and the compaction of tile k) was slower — the longer serial chain per tile costs more than the
  // third tile in flight brings.
  constexpr int IN_STAGES = 2;
  __shared__ __align__(8) unsigned long long s_full[IN_STAGES], s_agg[2], s_res[2];
  __shared__ int s_shift[IN_STAGES][2 + (NFX > 0 ? NFX : 1)];
  __shared__ int s_str_base[IN_STAGES], s_str_staged[IN_STAGES];
  __shared__ int s_cnt[2][T_WARPS], s_bytes[2][T_WARPS];
  __shared__ int s_tot[2][2];
  __shared__ long long s_excl[2][2];

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int n_tiles = P.n_tiles;
  const int str_stage = P.str_cap + 32;
  const int in_bytes_per = RING_PRED_BYTES + RING_OFFS_BYTES + NFX * RING_PRED_BYTES + str_stage;
  const int out_bytes_per = NF * TT * 8 + (TT * 4 + 16) + str_stage;
  uint8_t* const in_base = smem;
  uint8_t* const out_base = smem + IN_STAGES * in_bytes_per;
  auto tile_of = [&](int it) { return (int)blockIdx.x + it * (int)gridDim.x; };
  auto tile_rows = [&](int t) { const int64_t r = P.n_rows - (int64_t)t * TT; return (int)(r < TT ? r : TT); };
  // fixed-width inputs that are not the predicate column, in the order of the outputs that use them
  const unsigned long long* fx_src[NFX > 0 ? NFX : 1];
  {
    int k = 0;
#pragma unroll
    for (int c = 0; c < NF; ++c) if (!((P.fixed_is_pred >> c) & 1) && k < NFX) fx_src[k++] = P.fixed_in[c];
    if (NFX == 0) fx_src[0] = nullptr;
  }
  // producer: every bulk copy of tile t into input stage st; (o0, o1) = the tile's bounding string offsets
  auto issue_tile = [&](int st, int t, int32_t o0, int32_t o1) {
    const int rows = tile_rows(t);
    uint8_t* stage = in_base + (size_t)st * in_bytes_per;
    const int64_t r0 = (int64_t)t * TT;
    uintptr_t lo[4 + NFX], hi[4 + NFX];
    unsigned total = 0;
    {
      const uintptr_t a0 = reinterpret_cast<uintptr_t>(P.pred_in + r0), a1 = a0 + (uintptr_t)rows * 8;
      lo[0] = a0 & ~(uintptr_t)15; hi[0] = (a1 + 15) & ~(uintptr_t)15; s_shift[st][0] = (int)(a0 - lo[0]);
    }
    {
      const uintptr_t a0 = reinterpret_cast<uintptr_t>(P.offsets_in + r0), a1 = a0 + (uintptr_t)(rows + 1) * 4;
      lo[1] = a0 & ~(uintptr_t)15; hi[1] = (a1 + 15) & ~(uintptr_t)15; s_shift[st][1] = (int)(a0 - lo[1]);
    }
#pragma unroll
    for (int k = 0; k < NFX; ++k) {
      const uintptr_t a0 = reinterpret_cast<uintptr_t>(fx_src[k] + r0), a1 = a0 + (uintptr_t)rows * 8;
      lo[2 + k] = a0 & ~(uintptr_t)15; hi[2 + k] = (a1 + 15) & ~(uintptr_t)15; s_shift[st][2 + k] = (int)(a0 - lo[2 + k]);
    }
    const uintptr_t s0 = reinterpret_cast<uintptr_t>(P.data_in + o0), s1 = reinterpret_cast<uintptr_t>(P.data_in + o1);
    const uintptr_t slo = s0 & ~(uintptr_t)15, shi = (s1 + 15) & ~(uintptr_t)15;
    const int staged = (o1 > o0 && shi - slo <= (uintptr_t)P.str_cap) ? 1 : 0;
    s_str_base[st] = o0 - (int32_t)(s0 - slo); s_str_staged[st] = staged;
    for (int k = 0; k < 2 + NFX; ++k) total += (unsigned)(hi[k] - lo[k]);
    if (staged) total += (unsigned)(shi - slo);
    mbar_expect_tx(&s_full[st], total);
    tma_load_1d(stage, reinterpret_cast<const void*>(lo[0]), (unsigned)(hi[0] - lo[0]), &s_full[st]);
    tma_load_1d(stage + RING_PRED_BYTES, reinterpret_cast<const void*>(lo[1]), (unsigned)(hi[1] - lo[1]), &s_full[st]);
#pragma unroll
    for (int k = 0; k < NFX; ++k)
      tma_load_1d(stage + RING_PRED_BYTES + RING_OFFS_BYTES + k * RING_PRED_BYTES, reinterpret_cast<const void*>(lo[2 + k]), (unsigned)(hi[2 + k] - lo[2 + k]), &s_full[st]);
    if (staged) tma_load_1d(stage + RING_PRED_BYTES + RING_OFFS_BYTES + NFX * RING_PRED_BYTES, reinterpret_cast<const void*>(slo), (unsigned)(shi - slo), &s_full[st]);
  };
  auto bounds_of = [&](int t, int32_t* o0, int32_t* o1) {
    const int64_t r0 = (int64_t)t * TT;
    *o0 = P.offsets_in[r0]; *o1 = P.offsets_in[r0 + tile_rows(t)];
  };

  int32_t no0 = 0, no1 = 0;  // producer: bounds of the tile it will issue next
  if (tid == 0) {
    for (int k = 0; k < IN_STAGES; ++k) mbar_init(&s_full[k], 1);
    for (int k = 0; k < 2; ++k) { mbar_init(&s_agg[k], 1); mbar_init(&s_res[k], 1); }
    mbar_fence_init();
    for (int k = 0; k < IN_STAGES; ++k)
      if (tile_of(k) < n_tiles) { int32_t o0, o1; bounds_of(tile_of(k), &o0, &o1); issue_tile(k, tile_of(k), o0, o1); }
    if (tile_of(IN_STAGES) < n_tiles) bounds_of(tile_of(IN_STAGES), &no0, &no1);
  }
  __syncthreads();

  if (warp == LB_WARP) {  // ---- look-back of this CTA's tiles, one after the other ----
    for (int it = 0; tile_of(it) < n_tiles; ++it) {
      const int st = it & 1, tile = tile_of(it);
      mbar_wait(&s_agg[st], (it >> 1) & 1);
      const long long tile_cnt = s_tot[st][0], tb = s_tot[st][1];
      long long ex0, ex1;
      if (P.debug & 1) { ex0 = (long long)tile * (TT / 2); ex1 = ex0 * 12; }
      else lookback_two_level<true, TT>(P, tile, tile_cnt, tb, lane, &ex0, &ex1);
      if (lane == 0) { s_excl[st][0] = ex0; s_excl[st][1] = ex1; }
      __syncwarp();
      if (lane == 0) mbar_arrive(&s_res[st]);
    }
    return;
  }

  const int wrow0 = warp * 128;
  const unsigned lt_mask = (1u << lane) - 1u;
  // store of the tile whose outputs sit in output stage pst
  auto store_tile = [&](int pit) {
    const int pst = pit & 1, tile = tile_of(pit);
    uint8_t* ostage = out_base + (size_t)pst * out_bytes_per;
    mbar_wait(&s_res[pst], (pit >> 1) & 1);
    const long long base_cnt = s_excl[pst][0], bb = s_excl[pst][1];
    const int cnt = s_tot[pst][0], tb = s_tot[pst][1];
    const int32_t* ooff = reinterpret_cast<const int32_t*>(ostage + NF * TT * 8);
    const uint8_t* ostr = ostage + NF * TT * 8 + TT * 4 + 16;
#pragma unroll
    for (int c = 0; c < NF; ++c) {
      const unsigned long long* of = reinterpret_cast<const unsigned long long*>(ostage + c * TT * 8);
      unsigned long long* g = P.fixed_out[c] + base_cnt;
      for (int i = tid; i < cnt; i += T_THREADS) g[i] = of[i];
    }
    for (int i = tid; i < cnt; i += T_THREADS) P.offsets_out[base_cnt + i] = (int32_t)(bb + ooff[i]);
    if (tile == n_tiles - 1 && tid == 0) { P.totals[0] = base_cnt + cnt; P.totals[1] = bb + tb; P.offsets_out[base_cnt + cnt] = (int32_t)(bb + tb); }
    if (ooff[TT]) {  // staged flag, kept behind the offsets
      uint8_t* gdst = P.data_out + bb;
      const int head = (int)((16 - (bb & 15)) & 15) < tb ? (int)((16 - (bb & 15)) & 15) : tb;
      if (tid < head) gdst[tid] = ostr[tid];
      const int body = (tb - head) >> 4;
      const unsigned* sw = reinterpret_cast<const unsigned*>(ostr + (head & ~3));
      const unsigned sh = (head & 3) * 8;
      for (int g = tid; g < body; g += T_THREADS) {
        const unsigned* w = sw + g * 4;
        uint4 v;
        if (sh == 0) { v.x = w[0]; v.y = w[1]; v.z = w[2]; v.w = w[3]; }
        else {
          const unsigned a = w[0], b = w[1], c = w[2], d = w[3], e = w[4];
          v.x = __funnelshift_r(a, b, sh); v.y = __funnelshift_r(b, c, sh); v.z = __funnelshift_r(c, d, sh); v.w = __funnelshift_r(d, e, sh);
        }
        *reinterpret_cast<uint4*>(gdst + head + g * 16) = v;
      }
      const int done = head + body * 16;
      if (tid < tb - done) gdst[done + tid] = ostr[done + tid];
    } else {  // strings too long for the stage: the string region holds the source offset of every surviving row
      const int32_t* osrc = reinterpret_cast<const int32_t*>(ostr);
      for (int i = tid; i < cnt; i += T_THREADS) {
        const int len = (i + 1 < cnt ? ooff[i + 1] : tb) - ooff[i];
        const uint8_t* src = P.data_in + osrc[i];
        uint8_t* dst = P.data_out + bb + ooff[i];
        for (int b = 0; b < len; ++b) dst[b] = src[b];
      }
    }
  };

  int it = 0;
  for (; tile_of(it) < n_tiles; ++it) {
    const int st = it & 1, ist = it % IN_STAGES, tile = tile_of(it);
    const int rows = tile_rows(tile);
    const uint8_t* istage = in_base + (size_t)ist * in_bytes_per;
    uint8_t* ostage = out_base + (size_t)st * out_bytes_per;
    mbar_wait(&s_full[ist], (it / IN_STAGES) & 1);
    const unsigned long long* spred = reinterpret_cast<const unsigned long long*>(istage + s_shift[ist][0]);
    const int32_t* soff = reinterpret_cast<const int32_t*>(istage + RING_PRED_BYTES + s_shift[ist][1]);
    const bool staged = s_str_staged[ist];
    const uint8_t* sstr = istage + RING_PRED_BYTES + RING_OFFS_BYTES + NFX * RING_PRED_BYTES;
    const int str_base = s_str_base[ist];
    // ---- predicate, ranks, byte positions (rows striped over the warp) ----
    unsigned long long pv[4];
    int off[4], len[4];
    unsigned flags = 0;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int r = wrow0 + 32 * j + lane;
      const bool in = r < rows;
      pv[j] = in ? spred[r] : 0ull;
      off[j] = in ? soff[r] : 0;
      len[j] = in ? soff[r + 1] - off[j] : 0;
      const long long key = P.sp_is_f64 ? f64_total_key(pv[j]) : (long long)pv[j];
      bool f = (unsigned long long)(key - P.range_lo) <= P.range_span;
      f = (f != (bool)P.negate) && in;
      flags |= (unsigned)f << j;
    }
    int wpos[4], warp_cnt = 0;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const unsigned m = __ballot_sync(0xffffffffu, (flags >> j) & 1);
      wpos[j] = warp_cnt + __popc(m & lt_mask);
      warp_cnt += __popc(m);
    }
    int bpos[4] = {0, 0, 0, 0}, warp_bytes = 0;
    {
      const int len0 = __shfl_sync(0xffffffffu, len[0], 0);
      const bool same = (len[0] == len0 || wrow0 + lane >= rows) && (len[1] == len0 || wrow0 + 32 + lane >= rows) &&
                        (len[2] == len0 || wrow0 + 64 + lane >= rows) && (len[3] == len0 || wrow0 + 96 + lane >= rows);
      if (__all_sync(0xffffffffu, same)) {
#pragma unroll
        for (int j = 0; j < 4; ++j) bpos[j] = wpos[j] * len0;
        warp_bytes = warp_cnt * len0;
      } else {
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int sl = ((flags >> j) & 1) ? len[j] : 0;
          const int incl = warp_incl_scan(sl, lane);
          bpos[j] = warp_bytes + incl - sl;
          warp_bytes += __shfl_sync(0xffffffffu, incl, 31);
        }
      }
    }
    if (lane == 0) { s_cnt[st][warp] = warp_cnt; s_bytes[st][warp] = warp_bytes; }
    bar_sync(1, T_THREADS);  // (A')
    int w_cnt_excl, w_bytes_excl, tile_cnt, tb;
    {
      const int c = lane < T_WARPS ? s_cnt[st][lane] : 0;
      int incl = c;
#pragma unroll
      for (int o = 1; o < T_WARPS; o <<= 1) { const int t = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += t; }
      w_cnt_excl = __shfl_sync(0xffffffffu, incl - c, warp);
      tile_cnt = __shfl_sync(0xffffffffu, incl, T_WARPS - 1);
      const int b = lane < T_WARPS ? s_bytes[st][lane] : 0;
      int bi = b;
#pragma unroll
      for (int o = 1; o < T_WARPS; o <<= 1) { const int t = __shfl_up_sync(0xffffffffu, bi, o); if (lane >= o) bi += t; }
      w_bytes_excl = __shfl_sync(0xffffffffu, bi - b, warp);
      tb = __shfl_sync(0xffffffffu, bi, T_WARPS - 1);
    }
    if (tid == 0) {  // the aggregate is public before anything else happens to this tile
      st_volatile_u64(P.desc + (size_t)tile * P.desc_stride, desc_pack(tile == 0 ? DESC_PREFIX : DESC_AGG, tile_cnt, tb));
      s_tot[st][0] = tile_cnt; s_tot[st][1] = tb;
      mbar_arrive(&s_agg[st]);
    }
    // ---- compaction into output stage st at tile-local positions ----
    int32_t* ooff = reinterpret_cast<int32_t*>(ostage + NF * TT * 8);
    uint8_t* ostr = ostage + NF * TT * 8 + TT * 4 + 16;
    if (tid == 0) ooff[TT] = staged ? 1 : 0;
    {
      int kx = 0;
#pragma unroll
      for (int c = 0; c < NF; ++c) {
        unsigned long long* of = reinterpret_cast<unsigned long long*>(ostage + c * TT * 8);
        const bool is_pred = (P.fixed_is_pred >> c) & 1;
        const unsigned long long* sfx = nullptr;
        if (!is_pred && NFX > 0) { sfx = reinterpret_cast<const unsigned long long*>(istage + RING_PRED_BYTES + RING_OFFS_BYTES + kx * RING_PRED_BYTES + s_shift[ist][2 + (kx < NFX ? kx : 0)]); ++kx; }
#pragma unroll
        for (int j = 0; j < 4; ++j)
          if ((flags >> j) & 1) of[w_cnt_excl + wpos[j]] = is_pred ? pv[j] : sfx[wrow0 + 32 * j + lane];
      }
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      if (!((flags >> j) & 1)) continue;
      ooff[w_cnt_excl + wpos[j]] = w_bytes_excl + bpos[j];
      if (staged) smem_copy(ostr + w_bytes_excl + bpos[j], sstr + (off[j] - str_base), len[j]);
      else reinterpret_cast<int32_t*>(ostr)[w_cnt_excl + wpos[j]] = off[j];
    }
    bar_sync(1, T_THREADS);  // (A): input stage ist is consumed, the output stage is complete
    if (tid == 0) {
      const int t2 = tile_of(it + IN_STAGES);
      if (t2 < n_tiles) issue_tile(ist, t2, no0, no1);
      const int t3 = tile_of(it + IN_STAGES + 1);
      if (t3 < n_tiles) bounds_of(t3, &no0, &no1);
    }
    // ---- the previous tile's outputs leave now: its prefix was resolved while this tile was counted ----
    if (it > 0) store_tile(it - 1);
    bar_sync(2, T_THREADS);  // (B): output stage (it-1)&1 may be overwritten by tile it+1
  }
  if (it > 0) store_tile(it - 1);
}

}  // namespace

static std::atomic<double> g_avg_len_hint{12.8};
void filter_project_tma_note_avg_len(double avg) { if (avg > 0) g_avg_len_hint.store(avg); }
static int g_fp_threads = [] { const char* e = getenv("ARK_FP_THREADS"); const int v = e ? atoi(e) : 256; return v == 512 || v == 128 ? v : 256; }();
static int g_desc_stride = [] { const char* e = getenv("ARK_FP_DESC_STRIDE"); int v = e ? atoi(e) : 4; return v >= 1 && v <= 16 ? v : 4; }();  // one descriptor per 32-byte sector
int filter_project_tma_tile_rows() { return g_fp_threads * 4; }
int filter_project_tma_desc_stride() { return g_desc_stride; }
// u64 words of descriptor scratch for n_tiles tiles: the tile descriptors, then one descriptor per group of 32 tiles
size_t filter_project_tma_desc_words(int64_t n_tiles) { return (size_t)(n_tiles + (n_tiles + 31) / 32) * (size_t)g_desc_stride; }
int filter_project_tma_max_fixed_out() { return T_MAX_FIXED_OUT; }

// Returns false when the inputs do not meet the alignment rules of this path (caller falls back).
bool launch_filter_project_tma(int64_t n_rows, const void* pred_in, int n_fixed_out, const void* const* fixed_in, void* const* fixed_out,
                               const int32_t* offsets_in, const uint8_t* data_in, int64_t data_bytes, int32_t* offsets_out, uint8_t* data_out,
                               int cmp, int is_f64, uint64_t constant, unsigned long long* desc, unsigned int* ticket, long long* totals,
                               cudaStream_t stream) {
  if (reinterpret_cast<uintptr_t>(pred_in) & 7) return false;
  if (n_rows >= (1ll << 31) - 1) return false;  // 31-bit descriptor fields
  if (data_out && (reinterpret_cast<uintptr_t>(data_out) & 15)) return false;
  if (n_fixed_out > 2) return false;
  TmaParams P;
  memset(&P, 0, sizeof P);
  const int TT = g_fp_threads * 4;
  P.n_rows = n_rows; P.n_tiles = (int)ceil_div(n_rows, TT); P.n_fixed_out = n_fixed_out; P.has_varlen = offsets_in != nullptr;
  P.sp_is_f64 = is_f64;
  {  // comparison against a constant → range membership on the totally ordered int64 key
    long long c = (long long)constant;
    if (is_f64) c = c ^ (long long)(((unsigned long long)(c >> 63)) >> 1);  // f64 totalOrder key
    const long long MIN = INT64_MIN, MAX = INT64_MAX;
    long long lo = MIN, hi = MAX; int neg = 0;
    switch (cmp) {
      case CMP_EQ: lo = hi = c; break;
      case CMP_NE: lo = hi = c; neg = 1; break;
      case CMP_LT: if (c == MIN) neg = 1; else hi = c - 1; break;   // empty set = NOT(everything)
      case CMP_LE: hi = c; break;
      case CMP_GT: if (c == MAX) neg = 1; else lo = c + 1; break;
      default: lo = c; break;  // GE
    }
    P.range_lo = lo; P.range_span = (unsigned long long)hi - (unsigned long long)lo; P.negate = neg;
  }
  P.pred_in = (const unsigned long long*)pred_in;
  for (int c = 0; c < n_fixed_out; ++c) {
    P.fixed_in[c] = (const unsigned long long*)fixed_in[c]; P.fixed_out[c] = (unsigned long long*)fixed_out[c];
    if (fixed_in[c] == pred_in) P.fixed_is_pred |= 1u << c;
  }
  P.offsets_in = offsets_in; P.data_in = data_in; P.offsets_out = offsets_out; P.data_out = data_out;
  P.desc = desc; P.ticket = ticket; P.totals = totals;
  static const int debug = [] { const char* e = getenv("ARK_FP_DEBUG"); return e ? atoi(e) : 0; }();
  P.debug = debug;
  static const int lbw = [] { const char* e = getenv("ARK_FP_LB_WINDOWS"); const int v = e ? atoi(e) : 4; return v >= 1 && v <= 8 ? v : 4; }();
  P.lb_windows = lbw;
  static const int lb_mode = [] { const char* e = getenv("ARK_FP_LB"); return e && atoi(e) == 1 ? 1 : 2; }();
  P.lb_mode = lb_mode;
  static const int lb_sleep = [] { const char* e = getenv("ARK_FP_LB_SLEEP"); return e ? atoi(e) : 0; }();
  // the look-back warp sleeps this long before its first poll: the aggregates it needs belong to tiles whose loads were issued
  // at about the same time as its own, and the 60-odd descriptor loads of a poll that finds them missing are wasted L2
  // requests (measured on 2^24 rows over 0-1500 ns: shortest around 800-1000 ns)
  static const int lb_delay = [] { const char* e = getenv("ARK_FP_LB_DELAY"); return e ? atoi(e) : 800; }();
  P.lb_sleep = lb_sleep; P.lb_delay = lb_delay;
  // string staging sized from the batch's average string length (+25 %), 2 KB granules, 4..24 KB
  int cap = 0;
  if (P.has_varlen) {
    // exact when the extent is known; otherwise the average selected-string length of the previous launch
    double avg = n_rows > 0 && data_bytes >= 0 ? (double)data_bytes / (double)n_rows : g_avg_len_hint.load();
    static const double slack = [] { const char* e = getenv("ARK_FP_CAP_SLACK"); return e ? atof(e) : 1.0625; }();
    cap = (int)round_up((int64_t)(avg * TT * slack) + 64, 1024);
    cap = std::max(TT >= 1024 ? 4096 : 2048, std::min(cap, std::max(TT / 1024, 1) * 24 * 1024));
  }
  P.str_cap = cap;
  P.desc_stride = g_desc_stride;
  const bool v = P.has_varlen;
  // implementation: 2 = striped rows, one ticketed tile per CTA (default); 0 = persistent pipelined striped kernel;
  // 1 = the r1 kernel (blocked rows, tile = blockIdx).  0 and 1 are kept for A/B runs.
  static const int impl = [] { const char* e = getenv("ARK_FP_IMPL"); return e ? atoi(e) : 2; }();
  if (g_fp_threads == 128 && (impl != 3 || !v)) return false;  // 512-row tiles: the ring kernel only
  if (impl == 3 && v && ticket != nullptr && g_fp_threads <= 256) {
    int nfx = 0;
    for (int c = 0; c < n_fixed_out; ++c) if (!((P.fixed_is_pred >> c) & 1)) ++nfx;
    const int dt = g_fp_threads, tt = dt * 4;
    const size_t in_per = (size_t)ring_pred_bytes(tt) + ring_offs_bytes(tt) + (size_t)nfx * ring_pred_bytes(tt) + (size_t)cap + 32;
    const size_t out_per = (size_t)n_fixed_out * tt * 8 + tt * 4 + 16 + (size_t)cap + 32;
    const size_t smem = 2 * in_per + 2 * out_per;
    const void* fn = nullptr;
#define ARK_RING_FN(NF, NFX) (dt == 128 ? (const void*)filter_project_ring_kernel<NF, NFX, 128> : (const void*)filter_project_ring_kernel<NF, NFX, 256>)
    if (n_fixed_out == 0) fn = ARK_RING_FN(0, 0);
    else if (n_fixed_out == 1 && nfx == 0) fn = ARK_RING_FN(1, 0);
    else if (n_fixed_out == 1 && nfx == 1) fn = ARK_RING_FN(1, 1);
    else if (n_fixed_out == 2 && nfx == 1) fn = ARK_RING_FN(2, 1);
    if (fn && smem <= 112 * 1024) {   // at least two CTAs per SM; otherwise the one-tile-per-CTA kernel below
      static bool configured = false;
      if (!configured) {
        for (const void* f : {ARK_RING_FN(0, 0), ARK_RING_FN(1, 0), ARK_RING_FN(1, 1), ARK_RING_FN(2, 1)})
          ARK_CUDA(cudaFuncSetAttribute(f, cudaFuncAttributeMaxDynamicSharedMemorySize, 112 * 1024));
        configured = true;
      }
#undef ARK_RING_FN
      int occ = 0;
      ARK_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, fn, dt + 32, smem));
      if (occ >= 1) {
        const int sms = sm_count();
        static const int cap_per_sm = [] { const char* e = getenv("ARK_FP_CTAS_PER_SM"); return e ? atoi(e) : 0; }();
        if (cap_per_sm > 0) occ = std::min(occ, cap_per_sm);
        const int grid = std::max(1, std::min(P.n_tiles, sms * occ));
        KernelTimer t("filter_project_tma_kernel", stream, "filter_project_ring_kernel");
        void* args[] = {(void*)&P};
        ARK_CUDA(cudaLaunchKernel(fn, dim3(grid), dim3(dt + 32), args, smem, stream));
        return true;
      }
    }
    if (dt == 128) return false;  // 512-row tiles exist for this kernel only
  }
  if ((impl == 2 || impl == 3) && ticket != nullptr) {
    static const bool use_ticket = [] { const char* e = getenv("ARK_FP_TICKET"); return e && atoi(e) != 0; }();
    if (!use_ticket) P.ticket = nullptr;
    const size_t smem = v ? 2 * (size_t)(cap + 32) : 0;
    // data threads per CTA: g_fp_threads (ARK_FP_THREADS = 256 | 512); register cap: ARK_FP_MAXR (40 | 48 | 56)
    static const int maxr = [] { const char* e = getenv("ARK_FP_MAXR"); const int x = e ? atoi(e) : 40; return x == 32 || x == 48 || x == 56 ? x : 40; }();
    const int dt = g_fp_threads;
#define ARK_TILE_R(NF, V, D) (maxr == 56 ? (const void*)filter_project_tile_kernel<NF, V, 56, D> : maxr == 48 ? (const void*)filter_project_tile_kernel<NF, V, 48, D> \
                              : maxr == 32 ? (const void*)filter_project_tile_kernel<NF, V, 32, D> : (const void*)filter_project_tile_kernel<NF, V, 40, D>)
#define ARK_TILE_FN(NF, V) (dt == 512 ? ARK_TILE_R(NF, V, 512) : ARK_TILE_R(NF, V, 256))
    static bool configured = false;
    if (!configured) {
      for (const void* f : {ARK_TILE_FN(0, true), ARK_TILE_FN(1, true), ARK_TILE_FN(2, true)})
        ARK_CUDA(cudaFuncSetAttribute(f, cudaFuncAttributeMaxDynamicSharedMemorySize, 2 * (2 * 24 * 1024 + 32)));
      configured = true;
    }
    const void* fn = nullptr;
    if (n_fixed_out == 0 && v) fn = ARK_TILE_FN(0, true);
    else if (n_fixed_out == 1 && v) fn = ARK_TILE_FN(1, true);
    else if (n_fixed_out == 2 && v) fn = ARK_TILE_FN(2, true);
    else if (n_fixed_out == 1) fn = ARK_TILE_FN(1, false);
    else if (n_fixed_out == 2) fn = ARK_TILE_FN(2, false);
    else return false;
#undef ARK_TILE_FN
#undef ARK_TILE_R
    KernelTimer t("filter_project_tma_kernel", stream, "filter_project_tile_kernel");
    void* args[] = {(void*)&P};
    ARK_CUDA(cudaLaunchKernel(fn, dim3(P.n_tiles), dim3(dt + 32), args, smem, stream));
    return true;
  }
  if (impl == 0 && g_fp_threads == 256 && ticket != nullptr) {
    const size_t smem = v ? 3 * (size_t)(cap + 32) : 0;
    static int occ[2][3] = {{0, 0, 0}, {0, 0, 0}};   // CTAs per SM by (varlen, n_fixed) at the largest staging size seen
    static size_t occ_smem[2][3] = {{0, 0, 0}, {0, 0, 0}};
    static bool configured = false;
    const int max_smem = 3 * (48 * 1024 + 32);
    // CTAs per SM the kernel is compiled for: 4 (64 registers, the default) or 5 (48 registers, a few spilled words)
    static const int minb = [] { const char* e = getenv("ARK_FP_MINB"); const int v = e ? atoi(e) : 4; return v == 3 || v == 5 ? v : 4; }();
#define ARK_PIPE_FN(NF, V) (minb == 4 ? (const void*)filter_project_pipe_kernel<NF, V, 4> : minb == 3 ? (const void*)filter_project_pipe_kernel<NF, V, 3> : (const void*)filter_project_pipe_kernel<NF, V, 5>)
    if (!configured) {
      for (const void* f : {ARK_PIPE_FN(0, true), ARK_PIPE_FN(1, true), ARK_PIPE_FN(2, true)})
        ARK_CUDA(cudaFuncSetAttribute(f, cudaFuncAttributeMaxDynamicSharedMemorySize, max_smem));
      configured = true;
    }
    const void* fn = nullptr;
    if (n_fixed_out == 0 && v) fn = ARK_PIPE_FN(0, true);
    else if (n_fixed_out == 1 && v) fn = ARK_PIPE_FN(1, true);
    else if (n_fixed_out == 2 && v) fn = ARK_PIPE_FN(2, true);
    else if (n_fixed_out == 1) fn = ARK_PIPE_FN(1, false);
    else if (n_fixed_out == 2) fn = ARK_PIPE_FN(2, false);
    else return false;
#undef ARK_PIPE_FN
    int& o = occ[v ? 1 : 0][n_fixed_out];
    if (o == 0 || occ_smem[v ? 1 : 0][n_fixed_out] != smem) {
      ARK_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&o, fn, 256, smem));
      occ_smem[v ? 1 : 0][n_fixed_out] = smem;
      if (o < 1) o = 1;
    }
    const int sms = sm_count();
    static const int cap_per_sm = [] { const char* e = getenv("ARK_FP_CTAS_PER_SM"); return e ? atoi(e) : 0; }();
    const int per_sm = cap_per_sm > 0 ? std::min(cap_per_sm, o) : o;
    const int grid = std::max(1, std::min(P.n_tiles, sms * per_sm));
    KernelTimer t("filter_project_tma_kernel", stream, "filter_project_pipe_kernel");
    void* args[] = {(void*)&P};
    ARK_CUDA(cudaLaunchKernel(fn, dim3(grid), dim3(256), args, smem, stream));
    return true;
  }
  {
    static const bool use_ticket = [] { const char* e = getenv("ARK_FP_TICKET"); return e && atoi(e) != 0; }();
    if (!use_ticket) P.ticket = nullptr;
  }
  const size_t smem = P.has_varlen ? 2 * (size_t)(cap + 32) : 0;
  const int max_smem = 2 * (48 * 1024 + 32);
  static bool configured = false;
  if (!configured) {
    ARK_CUDA(cudaFuncSetAttribute(filter_project_tma_kernel<0, true, 256>, cudaFuncAttributeMaxDynamicSharedMemorySize, max_smem));
    ARK_CUDA(cudaFuncSetAttribute(filter_project_tma_kernel<1, true, 256>, cudaFuncAttributeMaxDynamicSharedMemorySize, max_smem));
    ARK_CUDA(cudaFuncSetAttribute(filter_project_tma_kernel<2, true, 256>, cudaFuncAttributeMaxDynamicSharedMemorySize, max_smem));
    ARK_CUDA(cudaFuncSetAttribute(filter_project_tma_kernel<0, true, 512>, cudaFuncAttributeMaxDynamicSharedMemorySize, max_smem));
    ARK_CUDA(cudaFuncSetAttribute(filter_project_tma_kernel<1, true, 512>, cudaFuncAttributeMaxDynamicSharedMemorySize, max_smem));
    ARK_CUDA(cudaFuncSetAttribute(filter_project_tma_kernel<2, true, 512>, cudaFuncAttributeMaxDynamicSharedMemorySize, max_smem));
    configured = true;
  }
  if (n_fixed_out == 0 && !v) return false;  // before the timer: a declined launch is not recorded
  KernelTimer t("filter_project_tma_kernel", stream, "filter_project_r1_kernel");
#define ARK_TMA_LAUNCH(NF, V, TH) filter_project_tma_kernel<NF, V, TH><<<P.n_tiles, TH, (V) ? smem : 0, stream>>>(P)
  if (g_fp_threads == 256) {
    if (n_fixed_out == 0 && v) ARK_TMA_LAUNCH(0, true, 256);
    else if (n_fixed_out == 1 && v) ARK_TMA_LAUNCH(1, true, 256);
    else if (n_fixed_out == 2 && v) ARK_TMA_LAUNCH(2, true, 256);
    else if (n_fixed_out == 1) ARK_TMA_LAUNCH(1, false, 256);
    else if (n_fixed_out == 2) ARK_TMA_LAUNCH(2, false, 256);
    else return false;
  } else {
    if (n_fixed_out == 0 && v) ARK_TMA_LAUNCH(0, true, 512);
    else if (n_fixed_out == 1 && v) ARK_TMA_LAUNCH(1, true, 512);
    else if (n_fixed_out == 2 && v) ARK_TMA_LAUNCH(2, true, 512);
    else if (n_fixed_out == 1) ARK_TMA_LAUNCH(1, false, 512);
    else if (n_fixed_out == 2) ARK_TMA_LAUNCH(2, false, 512);
    else return false;
  }
#undef ARK_TMA_LAUNCH
  return true;
}

}  // namespace ark
