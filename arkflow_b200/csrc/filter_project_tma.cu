// filter_project_tma.cu — the fast path of filter + project + compaction for the common shape
//   SELECT <fixed-width columns…> [, <one Utf8/Binary column>] FROM t WHERE <col> <cmp> <literal>
// (BASELINE config 2: SELECT sensor, value FROM flow WHERE value >= 10), no NULLs in the used columns.
//
// Same single-pass algorithm as filter_project.cu (tiles, ballot ranking, decoupled look-back) with the data movement
// rebuilt around what each buffer needs:
//   * fixed-width columns never touch shared memory: rows are striped over the warp, so one coalesced 8-byte load per
//     row lands in a register and the surviving lanes store to CONSECUTIVE output slots without staging;
//   * the tile's string bytes form one contiguous, arbitrarily aligned byte range: a single 1-D TMA bulk copy
//     (cp.async.bulk → UBLKCP, completion on an mbarrier) drops the 16-byte-aligned window around it into shared memory
//     while the data warps evaluate the predicate;
//   * strings are compacted shared→shared at word granularity (aligned source words funnel-shifted into destination
//     words) into a buffer that mirrors the destination's 16-byte alignment, then leave as 16-byte vector stores.
// One kernel, filter_project_tile_kernel: 2048-row tiles, 512 data threads + one look-back warp, 40 registers, three
// CTAs per SM; look-back and load latency are hidden by CTA-level parallelism (DESIGN.md §4.1, §8).
// Bulk copies only touch 16-byte blocks that contain at least one valid byte of the source buffer, so they never reach
// into an unmapped page.
#include <atomic>

#include "tma.cuh"
#include "batch.h"
#include "filter_project.cuh"
#include "vm.cuh"

namespace ark {

namespace {

constexpr int T_MAX_FIXED_OUT = 2;
constexpr int T_THREADS = 512;                // data threads per CTA; one more warp sets up the bulk copy and runs the look-back
constexpr int TT = T_THREADS * 4;             // rows per tile
constexpr int DESC_STRIDE = 4;                // u64 words between consecutive descriptors: one descriptor per 32-byte sector
constexpr int MAX_STR_CAP = 48 * 1024;        // largest string staging buffer (bytes per buffer, two buffers per CTA)

struct TmaParams {
  int64_t n_rows;
  int32_t n_tiles;
  int32_t n_fixed_out;
  int32_t has_varlen;
  int32_t str_cap;                          // bytes of shared memory per string buffer (multiple of 16)
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
  unsigned long long* desc_next;            // or null: its tile (and group) descriptor words are zeroed for the next launch
  long long* totals;
  int32_t debug;                            // measurement knob (ARK_FP_DEBUG): bit 0 = skip the look-back (results are garbage), bit 2 = force helping
  int32_t lb_delay;                         // ns the look-back warp sleeps before its first poll
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

// Forward progress without relying on CTA dispatch order.  A tile's look-back may only wait for tiles whose CTAs are
// running; with tile = blockIdx.x that holds when CTAs are dispatched in blockIdx order (what CUB's single-pass scans
// assume), but nothing in the programming model promises it (MPS, time slicing, a debugger, compute-sanitizer).  So a
// warp that has spun `spin_limit` times on an unpublished predecessor HELPS: it computes that tile's aggregate itself
// — the predicate over the tile's 2048 rows, 64 per lane — and publishes it with a CAS if it is still missing.  The
// aggregate is a pure function of the input, so helper and owner can only ever write the same value; the owner still
// publishes its inclusive prefix when it gets to run.  The fast path never executes this (`ARK_FP_DEBUG=4` forces it:
// tests/test_sql_filter_gpu.py, tests/test_filter_kernels_gpu.py).
template <bool VARLEN>
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
  if (lane == 0) atomicCAS(P.desc + (size_t)t * DESC_STRIDE, 0ull, desc_pack(t == 0 ? DESC_PREFIX : DESC_AGG, cnt, bytes));
}

// ---- two-level look-back -------------------------------------------------------------------------------
// A single chain of tile descriptors moves a prefix forward by one window per L2 round trip, and the CTAs of one wave
// publish their aggregates at about the same time — so the prefix would crawl through every wave at a fixed tile rate
// whatever the byte rate.  Here tiles form groups of 32.  A tile sums the aggregates of the tiles before it in its own
// group (one window) and, at the same time, looks back over GROUP descriptors (one window = 32 groups = 1024 tiles, more
// than a wave), which the last tile of every group publishes: first the group's aggregate, then — after its own
// group-level look-back — the inclusive prefix.  No descriptor waits for a PREFIX that is itself waiting: every tile
// resolves two or three round trips after the aggregates around it exist.
// Group descriptors live behind the tile descriptors (same stride); the trailing partial group is never published.
template <bool VARLEN>
__device__ __forceinline__ void help_publish_group(const TmaParams& P, unsigned long long* gdesc, int g, int lane) {
  const int t = g * 32 + lane;  // only complete groups are ever waited for
  unsigned long long d = ld_volatile_u64(P.desc + (size_t)t * DESC_STRIDE);
  unsigned miss = __ballot_sync(0xffffffffu, (d >> 62) == 0);
  while (miss) {
    help_publish_aggregate<VARLEN>(P, g * 32 + __ffs(miss) - 1, lane);
    miss &= miss - 1;
  }
  while ((d >> 62) == 0) d = ld_volatile_u64(P.desc + (size_t)t * DESC_STRIDE);  // owner or helper has published by now
  const unsigned c = __reduce_add_sync(0xffffffffu, (unsigned)((d >> 31) & DESC_FIELD));
  const unsigned b = __reduce_add_sync(0xffffffffu, (unsigned)(d & DESC_FIELD));
  if (lane == 0) atomicCAS(gdesc + (size_t)g * DESC_STRIDE, 0ull, desc_pack(g == 0 ? DESC_PREFIX : DESC_AGG, c, b));
}

// Resolve half (the look-back warp).  The tile's aggregate is already published.
template <bool VARLEN>
__device__ __forceinline__ void lookback_two_level(const TmaParams& P, int tile, long long agg_cnt, long long agg_bytes, int lane,
                                                   long long* ex_cnt, long long* ex_bytes) {
  unsigned long long* const desc = P.desc;
  unsigned long long* const gdesc = desc + (size_t)P.n_tiles * DESC_STRIDE;
  const int spin_limit = (P.debug & 4) ? 2 : 4096;
  const int g = tile >> 5, i = tile & 31;
  // both windows are requested before either is inspected
  if (P.lb_delay) __nanosleep(P.lb_delay);
  const int tidx = tile - 1 - lane;          // lanes < i: the tiles before this one in its group
  unsigned long long dt = DESC_AGG;          // other lanes: an empty aggregate
  if (lane < i) dt = ld_volatile_u64(desc + (size_t)tidx * DESC_STRIDE);
  int look = g - 1;
  unsigned long long dg = DESC_PREFIX;       // virtual group -1: prefix 0
  if (look - lane >= 0) dg = ld_volatile_u64(gdesc + (size_t)(look - lane) * DESC_STRIDE);
  for (int spins = 0;;) {
    const unsigned pending = __ballot_sync(0xffffffffu, (dt >> 62) == 0);
    if (!pending) break;
    if (++spins > spin_limit) { help_publish_aggregate<VARLEN>(P, tile - 1 - (__ffs(pending) - 1), lane); spins = 0; }
    if ((dt >> 62) == 0) dt = ld_volatile_u64(desc + (size_t)tidx * DESC_STRIDE);
  }
  const long long in_c = __reduce_add_sync(0xffffffffu, lane < i ? (unsigned)((dt >> 31) & DESC_FIELD) : 0u);
  const long long in_b = __reduce_add_sync(0xffffffffu, lane < i ? (unsigned)(dt & DESC_FIELD) : 0u);
  const bool closes_group = i == 31;
  if (closes_group && lane == 0) st_volatile_u64(gdesc + (size_t)g * DESC_STRIDE, desc_pack(g == 0 ? DESC_PREFIX : DESC_AGG, in_c + agg_cnt, in_b + agg_bytes));
  long long run_c = 0, run_b = 0;
  if (g > 0) {
    for (;;) {
      const int idx = look - lane;
      for (int spins = 0;;) {
        const unsigned pending = __ballot_sync(0xffffffffu, (dg >> 62) == 0);
        if (!pending) break;
        if (++spins > spin_limit) { help_publish_group<VARLEN>(P, gdesc, look - (__ffs(pending) - 1), lane); spins = 0; }
        if ((dg >> 62) == 0) dg = ld_volatile_u64(gdesc + (size_t)idx * DESC_STRIDE);
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
      if (look - lane >= 0) dg = ld_volatile_u64(gdesc + (size_t)(look - lane) * DESC_STRIDE);
    }
    if (closes_group && lane == 0) st_volatile_u64(gdesc + (size_t)g * DESC_STRIDE, desc_pack(DESC_PREFIX, run_c + in_c + agg_cnt, run_b + in_b + agg_bytes));
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

// Lane l of a warp loads rows wrow0 + 32 j + l, j = 0..3: predicate values and (VARLEN) the offsets where their strings
// start; lane 31 also loads the end of the warp's last string.
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

// ================================================================================================
// filter_project_tile_kernel.  ONE 2048-row tile per CTA (tile = blockIdx.x), rows striped over the warp (lane l of warp
// w owns rows 128w + 32j + l: coalesced 8-byte loads and stores, no shared-memory bank conflicts).  Sixteen data warps
// load, evaluate and rank the tile's rows and compact its strings in shared memory; a seventeenth warp sets up the bulk
// copy of the tile's string bytes, publishes the tile's aggregate and runs the two-level look-back meanwhile.
// What bounds it on config 2 (2^24 rows, H100): with the look-back stubbed out the kernel is the data path alone; the
// look-back adds the time a tile's CTA waits for the aggregates of the tiles before it (their loads were issued at the
// same time and some always land late), during which it holds its slot on the SM without having loads in flight.  At 40
// registers three CTAs fit per SM, 48 data warps.  The variants measured against this kernel are in DESIGN.md §8.
// Forward progress does not depend on CTA dispatch order: see help_publish_aggregate / help_publish_group.
// The register cap is __maxnreg__, not __launch_bounds__'s minBlocks: ptxas rounds a 544-thread CTA up when it derives
// the cap from minBlocks (3 blocks → 32 registers and spills instead of the 40 that fit).  __launch_bounds__ still tells
// ptxas the CTA size, and at the same cap that spills less (config 2's instance: 88 instead of 108 bytes of spill stores).
// nvcc accepts the two qualifiers together only when their arguments depend on template parameters: hence DT and MAXR,
// which are never given other values.
// ================================================================================================
template <int NF, bool VARLEN, int DT = T_THREADS, int MAXR = 40>
__global__ void __launch_bounds__(DT + 32) __maxnreg__(MAXR) filter_project_tile_kernel(const __grid_constant__ TmaParams P) {
  // warps 0..T_WARPS-1: the tile's rows; warp T_WARPS: bulk copy and look-back — nothing but its own few values is live
  // there, so the (rare) call into help_publish_aggregate costs the data warps no registers and no spills
  constexpr int T_WARPS = T_THREADS / 32, LB_WARP = T_WARPS;
  extern __shared__ __align__(16) uint8_t smem[];   // [in_bytes][out_bytes], each str_cap + 32
  __shared__ __align__(8) unsigned long long s_bar;
  __shared__ int s_str_base, s_str_staged;
  __shared__ int s_cnt[T_WARPS], s_bytes[T_WARPS];
  __shared__ long long s_excl[2];

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int wrow0 = warp * 128;
  const unsigned lt_mask = (1u << lane) - 1u;
  uint8_t* const in_bytes = smem;
  uint8_t* const out_bytes = smem + P.str_cap + 32;
  const int n_tiles = P.n_tiles;
  const int tile = blockIdx.x;
  // the data warps issue their loads at once; the window of string bytes is set up by the look-back warp meanwhile (its two
  // offset loads in front of a CTA-wide barrier would start every tile one memory latency late)
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
    if (lane == 0) st_volatile_u64(P.desc + (size_t)tile * DESC_STRIDE, desc_pack(tile == 0 ? DESC_PREFIX : DESC_AGG, tile_cnt, tb));
    long long ex0, ex1;
    if (P.debug & 1) { ex0 = (long long)tile * (TT / 2); ex1 = ex0 * 12; }
    else lookback_two_level<VARLEN>(P, tile, tile_cnt, tb, lane, &ex0, &ex1);
    if (lane == 0) { s_excl[0] = ex0; s_excl[1] = ex1; }
    __syncthreads();   // (2)
    if (P.desc_next && lane == 0) {  // no launch reads desc_next before this one has ended
      P.desc_next[(size_t)tile * DESC_STRIDE] = 0;
      if ((tile & 31) == 0) P.desc_next[((size_t)n_tiles + (tile >> 5)) * DESC_STRIDE] = 0;
    }
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

  // ---- D: tile scan over the per-warp totals (every warp, redundantly) ----
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

}  // namespace

static std::atomic<double> g_avg_len_hint{12.8};
void filter_project_tma_note_avg_len(double avg) { if (avg > 0) g_avg_len_hint.store(avg); }
int filter_project_tma_tile_rows() { return TT; }
// u64 words of descriptor scratch for n_tiles tiles: the tile descriptors, then one descriptor per group of 32 tiles
size_t filter_project_tma_desc_words(int64_t n_tiles) { return (size_t)(n_tiles + (n_tiles + 31) / 32) * (size_t)DESC_STRIDE; }
int filter_project_tma_max_fixed_out() { return T_MAX_FIXED_OUT; }

// Returns false when the inputs do not meet the alignment rules of this path, or when the query projects no column this
// kernel writes (caller falls back).  `desc` holds filter_project_tma_desc_words(tiles) zeroed words.  `desc_next` (may be
// null) is another buffer of that size: the kernel zeroes in it the descriptor words a launch with the same tile count reads.
bool launch_filter_project_tma(int64_t n_rows, const void* pred_in, int n_fixed_out, const void* const* fixed_in, void* const* fixed_out,
                               const int32_t* offsets_in, const uint8_t* data_in, int64_t data_bytes, int32_t* offsets_out, uint8_t* data_out,
                               int cmp, int is_f64, uint64_t constant, unsigned long long* desc, unsigned long long* desc_next,
                               long long* totals, cudaStream_t stream) {
  if (reinterpret_cast<uintptr_t>(pred_in) & 7) return false;
  if (n_rows >= (1ll << 31) - 1) return false;  // 31-bit descriptor fields
  if (data_out && (reinterpret_cast<uintptr_t>(data_out) & 15)) return false;
  if (n_fixed_out > 2) return false;
  TmaParams P;
  memset(&P, 0, sizeof P);
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
  P.desc = desc; P.desc_next = desc_next; P.totals = totals;
  static const int debug = [] { const char* e = getenv("ARK_FP_DEBUG"); return e ? atoi(e) : 0; }();
  P.debug = debug;
  // the look-back warp sleeps this long before its first poll: the aggregates it needs belong to tiles whose loads were issued
  // at about the same time as its own, and the 60-odd descriptor loads of a poll that finds them missing are wasted L2
  // requests (measured on 2^24 rows: shortest around 1500 ns with 2048-row tiles, DESIGN.md §8)
  static const int lb_delay = [] { const char* e = getenv("ARK_FP_LB_DELAY"); return e ? atoi(e) : 1500; }();
  P.lb_delay = lb_delay;
  // string staging sized from the batch's average string length (+6.25 %), 1 KB granules, 4..48 KB
  int cap = 0;
  if (P.has_varlen) {
    // exact when the extent is known; otherwise the average selected-string length of the previous launch
    double avg = n_rows > 0 && data_bytes >= 0 ? (double)data_bytes / (double)n_rows : g_avg_len_hint.load();
    cap = (int)round_up((int64_t)(avg * TT * 1.0625) + 64, 1024);
    cap = std::max(4096, std::min(cap, MAX_STR_CAP));
  }
  P.str_cap = cap;
  const bool v = P.has_varlen;
  const size_t smem = v ? 2 * (size_t)(cap + 32) : 0;
  static bool configured = false;
  if (!configured) {
    for (const void* f : {(const void*)filter_project_tile_kernel<0, true>, (const void*)filter_project_tile_kernel<1, true>,
                          (const void*)filter_project_tile_kernel<2, true>})
      ARK_CUDA(cudaFuncSetAttribute(f, cudaFuncAttributeMaxDynamicSharedMemorySize, 2 * (MAX_STR_CAP + 32)));
    configured = true;
  }
  const void* fn = nullptr;
  if (n_fixed_out == 0 && v) fn = (const void*)filter_project_tile_kernel<0, true>;
  else if (n_fixed_out == 1 && v) fn = (const void*)filter_project_tile_kernel<1, true>;
  else if (n_fixed_out == 2 && v) fn = (const void*)filter_project_tile_kernel<2, true>;
  else if (n_fixed_out == 1) fn = (const void*)filter_project_tile_kernel<1, false>;
  else if (n_fixed_out == 2) fn = (const void*)filter_project_tile_kernel<2, false>;
  else return false;  // before the timer: a declined launch is not recorded
  KernelTimer t("filter_project_tma_kernel", stream, "filter_project_tile_kernel");
  void* args[] = {(void*)&P};
  trace_kernel_begin(stream);
  ARK_CUDA(cudaLaunchKernel(fn, dim3(P.n_tiles), dim3(T_THREADS + 32), args, smem, stream));
  trace_kernel_end(stream);
  return true;
}

}  // namespace ark
