// hash_agg_stream.cu — GROUP BY for high-cardinality keys: the row kernel of hash_agg.cu rebuilt as a persistent,
// software-pipelined kernel with several probe chains in flight per thread.
//
// hash_agg_kernel (hash_agg.cu) walks one row per thread through three DEPENDENT memory latencies — offsets → key
// bytes → table slot — and resolves the probe chains of a thread one after the other, so its warps stall on long
// scoreboards with most issue slots and most of the HBM bandwidth idle.  Here:
//   * a CTA stays resident and takes 256·R-row tiles; the loads of the NEXT tile (offsets / Int64 keys / predicate
//     column into registers, the tile's key bytes by one 1-D TMA bulk copy into the other half of a two-stage ring)
//     are issued before the current tile is touched, so the only latency on a row's critical path is the table's;
//   * every thread owns R consecutive rows: the home BUCKETS of all R rows (four keys each, hash_agg.cuh) are requested
//     before any is inspected — R independent L2 requests per thread — and a row that is not settled by its home
//     bucket (4 % of the rows at load 0.48) continues with table_find_or_claim;
//   * aggregate arguments are fetched with 16-byte loads while the probes are in flight.
// Table layout, key encoding, claim protocol (128-bit CAS), accumulators (fire-and-forget REDs) and the overflow /
// group-count protocol are exactly hash_agg_kernel's, so everything downstream (compaction, emit, multi-GPU
// partition) is shared.  Algorithmic traffic: key + argument bytes read once (SURVEY.md §8(d): 24 B/row, config 3).
#include <atomic>

#include "agg_acc.cuh"
#include "engine.h"
#include "hash_agg.cuh"
#include "hashkey.cuh"
#include "tma.cuh"

namespace ark {

namespace {

constexpr int HS_THREADS = 256;
constexpr int HS_PRE = 2;  // aggregate arguments prefetched into registers per tile (further ones are loaded in place)


template <int R>
__device__ __forceinline__ void ld_vec_u64(const unsigned long long* src, bool fast, int lr0, int rows, unsigned long long (&v)[R]) {
  if constexpr (R == 1) {
    v[0] = 0;
    if (lr0 < rows) asm volatile("ld.global.nc.L1::no_allocate.u64 %0, [%1];" : "=l"(v[0]) : "l"(src));
  } else {
    if (fast) {
#pragma unroll
      for (int j = 0; j < R; j += 2)
        asm volatile("ld.global.nc.L1::no_allocate.v2.u64 {%0, %1}, [%2];" : "=l"(v[j]), "=l"(v[j + 1]) : "l"(src + j));
    } else {
#pragma unroll
      for (int j = 0; j < R; ++j) v[j] = (lr0 + j < rows) ? src[j] : 0;
    }
  }
}

template <int R>
__device__ __forceinline__ void ld_vec_off(const int32_t* os, bool fast, int lr0, int rows, int lane, int (&off)[R], int* offx) {
  if (fast) {
    if constexpr (R == 4) asm volatile("ld.global.nc.L1::no_allocate.v4.s32 {%0, %1, %2, %3}, [%4];" : "=r"(off[0]), "=r"(off[1]), "=r"(off[2]), "=r"(off[3]) : "l"(os));
    else if constexpr (R == 2) asm volatile("ld.global.nc.L1::no_allocate.v2.s32 {%0, %1}, [%2];" : "=r"(off[0]), "=r"(off[1]) : "l"(os));
    else asm volatile("ld.global.nc.L1::no_allocate.s32 %0, [%1];" : "=r"(off[0]) : "l"(os));
  } else {
#pragma unroll
    for (int j = 0; j < R; ++j) off[j] = (lr0 + j <= rows) ? os[j] : 0;
  }
  *offx = ((lane == 31 || lr0 + R >= rows) && lr0 + R <= rows) ? os[R] : 0;
}

// SIG 1: the accumulators are exactly {COUNT(*), SUM(<non-null Int64 column>)} (config 3): two REDs, no dispatch.
template <int KEYK, int PRED, int R, int SIG>
__global__ void __launch_bounds__(HS_THREADS) hash_agg_stream_kernel(const __grid_constant__ AggParams P, const int str_cap, const int dbg) {
  constexpr int TR = HS_THREADS * R;
  constexpr int PRODUCER = HS_THREADS - 32;
  extern __shared__ __align__(16) uint8_t smem[];  // KEY_BYTES: [key bytes stage 0][stage 1], each str_cap + 32
  __shared__ __align__(8) unsigned long long s_bar[2];
  __shared__ int s_str_base[2], s_str_staged[2];
  const int tid = threadIdx.x, lane = tid & 31;
  const int64_t n = P.n_rows;
  const int n_tiles = (int)((n + TR - 1) / TR);
  const int lr0 = R * tid;
  const int stage_bytes = str_cap + 32;
  const ColView& kc = P.cols[P.key_slot];
  const unsigned long long bmask = P.mask >> 2;
  const int bstride = P.bucket_stride;
  auto tile_rows = [&](int t) { const int64_t r = n - (int64_t)t * TR; return (int)(r < TR ? r : TR); };
  auto issue_window = [&](int st, int32_t o0, int32_t o1) {
    const uintptr_t a0 = reinterpret_cast<uintptr_t>((const uint8_t*)kc.data + o0), a1 = reinterpret_cast<uintptr_t>((const uint8_t*)kc.data + o1);
    const uintptr_t lo = a0 & ~(uintptr_t)15, hi = (a1 + 15) & ~(uintptr_t)15;
    int staged = 0;
    if (o1 > o0 && hi - lo <= (uintptr_t)str_cap) {
      staged = 1;
      mbar_expect_tx(&s_bar[st], (unsigned)(hi - lo));
      tma_load_1d(smem + st * stage_bytes, reinterpret_cast<const void*>(lo), (unsigned)(hi - lo), &s_bar[st]);
    }
    s_str_base[st] = o0 - (int32_t)(a0 - lo); s_str_staged[st] = staged;
  };
  // which accumulators get their argument prefetched (the first HS_PRE that read argument values; COUNT(x) reads only
  // x's validity)
  int pre_acc[HS_PRE];
  {
    int k = 0;
#pragma unroll
    for (int i = 0; i < HS_PRE; ++i) pre_acc[i] = -1;
    for (int a = 0; a < P.n_acc && k < HS_PRE; ++a)
      if (acc_reads_values(P.accs[a].kind)) pre_acc[k++] = a;
  }

  int tile = blockIdx.x;
  int32_t bo0 = 0, bo1 = 0;
  if (tid == PRODUCER) {
    if (KEYK == KEY_BYTES) {
      mbar_init(&s_bar[0], 1); mbar_init(&s_bar[1], 1); mbar_fence_init();
      if (tile < n_tiles) { const int64_t r0 = (int64_t)tile * TR; issue_window(0, kc.offsets[r0], kc.offsets[r0 + tile_rows(tile)]); }
      const int t1 = tile + (int)gridDim.x;
      if (t1 < n_tiles) { const int64_t r1 = (int64_t)t1 * TR; bo0 = kc.offsets[r1]; bo1 = kc.offsets[r1 + tile_rows(t1)]; }
    }
  }
  __syncthreads();
  // registers of the next tile
  int offn[R] = {}; int offxn = 0;
  unsigned long long kvn[R] = {}, pvn[R] = {};
  auto prefetch = [&](int t) {
    const int64_t r0 = (int64_t)t * TR;
    const int rows = tile_rows(t);
    const bool full = lr0 + R <= rows;
    if (KEYK == KEY_BYTES) {
      const int32_t* os = kc.offsets + r0 + lr0;
      ld_vec_off<R>(os, full && (reinterpret_cast<uintptr_t>(os) & (R * 4 - 1)) == 0, lr0, rows, lane, offn, &offxn);
    } else {
      const unsigned long long* ks = (const unsigned long long*)kc.data + r0 + lr0;
      ld_vec_u64<R>(ks, full && (reinterpret_cast<uintptr_t>(ks) & 15) == 0, lr0, rows, kvn);
    }
    if (PRED == 1) {
      const unsigned long long* ps = (const unsigned long long*)P.cols[P.sp_slot].data + r0 + lr0;
      ld_vec_u64<R>(ps, full && (reinterpret_cast<uintptr_t>(ps) & 15) == 0, lr0, rows, pvn);
    }
  };
  if (tile < n_tiles) prefetch(tile);

  unsigned int claimed = 0;
  unsigned ph = 0;
  int32_t err_overflow = 0, long_flag = 0;
  const long long pred_c = P.sp_is_f64 ? f64_total_key(P.sp_const) : (long long)P.sp_const;
  for (int it = 0; tile < n_tiles; ++it, tile += (int)gridDim.x) {
    const int st = it & 1;
    const int64_t row0 = (int64_t)tile * TR;
    const int rows = tile_rows(tile);
    const bool full = lr0 + R <= rows;
    int off[R + 1];
    unsigned long long kv[R], pv[R];
#pragma unroll
    for (int j = 0; j < R; ++j) { off[j] = offn[j]; kv[j] = kvn[j]; pv[j] = pvn[j]; }
    const int offx = offxn;
    // ---- A: the next tile's loads ----
    const int next = tile + (int)gridDim.x;
    int stop = 0;
    if (tid == PRODUCER) {
      stop = *reinterpret_cast<volatile int32_t*>(P.overflow);  // table too small: the host retries with 4× the slots
      if (KEYK == KEY_BYTES) {
        if (next < n_tiles) issue_window(st ^ 1, bo0, bo1);
        const int next2 = next + (int)gridDim.x;
        if (next2 < n_tiles) { const int64_t r2 = (int64_t)next2 * TR; bo0 = kc.offsets[r2]; bo1 = kc.offsets[r2 + tile_rows(next2)]; }
      }
    }
    if (next < n_tiles) prefetch(next);
    // ---- aggregate arguments of THIS tile: in flight while the keys are hashed and probed ----
    unsigned long long av[HS_PRE][R];
#pragma unroll
    for (int i = 0; i < HS_PRE; ++i) {
      if (pre_acc[i] >= 0) {
        const unsigned long long* as = (const unsigned long long*)P.cols[P.accs[pre_acc[i]].arg_slot].data + row0 + lr0;
        ld_vec_u64<R>(as, full && (reinterpret_cast<uintptr_t>(as) & 15) == 0, lr0, rows, av[i]);
      } else {
#pragma unroll
        for (int j = 0; j < R; ++j) av[i][j] = 0;
      }
    }
    // ---- predicate ----
    unsigned ok = 0;
#pragma unroll
    for (int j = 0; j < R; ++j) {
      bool f = lr0 + j < rows;
      if (PRED == 1 && f) {
        const ColView& c = P.cols[P.sp_slot];
        f = cmp_i64(P.sp_cmp, P.sp_is_f64 ? f64_total_key(pv[j]) : (long long)pv[j], pred_c) && col_valid(c, row0 + lr0 + j);
      }
      ok |= (unsigned)f << j;
    }
    // ---- keys ----
    Key16 mine[R];
    unsigned home[R];
    if (KEYK == KEY_BYTES) {
      off[R] = __shfl_down_sync(0xffffffffu, off[0], 1);
      if ((lane == 31 || lr0 + R >= rows) && lr0 + R <= rows) off[R] = offx;
      const bool staged = s_str_staged[st];
      const int base = s_str_base[st];
      if (staged) { mbar_wait(&s_bar[st], (ph >> st) & 1); ph ^= 1u << st; }
      const uint8_t* in_bytes = smem + st * stage_bytes;
#pragma unroll
      for (int j = 0; j < R; ++j) {
        home[j] = 0;
        if (!((ok >> j) & 1)) continue;
        const int64_t row = row0 + lr0 + j;
        unsigned h32;
        if (!col_valid(kc, row)) { mine[j].lo = 0; mine[j].hi = (unsigned long long)KEYTAG_NULL << 32; h32 = hash32_key16(mine[j]); }
        else if (staged) { make_key_smem(in_bytes + (off[j] - base), off[j + 1] - off[j], row, &mine[j], &h32); if (off[j + 1] - off[j] > 12) long_flag = 1; }
        else {
          int llen = 0;
          const uint8_t* lp = make_key_raw(KEY_BYTES, kc, row, &mine[j], &llen);
          if (lp) { const unsigned long long h = hash_bytes(lp, llen); h32 = (unsigned)(h >> 32) ^ (unsigned)h; long_flag = 1; }
          else h32 = hash32_key16(mine[j]);
        }
        home[j] = (unsigned)((h32 * 0x9E3779B1u) & bmask);
      }
    } else {
#pragma unroll
      for (int j = 0; j < R; ++j) {
        home[j] = 0;
        if (!((ok >> j) & 1)) continue;
        if (col_valid(kc, row0 + lr0 + j)) { mine[j].lo = kv[j]; mine[j].hi = (unsigned long long)KEYTAG_INT << 32; }
        else { mine[j].lo = 0; mine[j].hi = (unsigned long long)KEYTAG_NULL << 32; }
        home[j] = (unsigned)((hash32_key16(mine[j]) * 0x9E3779B1u) & bmask);
      }
    }
    // this stage's key bytes are in registers: the producer may refill it in the iteration after next.  The barrier
    // also carries the producer's poll of the overflow flag to every thread (CTA-uniform exit).
    if (__syncthreads_or(stop)) {
      // a bulk copy for the next tile may be in flight into this CTA's shared memory: let it land before leaving
      if (KEYK == KEY_BYTES && next < n_tiles && s_str_staged[st ^ 1]) mbar_wait(&s_bar[st ^ 1], (ph >> (st ^ 1)) & 1);
      break;
    }
    // ---- home buckets of all R rows requested at once ----
    Key16 kb[R][TBL_B];
#pragma unroll
    for (int j = 0; j < R; ++j) {
      if (!((ok >> j) & 1)) continue;
      if (dbg & 4) { kb[j][0].lo = home[j]; continue; }  // measurement: no table reads at all
      const Key16* b = reinterpret_cast<const Key16*>(P.table + (unsigned long long)home[j] * (unsigned long long)bstride);
      ld256_keys(b, &kb[j][0], &kb[j][1]);
      ld256_keys(b + 2, &kb[j][2], &kb[j][3]);
    }
    unsigned long long slot[R];
#pragma unroll
    for (int j = 0; j < R; ++j) {
      slot[j] = ~0ull;
      if (!((ok >> j) & 1)) continue;
      if (dbg & 2) { slot[j] = (unsigned long long)home[j] * TBL_B + (kb[j][0].lo & 3); continue; }  // measurement: no probing
      Key16* b = reinterpret_cast<Key16*>(P.table + (unsigned long long)home[j] * (unsigned long long)bstride);
      bool done = false;
#pragma unroll
      for (int i = 0; i < TBL_B; ++i) {
        if (done) continue;
        Key16 c = kb[j][i];
        if (c.hi == KEY_EMPTY) {
          c = cas128(b + i, Key16{KEY_EMPTY, KEY_EMPTY}, mine[j]);
          if (c.hi == KEY_EMPTY && c.lo == KEY_EMPTY) { ++claimed; done = true; slot[j] = (unsigned long long)home[j] * TBL_B + i; continue; }
        }
        if (key_equal(mine[j], c, kc, kc)) { done = true; slot[j] = (unsigned long long)home[j] * TBL_B + i; }
      }
      if (!done) {  // the home bucket is full of other keys: walk on
        slot[j] = table_find_or_claim(P.table, bmask, bstride, (unsigned long long)home[j] + 1, mine[j], kc, kc, &claimed);
        if (slot[j] == ~0ull) { err_overflow = 1; ok &= ~(1u << j); }  // table too loaded for this batch
      }
    }
    // ---- accumulate (fire-and-forget REDs) ----
    if (dbg & 1) continue;  // measurement: no accumulation
    if (SIG == 1) {
#pragma unroll
      for (int j = 0; j < R; ++j) {
        if (!((ok >> j) & 1)) continue;
        atomicAdd(tbl_acc(P.table, slot[j], 0, bstride), 1ull);
        atomicAdd(tbl_acc(P.table, slot[j], 1, bstride), av[0][j]);
      }
    } else {
      for (int a = 0; a < P.n_acc; ++a) {
        const AccParam& A = P.accs[a];
#pragma unroll
        for (int j = 0; j < R; ++j) {
          if (!((ok >> j) & 1)) continue;
          unsigned long long bits = 0;
          bool valid = true;
          if (A.kind != ACC_COUNT_STAR) {
            const ColView& c = P.cols[A.arg_slot];
            valid = col_valid(c, row0 + lr0 + j);
            if (A.kind != ACC_COUNT)
              bits = a == pre_acc[0] ? av[0][j] : (a == pre_acc[1] ? av[1][j] : __ldcs((const unsigned long long*)c.data + row0 + lr0 + j));
          }
          if (valid) accumulate(A.kind, A.arg_is_f64, tbl_acc(P.table, slot[j], a, bstride), bits);
        }
      }
    }
  }
  if (err_overflow) atomicExch(P.overflow, 1);
  if (long_flag) *P.long_seen = 1;
  claimed = (unsigned int)__reduce_add_sync(0xffffffffu, claimed);
  if (lane == 0 && claimed) atomicAdd(P.group_count, claimed);
}


// ================================================================================================
// hash_agg_staged_kernel — every input stream of a tile arrives by TMA.
//
// With the table out of the picture hash_agg_stream_kernel stays well below the HBM bandwidth: a 256-row tile
// prefetched into registers keeps only ~6 KB per CTA in flight.  Here a tile is
// 1024 rows and ALL of its inputs — key offsets, key bytes, the (first two) aggregate arguments, the predicate column —
// are 1-D bulk copies into a two-stage shared-memory ring issued by one thread a tile ahead (~25-33 KB per stage, 3-4
// CTAs per SM: ~100 KB per SM in flight, no registers spent on prefetching).  Rows are striped over the CTA (thread t
// owns rows t, t + 256, …: consecutive lanes read consecutive 12-byte keys, conflict-free) and taken R at a time:
// the home buckets of R rows are requested together, then resolved.
// Table protocol, key encoding and accumulators: exactly hash_agg_stream_kernel's.
// ================================================================================================
constexpr int HG_TILE = 1024;
constexpr int HG_MAX_STREAMS = 5;  // key offsets, key bytes | Int64 keys, arg 0, arg 1, predicate

struct StagedStream {  // one fixed-width input of a tile: element i of the tile sits at smem[base + shift + i * width]
  const uint8_t* src;  // column base (element 0 of the batch)
  int32_t width;       // bytes per element
  int32_t extra;       // elements past the tile's rows that are needed too (offsets: 1)
  int32_t smem_off;    // byte offset of this stream's window inside a stage
  int32_t pad;
};

struct StagedParams {
  StagedStream st[HG_MAX_STREAMS];
  int32_t n_streams;
  int32_t key_bytes_off, key_bytes_cap;  // KEY_BYTES: window of the key bytes inside a stage
  int32_t stage_bytes;
  int32_t i_off, i_key, i_arg0, i_arg1, i_pred;  // stream indices (-1: absent)
  int32_t dbg;
};

template <int KEYK, int PRED, int R, int SIG>
__global__ void __launch_bounds__(HS_THREADS, R == 1 ? 4 : 3) hash_agg_staged_kernel(const __grid_constant__ AggParams P, const __grid_constant__ StagedParams S) {
  constexpr int PRODUCER = HS_THREADS - 32;
  extern __shared__ __align__(16) uint8_t smem[];
  __shared__ __align__(8) unsigned long long s_bar[2];
  __shared__ int s_shift[2][HG_MAX_STREAMS];  // window start → element 0 of the tile
  __shared__ int s_str_base[2], s_str_staged[2];
  const int tid = threadIdx.x;
  const int64_t n = P.n_rows;
  const int n_tiles = (int)((n + HG_TILE - 1) / HG_TILE);
  const ColView& kc = P.cols[P.key_slot];
  const unsigned long long bmask = P.mask >> 2;
  const int bstride = P.bucket_stride;
  auto tile_rows = [&](int t) { const int64_t r = n - (int64_t)t * HG_TILE; return (int)(r < HG_TILE ? r : HG_TILE); };
  // producer: all bulk copies of tile t into stage st; (o0, o1) = the tile's bounding key offsets (KEY_BYTES)
  auto issue_tile = [&](int st, int t, int32_t o0, int32_t o1) {
    const int rows = tile_rows(t);
    uint8_t* stage = smem + (size_t)st * S.stage_bytes;
    unsigned total = 0;
    uintptr_t lo[HG_MAX_STREAMS + 1], hi[HG_MAX_STREAMS + 1];
    for (int k = 0; k < S.n_streams; ++k) {
      const uintptr_t a0 = reinterpret_cast<uintptr_t>(S.st[k].src) + (uintptr_t)((int64_t)t * HG_TILE) * S.st[k].width;
      const uintptr_t a1 = a0 + (uintptr_t)(rows + S.st[k].extra) * S.st[k].width;
      lo[k] = a0 & ~(uintptr_t)15; hi[k] = (a1 + 15) & ~(uintptr_t)15;
      s_shift[st][k] = (int)(a0 - lo[k]);
      total += (unsigned)(hi[k] - lo[k]);
    }
    int staged = 0;
    if (KEYK == KEY_BYTES) {
      const uintptr_t a0 = reinterpret_cast<uintptr_t>((const uint8_t*)kc.data + o0), a1 = reinterpret_cast<uintptr_t>((const uint8_t*)kc.data + o1);
      lo[HG_MAX_STREAMS] = a0 & ~(uintptr_t)15; hi[HG_MAX_STREAMS] = (a1 + 15) & ~(uintptr_t)15;
      if (o1 > o0 && hi[HG_MAX_STREAMS] - lo[HG_MAX_STREAMS] <= (uintptr_t)S.key_bytes_cap) { staged = 1; total += (unsigned)(hi[HG_MAX_STREAMS] - lo[HG_MAX_STREAMS]); }
      s_str_base[st] = o0 - (int32_t)(a0 - lo[HG_MAX_STREAMS]); s_str_staged[st] = staged;
    }
    mbar_expect_tx(&s_bar[st], total);
    for (int k = 0; k < S.n_streams; ++k)
      tma_load_1d(stage + S.st[k].smem_off, reinterpret_cast<const void*>(lo[k]), (unsigned)(hi[k] - lo[k]), &s_bar[st]);
    if (staged) tma_load_1d(stage + S.key_bytes_off, reinterpret_cast<const void*>(lo[HG_MAX_STREAMS]), (unsigned)(hi[HG_MAX_STREAMS] - lo[HG_MAX_STREAMS]), &s_bar[st]);
  };

  int tile = blockIdx.x;
  int32_t bo0 = 0, bo1 = 0;
  if (tid == PRODUCER) {
    mbar_init(&s_bar[0], 1); mbar_init(&s_bar[1], 1); mbar_fence_init();
    if (tile < n_tiles) {
      int32_t o0 = 0, o1 = 0;
      if (KEYK == KEY_BYTES) { const int64_t r0 = (int64_t)tile * HG_TILE; o0 = kc.offsets[r0]; o1 = kc.offsets[r0 + tile_rows(tile)]; }
      issue_tile(0, tile, o0, o1);
    }
    const int t1 = tile + (int)gridDim.x;
    if (KEYK == KEY_BYTES && t1 < n_tiles) { const int64_t r1 = (int64_t)t1 * HG_TILE; bo0 = kc.offsets[r1]; bo1 = kc.offsets[r1 + tile_rows(t1)]; }
  }
  __syncthreads();

  unsigned int claimed = 0;
  unsigned ph = 0;
  int32_t err_overflow = 0, long_flag = 0;
  const long long pred_c = P.sp_is_f64 ? f64_total_key(P.sp_const) : (long long)P.sp_const;
  for (int it = 0; tile < n_tiles; ++it, tile += (int)gridDim.x) {
    const int st = it & 1;
    const int64_t row0 = (int64_t)tile * HG_TILE;
    const int rows = tile_rows(tile);
    // ---- the next tile's bulk copies (its stage was released by the barrier that ended the previous iteration) ----
    const int next = tile + (int)gridDim.x;
    int stop = 0;
    if (tid == PRODUCER) {
      stop = *reinterpret_cast<volatile int32_t*>(P.overflow);  // table too small: the host retries with 4× the slots
      if (next < n_tiles && !stop) issue_tile(st ^ 1, next, bo0, bo1);
      const int next2 = next + (int)gridDim.x;
      if (KEYK == KEY_BYTES && next2 < n_tiles) { const int64_t r2 = (int64_t)next2 * HG_TILE; bo0 = kc.offsets[r2]; bo1 = kc.offsets[r2 + tile_rows(next2)]; }
    }
    mbar_wait(&s_bar[st], (ph >> st) & 1);  // this tile's streams have landed
    ph ^= 1u << st;
    const uint8_t* stage = smem + (size_t)st * S.stage_bytes;
    const bool staged = KEYK == KEY_BYTES && s_str_staged[st];
    const int str_base = s_str_base[st];
    auto elem = [&](int k, int i) -> const uint8_t* { return stage + S.st[k].smem_off + s_shift[st][k] + (size_t)i * S.st[k].width; };
#pragma unroll 1
    for (int q = 0; q < HG_TILE / HS_THREADS; q += R) {
      Key16 mine[R];
      unsigned home[R];
      unsigned long long av0[R], av1[R];
      unsigned ok = 0;
#pragma unroll
      for (int j = 0; j < R; ++j) {
        const int i = (q + j) * HS_THREADS + tid;  // striped: consecutive lanes, consecutive rows
        bool f = i < rows;
        const int64_t row = row0 + i;
        if (PRED == 1 && f) {
          const unsigned long long pv = *reinterpret_cast<const unsigned long long*>(elem(S.i_pred, i));
          f = cmp_i64(P.sp_cmp, P.sp_is_f64 ? f64_total_key(pv) : (long long)pv, pred_c) && col_valid(P.cols[P.sp_slot], row);
        }
        home[j] = 0; av0[j] = 0; av1[j] = 0;
        if (!f) continue;
        ok |= 1u << j;
        if (S.i_arg0 >= 0) av0[j] = *reinterpret_cast<const unsigned long long*>(elem(S.i_arg0, i));
        if (S.i_arg1 >= 0) av1[j] = *reinterpret_cast<const unsigned long long*>(elem(S.i_arg1, i));
        unsigned h32;
        if (!col_valid(kc, row)) { mine[j].lo = 0; mine[j].hi = (unsigned long long)KEYTAG_NULL << 32; h32 = hash32_key16(mine[j]); }
        else if (KEYK == KEY_BYTES) {
          const int o0 = *reinterpret_cast<const int32_t*>(elem(S.i_off, i)), o1 = *reinterpret_cast<const int32_t*>(elem(S.i_off, i + 1));
          if (staged) { make_key_smem(stage + S.key_bytes_off + (o0 - str_base), o1 - o0, row, &mine[j], &h32); if (o1 - o0 > 12) long_flag = 1; }
          else {
            int llen = 0;
            const uint8_t* lp = make_key_raw(KEY_BYTES, kc, row, &mine[j], &llen);
            if (lp) { const unsigned long long h = hash_bytes(lp, llen); h32 = (unsigned)(h >> 32) ^ (unsigned)h; long_flag = 1; }
            else h32 = hash32_key16(mine[j]);
          }
        } else {
          mine[j].lo = *reinterpret_cast<const unsigned long long*>(elem(S.i_key, i)); mine[j].hi = (unsigned long long)KEYTAG_INT << 32;
          h32 = hash32_key16(mine[j]);
        }
        home[j] = (unsigned)((h32 * 0x9E3779B1u) & bmask);
      }
      // ---- home buckets of the R rows requested together: first the two keys of the bucket's first sector, the second
      // sector only when neither of them is the row's key or free (a bucket fills from slot 0; at the usual load factor
      // of ≤ 0.5 three quarters of the rows are settled by the first 32 bytes — one L2 request instead of two) ----
      Key16 kb[R][2];
#pragma unroll
      for (int j = 0; j < R; ++j) {
        if (!((ok >> j) & 1)) continue;
        if (S.dbg & 4) { kb[j][0].lo = home[j]; continue; }  // measurement: no table reads at all
        const Key16* b = reinterpret_cast<const Key16*>(P.table + (unsigned long long)home[j] * (unsigned long long)bstride);
        ld256_keys(b, &kb[j][0], &kb[j][1]);
      }
      unsigned long long slot[R];
#pragma unroll
      for (int j = 0; j < R; ++j) {
        slot[j] = ~0ull;
        if (!((ok >> j) & 1)) continue;
        if (S.dbg & 2) { slot[j] = (unsigned long long)home[j] * TBL_B + (kb[j][0].lo & 3); continue; }  // measurement: no probing
        Key16* b = reinterpret_cast<Key16*>(P.table + (unsigned long long)home[j] * (unsigned long long)bstride);
        bool done = false;
#pragma unroll
        for (int half = 0; half < TBL_B / 2; ++half) {
          if (done) continue;
          Key16 k0 = kb[j][0], k1 = kb[j][1];
          if (half > 0) ld256_keys(b + 2 * half, &k0, &k1);
#pragma unroll
          for (int i = 0; i < 2; ++i) {
            if (done) continue;
            Key16 c = i == 0 ? k0 : k1;
            if (c.hi == KEY_EMPTY) {
              c = cas128(b + 2 * half + i, Key16{KEY_EMPTY, KEY_EMPTY}, mine[j]);
              if (c.hi == KEY_EMPTY && c.lo == KEY_EMPTY) { ++claimed; done = true; slot[j] = (unsigned long long)home[j] * TBL_B + 2 * half + i; continue; }
            }
            if (key_equal(mine[j], c, kc, kc)) { done = true; slot[j] = (unsigned long long)home[j] * TBL_B + 2 * half + i; }
          }
        }
        if (!done) {  // the home bucket is full of other keys: walk on
          slot[j] = table_find_or_claim(P.table, bmask, bstride, (unsigned long long)home[j] + 1, mine[j], kc, kc, &claimed);
          if (slot[j] == ~0ull) { err_overflow = 1; ok &= ~(1u << j); }
        }
      }
      // ---- accumulate (fire-and-forget REDs) ----
      if (S.dbg & 1) continue;  // measurement: no accumulation
      if (SIG == 1) {
#pragma unroll
        for (int j = 0; j < R; ++j) {
          if (!((ok >> j) & 1)) continue;
          atomicAdd(tbl_acc(P.table, slot[j], 0, bstride), 1ull);
          atomicAdd(tbl_acc(P.table, slot[j], 1, bstride), av0[j]);
        }
      } else {
        int pre = 0;
        for (int a = 0; a < P.n_acc; ++a) {
          const AccParam& A = P.accs[a];
          // the first two accumulators that read argument values are staged, numbered exactly as launch_staged adds them
          const int which = acc_reads_values(A.kind) ? pre++ : -1;
#pragma unroll
          for (int j = 0; j < R; ++j) {
            if (!((ok >> j) & 1)) continue;
            const int64_t row = row0 + (q + j) * HS_THREADS + tid;
            unsigned long long bits = 0;
            bool valid = true;
            if (A.kind != ACC_COUNT_STAR) {
              const ColView& c = P.cols[A.arg_slot];
              valid = col_valid(c, row);
              if (A.kind != ACC_COUNT) bits = which == 0 ? av0[j] : (which == 1 ? av1[j] : __ldcs((const unsigned long long*)c.data + row));
            }
            if (valid) accumulate(A.kind, A.arg_is_f64, tbl_acc(P.table, slot[j], a, bstride), bits);
          }
        }
      }
    }
    // every thread is done with this stage: the producer may refill it next iteration; the barrier also carries the
    // producer's poll of the overflow flag (CTA-uniform exit)
    if (__syncthreads_or(stop)) {
      // `stop` was read before this tile's successor was issued, so no bulk copy is in flight here
      break;
    }
  }
  if (err_overflow) atomicExch(P.overflow, 1);
  if (long_flag) *P.long_seen = 1;
  claimed = (unsigned int)__reduce_add_sync(0xffffffffu, claimed);
  if ((tid & 31) == 0 && claimed) atomicAdd(P.group_count, claimed);
}

bool launch_staged(const AggParams& P, int64_t key_bytes, int R, bool sig1, int dbg, cudaStream_t stream) {
  StagedParams S;
  memset(&S, 0, sizeof S);
  S.i_off = S.i_key = S.i_arg0 = S.i_arg1 = S.i_pred = -1;
  S.dbg = dbg;
  int off = 0;
  auto add = [&](const void* src, int width, int extra) {
    StagedStream& t = S.st[S.n_streams];
    t.src = (const uint8_t*)src; t.width = width; t.extra = extra; t.smem_off = off;
    off += (int)round_up((int64_t)(HG_TILE + extra) * width + 32, 16);  // aligned hull: up to 15 bytes before, 15 after
    return S.n_streams++;
  };
  const ColView& kc = P.cols[P.key_slot];
  if (P.key_kind == KEY_BYTES) S.i_off = add(kc.offsets, 4, 1);
  else S.i_key = add(kc.data, 8, 0);
  int pre = 0;  // hash_agg_staged_kernel numbers its staged arguments by the same rule
  for (int a = 0; a < P.n_acc && pre < 2; ++a) {
    if (!acc_reads_values(P.accs[a].kind)) continue;
    const int idx = add(P.cols[P.accs[a].arg_slot].data, 8, 0);
    if (pre == 0) S.i_arg0 = idx; else S.i_arg1 = idx;
    ++pre;
  }
  if (P.pred_kind == 1) S.i_pred = add(P.cols[P.sp_slot].data, 8, 0);
  if (P.key_kind == KEY_BYTES) {
    const double avg = (double)key_bytes / (double)P.n_rows;
    int cap = (int)round_up((int64_t)(avg * HG_TILE * 1.0625) + 64, 1024);
    cap = std::max(2048, std::min(cap, 40 * 1024));
    S.key_bytes_off = off; S.key_bytes_cap = cap;
    off += cap + 32;
  }
  S.stage_bytes = (int)round_up(off, 128);
  const size_t smem = 2 * (size_t)S.stage_bytes;
  if (smem > 200 * 1024) return false;
  const void* fn = nullptr;
#define ARK_HG_R(K, PR, SG) (R == 1 ? (const void*)hash_agg_staged_kernel<K, PR, 1, SG> : (const void*)hash_agg_staged_kernel<K, PR, 2, SG>)
#define ARK_HG_FN(K, PR) (sig1 ? ARK_HG_R(K, PR, 1) : ARK_HG_R(K, PR, 0))
  if (P.key_kind == KEY_BYTES) fn = P.pred_kind ? ARK_HG_FN(KEY_BYTES, 1) : ARK_HG_FN(KEY_BYTES, 0);
  else fn = P.pred_kind ? ARK_HG_FN(KEY_INT64, 1) : ARK_HG_FN(KEY_INT64, 0);
#undef ARK_HG_FN
#undef ARK_HG_R
  ARK_CUDA(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
  int occ = 0;
  ARK_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, fn, HS_THREADS, smem));
  if (occ < 1) return false;
  const int sms = sm_count();
  static const int cap_per_sm = [] { const char* e = getenv("ARK_AGG_STREAM_CTAS"); return e ? atoi(e) : 0; }();
  if (cap_per_sm > 0) occ = std::min(occ, cap_per_sm);
  const int n_tiles = (int)ceil_div(P.n_rows, HG_TILE);
  const int grid = std::max(1, std::min(n_tiles, sms * occ));
  // its own name, and hash_agg_kernel: the time of the GROUP BY table kernel, whichever ran (bench.py reads it)
  KernelTimer t("hash_agg_staged_kernel", stream, "hash_agg_kernel");
  void* args[] = {(void*)&P, (void*)&S};
  ARK_CUDA(cudaLaunchKernel(fn, dim3(grid), dim3(HS_THREADS), args, smem, stream));
  return true;
}

}  // namespace

// Returns false when the plan / batch shape is not covered (the caller then uses hash_agg_kernel).
bool launch_hash_agg_stream(const AggParams& P, unsigned long long capacity, int64_t key_bytes, cudaStream_t stream) {
  static const int enabled = [] { const char* e = getenv("ARK_AGG_STREAM"); return e ? atoi(e) : 1; }();
  if (!enabled) return false;
  if (P.pred_kind == 2 || (P.key_kind != KEY_BYTES && P.key_kind != KEY_INT64)) return false;
  if (capacity > (1ull << 31) || P.n_rows <= 0) return false;
  for (int a = 0; a < P.n_acc; ++a) if (P.accs[a].arg_prog >= 0) return false;
  if (P.pred_kind == 1 && (reinterpret_cast<uintptr_t>(P.cols[P.sp_slot].data) & 7)) return false;
  static const int rows_per_thread = [] { const char* e = getenv("ARK_AGG_STREAM_R"); const int v = e ? atoi(e) : 1; return v == 1 || v == 4 ? v : 2; }();
  const int R = rows_per_thread;
  static const int dbg_knob = [] { const char* e = getenv("ARK_AGG_DEBUG"); return e ? atoi(e) : 0; }();  // measurement knob, results void
  // 2: every stream by TMA, 1: register prefetch.  Unless ARK_AGG_STREAM_V says otherwise, the staged kernel runs while
  // the table fits in the L2 and the register-prefetch kernel once it does not: measured on H100 (50 MB L2), staged is
  // faster at 10^4-10^5 keys (tables of 1-8 MB) and slower at 10^6-4·10^6 keys (64-256 MB), DESIGN.md §8.
  static const int version_env = [] { const char* e = getenv("ARK_AGG_STREAM_V"); return e ? atoi(e) : 0; }();
  static const unsigned long long l2_bytes = [] { int d = 0, v = 0; cudaGetDevice(&d); cudaDeviceGetAttribute(&v, cudaDevAttrL2CacheSize, d); return (unsigned long long)v; }();
  const int version = version_env ? version_env : (table_bytes(capacity, P.n_acc) > l2_bytes ? 1 : 2);
  if (version == 2) {
    if (P.key_kind == KEY_BYTES && key_bytes < 0) return false;
    const bool sig1_ = P.n_acc == 2 && P.accs[0].kind == ACC_COUNT_STAR && P.accs[1].kind == ACC_SUM_I64 && P.cols[P.accs[1].arg_slot].validity == nullptr;
    if (launch_staged(P, key_bytes, R == 4 ? 2 : R, sig1_, dbg_knob, stream)) return true;
  }
  const int TR = HS_THREADS * R;
  int cap = 0;
  if (P.key_kind == KEY_BYTES) {
    if (key_bytes < 0) return false;  // the caller resolves the key column's extent first
    const double avg = (double)key_bytes / (double)P.n_rows;
    cap = (int)round_up((int64_t)(avg * TR * 1.0625) + 64, 1024);
    cap = std::max(2048, std::min(cap, 48 * 1024));
  }
  const size_t smem = cap ? 2 * (size_t)(cap + 32) : 0;
  // {COUNT(*), SUM(non-null Int64 column)}: the specialised accumulate
  const bool sig1 = P.n_acc == 2 && P.accs[0].kind == ACC_COUNT_STAR && P.accs[1].kind == ACC_SUM_I64 && P.cols[P.accs[1].arg_slot].validity == nullptr;
  const void* fn = nullptr;
#define ARK_HS_R(K, PR, S) (R == 1 ? (const void*)hash_agg_stream_kernel<K, PR, 1, S> : R == 4 ? (const void*)hash_agg_stream_kernel<K, PR, 4, S> : (const void*)hash_agg_stream_kernel<K, PR, 2, S>)
#define ARK_HS_FN(K, PR) (sig1 ? ARK_HS_R(K, PR, 1) : ARK_HS_R(K, PR, 0))
  if (P.key_kind == KEY_BYTES) fn = P.pred_kind ? ARK_HS_FN(KEY_BYTES, 1) : ARK_HS_FN(KEY_BYTES, 0);
  else fn = P.pred_kind ? ARK_HS_FN(KEY_INT64, 1) : ARK_HS_FN(KEY_INT64, 0);
#undef ARK_HS_FN
#undef ARK_HS_R
  ARK_CUDA(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, 2 * (48 * 1024 + 32)));
  int occ = 0;
  ARK_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, fn, HS_THREADS, smem));
  if (occ < 1) return false;
  const int sms = sm_count();
  static const int cap_per_sm = [] { const char* e = getenv("ARK_AGG_STREAM_CTAS"); return e ? atoi(e) : 0; }();
  if (cap_per_sm > 0) occ = std::min(occ, cap_per_sm);
  const int n_tiles = (int)ceil_div(P.n_rows, TR);
  const int grid = std::max(1, std::min(n_tiles, sms * occ));
  KernelTimer t("hash_agg_stream_kernel", stream, "hash_agg_kernel");  // as in launch_staged
  static const int dbg = [] { const char* e = getenv("ARK_AGG_DEBUG"); return e ? atoi(e) : 0; }();  // measurement knob, results void
  void* args[] = {(void*)&P, (void*)&cap, (void*)&dbg};
  ARK_CUDA(cudaLaunchKernel(fn, dim3(grid), dim3(HS_THREADS), args, smem, stream));
  return true;
}

}  // namespace ark
