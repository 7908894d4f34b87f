// hash_agg_stream.cu — GROUP BY for high-cardinality keys: the row kernel of hash_agg.cu rebuilt as a persistent,
// software-pipelined kernel.
//
// hash_agg_kernel (hash_agg.cu) walks one row per thread through three DEPENDENT memory latencies — offsets → key
// bytes → table slot — so its warps stall on long scoreboards with most issue slots and most of the HBM bandwidth
// idle.  Here:
//   * a CTA stays resident and takes 256-row tiles; the loads of the NEXT tile (offsets / Int64 keys / predicate
//     column into registers, the tile's key bytes by one 1-D TMA bulk copy into the other half of a two-stage ring)
//     are issued before the current tile is touched, so the only latency on a row's critical path is the table's;
//   * every thread owns one row of the tile: its home BUCKET (four keys, hash_agg.cuh) is read whole, and a row that
//     is not settled by its home bucket (4 % of the rows at load 0.48) continues with table_find_or_claim;
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


// one 8-byte value of row lr0 of a tile of `rows` rows (0 past the tile's end), read once
__device__ __forceinline__ unsigned long long ld_u64(const unsigned long long* src, int lr0, int rows) {
  unsigned long long v = 0;
  if (lr0 < rows) asm volatile("ld.global.nc.L1::no_allocate.u64 %0, [%1];" : "=l"(v) : "l"(src));
  return v;
}

// the key offset of row lr0; *offx: the one after it, where the next lane does not hold it (last lane, last row)
__device__ __forceinline__ void ld_off(const int32_t* os, bool fast, int lr0, int rows, int lane, int* off, int* offx) {
  if (fast) asm volatile("ld.global.nc.L1::no_allocate.s32 %0, [%1];" : "=r"(*off) : "l"(os));
  else *off = (lr0 <= rows) ? os[0] : 0;
  *offx = ((lane == 31 || lr0 + 1 >= rows) && lr0 + 1 <= rows) ? os[1] : 0;
}

// SIG 1: the accumulators are exactly {COUNT(*), SUM(<non-null Int64 column>)} (config 3): two REDs, no dispatch.
template <int KEYK, int PRED, int SIG>
__global__ void __launch_bounds__(HS_THREADS) hash_agg_stream_kernel(const __grid_constant__ AggParams P, const int str_cap) {
  constexpr int TR = HS_THREADS;
  constexpr int PRODUCER = HS_THREADS - 32;
  extern __shared__ __align__(16) uint8_t smem[];  // KEY_BYTES: [key bytes stage 0][stage 1], each str_cap + 32
  __shared__ __align__(8) unsigned long long s_bar[2];
  __shared__ int s_str_base[2], s_str_staged[2];
  const int tid = threadIdx.x, lane = tid & 31;
  const int64_t n = P.n_rows;
  const int n_tiles = (int)((n + TR - 1) / TR);
  const int lr0 = tid;
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
  int offn = 0, offxn = 0;
  unsigned long long kvn = 0, pvn = 0;
  auto prefetch = [&](int t) {
    const int64_t r0 = (int64_t)t * TR;
    const int rows = tile_rows(t);
    const bool full = lr0 + 1 <= rows;
    if (KEYK == KEY_BYTES) {
      const int32_t* os = kc.offsets + r0 + lr0;
      ld_off(os, full && (reinterpret_cast<uintptr_t>(os) & 3) == 0, lr0, rows, lane, &offn, &offxn);
    } else {
      kvn = ld_u64((const unsigned long long*)kc.data + r0 + lr0, lr0, rows);
    }
    if (PRED == 1) pvn = ld_u64((const unsigned long long*)P.cols[P.sp_slot].data + r0 + lr0, lr0, rows);
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
    const int64_t row = row0 + lr0;
    const int off0 = offn, offx = offxn;
    const unsigned long long kv = kvn, pv = pvn;
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
    unsigned long long av[HS_PRE];
#pragma unroll
    for (int i = 0; i < HS_PRE; ++i)
      av[i] = pre_acc[i] >= 0 ? ld_u64((const unsigned long long*)P.cols[P.accs[pre_acc[i]].arg_slot].data + row, lr0, rows) : 0;
    // ---- predicate ----
    bool ok = lr0 < rows;
    if (PRED == 1 && ok) {
      const ColView& c = P.cols[P.sp_slot];
      ok = cmp_i64(P.sp_cmp, P.sp_is_f64 ? f64_total_key(pv) : (long long)pv, pred_c) && col_valid(c, row);
    }
    // ---- key ----
    Key16 mine;
    unsigned home = 0;
    if (KEYK == KEY_BYTES) {
      int off1 = __shfl_down_sync(0xffffffffu, off0, 1);
      if ((lane == 31 || lr0 + 1 >= rows) && lr0 + 1 <= rows) off1 = offx;
      const bool staged = s_str_staged[st];
      const int base = s_str_base[st];
      if (staged) { mbar_wait(&s_bar[st], (ph >> st) & 1); ph ^= 1u << st; }
      const uint8_t* in_bytes = smem + st * stage_bytes;
      if (ok) {
        unsigned h32;
        if (!col_valid(kc, row)) { mine.lo = 0; mine.hi = (unsigned long long)KEYTAG_NULL << 32; h32 = hash32_key16(mine); }
        else if (staged) { make_key_smem(in_bytes + (off0 - base), off1 - off0, row, &mine, &h32); if (off1 - off0 > 12) long_flag = 1; }
        else {
          int llen = 0;
          const uint8_t* lp = make_key_raw(KEY_BYTES, kc, row, &mine, &llen);
          if (lp) { const unsigned long long h = hash_bytes(lp, llen); h32 = (unsigned)(h >> 32) ^ (unsigned)h; long_flag = 1; }
          else h32 = hash32_key16(mine);
        }
        home = (unsigned)((h32 * 0x9E3779B1u) & bmask);
      }
    } else if (ok) {
      if (col_valid(kc, row)) { mine.lo = kv; mine.hi = (unsigned long long)KEYTAG_INT << 32; }
      else { mine.lo = 0; mine.hi = (unsigned long long)KEYTAG_NULL << 32; }
      home = (unsigned)((hash32_key16(mine) * 0x9E3779B1u) & bmask);
    }
    // this stage's key bytes are in registers: the producer may refill it in the iteration after next.  The barrier
    // also carries the producer's poll of the overflow flag to every thread (CTA-uniform exit).
    if (__syncthreads_or(stop)) {
      // a bulk copy for the next tile may be in flight into this CTA's shared memory: let it land before leaving
      if (KEYK == KEY_BYTES && next < n_tiles && s_str_staged[st ^ 1]) mbar_wait(&s_bar[st ^ 1], (ph >> (st ^ 1)) & 1);
      break;
    }
    if (!ok) continue;
    // ---- the home bucket ----
    Key16* b = reinterpret_cast<Key16*>(P.table + (unsigned long long)home * (unsigned long long)bstride);
    Key16 kb[TBL_B];
    ld256_keys(b, &kb[0], &kb[1]);
    ld256_keys(b + 2, &kb[2], &kb[3]);
    unsigned long long slot = ~0ull;
    bool done = false;
#pragma unroll
    for (int i = 0; i < TBL_B; ++i) {
      if (done) continue;
      Key16 c = kb[i];
      if (c.hi == KEY_EMPTY) {
        c = cas128(b + i, Key16{KEY_EMPTY, KEY_EMPTY}, mine);
        if (c.hi == KEY_EMPTY && c.lo == KEY_EMPTY) { ++claimed; done = true; slot = (unsigned long long)home * TBL_B + i; continue; }
      }
      if (key_equal(mine, c, kc, kc)) { done = true; slot = (unsigned long long)home * TBL_B + i; }
    }
    if (!done) {  // the home bucket is full of other keys: walk on
      slot = table_find_or_claim(P.table, bmask, bstride, (unsigned long long)home + 1, mine, kc, kc, &claimed);
      if (slot == ~0ull) { err_overflow = 1; continue; }  // table too loaded for this batch
    }
    // ---- accumulate (fire-and-forget REDs) ----
    if (SIG == 1) {
      atomicAdd(tbl_acc(P.table, slot, 0, bstride), 1ull);
      atomicAdd(tbl_acc(P.table, slot, 1, bstride), av[0]);
    } else {
      for (int a = 0; a < P.n_acc; ++a) {
        const AccParam& A = P.accs[a];
        unsigned long long bits = 0;
        bool valid = true;
        if (A.kind != ACC_COUNT_STAR) {
          const ColView& c = P.cols[A.arg_slot];
          valid = col_valid(c, row);
          if (A.kind != ACC_COUNT) bits = a == pre_acc[0] ? av[0] : (a == pre_acc[1] ? av[1] : __ldcs((const unsigned long long*)c.data + row));
        }
        if (valid) accumulate(A.kind, A.arg_is_f64, tbl_acc(P.table, slot, a, bstride), bits);
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
// owns rows t, t + 256, …: consecutive lanes read consecutive 12-byte keys, conflict-free) and taken one at a time.
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
};

template <int KEYK, int PRED, int SIG>
__global__ void __launch_bounds__(HS_THREADS, 4) hash_agg_staged_kernel(const __grid_constant__ AggParams P, const __grid_constant__ StagedParams S) {
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
    for (int q = 0; q < HG_TILE / HS_THREADS; ++q) {
      const int i = q * HS_THREADS + tid;  // striped: consecutive lanes, consecutive rows
      const int64_t row = row0 + i;
      bool ok = i < rows;
      if (PRED == 1 && ok) {
        const unsigned long long pv = *reinterpret_cast<const unsigned long long*>(elem(S.i_pred, i));
        ok = cmp_i64(P.sp_cmp, P.sp_is_f64 ? f64_total_key(pv) : (long long)pv, pred_c) && col_valid(P.cols[P.sp_slot], row);
      }
      if (!ok) continue;
      const unsigned long long av0 = S.i_arg0 >= 0 ? *reinterpret_cast<const unsigned long long*>(elem(S.i_arg0, i)) : 0;
      const unsigned long long av1 = S.i_arg1 >= 0 ? *reinterpret_cast<const unsigned long long*>(elem(S.i_arg1, i)) : 0;
      Key16 mine;
      unsigned h32;
      if (!col_valid(kc, row)) { mine.lo = 0; mine.hi = (unsigned long long)KEYTAG_NULL << 32; h32 = hash32_key16(mine); }
      else if (KEYK == KEY_BYTES) {
        const int o0 = *reinterpret_cast<const int32_t*>(elem(S.i_off, i)), o1 = *reinterpret_cast<const int32_t*>(elem(S.i_off, i + 1));
        if (staged) { make_key_smem(stage + S.key_bytes_off + (o0 - str_base), o1 - o0, row, &mine, &h32); if (o1 - o0 > 12) long_flag = 1; }
        else {
          int llen = 0;
          const uint8_t* lp = make_key_raw(KEY_BYTES, kc, row, &mine, &llen);
          if (lp) { const unsigned long long h = hash_bytes(lp, llen); h32 = (unsigned)(h >> 32) ^ (unsigned)h; long_flag = 1; }
          else h32 = hash32_key16(mine);
        }
      } else {
        mine.lo = *reinterpret_cast<const unsigned long long*>(elem(S.i_key, i)); mine.hi = (unsigned long long)KEYTAG_INT << 32;
        h32 = hash32_key16(mine);
      }
      const unsigned home = (unsigned)((h32 * 0x9E3779B1u) & bmask);
      // ---- the home bucket: first the two keys of the bucket's first sector, the second sector only when neither of
      // them is the row's key or free (a bucket fills from slot 0; at the usual load factor of ≤ 0.5 three quarters of
      // the rows are settled by the first 32 bytes — one L2 request instead of two) ----
      Key16* b = reinterpret_cast<Key16*>(P.table + (unsigned long long)home * (unsigned long long)bstride);
      Key16 kb[2];
      ld256_keys(b, &kb[0], &kb[1]);
      unsigned long long slot = ~0ull;
      bool done = false;
#pragma unroll
      for (int half = 0; half < TBL_B / 2; ++half) {
        if (done) continue;
        Key16 k0 = kb[0], k1 = kb[1];
        if (half > 0) ld256_keys(b + 2 * half, &k0, &k1);
#pragma unroll
        for (int k = 0; k < 2; ++k) {
          if (done) continue;
          Key16 c = k == 0 ? k0 : k1;
          if (c.hi == KEY_EMPTY) {
            c = cas128(b + 2 * half + k, Key16{KEY_EMPTY, KEY_EMPTY}, mine);
            if (c.hi == KEY_EMPTY && c.lo == KEY_EMPTY) { ++claimed; done = true; slot = (unsigned long long)home * TBL_B + 2 * half + k; continue; }
          }
          if (key_equal(mine, c, kc, kc)) { done = true; slot = (unsigned long long)home * TBL_B + 2 * half + k; }
        }
      }
      if (!done) {  // the home bucket is full of other keys: walk on
        slot = table_find_or_claim(P.table, bmask, bstride, (unsigned long long)home + 1, mine, kc, kc, &claimed);
        if (slot == ~0ull) { err_overflow = 1; continue; }
      }
      // ---- accumulate (fire-and-forget REDs) ----
      if (SIG == 1) {
        atomicAdd(tbl_acc(P.table, slot, 0, bstride), 1ull);
        atomicAdd(tbl_acc(P.table, slot, 1, bstride), av0);
      } else {
        int pre = 0;
        for (int a = 0; a < P.n_acc; ++a) {
          const AccParam& A = P.accs[a];
          // the first two accumulators that read argument values are staged, numbered exactly as launch_staged adds them
          const int which = acc_reads_values(A.kind) ? pre++ : -1;
          unsigned long long bits = 0;
          bool valid = true;
          if (A.kind != ACC_COUNT_STAR) {
            const ColView& c = P.cols[A.arg_slot];
            valid = col_valid(c, row);
            if (A.kind != ACC_COUNT) bits = which == 0 ? av0 : (which == 1 ? av1 : __ldcs((const unsigned long long*)c.data + row));
          }
          if (valid) accumulate(A.kind, A.arg_is_f64, tbl_acc(P.table, slot, a, bstride), bits);
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

bool launch_staged(const AggParams& P, int64_t key_bytes, bool sig1, cudaStream_t stream) {
  StagedParams S;
  memset(&S, 0, sizeof S);
  S.i_off = S.i_key = S.i_arg0 = S.i_arg1 = S.i_pred = -1;
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
#define ARK_HG_FN(K, PR) (sig1 ? (const void*)hash_agg_staged_kernel<K, PR, 1> : (const void*)hash_agg_staged_kernel<K, PR, 0>)
  if (P.key_kind == KEY_BYTES) fn = P.pred_kind ? ARK_HG_FN(KEY_BYTES, 1) : ARK_HG_FN(KEY_BYTES, 0);
  else fn = P.pred_kind ? ARK_HG_FN(KEY_INT64, 1) : ARK_HG_FN(KEY_INT64, 0);
#undef ARK_HG_FN
  ARK_CUDA(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
  int occ = 0;
  ARK_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, fn, HS_THREADS, smem));
  if (occ < 1) return false;
  const int sms = sm_count();
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
// forced: AGG_KERNEL_STAGED or AGG_KERNEL_STREAM to take that kernel, AGG_KERNEL_AUTO to choose by the L2's size.
bool launch_hash_agg_stream(const AggParams& P, unsigned long long capacity, int64_t key_bytes, int forced, cudaStream_t stream) {
  if (P.pred_kind == 2 || (P.key_kind != KEY_BYTES && P.key_kind != KEY_INT64)) return false;
  if (capacity > (1ull << 31) || P.n_rows <= 0) return false;
  for (int a = 0; a < P.n_acc; ++a) if (P.accs[a].arg_prog >= 0) return false;
  if (P.pred_kind == 1 && (reinterpret_cast<uintptr_t>(P.cols[P.sp_slot].data) & 7)) return false;
  // {COUNT(*), SUM(non-null Int64 column)}: the specialised accumulate
  const bool sig1 = P.n_acc == 2 && P.accs[0].kind == ACC_COUNT_STAR && P.accs[1].kind == ACC_SUM_I64 && P.cols[P.accs[1].arg_slot].validity == nullptr;
  // Unless forced, the staged kernel runs while the table fits in the L2 and the register-prefetch kernel once it does
  // not: measured on H100 (50 MB L2), staged is faster at 10^4-10^5 keys (tables of 1-8 MB) and slower at 10^6-4·10^6
  // keys (64-256 MB), DESIGN.md §8.
  static const unsigned long long l2_bytes = [] { int d = 0, v = 0; cudaGetDevice(&d); cudaDeviceGetAttribute(&v, cudaDevAttrL2CacheSize, d); return (unsigned long long)v; }();
  const int kernel = forced ? forced : (table_bytes(capacity, P.n_acc) > l2_bytes ? AGG_KERNEL_STREAM : AGG_KERNEL_STAGED);
  if (kernel == AGG_KERNEL_STAGED) {
    if (P.key_kind == KEY_BYTES && key_bytes < 0) return false;
    if (launch_staged(P, key_bytes, sig1, stream)) return true;
  }
  int cap = 0;
  if (P.key_kind == KEY_BYTES) {
    if (key_bytes < 0) return false;  // the caller resolves the key column's extent first
    const double avg = (double)key_bytes / (double)P.n_rows;
    cap = (int)round_up((int64_t)(avg * HS_THREADS * 1.0625) + 64, 1024);
    cap = std::max(2048, std::min(cap, 48 * 1024));
  }
  const size_t smem = cap ? 2 * (size_t)(cap + 32) : 0;
  const void* fn = nullptr;
#define ARK_HS_FN(K, PR) (sig1 ? (const void*)hash_agg_stream_kernel<K, PR, 1> : (const void*)hash_agg_stream_kernel<K, PR, 0>)
  if (P.key_kind == KEY_BYTES) fn = P.pred_kind ? ARK_HS_FN(KEY_BYTES, 1) : ARK_HS_FN(KEY_BYTES, 0);
  else fn = P.pred_kind ? ARK_HS_FN(KEY_INT64, 1) : ARK_HS_FN(KEY_INT64, 0);
#undef ARK_HS_FN
  ARK_CUDA(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, 2 * (48 * 1024 + 32)));
  int occ = 0;
  ARK_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, fn, HS_THREADS, smem));
  if (occ < 1) return false;
  const int sms = sm_count();
  const int n_tiles = (int)ceil_div(P.n_rows, HS_THREADS);
  const int grid = std::max(1, std::min(n_tiles, sms * occ));
  KernelTimer t("hash_agg_stream_kernel", stream, "hash_agg_kernel");  // as in launch_staged
  void* args[] = {(void*)&P, (void*)&cap};
  ARK_CUDA(cudaLaunchKernel(fn, dim3(grid), dim3(HS_THREADS), args, smem, stream));
  return true;
}

}  // namespace ark
