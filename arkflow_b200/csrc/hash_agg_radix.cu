// hash_agg_radix.cu — GROUP BY by radix partitioning: an ALTERNATIVE to hash_agg_kernel that is kept, tested and
// measured, but is NOT taken by default (ARK_AGG_RADIX=1 enables it from 2^22 table slots, =2 from 2^16).
//
//   K1  agg_radix_partition_kernel: one CTA per 2048-row tile.  Predicate and key as in hash_agg_kernel;
//       the top bits of a 32-bit key hash name a *bucket* = one contiguous region of S table slots.
//       The tile is counting-sorted by bucket in shared memory and each bucket's run is appended to
//       that bucket's record array {Key16, value0, value1} (SoA; one atomicAdd per non-empty bucket
//       per tile reserves the range): sequential reads, run-coalesced writes.  (Scattering the
//       records straight from registers instead of sorting them first was measured 40 % slower.)
//   K2  agg_radix_bucket_kernel: one CTA per bucket.  The region's S slots live in shared memory
//       (smem_table.cuh); the bucket's records stream in coalesced, probe/claim/accumulate with
//       shared-memory atomics, and the finished region is written to the global table in the
//       layout hash_agg_kernel produces — so everything downstream (compaction, key/aggregate
//       emission, partition ordering for the multi-GPU exchange) is shared.
//
// History of the measurement (K1 + K2 vs hash_agg_kernel): while hash_agg_kernel still did one returning atomicAdd on a
// single counter per inserted group, it lost badly on large tables and this path won.  With that hot atomic gone the
// direct kernel is faster at 10^6 to 8·10^6 groups: moving every record through HBM twice costs more than the random
// table accesses it avoids, even with a 512 MB table.
// Covered shape = that of the tiled kernel (no VM programs), non-nullable argument columns, ≤ 2
// distinct argument columns.  A skewed key distribution overflows a bucket's record array; the
// kernels raise `skew`, and the caller reruns the batch through hash_agg_kernel.
#include <atomic>

#include "agg_acc.cuh"
#include "engine.h"
#include "hash_agg.cuh"
#include "hashkey.cuh"
#include "smem_table.cuh"

namespace ark {

namespace {

constexpr int RP_THREADS = 512;
constexpr int RP_ROWS = 4;
constexpr int RP_TILE = RP_THREADS * RP_ROWS;

struct RadixParams {
  Key16* rec_keys;             // [n_buckets * cap]
  unsigned long long* rec_v0;  // [n_buckets * cap] (nv ≥ 1)
  unsigned long long* rec_v1;  // (nv == 2)
  unsigned int* cursor;        // [n_buckets] records appended so far
  int32_t* skew;               // raised when a bucket's record array is full
  unsigned int cap;            // records per bucket
  int32_t log2_slots;          // S = 1 << log2_slots table slots per bucket
  int32_t log2_buckets;
  int32_t nv;
  int32_t v_slot[2];           // column slot of value 0 / 1
  int32_t acc_v[AGG_MAX_ACC];  // accumulator → value index, -1 = none (COUNT(*))
};

// bucket = top bits, slot inside the bucket's region = low bits of one 32-bit hash (disjoint: ≤ 12 + 12 bits)
__device__ __forceinline__ unsigned int bucket_of(unsigned int h32, int log2_buckets) { return h32 >> (32 - log2_buckets); }

template <int PRED>
__global__ void __launch_bounds__(RP_THREADS, 2) agg_radix_partition_kernel(const __grid_constant__ AggParams P, const __grid_constant__ RadixParams R) {
  extern __shared__ __align__(16) uint8_t smem[];
  const int NB = 1 << R.log2_buckets;
  Key16* s_keys = reinterpret_cast<Key16*>(smem);                                              // [RP_TILE] bucket-sorted
  unsigned long long* s_v0 = reinterpret_cast<unsigned long long*>(smem + RP_TILE * 16);          // [RP_TILE]
  unsigned long long* s_v1 = s_v0 + (R.nv >= 1 ? RP_TILE : 0);
  unsigned int* s_dst = reinterpret_cast<unsigned int*>(s_v1 + (R.nv >= 2 ? RP_TILE : 0));     // [RP_TILE] global record index
  unsigned int* s_cnt = s_dst + RP_TILE;                                                       // [NB] histogram, then reserved base
  unsigned int* s_start = s_cnt + NB;                                                          // [NB]
  __shared__ unsigned int s_warp_sums[RP_THREADS / 32];
  __shared__ unsigned int s_total;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int64_t n = P.n_rows;
  const int64_t row0 = (int64_t)blockIdx.x * RP_TILE;
  const ColView& kc = P.cols[P.key_slot];
  for (int i = tid; i < NB; i += RP_THREADS) s_cnt[i] = 0;
  __syncthreads();

  // ---- A: predicate, key, bucket, rank inside the bucket (shared-memory histogram) ----
  Key16 key[RP_ROWS];
  unsigned long long v0[RP_ROWS], v1[RP_ROWS];
  unsigned int br[RP_ROWS];  // bucket << 12 | rank; 0xFFFFFFFF = row dropped
  const long long pred_c = P.sp_is_f64 ? f64_total_key(P.sp_const) : (long long)P.sp_const;
#pragma unroll
  for (int j = 0; j < RP_ROWS; ++j) {
    const int64_t row = row0 + j * RP_THREADS + tid;
    bool ok = row < n;
    if (PRED == 1 && ok) {
      const ColView& c = P.cols[P.sp_slot];
      const unsigned long long v = __ldcs((const unsigned long long*)c.data + row);
      ok = cmp_i64(P.sp_cmp, P.sp_is_f64 ? f64_total_key(v) : (long long)v, pred_c) && col_valid(c, row);
    }
    br[j] = 0xFFFFFFFFu;
    v0[j] = 0; v1[j] = 0;
    if (ok) {
      int llen = 0;
      const uint8_t* lp = make_key_raw(P.key_kind, kc, row, &key[j], &llen);
      unsigned int h32;
      if (lp) { const unsigned long long h = hash_bytes(lp, llen); h32 = (unsigned)(h >> 32) ^ (unsigned)h; }
      else h32 = hash32_key16(key[j]);
      const unsigned int b = bucket_of(h32, R.log2_buckets);
      br[j] = (b << 12) | atomicAdd(&s_cnt[b], 1u);
      if (R.nv >= 1) v0[j] = __ldcs((const unsigned long long*)P.cols[R.v_slot[0]].data + row);
      if (R.nv >= 2) v1[j] = __ldcs((const unsigned long long*)P.cols[R.v_slot[1]].data + row);
    }
  }
  __syncthreads();

  // ---- B: exclusive scan of the histogram; reserve each non-empty bucket's run in its record array ----
  {
    const int per = (NB + RP_THREADS - 1) / RP_THREADS;
    const int lo = tid * per, hi = min(lo + per, NB);
    unsigned int sum = 0;
    for (int i = lo; i < hi; ++i) sum += s_cnt[i];
    unsigned int incl = sum;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const unsigned int t = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += t; }
    if (lane == 31) s_warp_sums[warp] = incl;
    __syncthreads();
    unsigned int wbase = 0;
#pragma unroll
    for (int w = 0; w < RP_THREADS / 32; ++w) wbase += (w < warp) ? s_warp_sums[w] : 0;
    unsigned int run = wbase + incl - sum;
    for (int i = lo; i < hi; ++i) {
      const unsigned int c = s_cnt[i];
      s_start[i] = run;
      run += c;
      if (c) {
        const unsigned int g = atomicAdd(R.cursor + i, c);
        s_cnt[i] = g;
        if (g + c > R.cap) atomicExch(R.skew, 1);
      }
    }
    if (tid == RP_THREADS - 1) s_total = run;
  }
  __syncthreads();

  // ---- C: records into bucket order ----
#pragma unroll
  for (int j = 0; j < RP_ROWS; ++j) {
    if (br[j] == 0xFFFFFFFFu) continue;
    const unsigned int b = br[j] >> 12, rank = br[j] & 0xFFFu;
    const unsigned int d = s_start[b] + rank;
    const unsigned int pos = s_cnt[b] + rank;
    s_keys[d] = key[j];
    if (R.nv >= 1) s_v0[d] = v0[j];
    if (R.nv >= 2) s_v1[d] = v1[j];
    s_dst[d] = pos < R.cap ? b * R.cap + pos : 0xFFFFFFFFu;
  }
  __syncthreads();

  // ---- D: runs out to the bucket record arrays ----
  const unsigned int total = s_total;
  for (unsigned int i = tid; i < total; i += RP_THREADS) {
    const unsigned int g = s_dst[i];
    if (g == 0xFFFFFFFFu) continue;
    R.rec_keys[g] = s_keys[i];
    if (R.nv >= 1) R.rec_v0[g] = s_v0[i];
    if (R.nv >= 2) R.rec_v1[g] = s_v1[i];
  }
}

constexpr int RB_U = 2;

__global__ void __launch_bounds__(1024) agg_radix_bucket_kernel(const __grid_constant__ AggParams P, const __grid_constant__ RadixParams R) {
  extern __shared__ __align__(16) uint8_t smem[];
  const int S = 1 << R.log2_slots;
  Key16* K = reinterpret_cast<Key16*>(smem);                                       // [S]
  unsigned long long* ACC = reinterpret_cast<unsigned long long*>(smem + S * 16);  // [n_acc][S]
  __shared__ unsigned int s_groups;
  const int tid = threadIdx.x, nthreads = blockDim.x;
  const unsigned int b = blockIdx.x;
  const ColView& kc = P.cols[P.key_slot];
  for (int s = tid; s < S; s += nthreads) {
    K[s] = Key16{KEY_EMPTY, KEY_EMPTY};
    for (int a = 0; a < P.n_acc; ++a) ACC[a * S + s] = acc_identity(P.accs[a].kind);
  }
  if (tid == 0) s_groups = 0;
  __syncthreads();

  const unsigned int cnt = min(R.cursor[b], R.cap);
  const Key16* rk = R.rec_keys + (size_t)b * R.cap;
  const unsigned long long* r0 = R.nv >= 1 ? R.rec_v0 + (size_t)b * R.cap : nullptr;
  const unsigned long long* r1 = R.nv >= 2 ? R.rec_v1 + (size_t)b * R.cap : nullptr;
  unsigned int claimed = 0;
  bool full = false;
  const int n_acc = P.n_acc;
  const int kind0 = P.accs[0].kind, f0 = P.accs[0].arg_is_f64, vi0 = R.acc_v[0];
  const int kind1 = P.accs[1].kind, f1 = P.accs[1].arg_is_f64, vi1 = R.acc_v[1];
  for (unsigned int i0 = tid; i0 < cnt; i0 += nthreads * RB_U) {
    Key16 key[RB_U];
    unsigned long long v0[RB_U], v1[RB_U];
    int slot[RB_U];
#pragma unroll
    for (int u = 0; u < RB_U; ++u) {
      const unsigned int i = i0 + u * nthreads;
      v0[u] = 0; v1[u] = 0;
      if (i < cnt) {
        const uint4 q = __ldcs(reinterpret_cast<const uint4*>(rk + i));
        key[u].lo = (unsigned long long)q.x | ((unsigned long long)q.y << 32);
        key[u].hi = (unsigned long long)q.z | ((unsigned long long)q.w << 32);
        if (r0) v0[u] = __ldcs(r0 + i);
        if (r1) v1[u] = __ldcs(r1 + i);
      }
    }
#pragma unroll
    for (int u = 0; u < RB_U; ++u) {
      slot[u] = -1;
      if (i0 + u * nthreads >= cnt) continue;
      const unsigned int h32 = stored_key_hash32(key[u], kc);
      slot[u] = region_find_or_claim(K, S, h32 & (unsigned int)(S - 1), key[u], kc, &claimed);
      if (slot[u] < 0) full = true;
    }
    if (n_acc <= 2) {
#pragma unroll
      for (int u = 0; u < RB_U; ++u) {
        if (slot[u] < 0) continue;
        accumulate(kind0, f0, ACC + slot[u], vi0 == 0 ? v0[u] : v1[u]);
        if (n_acc == 2) accumulate(kind1, f1, ACC + S + slot[u], vi1 == 0 ? v0[u] : v1[u]);
      }
    } else {
      for (int a = 0; a < n_acc; ++a) {
        const int kind = P.accs[a].kind, is_f64 = P.accs[a].arg_is_f64, vi = R.acc_v[a];
        unsigned long long* acc = ACC + a * S;
#pragma unroll
        for (int u = 0; u < RB_U; ++u)
          if (slot[u] >= 0) accumulate(kind, is_f64, acc + slot[u], vi == 0 ? v0[u] : v1[u]);
      }
    }
  }
  if (claimed) atomicAdd(&s_groups, claimed);
  if (full) atomicExch(P.overflow, 1);
  __syncthreads();

  // ---- region → global table (the layout hash_agg_kernel builds); empty slots carry the EMPTY key ----
  const unsigned long long region0 = (unsigned long long)b << R.log2_slots;  // first slot of this bucket's region
  for (int s = tid; s < S; s += nthreads) {
    *tbl_key(P.table, region0 + s, P.bucket_stride) = K[s];
    for (int a = 0; a < P.n_acc; ++a) *tbl_acc(P.table, region0 + s, a, P.bucket_stride) = ACC[a * S + s];
  }
  if (tid == 0) {
    const unsigned int g = s_groups;
    if (g) atomicAdd(P.group_count, g);
    if (g > (unsigned int)(S - S / 8)) atomicExch(P.overflow, 1);  // a region this loaded probes far: retry with a larger table
  }
}

std::atomic<int> g_skew_backoff{0};

}  // namespace

// Fills P.table (capacity slots, NOT pre-initialised) through the partitioned path.  Returns false when the
// shape is not covered; *skew_flag_host is where the caller finds the skew flag after its own sync
// (the kernels raise it in device memory at `skew_dev`).  When the flag is set the table is garbage and
// the caller reruns with hash_agg_kernel.
bool launch_hash_agg_radix(const AggParams& P, unsigned long long capacity, int32_t* skew_dev, std::vector<BufferPtr>* keep, cudaStream_t stream) {
  const char* mode_env = getenv("ARK_AGG_RADIX");  // read per call (tests flip it): 0 = never (default), 1 = from 2^22 slots, 2 = from 2^16 rows / slots
  const int mode = mode_env ? atoi(mode_env) : 0;
  static const int log2_slots_env = [] { const char* e = getenv("ARK_AGG_RADIX_S"); return e ? atoi(e) : 12; }();
  if (!mode) return false;
  const int64_t n = P.n_rows;
  if (P.pred_kind == 2 || (P.key_kind != KEY_INT64 && P.key_kind != KEY_BYTES)) return false;
  if (n < (mode == 2 ? 1 << 16 : 1 << 20) || n >= (1ll << 31) || capacity < (mode == 2 ? 1ull << 16 : 1ull << 22)) return false;
  if (mode != 2 && g_skew_backoff.load() > 0) { g_skew_backoff.fetch_sub(1); return false; }
  RadixParams R;
  memset(&R, 0, sizeof R);
  for (int a = 0; a < P.n_acc; ++a) {
    const AccParam& A = P.accs[a];
    R.acc_v[a] = -1;
    if (A.arg_prog >= 0) return false;
    if (A.kind == ACC_COUNT_STAR) continue;
    // an argument with a validity buffer declines the path: the records carry no validity.  COUNT(x) of an argument
    // without one (nullable by schema only) counts every row and records no values: x may be a Utf8 / Binary / Boolean
    // column, which holds no 8-byte values
    if (P.cols[A.arg_slot].validity) return false;
    if (!acc_reads_values(A.kind)) continue;
    int vi = -1;
    for (int v = 0; v < R.nv; ++v) if (R.v_slot[v] == A.arg_slot) vi = v;
    if (vi < 0) { if (R.nv == 2) return false; vi = R.nv; R.v_slot[R.nv++] = A.arg_slot; }
    R.acc_v[a] = vi;
  }
  int log2_slots = log2_slots_env;
  log2_slots = std::min(12, std::max(9, log2_slots));
  while (log2_slots > 9 && ((size_t)(16 + 8 * P.n_acc) << log2_slots) > 160 * 1024) --log2_slots;
  const unsigned long long n_buckets = capacity >> log2_slots;
  if (n_buckets < 16 || n_buckets > 4096) return false;
  int log2_buckets = 0;
  while ((1ull << log2_buckets) < n_buckets) ++log2_buckets;
  const unsigned long long cap = (unsigned long long)((double)n / (double)n_buckets * 1.25) + 1024;
  if (cap * n_buckets >= 0xFFFFFFFFull) return false;
  R.log2_slots = log2_slots;
  R.log2_buckets = log2_buckets;
  R.cap = (unsigned int)cap;
  BufferPtr keys = device_alloc((size_t)cap * n_buckets * 16);
  BufferPtr v0 = R.nv >= 1 ? device_alloc((size_t)cap * n_buckets * 8) : BufferPtr();
  BufferPtr v1 = R.nv >= 2 ? device_alloc((size_t)cap * n_buckets * 8) : BufferPtr();
  BufferPtr cursor = device_alloc((size_t)n_buckets * 4);
  keep->push_back(keys); keep->push_back(cursor);
  if (v0) keep->push_back(v0);
  if (v1) keep->push_back(v1);
  R.rec_keys = (Key16*)keys.get();
  R.rec_v0 = (unsigned long long*)v0.get();
  R.rec_v1 = (unsigned long long*)v1.get();
  R.cursor = (unsigned int*)cursor.get();
  R.skew = skew_dev;
  ARK_CUDA(cudaMemsetAsync(cursor.get(), 0, (size_t)n_buckets * 4, stream));
  const size_t smem1 = (size_t)RP_TILE * (16 + 8 * R.nv + 4) + (size_t)n_buckets * 8;
  const size_t smem2 = (size_t)(16 + 8 * P.n_acc) << log2_slots;
  static bool configured = false;
  if (!configured) {
    ARK_CUDA(cudaFuncSetAttribute(agg_radix_partition_kernel<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, 128 * 1024));
    ARK_CUDA(cudaFuncSetAttribute(agg_radix_partition_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, 128 * 1024));
    ARK_CUDA(cudaFuncSetAttribute(agg_radix_bucket_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    configured = true;
  }
  {
    KernelTimer t("agg_radix_partition_kernel", stream);
    const unsigned grid = (unsigned)ceil_div(n, RP_TILE);
    if (P.pred_kind == 0) agg_radix_partition_kernel<0><<<grid, RP_THREADS, smem1, stream>>>(P, R);
    else agg_radix_partition_kernel<1><<<grid, RP_THREADS, smem1, stream>>>(P, R);
  }
  {
    KernelTimer t("agg_radix_bucket_kernel", stream);
    agg_radix_bucket_kernel<<<(unsigned)n_buckets, (1 << log2_slots) / 4, smem2, stream>>>(P, R);
  }
  return true;
}

void hash_agg_radix_note_skew() { g_skew_backoff.store(16); }

}  // namespace ark
