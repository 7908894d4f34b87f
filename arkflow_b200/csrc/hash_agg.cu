// hash_agg.cu — GROUP BY hash-aggregate: WHERE + key hashing + accumulate in one pass over the
// input, against an open-addressing table in HBM whose hot part the L2 (50 MB on H100) keeps.
//
// Stands in for DataFusion's AggregateExec(Partial) → RepartitionExec(Hash) → AggregateExec(Final)
// (third-party; reached from crates/arkflow-plugin/src/processor/sql.rs:126-129).  The same kernel
// runs the *final* merge of partial states on the multi-GPU path (sum of sums / counts, min of mins).
//
// Table: buckets of four slots — four Key16 keys (two sectors) followed by one sector per accumulator (hash_agg.cuh);
// a probe reads a whole bucket, a key is claimed with a single 128-bit CAS (ATOMG.CAS.128), accumulators take
// fire-and-forget RED atomics; a warp whose lanes all hit the same group reduces with shuffles first.
// Algorithmic traffic = key + argument bytes read once (SURVEY.md §8(d): 24 B/row for config 3).
#include <cub/device/device_scan.cuh>

#include "agg_acc.cuh"
#include "engine.h"
#include "group_exchange.h"
#include "hash_agg.cuh"
#include "hashkey.cuh"
#include "vm.cuh"

namespace ark {

namespace {

__global__ void agg_init_kernel(uint8_t* table, unsigned long long capacity, int bstride, int n_acc, AccParam a0, AccParam a1, AccParam a2,
                                AccParam a3, AccParam a4, AccParam a5, AccParam a6, AccParam a7) {
  const AccParam accs[AGG_MAX_ACC] = {a0, a1, a2, a3, a4, a5, a6, a7};
  for (unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; i < capacity;
       i += (unsigned long long)gridDim.x * blockDim.x) {
    *tbl_key(table, i, bstride) = Key16{KEY_EMPTY, KEY_EMPTY};
    for (int a = 0; a < n_acc; ++a) {
      unsigned long long init = 0;
      if (accs[a].kind == ACC_MIN_I64 || accs[a].kind == ACC_MIN_F64) init = 0x7FFFFFFFFFFFFFFFull;
      if (accs[a].kind == ACC_MAX_I64 || accs[a].kind == ACC_MAX_F64) init = 0x8000000000000000ull;
      *tbl_acc(table, i, a, bstride) = init;
    }
  }
}

// a cached table starts its next batch: the keys stay, every accumulator goes back to its identity
__global__ void agg_reset_acc_kernel(uint8_t* table, unsigned long long capacity, int bstride, int n_acc, AccParam a0, AccParam a1, AccParam a2,
                                     AccParam a3, AccParam a4, AccParam a5, AccParam a6, AccParam a7) {
  const AccParam accs[AGG_MAX_ACC] = {a0, a1, a2, a3, a4, a5, a6, a7};
  const unsigned long long lanes = capacity * (unsigned long long)n_acc;
  for (unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; i < lanes; i += (unsigned long long)gridDim.x * blockDim.x) {
    const unsigned long long bucket = i / (4ull * n_acc), r = i % (4ull * n_acc);
    const int a = (int)(r / 4), lane = (int)(r % 4);
    unsigned long long init = 0;
    if (accs[a].kind == ACC_MIN_I64 || accs[a].kind == ACC_MIN_F64) init = 0x7FFFFFFFFFFFFFFFull;
    if (accs[a].kind == ACC_MAX_I64 || accs[a].kind == ACC_MAX_F64) init = 0x8000000000000000ull;
    *tbl_acc(table, bucket * 4 + lane, a, bstride) = init;
  }
}

constexpr int AGG_THREADS = 256;

// home-slot hash of this kernel's table: the 32-bit key hash spread over 64 bits (a quarter of hash_key16's
// instructions; the 64-bit hash stays what partitions groups across GPUs, see partition_of)
__device__ __forceinline__ unsigned long long table_hash(int key_kind, const ColView& c, int64_t row, Key16* key) {
  int llen = 0;
  const uint8_t* lp = make_key_raw(key_kind, c, row, key, &llen);
  if (key_kind == KEY_NONE) return 0;
  if (lp) return hash_bytes(lp, llen);
  const unsigned h = hash32_key16(*key);
  return ((unsigned long long)h << 32) | (h * 0x9E3779B1u);
}

// The general row kernel: one row per thread per iteration, any predicate (simple or VM program), any key kind,
// computed aggregate arguments.  High-cardinality plain-column queries take hash_agg_stream.cu instead.
template <int PRED>
__global__ void __launch_bounds__(AGG_THREADS) hash_agg_kernel(const __grid_constant__ AggParams P) {
  const int lane = threadIdx.x & 31;
  const int64_t n = P.n_rows;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  const int bstride = P.bucket_stride;
  const unsigned long long bmask = P.mask >> 2;
  int32_t err = 0;
  const ColView& kc = P.cols[P.key_kind == KEY_NONE ? 0 : P.key_slot];
  if (P.key_kind == KEY_NONE && blockIdx.x == 0 && threadIdx.x == 0) {
    // a global aggregate always yields one row, even when no row survives the filter
    Key16 mine; unsigned long long h;
    make_key(KEY_NONE, kc, 0, &mine, &h);
    unsigned int c = 0;
    table_find_or_claim(P.table, bmask, bstride, h, mine, kc, kc, &c);
    if (c) atomicAdd(P.group_count, c);
  }
  __shared__ volatile int32_t s_stop;
  if (threadIdx.x == 0) s_stop = 0;
  __syncthreads();
  unsigned int claimed = 0;
  for (int64_t base = (int64_t)blockIdx.x * blockDim.x; base < n; base += stride) {
    // A table that is too small (first batch of a high-cardinality stream): once some row has raised `overflow` the
    // launch is void (the host retries with 4× the slots), so stop instead of walking a full table with every
    // remaining row.  ONE thread per CTA polls the flag — every thread polling the same L2 line was measurably slower —
    // and the other warps pick it up from shared memory an iteration later.
    if (threadIdx.x == 0) s_stop = *reinterpret_cast<volatile int32_t*>(P.overflow);
    if (__any_sync(0xffffffffu, s_stop != 0)) break;  // warp-uniform: the full-mask shuffles below need every lane
    const int64_t row = base + threadIdx.x;
    bool ok = row < n;
    if (PRED == 1) {
      if (ok) {
        const ColView& c = P.cols[P.sp_slot];
        const unsigned long long v = __ldcs((const unsigned long long*)c.data + row);
        if (P.sp_is_f64) ok = cmp_i64(P.sp_cmp, f64_total_key(v), f64_total_key(P.sp_const));
        else ok = cmp_i64(P.sp_cmp, (int64_t)v, (int64_t)P.sp_const);
        ok = ok && col_valid(c, row);
      }
    } else if (PRED == 2) {
      if (ok) { VmVal v = vm_eval(P.pred, P.cols, row, &err); ok = v.valid && (v.bits & 1); }
    }
    unsigned long long slot = 0;
    if (ok) {
      Key16 mine;
      if (P.key_kind == KEY_PAIR) {
        const ColView& k2 = P.cols[P.key_slot2];
        *P.long_seen = 1;  // pair keys are stored by row reference
        const unsigned long long h = make_pair_key(P.key_kind1, kc, P.key_kind2, k2, row, &mine);
        slot = table_find_or_claim_pair(P.table, bmask, bstride, h, mine, P.key_kind1, kc, P.key_kind2, k2, &claimed);
      } else {
        const unsigned long long h = table_hash(P.key_kind, kc, row, &mine);
        if (key_is_long(mine)) *P.long_seen = 1;
        slot = table_find_or_claim(P.table, bmask, bstride, h, mine, kc, kc, &claimed);
      }
      if (slot == ~0ull) { atomicExch(P.overflow, 1); ok = false; }  // the table is too loaded for this batch
    }
    // ---- accumulate; a warp whose lanes all hit one group reduces with shuffles first ----
    const unsigned m = __ballot_sync(0xffffffffu, ok);
    if (m == 0) continue;
    const int leader = __ffs(m) - 1;
    const unsigned long long slot0 = __shfl_sync(0xffffffffu, slot, leader);
    const bool uniform = __all_sync(0xffffffffu, !ok || slot == slot0) && __popc(m) > 1;
    for (int a = 0; a < P.n_acc; ++a) {
      const AccParam& A = P.accs[a];
      unsigned long long bits = 0;
      bool valid = ok;
      if (ok && A.kind != ACC_COUNT_STAR) {
        if (A.arg_prog >= 0) { VmVal v = vm_eval(P.progs[A.arg_prog], P.cols, row, &err); bits = v.bits; valid = v.valid; }
        else {
          // COUNT(x) needs x's validity only: x may be a Utf8 / Binary / Boolean column, whose data buffer does not hold
          // 8-byte values
          const ColView& c = P.cols[A.arg_slot];
          valid = col_valid(c, row);
          bits = valid && A.kind != ACC_COUNT ? __ldcs((const unsigned long long*)c.data + row) : 0;
        }
      }
      unsigned long long* dst = tbl_acc(P.table, uniform ? slot0 : slot, a, bstride);
      switch (A.kind) {
        case ACC_COUNT_STAR:
        case ACC_COUNT: {
          if (uniform) { const int c = __popc(__ballot_sync(0xffffffffu, valid)); if (lane == leader && c) atomicAdd(dst, (unsigned long long)c); }
          else if (valid) atomicAdd(dst, 1ull);
          break;
        }
        case ACC_SUM_I64: {
          if (uniform) { const long long sm = warp_sum_ll(valid ? (long long)bits : 0); if (lane == leader) atomicAdd(dst, (unsigned long long)sm); }
          else if (valid) atomicAdd(dst, bits);
          break;
        }
        case ACC_SUM_F64: {
          double x = A.arg_is_f64 ? __longlong_as_double((long long)bits) : (double)(long long)bits;
          if (uniform) { const double sm = warp_sum_f64(valid ? x : 0.0); if (lane == leader) atomicAdd((double*)dst, sm); }
          else if (valid) atomicAdd((double*)dst, x);
          break;
        }
        case ACC_MIN_I64: case ACC_MIN_F64: {
          long long x = A.kind == ACC_MIN_F64 ? f64_total_key(bits) : (long long)bits;
          if (uniform) { const long long sm = warp_min_ll(valid ? x : 0x7FFFFFFFFFFFFFFFll); if (lane == leader) atomicMin((long long*)dst, sm); }
          else if (valid) atomicMin((long long*)dst, x);
          break;
        }
        default: {
          long long x = A.kind == ACC_MAX_F64 ? f64_total_key(bits) : (long long)bits;
          if (uniform) { const long long sm = warp_max_ll(valid ? x : (long long)0x8000000000000000ull); if (lane == leader) atomicMax((long long*)dst, sm); }
          else if (valid) atomicMax((long long*)dst, x);
          break;
        }
      }
    }
  }
  claimed = (unsigned int)__reduce_add_sync(0xffffffffu, claimed);
  if (lane == 0 && claimed) atomicAdd(P.group_count, claimed);
  if (err) atomicExch(P.error, err);
}

// ---- table → dense group list, ordered by partition = hash(key) mod n_parts -----------------------
// need_count: the table carries keys of earlier batches too (AggHints::CachedTable): a slot belongs to THIS batch's
// result iff its COUNT(*) accumulator (always accumulator 0) is non-zero
__global__ void agg_count_parts_kernel(const uint8_t* table, int stride, unsigned long long capacity, ColView kc, int key_kind, int n_parts,
                                       unsigned int* part_counts, int need_count) {
  for (unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; i < capacity;
       i += (unsigned long long)gridDim.x * blockDim.x) {
    Key16 k = *tbl_key(table, i, stride);
    if (k.hi == KEY_EMPTY) continue;
    if (need_count && *tbl_acc(table, i, 0, stride) == 0) continue;
    const int p = n_parts > 1 ? partition_of(key_kind == KEY_NONE ? 0 : stored_key_hash(k, kc), n_parts) : 0;
    atomicAdd(part_counts + p, 1u);
  }
}

// part_cursor[p] starts at the exclusive prefix of part_counts; slots[] receives table slot ids
__global__ void agg_compact_kernel(const uint8_t* table, int stride, unsigned long long capacity, ColView kc, int key_kind, int n_parts,
                                   unsigned int* part_cursor, unsigned int* slots, int need_count) {
  for (unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; i < capacity;
       i += (unsigned long long)gridDim.x * blockDim.x) {
    Key16 k = *tbl_key(table, i, stride);
    if (k.hi == KEY_EMPTY) continue;
    if (need_count && *tbl_acc(table, i, 0, stride) == 0) continue;
    const int p = n_parts > 1 ? partition_of(key_kind == KEY_NONE ? 0 : stored_key_hash(k, kc), n_parts) : 0;
    slots[atomicAdd(part_cursor + p, 1u)] = (unsigned int)i;
  }
}

__global__ void agg_key_lengths_kernel(const uint8_t* table, int stride, const unsigned int* slots, unsigned int n_groups, int32_t* lens) {
  unsigned int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= n_groups) return;
  Key16 k = *tbl_key(table, slots[g], stride);
  const unsigned tag = (unsigned)(k.hi >> 32);
  lens[g] = tag == KEYTAG_NULL ? 0 : (int32_t)(tag & 0x7FFFFFFFu);
}

// materialise the key column of the dense group list
__global__ void agg_emit_keys_kernel(const uint8_t* table, int stride, const unsigned int* slots, unsigned int n_groups, ColView kc, int key_kind,
                                     unsigned long long* out_fixed, uint8_t* out_bool_bytes, const int32_t* out_offsets,
                                     uint8_t* out_bytes, uint8_t* out_valid_bytes) {
  unsigned int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= n_groups) return;
  Key16 k = *tbl_key(table, slots[g], stride);
  const unsigned tag = (unsigned)(k.hi >> 32);
  const bool is_null = tag == KEYTAG_NULL;
  if (out_valid_bytes) out_valid_bytes[g] = !is_null;
  if (key_kind == KEY_INT64) out_fixed[g] = is_null ? 0 : k.lo;
  else if (key_kind == KEY_BOOL) out_bool_bytes[g] = is_null ? 0 : (uint8_t)(k.lo & 1);
  else if (key_kind == KEY_BYTES && !is_null) {
    uint8_t* d = out_bytes + out_offsets[g];
    const int len = (int)(tag & 0x7FFFFFFFu);
    if (tag & KEYTAG_LONG) {
      const uint8_t* s = (const uint8_t*)kc.data + kc.offsets[(int64_t)k.lo];
      for (int i = 0; i < len; ++i) d[i] = s[i];
    } else {
      for (int i = 0; i < len; ++i) d[i] = (uint8_t)((i < 8 ? (k.lo >> (8 * i)) : (k.hi >> (8 * (i - 8)))) & 0xff);
    }
  }
}

// dense accumulator columns: gather acc[slots[g]]
__global__ void agg_gather_acc_kernel(const uint8_t* table, int stride, int acc, const unsigned int* slots, unsigned int n_groups,
                                      unsigned long long* out) {
  unsigned int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g < n_groups) out[g] = *tbl_acc(table, slots[g], acc, stride);
}

enum FinalOp : int32_t { FIN_COPY = 0, FIN_AVG = 1, FIN_F64_KEY_BACK = 2, FIN_CONST = 3 };
// out[g] = op(a[g], b[g]); valid[g] = (nn == null || nn[g] > 0)
__global__ void agg_finalize_kernel(int op, const unsigned long long* a, const unsigned long long* cnt, unsigned long long constant,
                                    unsigned int n_groups, unsigned long long* out, uint8_t* out_valid_bytes) {
  unsigned int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= n_groups) return;
  const bool valid = cnt == nullptr || cnt[g] > 0;
  unsigned long long r = 0;
  if (op == FIN_CONST) r = constant;
  else if (valid) {
    if (op == FIN_COPY) r = a[g];
    else if (op == FIN_AVG) r = (unsigned long long)__double_as_longlong(__longlong_as_double((long long)a[g]) / (double)cnt[g]);
    else { long long s = (long long)a[g]; r = (unsigned long long)(s ^ (long long)(((unsigned long long)(s >> 63)) >> 1)); }
  }
  out[g] = r;
  if (out_valid_bytes) out_valid_bytes[g] = valid;
}

template <int PRED>
void launch_agg(const AggParams& P, int64_t n, cudaStream_t stream) {
  // hash_agg_kernel also counts the staged and register-prefetch launches (hash_agg_stream.cu), which carry their own
  // names too: this kernel's launches are hash_agg_kernel minus those two
  KernelTimer t("hash_agg_kernel", stream);
  const int grid = (int)std::max<int64_t>(1, std::min<int64_t>(ceil_div(n, (int64_t)AGG_THREADS), sm_count() * 8));
  hash_agg_kernel<PRED><<<grid, AGG_THREADS, 0, stream>>>(P);
}

struct AccPlan {  // host-side description of one accumulator
  AccKind kind;
  int arg_slot = -1;
  int arg_prog = -1;
  bool arg_is_f64 = false;
};

}  // namespace

// ---- executor ---------------------------------------------------------------------------------------
// AggExec: the physical aggregate — key, accumulators, how SELECT items derive from them.
struct AggExec {
  int key_kind = KEY_NONE;
  int key_slot = 0;
  DType key_type = DType::Null;
  // two GROUP BY keys: key_kind == KEY_PAIR, the columns' own kinds / slots / types here
  int key_kind1 = KEY_NONE, key_kind2 = KEY_NONE, key_slot2 = 0;
  DType key_type2 = DType::Null;
  std::vector<AccPlan> accs;
  std::vector<VmProgram> progs;
  int find_or_add(const AccPlan& a) {
    for (size_t i = 0; i < accs.size(); ++i)
      if (accs[i].kind == a.kind && accs[i].arg_slot == a.arg_slot && accs[i].arg_prog == a.arg_prog && accs[i].arg_is_f64 == a.arg_is_f64)
        return (int)i;
    if ((int)accs.size() >= AGG_MAX_ACC) fail(ARK_ERR_UNSUPPORTED, "too many aggregate accumulators in one query");
    accs.push_back(a);
    return (int)accs.size() - 1;
  }
};

struct AggOutput {  // one aggregate of the SELECT list expressed over accumulators
  int value_acc = -1;    // accumulator holding the value (sum / min / max / count)
  int count_acc = -1;    // accumulator whose >0 decides validity (and divides for AVG); -1 ⇒ always valid
  int final_op = FIN_COPY;
  DType type = DType::Int64;
  bool can_be_null = false;  // count_acc is a dedicated non-null counter (argument may be NULL)
};

struct DenseGroups {  // result of the hash pass: dense arrays of G groups, partition-ordered
  unsigned int n_groups = 0;
  std::vector<int64_t> part_rows;
  BufferPtr table, slots;                // table + dense slot list
  int stride = 128;   // bucket stride (hash_agg.cuh: table layout)
  // table reuse across batches (AggHints::CachedTable)
  bool count_filter = false;            // occupied slots may belong to earlier batches: a group of this batch has COUNT(*) > 0
  bool cacheable = false;               // may go back to the plan's cache after this call
  unsigned long long total_keys = 0;    // keys in the table (all batches)
  int n_acc = 0;
  unsigned long long capacity = 0;
};

bool launch_hash_agg_tile(const AggParams& P, unsigned long long capacity, unsigned int groups_hint, int64_t key_bytes, cudaStream_t stream);
bool launch_hash_agg_stream(const AggParams& P, unsigned long long capacity, int64_t key_bytes, cudaStream_t stream);
bool launch_hash_agg_radix(const AggParams& P, unsigned long long capacity, int32_t* skew_dev, std::vector<BufferPtr>* keep, cudaStream_t stream);
void hash_agg_radix_note_skew();


// dense, partition-ordered slot list of a built table (n_parts = 1: plain compaction)
static void compact_groups(DenseGroups& dg, const ColView& kc, int key_kind, int n_parts, BufferPtr ctl, BufferPtr hctl, cudaStream_t stream);

// compact == false: stop once the table is built (the device-side exchange pushes the slots themselves)
static DenseGroups hash_pass(const Plan& plan, const AggExec& ex, Batch& in, int n_parts, cudaStream_t stream, bool compact = true, bool merge_mode = false) {
  const int64_t n = in.num_rows;
  AggHints& hints = *plan.hints;  // per plan: the table size this query needed last time
  unsigned long long capacity = std::max<unsigned long long>(hints.capacity.load(), 1ull << 10);
  const unsigned long long cap_limit = 1ull << 31;
  DenseGroups dg;
  BufferPtr ctl = device_alloc(512);  // [group_count u32 | overflow i32 | error i32 | skew i32 | part_counts u32[32] | part_cursor u32[32]]
  BufferPtr hctl = pinned_alloc(512);
  bool allow_radix = true;
  if (n_parts > 32) fail(ARK_ERR_UNSUPPORTED, "more than 32 partitions");
  static const unsigned long long tile_max = [] { const char* e = getenv("ARK_AGG_TILE_MAX"); return e ? (unsigned long long)atoll(e) : 1024ull; }();  // 2048 slots (≈ 1000 groups): 1.65 ms in the tile kernel vs 1.34 ms in hash_agg_kernel
  static const bool cache_enabled = [] { const char* e = getenv("ARK_AGG_TABLE_CACHE"); return !e || atoi(e) != 0; }();
  // reuse needs self-contained keys (no row references) and a COUNT(*) accumulator that tells this batch's groups apart
  const bool can_cache = cache_enabled && (ex.key_kind == KEY_INT64 || ex.key_kind == KEY_BYTES || ex.key_kind == KEY_BOOL) &&
                         !ex.accs.empty() && (ex.accs[0].kind == ACC_COUNT_STAR || merge_mode);
  bool fresh_only = false;
  while (true) {
    const int stride = table_bucket_stride((int)ex.accs.size());
    dg.stride = stride;
    dg.n_acc = (int)ex.accs.size();
    AggHints::CachedTable ct;
    bool reused = false;
    // tables of the low-cardinality path (≤ tile_max slots: per-CTA shared-memory tables) are cheap to rebuild and must
    // not be probed row by row (hot keys would serialise on L2 atomics): they are never reused
    const bool cache_now = can_cache && capacity > tile_max;
    if (cache_now && !fresh_only) {
      std::lock_guard<std::mutex> l(hints.cache_mu);
      for (size_t i = 0; i < hints.cache.size(); ++i)
        if (hints.cache[i].capacity == capacity && hints.cache[i].n_acc == dg.n_acc) { ct = hints.cache[i]; hints.cache.erase(hints.cache.begin() + i); reused = true; break; }
      if (!reused) hints.cache.clear();  // other sizes are of no use any more
    }
    dg.table = reused ? ct.table : device_alloc((size_t)table_bytes(capacity, (int)ex.accs.size()));
    dg.count_filter = reused;  // a fresh table holds only this batch's keys
    AggParams P;
    memset(&P, 0, sizeof P);
    P.n_rows = n;
    P.pred_kind = !plan.has_pred ? 0 : (plan.simple.enabled ? 1 : 2);
    if (P.pred_kind == 1) { P.sp_slot = plan.simple.slot; P.sp_cmp = plan.simple.cmp; P.sp_is_f64 = plan.simple.is_f64; P.sp_const = plan.simple.constant; }
    if (P.pred_kind == 2) P.pred = plan.pred;
    P.key_kind = ex.key_kind; P.key_slot = ex.key_slot;
    P.key_slot2 = ex.key_slot2; P.key_kind1 = ex.key_kind1; P.key_kind2 = ex.key_kind2;
    for (size_t s = 0; s < plan.used_cols.size(); ++s) P.cols[s] = in.cols[plan.used_cols[s]].view();
    P.n_acc = (int)ex.accs.size();
    for (size_t a = 0; a < ex.accs.size(); ++a) {
      P.accs[a].kind = ex.accs[a].kind; P.accs[a].arg_slot = ex.accs[a].arg_slot; P.accs[a].arg_prog = ex.accs[a].arg_prog;
      P.accs[a].arg_is_f64 = ex.accs[a].arg_is_f64; P.accs[a].acc_index = (int)a;
    }
    for (size_t i = 0; i < ex.progs.size(); ++i) P.progs[i] = ex.progs[i];
    P.table = (uint8_t*)dg.table.get();
    P.bucket_stride = stride;
    P.mask = capacity - 1;
    P.group_count = (unsigned int*)ctl.get();
    P.overflow = (int32_t*)((char*)ctl.get() + 4);
    P.error = (int32_t*)((char*)ctl.get() + 8);
    P.long_seen = (int32_t*)((char*)ctl.get() + 280);
    P.max_groups = (unsigned int)std::min<unsigned long long>(capacity - capacity / 4, 0x7FFFFFFFull);  // retry above load 0.75
    ARK_CUDA(cudaMemsetAsync(ctl.get(), 0, 512, stream));
    // large tables: partition rows by table region, build each region in shared memory (hash_agg_radix.cu)
    std::vector<BufferPtr> radix_keep;
    const bool radix = !reused && allow_radix && n > 0 && ex.key_kind != KEY_PAIR && launch_hash_agg_radix(P, capacity, (int32_t*)((char*)ctl.get() + 12), &radix_keep, stream);
    if (reused) {
      KernelTimer t("agg_reset_acc_kernel", stream);
      const int grid = (int)std::min<unsigned long long>((capacity * P.n_acc + 255) / 256, 148ull * 8);
      agg_reset_acc_kernel<<<grid, 256, 0, stream>>>(P.table, capacity, stride, P.n_acc, P.accs[0], P.accs[1], P.accs[2], P.accs[3], P.accs[4],
                                                     P.accs[5], P.accs[6], P.accs[7]);
    } else if (!radix) {
      KernelTimer t("agg_init_kernel", stream);
      const int grid = (int)std::min<unsigned long long>((capacity + 255) / 256, 148ull * 8);
      agg_init_kernel<<<grid, 256, 0, stream>>>(P.table, capacity, stride, P.n_acc, P.accs[0], P.accs[1], P.accs[2], P.accs[3], P.accs[4],
                                                P.accs[5], P.accs[6], P.accs[7]);
    }
    // (A persisting L2 access-policy window on the table was tried: no gain for this kernel, and the set-aside it
    // needs, cudaLimitPersistingL2CacheSize, stays carved out of the L2 for every later kernel of the process, which
    // slowed a following concat.  Removed.)
    int64_t key_bytes = ex.key_kind == KEY_BYTES ? in.cols[plan.used_cols[ex.key_slot]].data_bytes : 0;
    if (ex.key_kind == KEY_BYTES) {
      // staging of the key bytes is sized from the column's average key length: the batch's own when its extent is
      // known, else what this plan saw last (a wrong guess only sends tiles down the unstaged path)
      if (key_bytes >= 0 && n > 0) hints.avg_key_len.store((double)key_bytes / (double)n);
      else if (hints.avg_key_len.load() >= 0) key_bytes = (int64_t)(hints.avg_key_len.load() * (double)n);
      else {
        resolve_varlen_extents(in, {plan.used_cols[ex.key_slot]}, stream);
        key_bytes = in.cols[plan.used_cols[ex.key_slot]].data_bytes;
        if (n > 0) hints.avg_key_len.store((double)key_bytes / (double)n);
      }
    }
    // low cardinality (table ≤ 1024 slots): per-CTA hash table in shared memory (hash_agg_tile.cu) — hot keys would
    // serialise on L2 atomics here.  Everything larger: this file's row kernel.
    if (radix) {
    } else if (n > 0 && !reused && capacity <= tile_max && ex.key_kind != KEY_PAIR && launch_hash_agg_tile(P, capacity, hints.groups.load(), key_bytes, stream)) {
    } else if (n > 0 && launch_hash_agg_stream(P, capacity, key_bytes, stream)) {
    } else {
      if (P.pred_kind == 0) launch_agg<0>(P, n, stream);
      else if (P.pred_kind == 1) launch_agg<1>(P, n, stream);
      else launch_agg<2>(P, n, stream);
    }
    ARK_CUDA(cudaGetLastError());
    ARK_CUDA(cudaMemcpyAsync(hctl.get(), ctl.get(), 16, cudaMemcpyDeviceToHost, stream));
    ARK_CUDA(cudaMemcpyAsync((char*)hctl.get() + 280, (char*)ctl.get() + 280, 4, cudaMemcpyDeviceToHost, stream));
    ARK_CUDA(cudaStreamSynchronize(stream));
    const unsigned int claimed_now = *(unsigned int*)hctl.get();  // keys claimed by THIS launch
    const unsigned long long keys_total = (reused ? ct.total_keys : 0) + claimed_now;
    const unsigned int groups = (unsigned int)std::min<unsigned long long>(keys_total, 0xFFFFFFFFull);
    const int overflow = *(int32_t*)((char*)hctl.get() + 4);
    const int err = *(int32_t*)((char*)hctl.get() + 8);
    const bool long_seen = *(int32_t*)((char*)hctl.get() + 280) != 0;
    if (reused && (overflow || groups > P.max_groups)) {  // the dictionary filled up with keys of past batches: start over at this size
      fresh_only = true;
      continue;
    }
    if (*(int32_t*)((char*)hctl.get() + 12)) {  // skewed keys overflowed a bucket's record array: same capacity, row kernel
      hash_agg_radix_note_skew();
      allow_radix = false;
      continue;
    }
    if (overflow || groups > P.max_groups) {
      if (capacity >= cap_limit) fail(ARK_ERR_PROCESS, "Collection query results error: group-by hash table exceeded 2^31 slots");
      capacity *= 4;
      hints.groups.store(0);  // the previous batch's group count undersized the shared-memory table: size it by capacity
      continue;
    }
    if (err) fail(ARK_ERR_PROCESS, std::string("Collection query results error: ") + vm_error_text(err));
    dg.n_groups = groups;  // upper bound when the table is reused (compact_groups counts this batch's groups)
    dg.capacity = capacity;
    dg.total_keys = keys_total;
    dg.cacheable = cache_now && !long_seen && keys_total * 10 <= capacity * 6;
    // next batch: the smallest power of two ≥ 2× the groups just seen (load ≤ 0.5), at least 2^12, so that
    // the table of config 3 (10^6 keys in 2^21 32-byte slots) is 64 MB, larger than H100's 50 MB L2 (hash_agg_stream.cu
    // picks its kernel by that)
    if (!reused) {  // a reused dictionary keeps its size (keys_total counts keys of past batches too)
      unsigned long long want = 1ull << 10;
      while (want < 2ull * groups) want <<= 1;
      hints.capacity.store(want);
      hints.groups.store(groups);
    }
    break;
  }
  if (!compact) return dg;
  const ColView kc = ex.key_kind == KEY_NONE ? ColView{} : in.cols[plan.used_cols[ex.key_slot]].view();
  compact_groups(dg, kc, ex.key_kind, n_parts, ctl, hctl, stream);
  return dg;
}

// After the call that used it: a table with self-contained keys goes back to its plan for the next batch.
static void return_table(AggHints& hints, DenseGroups& dg) {
  if (!dg.cacheable || !dg.table) return;
  std::lock_guard<std::mutex> l(hints.cache_mu);
  if (hints.cache.size() >= 4) return;
  AggHints::CachedTable ct;
  ct.table = dg.table; ct.capacity = dg.capacity; ct.total_keys = dg.total_keys; ct.n_acc = dg.n_acc;
  hints.cache.push_back(std::move(ct));
}
static void return_table(const Plan& plan, DenseGroups& dg) { return_table(*plan.hints, dg); }

static void compact_groups(DenseGroups& dg, const ColView& kc, int key_kind, int n_parts, BufferPtr ctl, BufferPtr hctl, cudaStream_t stream) {
  unsigned int* part_counts = (unsigned int*)((char*)ctl.get() + 16);
  unsigned int* part_cursor = (unsigned int*)((char*)ctl.get() + 16 + 128);
  ARK_CUDA(cudaMemsetAsync(part_counts, 0, 256, stream));
  const int need_count = dg.count_filter ? 1 : 0;
  dg.slots = device_alloc((size_t)std::max<unsigned int>(dg.n_groups, 1) * 4);  // n_groups: exact, or an upper bound when the table is reused
  dg.part_rows.assign(n_parts, 0);
  const int sgrid = (int)std::min<unsigned long long>((dg.capacity + 255) / 256, 148ull * 8);
  if (n_parts > 1) {
    {
      KernelTimer t("agg_count_parts_kernel", stream);
      agg_count_parts_kernel<<<sgrid, 256, 0, stream>>>((const uint8_t*)dg.table.get(), dg.stride, dg.capacity, kc, key_kind, n_parts, part_counts, need_count);
    }
    ARK_CUDA(cudaMemcpyAsync((char*)hctl.get() + 16, part_counts, 128, cudaMemcpyDeviceToHost, stream));
    ARK_CUDA(cudaStreamSynchronize(stream));
    unsigned int* hc = (unsigned int*)((char*)hctl.get() + 16);
    unsigned int* hcur = (unsigned int*)((char*)hctl.get() + 16 + 128);
    unsigned int run = 0;
    for (int p = 0; p < n_parts; ++p) { dg.part_rows[p] = hc[p]; hcur[p] = run; run += hc[p]; }
    if (need_count) dg.n_groups = run;
    ARK_CUDA(cudaMemcpyAsync(part_cursor, hcur, 128, cudaMemcpyHostToDevice, stream));
  }
  if (dg.n_groups > 0) {
    KernelTimer t("agg_compact_kernel", stream);
    agg_compact_kernel<<<sgrid, 256, 0, stream>>>((const uint8_t*)dg.table.get(), dg.stride, dg.capacity, kc, key_kind, n_parts, part_cursor,
                                                  (unsigned int*)dg.slots.get(), need_count);
  }
  if (n_parts == 1) {
    if (need_count && dg.n_groups > 0) {  // this batch's group count = where the cursor stopped
      ARK_CUDA(cudaMemcpyAsync((char*)hctl.get() + 16, part_cursor, 4, cudaMemcpyDeviceToHost, stream));
      ARK_CUDA(cudaStreamSynchronize(stream));
      dg.n_groups = *(unsigned int*)((char*)hctl.get() + 16);
    }
    dg.part_rows[0] = dg.n_groups;
  }
  ARK_CUDA(cudaGetLastError());
}

// key column of the dense groups
// kc: the column long keys (> 12 bytes) point into; may_null: emit a validity bitmap
static Column emit_key_column(const AggExec& ex, const DenseGroups& dg, const ColView& kc, bool may_null, const std::string& name,
                              bool nullable, cudaStream_t stream) {
  const unsigned int G = dg.n_groups;
  Column c;
  c.field.name = name; c.field.type = ex.key_type; c.field.nullable = nullable; c.length = G;
  BufferPtr valid_bytes = may_null ? device_alloc(std::max<size_t>(G, 1)) : BufferPtr();
  const unsigned grid = (unsigned)ceil_div(std::max<unsigned int>(G, 1), 256);
  const uint8_t* keys = (const uint8_t*)dg.table.get();
  const int kstride = dg.stride;
  const unsigned int* slots = (const unsigned int*)dg.slots.get();
  if (ex.key_kind == KEY_BYTES) {
    BufferPtr lens = device_alloc((size_t)(G + 1) * 4), offs = device_alloc((size_t)(G + 1) * 4);
    ARK_CUDA(cudaMemsetAsync(lens.get(), 0, (size_t)(G + 1) * 4, stream));
    if (G) {
      KernelTimer t("agg_key_lengths_kernel", stream);
      agg_key_lengths_kernel<<<grid, 256, 0, stream>>>(keys, kstride, slots, G, (int32_t*)lens.get());
    }
    size_t tmp_bytes = 0;
    cub::DeviceScan::ExclusiveSum(nullptr, tmp_bytes, (int32_t*)lens.get(), (int32_t*)offs.get(), (int)(G + 1), stream);
    BufferPtr tmp = device_alloc(tmp_bytes + 16);
    note_launch("cub::DeviceScan::ExclusiveSum");
    cub::DeviceScan::ExclusiveSum(tmp.get(), tmp_bytes, (int32_t*)lens.get(), (int32_t*)offs.get(), (int)(G + 1), stream);
    BufferPtr h = pinned_alloc(64);
    ARK_CUDA(cudaMemcpyAsync(h.get(), (int32_t*)offs.get() + G, 4, cudaMemcpyDeviceToHost, stream));
    ARK_CUDA(cudaStreamSynchronize(stream));
    const int32_t total = *(int32_t*)h.get();
    BufferPtr bytes = device_alloc((size_t)total + 16);
    if (G) {
      KernelTimer t("agg_emit_keys_kernel", stream);
      agg_emit_keys_kernel<<<grid, 256, 0, stream>>>(keys, kstride, slots, G, kc, ex.key_kind, nullptr, nullptr, (const int32_t*)offs.get(),
                                                     (uint8_t*)bytes.get(), (uint8_t*)valid_bytes.get());
    }
    c.offsets = (const int32_t*)offs.get(); c.data = (const uint8_t*)bytes.get(); c.data_bytes = total; c.first_offset = 0;
    c.owners = {offs, bytes};
  } else if (ex.key_kind == KEY_INT64) {
    BufferPtr vals = device_alloc((size_t)std::max<unsigned int>(G, 1) * 8);
    if (G) {
      KernelTimer t("agg_emit_keys_kernel", stream);
      agg_emit_keys_kernel<<<grid, 256, 0, stream>>>(keys, kstride, slots, G, kc, ex.key_kind, (unsigned long long*)vals.get(), nullptr, nullptr,
                                                     nullptr, (uint8_t*)valid_bytes.get());
    }
    c.data = (const uint8_t*)vals.get(); c.data_bytes = (int64_t)G * 8; c.owners = {vals};
  } else {  // KEY_BOOL
    BufferPtr bb = device_alloc(std::max<size_t>(G, 1)), bits = device_alloc((size_t)(G + 7) / 8 + 1);
    if (G) {
      KernelTimer t("agg_emit_keys_kernel", stream);
      agg_emit_keys_kernel<<<grid, 256, 0, stream>>>(keys, kstride, slots, G, kc, ex.key_kind, nullptr, (uint8_t*)bb.get(), nullptr, nullptr,
                                                     (uint8_t*)valid_bytes.get());
    }
    launch_pack_bits((const uint8_t*)bb.get(), G, (uint8_t*)bits.get(), nullptr, stream);
    c.data = (const uint8_t*)bits.get(); c.data_bytes = (G + 7) / 8; c.owners = {bits, bb};
  }
  if (may_null && G) {
    BufferPtr vbits = device_alloc((size_t)(G + 7) / 8 + 1);
    launch_pack_bits((const uint8_t*)valid_bytes.get(), G, (uint8_t*)vbits.get(), nullptr, stream);
    c.validity = (const uint8_t*)vbits.get(); c.null_count = -1;
    c.owners.push_back(vbits); c.owners.push_back(valid_bytes);
  }
  return c;
}

static Column emit_key_column(const AggExec& ex, const DenseGroups& dg, const Column& src, const std::string& name,
                              bool nullable, cudaStream_t stream) {
  return emit_key_column(ex, dg, src.view(), src.validity != nullptr, name, nullable, stream);
}

// pair keys: the row each group was first seen at (Key16.lo) → gather index for take_column
__global__ void agg_key_rows_kernel(const uint8_t* table, int stride, const unsigned int* slots, unsigned int n_groups, unsigned int* rows) {
  unsigned int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g < n_groups) rows[g] = (unsigned int)tbl_key(table, slots[g], stride)->lo;
}
static BufferPtr pair_key_rows(const DenseGroups& dg, cudaStream_t stream) {
  const unsigned int G = dg.n_groups;
  BufferPtr rows = device_alloc((size_t)std::max<unsigned int>(G, 1) * 4);
  if (G) {
    KernelTimer t("agg_key_rows_kernel", stream);
    agg_key_rows_kernel<<<(unsigned)ceil_div(G, 256), 256, 0, stream>>>((const uint8_t*)dg.table.get(), dg.stride, (const unsigned int*)dg.slots.get(), G,
                                                                        (unsigned int*)rows.get());
  }
  return rows;
}

static BufferPtr gather_acc(const DenseGroups& dg, int acc, cudaStream_t stream) {
  const unsigned int G = dg.n_groups;
  BufferPtr out = device_alloc((size_t)std::max<unsigned int>(G, 1) * 8);
  if (G) {
    KernelTimer t("agg_gather_acc_kernel", stream);
    agg_gather_acc_kernel<<<(unsigned)ceil_div(G, 256), 256, 0, stream>>>((const uint8_t*)dg.table.get(), dg.stride, acc,
                                                                         (const unsigned int*)dg.slots.get(), G, (unsigned long long*)out.get());
  }
  return out;
}

static Column finalize_column(const std::string& name, DType type, int op, BufferPtr a, BufferPtr cnt, uint64_t constant, bool nullable,
                              unsigned int G, cudaStream_t stream) {
  Column c;
  c.field.name = name; c.field.type = type; c.field.nullable = nullable; c.length = G;
  BufferPtr out = device_alloc((size_t)std::max<unsigned int>(G, 1) * 8);
  BufferPtr vb = (cnt && nullable) ? device_alloc(std::max<size_t>(G, 1)) : BufferPtr();
  if (G) {
    KernelTimer t("agg_finalize_kernel", stream);
    agg_finalize_kernel<<<(unsigned)ceil_div(G, 256), 256, 0, stream>>>(op, (const unsigned long long*)a.get(), (const unsigned long long*)cnt.get(),
                                                                       constant, G, (unsigned long long*)out.get(), (uint8_t*)vb.get());
  }
  c.data = (const uint8_t*)out.get(); c.data_bytes = (int64_t)G * 8; c.owners = {out};
  if (vb && G) {
    BufferPtr bits = device_alloc((size_t)(G + 7) / 8 + 1);
    launch_pack_bits((const uint8_t*)vb.get(), G, (uint8_t*)bits.get(), nullptr, stream);
    c.validity = (const uint8_t*)bits.get(); c.null_count = -1;
    c.owners.push_back(bits); c.owners.push_back(vb);
  }
  return c;
}

// Builds the physical aggregate of a bound plan.  merge == false: over raw rows.  merge == true:
// over partial-state rows (column layout produced by partial_state_batch below).
static void build_exec(const Plan& plan, const Batch* in, AggExec& ex, std::vector<AggOutput>& outs) {
  const bool schema_nullability = in == nullptr;
  if (plan.keys.size() > 2) fail(ARK_ERR_UNSUPPORTED, "more than two GROUP BY keys");
  auto kind_of = [](DType t) { return t == DType::Int64 ? KEY_INT64 : (t == DType::Bool ? KEY_BOOL : KEY_BYTES); };
  if (!plan.keys.empty()) {
    const ValueSource& k = plan.keys[0];
    ex.key_slot = k.slot; ex.key_type = k.type;
    ex.key_kind = kind_of(k.type);
    if (plan.keys.size() == 2) {
      ex.key_kind1 = ex.key_kind; ex.key_kind = KEY_PAIR;
      ex.key_slot2 = plan.keys[1].slot; ex.key_type2 = plan.keys[1].type; ex.key_kind2 = kind_of(plan.keys[1].type);
    }
  }
  auto arg_of = [&](const ValueSource& v, AccPlan& a, bool* nullable) {
    if (v.kind == ValueSource::PassThrough) {
      a.arg_slot = v.slot;
      // multi-GPU: every rank must build the same accumulator layout ⇒ decide from the schema, not the buffers
      *nullable = schema_nullability ? plan.input_fields[plan.used_cols[v.slot]].nullable : in->cols[plan.used_cols[v.slot]].validity != nullptr;
    } else {
      if ((int)ex.progs.size() >= AGG_MAX_PROGS) fail(ARK_ERR_UNSUPPORTED, "too many computed aggregate arguments");
      a.arg_prog = (int)ex.progs.size(); ex.progs.push_back(v.prog);
      *nullable = v.nullable;
    }
    a.arg_is_f64 = v.type == DType::Float64;
  };
  const int star = ex.find_or_add(AccPlan{ACC_COUNT_STAR});
  for (const AggSpec& s : plan.aggs) {
    AggOutput o;
    o.type = s.out_type;
    if (s.func == AggFunc::CountStar) { o.value_acc = star; outs.push_back(o); continue; }
    AccPlan a; bool nullable = false;
    arg_of(s.arg, a, &nullable);
    int nn = star;
    if (nullable) { AccPlan c = a; c.kind = ACC_COUNT; c.arg_is_f64 = false; nn = ex.find_or_add(c); o.can_be_null = true; }
    switch (s.func) {
      case AggFunc::Count: o.value_acc = nn; break;
      case AggFunc::Sum: a.kind = a.arg_is_f64 ? ACC_SUM_F64 : ACC_SUM_I64; o.value_acc = ex.find_or_add(a); o.count_acc = nn; break;
      case AggFunc::Avg: {
        const bool was_f64 = a.arg_is_f64;
        a.kind = ACC_SUM_F64; a.arg_is_f64 = was_f64;
        o.value_acc = ex.find_or_add(a); o.count_acc = nn; o.final_op = FIN_AVG; break;
      }
      case AggFunc::Min: a.kind = a.arg_is_f64 ? ACC_MIN_F64 : ACC_MIN_I64; o.value_acc = ex.find_or_add(a); o.count_acc = nn;
        o.final_op = a.arg_is_f64 ? FIN_F64_KEY_BACK : FIN_COPY; break;
      case AggFunc::Max: a.kind = a.arg_is_f64 ? ACC_MAX_F64 : ACC_MAX_I64; o.value_acc = ex.find_or_add(a); o.count_acc = nn;
        o.final_op = a.arg_is_f64 ? FIN_F64_KEY_BACK : FIN_COPY; break;
      default: break;
    }
    outs.push_back(o);
  }
}

static Batch project_groups(const Plan& plan, const AggExec& ex, const std::vector<AggOutput>& outs, const DenseGroups& dg,
                            const Column* key_src, cudaStream_t stream, const Column* key_src2 = nullptr) {
  const unsigned int G = dg.n_groups;
  Batch out;
  out.num_rows = G;
  std::vector<BufferPtr> dense(ex.accs.size());
  auto dense_acc = [&](int a) -> BufferPtr { if (!dense[a]) dense[a] = gather_acc(dg, a, stream); return dense[a]; };
  BufferPtr pair_rows;  // KEY_PAIR: keys are gathered from the rows that first held each pair
  for (const PostItem& pi : plan.post) {
    if (pi.kind == PostItem::Key && ex.key_kind == KEY_PAIR) {
      if (!pair_rows) pair_rows = pair_key_rows(dg, stream);
      const Column& src = pi.index == 0 ? *key_src : *key_src2;
      out.cols.push_back(take_column(src, (const unsigned int*)pair_rows.get(), G, pi.name, stream));
    } else if (pi.kind == PostItem::Key) {
      out.cols.push_back(emit_key_column(ex, dg, *key_src, pi.name, key_src->field.nullable, stream));
    } else if (pi.kind == PostItem::Agg) {
      const AggOutput& o = outs[pi.index];
      const AggSpec& s = plan.aggs[pi.index];
      const bool is_count = s.func == AggFunc::Count || s.func == AggFunc::CountStar;
      BufferPtr cnt = o.count_acc >= 0 ? dense_acc(o.count_acc) : BufferPtr();
      // a group exists only if it has ≥ 1 row, so COUNT(*) > 0: validity is needed only when the
      // argument itself can be NULL (dedicated ACC_COUNT accumulator)
      // … or when there is no key: the single group of a global aggregate may be empty (SUM → NULL)
      const bool can_be_null = !is_count && o.count_acc >= 0 && (o.can_be_null || ex.key_kind == KEY_NONE);
      Column col = finalize_column(pi.name, o.type, o.final_op, dense_acc(o.value_acc), cnt, 0, can_be_null, G, stream);
      col.field.nullable = !is_count;
      if (pi.cast_utf8) col = format_int64_column(col, pi.name, stream);  // CAST(<Int64 aggregate> AS STRING)
      out.cols.push_back(col);
    } else {
      if (pi.lit_type == DType::Utf8) fail(ARK_ERR_UNSUPPORTED, "string literal in an aggregate SELECT list");
      if (pi.lit_type == DType::Bool) fail(ARK_ERR_UNSUPPORTED, "boolean literal in an aggregate SELECT list");
      out.cols.push_back(finalize_column(pi.name, pi.lit_type, FIN_CONST, BufferPtr(), BufferPtr(), pi.lit_bits, false, G, stream));
    }
  }
  return out;
}

Batch run_aggregate(const Plan& plan, Batch& in, cudaStream_t stream) {
  AggExec ex;
  std::vector<AggOutput> outs;
  build_exec(plan, &in, ex, outs);
  DenseGroups dg = hash_pass(plan, ex, in, 1, stream);
  const Column* key_src = ex.key_kind == KEY_NONE ? nullptr : &in.cols[plan.used_cols[ex.key_slot]];
  const Column* key_src2 = ex.key_kind == KEY_PAIR ? &in.cols[plan.used_cols[ex.key_slot2]] : nullptr;
  Batch out = project_groups(plan, ex, outs, dg, key_src, stream, key_src2);
  ARK_CUDA(cudaStreamSynchronize(stream));
  return_table(plan, dg);
  return out;
}

// ---- multi-GPU building blocks (SURVEY.md §8(e)): partial states out, hash-partitioned; merge in ----
// Partial-state batch layout: [key column (if any)] + one 8-byte column per accumulator, in the
// accumulator order build_exec() derives from the plan alone (identical on every rank).
Batch run_partial_aggregate(const Plan& plan, Batch& in, int n_parts, std::vector<int64_t>& part_rows, cudaStream_t stream) {
  AggExec ex;
  std::vector<AggOutput> outs;
  build_exec(plan, nullptr, ex, outs);
  DenseGroups dg = hash_pass(plan, ex, in, n_parts, stream);
  part_rows = dg.part_rows;
  Batch out;
  out.num_rows = dg.n_groups;
  if (ex.key_kind == KEY_PAIR) {
    BufferPtr rows = pair_key_rows(dg, stream);
    out.cols.push_back(take_column(in.cols[plan.used_cols[ex.key_slot]], (const unsigned int*)rows.get(), dg.n_groups, plan.key_names[0], stream));
    out.cols.push_back(take_column(in.cols[plan.used_cols[ex.key_slot2]], (const unsigned int*)rows.get(), dg.n_groups, plan.key_names[1], stream));
  } else if (ex.key_kind != KEY_NONE) {
    const Column& src = in.cols[plan.used_cols[ex.key_slot]];
    out.cols.push_back(emit_key_column(ex, dg, src, plan.key_names[0], src.field.nullable, stream));
  }
  for (size_t a = 0; a < ex.accs.size(); ++a) {
    Column c;
    c.field.name = "__acc" + std::to_string(a);
    c.field.type = ex.accs[a].kind == ACC_SUM_F64 ? DType::Float64 : DType::Int64;
    c.field.nullable = false; c.length = dg.n_groups;
    BufferPtr d = gather_acc(dg, (int)a, stream);
    c.data = (const uint8_t*)d.get(); c.data_bytes = (int64_t)dg.n_groups * 8; c.owners = {d};
    out.cols.push_back(c);
  }
  ARK_CUDA(cudaStreamSynchronize(stream));
  return_table(plan, dg);
  return out;
}

Batch run_final_aggregate(const Plan& plan, Batch& partial, cudaStream_t stream) {
  AggExec ex;
  std::vector<AggOutput> outs;
  build_exec(plan, nullptr, ex, outs);  // same accumulator layout as the partial side
  const int key_cols = ex.key_kind == KEY_NONE ? 0 : (ex.key_kind == KEY_PAIR ? 2 : 1);
  if ((int)partial.cols.size() != key_cols + (int)ex.accs.size())
    fail(ARK_ERR_PROCESS, "final aggregate: partial-state batch has " + std::to_string(partial.cols.size()) + " columns, expected " +
                              std::to_string(key_cols + ex.accs.size()));
  AggExec mx;  // merge: aggregate the state columns
  mx.key_kind = ex.key_kind; mx.key_slot = 0; mx.key_type = ex.key_type;
  mx.key_kind1 = ex.key_kind1; mx.key_kind2 = ex.key_kind2; mx.key_slot2 = 1; mx.key_type2 = ex.key_type2;
  for (size_t a = 0; a < ex.accs.size(); ++a) {
    AccPlan m;
    m.arg_slot = key_cols + (int)a;
    switch (ex.accs[a].kind) {
      case ACC_COUNT_STAR: case ACC_COUNT: case ACC_SUM_I64: m.kind = ACC_SUM_I64; break;
      case ACC_SUM_F64: m.kind = ACC_SUM_F64; m.arg_is_f64 = true; break;
      case ACC_MIN_I64: case ACC_MIN_F64: m.kind = ACC_MIN_I64; break;   // F64 states travel as totalOrder keys
      default: m.kind = ACC_MAX_I64; break;
    }
    mx.accs.push_back(m);  // no dedup: positions must line up with `outs`
  }
  Plan mp;
  mp.kind = Plan::Aggregate;
  mp.hints = plan.final_hints;  // the merge table's size carries over from batch to batch like the partial side's
  for (size_t i = 0; i < partial.cols.size(); ++i) mp.used_cols.push_back((int)i);
  if ((int)mp.used_cols.size() > MAX_COLS) fail(ARK_ERR_UNSUPPORTED, "too many accumulator columns");
  DenseGroups dg = hash_pass(mp, mx, partial, 1, stream, true, /*merge_mode=*/true);
  Batch out = project_groups(plan, mx, outs, dg, key_cols ? &partial.cols[0] : nullptr, stream, key_cols == 2 ? &partial.cols[1] : nullptr);
  ARK_CUDA(cudaStreamSynchronize(stream));
  return_table(mp, dg);  // mp.hints is the plan's final_hints
  return out;
}

// ---- device-side exchange (group_exchange.cu): partial table → push over NVLink → merge → result --------------
// Push phase: build this rank's partial table and push its slots into the owners' receive regions.
void run_group_by_push(const Plan& plan, Batch& in, DistCtx& d, cudaStream_t stream) {
  AggExec ex;
  std::vector<AggOutput> outs;
  build_exec(plan, nullptr, ex, outs);  // accumulator layout from the schema alone: identical on every rank
  DenseGroups dg = hash_pass(plan, ex, in, 1, stream, /*compact=*/false);
  launch_exchange_push((const uint8_t*)dg.table.get(), dg.capacity, (int)ex.accs.size(), ex.key_kind, d.peers, d.world, d.rank, d.step, d.region_bytes,
                       dg.count_filter ? 1 : 0, stream);
  ARK_CUDA(cudaGetLastError());
  ARK_CUDA(cudaStreamSynchronize(stream));
  return_table(plan, dg);
}

// Merge phase: wait for every source's records, merge them into the final table, acknowledge, project the result.
// Returns false (on every rank alike) when some source held keys that cannot travel inline; the step is still
// acknowledged, so the caller can fall back to the descriptor exchange for this batch.
bool run_group_by_merge(const Plan& plan, DistCtx& d, Batch& out, cudaStream_t stream) {
  AggExec ex;
  std::vector<AggOutput> outs;
  build_exec(plan, nullptr, ex, outs);
  AggExec mx;  // same accumulators, merged instead of fed (sum of sums and counts, min of mins, …)
  mx.key_kind = ex.key_kind; mx.key_slot = 0; mx.key_type = ex.key_type;
  int32_t kinds[AGG_MAX_ACC] = {0};
  for (size_t a = 0; a < ex.accs.size(); ++a) {
    AccPlan m;
    switch (ex.accs[a].kind) {
      case ACC_COUNT_STAR: case ACC_COUNT: case ACC_SUM_I64: m.kind = ACC_SUM_I64; break;
      case ACC_SUM_F64: m.kind = ACC_SUM_F64; m.arg_is_f64 = true; break;
      case ACC_MIN_I64: case ACC_MIN_F64: m.kind = ACC_MIN_I64; break;
      default: m.kind = ACC_MAX_I64; break;
    }
    mx.accs.push_back(m);
    kinds[a] = m.kind;
  }
  AggHints& hints = *plan.final_hints;
  unsigned long long capacity = std::max<unsigned long long>(hints.capacity.load(), 1ull << 10);
  DenseGroups dg;
  dg.stride = table_bucket_stride((int)ex.accs.size());
  dg.n_acc = (int)ex.accs.size();
  BufferPtr ctl = device_alloc(512), hctl = pinned_alloc(512);
  bool poisoned = false, fresh_only = false;
  static const bool cache_env = [] { const char* e = getenv("ARK_AGG_TABLE_CACHE"); return !e || atoi(e) != 0; }();
  const bool cache_enabled = cache_env && mx.key_kind != KEY_NONE;  // a global aggregate's single group exists even with COUNT(*) = 0
  while (true) {
    // the owner meets the same keys step after step: keep the merge table's keys, reset its accumulators (AggHints::CachedTable)
    AggHints::CachedTable ct;
    bool reused = false;
    if (cache_enabled && !fresh_only) {
      std::lock_guard<std::mutex> l(hints.cache_mu);
      for (size_t i = 0; i < hints.cache.size(); ++i)
        if (hints.cache[i].capacity == capacity && hints.cache[i].n_acc == dg.n_acc) { ct = hints.cache[i]; hints.cache.erase(hints.cache.begin() + i); reused = true; break; }
      if (!reused) hints.cache.clear();
    }
    dg.table = reused ? ct.table : device_alloc((size_t)table_bytes(capacity, (int)ex.accs.size()));
    ARK_CUDA(cudaMemsetAsync(ctl.get(), 0, 512, stream));
    {
      AccParam ap[AGG_MAX_ACC];
      memset(ap, 0, sizeof ap);
      for (size_t a = 0; a < mx.accs.size(); ++a) { ap[a].kind = mx.accs[a].kind; ap[a].acc_index = (int)a; }
      KernelTimer t(reused ? "agg_reset_acc_kernel" : "agg_init_kernel", stream);
      if (reused) {
        const int grid = (int)std::min<unsigned long long>((capacity * mx.accs.size() + 255) / 256, 148ull * 8);
        agg_reset_acc_kernel<<<grid, 256, 0, stream>>>((uint8_t*)dg.table.get(), capacity, dg.stride, (int)mx.accs.size(), ap[0], ap[1], ap[2], ap[3], ap[4],
                                                       ap[5], ap[6], ap[7]);
      } else {
        const int grid = (int)std::min<unsigned long long>((capacity + 255) / 256, 148ull * 8);
        agg_init_kernel<<<grid, 256, 0, stream>>>((uint8_t*)dg.table.get(), capacity, dg.stride, (int)mx.accs.size(), ap[0], ap[1], ap[2], ap[3], ap[4],
                                                  ap[5], ap[6], ap[7]);
      }
    }
    // ctl: [group_count u32 | overflow i32 | status i32 | pad | total u64 @ 272]
    launch_exchange_merge((uint8_t*)dg.table.get(), capacity, (int)mx.accs.size(), kinds, d.comm, d.world, d.rank, d.step, d.region_bytes,
                          (unsigned int*)ctl.get(), (int32_t*)((char*)ctl.get() + 4), (int32_t*)((char*)ctl.get() + 8),
                          (unsigned long long*)((char*)ctl.get() + 272), stream);
    ARK_CUDA(cudaGetLastError());
    ARK_CUDA(cudaMemcpyAsync(hctl.get(), ctl.get(), 16, cudaMemcpyDeviceToHost, stream));
    ARK_CUDA(cudaMemcpyAsync((char*)hctl.get() + 16, (char*)ctl.get() + 272, 8, cudaMemcpyDeviceToHost, stream));
    ARK_CUDA(cudaStreamSynchronize(stream));
    const unsigned int claimed_now = *(unsigned int*)hctl.get();
    const unsigned long long keys_total = (reused ? ct.total_keys : 0) + claimed_now;
    const int overflow = *(int32_t*)((char*)hctl.get() + 4);
    const int status = *(int32_t*)((char*)hctl.get() + 8);
    const unsigned long long total = *(unsigned long long*)((char*)hctl.get() + 16);
    if (status & 2) {
      launch_exchange_ack(d.peers, d.world, d.rank, d.step, stream);
      ARK_CUDA(cudaStreamSynchronize(stream));
      fail(ARK_ERR_PROCESS, "Collection query results error: a rank's partial states exceed the exchange region (ark_dist_create region_bytes)");
    }
    if (status & 1) { poisoned = true; break; }
    const unsigned long long max_groups = capacity - capacity / 4;
    if (overflow || keys_total > max_groups) {  // the records stay in the receive region until the ack: merge again
      if (reused) { fresh_only = true; continue; }  // the dictionary filled up with keys of past steps: same size, fresh table
      if (capacity >= (1ull << 31)) fail(ARK_ERR_PROCESS, "Collection query results error: group-by hash table exceeded 2^31 slots");
      capacity = std::max(capacity * 4, (unsigned long long)1 << 10);
      while (capacity < 2 * total) capacity <<= 1;
      continue;
    }
    dg.n_groups = (unsigned int)keys_total;  // exact for a fresh table, an upper bound for a reused one (compact_groups counts)
    dg.capacity = capacity;
    dg.count_filter = reused;
    dg.total_keys = keys_total;
    dg.cacheable = cache_enabled && keys_total * 10 <= capacity * 6;
    d.last_recv_records = total; d.last_groups = keys_total;
    if (!reused) {
      unsigned long long want = 1ull << 10;
      while (want < 2ull * keys_total) want <<= 1;
      hints.capacity.store(want);
      hints.groups.store((unsigned int)keys_total);
    }
    break;
  }
  launch_exchange_ack(d.peers, d.world, d.rank, d.step, stream);
  ARK_CUDA(cudaGetLastError());
  if (poisoned) { ARK_CUDA(cudaStreamSynchronize(stream)); return false; }
  compact_groups(dg, ColView{}, mx.key_kind, 1, ctl, hctl, stream);
  // project: key column straight from the inline keys, aggregates from the merged accumulators
  const unsigned int G = dg.n_groups;
  out = Batch();
  out.num_rows = G;
  std::vector<BufferPtr> dense(mx.accs.size());
  auto dense_acc = [&](int a) -> BufferPtr { if (!dense[a]) dense[a] = gather_acc(dg, a, stream); return dense[a]; };
  for (const PostItem& pi : plan.post) {
    if (pi.kind == PostItem::Key) {
      const Field& kf = plan.input_fields[plan.used_cols[plan.keys[0].slot]];
      out.cols.push_back(emit_key_column(mx, dg, ColView{}, kf.nullable, pi.name, kf.nullable, stream));
    } else if (pi.kind == PostItem::Agg) {
      const AggOutput& o = outs[pi.index];
      const AggSpec& sp = plan.aggs[pi.index];
      const bool is_count = sp.func == AggFunc::Count || sp.func == AggFunc::CountStar;
      BufferPtr cnt = o.count_acc >= 0 ? dense_acc(o.count_acc) : BufferPtr();
      const bool can_be_null = !is_count && o.count_acc >= 0 && (o.can_be_null || mx.key_kind == KEY_NONE);
      Column col = finalize_column(pi.name, o.type, o.final_op, dense_acc(o.value_acc), cnt, 0, can_be_null, G, stream);
      col.field.nullable = !is_count;
      if (pi.cast_utf8) col = format_int64_column(col, pi.name, stream);
      out.cols.push_back(col);
    } else {
      if (pi.lit_type == DType::Utf8) fail(ARK_ERR_UNSUPPORTED, "string literal in an aggregate SELECT list");
      if (pi.lit_type == DType::Bool) fail(ARK_ERR_UNSUPPORTED, "boolean literal in an aggregate SELECT list");
      out.cols.push_back(finalize_column(pi.name, pi.lit_type, FIN_CONST, BufferPtr(), BufferPtr(), pi.lit_bits, false, G, stream));
    }
  }
  ARK_CUDA(cudaStreamSynchronize(stream));
  d.last_groups = G;
  return_table(hints, dg);
  return true;
}

}  // namespace ark
