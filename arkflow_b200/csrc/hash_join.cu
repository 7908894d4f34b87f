// hash_join.cu — equi-join (inner, LEFT / RIGHT outer: build + probe + gather) and hash repartition, device-resident.
//
// Stands in for DataFusion's HashJoinExec and RepartitionExec(Hash) reached from
// JoinOperation::join_operation (crates/arkflow-plugin/src/buffer/join.rs:111-118).
//   build : every non-NULL key of the smaller side claims a table slot with one 128-bit CAS; rows
//           with equal keys are chained through next[] (head exchange), so duplicates are handled;
//   probe : two passes over the probe side — count matches per row, exclusive scan, fill
//           (probe_row, build_row) pairs — then one gather per output column.
// NULL keys never match.  `SELECT *` = left columns then right columns (SQL order), whichever side
// was used to build.  Output row order is unspecified (as in DataFusion).
// LEFT / RIGHT [OUTER] JOIN (the shipped temporary_list example, examples/redis_temporary_example.yaml:29, is a
// RIGHT JOIN): the preserved side is the probe side; a probe row without a match yields one output row whose
// build-side index is NO_ROW, which the gathers turn into NULLs (validity bitmaps on every build-side column).
#include <cub/device/device_scan.cuh>

#include "agg_acc.cuh"
#include "bitmap.cuh"
#include "bitmap.h"
#include "engine.h"
#include "hashkey.cuh"
#include "stage_store.cuh"
#include "varlen.h"

namespace ark {

namespace {

constexpr unsigned int NO_ROW = 0xFFFFFFFFu;

// table hash of the join: 32 bits are plenty for ≤ 2^31 slots and cost a quarter of hash_key16
__device__ __forceinline__ unsigned long long join_key(int key_kind, const ColView& c, int64_t row, Key16* key) {
  int llen = 0;
  const uint8_t* lp = make_key_raw(key_kind, c, row, key, &llen);
  if (lp) return hash_bytes(lp, llen);
  const unsigned h = hash32_key16(*key);
  return ((unsigned long long)h << 32) | (h * 0x9E3779B1u);  // spread over 64 bits: masks wider than 32 bits stay usable
}

__global__ void join_init_kernel(Key16* keys, unsigned int* head, unsigned long long capacity) {
  for (unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; i < capacity;
       i += (unsigned long long)gridDim.x * blockDim.x) {
    keys[i] = Key16{KEY_EMPTY, KEY_EMPTY};
    head[i] = NO_ROW;
  }
}

__global__ void join_build_kernel(ColView kc, int key_kind, int64_t n, Key16* keys, unsigned int* head, unsigned int* next,
                                  unsigned long long mask) {
  for (int64_t row = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; row < n; row += (int64_t)gridDim.x * blockDim.x) {
    if (!col_valid(kc, row)) { next[row] = NO_ROW; continue; }  // NULL keys never match
    Key16 mine;
    const unsigned long long h = join_key(key_kind, kc, row, &mine);
    unsigned long long slot = h & mask;
    while (true) {
      Key16 cur = ld128(keys + slot);
      if (cur.hi == KEY_EMPTY) {
        cur = cas128(keys + slot, Key16{KEY_EMPTY, KEY_EMPTY}, mine);
        if (cur.hi == KEY_EMPTY && cur.lo == KEY_EMPTY) break;
      }
      if (key_equal(mine, cur, kc, kc)) break;
      slot = (slot + 1) & mask;
    }
    next[row] = atomicExch(head + slot, (unsigned int)row);
  }
}

// Probe pass: counts[row] = number of matches, match_slot[row] = table slot of the probe key (NO_ROW if none).
__global__ void join_probe_count_kernel(ColView pc, ColView bc, int key_kind, int64_t n, const Key16* keys, const unsigned int* head,
                                        const unsigned int* next, unsigned long long mask, long long* counts, unsigned int* match_slot, int outer) {
  for (int64_t row = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; row < n; row += (int64_t)gridDim.x * blockDim.x) {
    long long c = 0;
    unsigned int found = NO_ROW;
    if (col_valid(pc, row)) {
      Key16 mine;
      const unsigned long long h = join_key(key_kind, pc, row, &mine);
      unsigned long long slot = h & mask;
      while (true) {
        const Key16 cur = keys[slot];  // the table is read-only during the probe
        if (cur.hi == KEY_EMPTY) break;
        if (key_equal(mine, cur, pc, bc)) {
          found = (unsigned int)slot;
          for (unsigned int b = head[slot]; b != NO_ROW; b = next[b]) ++c;
          break;
        }
        slot = (slot + 1) & mask;
      }
    }
    counts[row] = (outer && c == 0) ? 1 : c;  // outer join: an unmatched probe row survives once, with NULLs
    match_slot[row] = found;
  }
}

// Fill pass: the (probe row, build row) pairs at offsets[row]; the slot comes from the count pass (no second
// hash + probe: 4 sequential bytes per row instead of a random table access).
__global__ void join_probe_fill_kernel(int64_t n, const unsigned int* head, const unsigned int* next, const unsigned int* match_slot,
                                       const long long* offsets, unsigned int* out_probe, unsigned int* out_build, int outer) {
  for (int64_t row = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; row < n; row += (int64_t)gridDim.x * blockDim.x) {
    const unsigned int slot = match_slot[row];
    long long o = offsets[row];
    if (slot == NO_ROW) {
      if (outer) { out_probe[o] = (unsigned int)row; out_build[o] = NO_ROW; }
      continue;
    }
    for (unsigned int b = head[slot]; b != NO_ROW; b = next[b]) { out_probe[o] = (unsigned int)row; out_build[o] = b; ++o; }
  }
}

// ---- gathers -----------------------------------------------------------------------------------------
__global__ void take_fixed8_kernel(const unsigned long long* src, const unsigned int* idx, long long n, unsigned long long* out) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) { const unsigned int r = idx[i]; out[i] = r == NO_ROW ? 0ull : src[r]; }
}
__global__ void take_bits_kernel(const uint8_t* bits, int bit0, const unsigned int* idx, long long n, uint8_t* out_bytes) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) {
    const unsigned int r = idx[i];
    const long long p = (long long)r + bit0;
    out_bytes[i] = r == NO_ROW ? 0 : bit_get(bits, p);  // NO_ROW (outer join, no match): NULL / false
  }
}
// validity of a gathered column that had none: only the NO_ROW rows are NULL
__global__ void take_matched_kernel(const unsigned int* idx, long long n, uint8_t* out_bytes) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out_bytes[i] = idx[i] != NO_ROW;
}
// The output offsets come from an int32 scan, which wraps silently once the bytes pass 2 GiB (and may wrap past 2^32
// back to a positive total).  The kernels that write the lengths therefore also add them up in 64 bits: one atomicAdd
// per warp into *total, which the host checks before it sizes the output.
__global__ void take_lengths_kernel(const int32_t* offsets, const unsigned int* idx, long long n, int32_t* lens, unsigned long long* total) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  int32_t l = 0;
  if (i < n) { const unsigned int r = idx[i]; l = r == NO_ROW ? 0 : offsets[r + 1] - offsets[r]; lens[i] = l; }
  const long long s = warp_sum_ll(l);
  if ((threadIdx.x & 31) == 0 && s) atomicAdd(total, (unsigned long long)s);
}
// All plain gathers of one output batch in ONE launch: every output row reads its (up to two) source row indices once,
// then copies the 8-byte value of every fixed-width column and records the length of every string column.  One launch per
// column read the index array again for each of them (a join of two schema-S tables has four fixed-width + two string
// columns).
constexpr int TAKE_MAX_FIXED = 8, TAKE_MAX_STR = 4;
struct TakeMultiParams {
  const unsigned int* idx[2];
  int32_t n_fixed, n_str;
  const unsigned long long* fsrc[TAKE_MAX_FIXED];
  unsigned long long* fdst[TAKE_MAX_FIXED];
  uint8_t fside[TAKE_MAX_FIXED];
  const int32_t* soff[TAKE_MAX_STR];
  int32_t* slen[TAKE_MAX_STR];
  unsigned long long* stotal;  // n_str words: each string column's 64-bit byte total (zeroed by the host)
  uint8_t sside[TAKE_MAX_STR];
};
// 5 CTAs per SM (48 registers, no spills): without the bound ptxas spends 74 registers on the string totals, 3 CTAs per SM
__global__ void __launch_bounds__(256, 5) take_multi_kernel(const __grid_constant__ TakeMultiParams P, long long n) {
  // a thread's bytes per column, saturated at 2^31 (no wrap in 32 bits): exact while the column's total fits int32, and
  // above 2^31 - 1 whenever the total does not
  unsigned tot[TAKE_MAX_STR] = {0, 0, 0, 0};
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    unsigned int r[2];
    r[0] = P.idx[0] ? P.idx[0][i] : NO_ROW;
    r[1] = P.idx[1] ? P.idx[1][i] : NO_ROW;
    unsigned long long v[TAKE_MAX_FIXED];
    int32_t l[TAKE_MAX_STR];
#pragma unroll
    for (int c = 0; c < TAKE_MAX_FIXED; ++c)
      if (c < P.n_fixed) { const unsigned int rr = r[P.fside[c]]; v[c] = rr == NO_ROW ? 0ull : P.fsrc[c][rr]; }
#pragma unroll
    for (int c = 0; c < TAKE_MAX_STR; ++c)
      if (c < P.n_str) { const unsigned int rr = r[P.sside[c]]; l[c] = rr == NO_ROW ? 0 : P.soff[c][rr + 1] - P.soff[c][rr]; }
#pragma unroll
    for (int c = 0; c < TAKE_MAX_FIXED; ++c) if (c < P.n_fixed) P.fdst[c][i] = v[c];
#pragma unroll
    for (int c = 0; c < TAKE_MAX_STR; ++c) if (c < P.n_str) { P.slen[c][i] = l[c]; tot[c] = min(tot[c] + (unsigned)l[c], 0x80000000u); }
  }
#pragma unroll
  for (int c = 0; c < TAKE_MAX_STR; ++c)
    if (c < P.n_str) {  // n_str is uniform: every lane of the warp takes part in the reduction
      const long long s = warp_sum_ll((long long)tot[c]);
      if ((threadIdx.x & 31) == 0 && s) atomicAdd(P.stotal + c, (unsigned long long)s);
    }
}
// global → shared copy of one string, word-granular on the (shared) destination: aligned source words are
// funnel-shifted into place, so a 12-byte key costs 3–4 loads and 3 stores instead of 12 + 12.
__device__ __forceinline__ void gather_string(uint8_t* dst, const uint8_t* src, int len) {
  const unsigned d0 = (unsigned)__cvta_generic_to_shared(dst);
  int i = 0;
  for (; i < len && ((d0 + i) & 3); ++i) dst[i] = src[i];  // head: up to 3 bytes
  const int words = (len - i) >> 2;
  if (words > 0) {
    const uintptr_t sa = reinterpret_cast<uintptr_t>(src + i);
    const unsigned sh = (unsigned)(sa & 3) * 8;
    const unsigned* sw = reinterpret_cast<const unsigned*>(sa & ~(uintptr_t)3);  // aligned word holding src[i]
    unsigned* d = reinterpret_cast<unsigned*>(dst + i);
    if (sh == 0) {
      for (int w = 0; w < words; ++w) d[w] = sw[w];
    } else {
      unsigned lo = sw[0];
      for (int w = 0; w < words; ++w) {  // sw[w + 1] holds source byte i + 4w + 3 < len: never past the string's last word
        const unsigned hi = sw[w + 1];
        d[w] = __funnelshift_r(lo, hi, sh);
        lo = hi;
      }
    }
    i += words * 4;
  }
  for (; i < len; ++i) dst[i] = src[i];  // tail
}

constexpr int TAKE_TILE = 1024;

// Gathers the bytes of TAKE_TILE output rows into shared memory (their output range is contiguous), then
// writes the range with destination-aligned 16-byte stores.  Replaces the warp-per-row kernel on the join's
// gather of string columns.
__global__ void __launch_bounds__(256) take_bytes_tile_kernel(const uint8_t* data, const int32_t* offsets, const unsigned int* idx, long long n,
                                                               const int32_t* out_offsets, uint8_t* out, int stage_bytes) {
  extern __shared__ __align__(16) uint8_t stage[];  // stage_bytes: sized to the column's average row (more CTAs per SM for short strings)
  const long long row0 = (long long)blockIdx.x * TAKE_TILE;
  const int rows = (int)((n - row0) < TAKE_TILE ? (n - row0) : TAKE_TILE);
  const int tid = threadIdx.x;
  const int32_t bb = out_offsets[row0];
  const int tb = out_offsets[row0 + rows] - bb;
  if (tb > stage_bytes - 16) {  // long strings: straight per-row copies, a warp per row (tb + 16 would overflow near 2 GiB)
    const int lane = tid & 31;
    for (int i = tid >> 5; i < rows; i += 8) {
      const unsigned int r = idx[row0 + i];
      if (r == NO_ROW) continue;
      const int32_t s0 = offsets[r], len = offsets[r + 1] - s0;
      uint8_t* d = out + out_offsets[row0 + i];
      for (int b = lane; b < len; b += 32) d[b] = data[s0 + b];
    }
    return;
  }
  // staging starts at the destination's misalignment so that shared and global addresses agree mod 16
  const int mis = stage_misalignment(out + bb);
  // all index / offset loads of a thread's 4 rows are issued before any string is copied (three dependent
  // levels — index → offsets → bytes — would otherwise serialise per row)
  constexpr int RPT = TAKE_TILE / 256;
  int32_t s0[RPT], len[RPT], dst[RPT];
#pragma unroll
  for (int k = 0; k < RPT; ++k) {
    const int i = k * 256 + tid;
    s0[k] = 0; len[k] = 0; dst[k] = 0;
    if (i < rows) {
      const unsigned int r = idx[row0 + i];
      if (r != NO_ROW) {
        s0[k] = offsets[r];
        len[k] = offsets[r + 1] - s0[k];
      }
      dst[k] = out_offsets[row0 + i] - bb;
    }
  }
#pragma unroll
  for (int k = 0; k < RPT; ++k)
    if (len[k] > 0) gather_string(stage + mis + dst[k], data + s0[k], len[k]);
  __syncthreads();
  stage_store(out + bb, stage, mis, tb, tid, 256);
}

// ---- hash repartition ----------------------------------------------------------------------------------
__global__ void partition_ids_kernel(ColView kc, int key_kind, int64_t n, int n_parts, uint8_t* part, unsigned int* part_counts) {
  __shared__ unsigned int s_cnt[32];
  if (threadIdx.x < 32) s_cnt[threadIdx.x] = 0;
  __syncthreads();
  for (int64_t row = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; row < n; row += (int64_t)gridDim.x * blockDim.x) {
    Key16 k; unsigned long long h;
    make_key(key_kind, kc, row, &k, &h);
    const int p = partition_of(h, n_parts);
    part[row] = (uint8_t)p;
    atomicAdd(&s_cnt[p], 1u);
  }
  __syncthreads();
  if (threadIdx.x < n_parts && s_cnt[threadIdx.x]) atomicAdd(part_counts + threadIdx.x, s_cnt[threadIdx.x]);
}

// stable within a block chunk is not required: DataFusion's repartition does not preserve order either
__global__ void partition_scatter_kernel(const uint8_t* part, int64_t n, int n_parts, unsigned int* part_cursor, unsigned int* idx) {
  __shared__ unsigned int s_cnt[32], s_base[32];
  const int64_t chunk = (int64_t)blockDim.x * 8;
  for (int64_t base = (int64_t)blockIdx.x * chunk; base < n; base += (int64_t)gridDim.x * chunk) {
    if (threadIdx.x < 32) s_cnt[threadIdx.x] = 0;
    __syncthreads();
    unsigned int local[8]; int p[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int64_t row = base + j * blockDim.x + threadIdx.x;
      p[j] = row < n ? part[row] : -1;
      if (p[j] >= 0) local[j] = atomicAdd(&s_cnt[p[j]], 1u);
    }
    __syncthreads();
    if (threadIdx.x < n_parts) s_base[threadIdx.x] = s_cnt[threadIdx.x] ? atomicAdd(part_cursor + threadIdx.x, s_cnt[threadIdx.x]) : 0;
    __syncthreads();
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int64_t row = base + j * blockDim.x + threadIdx.x;
      if (p[j] >= 0) idx[s_base[p[j]] + local[j]] = (unsigned int)row;
    }
    __syncthreads();
  }
}

int key_kind_of(DType t) {
  switch (t) {
    case DType::Int64: return KEY_INT64;
    case DType::Bool: return KEY_BOOL;
    case DType::Utf8: case DType::Binary: return KEY_BYTES;
    default: fail(ARK_ERR_UNSUPPORTED, std::string("hash key of type ") + dtype_name(t));
  }
}

const char* const OFFSET_OVERFLOW = "Collection query results error: Arrow error: offset overflow, result column exceeds 2 GiB";

unsigned grid_for(int64_t n, int threads = 256) { return (unsigned)std::max<int64_t>(1, std::min<int64_t>(ceil_div(n, threads), sm_count() * 16)); }

}  // namespace

// out[i] = column[idx[i]] for i < n  (idx on the device).  may_miss: idx may hold NO_ROW (outer join without a match):
// such rows come out NULL, so the column always gets a validity bitmap.
Column take_column(const Column& src, const unsigned int* idx, int64_t n, const std::string& name, cudaStream_t stream, bool may_miss) {
  if (n >= (1ll << 31) - 1) fail(ARK_ERR_UNSUPPORTED, "gather of 2^31 or more rows in one batch");
  Column c;
  c.field = src.field; c.field.name = name; c.length = n;
  const unsigned g = (unsigned)std::max<int64_t>(1, ceil_div(n, 256));
  switch (src.field.type) {
    case DType::Int64: case DType::Float64: {
      BufferPtr d = device_alloc((size_t)std::max<int64_t>(n, 1) * 8);
      if (n) { KernelTimer t("take_fixed8_kernel", stream); take_fixed8_kernel<<<g, 256, 0, stream>>>((const unsigned long long*)src.data, idx, n, (unsigned long long*)d.get()); }
      c.data = (const uint8_t*)d.get(); c.data_bytes = n * 8; c.owners = {d};
      break;
    }
    case DType::Bool: {
      BufferPtr bytes = device_alloc((size_t)std::max<int64_t>(n, 1));
      if (n) { KernelTimer t("take_bits_kernel", stream); take_bits_kernel<<<g, 256, 0, stream>>>(src.data, src.data_bit0, idx, n, (uint8_t*)bytes.get()); }
      set_bool_values(c, bytes, n, stream);
      break;
    }
    case DType::Utf8: case DType::Binary: {
      // lens[n] = 0 closes the scan; the 64-bit total sits in the 8 bytes after it
      BufferPtr lens = device_alloc((size_t)(n + 1) * 4 + 16);
      ARK_CUDA(cudaMemsetAsync(lens.get(), 0, (size_t)(n + 1) * 4 + 16, stream));
      unsigned long long* total64 = (unsigned long long*)((uint8_t*)lens.get() + round_up((int64_t)(n + 1) * 4, 8));
      if (n) { KernelTimer t("take_lengths_kernel", stream); take_lengths_kernel<<<g, 256, 0, stream>>>(src.offsets, idx, n, (int32_t*)lens.get(), total64); }
      const Varlen v = varlen_layout((const int32_t*)lens.get(), n, total64, -1, OFFSET_OVERFLOW, stream);
      if (n) {
        KernelTimer t("take_bytes_tile_kernel", stream);
        const int stage = stage_window(v.total, n, TAKE_TILE);
        take_bytes_tile_kernel<<<(unsigned)ceil_div(n, TAKE_TILE), 256, stage, stream>>>(src.data, src.offsets, idx, n, (const int32_t*)v.offsets.get(), (uint8_t*)v.bytes.get(), stage);
      }
      set_varlen(c, v);
      break;
    }
    default:
      if (src.field.format != "n") fail(ARK_ERR_UNSUPPORTED, "gather of a column with Arrow type '" + src.field.format + "'");
      break;
  }
  if (may_miss) c.field.nullable = true;
  if ((src.validity || may_miss) && n > 0) {
    BufferPtr vb = device_alloc((size_t)n);
    if (src.validity) { KernelTimer t("take_bits_kernel", stream); take_bits_kernel<<<g, 256, 0, stream>>>(src.validity, src.validity_bit0, idx, n, (uint8_t*)vb.get()); }
    else { KernelTimer t("take_matched_kernel", stream); take_matched_kernel<<<g, 256, 0, stream>>>(idx, n, (uint8_t*)vb.get()); }
    set_validity_unknown(c, vb, n, stream);
  }
  return c;
}

// Gathers several columns at once: specs[k] = (source column, which of the two index arrays, output name, may_miss).
// Fixed-width and string columns without a validity bitmap go through take_multi_kernel — one launch for all values and
// lengths, one host round trip for all string totals; anything else (Boolean, nullable, outer-join misses) takes take_column.
std::vector<Column> take_columns(const std::vector<TakeSpec>& specs, const unsigned int* idx0, const unsigned int* idx1, int64_t n, cudaStream_t stream) {
  if (n >= (1ll << 31) - 1) fail(ARK_ERR_UNSUPPORTED, "gather of 2^31 or more rows in one batch");
  std::vector<Column> out(specs.size());
  std::vector<int> fixed, strs;
  for (size_t k = 0; k < specs.size(); ++k) {
    const Column& src = *specs[k].src;
    const bool plain = !src.validity && !specs[k].may_miss && n > 0;
    const bool is_fixed = src.field.type == DType::Int64 || src.field.type == DType::Float64;
    const bool is_str = src.field.type == DType::Utf8 || src.field.type == DType::Binary;
    if (plain && is_fixed && (int)fixed.size() < TAKE_MAX_FIXED) fixed.push_back((int)k);
    else if (plain && is_str && (int)strs.size() < TAKE_MAX_STR) strs.push_back((int)k);
    else out[k] = take_column(src, specs[k].side == 0 ? idx0 : idx1, n, specs[k].name, stream, specs[k].may_miss);
  }
  if (fixed.empty() && strs.empty()) return out;
  TakeMultiParams P;
  memset(&P, 0, sizeof P);
  P.idx[0] = idx0; P.idx[1] = idx1;
  std::vector<BufferPtr> fbuf, lens;
  std::vector<Varlen> strv(strs.size());
  // each string column's 64-bit byte total: added up by take_multi_kernel, fetched in one round trip
  BufferPtr sums = device_alloc(8 * (size_t)std::max<size_t>(strs.size(), 1)), h = pinned_alloc(8 * (size_t)std::max<size_t>(strs.size(), 1));
  if (!strs.empty()) ARK_CUDA(cudaMemsetAsync(sums.get(), 0, 8 * strs.size(), stream));
  P.stotal = (unsigned long long*)sums.get();
  for (int k : fixed) {
    BufferPtr d = device_alloc((size_t)n * 8);
    P.fsrc[P.n_fixed] = (const unsigned long long*)specs[k].src->data; P.fdst[P.n_fixed] = (unsigned long long*)d.get(); P.fside[P.n_fixed] = (uint8_t)specs[k].side;
    ++P.n_fixed; fbuf.push_back(d);
  }
  for (int k : strs) {
    BufferPtr l = device_alloc((size_t)(n + 1) * 4);
    ARK_CUDA(cudaMemsetAsync((int32_t*)l.get() + n, 0, 4, stream));
    P.soff[P.n_str] = specs[k].src->offsets; P.slen[P.n_str] = (int32_t*)l.get(); P.sside[P.n_str] = (uint8_t)specs[k].side;
    ++P.n_str; lens.push_back(l);
  }
  {
    KernelTimer t("take_multi_kernel", stream);
    take_multi_kernel<<<grid_for(n), 256, 0, stream>>>(P, n);
  }
  // string columns: offsets by scan; every column's total comes back in one round trip
  if (!strs.empty()) ARK_CUDA(cudaMemcpyAsync(h.get(), sums.get(), 8 * strs.size(), cudaMemcpyDeviceToHost, stream));
  for (size_t j = 0; j < strs.size(); ++j) strv[j].offsets = varlen_scan((const int32_t*)lens[j].get(), n, stream);
  if (!strs.empty()) ARK_CUDA(cudaStreamSynchronize(stream));
  for (size_t j = 0; j < strs.size(); ++j) {
    Varlen& v = strv[j];
    v.total = varlen_guard(((const unsigned long long*)h.get())[j], OFFSET_OVERFLOW);
    v.bytes = device_alloc((size_t)v.total + 16);
    const TakeSpec& sp = specs[strs[j]];
    {
      KernelTimer t("take_bytes_tile_kernel", stream);
      const int stage = stage_window(v.total, n, TAKE_TILE);
      take_bytes_tile_kernel<<<(unsigned)ceil_div(n, TAKE_TILE), 256, stage, stream>>>(sp.src->data, sp.src->offsets, sp.side == 0 ? idx0 : idx1, n, (const int32_t*)v.offsets.get(),
                                                                                      (uint8_t*)v.bytes.get(), stage);
    }
    Column& c = out[strs[j]];
    c.field = sp.src->field; c.field.name = sp.name; c.length = n;
    set_varlen(c, v);
    c.validity = nullptr; c.null_count = 0;
  }
  for (size_t j = 0; j < fixed.size(); ++j) {
    const TakeSpec& sp = specs[fixed[j]];
    Column& c = out[fixed[j]];
    c.field = sp.src->field; c.field.name = sp.name; c.length = n;
    c.data = (const uint8_t*)fbuf[j].get(); c.data_bytes = n * 8; c.owners = {fbuf[j]}; c.validity = nullptr; c.null_count = 0;
  }
  return out;
}

Batch run_join(const Plan& plan, Batch& left, Batch& right, cudaStream_t stream) {
  // row counts travel through cub scans with 32-bit item counts and through 32-bit row indices
  if (left.num_rows >= (1ll << 31) - 1 || right.num_rows >= (1ll << 31) - 1) fail(ARK_ERR_UNSUPPORTED, "join input with 2^31 or more rows in one batch");
  Column& lk = left.cols[plan.left_key];
  Column& rk = right.cols[plan.right_key];
  const int key_kind = key_kind_of(lk.field.type);
  // outer joins probe with the preserved side (LEFT: left, RIGHT: right); inner joins build on the smaller side
  const int outer = plan.join_type != 0;
  const bool build_left = plan.join_type == 1 ? false : plan.join_type == 2 ? true : left.num_rows <= right.num_rows;
  Batch& B = build_left ? left : right;
  Batch& Pb = build_left ? right : left;
  const ColView bc = (build_left ? lk : rk).view(), pc = (build_left ? rk : lk).view();
  const int64_t nb = B.num_rows, np = Pb.num_rows;

  unsigned long long capacity = 1ull << 10;
  while (capacity < 2ull * (unsigned long long)std::max<int64_t>(nb, 1)) capacity <<= 1;
  BufferPtr keys = device_alloc((size_t)capacity * sizeof(Key16)), head = device_alloc((size_t)capacity * 4);
  BufferPtr next = device_alloc((size_t)std::max<int64_t>(nb, 1) * 4);
  {
    KernelTimer t("join_init_kernel", stream);
    join_init_kernel<<<grid_for((int64_t)capacity), 256, 0, stream>>>((Key16*)keys.get(), (unsigned int*)head.get(), capacity);
  }
  if (nb) {
    KernelTimer t("join_build_kernel", stream);
    join_build_kernel<<<grid_for(nb), 256, 0, stream>>>(bc, key_kind, nb, (Key16*)keys.get(), (unsigned int*)head.get(), (unsigned int*)next.get(), capacity - 1);
  }
  if (capacity >= (1ull << 32)) fail(ARK_ERR_UNSUPPORTED, "join build side with 2^31 or more distinct keys");
  BufferPtr counts = device_alloc((size_t)(np + 1) * 8), offsets = device_alloc((size_t)(np + 1) * 8), match_slot = device_alloc((size_t)std::max<int64_t>(np, 1) * 4);
  ARK_CUDA(cudaMemsetAsync((long long*)counts.get() + np, 0, 8, stream));
  if (np) {
    KernelTimer t("join_probe_count_kernel", stream);
    join_probe_count_kernel<<<grid_for(np), 256, 0, stream>>>(pc, bc, key_kind, np, (const Key16*)keys.get(), (const unsigned int*)head.get(),
                                                              (const unsigned int*)next.get(), capacity - 1, (long long*)counts.get(), (unsigned int*)match_slot.get(), outer);
  }
  size_t tb = 0;
  cub::DeviceScan::ExclusiveSum(nullptr, tb, (long long*)counts.get(), (long long*)offsets.get(), (int)(np + 1), stream);
  BufferPtr tmp = device_alloc(tb + 16);
  note_launch("cub::DeviceScan::ExclusiveSum");
  cub::DeviceScan::ExclusiveSum(tmp.get(), tb, (long long*)counts.get(), (long long*)offsets.get(), (int)(np + 1), stream);
  BufferPtr h = pinned_alloc(64);
  ARK_CUDA(cudaMemcpyAsync(h.get(), (long long*)offsets.get() + np, 8, cudaMemcpyDeviceToHost, stream));
  ARK_CUDA(cudaStreamSynchronize(stream));
  const long long pairs = *(long long*)h.get();
  if (pairs >= (1ll << 31)) fail(ARK_ERR_UNSUPPORTED, "join result with 2^31 or more rows in one batch");
  BufferPtr probe_idx = device_alloc((size_t)std::max<long long>(pairs, 1) * 4), build_idx = device_alloc((size_t)std::max<long long>(pairs, 1) * 4);
  if (np && pairs) {
    KernelTimer t("join_probe_fill_kernel", stream);
    join_probe_fill_kernel<<<grid_for(np), 256, 0, stream>>>(np, (const unsigned int*)head.get(), (const unsigned int*)next.get(), (const unsigned int*)match_slot.get(),
                                                             (const long long*)offsets.get(), (unsigned int*)probe_idx.get(), (unsigned int*)build_idx.get(), outer);
  }
  ARK_CUDA(cudaGetLastError());
  const unsigned int* lidx = (const unsigned int*)(build_left ? build_idx.get() : probe_idx.get());
  const unsigned int* ridx = (const unsigned int*)(build_left ? probe_idx.get() : build_idx.get());
  Batch out;
  out.num_rows = pairs;
  std::vector<TakeSpec> specs;
  for (const auto& jo : plan.join_out) {
    const Column& src = jo.side == 0 ? left.cols[jo.col] : right.cols[jo.col];
    if (!src.present) fail(ARK_ERR_UNSUPPORTED, "join output column '" + jo.name + "' has Arrow type '" + src.field.format + "'");
    const bool build_side = (jo.side == 0) == build_left;
    specs.push_back({&src, jo.side, jo.name, (bool)(outer && build_side)});
  }
  out.cols = take_columns(specs, lidx, ridx, pairs, stream);
  ARK_CUDA(cudaStreamSynchronize(stream));
  return out;
}

// RepartitionExec(Hash([key], n_parts)): rows reordered into n_parts contiguous ranges by key owner
Batch hash_partition(Batch& in, const std::string& key_column, int n_parts, std::vector<int64_t>& part_rows, cudaStream_t stream) {
  if (n_parts < 1 || n_parts > 32) fail(ARK_ERR_PROCESS, "n_parts must be in [1, 32]");
  const int ki = in.find(key_column);
  if (ki < 0) fail(ARK_ERR_PROCESS, "Schema error: No field named " + key_column + ".");
  const int64_t n = in.num_rows;
  if (n >= (1ll << 31) - 1) fail(ARK_ERR_UNSUPPORTED, "partition input with 2^31 or more rows in one batch");
  const int key_kind = key_kind_of(in.cols[ki].field.type);
  BufferPtr part = device_alloc((size_t)std::max<int64_t>(n, 1)), idx = device_alloc((size_t)std::max<int64_t>(n, 1) * 4);
  BufferPtr ctl = device_alloc(256), hctl = pinned_alloc(256);
  ARK_CUDA(cudaMemsetAsync(ctl.get(), 0, 256, stream));
  unsigned int* counts = (unsigned int*)ctl.get();
  unsigned int* cursor = counts + 32;
  if (n) {
    KernelTimer t("partition_ids_kernel", stream);
    partition_ids_kernel<<<grid_for(n), 256, 0, stream>>>(in.cols[ki].view(), key_kind, n, n_parts, (uint8_t*)part.get(), counts);
  }
  ARK_CUDA(cudaMemcpyAsync(hctl.get(), counts, 128, cudaMemcpyDeviceToHost, stream));
  ARK_CUDA(cudaStreamSynchronize(stream));
  unsigned int* hc = (unsigned int*)hctl.get();
  unsigned int* hcur = hc + 32;
  unsigned int run = 0;
  part_rows.assign(n_parts, 0);
  for (int p = 0; p < n_parts; ++p) { part_rows[p] = hc[p]; hcur[p] = run; run += hc[p]; }
  ARK_CUDA(cudaMemcpyAsync(cursor, hcur, 128, cudaMemcpyHostToDevice, stream));
  if (n) {
    KernelTimer t("partition_scatter_kernel", stream);
    partition_scatter_kernel<<<grid_for(ceil_div(n, 8)), 256, 0, stream>>>((const uint8_t*)part.get(), n, n_parts, cursor, (unsigned int*)idx.get());
  }
  ARK_CUDA(cudaGetLastError());
  Batch out;
  out.num_rows = n; out.input_name = in.input_name;
  // the partition-ordered columns are what the peers map (ipc_exchange.cu): one arena for all of them.  The output is a
  // permutation of the input, so its size is the input's (+ the gather's temporaries: lengths, offsets, scan scratch)
  size_t out_bytes = 1 << 20;
  for (auto& c : in.cols) {
    const bool vl = c.field.type == DType::Utf8 || c.field.type == DType::Binary;
    out_bytes += vl ? (size_t)(n + 1) * 12 + (size_t)std::max<int64_t>(varlen_bytes_bound(c), 0) + 4096 : (size_t)n * 8 + 1024;
    out_bytes += c.validity ? (size_t)n + (size_t)n / 8 + 2048 : 0;
  }
  ExportAllocScope exported(out_bytes);
  std::vector<TakeSpec> specs;
  for (auto& c : in.cols) {
    if (!c.present) fail(ARK_ERR_UNSUPPORTED, "partition of a column with Arrow type '" + c.field.format + "'");
    specs.push_back({&c, 0, c.field.name, false});
  }
  out.cols = take_columns(specs, (const unsigned int*)idx.get(), nullptr, n, stream);
  ARK_CUDA(cudaStreamSynchronize(stream));
  return out;
}

}  // namespace ark
