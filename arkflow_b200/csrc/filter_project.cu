// filter_project.cu — fused WHERE + SELECT-list + order-preserving compaction in ONE pass over HBM.
//
// Stands in for DataFusion's FilterExec → ProjectionExec → CoalesceBatchesExec and the final
// concat_batches of the reference (crates/arkflow-plugin/src/processor/sql.rs:126-129,145-148).
//
// Single pass: each CTA takes a 2048-row tile (dynamic ticket, so tile t-1 always started before
// tile t), evaluates the predicate, ranks the surviving rows with warp ballots, obtains its global
// output position from a decoupled look-back over per-tile descriptors (rows and string bytes are
// separate 62-bit channels), then stages every projected column through shared memory so that all
// global stores are coalesced.  Algorithmic traffic = every referenced input byte read once +
// every output byte written once (SURVEY.md §8(d): 36 B/row for config 2).
#include "batch.h"
#include "filter_project.cuh"
#include "utf8.cuh"
#include "vm.cuh"

namespace ark {

namespace {

constexpr unsigned long long DESC_AGG = 1ull << 62;
constexpr unsigned long long DESC_PREFIX = 2ull << 62;
constexpr unsigned long long DESC_MASK = (1ull << 62) - 1;

__device__ __forceinline__ unsigned long long ld_volatile_u64(const unsigned long long* p) {
  unsigned long long v;
  asm volatile("ld.volatile.global.u64 %0, [%1];" : "=l"(v) : "l"(p));
  return v;
}
__device__ __forceinline__ void st_volatile_u64(unsigned long long* p, unsigned long long v) {
  asm volatile("st.volatile.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ ulonglong2 ld_stream_v2(const unsigned long long* p) {
  ulonglong2 v;
  asm volatile("ld.global.nc.L1::no_allocate.v2.u64 {%0, %1}, [%2];" : "=l"(v.x), "=l"(v.y) : "l"(p));
  return v;
}
__device__ __forceinline__ long long warp_sum(long long v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// Decoupled look-back (Merrill & Garland) for one channel, executed by one full warp.
// Returns the exclusive prefix of `agg` over all earlier tiles.
__device__ long long lookback(unsigned long long* desc, int tile, int ch, long long agg, int lane) {
  unsigned long long* mine = desc + (size_t)tile * FP_CHANNELS + ch;
  if (tile == 0) {
    if (lane == 0) st_volatile_u64(mine, DESC_PREFIX | (unsigned long long)agg);
    return 0;
  }
  if (lane == 0) st_volatile_u64(mine, DESC_AGG | (unsigned long long)agg);
  long long running = 0;
  int look = tile - 1;
  while (true) {
    int idx = look - lane;
    unsigned long long d = DESC_PREFIX;  // virtual tile -1: inclusive prefix 0
    if (idx >= 0) {
      do { d = ld_volatile_u64(desc + (size_t)idx * FP_CHANNELS + ch); } while ((d >> 62) == 0);
    }
    __syncwarp();
    unsigned pm = __ballot_sync(0xffffffffu, (d >> 62) == 2);
    long long val = (long long)(d & DESC_MASK);
    if (pm) {
      int first = __ffs(pm) - 1;
      if (lane > first) val = 0;
      running += warp_sum(val);
      break;
    }
    running += warp_sum(val);
    look -= 32;
  }
  if (lane == 0) st_volatile_u64(mine, DESC_PREFIX | (unsigned long long)(running + agg));
  return running;
}

template <int PRED, int NV>
__global__ void __launch_bounds__(FP_THREADS) filter_project_kernel(const __grid_constant__ FpParams P) {
  extern __shared__ __align__(16) uint8_t smem[];
  __shared__ unsigned s_tile;
  __shared__ int s_cnt[FP_CHUNKS * FP_WARPS];
  __shared__ int s_bytes[FP_MAX_VARLEN][FP_CHUNKS * FP_WARPS];
  __shared__ long long s_excl[FP_CHANNELS];
  __shared__ int s_total[FP_CHANNELS];

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const unsigned lt_mask = (1u << lane) - 1;
  if (tid == 0) s_tile = atomicAdd(P.ticket, 1u);
  __syncthreads();
  const int tile = (int)s_tile;
  const int64_t row0 = (int64_t)tile * FP_TILE;
  const int64_t n = P.n_rows;
  int32_t err = 0;

  // ---- phase A: predicate → flags, per-warp counts ----
  unsigned flags = 0;
  unsigned b0[FP_CHUNKS], b1[FP_CHUNKS];
#pragma unroll
  for (int k = 0; k < FP_CHUNKS; ++k) {
    const int64_t r = row0 + k * FP_CHUNK_ROWS + 2 * tid;
    bool f0 = r < n, f1 = r + 1 < n;
    if (PRED == 1) {
      const ColView& c = P.cols[P.sp_slot];
      const unsigned long long* d = (const unsigned long long*)c.data;
      unsigned long long v0 = 0, v1 = 0;
      if (f1 && ((reinterpret_cast<uintptr_t>(d) & 15) == 0)) {
        ulonglong2 v = ld_stream_v2(d + r);
        v0 = v.x; v1 = v.y;
      } else {
        if (f0) v0 = d[r];
        if (f1) v1 = d[r + 1];
      }
      if (P.sp_is_f64) {
        const int64_t kc = f64_total_key(P.sp_const);
        f0 = f0 && cmp_i64(P.sp_cmp, f64_total_key(v0), kc);
        f1 = f1 && cmp_i64(P.sp_cmp, f64_total_key(v1), kc);
      } else {
        f0 = f0 && cmp_i64(P.sp_cmp, (int64_t)v0, (int64_t)P.sp_const);
        f1 = f1 && cmp_i64(P.sp_cmp, (int64_t)v1, (int64_t)P.sp_const);
      }
      if (c.validity) {
        f0 = f0 && bit_get(c.validity, r + c.validity_bit0);
        f1 = f1 && bit_get(c.validity, r + 1 + c.validity_bit0);
      }
    } else if (PRED == 2) {
      if (f0) { VmVal v = vm_eval(P.pred, P.cols, r, &err); f0 = v.valid && (v.bits & 1); }
      if (f1) { VmVal v = vm_eval(P.pred, P.cols, r + 1, &err); f1 = v.valid && (v.bits & 1); }
    }
    b0[k] = __ballot_sync(0xffffffffu, f0);
    b1[k] = __ballot_sync(0xffffffffu, f1);
    flags |= ((unsigned)f0 << (2 * k)) | ((unsigned)f1 << (2 * k + 1));
    if (lane == 0) s_cnt[k * FP_WARPS + warp] = __popc(b0[k]) + __popc(b1[k]);
  }

  // ---- phase A2: byte lengths of the surviving rows of each var-len output ----
  int bp[NV > 0 ? NV : 1][FP_CHUNKS][2];
#pragma unroll
  for (int v = 0; v < NV; ++v) {
    const int32_t* off = P.cols[P.varlen_slot[v]].offsets;
#pragma unroll
    for (int k = 0; k < FP_CHUNKS; ++k) {
      const int64_t r = row0 + k * FP_CHUNK_ROWS + 2 * tid;
      const bool f0 = (flags >> (2 * k)) & 1, f1 = (flags >> (2 * k + 1)) & 1;
      int len0 = 0, len1 = 0;
      if (f0 || f1) {
        int o1 = off[r + 1];
        if (f0) len0 = o1 - off[r];
        if (f1) len1 = off[r + 2] - o1;
      }
      int incl = len0 + len1;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        int t = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += t;
      }
      const int excl = incl - (len0 + len1);
      bp[v][k][0] = excl;
      bp[v][k][1] = excl + len0;
      if (lane == 31) s_bytes[v][k * FP_WARPS + warp] = incl;
    }
  }
  __syncthreads();

  // ---- phase B: tile-level scan of the 32 (chunk, warp) partials + decoupled look-back ----
  if (warp == 0) {
    {
      int c = s_cnt[lane], incl = c;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) { int t = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += t; }
      s_cnt[lane] = incl - c;
      const int total = __shfl_sync(0xffffffffu, incl, 31);
      const long long ex = lookback(P.desc, tile, 0, total, lane);
      if (lane == 0) { s_excl[0] = ex; s_total[0] = total; if (tile == P.n_tiles - 1) P.totals[0] = ex + total; }
    }
#pragma unroll
    for (int v = 0; v < NV; ++v) {
      int c = s_bytes[v][lane], incl = c;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) { int t = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += t; }
      s_bytes[v][lane] = incl - c;
      const int total = __shfl_sync(0xffffffffu, incl, 31);
      const long long ex = lookback(P.desc, tile, 1 + v, total, lane);
      if (lane == 0) { s_excl[1 + v] = ex; s_total[1 + v] = total; if (tile == P.n_tiles - 1) P.totals[1 + v] = ex + total; }
    }
  }
  __syncthreads();

  const int tile_cnt = s_total[0];
  const long long base_cnt = s_excl[0];
  int rank[FP_CHUNKS][2];
#pragma unroll
  for (int k = 0; k < FP_CHUNKS; ++k) {
    const int base = s_cnt[k * FP_WARPS + warp] + __popc(b0[k] & lt_mask) + __popc(b1[k] & lt_mask);
    rank[k][0] = base;
    rank[k][1] = base + ((flags >> (2 * k)) & 1);
  }

  // ---- phase D: stage each output column through shared memory, store coalesced ----
  for (int o = 0; o < P.n_out; ++o) {
    const FpOutput& out = P.outs[o];
    if (out.kind == FP_OUT_FIXED8 || out.kind == FP_OUT_COMPUTED8) {
      unsigned long long* st = reinterpret_cast<unsigned long long*>(smem);
      uint8_t* stv = smem + FP_TILE * 8;
#pragma unroll
      for (int k = 0; k < FP_CHUNKS; ++k) {
#pragma unroll
        for (int j = 0; j < 2; ++j) {
          if ((flags >> (2 * k + j)) & 1) {
            const int64_t r = row0 + k * FP_CHUNK_ROWS + 2 * tid + j;
            unsigned long long val; bool valid;
            if (out.kind == FP_OUT_FIXED8) {
              const ColView& c = P.cols[out.slot];
              val = ((const unsigned long long*)c.data)[r];
              valid = col_valid(c, r);
            } else {
              VmVal vv = vm_eval(P.progs[out.prog], P.cols, r, &err);
              val = vv.bits; valid = vv.valid;
            }
            st[rank[k][j]] = val;
            if (out.write_validity) stv[rank[k][j]] = valid;
          }
        }
      }
      __syncthreads();
      unsigned long long* dst = reinterpret_cast<unsigned long long*>(out.out_data) + base_cnt;
      for (int i = tid; i < tile_cnt; i += FP_THREADS) dst[i] = st[i];
      if (out.write_validity)
        for (int i = tid; i < tile_cnt; i += FP_THREADS) out.out_valid[base_cnt + i] = stv[i];
      __syncthreads();
    } else if (out.kind == FP_OUT_BOOL || out.kind == FP_OUT_COMPUTED_BOOL) {
      uint8_t* st = smem;
      uint8_t* stv = smem + FP_TILE;
#pragma unroll
      for (int k = 0; k < FP_CHUNKS; ++k) {
#pragma unroll
        for (int j = 0; j < 2; ++j) {
          if ((flags >> (2 * k + j)) & 1) {
            const int64_t r = row0 + k * FP_CHUNK_ROWS + 2 * tid + j;
            bool val, valid;
            if (out.kind == FP_OUT_BOOL) {
              const ColView& c = P.cols[out.slot];
              val = bit_get((const uint8_t*)c.data, r + c.data_bit0);
              valid = col_valid(c, r);
            } else {
              VmVal vv = vm_eval(P.progs[out.prog], P.cols, r, &err);
              val = vv.bits & 1; valid = vv.valid;
            }
            st[rank[k][j]] = val;
            if (out.write_validity) stv[rank[k][j]] = valid;
          }
        }
      }
      __syncthreads();
      uint8_t* dst = reinterpret_cast<uint8_t*>(out.out_data) + base_cnt;
      for (int i = tid; i < tile_cnt; i += FP_THREADS) dst[i] = st[i];
      if (out.write_validity)
        for (int i = tid; i < tile_cnt; i += FP_THREADS) out.out_valid[base_cnt + i] = stv[i];
      __syncthreads();
    } else if (NV > 0 && out.kind == FP_OUT_VARLEN) {
      const int v = out.varlen_idx < NV ? out.varlen_idx : 0;
      const ColView& c = P.cols[out.slot];
      const int tb = s_total[1 + v];
      const long long bb = s_excl[1 + v];
      // offsets (and validity bytes) of the surviving rows
      int32_t* st32 = reinterpret_cast<int32_t*>(smem);
      uint8_t* stv = smem + FP_TILE * 4;
#pragma unroll
      for (int k = 0; k < FP_CHUNKS; ++k) {
#pragma unroll
        for (int j = 0; j < 2; ++j) {
          if ((flags >> (2 * k + j)) & 1) {
            const int64_t r = row0 + k * FP_CHUNK_ROWS + 2 * tid + j;
            st32[rank[k][j]] = (int32_t)(bb + s_bytes[v][k * FP_WARPS + warp] + bp[v][k][j]);
            if (out.write_validity) stv[rank[k][j]] = col_valid(c, r);
          }
        }
      }
      __syncthreads();
      for (int i = tid; i < tile_cnt; i += FP_THREADS) out.out_offsets[base_cnt + i] = st32[i];
      if (out.write_validity)
        for (int i = tid; i < tile_cnt; i += FP_THREADS) out.out_valid[base_cnt + i] = stv[i];
      if (tile == P.n_tiles - 1 && tid == 0) out.out_offsets[base_cnt + tile_cnt] = (int32_t)(bb + tb);
      __syncthreads();
      // bytes
      uint8_t* gout = reinterpret_cast<uint8_t*>(out.out_data);
      const uint8_t* gin = reinterpret_cast<const uint8_t*>(c.data);
      if (tb <= FP_STR_STAGE - 16) {
        const int shift = (int)(bb & 15);
#pragma unroll
        for (int k = 0; k < FP_CHUNKS; ++k) {
#pragma unroll
          for (int j = 0; j < 2; ++j) {
            if ((flags >> (2 * k + j)) & 1) {
              const int64_t r = row0 + k * FP_CHUNK_ROWS + 2 * tid + j;
              const int32_t o0 = c.offsets[r], o1 = c.offsets[r + 1];
              uint8_t* d = smem + shift + s_bytes[v][k * FP_WARPS + warp] + bp[v][k][j];
              const uint8_t* s = gin + o0;
              for (int i = 0; i < o1 - o0; ++i) d[i] = __ldg(s + i);
            }
          }
        }
        __syncthreads();
        uint8_t* gbase = gout + (bb - shift);
        const int total = shift + tb;
        for (int p = tid * 16; p < total; p += FP_THREADS * 16) {
          if (p >= shift && p + 16 <= total) {
            *reinterpret_cast<uint4*>(gbase + p) = *reinterpret_cast<const uint4*>(smem + p);
          } else {
            const int q0 = p > shift ? p : shift, q1 = (p + 16 < total) ? p + 16 : total;
            for (int q = q0; q < q1; ++q) gbase[q] = smem[q];
          }
        }
        __syncthreads();
      } else {  // long strings: copy straight from global to global
#pragma unroll 1
        for (int k = 0; k < FP_CHUNKS; ++k) {
#pragma unroll 1
          for (int j = 0; j < 2; ++j) {
            if ((flags >> (2 * k + j)) & 1) {
              const int64_t r = row0 + k * FP_CHUNK_ROWS + 2 * tid + j;
              const int32_t o0 = c.offsets[r], o1 = c.offsets[r + 1];
              uint8_t* d = gout + bb + s_bytes[v][k * FP_WARPS + warp] + bp[v][k][j];
              const uint8_t* s = gin + o0;
              for (int i = 0; i < o1 - o0; ++i) d[i] = s[i];
            }
          }
        }
      }
    }
  }
  if (err) atomicExch(P.error, err);
}

// byte-per-row (0/1) → bitmap; counts zero bytes into *zeros (null count for validity maps)
__global__ void pack_bits_kernel(const uint8_t* bytes, int64_t n, uint8_t* bitmap, unsigned long long* zeros) {
  int64_t ob = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  int64_t nb = (n + 7) >> 3;
  int z = 0;
  if (ob < nb) {
    unsigned v = 0;
    for (int i = 0; i < 8; ++i) {
      int64_t r = ob * 8 + i;
      if (r < n) { if (bytes[r]) v |= 1u << i; else ++z; }
    }
    bitmap[ob] = (uint8_t)v;
  }
  z = (int)warp_sum(z);
  if ((threadIdx.x & 31) == 0 && z && zeros) atomicAdd(zeros, (unsigned long long)z);
}

// One thread validates one string (utf8_valid).  Raises *bad when any non-NULL string is invalid.
__global__ void utf8_validate_kernel(const int32_t* offsets, const uint8_t* data, const uint8_t* validity, int vbit0, long long n, int* bad) {
  const long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n) return;
  if (validity && !((validity[(r + vbit0) >> 3] >> ((r + vbit0) & 7)) & 1)) return;
  if (!utf8_valid(data + offsets[r], offsets[r + 1] - offsets[r])) atomicExch(bad, 1);
}

template <int PRED, int NV>
void launch_fp(const FpParams& P, cudaStream_t stream) {
  KernelTimer t("filter_project_kernel", stream);
  filter_project_kernel<PRED, NV><<<P.n_tiles, FP_THREADS, FP_STR_STAGE, stream>>>(P);
}

}  // namespace

void launch_filter_project(const FpParams& P, int pred_kind, cudaStream_t stream) {
  const int nv = P.n_varlen;
#define ARK_FP_CASE(PR, NV) if (pred_kind == PR && nv == NV) { launch_fp<PR, NV>(P, stream); return; }
  ARK_FP_CASE(0, 0) ARK_FP_CASE(0, 1) ARK_FP_CASE(0, 2)
  ARK_FP_CASE(1, 0) ARK_FP_CASE(1, 1) ARK_FP_CASE(1, 2)
  ARK_FP_CASE(2, 0) ARK_FP_CASE(2, 1) ARK_FP_CASE(2, 2)
#undef ARK_FP_CASE
  fail(ARK_ERR_PROCESS, "internal: bad filter_project specialisation");
}

void launch_utf8_validate(const int32_t* offsets, const uint8_t* data, const uint8_t* validity, int vbit0, int64_t n, int* bad, cudaStream_t stream) {
  if (n <= 0) return;
  KernelTimer t("utf8_validate_kernel", stream);
  utf8_validate_kernel<<<(unsigned)ceil_div(n, 256), 256, 0, stream>>>(offsets, data, validity, vbit0, n, bad);
}

void launch_pack_bits(const uint8_t* bytes, int64_t n, uint8_t* bitmap, unsigned long long* zeros, cudaStream_t stream) {
  if (n <= 0) return;
  KernelTimer t("pack_bits_kernel", stream);
  int64_t nb = (n + 7) >> 3;
  pack_bits_kernel<<<(unsigned)ceil_div(nb, 256), 256, 0, stream>>>(bytes, n, bitmap, zeros);
}

}  // namespace ark
