// group_exchange.cu — the GROUP BY repartition exchange as device code: partial states are PUSHED over NVLink into
// the owner rank's receive region by the kernel that scans the partial table, and the owner's merge kernel consumes
// them as soon as every source has signalled — no host round trip, no NCCL call, no staging copy on the data path.
//
// Stands in for DataFusion's RepartitionExec(Hash) between AggregateExec(Partial) and AggregateExec(FinalPartitioned)
// (in-process in the reference: crates/arkflow-plugin/src/processor/sql.rs:126-129).  SURVEY.md §8(e): "one
// all-to-all(v) of partial (key, sum, count) states".  One process per GPU; every rank owns one COMM BUFFER
// (cudaMalloc, exported once with CUDA IPC, mapped by every peer at connect time):
//
//   header  ready[src]        u64   last step whose records from `src` are complete      (written by src)
//           ack[dst]          u64   last step `dst` has finished reading MY records      (written by dst)
//           count[par][src]   u64   records in recv[par][src]; bit 63 = POISON, 62 = OVERFLOW (written by src)
//           cursor[dst], done, flags  local scratch of the push kernel
//   data    recv[par][src]    region_bytes each: records {Key16, accumulators…} (32 B for ≤ 2 accumulators)
//
// A transported record is a table slot — key and accumulators gathered from the bucket: keys up to 12 bytes, Int64/Boolean keys
// and the NULL key are inline in Key16.  Keys longer than 12 bytes reference the sender's input batch and cannot
// travel this way: the sender marks the step POISON, every receiver sees it and the call returns ARK_ERR_UNSUPPORTED on
// every rank alike, so the caller falls back (collectively, without another message) to the descriptor exchange of
// ipc_exchange.cu.
//
// Ordering: record stores → __threadfence_system() → grid-wide "last CTA" count → count → st.release.sys ready.  The
// receiver polls ready with ld.acquire.sys.  Regions are double-buffered by step parity; before writing parity p of
// step s a sender waits for ack ≥ s − 2 from every destination (always already true in lockstep operation).
#include "abi.h"
#include "agg_acc.cuh"
#include "group_exchange.h"
#include "hash_agg.cuh"
#include "hashkey.cuh"

namespace ark {

namespace {

constexpr int GX_THREADS = 256;
constexpr int GX_SLOTS = 4;  // table slots per thread of the push kernel

__device__ __forceinline__ unsigned long long ld_acquire_sys(const unsigned long long* p) {
  unsigned long long v;
  asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_release_sys(unsigned long long* p, unsigned long long v) {
  asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ void st_relaxed_sys(unsigned long long* p, unsigned long long v) {
  asm volatile("st.relaxed.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}

struct PushParams {
  const uint8_t* table;
  unsigned long long capacity;
  int32_t n_acc, rec_bytes, key_kind, world, rank;
  int32_t need_count;  // the table also holds keys of earlier batches: push only slots whose COUNT(*) accumulator is non-zero
  unsigned long long step;
  unsigned long long cap_records, region_bytes;
  uint8_t* peers[GX_MAX_WORLD];  // comm buffer of every rank as mapped here (peers[rank] = the local one)
};

__global__ void __launch_bounds__(GX_THREADS) exchange_push_kernel(const __grid_constant__ PushParams P) {
  __shared__ unsigned s_cnt[GX_MAX_WORLD], s_base[GX_MAX_WORLD];
  __shared__ int s_last;
  const int tid = threadIdx.x;
  GxHeader* hdr = reinterpret_cast<GxHeader*>(P.peers[P.rank]);
  if (tid < GX_MAX_WORLD) s_cnt[tid] = 0;
  // this parity's regions at every destination were last used by step − 2: wait until it has been consumed
  if (tid < P.world && P.step > 2) while (ld_acquire_sys(&hdr->ack[tid]) + 2 < P.step) { }
  __syncthreads();
  const unsigned long long slot0 = (unsigned long long)blockIdx.x * (GX_THREADS * GX_SLOTS);
  const int bstride = table_bucket_stride(P.n_acc);
  Key16 key[GX_SLOTS];
  int part[GX_SLOTS];
  unsigned local[GX_SLOTS];
  unsigned flags = 0;
#pragma unroll
  for (int j = 0; j < GX_SLOTS; ++j) {
    const unsigned long long s = slot0 + (unsigned long long)j * GX_THREADS + tid;
    part[j] = -1;
    if (s >= P.capacity) continue;
    key[j] = *tbl_key(P.table, s, bstride);
    if (key[j].hi == KEY_EMPTY) continue;
    if (P.need_count && *tbl_acc(P.table, s, 0, bstride) == 0) continue;
    if (key_is_long(key[j]) || key_is_pair(key[j])) { flags |= 1; continue; }  // keys that reference the sender's rows cannot travel inline
    part[j] = P.world > 1 ? partition_of(P.key_kind == KEY_NONE ? 0 : hash_key16(key[j]), P.world) : 0;
    local[j] = atomicAdd(&s_cnt[part[j]], 1u);
  }
  __syncthreads();
  if (tid < P.world) s_base[tid] = s_cnt[tid] ? atomicAdd(&hdr->cursor[tid], s_cnt[tid]) : 0;
  __syncthreads();
  const int parity = (int)(P.step & 1);
#pragma unroll
  for (int j = 0; j < GX_SLOTS; ++j) {
    if (part[j] < 0) continue;
    const unsigned long long idx = (unsigned long long)s_base[part[j]] + local[j];
    if (idx >= P.cap_records) { flags |= 2; continue; }
    const unsigned long long s = slot0 + (unsigned long long)j * GX_THREADS + tid;
    uint8_t* rec = P.peers[part[j]] + GX_HEADER_BYTES + ((unsigned long long)(parity * P.world + P.rank)) * P.region_bytes +
                   idx * (unsigned long long)P.rec_bytes;
    *reinterpret_cast<uint4*>(rec) = make_uint4((unsigned)key[j].lo, (unsigned)(key[j].lo >> 32), (unsigned)key[j].hi, (unsigned)(key[j].hi >> 32));
    unsigned long long* av = reinterpret_cast<unsigned long long*>(rec + 16);
    int a = 0;
    for (; a + 1 < P.n_acc; a += 2) {
      const unsigned long long v0 = *tbl_acc(P.table, s, a, bstride), v1 = *tbl_acc(P.table, s, a + 1, bstride);
      *reinterpret_cast<ulonglong2*>(av + a) = make_ulonglong2(v0, v1);
    }
    if (a < P.n_acc) av[a] = *tbl_acc(P.table, s, a, bstride);
  }
  if (flags) atomicOr(&hdr->flags, flags);
  __threadfence_system();
  __syncthreads();
  if (tid == 0) s_last = atomicAdd(&hdr->done, 1u) == gridDim.x - 1;
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  if (tid < P.world) {
    const unsigned f = *reinterpret_cast<volatile unsigned*>(&hdr->flags);
    unsigned long long c = *reinterpret_cast<volatile unsigned*>(&hdr->cursor[tid]);
    if (f & 1) c |= GX_POISON;
    if (f & 2) c |= GX_OVERFLOW;
    GxHeader* peer = reinterpret_cast<GxHeader*>(P.peers[tid]);
    st_relaxed_sys(&peer->count[parity][P.rank], c);
    __threadfence_system();
    st_release_sys(&peer->ready[P.rank], P.step);
  }
  __syncthreads();
  if (tid < GX_MAX_WORLD) hdr->cursor[tid] = 0;
  if (tid == 0) { hdr->done = 0; hdr->flags = 0; }
}

struct MergeParams {
  uint8_t* table;            // final table (initialised with the accumulators' identities)
  unsigned long long mask;
  int32_t rec_bytes, n_acc, world, rank;
  int32_t acc_kind[AGG_MAX_ACC];
  unsigned long long step, region_bytes;
  const uint8_t* comm;       // the local comm buffer
  unsigned int* group_count;
  int32_t* overflow;         // final table too small
  int32_t* status;           // bit 0: a source sent POISON, bit 1: a source overflowed its region
  unsigned long long* total; // records received (written by CTA 0)
};

__global__ void __launch_bounds__(GX_THREADS) exchange_merge_kernel(const __grid_constant__ MergeParams P) {
  __shared__ unsigned long long s_pref[GX_MAX_WORLD + 1];
  __shared__ int s_bad;
  const int tid = threadIdx.x, lane = tid & 31;
  const GxHeader* hdr = reinterpret_cast<const GxHeader*>(P.comm);
  const int parity = (int)(P.step & 1);
  if (tid == 0) {
    int bad = 0;
    unsigned long long run = 0;
    for (int s = 0; s < P.world; ++s) {
      while (ld_acquire_sys(&hdr->ready[s]) < P.step) { }
      const unsigned long long c = *reinterpret_cast<const volatile unsigned long long*>(&hdr->count[parity][s]);
      if (c & GX_POISON) bad |= 1;
      if (c & GX_OVERFLOW) bad |= 2;
      s_pref[s] = run;
      run += c & GX_COUNT_MASK;
    }
    s_pref[P.world] = run;
    s_bad = bad;
    if (blockIdx.x == 0) { *P.total = run; if (bad) atomicOr(P.status, bad); }
  }
  __syncthreads();
  if (s_bad) return;
  const unsigned long long total = s_pref[P.world];
  unsigned int claimed = 0;
  int32_t over = 0;
  const int bstride = table_bucket_stride(P.n_acc);
  const uint8_t* data = P.comm + GX_HEADER_BYTES + (unsigned long long)parity * P.world * P.region_bytes;
  for (unsigned long long g = (unsigned long long)blockIdx.x * GX_THREADS + tid; g < total; g += (unsigned long long)gridDim.x * GX_THREADS) {
    int src = 0;
    while (src + 1 < P.world && g >= s_pref[src + 1]) ++src;
    const uint8_t* rec = data + (unsigned long long)src * P.region_bytes + (g - s_pref[src]) * (unsigned long long)P.rec_bytes;
    const uint4 k4 = *reinterpret_cast<const uint4*>(rec);
    const Key16 mine{(unsigned long long)k4.x | ((unsigned long long)k4.y << 32), (unsigned long long)k4.z | ((unsigned long long)k4.w << 32)};
    const ColView none{};
    const unsigned long long slot = table_find_or_claim(P.table, P.mask >> 2, bstride, (unsigned long long)(hash32_key16(mine) * 0x9E3779B1u), mine,
                                                        none, none, &claimed);
    if (slot == ~0ull) { over = 1; continue; }
    const unsigned long long* av = reinterpret_cast<const unsigned long long*>(rec + 16);
    for (int a = 0; a < P.n_acc; ++a) {
      const unsigned long long v = av[a];
      if (v != acc_identity(P.acc_kind[a])) merge_acc(P.acc_kind[a], tbl_acc(P.table, slot, a, bstride), v);
    }
  }
  if (over) atomicExch(P.overflow, 1);
  claimed = (unsigned int)__reduce_add_sync(0xffffffffu, claimed);
  if (lane == 0 && claimed) atomicAdd(P.group_count, claimed);
}

__global__ void exchange_ack_kernel(GxPeers peers, int world, int rank, unsigned long long step) {
  const int t = threadIdx.x;
  if (t < world) st_release_sys(&reinterpret_cast<GxHeader*>(peers.p[t])->ack[rank], step);
}

}  // namespace

int exchange_record_bytes(int n_acc) { return 16 * ((16 + 8 * n_acc + 15) / 16); }

void launch_exchange_push(const uint8_t* table, unsigned long long capacity, int n_acc, int key_kind, const GxPeers& peers, int world, int rank,
                          unsigned long long step, unsigned long long region_bytes, int need_count, cudaStream_t stream) {
  PushParams P;
  memset(&P, 0, sizeof P);
  P.table = table; P.capacity = capacity; P.n_acc = n_acc; P.rec_bytes = exchange_record_bytes(n_acc); P.key_kind = key_kind;
  P.world = world; P.rank = rank; P.step = step; P.need_count = need_count;
  P.region_bytes = region_bytes; P.cap_records = region_bytes / (unsigned long long)P.rec_bytes;
  if (P.cap_records == 0) fail(ARK_ERR_PROCESS, "exchange region smaller than one record");
  for (int i = 0; i < world; ++i) P.peers[i] = peers.p[i];
  const unsigned grid = (unsigned)std::max<unsigned long long>(1, (capacity + GX_THREADS * GX_SLOTS - 1) / (GX_THREADS * GX_SLOTS));
  KernelTimer t("exchange_push_kernel", stream);
  exchange_push_kernel<<<grid, GX_THREADS, 0, stream>>>(P);
}

void launch_exchange_merge(uint8_t* table, unsigned long long capacity, int n_acc, const int32_t* acc_kind, const uint8_t* comm,
                           int world, int rank, unsigned long long step, unsigned long long region_bytes, unsigned int* group_count,
                           int32_t* overflow, int32_t* status, unsigned long long* total, cudaStream_t stream) {
  MergeParams P;
  memset(&P, 0, sizeof P);
  P.table = table; P.mask = capacity - 1; P.rec_bytes = exchange_record_bytes(n_acc); P.n_acc = n_acc; P.world = world; P.rank = rank;
  for (int a = 0; a < n_acc; ++a) P.acc_kind[a] = acc_kind[a];
  P.step = step; P.region_bytes = region_bytes; P.comm = comm;
  P.group_count = group_count; P.overflow = overflow; P.status = status; P.total = total;
  KernelTimer t("exchange_merge_kernel", stream);
  exchange_merge_kernel<<<sm_count() * 4, GX_THREADS, 0, stream>>>(P);
}

void launch_exchange_ack(const GxPeers& peers, int world, int rank, unsigned long long step, cudaStream_t stream) {
  KernelTimer t("exchange_ack_kernel", stream);
  exchange_ack_kernel<<<1, 32, 0, stream>>>(peers, world, rank, step);
}

}  // namespace ark

// ---- C ABI: exchange contexts and the exchanged GROUP BY ------------------------------------------------------------
#include <unistd.h>

using namespace ark;

struct ark_dist {
  DistCtx ctx;
};

namespace {

constexpr uint32_t GX_MAGIC = 0x41524B58u;  // "ARKX"
struct GxHandle {  // what ark_dist_export hands to the peers
  uint32_t magic;
  int32_t pid, device, rank;
  uint64_t raw;          // the owner's own pointer (used when importer and owner share a process and a device)
  uint64_t comm_bytes;
  uint8_t ipc[64];
};

}  // namespace

extern "C" {

int ark_dist_create(int rank, int world, int64_t region_bytes, ark_dist_t** out) {
  return guarded([&] {
    if (!out) fail(ARK_ERR_PROCESS, "null output handle");
    *out = nullptr;
    if (world < 1 || world > GX_MAX_WORLD || rank < 0 || rank >= world) fail(ARK_ERR_CONFIG, "ark_dist_create: rank/world out of range (world <= 16)");
    if (region_bytes < 4096) fail(ARK_ERR_CONFIG, "ark_dist_create: region_bytes must be at least 4096");
    ensure_device();
    auto d = std::make_unique<ark_dist>();
    DistCtx& c = d->ctx;
    c.rank = rank; c.world = world;
    ARK_CUDA(cudaGetDevice(&c.device));
    c.region_bytes = (size_t)round_up(region_bytes, 256);
    c.comm_bytes = GX_HEADER_BYTES + 2 * (size_t)world * c.region_bytes;
    // a dedicated allocation (not a pool block): it is exported once and stays mapped in the peers for its whole life
    ARK_CUDA(cudaMalloc((void**)&c.comm, c.comm_bytes));
    ARK_CUDA(cudaMemset(c.comm, 0, GX_HEADER_BYTES));
    ARK_CUDA(cudaDeviceSynchronize());
    *out = d.release();
  });
}

int64_t ark_dist_handle_bytes(void) { return (int64_t)sizeof(GxHandle); }

int ark_dist_export(ark_dist_t* d, uint8_t* blob, int64_t blob_cap, int64_t* blob_size) {
  return guarded([&] {
    if (!d || !blob) fail(ARK_ERR_PROCESS, "null argument");
    if (blob_size) *blob_size = (int64_t)sizeof(GxHandle);
    if (blob_cap < (int64_t)sizeof(GxHandle)) fail(ARK_ERR_PROCESS, "ark_dist_export: handle buffer too small");
    GxHandle h;
    memset(&h, 0, sizeof h);
    h.magic = GX_MAGIC; h.pid = (int32_t)getpid(); h.device = d->ctx.device; h.rank = d->ctx.rank;
    h.raw = (uint64_t)(uintptr_t)d->ctx.comm; h.comm_bytes = d->ctx.comm_bytes;
    cudaIpcMemHandle_t ipc;
    const cudaError_t e = cudaIpcGetMemHandle(&ipc, d->ctx.comm);
    if (e == cudaSuccess) memcpy(h.ipc, &ipc, 64);
    else cudaGetLastError();  // same-process peers do not need it
    memcpy(blob, &h, sizeof h);
  });
}

int ark_dist_connect(ark_dist_t* d, const uint8_t* blobs, int64_t blob_stride) {
  return guarded([&] {
    if (!d || !blobs) fail(ARK_ERR_PROCESS, "null argument");
    DistCtx& c = d->ctx;
    if (c.connected) fail(ARK_ERR_PROCESS, "ark_dist_connect: already connected");
    if (blob_stride < (int64_t)sizeof(GxHandle)) fail(ARK_ERR_PROCESS, "ark_dist_connect: handle stride too small");
    ensure_device();
    for (int r = 0; r < c.world; ++r) {
      GxHandle h;
      memcpy(&h, blobs + (size_t)r * blob_stride, sizeof h);
      if (h.magic != GX_MAGIC || h.rank != r) fail(ARK_ERR_PROCESS, "ark_dist_connect: malformed handle for rank " + std::to_string(r));
      if (h.comm_bytes != c.comm_bytes) fail(ARK_ERR_CONFIG, "ark_dist_connect: rank " + std::to_string(r) + " was created with a different region size");
      if (r == c.rank) { c.peers.p[r] = c.comm; continue; }
      if (h.pid == (int32_t)getpid()) {
        if (h.device != c.device) {
          int can = 0;
          ARK_CUDA(cudaDeviceCanAccessPeer(&can, c.device, h.device));
          if (!can) fail(ARK_ERR_UNSUPPORTED, "ark_dist_connect: no peer access between devices " + std::to_string(c.device) + " and " + std::to_string(h.device));
          const cudaError_t e = cudaDeviceEnablePeerAccess(h.device, 0);
          if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) ARK_CUDA(e);
          cudaGetLastError();
        }
        c.peers.p[r] = (uint8_t*)(uintptr_t)h.raw;
      } else {
        cudaIpcMemHandle_t ipc;
        memcpy(&ipc, h.ipc, 64);
        void* base = nullptr;
        ARK_CUDA(cudaIpcOpenMemHandle(&base, ipc, cudaIpcMemLazyEnablePeerAccess));
        c.opened.push_back(base);
        c.peers.p[r] = (uint8_t*)base;
      }
    }
    c.connected = true;
  });
}

int ark_dist_stats(ark_dist_t* d, int64_t* out4) {
  return guarded([&] {
    if (!d || !out4) fail(ARK_ERR_PROCESS, "null argument");
    std::lock_guard<std::mutex> l(d->ctx.mu);
    out4[0] = (int64_t)d->ctx.step; out4[1] = (int64_t)d->ctx.last_recv_records; out4[2] = (int64_t)d->ctx.last_groups;
    out4[3] = (int64_t)d->ctx.region_bytes;
  });
}

void ark_dist_destroy(ark_dist_t* d) {
  if (!d) return;
  cudaDeviceSynchronize();
  for (void* b : d->ctx.opened) cudaIpcCloseMemHandle(b);
  if (d->ctx.comm) cudaFree(d->ctx.comm);
  cudaGetLastError();
  delete d;
}

int ark_sql_group_by_push_device(ark_proc_t* p, ark_dist_t* d, ArrowDeviceArray* in, ArrowSchema* in_schema) {
  BufferPtr in_owner = adopt_array(&in->array);
  return guarded([&] {
    SqlProcessor* sp = as_sql(p);
    if (!d || !d->ctx.connected) fail(ARK_ERR_PROCESS, "exchange context is not connected");
    ArrowDeviceArray view = device_view(*in, in_owner);
    DistCtx& c = d->ctx;
    std::lock_guard<std::mutex> l(c.mu);
    if (c.pushed) fail(ARK_ERR_PROCESS, "ark_sql_group_by_push_device: the previous step has not been merged");
    auto bound = sp->bind(in_schema);
    if (bound->plan->kind != Plan::Aggregate) fail(ARK_ERR_PROCESS, "not an aggregate query");
    refuse_limit_across_ranks(*bound->plan);
    StreamLease lease;
    Batch b = import_device(&view, in_schema, &bound->mask, in_owner, false, &bound->fields);
    if (!bound->plan->derived.empty()) b = append_json_columns(*bound->plan, b, lease.s);
    ++c.step;
    c.pushed = true;
    run_group_by_push(*bound->plan, b, c, lease.s);
  });
}

int ark_sql_group_by_merge_device(ark_proc_t* p, ark_dist_t* d, ArrowDeviceArray* out, ArrowSchema* out_schema) {
  return guarded([&] {
    zero_out(out, out_schema);
    SqlProcessor* sp = as_sql(p);
    if (!d || !d->ctx.connected) fail(ARK_ERR_PROCESS, "exchange context is not connected");
    DistCtx& c = d->ctx;
    std::lock_guard<std::mutex> l(c.mu);
    if (!c.pushed) fail(ARK_ERR_PROCESS, "ark_sql_group_by_merge_device: nothing was pushed for this step");
    auto plan = sp->last_aggregate_plan();
    if (!plan) fail(ARK_ERR_PROCESS, "final aggregate before any partial aggregate");
    refuse_limit_across_ranks(*plan);
    c.pushed = false;
    StreamLease lease;
    Batch r;
    if (!run_group_by_merge(*plan, c, r, lease.s))
      fail(ARK_ERR_UNSUPPORTED, "device-side exchange: a GROUP BY key longer than 12 bytes cannot travel inline (use the descriptor exchange)");
    export_device(r, out, out_schema, lease);
  });
}

int ark_sql_group_by_exchange_device(ark_proc_t* p, ark_dist_t* d, ArrowDeviceArray* in, ArrowSchema* in_schema, ArrowDeviceArray* out,
                                     ArrowSchema* out_schema) {
  const int rc = ark_sql_group_by_push_device(p, d, in, in_schema);
  if (rc != ARK_OK) return rc;
  return ark_sql_group_by_merge_device(p, d, out, out_schema);
}

}  // extern "C"
