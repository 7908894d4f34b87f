// string_funcs.cu — string-valued scalar functions of the `sql` processor and of expr::evaluate_expr.
//
// concat(a, b, …): datafusion-functions 47 `ConcatFunc` (third-party; reached from
// crates/arkflow-plugin/src/expr/mod.rs:92-122 — the reference's own test is `concat(name, ' is here')`,
// expr/mod.rs:148-166 — and from any SELECT list, processor/sql.rs:188-204).  NULL arguments count as
// empty strings and the result is never NULL.  Runs after the row kernels on the surviving rows:
// lengths → exclusive scan → one thread per row writes its parts.
#include <cub/device/device_scan.cuh>

#include "agg_acc.cuh"
#include "engine.h"
#include "stage_store.cuh"

namespace ark {

namespace {

constexpr int CONCAT_MAX_PARTS = 8;

enum : int32_t { PART_LITERAL = 0, PART_UTF8 = 1, PART_INT64 = 2, PART_BOOL = 3 };

struct ConcatPartView {
  const uint8_t* data;      // column bytes base / values / bit-packed booleans, or the literal's bytes
  const int32_t* offsets;   // Utf8 columns only
  const uint8_t* validity;
  int32_t validity_bit0;
  int32_t lit_len;
  int32_t kind;
  int32_t data_bit0;
};

struct ConcatParams {
  int32_t n_parts;
  int64_t n_rows;
  ConcatPartView parts[CONCAT_MAX_PARTS];
};

// decimal text of an i64, as arrow-cast / lexical write it; returns the length (≤ 20)
__device__ __forceinline__ int format_i64(long long v, uint8_t* out) {
  unsigned long long u = v < 0 ? 0ull - (unsigned long long)v : (unsigned long long)v;
  uint8_t rev[20];
  int n = 0;
  do { rev[n++] = (uint8_t)('0' + u % 10); u /= 10; } while (u);
  int k = 0;
  if (v < 0) out[k++] = '-';
  while (n) out[k++] = rev[--n];
  return k;
}

// bytes of part p for row r: *src points at them (literal / column bytes) or they are rendered into scratch
__device__ __forceinline__ int part_len(const ConcatPartView& p, int64_t r, const uint8_t** src, uint8_t* scratch) {
  if (p.kind == PART_LITERAL) { *src = p.data; return p.lit_len; }
  if (p.validity) { const int64_t b = r + p.validity_bit0; if (!((p.validity[b >> 3] >> (b & 7)) & 1)) return 0; }
  if (p.kind == PART_INT64) { *src = scratch; return format_i64(reinterpret_cast<const long long*>(p.data)[r], scratch); }
  if (p.kind == PART_BOOL) {
    const int64_t b = r + p.data_bit0;
    const bool t = (p.data[b >> 3] >> (b & 7)) & 1;
    const char* w = t ? "true" : "false";
    const int n = t ? 4 : 5;
    for (int i = 0; i < n; ++i) scratch[i] = (uint8_t)w[i];
    *src = scratch;
    return n;
  }
  const int32_t o0 = p.offsets[r];
  *src = p.data + o0;
  return p.offsets[r + 1] - o0;
}

// lens[r] = bytes of row r; *sum += all of them in 64 bits (the int32 scan of lens wraps silently past 2 GiB, and a
// literal repeated on every row can take the total past 2^32 back to a positive int32)
__global__ void concat_lengths_kernel(const __grid_constant__ ConcatParams P, int32_t* lens, unsigned long long* sum) {
  const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  int total = 0;
  if (r < P.n_rows) {
    const uint8_t* src;
    uint8_t scratch[24];
    for (int k = 0; k < P.n_parts; ++k) total += part_len(P.parts[k], r, &src, scratch);
    lens[r] = total;
  }
  const long long s = warp_sum_ll(total);
  if ((threadIdx.x & 31) == 0 && s) atomicAdd(sum, (unsigned long long)s);
}

__device__ __forceinline__ void concat_row(const ConcatParams& P, int64_t r, uint8_t* d) {
  uint8_t scratch[24];
  for (int k = 0; k < P.n_parts; ++k) {
    const uint8_t* src = nullptr;
    const int len = part_len(P.parts[k], r, &src, scratch);
    for (int i = 0; i < len; ++i) d[i] = src[i];
    d += len;
  }
}

// The rows of a CTA are contiguous in the output: build them in shared memory, store them 16 bytes at a time.
constexpr int CONCAT_THREADS = 256;
__global__ void __launch_bounds__(CONCAT_THREADS) concat_write_kernel(const __grid_constant__ ConcatParams P, const int32_t* out_offsets, uint8_t* out,
                                                                       int stage_bytes) {
  extern __shared__ __align__(16) uint8_t cc_stage[];
  const int64_t r0 = (int64_t)blockIdx.x * CONCAT_THREADS;
  const int rows = (int)((P.n_rows - r0) < CONCAT_THREADS ? (P.n_rows - r0) : CONCAT_THREADS);
  const int64_t r = r0 + threadIdx.x;
  const int32_t bb = out_offsets[r0];
  const int tb = out_offsets[r0 + rows] - bb;
  if (tb > stage_bytes - 16) {  // (tb + 16 would overflow near 2 GiB)
    if (r < P.n_rows) concat_row(P, r, out + out_offsets[r]);
    return;
  }
  const int mis = stage_misalignment(out + bb);
  if (r < P.n_rows) concat_row(P, r, cc_stage + mis + (out_offsets[r] - bb));
  __syncthreads();
  stage_store(out + bb, cc_stage, mis, tb, threadIdx.x, CONCAT_THREADS);
}

}  // namespace

// lengths → scan → bytes for one string column described by P; returns the offsets / bytes of the n_rows strings
static void render_strings(const ConcatParams& P, int64_t n, cudaStream_t stream, BufferPtr* out_offs, BufferPtr* out_bytes, int32_t* out_total) {
  // lens[n] = 0 closes the scan; the 64-bit total sits in the 8 bytes after it
  BufferPtr lens = device_alloc((size_t)(n + 1) * 4 + 16), offs = device_alloc((size_t)(n + 1) * 4);
  const int64_t sum_at = round_up((int64_t)(n + 1) * 4, 8);
  ARK_CUDA(cudaMemsetAsync((int32_t*)lens.get() + n, 0, (size_t)(sum_at + 8 - n * 4), stream));
  unsigned long long* sum = (unsigned long long*)((uint8_t*)lens.get() + sum_at);
  const unsigned grid = (unsigned)std::max<int64_t>(1, ceil_div(n, 256));
  if (n) { KernelTimer t("concat_lengths_kernel", stream); concat_lengths_kernel<<<grid, 256, 0, stream>>>(P, (int32_t*)lens.get(), sum); }
  size_t tb = 0;
  cub::DeviceScan::ExclusiveSum(nullptr, tb, (int32_t*)lens.get(), (int32_t*)offs.get(), (int)(n + 1), stream);
  BufferPtr tmp = device_alloc(tb + 16);
  note_launch("cub::DeviceScan::ExclusiveSum");
  cub::DeviceScan::ExclusiveSum(tmp.get(), tb, (int32_t*)lens.get(), (int32_t*)offs.get(), (int)(n + 1), stream);
  BufferPtr h = pinned_alloc(64);
  ARK_CUDA(cudaMemcpyAsync(h.get(), sum, 8, cudaMemcpyDeviceToHost, stream));
  ARK_CUDA(cudaStreamSynchronize(stream));
  const unsigned long long total64 = *(const unsigned long long*)h.get();
  if (total64 > 2147483647ull) fail(ARK_ERR_PROCESS, "Collection query results error: Arrow error: offset overflow, string result exceeds 2 GiB");
  const int32_t total = (int32_t)total64;  // = offs[n]: the scan did not wrap
  BufferPtr bytes = device_alloc((size_t)total + 16);
  if (n) {
    const int stage = (int)std::min<int64_t>(44 * 1024, round_up((int64_t)((double)total / (double)n * CONCAT_THREADS * 1.5) + 256, 1024));
    KernelTimer t("concat_write_kernel", stream);
    concat_write_kernel<<<grid, CONCAT_THREADS, stage, stream>>>(P, (const int32_t*)offs.get(), (uint8_t*)bytes.get(), stage);
  }
  ARK_CUDA(cudaGetLastError());
  *out_offs = offs; *out_bytes = bytes; *out_total = total;
}

// CAST(<Int64 column> AS STRING) of an already materialised column (aggregate results): decimal text, NULL stays NULL
Column format_int64_column(const Column& src, const std::string& name, cudaStream_t stream) {
  ConcatParams P;
  memset(&P, 0, sizeof P);
  P.n_parts = 1; P.n_rows = src.length;
  P.parts[0].data = src.data; P.parts[0].validity = src.validity; P.parts[0].validity_bit0 = (int32_t)src.validity_bit0; P.parts[0].kind = PART_INT64;
  BufferPtr offs, bytes;
  int32_t total = 0;
  render_strings(P, src.length, stream, &offs, &bytes, &total);
  Column c;
  c.field.name = name; c.field.type = DType::Utf8; c.field.nullable = src.field.nullable; c.length = src.length;
  c.offsets = (const int32_t*)offs.get(); c.data = (const uint8_t*)bytes.get(); c.data_bytes = total; c.first_offset = 0;
  c.validity = src.validity; c.validity_bit0 = src.validity_bit0; c.null_count = src.null_count;
  c.owners = {offs, bytes};
  for (auto& o : src.owners) c.owners.push_back(o);
  return c;
}

// Builds the result of a FilterProject plan that holds concat() items: `r` carries plan.outputs (visible
// columns first, hidden concat sources after them).
Batch apply_concats(const Plan& plan, Batch& r, cudaStream_t stream) {
  const int64_t n = r.num_rows;
  std::vector<Column> made(plan.concats.size());
  for (size_t ci = 0; ci < plan.concats.size(); ++ci) {
    const ConcatItem& item = plan.concats[ci];
    if ((int)item.parts.size() > CONCAT_MAX_PARTS) fail(ARK_ERR_UNSUPPORTED, "concat() with more than 8 arguments");
    ConcatParams P;
    memset(&P, 0, sizeof P);
    P.n_parts = (int)item.parts.size();
    P.n_rows = n;
    size_t lit_bytes = 0;
    for (auto& part : item.parts) if (part.is_literal) lit_bytes += part.literal.size();
    BufferPtr lit_host = pinned_alloc(lit_bytes + 16), lit_dev = device_alloc(lit_bytes + 16);
    size_t pos = 0;
    for (size_t k = 0; k < item.parts.size(); ++k) {
      const ConcatPart& part = item.parts[k];
      ConcatPartView& v = P.parts[k];
      if (part.is_literal) {
        memcpy((char*)lit_host.get() + pos, part.literal.data(), part.literal.size());
        v.data = (const uint8_t*)lit_dev.get() + pos; v.offsets = nullptr; v.lit_len = (int32_t)part.literal.size();
        v.kind = PART_LITERAL;
        pos += part.literal.size();
      } else {
        const Column& c = r.cols[part.out_index];
        v.data = c.data; v.offsets = c.offsets; v.validity = c.validity; v.validity_bit0 = (int32_t)c.validity_bit0;
        v.data_bit0 = (int32_t)c.data_bit0;
        v.kind = part.col_type == DType::Int64 ? PART_INT64 : part.col_type == DType::Bool ? PART_BOOL : PART_UTF8;
      }
    }
    if (lit_bytes) ARK_CUDA(cudaMemcpyAsync(lit_dev.get(), lit_host.get(), lit_bytes, cudaMemcpyHostToDevice, stream));
    BufferPtr offs, bytes;
    int32_t total = 0;
    render_strings(P, n, stream, &offs, &bytes, &total);
    ARK_CUDA(cudaStreamSynchronize(stream));  // the literal staging blocks go back to the pool
    Column& c = made[ci];
    c.field.name = item.name; c.field.type = DType::Utf8; c.field.nullable = true; c.length = n;
    c.offsets = (const int32_t*)offs.get(); c.data = (const uint8_t*)bytes.get(); c.data_bytes = total; c.first_offset = 0;
    c.validity = nullptr; c.null_count = 0;
    c.owners = {offs, bytes};
    if (item.is_cast && !item.parts.empty() && !item.parts[0].is_literal) {  // CAST: NULL in ⇒ NULL out — the source's bitmap is the result's
      const Column& src = r.cols[item.parts[0].out_index];
      c.field.nullable = src.field.nullable;
      if (src.validity) {
        c.validity = src.validity; c.validity_bit0 = src.validity_bit0; c.null_count = src.null_count;
        for (auto& o : src.owners) c.owners.push_back(o);
      }
    }
  }
  Batch out;
  out.num_rows = n;
  out.input_name = r.input_name;
  for (auto& fi : plan.final_items) out.cols.push_back(fi.is_concat ? made[fi.index] : r.cols[fi.index]);
  return out;
}

}  // namespace ark
