// concat.cu — concat_batches on the device: one segmented-copy launch for every data buffer of every
// column, one offset-rebase launch per var-len column, one bit-gather launch per nullable column.
//
// Stands in for arrow::compute::concat_batches at the reference's call sites
// (buffer/memory.rs:130, buffer/window.rs:131,159, processor/sql.rs:146, component/json.rs:54).
// Algorithmic traffic: every byte of every input buffer read once and written once
// (SURVEY.md §8(d) config 5: 2 × 32 B/row for decoded S, 134 B/msg for raw Binary payloads).
#include <algorithm>

#include "abi.h"
#include "bitmap.cuh"

namespace ark {

namespace {

struct CopySpan {
  const uint8_t* src;
  uint8_t* dst;
  unsigned long long bytes;
  unsigned long long chunk0;  // index of this span's first chunk in the global chunk space
};

constexpr unsigned long long CONCAT_CHUNK = 64 * 1024;  // bytes per CTA work item
constexpr int CONCAT_THREADS = 256;

// copy [src, src+n) → [dst, dst+n) with the widest access the mutual alignment allows
__device__ void copy_span(uint8_t* dst, const uint8_t* src, unsigned long long n, int tid, int nthreads) {
  const uintptr_t a = reinterpret_cast<uintptr_t>(src), b = reinterpret_cast<uintptr_t>(dst);
  if (((a ^ b) & 15) == 0) {
    unsigned long long head = (16 - (a & 15)) & 15;
    if (head > n) head = n;
    for (unsigned long long i = tid; i < head; i += nthreads) dst[i] = src[i];
    const unsigned long long body = (n - head) / 16;
    const uint4* s4 = reinterpret_cast<const uint4*>(src + head);
    uint4* d4 = reinterpret_cast<uint4*>(dst + head);
    for (unsigned long long i = tid; i < body; i += nthreads) d4[i] = s4[i];
    for (unsigned long long i = head + body * 16 + tid; i < n; i += nthreads) dst[i] = src[i];
  } else if (((a ^ b) & 7) == 0) {
    unsigned long long head = (8 - (a & 7)) & 7;
    if (head > n) head = n;
    for (unsigned long long i = tid; i < head; i += nthreads) dst[i] = src[i];
    const unsigned long long body = (n - head) / 8;
    const unsigned long long* s8 = reinterpret_cast<const unsigned long long*>(src + head);
    unsigned long long* d8 = reinterpret_cast<unsigned long long*>(dst + head);
    for (unsigned long long i = tid; i < body; i += nthreads) d8[i] = s8[i];
    for (unsigned long long i = head + body * 8 + tid; i < n; i += nthreads) dst[i] = src[i];
  } else if (((a ^ b) & 3) == 0) {
    unsigned long long head = (4 - (a & 3)) & 3;
    if (head > n) head = n;
    for (unsigned long long i = tid; i < head; i += nthreads) dst[i] = src[i];
    const unsigned long long body = (n - head) / 4;
    const unsigned* s4 = reinterpret_cast<const unsigned*>(src + head);
    unsigned* d4 = reinterpret_cast<unsigned*>(dst + head);
    for (unsigned long long i = tid; i < body; i += nthreads) d4[i] = s4[i];
    for (unsigned long long i = head + body * 4 + tid; i < n; i += nthreads) dst[i] = src[i];
  } else {
    for (unsigned long long i = tid; i < n; i += nthreads) dst[i] = src[i];
  }
}

__global__ void __launch_bounds__(CONCAT_THREADS) concat_copy_kernel(const CopySpan* spans, int n_spans, unsigned long long n_chunks) {
  for (unsigned long long chunk = blockIdx.x; chunk < n_chunks; chunk += gridDim.x) {
    int lo = 0, hi = n_spans - 1;  // last span with chunk0 <= chunk
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (spans[mid].chunk0 <= chunk) lo = mid; else hi = mid - 1;
    }
    const CopySpan s = spans[lo];
    const unsigned long long off = (chunk - s.chunk0) * CONCAT_CHUNK;
    if (off >= s.bytes) continue;
    const unsigned long long n = s.bytes - off < CONCAT_CHUNK ? s.bytes - off : CONCAT_CHUNK;
    copy_span(s.dst + off, s.src + off, n, threadIdx.x, CONCAT_THREADS);
  }
}

struct OffsetSeg {
  const int32_t* offsets;  // element 0 of the segment
  long long row0;          // first output row of the segment
  long long byte_base;     // output byte position of the segment's first value
  int first;               // offsets[0] of the segment
};

__global__ void concat_offsets_kernel(const OffsetSeg* segs, int n_segs, long long total_rows, long long total_bytes, int32_t* out) {
  const long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (r > total_rows) return;
  if (r == total_rows) { out[r] = (int32_t)total_bytes; return; }
  int lo = 0, hi = n_segs - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (segs[mid].row0 <= r) lo = mid; else hi = mid - 1;
  }
  const OffsetSeg s = segs[lo];
  out[r] = (int32_t)((long long)s.offsets[r - s.row0] - s.first + s.byte_base);
}

struct BitSeg {
  const uint8_t* bits;  // nullptr ⇒ all ones
  long long row0;
  int bit0;
};

// `zeros` (may be null): incremented by the number of clear bits gathered, i.e. the NULLs of a validity bitmap
__global__ void concat_bits_kernel(const BitSeg* segs, int n_segs, long long total_rows, uint8_t* out, unsigned long long* zeros) {
  const long long ob = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (ob >= (total_rows + 7) / 8) return;
  unsigned v = 0;
  long long r = ob * 8;
  int lo = 0, hi = n_segs - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (segs[mid].row0 <= r) lo = mid; else hi = mid - 1;
  }
  int seg = lo, i = 0;
  for (; i < 8 && r < total_rows; ++i, ++r) {
    while (seg + 1 < n_segs && segs[seg + 1].row0 <= r) ++seg;
    const BitSeg s = segs[seg];
    const long long p = r - s.row0 + s.bit0;
    const unsigned bit = s.bits ? bit_get(s.bits, p) : 1u;
    v |= bit << i;
  }
  out[ob] = (uint8_t)v;
  if (zeros && i != __popc(v)) atomicAdd(zeros, (unsigned long long)(i - __popc(v)));
}

}  // namespace

// Concatenates batches that already live in HBM.  Var-len extents must be resolved.
Batch concat_device(std::vector<Batch>& ins, cudaStream_t stream) {
  if (ins.empty()) fail(ARK_ERR_PROCESS, "Merge batches failed: no batches");
  const size_t ncol = ins[0].cols.size();
  for (size_t b = 1; b < ins.size(); ++b) {
    if (ins[b].cols.size() != ncol) fail(ARK_ERR_PROCESS, "Merge batches failed: Invalid argument error: batches have different column counts");
    for (size_t c = 0; c < ncol; ++c) {
      if (ins[b].cols[c].field.type != ins[0].cols[c].field.type || ins[b].cols[c].field.format != ins[0].cols[c].field.format)
        fail(ARK_ERR_PROCESS, "Merge batches failed: Invalid argument error: column types must match schema types, expected " +
                                  std::string(dtype_name(ins[0].cols[c].field.type)) + " but found " +
                                  dtype_name(ins[b].cols[c].field.type) + " at column index " + std::to_string(c));
    }
  }
  // A Null column is a length without buffers: the import marks it not present, as it does every type it holds no
  // buffers for, so it is told apart by its format.
  auto null_column = [](const Column& c) { return c.field.type == DType::Null && (c.present || c.field.format == "n"); };
  for (size_t c = 0; c < ncol; ++c) {
    const Column& c0 = ins[0].cols[c];
    const DType t = c0.field.type;
    if (null_column(c0)) continue;
    if (!c0.present || (!fixed_width(t) && t != DType::Bool && t != DType::Utf8 && t != DType::Binary))
      fail(ARK_ERR_UNSUPPORTED, "concat of a column with Arrow type '" + (c0.field.format.empty() ? std::string(dtype_arrow_format(t)) : c0.field.format) + "'");
  }
  // RecordBatch::try_new: a field the schema batch declares non-nullable may hold no NULL.  A known null count settles
  // it here; members whose count is unknown (-1) are counted by concat_bits_kernel, which the one-batch return skips.
  std::vector<char> count_nulls(ncol, 0);
  bool any_count = false;
  auto non_nullable = [&](size_t c) {
    fail(ARK_ERR_PROCESS, "Merge batches failed: Invalid argument error: Column '" + ins[0].cols[c].field.name +
                              "' is declared as non-nullable but contains null values");
  };
  for (size_t c = 0; c < ncol; ++c) {
    if (ins[0].cols[c].field.nullable) continue;
    for (auto& b : ins) {
      const Column& m = b.cols[c];
      if (!m.validity || b.num_rows == 0) continue;
      if (m.null_count > 0) non_nullable(c);
      if (m.null_count < 0) count_nulls[c] = any_count = true;
    }
  }
  {
    std::vector<Column*> all;  // one round trip for the extents of every batch
    for (auto& b : ins) for (auto& c : b.cols) all.push_back(&c);
    resolve_varlen_extents_many(all, stream);
  }
  if (ins.size() == 1 && !any_count) return ins[0];
  int64_t total_rows = 0;
  std::vector<int64_t> row0(ins.size());
  for (size_t b = 0; b < ins.size(); ++b) { row0[b] = total_rows; total_rows += ins[b].num_rows; }

  Batch out;
  out.num_rows = total_rows;
  out.input_name = ins[0].input_name;
  std::vector<CopySpan> spans;
  std::vector<BufferPtr> keep;
  struct PendingOffsets { std::vector<OffsetSeg> segs; int32_t* out; int64_t total_bytes; };
  struct PendingBits { std::vector<BitSeg> segs; uint8_t* out; int counter; };  // counter: slot in `zeros`, or -1
  std::vector<PendingOffsets> poffs;
  std::vector<PendingBits> pbits;
  std::vector<size_t> counted;  // column of each `zeros` slot
  auto add_span = [&](const uint8_t* src, uint8_t* dst, int64_t bytes) {
    if (bytes > 0) spans.push_back({src, dst, (unsigned long long)bytes, 0});
  };
  for (size_t c = 0; c < ncol; ++c) {
    const Column& c0 = ins[0].cols[c];
    Column oc;
    oc.field = c0.field; oc.length = total_rows;
    if (null_column(c0)) { out.cols.push_back(std::move(oc)); continue; }
    bool any_null = false;
    for (auto& b : ins) any_null = any_null || (b.cols[c].validity != nullptr);
    switch (c0.field.type) {
      case DType::Int64: case DType::Float64:
      case DType::Int32: case DType::UInt32: case DType::UInt64: case DType::Float32: {
        const int w = fixed_width(c0.field.type);
        BufferPtr d = device_alloc((size_t)total_rows * w + 16);
        for (size_t b = 0; b < ins.size(); ++b) add_span(ins[b].cols[c].data, (uint8_t*)d.get() + row0[b] * w, ins[b].num_rows * w);
        oc.data = (const uint8_t*)d.get(); oc.data_bytes = total_rows * w; oc.owners.push_back(d);
        break;
      }
      case DType::Bool: {
        BufferPtr d = device_alloc((size_t)(total_rows + 7) / 8 + 16);
        PendingBits pb; pb.out = (uint8_t*)d.get(); pb.counter = -1;
        for (size_t b = 0; b < ins.size(); ++b) if (ins[b].num_rows) pb.segs.push_back({ins[b].cols[c].data, row0[b], ins[b].cols[c].data_bit0});
        pbits.push_back(std::move(pb));
        oc.data = (const uint8_t*)d.get(); oc.data_bit0 = 0; oc.data_bytes = (total_rows + 7) / 8; oc.owners.push_back(d);
        break;
      }
      case DType::Utf8: case DType::Binary: {
        int64_t total_bytes = 0;
        for (auto& b : ins) total_bytes += std::max<int64_t>(b.cols[c].data_bytes, 0);
        if (total_bytes > 2147483647ll)
          fail(ARK_ERR_PROCESS, "Merge batches failed: Invalid argument error: offset overflow, concatenated Utf8 column exceeds 2 GiB");
        BufferPtr o = device_alloc((size_t)(total_rows + 1) * 4 + 16), d = device_alloc((size_t)total_bytes + 16);
        PendingOffsets po; po.out = (int32_t*)o.get(); po.total_bytes = total_bytes;
        int64_t byte_base = 0;
        for (size_t b = 0; b < ins.size(); ++b) {
          const Column& sc = ins[b].cols[c];
          if (ins[b].num_rows == 0) continue;
          po.segs.push_back({sc.offsets, row0[b], byte_base, (int)sc.first_offset});
          add_span(sc.data + sc.first_offset, (uint8_t*)d.get() + byte_base, sc.data_bytes);
          byte_base += sc.data_bytes;
        }
        poffs.push_back(std::move(po));
        oc.offsets = (const int32_t*)o.get(); oc.data = (const uint8_t*)d.get(); oc.data_bytes = total_bytes; oc.first_offset = 0;
        oc.owners = {o, d};
        break;
      }
      default: break;  // not reached: the types checked above
    }
    if (any_null && total_rows > 0) {
      BufferPtr v = device_alloc((size_t)(total_rows + 7) / 8 + 16);
      PendingBits pb; pb.out = (uint8_t*)v.get(); pb.counter = -1;
      for (size_t b = 0; b < ins.size(); ++b) if (ins[b].num_rows) pb.segs.push_back({ins[b].cols[c].validity, row0[b], ins[b].cols[c].validity_bit0});
      if (count_nulls[c]) { pb.counter = (int)counted.size(); counted.push_back(c); }
      pbits.push_back(std::move(pb));
      oc.validity = (const uint8_t*)v.get(); oc.validity_bit0 = 0; oc.null_count = -1; oc.owners.push_back(v);
    }
    out.cols.push_back(std::move(oc));
  }
  // one upload for all descriptors
  unsigned long long n_chunks = 0;
  for (auto& s : spans) { s.chunk0 = n_chunks; n_chunks += (s.bytes + CONCAT_CHUNK - 1) / CONCAT_CHUNK; }
  size_t desc_bytes = spans.size() * sizeof(CopySpan);
  for (auto& p : poffs) desc_bytes += p.segs.size() * sizeof(OffsetSeg);
  for (auto& p : pbits) desc_bytes += p.segs.size() * sizeof(BitSeg);
  desc_bytes += counted.size() * sizeof(unsigned long long);
  BufferPtr hdesc = pinned_alloc(desc_bytes + 64), ddesc = device_alloc(desc_bytes + 64);
  size_t pos = 0;
  auto put = [&](const void* src, size_t n) -> const void* {
    memcpy((char*)hdesc.get() + pos, src, n);
    const void* dptr = (char*)ddesc.get() + pos;
    pos += n;
    return dptr;
  };
  // the NULL counters go first: 8-byte aligned, and uploaded as zeros with the descriptors
  const std::vector<unsigned long long> zero_counts(counted.size(), 0);
  unsigned long long* d_zeros = (unsigned long long*)put(zero_counts.data(), zero_counts.size() * sizeof(unsigned long long));
  const unsigned long long* h_zeros = (const unsigned long long*)hdesc.get();
  const CopySpan* d_spans = (const CopySpan*)put(spans.data(), spans.size() * sizeof(CopySpan));
  std::vector<const OffsetSeg*> d_offs;
  std::vector<const BitSeg*> d_bits;
  for (auto& p : poffs) d_offs.push_back((const OffsetSeg*)put(p.segs.data(), p.segs.size() * sizeof(OffsetSeg)));
  for (auto& p : pbits) d_bits.push_back((const BitSeg*)put(p.segs.data(), p.segs.size() * sizeof(BitSeg)));
  if (pos) ARK_CUDA(cudaMemcpyAsync(ddesc.get(), hdesc.get(), pos, cudaMemcpyHostToDevice, stream));
  if (n_chunks) {
    KernelTimer t("concat_copy_kernel", stream);
    const unsigned grid = (unsigned)std::min<unsigned long long>(n_chunks, 148ull * 16);
    concat_copy_kernel<<<grid, CONCAT_THREADS, 0, stream>>>(d_spans, (int)spans.size(), n_chunks);
  }
  for (size_t i = 0; i < poffs.size(); ++i) {
    if (poffs[i].segs.empty()) { ARK_CUDA(cudaMemsetAsync(poffs[i].out, 0, 4, stream)); continue; }
    KernelTimer t("concat_offsets_kernel", stream);
    concat_offsets_kernel<<<(unsigned)ceil_div(total_rows + 1, 256), 256, 0, stream>>>(d_offs[i], (int)poffs[i].segs.size(), total_rows,
                                                                                       poffs[i].total_bytes, poffs[i].out);
  }
  for (size_t i = 0; i < pbits.size(); ++i) {
    if (pbits[i].segs.empty()) continue;
    KernelTimer t("concat_bits_kernel", stream);
    concat_bits_kernel<<<(unsigned)ceil_div((total_rows + 7) / 8, 256), 256, 0, stream>>>(d_bits[i], (int)pbits[i].segs.size(), total_rows, pbits[i].out,
                                                                                       pbits[i].counter < 0 ? nullptr : d_zeros + pbits[i].counter);
  }
  ARK_CUDA(cudaGetLastError());
  if (!counted.empty())
    ARK_CUDA(cudaMemcpyAsync((void*)h_zeros, d_zeros, counted.size() * sizeof(unsigned long long), cudaMemcpyDeviceToHost, stream));
  ARK_CUDA(cudaStreamSynchronize(stream));  // descriptors live in pooled blocks: finish before they are recycled
  for (size_t k = 0; k < counted.size(); ++k) {
    if (h_zeros[k]) non_nullable(counted[k]);
    out.cols[counted[k]].null_count = 0;
  }
  return out;
}

}  // namespace ark

using namespace ark;

extern "C" int ark_concat_batches(int n, ArrowArray* ins, ArrowSchema* in_schemas, ArrowArray* out, ArrowSchema* out_schema) {
  std::vector<BufferPtr> owners;
  for (int i = 0; i < n; ++i) owners.push_back(adopt_array(&ins[i]));
  return guarded([&] {
    zero_out(out, out_schema);
    if (n <= 0) fail(ARK_ERR_PROCESS, "Merge batches failed: no batches");
    StreamLease lease;
    std::vector<Batch> bs;
    for (int i = 0; i < n; ++i) bs.push_back(import_host(adopted(owners[i]), &in_schemas[i], nullptr, lease.s, nullptr, true));
    Batch r = concat_device(bs, lease.s);
    export_host(r, lease.s, out, out_schema);
  });
}

extern "C" int ark_concat_batches_device(int n, ArrowDeviceArray* ins, ArrowSchema* in_schemas, ArrowDeviceArray* out, ArrowSchema* out_schema) {
  std::vector<BufferPtr> owners;
  for (int i = 0; i < n; ++i) owners.push_back(adopt_array(&ins[i].array));
  return guarded([&] {
    zero_out(out, out_schema);
    if (n <= 0) fail(ARK_ERR_PROCESS, "Merge batches failed: no batches");
    StreamLease lease;
    std::vector<Batch> bs;
    for (int i = 0; i < n; ++i) {
      ArrowDeviceArray view = device_view(ins[i], owners[i]);
      bs.push_back(import_device(&view, &in_schemas[i], nullptr, owners[i], true));
    }
    Batch r = concat_device(bs, lease.s);
    export_device(r, out, out_schema, lease);
  });
}
