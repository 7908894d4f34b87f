// decoded.cu — decoder columns staged, settled and built into Arrow columns (decoded.h).
#include <algorithm>

#include "bitmap.h"
#include "decoded.h"
#include "varlen.h"

namespace ark {

StagedColumn stage_column(DType type, int64_t rows, bool nullable, bool wants_raw, cudaStream_t stream) {
  StagedColumn s;
  s.type = type; s.rows = rows;
  const size_t r = (size_t)std::max<int64_t>(rows, 1);
  const bool str = type == DType::Utf8 || type == DType::Binary;
  if (nullable) s.valid = device_alloc(r);
  if (str) {
    s.len = device_alloc((size_t)(rows + 1) * 4);
    ARK_CUDA(cudaMemsetAsync((int32_t*)s.len.get() + rows, 0, 4, stream));  // the scan reads rows + 1 entries
  }
  if (str || type == DType::List || type == DType::Struct) {
    s.src = device_alloc(r * 8);
    if (wants_raw) s.raw = device_alloc(r * 4);
  } else if (type == DType::Bool || fixed_width(type)) {
    s.values = device_alloc(r * (type == DType::Bool ? 1 : fixed_width(type)));
  }
  return s;
}

void settle_columns(std::vector<StagedColumn>& cols, const void* err, size_t err_bytes,
                    const std::function<void(const void*)>& check, cudaStream_t stream) {
  const size_t nc = cols.size();
  BufferPtr h = pinned_alloc(16 + 12 * nc), zeros = device_alloc(8 * nc + 8);  // h: error word, null counts, totals
  unsigned long long* nulls = (unsigned long long*)((char*)h.get() + 16);
  int32_t* totals = (int32_t*)(nulls + nc);
  if (std::any_of(cols.begin(), cols.end(), [](const StagedColumn& s) { return s.len && s.bound > INT32_MAX; })) {
    if (err) {
      ARK_CUDA(cudaMemcpyAsync(h.get(), err, err_bytes, cudaMemcpyDeviceToHost, stream));
      ARK_CUDA(cudaStreamSynchronize(stream));
      check(h.get());
    }
    for (auto& s : cols)
      if (s.len) varlen_guard((const int32_t*)s.len.get(), s.rows, s.bound, s.what, stream);
  }
  ARK_CUDA(cudaMemsetAsync(zeros.get(), 0, 8 * nc + 8, stream));
  bool reads = err != nullptr;
  for (size_t k = 0; k < nc; ++k) {
    StagedColumn& s = cols[k];
    if (s.len) {
      s.offsets = varlen_scan((const int32_t*)s.len.get(), s.rows, stream);
      ARK_CUDA(cudaMemcpyAsync(totals + k, (const int32_t*)s.offsets.get() + s.rows, 4, cudaMemcpyDeviceToHost, stream));
      reads = true;
    }
    if (s.valid && s.type != DType::Null && s.rows > 0) {
      s.bits = pack_bits((const uint8_t*)s.valid.get(), s.rows, (unsigned long long*)zeros.get() + k, stream);
      reads = true;
    }
  }
  if (!reads) return;
  ARK_CUDA(cudaMemcpyAsync(nulls, zeros.get(), 8 * nc, cudaMemcpyDeviceToHost, stream));
  if (err) ARK_CUDA(cudaMemcpyAsync(h.get(), err, err_bytes, cudaMemcpyDeviceToHost, stream));
  ARK_CUDA(cudaStreamSynchronize(stream));
  if (err) check(h.get());
  for (size_t k = 0; k < nc; ++k) {
    if (cols[k].offsets) cols[k].total = totals[k];
    cols[k].null_count = (int64_t)nulls[k];
  }
}

Column finish_column(const StagedColumn& s, Field f, const std::function<void(const StagedColumn&, uint8_t*)>& copy_bytes,
                     cudaStream_t stream) {
  Column c;
  c.field = std::move(f);
  c.length = s.rows;
  if (s.offsets) {
    BufferPtr bytes = device_alloc((size_t)s.total + 16);
    copy_bytes(s, (uint8_t*)bytes.get());
    set_varlen(c, {s.offsets, bytes, s.total});
  } else if (s.type == DType::Bool) {
    set_bool_values(c, s.values, s.rows, stream);
  } else if (s.values) {
    c.data = (const uint8_t*)s.values.get(); c.data_bytes = s.rows * fixed_width(s.type); c.owners = {s.values};
  }
  if (s.bits) set_validity(c, s.bits, s.null_count);
  return c;
}

}  // namespace ark
