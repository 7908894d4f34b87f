// varlen.cu — int32 offsets and bytes of Binary / Utf8 columns built from per-row lengths, and their 2 GiB guard
// (varlen.h).
#include <cub/device/device_scan.cuh>

#include <algorithm>

#include "varlen.h"

namespace ark {

namespace {

// string / bytes column bytes: thread per row, from the payload column or from the default blob
__global__ void protobuf_strings_kernel(const uint8_t* data, const uint8_t* dflt, const long long* src, const int32_t* offsets,
                                        int64_t n_rows, uint8_t* out) {
  const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n_rows) return;
  const int len = offsets[r + 1] - offsets[r];
  if (len == 0) return;
  const long long s = src[r];
  const uint8_t* from = s >= 0 ? data + s : dflt + (-1 - s);
  uint8_t* d = out + offsets[r];
  for (int k = 0; k < len; ++k) d[k] = from[k];
}

// Sum of n non-negative int32 lengths, accumulated in 64 bits.
__global__ void protobuf_sum64_kernel(const int32_t* lens, int64_t n, unsigned long long* total) {
  long long acc = 0;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    acc += lens[i] >= 0 ? lens[i] : (1ll << 40);  // a negative length is a row that itself passed 2^31
  for (int o = 16; o; o >>= 1) acc += __shfl_down_sync(0xffffffffu, acc, o);
  if ((threadIdx.x & 31) == 0) atomicAdd(total, (unsigned long long)acc);
}

}  // namespace

BufferPtr varlen_scan(const int32_t* lens, int64_t n, cudaStream_t stream) {
  BufferPtr offs = device_alloc((size_t)(n + 1) * 4);
  size_t tb = 0;
  cub::DeviceScan::ExclusiveSum(nullptr, tb, lens, (int32_t*)offs.get(), (int)(n + 1), stream);
  BufferPtr tmp = device_alloc(tb + 16);
  note_launch("cub::DeviceScan::ExclusiveSum");
  cub::DeviceScan::ExclusiveSum(tmp.get(), tb, lens, (int32_t*)offs.get(), (int)(n + 1), stream);
  return offs;
}

int32_t varlen_guard(unsigned long long total, const std::string& msg) {
  if (total > (unsigned long long)INT32_MAX) fail(ARK_ERR_PROCESS, msg);
  return (int32_t)total;
}

void varlen_guard(const int32_t* lens, int64_t n, int64_t bound, const std::string& what, cudaStream_t stream) {
  if (bound >= 0 && bound <= INT32_MAX) return;
  BufferPtr d = device_alloc(8), h = pinned_alloc(8);
  ARK_CUDA(cudaMemsetAsync(d.get(), 0, 8, stream));
  if (n > 0) {
    KernelTimer t("protobuf_sum64_kernel", stream);
    protobuf_sum64_kernel<<<(unsigned)std::min<int64_t>(ceil_div(n, 256), 8 * sm_count()), 256, 0, stream>>>(lens, n, (unsigned long long*)d.get());
  }
  ARK_CUDA(cudaMemcpyAsync(h.get(), d.get(), 8, cudaMemcpyDeviceToHost, stream));
  ARK_CUDA(cudaStreamSynchronize(stream));
  const unsigned long long total = *(const unsigned long long*)h.get();
  if (total > (unsigned long long)INT32_MAX) fail(ARK_ERR_PROCESS, what + " holds " + std::to_string(total) + " bytes: more than a Binary / Utf8 column's 2 GiB");
}

Varlen varlen_layout(const int32_t* lens, int64_t n, const unsigned long long* exact, int64_t bound, const std::string& what,
                     cudaStream_t stream) {
  if (!exact) varlen_guard(lens, n, bound, what, stream);
  Varlen v;
  v.offsets = varlen_scan(lens, n, stream);
  BufferPtr h = pinned_alloc(8);
  if (exact) ARK_CUDA(cudaMemcpyAsync(h.get(), exact, 8, cudaMemcpyDeviceToHost, stream));
  else ARK_CUDA(cudaMemcpyAsync(h.get(), (const int32_t*)v.offsets.get() + n, 4, cudaMemcpyDeviceToHost, stream));
  ARK_CUDA(cudaStreamSynchronize(stream));
  v.total = exact ? varlen_guard(*(const unsigned long long*)h.get(), what) : *(const int32_t*)h.get();
  v.bytes = device_alloc((size_t)v.total + 16);
  return v;
}

void set_varlen(Column& c, const Varlen& v) {
  c.offsets = (const int32_t*)v.offsets.get(); c.data = (const uint8_t*)v.bytes.get(); c.data_bytes = v.total; c.first_offset = 0;
  c.owners = {v.offsets, v.bytes};
}

void launch_span_copy(const uint8_t* data, const uint8_t* dflt, const long long* src, const int32_t* offsets, int64_t n_rows,
                      uint8_t* out, cudaStream_t stream) {
  if (n_rows == 0) return;
  KernelTimer t("protobuf_strings_kernel", stream);
  protobuf_strings_kernel<<<(unsigned)ceil_div(n_rows, 256), 256, 0, stream>>>(data, dflt, src, offsets, n_rows, out);
}

}  // namespace ark
