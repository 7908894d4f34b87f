// synth.cu — synthetic batches of schema S generated directly in HBM (bench/test support).
// Twin of oracle/synth.py (same splitmix64 counter RNG), so host and device inputs are identical.
// Schema S: examples/generate_example.yaml:6 and examples/stream_data.json:1-21 of the reference.
#include "abi.h"

namespace ark {

namespace {

__device__ __forceinline__ uint64_t splitmix64_at(uint64_t seed, uint64_t idx) {
  uint64_t z = seed + (idx + 1) * 0x9E3779B97F4A7C15ull;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}

__global__ void synth_kernel(int64_t n, int64_t row0, uint64_t seed, int value_kind, uint64_t key_space,
                             int64_t* ts, uint64_t* value, int32_t* offsets, uint32_t* sensor_words) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i > n) return;
  if (i == n) { offsets[n] = (int32_t)(n * 12); return; }
  const uint64_t g = (uint64_t)(row0 + i);
  ts[i] = 1625000000000ll + 1000ll * (int64_t)g;
  const uint64_t rv = splitmix64_at(seed, g);
  if (value_kind == 0) value[i] = rv % 20ull;
  else {
    double d = (double)(rv >> 11) * (20.0 * 1.1102230246251565e-16);  // 20 * 2^-53
    value[i] = (uint64_t)__double_as_longlong(d);
  }
  uint64_t k = splitmix64_at(seed ^ 0x9E37ull, g) % key_space;
  offsets[i] = (int32_t)(i * 12);
  uint8_t s[12] = {'t', 'e', 'm', 'p', '_', 0, 0, 0, 0, 0, 0, 0};
#pragma unroll
  for (int d = 6; d >= 0; --d) { s[5 + d] = (uint8_t)('0' + (k % 10)); k /= 10; }
  uint32_t w0 = s[0] | (s[1] << 8) | (s[2] << 16) | ((uint32_t)s[3] << 24);
  uint32_t w1 = s[4] | (s[5] << 8) | (s[6] << 16) | ((uint32_t)s[7] << 24);
  uint32_t w2 = s[8] | (s[9] << 8) | (s[10] << 16) | ((uint32_t)s[11] << 24);
  sensor_words[3 * i] = w0; sensor_words[3 * i + 1] = w1; sensor_words[3 * i + 2] = w2;
}

}  // namespace

Batch synth_batch(int64_t n, int64_t row0, uint64_t seed, int value_kind, int64_t key_space, cudaStream_t stream) {
  if (n < 0 || n * 12 > 2147483647ll) fail(ARK_ERR_PROCESS, "synthetic batch too large for Utf8 int32 offsets");
  if (key_space <= 0 || key_space > 10000000) fail(ARK_ERR_PROCESS, "key_space must be in [1, 10^7]");
  Batch b;
  b.num_rows = n;
  BufferPtr ts = device_alloc((size_t)n * 8), val = device_alloc((size_t)n * 8);
  BufferPtr off = device_alloc((size_t)(n + 1) * 4), data = device_alloc((size_t)n * 12 + 16);
  {
    KernelTimer t("synth_kernel", stream);
    synth_kernel<<<(unsigned)ceil_div(n + 1, 256), 256, 0, stream>>>(n, row0, seed, value_kind, (uint64_t)key_space,
                                                                     (int64_t*)ts.get(), (uint64_t*)val.get(),
                                                                     (int32_t*)off.get(), (uint32_t*)data.get());
  }
  ARK_CUDA(cudaGetLastError());
  auto mk = [&](const char* name, DType t) { Column c; c.field.name = name; c.field.type = t; c.field.nullable = true; c.length = n; return c; };
  Column c0 = mk("timestamp", DType::Int64); c0.data = (const uint8_t*)ts.get(); c0.data_bytes = n * 8; c0.owners = {ts};
  Column c1 = mk("value", value_kind == 0 ? DType::Int64 : DType::Float64); c1.data = (const uint8_t*)val.get(); c1.data_bytes = n * 8; c1.owners = {val};
  Column c2 = mk("sensor", DType::Utf8); c2.offsets = (const int32_t*)off.get(); c2.data = (const uint8_t*)data.get();
  c2.data_bytes = n * 12; c2.first_offset = 0; c2.owners = {off, data};
  b.cols = {c0, c1, c2};
  return b;
}

}  // namespace ark

extern "C" int ark_synth_batch_device(int64_t n_rows, int64_t row0, uint64_t seed, int value_kind, int64_t key_space,
                                      ArrowDeviceArray* out, ArrowSchema* out_schema) {
  return ark::guarded([&] {
    ark::zero_out(out, out_schema);
    ark::StreamLease lease;
    ark::Batch b = ark::synth_batch(n_rows, row0, seed, value_kind, key_space, lease.s);
    ark::export_device(b, out, out_schema, lease);
  });
}
