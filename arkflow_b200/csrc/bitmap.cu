// bitmap.cu — Arrow bitmaps built on the device from one byte per row, and the null-count policy of validity bitmaps
// (bitmap.h).
#include "bitmap.h"

namespace ark {

namespace {

__device__ __forceinline__ long long warp_sum(long long v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
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

// copy `n` bits starting at bit `bit0` of `in` into a fresh bitmap starting at bit 0
__global__ void realign_bits_kernel(const uint8_t* in, uint8_t* out, int64_t n, int32_t bit0) {
  int64_t byte = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  int64_t nbytes = (n + 7) >> 3;
  if (byte >= nbytes) return;
  int64_t src_bit = byte * 8 + bit0;
  uint32_t lo = in[src_bit >> 3];
  uint32_t hi = (((src_bit & 7) != 0) && ((src_bit >> 3) + 1 <= ((bit0 + n - 1) >> 3))) ? in[(src_bit >> 3) + 1] : 0;
  uint32_t v = ((lo | (hi << 8)) >> (src_bit & 7)) & 0xff;
  int64_t rem = n - byte * 8;
  if (rem < 8) v &= (1u << rem) - 1;
  out[byte] = (uint8_t)v;
}

// zero bits of `bits` over [bit0, bit0 + n), 32 bits per thread
__global__ void count_zeros_kernel(const uint8_t* bits, int64_t bit0, int64_t n, unsigned long long* zeros) {
  const int64_t i0 = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) * 32;
  int z = 0;
  for (int64_t i = i0; i < n && i < i0 + 32; ++i) {
    const int64_t b = bit0 + i;
    z += ((bits[b >> 3] >> (b & 7)) & 1) ^ 1;
  }
  z = (int)warp_sum(z);
  if ((threadIdx.x & 31) == 0 && z) atomicAdd(zeros, (unsigned long long)z);
}

}  // namespace

BufferPtr pack_bits(const uint8_t* bytes, int64_t n, unsigned long long* zeros, cudaStream_t stream) {
  BufferPtr bits = device_alloc((size_t)(n + 7) / 8 + 1);
  if (n > 0) {
    KernelTimer t("pack_bits_kernel", stream);
    int64_t nb = (n + 7) >> 3;
    pack_bits_kernel<<<(unsigned)ceil_div(nb, 256), 256, 0, stream>>>(bytes, n, (uint8_t*)bits.get(), zeros);
  }
  return bits;
}

void set_bool_values(Column& c, const BufferPtr& bytes, int64_t n, cudaStream_t stream) {
  BufferPtr bits = pack_bits((const uint8_t*)bytes.get(), n, nullptr, stream);
  c.data = (const uint8_t*)bits.get(); c.data_bit0 = 0; c.data_bytes = (n + 7) / 8;
  c.owners = {bits, bytes};
}

void set_validity(Column& c, const BufferPtr& bits, int64_t null_count) {
  if (null_count == 0) { c.validity = nullptr; c.null_count = 0; return; }
  c.validity = (const uint8_t*)bits.get(); c.validity_bit0 = 0; c.null_count = null_count;
  c.owners.push_back(bits);
}

void set_validity_unknown(Column& c, const BufferPtr& bytes, int64_t n, cudaStream_t stream) {
  if (n == 0) { set_validity(c, nullptr, 0); return; }
  set_validity(c, pack_bits((const uint8_t*)bytes.get(), n, nullptr, stream), -1);
  c.owners.push_back(bytes);
}

void count_zeros(const uint8_t* bits, int32_t bit0, int64_t n, unsigned long long* zeros, cudaStream_t stream) {
  if (n <= 0) return;
  KernelTimer t("count_zeros_kernel", stream);
  count_zeros_kernel<<<(unsigned)ceil_div(ceil_div(n, 32), 256), 256, 0, stream>>>(bits, bit0, n, zeros);
}

BufferPtr realign_bits(const uint8_t* in, int32_t bit0, int64_t n, cudaStream_t stream) {
  const int64_t nbytes = (n + 7) / 8;
  BufferPtr out = device_alloc((size_t)nbytes);
  KernelTimer t("realign_bits_kernel", stream);
  realign_bits_kernel<<<(unsigned)ceil_div(nbytes, 256), 256, 0, stream>>>(in, (uint8_t*)out.get(), n, bit0);
  return out;
}

}  // namespace ark
