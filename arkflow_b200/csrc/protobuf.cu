// protobuf.cu — `protobuf_to_arrow` and `arrow_to_protobuf` on the device.
//
// Stands in for ProtobufProcessor (crates/arkflow-plugin/src/processor/protobuf.rs:33-244) and protobuf_to_arrow /
// arrow_to_protobuf (crates/arkflow-plugin/src/component/protobuf.rs:115-339), i.e. prost-reflect 0.16's
// DynamicMessage decode / encode (a third-party crate) over the descriptor proto_schema.cc builds.
//
// protobuf_to_arrow: one message per thread (the MODE 2 pattern of json_parse_kernel: the CTA's payload bytes arrive
// in shared memory through one 1-D TMA bulk copy).  Fixed-width fields go straight to their output rows; string /
// bytes fields record the span of their last occurrence, and an exclusive scan + copy kernel builds the column.
//   * one non-nullable column per descriptor field, in declaration order; NULL payloads are dropped (to_binary);
//   * an absent field takes its default; the last occurrence of a field wins, and of a oneof only its last member read
//     keeps a value (the others take their defaults, as merging a oneof member clears the others); unknown fields
//     (groups included) are skipped;
//   * a truncated buffer, a varint longer than 10 bytes, a field number of 0 or a key beyond 32 bits, a known field
//     with the wrong wire type, an end-group that closes no group, more than 100 nested unknown groups, or a `string`
//     field that is not UTF-8 raise Process "Protobuf message parsing failed: …" (the first failing payload);
//   * a repeated / map / message field fails every non-empty batch with Process "Unsupported field type: <name>",
//     the first such field in declaration order (component/protobuf.rs:178-183 raises it while walking the fields);
//   * deviation: a batch whose payloads are all NULL gives zero rows with the message's columns (the reference indexes
//     the first decoded message of an empty list, processor/protobuf.rs:135, and panics).
// arrow_to_protobuf: measure → exclusive scan → write, one thread per row (the arrow_to_json pattern):
//   * a column is encoded when its name is a descriptor field and its Arrow type is that field's (Int32 for int32 /
//     sint32 / sfixed32 / enum, Int64, UInt32, UInt64, Float32, Float64, Boolean, Utf8, Binary); other columns are
//     skipped; a later column for the same field (or for another member of the same oneof) replaces an earlier one,
//     as set_field_by_name does;
//   * a matching column whose field is a message, a group or a map raises Process "Unsupported Protobuf type: …"
//     (the reference's `_` arm).  Map fields deliberately keep this Process error rather than ARK_ERR_UNSUPPORTED:
//     prost-reflect's Kind of a map field is Message, so the reference raises it before any value is set.  A column
//     whose field is a repeated scalar raises ARK_ERR_UNSUPPORTED (the reference panics in set_field there);
//   * fields in ascending number order; a field without explicit presence is left out when it holds its zero value
//     (0, false, "", and for float / double anything == 0.0, -0.0 included); NULL slots encode the value buffer;
//   * the output carries every input column, so an input column of a type the library does not hold (e.g. Date32)
//     raises ARK_ERR_UNSUPPORTED, as in arrow_to_json.
// Library limits, ARK_ERR_UNSUPPORTED: more than 64 fields in a decoded message, more than 64 encoded fields.  A string /
// bytes column or an encoded message column of 2 GiB or more (int32 offsets) raises Process before anything is written.
#include <cub/device/device_scan.cuh>

#include <algorithm>

#include "engine.h"
#include "json_mini.h"
#include "proto_schema.h"
#include "stage_store.cuh"
#include "tma.cuh"
#include "utf8.cuh"

namespace ark {

namespace {

constexpr int PB_MAX_FIELDS = 64;       // the per-message `seen` mask is 64 bits wide; the field tables travel in the parameter block
constexpr int PB_THREADS = 128;
constexpr int PB_MAX_GROUP_DEPTH = 100; // nested unknown groups a message may hold (prost's recursion limit)
constexpr int PB_BY_NUMBER = 128;       // field numbers below this are looked up in a table

enum PbErr : int { PE_NONE = 0, PE_TRUNCATED, PE_VARINT, PE_KEY, PE_WIRE_VALUE, PE_WIRE, PE_END_GROUP, PE_DEPTH, PE_UTF8 };

const char* pb_err_text(int code) {
  switch (code) {
    case PE_TRUNCATED: return "buffer underflow";
    case PE_VARINT: return "invalid varint";
    case PE_KEY: return "invalid key value (field number 0 or above 2^29-1)";
    case PE_WIRE_VALUE: return "invalid wire type value";
    case PE_WIRE: return "invalid wire type for a known field";
    case PE_END_GROUP: return "unexpected end group tag";
    case PE_DEPTH: return "recursion limit reached";
    case PE_UTF8: return "invalid string value: data is not UTF-8 encoded";
    default: return "malformed message";
  }
}

int wire_of(PbKind k) {
  switch (k) {
    case PbKind::Double: case PbKind::Fixed64: case PbKind::SFixed64: return 1;
    case PbKind::Float: case PbKind::Fixed32: case PbKind::SFixed32: return 5;
    case PbKind::String: case PbKind::Bytes: return 2;
    default: return 0;
  }
}

// the Arrow type a scalar kind maps to (component/protobuf.rs:138-177, 215-318)
DType arrow_type_of(PbKind k) {
  switch (k) {
    case PbKind::Bool: return DType::Bool;
    case PbKind::Int32: case PbKind::SInt32: case PbKind::SFixed32: case PbKind::Enum: return DType::Int32;
    case PbKind::Int64: case PbKind::SInt64: case PbKind::SFixed64: return DType::Int64;
    case PbKind::UInt32: case PbKind::Fixed32: return DType::UInt32;
    case PbKind::UInt64: case PbKind::Fixed64: return DType::UInt64;
    case PbKind::Float: return DType::Float32;
    case PbKind::Double: return DType::Float64;
    case PbKind::String: return DType::Utf8;
    case PbKind::Bytes: return DType::Binary;
    default: return DType::Null;
  }
}

// ---- decode -----------------------------------------------------------------------------------------------------
struct PbDecField {
  int32_t number;
  uint8_t kind;       // PbKind
  uint8_t wire;       // the wire type the kind travels with
  uint8_t width;      // bytes per output value: 1 (Boolean, bit-packed afterwards), 4 or 8; 0 for string / bytes
  uint8_t pad;
  uint64_t dflt;      // absent field: the value (fixed width), or (offset in the default blob << 32 | length)
  uint64_t others;    // bits of the other members of the field's oneof: reading this field clears them
  void* values;
  long long* str_src; // string / bytes: payload-column offset of the last occurrence's bytes; absent: -1 - blob offset
  int32_t* str_len;
};

struct PbDecParams {
  const uint8_t* data;       // payload bytes base
  const int32_t* offsets;    // payload i = data[offsets[i] .. offsets[i+1])
  const uint8_t* validity;   // payload validity: NULL payloads produce no row
  int32_t validity_bit0;
  int32_t n_fields;
  int64_t n_payloads;
  const int32_t* row_of;     // output row of payload i when some payloads are NULL (else nullptr: row i)
  unsigned long long* error; // min over failing payloads of (payload << 8 | PbErr)
  int32_t stage_bytes;       // shared-memory staging window per CTA (0 = parse from global memory)
  int8_t by_number[PB_BY_NUMBER];
  PbDecField fields[PB_MAX_FIELDS];
};

__device__ __forceinline__ bool pb_varint(const uint8_t*& p, const uint8_t* end, unsigned long long& v, int& err) {
  if (p < end && *p < 0x80) { v = *p++; return true; }
  v = 0;
#pragma unroll 1
  for (int s = 0; s < 10; ++s) {
    if (p >= end) { err = PE_TRUNCATED; return false; }
    const unsigned b = *p++;
    if (s == 9 && b > 1) { err = PE_VARINT; return false; }  // an 11th byte, or bits beyond 64
    v |= (unsigned long long)(b & 0x7F) << (7 * s);
    if (b < 0x80) return true;
  }
  err = PE_VARINT;
  return false;
}

// prost's decode_key: key ≤ u32::MAX, wire type 0..5, field number ≥ 1
__device__ __forceinline__ bool pb_key(const uint8_t*& p, const uint8_t* end, uint32_t& number, int& wire, int& err) {
  unsigned long long k;
  if (!pb_varint(p, end, k, err)) return false;
  if (k > 0xFFFFFFFFull) { err = PE_KEY; return false; }
  wire = (int)(k & 7);
  if (wire > 5) { err = PE_WIRE_VALUE; return false; }
  number = (uint32_t)(k >> 3);
  if (number == 0) { err = PE_KEY; return false; }
  return true;
}

// Skips the value of an unknown field (a group up to its matching end-group).  Out of line: the tag stack stays off the
// main loop's frame.
__device__ __noinline__ bool pb_skip(const uint8_t*& p, const uint8_t* end, uint32_t number, int wire, int& err) {
  uint32_t open[PB_MAX_GROUP_DEPTH];
  int depth = 0;
  while (true) {
    if (wire == 0) { unsigned long long v; if (!pb_varint(p, end, v, err)) return false; }
    else if (wire == 1 || wire == 5) {
      const int w = wire == 1 ? 8 : 4;
      if (end - p < w) { err = PE_TRUNCATED; return false; }
      p += w;
    } else if (wire == 2) {
      unsigned long long len;
      if (!pb_varint(p, end, len, err)) return false;
      if (len > (unsigned long long)(end - p)) { err = PE_TRUNCATED; return false; }
      p += len;
    } else if (wire == 3) {
      if (depth == PB_MAX_GROUP_DEPTH) { err = PE_DEPTH; return false; }
      open[depth++] = number;
    } else {  // 4: end-group
      if (depth == 0 || open[depth - 1] != number) { err = PE_END_GROUP; return false; }
      --depth;
    }
    if (depth == 0) return true;
    if (!pb_key(p, end, number, wire, err)) return false;
  }
}

__device__ __forceinline__ void pb_store(const PbDecField& F, int64_t row, unsigned long long v) {
  if (F.width == 8) ((unsigned long long*)F.values)[row] = v;
  else if (F.width == 4) ((uint32_t*)F.values)[row] = (uint32_t)v;
  else ((uint8_t*)F.values)[row] = (uint8_t)v;
}

__global__ void __launch_bounds__(PB_THREADS) protobuf_decode_kernel(const __grid_constant__ PbDecParams P) {
  extern __shared__ __align__(16) uint8_t pb_stage[];
  __shared__ __align__(8) unsigned long long s_bar;
  __shared__ long long s_stage_off;  // payload-column byte offset of pb_stage[0] (may be slightly negative)
  __shared__ int s_staged;
  const int64_t i0 = (int64_t)blockIdx.x * PB_THREADS;
  const int64_t i = i0 + threadIdx.x;
  if (threadIdx.x == 0) {
    s_staged = 0;
    if (P.stage_bytes > 0) {
      const int rows = (int)((P.n_payloads - i0) < PB_THREADS ? (P.n_payloads - i0) : PB_THREADS);
      const int32_t o0 = P.offsets[i0], o1 = P.offsets[i0 + rows];
      const uintptr_t a0 = reinterpret_cast<uintptr_t>(P.data + o0), a1 = reinterpret_cast<uintptr_t>(P.data + o1);
      const uintptr_t lo = a0 & ~(uintptr_t)15, hi = (a1 + 15) & ~(uintptr_t)15;
      if (o1 > o0 && hi - lo <= (uintptr_t)P.stage_bytes) {
        mbar_init(&s_bar, 1);
        mbar_fence_init();
        mbar_expect_tx(&s_bar, (unsigned)(hi - lo));
        tma_load_1d(pb_stage, reinterpret_cast<const void*>(lo), (unsigned)(hi - lo), &s_bar);
        s_stage_off = (long long)o0 - (long long)(a0 - lo);
        s_staged = 1;
      }
    }
  }
  __syncthreads();
  const bool staged = s_staged != 0;
  if (staged) mbar_wait(&s_bar, 0);
  if (i >= P.n_payloads) return;
  if (P.validity && !((P.validity[(i + P.validity_bit0) >> 3] >> ((i + P.validity_bit0) & 7)) & 1)) return;
  const int64_t row = P.row_of ? P.row_of[i] : i;
  // `origin` + column byte offset = address of that byte (in the staging window or in global memory)
  const uint8_t* origin = staged ? pb_stage - s_stage_off : P.data;
  const uint8_t* p = origin + P.offsets[i];
  const uint8_t* const end = origin + P.offsets[i + 1];
  unsigned long long seen = 0;
  int err = PE_NONE;
  while (p < end) {
    uint32_t num;
    int wire;
    if (!pb_key(p, end, num, wire, err)) break;
    int f = -1;
    if (num < PB_BY_NUMBER) f = P.by_number[num];
    else for (int k = 0; k < P.n_fields; ++k) if ((uint32_t)P.fields[k].number == num) { f = k; break; }
    if (f < 0) { if (!pb_skip(p, end, num, wire, err)) break; continue; }
    const PbDecField& F = P.fields[f];
    if (wire != F.wire) { err = PE_WIRE; break; }
    unsigned long long v = 0;
    if (wire == 0) {
      if (!pb_varint(p, end, v, err)) break;
      if (F.kind == (uint8_t)PbKind::SInt32) { const uint32_t n = (uint32_t)v; v = (n >> 1) ^ (0u - (n & 1)); }
      else if (F.kind == (uint8_t)PbKind::SInt64) v = (v >> 1) ^ (0ull - (v & 1));
      else if (F.kind == (uint8_t)PbKind::Bool) v = v != 0;
      // int32 / uint32 / enum keep the low 32 bits (`as i32` / `as u32`): pb_store truncates
    } else if (wire == 1 || wire == 5) {
      const int w = wire == 1 ? 8 : 4;
      if (end - p < w) { err = PE_TRUNCATED; break; }
      for (int b = w - 1; b >= 0; --b) v = (v << 8) | p[b];
      p += w;
    } else {  // 2: string / bytes
      unsigned long long len;
      if (!pb_varint(p, end, len, err)) break;
      if (len > (unsigned long long)(end - p)) { err = PE_TRUNCATED; break; }
      if (F.kind == (uint8_t)PbKind::String && !utf8_valid(p, (long long)len)) { err = PE_UTF8; break; }
      F.str_src[row] = (long long)(p - origin);
      F.str_len[row] = (int32_t)len;
      p += len;
      seen = (seen & ~F.others) | (1ull << f);
      continue;
    }
    pb_store(F, row, v);
    seen = (seen & ~F.others) | (1ull << f);  // a oneof keeps its last member: the others fall back to their defaults
  }
  if (err != PE_NONE) { atomicMin(P.error, ((unsigned long long)i << 8) | (unsigned)err); return; }
  for (int k = 0; k < P.n_fields; ++k) {
    if ((seen >> k) & 1) continue;
    const PbDecField& F = P.fields[k];
    if (F.width) pb_store(F, row, F.dflt);
    else { F.str_src[row] = -1 - (long long)(F.dflt >> 32); F.str_len[row] = (int32_t)(F.dflt & 0xFFFFFFFFu); }
  }
}

// 1 per non-NULL payload (the row count scan of a payload column with NULLs)
__global__ void protobuf_valid_kernel(const uint8_t* validity, int32_t bit0, int64_t n, int32_t* flags) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) flags[i] = (validity[(i + bit0) >> 3] >> ((i + bit0) & 7)) & 1;
}

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

// ---- encode -----------------------------------------------------------------------------------------------------
struct PbEncCol {
  uint8_t kind;      // PbKind
  uint8_t always;    // explicit presence: written even when it holds the zero value
  uint8_t key_len;
  uint8_t key[5];    // the field's tag as a varint
  ColView view;
};

struct PbEncParams {
  int64_t n_rows;
  int32_t n_cols;
  PbEncCol cols[PB_MAX_FIELDS];  // ascending field number
};

struct Sink {
  uint8_t* p;  // nullptr ⇒ counting only
  int n;
  __device__ __forceinline__ void put(uint8_t c) { if (p) p[n] = c; ++n; }
  __device__ __forceinline__ void varint(unsigned long long v) { while (v >= 0x80) { put((uint8_t)(v | 0x80)); v >>= 7; } put((uint8_t)v); }
  __device__ __forceinline__ void le(unsigned long long v, int w) { for (int b = 0; b < w; ++b) put((uint8_t)(v >> (8 * b))); }
};

__device__ __forceinline__ int pb_emit_row(const PbEncParams& P, int64_t row, uint8_t* out) {
  Sink s{out, 0};
  for (int c = 0; c < P.n_cols; ++c) {
    const PbEncCol& col = P.cols[c];
    const ColView& v = col.view;
    const PbKind k = (PbKind)col.kind;
    if (k == PbKind::String || k == PbKind::Bytes) {
      const int32_t o0 = v.offsets[row], len = v.offsets[row + 1] - o0;
      if (len == 0 && !col.always) continue;
      for (int b = 0; b < col.key_len; ++b) s.put(col.key[b]);
      s.varint((unsigned)len);
      const uint8_t* src = (const uint8_t*)v.data + o0;
      for (int b = 0; b < len; ++b) s.put(src[b]);
      continue;
    }
    unsigned long long raw;
    bool zero;
    switch (k) {
      case PbKind::Bool: {
        const int64_t b = row + v.data_bit0;
        raw = (((const uint8_t*)v.data)[b >> 3] >> (b & 7)) & 1;
        zero = raw == 0;
        break;
      }
      case PbKind::Int32: case PbKind::SInt32: case PbKind::SFixed32: case PbKind::Enum:
      case PbKind::UInt32: case PbKind::Fixed32:
        raw = ((const uint32_t*)v.data)[row]; zero = raw == 0; break;
      case PbKind::Float: raw = ((const uint32_t*)v.data)[row]; zero = __uint_as_float((unsigned)raw) == 0.0f; break;
      case PbKind::Double: raw = ((const unsigned long long*)v.data)[row]; zero = __longlong_as_double((long long)raw) == 0.0; break;
      default: raw = ((const unsigned long long*)v.data)[row]; zero = raw == 0; break;  // 64-bit integers
    }
    if (zero && !col.always) continue;
    for (int b = 0; b < col.key_len; ++b) s.put(col.key[b]);
    switch (k) {
      case PbKind::Int32: case PbKind::Enum: s.varint((unsigned long long)(long long)(int32_t)(uint32_t)raw); break;  // sign-extended: 10 bytes when negative
      case PbKind::SInt32: { const int32_t n = (int32_t)(uint32_t)raw; s.varint((uint32_t)((uint32_t)n << 1) ^ (uint32_t)(n >> 31)); break; }
      case PbKind::SInt64: { const long long n = (long long)raw; s.varint(((unsigned long long)n << 1) ^ (unsigned long long)(n >> 63)); break; }
      case PbKind::Fixed32: case PbKind::SFixed32: case PbKind::Float: s.le(raw, 4); break;
      case PbKind::Fixed64: case PbKind::SFixed64: case PbKind::Double: s.le(raw, 8); break;
      default: s.varint(raw); break;  // int64, uint64, uint32, bool
    }
  }
  return s.n;
}

__global__ void protobuf_encode_measure_kernel(const __grid_constant__ PbEncParams P, int32_t* lens) {
  const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r < P.n_rows) lens[r] = pb_emit_row(P, r, nullptr);
}

// The messages of one CTA's rows are contiguous in the output: each thread encodes its row into a shared-memory image of
// that range, which leaves with 16-byte stores (as arrow_to_json_write_kernel does).  The minimum of 8 CTAs per SM is
// there for ptxas: without it the kernel was held to 32 registers and spilled.
__global__ void __launch_bounds__(PB_THREADS, 8) protobuf_encode_write_kernel(const __grid_constant__ PbEncParams P, const int32_t* offsets, uint8_t* out,
                                                                            int stage_bytes) {
  extern __shared__ __align__(16) uint8_t pe_stage[];
  const int64_t r0 = (int64_t)blockIdx.x * PB_THREADS;
  const int rows = (int)((P.n_rows - r0) < PB_THREADS ? (P.n_rows - r0) : PB_THREADS);
  const int64_t r = r0 + threadIdx.x;
  const int32_t bb = offsets[r0];
  const int tb = offsets[r0 + rows] - bb;
  if (tb + 16 > stage_bytes) {  // long rows: encode straight into global memory
    if (r < P.n_rows) pb_emit_row(P, r, out + offsets[r]);
    return;
  }
  const int mis = stage_misalignment(out + bb);
  if (r < P.n_rows) pb_emit_row(P, r, pe_stage + mis + (offsets[r] - bb));
  __syncthreads();
  stage_store(out + bb, pe_stage, mis, tb, threadIdx.x, PB_THREADS);
}

// Sum of n non-negative int32 lengths, accumulated in 64 bits.
__global__ void protobuf_sum64_kernel(const int32_t* lens, int64_t n, unsigned long long* total) {
  long long acc = 0;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    acc += lens[i] >= 0 ? lens[i] : (1ll << 40);  // a negative length is a row that itself passed 2^31
  for (int o = 16; o; o >>= 1) acc += __shfl_down_sync(0xffffffffu, acc, o);
  if ((threadIdx.x & 31) == 0) atomicAdd(total, (unsigned long long)acc);
}

// The offsets of a Binary / Utf8 column are int32, and so is pb_scan: when lengths add up to 2^31 or more the scan wraps,
// and once it wraps past 2^32 its last entry looks valid again while earlier offsets point outside the allocation.  When
// the host's bound on the total (`bound`) does not rule that out, the total is summed exactly first (one more launch and
// synchronisation, taken only by batches near the limit) and a total beyond the int32 range fails before anything is
// written.
void pb_check_total(const int32_t* lens, int64_t n, int64_t bound, const std::string& what, cudaStream_t stream) {
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

// exclusive scan of n + 1 int32 lengths (pb_check_total guards the int32 range)
BufferPtr pb_scan(const int32_t* lens, int64_t n, cudaStream_t stream) {
  BufferPtr offs = device_alloc((size_t)(n + 1) * 4);
  size_t tb = 0;
  cub::DeviceScan::ExclusiveSum(nullptr, tb, lens, (int32_t*)offs.get(), (int)(n + 1), stream);
  BufferPtr tmp = device_alloc(tb + 16);
  note_launch("cub::DeviceScan::ExclusiveSum");
  cub::DeviceScan::ExclusiveSum(tmp.get(), tb, lens, (int32_t*)offs.get(), (int)(n + 1), stream);
  return offs;
}

// ---- configuration ----------------------------------------------------------------------------------------------
std::vector<std::string> string_list(const JsonValue& v, const char* key) {
  if (v.kind != JsonValue::Array) fail(ARK_ERR_SERIALIZATION, std::string("invalid type for `") + key + "`: expected a sequence");
  std::vector<std::string> out;
  for (auto& e : v.arr) {
    if (e.kind != JsonValue::String) fail(ARK_ERR_SERIALIZATION, std::string("invalid type in `") + key + "`: expected a string");
    out.push_back(e.str);
  }
  return out;
}

// CommonProtobufProcessorConfig (processor/protobuf.rs:157-163) read from the flat shape the reference's documentation
// and example use, then parse_proto_file + get_message_by_name (processor/protobuf.rs:73-95).
PbMessage load_config_message(const char* config_json, const char* name, JsonValue& cfg) {
  const std::string missing = std::string(name) + " processor configuration is missing";
  if (!config_json) fail(ARK_ERR_CONFIG, missing);
  cfg = parse_json(config_json);
  if (cfg.kind == JsonValue::Null) fail(ARK_ERR_CONFIG, missing);
  if (cfg.kind != JsonValue::Object) fail(ARK_ERR_SERIALIZATION, std::string("invalid type: expected struct ") + name + "ProcessorConfig");
  const JsonValue* in = cfg.get("proto_inputs");
  if (!in) fail(ARK_ERR_SERIALIZATION, "missing field `proto_inputs`");
  std::vector<std::string> inputs = string_list(*in, "proto_inputs"), includes = inputs;
  if (const JsonValue* v = cfg.get("proto_includes")) if (v->kind != JsonValue::Null) includes = string_list(*v, "proto_includes");
  const JsonValue* mt = cfg.get("message_type");
  if (!mt) fail(ARK_ERR_SERIALIZATION, "missing field `message_type`");
  if (mt->kind != JsonValue::String) fail(ARK_ERR_SERIALIZATION, "invalid type for `message_type`: expected a string");
  return load_proto_message(inputs, includes, mt->str);
}

}  // namespace

struct ProtobufToArrowProcessor : Processor {
  const char* type() const override { return "protobuf_to_arrow"; }
  PbMessage msg;
  std::string value_field = "__value__";  // DEFAULT_BINARY_VALUE_FIELD
  std::string unsupported;                 // the first repeated / map / message field, if any
  std::string default_blob;                // default bytes of the string / bytes fields
  std::vector<uint32_t> default_off;       // per field: offset of its default in default_blob
};

struct ArrowToProtobufProcessor : Processor {
  const char* type() const override { return "arrow_to_protobuf"; }
  PbMessage msg;
  bool has_include = false;
  std::vector<std::string> include;
};

std::unique_ptr<Processor> make_protobuf_to_arrow(const char* config_json) {
  JsonValue cfg;
  auto p = std::make_unique<ProtobufToArrowProcessor>();
  p->msg = load_config_message(config_json, "ProtobufToArrow", cfg);
  if (const JsonValue* v = cfg.get("value_field")) {
    if (v->kind == JsonValue::String) p->value_field = v->str;
    else if (v->kind != JsonValue::Null) fail(ARK_ERR_SERIALIZATION, "invalid type for `value_field`: expected a string");
  }
  for (auto& f : p->msg.fields) {
    if (p->unsupported.empty() && (f.repeated || f.kind == PbKind::Message || f.kind == PbKind::Group)) p->unsupported = f.name;
    p->default_off.push_back((uint32_t)p->default_blob.size());
    p->default_blob += f.default_bytes;
  }
  return p;
}

const std::string& protobuf_to_arrow_value_field(const Processor& p) { return static_cast<const ProtobufToArrowProcessor&>(p).value_field; }

std::unique_ptr<Processor> make_arrow_to_protobuf(const char* config_json) {
  JsonValue cfg;
  auto p = std::make_unique<ArrowToProtobufProcessor>();
  p->msg = load_config_message(config_json, "ArrowToProtobuf", cfg);
  if (const JsonValue* v = cfg.get("fields_to_include")) {
    if (v->kind != JsonValue::Null) { p->has_include = true; p->include = string_list(*v, "fields_to_include"); }
  }
  return p;
}

// `in` holds the payload column (device-resident) and at least one row.
Batch protobuf_to_arrow_device(const Processor& proc, Batch& in, cudaStream_t stream) {
  const auto& pp = static_cast<const ProtobufToArrowProcessor&>(proc);
  const int ci = in.find(pp.value_field);
  if (ci < 0) fail(ARK_ERR_PROCESS, "not found column");                                  // core/lib.rs:357-359
  Column& col = in.cols[ci];
  if (col.field.format != "z" || !col.present) fail(ARK_ERR_PROCESS, "not support data type");  // core/lib.rs:363-367
  if (!pp.unsupported.empty()) fail(ARK_ERR_PROCESS, "Unsupported field type: " + pp.unsupported);
  const std::vector<PbField>& fields = pp.msg.fields;
  if ((int)fields.size() > PB_MAX_FIELDS) fail(ARK_ERR_UNSUPPORTED, "protobuf_to_arrow: more than 64 fields in one message");
  std::vector<int> vl = {ci};
  resolve_varlen_extents(in, vl, stream);
  const int64_t n = col.length;
  BufferPtr h = pinned_alloc(16 + 4 * PB_MAX_FIELDS);

  // ---- output rows: the non-NULL payloads ----
  int64_t rows = n;
  BufferPtr row_of;
  if (col.validity && col.null_count != 0 && n > 0) {
    BufferPtr flags = device_alloc((size_t)(n + 1) * 4);
    ARK_CUDA(cudaMemsetAsync((int32_t*)flags.get() + n, 0, 4, stream));
    {
      KernelTimer t("protobuf_valid_kernel", stream);
      protobuf_valid_kernel<<<(unsigned)ceil_div(n, 256), 256, 0, stream>>>(col.validity, col.validity_bit0, n, (int32_t*)flags.get());
    }
    row_of = pb_scan((const int32_t*)flags.get(), n, stream);
    ARK_CUDA(cudaMemcpyAsync(h.get(), (int32_t*)row_of.get() + n, 4, cudaMemcpyDeviceToHost, stream));
    ARK_CUDA(cudaStreamSynchronize(stream));
    rows = *(const int32_t*)h.get();
  }
  // RecordBatch::try_new of a message without fields (component/protobuf.rs:188-190)
  if (fields.empty() && rows > 0) fail(ARK_ERR_PROCESS, "Creating an Arrow record batch failed: Invalid argument error: must either specify a row count or at least one column");

  // ---- decode ----
  PbDecParams P;
  memset(&P, 0, sizeof P);
  P.data = col.data; P.offsets = col.offsets; P.validity = col.validity; P.validity_bit0 = col.validity_bit0;
  P.n_payloads = n; P.n_fields = (int)fields.size();
  P.row_of = (const int32_t*)row_of.get();
  memset(P.by_number, -1, sizeof P.by_number);
  const size_t nf = fields.size();
  std::vector<BufferPtr> values(nf), src(nf), lens(nf);
  for (size_t k = 0; k < nf; ++k) {
    const PbField& f = fields[k];
    PbDecField& F = P.fields[k];
    F.number = f.number; F.kind = (uint8_t)f.kind; F.wire = (uint8_t)wire_of(f.kind);
    if (f.oneof >= 0)
      for (size_t j = 0; j < nf; ++j) if (j != k && fields[j].oneof == f.oneof) F.others |= 1ull << j;
    if (f.number < PB_BY_NUMBER) P.by_number[f.number] = (int8_t)k;
    const DType t = arrow_type_of(f.kind);
    if (t == DType::Utf8 || t == DType::Binary) {
      src[k] = device_alloc((size_t)std::max<int64_t>(rows, 1) * 8);
      lens[k] = device_alloc((size_t)(rows + 1) * 4);
      ARK_CUDA(cudaMemsetAsync((int32_t*)lens[k].get() + rows, 0, 4, stream));  // the scan reads rows + 1 entries
      F.str_src = (long long*)src[k].get(); F.str_len = (int32_t*)lens[k].get();
      F.dflt = ((uint64_t)pp.default_off[k] << 32) | (uint64_t)f.default_bytes.size();
    } else {
      F.width = t == DType::Bool ? 1 : (uint8_t)fixed_width(t);
      values[k] = device_alloc((size_t)std::max<int64_t>(rows, 1) * F.width);
      F.values = values[k].get();
      F.dflt = f.default_bits;
    }
  }
  BufferPtr err = device_alloc(8), blob;
  ARK_CUDA(cudaMemsetAsync(err.get(), 0xFF, 8, stream));
  P.error = (unsigned long long*)err.get();
  if (!pp.default_blob.empty()) {
    blob = device_alloc(pp.default_blob.size());
    ARK_CUDA(cudaMemcpyAsync(blob.get(), pp.default_blob.data(), pp.default_blob.size(), cudaMemcpyHostToDevice, stream));
  }
  if (rows > 0) {
    // staging window: the CTA's payload bytes + alignment slack; payloads that average more than 256 bytes are parsed in place
    const double avg = (double)col.data_bytes / (double)n;
    P.stage_bytes = avg <= 256.0 ? (int)round_up((int64_t)(avg * PB_THREADS * 1.25) + 256, 1024) : 0;
    KernelTimer t("protobuf_decode_kernel", stream);
    protobuf_decode_kernel<<<(unsigned)ceil_div(n, PB_THREADS), PB_THREADS, (size_t)P.stage_bytes + 32, stream>>>(P);
  }
  ARK_CUDA(cudaGetLastError());
  // the error word and every string column's byte total come back in one round trip
  std::vector<BufferPtr> str_offs(nf);
  ARK_CUDA(cudaMemcpyAsync(h.get(), err.get(), 8, cudaMemcpyDeviceToHost, stream));
  for (size_t k = 0; k < nf; ++k) {
    if (!lens[k]) continue;
    str_offs[k] = pb_scan((const int32_t*)lens[k].get(), rows, stream);
    ARK_CUDA(cudaMemcpyAsync((char*)h.get() + 16 + 4 * k, (int32_t*)str_offs[k].get() + rows, 4, cudaMemcpyDeviceToHost, stream));
  }
  ARK_CUDA(cudaStreamSynchronize(stream));
  const unsigned long long e = *(const unsigned long long*)h.get();
  if (e != ~0ull)
    fail(ARK_ERR_PROCESS, std::string("Protobuf message parsing failed: ") + pb_err_text((int)(e & 0xFF)) + " (payload " + std::to_string(e >> 8) + ")");
  // a row's span lies inside its own payload, so the payload bytes plus one default per row bound a string column's total
  for (size_t k = 0; k < nf; ++k)
    if (lens[k])
      pb_check_total((const int32_t*)lens[k].get(), rows, col.data_bytes + rows * (int64_t)fields[k].default_bytes.size(),
                     "protobuf_to_arrow: column '" + fields[k].name + "'", stream);

  // ---- columns ----
  Batch out;
  out.num_rows = rows;
  for (size_t k = 0; k < nf; ++k) {
    const DType t = arrow_type_of(fields[k].kind);
    Column c;
    c.field.name = fields[k].name; c.field.type = t; c.field.nullable = false; c.field.format = dtype_arrow_format(t);
    c.length = rows;
    if (str_offs[k]) {
      const int32_t total = *(const int32_t*)((char*)h.get() + 16 + 4 * k);
      BufferPtr bytes = device_alloc((size_t)total + 16);
      if (rows && total) {
        KernelTimer tm("protobuf_strings_kernel", stream);
        protobuf_strings_kernel<<<(unsigned)ceil_div(rows, 256), 256, 0, stream>>>(col.data, (const uint8_t*)blob.get(), (const long long*)src[k].get(),
                                                                                 (const int32_t*)str_offs[k].get(), rows, (uint8_t*)bytes.get());
      }
      c.offsets = (const int32_t*)str_offs[k].get(); c.data = (const uint8_t*)bytes.get(); c.data_bytes = total; c.first_offset = 0;
      c.owners = {str_offs[k], bytes};
    } else if (t == DType::Bool) {
      BufferPtr bits = device_alloc((size_t)(rows + 7) / 8 + 1);
      if (rows) launch_pack_bits((const uint8_t*)values[k].get(), rows, (uint8_t*)bits.get(), nullptr, stream);
      c.data = (const uint8_t*)bits.get(); c.data_bytes = (rows + 7) / 8; c.owners = {bits, values[k]};
    } else {
      c.data = (const uint8_t*)values[k].get(); c.data_bytes = rows * fixed_width(t); c.owners = {values[k]};
    }
    out.cols.push_back(std::move(c));
  }
  ARK_CUDA(cudaGetLastError());
  ARK_CUDA(cudaStreamSynchronize(stream));
  return out;
}

// `in` was imported with codec_types (Int32 / UInt32 / UInt64 / Float32 columns present) and holds at least one row.
Batch arrow_to_protobuf_device(const Processor& proc, Batch& in, cudaStream_t stream) {
  const auto& ap = static_cast<const ArrowToProtobufProcessor&>(proc);
  const std::vector<PbField>& fields = ap.msg.fields;
  const int64_t n = in.num_rows;
  // which column sets each field: set_field_by_name in column order (component/protobuf.rs:209-327)
  std::vector<int> from(fields.size(), -1);
  int kept = 0;
  for (size_t i = 0; i < in.cols.size(); ++i) {
    const Column& c = in.cols[i];
    if (!c.present && c.field.format != "n") fail(ARK_ERR_UNSUPPORTED, "arrow_to_protobuf: column '" + c.field.name + "' has Arrow type '" + c.field.format + "'");
    if (ap.has_include && std::find(ap.include.begin(), ap.include.end(), c.field.name) == ap.include.end()) continue;  // filter_columns, lib.rs:304-328
    ++kept;
    int k = -1;
    for (size_t j = 0; j < fields.size(); ++j) if (fields[j].name == c.field.name) { k = (int)j; break; }
    if (k < 0) continue;
    const PbField& f = fields[k];
    if (f.kind == PbKind::Message || f.kind == PbKind::Group) fail(ARK_ERR_PROCESS, "Unsupported Protobuf type: " + pb_kind_debug(f));
    if (!c.present || c.field.type != arrow_type_of(f.kind)) continue;  // the reference's downcast_ref fails: skipped
    if (f.repeated) fail(ARK_ERR_UNSUPPORTED, "arrow_to_protobuf: column '" + c.field.name + "' sets repeated field '" + f.name + "'");
    if (f.oneof >= 0) for (size_t j = 0; j < fields.size(); ++j) if (fields[j].oneof == f.oneof) from[j] = -1;  // one member of a oneof at a time
    from[k] = (int)i;
  }
  if (ap.has_include && kept == 0) fail_filtered_to_no_columns();
  std::vector<int> order;
  for (size_t j = 0; j < fields.size(); ++j) if (from[j] >= 0) order.push_back((int)j);
  std::sort(order.begin(), order.end(), [&](int a, int b) { return fields[a].number < fields[b].number; });
  if ((int)order.size() > PB_MAX_FIELDS) fail(ARK_ERR_UNSUPPORTED, "arrow_to_protobuf: more than 64 encoded fields");
  PbEncParams P;
  memset(&P, 0, sizeof P);
  P.n_rows = n;
  int64_t bound = 0;  // on the output bytes: per row a key and the widest value, string bytes counted once
  for (int j : order) {
    const PbField& f = fields[j];
    const Column& c = in.cols[from[j]];
    const int w = wire_of(f.kind);
    bound += n * (5 + (w == 0 ? 10 : w == 1 ? 8 : w == 5 ? 4 : 5));
    if (w == 2) bound = c.data_bytes < 0 ? -1 : (bound < 0 ? -1 : bound + c.data_bytes);
    if (bound < 0) break;
  }
  for (int j : order) {
    const PbField& f = fields[j];
    PbEncCol& e = P.cols[P.n_cols++];
    e.kind = (uint8_t)f.kind; e.always = f.presence ? 1 : 0;
    unsigned long long key = ((unsigned long long)f.number << 3) | (unsigned)wire_of(f.kind);
    while (key >= 0x80) { e.key[e.key_len++] = (uint8_t)(key | 0x80); key >>= 7; }
    e.key[e.key_len++] = (uint8_t)key;
    e.view = in.cols[from[j]].view();
  }
  BufferPtr lens = device_alloc((size_t)(n + 1) * 4);
  ARK_CUDA(cudaMemsetAsync(lens.get(), 0, (size_t)(n + 1) * 4, stream));
  const unsigned grid = (unsigned)std::max<int64_t>(1, ceil_div(n, PB_THREADS));
  if (n) {
    KernelTimer t("protobuf_encode_measure_kernel", stream);
    protobuf_encode_measure_kernel<<<grid, PB_THREADS, 0, stream>>>(P, (int32_t*)lens.get());
  }
  pb_check_total((const int32_t*)lens.get(), n, bound, "arrow_to_protobuf: the encoded messages", stream);
  BufferPtr offs = pb_scan((const int32_t*)lens.get(), n, stream);
  BufferPtr h = pinned_alloc(16);
  ARK_CUDA(cudaMemcpyAsync(h.get(), (int32_t*)offs.get() + n, 4, cudaMemcpyDeviceToHost, stream));
  ARK_CUDA(cudaStreamSynchronize(stream));
  const int32_t total = *(const int32_t*)h.get();
  BufferPtr bytes = device_alloc((size_t)total + 16);
  if (n && total) {
    KernelTimer t("protobuf_encode_write_kernel", stream);
    // staging window: the average CTA's bytes + 50 %; CTAs whose rows are longer take the direct path
    const int stage = (int)std::min<int64_t>(44 * 1024, round_up((int64_t)((double)total / (double)n * PB_THREADS * 1.5) + 256, 1024));
    protobuf_encode_write_kernel<<<grid, PB_THREADS, stage, stream>>>(P, (const int32_t*)offs.get(), (uint8_t*)bytes.get(), stage);
  }
  ARK_CUDA(cudaGetLastError());
  Batch out;
  out.num_rows = n;  // new_binary_with_origin → MessageBatch::new_arrow: no input name
  out.cols = in.cols;
  Column v;
  v.field.name = "__value__"; v.field.type = DType::Binary; v.field.nullable = false; v.field.format = "z";
  v.length = n;
  v.offsets = (const int32_t*)offs.get(); v.data = (const uint8_t*)bytes.get(); v.data_bytes = total; v.first_offset = 0;
  v.owners = {offs, bytes};
  out.cols.push_back(v);
  ARK_CUDA(cudaStreamSynchronize(stream));
  return out;
}

}  // namespace ark
