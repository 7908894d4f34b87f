// avro.cu — the `file` input's `avro` type: Avro object container files (spec 1.11) decoded on the device.
//
// The file's bytes go to HBM once (the file driver's upload); on the host, while the chunks stream past, avro_scan walks
// the header and every block header and builds the block table {data offset, size, count, first row, uncompressed
// length}.  A batch of rows [r0, r0 + n) then runs:
//   avro_snappy_kernel  (codec snappy) one warp per block of the batch decompresses into an arena laid out by a host scan
//                       of the uncompressed lengths, and checks the block's big-endian CRC-32; with codec null the arena is
//                       the file itself and nothing is copied;
//   avro_index_kernel   one thread per block walks its records, skipping fields by schema, and writes where each record of
//                       the batch starts and ends;
//   avro_decode_kernel  one thread per record (the records of a CTA arrive in shared memory by one 1-D TMA bulk copy):
//                       fixed-width values and validity go to their rows, string / bytes record their spans, and strings
//                       are checked for UTF-8 in the same pass;
//   columns             settled and built by decoded.h (the error word before the 2 GiB guard; scans, validity and null
//                       counts in one round trip), string bytes by a span copy (varlen.h's launch_span_copy).
// Schema: a record whose fields are null, boolean, int, long, float, double, bytes or string, or a two-branch union of
// null and one of these in either order → Null, Boolean, Int32, Int64, Float32, Float64, Binary, Utf8 (DataFusion's Avro
// reader's mapping); a plain field is non-nullable, a union field nullable.  Anything else (nested record, array, map,
// enum, fixed, a logicalType, other unions, a top level that is not a record) and the codecs deflate / zstandard / bzip2
// / xz are ARK_ERR_UNSUPPORTED from connect(), decided from the header before the device is touched.
// Errors are Process "Read input failed: Avro error: …":
//   * the container's structure (bad magic, sync-marker mismatch, truncated block, negative count or size, a block
//     header varint longer than 10 bytes, a snappy length preamble that does not fit its block) fails connect() and
//     names the block's file offset;
//   * the data (a varint longer than 10 bytes, an `int` outside i32, a boolean byte other than 0 / 1, a union index
//     other than 0 / 1, a negative or overrunning length, a `string` that is not UTF-8, a record that runs past its
//     block, a snappy stream that overruns or underfills its declared length or copies from before its start, a CRC
//     mismatch) fails the read() of the batch that holds the first failing record in file order, and names that record
//     (0-based in the file) and its block's offset.  Within a record the first failing field in order decides the text.
//     A snappy or CRC failure is the failure of its block's first record.
// oracle/avro_oracle.py restates all of this in Python; tests/test_avro_input_gpu.py compares the two.
#include <algorithm>
#include <cstdio>

#include "decoded.h"
#include "file_input.h"
#include "json_mini.h"
#include "stage_store.cuh"
#include "tma.cuh"
#include "utf8.cuh"
#include "varlen.h"

namespace ark {

namespace {

constexpr int AV_THREADS = 128;
constexpr int AV_MAX_FIELDS = 64;
constexpr uint32_t CRC_POLY = 0xEDB88320u;  // CRC-32 (zlib's), reflected

enum AvKind : uint8_t { AK_NULL = 0, AK_BOOL, AK_INT, AK_LONG, AK_FLOAT, AK_DOUBLE, AK_BYTES, AK_STRING };

enum AvErr : int { AE_NONE = 0, AE_VARINT, AE_TRUNCATED, AE_INT, AE_BOOL, AE_UNION, AE_LEN, AE_UTF8,
                   AE_SNAPPY_OVERRUN, AE_SNAPPY_UNDERFILL, AE_SNAPPY_BAD, AE_CRC };

const char* av_err_text(int code) {
  switch (code) {
    case AE_VARINT: return "varint longer than 10 bytes";
    case AE_TRUNCATED: return "record runs past the end of its block";
    case AE_INT: return "int value out of the i32 range";
    case AE_BOOL: return "boolean byte other than 0 or 1";
    case AE_UNION: return "union index out of range";
    case AE_LEN: return "negative or overrunning length";
    case AE_UTF8: return "string is not valid UTF-8";
    case AE_SNAPPY_OVERRUN: return "snappy stream overruns its declared length";
    case AE_SNAPPY_UNDERFILL: return "snappy stream underfills its declared length";
    case AE_SNAPPY_BAD: return "malformed snappy stream";
    case AE_CRC: return "snappy block CRC-32 mismatch";
    default: return "malformed data";
  }
}

DType av_dtype(uint8_t k) {
  switch (k) {
    case AK_BOOL: return DType::Bool;
    case AK_INT: return DType::Int32;
    case AK_LONG: return DType::Int64;
    case AK_FLOAT: return DType::Float32;
    case AK_DOUBLE: return DType::Float64;
    case AK_BYTES: return DType::Binary;
    case AK_STRING: return DType::Utf8;
    default: return DType::Null;
  }
}

}  // namespace

struct AvroField {
  std::string name;
  uint8_t kind;
  int8_t null_branch;  // -1: a plain field; 0 / 1: the union branch that is null
};

// one block of the file: data = file[data_off, data_off + size), followed by the 16-byte sync marker
struct AvroBlock {
  int64_t offset;     // file offset of the block (its count varint)
  int64_t data_off;
  int64_t size;
  int64_t count;
  int64_t first_row;
  int64_t ulen;       // uncompressed bytes (snappy: the stream's preamble; null: size)
  int64_t pre;        // snappy: bytes of the length preamble
};

struct AvroFile {
  std::vector<AvroField> fields;
  bool snappy = false;
  uint8_t sync[16];
  int64_t header_bytes = 0;
  std::vector<AvroBlock> blocks;
  int64_t rows = 0;
  // scanner state: `win` holds the file's bytes [pos, pos + win.size()) not yet parsed
  enum State { BlockHeader, Data, Sync } state = BlockHeader;
  int64_t pos = 0;
  std::string win;
  int64_t cur = -1;  // the block being scanned
};

namespace {

[[noreturn]] void av_fail(const std::string& what) { fail(ARK_ERR_PROCESS, "Read input failed: Avro error: " + what); }

// Avro's long: zig-zag varint of at most 10 bytes (apache-avro's decode_variable: bits past 64 are dropped).
// Returns bytes used, 0 when `n` bytes do not finish it, -1 when it runs past 10 bytes.
int host_varint(const uint8_t* p, size_t n, int64_t* out) {
  uint64_t v = 0;
  for (int i = 0; i < 10; ++i) {
    if ((size_t)i >= n) return 0;
    v |= (uint64_t)(p[i] & 0x7F) << (7 * i);
    if (p[i] < 0x80) { *out = (int64_t)(v >> 1) ^ -(int64_t)(v & 1); return i + 1; }
  }
  return -1;
}

std::string type_desc(const JsonValue& t) {
  if (t.kind == JsonValue::String) return t.str;
  if (t.kind == JsonValue::Array) return "union";
  if (t.kind == JsonValue::Object) {
    if (t.get("logicalType")) return "logicalType " + (t.get("logicalType")->kind == JsonValue::String ? t.get("logicalType")->str : std::string("?"));
    if (const JsonValue* ty = t.get("type")) if (ty->kind == JsonValue::String) return ty->str;
  }
  return "?";
}

// a primitive this decoder reads, or -1
int prim_kind(const JsonValue& t) {
  const JsonValue* s = &t;
  if (t.kind == JsonValue::Object) {
    if (t.get("logicalType")) return -1;
    s = t.get("type");
    if (!s) return -1;
  }
  if (s->kind != JsonValue::String) return -1;
  static const char* names[] = {"null", "boolean", "int", "long", "float", "double", "bytes", "string"};
  for (int k = 0; k < 8; ++k) if (s->str == names[k]) return k;
  return -1;
}

void parse_schema(AvroFile& f, const std::string& text) {
  JsonValue s;
  try { s = parse_json(text); } catch (const ArkError& e) { av_fail(std::string("invalid schema: ") + e.what()); }
  const JsonValue* ty = s.kind == JsonValue::Object ? s.get("type") : nullptr;
  if (!ty || ty->kind != JsonValue::String || ty->str != "record")
    fail(ARK_ERR_UNSUPPORTED, "avro input: the top-level schema is " + type_desc(s) + ", not a record");
  const JsonValue* fs = s.get("fields");
  if (!fs || fs->kind != JsonValue::Array) av_fail("invalid schema: a record without `fields`");
  for (auto& fv : fs->arr) {
    const JsonValue* nm = fv.kind == JsonValue::Object ? fv.get("name") : nullptr;
    const JsonValue* t = fv.kind == JsonValue::Object ? fv.get("type") : nullptr;
    if (!nm || nm->kind != JsonValue::String || !t) av_fail("invalid schema: a field without `name` or `type`");
    AvroField F{nm->str, 0, -1};
    int k = prim_kind(*t);
    if (t->kind == JsonValue::Array && t->arr.size() == 2) {
      const int a = prim_kind(t->arr[0]), b = prim_kind(t->arr[1]);
      if (a == AK_NULL && b > AK_NULL) { k = b; F.null_branch = 0; }
      else if (b == AK_NULL && a > AK_NULL) { k = a; F.null_branch = 1; }
    }
    if (k < 0) fail(ARK_ERR_UNSUPPORTED, "avro input: field '" + F.name + "' has type " + type_desc(*t) + ", which is not decoded on the GPU");
    F.kind = (uint8_t)k;
    f.fields.push_back(F);
  }
  if ((int)f.fields.size() > AV_MAX_FIELDS) fail(ARK_ERR_UNSUPPORTED, "avro input: more than 64 fields in a record");
}

// Parses the header at the start of `h`: returns its length, or 0 when more bytes are needed (`eof`: there are none).
int64_t parse_header(AvroFile& f, const std::string& h, bool eof) {
  const uint8_t* p = (const uint8_t*)h.data();
  const size_t n = h.size();
  if (n < 4) { if (eof) av_fail("not an Avro object container file (bad magic)"); return 0; }
  if (memcmp(p, "Obj\x01", 4) != 0) av_fail("not an Avro object container file (bad magic)");
  size_t q = 4;
  std::string schema, codec = "null";
  bool have_schema = false;
  auto need_more = [&]() -> int64_t { if (eof) av_fail("truncated header"); return 0; };
  while (true) {
    int64_t cnt;
    int u = host_varint(p + q, n - q, &cnt);
    if (u == 0) return need_more();
    if (u < 0) av_fail("varint longer than 10 bytes in the header");
    q += (size_t)u;
    if (cnt == 0) break;
    if (cnt < 0) {
      cnt = -cnt;
      int64_t bytes;
      u = host_varint(p + q, n - q, &bytes);
      if (u == 0) return need_more();
      if (u < 0) av_fail("varint longer than 10 bytes in the header");
      q += (size_t)u;
    }
    for (int64_t i = 0; i < cnt; ++i) {
      std::string kv[2];
      for (auto& s : kv) {
        int64_t len;
        u = host_varint(p + q, n - q, &len);
        if (u == 0) return need_more();
        if (u < 0) av_fail("varint longer than 10 bytes in the header");
        if (len < 0) av_fail("negative length in the header");
        q += (size_t)u;
        if ((uint64_t)len > n - q) return need_more();
        s.assign((const char*)p + q, (size_t)len);
        q += (size_t)len;
      }
      if (kv[0] == "avro.schema") { schema = kv[1]; have_schema = true; }
      else if (kv[0] == "avro.codec") codec = kv[1];
    }
  }
  if (n - q < 16) return need_more();
  memcpy(f.sync, p + q, 16);
  q += 16;
  if (!have_schema) av_fail("the header has no avro.schema");
  if (codec == "snappy") f.snappy = true;
  else if (codec != "null" && !codec.empty())
    fail(ARK_ERR_UNSUPPORTED, "avro input: codec '" + codec + "' is not decoded on the GPU (null and snappy are)");
  parse_schema(f, schema);
  return (int64_t)q;
}

// The file's bytes [base, base + n), in order, after the header.  Block headers and sync markers may straddle two calls.
void avro_scan(AvroFile& f, const uint8_t* p, size_t n, int64_t base) {
  const int64_t end = base + (int64_t)n;
  while (true) {
    if (f.state == AvroFile::Data) {  // skip to the end of the block's data
      AvroBlock& b = f.blocks[(size_t)f.cur];
      const int64_t t = b.data_off + b.size;
      const int64_t have = f.pos + (int64_t)f.win.size();
      if (t <= have) { f.win.erase(0, (size_t)(t - f.pos)); f.pos = t; }
      else { if (t > end) { f.pos = end; f.win.clear(); return; } f.pos = t; f.win.clear(); }
      f.state = AvroFile::Sync;
    }
    // top up the window from this chunk (64 bytes decide a block header or a sync marker)
    const int64_t q = f.pos + (int64_t)f.win.size();
    if (f.win.size() < 64 && q >= base && q < end) f.win.append((const char*)p + (q - base), (size_t)std::min<int64_t>(64 - (int64_t)f.win.size(), end - q));
    const uint8_t* w = (const uint8_t*)f.win.data();
    const size_t wn = f.win.size();
    if (f.state == AvroFile::Sync) {
      if (wn < 16) return;
      if (memcmp(w, f.sync, 16) != 0) av_fail("sync marker mismatch (block at offset " + std::to_string(f.blocks[(size_t)f.cur].offset) + ")");
      f.win.erase(0, 16); f.pos += 16;
      f.state = AvroFile::BlockHeader;
      continue;
    }
    // block header: count, size, and for snappy the stream's length preamble
    if (wn == 0) return;
    const std::string at = " (block at offset " + std::to_string(f.pos) + ")";
    int64_t count, size, ulen = 0;
    int u1 = host_varint(w, wn, &count);
    if (u1 < 0) av_fail("varint longer than 10 bytes" + at);
    if (u1 == 0) return;
    int u2 = host_varint(w + u1, wn - (size_t)u1, &size);
    if (u2 < 0) av_fail("varint longer than 10 bytes" + at);
    if (u2 == 0) return;
    if (count < 0) av_fail("negative block count" + at);
    if (size < 0) av_fail("negative block size" + at);
    int pre = 0;
    if (f.snappy) {
      // the preamble: a plain (not zig-zag) varint of at most 32 bits, inside the block's data before its 4-byte CRC
      const size_t avail = (size_t)std::min<int64_t>((int64_t)(wn - u1 - u2), size);
      uint64_t v = 0;
      for (int i = 0;; ++i) {
        if (i == 5 || (int64_t)i >= size - 4) av_fail("snappy block without a valid length preamble" + at);
        if ((size_t)i >= avail) return;
        const uint8_t c = w[u1 + u2 + i];
        v |= (uint64_t)(c & 0x7F) << (7 * i);
        if (c < 0x80) { pre = i + 1; break; }
      }
      if (v > 0xFFFFFFFFull) av_fail("snappy block without a valid length preamble" + at);
      ulen = (int64_t)v;
    }
    AvroBlock b{f.pos, f.pos + u1 + u2, size, count, f.rows, f.snappy ? ulen : size, pre};
    f.blocks.push_back(b);
    f.rows += count;
    f.cur = (int64_t)f.blocks.size() - 1;
    f.win.erase(0, (size_t)(u1 + u2)); f.pos += u1 + u2;
    f.state = AvroFile::Data;
  }
}

void avro_scan_end(AvroFile& f) {
  if (f.state == AvroFile::BlockHeader && f.win.empty()) return;
  const int64_t off = f.state == AvroFile::BlockHeader ? f.pos : f.blocks[(size_t)f.cur].offset;
  av_fail("truncated block (block at offset " + std::to_string(off) + ")");
}

// ---- device --------------------------------------------------------------------------------------------------------
struct AvBlockDev {
  long long start, end;   // the block's records in the arena
  long long first_row;    // file row of its first record
  long long src;          // snappy: file offset of the compressed stream (after the preamble)
  long long src_len;      // snappy: bytes of that stream (the CRC follows)
  long long count;
};

struct AvField {
  uint8_t kind;
  int8_t null_branch;
  uint8_t width;          // bytes per stored value (Boolean 1, bit-packed afterwards); 0: no value buffer
  void* values;
  uint8_t* valid;         // union fields: byte per row
  long long* str_src;     // string / bytes: arena offset of the value
  int32_t* str_len;
};

struct AvParams {
  const uint8_t* arena;
  const long long* rec_start;  // arena offset of record row0 + i, or -1 when its block could not be walked to it
  const long long* rec_end;
  long long n;
  long long row0;              // file row of the batch's first record
  int32_t n_fields;
  int32_t stage_bytes;
  unsigned long long* error;   // min over failing records of (file row << 8 | AvErr)
  AvField f[AV_MAX_FIELDS];
};

__device__ __forceinline__ bool av_long(const uint8_t*& p, const uint8_t* end, long long& v, int& err) {
  unsigned long long u = 0;
#pragma unroll 1
  for (int s = 0; s < 10; ++s) {
    if (p >= end) { err = AE_TRUNCATED; return false; }
    const unsigned b = *p++;
    u |= (unsigned long long)(b & 0x7F) << (7 * s);
    if (b < 0x80) { v = (long long)(u >> 1) ^ -(long long)(u & 1); return true; }
  }
  err = AE_VARINT;
  return false;
}

// Walks one record.  With STORE it checks every value and stores row `row`'s; without, it checks only what finding the
// record's end needs (varints, union indexes, lengths).
template <bool STORE>
__device__ __forceinline__ bool av_record(const AvParams& P, const uint8_t*& p, const uint8_t* end, const uint8_t* origin, long long row, int& err) {
  for (int k = 0; k < P.n_fields; ++k) {
    const AvField& F = P.f[k];
    bool present = F.kind != AK_NULL;
    if (F.null_branch >= 0) {
      long long b;
      if (!av_long(p, end, b, err)) return false;
      if (b != 0 && b != 1) { err = AE_UNION; return false; }
      if (b == F.null_branch) present = false;
      if (STORE) F.valid[row] = present;
    }
    if (!present) {
      if (STORE) {
        if (F.str_len) { F.str_len[row] = 0; F.str_src[row] = 0; }
        else if (F.width == 8) ((unsigned long long*)F.values)[row] = 0;
        else if (F.width == 4) ((uint32_t*)F.values)[row] = 0;
        else if (F.width == 1) ((uint8_t*)F.values)[row] = 0;
      }
      continue;
    }
    switch (F.kind) {
      case AK_BOOL: {
        if (p >= end) { err = AE_TRUNCATED; return false; }
        const uint8_t v = *p++;
        if (STORE) { if (v > 1) { err = AE_BOOL; return false; } ((uint8_t*)F.values)[row] = v; }
        break;
      }
      case AK_INT: case AK_LONG: {
        long long v;
        if (!av_long(p, end, v, err)) return false;
        if (STORE) {
          if (F.kind == AK_INT) { if (v < INT32_MIN || v > INT32_MAX) { err = AE_INT; return false; } ((int32_t*)F.values)[row] = (int32_t)v; }
          else ((long long*)F.values)[row] = v;
        }
        break;
      }
      case AK_FLOAT: case AK_DOUBLE: {
        const int w = F.kind == AK_FLOAT ? 4 : 8;
        if (end - p < w) { err = AE_TRUNCATED; return false; }
        if (STORE) {
          unsigned long long v = 0;
          for (int b = w - 1; b >= 0; --b) v = (v << 8) | p[b];
          if (w == 8) ((unsigned long long*)F.values)[row] = v;
          else ((uint32_t*)F.values)[row] = (uint32_t)v;
        }
        p += w;
        break;
      }
      default: {  // bytes / string
        long long len;
        if (!av_long(p, end, len, err)) return false;
        if (len < 0 || len > end - p) { err = AE_LEN; return false; }
        if (STORE) {
          if (F.kind == AK_STRING && !utf8_valid(p, len)) { err = AE_UTF8; return false; }
          F.str_src[row] = (long long)(p - origin);
          F.str_len[row] = (int32_t)len;
        }
        p += len;
        break;
      }
    }
  }
  return true;
}

// ---- snappy ----
__host__ __device__ inline uint32_t crc_multmodp(uint32_t a, uint32_t b) {  // a·b mod the CRC polynomial (zlib's multmodp)
  uint32_t m = 1u << 31, p = 0;
  for (;;) {
    if (a & m) { p ^= b; if ((a & (m - 1)) == 0) break; }
    m >>= 1;
    b = b & 1 ? (b >> 1) ^ CRC_POLY : b >> 1;
  }
  return p;
}

// CRC-32 of A‖B from crc(A), crc(B) and |B| (zlib's crc32_combine): crc(A)·x^(8|B|) ⊕ crc(B)
__host__ __device__ inline uint32_t crc_combine(uint32_t c1, uint32_t c2, long long len2) {
  uint32_t sq = 1u << 23;  // x^8 (one byte); x^k is bit 31 - k
  uint32_t p = 1u << 31;   // x^0
  for (unsigned long long n = (unsigned long long)len2; n; n >>= 1) {
    if (n & 1) p = crc_multmodp(sq, p);
    sq = crc_multmodp(sq, sq);
  }
  return crc_multmodp(p, c1) ^ c2;
}

// One warp per block.  Every lane parses the same element (the tag bytes are broadcast loads), and the lanes copy its
// bytes; a copy whose offset is smaller than its length repeats the offset's period, so lane i reads from
// pos - offset + i mod offset, all before pos.  Every write is bounded by the block's declared length.  Then each lane
// takes the CRC-32 of one 32nd of the output and lane 0's combination is compared with the block's stored CRC.
__global__ void __launch_bounds__(AV_THREADS) avro_snappy_kernel(const uint8_t* file, const AvBlockDev* blk, int nb, uint8_t* arena, int32_t* status) {
  __shared__ uint32_t tab[256];
  for (int i = threadIdx.x; i < 256; i += blockDim.x) {
    uint32_t c = (uint32_t)i;
    for (int k = 0; k < 8; ++k) c = c & 1 ? (c >> 1) ^ CRC_POLY : c >> 1;
    tab[i] = c;
  }
  __syncthreads();
  const int b = blockIdx.x * (AV_THREADS / 32) + (int)(threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (b >= nb) return;
  const AvBlockDev B = blk[b];
  const uint8_t* in = file + B.src;
  const uint8_t* const iend = in + B.src_len;
  uint8_t* const out = arena + B.start;
  const long long ulen = B.end - B.start;
  long long pos = 0;
  int code = AE_NONE;
  while (in < iend) {
    const unsigned t = *in++;
    long long len;
    if ((t & 3) == 0) {
      unsigned long long l = t >> 2;
      if (l >= 60) {
        const int nx = (int)l - 59;
        if (iend - in < nx) { code = AE_SNAPPY_BAD; break; }
        l = 0;
        for (int k = 0; k < nx; ++k) l |= (unsigned long long)in[k] << (8 * k);
        in += nx;
      }
      len = (long long)l + 1;
      if (iend - in < len) { code = AE_SNAPPY_BAD; break; }
      if (len > ulen - pos) { code = AE_SNAPPY_OVERRUN; break; }
      for (long long i = lane; i < len; i += 32) out[pos + i] = in[i];
      in += len;
    } else {
      long long off;
      if ((t & 3) == 1) {
        if (iend - in < 1) { code = AE_SNAPPY_BAD; break; }
        len = 4 + ((t >> 2) & 7); off = ((long long)(t >> 5) << 8) | in[0]; in += 1;
      } else if ((t & 3) == 2) {
        if (iend - in < 2) { code = AE_SNAPPY_BAD; break; }
        len = (t >> 2) + 1; off = in[0] | (in[1] << 8); in += 2;
      } else {
        if (iend - in < 4) { code = AE_SNAPPY_BAD; break; }
        len = (t >> 2) + 1; off = (long long)(in[0] | (in[1] << 8) | (in[2] << 16) | ((unsigned)in[3] << 24)); in += 4;
      }
      if (off == 0 || off > pos) { code = AE_SNAPPY_BAD; break; }
      if (len > ulen - pos) { code = AE_SNAPPY_OVERRUN; break; }
      for (long long i = lane; i < len; i += 32) out[pos + i] = out[pos - off + (i < off ? i : i % off)];
    }
    pos += len;
    __syncwarp();  // the next element may copy these bytes
  }
  if (code == AE_NONE && pos != ulen) code = AE_SNAPPY_UNDERFILL;
  if (code == AE_NONE) {
    const long long per = (ulen + 31) / 32, a = lane * per, e = min(ulen, a + per);
    uint32_t c = 0xFFFFFFFFu;
    for (long long k = a; k < e; ++k) c = tab[(c ^ out[k]) & 0xFF] ^ (c >> 8);
    c ^= 0xFFFFFFFFu;
    uint32_t crc = __shfl_sync(0xffffffffu, c, 0);
    for (int l = 1; l < 32; ++l) {
      const uint32_t cl = __shfl_sync(0xffffffffu, c, l);
      const long long la = min(ulen, l * per), le = min(ulen, (l + 1) * per);
      crc = crc_combine(crc, cl, le - la);
    }
    const uint8_t* s = iend;  // big-endian CRC-32 of the uncompressed data
    const uint32_t want = ((uint32_t)s[0] << 24) | ((uint32_t)s[1] << 16) | ((uint32_t)s[2] << 8) | s[3];
    if (crc != want) code = AE_CRC;
  }
  if (lane == 0) status[b] = code;
}

// One thread per block: walk its records up to the batch's end, recording where each record of the batch starts and ends.
// A record the walk cannot get past is handed to avro_decode_kernel with the block's end as its end (it finds the first
// failing field); the records after it are unlocated (-1).  When that record lies before the batch, or the block failed
// to decompress, the error is reported here.
__global__ void avro_index_kernel(const __grid_constant__ AvParams P, const AvBlockDev* blk, int nb, const int32_t* status, long long* rec_start, long long* rec_end) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= nb) return;
  const AvBlockDev B = blk[b];
  const long long row_end = P.row0 + P.n;
  const int st = status ? status[b] : 0;
  if (st != AE_NONE) {
    atomicMin(P.error, ((unsigned long long)B.first_row << 8) | (unsigned)st);
    for (long long r = max(B.first_row, P.row0); r < min(B.first_row + B.count, row_end); ++r) rec_start[r - P.row0] = -1;
    return;
  }
  const uint8_t* p = P.arena + B.start;
  const uint8_t* const end = P.arena + B.end;
  for (long long j = 0; j < B.count; ++j) {
    const long long r = B.first_row + j;
    if (r >= row_end) break;
    const uint8_t* s = p;
    int err = AE_NONE;
    const bool ok = av_record<false>(P, p, end, P.arena, 0, err);
    if (r >= P.row0) { rec_start[r - P.row0] = s - P.arena; rec_end[r - P.row0] = ok ? p - P.arena : B.end; }
    if (!ok) {
      if (r < P.row0) atomicMin(P.error, ((unsigned long long)r << 8) | (unsigned)err);
      for (long long q = max(r + 1, P.row0); q < min(B.first_row + B.count, row_end); ++q) rec_start[q - P.row0] = -1;
      return;
    }
  }
}

// One thread per record; the CTA's records (one contiguous arena range) are staged in shared memory by one TMA copy.
__global__ void __launch_bounds__(AV_THREADS) avro_decode_kernel(const __grid_constant__ AvParams P) {
  extern __shared__ __align__(16) uint8_t av_stage[];
  __shared__ __align__(8) unsigned long long s_bar;
  __shared__ long long s_stage_off;  // arena offset of av_stage[0]
  __shared__ int s_staged;
  const long long i0 = (long long)blockIdx.x * AV_THREADS;
  const long long i = i0 + threadIdx.x;
  if (threadIdx.x == 0) {
    s_staged = 0;
    if (P.stage_bytes > 0) {
      const int rows = (int)((P.n - i0) < AV_THREADS ? (P.n - i0) : AV_THREADS);
      const long long o0 = P.rec_start[i0], o1 = P.rec_end[i0 + rows - 1];
      if (o0 >= 0 && P.rec_start[i0 + rows - 1] >= 0 && o1 > o0) {
        const uintptr_t a0 = reinterpret_cast<uintptr_t>(P.arena + o0), a1 = reinterpret_cast<uintptr_t>(P.arena + o1);
        const uintptr_t lo = a0 & ~(uintptr_t)15, hi = (a1 + 15) & ~(uintptr_t)15;
        if (hi - lo <= (uintptr_t)P.stage_bytes) {
          mbar_init(&s_bar, 1);
          mbar_fence_init();
          mbar_expect_tx(&s_bar, (unsigned)(hi - lo));
          tma_load_1d(av_stage, reinterpret_cast<const void*>(lo), (unsigned)(hi - lo), &s_bar);
          s_stage_off = o0 - (long long)(a0 - lo);
          s_staged = 1;
        }
      }
    }
  }
  __syncthreads();
  const bool staged = s_staged != 0;
  if (staged) mbar_wait(&s_bar, 0);
  if (i >= P.n) return;
  const long long s = P.rec_start[i];
  if (s < 0) return;
  const uint8_t* const origin = staged ? av_stage - s_stage_off : P.arena;
  const uint8_t* p = origin + s;
  const uint8_t* const end = origin + P.rec_end[i];
  int err = AE_NONE;
  if (!av_record<true>(P, p, end, origin, i, err)) atomicMin(P.error, ((unsigned long long)(P.row0 + i) << 8) | (unsigned)err);
}

Batch avro_batch(AvroFile& f, const BufferPtr& file_dev, int64_t r0, int64_t n, cudaStream_t stream) {
  // the blocks that hold rows [r0, r0 + n): the first whose rows reach past r0, up to the first that starts at r0 + n
  auto by_row = [](const AvroBlock& b, int64_t r) { return b.first_row + b.count <= r; };
  const size_t b0 = (size_t)(std::lower_bound(f.blocks.begin(), f.blocks.end(), r0, by_row) - f.blocks.begin());
  size_t b1 = b0;
  while (b1 < f.blocks.size() && f.blocks[b1].first_row < r0 + n) ++b1;
  std::vector<AvBlockDev> hb;
  int64_t arena_bytes = 0;
  for (size_t k = b0; k < b1; ++k) {
    const AvroBlock& a = f.blocks[k];
    if (a.count == 0) continue;  // no rows: its data is not decoded
    hb.emplace_back();
    AvBlockDev& d = hb.back();
    d.first_row = a.first_row; d.count = a.count;
    if (f.snappy) { d.start = arena_bytes; d.end = arena_bytes + a.ulen; d.src = a.data_off + a.pre; d.src_len = a.size - 4 - a.pre; arena_bytes += a.ulen; }
    else { d.start = a.data_off; d.end = a.data_off + a.size; d.src = 0; d.src_len = 0; }
  }
  const int nb = (int)hb.size();
  BufferPtr dblk = device_alloc(sizeof(AvBlockDev) * (size_t)std::max(nb, 1));
  BufferPtr hblk = pinned_alloc(sizeof(AvBlockDev) * (size_t)std::max(nb, 1));
  memcpy(hblk.get(), hb.data(), sizeof(AvBlockDev) * (size_t)nb);
  ARK_CUDA(cudaMemcpyAsync(dblk.get(), hblk.get(), sizeof(AvBlockDev) * (size_t)nb, cudaMemcpyHostToDevice, stream));
  BufferPtr arena = file_dev, status;
  if (f.snappy) {
    arena = device_alloc((size_t)arena_bytes + 64);
    status = device_alloc((size_t)std::max(nb, 1) * 4);
    KernelTimer t("avro_snappy_kernel", stream);
    avro_snappy_kernel<<<(unsigned)ceil_div(nb, AV_THREADS / 32), AV_THREADS, 0, stream>>>((const uint8_t*)file_dev.get(), (const AvBlockDev*)dblk.get(), nb,
                                                                                         (uint8_t*)arena.get(), (int32_t*)status.get());
  }
  const size_t nf = f.fields.size();
  AvParams P;
  memset(&P, 0, sizeof P);
  P.arena = (const uint8_t*)arena.get(); P.n = n; P.row0 = r0; P.n_fields = (int)nf;
  BufferPtr rs = device_alloc((size_t)n * 8), re = device_alloc((size_t)n * 8), err = device_alloc(8);
  ARK_CUDA(cudaMemsetAsync(err.get(), 0xFF, 8, stream));
  ARK_CUDA(cudaMemsetAsync(rs.get(), 0xFF, (size_t)n * 8, stream));  // unlocated until avro_index_kernel finds it
  P.rec_start = (const long long*)rs.get(); P.rec_end = (const long long*)re.get(); P.error = (unsigned long long*)err.get();
  // a record's strings lie inside the record, so the bytes the batch's blocks span bound every string column's total
  int64_t bound = 0;
  for (auto& d : hb) bound += d.end - d.start;
  std::vector<StagedColumn> cols;
  for (size_t k = 0; k < nf; ++k) {
    const AvroField& a = f.fields[k];
    cols.push_back(stage_column(av_dtype(a.kind), n, a.null_branch >= 0, false, stream));
    StagedColumn& s = cols.back();
    s.bound = bound; s.what = "avro input: column '" + a.name + "'";
    AvField& F = P.f[k];
    F.kind = a.kind; F.null_branch = a.null_branch;
    F.values = s.values.get(); F.valid = (uint8_t*)s.valid.get(); F.str_src = (long long*)s.src.get(); F.str_len = (int32_t*)s.len.get();
    if (s.values) F.width = a.kind == AK_BOOL ? 1 : (uint8_t)fixed_width(s.type);
  }
  {
    KernelTimer t("avro_index_kernel", stream);
    avro_index_kernel<<<(unsigned)ceil_div(nb, 128), 128, 0, stream>>>(P, (const AvBlockDev*)dblk.get(), nb, (const int32_t*)status.get(), (long long*)rs.get(), (long long*)re.get());
  }
  {
    P.stage_bytes = record_stage_window(hb.empty() ? 0 : hb.back().end - hb.front().start, n, AV_THREADS);
    KernelTimer t("avro_decode_kernel", stream);
    avro_decode_kernel<<<(unsigned)ceil_div(n, AV_THREADS), AV_THREADS, (size_t)P.stage_bytes + 32, stream>>>(P);
  }
  ARK_CUDA(cudaGetLastError());
  settle_columns(cols, err.get(), 8, [&](const void* h) {
    const unsigned long long e = *(const unsigned long long*)h;
    if (e == ~0ull) return;
    const int64_t row = (int64_t)(e >> 8);
    auto it = std::lower_bound(f.blocks.begin(), f.blocks.end(), row, by_row);
    av_fail(std::string(av_err_text((int)(e & 0xFF))) + " in record " + std::to_string(row) + " (block at offset " + std::to_string(it->offset) + ")");
  }, stream);

  Batch out;
  out.num_rows = n;
  for (size_t k = 0; k < nf; ++k) {
    const AvroField& a = f.fields[k];
    const DType t = av_dtype(a.kind);
    Column c = finish_column(cols[k], Field{a.name, t, a.null_branch >= 0 || a.kind == AK_NULL, dtype_arrow_format(t)}, [&](const StagedColumn& s, uint8_t* bytes) {
      if (s.total) launch_span_copy(P.arena, nullptr, (const long long*)s.src.get(), (const int32_t*)s.offsets.get(), n, bytes, stream);
    }, stream);
    if (a.kind == AK_NULL) c.null_count = n;
    out.cols.push_back(std::move(c));
  }
  ARK_CUDA(cudaGetLastError());
  ARK_CUDA(cudaStreamSynchronize(stream));
  return out;
}

struct AvroFormat : FileFormat {
  AvroFile f;
  BufferPtr file_dev;

  // the header (schema and codec), whose errors need no device
  void open(const HostFile& file) override {
    f = AvroFile();
    std::string h;
    char buf[1 << 16];
    while (true) {
      const size_t got = file.read_some((int64_t)h.size(), buf, sizeof buf);
      h.append(buf, got);
      const int64_t len = parse_header(f, h, got < sizeof buf);
      if (len > 0) { f.header_bytes = len; f.pos = len; return; }
    }
  }
  // the block table, built while the upload's chunks pass
  void scan(const uint8_t* p, size_t n, int64_t base) override { avro_scan(f, p, n, base); }
  int64_t prepare(const BufferPtr& dev, int64_t, cudaStream_t) override {
    avro_scan_end(f);
    file_dev = dev;
    return f.rows;
  }
  Batch batch(int64_t r0, int64_t n, cudaStream_t stream) override { return avro_batch(f, file_dev, r0, n, stream); }
};

}  // namespace

std::unique_ptr<FileFormat> make_avro_format() { return std::make_unique<AvroFormat>(); }

}  // namespace ark
