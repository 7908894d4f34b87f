// arrow_ipc.cu — the `file` input's `arrow` type: Arrow IPC files (format 1.x, the footer-indexed "file" form), read on
// the device.
//
// An IPC file's body buffers already are Arrow columns, so the device work is validation, re-batching and, for
// compressed bodies, LZ4 decompression.  connect() (ipc_open) reads every piece of metadata with pread before the device
// is touched: the leading and trailing `ARROW1` magic, the footer, the schema, and for every record batch its message
// (continuation-marker or legacy pre-0.15 length prefix), its field nodes and buffers and, in a compressed body, the
// 8-byte uncompressed-length prefix of every buffer.  The flatbuffers are read by the bounds-checked reader below.  Every
// buffer's range, node length and (uncompressed) size is checked against the body, the file and what its type needs.
// The file's bytes then go to HBM once (the file driver's upload).
//
// A read of rows [r0, r0 + n) decodes every stored record batch it touches for the first time, as a whole, and keeps
// the last one when it reaches into the next read:
//   ipc_lz4_kernel       one warp per LZ4 frame, every compressed buffer of those batches in one launch, into an arena
//                        laid out from the prefixes read at connect; uncompressed and raw (-1) buffers are not copied;
//   ipc_validate_kernel  one launch over the Utf8 / Binary columns (offsets non-negative, non-decreasing and inside the
//                        data buffer; Utf8 slots, NULL ones too, valid UTF-8) and the columns whose node has
//                        null_count > 0 (the bitmap's zero bits over [0, length) equal it).  A node with null_count 0
//                        carries no validity: its bitmap is ignored, as arrow-rs and Arrow C++ do.
// Both report into one error word per read: atomicMin of (batch, column, row, code), so the first failure in file order
// wins.  The output batch is then a view of one decoded batch (no copy: its buffers point into the uploaded file or the
// arena) or, when it spans stored batches, their slices joined by concat_device.
// Types: Null, Boolean, Int32, Int64, UInt32, UInt64, Float32, Float64, Utf8 and Binary, nullable or not.  Every other
// type (dictionary-encoded, nested, Large* / View, Int8 / Int16, temporal, decimal, …), a big-endian schema and a ZSTD
// body are ARK_ERR_UNSUPPORTED from connect().  Custom metadata is not carried.
// Errors are Process "Read input failed: Arrow IPC error: <what> (record batch k[, column 'c'][, row r])": a check that
// needs only metadata and length prefixes fails connect(), one that needs body bytes fails the read of the batch.
// oracle/arrow_ipc_oracle.py restates all of this in Python; tests/test_arrow_ipc_input_gpu.py compares the two.
#include <algorithm>
#include <array>
#include <climits>
#include <cstring>

#include "bitmap.h"
#include "file_input.h"
#include "utf8.cuh"
#include "varlen.h"

namespace ark {

namespace {

constexpr int IPC_MAX_FIELDS = 1024;           // the column's 10 bits of the error key
constexpr int64_t IPC_MAX_ROWS = INT32_MAX;    // the row's 31 bits
constexpr int IPC_GROUP = 1 << 19;             // stored batches decoded per launch: the batch's 19 bits
constexpr int LZ_THREADS = 128;
constexpr int VAL_THREADS = 256;
constexpr int64_t VAL_CHUNK = VAL_THREADS * 32;  // rows per CTA of ipc_validate_kernel

// error codes, in their order of precedence within one (batch, column, row)
enum IpcErr : int { IE_NONE = 0, IE_LZ4_BAD, IE_LZ4_CSIZE, IE_LZ4_TRUNC, IE_LZ4_ZERO, IE_LZ4_OFFSET, IE_LZ4_OVERRUN,
                    IE_LZ4_UNDERFILL, IE_LZ4_CHECKSUM, IE_LZ4_TRAIL, IE_OFFSETS, IE_UTF8, IE_NULLS };

const char* ipc_err_text(int code) {
  switch (code) {
    case IE_LZ4_BAD: return "malformed LZ4 frame header";
    case IE_LZ4_CSIZE: return "LZ4 frame content size differs from the buffer's uncompressed length";
    case IE_LZ4_TRUNC: return "truncated LZ4 frame";
    case IE_LZ4_ZERO: return "LZ4 match with offset 0";
    case IE_LZ4_OFFSET: return "LZ4 match reaches before the start of its output";
    case IE_LZ4_OVERRUN: return "LZ4 frame overruns the buffer's uncompressed length";
    case IE_LZ4_UNDERFILL: return "LZ4 frame underfills the buffer's uncompressed length";
    case IE_LZ4_CHECKSUM: return "LZ4 frame checksum mismatch";
    case IE_LZ4_TRAIL: return "bytes after the end of the LZ4 frame";
    case IE_OFFSETS: return "offsets are negative, decreasing or past the end of the data buffer";
    case IE_UTF8: return "invalid UTF-8 in a Utf8 value";
    case IE_NULLS: return "null count differs from the validity bitmap";
    default: return "malformed data";
  }
}

// error key: batch (relative to the launch group) << 45 | column << 35 | row << 4 | code; a whole-column failure has row 0
// (LZ4: before every row check) or the largest row (null count: after every row check)
__host__ __device__ inline unsigned long long ipc_key(long long batch, int col, long long row, int code) {
  return ((unsigned long long)batch << 45) | ((unsigned long long)col << 35) | ((unsigned long long)row << 4) | (unsigned)code;
}
constexpr long long IPC_ROW_LAST = (1ll << 31) - 1;

// xxHash32 (the LZ4 frame format's checksum), seed 0
__host__ __device__ inline uint32_t rotl32(uint32_t x, int r) { return (x << r) | (x >> (32 - r)); }
__host__ __device__ inline uint32_t rd32(const uint8_t* p) { return (uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) | ((uint32_t)p[3] << 24); }
__host__ __device__ inline uint32_t xxh32(const uint8_t* p, long long len) {
  const uint32_t P1 = 2654435761u, P2 = 2246822519u, P3 = 3266489917u, P4 = 668265263u, P5 = 374761393u;
  const uint8_t* const end = p + len;
  uint32_t h;
  if (len >= 16) {
    uint32_t v1 = P1 + P2, v2 = P2, v3 = 0, v4 = 0u - P1;
    for (; end - p >= 16; p += 16) {
      v1 = rotl32(v1 + rd32(p) * P2, 13) * P1;
      v2 = rotl32(v2 + rd32(p + 4) * P2, 13) * P1;
      v3 = rotl32(v3 + rd32(p + 8) * P2, 13) * P1;
      v4 = rotl32(v4 + rd32(p + 12) * P2, 13) * P1;
    }
    h = rotl32(v1, 1) + rotl32(v2, 7) + rotl32(v3, 12) + rotl32(v4, 18);
  } else {
    h = P5;
  }
  h += (uint32_t)len;
  for (; end - p >= 4; p += 4) h = rotl32(h + rd32(p) * P3, 17) * P4;
  for (; p < end; ++p) h = rotl32(h + *p * P5, 11) * P1;
  h ^= h >> 15; h *= P2; h ^= h >> 13; h *= P3; h ^= h >> 16;
  return h;
}

// ---- flatbuffers ---------------------------------------------------------------------------------------------------
// A bounds-checked reader of the few tables the footer and the messages use.  Any read outside the buffer throws
// FbError, which the caller turns into its own message.
struct FbError {};

struct Fb {
  const uint8_t* p;
  size_t n;
  template <class T> T rd(size_t at) const {
    if (at > n || sizeof(T) > n - at) throw FbError{};
    T v;
    memcpy(&v, p + at, sizeof(T));
    return v;
  }
};

struct FbTable {
  const Fb* fb = nullptr;
  size_t pos = 0, vt = 0;
  uint16_t vlen = 0;
  bool present = false;

  static FbTable at(const Fb& fb, size_t pos) {
    FbTable t;
    t.fb = &fb; t.pos = pos; t.present = true;
    const int64_t vt = (int64_t)pos - fb.rd<int32_t>(pos);
    if (vt < 0 || (size_t)vt >= fb.n) throw FbError{};
    t.vt = (size_t)vt;
    t.vlen = fb.rd<uint16_t>(t.vt);
    if (t.vlen < 4 || (t.vlen & 1)) throw FbError{};
    return t;
  }
  size_t field(int i) const {  // the field's position, or 0 when absent
    if (4 + 2 * (size_t)i + 2 > vlen) return 0;
    const uint16_t o = fb->rd<uint16_t>(vt + 4 + 2 * (size_t)i);
    return o ? pos + o : 0;
  }
  template <class T> T scalar(int i, T dflt) const { const size_t f = field(i); return f ? fb->rd<T>(f) : dflt; }
  FbTable table(int i) const {
    const size_t f = field(i);
    if (!f) return FbTable{};
    return at(*fb, f + fb->rd<uint32_t>(f));
  }
  // a vector of `elem`-byte elements: (position of element 0, count); count 0 when absent
  std::pair<size_t, size_t> vec(int i, size_t elem) const {
    const size_t f = field(i);
    if (!f) return {0, 0};
    const size_t v = f + fb->rd<uint32_t>(f);
    const size_t cnt = fb->rd<uint32_t>(v);
    if (v + 4 > fb->n || cnt > (fb->n - v - 4) / elem) throw FbError{};
    return {v + 4, cnt};
  }
  FbTable elem_table(std::pair<size_t, size_t> v, size_t k) const { const size_t e = v.first + 4 * k; return at(*fb, e + fb->rd<uint32_t>(e)); }
  std::string str(int i) const {
    const auto v = vec(i, 1);
    return v.second ? std::string((const char*)fb->p + v.first, v.second) : std::string();
  }
};

FbTable fb_root(const Fb& fb) { return FbTable::at(fb, fb.rd<uint32_t>(0)); }

// Schema.fbs: the Type union's members
const char* type_name(int t) {
  static const char* names[] = {"NONE", "Null", "Int", "FloatingPoint", "Binary", "Utf8", "Bool", "Decimal", "Date", "Time",
                                "Timestamp", "Interval", "List", "Struct", "Union", "FixedSizeBinary", "FixedSizeList", "Map",
                                "Duration", "LargeBinary", "LargeUtf8", "LargeList", "RunEndEncoded", "BinaryView", "Utf8View",
                                "ListView", "LargeListView"};
  return t >= 0 && t < (int)(sizeof names / sizeof names[0]) ? names[t] : "unknown";
}

}  // namespace

struct IpcField {
  std::string name;
  DType type;
  bool nullable;
};

// one body buffer: `len` stored bytes at file offset `src`, `size` bytes once decoded (LZ4 frame when `lz4`)
struct IpcBuf {
  int64_t src = 0, len = 0, size = 0;
  bool lz4 = false;
};

struct IpcNode {
  int64_t length = 0, null_count = 0;
  IpcBuf buf[3];  // validity, then values (Bool and fixed width) or offsets and data (Utf8 / Binary)
};

struct IpcStored {
  int64_t offset = 0;   // file offset of the block's message
  int64_t rows = 0, first_row = 0;
  std::vector<IpcNode> nodes;
};

struct IpcFile {
  std::vector<IpcField> fields;
  std::vector<IpcStored> batches;
  int64_t rows = 0;
  // the stored batch the last read decoded and did not finish, as a batch of all its rows
  int64_t carry_index = -1;
  Batch carry;
};

namespace {

[[noreturn]] void ipc_fail(const std::string& what) { fail(ARK_ERR_PROCESS, "Read input failed: Arrow IPC error: " + what); }

std::string at_batch(size_t k) { return " (record batch " + std::to_string(k) + ")"; }
std::string at_col(size_t k, const std::string& c) { return " (record batch " + std::to_string(k) + ", column '" + c + "')"; }

int n_buffers(DType t) { return t == DType::Null ? 0 : (t == DType::Utf8 || t == DType::Binary) ? 3 : 2; }

// a field's Arrow type → the column type, or a description of what is not read
bool field_type(const FbTable& f, DType* out, std::string* desc) {
  const int tt = f.scalar<uint8_t>(2, 0);
  const FbTable t = f.table(3);
  std::string d = type_name(tt);
  DType r = DType::Null;
  bool ok = true;
  switch (tt) {
    case 1: r = DType::Null; break;
    case 2: {
      const int bits = t.present ? t.scalar<int32_t>(0, 0) : 0;
      const bool sig = t.present && t.scalar<uint8_t>(1, 0) != 0;
      d = std::string(sig ? "Int" : "UInt") + std::to_string(bits);
      if (bits == 32) r = sig ? DType::Int32 : DType::UInt32;
      else if (bits == 64) r = sig ? DType::Int64 : DType::UInt64;
      else ok = false;
      break;
    }
    case 3: {
      const int prec = t.present ? t.scalar<int16_t>(0, 0) : 0;
      d = prec == 0 ? "Float16" : prec == 1 ? "Float32" : "Float64";
      if (prec == 1) r = DType::Float32;
      else if (prec == 2) r = DType::Float64;
      else ok = false;
      break;
    }
    case 4: r = DType::Binary; break;
    case 5: r = DType::Utf8; break;
    case 6: r = DType::Bool; break;
    default: ok = false;
  }
  if (f.table(4).present) { d = "dictionary-encoded " + d; ok = false; }
  *out = r;
  *desc = d;
  return ok;
}

int64_t le64(const std::string& s, size_t at) { int64_t v; memcpy(&v, s.data() + at, 8); return v; }
int32_t le32(const std::string& s, size_t at) { int32_t v; memcpy(&v, s.data() + at, 4); return v; }

void read_batch_meta(IpcFile& f, const HostFile& fd, size_t k, int64_t off, int64_t meta_len, int64_t body_len, int64_t end) {
  IpcStored S;
  S.offset = off;
  const std::string kb = at_batch(k);
  if (off < 8 || meta_len < 8 || body_len < 0 || meta_len > end - off || body_len > end - off - meta_len) ipc_fail("block outside the file" + kb);
  const std::string meta = fd.read(off, meta_len);
  // continuation marker 0xFFFFFFFF then the length, or (before format 0.15) the length alone
  size_t fb0 = 4;
  int64_t len = le32(meta, 0);
  if (len == -1) { len = le32(meta, 4); fb0 = 8; }
  if (len <= 0 || len > meta_len - (int64_t)fb0) ipc_fail("malformed message" + kb);
  const Fb fb{(const uint8_t*)meta.data() + fb0, (size_t)len};
  const int64_t body = off + meta_len;
  const size_t nf = f.fields.size();
  int64_t nbuf = 0;
  for (auto& fl : f.fields) nbuf += n_buffers(fl.type);
  std::vector<std::pair<int64_t, int64_t>> bufs;
  bool lz4 = false;
  try {
    const FbTable msg = fb_root(fb);
    if (msg.scalar<uint8_t>(1, 0) != 3) ipc_fail("message is not a record batch" + kb);
    const FbTable rb = msg.table(2);
    if (!rb.present) throw FbError{};
    S.rows = rb.scalar<int64_t>(0, 0);
    if (S.rows < 0) ipc_fail("negative row count" + kb);
    if (S.rows > IPC_MAX_ROWS) fail(ARK_ERR_UNSUPPORTED, "arrow input: record batch " + std::to_string(k) + " holds more than 2^31 - 1 rows");
    const auto nodes = rb.vec(1, 16), buffers = rb.vec(2, 16);
    if (nodes.second != nf) ipc_fail("field node count differs from the schema" + kb);
    if ((int64_t)buffers.second != nbuf) ipc_fail("buffer count differs from the schema" + kb);
    S.nodes.resize(nf);
    for (size_t c = 0; c < nf; ++c) { S.nodes[c].length = fb.rd<int64_t>(nodes.first + 16 * c); S.nodes[c].null_count = fb.rd<int64_t>(nodes.first + 16 * c + 8); }
    for (size_t j = 0; j < buffers.second; ++j) bufs.push_back({fb.rd<int64_t>(buffers.first + 16 * j), fb.rd<int64_t>(buffers.first + 16 * j + 8)});
    const FbTable comp = rb.table(3);
    if (comp.present) {
      const int codec = comp.scalar<int8_t>(0, 0);
      if (codec == 1) fail(ARK_ERR_UNSUPPORTED, "arrow input: record batch " + std::to_string(k) + " has a ZSTD body, which is not decoded on the GPU (uncompressed and LZ4_FRAME are)");
      if (codec != 0 || comp.scalar<int8_t>(1, 0) != 0) ipc_fail("unknown body compression" + kb);
      lz4 = true;
    }
  } catch (const FbError&) {
    ipc_fail("malformed message" + kb);
  }
  size_t j = 0;
  for (size_t c = 0; c < nf; ++c) {
    const IpcField& F = f.fields[c];
    IpcNode& N = S.nodes[c];
    const std::string kc = at_col(k, F.name);
    if (N.length != S.rows) ipc_fail("node length differs from the batch length" + kc);
    if (N.null_count < 0 || N.null_count > N.length) ipc_fail("invalid null count" + kc);
    if (!F.nullable && N.null_count > 0 && F.type != DType::Null) ipc_fail("null values in a non-nullable field" + kc);
    for (int b = 0; b < n_buffers(F.type); ++b, ++j) {
      const int64_t o = bufs[j].first, l = bufs[j].second;
      if (o < 0 || l < 0 || o > body_len || l > body_len - o) ipc_fail("buffer outside the body" + kc);
      if ((body + o) % 8) ipc_fail("buffer not 8-byte aligned" + kc);
      IpcBuf& B = N.buf[b];
      B.src = body + o; B.len = l; B.size = l;
      if (lz4 && l > 0) {
        if (l < 8) ipc_fail("buffer shorter than its length prefix" + kc);
        const int64_t u = le64(fd.read(body + o, 8), 0);
        B.src += 8; B.len -= 8;
        if (u == -1) B.size = B.len;                 // stored raw
        else if (u == 0) B.size = B.len = 0;         // empty: the frame is not read
        else if (u < 0) ipc_fail("invalid uncompressed length" + kc);
        else { B.size = u; B.lz4 = true; }
      }
    }
    const int64_t n = N.length, bits = (n + 7) / 8;
    bool short_buf = F.type != DType::Null && N.null_count > 0 && N.buf[0].size < bits;
    const int w = fixed_width(F.type);
    if (w) short_buf = short_buf || N.buf[1].size < n * w;
    if (F.type == DType::Bool) short_buf = short_buf || N.buf[1].size < bits;
    if ((F.type == DType::Utf8 || F.type == DType::Binary) && n > 0) short_buf = short_buf || N.buf[1].size < (n + 1) * 4;
    if (short_buf) ipc_fail("buffer too short for its node" + kc);
  }
  S.first_row = f.rows;
  f.rows += S.rows;
  f.batches.push_back(std::move(S));
}

void ipc_open(IpcFile& f, const HostFile& fd) {
  const int64_t n = fd.size;
  if (n < 18 || fd.read(0, 6) != "ARROW1" || fd.read(n - 6, 6) != "ARROW1") ipc_fail("not an Arrow IPC file (bad magic)");
  const int64_t flen = le32(fd.read(n - 10, 4), 0);
  if (flen <= 0 || flen > n - 18) ipc_fail("footer out of range");
  const int64_t foot = n - 10 - flen;
  const std::string fbytes = fd.read(foot, flen);
  const Fb fb{(const uint8_t*)fbytes.data(), fbytes.size()};
  struct Block { int64_t off, meta, body; };
  std::vector<Block> blocks;
  try {
    const FbTable footer = fb_root(fb);
    const FbTable schema = footer.table(1);
    if (!schema.present) ipc_fail("the footer has no schema");
    if (schema.scalar<int16_t>(0, 0) != 0) fail(ARK_ERR_UNSUPPORTED, "arrow input: the schema is big-endian, which is not decoded on the GPU");
    const auto fields = schema.vec(1, 4);
    if (fields.second > (size_t)IPC_MAX_FIELDS) fail(ARK_ERR_UNSUPPORTED, "arrow input: more than 1024 fields in a schema");
    for (size_t i = 0; i < fields.second; ++i) {
      const FbTable fl = schema.elem_table(fields, i);
      IpcField F;
      F.name = fl.str(0);
      F.nullable = fl.scalar<uint8_t>(1, 0) != 0;
      std::string desc;
      if (!field_type(fl, &F.type, &desc)) fail(ARK_ERR_UNSUPPORTED, "arrow input: field '" + F.name + "' has type " + desc + ", which is not decoded on the GPU");
      f.fields.push_back(F);
    }
    const auto rbs = footer.vec(3, 24);
    for (size_t k = 0; k < rbs.second; ++k)
      blocks.push_back({fb.rd<int64_t>(rbs.first + 24 * k), (int64_t)fb.rd<int32_t>(rbs.first + 24 * k + 8), fb.rd<int64_t>(rbs.first + 24 * k + 16)});
  } catch (const FbError&) {
    ipc_fail("malformed footer");
  }
  for (size_t k = 0; k < blocks.size(); ++k) read_batch_meta(f, fd, k, blocks[k].off, blocks[k].meta, blocks[k].body, foot);
}

}  // namespace


namespace {

// ---- device --------------------------------------------------------------------------------------------------------
struct IpcFrame {
  long long src, src_len;  // file offset and bytes of the frame
  long long dst, ulen;     // arena offset and the declared uncompressed length
  unsigned long long key;  // ipc_key(batch, column, 0, 0)
};

// One warp per frame.  Every lane parses the same bytes (broadcast loads) and the lanes copy literals and matches; a
// match whose offset is smaller than its length repeats the offset's period, so lane i reads pos - off + i mod off, all
// written before (a __syncwarp follows every copy).  Every write is bounded by the declared length, every read by the
// frame.  A failure folds its key into *err.
__global__ void __launch_bounds__(LZ_THREADS) ipc_lz4_kernel(const uint8_t* file, const IpcFrame* frames, int nf, uint8_t* arena, unsigned long long* err) {
  const int w = blockIdx.x * (LZ_THREADS / 32) + (int)(threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (w >= nf) return;
  const IpcFrame F = frames[w];
  const uint8_t* in = file + F.src;
  const uint8_t* const iend = in + F.src_len;
  uint8_t* const out = arena + F.dst;
  const long long ulen = F.ulen;
  long long pos = 0;
  int code = IE_NONE;
  do {
    if (iend - in < 7) { code = IE_LZ4_TRUNC; break; }
    if (rd32(in) != 0x184D2204u) { code = IE_LZ4_BAD; break; }
    const unsigned flg = in[4], bd = in[5];
    if ((flg >> 6) != 1 || (flg & 3) || (bd & 0x8F) || ((bd >> 4) & 7) < 4) { code = IE_LZ4_BAD; break; }
    const bool indep = flg & 0x20, bsum = flg & 0x10, csize = flg & 0x08, csum = flg & 0x04;
    const long long max_block = 1ll << (8 + 2 * ((bd >> 4) & 7));
    const int desc = 2 + (csize ? 8 : 0);
    if (iend - in < 4 + desc + 1) { code = IE_LZ4_TRUNC; break; }
    if (((xxh32(in + 4, desc) >> 8) & 0xFF) != in[4 + desc]) { code = IE_LZ4_CHECKSUM; break; }
    if (csize) {
      unsigned long long cs = 0;
      for (int b = 7; b >= 0; --b) cs = (cs << 8) | in[6 + b];
      if (cs != (unsigned long long)ulen) { code = IE_LZ4_CSIZE; break; }
    }
    in += 4 + desc + 1;
    while (code == IE_NONE) {
      if (iend - in < 4) { code = IE_LZ4_TRUNC; break; }
      const uint32_t word = rd32(in);
      in += 4;
      if (word == 0) break;  // end mark
      const bool stored = word >> 31;
      const long long bsz = word & 0x7FFFFFFFu;
      if (bsz > max_block) { code = IE_LZ4_BAD; break; }
      if (iend - in < bsz + (bsum ? 4 : 0)) { code = IE_LZ4_TRUNC; break; }
      const uint8_t* const bend = in + bsz;
      if (bsum && xxh32(in, bsz) != rd32(bend)) { code = IE_LZ4_CHECKSUM; break; }
      const long long block0 = pos;
      if (stored) {
        if (bsz > ulen - pos) { code = IE_LZ4_OVERRUN; break; }
        for (long long i = lane; i < bsz; i += 32) out[pos + i] = in[i];
        pos += bsz;
      } else {
        const uint8_t* q = in;
        while (true) {
          if (q >= bend) { code = IE_LZ4_TRUNC; break; }
          const unsigned tok = *q++;
          long long lit = tok >> 4;
          if (lit == 15) {
            unsigned b;
            do { if (q >= bend) { code = IE_LZ4_TRUNC; break; } b = *q++; lit += b; } while (b == 255);
            if (code) break;
          }
          if (lit > bend - q) { code = IE_LZ4_TRUNC; break; }
          if (lit > ulen - pos) { code = IE_LZ4_OVERRUN; break; }
          for (long long i = lane; i < lit; i += 32) out[pos + i] = q[i];
          q += lit;
          pos += lit;
          __syncwarp();
          if (q == bend) break;  // the last sequence has literals only
          if (bend - q < 2) { code = IE_LZ4_TRUNC; break; }
          const long long off = q[0] | (q[1] << 8);
          q += 2;
          if (off == 0) { code = IE_LZ4_ZERO; break; }
          if (off > pos - (indep ? block0 : 0)) { code = IE_LZ4_OFFSET; break; }
          long long ml = tok & 15;
          if (ml == 15) {
            unsigned b;
            do { if (q >= bend) { code = IE_LZ4_TRUNC; break; } b = *q++; ml += b; } while (b == 255);
            if (code) break;
          }
          ml += 4;
          if (ml > ulen - pos) { code = IE_LZ4_OVERRUN; break; }
          // lane i reads pos - off + (i mod off); the phase advances by 32 mod off per round (no 64-bit division)
          const unsigned o = (unsigned)off, step = 32u % o;
          unsigned j = (unsigned)lane % o;
          for (long long i = lane; i < ml; i += 32) {
            out[pos + i] = out[pos - off + j];
            j += step;
            if (j >= o) j -= o;
          }
          pos += ml;
          __syncwarp();
        }
      }
      in = bend + (bsum ? 4 : 0);
    }
    if (code != IE_NONE) break;
    if (pos != ulen) { code = IE_LZ4_UNDERFILL; break; }
    if (csum) {
      if (iend - in < 4) { code = IE_LZ4_TRUNC; break; }
      if (xxh32(out, ulen) != rd32(in)) { code = IE_LZ4_CHECKSUM; break; }
      in += 4;
    }
    if (in != iend) code = IE_LZ4_TRAIL;
  } while (false);
  if (code != IE_NONE && lane == 0) atomicMin(err, F.key | (unsigned)code);
}

struct IpcCheck {
  const int32_t* offsets;   // Utf8 / Binary, or nullptr
  const uint8_t* data;
  long long data_len;
  const uint8_t* validity;  // checked against null_count when not nullptr
  long long n, null_count;
  long long chunk0;         // first chunk of this column in the launch's chunk space
  unsigned long long key;   // ipc_key(batch, column, 0, 0)
  int utf8;
};

// One CTA per VAL_CHUNK rows of one column.  Rows r of a string column: offsets[r] >= 0, offsets[r] <= offsets[r + 1] <=
// data_len, and (Utf8) the value is valid UTF-8.  A nullable column's zero bits are added to zeros[item]; the CTA that
// finishes the column last compares the total with the node's null count.
__global__ void __launch_bounds__(VAL_THREADS) ipc_validate_kernel(const IpcCheck* items, int ni, unsigned long long* zeros, unsigned* done, unsigned long long* err) {
  const long long chunk = blockIdx.x;
  int lo = 0, hi = ni - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (items[mid].chunk0 <= chunk) lo = mid; else hi = mid - 1;
  }
  const IpcCheck C = items[lo];
  const long long r0 = (chunk - C.chunk0) * VAL_CHUNK;
  if (C.offsets) {
    long long bad = LLONG_MAX;
    int bcode = IE_NONE;
    for (long long r = r0 + threadIdx.x; r < min(C.n, r0 + VAL_CHUNK); r += VAL_THREADS) {
      const long long a = C.offsets[r], b = C.offsets[r + 1];
      if (a < 0 || b < a || b > C.data_len) { bad = r; bcode = IE_OFFSETS; break; }
      if (C.utf8 && !utf8_valid(C.data + a, b - a)) { bad = r; bcode = IE_UTF8; break; }
    }
    if (bcode != IE_NONE) atomicMin(err, C.key | ((unsigned long long)bad << 4) | (unsigned)bcode);
  }
  if (C.validity) {
    __shared__ unsigned s_z;
    if (threadIdx.x == 0) s_z = 0;
    __syncthreads();
    unsigned z = 0;
    for (long long r = r0 + threadIdx.x * 32; r < min(C.n, r0 + (threadIdx.x + 1) * 32ll); ++r) z += ((C.validity[r >> 3] >> (r & 7)) & 1) ^ 1;
    if (z) atomicAdd(&s_z, z);
    __syncthreads();
    if (threadIdx.x == 0) {
      if (s_z) atomicAdd(&zeros[lo], (unsigned long long)s_z);
      __threadfence();
      const long long chunks = (C.n + VAL_CHUNK - 1) / VAL_CHUNK;
      if (atomicAdd(&done[lo], 1u) == (unsigned)(chunks - 1)) {
        __threadfence();
        const unsigned long long total = *(volatile unsigned long long*)&zeros[lo];
        if ((long long)total != C.null_count) atomicMin(err, C.key | ((unsigned long long)IPC_ROW_LAST << 4) | (unsigned)IE_NULLS);
      }
    }
  }
}

// A column of `rows` rows [a, a + m) as a view of `c` (the decoded stored batch's column, which starts at bit 0).
Column slice_column(const Column& c, int64_t a, int64_t m) {
  Column s = c;
  s.length = m;
  const int w = fixed_width(c.field.type);
  if (w) { s.data = c.data + a * w; s.data_bytes = m * w; }
  else if (c.field.type == DType::Bool) { s.data = c.data + a / 8; s.data_bit0 = (int32_t)(a % 8); s.data_bytes = (m + (a % 8) + 7) / 8; }
  else if (c.field.type == DType::Utf8 || c.field.type == DType::Binary) { s.offsets = c.offsets + a; s.data_bytes = -1; s.first_offset = 0; }
  if (c.field.type == DType::Null) s.null_count = m;
  else if (c.validity && m != c.length) { s.validity = c.validity + a / 8; s.validity_bit0 = (int32_t)(a % 8); s.null_count = -1; }
  return s;
}

}  // namespace

// Decodes stored batches `ks` (at most IPC_GROUP, each with rows): one LZ4 launch, one validation launch, one
// synchronisation; returns each as a batch of all its rows.
std::vector<Batch> ipc_decode(IpcFile& f, const BufferPtr& file_dev, const std::vector<size_t>& ks, cudaStream_t stream) {
  const size_t nf = f.fields.size();
  std::vector<IpcFrame> frames;
  int64_t arena_bytes = 0;
  std::vector<std::vector<std::array<int64_t, 3>>> aoff(ks.size());  // arena offset of each LZ4 buffer, else -1
  for (size_t g = 0; g < ks.size(); ++g) {
    const IpcStored& S = f.batches[ks[g]];
    aoff[g].assign(nf, {-1, -1, -1});
    for (size_t c = 0; c < nf; ++c)
      for (int b = 0; b < 3; ++b) {
        const IpcBuf& B = S.nodes[c].buf[b];
        if (!B.lz4) continue;
        aoff[g][c][b] = arena_bytes;
        frames.push_back({B.src, B.len, arena_bytes, B.size, ipc_key((long long)g, (int)c, 0, 0)});
        arena_bytes += round_up(B.size, 64);
      }
  }
  BufferPtr arena = frames.empty() ? nullptr : device_alloc((size_t)arena_bytes + 64);
  const uint8_t* file = (const uint8_t*)file_dev.get();
  auto ptr = [&](size_t g, size_t c, int b) -> const uint8_t* {
    return aoff[g][c][b] >= 0 ? (const uint8_t*)arena.get() + aoff[g][c][b] : file + f.batches[ks[g]].nodes[c].buf[b].src;
  };
  std::vector<IpcCheck> checks;
  long long chunks = 0;
  for (size_t g = 0; g < ks.size(); ++g) {
    const IpcStored& S = f.batches[ks[g]];
    for (size_t c = 0; c < nf; ++c) {
      const IpcField& F = f.fields[c];
      const IpcNode& N = S.nodes[c];
      const bool str = F.type == DType::Utf8 || F.type == DType::Binary;
      if (!str && N.null_count == 0) continue;
      if (F.type == DType::Null) continue;
      IpcCheck k{};
      k.offsets = str ? (const int32_t*)ptr(g, c, 1) : nullptr;
      k.data = str ? ptr(g, c, 2) : nullptr;
      k.data_len = str ? N.buf[2].size : 0;
      k.validity = N.null_count > 0 ? ptr(g, c, 0) : nullptr;
      k.n = N.length; k.null_count = N.null_count; k.chunk0 = chunks; k.key = ipc_key((long long)g, (int)c, 0, 0);
      k.utf8 = F.type == DType::Utf8;
      chunks += ceil_div(N.length, VAL_CHUNK);
      if (N.length > 0) checks.push_back(k);
    }
  }
  const size_t nc = checks.size();
  // one upload: [error word][zeros nc][done nc (u32)][frames][checks]
  const size_t zoff = 8, doff = zoff + 8 * nc, foff = round_up((int64_t)(doff + 4 * nc), 16), coff = foff + sizeof(IpcFrame) * frames.size();
  const size_t bytes = coff + sizeof(IpcCheck) * nc;
  BufferPtr h = pinned_alloc(bytes + 16), d = device_alloc(bytes + 16);
  memset(h.get(), 0, doff + 4 * nc);
  *(unsigned long long*)h.get() = ~0ull;
  memcpy((char*)h.get() + foff, frames.data(), sizeof(IpcFrame) * frames.size());
  memcpy((char*)h.get() + coff, checks.data(), sizeof(IpcCheck) * nc);
  ARK_CUDA(cudaMemcpyAsync(d.get(), h.get(), bytes, cudaMemcpyHostToDevice, stream));
  unsigned long long* derr = (unsigned long long*)d.get();
  if (!frames.empty()) {
    KernelTimer t("ipc_lz4_kernel", stream);
    ipc_lz4_kernel<<<(unsigned)ceil_div((int64_t)frames.size(), LZ_THREADS / 32), LZ_THREADS, 0, stream>>>(
        file, (const IpcFrame*)((char*)d.get() + foff), (int)frames.size(), (uint8_t*)arena.get(), derr);
  }
  if (nc) {
    KernelTimer t("ipc_validate_kernel", stream);
    ipc_validate_kernel<<<(unsigned)chunks, VAL_THREADS, 0, stream>>>((const IpcCheck*)((char*)d.get() + coff), (int)nc,
                                                                      (unsigned long long*)((char*)d.get() + zoff), (unsigned*)((char*)d.get() + doff), derr);
  }
  ARK_CUDA(cudaGetLastError());
  ARK_CUDA(cudaMemcpyAsync(h.get(), derr, 8, cudaMemcpyDeviceToHost, stream));
  ARK_CUDA(cudaStreamSynchronize(stream));
  const unsigned long long e = *(const unsigned long long*)h.get();
  if (e != ~0ull) {
    const size_t k = ks[(size_t)(e >> 45)];
    const size_t c = (size_t)((e >> 35) & 1023);
    const long long row = (long long)((e >> 4) & IPC_ROW_LAST);
    const int code = (int)(e & 15);
    std::string where = " (record batch " + std::to_string(k) + ", column '" + f.fields[c].name + "'";
    if (code == IE_OFFSETS || code == IE_UTF8) where += ", row " + std::to_string(row);
    ipc_fail(ipc_err_text(code) + where + ")");
  }
  std::vector<Batch> out(ks.size());
  for (size_t g = 0; g < ks.size(); ++g) {
    const IpcStored& S = f.batches[ks[g]];
    Batch& b = out[g];
    b.num_rows = S.rows;
    for (size_t c = 0; c < nf; ++c) {
      const IpcField& F = f.fields[c];
      const IpcNode& N = S.nodes[c];
      Column col;
      col.field.name = F.name; col.field.type = F.type; col.field.format = dtype_arrow_format(F.type); col.field.nullable = F.nullable;
      col.length = S.rows;
      bool from_arena = false;
      for (int j = 0; j < 3; ++j) from_arena = from_arena || aoff[g][c][j] >= 0;
      col.owners = {from_arena ? arena : file_dev};
      if (from_arena) col.owners.push_back(file_dev);  // raw buffers of the same column
      if (F.type == DType::Null) { col.null_count = S.rows; b.cols.push_back(std::move(col)); continue; }
      if (N.null_count > 0) { col.validity = ptr(g, c, 0); col.null_count = N.null_count; }
      if (F.type == DType::Utf8 || F.type == DType::Binary) {
        col.offsets = (const int32_t*)ptr(g, c, 1); col.data = ptr(g, c, 2); col.data_bytes = -1;
      } else {
        col.data = ptr(g, c, 1);
        col.data_bytes = F.type == DType::Bool ? (S.rows + 7) / 8 : S.rows * fixed_width(F.type);
      }
      b.cols.push_back(std::move(col));
    }
  }
  return out;
}

Batch ipc_batch(IpcFile& f, const BufferPtr& file_dev, int64_t r0, int64_t n, cudaStream_t stream) {
  // the stored batches with rows in [r0, r0 + n)
  auto by_row = [](const IpcStored& b, int64_t r) { return b.first_row + b.rows <= r; };
  size_t k = (size_t)(std::lower_bound(f.batches.begin(), f.batches.end(), r0, by_row) - f.batches.begin());
  std::vector<size_t> touched;
  for (; k < f.batches.size() && f.batches[k].first_row < r0 + n; ++k)
    if (f.batches[k].rows > 0) touched.push_back(k);
  std::vector<Batch> whole(touched.size());
  std::vector<size_t> todo, slot;
  for (size_t i = 0; i < touched.size(); ++i) {
    if ((int64_t)touched[i] == f.carry_index) whole[i] = f.carry;
    else { todo.push_back(touched[i]); slot.push_back(i); }
  }
  for (size_t g0 = 0; g0 < todo.size(); g0 += IPC_GROUP) {
    const std::vector<size_t> ks(todo.begin() + g0, todo.begin() + std::min(todo.size(), g0 + IPC_GROUP));
    std::vector<Batch> dec = ipc_decode(f, file_dev, ks, stream);
    for (size_t j = 0; j < ks.size(); ++j) whole[slot[g0 + j]] = std::move(dec[j]);
  }
  // slices; a NULL count of a partial slice is counted from its bitmap
  std::vector<Batch> pieces;
  std::vector<Column*> counted;
  for (size_t i = 0; i < touched.size(); ++i) {
    const IpcStored& S = f.batches[touched[i]];
    const int64_t a = std::max<int64_t>(r0, S.first_row) - S.first_row, e = std::min<int64_t>(r0 + n, S.first_row + S.rows) - S.first_row;
    Batch p;
    p.num_rows = e - a;
    for (auto& c : whole[i].cols) p.cols.push_back(slice_column(c, a, e - a));
    pieces.push_back(std::move(p));
  }
  for (auto& p : pieces) for (auto& c : p.cols) if (c.null_count < 0) counted.push_back(&c);
  if (!counted.empty()) {
    BufferPtr z = device_alloc(8 * counted.size()), hz = pinned_alloc(8 * counted.size());
    ARK_CUDA(cudaMemsetAsync(z.get(), 0, 8 * counted.size(), stream));
    for (size_t j = 0; j < counted.size(); ++j)
      count_zeros(counted[j]->validity, counted[j]->validity_bit0, counted[j]->length, (unsigned long long*)z.get() + j, stream);
    ARK_CUDA(cudaMemcpyAsync(hz.get(), z.get(), 8 * counted.size(), cudaMemcpyDeviceToHost, stream));
    ARK_CUDA(cudaStreamSynchronize(stream));
    for (size_t j = 0; j < counted.size(); ++j) {
      counted[j]->null_count = (int64_t)((const unsigned long long*)hz.get())[j];
      if (counted[j]->null_count == 0) counted[j]->validity = nullptr;
    }
  }
  {
    std::vector<Column*> all;  // one round trip for every string slice's extent
    for (auto& p : pieces) for (auto& c : p.cols) all.push_back(&c);
    resolve_varlen_extents_many(all, stream);
  }
  // keep the last stored batch when the next read starts inside it
  if (!touched.empty()) {
    const IpcStored& L = f.batches[touched.back()];
    if (L.first_row + L.rows > r0 + n) { f.carry_index = (int64_t)touched.back(); f.carry = whole.back(); }
    else { f.carry_index = -1; f.carry = Batch(); }
  }
  if (pieces.size() == 1) return std::move(pieces[0]);
  const size_t nf = f.fields.size();
  std::vector<int64_t> nulls(nf, 0);
  for (size_t c = 0; c < nf; ++c) {
    int64_t bytes = 0;
    for (auto& p : pieces) { bytes += std::max<int64_t>(p.cols[c].data_bytes, 0); nulls[c] += p.cols[c].null_count; }
    if ((f.fields[c].type == DType::Utf8 || f.fields[c].type == DType::Binary) && bytes > INT32_MAX)
      fail(ARK_ERR_PROCESS, "file input: column '" + f.fields[c].name + "' of a batch of " + std::to_string(n) + " rows exceeds 2 GiB; lower batch_size");
  }
  Batch out = concat_device(pieces, stream);
  for (size_t c = 0; c < nf; ++c) {
    Column& oc = out.cols[c];
    oc.null_count = nulls[c];
    if (nulls[c] == 0) oc.validity = nullptr;
  }
  return out;
}

namespace {

struct IpcFormat : FileFormat {
  IpcFile f;
  BufferPtr file_dev;

  // every piece of metadata, whose errors need no device
  void open(const HostFile& file) override {
    f = IpcFile();
    ipc_open(f, file);
  }
  int64_t prepare(const BufferPtr& dev, int64_t, cudaStream_t) override {
    file_dev = dev;
    return f.rows;
  }
  Batch batch(int64_t r0, int64_t n, cudaStream_t stream) override { return ipc_batch(f, file_dev, r0, n, stream); }
};

}  // namespace

std::unique_ptr<FileFormat> make_arrow_ipc_format() { return std::make_unique<IpcFormat>(); }

}  // namespace ark
