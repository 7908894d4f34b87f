// ipc_exchange.cu — the repartition exchange of GROUP BY / JOIN over peer memory (one process per GPU, one
// node): each rank publishes its hash-partitioned batch as CUDA IPC handles; every receiver then PULLS its
// slice of every peer's batch with ONE segmented-copy launch (concat_copy_kernel + offset rebase) whose
// sources are peer-mapped pointers, i.e. the transfer over NVLink and the concatenation / offset rebasing
// of the received partitions are the same kernel.  Replaces one ncclSend/Recv group per column buffer
// (SURVEY.md §8(e); DataFusion's RepartitionExec(Hash) is in-process in the reference,
// crates/arkflow-plugin/src/processor/sql.rs:126-129).  The NCCL all-to-all in arkflow_b200/dist.py stays as
// the fallback (memory that cannot be exported, e.g. torch's expandable segments) and as the test oracle.
#include <unistd.h>

#include <map>
#include <mutex>

#include "abi.h"

namespace ark {

Batch concat_device(std::vector<Batch>& ins, cudaStream_t stream);
bool device_alloc_range(const void* p, unsigned long long* base, size_t* size);

namespace {

constexpr uint32_t IPC_MAGIC = 0x41524B49u;  // "ARKI"

struct IpcBuf {
  uint8_t handle[64];   // cudaIpcMemHandle_t of the allocation that holds the buffer
  uint64_t offset;      // of the buffer inside that allocation
  uint64_t raw;         // the exporter's own device pointer (used when importer == exporter)
  int32_t present;
  int32_t pad;
};
struct IpcCol {
  char name[64];
  char format[8];
  int32_t dtype, nullable;
  int64_t length, null_count;
  int32_t validity_bit0, data_bit0;
  IpcBuf validity, first, second;  // first = values (fixed / bool) or offsets (var-len); second = var-len bytes
};
struct IpcHeader {
  uint32_t magic;
  int32_t pid, device, n_cols;
  int64_t num_rows;
};
static_assert(sizeof(cudaIpcMemHandle_t) == 64, "cudaIpcMemHandle_t is 64 bytes");

void export_buf(const void* p, IpcBuf* b) {
  memset(b, 0, sizeof *b);
  if (!p) return;
  unsigned long long base = 0;
  size_t size = 0;
  if (!device_alloc_range(p, &base, &size)) fail(ARK_ERR_UNSUPPORTED, "ipc export: pointer is not inside a CUDA allocation");
  cudaIpcMemHandle_t h;
  cudaError_t e = cudaIpcGetMemHandle(&h, (void*)(uintptr_t)base);
  if (e != cudaSuccess) {
    cudaGetLastError();
    fail(ARK_ERR_UNSUPPORTED, std::string("ipc export: ") + cudaGetErrorString(e) + " (memory not created by cudaMalloc?)");
  }
  device_pool().mark_exported((const void*)(uintptr_t)base);  // peers cache the mapping: the block must outlive trim()
  export_pool().mark_exported((const void*)(uintptr_t)base);
  memcpy(b->handle, &h, 64);
  b->offset = (uint64_t)((unsigned long long)(uintptr_t)p - base);
  b->raw = (uint64_t)(uintptr_t)p;
  b->present = 1;
}

// opened peer allocations, by handle bytes.  An exported pool block is never returned to the driver while the
// process lives (export_buf marks it; BlockPool::trim skips marked blocks), so a cached mapping stays valid.
const uint8_t* open_buf(const IpcBuf& b, bool same_process) {
  if (!b.present) return nullptr;
  if (same_process) return (const uint8_t*)(uintptr_t)b.raw;
  static std::mutex mu;
  static std::map<std::string, void*> opened;
  std::lock_guard<std::mutex> l(mu);
  const std::string key((const char*)b.handle, 64);
  auto it = opened.find(key);
  void* base = nullptr;
  if (it != opened.end()) base = it->second;
  else {
    cudaIpcMemHandle_t h;
    memcpy(&h, b.handle, 64);
    ARK_CUDA(cudaIpcOpenMemHandle(&base, h, cudaIpcMemLazyEnablePeerAccess));
    opened[key] = base;
  }
  return (const uint8_t*)base + b.offset;
}

}  // namespace

std::vector<uint8_t> ipc_export(const Batch& b) {
  int dev = 0;
  ARK_CUDA(cudaGetDevice(&dev));
  std::vector<uint8_t> blob(sizeof(IpcHeader) + b.cols.size() * sizeof(IpcCol));
  IpcHeader* h = (IpcHeader*)blob.data();
  h->magic = IPC_MAGIC; h->pid = (int32_t)getpid(); h->device = dev; h->n_cols = (int32_t)b.cols.size(); h->num_rows = b.num_rows;
  IpcCol* cols = (IpcCol*)(blob.data() + sizeof(IpcHeader));
  for (size_t i = 0; i < b.cols.size(); ++i) {
    const Column& c = b.cols[i];
    if (!c.present) fail(ARK_ERR_UNSUPPORTED, "ipc export: column '" + c.field.name + "' has Arrow type '" + c.field.format + "'");
    IpcCol& o = cols[i];
    memset(&o, 0, sizeof o);
    if (c.field.name.size() >= sizeof o.name) fail(ARK_ERR_UNSUPPORTED, "ipc export: column name longer than 63 bytes");
    memcpy(o.name, c.field.name.data(), c.field.name.size());
    strncpy(o.format, c.field.format.c_str(), sizeof o.format - 1);
    o.dtype = (int32_t)c.field.type; o.nullable = c.field.nullable; o.length = c.length; o.null_count = c.null_count;
    o.validity_bit0 = c.validity_bit0; o.data_bit0 = c.data_bit0;
    export_buf(c.validity, &o.validity);
    const bool varlen = c.field.type == DType::Utf8 || c.field.type == DType::Binary;
    export_buf(varlen ? (const void*)c.offsets : (const void*)c.data, &o.first);
    export_buf(varlen ? (const void*)c.data : nullptr, &o.second);
  }
  return blob;
}

// rows [row0[s], row0[s] + n_rows[s]) of every source, concatenated in source order
Batch ipc_concat_slices(int n_src, const uint8_t* const* blobs, const int64_t* blob_sizes, const int64_t* row0, const int64_t* n_rows,
                        cudaStream_t stream) {
  int dev = 0;
  ARK_CUDA(cudaGetDevice(&dev));
  std::vector<Batch> parts;
  for (int s = 0; s < n_src; ++s) {
    if (blob_sizes[s] < (int64_t)sizeof(IpcHeader)) fail(ARK_ERR_PROCESS, "ipc import: truncated descriptor");
    const IpcHeader* h = (const IpcHeader*)blobs[s];
    if (h->magic != IPC_MAGIC || blob_sizes[s] < (int64_t)(sizeof(IpcHeader) + (size_t)h->n_cols * sizeof(IpcCol)))
      fail(ARK_ERR_PROCESS, "ipc import: malformed descriptor");
    if (row0[s] < 0 || n_rows[s] < 0 || row0[s] + n_rows[s] > h->num_rows) fail(ARK_ERR_PROCESS, "ipc import: slice outside the source batch");
    const bool same = h->pid == (int32_t)getpid() && h->device == dev;
    const IpcCol* cols = (const IpcCol*)(blobs[s] + sizeof(IpcHeader));
    Batch b;
    b.num_rows = n_rows[s];
    for (int i = 0; i < h->n_cols; ++i) {
      const IpcCol& o = cols[i];
      Column c;
      c.field.name = o.name; c.field.format = o.format; c.field.type = (DType)o.dtype; c.field.nullable = o.nullable != 0;
      c.length = n_rows[s];
      c.validity = open_buf(o.validity, same);
      c.validity_bit0 = (int32_t)(o.validity_bit0 + row0[s]);
      c.null_count = c.validity ? -1 : 0;
      const uint8_t* first = open_buf(o.first, same);
      switch (c.field.type) {
        case DType::Int64: case DType::Float64:
          c.data = first ? first + row0[s] * 8 : nullptr; c.data_bytes = n_rows[s] * 8; break;
        case DType::Bool:
          c.data = first; c.data_bit0 = (int32_t)(o.data_bit0 + row0[s]); c.data_bytes = (n_rows[s] + 7) / 8; break;
        case DType::Utf8: case DType::Binary:
          c.offsets = first ? (const int32_t*)first + row0[s] : nullptr;
          c.data = open_buf(o.second, same);
          c.data_bytes = -1;  // offsets[0] / offsets[n] are read from the peer by gather_extents_kernel
          break;
        default: break;
      }
      b.cols.push_back(std::move(c));
    }
    parts.push_back(std::move(b));
  }
  if (parts.size() == 1) {  // concat_device would hand the (peer-resident) slice back: force a local copy
    Batch empty = parts[0];
    empty.num_rows = 0;
    for (auto& c : empty.cols) { c.length = 0; if (c.field.type == DType::Utf8 || c.field.type == DType::Binary) c.data_bytes = 0; }
    parts.push_back(std::move(empty));
  }
  return concat_device(parts, stream);
}

}  // namespace ark

using namespace ark;

extern "C" {

int ark_ipc_export_device(ArrowDeviceArray* in, ArrowSchema* in_schema, uint8_t* blob, int64_t blob_cap, int64_t* blob_size) {
  BufferPtr in_owner = adopt_array(&in->array);
  return guarded([&] {
    ArrowDeviceArray view = device_view(*in, in_owner);
    Batch b = import_device(&view, in_schema, nullptr, in_owner);
    std::vector<uint8_t> out = ipc_export(b);
    if (blob_size) *blob_size = (int64_t)out.size();
    if ((int64_t)out.size() > blob_cap) fail(ARK_ERR_PROCESS, "ipc export: descriptor buffer too small");
    memcpy(blob, out.data(), out.size());
  });
}

int ark_ipc_concat_slices_device(int n_src, const uint8_t* const* blobs, const int64_t* blob_sizes, const int64_t* row0, const int64_t* n_rows,
                                 ArrowDeviceArray* out, ArrowSchema* out_schema) {
  return guarded([&] {
    zero_out(out, out_schema);
    if (n_src <= 0 || !blobs || !blob_sizes || !row0 || !n_rows || !out) fail(ARK_ERR_PROCESS, "null argument");
    StreamLease lease;
    Batch r = ipc_concat_slices(n_src, blobs, blob_sizes, row0, n_rows, lease.s);
    export_device(r, out, out_schema, lease);
  });
}

}  // extern "C"
