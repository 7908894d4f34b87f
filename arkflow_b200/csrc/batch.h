// batch.h — HBM-resident record batch (the MessageBatch stand-in, crates/arkflow-core/src/lib.rs:236-240),
// the device/pinned memory pools behind it, and the Arrow C Data Interface import/export.
//
// Layout in HBM (same as Arrow's columnar format, so a batch can be handed to the next processor
// without reshaping): fixed-width columns = one contiguous values buffer; Utf8/Binary = int32
// offsets[n+1] + contiguous bytes; Boolean = bit-packed; optional validity bitmap per column.
#pragma once
#include <memory>
#include <mutex>
#include <string>
#include <vector>

#include "common.h"
#include "sql.h"
#include "vm.h"

namespace ark {

// ---- memory pools -------------------------------------------------------------------------------
// Caching allocators.  A block freed inside a call is parked until that call's stream has been synchronised
// (~StreamLease); Arrow's contract is that a consumer releases an array only when it is done with it.  So a
// block in the free list is idle and can be handed to any stream without event tracking.
class BlockPool {
 public:
  enum Kind { Device, Pinned };
  explicit BlockPool(Kind k) : kind_(k) {}
  ~BlockPool();
  void* alloc(size_t bytes);
  void free(void* p);      // parks the block while the calling thread is inside a call (see batch.cu)
  void free_now(void* p);
  size_t bytes_reserved() const { return reserved_; }
  void trim();
  // A block whose CUDA IPC handle has been given to a peer stays mapped there for the life of the process
  // (ipc_exchange.cu caches the mappings): it must never go back to the driver, so trim() keeps it.
  void mark_exported(const void* base);

 private:
  struct Block { void* p; size_t size; };
  Kind kind_;
  std::mutex mu_;
  std::vector<Block> free_;    // sorted by size
  std::vector<Block> live_;
  std::vector<const void*> exported_;
  size_t reserved_ = 0;
};

BlockPool& device_pool();
BlockPool& pinned_pool();
BlockPool& export_pool();  // device blocks whose IPC handles go to peers (see ExportAllocScope)

using BufferPtr = std::shared_ptr<void>;  // owner of one allocation; get() = base pointer
BufferPtr device_alloc(size_t bytes);
BufferPtr pinned_alloc(size_t bytes);

// While one of these is alive on a thread, device_alloc() on that thread serves buffers that are going to be published to
// the other ranks as CUDA IPC handles (the outputs of a hash partition / partial aggregate).  Every peer caches its mapping of
// a block, and a new block costs every peer a cudaIpcOpenMemHandle (~1.5 ms): taken from the general pool, a different block
// served the same buffer from step to step, and the opens dominated a distributed join step.  So:
//  * with `expected_bytes` > 0 the scope bump-allocates from ONE arena block that holds the whole output (and the few
//    temporaries allocated next to it); an arena is reused as soon as every buffer cut from it has been released, the
//    lowest-numbered free arena first — consecutive batches of a stream land in the same one or two blocks;
//  * otherwise (or when the arena is full) from export_pool(), a pool that only such outputs use.
struct ExportAllocScope {
  explicit ExportAllocScope(size_t expected_bytes = 0);
  ~ExportAllocScope();
  ExportAllocScope(const ExportAllocScope&) = delete;
  ExportAllocScope& operator=(const ExportAllocScope&) = delete;
};

// ---- streams ------------------------------------------------------------------------------------
// RAII lease of a non-blocking stream from a small pool (replaces the reference's
// SessionContextPool::acquire/release, context_pool.rs:91-119, without its leak-on-error).
struct StreamLease {
  StreamLease();
  ~StreamLease();
  cudaStream_t s;
  StreamLease(const StreamLease&) = delete;
  StreamLease& operator=(const StreamLease&) = delete;
};

// ---- columns and batches ------------------------------------------------------------------------
struct Field {
  std::string name;
  DType type = DType::Null;
  bool nullable = true;
  std::string format;  // original Arrow format string (kept for unsupported types)
};

struct Column {
  Field field;
  int64_t length = 0;
  int64_t null_count = 0;
  const uint8_t* validity = nullptr;  // device bitmap or nullptr
  int32_t validity_bit0 = 0;
  const int32_t* offsets = nullptr;   // element 0 (already shifted by the Arrow offset)
  const uint8_t* data = nullptr;      // values of element 0 / byte base that offsets index into
  int32_t data_bit0 = 0;              // Boolean
  int64_t data_bytes = 0;             // var-len: bytes referenced (offsets[n]-offsets[0]); fixed: n*width
  int64_t first_offset = 0;           // var-len: offsets[0] value (0 for batches we produced)
  int64_t data_bound = -1;            // var-len, extent unknown: upper bound on offsets[n] (end of the allocation), or -1
  std::vector<BufferPtr> owners;      // keep-alive for everything referenced above
  bool present = true;                // false ⇒ column was not imported (projection push-down)
  // List: children[0] = the elements (offsets index into it); Struct: one child per field, each of `length` rows.
  // Only json_to_arrow produces these (one nesting level); they can be exported, not queried.
  std::vector<Column> children;

  ColView view() const {
    ColView v;
    v.data = data; v.offsets = offsets; v.validity = validity;
    v.validity_bit0 = validity_bit0; v.data_bit0 = data_bit0;
    return v;
  }
};

struct Batch {
  std::vector<Column> cols;
  int64_t num_rows = 0;
  std::string input_name;  // MessageBatch::input_name (lib.rs:239)
  int find(const std::string& name) const {
    for (size_t i = 0; i < cols.size(); ++i) if (cols[i].field.name == name) return (int)i;
    return -1;
  }
};

std::vector<Field> schema_fields(const ArrowSchema* s);  // struct schema → fields (no data needed)
std::string schema_fingerprint(const std::vector<Field>& f);

// Bytes per value of a fixed-width column type other than Boolean; 0 for the rest.
inline int fixed_width(DType t) {
  switch (t) {
    case DType::Int64: case DType::Float64: case DType::UInt64: return 8;
    case DType::Int32: case DType::UInt32: case DType::Float32: return 4;
    default: return 0;
  }
}

// Import a struct array.  `needed`: per top-level column, whether its buffers are required (others
// get present=false and are not copied); nullptr ⇒ all.  Host import copies buffers to HBM on
// `stream` (the source is read asynchronously when pinned; the caller synchronizes before
// releasing `arr`).  Device import wraps the pointers without copying; `keep` (may be null) is
// attached to every column as an owner.  `codec_types` also imports Int32 / UInt32 / UInt64 / Float32
// columns (formats i, I, L, f): only arrow_to_protobuf reads them; every other caller leaves them not present.
Batch import_host(const ArrowArray* arr, const ArrowSchema* schema, const std::vector<bool>* needed,
                  cudaStream_t stream, int64_t* h2d_bytes = nullptr, bool codec_types = false);
Batch import_device(const ArrowDeviceArray* arr, const ArrowSchema* schema, const std::vector<bool>* needed,
                    BufferPtr keep, bool codec_types = false);

// Export: builds a struct ArrowArray/ArrowSchema whose release callbacks drop the owners.
// Host export copies HBM → pinned host on `stream` and synchronizes it.
void export_schema(const Batch& b, ArrowSchema* out);
void export_empty_schema(ArrowSchema* out);  // RecordBatch::new_empty(Schema::empty()), sql.rs:137-139
void export_host(const Batch& b, cudaStream_t stream, ArrowArray* out, ArrowSchema* out_schema,
                 int64_t* d2h_bytes = nullptr);
void export_device(const Batch& b, ArrowDeviceArray* out, ArrowSchema* out_schema);

// Moves an ArrowArray into shared ownership: the returned pointer releases it when dropped.
BufferPtr adopt_array(ArrowArray* arr);

// Bytes from p to the end of the device allocation that contains it (driver cuMemGetAddressRange), or -1.
int64_t device_alloc_remaining(const void* p);
// Upper bound on the bytes a var-len column references: exact when known, else the allocation bound
// (clamped to the 2 GiB an int32-offset column can address); -1 when neither is available.
int64_t varlen_bytes_bound(const Column& c);

}  // namespace ark
