// decoded.h — the per-row buffers a decode kernel fills for one output column (CSV, NDJSON / json_to_arrow, Avro,
// protobuf_to_arrow), and the step that turns them into Arrow columns: stage_column before the kernel, settle_columns
// after it for the whole batch, then finish_column per column.
//
// Only len[rows] is zeroed up front.  The kernel writes every row of a batch that succeeds, and a failing batch's
// lengths are read only by scans whose totals are dropped with it: the exact 2 GiB sum runs after its error check.
#pragma once
#include <functional>
#include <string>
#include <vector>

#include "batch.h"

namespace ark {

struct StagedColumn {
  DType type = DType::Null;
  int64_t rows = 0;
  BufferPtr values;  // fixed_width(type) bytes per row; Boolean: one byte (0 / 1) per row
  BufferPtr valid;   // nullable: one byte (0: NULL) per row
  BufferPtr len;     // Utf8 / Binary: rows + 1 int32 lengths
  BufferPtr src;     // Utf8 / Binary: int64 source position of each row's bytes; List / Struct: of its raw value
  BufferPtr raw;     // wants_raw: int32 raw length per row (formats that unescape; List / Struct spans)
  int64_t bound = 0;  // Utf8 / Binary: host bound on the column's bytes, and the "<what>" of its 2 GiB error
  std::string what;
  BufferPtr offsets, bits;  // set by settle_columns, with total and null_count
  int32_t total = 0;
  int64_t null_count = 0;
};

StagedColumn stage_column(DType type, int64_t rows, bool nullable, bool wants_raw, cudaStream_t stream);

// `err` (may be null): a device error word of at most 16 bytes; `check` raises the decoder's error from its host copy.
// When a bound exceeds INT32_MAX, the error word is checked before varlen_guard, so a decode error wins over the 2 GiB
// error.  Then every string column is scanned and every validity packed, one synchronisation brings back the error
// word, the totals and the null counts, and `check` runs again.
void settle_columns(std::vector<StagedColumn>& cols, const void* err, size_t err_bytes,
                    const std::function<void(const void*)>& check, cudaStream_t stream);

// The Column of a settled `s`; `copy_bytes(s, out)` writes a string column's bytes.  Owners: values (Boolean: bitmap
// and bytes) or {offsets, bytes}, then the validity bitmap.  A Null column gets no buffers.
Column finish_column(const StagedColumn& s, Field f, const std::function<void(const StagedColumn&, uint8_t*)>& copy_bytes,
                     cudaStream_t stream);

}  // namespace ark
