// bitmap.h — the Arrow bitmaps (validity and Boolean values) the library builds on the device from one byte per row,
// and the null count that goes with a validity bitmap.  bitmap.cuh reads them on the device.
//
// A bitmap of n rows starts at bit 0, and the unused bits of its last byte are zero.  It is allocated with
// (n + 7) / 8 + 1 bytes, of which the first (n + 7) / 8 are the bitmap.
//
// A column's null_count is exact or -1 (unknown), and a column whose count is 0 carries no validity bitmap.  Which of
// the two a producer gives depends on what the count costs it:
//   * exact: the decoders (CSV, JSON, Avro) count the zero bytes while packing, in a counter slot of the one round trip
//     that settles all the columns of a batch (decoded.h), and call set_validity after its synchronisation.
//   * unknown: query outputs (SQL projection, join gathers, GROUP BY keys and aggregates) take no read-back and no
//     synchronisation; set_validity_unknown attaches the bitmap whenever there are rows.
#pragma once
#include "batch.h"

namespace ark {

// bytes[0 .. n) (0 / non-zero) packed into a fresh bitmap.  `zeros` (may be null): a device counter the number of zero
// bytes is added to.
BufferPtr pack_bits(const uint8_t* bytes, int64_t n, unsigned long long* zeros, cudaStream_t stream);

// c.data / data_bit0 / data_bytes: bytes[0 .. n) packed; owners = {bitmap, bytes}: validity owners go after.
void set_bool_values(Column& c, const BufferPtr& bytes, int64_t n, cudaStream_t stream);

// Attaches `bits` as c's validity with `null_count` (-1: unknown); a count of 0 attaches nothing.
void set_validity(Column& c, const BufferPtr& bits, int64_t null_count);

// c's validity from bytes[0 .. n) with null_count -1, attached when n > 0 and kept alive with `bytes`.
void set_validity_unknown(Column& c, const BufferPtr& bytes, int64_t n, cudaStream_t stream);

// Adds the number of zero bits among the n bits of `bits` from bit `bit0` on to the device counter `zeros`: the null count
// of a validity bitmap that a column shares with a larger one (a slice).
void count_zeros(const uint8_t* bits, int32_t bit0, int64_t n, unsigned long long* zeros, cudaStream_t stream);

// The n bits of `in` from bit `bit0` on, copied into a fresh bitmap of (n + 7) / 8 bytes that starts at bit 0.  n > 0.
BufferPtr realign_bits(const uint8_t* in, int32_t bit0, int64_t n, cudaStream_t stream);

}  // namespace ark
