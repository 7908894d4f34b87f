// varlen.h — the int32 offsets and bytes of a Binary / Utf8 column built on the device from per-row lengths, and the
// guard that keeps such a column inside its 2 GiB.
//
// The offsets come from an int32 exclusive scan of the lengths.  Once the lengths add up past 2^31 - 1 that scan wraps
// silently, and past 2^32 its last entry looks valid again while earlier offsets point outside the allocation.  So no
// scan of lengths is trusted before varlen_guard has shown that their total fits.
#pragma once
#include <string>

#include "batch.h"

namespace ark {

// Exclusive scan of lens[0 .. n] (n + 1 entries, lens[n] = 0) into a fresh buffer of n + 1 int32 offsets.
BufferPtr varlen_scan(const int32_t* lens, int64_t n, cudaStream_t stream);

// The 2 GiB guard, in whichever form is cheaper where it is used:
//   * `total`: the lengths' sum, added up exactly in 64 bits by the kernel that wrote them and read back.  A total past
//     INT32_MAX fails with Process `msg`; otherwise it is returned (it equals the scan's last offset).
//   * `bound`: a host bound on the sum of lens[0 .. n).  When 0 <= bound <= INT32_MAX nothing runs.  Otherwise
//     protobuf_sum64_kernel adds the lengths up exactly first (one launch and one synchronisation, taken only by batches
//     near the limit), and a total past INT32_MAX fails with Process "<what> holds N bytes: …" before anything is written.
int32_t varlen_guard(unsigned long long total, const std::string& msg);
void varlen_guard(const int32_t* lens, int64_t n, int64_t bound, const std::string& what, cudaStream_t stream);

struct Varlen {
  BufferPtr offsets, bytes;  // n + 1 offsets; total + 16 bytes, not yet written
  int32_t total = 0;
};

// One column's lengths → its offsets and an unwritten bytes buffer: the guard, the scan, one read-back of the total and
// one synchronisation.  `exact` is a device word holding the lengths' 64-bit sum (read back in place of the last offset,
// `what` is then the whole error text); without it `bound` and `what` go to the bound form of varlen_guard.
Varlen varlen_layout(const int32_t* lens, int64_t n, const unsigned long long* exact, int64_t bound, const std::string& what,
                     cudaStream_t stream);

// c.offsets / data / data_bytes from v, first_offset = 0, owners = {offsets, bytes}: validity owners go after.
void set_varlen(Column& c, const Varlen& v);

// The bytes of a column whose row r is the span [src[r], src[r] + offsets[r + 1] - offsets[r]) of `data`, or, when
// src[r] < 0, of `dflt` from -1 - src[r].
void launch_span_copy(const uint8_t* data, const uint8_t* dflt, const long long* src, const int32_t* offsets, int64_t n_rows,
                      uint8_t* out, cudaStream_t stream);

}  // namespace ark
