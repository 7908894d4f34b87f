// file_input.h — the `file` input's formats behind one driver (inputs.cu).
//
// The driver owns what every format shares: it opens the file once, uploads it to HBM through two pinned chunks, cuts
// reads into `batch_size` rows, skips batches without rows and runs the optional query.  A format knows only its own
// bytes: the metadata it reads before the device is touched, what it learns from the upload's chunks, how many rows the
// uploaded file holds and how to decode rows [r0, r0 + n) of it.
#pragma once
#include <memory>
#include <string>
#include <utility>
#include <vector>

#include "engine.h"

namespace ark {

// The file on the host, opened once per connect(): "not found" and "cannot open" are reported here, before any device
// work.
struct HostFile {
  explicit HostFile(const std::string& path);
  ~HostFile();
  HostFile(const HostFile&) = delete;
  HostFile& operator=(const HostFile&) = delete;
  // up to n bytes at `off`, fewer only at the end of the file or on a read error
  size_t read_some(int64_t off, void* dst, size_t n) const;
  // exactly n bytes at `off`, or Process "short read"
  std::string read(int64_t off, int64_t n) const;
  std::string path;
  int fd = -1;
  int64_t size = 0;
};

struct FileFormat {
  virtual ~FileFormat() {}
  // host-only metadata, read before the device is touched
  virtual void open(const HostFile&) {}
  // the upload's bytes [file_offset, file_offset + n), in file order
  virtual void scan(const uint8_t*, size_t, int64_t) {}
  // after the upload: the rows the file holds
  virtual int64_t prepare(const BufferPtr& file_dev, int64_t bytes, cudaStream_t stream) = 0;
  // rows [r0, r0 + n)
  virtual Batch batch(int64_t r0, int64_t n, cudaStream_t stream) = 0;
};

std::unique_ptr<FileFormat> make_csv_format(bool has_header);  // csv.cu
std::unique_ptr<FileFormat> make_avro_format();                // avro.cu
std::unique_ptr<FileFormat> make_arrow_ipc_format();           // arrow_ipc.cu

inline unsigned grid_of(long long n, int threads = 256) { return (unsigned)std::max<long long>(1, std::min<long long>((n + threads - 1) / threads, sm_count() * 16)); }

// The lines of an uploaded text file (CSV, NDJSON) that are not empty: a line ends at `\n` or at the end of the file,
// and a line with nothing but `\r` before its end is left out, so it is never a record.
struct LineIndex {
  BufferPtr file;    // the file in HBM
  int64_t bytes = 0;
  BufferPtr starts;  // int64 starts of the lines, then the file's end
  int64_t lines = 0;

  void build(const BufferPtr& file_dev, int64_t file_bytes, cudaStream_t stream);
  // the byte span [first byte of line l0, first byte of line l0 + n), at most 2 GiB: one read-back
  std::pair<int64_t, int64_t> span(int64_t l0, int64_t n, cudaStream_t stream) const;
  // int32 starts of lines [l0, l0 + n) and their end, relative to the start of line l0
  BufferPtr rebased(int64_t l0, int64_t n, cudaStream_t stream) const;
  // the first k lines on the host, terminators kept; *first: the file offset of the first
  std::vector<std::string> sample(int64_t k, cudaStream_t stream, int64_t* first = nullptr) const;
  // the 1-based physical line that holds byte `off`: the line terminators before it, empty lines included
  long long physical_line(long long off, cudaStream_t stream) const;
};

}  // namespace ark
