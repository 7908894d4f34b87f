// common.h — status/error plumbing, CUDA checks, launch accounting shared by every translation unit.
#pragma once
#include <cuda_runtime.h>

#include <cstdint>
#include <cstdio>
#include <cstring>
#include <stdexcept>
#include <string>

#include "../../include/arkflow_b200.h"

namespace ark {

// Exception carrying an ark_status; every C-ABI entry point catches it and stores the message in
// the thread-local last-error slot (mirrors `Result<_, Error>` of crates/arkflow-core/src/lib.rs:66-110).
struct ArkError : std::runtime_error {
  int code;
  ArkError(int c, const std::string& m) : std::runtime_error(m), code(c) {}
};

[[noreturn]] inline void fail(int code, const std::string& msg) { throw ArkError(code, msg); }

void set_last_error(const std::string& msg);

#define ARK_CUDA(expr)                                                                      \
  do {                                                                                      \
    cudaError_t _e = (expr);                                                                \
    if (_e != cudaSuccess) {                                                                \
      throw ::ark::ArkError(ARK_ERR_CUDA, std::string("CUDA error: ") + cudaGetErrorString(_e) + \
                                              " at " + __FILE__ + ":" + std::to_string(__LINE__)); \
    }                                                                                       \
  } while (0)

// ---- kernel launch accounting (ark_kernel_launch_count / ark_kernel_timing_*) ----
void note_launch(const char* name);
struct KernelTimer {  // RAII: records CUDA events around one launch when timing is enabled
  // `also`: a second name the same launch is recorded under (a group of kernels timed together, e.g. hash_agg_kernel)
  KernelTimer(const char* name, cudaStream_t s, const char* also = nullptr);
  ~KernelTimer();
  const char* name;
  const char* also;
  cudaStream_t stream;
  cudaEvent_t e0 = nullptr, e1 = nullptr;
};

void bind_device(int device);   // remembered by ark_b200_init
void ensure_device();           // re-binds the calling host thread to that device

inline int64_t ceil_div(int64_t a, int64_t b) { return (a + b - 1) / b; }
inline int64_t round_up(int64_t a, int64_t b) { return ceil_div(a, b) * b; }

// SMs of the device the process first asked from (132 on an H100 SXM); grid caps of grid-stride kernels scale with it
inline int sm_count() {
  static const int n = [] { int d = 0, v = 0; cudaGetDevice(&d); cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, d); return v > 0 ? v : 132; }();
  return n;
}

}  // namespace ark
