// batch.cu — pools, stream leases, Arrow C Data Interface import/export (see batch.h).
#include <chrono>
#include <algorithm>
#include <atomic>
#include <condition_variable>
#include <deque>
#include <functional>
#include <map>
#include <thread>

#include "batch.h"
#include "bitmap.h"

namespace ark {

// ---- error slot + launch accounting ---------------------------------------------------------------
static thread_local std::string g_last_error;
void set_last_error(const std::string& msg) { g_last_error = msg; }
const std::string& last_error_ref() { return g_last_error; }

static std::atomic<int64_t> g_launches{0};
static std::atomic<int> g_timing{0};
struct TimingEntry { double ms = 0; int64_t n = 0; };
static std::mutex g_timing_mu;
static std::map<std::string, TimingEntry> g_timing_map;

void note_launch(const char*) { g_launches.fetch_add(1, std::memory_order_relaxed); }
int64_t launch_count() { return g_launches.load(); }
static void resolve_pending_locked();
struct PendingTiming { const char* name; const char* also; cudaEvent_t e0, e1; };
static std::vector<PendingTiming> g_pending;
static std::vector<cudaEvent_t> g_event_pool;
// Creating an event costs about as much as two records (measured on H100), so timed launches never create theirs: the
// pool is stocked when timing is switched on, and each timed launch hands back the events of launches that have ended.
constexpr size_t EVENT_STOCK = 16;
void timing_enable(int on) {
  if (on) {
    std::lock_guard<std::mutex> l(g_timing_mu);
    while (g_event_pool.size() < EVENT_STOCK) {
      cudaEvent_t e = nullptr;
      if (cudaEventCreate(&e) != cudaSuccess) { cudaGetLastError(); break; }
      g_event_pool.push_back(e);
    }
  }
  g_timing.store(on);
}
static cudaEvent_t g_gap_open = nullptr;  // ARK_TRACE: recorded after the last filter kernel, closed by the next one's start
void timing_reset() {
  std::lock_guard<std::mutex> l(g_timing_mu);
  resolve_pending_locked();
  g_timing_map.clear();
  if (g_gap_open) { g_event_pool.push_back(g_gap_open); g_gap_open = nullptr; }  // a gap starts inside the measured window
}
bool timing_get(const char* name, double* ms, int64_t* n) {
  std::lock_guard<std::mutex> l(g_timing_mu);
  resolve_pending_locked();
  auto it = g_timing_map.find(name);
  if (it == g_timing_map.end()) { *ms = 0; *n = 0; return false; }
  *ms = it->second.ms; *n = it->second.n; return true;
}

// Timed launches record an event pair and resolve it lazily (no synchronisation on the launch path):
// ark_kernel_timing_get() is called after the caller has synchronised the device.

static cudaEvent_t take_event() {
  {
    std::lock_guard<std::mutex> l(g_timing_mu);
    if (!g_event_pool.empty()) { cudaEvent_t e = g_event_pool.back(); g_event_pool.pop_back(); return e; }
  }
  cudaEvent_t e = nullptr;
  cudaEventCreate(&e);
  return e;
}

static void resolve_one_locked(const PendingTiming& p, bool ended) {
  float ms = 0;
  if (ended && cudaEventElapsedTime(&ms, p.e0, p.e1) == cudaSuccess) {
    auto& e = g_timing_map[p.name]; e.ms += ms; e.n += 1;
    if (p.also) { auto& a = g_timing_map[p.also]; a.ms += ms; a.n += 1; }
  } else cudaGetLastError();
  g_event_pool.push_back(p.e0); g_event_pool.push_back(p.e1);
}

static void resolve_pending_locked() {
  for (auto& p : g_pending) resolve_one_locked(p, cudaEventSynchronize(p.e1) == cudaSuccess);
  g_pending.clear();
}

// The pairs whose launch has ended, without waiting for the others.
static void resolve_ended_locked() {
  size_t keep = 0;
  for (size_t i = 0; i < g_pending.size(); ++i) {
    const cudaError_t q = cudaEventQuery(g_pending[i].e1);
    if (q == cudaErrorNotReady) { g_pending[keep++] = g_pending[i]; continue; }
    resolve_one_locked(g_pending[i], q == cudaSuccess);
  }
  g_pending.resize(keep);
  if (keep && cudaPeekAtLastError() == cudaErrorNotReady) cudaGetLastError();  // "not ready" is an answer, not an error
}

KernelTimer::KernelTimer(const char* n, cudaStream_t s, const char* a) : name(n), also(a), stream(s) {
  note_launch(n);
  if (g_timing.load(std::memory_order_relaxed)) {
    {
      std::lock_guard<std::mutex> l(g_timing_mu);  // both events in one visit to the pool
      if (g_event_pool.size() >= 2) { e0 = g_event_pool.back(); g_event_pool.pop_back(); e1 = g_event_pool.back(); g_event_pool.pop_back(); }
    }
    if (!e0) { e0 = take_event(); e1 = take_event(); }
    cudaEventRecord(e0, stream);
  }
}
KernelTimer::~KernelTimer() {
  if (e0) {
    cudaEventRecord(e1, stream);
    std::lock_guard<std::mutex> l(g_timing_mu);
    g_pending.push_back({name, also, e0, e1});
    resolve_ended_locked();  // the kernel is queued: this host time is not between kernels
  }
}

bool trace_enabled() { static const bool on = getenv("ARK_TRACE") != nullptr; return on; }
thread_local CallTrace tl_call_trace;

void trace_kernel_begin(cudaStream_t s) {
  if (!trace_enabled()) return;
  cudaEvent_t e = take_event();
  cudaEventRecord(e, s);
  std::lock_guard<std::mutex> l(g_timing_mu);
  if (g_gap_open) g_pending.push_back({"filter_call_gap", nullptr, g_gap_open, e});
  else g_event_pool.push_back(e);
  g_gap_open = nullptr;
}
void trace_kernel_end(cudaStream_t s) {
  if (!trace_enabled()) return;
  cudaEvent_t e = take_event();
  cudaEventRecord(e, s);
  std::lock_guard<std::mutex> l(g_timing_mu);
  if (g_gap_open) g_event_pool.push_back(g_gap_open);
  g_gap_open = e;
}

// ---- device binding ---------------------------------------------------------------------------------
// One process drives one GPU (ark_b200_init).  CUDA's "current device" is per host thread and defaults
// to 0, so worker threads that never called cudaSetDevice (tokio blocking threads, Python thread pools)
// are re-bound to the library's device on entry.
static std::atomic<int> g_device{-1};
void bind_device(int device) { g_device.store(device); }
void ensure_device() {
  const int want = g_device.load(std::memory_order_relaxed);
  if (want < 0) return;
  int cur = -1;
  if (cudaGetDevice(&cur) == cudaSuccess && cur != want) cudaSetDevice(want);
}

// ---- pools ------------------------------------------------------------------------------------------
BlockPool::~BlockPool() {}  // process teardown: the driver reclaims; freeing here races CUDA shutdown

void* BlockPool::alloc(size_t bytes) {
  ensure_device();
  if (bytes == 0) bytes = 1;
  size_t want = (size_t)round_up((int64_t)bytes, kind_ == Device ? 512 : 4096);
  // size classes for large blocks (eight per power of two, ≤ 12.5 % slack): the buffers of consecutive batches differ by a few
  // KB (a hash partition of 2^24 rows, the slice a rank receives), and with exact sizes a request took a slightly larger
  // free block, the next request for that size found none and went to cudaMalloc — and, for exported blocks, made every
  // peer open a new IPC mapping, which costs several times the exchange itself
  if (want >= (1u << 20)) {
    size_t step = (size_t)1 << 17;
    while ((step << 4) <= want) step <<= 1;  // step = 2^(floor(log2(want)) - 3)
    want = (size_t)round_up((int64_t)want, (int64_t)step);
  }
  {
    std::lock_guard<std::mutex> l(mu_);
    auto it = std::lower_bound(free_.begin(), free_.end(), want, [](const Block& b, size_t w) { return b.size < w; });
    if (it != free_.end() && it->size <= std::max(want + (want >> 2), want + (1u << 20))) {
      // among the free blocks of that size, the lowest address: the same buffer of consecutive batches tends to land in
      // the same block whatever order the previous batch's buffers were released in (peers cache their IPC mappings)
      auto best = it;
      for (auto j = it; j != free_.end() && j->size == it->size; ++j) if (j->p < best->p) best = j;
      Block b = *best; free_.erase(best); live_.push_back(b); return b.p;
    }
  }
  void* p = nullptr;
  cudaError_t e = kind_ == Device ? cudaMalloc(&p, want) : cudaHostAlloc(&p, want, cudaHostAllocDefault);
  if (e != cudaSuccess) {
    cudaGetLastError();
    trim();
    if (kind_ == Device) { device_pool().trim(); export_pool().trim(); }  // either device pool may hold the idle blocks
    e = kind_ == Device ? cudaMalloc(&p, want) : cudaHostAlloc(&p, want, cudaHostAllocDefault);
    if (e != cudaSuccess) {
      cudaGetLastError();
      fail(ARK_ERR_CUDA, std::string(kind_ == Device ? "device" : "pinned host") + " allocation of " +
                             std::to_string(want) + " bytes failed: " + cudaGetErrorString(e));
    }
  }
  std::lock_guard<std::mutex> l(mu_);
  live_.push_back({p, want}); reserved_ += want;
  return p;
}

// A block released while the calling thread is inside a C-ABI call (it holds a StreamLease) may still be read or
// written by work that call has queued on its stream — cub temporaries, staging blocks and the like go out of scope
// right after the launch.  Handing such a block to ANOTHER thread's call would corrupt both, so it is parked here
// and returns to the pool when the thread's outermost lease ends, after the stream synchronize in ~StreamLease.
// (Blocks released outside a call — an Arrow consumer dropping a result — belong to calls that completed.)
static thread_local int tl_lease_depth = 0;
static thread_local std::vector<std::pair<BlockPool*, void*>> tl_parked;

void BlockPool::free(void* p) {
  if (!p) return;
  if (tl_lease_depth > 0) { tl_parked.push_back({this, p}); return; }
  free_now(p);
}

void BlockPool::free_now(void* p) {
  std::lock_guard<std::mutex> l(mu_);
  for (size_t i = 0; i < live_.size(); ++i) {
    if (live_[i].p == p) {
      Block b = live_[i];
      live_[i] = live_.back(); live_.pop_back();
      auto it = std::lower_bound(free_.begin(), free_.end(), b.size, [](const Block& x, size_t w) { return x.size < w; });
      free_.insert(it, b);
      return;
    }
  }
}

void BlockPool::mark_exported(const void* base) {
  std::lock_guard<std::mutex> l(mu_);
  if (std::find(exported_.begin(), exported_.end(), base) == exported_.end()) exported_.push_back(base);
}

void BlockPool::trim() {
  std::vector<Block> drop;
  {
    std::lock_guard<std::mutex> l(mu_);
    std::vector<Block> keep;
    for (auto& b : free_) {
      if (std::find(exported_.begin(), exported_.end(), (const void*)b.p) != exported_.end()) keep.push_back(b);  // peers may still have it mapped
      else { drop.push_back(b); reserved_ -= b.size; }
    }
    free_.swap(keep);
  }
  for (auto& b : drop) { if (kind_ == Device) cudaFree(b.p); else cudaFreeHost(b.p); }
}

BlockPool& device_pool() { static BlockPool* p = new BlockPool(BlockPool::Device); return *p; }
BlockPool& pinned_pool() { static BlockPool* p = new BlockPool(BlockPool::Pinned); return *p; }

BlockPool& export_pool() { static BlockPool* p = new BlockPool(BlockPool::Device); return *p; }

// ---- arenas for exported outputs (see ExportAllocScope) ----
namespace {
struct Arena {
  uint8_t* base = nullptr;
  size_t size = 0, used = 0;
  std::atomic<int> live{0};   // buffers cut from the arena that are still referenced (+1 while a scope holds it)
};
std::mutex g_arena_mu;
std::vector<Arena*> g_arenas;  // never freed: peers keep them mapped

Arena* arena_acquire(size_t bytes) {
  std::lock_guard<std::mutex> l(g_arena_mu);
  for (Arena* a : g_arenas)
    if (a->live.load() == 0 && a->size >= bytes) { a->used = 0; a->live.store(1); return a; }
  ensure_device();
  size_t want = bytes + (bytes >> 2);
  size_t step = (size_t)1 << 20;
  while ((step << 3) <= want) step <<= 1;
  want = (size_t)round_up((int64_t)want, (int64_t)step);
  void* p = nullptr;
  if (cudaMalloc(&p, want) != cudaSuccess) {
    cudaGetLastError();
    device_pool().trim(); export_pool().trim();
    if (cudaMalloc(&p, want) != cudaSuccess) { cudaGetLastError(); return nullptr; }  // the scope falls back to the pool
  }
  Arena* a = new Arena;
  a->base = (uint8_t*)p; a->size = want; a->live.store(1);
  g_arenas.push_back(a);
  return a;
}
}  // namespace

static thread_local int tl_export_alloc = 0;
static thread_local Arena* tl_arena = nullptr;
ExportAllocScope::ExportAllocScope(size_t expected_bytes) {
  ++tl_export_alloc;
  if (expected_bytes > 0 && tl_arena == nullptr) tl_arena = arena_acquire(expected_bytes);
}
ExportAllocScope::~ExportAllocScope() {
  if (--tl_export_alloc == 0 && tl_arena) { tl_arena->live.fetch_sub(1); tl_arena = nullptr; }
}

BufferPtr device_alloc(size_t bytes) {
  if (tl_export_alloc > 0) {
    if (Arena* a = tl_arena) {
      const size_t need = (size_t)round_up((int64_t)std::max<size_t>(bytes, 1), 512);
      if (a->used + need <= a->size) {
        void* p = a->base + a->used;
        a->used += need;
        a->live.fetch_add(1);
        return BufferPtr(p, [a](void*) { a->live.fetch_sub(1); });
      }
    }
    void* p = export_pool().alloc(bytes);
    return BufferPtr(p, [](void* q) { export_pool().free(q); });
  }
  void* p = device_pool().alloc(bytes);
  return BufferPtr(p, [](void* q) { device_pool().free(q); });
}
BufferPtr pinned_alloc(size_t bytes) {
  void* p = pinned_pool().alloc(bytes);
  return BufferPtr(p, [](void* q) { pinned_pool().free(q); });
}

// ---- streams ------------------------------------------------------------------------------------------
static std::mutex g_stream_mu;
static thread_local std::vector<StreamLease*> tl_leases;  // the leases this thread holds, innermost last
static std::vector<std::pair<cudaStream_t, FilterScratch*>> g_streams;  // the scratch is never freed, like the stream
StreamLease::StreamLease() {
  ensure_device();
  {
    std::lock_guard<std::mutex> l(g_stream_mu);
    if (!g_streams.empty()) {
      s = g_streams.back().first; filter = g_streams.back().second; g_streams.pop_back();
      ++tl_lease_depth;
      tl_leases.push_back(this);
      return;
    }
  }
  ARK_CUDA(cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking));
  filter = new FilterScratch();
  ++tl_lease_depth;
  tl_leases.push_back(this);
}
FilterScratch* lease_filter_scratch(cudaStream_t s) {
  for (auto it = tl_leases.rbegin(); it != tl_leases.rend(); ++it) if ((*it)->s == s) return (*it)->filter;
  return nullptr;
}
void StreamLease::synchronize_last() {
  ARK_CUDA(cudaStreamSynchronize(s));
  synced = true;
}
StreamLease::~StreamLease() {
  if (!synced) cudaStreamSynchronize(s);  // whatever this call queued is done: its temporaries may now serve any other call
  tl_leases.erase(std::find(tl_leases.begin(), tl_leases.end(), this));
  {
    std::lock_guard<std::mutex> l(g_stream_mu);
    g_streams.push_back({s, filter});
  }
  if (--tl_lease_depth == 0 && !tl_parked.empty()) {
    std::vector<std::pair<BlockPool*, void*>> v;
    v.swap(tl_parked);
    for (auto& e : v) e.first->free_now(e.second);
  }
}

// ---- schema helpers -------------------------------------------------------------------------------------
static DType dtype_from_format(const char* f) {
  if (!f) return DType::Null;
  if (!strcmp(f, "l")) return DType::Int64;
  if (!strcmp(f, "g")) return DType::Float64;
  if (!strcmp(f, "u")) return DType::Utf8;
  if (!strcmp(f, "z")) return DType::Binary;
  if (!strcmp(f, "b")) return DType::Bool;
  return DType::Null;
}

std::vector<Field> schema_fields(const ArrowSchema* s) {
  if (!s || !s->format || strcmp(s->format, "+s") != 0)
    fail(ARK_ERR_PROCESS, "Registration failed: expected a struct (RecordBatch) schema");
  std::vector<Field> out;
  for (int64_t i = 0; i < s->n_children; ++i) {
    const ArrowSchema* c = s->children[i];
    Field f;
    f.name = c->name ? c->name : "";
    f.format = c->format ? c->format : "";
    f.type = dtype_from_format(c->format);
    f.nullable = (c->flags & ARROW_FLAG_NULLABLE) != 0;
    out.push_back(f);
  }
  return out;
}

std::string schema_fingerprint(const std::vector<Field>& f) {
  std::string s;
  for (auto& x : f) { s += x.name; s += '\x1f'; s += x.format; s += x.nullable ? "?" : "!"; s += '\x1e'; }
  return s;
}

static bool format_supported(const std::string& f) {
  return f == "l" || f == "g" || f == "u" || f == "z" || f == "b";
}

// the fixed-width types only the protobuf codec reads (import_*'s codec_types)
static DType codec_dtype(const std::string& f) {
  if (f == "i") return DType::Int32;
  if (f == "I") return DType::UInt32;
  if (f == "L") return DType::UInt64;
  if (f == "f") return DType::Float32;
  return DType::Null;
}

// ---- import ---------------------------------------------------------------------------------------------
// Host → device copy of one Arrow buffer.  A Rust shim hands over arrow-rs heap buffers, i.e. PAGEABLE memory: a plain
// cudaMemcpyAsync from such a pointer is staged by the driver through one small pinned buffer, synchronously, at a
// fraction of the link rate.  Large pageable sources are therefore staged here: a small pool of host threads copies
// 2 MB chunks into pinned slots (two per thread, from the pinned pool) and queues each chunk's H2D as soon as it is
// filled, so host memcpy, PCIe transfer and — across concurrent callers — the kernels of other calls overlap.
// Pinned or registered sources (cudaPointerGetAttributes ≠ unregistered) take the direct copy.
int host_copy_stream(void* dst, const void* src, size_t n, int kind);  // host_copy.cpp

namespace {

struct StagePool {
  std::vector<std::thread> threads;
  std::mutex mu;
  std::condition_variable cv;
  std::deque<std::function<void()>> q;
  bool stop = false;
  explicit StagePool(int n) {
    for (int i = 0; i < n; ++i)
      threads.emplace_back([this] {
        for (;;) {
          std::function<void()> f;
          {
            std::unique_lock<std::mutex> l(mu);
            cv.wait(l, [&] { return stop || !q.empty(); });
            if (stop && q.empty()) return;
            f = std::move(q.front());
            q.pop_front();
          }
          f();
        }
      });
  }
  ~StagePool() {
    { std::lock_guard<std::mutex> l(mu); stop = true; }
    cv.notify_all();
    for (auto& t : threads) t.detach();  // process teardown: do not wait on threads that may sit in the CUDA runtime
  }
  void submit(std::function<void()> f) {
    { std::lock_guard<std::mutex> l(mu); q.push_back(std::move(f)); }
    cv.notify_one();
  }
};

int stage_threads() {
  static const int n = [] {
    const char* e = getenv("ARK_STAGE_THREADS");
    int v = e ? atoi(e) : 12;
    return std::max(0, std::min(v, 32));
  }();
  return n;
}
StagePool& stage_pool() {
  static StagePool* p = new StagePool(stage_threads());  // leaked on purpose (see ~BlockPool)
  return *p;
}

// Pageable inputs are staged through pinned chunks by host threads.  With glibc's memcpy those threads, not the PCIe
// copies, bounded the end-to-end rate whatever the chunk size or thread count; with non-temporal copies (host_copy.cpp)
// the threads wait for the PCIe copies, not the other way round.
size_t stage_chunk() {
  static const size_t v = [] {
    if (const char* k = getenv("ARK_STAGE_CHUNK_KB")) return (size_t)std::max(64, std::min(atoi(k), 65536)) << 10;
    const char* e = getenv("ARK_STAGE_CHUNK_MB");
    const int mb = e ? atoi(e) : 4;
    return (size_t)std::max(1, std::min(mb, 64)) << 20;
  }();
  return v;
}
constexpr size_t STAGE_MIN = 8u << 20;  // smaller sources are not worth the hand-off

bool is_pageable(const void* p) {
  cudaPointerAttributes at;
  if (cudaPointerGetAttributes(&at, p) != cudaSuccess) { cudaGetLastError(); return false; }
  return at.type == cudaMemoryTypeUnregistered;
}

void staged_h2d(void* dst, const void* src, size_t n, cudaStream_t s) {
  using clk = std::chrono::steady_clock;
  static const bool trace = getenv("ARK_STAGE_TRACE") != nullptr;
  static const int copy_kind = [] { const char* e = getenv("ARK_STAGE_COPY"); return e ? atoi(e) : -1; }();  // 0 memcpy, 1 AVX2 NT, 2 AVX-512 NT
  const auto t_begin = clk::now();
  const size_t STAGE_CHUNK = stage_chunk();
  const size_t n_chunks = (n + STAGE_CHUNK - 1) / STAGE_CHUNK;
  const int T = (int)std::min<size_t>((size_t)stage_threads(), n_chunks);
  BufferPtr ring = pinned_alloc((size_t)T * 2 * STAGE_CHUNK);
  std::mutex mu;
  std::condition_variable cv;
  int done = 0;
  cudaError_t first_err = cudaSuccess;
  double us_copy = 0, us_wait = 0, us_issue = 0, us_start = 0;
  for (int w = 0; w < T; ++w) {
    stage_pool().submit([&, w] {
      ensure_device();
      const auto t_start = clk::now();
      double my_copy = 0, my_wait = 0, my_issue = 0;
      cudaEvent_t ev[2] = {nullptr, nullptr};
      cudaError_t err = cudaSuccess;
      bool used[2] = {false, false};
      for (int k = 0; k < 2 && err == cudaSuccess; ++k) err = cudaEventCreateWithFlags(&ev[k], cudaEventDisableTiming);
      int turn = 0;
      for (size_t c = (size_t)w; c < n_chunks && err == cudaSuccess; c += (size_t)T, turn ^= 1) {
        uint8_t* slot = (uint8_t*)ring.get() + ((size_t)w * 2 + turn) * STAGE_CHUNK;
        const size_t off = c * STAGE_CHUNK, len = std::min(STAGE_CHUNK, n - off);
        const auto t0 = clk::now();
        if (used[turn]) err = cudaEventSynchronize(ev[turn]);  // the slot's previous chunk has left for the device
        if (err != cudaSuccess) break;
        const auto t1 = clk::now();
        host_copy_stream(slot, (const uint8_t*)src + off, len, copy_kind);
        const auto t2 = clk::now();
        err = cudaMemcpyAsync((uint8_t*)dst + off, slot, len, cudaMemcpyHostToDevice, s);
        if (err == cudaSuccess) err = cudaEventRecord(ev[turn], s);
        used[turn] = true;
        if (trace) {
          const auto t3 = clk::now();
          my_wait += std::chrono::duration<double, std::micro>(t1 - t0).count();
          my_copy += std::chrono::duration<double, std::micro>(t2 - t1).count();
          my_issue += std::chrono::duration<double, std::micro>(t3 - t2).count();
        }
      }
      for (int k = 0; k < 2; ++k) if (ev[k]) cudaEventDestroy(ev[k]);
      std::lock_guard<std::mutex> l(mu);
      if (err != cudaSuccess && first_err == cudaSuccess) first_err = err;
      us_copy += my_copy; us_wait += my_wait; us_issue += my_issue;
      us_start += std::chrono::duration<double, std::micro>(t_start - t_begin).count();
      ++done;
      cv.notify_one();
    });
  }
  {
    std::unique_lock<std::mutex> l(mu);
    cv.wait(l, [&] { return done == T; });
  }
  ARK_CUDA(first_err);
  if (trace) {
    const double wall = std::chrono::duration<double, std::micro>(clk::now() - t_begin).count();
    fprintf(stderr, "[stage] %.1f MB in %.0f us (%.1f GB/s) by %d threads: per thread copy %.0f us (%.1f GB/s each) wait %.0f us issue %.0f us start-lag %.0f us\n",
            n / 1e6, wall, n / 1e3 / wall, T, us_copy / T, n / 1e3 / std::max(us_copy, 1.0), us_wait / T, us_issue / T, us_start / T);
  }
  // `ring` returns to the pinned pool when this call's stream has been synchronised (blocks freed inside a call are
  // parked until then), i.e. after the queued copies have read it
}

}  // namespace

static void h2d(void* dst, const void* src, size_t n, cudaStream_t s, int64_t* acc) {
  if (n == 0) return;
  if (acc) *acc += (int64_t)n;
  if (n >= STAGE_MIN && stage_threads() > 0 && is_pageable(src)) { staged_h2d(dst, src, n, s); return; }
  ARK_CUDA(cudaMemcpyAsync(dst, src, n, cudaMemcpyHostToDevice, s));
}

Batch import_host(const ArrowArray* arr, const ArrowSchema* schema, const std::vector<bool>* needed,
                  cudaStream_t stream, int64_t* h2d_bytes, bool codec_types) {
  std::vector<Field> fields = schema_fields(schema);
  if (arr->n_children != (int64_t)fields.size())
    fail(ARK_ERR_PROCESS, "Registration failed: array/schema child count mismatch");
  if (arr->offset != 0) fail(ARK_ERR_UNSUPPORTED, "struct array with non-zero offset");
  Batch b;
  b.num_rows = arr->length;
  for (size_t i = 0; i < fields.size(); ++i) {
    Column c;
    c.field = fields[i];
    if (codec_types && codec_dtype(c.field.format) != DType::Null) c.field.type = codec_dtype(c.field.format);
    const ArrowArray* a = arr->children[i];
    c.length = a->length;
    bool want = (!needed || (*needed)[i]) && (format_supported(fields[i].format) || c.field.type != fields[i].type);
    if (!want) { c.present = false; b.cols.push_back(std::move(c)); continue; }
    if (a->length != arr->length) fail(ARK_ERR_PROCESS, "Registration failed: column length mismatch");
    int64_t off = a->offset, n = a->length;
    c.null_count = a->null_count;
    if (a->buffers[0] != nullptr && a->null_count != 0 && n > 0) {
      int64_t byte0 = off >> 3, byte1 = (off + n + 7) >> 3;
      BufferPtr v = device_alloc((size_t)(byte1 - byte0));
      h2d(v.get(), (const uint8_t*)a->buffers[0] + byte0, (size_t)(byte1 - byte0), stream, h2d_bytes);
      c.validity = (const uint8_t*)v.get();
      c.validity_bit0 = (int32_t)(off & 7);
      c.null_count = a->null_count;  // may be -1 (unknown): treated as "has nulls"
      c.owners.push_back(v);
    } else {
      c.null_count = 0;
    }
    switch (c.field.type) {
      case DType::Int64: case DType::Float64:
      case DType::Int32: case DType::UInt32: case DType::UInt64: case DType::Float32: {
        const int w = fixed_width(c.field.type);
        BufferPtr d = device_alloc((size_t)n * w);
        if (n) h2d(d.get(), (const uint8_t*)a->buffers[1] + off * w, (size_t)n * w, stream, h2d_bytes);
        c.data = (const uint8_t*)d.get(); c.data_bytes = n * w; c.owners.push_back(d);
        break;
      }
      case DType::Bool: {
        int64_t byte0 = off >> 3, byte1 = (off + n + 7) >> 3;
        BufferPtr d = device_alloc((size_t)(byte1 - byte0));
        if (n) h2d(d.get(), (const uint8_t*)a->buffers[1] + byte0, (size_t)(byte1 - byte0), stream, h2d_bytes);
        c.data = (const uint8_t*)d.get(); c.data_bit0 = (int32_t)(off & 7); c.data_bytes = byte1 - byte0;
        c.owners.push_back(d);
        break;
      }
      case DType::Utf8:
      case DType::Binary: {
        BufferPtr o = device_alloc((size_t)(n + 1) * 4);
        int32_t first = 0, last = 0;
        if (a->buffers[1] != nullptr) {
          const int32_t* ho = (const int32_t*)a->buffers[1] + off;
          first = ho[0]; last = ho[n];
          h2d(o.get(), ho, (size_t)(n + 1) * 4, stream, h2d_bytes);
        } else {
          ARK_CUDA(cudaMemsetAsync(o.get(), 0, (size_t)(n + 1) * 4, stream));
        }
        BufferPtr d = device_alloc((size_t)(last - first));
        if (last > first) h2d(d.get(), (const uint8_t*)a->buffers[2] + first, (size_t)(last - first), stream, h2d_bytes);
        c.offsets = (const int32_t*)o.get();
        c.data = (const uint8_t*)d.get() - first;
        c.data_bytes = last - first; c.first_offset = first;
        c.owners.push_back(o); c.owners.push_back(d);
        break;
      }
      default: break;
    }
    b.cols.push_back(std::move(c));
  }
  return b;
}

__global__ void gather_extents_kernel(const int32_t* const* offs, const int64_t* lens, int32_t* out, int n) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) { out[2 * i] = offs[i][0]; out[2 * i + 1] = offs[i][lens[i]]; }
}

Batch import_device(const ArrowDeviceArray* darr, const ArrowSchema* schema, const std::vector<bool>* needed,
                    BufferPtr keep, bool codec_types, const std::vector<Field>* known_fields) {
  if (darr->device_type != ARROW_DEVICE_CUDA && darr->device_type != ARROW_DEVICE_CUDA_HOST)
    fail(ARK_ERR_PROCESS, "Registration failed: ArrowDeviceArray is not on a CUDA device");
  const ArrowArray* arr = &darr->array;
  if (darr->sync_event) ARK_CUDA(cudaEventSynchronize(*(cudaEvent_t*)darr->sync_event));
  std::vector<Field> parsed;
  if (!known_fields) parsed = schema_fields(schema);
  const std::vector<Field>& fields = known_fields ? *known_fields : parsed;
  if (arr->n_children != (int64_t)fields.size())
    fail(ARK_ERR_PROCESS, "Registration failed: array/schema child count mismatch");
  if (arr->offset != 0) fail(ARK_ERR_UNSUPPORTED, "struct array with non-zero offset");
  Batch b;
  b.num_rows = arr->length;
  std::vector<int> varlen_idx;
  for (size_t i = 0; i < fields.size(); ++i) {
    Column c;
    c.field = fields[i];
    if (codec_types && codec_dtype(c.field.format) != DType::Null) c.field.type = codec_dtype(c.field.format);
    const ArrowArray* a = arr->children[i];
    c.length = a->length;
    bool want = (!needed || (*needed)[i]) && (format_supported(fields[i].format) || c.field.type != fields[i].type);
    if (!want) { c.present = false; b.cols.push_back(std::move(c)); continue; }
    if (a->length != arr->length) fail(ARK_ERR_PROCESS, "Registration failed: column length mismatch");
    int64_t off = a->offset, n = a->length;
    if (keep) c.owners.push_back(keep);
    if (a->buffers[0] != nullptr && a->null_count != 0) {
      c.validity = (const uint8_t*)a->buffers[0] + (off >> 3);
      c.validity_bit0 = (int32_t)(off & 7);
      c.null_count = a->null_count;
    } else c.null_count = 0;
    switch (c.field.type) {
      case DType::Int64: case DType::Float64:
      case DType::Int32: case DType::UInt32: case DType::UInt64: case DType::Float32: {
        const int w = fixed_width(c.field.type);
        c.data = (const uint8_t*)a->buffers[1] + off * w; c.data_bytes = n * w; break;
      }
      case DType::Bool:
        c.data = (const uint8_t*)a->buffers[1] + (off >> 3); c.data_bit0 = (int32_t)(off & 7);
        c.data_bytes = (n + 7) / 8 + 1; break;
      case DType::Utf8: case DType::Binary:
        c.offsets = (const int32_t*)a->buffers[1] + off;
        c.data = (const uint8_t*)a->buffers[2];
        c.data_bytes = -1;  // unknown until resolve_varlen_extents(); most paths only need an upper bound
        c.data_bound = a->buffers[2] ? std::min<int64_t>(device_alloc_remaining(a->buffers[2]), 2147483647ll) : 0;
        break;
      default: break;
    }
    b.cols.push_back(std::move(c));
  }
  return b;
}

int64_t device_alloc_remaining(const void* p) {
  typedef int (*fn_t)(unsigned long long*, size_t*, unsigned long long);
  static fn_t fn = [] {
    void* f = nullptr;
    cudaDriverEntryPointQueryResult st;
    if (cudaGetDriverEntryPoint("cuMemGetAddressRange", &f, cudaEnableDefault, &st) != cudaSuccess || st != cudaDriverEntryPointSuccess) {
      cudaGetLastError();
      f = nullptr;
    }
    return (fn_t)f;
  }();
  if (!fn || !p) return -1;
  unsigned long long base = 0;
  size_t size = 0;
  if (fn(&base, &size, (unsigned long long)(uintptr_t)p) != 0) return -1;
  return (int64_t)(base + size - (unsigned long long)(uintptr_t)p);
}

// base address and size of the CUDA allocation that contains p
bool device_alloc_range(const void* p, unsigned long long* base, size_t* size) {
  const int64_t rest = device_alloc_remaining(p);
  if (rest < 0) return false;
  typedef int (*fn_t)(unsigned long long*, size_t*, unsigned long long);
  void* f = nullptr;
  cudaDriverEntryPointQueryResult st;
  if (cudaGetDriverEntryPoint("cuMemGetAddressRange", &f, cudaEnableDefault, &st) != cudaSuccess || st != cudaDriverEntryPointSuccess) { cudaGetLastError(); return false; }
  return ((fn_t)f)(base, size, (unsigned long long)(uintptr_t)p) == 0;
}

int64_t varlen_bytes_bound(const Column& c) {
  if (c.data_bytes >= 0) return c.data_bytes;
  return c.data_bound;
}

// Fetch offsets[0] / offsets[n] of device-resident var-len columns whose extent is still unknown.
// Reads offsets[0] and offsets[length] of every var-len column whose byte extent is still unknown — all
// of them (across batches) with ONE kernel, one D2H copy and one stream synchronize.
void resolve_varlen_extents_many(std::vector<Column*>& cols, cudaStream_t stream) {
  std::vector<Column*> todo;
  for (Column* c : cols) {
    if (c->present && (c->field.type == DType::Utf8 || c->field.type == DType::Binary) && c->data_bytes < 0) {
      if (c->length == 0 || c->offsets == nullptr) { c->data_bytes = 0; c->first_offset = 0; }
      else todo.push_back(c);
    }
  }
  if (todo.empty()) return;
  const size_t n = todo.size();
  // layout (pinned & device): [pointers n×8][lens n×8][out n×8]
  BufferPtr hp = pinned_alloc(n * 24 + 64);
  BufferPtr dp = device_alloc(n * 24 + 64);
  const int32_t** hptr = (const int32_t**)hp.get();
  int64_t* hlen = (int64_t*)((char*)hp.get() + n * 8);
  int32_t* hout = (int32_t*)((char*)hp.get() + n * 16);
  for (size_t k = 0; k < n; ++k) { hptr[k] = todo[k]->offsets; hlen[k] = todo[k]->length; }
  ARK_CUDA(cudaMemcpyAsync(dp.get(), hp.get(), n * 16, cudaMemcpyHostToDevice, stream));
  {
    KernelTimer t("gather_extents_kernel", stream);
    gather_extents_kernel<<<(unsigned)ceil_div((int64_t)n, 32), 32, 0, stream>>>((const int32_t* const*)dp.get(), (const int64_t*)((char*)dp.get() + n * 8),
                                                                            (int32_t*)((char*)dp.get() + n * 16), (int)n);
  }
  ARK_CUDA(cudaMemcpyAsync(hout, (char*)dp.get() + n * 16, n * 8, cudaMemcpyDeviceToHost, stream));
  ARK_CUDA(cudaStreamSynchronize(stream));
  for (size_t k = 0; k < n; ++k) {
    todo[k]->first_offset = hout[2 * k];
    todo[k]->data_bytes = (int64_t)hout[2 * k + 1] - hout[2 * k];
  }
}

void resolve_varlen_extents(Batch& b, const std::vector<int>& col_idx, cudaStream_t stream) {
  std::vector<Column*> cols;
  for (int i : col_idx) cols.push_back(&b.cols[i]);
  resolve_varlen_extents_many(cols, stream);
}

// ---- export ---------------------------------------------------------------------------------------------
void resolve_varlen_extents(Batch& b, const std::vector<int>& col_idx, cudaStream_t stream);
namespace {

struct SchemaPriv {
  std::string format, name;
  std::vector<ArrowSchema> child_storage;
  std::vector<ArrowSchema*> child_ptrs;
};
void release_schema(ArrowSchema* s) {
  if (!s || !s->release) return;
  auto* p = (SchemaPriv*)s->private_data;
  for (auto& c : p->child_storage) if (c.release) c.release(&c);
  delete p;
  s->release = nullptr;
}
void fill_schema(ArrowSchema* s, const char* fmt, const std::string& name, bool nullable) {
  auto* p = new SchemaPriv();
  p->format = fmt; p->name = name;
  memset(s, 0, sizeof(*s));
  s->format = p->format.c_str(); s->name = p->name.c_str(); s->metadata = nullptr;
  s->flags = nullable ? ARROW_FLAG_NULLABLE : 0;
  s->release = release_schema; s->private_data = p;
}

struct ArrayPriv {
  std::vector<BufferPtr> owners;
  std::vector<const void*> buffers;
  std::vector<ArrowArray> child_storage;
  std::vector<ArrowArray*> child_ptrs;
};
void release_array(ArrowArray* a) {
  if (!a || !a->release) return;
  auto* p = (ArrayPriv*)a->private_data;
  for (auto& c : p->child_storage) if (c.release) c.release(&c);
  delete p;
  a->release = nullptr;
}

__global__ void rebase_offsets_kernel(const int32_t* in, int32_t* out, int64_t n1, int32_t first) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n1) out[i] = in[i] - first;
}
}  // namespace

static void fill_column_schema(ArrowSchema* s, const Column& c) {
  fill_schema(s, dtype_arrow_format(c.field.type), c.field.name, c.field.nullable);
  if (c.children.empty()) return;
  auto* p = (SchemaPriv*)s->private_data;
  p->child_storage.resize(c.children.size());
  p->child_ptrs.resize(c.children.size());
  for (size_t i = 0; i < c.children.size(); ++i) {
    fill_column_schema(&p->child_storage[i], c.children[i]);
    p->child_ptrs[i] = &p->child_storage[i];
  }
  s->n_children = (int64_t)c.children.size();
  s->children = p->child_ptrs.data();
}

void export_schema(const Batch& b, ArrowSchema* out) {
  fill_schema(out, "+s", "", false);
  auto* p = (SchemaPriv*)out->private_data;
  p->child_storage.resize(b.cols.size());
  p->child_ptrs.resize(b.cols.size());
  for (size_t i = 0; i < b.cols.size(); ++i) {
    fill_column_schema(&p->child_storage[i], b.cols[i]);
    p->child_ptrs[i] = &p->child_storage[i];
  }
  out->n_children = (int64_t)b.cols.size();
  out->children = p->child_ptrs.data();
}

void export_empty_schema(ArrowSchema* out) {
  Batch b;
  export_schema(b, out);
}

// Normalised device view of a column for export: offsets rebased to 0, bitmaps starting at bit 0.
struct ExportCol {
  const uint8_t* validity = nullptr; int64_t validity_bytes = 0;
  const void* buf1 = nullptr; int64_t buf1_bytes = 0;
  const void* buf2 = nullptr; int64_t buf2_bytes = 0;
  int n_buffers = 2;
  std::vector<BufferPtr> owners;
};

static ExportCol normalise_for_export(const Column& c_in, bool to_host, cudaStream_t stream) {
  Column c = c_in;
  if (to_host && c.present && (c.field.type == DType::Utf8 || c.field.type == DType::Binary) && c.data_bytes < 0) {
    Batch tmp;  // the extent is needed to size the D2H copy
    tmp.cols.push_back(c);
    tmp.num_rows = c.length;
    resolve_varlen_extents(tmp, {0}, stream);
    c = tmp.cols[0];
  }
  ExportCol e;
  e.owners = c.owners;
  int64_t n = c.length;
  if (c.validity && c.null_count != 0 && n > 0) {
    e.validity_bytes = (n + 7) / 8;
    if (c.validity_bit0 != 0) {
      BufferPtr v = realign_bits(c.validity, c.validity_bit0, n, stream);
      e.validity = (const uint8_t*)v.get(); e.owners.push_back(v);
    } else e.validity = c.validity;
  }
  switch (c.field.type) {
    case DType::Int64: case DType::Float64:
    case DType::Int32: case DType::UInt32: case DType::UInt64: case DType::Float32:
      e.buf1 = c.data; e.buf1_bytes = n * fixed_width(c.field.type); e.n_buffers = 2; break;
    case DType::Bool:
      e.buf1_bytes = (n + 7) / 8;
      if (c.data_bit0 != 0 && n > 0) {
        BufferPtr v = realign_bits(c.data, c.data_bit0, n, stream);
        e.buf1 = v.get(); e.owners.push_back(v);
      } else e.buf1 = c.data;
      e.n_buffers = 2; break;
    case DType::Utf8: case DType::Binary: {
      e.n_buffers = 3;
      e.buf1_bytes = (n + 1) * 4;
      // device export: Arrow does not require offsets[0] == 0; hand the buffers over as they are, unless offsets[0] != 0 is
      // known.  A host import points `data` offsets[0] bytes before its allocation, which no consumer may be handed.
      if (!to_host && c.first_offset == 0) {
        if (c.offsets) e.buf1 = c.offsets;
        else { BufferPtr o = device_alloc(4); ARK_CUDA(cudaMemsetAsync(o.get(), 0, 4, stream)); e.buf1 = o.get(); e.owners.push_back(o); }
        e.buf2 = c.data; e.buf2_bytes = std::max<int64_t>(c.data_bytes, 0);
        break;
      }
      if (c.first_offset != 0 && c.offsets) {
        BufferPtr o = device_alloc((size_t)e.buf1_bytes);
        KernelTimer t("rebase_offsets_kernel", stream);
        rebase_offsets_kernel<<<(unsigned)ceil_div(n + 1, 256), 256, 0, stream>>>(c.offsets, (int32_t*)o.get(), n + 1, (int32_t)c.first_offset);
        e.buf1 = o.get(); e.owners.push_back(o);
      } else if (c.offsets) e.buf1 = c.offsets;
      else {
        BufferPtr o = device_alloc(4);
        ARK_CUDA(cudaMemsetAsync(o.get(), 0, 4, stream));
        e.buf1 = o.get(); e.owners.push_back(o);
      }
      e.buf2 = c.data ? c.data + c.first_offset : nullptr; e.buf2_bytes = c.data_bytes;
      break;
    }
    case DType::List:  // offsets (library-produced: first offset 0) + one child
      e.buf1 = c.offsets; e.buf1_bytes = (n + 1) * 4; e.n_buffers = 2; break;
    case DType::Struct:
      e.n_buffers = 1; break;
    default: e.n_buffers = 0; break;
  }
  return e;
}

// one column (and, for List / Struct, its children) as an ArrowArray
static void build_column_array(const Column& c, ExportCol& e, bool to_host, cudaStream_t stream, ArrowArray* ca, int64_t* d2h_bytes) {
  auto* cp = new ArrayPriv();
  memset(ca, 0, sizeof(*ca));
  ca->length = c.length; ca->offset = 0;
  ca->null_count = e.validity ? (c.null_count < 0 ? -1 : c.null_count) : 0;
  auto place = [&](const void* dptr, int64_t bytes) -> const void* {
    if (!to_host) return dptr;
    if (!dptr && bytes == 0) {
      BufferPtr h = pinned_alloc(64);
      cp->owners.push_back(h);
      return h.get();
    }
    BufferPtr h = pinned_alloc((size_t)std::max<int64_t>(bytes, 1));
    if (bytes > 0) {
      ARK_CUDA(cudaMemcpyAsync(h.get(), dptr, (size_t)bytes, cudaMemcpyDeviceToHost, stream));
      if (d2h_bytes) *d2h_bytes += bytes;
    }
    cp->owners.push_back(h);
    return h.get();
  };
  if (c.field.type == DType::Null) {
    ca->n_buffers = 0; ca->null_count = c.length;
  } else {
    cp->buffers.push_back(e.validity ? place(e.validity, e.validity_bytes) : nullptr);
    if (e.n_buffers >= 2) cp->buffers.push_back(place(e.buf1, e.buf1_bytes));
    if (e.n_buffers == 3) cp->buffers.push_back(place(e.buf2, e.buf2_bytes));
    ca->n_buffers = (int64_t)cp->buffers.size();
  }
  ca->buffers = cp->buffers.data();
  if (!to_host) cp->owners = e.owners;  // device export keeps the HBM blocks alive
  if (!c.children.empty()) {
    cp->child_storage.resize(c.children.size());
    cp->child_ptrs.resize(c.children.size());
    for (size_t k = 0; k < c.children.size(); ++k) {
      ExportCol ce = normalise_for_export(c.children[k], to_host, stream);
      build_column_array(c.children[k], ce, to_host, stream, &cp->child_storage[k], d2h_bytes);
      cp->child_ptrs[k] = &cp->child_storage[k];
    }
    ca->n_children = (int64_t)c.children.size();
    ca->children = cp->child_ptrs.data();
  }
  ca->release = release_array; ca->private_data = cp;
}

static void build_struct_array(const Batch& b, std::vector<ExportCol>& cols, bool to_host, cudaStream_t stream,
                               ArrowArray* out, int64_t* d2h_bytes) {
  auto* top = new ArrayPriv();
  memset(out, 0, sizeof(*out));
  out->length = b.num_rows; out->null_count = 0; out->offset = 0;
  top->buffers.push_back(nullptr);
  out->n_buffers = 1; out->buffers = top->buffers.data();
  top->child_storage.resize(cols.size());
  top->child_ptrs.resize(cols.size());
  for (size_t i = 0; i < cols.size(); ++i) {
    build_column_array(b.cols[i], cols[i], to_host, stream, &top->child_storage[i], d2h_bytes);
    top->child_ptrs[i] = &top->child_storage[i];
  }
  out->n_children = (int64_t)cols.size();
  out->children = top->child_ptrs.data();
  out->release = release_array; out->private_data = top;
}

void export_host(const Batch& b, cudaStream_t stream, ArrowArray* out, ArrowSchema* out_schema, int64_t* d2h_bytes) {
  std::vector<ExportCol> cols;
  for (auto& c : b.cols) cols.push_back(normalise_for_export(c, true, stream));
  build_struct_array(b, cols, true, stream, out, d2h_bytes);
  ARK_CUDA(cudaStreamSynchronize(stream));
  export_schema(b, out_schema);
}

void export_device(const Batch& b, ArrowDeviceArray* out, ArrowSchema* out_schema, StreamLease& lease) {
  std::vector<ExportCol> cols;
  for (auto& c : b.cols) cols.push_back(normalise_for_export(c, false, lease.s));
  memset(out, 0, sizeof(*out));
  build_struct_array(b, cols, false, lease.s, &out->array, nullptr);
  lease.synchronize_last();
  int dev = 0; cudaGetDevice(&dev);
  out->device_id = dev; out->device_type = ARROW_DEVICE_CUDA; out->sync_event = nullptr;
  export_schema(b, out_schema);
}

BufferPtr adopt_array(ArrowArray* arr) {
  if (!arr || !arr->release) return BufferPtr();
  auto* moved = new ArrowArray(*arr);
  arr->release = nullptr;  // moved
  return BufferPtr(moved, [](void* p) {
    auto* a = (ArrowArray*)p;
    if (a->release) a->release(a);
    delete a;
  });
}

}  // namespace ark
