// runtime.cu -- contexts, CUDA-IPC regions, staging pipelines, graphs and the
// extern "C" surface declared in include/tb200.h.
//
// Reference behaviour this file restates (paths under the reference root,
// PY = src/python/library/tritonclient):
//   PY/utils/cuda_shared_memory/__init__.py:107-149  region create (cudaMalloc + IPC handle)
//   PY/utils/cuda_shared_memory/__init__.py:173-239  host arrays -> region (H2D + sync)
//   PY/utils/cuda_shared_memory/__init__.py:242-325  region -> host
//   PY/utils/cuda_shared_memory/_utils.py:67-121     region / stream lifetime
// The device work itself lives in kernels.cu.
#include <cuda_runtime.h>

#include <algorithm>
#include <atomic>
#include <condition_variable>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cmath>
#include <cstring>
#include <functional>
#include <mutex>
#include <string>
#include <thread>
#include <vector>

#include "kernels.cuh"
#include "resample.h"

namespace {

thread_local std::string g_last_error;

int fail(int code, const char* fmt, ...) {
  char buf[512];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  g_last_error = buf;
  return code;
}

#define TB200_CUDA(expr)                                                              \
  do {                                                                                \
    cudaError_t e__ = (expr);                                                         \
    if (e__ != cudaSuccess) {                                                         \
      return fail(TB200_ERR_CUDA, "%s failed: %s", #expr, cudaGetErrorString(e__));   \
    }                                                                                 \
  } while (0)

// switch to a device for the duration of a call and switch back (the reference
// does the same around every runtime call, cuda_shared_memory/__init__.py:128-147)
class DeviceGuard {
 public:
  explicit DeviceGuard(int dev) {
    if (cudaGetDevice(&prev_) != cudaSuccess) prev_ = -1;
    if (prev_ != dev) {
      err_ = cudaSetDevice(dev);
      switched_ = (err_ == cudaSuccess);
    }
  }
  ~DeviceGuard() {
    if (switched_ && prev_ >= 0) cudaSetDevice(prev_);
  }
  cudaError_t error() const { return err_; }

 private:
  int prev_ = -1;
  bool switched_ = false;
  cudaError_t err_ = cudaSuccess;
};

// ---- a tiny fork/join pool for the host side of the staging pipeline ----------
class CopyPool {
 public:
  static CopyPool& instance() {
    static CopyPool pool;
    return pool;
  }
  int threads() const { return static_cast<int>(workers_.size()) + 1; }
  // split [0, n) into contiguous pieces and memcpy them in parallel
  void parallel_memcpy(void* dst, const void* src, size_t n) {
    const int parts = (n < (1u << 20)) ? 1 : std::min<int>(threads(), static_cast<int>(n >> 18));
    if (parts <= 1) {
      memcpy(dst, src, n);
      return;
    }
    const size_t piece = ((n / parts) + 63) & ~static_cast<size_t>(63);
    std::unique_lock<std::mutex> lk(mu_);
    pending_ = 0;
    for (int p = 1; p < parts; ++p) {
      const size_t off = piece * p;
      if (off >= n) break;
      const size_t len = std::min(piece, n - off);
      tasks_.push_back({static_cast<char*>(dst) + off, static_cast<const char*>(src) + off, len});
      ++pending_;
    }
    lk.unlock();
    cv_.notify_all();
    memcpy(dst, src, std::min(piece, n));
    lk.lock();
    done_cv_.wait(lk, [&] { return pending_ == 0; });
  }

 private:
  struct Task {
    char* dst;
    const char* src;
    size_t len;
  };
  CopyPool() {
    int n = 4;
    if (const char* env = getenv("TB200_COPY_THREADS")) n = atoi(env);
    else {
      const unsigned hc = std::thread::hardware_concurrency();
      n = static_cast<int>(std::max(1u, std::min(16u, hc / 2)));
    }
    n = std::max(1, std::min(n, 64));
    for (int i = 1; i < n; ++i) workers_.emplace_back([this] { run(); });
  }
  ~CopyPool() {
    {
      std::lock_guard<std::mutex> lk(mu_);
      stop_ = true;
    }
    cv_.notify_all();
    for (auto& t : workers_) t.join();
  }
  void run() {
    std::unique_lock<std::mutex> lk(mu_);
    for (;;) {
      cv_.wait(lk, [&] { return stop_ || !tasks_.empty(); });
      if (stop_) return;
      Task t = tasks_.back();
      tasks_.pop_back();
      lk.unlock();
      memcpy(t.dst, t.src, t.len);
      lk.lock();
      if (--pending_ == 0) done_cv_.notify_all();
    }
  }
  std::mutex mu_;
  std::condition_variable cv_, done_cv_;
  std::vector<Task> tasks_;
  std::vector<std::thread> workers_;
  int pending_ = 0;
  bool stop_ = false;
};

constexpr size_t kStageBytes = 8u << 20;  // one pinned staging buffer
static size_t kDirectBytes = 2u << 20;    // up to this size the driver's own staging is used: it holds up better when many client
                                           // processes contend; "h2d_direct_kb" knob
constexpr int kStageCount = 4;            // in flight per context
constexpr size_t kJobSlotBytes = 64u << 10;
constexpr int kJobSlots = 32;
constexpr size_t kFlushBytes = 256u << 20;  // > the 50 MB L2 of an H100

}  // namespace

struct tb200_graph {
  cudaGraph_t graph = nullptr;
  cudaGraphExec_t exec = nullptr;
  int device = 0;
  uint64_t kernels_per_launch = 0;
  std::vector<void*> device_allocs;  // job tables owned by the graph
};

struct tb200_ctx {
  int device = 0;
  int sm_count = 0;
  cudaStream_t stream = nullptr;   // main stream
  cudaStream_t cur = nullptr;      // stream launches go to (main, or side between fork/join)
  cudaStream_t side = nullptr;
  cudaEvent_t ev_fork = nullptr, ev_join = nullptr;
  // pipelined steps (tb200_step_submit / tb200_step_wait): per ring entry the event after the
  // fill (main stream) and after the validation (side stream)
  cudaEvent_t step_ev[TB200_STEP_DEPTH][2] = {};
  uint64_t step_ticket[TB200_STEP_DEPTH] = {};  // ticket occupying the entry, 0 = free
  bool step_has_side[TB200_STEP_DEPTH] = {};
  uint64_t step_next = 1;
  bool own_stream = true;
  bool forked = false;
  uint64_t launches = 0;
  // pinned staging ring for host <-> region copies
  void* stage[kStageCount] = {nullptr, nullptr, nullptr, nullptr};
  cudaEvent_t stage_ev[kStageCount] = {nullptr, nullptr, nullptr, nullptr};
  int stage_next = 0;
  // job-table upload ring (pinned host mirror + device copy)
  char* job_host = nullptr;
  char* job_dev = nullptr;
  // a slot may be rewritten once a full synchronisation happened after its last use:
  // job_epoch[slot] < sync_epoch; otherwise the stream it went to is synchronised first
  uint64_t sync_epoch = 1;
  uint64_t job_epoch[kJobSlots];
  // ... or when a pipelined step submitted after it has been waited for (tb200_step_wait)
  uint64_t upload_seq = 0, uploads_done = 0;
  uint64_t job_seq[kJobSlots] = {};
  uint64_t step_upload_mark[TB200_STEP_DEPTH] = {};
  cudaStream_t job_stream[kJobSlots];
  int job_next = 0;
  // check scratch
  tb200::CheckAccum* accum = nullptr;
  uint32_t accum_cap = 0;
  // epoch + flush scratch
  uint64_t* dev_epoch = nullptr;       // [0] epoch, [1] CTA-done counter of the fill kernel
  void* flush_buf = nullptr;
  // resize coefficient tables, keyed by (src_h, src_w, dst_h, dst_w); device resident
  struct ResizeTables {
    int sh, sw, dh, dw, hk, vk, max_rows[6];  // max source rows a tile of 32/16/8/4/2/1 output rows needs
    int max_span;                             // max source columns a 32-column output tile needs
    void* dev;                                // hbounds | vbounds | hcoeffs | vcoeffs
    size_t off_vb, off_hc, off_vc;
  };
  std::vector<ResizeTables> resize_tables;
  // deflate scratch: per-chunk output slots + metadata
  void* deflate_scratch = nullptr;
  void* deflate_meta = nullptr;
  uint64_t deflate_chunks_cap = 0;
  // BYTES decode scratch: where each payload starts in the source
  uint64_t* bytes_src_off = nullptr;
  uint64_t bytes_src_off_cap = 0;
  // capture state
  tb200_graph* capture = nullptr;
  uint64_t capture_launches0 = 0;
  uint64_t capture_epoch = 0;  // device-epoch advance accumulated by the capture's fill_epoch calls (applied by its last node)
  // programmatic dependent launch of back-to-back homogeneous fills: the previous launch on
  // stream s (0 main, 1 side) was a fill_uniform_kernel writing [pdl_lo[s], pdl_hi[s]) iff pdl_mark[s] == stream_seq[s]
  uint64_t stream_seq[2] = {0, 0};
  uint64_t pdl_mark[2] = {~0ull, ~0ull};
  struct PdlEntry {
    std::vector<std::pair<uint64_t, uint64_t>> spans;  // [lo, hi) written, sorted and merged
    uint32_t grid;
  };
  std::vector<PdlEntry> pdl_chain[2];  // most recent last; the launches of the current overlap chain
};

struct tb200_timer {
  tb200_ctx* ctx = nullptr;
  cudaEvent_t start = nullptr, stop = nullptr;
};

struct tb200_region {
  std::string name;
  void* base = nullptr;
  uint64_t size = 0;
  int device = 0;
  bool opened = false;  // mapped from another process's handle
  cudaIpcMemHandle_t handle;
};

namespace {

// every kernel launch is counted per context and per stream (main / side); the per-stream
// count tells a fill whether the previous kernel of ITS stream was a fill as well
inline void count_launch(tb200_ctx* ctx, uint64_t n = 1) {
  ctx->launches += n;
  ctx->stream_seq[ctx->cur == ctx->side && ctx->side != nullptr ? 1 : 0] += n;
}
inline uint64_t stream_seq(const tb200_ctx* ctx) { return ctx->stream_seq[ctx->cur == ctx->side && ctx->side != nullptr ? 1 : 0]; }

int ensure_stage(tb200_ctx* ctx) {
  if (ctx->stage[0] != nullptr) return TB200_OK;
  for (int i = 0; i < kStageCount; ++i) {
    TB200_CUDA(cudaHostAlloc(&ctx->stage[i], kStageBytes, cudaHostAllocDefault));
    TB200_CUDA(cudaEventCreateWithFlags(&ctx->stage_ev[i], cudaEventDisableTiming));
  }
  return TB200_OK;
}

int ensure_jobs(tb200_ctx* ctx) {
  if (ctx->job_host != nullptr) return TB200_OK;
  void* h = nullptr;
  void* d = nullptr;
  TB200_CUDA(cudaHostAlloc(&h, kJobSlotBytes * kJobSlots, cudaHostAllocDefault));
  TB200_CUDA(cudaMalloc(&d, kJobSlotBytes * kJobSlots));
  ctx->job_host = static_cast<char*>(h);
  ctx->job_dev = static_cast<char*>(d);
  for (int i = 0; i < kJobSlots; ++i) {
    ctx->job_epoch[i] = 0;
    ctx->job_stream[i] = nullptr;
  }
  return TB200_OK;
}

// Make `bytes` of host data available on the device for the next kernel on the
// context's stream.  Outside capture: pinned ring slot + async H2D.  During
// capture: a dedicated device buffer owned by the graph, filled synchronously now
// (job tables are constants of the graph, replays upload nothing).
int upload(tb200_ctx* ctx, const void* host, size_t bytes, const void** dev_out) {
  if (bytes > kJobSlotBytes) return fail(TB200_ERR_INVALID, "job table of %zu bytes exceeds %zu", bytes, kJobSlotBytes);
  if (ctx->capture != nullptr) {
    void* d = nullptr;
    TB200_CUDA(cudaMalloc(&d, bytes == 0 ? 16 : bytes));
    ctx->capture->device_allocs.push_back(d);
    TB200_CUDA(cudaMemcpy(d, host, bytes, cudaMemcpyHostToDevice));
    *dev_out = d;
    return TB200_OK;
  }
  int rc = ensure_jobs(ctx);
  if (rc != TB200_OK) return rc;
  const int slot = ctx->job_next;
  ctx->job_next = (slot + 1) % kJobSlots;
  if (ctx->job_epoch[slot] == ctx->sync_epoch && ctx->job_seq[slot] > ctx->uploads_done) {
    // 32 uploads without a synchronisation in between: wait for the slot's previous copy
    TB200_CUDA(cudaStreamSynchronize(ctx->job_stream[slot]));
  }
  char* h = ctx->job_host + slot * kJobSlotBytes;
  char* d = ctx->job_dev + slot * kJobSlotBytes;
  memcpy(h, host, bytes);
  TB200_CUDA(cudaMemcpyAsync(d, h, bytes, cudaMemcpyHostToDevice, ctx->cur));
  ctx->job_epoch[slot] = ctx->sync_epoch;
  ctx->job_seq[slot] = ++ctx->upload_seq;
  ctx->job_stream[slot] = ctx->cur;
  *dev_out = d;
  return TB200_OK;
}

int check_range(const tb200_region* r, uint64_t offset, uint64_t nbytes) {
  if (offset > r->size || nbytes > r->size - offset) {
    return fail(TB200_ERR_RANGE, "range [%llu, +%llu) outside region '%s' of %llu bytes",
                static_cast<unsigned long long>(offset), static_cast<unsigned long long>(nbytes),
                r->name.c_str(), static_cast<unsigned long long>(r->size));
  }
  return TB200_OK;
}

// host -> device through the pinned ring; does not synchronise at the end
int staged_h2d(tb200_ctx* ctx, char* dst, const char* src, uint64_t nbytes) {
  if (nbytes <= kDirectBytes) {
    // small tensors (C1 / C4 / C5): the copy from pageable memory is staged by the driver
    // before cudaMemcpyAsync returns; nothing to gain from our own ring
    TB200_CUDA(cudaMemcpyAsync(dst, src, nbytes, cudaMemcpyHostToDevice, ctx->cur));
    return TB200_OK;
  }
  int rc = ensure_stage(ctx);
  if (rc != TB200_OK) return rc;
  uint64_t done = 0;
  while (done < nbytes) {
    const size_t n = static_cast<size_t>(std::min<uint64_t>(kStageBytes, nbytes - done));
    const int b = ctx->stage_next;
    ctx->stage_next = (b + 1) % kStageCount;
    TB200_CUDA(cudaEventSynchronize(ctx->stage_ev[b]));  // buffer free again?
    CopyPool::instance().parallel_memcpy(ctx->stage[b], src + done, n);
    TB200_CUDA(cudaMemcpyAsync(dst + done, ctx->stage[b], n, cudaMemcpyHostToDevice, ctx->cur));
    TB200_CUDA(cudaEventRecord(ctx->stage_ev[b], ctx->cur));
    done += n;
  }
  return TB200_OK;
}

}  // namespace

using namespace tb200;

namespace tb200 {
void set_last_error(const char* msg) { g_last_error = msg ? msg : ""; }
}  // namespace tb200

extern "C" {

// ---------------------------------------------------------------------------
// misc
// ---------------------------------------------------------------------------
uint32_t tb200_dtype_size(uint32_t dtype) {
  switch (dtype) {
    case TB200_BOOL: case TB200_UINT8: case TB200_INT8: return 1;
    case TB200_UINT16: case TB200_INT16: case TB200_FP16: case TB200_BF16: return 2;
    case TB200_UINT32: case TB200_INT32: case TB200_FP32: return 4;
    case TB200_UINT64: case TB200_INT64: case TB200_FP64: return 8;
    default: return 0;
  }
}

static const char* const kDtypeNames[] = {"",      "BOOL",  "UINT8", "UINT16", "UINT32",
                                          "UINT64", "INT8",  "INT16", "INT32",  "INT64",
                                          "FP16",  "FP32",  "FP64",  "BYTES",  "BF16"};

uint32_t tb200_dtype_from_name(const char* name) {
  if (name == nullptr) return TB200_INVALID;
  for (uint32_t i = 1; i <= TB200_BF16; ++i) {
    if (strcmp(name, kDtypeNames[i]) == 0) return i;
  }
  return TB200_INVALID;
}
const char* tb200_dtype_name(uint32_t dtype) {
  return (dtype >= 1 && dtype <= TB200_BF16) ? kDtypeNames[dtype] : "";
}

int tb200_abi_version(void) { return TB200_ABI_VERSION; }
const char* tb200_last_error(void) { return g_last_error.c_str(); }

int tb200_device_count(int* count) {
  if (count == nullptr) return fail(TB200_ERR_INVALID, "count is NULL");
  *count = 0;
  TB200_CUDA(cudaGetDeviceCount(count));
  return TB200_OK;
}

// ---------------------------------------------------------------------------
// contexts
// ---------------------------------------------------------------------------
int tb200_ctx_create(int device_id, tb200_ctx** out) {
  if (out == nullptr) return fail(TB200_ERR_INVALID, "out is NULL");
  *out = nullptr;
  int n = 0;
  TB200_CUDA(cudaGetDeviceCount(&n));
  if (device_id < 0 || device_id >= n) return fail(TB200_ERR_INVALID, "device %d not in [0,%d)", device_id, n);
  DeviceGuard g(device_id);
  TB200_CUDA(g.error());
  tb200_ctx* ctx = new tb200_ctx();
  ctx->device = device_id;
  cudaError_t e = cudaDeviceGetAttribute(&ctx->sm_count, cudaDevAttrMultiProcessorCount, device_id);
  if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking);
  void* ep = nullptr;
  if (e == cudaSuccess) e = cudaMalloc(&ep, 2 * sizeof(uint64_t));
  if (e == cudaSuccess) e = cudaMemset(ep, 0, 2 * sizeof(uint64_t));
  if (e != cudaSuccess) {
    delete ctx;
    return fail(TB200_ERR_CUDA, "context setup failed: %s", cudaGetErrorString(e));
  }
  ctx->dev_epoch = static_cast<uint64_t*>(ep);
  ctx->cur = ctx->stream;
  *out = ctx;
  return TB200_OK;
}

int tb200_ctx_destroy(tb200_ctx* ctx) {
  if (ctx == nullptr) return TB200_OK;
  DeviceGuard g(ctx->device);
  cudaStreamSynchronize(ctx->stream);
  for (int i = 0; i < kStageCount; ++i) {
    if (ctx->stage[i]) cudaFreeHost(ctx->stage[i]);
    if (ctx->stage_ev[i]) cudaEventDestroy(ctx->stage_ev[i]);
  }
  if (ctx->job_host) {
    cudaFreeHost(ctx->job_host);
    cudaFree(ctx->job_dev);
  }
  if (ctx->accum) cudaFree(ctx->accum);
  if (ctx->dev_epoch) cudaFree(ctx->dev_epoch);
  if (ctx->flush_buf) cudaFree(ctx->flush_buf);
  for (auto& t : ctx->resize_tables) cudaFree(t.dev);
  if (ctx->deflate_scratch) cudaFree(ctx->deflate_scratch);
  if (ctx->deflate_meta) cudaFree(ctx->deflate_meta);
  if (ctx->side) cudaStreamDestroy(ctx->side);
  for (auto& pair : ctx->step_ev) {
    for (cudaEvent_t e : pair) {
      if (e) cudaEventDestroy(e);
    }
  }
  if (ctx->ev_fork) cudaEventDestroy(ctx->ev_fork);
  if (ctx->ev_join) cudaEventDestroy(ctx->ev_join);
  if (ctx->own_stream && ctx->stream) cudaStreamDestroy(ctx->stream);
  delete ctx;
  return TB200_OK;
}

int tb200_ctx_set_stream(tb200_ctx* ctx, void* cuda_stream) {
  if (ctx == nullptr) return fail(TB200_ERR_INVALID, "ctx is NULL");
  DeviceGuard g(ctx->device);
  cudaStreamSynchronize(ctx->stream);
  if (ctx->own_stream && ctx->stream) cudaStreamDestroy(ctx->stream);
  ctx->stream = static_cast<cudaStream_t>(cuda_stream);
  ctx->cur = ctx->stream;
  ctx->own_stream = false;
  return TB200_OK;
}
void* tb200_ctx_stream(tb200_ctx* ctx) { return ctx ? ctx->stream : nullptr; }
int tb200_ctx_device(tb200_ctx* ctx) { return ctx ? ctx->device : -1; }
int tb200_ctx_sm_count(tb200_ctx* ctx) { return ctx ? ctx->sm_count : 0; }
uint64_t tb200_ctx_launch_count(tb200_ctx* ctx) { return ctx ? ctx->launches : 0; }

int tb200_ctx_sync(tb200_ctx* ctx) {
  if (ctx == nullptr) return fail(TB200_ERR_INVALID, "ctx is NULL");
  DeviceGuard g(ctx->device);
  TB200_CUDA(cudaStreamSynchronize(ctx->stream));
  // after a join the main stream already waited for the side stream
  if (ctx->side != nullptr && ctx->capture == nullptr && ctx->forked) TB200_CUDA(cudaStreamSynchronize(ctx->side));
  ctx->sync_epoch += 1;  // every job-table slot is free again
  return TB200_OK;
}

// fork: later launches go to a side stream that starts after everything issued so far;
// join: the main stream waits for the side stream.  Works eagerly and inside a graph
// capture (it becomes a parallel branch of the graph).
int tb200_ctx_fork(tb200_ctx* ctx) {
  if (ctx == nullptr) return fail(TB200_ERR_INVALID, "ctx is NULL");
  if (ctx->forked) return fail(TB200_ERR_STATE, "already forked");
  DeviceGuard g(ctx->device);
  if (ctx->side == nullptr) {
    TB200_CUDA(cudaStreamCreateWithFlags(&ctx->side, cudaStreamNonBlocking));
    TB200_CUDA(cudaEventCreateWithFlags(&ctx->ev_fork, cudaEventDisableTiming));
    TB200_CUDA(cudaEventCreateWithFlags(&ctx->ev_join, cudaEventDisableTiming));
  }
  TB200_CUDA(cudaEventRecord(ctx->ev_fork, ctx->stream));
  TB200_CUDA(cudaStreamWaitEvent(ctx->side, ctx->ev_fork, 0));
  ctx->forked = true;
  ctx->cur = ctx->side;
  return TB200_OK;
}
int tb200_ctx_select(tb200_ctx* ctx, int side) {
  if (ctx == nullptr) return fail(TB200_ERR_INVALID, "ctx is NULL");
  if (!ctx->forked) return fail(TB200_ERR_STATE, "not forked");
  ctx->cur = side ? ctx->side : ctx->stream;
  return TB200_OK;
}
int tb200_ctx_join(tb200_ctx* ctx) {
  if (ctx == nullptr) return fail(TB200_ERR_INVALID, "ctx is NULL");
  if (!ctx->forked) return fail(TB200_ERR_STATE, "not forked");
  DeviceGuard g(ctx->device);
  TB200_CUDA(cudaEventRecord(ctx->ev_join, ctx->side));
  TB200_CUDA(cudaStreamWaitEvent(ctx->stream, ctx->ev_join, 0));
  ctx->forked = false;
  ctx->cur = ctx->stream;
  return TB200_OK;
}

int tb200_timer_create(tb200_ctx* ctx, tb200_timer** out) {
  if (ctx == nullptr || out == nullptr) return fail(TB200_ERR_INVALID, "NULL argument");
  DeviceGuard g(ctx->device);
  tb200_timer* t = new tb200_timer();
  t->ctx = ctx;
  cudaError_t e = cudaEventCreate(&t->start);
  if (e == cudaSuccess) e = cudaEventCreate(&t->stop);
  if (e != cudaSuccess) {
    delete t;
    return fail(TB200_ERR_CUDA, "cudaEventCreate failed: %s", cudaGetErrorString(e));
  }
  *out = t;
  return TB200_OK;
}
int tb200_timer_start(tb200_timer* t) {
  if (t == nullptr) return fail(TB200_ERR_INVALID, "timer is NULL");
  DeviceGuard g(t->ctx->device);
  TB200_CUDA(cudaEventRecord(t->start, t->ctx->stream));
  return TB200_OK;
}
int tb200_timer_stop(tb200_timer* t) {
  if (t == nullptr) return fail(TB200_ERR_INVALID, "timer is NULL");
  DeviceGuard g(t->ctx->device);
  TB200_CUDA(cudaEventRecord(t->stop, t->ctx->stream));
  return TB200_OK;
}
int tb200_timer_elapsed_ms(tb200_timer* t, float* ms) {
  if (t == nullptr || ms == nullptr) return fail(TB200_ERR_INVALID, "NULL argument");
  DeviceGuard g(t->ctx->device);
  TB200_CUDA(cudaEventSynchronize(t->stop));
  TB200_CUDA(cudaEventElapsedTime(ms, t->start, t->stop));
  return TB200_OK;
}
int tb200_timer_destroy(tb200_timer* t) {
  if (t == nullptr) return TB200_OK;
  DeviceGuard g(t->ctx->device);
  cudaEventDestroy(t->start);
  cudaEventDestroy(t->stop);
  delete t;
  return TB200_OK;
}

// ---------------------------------------------------------------------------
// regions
// ---------------------------------------------------------------------------
int tb200_region_create(const char* name, uint64_t byte_size, int device_id, tb200_region** out) {
  if (out == nullptr) return fail(TB200_ERR_INVALID, "out is NULL");
  *out = nullptr;
  int n = 0;
  TB200_CUDA(cudaGetDeviceCount(&n));
  if (device_id < 0 || device_id >= n) return fail(TB200_ERR_INVALID, "device %d not in [0,%d)", device_id, n);
  DeviceGuard g(device_id);
  TB200_CUDA(g.error());
  tb200_region* r = new tb200_region();
  r->name = name ? name : "";
  r->size = byte_size;
  r->device = device_id;
  // cudaMalloc(0) yields no allocation to export; keep one granule so that an
  // empty region still has a valid handle (the reference would fail here)
  cudaError_t e = cudaMalloc(&r->base, byte_size == 0 ? 256 : byte_size);
  if (e == cudaSuccess) e = cudaIpcGetMemHandle(&r->handle, r->base);
  if (e != cudaSuccess) {
    if (r->base) cudaFree(r->base);
    delete r;
    return fail(TB200_ERR_CUDA, "unable to create cuda shared memory handle: %s", cudaGetErrorString(e));
  }
  *out = r;
  return TB200_OK;
}

int tb200_region_open(const uint8_t ipc_handle[TB200_IPC_HANDLE_BYTES], uint64_t byte_size,
                      int device_id, tb200_region** out) {
  if (out == nullptr || ipc_handle == nullptr) return fail(TB200_ERR_INVALID, "NULL argument");
  *out = nullptr;
  static_assert(sizeof(cudaIpcMemHandle_t) == TB200_IPC_HANDLE_BYTES, "IPC handle size");
  DeviceGuard g(device_id);
  TB200_CUDA(g.error());
  tb200_region* r = new tb200_region();
  r->size = byte_size;
  r->device = device_id;
  r->opened = true;
  memcpy(&r->handle, ipc_handle, TB200_IPC_HANDLE_BYTES);
  cudaError_t e = cudaIpcOpenMemHandle(&r->base, r->handle, cudaIpcMemLazyEnablePeerAccess);
  if (e != cudaSuccess) {
    delete r;
    return fail(TB200_ERR_CUDA, "cudaIpcOpenMemHandle failed: %s", cudaGetErrorString(e));
  }
  *out = r;
  return TB200_OK;
}

int tb200_region_destroy(tb200_region* r) {
  if (r == nullptr) return TB200_OK;
  DeviceGuard g(r->device);
  cudaError_t e = r->opened ? cudaIpcCloseMemHandle(r->base) : cudaFree(r->base);
  delete r;
  if (e != cudaSuccess) return fail(TB200_ERR_CUDA, "region release failed: %s", cudaGetErrorString(e));
  return TB200_OK;
}

int tb200_region_ipc_handle(const tb200_region* r, uint8_t out[TB200_IPC_HANDLE_BYTES]) {
  if (r == nullptr || out == nullptr) return fail(TB200_ERR_INVALID, "NULL argument");
  memcpy(out, &r->handle, TB200_IPC_HANDLE_BYTES);
  return TB200_OK;
}
uint64_t tb200_region_base(const tb200_region* r) { return r ? reinterpret_cast<uint64_t>(r->base) : 0; }
uint64_t tb200_region_size(const tb200_region* r) { return r ? r->size : 0; }
int tb200_region_device(const tb200_region* r) { return r ? r->device : -1; }
const char* tb200_region_name(const tb200_region* r) { return r ? r->name.c_str() : ""; }

int tb200_region_write_host_gather(tb200_ctx* ctx, tb200_region* r, uint64_t offset, int nchunks,
                                   const void* const* srcs, const uint64_t* sizes) {
  if (ctx == nullptr || r == nullptr || nchunks < 0 || (nchunks > 0 && (srcs == nullptr || sizes == nullptr))) {
    return fail(TB200_ERR_INVALID, "bad argument");
  }
  if (ctx->device != r->device) return fail(TB200_ERR_INVALID, "context on device %d, region on %d", ctx->device, r->device);
  uint64_t total = 0;
  for (int i = 0; i < nchunks; ++i) total += sizes[i];
  int rc = check_range(r, offset, total);
  if (rc != TB200_OK) return rc;
  DeviceGuard g(ctx->device);
  char* dst = static_cast<char*>(r->base) + offset;
  for (int i = 0; i < nchunks; ++i) {
    if (sizes[i] == 0) continue;
    if (srcs[i] == nullptr) return fail(TB200_ERR_INVALID, "chunk %d is NULL", i);
    rc = staged_h2d(ctx, dst, static_cast<const char*>(srcs[i]), sizes[i]);
    if (rc != TB200_OK) return rc;
    dst += sizes[i];
  }
  TB200_CUDA(cudaStreamSynchronize(ctx->cur));
  return TB200_OK;
}

int tb200_region_write_host(tb200_ctx* ctx, tb200_region* r, uint64_t offset, const void* src, uint64_t nbytes) {
  const void* srcs[1] = {src};
  const uint64_t sizes[1] = {nbytes};
  return tb200_region_write_host_gather(ctx, r, offset, 1, srcs, sizes);
}

int tb200_region_read_host(tb200_ctx* ctx, const tb200_region* r, uint64_t offset, void* dst, uint64_t nbytes) {
  if (ctx == nullptr || r == nullptr || (dst == nullptr && nbytes != 0)) return fail(TB200_ERR_INVALID, "bad argument");
  if (ctx->device != r->device) return fail(TB200_ERR_INVALID, "context on device %d, region on %d", ctx->device, r->device);
  int rc = check_range(r, offset, nbytes);
  if (rc != TB200_OK) return rc;
  if (nbytes == 0) return TB200_OK;
  DeviceGuard g(ctx->device);
  if (nbytes <= kDirectBytes) {
    TB200_CUDA(cudaMemcpyAsync(dst, static_cast<const char*>(r->base) + offset, nbytes, cudaMemcpyDeviceToHost, ctx->cur));
    TB200_CUDA(cudaStreamSynchronize(ctx->cur));
    return TB200_OK;
  }
  rc = ensure_stage(ctx);
  if (rc != TB200_OK) return rc;
  const char* src = static_cast<const char*>(r->base) + offset;
  char* out = static_cast<char*>(dst);
  // two-deep pipeline: D2H of chunk k+1 overlaps the host memcpy of chunk k
  uint64_t issued = 0, copied = 0;
  int qb[kStageCount];
  size_t qn[kStageCount];
  int qhead = 0, qlen = 0;
  while (copied < nbytes) {
    while (issued < nbytes && qlen < kStageCount) {
      const size_t n = static_cast<size_t>(std::min<uint64_t>(kStageBytes, nbytes - issued));
      const int b = ctx->stage_next;
      ctx->stage_next = (b + 1) % kStageCount;
      TB200_CUDA(cudaEventSynchronize(ctx->stage_ev[b]));
      TB200_CUDA(cudaMemcpyAsync(ctx->stage[b], src + issued, n, cudaMemcpyDeviceToHost, ctx->cur));
      TB200_CUDA(cudaEventRecord(ctx->stage_ev[b], ctx->cur));
      qb[(qhead + qlen) % kStageCount] = b;
      qn[(qhead + qlen) % kStageCount] = n;
      ++qlen;
      issued += n;
    }
    const int b = qb[qhead];
    const size_t n = qn[qhead];
    qhead = (qhead + 1) % kStageCount;
    --qlen;
    TB200_CUDA(cudaEventSynchronize(ctx->stage_ev[b]));
    CopyPool::instance().parallel_memcpy(out + copied, ctx->stage[b], n);
    copied += n;
  }
  return TB200_OK;
}

int tb200_region_write_ptr(tb200_ctx* ctx, tb200_region* r, uint64_t offset, const void* src, uint64_t nbytes) {
  if (ctx == nullptr || r == nullptr || (src == nullptr && nbytes != 0)) return fail(TB200_ERR_INVALID, "bad argument");
  int rc = check_range(r, offset, nbytes);
  if (rc != TB200_OK) return rc;
  if (nbytes == 0) return TB200_OK;
  DeviceGuard g(ctx->device);
  TB200_CUDA(cudaMemcpyAsync(static_cast<char*>(r->base) + offset, src, nbytes, cudaMemcpyDefault, ctx->cur));
  TB200_CUDA(cudaStreamSynchronize(ctx->cur));
  return TB200_OK;
}

int tb200_host_alloc(uint64_t nbytes, void** host_ptr, void** device_ptr) {
  if (host_ptr == nullptr) return fail(TB200_ERR_INVALID, "host_ptr is NULL");
  void* h = nullptr;
  TB200_CUDA(cudaHostAlloc(&h, nbytes == 0 ? 16 : nbytes, cudaHostAllocMapped | cudaHostAllocPortable));
  *host_ptr = h;
  if (device_ptr != nullptr) {
    void* d = nullptr;
    cudaError_t e = cudaHostGetDevicePointer(&d, h, 0);
    if (e != cudaSuccess) {
      cudaFreeHost(h);
      return fail(TB200_ERR_CUDA, "cudaHostGetDevicePointer failed: %s", cudaGetErrorString(e));
    }
    *device_ptr = d;
  }
  return TB200_OK;
}
int tb200_host_free(void* host_ptr) {
  if (host_ptr == nullptr) return TB200_OK;
  TB200_CUDA(cudaFreeHost(host_ptr));
  return TB200_OK;
}
int tb200_device_alloc(int device_id, uint64_t nbytes, void** device_ptr) {
  if (device_ptr == nullptr) return fail(TB200_ERR_INVALID, "device_ptr is NULL");
  DeviceGuard g(device_id);
  TB200_CUDA(g.error());
  TB200_CUDA(cudaMalloc(device_ptr, nbytes == 0 ? 16 : nbytes));
  return TB200_OK;
}
int tb200_device_free(int device_id, void* device_ptr) {
  if (device_ptr == nullptr) return TB200_OK;
  DeviceGuard g(device_id);
  TB200_CUDA(cudaFree(device_ptr));
  return TB200_OK;
}
int tb200_memcpy_h2d_async(tb200_ctx* ctx, void* dst, const void* src, uint64_t nbytes) {
  if (ctx == nullptr) return fail(TB200_ERR_INVALID, "ctx is NULL");
  DeviceGuard g(ctx->device);
  TB200_CUDA(cudaMemcpyAsync(dst, src, nbytes, cudaMemcpyHostToDevice, ctx->cur));
  return TB200_OK;
}
int tb200_memcpy_d2h_async(tb200_ctx* ctx, void* dst, const void* src, uint64_t nbytes) {
  if (ctx == nullptr) return fail(TB200_ERR_INVALID, "ctx is NULL");
  DeviceGuard g(ctx->device);
  TB200_CUDA(cudaMemcpyAsync(dst, src, nbytes, cudaMemcpyDeviceToHost, ctx->cur));
  return TB200_OK;
}

// ---------------------------------------------------------------------------
// fill
// ---------------------------------------------------------------------------
// the byte ranges a launch writes, sorted and merged (the 64 slots of one region set: one span)
static void written_spans(const tb200_fill_job* jobs, int n, std::vector<std::pair<uint64_t, uint64_t>>* out) {
  out->clear();
  out->reserve(static_cast<size_t>(n));
  bool sorted = true;
  for (int i = 0; i < n; ++i) {
    if (jobs[i].nbytes == 0) continue;
    if (!out->empty() && jobs[i].dst < out->back().first) sorted = false;
    out->emplace_back(jobs[i].dst, jobs[i].dst + jobs[i].nbytes);
  }
  if (!sorted) std::sort(out->begin(), out->end());
  size_t w = 0;
  for (size_t i = 0; i < out->size(); ++i) {
    if (w != 0 && (*out)[i].first <= (*out)[w - 1].second) {
      (*out)[w - 1].second = std::max((*out)[w - 1].second, (*out)[i].second);
    } else {
      (*out)[w++] = (*out)[i];
    }
  }
  out->resize(w);
}
static bool spans_overlap(const std::vector<std::pair<uint64_t, uint64_t>>& a, const std::vector<std::pair<uint64_t, uint64_t>>& b) {
  size_t i = 0, j = 0;
  while (i < a.size() && j < b.size()) {
    if (a[i].second <= b[j].first) ++i;
    else if (b[j].second <= a[i].first) ++j;
    else return true;
  }
  return false;
}

static bool g_fill_uniform = true;  // homogeneous launches take fill_uniform_kernel ("fill_uniform" knob)
static bool g_fill_pdl = true;      // ... and overlap with the previous one when they write disjoint memory ("fill_pdl" knob)

static int fill_impl(tb200_ctx* ctx, const tb200_fill_job* jobs, int njobs, uint64_t seed,
                     uint64_t epoch, bool use_dev_epoch, uint64_t bump) {
  if (ctx == nullptr || njobs < 0 || (njobs > 0 && jobs == nullptr)) return fail(TB200_ERR_INVALID, "bad argument");
  if (njobs == 0) return TB200_OK;
  DeviceGuard g(ctx->device);
  const int max_jobs = static_cast<int>(kJobSlotBytes / (sizeof(tb200_fill_job) + sizeof(uint64_t))) - 1;
  RoundKeys rk;
  make_round_keys(seed, &rk);
  for (int base = 0; base < njobs; base += max_jobs) {
    const int n = std::min(max_jobs, njobs - base);
    const bool last = base + n >= njobs;
    std::vector<uint64_t> prefix(n + 1, 0);
    bool uniform = true;
    bool homogeneous = true;
    uint64_t total = 0;
    uint32_t unaligned = 0;
    for (int i = 0; i < n; ++i) {
      const tb200_fill_job& jb = jobs[base + i];
      if ((jb.dst & 15) != 0 && jb.nbytes != 0) ++unaligned;
      const bool strings = jb.dtype == TB200_BYTES;
      const uint32_t es = strings ? 1u : tb200_dtype_size(jb.dtype);
      if (es == 0) return fail(TB200_ERR_INVALID, "job %d: dtype %u cannot be filled", base + i, jb.dtype);
      if (strings && jb.mode == TB200_FILL_RANDOM) {
        // fixed-length strings: irange = string length, nbytes = count * (4 + length)
        if (jb.irange >= (1ull << 31) || jb.nbytes % (jb.irange + 4) != 0) {
          return fail(TB200_ERR_INVALID, "job %d: BYTES fill needs nbytes = count * (4 + string length %llu)", base + i,
                      static_cast<unsigned long long>(jb.irange));
        }
      } else if (strings) {
        return fail(TB200_ERR_INVALID, "job %d: BYTES tensors take TB200_FILL_RANDOM only", base + i);
      }
      if (jb.mode > TB200_FILL_BYTE) return fail(TB200_ERR_INVALID, "job %d: unknown fill mode %u", base + i, jb.mode);
      if (jb.nbytes != 0 && jb.dst == 0) return fail(TB200_ERR_INVALID, "job %d: dst is NULL", base + i);
      if (jb.mode == TB200_FILL_RANDOM) {
        const uint64_t lim = es == 1 ? 256ull : (es == 2 ? 65536ull : (es == 4 ? (1ull << 32) : 0ull));
        const bool is_int = jb.dtype != TB200_FP16 && jb.dtype != TB200_FP32 && jb.dtype != TB200_FP64 &&
                            jb.dtype != TB200_BF16 && jb.dtype != TB200_BOOL && !strings;
        if (is_int && lim != 0 && jb.irange > lim) {
          return fail(TB200_ERR_INVALID, "job %d: irange %llu exceeds the %u-byte element range", base + i,
                      static_cast<unsigned long long>(jb.irange), es);
        }
      }
      const uint64_t groups = (jb.nbytes + 15) / 16;
      const tb200_fill_job& f = jobs[base];
      if (strings || jb.mode != TB200_FILL_RANDOM || jb.dtype != f.dtype || jb.lo != f.lo || jb.span != f.span ||
          jb.ilo != f.ilo || jb.irange != f.irange || (jb.nbytes & 15) != 0 || (jb.dst & 15) != 0) {
        homogeneous = false;
      }
      total += groups;
      if (total > (1ull << 44)) return fail(TB200_ERR_INVALID, "fill launch too large");
      prefix[i + 1] = total;
      if (groups != (jobs[base].nbytes + 15) / 16) uniform = false;
    }
    if (total == 0 && !(last && bump != 0 && use_dev_epoch)) continue;
    // graphs: every captured fill reads the device epoch plus the advance the capture has
    // accumulated so far; the capture's last node applies the sum (tb200_graph_end), so the
    // fills of one graph never wait for each other's epoch update
    uint64_t launch_epoch = epoch, launch_bump = (last && use_dev_epoch) ? bump : 0;
    if (ctx->capture != nullptr && use_dev_epoch) {
      launch_epoch += ctx->capture_epoch;
      if (last) ctx->capture_epoch += bump;
      launch_bump = 0;
    }
    if (g_fill_uniform && homogeneous && uniform && total != 0 && unaligned == 0 && n <= kFillTabLarge && prefix[1] < (1ull << 31)) {
      const tb200_fill_job& f = jobs[base];
      FillUniform U;
      U.rk = rk;
      U.p.lo_f = static_cast<float>(f.lo);
      U.p.span_f = static_cast<float>(f.span);
      U.p.lo_d = f.lo;
      U.p.span_d = f.span;
      U.p.ilo = f.ilo;
      U.p.irange = f.irange;
      U.p.unit = (f.span == 0.0) ? 1u : 0u;
      U.dev_epoch = use_dev_epoch ? ctx->dev_epoch : nullptr;
      U.epoch = launch_epoch;
      U.total_groups = total;
      U.njobs = static_cast<uint32_t>(n);
      U.groups_per_job = static_cast<uint32_t>(prefix[1]);
      plan_fill_uniform(&U, ctx->sm_count);
      tb200_ctx::PdlEntry mine;
      written_spans(jobs + base, n, &mine.spans);
      // overlap with the previous launch only if that was a homogeneous fill on this stream
      // writing other memory (same memory: the later launch must win)
      // Which earlier launches of the chain can still be running when this one starts?  A
      // launch starts only after every CTA of its predecessor started, and no CTA of a launch
      // exits before the launch it overlapped with completed (griddepcontrol.wait at the end of
      // the kernel).  So launch -k is still running only if the grids of launches -1 .. -(k-1)
      // plus one of its own CTAs are resident together: at most 8 CTAs of 256 threads per SM.
      const int si = (ctx->cur == ctx->side && ctx->side != nullptr) ? 1 : 0;
      std::vector<tb200_ctx::PdlEntry>& chain = ctx->pdl_chain[si];
      bool pdl = g_fill_pdl && ctx->pdl_mark[si] == stream_seq(ctx) && !chain.empty();
      if (pdl) {
        const uint64_t capacity = static_cast<uint64_t>(ctx->sm_count) * 8;
        uint64_t newer = 0;
        size_t live = 0;
        for (size_t k = chain.size(); k-- > 0;) {
          if (newer + 1 > capacity) break;  // this one and everything older completed
          ++live;
          if (spans_overlap(mine.spans, chain[k].spans)) pdl = false;  // same memory: the later launch must win
          newer += chain[k].grid;
        }
        if (live == chain.size() && chain.size() >= 16) pdl = false;  // bounded history
        if (pdl && live < chain.size()) chain.erase(chain.begin(), chain.end() - live);
      }
      if (!pdl) chain.clear();  // a plain launch waits for the whole chain
      TB200_CUDA(launch_fill_uniform(U, jobs + base, f.dtype, ctx->cur, pdl));
      count_launch(ctx);
      ctx->pdl_mark[si] = stream_seq(ctx);
      mine.grid = U.grid;
      chain.push_back(std::move(mine));
      if (launch_bump != 0) {  // eager fill_epoch: advance the device epoch behind the fill
        TB200_CUDA(launch_epoch_bump(ctx->dev_epoch, launch_bump, ctx->cur));
        count_launch(ctx);
      }
      continue;
    }
    // one upload: [jobs | prefix]
    const size_t jbytes = sizeof(tb200_fill_job) * n;
    const size_t pbytes = sizeof(uint64_t) * (n + 1);
    std::vector<char> blob(jbytes + pbytes);
    memcpy(blob.data(), jobs + base, jbytes);
    memcpy(blob.data() + jbytes, prefix.data(), pbytes);
    const void* dev = nullptr;
    int rc = upload(ctx, blob.data(), blob.size(), &dev);
    if (rc != TB200_OK) return rc;
    FillLaunch L;
    L.jobs = static_cast<const tb200_fill_job*>(dev);
    L.group_prefix = reinterpret_cast<const uint64_t*>(static_cast<const char*>(dev) + jbytes);
    L.dev_epoch = use_dev_epoch ? ctx->dev_epoch : nullptr;
    L.done_counter = reinterpret_cast<unsigned int*>(ctx->dev_epoch + 1);
    L.seed = seed;
    L.epoch = launch_epoch;
    L.bump = launch_bump;
    L.njobs = static_cast<uint32_t>(n);
    L.total_groups = total;
    L.uniform_groups = (uniform && total != 0) ? prefix[1] : 0;
    L.homogeneous = (homogeneous && L.uniform_groups != 0) ? 1u : 0u;
    L.unaligned_jobs = unaligned;
    L.div_magic = 0;
    L.dtype0 = jobs[base].dtype;
    // exact g / d by multiply-high needs g * d < 2^64
    if (L.homogeneous && (L.uniform_groups < 2 || static_cast<unsigned __int128>(total) * L.uniform_groups >= (static_cast<unsigned __int128>(1) << 63))) {
      L.homogeneous = 0;
    }
    if (L.homogeneous) {
      L.div_magic = static_cast<uint64_t>((static_cast<unsigned __int128>(1) << 64) / L.uniform_groups) + 1;
    }
    L.rk = rk;
    TB200_CUDA(launch_fill(L, ctx->sm_count, ctx->cur));
    count_launch(ctx);
  }
  return TB200_OK;
}

int tb200_fill_async(tb200_ctx* ctx, const tb200_fill_job* jobs, int njobs, uint64_t seed, uint64_t stream_epoch) {
  return fill_impl(ctx, jobs, njobs, seed, stream_epoch, false, 0);
}
int tb200_fill_epoch_async(tb200_ctx* ctx, const tb200_fill_job* jobs, int njobs, uint64_t seed, uint64_t bump) {
  return fill_impl(ctx, jobs, njobs, seed, 0, true, bump);
}

int tb200_ctx_epoch_set(tb200_ctx* ctx, uint64_t value) {
  if (ctx == nullptr) return fail(TB200_ERR_INVALID, "ctx is NULL");
  DeviceGuard g(ctx->device);
  TB200_CUDA(cudaStreamSynchronize(ctx->stream));
  TB200_CUDA(cudaMemcpy(ctx->dev_epoch, &value, sizeof(value), cudaMemcpyHostToDevice));
  return TB200_OK;
}
int tb200_ctx_epoch_bump_async(tb200_ctx* ctx, uint64_t delta) {
  if (ctx == nullptr) return fail(TB200_ERR_INVALID, "ctx is NULL");
  DeviceGuard g(ctx->device);
  TB200_CUDA(launch_epoch_bump(ctx->dev_epoch, delta, ctx->cur));
  count_launch(ctx);
  return TB200_OK;
}

// ---------------------------------------------------------------------------
// pack / cast
// ---------------------------------------------------------------------------
int tb200_pack_image_async(tb200_ctx* ctx, void* dst, uint32_t dst_dtype, uint32_t dst_layout,
                           const void* src_u8_nhwc, int n, int h, int w, int c, uint32_t scaling) {
  if (ctx == nullptr || dst == nullptr || src_u8_nhwc == nullptr) return fail(TB200_ERR_INVALID, "NULL argument");
  if (dst_layout != TB200_NCHW && dst_layout != TB200_NHWC) return fail(TB200_ERR_INVALID, "unknown layout %u", dst_layout);
  DeviceGuard g(ctx->device);
  ImagePack p;
  p.dst = dst;
  p.src = static_cast<const uint8_t*>(src_u8_nhwc);
  p.dst_dtype = dst_dtype;
  p.layout = dst_layout;
  p.scaling = scaling;
  p.n = n; p.h = h; p.w = w; p.c = c;
  int launches = 0;
  cudaError_t e = launch_pack_image(p, ctx->sm_count, ctx->cur, &launches);
  if (e == cudaErrorInvalidValue) {
    return fail(TB200_ERR_INVALID, "pack_image: unsupported combination (dtype %u, n=%d h=%d w=%d c=%d, scaling %u)",
                dst_dtype, n, h, w, c, scaling);
  }
  TB200_CUDA(e);
  count_launch(ctx, launches);
  return TB200_OK;
}

// ---------------------------------------------------------------------------
// resize + pack.  Coefficients as Pillow computes them (libImaging/Resample.c,
// precompute_coeffs + normalize_coeffs_8bpc; third-party to the reference, which calls it
// through Image.resize at src/python/examples/image_client.py:166): for output index xx,
// center = (xx + 0.5) * scale, triangle filter of half-width support = max(scale, 1),
// taps [xmin, xmax) rounded to the nearest source index, weights normalised to sum 1 in
// double precision and quantised to 22-bit fixed point with round-half-up.
// ---------------------------------------------------------------------------

int tb200_resize_pack_image_async(tb200_ctx* ctx, void* dst, uint32_t dst_dtype, uint32_t dst_layout, const void* src_u8_nhwc,
                                  int n, int src_h, int src_w, int c, int dst_h, int dst_w, uint32_t scaling) {
  if (ctx == nullptr || dst == nullptr || src_u8_nhwc == nullptr) return fail(TB200_ERR_INVALID, "NULL argument");
  if (dst_layout != TB200_NCHW && dst_layout != TB200_NHWC) return fail(TB200_ERR_INVALID, "unknown layout %u", dst_layout);
  if (n <= 0 || src_h <= 0 || src_w <= 0 || dst_h <= 0 || dst_w <= 0 || (c != 1 && c != 3) || n > 65535) {
    return fail(TB200_ERR_INVALID, "resize_pack: bad shape (n=%d, %dx%dx%d -> %dx%d)", n, src_h, src_w, c, dst_h, dst_w);
  }
  if (dst_dtype != TB200_FP32 && dst_dtype != TB200_FP16 && dst_dtype != TB200_BF16 && dst_dtype != TB200_UINT8) {
    return fail(TB200_ERR_INVALID, "resize_pack: destination dtype %s is not supported", tb200_dtype_name(dst_dtype));
  }
  if (dst_dtype == TB200_UINT8 && scaling != TB200_SCALE_NONE) return fail(TB200_ERR_INVALID, "resize_pack: UINT8 output takes no scaling");
  if (scaling > TB200_SCALE_VGG) return fail(TB200_ERR_INVALID, "unknown scaling %u", scaling);
  if (static_cast<int64_t>(src_h) > 100ll * src_w) {
    return fail(TB200_ERR_INVALID, "resize_pack: source taller than 100:1 (%dx%d); Pillow resamples those vertically first", src_h, src_w);
  }
  DeviceGuard g(ctx->device);
  tb200_ctx::ResizeTables* tab = nullptr;
  for (auto& t : ctx->resize_tables) {
    if (t.sh == src_h && t.sw == src_w && t.dh == dst_h && t.dw == dst_w) tab = &t;
  }
  if (tab == nullptr) {
    std::vector<tb200::ResampleBound> hb, vb;  // layout-compatible with int2
    std::vector<int32_t> hc, vc;
    tb200_ctx::ResizeTables t{};
    t.sh = src_h; t.sw = src_w; t.dh = dst_h; t.dw = dst_w;
    tb200::resample_coefficients(src_w, dst_w, &hb, &hc, &t.hk);
    tb200::resample_coefficients(src_h, dst_h, &vb, &vc, &t.vk);
    const int tiles[6] = {32, 16, 8, 4, 2, 1};
    for (int i = 0; i < 6; ++i) {
      int mr = 0;
      for (int y0 = 0; y0 < dst_h; y0 += tiles[i]) {
        const int y1 = std::min(y0 + tiles[i], dst_h) - 1;
        mr = std::max(mr, vb[static_cast<size_t>(y1)].first + vb[static_cast<size_t>(y1)].count - vb[static_cast<size_t>(y0)].first);
      }
      t.max_rows[i] = mr;
    }
    static_assert(sizeof(tb200::ResampleBound) == sizeof(int2), "bounds are read as int2 on the device");
    for (int x0 = 0; x0 < dst_w; x0 += 32) {
      const int xe = std::min(x0 + 32, dst_w) - 1;
      t.max_span = std::max(t.max_span, hb[static_cast<size_t>(xe)].first + hb[static_cast<size_t>(xe)].count - hb[static_cast<size_t>(x0)].first);
    }
    t.off_vb = hb.size() * sizeof(int2);
    t.off_hc = t.off_vb + vb.size() * sizeof(int2);
    t.off_vc = t.off_hc + hc.size() * sizeof(int32_t);
    const size_t total = t.off_vc + vc.size() * sizeof(int32_t);
    std::vector<char> host(total);
    memcpy(host.data(), hb.data(), hb.size() * sizeof(int2));
    memcpy(host.data() + t.off_vb, vb.data(), vb.size() * sizeof(int2));
    memcpy(host.data() + t.off_hc, hc.data(), hc.size() * sizeof(int32_t));
    memcpy(host.data() + t.off_vc, vc.data(), vc.size() * sizeof(int32_t));
    TB200_CUDA(cudaMalloc(&t.dev, total));
    // synchronous and outside any capture: the table outlives graphs that use it
    cudaStreamCaptureMode mode = cudaStreamCaptureModeRelaxed;
    cudaThreadExchangeStreamCaptureMode(&mode);
    const cudaError_t e = cudaMemcpy(t.dev, host.data(), total, cudaMemcpyHostToDevice);
    cudaThreadExchangeStreamCaptureMode(&mode);
    if (e != cudaSuccess) {
      cudaFree(t.dev);
      return fail(TB200_ERR_CUDA, "resize table upload failed: %s", cudaGetErrorString(e));
    }
    if (ctx->resize_tables.size() >= 64) {  // bounded cache: drop the oldest
      TB200_CUDA(cudaStreamSynchronize(ctx->cur));
      cudaFree(ctx->resize_tables.front().dev);
      ctx->resize_tables.erase(ctx->resize_tables.begin());
    }
    ctx->resize_tables.push_back(t);
    tab = &ctx->resize_tables.back();
  }
  ResizePack p;
  p.dst = dst;
  p.src = static_cast<const uint8_t*>(src_u8_nhwc);
  const char* base = static_cast<const char*>(tab->dev);
  p.hbounds = reinterpret_cast<const int2*>(base);
  p.vbounds = reinterpret_cast<const int2*>(base + tab->off_vb);
  p.hcoeffs = reinterpret_cast<const int32_t*>(base + tab->off_hc);
  p.vcoeffs = reinterpret_cast<const int32_t*>(base + tab->off_vc);
  p.dst_dtype = dst_dtype; p.layout = dst_layout; p.scaling = scaling;
  p.n = n; p.sh = src_h; p.sw = src_w; p.c = c; p.dh = dst_h; p.dw = dst_w; p.hk = tab->hk; p.vk = tab->vk;
  // the tallest tile whose block fits: taller tiles repeat less of the horizontal pass, but
  // stay within 40 KB while possible so that several CTAs share an SM
  const int tiles[6] = {32, 16, 8, 4, 2, 1};
  p.tile_h = 0;
  p.raw_stride = static_cast<uint32_t>((tab->max_span * c + 15 + 15) & ~15);  // whole 16-byte granules: + the row's offset in its first one
  for (int pass = 0; pass < 2 && p.tile_h == 0; ++pass) {
    const size_t limit = pass == 0 ? 40u * 1024u : 200u * 1024u;
    for (int i = 0; i < 6 && p.tile_h == 0; ++i) {
      // mbarrier | staged rows | 8-bit intermediate (+ vk slack rows: short output rows read zero-weighted taps
      // past their own) | vertical coefficients | per-row shifts -- the layout resize_pack_kernel walks
      const size_t tmp_bytes = (static_cast<size_t>(tab->max_rows[i] + tab->vk) * 32 * c + 15) & ~static_cast<size_t>(15);
      const size_t bytes = 16 + static_cast<size_t>(tab->max_rows[i]) * p.raw_stride + tmp_bytes +
                           static_cast<size_t>(tiles[i]) * tab->vk * sizeof(int32_t) +
                           ((static_cast<size_t>(tab->max_rows[i]) + 15) & ~static_cast<size_t>(15));
      if (bytes <= limit) {
        p.tile_h = tiles[i];
        p.max_rows = tab->max_rows[i];
        p.smem_bytes = static_cast<uint32_t>(bytes);
      }
    }
  }
  if (p.tile_h == 0) return fail(TB200_ERR_INVALID, "resize_pack: down-scale %dx%d -> %dx%d needs a larger source block per tile than shared memory holds", src_h, src_w, dst_h, dst_w);
  TB200_CUDA(launch_resize_pack(p, ctx->cur));
  count_launch(ctx);
  return TB200_OK;
}

int tb200_cast_async(tb200_ctx* ctx, void* dst, uint32_t dst_dtype, const void* src, uint32_t src_dtype, uint64_t nelem) {
  if (ctx == nullptr) return fail(TB200_ERR_INVALID, "ctx is NULL");
  if (nelem == 0) return TB200_OK;
  if (dst == nullptr || src == nullptr) return fail(TB200_ERR_INVALID, "NULL argument");
  if (!cast_supported(src_dtype, dst_dtype)) {
    return fail(TB200_ERR_INVALID, "cast %s -> %s is not supported", tb200_dtype_name(src_dtype), tb200_dtype_name(dst_dtype));
  }
  DeviceGuard g(ctx->device);
  TB200_CUDA(launch_cast(dst, dst_dtype, src, src_dtype, nelem, ctx->sm_count, ctx->cur));
  count_launch(ctx);
  return TB200_OK;
}

int tb200_pack_strided_async(tb200_ctx* ctx, void* dst, const void* src, uint32_t elem_size, int ndim,
                             const int64_t* shape, const int64_t* src_strides) {
  if (ctx == nullptr) return fail(TB200_ERR_INVALID, "ctx is NULL");
  if (ndim < 0 || ndim > TB200_MAX_DIMS) return fail(TB200_ERR_INVALID, "ndim %d not in [0,%d]", ndim, TB200_MAX_DIMS);
  if (elem_size != 1 && elem_size != 2 && elem_size != 4 && elem_size != 8) return fail(TB200_ERR_INVALID, "elem_size %u", elem_size);
  if (ndim > 0 && (shape == nullptr || src_strides == nullptr)) return fail(TB200_ERR_INVALID, "NULL shape/strides");
  StridedPack p;
  memset(&p, 0, sizeof(p));
  p.dst = dst;
  p.src = src;
  p.elem_size = elem_size;
  p.ndim = ndim;
  p.nelem = 1;
  for (int d = 0; d < ndim; ++d) {
    if (shape[d] < 0) return fail(TB200_ERR_INVALID, "negative extent");
    p.shape[d] = shape[d];
    p.strides[d] = src_strides[d];
    p.nelem *= static_cast<uint64_t>(shape[d]);
  }
  if (p.nelem == 0) return TB200_OK;
  if (dst == nullptr || src == nullptr) return fail(TB200_ERR_INVALID, "NULL argument");
  DeviceGuard g(ctx->device);
  TB200_CUDA(launch_pack_strided(p, ctx->sm_count, ctx->cur));
  count_launch(ctx);
  return TB200_OK;
}

int tb200_concat_async(tb200_ctx* ctx, const tb200_copy_job* jobs, int njobs) {
  if (ctx == nullptr || njobs < 0 || (njobs > 0 && jobs == nullptr)) return fail(TB200_ERR_INVALID, "bad argument");
  if (njobs == 0) return TB200_OK;
  DeviceGuard g(ctx->device);
  const int max_jobs = static_cast<int>(kJobSlotBytes / (sizeof(tb200_copy_job) + sizeof(uint32_t))) - 1;
  for (int base = 0; base < njobs; base += max_jobs) {
    const int n = std::min(max_jobs, njobs - base);
    std::vector<uint32_t> prefix(n + 1, 0);
    uint64_t total = 0;
    for (int i = 0; i < n; ++i) {
      const tb200_copy_job& jb = jobs[base + i];
      if (jb.nbytes != 0 && (jb.dst == 0 || jb.src == 0)) return fail(TB200_ERR_INVALID, "job %d: NULL pointer", base + i);
      total += (jb.nbytes + kCopyTileBytes - 1) / kCopyTileBytes;
      if (total > 0xFFFFFFF0ull) return fail(TB200_ERR_INVALID, "concat launch too large");
      prefix[i + 1] = static_cast<uint32_t>(total);
    }
    if (total == 0) continue;
    const size_t jbytes = sizeof(tb200_copy_job) * n;
    const size_t pbytes = sizeof(uint32_t) * (n + 1);
    std::vector<char> blob(jbytes + pbytes);
    memcpy(blob.data(), jobs + base, jbytes);
    memcpy(blob.data() + jbytes, prefix.data(), pbytes);
    const void* dev = nullptr;
    int rc = upload(ctx, blob.data(), blob.size(), &dev);
    if (rc != TB200_OK) return rc;
    CopyLaunch L;
    L.jobs = static_cast<const tb200_copy_job*>(dev);
    L.tile_prefix = reinterpret_cast<const uint32_t*>(static_cast<const char*>(dev) + jbytes);
    L.njobs = static_cast<uint32_t>(n);
    L.total_tiles = static_cast<uint32_t>(total);
    TB200_CUDA(launch_concat(L, ctx->sm_count, ctx->cur));
    count_launch(ctx);
  }
  return TB200_OK;
}

// ---------------------------------------------------------------------------
// check
// ---------------------------------------------------------------------------
int tb200_check_async(tb200_ctx* ctx, const tb200_check_job* jobs, int njobs, tb200_check_result* results) {
  if (ctx == nullptr || njobs < 0 || (njobs > 0 && (jobs == nullptr || results == nullptr))) return fail(TB200_ERR_INVALID, "bad argument");
  if (njobs == 0) return TB200_OK;
  DeviceGuard g(ctx->device);
  const int max_jobs = std::min<int>(static_cast<int>(kJobSlotBytes / sizeof(tb200_check_job)), 65535);
  if (ctx->capture == nullptr && ctx->accum_cap < static_cast<uint32_t>(std::min(njobs, max_jobs))) {
    TB200_CUDA(cudaStreamSynchronize(ctx->cur));
    if (ctx->accum) cudaFree(ctx->accum);
    ctx->accum = nullptr;
    ctx->accum_cap = 0;
    const uint32_t cap = std::max<uint32_t>(1024, static_cast<uint32_t>(std::min(njobs, max_jobs)));
    void* p = nullptr;
    TB200_CUDA(cudaMalloc(&p, sizeof(CheckAccum) * cap));
    TB200_CUDA(cudaMemset(p, 0, sizeof(CheckAccum) * cap));  // kept zero by the kernel itself
    ctx->accum = static_cast<CheckAccum*>(p);
    ctx->accum_cap = cap;
  }
  for (int base = 0; base < njobs; base += max_jobs) {
    const int n = std::min(max_jobs, njobs - base);
    uint64_t max_bytes = 0;
    for (int i = 0; i < n; ++i) {
      const tb200_check_job& jb = jobs[base + i];
      if (jb.kind > TB200_CHECK_TOP1) return fail(TB200_ERR_INVALID, "job %d: unknown check kind %u", base + i, jb.kind);
      if (jb.nbytes != 0 && jb.a == 0) return fail(TB200_ERR_INVALID, "job %d: a is NULL", base + i);
      if ((jb.kind == TB200_CHECK_EQUAL || jb.kind == TB200_CHECK_ADDSUB) && jb.nbytes != 0 && jb.b == 0) return fail(TB200_ERR_INVALID, "job %d: b is NULL", base + i);
      if (jb.kind == TB200_CHECK_ADDSUB && jb.nbytes != 0 && (jb.c == 0 || jb.d == 0)) return fail(TB200_ERR_INVALID, "job %d: c/d is NULL", base + i);
      if ((jb.kind == TB200_CHECK_ADDSUB || jb.kind == TB200_CHECK_TOP1) && (jb.nbytes % 4) != 0) return fail(TB200_ERR_INVALID, "job %d: nbytes must be a multiple of 4", base + i);
      max_bytes = std::max(max_bytes, jb.nbytes);
    }
    const void* dev = nullptr;
    int rc = upload(ctx, jobs + base, sizeof(tb200_check_job) * n, &dev);
    if (rc != TB200_OK) return rc;
    CheckAccum* accum = ctx->accum;
    if (ctx->capture != nullptr) {  // graph-owned scratch
      void* p = nullptr;
      TB200_CUDA(cudaMalloc(&p, sizeof(CheckAccum) * n));
      TB200_CUDA(cudaMemset(p, 0, sizeof(CheckAccum) * n));
      ctx->capture->device_allocs.push_back(p);
      accum = static_cast<CheckAccum*>(p);
    }
    CheckLaunch L;
    L.jobs = static_cast<const tb200_check_job*>(dev);
    L.accum = accum;
    L.results = results + base;
    L.njobs = static_cast<uint32_t>(n);
    L.max_chunks = static_cast<uint32_t>((max_bytes + kCheckChunkBytes - 1) / kCheckChunkBytes);
    if (L.max_chunks > 65535u * 32u) return fail(TB200_ERR_INVALID, "check job too large");
    TB200_CUDA(launch_check(L, ctx->cur));
    count_launch(ctx);
  }
  return TB200_OK;
}

int tb200_topk_async(tb200_ctx* ctx, const tb200_topk_job* jobs, int njobs, int k, tb200_topk_entry* out) {
  if (ctx == nullptr || njobs < 0 || (njobs > 0 && (jobs == nullptr || out == nullptr))) return fail(TB200_ERR_INVALID, "bad argument");
  if (k < 1 || k > 1024) return fail(TB200_ERR_INVALID, "k must be in [1, 1024], got %d", k);
  if (njobs == 0) return TB200_OK;
  DeviceGuard g(ctx->device);
  const int max_jobs = static_cast<int>(kJobSlotBytes / sizeof(tb200_topk_job));
  for (int base = 0; base < njobs; base += max_jobs) {
    const int n = std::min(max_jobs, njobs - base);
    for (int i = 0; i < n; ++i) {
      const tb200_topk_job& jb = jobs[base + i];
      if (jb.dtype != TB200_FP32 && jb.dtype != TB200_FP16 && jb.dtype != TB200_BF16) {
        return fail(TB200_ERR_INVALID, "job %d: top-k takes FP32, FP16 or BF16 vectors", base + i);
      }
      if (jb.count >= 0xFFFFFFFFull) return fail(TB200_ERR_INVALID, "job %d: vector too long", base + i);
      if (jb.count != 0 && jb.src == 0) return fail(TB200_ERR_INVALID, "job %d: src is NULL", base + i);
    }
    const void* dev = nullptr;
    int rc = upload(ctx, jobs + base, sizeof(tb200_topk_job) * n, &dev);
    if (rc != TB200_OK) return rc;
    TB200_CUDA(launch_topk(static_cast<const tb200_topk_job*>(dev), static_cast<uint32_t>(n), static_cast<uint32_t>(k),
                           out + static_cast<size_t>(base) * k, ctx->cur));
    count_launch(ctx);
  }
  return TB200_OK;
}

int tb200_bytes_decode_async(tb200_ctx* ctx, const void* src, uint64_t src_bytes, uint64_t count, uint32_t* offsets, void* packed,
                             uint64_t packed_capacity, uint64_t* status) {
  if (ctx == nullptr || offsets == nullptr || status == nullptr || (src_bytes != 0 && src == nullptr)) return fail(TB200_ERR_INVALID, "bad argument");
  if (count != 0 && packed == nullptr && packed_capacity != 0) return fail(TB200_ERR_INVALID, "packed is NULL");
  if (ctx->capture != nullptr) return fail(TB200_ERR_STATE, "BYTES decode cannot be captured (it sizes its scratch per call)");
  DeviceGuard g(ctx->device);
  if (count > ctx->bytes_src_off_cap) {
    TB200_CUDA(cudaStreamSynchronize(ctx->cur));
    if (ctx->bytes_src_off != nullptr) cudaFree(ctx->bytes_src_off);
    ctx->bytes_src_off = nullptr;
    const uint64_t cap = std::max<uint64_t>(count, 4096);
    TB200_CUDA(cudaMalloc(reinterpret_cast<void**>(&ctx->bytes_src_off), cap * sizeof(uint64_t)));
    ctx->bytes_src_off_cap = cap;
  }
  if (ctx->bytes_src_off == nullptr) {
    TB200_CUDA(cudaMalloc(reinterpret_cast<void**>(&ctx->bytes_src_off), 4096 * sizeof(uint64_t)));
    ctx->bytes_src_off_cap = 4096;
  }
  TB200_CUDA(launch_bytes_decode(static_cast<const uint8_t*>(src), src_bytes, count, ctx->bytes_src_off, offsets, static_cast<uint8_t*>(packed),
                                 packed_capacity, status, ctx->sm_count, ctx->cur));
  count_launch(ctx, count != 0 ? 2 : 1);
  return TB200_OK;
}

// ---------------------------------------------------------------------------
// deflate
// ---------------------------------------------------------------------------
static constexpr uint64_t kDeflateChunkBytes = 8192, kDeflateChunkOutBytes = 8192 + 16;

uint64_t tb200_deflate_bound(uint64_t nbytes) {
  const uint64_t chunks = (nbytes + kDeflateChunkBytes - 1) / kDeflateChunkBytes;
  return 10 + chunks * kDeflateChunkOutBytes + 5 + 8;
}

int tb200_deflate_async(tb200_ctx* ctx, void* dst, uint64_t dst_capacity, const void* src, uint64_t nbytes, uint32_t format,
                        uint64_t* out_size) {
  if (ctx == nullptr || dst == nullptr || out_size == nullptr || (src == nullptr && nbytes != 0)) return fail(TB200_ERR_INVALID, "NULL argument");
  if (format != TB200_DEFLATE_ZLIB && format != TB200_DEFLATE_GZIP) return fail(TB200_ERR_INVALID, "unknown deflate format %u", format);
  if (dst_capacity < tb200_deflate_bound(nbytes)) {
    return fail(TB200_ERR_RANGE, "deflate: dst holds %llu bytes, tb200_deflate_bound(%llu) = %llu", static_cast<unsigned long long>(dst_capacity),
                static_cast<unsigned long long>(nbytes), static_cast<unsigned long long>(tb200_deflate_bound(nbytes)));
  }
  if (ctx->capture != nullptr) return fail(TB200_ERR_STATE, "deflate is not capturable (scratch may be reallocated)");
  const uint64_t chunks = (nbytes + kDeflateChunkBytes - 1) / kDeflateChunkBytes;
  if (chunks >= (1ull << 31)) return fail(TB200_ERR_INVALID, "deflate: input too large");
  DeviceGuard g(ctx->device);
  if (chunks > ctx->deflate_chunks_cap || ctx->deflate_meta == nullptr) {
    TB200_CUDA(cudaStreamSynchronize(ctx->cur));
    if (ctx->deflate_scratch) cudaFree(ctx->deflate_scratch);
    if (ctx->deflate_meta) cudaFree(ctx->deflate_meta);
    ctx->deflate_scratch = ctx->deflate_meta = nullptr;
    ctx->deflate_chunks_cap = 0;
    const uint64_t cap = std::max<uint64_t>(chunks, 64);
    TB200_CUDA(cudaMalloc(&ctx->deflate_scratch, cap * kDeflateChunkOutBytes));
    TB200_CUDA(cudaMalloc(&ctx->deflate_meta, cap * sizeof(DeflateChunkMeta)));
    ctx->deflate_chunks_cap = cap;
  }
  TB200_CUDA(launch_deflate(static_cast<const uint8_t*>(src), nbytes, format, static_cast<uint8_t*>(ctx->deflate_scratch),
                            static_cast<DeflateChunkMeta*>(ctx->deflate_meta), static_cast<uint8_t*>(dst), out_size, ctx->cur));
  count_launch(ctx, chunks > 0 ? 3 : 1);
  return TB200_OK;
}

// ---------------------------------------------------------------------------
// graphs
// ---------------------------------------------------------------------------
int tb200_graph_begin(tb200_ctx* ctx) {
  if (ctx == nullptr) return fail(TB200_ERR_INVALID, "ctx is NULL");
  if (ctx->capture != nullptr) return fail(TB200_ERR_STATE, "capture already in progress");
  if (ctx->forked) return fail(TB200_ERR_STATE, "join the side stream before capturing");
  DeviceGuard g(ctx->device);
  TB200_CUDA(cudaStreamSynchronize(ctx->stream));
  tb200_graph* gr = new tb200_graph();
  gr->device = ctx->device;
  cudaError_t e = cudaStreamBeginCapture(ctx->stream, cudaStreamCaptureModeRelaxed);
  if (e != cudaSuccess) {
    delete gr;
    return fail(TB200_ERR_CUDA, "cudaStreamBeginCapture failed: %s", cudaGetErrorString(e));
  }
  ctx->capture = gr;
  ctx->capture_launches0 = ctx->launches;
  ctx->capture_epoch = 0;
  ctx->pdl_mark[0] = ctx->pdl_mark[1] = ~0ull;
  return TB200_OK;
}

int tb200_graph_end(tb200_ctx* ctx, tb200_graph** out) {
  if (ctx == nullptr || out == nullptr) return fail(TB200_ERR_INVALID, "NULL argument");
  if (ctx->capture == nullptr) return fail(TB200_ERR_STATE, "no capture in progress");
  if (ctx->forked) return fail(TB200_ERR_STATE, "join the side stream before ending the capture");
  DeviceGuard g(ctx->device);
  tb200_graph* gr = ctx->capture;
  if (ctx->capture_epoch != 0) {
    // last node: the device epoch moves on by what the capture's fill_epoch calls asked for.
    // Every fill read the epoch before it released its successor, so all reads of this replay
    // precede this node and all reads of the next replay follow it.
    const cudaError_t eb = launch_epoch_bump(ctx->dev_epoch, ctx->capture_epoch, ctx->stream);
    if (eb != cudaSuccess) return fail(TB200_ERR_CUDA, "epoch node failed: %s", cudaGetErrorString(eb));
    count_launch(ctx);
    ctx->capture_epoch = 0;
  }
  ctx->capture = nullptr;
  ctx->pdl_mark[0] = ctx->pdl_mark[1] = ~0ull;
  gr->kernels_per_launch = ctx->launches - ctx->capture_launches0;
  ctx->launches = ctx->capture_launches0;  // captured kernels did not run yet
  cudaError_t e = cudaStreamEndCapture(ctx->stream, &gr->graph);
  if (e == cudaSuccess) e = cudaGraphInstantiate(&gr->exec, gr->graph, 0);
  if (e != cudaSuccess) {
    tb200_graph_destroy(gr);
    return fail(TB200_ERR_CUDA, "graph capture failed: %s", cudaGetErrorString(e));
  }
  *out = gr;
  return TB200_OK;
}

int tb200_graph_launch(tb200_ctx* ctx, tb200_graph* gr) {
  if (ctx == nullptr || gr == nullptr) return fail(TB200_ERR_INVALID, "NULL argument");
  DeviceGuard g(ctx->device);
  TB200_CUDA(cudaGraphLaunch(gr->exec, ctx->stream));
  count_launch(ctx, gr->kernels_per_launch);
  return TB200_OK;
}

int tb200_graph_destroy(tb200_graph* gr) {
  if (gr == nullptr) return TB200_OK;
  DeviceGuard g(gr->device);
  if (gr->exec) cudaGraphExecDestroy(gr->exec);
  if (gr->graph) cudaGraphDestroy(gr->graph);
  for (void* p : gr->device_allocs) cudaFree(p);
  delete gr;
  return TB200_OK;
}

static uint64_t g_step_parallel_min_bytes = 0;  // measured: the parallel form wins even for the 38.5 MB C2 step

int tb200_step_sync(tb200_ctx* ctx, const tb200_fill_job* fill_jobs, int nfill, uint64_t seed,
                    uint64_t stream_epoch, const tb200_check_job* check_jobs, int ncheck,
                    tb200_check_result* results) {
  if (ctx == nullptr) return fail(TB200_ERR_INVALID, "ctx is NULL");
  if (ctx->forked || ctx->capture != nullptr) return fail(TB200_ERR_STATE, "step inside a fork / capture");
  int rc = TB200_OK;
  // Validation of the previous responses runs beside the generation of the next inputs
  // (2.19 M vs 1.59 M infer/s for the C2 step when both go down one stream); the
  // "step_parallel_min_mb" knob keeps the one-stream form for experiments.
  uint64_t fill_bytes = 0;
  for (int i = 0; i < nfill; ++i) fill_bytes += fill_jobs[i].nbytes;
  if (ncheck > 0 && fill_bytes < g_step_parallel_min_bytes) {
    rc = tb200_check_async(ctx, check_jobs, ncheck, results);
    if (rc == TB200_OK) rc = tb200_fill_async(ctx, fill_jobs, nfill, seed, stream_epoch);
    if (rc != TB200_OK) return rc;
    return tb200_ctx_sync(ctx);
  }
  if (ncheck == 0) {
    rc = tb200_fill_async(ctx, fill_jobs, nfill, seed, stream_epoch);
    return rc != TB200_OK ? rc : tb200_ctx_sync(ctx);
  }
  // Neither launch depends on anything issued before (the server wrote the outputs, the
  // inputs are write-only), so the side stream needs no fork event: the fill -- the long
  // pole -- goes out first on the main stream, the check on the side stream, and the call
  // returns when both streams are idle.
  DeviceGuard g(ctx->device);
  if (ctx->side == nullptr) {
    TB200_CUDA(cudaStreamCreateWithFlags(&ctx->side, cudaStreamNonBlocking));
    TB200_CUDA(cudaEventCreateWithFlags(&ctx->ev_fork, cudaEventDisableTiming));
    TB200_CUDA(cudaEventCreateWithFlags(&ctx->ev_join, cudaEventDisableTiming));
  }
  rc = tb200_fill_async(ctx, fill_jobs, nfill, seed, stream_epoch);
  if (rc != TB200_OK) return rc;
  ctx->forked = true;  // uploads and launches below go to the side stream
  ctx->cur = ctx->side;
  rc = tb200_check_async(ctx, check_jobs, ncheck, results);
  ctx->cur = ctx->stream;
  const cudaError_t e_side = cudaStreamSynchronize(ctx->side);
  ctx->forked = false;
  if (rc != TB200_OK) return rc;
  if (e_side != cudaSuccess) return fail(TB200_ERR_CUDA, "cudaStreamSynchronize(side) failed: %s", cudaGetErrorString(e_side));
  return tb200_ctx_sync(ctx);
}

int tb200_step_wait(tb200_ctx* ctx, uint64_t ticket) {
  if (ctx == nullptr) return fail(TB200_ERR_INVALID, "ctx is NULL");
  if (ticket == 0 || ticket >= ctx->step_next) return fail(TB200_ERR_INVALID, "unknown step ticket");
  const int k = static_cast<int>(ticket % TB200_STEP_DEPTH);
  if (ctx->step_ticket[k] != ticket) return TB200_OK;  // already waited for (or displaced, which waited)
  DeviceGuard g(ctx->device);
  TB200_CUDA(cudaEventSynchronize(ctx->step_ev[k][0]));
  if (ctx->step_has_side[k]) TB200_CUDA(cudaEventSynchronize(ctx->step_ev[k][1]));
  ctx->step_ticket[k] = 0;
  // both streams are past this step's events: every job table uploaded up to its submit is consumed
  if (ctx->step_upload_mark[k] > ctx->uploads_done) ctx->uploads_done = ctx->step_upload_mark[k];
  return TB200_OK;
}

// One pipelined step: `write_inputs` issues the input side (a fill, or the copies of replayed
// entries) on the main stream, the checks go to the side stream, and the ring entry's events
// follow both.
extern "C++" {
namespace {
template <typename WriteInputs>
int step_submit_with(tb200_ctx* ctx, WriteInputs&& write_inputs, const tb200_check_job* check_jobs, int ncheck,
                     tb200_check_result* results, uint64_t* ticket) {
  if (ctx == nullptr || ticket == nullptr) return fail(TB200_ERR_INVALID, "ctx / ticket is NULL");
  if (ctx->forked || ctx->capture != nullptr) return fail(TB200_ERR_STATE, "step inside a fork / capture");
  DeviceGuard g(ctx->device);
  const uint64_t t = ctx->step_next;
  const int k = static_cast<int>(t % TB200_STEP_DEPTH);
  if (ctx->step_ticket[k] != 0) {
    const int rc = tb200_step_wait(ctx, ctx->step_ticket[k]);
    if (rc != TB200_OK) return rc;
  }
  if (ctx->step_ev[k][0] == nullptr) {
    TB200_CUDA(cudaEventCreateWithFlags(&ctx->step_ev[k][0], cudaEventDisableTiming));
    TB200_CUDA(cudaEventCreateWithFlags(&ctx->step_ev[k][1], cudaEventDisableTiming));
  }
  if (ctx->side == nullptr) {
    TB200_CUDA(cudaStreamCreateWithFlags(&ctx->side, cudaStreamNonBlocking));
    TB200_CUDA(cudaEventCreateWithFlags(&ctx->ev_fork, cudaEventDisableTiming));
    TB200_CUDA(cudaEventCreateWithFlags(&ctx->ev_join, cudaEventDisableTiming));
  }
  int rc = write_inputs();
  if (rc != TB200_OK) return rc;
  TB200_CUDA(cudaEventRecord(ctx->step_ev[k][0], ctx->stream));
  ctx->step_has_side[k] = ncheck > 0;
  if (ncheck > 0) {
    ctx->forked = true;  // uploads and launches below go to the side stream
    ctx->cur = ctx->side;
    rc = tb200_check_async(ctx, check_jobs, ncheck, results);
    cudaError_t e = cudaSuccess;
    if (rc == TB200_OK) e = cudaEventRecord(ctx->step_ev[k][1], ctx->side);
    ctx->cur = ctx->stream;
    ctx->forked = false;
    if (rc != TB200_OK) return rc;
    if (e != cudaSuccess) return fail(TB200_ERR_CUDA, "cudaEventRecord failed: %s", cudaGetErrorString(e));
  }
  ctx->step_ticket[k] = t;
  ctx->step_upload_mark[k] = ctx->upload_seq;
  ctx->step_next = t + 1;
  *ticket = t;
  return TB200_OK;
}
}  // namespace
}  // extern "C++"

int tb200_step_submit(tb200_ctx* ctx, const tb200_fill_job* fill_jobs, int nfill, uint64_t seed,
                      uint64_t stream_epoch, const tb200_check_job* check_jobs, int ncheck,
                      tb200_check_result* results, uint64_t* ticket) {
  return step_submit_with(
      ctx, [&] { return tb200_fill_async(ctx, fill_jobs, nfill, seed, stream_epoch); }, check_jobs, ncheck, results, ticket);
}

int tb200_step_submit_copy(tb200_ctx* ctx, const tb200_copy_job* copies, int ncopy, const tb200_check_job* check_jobs,
                           int ncheck, tb200_check_result* results, uint64_t* ticket) {
  return step_submit_with(ctx, [&] { return tb200_concat_async(ctx, copies, ncopy); }, check_jobs, ncheck, results, ticket);
}

int tb200_tune(const char* key, int value) {
  if (key != nullptr && strcmp(key, "fill_variant") == 0) {
    set_fill_variant(value);
    g_fill_uniform = value == 0;  // the experiment matrix addresses the general kernels
    return TB200_OK;
  }
  if (key != nullptr && strcmp(key, "h2d_direct_kb") == 0) {
    kDirectBytes = static_cast<size_t>(value) << 10;
    return TB200_OK;
  }
  if (key != nullptr && strcmp(key, "fill_uniform") == 0) {
    g_fill_uniform = value != 0;
    return TB200_OK;
  }
  if (key != nullptr && strcmp(key, "fill_pdl") == 0) {
    g_fill_pdl = value != 0;
    return TB200_OK;
  }
  if (key != nullptr && strcmp(key, "step_parallel_min_mb") == 0) {
    g_step_parallel_min_bytes = static_cast<uint64_t>(value) << 20;
    return TB200_OK;
  }
  return fail(TB200_ERR_INVALID, "unknown tuning key");
}

int tb200_l2_flush_async(tb200_ctx* ctx) {
  if (ctx == nullptr) return fail(TB200_ERR_INVALID, "ctx is NULL");
  DeviceGuard g(ctx->device);
  if (ctx->flush_buf == nullptr) TB200_CUDA(cudaMalloc(&ctx->flush_buf, kFlushBytes));
  TB200_CUDA(cudaMemsetAsync(ctx->flush_buf, 0, kFlushBytes, ctx->cur));
  return TB200_OK;
}

}  // extern "C"
