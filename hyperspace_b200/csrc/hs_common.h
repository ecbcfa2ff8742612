// hs_common.h -- context, error plumbing, pooled device/pinned buffers shared by every translation unit.
#pragma once
#include <cuda_runtime.h>

#include <cstdarg>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <map>
#include <memory>
#include <set>
#include <mutex>
#include <stdexcept>
#include <string>
#include <vector>

#include "../../include/hs_gpu.h"

namespace hs {

// Exception carrying an HS_E* code; converted to a return code + message at the C-ABI boundary.
struct Error : std::runtime_error {
  int code;
  Error(int c, const std::string& m) : std::runtime_error(m), code(c) {}
};

[[noreturn]] inline void fail(int code, const char* fmt, ...) {
  char buf[1024];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof buf, fmt, ap);
  va_end(ap);
  throw Error(code, buf);
}

#define HS_CUDA(expr)                                                                              \
  do {                                                                                             \
    cudaError_t _e = (expr);                                                                       \
    if (_e != cudaSuccess)                                                                         \
      ::hs::fail(HS_ECUDA, "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__); \
  } while (0)

inline size_t round_up(size_t v, size_t a) { return (v + a - 1) / a * a; }
inline int64_t ceil_div(int64_t a, int64_t b) { return (a + b - 1) / b; }

// Size-keyed cache of device and pinned-host allocations: a build allocates tens of GB per call and
// cudaMalloc/cudaHostAlloc of that size costs far more than the kernels, so buffers are recycled across calls.
class BufferPool {
 public:
  void* get(size_t bytes, bool pinned) {
    bytes = round_up(bytes ? bytes : 1, 1 << 16);
    auto& free_map = pinned ? free_pinned_ : free_dev_;
    auto it = free_map.lower_bound(bytes);
    // accept a cached block up to 25% larger than asked
    if (it != free_map.end() && it->first <= bytes + bytes / 4) {
      void* p = it->second;
      size_t sz = it->first;
      free_map.erase(it);
      live_[p] = {sz, pinned};
      return p;
    }
    void* p = nullptr;
    cudaError_t e = pinned ? cudaHostAlloc(&p, bytes, cudaHostAllocDefault) : cudaMalloc(&p, bytes);
    if (e != cudaSuccess) {
      cudaGetLastError();
      trim();  // give cached blocks back and retry once
      e = pinned ? cudaHostAlloc(&p, bytes, cudaHostAllocDefault) : cudaMalloc(&p, bytes);
      if (e != cudaSuccess) {
        cudaGetLastError();
        fail(HS_ENOMEM, "%s of %zu bytes failed: %s", pinned ? "cudaHostAlloc" : "cudaMalloc", bytes,
             cudaGetErrorString(e));
      }
    }
    live_[p] = {bytes, pinned};
    return p;
  }
  void put(void* p) {
    if (!p) return;
    auto it = live_.find(p);
    if (it == live_.end()) return;
    (it->second.pinned ? free_pinned_ : free_dev_).emplace(it->second.bytes, p);
    live_.erase(it);
  }
  // Buffers whose IPC handle was given to a peer process stay allocated until the pool dies (a peer may hold a mapping).
  void mark_exported(void* p) { exported_.insert(p); }
  void trim() {
    for (auto it = free_dev_.begin(); it != free_dev_.end();) {
      if (exported_.count(it->second)) {
        ++it;
        continue;
      }
      cudaFree(it->second);
      it = free_dev_.erase(it);
    }
    for (auto& kv : free_pinned_) cudaFreeHost(kv.second);
    free_pinned_.clear();
  }
  ~BufferPool() {
    exported_.clear();
    trim();
    for (auto& kv : live_) kv.second.pinned ? cudaFreeHost(kv.first) : cudaFree(kv.first);
  }

 private:
  struct Live {
    size_t bytes;
    bool pinned;
  };
  std::multimap<size_t, void*> free_dev_, free_pinned_;
  std::map<void*, Live> live_;
  std::set<void*> exported_;
};

}  // namespace hs

struct hs_comm_state;  // exchange.cu
namespace hs {
namespace pq {
struct FileMeta;  // parquet_meta.h
}
}  // namespace hs

struct hs_ctx {
  int device = 0;
  cudaStream_t stream = nullptr;
  bool own_stream = false;
  // Copy engines of their own, so that the host->device staging of the NEXT call's source files and the device->host
  // drain of the PREVIOUS call's index files overlap this call's kernels and each other (PCIe is full duplex).
  cudaStream_t h2d_stream = nullptr;   // hs_stage_sources
  cudaStream_t d2h_stream = nullptr;   // hs_create_index_async -> hs_pending_wait
  // device images staged by hs_stage_sources, by address: the footer parsed from host memory on the way, and the event
  // behind the copy (a call that reads the image makes its stream wait for exactly that event -- not for the copies of
  // images staged for LATER calls, which are already in flight at that point)
  struct StagedImage {
    std::shared_ptr<hs::pq::FileMeta> meta;
    cudaEvent_t ready;
  };
  std::map<const void*, StagedImage> staged;
  int sm_count = 132;  // H100 SXM; hs_init reads the device's own count
  hs::BufferPool pool;
  int launches = 0;  // kernels launched by the current call (hs_stats.gpu_launches)
  // per-kernel CUDA-event timing (hs_profile_enable): one (start, stop) event pair per profiled launch
  bool profile = false;
  struct KEvent {
    const char* name;
    cudaEvent_t a, b;
    int64_t items;  // work items of the launch, for kernels that report them (0: none)
  };
  std::vector<KEvent> kevents;
  std::vector<cudaEvent_t> event_pool;
  hs_comm_state* comm = nullptr;
  int rank = 0, world = 1;
  // small host <-> device transfers that bypass the copy engines (xfer.cu)
  struct PendingD2H {
    void* dst;
    const uint8_t* slot;
    size_t bytes;
  };
  uint8_t* xfer_ring = nullptr;       // pinned, device-accessible
  size_t xfer_cap = 0, xfer_head = 0;
  std::vector<uint8_t*> xfer_retired; // outgrown rings, recycled at the next synchronisation
  std::vector<PendingD2H> xfer_pending;
  uint64_t sync_count = 0;            // sync_stream calls so far: a copy_d2h queued at count c has been delivered once sync_count > c
  // what the ranks agreed on when the same dictionaries were last seen (engine.cu: DecodeCache); freed by hs_shutdown
  void* decode_cache = nullptr;
  void (*decode_cache_free)(void*) = nullptr;
};

namespace hs {

// Small transfers on the ctx stream without the copy engines (xfer.cu).  copy_h2d snapshots the host bytes at once; the
// result of copy_d2h is in place after the next sync_stream(ctx).  Every synchronisation of ctx->stream inside a call goes
// through sync_stream; error paths use xfer_abort (synchronises, drops undelivered results).
void copy_h2d(hs_ctx* ctx, void* dst_dev, const void* src_host, size_t bytes);
void copy_d2h(hs_ctx* ctx, void* dst_host, const void* src_dev, size_t bytes);
// Always on the copy engine, whatever the size: for results copied into pinned memory the caller owns (copy_d2h sends
// copies up to 16 MB through the small-transfer ring: a copy kernel writing over PCIe, then a host memcpy at sync_stream).
void copy_d2h_engine(hs_ctx* ctx, void* dst_host, const void* src_dev, size_t bytes);
void fill_bytes(hs_ctx* ctx, void* dst, int value, size_t bytes);  // cudaMemsetAsync without a copy engine
void sync_stream(hs_ctx* ctx);
void xfer_abort(hs_ctx* ctx);
void xfer_release(hs_ctx* ctx);

// RAII handle on a pooled buffer.
template <typename T>
class Buf {
 public:
  Buf() = default;
  Buf(hs_ctx* ctx, size_t n, bool pinned = false) { alloc(ctx, n, pinned); }
  Buf(const Buf&) = delete;
  Buf& operator=(const Buf&) = delete;
  Buf(Buf&& o) noexcept { *this = std::move(o); }
  Buf& operator=(Buf&& o) noexcept {
    if (this != &o) {
      release();
      ctx_ = o.ctx_;
      p_ = o.p_;
      n_ = o.n_;
      o.p_ = nullptr;
      o.n_ = 0;
    }
    return *this;
  }
  ~Buf() { release(); }
  void alloc(hs_ctx* ctx, size_t n, bool pinned = false) {
    release();
    ctx_ = ctx;
    n_ = n;
    p_ = static_cast<T*>(ctx->pool.get(n * sizeof(T), pinned));
  }
  void release() {
    if (p_ && ctx_) ctx_->pool.put(p_);
    p_ = nullptr;
    n_ = 0;
  }
  T* get() const { return p_; }
  T* detach() {
    T* p = p_;
    p_ = nullptr;
    return p;
  }
  size_t size() const { return n_; }
  T& operator[](size_t i) const { return p_[i]; }
  explicit operator bool() const { return p_ != nullptr; }

 private:
  hs_ctx* ctx_ = nullptr;
  T* p_ = nullptr;
  size_t n_ = 0;
};

// CUDA-event stage timer on the ctx stream.
struct StageTimer {
  hs_ctx* ctx;
  cudaEvent_t a = nullptr, b = nullptr;
  explicit StageTimer(hs_ctx* c) : ctx(c) {
    cudaEventCreate(&a);
    cudaEventCreate(&b);
  }
  ~StageTimer() {
    cudaEventDestroy(a);
    cudaEventDestroy(b);
  }
  void start() { cudaEventRecord(a, ctx->stream); }
  // records the end; the elapsed time is read later with ms() after a sync
  void stop() { cudaEventRecord(b, ctx->stream); }
  float ms() {
    float t = 0;
    cudaEventSynchronize(b);
    cudaEventElapsedTime(&t, a, b);
    return t;
  }
};

// RAII: brackets the kernel launches issued in its scope with CUDA events on the ctx stream when profiling is on.
// Per-device "done once" flag for settings that live in a device's context (cudaFuncSetAttribute): one process may hold
// contexts on several GPUs (one hs_ctx per host thread), and an attribute set for device 0 says nothing about device 1.
struct DeviceOnce {
  bool done[64] = {};
  bool& operator()(int device) { return done[device & 63]; }
};

struct KernelScope {
  hs_ctx* ctx;
  size_t idx = (size_t)-1;
  // items: the launch's work items, reported by hs_profile_report when nonzero
  KernelScope(hs_ctx* c, const char* name, int64_t items = 0) : ctx(c) {
    if (!c->profile) return;
    auto take = [&]() {
      cudaEvent_t e;
      if (!c->event_pool.empty()) {
        e = c->event_pool.back();
        c->event_pool.pop_back();
      } else {
        cudaEventCreate(&e);
      }
      return e;
    };
    hs_ctx::KEvent ke{name, take(), take(), items};
    cudaEventRecord(ke.a, c->stream);
    idx = c->kevents.size();
    c->kevents.push_back(ke);
  }
  ~KernelScope() {
    if (idx != (size_t)-1) cudaEventRecord(ctx->kevents[idx].b, ctx->stream);
  }
};

#define HS_LAUNCH_CHECK(ctx)                \
  do {                                      \
    (ctx)->launches++;                      \
    HS_CUDA(cudaGetLastError());            \
  } while (0)

}  // namespace hs
