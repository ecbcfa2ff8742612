// xfer.cu -- small host <-> device transfers of the build path, kept OFF the copy engines.
//
// A createIndex issues dozens of small copies (chunk descriptors, page plans, counters, flags).  cudaMemcpyAsync puts them
// on the GPU's copy engines, which serve their queue in order ACROSS streams: with the staged source images of the next call
// (hs_stage_sources, gigabytes) already queued on the H2D engine, each 100-byte descriptor copy of the running build waited for
// all of them, and the build finished only when the next call's copy had -- the software pipeline degenerated into
// lockstep.  Here small transfers go through a pinned ring buffer that kernels read and
// write directly over PCIe (unified addressing makes pinned host memory device-accessible): host data is snapshot into the
// ring at once (the caller's buffer may die immediately -- no "keep the vector alive" synchronisation), a copy kernel on the
// ctx stream moves it; device -> host results land in the ring and are handed to their destination by sync_stream().
// Large transfers (file images) and query results (copy_d2h_engine, any size) use the copy engines, which is what they are for.
#include "hs_common.h"

namespace hs {

namespace {

constexpr size_t kSmallCopy = 16 << 20;  // up to here a copy kernel moves the bytes (page plans of a 1 B-row build: ~2 MB)
constexpr size_t kFirstRing = 8 << 20;

__global__ void k_xfer(uint8_t* __restrict__ dst, const uint8_t* __restrict__ src, size_t n) {
  const size_t tid = (size_t)blockIdx.x * blockDim.x + threadIdx.x, stride = (size_t)gridDim.x * blockDim.x;
  if ((((uintptr_t)dst | (uintptr_t)src) & 15) == 0) {
    const size_t nv = n / 16;
    for (size_t i = tid; i < nv; i += stride) ((uint4*)dst)[i] = ((const uint4*)src)[i];
    for (size_t i = nv * 16 + tid; i < n; i += stride) dst[i] = src[i];
  } else {
    for (size_t i = tid; i < n; i += stride) dst[i] = src[i];
  }
}

__global__ void k_fill(uint8_t* __restrict__ dst, uint8_t value, size_t n) {
  const size_t tid = (size_t)blockIdx.x * blockDim.x + threadIdx.x, stride = (size_t)gridDim.x * blockDim.x;
  const uint32_t w = 0x01010101u * value;
  size_t head = (16 - ((uintptr_t)dst & 15)) & 15;
  if (head > n) head = n;
  for (size_t i = tid; i < head; i += stride) dst[i] = value;
  uint4* v = (uint4*)(dst + head);
  const size_t nv = (n - head) / 16;
  for (size_t i = tid; i < nv; i += stride) v[i] = make_uint4(w, w, w, w);
  for (size_t i = head + nv * 16 + tid; i < n; i += stride) dst[i] = value;
}

uint8_t* ring_slot(hs_ctx* ctx, size_t bytes) {
  bytes = round_up(std::max<size_t>(bytes, 1), 16);
  if (!ctx->xfer_ring || ctx->xfer_head + bytes > ctx->xfer_cap) {
    // a bigger ring; the old one stays alive until the kernels that read it have run (next sync_stream)
    size_t cap = std::max(kFirstRing, ctx->xfer_cap * 2);
    while (cap < bytes) cap *= 2;
    if (ctx->xfer_ring) ctx->xfer_retired.push_back(ctx->xfer_ring);
    ctx->xfer_ring = (uint8_t*)ctx->pool.get(cap, /*pinned=*/true);
    ctx->xfer_cap = cap;
    ctx->xfer_head = 0;
  }
  uint8_t* p = ctx->xfer_ring + ctx->xfer_head;
  ctx->xfer_head += bytes;
  return p;
}

void launch_xfer(hs_ctx* ctx, void* dst, const void* src, size_t bytes) {
  const int grid = (int)std::min<size_t>(128, std::max<size_t>(1, bytes / 4096));
  k_xfer<<<grid, 256, 0, ctx->stream>>>((uint8_t*)dst, (const uint8_t*)src, bytes);
  HS_CUDA(cudaGetLastError());
}

}  // namespace

void copy_h2d(hs_ctx* ctx, void* dst_dev, const void* src_host, size_t bytes) {
  if (bytes == 0) return;
  if (bytes > kSmallCopy) {  // the caller keeps src alive until the stream has been synchronised, as with any async copy
    HS_CUDA(cudaMemcpyAsync(dst_dev, src_host, bytes, cudaMemcpyHostToDevice, ctx->stream));
    return;
  }
  uint8_t* slot = ring_slot(ctx, bytes);
  memcpy(slot, src_host, bytes);
  launch_xfer(ctx, dst_dev, slot, bytes);
}

void copy_d2h(hs_ctx* ctx, void* dst_host, const void* src_dev, size_t bytes) {
  if (bytes == 0) return;
  if (bytes > kSmallCopy) {
    HS_CUDA(cudaMemcpyAsync(dst_host, src_dev, bytes, cudaMemcpyDeviceToHost, ctx->stream));
    return;
  }
  uint8_t* slot = ring_slot(ctx, bytes);
  launch_xfer(ctx, slot, src_dev, bytes);
  ctx->xfer_pending.push_back(hs_ctx::PendingD2H{dst_host, slot, bytes});
}

void copy_d2h_engine(hs_ctx* ctx, void* dst_host, const void* src_dev, size_t bytes) {
  if (bytes == 0) return;
  HS_CUDA(cudaMemcpyAsync(dst_host, src_dev, bytes, cudaMemcpyDeviceToHost, ctx->stream));
}

// cudaMemsetAsync may be served by a copy engine too: the build path fills with a kernel
void fill_bytes(hs_ctx* ctx, void* dst, int value, size_t bytes) {
  if (bytes == 0) return;
  const int grid = (int)std::min<size_t>((size_t)ctx->sm_count * 8, std::max<size_t>(1, bytes / 8192));
  k_fill<<<grid, 256, 0, ctx->stream>>>((uint8_t*)dst, (uint8_t)value, bytes);
  HS_CUDA(cudaGetLastError());
}

static void recycle(hs_ctx* ctx) {
  for (uint8_t* r : ctx->xfer_retired) ctx->pool.put(r);
  ctx->xfer_retired.clear();
  ctx->xfer_head = 0;
}

void sync_stream(hs_ctx* ctx) {
  HS_CUDA(cudaStreamSynchronize(ctx->stream));
  for (const hs_ctx::PendingD2H& p : ctx->xfer_pending) memcpy(p.dst, p.slot, p.bytes);
  ctx->xfer_pending.clear();
  ctx->sync_count++;
  recycle(ctx);
}

void xfer_abort(hs_ctx* ctx) {
  cudaStreamSynchronize(ctx->stream);
  ctx->xfer_pending.clear();  // their destinations may be gone (exception unwinding)
  recycle(ctx);
}

void xfer_release(hs_ctx* ctx) {
  xfer_abort(ctx);
  if (ctx->xfer_ring) ctx->pool.put(ctx->xfer_ring);
  ctx->xfer_ring = nullptr;
  ctx->xfer_cap = 0;
}

}  // namespace hs
