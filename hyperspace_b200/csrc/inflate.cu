// inflate.cu -- GZIP page decompression on the GPU.
//
// Spark before 2.0, `spark.sql.parquet.compression.codec=gzip`, Hive and older parquet-mr jobs write GZIP column chunks:
// every page body (dictionary pages included) is one or more gzip members.  DEFLATE blocks depend on each other (a 32 KB
// window, bit-aligned block boundaries known only by decoding), so the unit of parallelism is the page: one warp per page,
// four warps per CTA, each warp's Huffman tables in shared memory (gz::InflateTables, 3.5 KB).
//
//  * Lane 0 decodes the members (inflate.h: bit reader, header, table construction, symbol decoding, match copies): a
//    page of pyarrow or Spark is ~1 MB, so a table holds thousands of independent streams and the GPU runs one per warp.
//    Symbols are decoded serially -- each depends on the bits the previous one consumed -- so the kernel is bound by the
//    latency of lane 0's dependent loads and stores, not by bandwidth.
//  * The whole warp checks each member's CRC-32 in a pass of its own, once lane 0 has written the member: lane i takes the
//    i-th 32nd of the output, CRCs it with a table in shared memory, and the pieces are combined with the CRC's linearity
//    (gz::crc32_piece / crc32_finish).  It reads the member's output once more, from L1 / L2, in parallel.
//  * The warp also copies what is stored verbatim: the level bytes in front of a v2 page's values, and v2 pages stored
//    uncompressed inside a GZIP chunk.
//
// The decoder never reads past a page's compressed bytes (the bit reader shifts in zeros there and reports truncation).
#include "device_utils.cuh"
#include "inflate.h"
#include "page_codec_kernels.h"

namespace hs {

namespace {

constexpr int kWarpsPerCta = 4;

__global__ void __launch_bounds__(kWarpsPerCta * 32) k_inflate(const PageBlob* __restrict__ blobs, int64_t n,
                                                                uint8_t* __restrict__ scratch, uint32_t* __restrict__ d_error) {
  __shared__ gz::InflateTables s_tables[kWarpsPerCta];
  __shared__ uint32_t s_crc[256];
  for (uint32_t i = threadIdx.x; i < 256; i += blockDim.x) s_crc[i] = gz::crc32_table_entry(i);
  __syncthreads();
  const unsigned lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
  const int64_t w = (int64_t)blockIdx.x * kWarpsPerCta + wib;
  if (w >= n) return;
  const PageBlob b = blobs[w];
  uint8_t* dst = scratch + b.dst_off;
  const uint32_t verbatim = b.compressed ? b.prefix : min(b.src_len, b.dst_len);
  for (uint32_t j = lane; j < verbatim; j += 32) dst[j] = b.src[j];
  if (!b.compressed) return;
  const uint8_t* src = b.src + b.prefix;
  const uint32_t n_src = b.src_len - b.prefix, len = b.dst_len - b.prefix;
  uint8_t* body = dst + b.prefix;
  uint32_t p = 0, out = 0, err = 0;
  for (bool first = true;; first = false) {
    gz::Member m{0, 0, 0, 0};
    if (lane == 0) err = gz::inflate_member(src, n_src, p, first, body, len, out, s_tables[wib], m);
    err = __shfl_sync(0xffffffffu, err, 0);
    if (err) break;
    p = __shfl_sync(0xffffffffu, p, 0);
    const uint32_t begin = __shfl_sync(0xffffffffu, m.out_begin, 0), end = __shfl_sync(0xffffffffu, m.out_end, 0);
    const uint32_t want = __shfl_sync(0xffffffffu, m.crc, 0);
    __syncwarp();  // lane 0's stores are visible to the warp
    uint32_t x = gz::crc32_piece(s_crc, body + begin, end - begin, 32, lane);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) x ^= __shfl_xor_sync(0xffffffffu, x, o);
    if (gz::crc32_finish(x, end - begin) != want) {
      err = gz::GZ_CRC;
      break;
    }
    if (p >= n_src) break;
  }
  out = __shfl_sync(0xffffffffu, out, 0);
  if (!err && out != len) err = gz::GZ_OUTPUT_SHORT;
  if (err && lane == 0) atomicCAS(d_error, 0u, ((uint32_t)DERR_GZIP << 24) | err);
}

}  // namespace

void launch_inflate(hs_ctx* ctx, const PageBlob* blobs, int64_t n, uint8_t* scratch, uint32_t* d_error) {
  if (n == 0) return;
  KernelScope _ks(ctx, "k_inflate");
  k_inflate<<<(unsigned)ceil_div(n, kWarpsPerCta), kWarpsPerCta * 32, 0, ctx->stream>>>(blobs, n, scratch, d_error);
  HS_LAUNCH_CHECK(ctx);
}

}  // namespace hs
