// lz4.cu -- LZ4 and LZ4_RAW page decompression on the GPU.
//
// Spark 2.4 - 3.1 with `spark.sql.parquet.compression.codec=lz4` write Parquet codec 5 (Hadoop's Lz4Codec: LZ4 blocks
// inside Hadoop's framing); newer parquet-mr and Spark (`lz4_raw`) and Arrow write codec 7, one bare block per page.  An
// LZ4 page is one block (or a few, under codec 5) whose matches reach up to 65 535 bytes back anywhere in it, so the unit
// of work is the page: one warp per page, four warps per CTA.  Per batch of up to 32 sequences:
//
//  * Lane 0 parses the sequences (lz4_block.h: parse_sequence, with every check) into the warp's table in shared memory.
//    Parsing touches a few bytes per sequence; copying is the work.
//  * Phase A: the whole warp copies, flattened over bytes through a prefix sum of their lengths, every literal run of the
//    batch and every match whose source lies before the batch's first output byte.  These writes are disjoint and read
//    only input bytes or output that is already final.
//  * Phase B: the other matches, in order, each by the whole warp as dst[p + j] = dst[p - off + j mod off], which reads
//    only bytes before p (final by then), so overlapping copies repeat their period as the format asks.
//
// The warp also copies what is stored verbatim: the level bytes in front of a v2 page's values, and v2 pages stored
// uncompressed inside an LZ4 chunk.  Under codec 5 lane 0 walks the groups and chunks (hadoop_next) and the warp decodes
// each chunk; a body that fails as groups is decoded again as one raw block, over whatever the attempt wrote.
#include "device_utils.cuh"
#include "lz4_block.h"
#include "lz77.cuh"
#include "page_codec_kernels.h"

namespace hs {

namespace {

constexpr int kWarpsPerCta = 4;
constexpr int kBatch = 32;  // sequences per batch: one per lane

struct WarpTable {
  lz4::Seq seq[kBatch];
  uint32_t start[kBatch + 1];  // phase A: first flattened byte of each sequence's literals (+ match), and the total
};

// The block src[ip, n) into dst from `out` with capacity cap, by the whole warp; returns an Lz4Error (the same in every
// lane) and leaves out past the block's output.
__device__ __forceinline__ uint32_t decode_block(const uint8_t* __restrict__ src, uint32_t ip, uint32_t n, uint8_t* __restrict__ dst,
                                 uint32_t& out, uint32_t cap, WarpTable& t, unsigned lane) {
  const uint32_t block_start = out;
  for (;;) {
    const uint32_t batch_start = out;
    uint32_t cnt = 0, err = 0, last_seen = 0;
    if (lane == 0) {
      bool last = false;
      while (cnt < kBatch && !last) {
        err = lz4::parse_sequence(src, n, ip, out, block_start, cap, t.seq[cnt], last);
        if (err) break;
        cnt++;
      }
      last_seen = last ? 1u : 0u;
    }
    err = __shfl_sync(0xffffffffu, err, 0);
    if (err) return err;
    cnt = __shfl_sync(0xffffffffu, cnt, 0);
    last_seen = __shfl_sync(0xffffffffu, last_seen, 0);
    ip = __shfl_sync(0xffffffffu, ip, 0);
    out = __shfl_sync(0xffffffffu, out, 0);
    __syncwarp();  // lane 0's table is visible to the warp

    // phase A: lane i sizes sequence i's share, and the shares are laid end to end
    lz4::Seq s{0, 0, 0, 0, 0};
    if (lane < cnt) s = t.seq[lane];
    const uint32_t p = s.out + s.lit_len;  // the match's first output byte
    const bool early = s.match_len == 0 || p - s.offset + min(s.match_len, s.offset) <= batch_start;
    const uint32_t share = s.lit_len + (early ? s.match_len : 0u);
    uint32_t incl = share;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const uint32_t v = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= (unsigned)o) incl += v;
    }
    t.start[lane] = incl - share;
    if (lane == 31) t.start[kBatch] = incl;
    const unsigned late = __ballot_sync(0xffffffffu, lane < cnt && !early);
    __syncwarp();
    const uint32_t total = t.start[kBatch];
    uint32_t k = 0;  // the sequence of this lane's byte: advances with it
    for (uint32_t g = lane; g < total; g += 32) {
      while (g >= t.start[k + 1]) k++;
      const lz4::Seq& q = t.seq[k];
      const uint32_t j = g - t.start[k];
      if (j < q.lit_len) {
        dst[q.out + j] = src[q.lit_src + j];
      } else {
        const uint32_t m = j - q.lit_len, at = q.out + q.lit_len;
        dst[at + m] = dst[at - q.offset + (m < q.offset ? m : m % q.offset)];
      }
    }
    // phase B: the matches that read this batch's output, in order
    for (unsigned rest = late; rest; rest &= rest - 1) {
      __syncwarp();
      const lz4::Seq& q = t.seq[__ffs(rest) - 1];
      const uint32_t at = q.out + q.lit_len;
      for (uint32_t m = lane; m < q.match_len; m += 32) dst[at + m] = dst[at - q.offset + (m < q.offset ? m : m % q.offset)];
    }
    __syncwarp();  // the batch is written before the next one reads it, and lane 0 may rewrite the table
    if (last_seen) return lz4::LZ4_OK;
  }
}

__global__ void __launch_bounds__(kWarpsPerCta * 32, 8) k_lz4(const PageBlob* __restrict__ blobs, int64_t n,
                                                            uint8_t* __restrict__ scratch, uint32_t* __restrict__ d_error) {
  __shared__ WarpTable s_tables[kWarpsPerCta];
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
  WarpTable& t = s_tables[wib];
  // codec 5 tries Hadoop's groups and chunks first; a body that fails as groups is decoded as one raw block
  bool groups = b.codec == lz4::kCodecLz4;
  lz4::HadoopCursor c{0, 0, 0};
  uint32_t out = 0, err = 0;
  for (;;) {
    uint32_t cs = 0, cl = n_src, cap = len;
    if (groups) {
      uint32_t r = 0;
      if (lane == 0) r = lz4::hadoop_next(src, n_src, out, len, c, cs, cl);
      r = __shfl_sync(0xffffffffu, r, 0);
      if (r == lz4::HADOOP_DONE) return;
      cs = __shfl_sync(0xffffffffu, cs, 0);
      cl = __shfl_sync(0xffffffffu, cl, 0);
      cap = __shfl_sync(0xffffffffu, c.group_end, 0);
      if (r == lz4::HADOOP_NOT) {
        groups = false;
        out = 0;
        continue;
      }
    }
    err = decode_block(src, cs, cs + cl, body, out, cap, t, lane);
    if (!groups) break;
    if (err) {
      groups = false;
      out = 0;
    }
  }
  if (!err && out != len) err = lz4::LZ4_OUTPUT_SHORT;
  if (err && lane == 0) atomicCAS(d_error, 0u, ((uint32_t)DERR_LZ4 << 24) | err);
}

}  // namespace

void launch_lz4(hs_ctx* ctx, const PageBlob* blobs, int64_t n, uint8_t* scratch, uint32_t* d_error) {
  if (n == 0) return;
  KernelScope _ks(ctx, "k_lz4");
  k_lz4<<<(unsigned)ceil_div(n, kWarpsPerCta), kWarpsPerCta * 32, 0, ctx->stream>>>(blobs, n, scratch, d_error);
  HS_LAUNCH_CHECK(ctx);
}

}  // namespace hs

// =====================================================================================================================
// LZ4 compression of index pages (Spark 2.4-3.1's spark.sql.parquet.compression.codec=lz4: codec 5, Hadoop's Lz4Codec
// framing), one warp per 64 KB fragment of a page body, four warps per CTA.  A fragment is parsed by lz77_parse (lz77.cuh)
// under LZ4's end-of-block rules and becomes one block in a Hadoop group of one chunk -- what Arrow's Lz4HadoopCodec
// requires, and far below the 256 KB buffer of Hadoop's BlockDecompressorStream.  A page body is its fragments' groups
// back to back.
// =====================================================================================================================
namespace hs {
namespace {

constexpr int kCompWarps = 4;

struct Lz4Emitter {
  const uint8_t* __restrict__ in;
  uint8_t* __restrict__ out;  // the block
  uint32_t op;
  unsigned lane;

  __device__ __forceinline__ void literals(uint32_t from, uint32_t to) {
    for (uint32_t j = lane; j < to - from; j += 32) out[op + j] = in[from + j];
    op += to - from;
  }
  __device__ __forceinline__ void sequence(uint32_t lit, uint32_t q, uint32_t offset, uint32_t mlen) {
    op = lz4::put_sequence_head(out, op, q - lit, mlen, lane == 0);
    literals(lit, q);
    op = lz4::put_match(out, op, offset, mlen, lane == 0);
  }
  __device__ __forceinline__ void finish(uint32_t lit, uint32_t len) {
    op = lz4::put_sequence_head(out, op, len - lit, 0, lane == 0);
    literals(lit, len);
  }
};

__global__ void __launch_bounds__(kCompWarps * 32) k_lz4_compress(const PageFragment* __restrict__ frags, int64_t n,
                                                                   const uint8_t* __restrict__ raw, uint8_t* __restrict__ scratch,
                                                                   uint32_t* __restrict__ out_len) {
  __shared__ uint32_t s_table[kCompWarps][kLz77Table];
  const unsigned lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
  const int64_t f = (int64_t)blockIdx.x * kCompWarps + wib;
  if (f >= n) return;
  const PageFragment fr = frags[f];
  uint8_t* group = scratch + fr.dst_off;
  Lz4Emitter emit{raw + fr.src_off, group + lz4::kHadoopGroupHeader, 0u, lane};
  lz77_parse(raw + fr.src_off, fr.len, s_table[wib], lane,
             Lz77Limits{0xffffu, 0xffffffffu, lz4::kMatchStartMargin, lz4::kLastLiterals}, emit);
  if (lane == 0) {
    lz4::put_be32(group, fr.len);
    lz4::put_be32(group + 4, emit.op);
    out_len[f] = lz4::kHadoopGroupHeader + emit.op;
  }
}

}  // namespace

void launch_lz4_compress(hs_ctx* ctx, const PageFragment* frags, int64_t n, const uint8_t* raw, uint8_t* scratch,
                         uint32_t* out_len) {
  KernelScope _ks(ctx, "k_lz4_compress");
  if (n == 0) return;
  k_lz4_compress<<<(unsigned)ceil_div(n, kCompWarps), kCompWarps * 32, 0, ctx->stream>>>(frags, n, raw, scratch, out_len);
  HS_LAUNCH_CHECK(ctx);
}

}  // namespace hs
