// snappy.cu -- Snappy (raw block format) page decompression on the GPU.
//
// Spark writes Parquet with the SNAPPY codec by default, so the source tables (and index files written by the reference)
// that users hand to createIndex / refreshIndex / the index scans are usually snappy-compressed; the reference reads them
// through parquet-mr + snappy-java (index/covering/CoveringIndexTrait.scala:82-84, CoveringIndexRuleUtils.scala:113-123).
//
// Numeric columns compress into very short elements (a 4-byte copy and a 4-byte literal per 8-byte value is typical), so a
// billion-row table is several billion elements and the decoder is bound by instructions per element, not by bytes: a
// single thread retires one dependent instruction every ~6 cycles, a warp that walks ONE stream spends 32 lanes on one
// element.  Here every LANE walks its own piece of a stream:
//
//  * Every snappy compressor in use (the C++ library behind snappy-java and pyarrow, and k_snappy_compress below) works on
//    64 KB blocks of the input with a fresh hash table per block: no element straddles a 64 KB boundary of the OUTPUT and no
//    back-reference leaves its block.  k_snappy_index (one warp per page) finds where in the compressed stream each output
//    block starts, and checks that property; a page that does not have it (legal snappy, never seen from those writers) is
//    flagged and decoded front to back by a single lane.  Element boundaries are only known by walking the tags, so the
//    walk is speculative: the 32 lanes take 32 consecutive segments (256..1024 bytes) of the stream, each walks its segment from a
//    GUESSED start, then every lane whose true entry point (the exit of the lane before it) differs from what it walked
//    from walks again -- until nothing changes.  Wrong starts fall back onto the true element chain within a few elements,
//    so two rounds is the norm; after round r the first r lanes are certainly right, which bounds it.  No bytes are copied.
//  * k_snappy_blocks (one LANE per 64 KB block, the 32 lanes of a warp in lock step, one element each per round) parses and
//    copies.  Literals of 64 bytes or more -- incompressible data -- are handed to the whole warp: the lanes that hold one
//    are served in turn with coalesced copies.
//  * k_snappy_levels (one warp per page, launched only when needed) copies what is stored verbatim: the level bytes in front
//    of a v2 page's values and pages stored uncompressed inside a compressed chunk.
//
// Reads run up to 8 bytes past the element being parsed: a page body inside a Parquet file is always followed by at least
// the footer length and the magic.
#include <climits>

#include "device_utils.cuh"
#include "lz77.cuh"
#include "page_codec_kernels.h"

namespace hs {

namespace {

constexpr int kWarpsPerCta = 4;
constexpr uint32_t kBlockBytes = 65536;  // snappy's kBlockSize
constexpr uint32_t kCoopLiteral = 64;    // literals from this length on are copied by the whole warp
constexpr uint32_t kSeg = 256;           // least compressed bytes per lane and round of the speculative walk
constexpr uint32_t kBroken = 0xffffffffu;

struct Element {
  uint32_t len, offset, hdr;  // offset == 0: literal of len bytes following hdr tag bytes
};                            // len 0: a literal's length field overflows, or a copy has offset 0 -- the callers reject it

// the element whose tag is at p: two aligned words cover the tag and its (up to) four trailing bytes.  Written with
// selects, not branches: the lanes of a warp parse elements of different kinds in the same instructions.
__device__ __forceinline__ Element parse_element(const uint8_t* __restrict__ p) {
  const uintptr_t a = (uintptr_t)p;
  const uint32_t* w = (const uint32_t*)(a & ~(uintptr_t)3);
  const uint64_t pair = ((uint64_t)w[1] << 32) | w[0];
  const uint64_t v = pair >> (8 * (unsigned)(a & 3));
  const uint32_t tag = (uint32_t)v & 0xffu, trailer = (uint32_t)(v >> 8);
  const uint32_t kind = tag & 3, upper = tag >> 2;
  const bool lit = kind == 0;
  const uint32_t nb = (lit && upper >= 60) ? upper - 59 : 0u;     // length bytes of a long literal
  const uint32_t tail = lit ? nb : (kind == 3 ? 4u : kind);        // bytes after the tag: 0..4
  const uint32_t t = trailer & (tail >= 4 ? 0xffffffffu : ((1u << (8 * tail)) - 1u));
  Element e;
  e.hdr = 1 + tail;
  e.offset = lit ? 0u : (kind == 1 ? ((tag >> 5) << 8) | t : t);
  const uint32_t copy_len = e.offset == 0 ? 0u : (kind == 1 ? (upper & 7) + 4 : upper + 1);  // a copy of offset 0 is invalid
  e.len = lit ? (nb ? t : upper) + 1 : copy_len;  // 0 for a 0xffffffff length field too
  return e;
}

struct Walk {
  uint32_t exit;     // first element start >= the segment's end (kBroken: an element runs past the stream)
  uint32_t out_len;  // bytes the walked elements produce
  int32_t reach;     // max over copies of (offset - bytes produced before the copy since the entry); INT_MIN without copies
};

// walks the elements from `pos` while they start inside [.., seg_hi)
__device__ __forceinline__ Walk walk_segment(const uint8_t* __restrict__ src, uint32_t n_src, uint32_t pos, uint32_t seg_hi) {
  Walk w{pos, 0u, INT_MIN};
  while (pos < seg_hi) {
    const Element e = parse_element(src + pos);
    const uint32_t adv = e.hdr + (e.offset == 0 ? e.len : 0u);
    if (e.len == 0 || adv < e.hdr || adv > n_src - pos) {
      pos = kBroken;
      break;
    }
    if (e.offset != 0) w.reach = max(w.reach, e.offset > 0xffffu ? INT_MAX : (int32_t)e.offset - (int32_t)w.out_len);
    w.out_len += e.len;
    pos += adv;
  }
  w.exit = pos;
  return w;
}

// Pass 1: block_in[first_block + b] = position in the compressed stream (after the v2 prefix) of output block b;
// sequential[w] = 1 when the page's blocks are not independent (or the stream looks damaged: the decoder reports it).
__global__ void __launch_bounds__(kWarpsPerCta * 32) k_snappy_index(const PageBlob* __restrict__ blobs, int64_t n,
                                                                     uint32_t* __restrict__ block_in, uint32_t* __restrict__ sequential) {
  const unsigned lane = threadIdx.x & 31;
  const int64_t w = (int64_t)blockIdx.x * kWarpsPerCta + (threadIdx.x >> 5);
  if (w >= n) return;
  const PageBlob b = blobs[w];
  if (!b.compressed) {
    if (lane == 0) sequential[w] = 0;
    return;
  }
  const uint32_t n_src = b.src_len - b.prefix, dst_len = b.dst_len - b.prefix;
  uint32_t* my_in = block_in + b.first_block;
  const uint8_t* __restrict__ src = b.src + b.prefix;
  uint32_t pos0 = 0, out0 = 0;
  while (pos0 < n_src && pos0 < 5) {  // preamble: uncompressed length as a varint (checked by the decoder)
    if (!(src[pos0++] & 0x80)) break;
  }
  if (lane == 0) my_in[0] = pos0;
  bool seq = false;
  // compressed bytes per lane and round: long segments need fewer rounds to settle (simulation on a double column written by
  // the C++ library: 5 rounds with 256 bytes, 3 with 1024), short ones keep the lanes of a small page busy
  const uint32_t seg = n_src >= 32u * 1024u ? 1024u : (n_src >= 32u * 512u ? 512u : kSeg);
  for (uint32_t base = 0; base < n_src && !seq; base += 32 * seg) {
    base = max(base, pos0 & ~(seg - 1));  // a long literal may have carried the chain past whole rounds
    if (base >= n_src) break;
    const uint32_t seg_lo = min(base + lane * seg, n_src), seg_hi = min(seg_lo + seg, n_src);
    uint32_t entry = lane == 0 ? pos0 : seg_lo, walked_from = kBroken;
    Walk wk{kBroken, 0u, INT_MIN};
    while (true) {
      if (entry != walked_from) {
        wk = entry < seg_hi ? walk_segment(src, n_src, entry, seg_hi) : Walk{entry, 0u, INT_MIN};
        walked_from = entry;
      }
      // lanes [0, trusted) walked from their true entries: lane 0 always did, lane i did if it started where lane i-1,
      // itself trusted, came out
      const uint32_t before = __shfl_up_sync(0xffffffffu, wk.exit, 1);
      const unsigned agree = __ballot_sync(0xffffffffu, entry == (lane == 0 ? pos0 : before));
      if (agree == 0xffffffffu) break;
      const unsigned trusted = __ffs(~agree) - 1;  // >= 1
      const uint32_t chain = __shfl_sync(0xffffffffu, wk.exit, trusted - 1);
      if (lane >= trusted) {
        if (lane == trusted || seg_hi <= chain) {
          entry = chain;  // the first lane after the trusted ones, and every lane a trusted long literal skips entirely
        } else if (before <= seg_lo + 64) {
          entry = before;
        }  // else: a guessed walk that left through a long literal -- usually a data byte read as a tag; wait until that
           // lane is trusted rather than let a wrong position ripple through the lanes behind it
      }
    }
    // the chain is the true one now: output position at every lane's entry
    uint32_t incl = wk.out_len;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const uint32_t up = __shfl_up_sync(0xffffffffu, incl, d);
      if ((int)lane >= d) incl += up;
    }
    const uint32_t out_entry = out0 + incl - wk.out_len;
    const uint32_t in_block = out_entry & (kBlockBytes - 1);
    bool bad = false;
    if (wk.out_len != 0) {
      if (wk.out_len > dst_len - min(out_entry, dst_len)) {
        bad = true;
      } else if (in_block + wk.out_len < kBlockBytes) {
        bad = wk.reach > (int32_t)in_block;  // some copy reaches back past the start of its block
      } else {  // a block ends inside this lane's elements: walk them once more with absolute positions
        uint32_t pos = entry, out = out_entry;
        while (pos < seg_hi) {
          const Element e = parse_element(src + pos);
          const uint32_t ib = out & (kBlockBytes - 1);
          if (e.len > kBlockBytes - ib || e.offset > ib) {
            bad = true;
            break;
          }
          out += e.len;
          pos += e.hdr + (e.offset == 0 ? e.len : 0u);
          if ((out & (kBlockBytes - 1)) == 0 && out < dst_len) my_in[out >> 16] = pos;
        }
      }
    }
    pos0 = __shfl_sync(0xffffffffu, wk.exit, 31);
    out0 += __shfl_sync(0xffffffffu, incl, 31);
    seq = __any_sync(0xffffffffu, bad) || pos0 == kBroken;
  }
  // the reference decoder insists on consuming the whole stream; anything else goes to the front-to-back decoder, which names it
  if (pos0 != n_src || out0 != dst_len) seq = true;
  if (lane == 0) sequential[w] = seq ? 1u : 0u;
}

// len bytes from `from` to `o`; `far`: the ranges do not overlap within 8 bytes (loads of a chunk may go before its stores)
__device__ __forceinline__ void copy_bytes(uint8_t* o, const uint8_t* from, uint32_t len, bool far) {
  if (!far) {  // offsets 1..7: bytes just written are the source (run-length patterns)
    for (uint32_t j = 0; j < len; j++) o[j] = from[j];
    return;
  }
  for (uint32_t j = 0; j < len; j += 8) {
    uint8_t r[8];
#pragma unroll
    for (uint32_t k = 0; k < 8; k++)
      if (j + k < len) r[k] = from[j + k];
#pragma unroll
    for (uint32_t k = 0; k < 8; k++)
      if (j + k < len) o[j + k] = r[k];
  }
}

// len bytes from lit to o by the whole warp.  Byte-wide accesses saturate the load/store unit long before they saturate
// memory (ncu: lg_throttle), so the body moves 16 bytes per lane and step: the destination is brought to 16-byte alignment,
// the source is read as aligned words and realigned with funnel shifts (reads stay inside [lit & ~3, lit + len + 4)).
__device__ __forceinline__ void warp_copy(uint8_t* o, const uint8_t* lit, uint32_t len, unsigned lane) {
  const uint32_t head = min(len, (uint32_t)((16 - ((uintptr_t)o & 15)) & 15));
  if (lane < head) o[lane] = lit[lane];
  o += head;
  lit += head;
  len -= head;
  const unsigned sh = 8 * (unsigned)((uintptr_t)lit & 3);
  const uint32_t* ws = (const uint32_t*)((uintptr_t)lit & ~(uintptr_t)3);
  const uint32_t nvec = len / 16;
  uint4* ov = (uint4*)o;
  uint32_t v = lane;
  for (; v + 32 < nvec; v += 64) {  // two vectors in flight per lane
    const uint32_t* w0 = ws + 4 * v;
    const uint32_t* w1 = w0 + 128;
    const uint32_t a0 = w0[0], a1 = w0[1], a2 = w0[2], a3 = w0[3], a4 = w0[4];
    const uint32_t b0 = w1[0], b1 = w1[1], b2 = w1[2], b3 = w1[3], b4 = w1[4];
    ov[v] = make_uint4(__funnelshift_r(a0, a1, sh), __funnelshift_r(a1, a2, sh), __funnelshift_r(a2, a3, sh), __funnelshift_r(a3, a4, sh));
    ov[v + 32] = make_uint4(__funnelshift_r(b0, b1, sh), __funnelshift_r(b1, b2, sh), __funnelshift_r(b2, b3, sh), __funnelshift_r(b3, b4, sh));
  }
  for (; v < nvec; v += 32) {
    const uint32_t* w0 = ws + 4 * v;
    const uint32_t a0 = w0[0], a1 = w0[1], a2 = w0[2], a3 = w0[3], a4 = w0[4];
    ov[v] = make_uint4(__funnelshift_r(a0, a1, sh), __funnelshift_r(a1, a2, sh), __funnelshift_r(a2, a3, sh), __funnelshift_r(a3, a4, sh));
  }
  for (uint32_t j = nvec * 16 + lane; j < len; j += 32) o[j] = lit[j];
}

// Pass 2: one lane per 64 KB output block (or per page, for a page flagged sequential).
__global__ void __launch_bounds__(kWarpsPerCta * 32) k_snappy_blocks(const PageBlob* __restrict__ blobs, int64_t n,
                                                                      int64_t total_blocks, const uint32_t* __restrict__ block_in,
                                                                      const uint32_t* __restrict__ sequential,
                                                                      uint8_t* __restrict__ scratch, uint32_t* __restrict__ d_error) {
  const unsigned lane = threadIdx.x & 31;
  const int64_t blk = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const uint8_t* src = nullptr;
  uint8_t* dst = nullptr;
  uint32_t pos = 0, in_hi = 0, out = 0, out_lo = 0, out_hi = 0, error = 0;
  bool live = blk < total_blocks;
  if (live) {
    // the page this block belongs to: last blob with first_block <= blk
    int64_t lo = 0, hi = n - 1;
    while (lo < hi) {
      const int64_t mid = (lo + hi + 1) >> 1;
      if ((int64_t)blobs[mid].first_block <= blk) lo = mid; else hi = mid - 1;
    }
    const PageBlob b = blobs[lo];
    const uint32_t bi = (uint32_t)(blk - b.first_block);
    const bool seq = b.compressed && sequential[lo] != 0;
    live = b.compressed && !(seq && bi > 0);
    if (live) {
      src = b.src + b.prefix;
      dst = scratch + b.dst_off + b.prefix;
      const uint32_t n_src = b.src_len - b.prefix, dst_len = b.dst_len - b.prefix;
      const uint32_t n_blocks = snappy_blocks_of(b.dst_len, b.prefix);
      const uint32_t* my_in = block_in + b.first_block;
      out_lo = seq ? 0u : bi * kBlockBytes;
      out_hi = seq ? dst_len : min(out_lo + kBlockBytes, dst_len);
      pos = my_in[bi];
      in_hi = (seq || bi + 1 >= n_blocks) ? n_src : min(my_in[bi + 1], n_src);
      out = out_lo;
      if (bi == 0) {  // preamble: the uncompressed length must be the page header's, a varint of 32 bits at most
        uint32_t p = 0, ulen = 0;
        int shift = 0;
        bool ended = false;
        while (p < n_src && p < 5) {
          const uint8_t c = src[p++];
          ulen |= (uint32_t)(c & 0x7f) << shift;
          ended = !(c & 0x80);
          if (ended) break;
          shift += 7;
        }
        if (!ended || (p == 5 && src[4] >= 16) || ulen != dst_len || p != pos) error = 1;
      }
    }
  }
  while (true) {
    const bool active = live && !error && out < out_hi && pos < in_hi;
    if (!__any_sync(0xffffffffu, active)) break;
    Element e{0, 0, 0};
    bool coop = false;
    if (active) {
      e = parse_element(src + pos);
      if (e.len == 0 || e.len > out_hi - out) {
        error = 2;
      } else if (e.hdr + (e.offset == 0 ? e.len : 0u) > in_hi - pos) {
        error = 3;
      } else if (e.offset > out - out_lo) {
        error = 4;
      } else if (e.offset == 0 && e.len >= kCoopLiteral) {
        coop = true;
      } else {
        // one path for short literals and copies.  A lane sees its own earlier stores, so a byte-by-byte copy of an
        // overlapping back-reference (offset < len) repeats the pattern as the format asks.
        uint8_t* o = dst + out;
        copy_bytes(o, e.offset == 0 ? src + pos + e.hdr : o - e.offset, e.len, e.offset == 0 || e.offset >= 8);
      }
    }
    unsigned turn = __ballot_sync(0xffffffffu, coop);
    while (turn) {  // long literals: the whole warp copies for one lane at a time
      const int l = __ffs(turn) - 1;
      turn &= turn - 1;
      const uint8_t* lit = (const uint8_t*)__shfl_sync(0xffffffffu, (unsigned long long)(src + pos + e.hdr), l);
      uint8_t* o = (uint8_t*)__shfl_sync(0xffffffffu, (unsigned long long)(dst + out), l);
      const uint32_t len = __shfl_sync(0xffffffffu, e.len, l);
      warp_copy(o, lit, len, lane);
    }
    __syncwarp();  // a lane's later back-references may read what the warp just wrote for it
    if (active && !error) {
      out += e.len;
      pos += e.hdr + (e.offset == 0 ? e.len : 0u);
    }
  }
  // the block's bytes are all there, and so is nothing else: as the reference decoder, refuse elements after a full output
  if (live && !error) error = out != out_hi ? 5u : (pos != in_hi ? 6u : 0u);
  if (error) atomicCAS(d_error, 0u, ((uint32_t)DERR_SNAPPY << 24) | error);
}

// what is stored verbatim: v2 level bytes in front of the values, and pages stored uncompressed inside a compressed chunk
__global__ void __launch_bounds__(256) k_snappy_levels(const PageBlob* __restrict__ blobs, int64_t n, uint8_t* __restrict__ scratch) {
  const unsigned lane = threadIdx.x & 31;
  const int64_t w = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (w >= n) return;
  const PageBlob b = blobs[w];
  const uint32_t bytes = b.compressed ? b.prefix : min(b.src_len, b.dst_len);
  uint8_t* __restrict__ dst = scratch + b.dst_off;
  for (uint32_t j = lane; j < bytes; j += 32) dst[j] = b.src[j];
}

}  // namespace

void launch_snappy_decompress(hs_ctx* ctx, const PageBlob* blobs, int64_t n, int64_t total_blocks, bool any_verbatim,
                              uint32_t* block_in, uint32_t* sequential, uint8_t* scratch, uint32_t* d_error) {
  if (n == 0) return;
  if (any_verbatim) {
    KernelScope _ks(ctx, "k_snappy_levels");
    k_snappy_levels<<<(unsigned)ceil_div(n, 8), 256, 0, ctx->stream>>>(blobs, n, scratch);
    HS_LAUNCH_CHECK(ctx);
  }
  {
    KernelScope _ks(ctx, "k_snappy_index");
    k_snappy_index<<<(unsigned)ceil_div(n, kWarpsPerCta), kWarpsPerCta * 32, 0, ctx->stream>>>(blobs, n, block_in, sequential);
    HS_LAUNCH_CHECK(ctx);
  }
  KernelScope _ks(ctx, "k_snappy_blocks");
  k_snappy_blocks<<<(unsigned)ceil_div(total_blocks, kWarpsPerCta * 32), kWarpsPerCta * 32, 0, ctx->stream>>>(
      blobs, n, total_blocks, block_in, sequential, scratch, d_error);
  HS_LAUNCH_CHECK(ctx);
}

}  // namespace hs

// =====================================================================================================================
// Snappy compression of index pages (raw block format), one warp per 64 KB fragment of a page.
//
// Spark writes its Parquet -- and therefore the reference's index files -- with the SNAPPY codec by default
// (index/DataFrameWriterExtensions.scala:59-66 goes through DataFrameWriter; file names ...c000.snappy.parquet,
// T/index/VacuumOutdatedActionTest.scala:67).  A page's compressed body is the varint of its uncompressed length followed by
// the element streams of its fragments, which are compressed independently (back-references never leave a fragment, as in
// snappy's own 64 KB blocks) and therefore in parallel.  The fragment is parsed by lz77_parse (lz77.cuh); its sequences
// become a literal element and copies with 2-byte offsets.
// =====================================================================================================================
namespace hs {
namespace {

constexpr int kCompWarps = 4;

// literal [from, to) of `in` -> out; returns the new output position (all lanes take part)
__device__ __forceinline__ uint32_t emit_literal(const uint8_t* __restrict__ in, uint32_t from, uint32_t to, uint8_t* __restrict__ out,
                                                 uint32_t op, unsigned lane) {
  const uint32_t len = to - from;
  if (len == 0) return op;
  uint32_t hdr;
  if (len <= 60) {
    if (lane == 0) out[op] = (uint8_t)((len - 1) << 2);
    hdr = 1;
  } else if (len <= 256) {
    if (lane == 0) {
      out[op] = (uint8_t)(60 << 2);
      out[op + 1] = (uint8_t)(len - 1);
    }
    hdr = 2;
  } else {  // len <= 65536 (a fragment)
    if (lane == 0) {
      out[op] = (uint8_t)(61 << 2);
      out[op + 1] = (uint8_t)((len - 1) & 0xff);
      out[op + 2] = (uint8_t)((len - 1) >> 8);
    }
    hdr = 3;
  }
  for (uint32_t j = lane; j < len; j += 32) out[op + hdr + j] = in[from + j];
  return op + hdr + len;
}

struct SnappyEmitter {
  const uint8_t* __restrict__ in;
  uint8_t* __restrict__ out;
  uint32_t op;
  unsigned lane;

  __device__ __forceinline__ void sequence(uint32_t lit, uint32_t q, uint32_t offset, uint32_t mlen) {
    op = emit_literal(in, lit, q, out, op, lane);
    if (mlen <= 11 && offset < 2048) {  // short match nearby: the 2-byte copy element (4..11 bytes, 11-bit offset)
      if (lane == 0) {
        out[op] = (uint8_t)(1u | ((mlen - 4) << 2) | ((offset >> 8) << 5));
        out[op + 1] = (uint8_t)(offset & 0xff);
      }
      op += 2;
    } else {
      if (lane == 0) {  // copies with a 2-byte offset carry 1..64 bytes each
        uint32_t left = mlen, o = op;
        while (left > 0) {
          const uint32_t l = left > 64 ? 64 : left;
          out[o] = (uint8_t)(2u | ((l - 1) << 2));
          out[o + 1] = (uint8_t)(offset & 0xff);
          out[o + 2] = (uint8_t)(offset >> 8);
          o += 3;
          left -= l;
        }
      }
      op += 3 * ((mlen + 63) / 64);
    }
  }
  __device__ __forceinline__ void finish(uint32_t lit, uint32_t len) { op = emit_literal(in, lit, len, out, op, lane); }
};

__global__ void __launch_bounds__(kCompWarps * 32) k_snappy_compress(const PageFragment* __restrict__ frags, int64_t n,
                                                                      const uint8_t* __restrict__ raw, uint8_t* __restrict__ scratch,
                                                                      uint32_t* __restrict__ out_len) {
  __shared__ uint32_t s_table[kCompWarps][kLz77Table];
  const unsigned lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
  const int64_t f = (int64_t)blockIdx.x * kCompWarps + wib;
  if (f >= n) return;
  const PageFragment fr = frags[f];
  SnappyEmitter emit{raw + fr.src_off, scratch + fr.dst_off, 0u, lane};
  // every offset of a fragment fits the 2-byte copy, and a copy may end anywhere
  lz77_parse(raw + fr.src_off, fr.len, s_table[wib], lane, Lz77Limits{0xffffu, 0xffffffffu, 4u, 0u}, emit);
  if (lane == 0) out_len[f] = emit.op;
}

}  // namespace

void launch_snappy_compress(hs_ctx* ctx, const PageFragment* frags, int64_t n, const uint8_t* raw, uint8_t* scratch,
                            uint32_t* out_len) {
  KernelScope _ks(ctx, "k_snappy_compress");
  if (n == 0) return;
  k_snappy_compress<<<(unsigned)ceil_div(n, kCompWarps), kCompWarps * 32, 0, ctx->stream>>>(frags, n, raw, scratch, out_len);
  HS_LAUNCH_CHECK(ctx);
}

}  // namespace hs
