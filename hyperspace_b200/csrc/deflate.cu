// deflate.cu -- GZIP compression of index pages (Spark's spark.sql.parquet.compression.codec=gzip), one warp per 64 KB
// fragment of a page body, four warps per CTA.
//
// A fragment is parsed twice by lz77_parse (lz77.cuh), with DEFLATE's limits: the parse is deterministic, so the second
// pass sees the symbols the first one counted.
//  * Pass 1 counts literal/length and distance symbols in shared memory.  Lane 0 then builds both codes (deflate.h:
//    lengths limited to 15 bits, ties broken by symbol index) and sizes three encodings of the fragment: one dynamic-Huffman
//    block, one fixed-Huffman block, stored blocks.  The smallest is written.
//  * Pass 2 writes the Huffman block's symbols by the warp: each lane takes one symbol (a literal, or a length with its
//    distance), a prefix sum of their bit lengths places them, the lanes OR their bits into a staging buffer in shared
//    memory, and the complete words go out as disjoint word stores.
//  * Every fragment ends non-final and byte-aligned with a sync flush, so the fragments of a page are concatenated as
//    they are.  The warp also computes the fragment's CRC-32 (one piece per lane, combined by linearity as k_inflate does);
//    the host combines the fragments' CRCs into the member's trailer (page_codec.cu).
#include "deflate.h"
#include "device_utils.cuh"
#include "lz77.cuh"
#include "page_codec_kernels.h"

namespace hs {

namespace {

constexpr int kWarpsPerCta = 4;
constexpr uint32_t kStageWords = 64;  // a batch of 32 symbols of at most 48 bits, behind at most 31 pending bits
constexpr int kModeStored = 0, kModeFixed = 1, kModeDynamic = 2;

struct DeflateShared {
  // the parse's hash table; between the passes, the Huffman builder's work area and (from word kHeaderAt) the block header
  uint32_t table[kLz77Table];
  uint32_t hist[gz::kLitCodes + gz::kDistCodes];  // literal/length symbols, then distance symbols
  uint32_t stage[kStageWords];
  uint16_t codes[gz::kLitCodes + gz::kDistCodes];
  uint8_t lens[gz::kLitCodes + gz::kDistCodes + 4];
};
constexpr uint32_t kHeaderAt = 1536;  // > 5 * 286 words of huffman_lengths' work area
static_assert(kHeaderAt * 4 + sizeof(gz::DynamicHeader) <= kLz77Table * 4, "the block header fits the table");

// the warp's bit stream: stage[0] holds the bits of output word `word` written so far (`used` of them)
struct WarpBits {
  uint32_t* stage;
  uint32_t* out;
  uint32_t word, used;

  // appends lane's n bits v (n <= 48; 0: nothing) after those of the lanes before it
  __device__ __forceinline__ void put(uint64_t v, uint32_t n, unsigned lane) {
    uint32_t incl = n;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const uint32_t up = __shfl_up_sync(0xffffffffu, incl, d);
      if ((int)lane >= d) incl += up;
    }
    const uint32_t total = __shfl_sync(0xffffffffu, incl, 31);
    if (n) {
      const uint32_t at = used + incl - n, w = at >> 5, sh = at & 31;
      const uint64_t rest = sh ? v >> (32 - sh) : v >> 32;
      atomicOr(&stage[w], (uint32_t)(v << sh));
      if ((uint32_t)rest) atomicOr(&stage[w + 1], (uint32_t)rest);
      if (rest >> 32) atomicOr(&stage[w + 2], (uint32_t)(rest >> 32));
    }
    __syncwarp();
    used += total;
    const uint32_t full = used >> 5;
    for (uint32_t j = lane; j < full; j += 32) out[word + j] = stage[j];
    const uint32_t part = stage[full];
    __syncwarp();
    for (uint32_t j = lane; j < full + 3 && j < kStageWords; j += 32) stage[j] = j == 0 ? part : 0u;
    __syncwarp();
    word += full;
    used &= 31;
  }
};

// pass 1's emitter: counts the symbols of the fragment's sequences
struct DeflateCounter {
  const uint8_t* __restrict__ in;
  uint32_t* hist;
  unsigned lane;

  __device__ __forceinline__ void literals(uint32_t from, uint32_t to) {
    for (uint32_t j = from + lane; j < to; j += 32) atomicAdd(&hist[in[j]], 1u);
  }
  __device__ __forceinline__ void sequence(uint32_t lit, uint32_t q, uint32_t offset, uint32_t mlen) {
    literals(lit, q);
    if (lane == 0) {
      atomicAdd(&hist[257 + gz::length_index(mlen)], 1u);
      atomicAdd(&hist[gz::kLitCodes + gz::distance_symbol(offset)], 1u);
    }
  }
  __device__ __forceinline__ void finish(uint32_t lit, uint32_t len) { literals(lit, len); }
};

struct DeflateWriter {
  const uint8_t* __restrict__ in;
  const uint16_t* codes;
  const uint8_t* lens;
  WarpBits& bits;
  unsigned lane;

  // literals in[lit, to), then the match (mlen, offset) -- or, mlen 0, the end-of-block symbol
  __device__ __forceinline__ void symbols(uint32_t lit, uint32_t to, uint32_t offset, uint32_t mlen) {
    const uint32_t n = to - lit + 1;
    for (uint32_t base = 0; base < n; base += 32) {
      const uint32_t i = base + lane;
      uint64_t v = 0;
      uint32_t nb = 0;
      if (i + 1 < n) {
        const uint8_t s = in[lit + i];
        v = codes[s];
        nb = lens[s];
      } else if (i + 1 == n && mlen == 0) {
        v = codes[256];
        nb = lens[256];
      } else if (i + 1 == n) {
        const int li = gz::length_index(mlen), ds = gz::distance_symbol(offset);
        v = codes[257 + li];
        nb = lens[257 + li];
        v |= (uint64_t)(mlen - gz::len_base(li)) << nb;
        nb += gz::len_extra(li);
        v |= (uint64_t)codes[gz::kLitCodes + ds] << nb;
        nb += lens[gz::kLitCodes + ds];
        v |= (uint64_t)(offset - gz::dist_base(ds)) << nb;
        nb += gz::dist_extra(ds);
      }
      bits.put(v, nb, lane);
    }
  }
  __device__ __forceinline__ void sequence(uint32_t lit, uint32_t q, uint32_t offset, uint32_t mlen) {
    symbols(lit, q, offset, mlen);
  }
  __device__ __forceinline__ void finish(uint32_t lit, uint32_t len) { symbols(lit, len, 0, 0); }
};

// bits of the symbols counted in hist under code lengths lit_len(s) / dist_len(d), extra bits included
template <class L, class D>
__device__ uint64_t symbol_bits(const uint32_t* hist, L lit_len, D dist_len) {
  uint64_t bits = 0;
  for (int s = 0; s < (int)gz::kLitCodes; s++)
    bits += (uint64_t)hist[s] * (lit_len(s) + (s >= 257 ? gz::len_extra(s - 257) : 0u));
  for (int d = 0; d < (int)gz::kDistCodes; d++) bits += (uint64_t)hist[gz::kLitCodes + d] * (dist_len(d) + gz::dist_extra(d));
  return bits;
}

__global__ void __launch_bounds__(kWarpsPerCta * 32) k_deflate_compress(const PageFragment* __restrict__ frags, int64_t n,
                                                                         const uint8_t* __restrict__ raw,
                                                                         uint8_t* __restrict__ scratch,
                                                                         uint32_t* __restrict__ out_len,
                                                                         uint32_t* __restrict__ out_crc) {
  __shared__ DeflateShared s_warp[kWarpsPerCta];
  __shared__ uint32_t s_crc[256];
  for (uint32_t i = threadIdx.x; i < 256; i += blockDim.x) s_crc[i] = gz::crc32_table_entry(i);
  __syncthreads();
  const unsigned lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
  const int64_t f = (int64_t)blockIdx.x * kWarpsPerCta + wib;
  if (f >= n) return;
  DeflateShared& sh = s_warp[wib];
  const PageFragment fr = frags[f];
  const uint8_t* __restrict__ in = raw + fr.src_off;
  uint8_t* __restrict__ out = scratch + fr.dst_off;
  const uint32_t len = fr.len;
  const Lz77Limits limits{32768u, 258u, 4u, 0u};

  // the fragment's CRC-32 without pre- and post-inversion
  uint32_t x = gz::crc32_piece(s_crc, in, len, 32, lane);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) x ^= __shfl_xor_sync(0xffffffffu, x, o);
  if (lane == 0) out_crc[f] = x;

  // pass 1: symbol counts
  for (uint32_t i = lane; i < gz::kLitCodes + gz::kDistCodes; i += 32) sh.hist[i] = i == 256 ? 1u : 0u;
  for (uint32_t i = lane; i < kStageWords; i += 32) sh.stage[i] = 0;
  __syncwarp();
  DeflateCounter counter{in, sh.hist, lane};
  lz77_parse(in, len, sh.table, lane, limits, counter);
  __syncwarp();

  // lane 0: the codes, the smallest encoding, and the block header
  int mode = kModeStored;
  uint32_t word = 0, used = 0;
  if (lane == 0) {
    uint8_t* lens = sh.lens;
    gz::DynamicHeader& hdr = *reinterpret_cast<gz::DynamicHeader*>(sh.table + kHeaderAt);
    gz::huffman_lengths(sh.hist, gz::kLitCodes, gz::kMaxBits, lens, sh.table);
    gz::huffman_lengths(sh.hist + gz::kLitCodes, gz::kDistCodes, gz::kMaxBits, lens + gz::kLitCodes, sh.table);
    const uint64_t dyn = 3 + gz::plan_dynamic_header(lens, lens + gz::kLitCodes, hdr, sh.table) +
                         symbol_bits(sh.hist, [&](int s) { return (uint32_t)lens[s]; },
                                     [&](int d) { return (uint32_t)lens[gz::kLitCodes + d]; });
    const uint64_t fixed = 3 + symbol_bits(sh.hist, [](int s) { return (uint32_t)gz::fixed_lit_len(s); }, [](int) { return 5u; });
    // bytes with the sync flush: a Huffman block, then 3 bits, a byte boundary and 4 bytes; stored blocks, then 5 bytes
    auto total = [](uint64_t b) { return (b + 3 + 7) / 8 + 4; };
    const uint64_t stored = gz::deflate_fragment_bound(len);
    if (total(dyn) <= total(fixed) && total(dyn) < stored) {
      mode = kModeDynamic;
    } else if (total(fixed) < stored) {
      mode = kModeFixed;
      for (int s = 0; s < (int)gz::kLitCodes; s++) lens[s] = gz::fixed_lit_len(s);
      for (int d = 0; d < (int)gz::kDistCodes; d++) lens[gz::kLitCodes + d] = 5;
    }
    if (mode != kModeStored) {
      if (mode == kModeDynamic) {
        gz::huffman_codes(lens, gz::kLitCodes, sh.codes);
      } else {  // the fixed code has 288 symbols: the 9-bit codes come after those of 286 and 287
        for (int s = 0; s < (int)gz::kLitCodes; s++) sh.codes[s] = gz::fixed_lit_code(s);
      }
      gz::huffman_codes(lens + gz::kLitCodes, gz::kDistCodes, sh.codes + gz::kLitCodes);
      gz::BitWriter bw{out, 0, 0, 0};
      bw.put(mode == kModeDynamic ? 4u : 2u, 3);  // BFINAL 0, BTYPE 10 or 01
      if (mode == kModeDynamic) gz::write_dynamic_header(bw, hdr);
      word = bw.pos >> 2;
      uint32_t part = 0;
      for (uint32_t b = word * 4; b < bw.pos; b++) part |= (uint32_t)out[b] << (8 * (b & 3));
      sh.stage[0] = part | (uint32_t)bw.acc << (8 * (bw.pos & 3));
      used = 8 * (bw.pos & 3) + bw.cnt;
    }
  }
  mode = __shfl_sync(0xffffffffu, mode, 0);
  word = __shfl_sync(0xffffffffu, word, 0);
  used = __shfl_sync(0xffffffffu, used, 0);
  __syncwarp();

  if (mode == kModeStored) {
    uint32_t op = 0;
    for (uint32_t o = 0; o < len; o += 65535) {
      const uint32_t bl = min(65535u, len - o);
      if (lane == 0) gz::put_stored_header(out + op, bl);
      for (uint32_t j = lane; j < bl; j += 32) out[op + 5 + j] = in[o + j];
      op += 5 + bl;
    }
    if (lane == 0) gz::put_stored_header(out + op, 0);  // the sync flush
    if (lane == 0) out_len[f] = op + 5;
    return;
  }
  // pass 2: the symbols
  WarpBits bits{sh.stage, reinterpret_cast<uint32_t*>(out), word, used};
  DeflateWriter writer{in, sh.codes, sh.lens, bits, lane};
  lz77_parse(in, len, sh.table, lane, limits, writer);
  // the sync flush: an empty stored block -- 3 bits, the byte boundary, LEN 0000 and NLEN ffff
  const uint32_t pad = (8 - ((bits.used + 3) & 7)) & 7;
  bits.put(lane == 0 ? (uint64_t)gz::kSyncFlush << (3 + pad) : 0ull, lane == 0 ? 3 + pad + 32 : 0u, lane);
  if (lane == 0) {
    if (bits.used) reinterpret_cast<uint32_t*>(out)[bits.word] = sh.stage[0];
    out_len[f] = bits.word * 4 + bits.used / 8;
  }
}

}  // namespace

void launch_deflate_compress(hs_ctx* ctx, const PageFragment* frags, int64_t n, const uint8_t* raw, uint8_t* scratch,
                             uint32_t* out_len, uint32_t* out_crc) {
  KernelScope _ks(ctx, "k_deflate_compress");
  if (n == 0) return;
  k_deflate_compress<<<(unsigned)ceil_div(n, kWarpsPerCta), kWarpsPerCta * 32, 0, ctx->stream>>>(frags, n, raw, scratch, out_len,
                                                                                                  out_crc);
  HS_LAUNCH_CHECK(ctx);
}

}  // namespace hs
