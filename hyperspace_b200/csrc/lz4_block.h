// lz4_block.h -- LZ4 blocks (the LZ4 block format) and the two ways Parquet stores them: the per-stream pieces of the LZ4
// page decoder.  __host__ __device__ like inflate.h: the GPU kernel (lz4.cu) parses sequences in one lane per page, and
// tests/native/lz4.cu runs the same code on the CPU against pyarrow.
//
//  * LZ4_RAW (codec 7): a page body (after the v2 level bytes) is one block that decodes to exactly the page's size.
//  * LZ4 (codec 5, Hadoop's Lz4Codec framing): the body is one or more groups, a group being a big-endian u32 uncompressed
//    length U and then one or more chunks (a big-endian u32 compressed length C and C bytes of an independent block) that
//    decode to U bytes in total.  A body that does not decode as groups anywhere is decoded as one raw block: older Parquet
//    C++ wrote raw blocks under codec 5 (Arrow's rule).  When that fails too, the raw attempt's check is reported.
//
// A block is accepted exactly when LZ4_decompress_safe accepts it with the page's size as capacity and returns that size,
// with one exception: a match offset of 0, which the format declares invalid, is refused (LZ4_decompress_safe writes
// zeros for it).  Its end-of-block rules, in terms of the capacity `cap`:
//  * the last sequence is literals only and ends exactly at the end of the input;
//  * any other sequence's literals end at most 12 bytes before cap and 8 bytes before the input's end, and its match
//    ends at most 5 bytes before cap.  The decoder's short-sequence path skips these margins: a sequence of at most 14
//    literals that starts with 32 bytes of capacity and 17 bytes of input left after its token is not held to the
//    literal margins, and when its match is also at most 18 bytes long at an offset of 8 or more, not to the match's;
//  * a match-length extension leaves at least 5 bytes of input.
// Every check returns an Lz4Error; no check reads outside [src, src + n) or lets a write leave [dst, dst + cap), and every
// loop ends (each sequence consumes input).
#pragma once
#include <cstdint>

#ifdef __CUDACC__
#define HS_HD __host__ __device__ __forceinline__
#else
#define HS_HD inline
#endif

namespace hs {
namespace lz4 {

constexpr uint32_t kCodecLz4 = 5;  // pq::LZ4, Hadoop's framing (pq::LZ4_RAW, 7, is a bare block)

enum Lz4Error : uint32_t {
  LZ4_OK = 0,
  LZ4_TRUNCATED = 1,        // the input ends inside a sequence
  LZ4_OFFSET_ZERO = 2,      // match offset 0
  LZ4_BEFORE_START = 3,     // a match reaches before the block's first output byte
  LZ4_OUTPUT_OVERRUN = 4,   // more output than declared
  LZ4_OUTPUT_SHORT = 5,     // less output than declared
  LZ4_END_OF_BLOCK = 6,     // an end-of-block margin is broken
};

HS_HD const char* lz4_error_text(uint32_t e) {
  switch (e) {
    case LZ4_TRUNCATED: return "input ends inside a sequence";
    case LZ4_OFFSET_ZERO: return "match offset 0";
    case LZ4_BEFORE_START: return "match reaches before the start of the block";
    case LZ4_OUTPUT_OVERRUN: return "output longer than the page's uncompressed size";
    case LZ4_OUTPUT_SHORT: return "output shorter than the page's uncompressed size";
    case LZ4_END_OF_BLOCK: return "end-of-block rule broken (last literals, or a match too close to the end)";
    default: return "ok";
  }
}

// One sequence: literals src[lit_src, + lit_len) to dst[out, + lit_len), then match_len bytes at dst[out + lit_len] copied
// from `offset` bytes back (match_len 0: the block's last sequence).
struct Seq {
  uint32_t lit_src, lit_len, out, offset, match_len;
};

// The sequence at src[ip] of the block src[.., n) whose output began at dst offset `start` and has reached `out`; the
// output may not pass `cap`.  On success ip and out are past the sequence and `last` says it ended the block.
HS_HD uint32_t parse_sequence(const uint8_t* src, uint32_t n, uint32_t& ip, uint32_t& out, uint32_t start, uint32_t cap, Seq& s,
                              bool& last) {
  if (ip >= n) return LZ4_TRUNCATED;
  const uint32_t token = src[ip++];
  const uint32_t ip1 = ip;  // the byte after the token
  uint32_t lit = token >> 4;
  if (lit == 15) {
    uint32_t b;
    do {
      if (ip >= n) return LZ4_TRUNCATED;
      b = src[ip++];
      lit += b;
    } while (b == 255 && lit < n);  // a longer run cannot fit the input: the check below says so
  }
  if (lit > n - ip) return LZ4_TRUNCATED;
  s.lit_src = ip;
  s.lit_len = lit;
  s.out = out;
  s.offset = 0;
  s.match_len = 0;
  if (lit > cap - out) return LZ4_OUTPUT_OVERRUN;
  ip += lit;
  out += lit;
  if (ip == n) {  // literals up to the end of the input: the last sequence
    last = true;
    return LZ4_OK;
  }
  last = false;
  if (n - ip < 2) return LZ4_TRUNCATED;
  const uint32_t off = src[ip] | (uint32_t)src[ip + 1] << 8;
  ip += 2;
  uint32_t len = token & 15u;
  if (len == 15) {
    uint32_t b;
    do {
      if (ip >= n) return LZ4_TRUNCATED;
      b = src[ip++];
      len += b;
    } while (b == 255 && len < cap);
    if (n - ip < 5) return LZ4_END_OF_BLOCK;
  }
  len += 4;
  // the short-sequence path: its literal step skips the literal margins, its match step (when it applies too) the match's
  const bool short_lits = (token >> 4) < 15 && cap - s.out >= 32 && n - ip1 >= 17;
  const bool short_match = short_lits && (token & 15u) < 15 && off >= 8;
  if (!short_lits && (cap - out < 12 || n - (s.lit_src + lit) < 8)) return LZ4_END_OF_BLOCK;
  if (off == 0) return LZ4_OFFSET_ZERO;
  if (off > out - start) return LZ4_BEFORE_START;
  if (len > cap - out) return LZ4_OUTPUT_OVERRUN;
  if (!short_match && cap - out - len < 5) return LZ4_END_OF_BLOCK;
  s.offset = off;
  s.match_len = len;
  out += len;
  return LZ4_OK;
}

// ---- codec 5: Hadoop's groups and chunks ----------------------------------------------------------------------------------
enum : uint32_t { HADOOP_CHUNK = 0, HADOOP_DONE = 1, HADOOP_NOT = 2 };
struct HadoopCursor {
  uint32_t p;          // input position
  uint32_t group_end;  // output position where the current group ends
  uint32_t fresh;      // a group header was just read: its first chunk is due
};
HS_HD uint32_t be32(const uint8_t* p) { return (uint32_t)p[0] << 24 | (uint32_t)p[1] << 16 | (uint32_t)p[2] << 8 | p[3]; }

// With the output at `out`: the next chunk [cs, cs + cl) of the body src[0, n), to be decoded with capacity c.group_end;
// HADOOP_DONE when the groups consumed the body and made dst_len bytes; HADOOP_NOT when the body is not such groups.
HS_HD uint32_t hadoop_next(const uint8_t* src, uint32_t n, uint32_t out, uint32_t dst_len, HadoopCursor& c, uint32_t& cs,
                           uint32_t& cl) {
  if (!c.fresh && out == c.group_end) {  // between groups
    if (c.p == n) return out == dst_len ? HADOOP_DONE : HADOOP_NOT;
    if (n - c.p < 4) return HADOOP_NOT;
    const uint32_t u = be32(src + c.p);
    c.p += 4;
    if (u > dst_len - out) return HADOOP_NOT;
    c.group_end = out + u;
    c.fresh = 1;
  }
  if (n - c.p < 4) return HADOOP_NOT;
  cl = be32(src + c.p);
  c.p += 4;
  if (cl > n - c.p) return HADOOP_NOT;
  cs = c.p;
  c.p += cl;
  c.fresh = 0;
  return HADOOP_CHUNK;
}

// ---- encoding (lz4.cu's compressor, and the host build of the tests) ---------------------------------------------------------
// A block the compressor writes keeps the end-of-block rules without the decoder's short-sequence exceptions: no match
// starts in the last kMatchStartMargin bytes of the block, and the last kLastLiterals bytes are literals of the final
// sequence.
constexpr uint32_t kMatchStartMargin = 12, kLastLiterals = 5;
constexpr uint32_t kHadoopGroupHeader = 8;  // a group of one chunk: [BE u32 raw length][BE u32 compressed length][block]

// the largest block of len bytes: literals only, one token and len / 255 + 1 length bytes
HS_HD uint64_t block_bound(uint64_t len) { return len + len / 255 + 16; }

HS_HD void put_be32(uint8_t* p, uint32_t v) {
  p[0] = (uint8_t)(v >> 24);
  p[1] = (uint8_t)(v >> 16);
  p[2] = (uint8_t)(v >> 8);
  p[3] = (uint8_t)v;
}
// 15 in a nibble, then bytes of 255 and the rest: the length fields of literals and matches
HS_HD uint32_t put_length_bytes(uint8_t* out, uint32_t op, uint32_t v, bool write) {
  for (; v >= 255; v -= 255) {
    if (write) out[op] = 255;
    op++;
  }
  if (write) out[op] = (uint8_t)v;
  return op + 1;
}
// The token and literal-length bytes at out[op] of a sequence of lit_len literals and a match of match_len >= 4 bytes
// (0: the block's last sequence, literals only).  Returns where its literals go.  Only the lane with `write` stores.
HS_HD uint32_t put_sequence_head(uint8_t* out, uint32_t op, uint32_t lit_len, uint32_t match_len, bool write) {
  const uint32_t ml = match_len ? match_len - 4 : 0;
  if (write) out[op] = (uint8_t)((lit_len < 15 ? lit_len : 15) << 4 | (ml < 15 ? ml : 15));
  op++;
  return lit_len >= 15 ? put_length_bytes(out, op, lit_len - 15, write) : op;
}
// The offset and match-length bytes after the sequence's literals, at out[op]; returns the position after them.
HS_HD uint32_t put_match(uint8_t* out, uint32_t op, uint32_t offset, uint32_t match_len, bool write) {
  if (write) {
    out[op] = (uint8_t)offset;
    out[op + 1] = (uint8_t)(offset >> 8);
  }
  op += 2;
  return match_len - 4 >= 15 ? put_length_bytes(out, op, match_len - 4 - 15, write) : op;
}

// ---- serial decoding (the host build of the tests) -------------------------------------------------------------------------
// The block src[ip, n) into dst from `out` (its start) with capacity cap; out ends past the block's output.
inline uint32_t decode_block_serial(const uint8_t* src, uint32_t ip, uint32_t n, uint8_t* dst, uint32_t& out, uint32_t cap) {
  const uint32_t start = out;
  for (bool last = false; !last;) {
    Seq s;
    const uint32_t e = parse_sequence(src, n, ip, out, start, cap, s, last);
    if (e) return e;
    for (uint32_t j = 0; j < s.lit_len; j++) dst[s.out + j] = src[s.lit_src + j];
    const uint32_t p = s.out + s.lit_len;
    for (uint32_t j = 0; j < s.match_len; j++) dst[p + j] = dst[p - s.offset + j];  // byte by byte: overlap repeats
  }
  return LZ4_OK;
}

// A page body of codec 5 or 7 into dst[0, dst_len).
inline uint32_t decode_page_serial(uint32_t codec, const uint8_t* src, uint32_t n, uint8_t* dst, uint32_t dst_len) {
  if (codec == kCodecLz4) {
    HadoopCursor c{0, 0, 0};
    uint32_t out = 0, cs = 0, cl = 0, r;
    while ((r = hadoop_next(src, n, out, dst_len, c, cs, cl)) == HADOOP_CHUNK) {
      // the chunk's output starts at `out`: its matches never reach before it
      if (decode_block_serial(src, cs, cs + cl, dst, out, c.group_end)) break;
    }
    if (r == HADOOP_DONE) return LZ4_OK;
  }
  uint32_t out = 0;
  const uint32_t e = decode_block_serial(src, 0, n, dst, out, dst_len);
  return e ? e : out == dst_len ? LZ4_OK : LZ4_OUTPUT_SHORT;
}

}  // namespace lz4
}  // namespace hs
