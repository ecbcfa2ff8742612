// inflate.h -- GZIP members (RFC 1952) and the DEFLATE streams inside them (RFC 1951): the per-stream pieces of the
// GZIP page decoder.  __host__ __device__ like thrift_compact.h: the GPU kernel (inflate.cu) runs them in one lane per
// page, and tests/native/inflate.cu runs the same code on the CPU against zlib.
//
// A Parquet GZIP page body is one or more gzip members back to back.  inflate_member decodes one member -- header, blocks,
// trailer -- into dst; the caller checks the member's CRC-32 (crc32_piece / crc32_finish: one piece per lane on the GPU)
// and calls it again while input is left.  Every check returns an InflateError; no check reads outside
// [src, src + n_src) or writes outside [dst, dst + dst_len), and every loop ends (each block consumes input, each symbol
// either ends its block or produces output, and both are bounded).
#pragma once
#include <cstdint>

#ifdef __CUDACC__
#define HS_HD __host__ __device__ __forceinline__
#else
#define HS_HD inline
#endif

namespace hs {
namespace gz {

enum InflateError : uint32_t {
  GZ_OK = 0,
  GZ_BAD_MAGIC = 1,        // not a gzip member (a zlib-wrapped or raw-deflate body lands here)
  GZ_BAD_METHOD = 2,       // CM != 8
  GZ_BAD_FLAGS = 3,        // reserved flag bits set
  GZ_HEADER_CRC = 4,       // FHCRC does not match the header
  GZ_STORED_LEN = 5,       // stored block: LEN != ~NLEN
  GZ_BLOCK_TYPE = 6,       // block type 3
  GZ_BAD_LENGTHS = 7,      // code-length set over-subscribed, incomplete, too many symbols, or without end-of-block
  GZ_BAD_SYMBOL = 8,       // literal/length 286-287, distance 30-31, or a code outside an incomplete set
  GZ_FAR_DISTANCE = 9,     // a match reaches before the start of the member's output
  GZ_OUTPUT_OVERRUN = 10,  // more output than the page's uncompressed size
  GZ_OUTPUT_SHORT = 11,    // less output than the page's uncompressed size
  GZ_TRUNCATED = 12,       // the stream runs past the compressed bytes
  GZ_CRC = 13,             // CRC-32 of the member's output differs from its trailer
  GZ_ISIZE = 14,           // ISIZE differs from the member's output length
  GZ_TRAILING = 15,        // bytes after a member that do not start a valid member
};

HS_HD const char* inflate_error_text(uint32_t e) {
  switch (e) {
    case GZ_BAD_MAGIC: return "not a gzip member (bad magic)";
    case GZ_BAD_METHOD: return "compression method is not deflate";
    case GZ_BAD_FLAGS: return "reserved header flag bits set";
    case GZ_HEADER_CRC: return "header CRC-16 mismatch";
    case GZ_STORED_LEN: return "stored block LEN does not match NLEN";
    case GZ_BLOCK_TYPE: return "invalid block type 3";
    case GZ_BAD_LENGTHS: return "invalid code-length set";
    case GZ_BAD_SYMBOL: return "invalid literal/length or distance symbol";
    case GZ_FAR_DISTANCE: return "distance reaches before the start of the output";
    case GZ_OUTPUT_OVERRUN: return "output longer than the page's uncompressed size";
    case GZ_OUTPUT_SHORT: return "output shorter than the page's uncompressed size";
    case GZ_TRUNCATED: return "stream runs past the compressed bytes";
    case GZ_CRC: return "CRC-32 mismatch";
    case GZ_ISIZE: return "ISIZE mismatch";
    case GZ_TRAILING: return "trailing bytes after the last member";
    default: return "ok";
  }
}

// ---- CRC-32 (the gzip / zlib polynomial, reflected 0xedb88320) --------------------------------------------------------
// table: 256 entries made by crc32_table_entry; crc is the running value with gzip's pre/post inversion applied by the caller
HS_HD uint32_t crc32_table_entry(uint32_t n) {
  uint32_t c = n;
  for (int k = 0; k < 8; k++) c = (c & 1) ? 0xedb88320u ^ (c >> 1) : c >> 1;
  return c;
}
HS_HD uint32_t crc32_raw(const uint32_t* table, uint32_t crc, const uint8_t* p, uint32_t n) {
  for (uint32_t i = 0; i < n; i++) crc = table[(crc ^ p[i]) & 0xffu] ^ (crc >> 8);
  return crc;
}
// a * b modulo the CRC polynomial (reflected bit order: bit 31 is x^0)
HS_HD uint32_t crc32_multmodp(uint32_t a, uint32_t b) {
  uint32_t m = 1u << 31, p = 0;
  for (;;) {
    if (a & m) {
      p ^= b;
      if ((a & (m - 1)) == 0) break;
    }
    m >>= 1;
    b = (b & 1) ? (b >> 1) ^ 0xedb88320u : b >> 1;
  }
  return p;
}
// x^(8 n) modulo the polynomial: what appending n zero bytes multiplies a raw CRC by
HS_HD uint32_t crc32_x8n(uint64_t n) {
  uint32_t p = 1u << 31, sq = 1u << 23;  // sq = x^8, squared at every bit of n
  while (n) {
    if (n & 1) p = crc32_multmodp(sq, p);
    sq = crc32_multmodp(sq, sq);
    n >>= 1;
  }
  return p;
}
// gzip's CRC-32 of p[0, n)
HS_HD uint32_t crc32_of(const uint32_t* table, const uint8_t* p, uint32_t n) { return ~crc32_raw(table, 0xffffffffu, p, n); }
// the same without a table (short inputs: header CRCs)
HS_HD uint32_t crc32_bitwise(uint32_t crc, const uint8_t* p, uint32_t n) {
  crc = ~crc;
  for (uint32_t i = 0; i < n; i++) {
    crc ^= p[i];
    for (int k = 0; k < 8; k++) crc = (crc & 1) ? 0xedb88320u ^ (crc >> 1) : crc >> 1;
  }
  return ~crc;
}

// ---- Huffman tables ----------------------------------------------------------------------------------------------------
// Codes up to root_bits long are looked up in one step: root[bits] = symbol << 4 | length.  Longer codes (rare: they belong
// to rare symbols) leave their root entries 0 and are decoded canonically from count[] and sym[], as RFC 1951 defines them.
constexpr int kLitRootBits = 10, kDistRootBits = 8, kMaxBits = 15;
constexpr int kLitSyms = 288, kDistSyms = 32, kCodeLenSyms = 19;

struct Huffman {
  uint16_t* root;
  uint16_t* count;  // [kMaxBits + 1]: codes of each length
  uint16_t* sym;    // symbols in canonical order
  int root_bits;
};

// A warp's (or the host's) working set: one per stream in flight.
struct InflateTables {
  uint16_t lit_root[1 << kLitRootBits];
  uint16_t dist_root[1 << kDistRootBits];  // also the code-length code's table
  uint16_t lit_count[kMaxBits + 1], dist_count[kMaxBits + 1];
  uint16_t lit_sym[kLitSyms], dist_sym[kDistSyms];
  uint8_t lens[kLitSyms + kDistSyms];
};

// Builds h from lens[0, n).  Returns false for an over-subscribed set, and for an incomplete one unless allow_incomplete and
// the set is a single code of length 1 (RFC 1951 3.2.7; zlib's rule).  An empty set is accepted when allow_empty.
HS_HD bool build_huffman(Huffman& h, const uint8_t* lens, int n, bool allow_incomplete, bool allow_empty) {
  for (int l = 0; l <= kMaxBits; l++) h.count[l] = 0;
  for (int s = 0; s < n; s++) h.count[lens[s]]++;
  h.count[0] = 0;
  int left = 1, used = 0;
  for (int l = 1; l <= kMaxBits; l++) {
    left <<= 1;
    left -= h.count[l];
    if (left < 0) return false;
    used += h.count[l];
  }
  if (used == 0) {
    if (!allow_empty) return false;
  } else if (left > 0 && !(allow_incomplete && used == 1 && h.count[1] == 1)) {
    return false;
  }
  uint16_t offs[kMaxBits + 2];
  offs[1] = 0;
  for (int l = 1; l <= kMaxBits; l++) offs[l + 1] = offs[l] + h.count[l];
  const int root_size = 1 << h.root_bits;
  for (int i = 0; i < root_size; i++) h.root[i] = 0;
  uint32_t code = 0;  // canonical code of the first symbol of each length, MSB first
  uint32_t next[kMaxBits + 1];
  for (int l = 1; l <= kMaxBits; l++) {
    code = (code + h.count[l - 1]) << 1;
    next[l] = code;
  }
  for (int s = 0; s < n; s++) {
    const int l = lens[s];
    if (l == 0) continue;
    h.sym[offs[l]++] = (uint16_t)s;
    const uint32_t c = next[l]++;
    if (l > h.root_bits) continue;
    uint32_t r = 0;  // the code's bits in stream order (LSB first)
    for (int b = 0; b < l; b++) r |= ((c >> b) & 1u) << (l - 1 - b);
    for (uint32_t i = r; i < (uint32_t)root_size; i += 1u << l) h.root[i] = (uint16_t)(s << 4 | l);
  }
  return true;
}

// ---- bit reader ----------------------------------------------------------------------------------------------------------
// A 64-bit buffer, refilled byte by byte from [src, src + n).  Past n it shifts in zeros and counts them: a stream that
// needs them is truncated, which the block and member loops check (consumed() > 8 n).
struct BitReader {
  const uint8_t* src;
  uint32_t n, pos;  // pos: bytes taken into the buffer, real or zero
  uint64_t buf;
  uint32_t cnt;

  HS_HD void refill() {
    while (cnt <= 56) {
      const uint64_t b = pos < n ? src[pos] : 0u;
      buf |= b << cnt;
      pos++;
      cnt += 8;
    }
  }
  HS_HD uint32_t peek(int k) const { return (uint32_t)(buf & ((1ull << k) - 1)); }
  HS_HD void drop(int k) {
    buf >>= k;
    cnt -= k;
  }
  HS_HD uint32_t bits(int k) {  // k <= 32, buffer refilled before
    const uint32_t v = peek(k);
    drop(k);
    return v;
  }
  HS_HD uint64_t consumed() const { return (uint64_t)pos * 8 - cnt; }
  HS_HD bool overrun() const { return consumed() > (uint64_t)n * 8; }
  // to the next byte boundary; returns the byte position there
  HS_HD uint32_t align() {
    drop(cnt & 7);
    return pos - cnt / 8;
  }
  HS_HD void seek(uint32_t p) {
    pos = p;
    buf = 0;
    cnt = 0;
  }
};

// one symbol of h; needs 15 bits in the buffer.  Returns -1 for a code outside the set.
HS_HD int decode_symbol(BitReader& br, const Huffman& h) {
  const uint32_t e = h.root[br.peek(h.root_bits)];
  if (e & 15) {
    br.drop(e & 15);
    return (int)(e >> 4);
  }
  // canonical decode, one bit at a time (puff's loop): codes longer than the root, or none at all
  uint32_t code = 0, first = 0, index = 0;
  const uint32_t v = br.peek(kMaxBits);
  for (int l = 1; l <= kMaxBits; l++) {
    code |= (v >> (l - 1)) & 1u;
    const uint32_t count = h.count[l];
    if (code - first < count) {
      br.drop(l);
      return h.sym[index + (code - first)];
    }
    index += count;
    first = (first + count) << 1;
    code <<= 1;
  }
  return -1;
}

// RFC 1951 3.2.5: base and extra bits of length symbols 257..285 (index s - 257) and distance symbols 0..29, by formula
HS_HD uint32_t len_extra(int i) { return i < 8 || i == 28 ? 0u : (uint32_t)(i - 4) >> 2; }
HS_HD uint32_t len_base(int i) { return i < 8 ? 3u + i : i == 28 ? 258u : ((4u + (i & 3)) << len_extra(i)) + 3u; }
HS_HD uint32_t dist_extra(int d) { return d < 4 ? 0u : (uint32_t)(d - 2) >> 1; }
HS_HD uint32_t dist_base(int d) { return d < 4 ? 1u + d : ((2u + (d & 1)) << dist_extra(d)) + 1u; }

// ---- one member ----------------------------------------------------------------------------------------------------------
struct Member {
  uint32_t out_begin, out_end;  // the member's output in dst
  uint32_t crc, isize;          // from its trailer
};

// Header at src[p]; on success p is the first byte of the deflate stream.
HS_HD uint32_t parse_header(const uint8_t* src, uint32_t n, uint32_t& p) {
  const uint32_t h0 = p;
  if (n - p < 2) return GZ_TRUNCATED;
  if (src[p] != 0x1f || src[p + 1] != 0x8b) return GZ_BAD_MAGIC;
  if (n - p < 10) return GZ_TRUNCATED;
  if (src[p + 2] != 8) return GZ_BAD_METHOD;
  const uint8_t flg = src[p + 3];
  if (flg & 0xe0) return GZ_BAD_FLAGS;
  p += 10;
  if (flg & 4) {  // FEXTRA
    if (n - p < 2) return GZ_TRUNCATED;
    const uint32_t xlen = src[p] | (uint32_t)src[p + 1] << 8;
    p += 2;
    if (n - p < xlen) return GZ_TRUNCATED;
    p += xlen;
  }
  for (int z = 0; z < 2; z++) {  // FNAME, FCOMMENT: zero-terminated
    if (!(flg & (8 << z))) continue;
    while (p < n && src[p] != 0) p++;
    if (p >= n) return GZ_TRUNCATED;
    p++;
  }
  if (flg & 2) {  // FHCRC: the low 16 bits of the CRC-32 of the header so far
    if (n - p < 2) return GZ_TRUNCATED;
    const uint32_t want = src[p] | (uint32_t)src[p + 1] << 8;
    if ((crc32_bitwise(0, src + h0, p - h0) & 0xffffu) != want) return GZ_HEADER_CRC;
    p += 2;
  }
  return GZ_OK;
}

HS_HD void fixed_tables(InflateTables& t, Huffman& lit, Huffman& dist) {
  for (int s = 0; s < kLitSyms; s++) t.lens[s] = s < 144 ? 8 : s < 256 ? 9 : s < 280 ? 7 : 8;
  build_huffman(lit, t.lens, kLitSyms, false, false);
  for (int s = 0; s < kDistSyms; s++) t.lens[s] = 5;
  build_huffman(dist, t.lens, kDistSyms, false, false);
}

// a dynamic block's header: HLIT, HDIST, HCLEN, the code-length code, then both code-length sets
HS_HD uint32_t dynamic_tables(BitReader& br, InflateTables& t, Huffman& lit, Huffman& dist) {
  br.refill();
  const int nlen = (int)br.bits(5) + 257, ndist = (int)br.bits(5) + 1, ncode = (int)br.bits(4) + 4;
  if (nlen > 286 || ndist > 30) return GZ_BAD_LENGTHS;
  // the code-length code's lengths, 3 bits each, in the order 16 17 18 0 8 7 9 6 10 5 11 4 12 3 13 2 14 1 15
  uint8_t cl[kCodeLenSyms];
  br.refill();
  const uint64_t raw = br.buf;  // 57 bits or more: all 19 fields
  br.drop(3 * ncode);
  for (int i = 0; i < kCodeLenSyms; i++) {
    const int sym = i < 3 ? 16 + i : i == 3 ? 0 : ((i - 4) & 1) ? 8 - ((i - 3) >> 1) : 8 + ((i - 4) >> 1);
    cl[sym] = i < ncode ? (uint8_t)((raw >> (3 * i)) & 7u) : (uint8_t)0;
  }
  Huffman clh{t.dist_root, t.dist_count, t.dist_sym, 7};
  if (!build_huffman(clh, cl, kCodeLenSyms, false, false)) return GZ_BAD_LENGTHS;
  int i = 0;
  while (i < nlen + ndist) {
    br.refill();
    if (br.overrun()) return GZ_TRUNCATED;
    const int s = decode_symbol(br, clh);
    if (s < 0) return GZ_BAD_LENGTHS;
    if (s < 16) {
      t.lens[i++] = (uint8_t)s;
      continue;
    }
    uint8_t v = 0;
    int rep;
    if (s == 16) {
      if (i == 0) return GZ_BAD_LENGTHS;
      v = t.lens[i - 1];
      rep = 3 + (int)br.bits(2);
    } else if (s == 17) {
      rep = 3 + (int)br.bits(3);
    } else {
      rep = 11 + (int)br.bits(7);
    }
    if (i + rep > nlen + ndist) return GZ_BAD_LENGTHS;
    while (rep--) t.lens[i++] = v;
  }
  if (t.lens[256] == 0) return GZ_BAD_LENGTHS;  // no end-of-block code
  if (!build_huffman(lit, t.lens, nlen, true, false)) return GZ_BAD_LENGTHS;
  // the distance set may be empty (a block of literals only) or a single code; it overwrites the code-length code
  if (!build_huffman(dist, t.lens + nlen, ndist, true, true)) return GZ_BAD_LENGTHS;
  return GZ_OK;
}

// The blocks of the deflate stream at src[p] (after a member header), then the trailer: dst[out, ..) gets the output.  On
// success p is past the trailer, out past the output, and m holds what the caller checks: the CRC-32 over
// dst[m.out_begin, m.out_end) against m.crc.  ISIZE is checked here.
HS_HD uint32_t inflate_blocks(BitReader& br, uint8_t* dst, uint32_t dst_len, uint32_t& out, InflateTables& t, Member& m) {
  const uint8_t* src = br.src;
  const uint32_t n = br.n;
  Huffman lit{t.lit_root, t.lit_count, t.lit_sym, kLitRootBits};
  Huffman dist{t.dist_root, t.dist_count, t.dist_sym, kDistRootBits};
  bool last = false;
  while (!last) {
    br.refill();
    if (br.overrun()) return GZ_TRUNCATED;
    last = br.bits(1) != 0;
    const uint32_t type = br.bits(2);
    if (type == 3) return GZ_BLOCK_TYPE;
    if (type == 0) {  // stored: LEN, NLEN at the next byte boundary, then LEN bytes
      uint32_t q = br.align();
      if (q > n || n - q < 4) return GZ_TRUNCATED;
      const uint32_t len = src[q] | (uint32_t)src[q + 1] << 8, nlen = src[q + 2] | (uint32_t)src[q + 3] << 8;
      if (len != (~nlen & 0xffffu)) return GZ_STORED_LEN;
      q += 4;
      if (n - q < len) return GZ_TRUNCATED;
      if (len > dst_len - out) return GZ_OUTPUT_OVERRUN;
      for (uint32_t j = 0; j < len; j++) dst[out + j] = src[q + j];
      out += len;
      br.seek(q + len);
      continue;
    }
    if (type == 1) {
      fixed_tables(t, lit, dist);
    } else {
      const uint32_t e = dynamic_tables(br, t, lit, dist);
      if (e) return e;
    }
    for (;;) {
      br.refill();  // 57+ bits: a length code and its extra bits (15 + 5), a distance code and its extra bits (15 + 13)
      const int s = decode_symbol(br, lit);
      if ((unsigned)s < 256u) {
        if (out >= dst_len) return GZ_OUTPUT_OVERRUN;
        dst[out++] = (uint8_t)s;
        continue;
      }
      if (s == 256) break;
      if (s < 0 || s > 285) return GZ_BAD_SYMBOL;
      const uint32_t len = len_base(s - 257) + br.bits(len_extra(s - 257));
      const int ds = decode_symbol(br, dist);
      if (ds < 0 || ds >= 30) return GZ_BAD_SYMBOL;
      const uint32_t d = dist_base(ds) + br.bits(dist_extra(ds));
      if (d > out - m.out_begin) return GZ_FAR_DISTANCE;
      if (len > dst_len - out) return GZ_OUTPUT_OVERRUN;
      uint8_t* o = dst + out;
      const uint8_t* from = o - d;
      if (d >= 8) {  // chunks of 8: each chunk's loads come before its stores, and no chunk reads what it writes
        uint32_t j = 0;
        for (; j + 8 <= len; j += 8) {
          uint8_t r[8];
          for (int k = 0; k < 8; k++) r[k] = from[j + k];
          for (int k = 0; k < 8; k++) o[j + k] = r[k];
        }
        for (; j < len; j++) o[j] = from[j];
      } else {  // a short period: byte by byte repeats the pattern as the format asks
        for (uint32_t j = 0; j < len; j++) o[j] = from[j];
      }
      out += len;
    }
  }
  if (br.overrun()) return GZ_TRUNCATED;
  // trailer: CRC-32 and ISIZE at the next byte boundary
  const uint32_t q = br.align();
  if (q > n || n - q < 8) return GZ_TRUNCATED;
  m.crc = src[q] | (uint32_t)src[q + 1] << 8 | (uint32_t)src[q + 2] << 16 | (uint32_t)src[q + 3] << 24;
  m.isize = src[q + 4] | (uint32_t)src[q + 5] << 8 | (uint32_t)src[q + 6] << 16 | (uint32_t)src[q + 7] << 24;
  m.out_end = out;
  br.seek(q + 8);
  if (m.isize != m.out_end - m.out_begin) return GZ_ISIZE;
  return GZ_OK;
}

// One member at src[p]: header, blocks, trailer.  `first`: the page's first member (a later one that does not parse as a
// member is trailing garbage).  A check that fails after the stream ran out of bytes is reported as truncation: the bits it
// read past the end were zeros, not the stream.
HS_HD uint32_t inflate_member(const uint8_t* src, uint32_t n, uint32_t& p, bool first, uint8_t* dst, uint32_t dst_len,
                              uint32_t& out, InflateTables& t, Member& m) {
  const uint32_t e = parse_header(src, n, p);
  if (e) return first ? e : GZ_TRAILING;
  m.out_begin = out;
  BitReader br{src, n, 0, 0, 0};
  br.seek(p);
  uint32_t r = inflate_blocks(br, dst, dst_len, out, t, m);
  if (r && br.overrun()) r = GZ_TRUNCATED;
  p = br.pos;
  return r;
}

// The CRC-32 of dst[m.out_begin, m.out_end) in `parts` pieces: piece i's raw CRC (no inversions) is shifted past the bytes
// after it and the pieces are XORed (the CRC is linear), then gzip's initial value is shifted past the whole member.  The
// warp-parallel pass in inflate.cu computes exactly this with one piece per lane.
HS_HD uint32_t crc32_piece(const uint32_t* table, const uint8_t* p, uint32_t len, uint32_t parts, uint32_t i) {
  const uint32_t per = (len + parts - 1) / parts;
  const uint32_t lo = per * i < len ? per * i : len, hi = lo + per < len ? lo + per : len;
  return crc32_multmodp(crc32_x8n(len - hi), crc32_raw(table, 0u, p + lo, hi - lo));
}
HS_HD uint32_t crc32_finish(uint32_t xor_of_pieces, uint32_t len) {
  return ~(xor_of_pieces ^ crc32_multmodp(crc32_x8n(len), 0xffffffffu));
}

// The whole page body, serially (the host build of the tests): every member, its CRC-32 in `parts` pieces, the output length.
inline uint32_t inflate_gzip_serial(const uint8_t* src, uint32_t n, uint8_t* dst, uint32_t dst_len, InflateTables& t,
                                    const uint32_t* crc_table, uint32_t parts) {
  uint32_t p = 0, out = 0;
  for (bool first = true; first || p < n; first = false) {
    Member m{0, 0, 0, 0};
    const uint32_t e = inflate_member(src, n, p, first, dst, dst_len, out, t, m);
    if (e) return e;
    const uint32_t len = m.out_end - m.out_begin;
    uint32_t x = 0;
    for (uint32_t i = 0; i < parts; i++) x ^= crc32_piece(crc_table, dst + m.out_begin, len, parts, i);
    if (crc32_finish(x, len) != m.crc) return GZ_CRC;
  }
  return out == dst_len ? GZ_OK : GZ_OUTPUT_SHORT;
}

}  // namespace gz
}  // namespace hs
