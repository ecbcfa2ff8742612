// deflate.h -- the per-stream pieces of the GZIP page compressor (deflate.cu): length-limited Huffman codes, the header of a
// dynamic block, the gzip member's header and trailer, and the worst-case sizes.  __host__ __device__ like inflate.h, whose
// tables, code-length order and CRC-32 helpers it shares: lane 0 of a warp runs them on the GPU, and
// tests/native/index_codecs.cu runs the same code on the CPU.
//
// A page body becomes one gzip member: kGzipHeader, then every 64 KB fragment's DEFLATE blocks -- each fragment ends
// non-final and byte-aligned with an empty stored block (a sync flush), so the fragments compress independently and are
// concatenated as they are -- then an empty final block and the trailer (CRC-32, ISIZE).
#pragma once
#include "inflate.h"

namespace hs {
namespace gz {

constexpr uint32_t kLitCodes = 286, kDistCodes = 30;      // the symbols a block may use
constexpr int kCodeLenLimit = 7;                          // the code-length code's longest code
constexpr uint8_t kGzipHeader[10] = {0x1f, 0x8b, 8, 0, 0, 0, 0, 0, 0, 0xff};  // no optional fields, MTIME 0, OS unknown
constexpr uint8_t kFinalBlock[2] = {0x03, 0x00};         // BFINAL=1, fixed Huffman, end-of-block
constexpr uint32_t kSyncFlush = 0xffff0000u;              // LEN 0000, NLEN ffff of the sync flush's empty stored block
// the code-length code's lengths are stored in the order 16 17 18 0 8 7 9 6 10 5 11 4 12 3 13 2 14 1 15
HS_HD int cl_order(int i) { return i < 3 ? 16 + i : i == 3 ? 0 : ((i - 4) & 1) ? 8 - ((i - 3) >> 1) : 8 + ((i - 4) >> 1); }

// ---- worst-case sizes ----------------------------------------------------------------------------------------------------
// A fragment of len bytes is never larger than its stored form: stored blocks of at most 65 535 bytes (5 bytes of header
// each, the first starting byte-aligned), then the sync flush (5 bytes).
HS_HD uint64_t deflate_fragment_bound(uint64_t len) { return len + 5 * (len > 65535 ? (len + 65534) / 65535 : 1) + 5; }
// the member of a body of len bytes cut into fragments of `fragment` bytes
HS_HD uint64_t gzip_body_bound(uint64_t len, uint64_t fragment) {
  const uint64_t full = len / fragment, rest = len % fragment;
  return sizeof(kGzipHeader) + full * deflate_fragment_bound(fragment) + (rest ? deflate_fragment_bound(rest) : 0) +
         sizeof(kFinalBlock) + 8;
}

// ---- bit writer (LSB first, as DEFLATE packs bits) -----------------------------------------------------------------------
struct BitWriter {
  uint8_t* out;
  uint32_t pos;  // bytes written
  uint64_t acc;  // pending bits
  uint32_t cnt;

  HS_HD void put(uint32_t v, int n) {  // n <= 32
    acc |= (uint64_t)v << cnt;
    cnt += n;
    while (cnt >= 8) {
      out[pos++] = (uint8_t)acc;
      acc >>= 8;
      cnt -= 8;
    }
  }
  HS_HD void align() {
    if (cnt) put(0, 8 - cnt);
  }
};

// ---- length-limited Huffman codes ------------------------------------------------------------------------------------------
HS_HD void sift_down(uint32_t* key, int r, int size) {
  for (;;) {
    int c = 2 * r + 1;
    if (c >= size) return;
    if (c + 1 < size && key[c + 1] > key[c]) c++;
    if (key[r] >= key[c]) return;
    const uint32_t t = key[r];
    key[r] = key[c];
    key[c] = t;
    r = c;
  }
}

// lens[0, n) for the frequencies freq[0, n): a Huffman code whose lengths are capped at `limit` and fixed up so that the
// code stays complete (Kraft sum 1).  Every code has at least two symbols: a set with fewer gets symbols of frequency 0,
// lowest index first, so decoders never meet the one-code special case.  Ties break by symbol index, so the result depends
// on the frequencies alone.  work: 5 n uint32.  Needs 2 <= n <= min(512, 2^limit), frequencies below
// 2^23 and their sum below 2^32 (a fragment's counts are at most 65 537).
HS_HD void huffman_lengths(const uint32_t* freq, int n, int limit, uint8_t* lens, uint32_t* work) {
  uint32_t* key = work;  // leaves, (freq << 9 | symbol), sorted ascending
  int m = 0;
  for (int s = 0; s < n; s++) {
    lens[s] = 0;
    if (freq[s]) key[m++] = freq[s] << 9 | (uint32_t)s;
  }
  for (int s = 0; m < 2 && s < n; s++)
    if (!freq[s]) key[m++] = (uint32_t)s;
  for (int i = m / 2 - 1; i >= 0; i--) sift_down(key, i, m);  // heap sort
  for (int size = m - 1; size > 0; size--) {
    const uint32_t t = key[0];
    key[0] = key[size];
    key[size] = t;
    sift_down(key, 0, size);
  }
  // Huffman's tree by two queues: leaves 0..m-1 in order, internal nodes m..2m-2 in the order they are made
  uint32_t* weight = work + m;         // [2m - 1], then depths
  uint32_t* parent = work + 3 * m;     // [2m - 1]
  for (int i = 0; i < m; i++) weight[i] = key[i] >> 9;
  int li = 0, ii = m;
  for (int next = m; next < 2 * m - 1; next++) {
    uint32_t w = 0;
    for (int k = 0; k < 2; k++) {
      const int c = (li < m && (ii >= next || weight[li] <= weight[ii])) ? li++ : ii++;
      w += weight[c];
      parent[c] = (uint32_t)next;
    }
    weight[next] = w;
  }
  weight[2 * m - 2] = 0;  // depths, from the root down (a parent is made after its children)
  for (int i = 2 * m - 3; i >= 0; i--) weight[i] = weight[parent[i]] + 1;
  // lengths per count, capped; then codes move down one level at a time until the Kraft sum is exactly 1
  uint32_t count[16] = {0};
  for (int i = 0; i < m; i++) count[weight[i] < (uint32_t)limit ? weight[i] : limit]++;
  uint32_t total = 0;
  for (int l = 1; l <= limit; l++) total += count[l] << (limit - l);
  while (total != (1u << limit)) {
    count[limit]--;
    for (int l = limit - 1; l > 0; l--) {
      if (count[l]) {
        count[l]--;
        count[l + 1] += 2;
        break;
      }
    }
    total--;
  }
  // the longest codes go to the least frequent symbols
  int j = 0;
  for (int l = limit; l > 0; l--)
    for (uint32_t k = 0; k < count[l]; k++) lens[key[j++] & 511] = (uint8_t)l;
}

// Canonical codes for lens[0, n), bit-reversed: the value to put() LSB first.
HS_HD void huffman_codes(const uint8_t* lens, int n, uint16_t* codes) {
  uint32_t count[kMaxBits + 1] = {0}, next[kMaxBits + 1];
  for (int s = 0; s < n; s++) count[lens[s]]++;
  count[0] = 0;
  uint32_t code = 0;
  for (int l = 1; l <= kMaxBits; l++) {
    code = (code + count[l - 1]) << 1;
    next[l] = code;
  }
  for (int s = 0; s < n; s++) {
    const int l = lens[s];
    uint32_t r = 0;
    if (l) {
      const uint32_t c = next[l]++;
      for (int b = 0; b < l; b++) r |= ((c >> b) & 1u) << (l - 1 - b);
    }
    codes[s] = (uint16_t)r;
  }
}

// ---- the header of a dynamic block ---------------------------------------------------------------------------------------
// The code lengths, run-length coded with the code-length code: symbols 0..15 are lengths, 16 repeats the previous length
// 3..6 times (2 extra bits), 17 and 18 give 3..10 and 11..138 zeros (3 and 7 extra bits).  items: symbol | extra << 5.
HS_HD int rle_lengths(const uint8_t* lens, int n, uint16_t* items) {
  int k = 0;
  for (int i = 0; i < n;) {
    const uint8_t v = lens[i];
    int run = 1;
    while (i + run < n && lens[i + run] == v) run++;
    int r = run;
    if (v == 0) {
      for (; r >= 11; r -= r < 138 ? r : 138) items[k++] = (uint16_t)(18 | ((r < 138 ? r : 138) - 11) << 5);
      if (r >= 3) {
        items[k++] = (uint16_t)(17 | (r - 3) << 5);
        r = 0;
      }
    } else {
      items[k++] = v;
      for (r--; r >= 3; r -= r < 6 ? r : 6) items[k++] = (uint16_t)(16 | ((r < 6 ? r : 6) - 3) << 5);
    }
    for (; r > 0; r--) items[k++] = v;
    i += run;
  }
  return k;
}
HS_HD int cl_extra_bits(int sym) { return sym == 16 ? 2 : sym == 17 ? 3 : sym == 18 ? 7 : 0; }

struct DynamicHeader {
  uint16_t nlit, ndist, ncl, nitems;
  uint8_t cl_lens[kCodeLenSyms];
  uint16_t cl_codes[kCodeLenSyms];
  uint8_t seq[kLitCodes + kDistCodes];    // the literal/length lengths, then the distance lengths
  uint16_t items[kLitCodes + kDistCodes];
};

// The header for lit_lens[0, 286) and dist_lens[0, 30); work: 5 * 19 uint32.  Returns its size in bits (after BTYPE).
HS_HD uint32_t plan_dynamic_header(const uint8_t* lit_lens, const uint8_t* dist_lens, DynamicHeader& h, uint32_t* work) {
  int nlit = kLitCodes, ndist = kDistCodes;
  while (nlit > 257 && lit_lens[nlit - 1] == 0) nlit--;
  while (ndist > 1 && dist_lens[ndist - 1] == 0) ndist--;
  for (int s = 0; s < nlit; s++) h.seq[s] = lit_lens[s];
  for (int d = 0; d < ndist; d++) h.seq[nlit + d] = dist_lens[d];
  const int nitems = rle_lengths(h.seq, nlit + ndist, h.items);
  uint32_t freq[kCodeLenSyms] = {0};
  for (int i = 0; i < nitems; i++) freq[h.items[i] & 31]++;
  huffman_lengths(freq, kCodeLenSyms, kCodeLenLimit, h.cl_lens, work);
  huffman_codes(h.cl_lens, kCodeLenSyms, h.cl_codes);
  int ncl = kCodeLenSyms;
  while (ncl > 4 && h.cl_lens[cl_order(ncl - 1)] == 0) ncl--;
  h.nlit = (uint16_t)nlit;
  h.ndist = (uint16_t)ndist;
  h.ncl = (uint16_t)ncl;
  h.nitems = (uint16_t)nitems;
  uint32_t bits = 5 + 5 + 4 + 3 * ncl;
  for (int i = 0; i < nitems; i++) bits += h.cl_lens[h.items[i] & 31] + cl_extra_bits(h.items[i] & 31);
  return bits;
}

HS_HD void write_dynamic_header(BitWriter& bw, const DynamicHeader& h) {
  bw.put(h.nlit - 257u, 5);
  bw.put(h.ndist - 1u, 5);
  bw.put(h.ncl - 4u, 4);
  for (int i = 0; i < h.ncl; i++) bw.put(h.cl_lens[cl_order(i)], 3);
  for (int i = 0; i < h.nitems; i++) {
    const int s = h.items[i] & 31;
    bw.put(h.cl_codes[s], h.cl_lens[s]);
    if (cl_extra_bits(s)) bw.put(h.items[i] >> 5, cl_extra_bits(s));
  }
}

// ---- symbols ---------------------------------------------------------------------------------------------------------------
HS_HD int floor_log2(uint32_t x) {
  int l = 0;
  while (x >>= 1) l++;
  return l;
}
// length 3..258 -> index i of symbol 257 + i (len_base / len_extra in inflate.h are its inverse)
HS_HD int length_index(uint32_t len) {
  const uint32_t x = len - 3;
  if (x < 8) return (int)x;
  if (len == 258) return 28;
  const int e = floor_log2(x) - 2;
  return 4 * e + 4 + (int)((x >> e) & 3);
}
// distance 1..32768 -> distance symbol
HS_HD int distance_symbol(uint32_t d) {
  const uint32_t x = d - 1;
  if (x < 4) return (int)x;
  const int e = floor_log2(x) - 1;
  return 2 * e + 2 + (int)((x >> e) & 1);
}
HS_HD uint8_t fixed_lit_len(int s) { return s < 144 ? 8 : s < 256 ? 9 : s < 280 ? 7 : 8; }
// the fixed literal/length code of s (RFC 1951 3.2.6), bit-reversed as huffman_codes gives it
HS_HD uint16_t fixed_lit_code(int s) {
  const uint32_t c = s < 144 ? 0x30u + s : s < 256 ? 0x190u + (s - 144) : s < 280 ? (uint32_t)(s - 256) : 0xc0u + (s - 280);
  const int l = fixed_lit_len(s);
  uint32_t r = 0;
  for (int b = 0; b < l; b++) r |= ((c >> b) & 1u) << (l - 1 - b);
  return (uint16_t)r;
}

// ---- the member around the fragments -------------------------------------------------------------------------------------
// crc_of_fragments: XOR over fragments of crc32_multmodp(crc32_x8n(bytes after the fragment), its CRC with no pre- or
// post-inversion); len: the body's length.  out: 10 bytes of trailer (final block, CRC-32, ISIZE).
HS_HD void gzip_trailer(uint32_t crc_of_fragments, uint64_t len, uint8_t* out) {
  const uint32_t crc = crc32_finish(crc_of_fragments, (uint32_t)len), isize = (uint32_t)len;
  out[0] = 0x03;  // kFinalBlock
  out[1] = 0x00;
  for (int i = 0; i < 4; i++) {
    out[2 + i] = (uint8_t)(crc >> (8 * i));
    out[6 + i] = (uint8_t)(isize >> (8 * i));
  }
}
// the 5 header bytes of a non-final stored block of len <= 65 535 bytes, at a byte boundary (the sync flush is one of len 0)
HS_HD uint32_t put_stored_header(uint8_t* out, uint32_t len) {
  out[0] = 0;
  out[1] = (uint8_t)len;
  out[2] = (uint8_t)(len >> 8);
  out[3] = (uint8_t)~len;
  out[4] = (uint8_t)(~len >> 8);
  return 5;
}

}  // namespace gz
}  // namespace hs
