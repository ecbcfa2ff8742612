// string_match.h -- the string patterns of filter terms that are not a range of values: Spark's EndsWith, Contains and
// Like.  __host__ __device__ like inflate.h and lz4_block.h: k_pattern_mask (read_side.cu) runs it one thread per row, and
// tests/native/filter_terms.cu runs the same code on the CPU against Python's re.
//
// A pattern is compiled on the host (predicates.h: compile_pattern) into items and segments.  An item is one literal byte
// (0..255) or kAnyChar, LIKE's `_`: one UTF-8 character, whose length the lead byte gives.  The segments are the runs of
// items between LIKE's `%`s.  Without a `%` the one segment must span the whole value; otherwise the first segment is
// anchored at the start, the last at the end, and every segment between them is placed at its leftmost match after the
// previous one.  A segment consumes a fixed number of characters from any start, so its end grows with its start and the
// leftmost placement leaves the most room for the rest: the greedy walk is exact and never backtracks.  Segments without
// `_` are searched byte by byte with Knuth-Morris-Pratt (EndsWith and Contains compare bytes, as UTF8String does), so a
// value of n bytes costs O(n + pattern length) whatever the pattern (the segments' searches cover the value once).
// Middle segments with `_` are tried at every character start, O(n x segment length) in the worst case; that bound is the
// one pattern shape (a LIKE with `_` between two `%`s) whose cost grows with the product.  On values that are not valid
// UTF-8, LIKE's `_` follows the lead bytes and may differ from Spark, which matches the decoded String.
#pragma once
#include <cstdint>

#ifdef __CUDACC__
#define HS_HD __host__ __device__ __forceinline__
#else
#define HS_HD inline
#endif

namespace hs {

constexpr uint16_t kAnyChar = 256;  // LIKE's `_` among the items

// items[off, off + len); any_char: the segment holds a `_`
struct PatSeg {
  uint32_t off, len;
  int32_t any_char;
};

// bytes of the UTF-8 character whose lead byte is b (a stray continuation byte counts as one)
HS_HD uint32_t utf8_char_len(uint8_t b) { return b < 0xc0 ? 1u : (b < 0xe0 ? 2u : (b < 0xf0 ? 3u : 4u)); }

// the segment matched forward from s[i]: the position after it, or -1
HS_HD int64_t match_forward(const uint8_t* s, int64_t n, int64_t i, const uint16_t* items, const PatSeg& g) {
  for (uint32_t k = 0; k < g.len; k++) {
    const uint16_t it = items[g.off + k];
    if (i >= n) return -1;
    if (it == kAnyChar) {
      i += utf8_char_len(s[i]);
      if (i > n) return -1;
    } else if (s[i++] != it) {
      return -1;
    }
  }
  return i;
}

// the segment matched backward so that it ends at s[e]: its start, or -1
HS_HD int64_t match_backward(const uint8_t* s, int64_t e, const uint16_t* items, const PatSeg& g) {
  for (uint32_t k = g.len; k-- > 0;) {
    const uint16_t it = items[g.off + k];
    if (e <= 0) return -1;
    if (it == kAnyChar) {
      e--;
      while (e > 0 && (s[e] & 0xc0) == 0x80) e--;
    } else if (s[--e] != it) {
      return -1;
    }
  }
  return e;
}

// The end of the leftmost occurrence of the literal segment g (no `_`, len >= 1) inside s[from, to), or -1: KMP with
// fail[g.off + j], the longest proper border of the segment's first j + 1 items.
HS_HD int64_t find_literal(const uint8_t* s, int64_t from, int64_t to, const uint16_t* items, const int32_t* fail, const PatSeg& g) {
  uint32_t k = 0;  // items of g matched so far
  for (int64_t i = from; i < to; i++) {
    while (k > 0 && s[i] != items[g.off + k]) k = (uint32_t)fail[g.off + k - 1];
    if (s[i] == items[g.off + k] && ++k == g.len) return i + 1;
  }
  return -1;
}

// Does the value s[0, n) match the compiled pattern (nseg >= 1 segments; whole: no `%`, one segment spanning the value)?
// fail: the segments' KMP tables (predicates.h: compile_pattern).
HS_HD bool pattern_matches(const uint8_t* s, int64_t n, const uint16_t* items, const int32_t* fail, const PatSeg* segs, int nseg,
                           bool whole) {
  if (whole) return match_forward(s, n, 0, items, segs[0]) == n;
  int64_t p = match_forward(s, n, 0, items, segs[0]);
  if (p < 0) return false;
  const int64_t q = match_backward(s, n, items, segs[nseg - 1]);
  if (q < p) return false;  // also q < 0
  for (int g = 1; g + 1 < nseg; g++) {
    const PatSeg seg = segs[g];
    if (seg.len == 0) continue;
    int64_t e = -1;
    if (!seg.any_char) {
      e = find_literal(s, p, q, items, fail, seg);
    } else {
      for (int64_t i = p; i + (int64_t)seg.len <= q; i += utf8_char_len(s[i])) {  // every item takes at least one byte
        e = match_forward(s, q, i, items, seg);
        if (e >= 0) break;
      }
    }
    if (e < 0) return false;
    p = e;
  }
  return true;
}

}  // namespace hs
