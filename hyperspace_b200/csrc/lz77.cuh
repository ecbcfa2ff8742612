// lz77.cuh -- the match finder of the page compressors (snappy.cu, deflate.cu, lz4.cu): one warp parses one fragment
// (<= 64 KB) of a page body into sequences -- literals, then a back-reference -- and hands each to the codec's emitter.
//
// The 32 lanes probe 32 consecutive positions at a time against a 2048-entry hash table of earlier positions (4-byte
// hashes); the first lane whose candidate matches wins, the match is extended 32 bytes per ballot.  Windows without a match
// make the stride grow (snappy's own heuristic), so incompressible data costs little more than the literal copy.  The
// table takes atomicMax updates: the parse, and so every codec's output, is the same on every run.
#pragma once
#include <cstdint>

namespace hs {

constexpr uint32_t kLz77Table = 2048;  // uint32 entries of a warp's hash table

// What a codec allows of a back-reference in a fragment of `len` bytes.
struct Lz77Limits {
  uint32_t max_offset;    // farthest reach back (DEFLATE 32 768, LZ4 65 535)
  uint32_t max_match;     // longest match (DEFLATE 258)
  uint32_t start_margin;  // a match starts at q only when q + start_margin <= len (at least 4; LZ4: 12)
  uint32_t end_margin;    // and ends at least end_margin bytes before len (LZ4: 5, the last literals)
};

__device__ __forceinline__ uint32_t load32_any(const uint8_t* p) {
  return (uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) | ((uint32_t)p[3] << 24);
}

// Parses in[0, len) with the warp's `table` (kLz77Table entries).  The emitter is called by all lanes:
//   emit.sequence(lit_from, q, offset, mlen): literals in[lit_from, q), then mlen bytes from offset back;
//   emit.finish(lit_from, len): the literals after the last match.
template <class Emitter>
__device__ __forceinline__ void lz77_parse(const uint8_t* __restrict__ in, uint32_t len, uint32_t* table, unsigned lane,
                                           const Lz77Limits lim, Emitter& emit) {
  for (uint32_t i = lane; i < kLz77Table; i += 32) table[i] = 0;
  __syncwarp();
  const uint32_t match_end = len - min(len, lim.end_margin);
  uint32_t ip = 0, lit = 0, misses = 0;
  while (ip + lim.start_margin <= len) {
    const uint32_t pos = ip + lane;
    const bool can = pos + lim.start_margin <= len;
    uint32_t w = 0, h = 0, cand = 0;
    if (can) {
      w = load32_any(in + pos);
      h = (w * 0x1e35a7bdu) >> 21;  // 11 bits
      cand = table[h];
    }
    __syncwarp();
    const bool match = can && cand < pos && pos - cand <= lim.max_offset && load32_any(in + cand) == w;
    const unsigned m = __ballot_sync(0xffffffffu, match);
    // only positions up to the match enter the table: the scan resumes right behind the match, and an entry that points
    // past the scan position can never be a candidate (it would shadow the useful, earlier one)
    const int fl = m ? __ffs(m) - 1 : 31;
    if (can && (int)lane <= fl) atomicMax(&table[h], pos);
    __syncwarp();
    if (m == 0) {
      misses++;
      ip += 32u << min(misses >> 2, 4u);
      continue;
    }
    misses = 0;
    const uint32_t q = ip + fl;
    const uint32_t c = __shfl_sync(0xffffffffu, cand, fl);
    // extend the match 32 bytes at a time
    const uint32_t room = min(match_end - q, lim.max_match);
    uint32_t mlen = 4;
    for (;;) {
      const bool eq = mlen + lane < room && in[q + mlen + lane] == in[c + mlen + lane];
      const unsigned e = __ballot_sync(0xffffffffu, eq);
      const uint32_t run = e == 0xffffffffu ? 32u : (uint32_t)(__ffs(~e) - 1);
      mlen += run;
      if (run < 32) break;
    }
    emit.sequence(lit, q, q - c, mlen);
    ip = q + mlen;
    lit = ip;
    __syncwarp();
  }
  emit.finish(lit, len);
}

}  // namespace hs
