// device_utils.cuh -- device helpers shared by the kernels: Spark Murmur3, order-preserving key encodings,
// unaligned little-endian loads / warp-cooperative unaligned stores, block scans.
#pragma once
#include <cuda_runtime.h>

#include <cstdint>

#ifndef HS_HD
#ifdef __CUDACC__
#define HS_HD __host__ __device__ __forceinline__
#else
#define HS_HD inline
#endif
#endif

namespace hs {

// ---- Spark Murmur3_x86_32 (seed 42 fold; CoveringIndex.scala:60 -> HashPartitioning) -----------------------------
HS_HD uint32_t rotl32(uint32_t x, int r) { return (x << r) | (x >> (32 - r)); }
HS_HD uint32_t mm3_mix_k1(uint32_t k1) {
  k1 *= 0xcc9e2d51u;
  k1 = rotl32(k1, 15);
  k1 *= 0x1b873593u;
  return k1;
}
HS_HD uint32_t mm3_mix_h1(uint32_t h1, uint32_t k1) {
  h1 ^= k1;
  h1 = rotl32(h1, 13);
  return h1 * 5u + 0xe6546b64u;
}
HS_HD uint32_t mm3_fmix(uint32_t h1, uint32_t len) {
  h1 ^= len;
  h1 ^= h1 >> 16;
  h1 *= 0x85ebca6bu;
  h1 ^= h1 >> 13;
  h1 *= 0xc2b2ae35u;
  h1 ^= h1 >> 16;
  return h1;
}
HS_HD uint32_t mm3_hash_int(uint32_t v, uint32_t seed) { return mm3_fmix(mm3_mix_h1(seed, mm3_mix_k1(v)), 4); }
HS_HD uint32_t mm3_hash_long(uint64_t v, uint32_t seed) {
  uint32_t h1 = mm3_mix_h1(seed, mm3_mix_k1((uint32_t)v));
  h1 = mm3_mix_h1(h1, mm3_mix_k1((uint32_t)(v >> 32)));
  return mm3_fmix(h1, 8);
}
// Spark Pmod on the signed hash
HS_HD int32_t spark_pmod(uint32_t h, int32_t n) {
  int32_t r = (int32_t)h % n;
  return r < 0 ? r + n : r;
}

// ---- strings (Parquet BYTE_ARRAY) --------------------------------------------------------------------------------------
// A string never moves between decode and encode: a row's value is a 64-bit REFERENCE into the source file image (the
// PLAIN page body or the dictionary page it was read from): device address in the low 48 bits (canonical on every CUDA
// platform), length in the high 16 (longer values are rejected with HS_EUNSUPPORTED when they are decoded).  References
// are ordinary 8-byte column values for the partition and the sort's row bookkeeping.
constexpr uint32_t kMaxStringLen = 0xffffu;
HS_HD uint64_t string_ref(const void* p, uint32_t len) { return ((uint64_t)(uintptr_t)p & 0xffffffffffffull) | ((uint64_t)len << 48); }
HS_HD const uint8_t* ref_ptr(uint64_t ref) { return (const uint8_t*)(uintptr_t)(ref & 0xffffffffffffull); }
HS_HD uint32_t ref_len(uint64_t ref) { return (uint32_t)(ref >> 48); }

// Spark's Murmur3_x86_32.hashUnsafeBytes (the function Murmur3Hash applies to StringType / BinaryType): whole little-endian
// 4-byte words first, then EVERY tail byte mixed on its own as a sign-extended int -- Spark's legacy, non-standard tail
// (oracle: hso_hash_bytes; golden vector hash('Spark', array(123), 2) in tests/test_oracle.py).
HS_HD uint32_t mm3_hash_bytes(const uint8_t* p, uint32_t len, uint32_t seed) {
  uint32_t h1 = seed;
  const uint32_t aligned = len & ~3u;
  for (uint32_t i = 0; i < aligned; i += 4) {
    const uint32_t w = (uint32_t)p[i] | ((uint32_t)p[i + 1] << 8) | ((uint32_t)p[i + 2] << 16) | ((uint32_t)p[i + 3] << 24);
    h1 = mm3_mix_h1(h1, mm3_mix_k1(w));
  }
  for (uint32_t i = aligned; i < len; i++) h1 = mm3_mix_h1(h1, mm3_mix_k1((uint32_t)(int32_t)(int8_t)p[i]));
  return mm3_fmix(h1, len);
}

// UTF8String.compareTo: unsigned byte-wise, a proper prefix sorts first.  -1 / 0 / +1
HS_HD int string_compare(uint64_t ra, uint64_t rb) {
  const uint8_t *a = ref_ptr(ra), *b = ref_ptr(rb);
  const uint32_t la = ref_len(ra), lb = ref_len(rb), n = la < lb ? la : lb;
  for (uint32_t i = 0; i < n; i++)
    if (a[i] != b[i]) return a[i] < b[i] ? -1 : 1;
  return la == lb ? 0 : (la < lb ? -1 : 1);
}

// the `chunk`-th 8-byte piece of a string as a big-endian integer, zero-padded: comparing the pieces in order, then the
// lengths, is the byte-wise order above (this is how the radix sort sees a string key)
HS_HD uint64_t string_chunk(uint64_t ref, uint32_t chunk) {
  const uint8_t* p = ref_ptr(ref);
  const uint32_t len = ref_len(ref), begin = chunk * 8;
  uint64_t v = 0;
  for (uint32_t i = 0; i < 8; i++) v = (v << 8) | (begin + i < len ? (uint64_t)p[begin + i] : 0ull);
  return v;
}

// Hash kind of a Spark decimal(p <= 9) column: its unscaled value is an int32 in HBM, but Murmur3Hash hashes every decimal
// of precision <= 18 as hashLong(unscaled) -- so the int32 is sign-extended and hashed as a long.
constexpr int kHashDecimalInt = 6;

// raw bits of one key value, as stored in the decoded column; type = HS_TYPE_* or kHashDecimalInt (KeyColumn::hash)
HS_HD uint32_t mm3_hash_value(int type, uint64_t raw, uint32_t seed) {
  switch (type) {
    case 0: return mm3_hash_int((uint32_t)raw, seed);   // int32
    case 1: return mm3_hash_long(raw, seed);            // int64
    case 2: {                                           // float: -0.0 -> 0.0, canonical NaN
      uint32_t b = (uint32_t)raw;
      if ((b & 0x7fffffffu) == 0) b = 0;
      else if ((b & 0x7fffffffu) > 0x7f800000u) b = 0x7fc00000u;
      return mm3_hash_int(b, seed);
    }
    case 3: {
      uint64_t b = raw;
      if ((b & 0x7fffffffffffffffull) == 0) b = 0;
      else if ((b & 0x7fffffffffffffffull) > 0x7ff0000000000000ull) b = 0x7ff8000000000000ull;
      return mm3_hash_long(b, seed);
    }
    case 4: return mm3_hash_int((raw & 0xff) ? 1u : 0u, seed);
    case 5: return mm3_hash_bytes(ref_ptr(raw), ref_len(raw), seed);  // string / binary: raw is a reference
    case kHashDecimalInt: return mm3_hash_long((uint64_t)(int64_t)(int32_t)(uint32_t)raw, seed);
  }
  return seed;
}

// ---- order-preserving unsigned encodings (ascending; Spark SortOrder asc, NaN greatest, -0.0 == 0.0) ----------------
HS_HD uint64_t sort_encode(int type, uint64_t raw) {
  switch (type) {
    case 0: return (uint64_t)((uint32_t)raw ^ 0x80000000u);
    case 1: return raw ^ 0x8000000000000000ull;
    case 2: {
      uint32_t b = (uint32_t)raw;
      if ((b & 0x7fffffffu) == 0) b = 0;
      else if ((b & 0x7fffffffu) > 0x7f800000u) b = 0x7fc00000u;
      return (uint64_t)((b & 0x80000000u) ? ~b : (b | 0x80000000u));
    }
    case 3: {
      uint64_t b = raw;
      if ((b & 0x7fffffffffffffffull) == 0) b = 0;
      else if ((b & 0x7fffffffffffffffull) > 0x7ff0000000000000ull) b = 0x7ff8000000000000ull;
      return (b & 0x8000000000000000ull) ? ~b : (b | 0x8000000000000000ull);
    }
    case 4: return (raw & 0xff) ? 1 : 0;
  }
  return raw;
}
// inverse of sort_encode for the integer types (type 1: int64, else int32)
__device__ __forceinline__ uint64_t sort_decode_int(int type, uint64_t e) {
  return type == 1 ? (e ^ 0x8000000000000000ull) : (uint64_t)((uint32_t)e ^ 0x80000000u);
}

// Fibonacci hashing of a dictionary value's raw bits: one 64-bit multiply; the top bits of the product depend on every
// input bit.  Shared by the device hash sets / look-up tables and the host code that builds the compact look-up table.
HS_HD uint32_t dict_hash_u64(uint64_t v) { return (uint32_t)((v * 0x9E3779B97F4A7C15ull) >> 32); }

HS_HD int type_width(int type) {
  switch (type) {
    case 0: case 2: return 4;
    case 1: case 3: return 8;
    case 4: return 1;
    case 5: return 8;  // a string column holds 8-byte references
  }
  return 0;
}

#ifdef __CUDACC__

// ---- unaligned little-endian loads ---------------------------------------------------------------------------
// The enclosing allocation is at least 8-byte aligned and padded, so the aligned words that contain [p, p+W) are
// always readable.
__device__ __forceinline__ uint64_t load_le64_unaligned(const uint8_t* p) {
  uintptr_t a = (uintptr_t)p;
  const uint64_t* w = (const uint64_t*)(a & ~(uintptr_t)7);
  unsigned s = (unsigned)(a & 7) * 8;
  uint64_t lo = __ldg(w);
  if (s == 0) return lo;
  uint64_t hi = __ldg(w + 1);
  return (lo >> s) | (hi << (64 - s));
}
__device__ __forceinline__ uint32_t load_le32_unaligned(const uint8_t* p) {
  uintptr_t a = (uintptr_t)p;
  const uint32_t* w = (const uint32_t*)(a & ~(uintptr_t)3);
  unsigned s = (unsigned)(a & 3) * 8;
  uint32_t lo = __ldg(w);
  if (s == 0) return lo;
  uint32_t hi = __ldg(w + 1);
  return __funnelshift_r(lo, hi, s);
}

// `bw`-bit value number `idx` of a bit-packed run whose first byte is `base` (Parquet RLE/bit-packing hybrid:
// values packed LSB first).  Reads only bytes that belong to the run.
__device__ __forceinline__ uint32_t extract_bits(const uint8_t* base, uint64_t idx, uint32_t bw) {
  uint64_t bit = idx * bw;
  const uint8_t* p = base + (bit >> 3);
  uintptr_t a = (uintptr_t)p;
  const uint32_t* w = (const uint32_t*)(a & ~(uintptr_t)3);
  unsigned s = (unsigned)(a & 3) * 8 + (unsigned)(bit & 7);
  uint64_t v = __ldg(w);
  if (s + bw > 32) v |= (uint64_t)__ldg(w + 1) << 32;
  // s <= 31 and bw <= 32, so the value never spans more than these two words
  return (uint32_t)((v >> s) & ((bw >= 32) ? 0xffffffffull : ((1ull << bw) - 1)));
}

// ---- warp-cooperative unaligned stores ---------------------------------------------------------------------------
// Every active lane holds one W-byte value `v` destined for byte address `dst` (any alignment).  Lanes whose
// destinations are consecutive (dst[l] == dst[l-1] + W) cooperate: each aligned word that lies completely inside a
// run of consecutive destinations is written once with a full-width store assembled from two neighbouring lanes;
// the ragged head and tail of each run fall back to byte stores.  Must be called by all 32 lanes of the warp.
template <int W>
__device__ __forceinline__ void warp_store_unaligned(uint8_t* dst, uint64_t v, bool active) {
  static_assert(W == 4 || W == 8, "W");
  const unsigned lane = threadIdx.x & 31;
  unsigned long long d = active ? (unsigned long long)(uintptr_t)dst : 0ull;
  unsigned long long d_prev = __shfl_up_sync(0xffffffffu, d, 1);
  uint64_t v_prev = __shfl_up_sync(0xffffffffu, (unsigned long long)v, 1);
  unsigned long long d_next = __shfl_down_sync(0xffffffffu, d, 1);
  if (!active) return;
  const unsigned a = (unsigned)(d & (W - 1));
  if (a == 0) {  // aligned destination: plain store
    if (W == 8) *(uint64_t*)dst = v;
    else *(uint32_t*)dst = (uint32_t)v;
    return;
  }
  const bool has_prev = lane > 0 && d_prev != 0 && d_prev + W == d;
  const bool has_next = lane < 31 && d_next != 0 && d + W == d_next;
  uint8_t* word = dst - a;  // aligned word that holds the first W-a bytes of v
  const unsigned s = a * 8;
  if (has_prev) {
    // word = high bytes of v_prev | low bytes of v
    if (W == 8) *(uint64_t*)word = (v_prev >> (64 - s)) | (v << s);
    else *(uint32_t*)word = (uint32_t)(((uint32_t)v_prev >> (32 - s)) | ((uint32_t)v << s));
  } else {
    for (unsigned i = 0; i < W - a; i++) dst[i] = (uint8_t)(v >> (8 * i));
  }
  if (!has_next) {
    for (unsigned i = W - a; i < W; i++) dst[i] = (uint8_t)(v >> (8 * i));
  }
}

// ---- warp multi-split -------------------------------------------------------------------------------------------
// Mask of the lanes in `amask` whose `v` equals this lane's, from NBITS ballots.  __match_any_sync does the same in one
// instruction, but MATCH runs on the ADU pipe at roughly one lane per cycle and made the radix scatter kernel
// ADU-bound, while VOTE + LOP3 issue at full rate.
__device__ __forceinline__ unsigned match_any_bits(unsigned amask, unsigned v, int nbits) {
  unsigned peers = amask;
  for (int b = 0; b < nbits; b++) {
    const bool bit = (v >> b) & 1u;
    const unsigned m = __ballot_sync(amask, bit);
    peers &= bit ? m : ~m;
  }
  return peers;
}
template <int NBITS>
__device__ __forceinline__ unsigned match_any_bits(unsigned amask, unsigned v) {
  unsigned peers = amask;
#pragma unroll
  for (int b = 0; b < NBITS; b++) {
    const bool bit = (v & (1u << b)) != 0;  // one LOP3 with predicate output
    const unsigned m = __ballot_sync(amask, bit);
    peers &= m ^ (bit ? 0u : ~0u);          // SEL + one three-input LOP3
  }
  return peers;
}

// Full-warp variant (every lane takes part, no branch around it): bit test, ballot and the select of m / ~m are spelled
// out in PTX; ptxas then moves the digit's bits into predicates with one R2P and spends VOTE + predicated LOP3 (NOT) +
// LOP3 (AND) per bit -- half of what it emits for the C++ form above.
template <int NBITS>
__device__ __forceinline__ unsigned match_any_full(unsigned v) {
  unsigned peers = 0xffffffffu;
#pragma unroll
  for (int b = 0; b < NBITS; b++) {
    unsigned m, x;
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        ".reg .b32 t;\n\t"
        "and.b32 t, %2, %3;\n\t"
        "setp.ne.u32 p, t, 0;\n\t"
        "vote.sync.ballot.b32 %0, p, 0xffffffff;\n\t"
        "selp.b32 %1, 0, 0xffffffff, p;\n\t"
        "}"
        : "=r"(m), "=r"(x)
        : "r"(v), "r"(1u << b));
    peers &= m ^ x;
  }
  return peers;
}

// ---- block-level exclusive scan of one uint32 per thread (blockDim.x <= 1024, multiple of 32) ------------------------
// Returns the exclusive prefix; *total receives the block sum.  `warp_sums` is >= 32 words of shared memory.
__device__ __forceinline__ uint32_t block_exclusive_scan(uint32_t x, uint32_t* warp_sums, uint32_t* total) {
  const unsigned lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = (blockDim.x + 31) >> 5;
  uint32_t incl = x;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    uint32_t y = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= (unsigned)o) incl += y;
  }
  __syncthreads();  // protect warp_sums reuse across calls
  if (lane == 31) warp_sums[warp] = incl;
  __syncthreads();
  if (warp == 0) {
    uint32_t w = lane < nwarps ? warp_sums[lane] : 0;
    uint32_t wi = w;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      uint32_t y = __shfl_up_sync(0xffffffffu, wi, o);
      if (lane >= (unsigned)o) wi += y;
    }
    warp_sums[lane] = wi - w;  // exclusive warp offsets
    if (lane == 31) warp_sums[32] = wi;
  }
  __syncthreads();
  uint32_t res = warp_sums[warp] + incl - x;
  if (total) *total = warp_sums[32];
  return res;
}

#endif  // __CUDACC__

}  // namespace hs
