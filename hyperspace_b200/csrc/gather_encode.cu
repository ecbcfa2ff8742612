// gather_encode.cu -- K5 payload gather fused with K6 PLAIN Parquet page encode, plus the synthetic-table generator.
//
// Replaces Spark's DynamicPartitionDataWriter -> ParquetOutputWriter (parquet-mr column writers) that the reference
// reaches through DataSource.planForWriting (index/DataFrameWriterExtensions.scala:58-67; SURVEY.md 3.1 HOT LOOP 3).
// The host lays every bucket file out up front (page headers, definition-level blocks and footers are tiny and are
// serialised on the host into a "skeleton" byte stream); the kernel below writes each sorted value straight into its
// page body inside the file image, so the index is encoded in the same pass that gathers the payload.  Page bodies
// start at arbitrary byte offsets (Thrift headers have odd sizes): warp_store_unaligned assembles full-width stores
// from neighbouring lanes.
#include "device_utils.cuh"
#include "kernels.h"

namespace hs {

namespace {

constexpr int kThreads = 256;

template <int W>
__global__ void __launch_bounds__(kThreads) k_gather_encode(const SortTile* __restrict__ tiles,
                                                             const uint64_t* __restrict__ seg_start,
                                                             const uint32_t* __restrict__ perm, GatherColumn col,
                                                             const uint32_t* __restrict__ bucket_page_begin,
                                                             int64_t rows_per_page, uint8_t* __restrict__ arena) {
  // tiles are kSortTile-aligned inside their bucket and rows_per_page is a multiple of kSortTile, so a tile lies inside
  // one page: the destination is one base pointer per CTA plus i * W
  const SortTile t = tiles[blockIdx.x];
  const uint64_t lr0 = t.start - seg_start[t.seg];
  const uint64_t page = lr0 / (uint64_t)rows_per_page;
  uint8_t* const base = arena + col.page_value_offset[bucket_page_begin[t.seg] + page] + (lr0 - page * (uint64_t)rows_per_page) * W;
  // the host pads the definition-level block so that page bodies are 8-byte aligned whenever the page is large enough
  const bool aligned = ((uintptr_t)base & (W - 1)) == 0;
  if (aligned && t.count == kSortTile) {
    // Full tile, aligned body (all but a bucket's last tile): every thread's row indices are loaded first, then all its
    // gathers are in flight together, then the stores -- the gather is latency-bound (stalls on the dependent
    // perm -> value load pair with one pair per thread in flight)
    constexpr int kPer = kSortTile / kThreads;
    uint64_t v[kPer];
    if (col.sorted_keys) {
#pragma unroll
      for (int it = 0; it < kPer; it++) v[it] = sort_decode_int(col.key_type, col.sorted_keys[t.start + it * kThreads + threadIdx.x]);
    } else {
      uint32_t r[kPer];
#pragma unroll
      for (int it = 0; it < kPer; it++) r[it] = perm[t.start + it * kThreads + threadIdx.x];
#pragma unroll
      for (int it = 0; it < kPer; it++) v[it] = W == 8 ? ((const uint64_t*)col.src)[r[it]] : ((const uint32_t*)col.src)[r[it]];
    }
#pragma unroll
    for (int it = 0; it < kPer; it++) {
      const uint32_t i = it * kThreads + threadIdx.x;
      if (W == 8) reinterpret_cast<uint64_t*>(base)[i] = v[it];
      else reinterpret_cast<uint32_t*>(base)[i] = (uint32_t)v[it];
    }
    return;
  }
  const uint32_t iters = (t.count + kThreads - 1) / kThreads;
  for (uint32_t it = 0; it < iters; it++) {
    const uint32_t i = it * kThreads + threadIdx.x;
    const bool active = i < t.count;
    uint64_t v = 0;
    if (active) {
      const uint64_t p = t.start + i;
      if (col.sorted_keys) {
        v = sort_decode_int(col.key_type, col.sorted_keys[p]);
      } else {
        const uint32_t src_row = perm[p];
        v = W == 8 ? ((const uint64_t*)col.src)[src_row] : ((const uint32_t*)col.src)[src_row];
      }
    }
    if (aligned) {
      if (active) {
        if (W == 8) reinterpret_cast<uint64_t*>(base)[i] = v;
        else reinterpret_cast<uint32_t*>(base)[i] = (uint32_t)v;
      }
    } else {
      warp_store_unaligned<W>(base + (size_t)i * W, v, active);
    }
  }
}

// ---- nullable columns ---------------------------------------------------------------------------------------------
// valid flags of the rows at the tile's sorted positions, counted (the host turns the per-tile counts into the page
// layout: a page stores only its non-null values)
__global__ void __launch_bounds__(kThreads) k_tile_valid_counts(const SortTile* __restrict__ tiles,
                                                                 const uint32_t* __restrict__ perm,
                                                                 const uint8_t* __restrict__ valid,
                                                                 uint32_t* __restrict__ counts) {
  __shared__ uint32_t s_total;
  if (threadIdx.x == 0) s_total = 0;
  __syncthreads();
  const SortTile t = tiles[blockIdx.x];
  uint32_t local = 0;
  for (uint32_t i = threadIdx.x; i < t.count; i += kThreads) local += valid[perm[t.start + i]] ? 1u : 0u;
  for (int o = 16; o > 0; o >>= 1) local += __shfl_xor_sync(0xffffffffu, local, o);
  if ((threadIdx.x & 31) == 0 && local) atomicAdd(&s_total, local);
  __syncthreads();
  if (threadIdx.x == 0) counts[blockIdx.x] = s_total;
}

// Per tile: definition levels as bits (one bit-packed hybrid run per page, written 32 levels per warp ballot) and the
// non-null values compacted through shared memory into the page's dense value region.
template <int W>
__global__ void __launch_bounds__(kThreads) k_gather_encode_nullable(const SortTile* __restrict__ tiles,
                                                                      const uint32_t* __restrict__ perm,
                                                                      const void* __restrict__ src,
                                                                      const uint8_t* __restrict__ valid,
                                                                      const uint64_t* __restrict__ tile_value_offset,
                                                                      const uint64_t* __restrict__ tile_def_offset,
                                                                      uint8_t* __restrict__ arena) {
  __shared__ uint64_t s_vals[kSortTile];
  __shared__ uint32_t warp_sums[40];
  const SortTile t = tiles[blockIdx.x];
  uint8_t* const def_out = arena + tile_def_offset[blockIdx.x];
  uint32_t base = 0;
  const uint32_t iters = (t.count + kThreads - 1) / kThreads;
  for (uint32_t it = 0; it < iters; it++) {
    const uint32_t i = it * kThreads + threadIdx.x;
    const bool active = i < t.count;
    uint32_t flag = 0;
    uint64_t v = 0;
    if (active) {
      const uint32_t row = perm[t.start + i];
      flag = valid[row] ? 1u : 0u;
      if (flag) v = W == 8 ? ((const uint64_t*)src)[row] : ((const uint32_t*)src)[row];
    }
    const unsigned bits = __ballot_sync(0xffffffffu, flag != 0);
    if ((threadIdx.x & 31) == 0) {  // 32 levels = 4 bytes, LSB first; the last warp of a page may own fewer bytes
      const uint32_t first = it * kThreads + (threadIdx.x & ~31u);
      if (first < t.count) {
        const uint32_t nbytes = min(4u, (t.count - first + 7) / 8);
        for (uint32_t b = 0; b < nbytes; b++) def_out[first / 8 + b] = (uint8_t)(bits >> (8 * b));
      }
    }
    uint32_t total = 0;
    const uint32_t pos = block_exclusive_scan(flag, warp_sums, &total);
    if (flag) s_vals[base + pos] = v;
    base += total;
  }
  __syncthreads();
  uint8_t* const val_out = arena + tile_value_offset[blockIdx.x];
  const uint32_t viters = (base + kThreads - 1) / kThreads;
  for (uint32_t it = 0; it < viters; it++) {
    const uint32_t j = it * kThreads + threadIdx.x;
    const bool active = j < base;
    warp_store_unaligned<W>(val_out + (size_t)j * W, active ? s_vals[j] : 0, active);
  }
}

// ---- boolean columns ----------------------------------------------------------------------------------------------
// PLAIN BOOLEAN is bit-packed, LSB first.  A page starts on a multiple of kSortTile rows, so a tile of a null-free page
// starts on a byte of the page body ((lr0 mod P) / 8) and ends on one unless it is its bucket's last: no two tiles share
// a byte.  Each warp ballot packs 32 rows into one word of shared memory; the tile's bytes leave as unaligned words, the
// ragged tail as single bytes (the byte after a page body belongs to the next page header).
static_assert(kSortTile % 32 == 0, "a tile packs into whole words and starts on a byte boundary");
__global__ void __launch_bounds__(kThreads) k_gather_encode_bool(const SortTile* __restrict__ tiles,
                                                                  const uint64_t* __restrict__ seg_start,
                                                                  const uint32_t* __restrict__ perm,
                                                                  const uint8_t* __restrict__ src,
                                                                  const uint64_t* __restrict__ page_value_offset,
                                                                  const uint32_t* __restrict__ bucket_page_begin,
                                                                  int64_t rows_per_page, uint8_t* __restrict__ arena) {
  constexpr int kPer = kSortTile / kThreads;
  __shared__ uint32_t s_words[kSortTile / 32];
  const SortTile t = tiles[blockIdx.x];
  const uint64_t lr0 = t.start - seg_start[t.seg];
  const uint64_t page = lr0 / (uint64_t)rows_per_page;
  uint8_t* const base = arena + page_value_offset[bucket_page_begin[t.seg] + page] + (lr0 - page * (uint64_t)rows_per_page) / 8;
  // all of a thread's row indices first, then all its value loads in flight together (as k_gather_encode does)
  uint32_t r[kPer];
#pragma unroll
  for (int it = 0; it < kPer; it++) {
    const uint32_t i = it * kThreads + threadIdx.x;
    r[it] = i < t.count ? perm[t.start + i] : 0u;
  }
  uint8_t v[kPer];
#pragma unroll
  for (int it = 0; it < kPer; it++) v[it] = it * kThreads + threadIdx.x < t.count ? src[r[it]] : (uint8_t)0;
#pragma unroll
  for (int it = 0; it < kPer; it++) {
    const unsigned bits = __ballot_sync(0xffffffffu, v[it] != 0);
    if ((threadIdx.x & 31) == 0) s_words[(it * kThreads + threadIdx.x) / 32] = bits;
  }
  __syncthreads();
  const uint32_t nbytes = (t.count + 7) / 8, nwords = nbytes / 4;
  for (uint32_t w0 = 0; w0 < kSortTile / 32; w0 += kThreads) {
    const uint32_t w = w0 + threadIdx.x;
    warp_store_unaligned<4>(base + 4 * (size_t)w, w < nwords ? s_words[w] : 0u, w < nwords);
  }
  if (threadIdx.x < nbytes - 4 * nwords) base[4 * nwords + threadIdx.x] = (uint8_t)(s_words[nwords] >> (8 * threadIdx.x));
}

// Nullable boolean columns, one CTA per page.  The non-null values of a page are one bit stream that crosses its tiles at
// any bit, and the page's definition bits end in the middle of a word: a CTA that owns the whole page writes every byte of
// it, so no two CTAs touch the same byte.  The grid is the tile list; the CTA of a page's first tile walks the page's
// tiles (those of its segment whose definition bits follow on, kSortTile / 8 bytes apart), the others return at once.  Per
// step of kBoolStep rows: definition bits by warp ballot (as k_gather_encode_nullable writes them), positions of the
// non-null rows by block scan, their value bits OR-ed into a shared bit buffer that carries its partial last word from one
// step to the next; whole words are stored as they fill.  The value bits follow the definition bits of the page.
constexpr int kBoolStep = 1024;  // rows per step: four gathers in flight per thread
__global__ void __launch_bounds__(kThreads) k_gather_encode_bool_nullable(const SortTile* __restrict__ tiles, int64_t ntiles,
                                                                           const uint32_t* __restrict__ perm,
                                                                           const uint8_t* __restrict__ src,
                                                                           const uint8_t* __restrict__ valid,
                                                                           const uint64_t* __restrict__ tile_def_offset,
                                                                           uint8_t* __restrict__ arena) {
  constexpr int kPer = kBoolStep / kThreads;
  constexpr uint32_t kWords = kBoolStep / 32 + 2;
  __shared__ uint32_t s_bits[kWords];
  __shared__ uint32_t warp_sums[40];
  const int64_t t0 = blockIdx.x;
  const uint32_t seg = tiles[t0].seg;
  auto follows = [&](int64_t t) {  // tile t continues the page of tile t - 1
    return tiles[t].seg == seg && tile_def_offset[t] == tile_def_offset[t - 1] + kSortTile / 8;
  };
  if (t0 > 0 && follows(t0)) return;
  int64_t t1 = t0 + 1;
  uint32_t count = tiles[t0].count;
  while (t1 < ntiles && follows(t1)) count += tiles[t1++].count;
  const uint64_t start = tiles[t0].start;
  uint8_t* const def_out = arena + tile_def_offset[t0];
  uint8_t* const val_out = def_out + (count + 7) / 8;
  for (uint32_t j = threadIdx.x; j < kWords; j += kThreads) s_bits[j] = 0;
  uint32_t carry_bits = 0;  // value bits in s_bits[0] not yet stored
  uint64_t stored_words = 0;
  for (uint32_t step = 0; step < count; step += kBoolStep) {
    uint32_t flag[kPer];
    uint8_t v[kPer];
#pragma unroll
    for (int k = 0; k < kPer; k++) {
      const uint32_t i = step + k * kThreads + threadIdx.x;
      const uint32_t row = i < count ? perm[start + i] : 0u;
      flag[k] = i < count && valid[row] ? 1u : 0u;
      v[k] = flag[k] ? src[row] : (uint8_t)0;
    }
#pragma unroll
    for (int k = 0; k < kPer; k++) {
      const uint32_t first = step + k * kThreads + (threadIdx.x & ~31u);
      const unsigned bits = __ballot_sync(0xffffffffu, flag[k] != 0);
      if ((threadIdx.x & 31) == 0 && first < count) {  // 32 levels = 4 bytes, LSB first
        const uint32_t nb = min(4u, (count - first + 7) / 8);
        for (uint32_t b = 0; b < nb; b++) def_out[first / 8 + b] = (uint8_t)(bits >> (8 * b));
      }
      uint32_t total = 0;
      const uint32_t pos = carry_bits + block_exclusive_scan(flag[k], warp_sums, &total);
      if (flag[k] && v[k]) atomicOr(&s_bits[pos / 32], 1u << (pos % 32));
      carry_bits += total;
    }
    __syncthreads();
    const uint32_t full = carry_bits / 32;
    for (uint32_t w0 = 0; w0 < kWords; w0 += kThreads) {
      const uint32_t w = w0 + threadIdx.x;
      warp_store_unaligned<4>(val_out + 4 * (stored_words + w), w < full ? s_bits[w] : 0u, w < full);
    }
    __syncthreads();
    const uint32_t tail = s_bits[full];
    __syncthreads();
    for (uint32_t j = threadIdx.x; j < kWords; j += kThreads) s_bits[j] = j == 0 ? tail : 0u;
    __syncthreads();
    stored_words += full;
    carry_bits %= 32;
  }
  if (threadIdx.x < (carry_bits + 7) / 8) val_out[4 * stored_words + threadIdx.x] = (uint8_t)(s_bits[0] >> (8 * threadIdx.x));
}

// ---- string columns -----------------------------------------------------------------------------------------------
// PLAIN BYTE_ARRAY: every non-null value is [u32 length][bytes].  First the tiles are measured (the host needs every
// page's byte size to lay the files out), then each tile writes its definition bits and its values: a block scan of the
// value sizes gives every row its place, and each thread copies its own string out of the source image.
__global__ void __launch_bounds__(kThreads) k_tile_string_sizes(const SortTile* __restrict__ tiles, const uint32_t* __restrict__ perm,
                                                                 const uint64_t* __restrict__ refs,
                                                                 const uint8_t* __restrict__ valid,
                                                                 uint32_t* __restrict__ bytes, uint32_t* __restrict__ counts) {
  __shared__ uint32_t s_bytes, s_count;
  if (threadIdx.x == 0) s_bytes = s_count = 0;
  __syncthreads();
  const SortTile t = tiles[blockIdx.x];
  uint32_t b = 0, c = 0;
  for (uint32_t i = threadIdx.x; i < t.count; i += kThreads) {
    const uint32_t row = perm[t.start + i];
    if (!valid || valid[row]) {
      b += 4u + ref_len(refs[row]);
      c++;
    }
  }
  for (int o = 16; o > 0; o >>= 1) {
    b += __shfl_xor_sync(0xffffffffu, b, o);
    c += __shfl_xor_sync(0xffffffffu, c, o);
  }
  if ((threadIdx.x & 31) == 0 && c) {
    atomicAdd(&s_bytes, b);
    atomicAdd(&s_count, c);
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    bytes[blockIdx.x] = s_bytes;
    counts[blockIdx.x] = s_count;
  }
}

__global__ void __launch_bounds__(kThreads) k_gather_encode_strings(const SortTile* __restrict__ tiles,
                                                                     const uint32_t* __restrict__ perm,
                                                                     const uint64_t* __restrict__ refs,
                                                                     const uint8_t* __restrict__ valid,
                                                                     const uint64_t* __restrict__ tile_value_offset,
                                                                     const uint64_t* __restrict__ tile_def_offset,
                                                                     uint8_t* __restrict__ arena) {
  __shared__ uint32_t warp_sums[40];
  const SortTile t = tiles[blockIdx.x];
  uint8_t* const def_out = arena + tile_def_offset[blockIdx.x];
  uint8_t* const val_out = arena + tile_value_offset[blockIdx.x];
  uint32_t base = 0;
  const uint32_t iters = (t.count + kThreads - 1) / kThreads;
  for (uint32_t it = 0; it < iters; it++) {
    const uint32_t i = it * kThreads + threadIdx.x;
    const bool active = i < t.count;
    uint32_t flag = 0;
    uint64_t r = 0;
    if (active) {
      const uint32_t row = perm[t.start + i];
      flag = (!valid || valid[row]) ? 1u : 0u;
      if (flag) r = refs[row];
    }
    const unsigned bits = __ballot_sync(0xffffffffu, flag != 0);
    if ((threadIdx.x & 31) == 0) {  // 32 levels = 4 bytes, LSB first; the last warp of a page may own fewer bytes
      const uint32_t first = it * kThreads + (threadIdx.x & ~31u);
      if (first < t.count) {
        const uint32_t nbytes = min(4u, (t.count - first + 7) / 8);
        for (uint32_t b = 0; b < nbytes; b++) def_out[first / 8 + b] = (uint8_t)(bits >> (8 * b));
      }
    }
    const uint32_t len = ref_len(r), size = flag ? 4u + len : 0u;
    uint32_t total = 0;
    const uint32_t pos = block_exclusive_scan(size, warp_sums, &total);
    if (flag) {
      uint8_t* o = val_out + base + pos;
      o[0] = (uint8_t)len;
      o[1] = (uint8_t)(len >> 8);
      o[2] = (uint8_t)(len >> 16);
      o[3] = (uint8_t)(len >> 24);
      const uint8_t* src = ref_ptr(r);
      for (uint32_t b = 0; b < len; b++) o[4 + b] = src[b];
    }
    base += total;
  }
}

// fixed-width values through a permutation (width 1: the read side's boolean columns, one byte per row)
template <typename T>
__global__ void k_gather_plain(const T* __restrict__ src, const uint32_t* __restrict__ perm, int64_t n,
                               T* __restrict__ out) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) out[i] = src[perm[i]];
}

__global__ void k_scatter_bytes(const ByteCopy* __restrict__ copies, int64_t n, const uint8_t* __restrict__ skeleton,
                                uint8_t* __restrict__ arena) {
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (warp >= n) return;
  const ByteCopy c = copies[warp];
  for (uint32_t i = lane; i < c.len; i += 32) arena[c.dst + i] = skeleton[c.src + i];
}

__global__ void __launch_bounds__(256) k_copy_blobs(const BlobCopy* __restrict__ blobs, const uint8_t* __restrict__ src_base,
                                                     uint8_t* __restrict__ dst_base) {
  const BlobCopy b = blobs[blockIdx.x];
  const uint8_t* src = src_base + b.src;
  uint8_t* dst = dst_base + b.dst;
  // bytes up to the destination's first 4-byte boundary, then whole words assembled from the two aligned source words
  // around them, then the tail
  const uint32_t head = min(b.len, (uint32_t)((4 - ((uintptr_t)dst & 3)) & 3));
  for (uint32_t i = threadIdx.x; i < head; i += 256) dst[i] = src[i];
  const uint32_t nwords = (b.len - head) / 4;
  uint32_t* d32 = reinterpret_cast<uint32_t*>(dst + head);
  const uint8_t* s0 = src + head;
  for (uint32_t w = threadIdx.x; w < nwords; w += 256) d32[w] = load_le32_unaligned(s0 + 4 * (size_t)w);
  for (uint32_t i = head + 4 * nwords + threadIdx.x; i < b.len; i += 256) dst[i] = src[i];
}

// min / max statistics of the (sorted) indexed column: first and last key of every row group, written over the
// placeholders the host left in the footer.  The values come from the partitioned column through the permutation, which
// every sort path writes (the page bodies would hold codes when the key is dictionary-encoded).
__global__ void k_patch_key_stats(const StatPatch* __restrict__ patches, int64_t n, const uint32_t* __restrict__ perm,
                                  const void* __restrict__ keys, uint8_t* __restrict__ arena) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const StatPatch p = patches[i];
  const uint32_t rmin = perm[p.first_pos], rmax = perm[p.last_pos];
  const uint64_t vmin = p.width == 8 ? ((const uint64_t*)keys)[rmin] : ((const uint32_t*)keys)[rmin];
  const uint64_t vmax = p.width == 8 ? ((const uint64_t*)keys)[rmax] : ((const uint32_t*)keys)[rmax];
  for (int b = 0; b < p.width; b++) {
    const uint8_t lo = (uint8_t)(vmin >> (8 * b)), hi = (uint8_t)(vmax >> (8 * b));
    arena[p.min_off[0] + b] = lo;
    arena[p.min_off[1] + b] = lo;
    arena[p.max_off[0] + b] = hi;
    arena[p.max_off[1] + b] = hi;
  }
}

__device__ __forceinline__ uint64_t splitmix64(uint64_t seed, uint64_t i) {
  uint64_t z = seed + (i + 1) * 0x9E3779B97F4A7C15ull;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}

__global__ void k_synth_column(int col, int64_t first_row, int64_t n, void* __restrict__ out) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; j < n; j += stride) {
    const uint64_t i = (uint64_t)(first_row + j);
    switch (col) {
      case 0: ((uint64_t*)out)[j] = splitmix64(42, i); break;
      case 1: ((int64_t*)out)[j] = (int64_t)(splitmix64(43, i) % 1000ull); break;
      case 2: ((double*)out)[j] = (double)i * 1e-3; break;
      case 3: ((int32_t*)out)[j] = (int32_t)(i % 100ull); break;
      case 4: ((float*)out)[j] = (float)(i % 4096ull) * 0.25f; break;
    }
  }
}

inline int grid_for(hs_ctx* ctx, int64_t n, int threads, int per_sm) {
  int64_t want = ceil_div(n, threads);
  int64_t cap = (int64_t)ctx->sm_count * per_sm;
  return (int)std::max<int64_t>(1, std::min(want, cap));
}

}  // namespace

void launch_gather_encode(hs_ctx* ctx, const SortTile* tiles, int64_t ntiles, const uint64_t* seg_start,
                          const uint32_t* perm, const GatherColumn& col, const uint32_t* bucket_page_begin,
                          int64_t rows_per_page, uint8_t* arena) {
  KernelScope _ks(ctx, col.width == 1 ? "k_gather_encode_bool" : "k_gather_encode");
  if (ntiles == 0) return;
  if (col.width == 1)
    k_gather_encode_bool<<<(unsigned)ntiles, kThreads, 0, ctx->stream>>>(tiles, seg_start, perm, (const uint8_t*)col.src,
                                                                         col.page_value_offset, bucket_page_begin, rows_per_page, arena);
  else if (col.width == 8)
    k_gather_encode<8><<<(unsigned)ntiles, kThreads, 0, ctx->stream>>>(tiles, seg_start, perm, col, bucket_page_begin,
                                                                        rows_per_page, arena);
  else if (col.width == 4)
    k_gather_encode<4><<<(unsigned)ntiles, kThreads, 0, ctx->stream>>>(tiles, seg_start, perm, col, bucket_page_begin,
                                                                        rows_per_page, arena);
  else
    fail(HS_EUNSUPPORTED, "gather_encode: column width %d", col.width);
  HS_LAUNCH_CHECK(ctx);
}

void launch_tile_valid_counts(hs_ctx* ctx, const SortTile* tiles, int64_t ntiles, const uint32_t* perm,
                              const uint8_t* valid, uint32_t* counts) {
  KernelScope _ks(ctx, "k_tile_valid_counts");
  if (ntiles == 0) return;
  k_tile_valid_counts<<<(unsigned)ntiles, kThreads, 0, ctx->stream>>>(tiles, perm, valid, counts);
  HS_LAUNCH_CHECK(ctx);
}

void launch_gather_encode_nullable(hs_ctx* ctx, const SortTile* tiles, int64_t ntiles, const uint32_t* perm,
                                   const void* src, const uint8_t* valid, int width, const uint64_t* tile_value_offset,
                                   const uint64_t* tile_def_offset, uint8_t* arena) {
  KernelScope _ks(ctx, width == 1 ? "k_gather_encode_bool_nullable" : "k_gather_encode_nullable");
  if (ntiles == 0) return;
  if (width == 1)
    k_gather_encode_bool_nullable<<<(unsigned)ntiles, kThreads, 0, ctx->stream>>>(tiles, ntiles, perm, (const uint8_t*)src, valid,
                                                                                   tile_def_offset, arena);
  else if (width == 8)
    k_gather_encode_nullable<8><<<(unsigned)ntiles, kThreads, 0, ctx->stream>>>(tiles, perm, src, valid, tile_value_offset,
                                                                                 tile_def_offset, arena);
  else if (width == 4)
    k_gather_encode_nullable<4><<<(unsigned)ntiles, kThreads, 0, ctx->stream>>>(tiles, perm, src, valid, tile_value_offset,
                                                                                 tile_def_offset, arena);
  else
    fail(HS_EUNSUPPORTED, "gather_encode_nullable: column width %d", width);
  HS_LAUNCH_CHECK(ctx);
}

void launch_tile_string_sizes(hs_ctx* ctx, const SortTile* tiles, int64_t ntiles, const uint32_t* perm, const uint64_t* refs,
                              const uint8_t* valid, uint32_t* bytes, uint32_t* counts) {
  KernelScope _ks(ctx, "k_tile_string_sizes");
  if (ntiles == 0) return;
  k_tile_string_sizes<<<(unsigned)ntiles, kThreads, 0, ctx->stream>>>(tiles, perm, refs, valid, bytes, counts);
  HS_LAUNCH_CHECK(ctx);
}

void launch_gather_encode_strings(hs_ctx* ctx, const SortTile* tiles, int64_t ntiles, const uint32_t* perm, const uint64_t* refs,
                                  const uint8_t* valid, const uint64_t* tile_value_offset, const uint64_t* tile_def_offset,
                                  uint8_t* arena) {
  KernelScope _ks(ctx, "k_gather_encode_strings");
  if (ntiles == 0) return;
  k_gather_encode_strings<<<(unsigned)ntiles, kThreads, 0, ctx->stream>>>(tiles, perm, refs, valid, tile_value_offset,
                                                                          tile_def_offset, arena);
  HS_LAUNCH_CHECK(ctx);
}

void launch_copy_blobs(hs_ctx* ctx, const BlobCopy* blobs, int64_t n, const uint8_t* src_base, uint8_t* dst_base) {
  KernelScope _ks(ctx, "k_copy_blobs");
  if (n == 0) return;
  k_copy_blobs<<<(unsigned)n, 256, 0, ctx->stream>>>(blobs, src_base, dst_base);
  HS_LAUNCH_CHECK(ctx);
}

void launch_gather_plain(hs_ctx* ctx, const void* src, const uint32_t* perm, int64_t n, int width, void* out) {
  KernelScope _ks(ctx, "k_gather_plain");
  if (n == 0) return;
  const int grid = grid_for(ctx, n, 256, 16);
  switch (width) {
    case 8: k_gather_plain<uint64_t><<<grid, 256, 0, ctx->stream>>>((const uint64_t*)src, perm, n, (uint64_t*)out); break;
    case 4: k_gather_plain<uint32_t><<<grid, 256, 0, ctx->stream>>>((const uint32_t*)src, perm, n, (uint32_t*)out); break;
    case 1: k_gather_plain<uint8_t><<<grid, 256, 0, ctx->stream>>>((const uint8_t*)src, perm, n, (uint8_t*)out); break;
    default: fail(HS_EINVAL, "gather: unsupported width %d", width);
  }
  HS_LAUNCH_CHECK(ctx);
}

void launch_scatter_bytes(hs_ctx* ctx, const ByteCopy* copies, int64_t n, const uint8_t* skeleton, uint8_t* arena) {
  if (n == 0) return;
  const int64_t threads = n * 32;
  k_scatter_bytes<<<(unsigned)ceil_div(threads, 256), 256, 0, ctx->stream>>>(copies, n, skeleton, arena);
  HS_LAUNCH_CHECK(ctx);
}

void launch_patch_key_stats(hs_ctx* ctx, const StatPatch* patches, int64_t n, const uint32_t* perm, const void* keys,
                            uint8_t* arena) {
  if (n == 0) return;
  k_patch_key_stats<<<(unsigned)ceil_div(n, 128), 128, 0, ctx->stream>>>(patches, n, perm, keys, arena);
  HS_LAUNCH_CHECK(ctx);
}

void launch_synth_column(hs_ctx* ctx, int col, int64_t first_row, int64_t n, void* out) {
  KernelScope _ks(ctx, "k_synth_column");
  if (n == 0) return;
  k_synth_column<<<grid_for(ctx, n, 256, 16), 256, 0, ctx->stream>>>(col, first_row, n, out);
  HS_LAUNCH_CHECK(ctx);
}

}  // namespace hs
