// dict_encode.cu -- dictionary encoding on the GPU (PLAIN_DICTIONARY pages with bit-packed indices).
//
// parquet-mr, which writes the reference's index files (index/DataFrameWriterExtensions.scala:58-67 -> ParquetOutputWriter),
// dictionary-encodes every column chunk whose distinct values fit its dictionary page and falls back to PLAIN otherwise.
// Here: one open-addressing hash set per candidate column (64-bit CAS on the raw value bits, no locks) collects the
// distinct values of the whole column and gives up as soon as more than kMaxDictEntries are seen; the host sorts the
// (small) dictionary, maps every table slot to its dictionary index, and k_dict_encode looks each gathered value up and
// bit-packs the indices of a 4096-row tile in shared memory.  For the benchmark table this shrinks v1/v3/v4 from
// 8/4/4 bytes per row to 10/7/12 bits, i.e. 32 -> 19.7 bytes per row over PCIe and on disk.
#include "device_utils.cuh"
#include "kernels.h"

namespace hs {

namespace {

constexpr unsigned long long kEmpty = 0xFFFFFFFFFFFFFFFFull;
constexpr int kThreads = 256;

// Fibonacci hashing: one 64-bit multiply; the top bits of the product depend on every input bit
__device__ __forceinline__ uint32_t dict_hash(uint64_t v) { return dict_hash_u64(v); }

// Column values are read exactly once: streaming (evict-first) loads keep them from evicting the few hot lines of the
// hash table out of L1 (with default caching the look-ups went to L2: ~6 sector requests per row, L2-request bound).
__device__ __forceinline__ uint64_t load_raw_value(const void* src, int width, int64_t i) {
  return width == 8 ? __ldcs((const unsigned long long*)src + i) : (uint64_t)__ldcs((const unsigned int*)src + i);
}

// state[0] = number of distinct values inserted, state[1] = overflow flag, state[2] = the value kEmpty itself occurs
__global__ void __launch_bounds__(kThreads) k_dict_build(const void* __restrict__ src, int width, int64_t begin, int64_t end,
                                                          unsigned long long* __restrict__ keys, uint32_t mask,
                                                          uint32_t max_distinct, uint32_t* __restrict__ state) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  uint32_t it = 0;
  for (int64_t i0 = begin + (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i0 < end; i0 += 2 * stride, it++) {
    // the overflow flag lives in one L2 line: polling it for every element serialises the whole grid on that line,
    // so look only every 32 iterations
    if ((it & 31) == 0 && *(volatile uint32_t*)&state[1]) return;
    const int64_t i1 = i0 + stride;
    uint64_t vals[2];
    vals[0] = load_raw_value(src, width, i0);
    vals[1] = i1 < end ? load_raw_value(src, width, i1) : vals[0];  // two independent loads in flight
#pragma unroll
    for (int u = 0; u < 2; u++) {
      const uint64_t v = vals[u];
      if (v == kEmpty) {
        state[2] = 1;
        continue;
      }
      uint32_t h = dict_hash(v) & mask;
      // A thread counts an insert only while the distinct count is still below max_distinct; threads that passed that
      // check concurrently can overshoot by at most two inserts each, and the launcher caps the grid so that
      // max_distinct + 2 * #threads stays below the table capacity: the table never fills, probing terminates.  At the
      // limit only a value that wins an empty slot is new: another thread may be inserting the same value right now.
      for (uint32_t probes = 0; probes <= mask; probes++) {
        const unsigned long long cur = keys[h];
        if (cur == v) break;
        if (cur == kEmpty) {
          const bool full = *(volatile uint32_t*)&state[0] >= max_distinct;
          const unsigned long long old = atomicCAS(&keys[h], kEmpty, (unsigned long long)v);
          if (old == kEmpty) {
            if (full) {
              state[1] = 1;
              return;
            }
            atomicAdd(&state[0], 1u);
            break;
          }
          if (old == v) break;
        }
        h = (h + 1) & mask;
      }
    }
  }
}

// Hash set filled from the dictionary pages of the source chunks (one CTA per data page; pages of one chunk insert the same
// few values again).  Used when every page of a column was dictionary-encoded; entries no row uses stay in the set.
__global__ void __launch_bounds__(kThreads) k_dict_build_from_pages(const PageDesc* __restrict__ pages, int col, int width,
                                                                     unsigned long long* __restrict__ keys, uint32_t mask,
                                                                     uint32_t max_distinct, uint32_t* __restrict__ state) {
  const PageDesc pg = pages[blockIdx.x];
  if (pg.col != col || pg.dict == nullptr) return;
  for (int i = threadIdx.x; i < pg.dict_count; i += kThreads) {
    if (*(volatile uint32_t*)&state[1]) return;
    const uint8_t* p = pg.dict + (size_t)i * width;
    const uint64_t v = width == 8 ? load_le64_unaligned(p) : (uint64_t)load_le32_unaligned(p);
    if (v == kEmpty) {
      state[2] = 1;
      continue;
    }
    uint32_t h = dict_hash(v) & mask;
    for (uint32_t probes = 0; probes <= mask; probes++) {  // the insert of k_dict_build
      const unsigned long long cur = keys[h];
      if (cur == v) break;
      if (cur == kEmpty) {
        const bool full = *(volatile uint32_t*)&state[0] >= max_distinct;
        const unsigned long long old = atomicCAS(&keys[h], kEmpty, (unsigned long long)v);
        if (old == kEmpty) {
          if (full) {
            state[1] = 1;
            return;
          }
          atomicAdd(&state[0], 1u);
          break;
        }
        if (old == v) break;
      }
      h = (h + 1) & mask;
    }
  }
}

// distinct values out of the hash set (order arbitrary; the host sorts the small list)
__global__ void k_dict_collect(const unsigned long long* __restrict__ keys, uint32_t capacity,
                               unsigned long long* __restrict__ out, uint32_t* __restrict__ counter, uint32_t max_out) {
  const uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= capacity) return;
  const unsigned long long v = keys[s];
  if (v != kEmpty) {
    const uint32_t at = atomicAdd(counter, 1u);
    if (at < max_out) out[at] = v;
  }
}

// ---- all dictionary columns at once ---------------------------------------------------------------------------------
// k_dict_map_all writes ONE record per row holding the 16-bit indices of every dictionary column (4 or 8 slots), so
// that k_dict_pack_all fetches all of a row's indices with a single 32-byte L2 sector request instead of one request per
// column (the single-column pack kernel was bound by L2 sector requests, not by DRAM).
template <int SLOTS>
__global__ void __launch_bounds__(kThreads) k_dict_map_all(DictMapArgs a, int64_t n, uint16_t* __restrict__ rec) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    uint64_t v[SLOTS];
#pragma unroll
    for (int c = 0; c < SLOTS; c++) v[c] = c < a.ncols ? load_raw_value(a.src[c], a.width[c], i) : kEmpty;
    uint16_t ix[SLOTS];
#pragma unroll
    for (int c = 0; c < SLOTS; c++) {
      uint32_t x = 0;
      if (c < a.ncols) {
        x = a.empty_index[c];
        if (v[c] != kEmpty) {
          const uint32_t mask = a.mask[c];
          uint32_t h = dict_hash(v[c]) & mask;
          const uint4* tab = reinterpret_cast<const uint4*>(a.entries[c]);
          const uint32_t vlo = (uint32_t)v[c], vhi = (uint32_t)(v[c] >> 32);
          uint4 e = tab[h];
          uint32_t probes = 0;
          while ((e.x != vlo || e.y != vhi) && probes++ <= mask) {  // present by construction; bounded regardless
            h = (h + 1) & mask;
            e = tab[h];
          }
          x = e.z;
        }
      }
      ix[c] = (uint16_t)x;
    }
    if (SLOTS == 4) {
      __stcs(reinterpret_cast<uint2*>(rec) + i, make_uint2((uint32_t)ix[0] | ((uint32_t)ix[1] << 16), (uint32_t)ix[2] | ((uint32_t)ix[3] << 16)));
    } else {
      __stcs(reinterpret_cast<uint4*>(rec) + i, make_uint4((uint32_t)ix[0] | ((uint32_t)ix[1] << 16), (uint32_t)ix[2] | ((uint32_t)ix[3] << 16),
                                                   (uint32_t)ix[SLOTS > 4 ? 4 : 0] | ((uint32_t)ix[SLOTS > 5 ? 5 : 0] << 16),
                                                   (uint32_t)ix[SLOTS > 6 ? 6 : 0] | ((uint32_t)ix[SLOTS > 7 ? 7 : 0] << 16)));
    }
  }
}

template <int SLOTS>
__global__ void __launch_bounds__(kThreads, 4) k_dict_pack_all(const SortTile* __restrict__ tiles,
                                                                const uint64_t* __restrict__ seg_start,
                                                                const uint32_t* __restrict__ perm,
                                                                const uint16_t* __restrict__ rec, DictPackArgs a,
                                                                const uint32_t* __restrict__ bucket_page_begin,
                                                                int64_t rows_per_page, uint8_t* __restrict__ arena) {
  extern __shared__ __align__(16) uint8_t s_all[];  // ncols x (kSortTile / 8 * 16) bytes
  constexpr uint32_t kColBytes = kSortTile / 8 * 16;
  constexpr int kWords = SLOTS / 2;  // 32-bit words per record
  const SortTile t = tiles[blockIdx.x];
  const uint32_t ngroups = (t.count + 7) / 8;
  for (uint32_t g = threadIdx.x; g < ngroups; g += kThreads) {
    uint32_t r[8][kWords];  // the eight records of the group, still packed (two 16-bit indices per word)
#pragma unroll
    for (int j = 0; j < 8; j++) {
      const uint32_t i = g * 8 + j;
#pragma unroll
      for (int w = 0; w < kWords; w++) r[j][w] = 0;  // padding indices of the last group are zero
      if (i < t.count) {
        const uint32_t row = perm[t.start + i];
        if (SLOTS == 4) {
          const uint2 q = reinterpret_cast<const uint2*>(rec)[row];
          r[j][0] = q.x;
          r[j][1] = q.y;
        } else {
          const uint4 q = reinterpret_cast<const uint4*>(rec)[row];
          r[j][0] = q.x;
          r[j][1] = q.y;
          r[j][kWords > 2 ? 2 : 0] = q.z;
          r[j][kWords > 3 ? 3 : 0] = q.w;
        }
      }
    }
#pragma unroll
    for (int c = 0; c < SLOTS; c++) {
      if (c < a.ncols) {
        const uint32_t bw = a.bw[c];
        unsigned long long lo = 0, hi = 0;  // 8 x bw <= 128 bits, LSB first
#pragma unroll
        for (int j = 0; j < 8; j++) {
          const unsigned long long ix = (r[j][c >> 1] >> ((c & 1) * 16)) & 0xffffu;
          const uint32_t bit = j * bw;
          if (bit < 64) {
            lo |= ix << bit;
            if (bit + bw > 64) hi |= ix >> (64 - bit);
          } else {
            hi |= ix << (bit - 64);
          }
        }
        uint8_t* dst = s_all + (size_t)c * kColBytes + (size_t)g * bw;
        for (uint32_t b = 0; b < bw; b++) dst[b] = (uint8_t)(b < 8 ? (lo >> (8 * b)) : (hi >> (8 * (b - 8))));
      }
    }
  }
  __syncthreads();
  const uint64_t lr0 = t.start - seg_start[t.seg];
  const uint64_t page = lr0 / (uint64_t)rows_per_page;
  const uint64_t in_page = lr0 - page * (uint64_t)rows_per_page;
  const uint32_t gpage = bucket_page_begin[t.seg] + (uint32_t)page;
#pragma unroll
  for (int c = 0; c < SLOTS; c++) {
    if (c < a.ncols) {
      const uint32_t bw = a.bw[c];
      const uint8_t* sb = s_all + (size_t)c * kColBytes;
      uint8_t* const out = arena + a.page_value_offset[c][gpage] + in_page * bw / 8;
      const uint32_t nbytes = ngroups * bw;
      const uint32_t head = min(nbytes, (uint32_t)((4 - ((uintptr_t)out & 3)) & 3));
      for (uint32_t b = threadIdx.x; b < head; b += kThreads) out[b] = sb[b];
      const uint32_t nwords = (nbytes - head) / 4;
      uint32_t* out32 = reinterpret_cast<uint32_t*>(out + head);
      for (uint32_t w = threadIdx.x; w < nwords; w += kThreads) {
        const uint8_t* p = sb + head + 4 * w;
        out32[w] = (uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) | ((uint32_t)p[3] << 24);
      }
      for (uint32_t b = head + 4 * nwords + threadIdx.x; b < nbytes; b += kThreads) out[b] = sb[b];
    }
  }
}

inline int grid_for(hs_ctx* ctx, int64_t n, int threads, int per_sm) {
  int64_t want = ceil_div(n, threads);
  int64_t cap = (int64_t)ctx->sm_count * per_sm;
  return (int)std::max<int64_t>(1, std::min(want, cap));
}

}  // namespace

void launch_dict_build(hs_ctx* ctx, const void* src, int width, int64_t begin, int64_t end, unsigned long long* keys,
                       uint32_t capacity, uint32_t max_distinct, uint32_t* state) {
  KernelScope _ks(ctx, "k_dict_build");
  if (end <= begin) return;
  // grid * 256 threads * 2 values + max_distinct < capacity: see the capacity argument in k_dict_build
  int grid = grid_for(ctx, end - begin, kThreads * 2, 6);
  while ((uint64_t)grid * kThreads * 2 + max_distinct >= capacity && grid > 1) grid /= 2;
  k_dict_build<<<grid, kThreads, 0, ctx->stream>>>(src, width, begin, end, keys, capacity - 1, max_distinct, state);
  HS_LAUNCH_CHECK(ctx);
}

void launch_dict_build_from_pages(hs_ctx* ctx, const PageDesc* pages, int64_t n_pages, int col, int width,
                                  unsigned long long* keys, uint32_t capacity, uint32_t max_distinct, uint32_t* state) {
  KernelScope _ks(ctx, "k_dict_build_from_pages");
  if (n_pages == 0) return;
  // one CTA per page, 256 threads: at most n_pages * 256 concurrent inserts; the table has capacity - max_distinct spare
  // slots and a dictionary page rarely has more than a few thousand entries, but keep the bound explicit:
  const int64_t max_ctas = (capacity - max_distinct) / kThreads - 1;
  for (int64_t p0 = 0; p0 < n_pages; p0 += max_ctas) {
    const unsigned grid = (unsigned)std::min<int64_t>(max_ctas, n_pages - p0);
    k_dict_build_from_pages<<<grid, kThreads, 0, ctx->stream>>>(pages + p0, col, width, keys, capacity - 1, max_distinct, state);
    HS_LAUNCH_CHECK(ctx);
  }
}

void launch_dict_collect(hs_ctx* ctx, const unsigned long long* keys, uint32_t capacity, unsigned long long* out,
                         uint32_t* counter, uint32_t max_out) {
  k_dict_collect<<<(capacity + 255) / 256, 256, 0, ctx->stream>>>(keys, capacity, out, counter, max_out);
  HS_LAUNCH_CHECK(ctx);
}

void launch_dict_pack(hs_ctx* ctx, const SortTile* tiles, int64_t ntiles, const uint64_t* seg_start, const uint32_t* perm,
                      const DictPackArgs& pack_args, int slots, const uint16_t* rec, const uint32_t* bucket_page_begin,
                      int64_t rows_per_page, uint8_t* arena) {
  KernelScope _ks(ctx, "k_dict_pack");
  if (ntiles == 0) return;
  const size_t smem = (size_t)pack_args.ncols * (kSortTile / 8 * 16);
  static DeviceOnce attr_once;
  bool& attr = attr_once(ctx->device);
  if (!attr) {
    HS_CUDA(cudaFuncSetAttribute(k_dict_pack_all<4>, cudaFuncAttributeMaxDynamicSharedMemorySize, 4 * (kSortTile / 8 * 16)));
    HS_CUDA(cudaFuncSetAttribute(k_dict_pack_all<8>, cudaFuncAttributeMaxDynamicSharedMemorySize, 8 * (kSortTile / 8 * 16)));
    attr = true;
  }
  if (slots == 4)
    k_dict_pack_all<4><<<(unsigned)ntiles, kThreads, smem, ctx->stream>>>(tiles, seg_start, perm, rec, pack_args,
                                                                         bucket_page_begin, rows_per_page, arena);
  else
    k_dict_pack_all<8><<<(unsigned)ntiles, kThreads, smem, ctx->stream>>>(tiles, seg_start, perm, rec, pack_args,
                                                                         bucket_page_begin, rows_per_page, arena);
  HS_LAUNCH_CHECK(ctx);
}

void launch_dict_encode_all(hs_ctx* ctx, const SortTile* tiles, int64_t ntiles, const uint64_t* seg_start, const uint32_t* perm,
                            const DictMapArgs& map_args, const DictPackArgs& pack_args, int64_t nrows, uint32_t capacity,
                            uint16_t* rec_scratch, const uint32_t* bucket_page_begin, int64_t rows_per_page, uint8_t* arena) {
  if (ntiles == 0) return;
  (void)capacity;
  const int slots = map_args.ncols <= 4 ? 4 : 8;
  {
    KernelScope _ks(ctx, "k_dict_map");
    const int grid = grid_for(ctx, nrows, kThreads, 16);
    if (slots == 4) k_dict_map_all<4><<<grid, kThreads, 0, ctx->stream>>>(map_args, nrows, rec_scratch);
    else k_dict_map_all<8><<<grid, kThreads, 0, ctx->stream>>>(map_args, nrows, rec_scratch);
    HS_LAUNCH_CHECK(ctx);
  }
  launch_dict_pack(ctx, tiles, ntiles, seg_start, perm, pack_args, slots, rec_scratch, bucket_page_begin, rows_per_page, arena);
}

}  // namespace hs
