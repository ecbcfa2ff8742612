// radix_sort.cu -- K4: segmented stable LSD radix sort of (encoded key u64, row index u32) pairs.
//
// Replaces the per-bucket SortExec Spark's FileFormatWriter adds for BucketSpec(n, cols, cols)
// (index/DataFrameWriterExtensions.scala:64; SURVEY.md section 3.1 HOT LOOP 2: UnsafeExternalRowSorter).  Each bucket is a
// segment; tiles of 4096 pairs never straddle segments, so one launch per pass sorts all buckets at once.
//
// Per 8-bit digit pass:  k_sort_hist (tile digit histograms) -> k_seg_* (per-segment column scan giving every
// (tile, digit) its global destination) -> k_sort_scatter (stable in-tile ranking with __match_any_sync, exchange
// through shared memory so each digit's items leave the tile as one contiguous run).  Passes whose digit is constant
// over the whole input (OR == AND on those bits) are skipped.
//
// k_local_sort finishes ranges that fit one CTA in shared memory: whole small segments straight from the raw column, or
// the (segment, digit) sub-buckets of one MSD pass -- two HBM passes for keys whose LSD sort would take three or more.
//
// sort_rows() is the module's one entry point and makes every choice between these paths, from shapes the host knows:
// a null-free int32 / int64 / float / double first key column takes k_local_sort when it can (HS_LSD_SORT=1 turns that
// off for A/B measurements); other keys take LSD passes over their top varying bytes plus k_fix_runs, or over every
// varying byte.  When k_fix_runs gives up on a long run, the rows are sorted again with full passes -- at once, or in
// settle_sorted_rows() when the caller let the verdict wait for its next synchronisation.
#include <cmath>

#include "device_utils.cuh"
#include "kernels.h"

namespace hs {

struct SortChunk {  // up to kChunkTiles consecutive tiles of one segment: the unit of the per-segment scan
  uint32_t seg;
  uint32_t tile_begin, tile_end;
};

namespace {

constexpr int kThreads = 512;                  // 512 x 8 items: <= 64 registers -> 2 CTAs (32 warps) per SM
constexpr int kWarps = kThreads / 32;
constexpr int kItems = kSortTile / kThreads;   // 8
constexpr int kWarpRows = kSortTile / kWarps;  // 256 consecutive pairs per warp
constexpr int kChunkTiles = 128;
constexpr int kHistThreads = 256;

struct DigitShift {
  int shift;
  __device__ __forceinline__ uint32_t operator()(uint64_t key, uint32_t) const { return (uint32_t)(key >> shift) & 255u; }
};
struct DigitTable {
  const uint8_t* table;
  __device__ __forceinline__ uint32_t operator()(uint64_t, uint32_t val) const { return table[val]; }
};

// Where a pass reads its (key, row) pairs from: the ping-pong arrays, or -- for the first pass over a freshly partitioned
// key column -- the raw column itself, encoded on the fly with the row's own position as its value (so the encoded-key
// and iota arrays are never materialised).
struct SrcPairs {
  const uint64_t* __restrict__ keys;
  const uint32_t* __restrict__ vals;
  __device__ __forceinline__ void load(uint64_t p, uint64_t& k, uint32_t& v) const {
    k = keys[p];
    v = vals[p];
  }
};
template <int TYPE>  // HS_TYPE_*: a compile-time type keeps the loads of a thread's items back to back
struct SrcRaw {
  const void* __restrict__ raw;
  __device__ __forceinline__ void load(uint64_t p, uint64_t& k, uint32_t& v) const {
    const uint64_t r = (TYPE == HS_TYPE_INT64 || TYPE == HS_TYPE_DOUBLE) ? ((const uint64_t*)raw)[p]
                                                                          : (uint64_t)((const uint32_t*)raw)[p];
    k = sort_encode(TYPE, r);
    v = (uint32_t)p;
  }
};

template <typename Src, typename Digit>
__global__ void __launch_bounds__(kHistThreads) k_sort_hist(const SortTile* __restrict__ tiles, Src src, Digit digit,
                                                         uint32_t* __restrict__ tile_hist) {
  __shared__ uint32_t s_hist[256];
  s_hist[threadIdx.x] = 0;
  __syncthreads();
  const SortTile t = tiles[blockIdx.x];
  for (uint32_t i = threadIdx.x; i < t.count; i += kHistThreads) {
    uint64_t k;
    uint32_t v;
    src.load(t.start + i, k, v);
    atomicAdd(&s_hist[digit(k, v)], 1u);
  }
  __syncthreads();
  tile_hist[(size_t)blockIdx.x * 256 + threadIdx.x] = s_hist[threadIdx.x];
}

// A: per chunk, per digit sums
__global__ void __launch_bounds__(256) k_seg_chunk_sums(const SortChunk* __restrict__ chunks,
                                                         const uint32_t* __restrict__ tile_hist,
                                                         uint32_t* __restrict__ chunk_sums) {
  const SortChunk c = chunks[blockIdx.x];
  uint32_t s = 0;
  for (uint32_t t = c.tile_begin; t < c.tile_end; t++) s += tile_hist[(size_t)t * 256 + threadIdx.x];
  chunk_sums[(size_t)blockIdx.x * 256 + threadIdx.x] = s;
}

// B: one CTA per segment: prefix over the segment's chunks, then digit bases (also written to digit_base[seg * 256 + digit]
// when it is given: the first position of every (segment, digit) sub-bucket)
__global__ void __launch_bounds__(256) k_seg_scan(const uint32_t* __restrict__ seg_chunk_begin,
                                                   const uint64_t* __restrict__ seg_start,
                                                   uint32_t* __restrict__ chunk_sums, uint32_t* __restrict__ digit_base) {
  __shared__ uint32_t warp_sums[40];
  const uint32_t seg = blockIdx.x;
  const uint32_t c0 = seg_chunk_begin[seg], c1 = seg_chunk_begin[seg + 1];
  uint32_t tot = 0;
  for (uint32_t c = c0; c < c1; c++) {
    const uint32_t v = chunk_sums[(size_t)c * 256 + threadIdx.x];
    chunk_sums[(size_t)c * 256 + threadIdx.x] = tot;
    tot += v;
  }
  const uint32_t dbase = block_exclusive_scan(tot, warp_sums, nullptr) + (uint32_t)seg_start[seg];
  if (digit_base) digit_base[(size_t)seg * 256 + threadIdx.x] = dbase;
  for (uint32_t c = c0; c < c1; c++) chunk_sums[(size_t)c * 256 + threadIdx.x] += dbase;
}

// C: per chunk, turn tile histograms into destinations.  1024 threads = 4 groups x 256 digits; each group owns a
// quarter of the chunk's tiles.  Input and output are distinct arrays so the loads can be issued ahead of the stores.
__global__ void __launch_bounds__(1024) k_seg_apply(const SortChunk* __restrict__ chunks,
                                                     const uint32_t* __restrict__ tile_hist,
                                                     uint32_t* __restrict__ tile_dst,
                                                     const uint32_t* __restrict__ chunk_sums) {
  __shared__ uint32_t s_group[4][256];
  const SortChunk c = chunks[blockIdx.x];
  const uint32_t d = threadIdx.x & 255, g = threadIdx.x >> 8;
  const uint32_t n = c.tile_end - c.tile_begin;
  const uint32_t per = (n + 3) / 4;
  const uint32_t t0 = c.tile_begin + min(g * per, n), t1 = c.tile_begin + min((g + 1) * per, n);
  uint32_t s = 0;
#pragma unroll 8
  for (uint32_t t = t0; t < t1; t++) s += tile_hist[(size_t)t * 256 + d];
  s_group[g][d] = s;
  __syncthreads();
  uint32_t run = chunk_sums[(size_t)blockIdx.x * 256 + d];
  for (uint32_t gg = 0; gg < g; gg++) run += s_group[gg][d];
#pragma unroll 8
  for (uint32_t t = t0; t < t1; t++) {
    const uint32_t v = tile_hist[(size_t)t * 256 + d];
    tile_dst[(size_t)t * 256 + d] = run;
    run += v;
  }
}

// Stable ranking of a tile's items on their 8-bit digits, shared by k_sort_scatter and local_pass.  W warps, I items per
// lane: item j of a lane is the tile's item warp * I * 32 + j * 32 + lane, with digit bin(j).  On return rank[j] is the
// item's rank among its warp's earlier items with the same digit and cnt[w][d] the first tile position of (warp w,
// digit d); the result is the first tile position of digit threadIdx.x (threads below 256).  cnt must be zero, and the
// block synchronised since it was zeroed.  kGuard: only items below `count` are ranked, tested per warp row (warp-
// uniform); otherwise every slot is, and slots past the end must carry the digit 255 (see k_sort_scatter).
template <int W, int I, bool kGuard, typename Bin>
__device__ __forceinline__ uint32_t rank_tile(uint16_t (&cnt)[W][256], uint32_t* warp_sums, Bin bin, uint32_t count,
                                              uint32_t (&rank)[I]) {
  const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const unsigned lt = (1u << lane) - 1;
  uint16_t* wcnt = cnt[warp];
#pragma unroll
  for (int j = 0; j < I; j++) {
    rank[j] = 0;
    if (!kGuard || warp * (I * 32) + j * 32 < count) {
      const uint32_t b = bin(j);
      const unsigned peers = match_any_full<8>(b);
      const uint32_t before = __popc(peers & lt);
      const uint32_t pre = wcnt[b];   // every peer reads the same counter (broadcast)
      __syncwarp();
      if (before == 0) wcnt[b] = (uint16_t)(pre + __popc(peers));
      __syncwarp();
      rank[j] = pre + before;
    }
  }
  __syncthreads();
  // per digit: exclusive prefix over warps and digits -> first in-tile position of every (warp, digit)
  uint32_t total = 0;
  if (threadIdx.x < 256) {
#pragma unroll
    for (int w = 0; w < W; w++) total += cnt[w][threadIdx.x];
  }
  const uint32_t start = block_exclusive_scan(total, warp_sums, nullptr);
  if (threadIdx.x < 256) {
    uint32_t run = start;
#pragma unroll
    for (int w = 0; w < W; w++) {
      const uint16_t c = cnt[w][threadIdx.x];
      cnt[w][threadIdx.x] = (uint16_t)run;
      run += c;
    }
  }
  return start;
}

struct ScatterShared {
  uint64_t keys[kSortTile];
  uint32_t vals[kSortTile];
  uint16_t cnt[kWarps][256];   // ranking: per-warp digit counts; afterwards: first in-tile position of (warp, digit)
  uint32_t out_adj[256];       // global destination of a digit's run minus its first in-tile position
  uint32_t warp_sums[40];
};

// All warp-collectives below run with the full mask and outside any branch: slots past the end of a partial tile carry
// digit 255 and, being the last slots of the tile, rank behind every real item of that digit, so they never disturb a
// real item's position and are simply not written out.
template <typename Src, typename Digit>
__global__ void __launch_bounds__(kThreads, 2) k_sort_scatter(const SortTile* __restrict__ tiles, Src src, Digit digit,
                                                               const uint32_t* __restrict__ tile_dst,
                                                               uint64_t* __restrict__ out_keys,
                                                               uint32_t* __restrict__ out_vals) {
  extern __shared__ __align__(16) uint8_t smem_raw[];
  ScatterShared& sm = *reinterpret_cast<ScatterShared*>(smem_raw);
  const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  {
    uint32_t* z = reinterpret_cast<uint32_t*>(&sm.cnt[0][0]);
#pragma unroll
    for (int i = 0; i < kWarps * 256 / 2 / kThreads; i++) z[threadIdx.x + i * kThreads] = 0;
  }
  const SortTile t = tiles[blockIdx.x];
  uint32_t dst0 = 0;
  if (threadIdx.x < 256) dst0 = tile_dst[(size_t)blockIdx.x * 256 + threadIdx.x];
  const uint32_t first = warp * kWarpRows + lane;
  const uint64_t p0 = t.start + first;
  uint64_t k[kItems];
  uint32_t v[kItems];
  uint32_t bin[kItems];
#pragma unroll
  for (int j = 0; j < kItems; j++) {
    const bool a = first + j * 32 < t.count;
    k[j] = ~0ull;
    v[j] = 0;
    if (a) src.load(p0 + j * 32, k[j], v[j]);
    bin[j] = a ? digit(k[j], v[j]) : 255u;
  }
  __syncthreads();
  uint32_t rank[kItems];
  const uint32_t start = rank_tile<kWarps, kItems, false>(sm.cnt, sm.warp_sums, [&](int j) { return bin[j]; }, 0, rank);
  if (threadIdx.x < 256) sm.out_adj[threadIdx.x] = dst0 - start;
  __syncthreads();
  // exchange: digit-sorted order inside the tile
  const uint16_t* cnt = sm.cnt[warp];
#pragma unroll
  for (int j = 0; j < kItems; j++) {
    const uint32_t pos = cnt[bin[j]] + rank[j];
    sm.keys[pos] = k[j];
    sm.vals[pos] = v[j];
  }
  __syncthreads();
#pragma unroll
  for (int j = 0; j < kItems; j++) {
    const uint32_t i = threadIdx.x + j * kThreads;
    if (i < t.count) {
      const uint64_t key = sm.keys[i];
      const uint32_t val = sm.vals[i];
      const uint32_t dst = sm.out_adj[digit(key, val)] + i;
      out_keys[dst] = key;
      out_vals[dst] = val;
    }
  }
}

// ---- tie-run fix-up ---------------------------------------------------------------------------------------------
// After the stable LSD passes over the HIGH bytes of the key, rows are ordered by (key & high_mask) and rows that share
// those bits still sit in their original relative order.  For high-entropy keys such runs are rare and tiny, so instead
// of four more full passes over the data the head of every run insertion-sorts it (stably) on (key & low_mask).  A run
// longer than max_run raises `flag`; the caller then falls back to full LSD passes, which is still correct because equal
// full keys are in original order both inside untouched runs and inside insertion-sorted ones.
//
// Two phases per tile so that the divergent part runs with full warps: (1) every thread tests its rows for "head of a
// run of two or more" -- a straight-line compare against both neighbours -- and the heads are compacted into a list in
// shared memory; (2) the threads walk that list, one run each.  With 24 sorted bits and 5 M-row buckets about a quarter
// of the rows head such a run; testing and sorting in the same loop left three quarters of every warp idle.
constexpr uint32_t kFixMaxRun = 64;
__global__ void __launch_bounds__(256) k_fix_runs(const SortTile* __restrict__ tiles, const uint64_t* __restrict__ seg_start,
                                                   uint64_t* __restrict__ keys, uint32_t* __restrict__ vals,
                                                   uint64_t high_mask, uint64_t low_mask, uint32_t max_run,
                                                   uint32_t* __restrict__ flag) {
  // The tile's keys are staged in shared memory with all of a thread's loads in flight at once: s_key[1 + i] = key of row i
  // of the tile, [0] / [count + 1] = the rows just outside it (or a key with a different prefix where the segment ends).
  // Run detection, the walk to the end of a run and the order test then never leave shared memory; global memory is touched
  // again only for the rows an out-of-order run actually moves.  With 5 M-row buckets one row in eight heads a run: doing
  // all of that through dependent global loads was latency-bound.
  __shared__ uint64_t s_key[kSortTile + 2];
  __shared__ uint16_t s_heads[kSortTile / 2], s_len[kSortTile / 2];  // 8 warps x 256 entries
  const SortTile t = tiles[blockIdx.x];
  const uint64_t segb = seg_start[t.seg], sege = seg_start[t.seg + 1];
  const unsigned lane = threadIdx.x & 31, lt = (1u << lane) - 1;
  constexpr int kPer = kSortTile / 256;
  {
    uint64_t k[kPer];
#pragma unroll
    for (int j = 0; j < kPer; j++) {
      const uint32_t i = j * 256 + threadIdx.x;
      k[j] = i < t.count ? keys[t.start + i] : 0;
    }
#pragma unroll
    for (int j = 0; j < kPer; j++) s_key[1 + j * 256 + threadIdx.x] = k[j];
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    const uint64_t flip = high_mask & (~high_mask + 1);  // lowest bit of the prefix: flipping it makes a different prefix
    s_key[0] = t.start > segb ? keys[t.start - 1] : (s_key[1] ^ flip);
    s_key[t.count + 1] = t.start + t.count < sege ? keys[t.start + t.count] : (s_key[t.count] ^ flip);
  }
  __syncthreads();
  // every warp keeps its own list of heads (a warp's rows give at most 256: a head needs a row behind it), so building the
  // lists takes no atomics and no block-wide counter -- 128 contended shared-memory atomics per tile, each followed by a
  // dependent shuffle, were a third of this kernel's time
  const uint32_t wid = threadIdx.x >> 5;
  uint16_t* my_heads = s_heads + wid * (kSortTile / 16);
  uint16_t* my_len = s_len + wid * (kSortTile / 16);
  uint32_t my_n = 0;
#pragma unroll 4
  for (uint32_t i0 = 0; i0 < kSortTile; i0 += 256) {  // uniform trip count: the ballot below needs whole warps
    const uint32_t i = i0 + threadIdx.x;
    bool head = false;
    if (i < t.count) {
      const uint64_t kh = s_key[1 + i] & high_mask;
      head = (s_key[i] & high_mask) != kh && (s_key[2 + i] & high_mask) == kh;
    }
    const unsigned m = __ballot_sync(0xffffffffu, head);
    if (head) my_heads[my_n + __popc(m & lt)] = (uint16_t)i;
    my_n += __popc(m);
  }
  __syncwarp();
  // first every run is measured (reads only: a walk looks one key past its run, i.e. at the head of the next one), then,
  // behind a barrier, every run is sorted (writes stay inside the run)
  for (uint32_t e = lane; e < my_n; e += 32) {
    const uint32_t i = my_heads[e];
    const uint64_t* sk = s_key + 1 + i;
    const uint64_t kh = sk[0] & high_mask;
    uint32_t len = 1;
    while (i + len < t.count && len <= max_run && (sk[len] & high_mask) == kh) len++;
    const bool crosses = i + len == t.count && (sk[len] & high_mask) == kh;  // sk[len] is the next tile's first key here
    my_len[e] = crosses ? (uint16_t)0xffffu : (uint16_t)len;
  }
  __syncthreads();
  for (uint32_t e = lane; e < my_n; e += 32) {
    const uint32_t i = my_heads[e];
    const uint64_t p = t.start + i;
    uint64_t* sk = s_key + 1 + i;  // the run starts at sk[0]
    const uint64_t kh = sk[0] & high_mask;
    uint32_t len = my_len[e];
    if (len == 0xffffu) {
      len = t.count - i;
      // the run continues into the next tile (at most one per tile): settle it in global memory, as a whole.  The next
      // tile never touches these rows -- none of them heads a run there -- and reads only their (unchanging) prefixes.
      uint64_t q = p + len;
      while (q < sege && q - p <= max_run && (keys[q] & high_mask) == kh) q++;
      const uint32_t glen = (uint32_t)(q - p);
      if (glen > max_run) {
        *flag = 1;
        continue;
      }
      for (uint32_t a = 1; a < glen; a++) {  // stable insertion sort on the low bits
        const uint64_t ka = keys[p + a];
        const uint32_t va = vals[p + a];
        const uint64_t la = ka & low_mask;
        uint32_t b = a;
        while (b > 0 && (keys[p + b - 1] & low_mask) > la) {
          keys[p + b] = keys[p + b - 1];
          vals[p + b] = vals[p + b - 1];
          b--;
        }
        if (b != a) {
          keys[p + b] = ka;
          vals[p + b] = va;
        }
      }
      continue;
    }
    if (len > max_run) {
      *flag = 1;
      continue;
    }
    // the run lies inside the tile: stable insertion sort on the low bits, keys in shared memory; the rows that move are
    // written through to global memory (their row indices are fetched only then)
    for (uint32_t a = 1; a < len; a++) {
      const uint64_t ka = sk[a];
      const uint64_t la = ka & low_mask;
      uint32_t b = a;
      while (b > 0 && (sk[b - 1] & low_mask) > la) b--;
      if (b == a) continue;
      const uint32_t va = vals[p + a];
      for (uint32_t c = a; c > b; c--) {
        const uint64_t kc = sk[c - 1];
        sk[c] = kc;
        keys[p + c] = kc;
        vals[p + c] = vals[p + c - 1];
      }
      sk[b] = ka;
      keys[p + b] = ka;
      vals[p + b] = va;
    }
  }
}

// ---- local sort ---------------------------------------------------------------------------------------------------
// One CTA sorts one work item -- a range of at most kLocalSortCap pairs that the caller knows to be final as a whole: a
// whole segment, or consecutive whole (segment, MSD digit) sub-buckets of one segment after the MSD scatter -- completely
// and stably on its key, in shared memory: one HBM read and one HBM write per pair.
//
// The keys and row indices stay where they were loaded; the passes move 16-bit slot numbers.  Stable LSD passes on the
// item's top varying 8-bit digits, enough of them that the item spreads over more prefixes than twice its rows, then the
// (short, rare) runs of rows that share that prefix are insertion-sorted on the whole key.  When a run is longer than
// kLocalMaxRun (low-entropy high bits, heavy ties), the item is sorted again from its load order with LSD passes over all of
// its varying digits: the result is the same stable order either way.
constexpr int kLocalSortCap = 12288;
struct LocalSortItem {
  uint32_t start, count;  // a range of pairs that is sorted as a whole
  uint32_t seg, seg_row;  // its segment, and the position of its first pair inside the segment
};
constexpr int kLocalThreads = 1024;
constexpr int kLocalWarps = kLocalThreads / 32;
constexpr int kLocalItems = kLocalSortCap / kLocalThreads;  // 12 slots per thread
constexpr int kLocalWarpRows = kLocalSortCap / kLocalWarps; // 384 consecutive slots per warp
constexpr uint32_t kLocalMaxRun = 64;
static_assert(kLocalSortCap % kLocalThreads == 0 && kLocalSortCap <= 65536, "slot numbers are 16-bit");

struct LocalShared {
  uint64_t keys[kLocalSortCap];        // in load order
  uint32_t vals[kLocalSortCap];        // in load order
  uint16_t slot[kLocalSortCap];        // sorted position -> load-order slot
  uint16_t cnt[kLocalWarps][256];
  uint32_t warp_sums[40];
  unsigned long long or_bits, and_bits;
  uint32_t long_run;
};

// One stable pass on digit (key >> shift) & 255 over sm.slot[0, count).  Ranking as in k_sort_scatter; warps whose slots
// all lie past the end skip it (their counters stay zero), so small items cost little.
__device__ __forceinline__ void local_pass(LocalShared& sm, uint32_t count, int shift) {
  const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  {
    uint32_t* z = reinterpret_cast<uint32_t*>(&sm.cnt[0][0]);
#pragma unroll
    for (int i = 0; i < kLocalWarps * 256 / 2 / kLocalThreads; i++) z[threadIdx.x + i * kLocalThreads] = 0;
  }
  const uint32_t first = warp * kLocalWarpRows + lane;
  uint32_t slot_bin[kLocalItems], rank[kLocalItems];  // slot << 8 | digit: one register per row
#pragma unroll
  for (int j = 0; j < kLocalItems; j++) {
    const uint32_t pos = first + j * 32;
    const uint32_t s = pos < count ? sm.slot[pos] : pos;
    slot_bin[j] = s << 8 | (pos < count ? (uint32_t)(sm.keys[s] >> shift) & 255u : 255u);
  }
  __syncthreads();
  rank_tile<kLocalWarps, kLocalItems, true>(sm.cnt, sm.warp_sums, [&](int j) { return slot_bin[j] & 255u; }, count, rank);
  __syncthreads();
  const uint16_t* cnt = sm.cnt[warp];
#pragma unroll
  for (int j = 0; j < kLocalItems; j++)
    if (warp * kLocalWarpRows + j * 32 < count) sm.slot[cnt[slot_bin[j] & 255u] + rank[j]] = (uint16_t)(slot_bin[j] >> 8);
  __syncthreads();
}

// out_keys == nullptr: each sorted key is decoded and stored into its PLAIN page body instead (KeyPageDest).  Bodies are
// width-aligned except on tiny pages (Thrift headers have odd sizes), where the value is stored byte by byte.
template <typename Src>
__global__ void __launch_bounds__(kLocalThreads, 1) k_local_sort(const LocalSortItem* __restrict__ items, Src src,
                                                                 uint64_t* __restrict__ out_keys,
                                                                 uint32_t* __restrict__ out_vals, KeyPageDest pages) {
  extern __shared__ __align__(16) uint8_t smem_raw[];
  LocalShared& sm = *reinterpret_cast<LocalShared*>(smem_raw);
  const LocalSortItem it = items[blockIdx.x];
  const uint32_t count = it.count;
  if (threadIdx.x == 0) {
    sm.or_bits = 0;
    sm.and_bits = ~0ull;
    sm.long_run = 0;
  }
  // load: half of a thread's loads in flight at once (all of them would not fit in 64 registers); OR / AND of the item's
  // keys on the way
  uint64_t k_or = 0, k_and = ~0ull;
  constexpr int kHalf = kLocalItems / 2;
#pragma unroll 1
  for (int h = 0; h < 2; h++) {
    uint64_t k[kHalf];
    uint32_t v[kHalf];
#pragma unroll
    for (int j = 0; j < kHalf; j++) {
      const uint32_t i = (h * kHalf + j) * kLocalThreads + threadIdx.x;
      if (i < count) src.load((uint64_t)it.start + i, k[j], v[j]);
    }
#pragma unroll
    for (int j = 0; j < kHalf; j++) {
      const uint32_t i = (h * kHalf + j) * kLocalThreads + threadIdx.x;
      if (i < count) {
        sm.keys[i] = k[j];
        sm.vals[i] = v[j];
        sm.slot[i] = (uint16_t)i;
        k_or |= k[j];
        k_and &= k[j];
      }
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    k_or |= __shfl_xor_sync(0xffffffffu, k_or, o);
    k_and &= __shfl_xor_sync(0xffffffffu, k_and, o);
  }
  __syncthreads();
  if ((threadIdx.x & 31) == 0) {
    atomicOr(&sm.or_bits, k_or);
    atomicAnd(&sm.and_bits, k_and);
  }
  __syncthreads();
  const uint64_t varying = sm.or_bits ^ sm.and_bits;
  if (varying != 0) {
    const int top = 63 - __clzll((long long)varying);
    int pbits = 1;  // prefix bits: at least twice as many prefixes as rows
    while ((1u << pbits) < 2 * count) pbits++;
    const int ndig = (min(pbits, top + 1) + 7) / 8;
    const int low = max(0, top + 1 - 8 * ndig);  // lowest digit: bits [low, low + 8); may overlap the next one
    for (int d = ndig - 1; d >= 0; d--) {
      const int shift = max(0, top + 1 - 8 * (d + 1));
      if ((varying >> shift) & 0xff) local_pass(sm, count, shift);
    }
    const uint64_t high_mask = ~0ull << low;
    if (varying & ~high_mask) {
      // rows that share the prefix are still in load order: stable insertion sort of every such run on the whole key.
      // Other threads' runs are being reordered meanwhile, but every row of a run has the run's prefix, so the head test
      // and the walk (which look one row past a run) read the same prefixes whatever the order inside it.
      for (uint32_t i = threadIdx.x; i < count; i += kLocalThreads) {
        const uint64_t kh = sm.keys[sm.slot[i]] & high_mask;
        if (i > 0 && (sm.keys[sm.slot[i - 1]] & high_mask) == kh) continue;               // not the head of a run
        if (i + 1 >= count || (sm.keys[sm.slot[i + 1]] & high_mask) != kh) continue;      // a run of one
        uint32_t len = 2;
        while (i + len < count && len <= kLocalMaxRun && (sm.keys[sm.slot[i + len]] & high_mask) == kh) len++;
        if (len > kLocalMaxRun) {
          sm.long_run = 1;
          continue;
        }
        uint16_t* s = sm.slot + i;
        for (uint32_t a = 1; a < len; a++) {
          const uint16_t sa = s[a];
          const uint64_t ka = sm.keys[sa];
          uint32_t b = a;
          while (b > 0 && sm.keys[s[b - 1]] > ka) {
            s[b] = s[b - 1];
            b--;
          }
          s[b] = sa;
        }
      }
      __syncthreads();
      if (sm.long_run) {
        for (uint32_t i = threadIdx.x; i < count; i += kLocalThreads) sm.slot[i] = (uint16_t)i;
        __syncthreads();
        for (int shift = 0; shift < 64; shift += 8)
          if ((varying >> shift) & 0xff) local_pass(sm, count, shift);
      }
    }
  }
  __syncthreads();
  if (out_keys) {
#pragma unroll
    for (int j = 0; j < kLocalItems; j++) {
      const uint32_t i = j * kLocalThreads + threadIdx.x;
      if (i < count) {
        const uint32_t s = sm.slot[i];
        out_keys[(uint64_t)it.start + i] = sm.keys[s];
        out_vals[(uint64_t)it.start + i] = sm.vals[s];
      }
    }
    return;
  }
  const uint64_t* pvo = pages.page_value_offset + pages.seg_page_begin[it.seg];
  const uint32_t P = pages.rows_per_page;
#pragma unroll
  for (int j = 0; j < kLocalItems; j++) {
    const uint32_t i = j * kLocalThreads + threadIdx.x;
    if (i < count) {
      const uint32_t s = sm.slot[i];
      out_vals[(uint64_t)it.start + i] = sm.vals[s];
      const uint32_t lr = it.seg_row + i, page = lr / P;
      uint8_t* dst = pages.arena + pvo[page] + (uint64_t)(lr - page * P) * pages.width;
      const uint64_t v = sort_decode_int(pages.type, sm.keys[s]);
      if (((uintptr_t)dst & (pages.width - 1)) != 0) {
        for (int b = 0; b < pages.width; b++) dst[b] = (uint8_t)(v >> (8 * b));
      } else if (pages.width == 8) {
        *reinterpret_cast<uint64_t*>(dst) = v;
      } else {
        *reinterpret_cast<uint32_t*>(dst) = (uint32_t)v;
      }
    }
  }
}

// pages != nullptr: the keys go into their pages, out_keys is not written
template <typename Src>
void launch_local_sort(hs_ctx* ctx, const std::vector<LocalSortItem>& items, Src src, uint64_t* out_keys,
                       uint32_t* out_vals, const KeyPageDest* pages) {
  if (items.empty()) return;
  KeyPageDest dest{};
  if (pages) {
    dest = *pages;
    out_keys = nullptr;
  } else if (!out_keys) {
    fail(HS_EINVAL, "internal: local sort without a key destination");
  }
  Buf<LocalSortItem> d_items(ctx, items.size());
  copy_h2d(ctx, d_items.get(), items.data(), items.size() * sizeof(LocalSortItem));
  static DeviceOnce attr_once;  // one per Src instantiation
  bool& attr = attr_once(ctx->device);
  if (!attr) {
    HS_CUDA(cudaFuncSetAttribute(k_local_sort<Src>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(LocalShared)));
    attr = true;
  }
  KernelScope _ks(ctx, "k_local_sort");
  k_local_sort<Src><<<(unsigned)items.size(), kLocalThreads, sizeof(LocalShared), ctx->stream>>>(d_items.get(), src,
                                                                                                 out_keys, out_vals, dest);
  HS_LAUNCH_CHECK(ctx);
}

// histogram of one pass and the (segment, digit) bases; digit_base (optional) receives the bases, see k_seg_scan
template <typename Src, typename Digit>
void run_hist(hs_ctx* ctx, SortPlan* plan, Src src, Digit digit, uint32_t* digit_base) {
  {
    KernelScope _ks(ctx, "k_sort_hist");
    k_sort_hist<Src, Digit><<<(unsigned)plan->ntiles, kHistThreads, 0, ctx->stream>>>(plan->tiles.get(), src, digit,
                                                                                 plan->tile_hist.get());
    HS_LAUNCH_CHECK(ctx);
  }
  KernelScope _ks(ctx, "k_seg_scan");
  k_seg_chunk_sums<<<(unsigned)plan->nchunks, 256, 0, ctx->stream>>>(plan->chunks.get(), plan->tile_hist.get(),
                                                                     plan->chunk_sums.get());
  HS_LAUNCH_CHECK(ctx);
  k_seg_scan<<<(unsigned)plan->nseg, 256, 0, ctx->stream>>>(plan->seg_chunk_begin.get(), plan->seg_start.get(),
                                                            plan->chunk_sums.get(), digit_base);
  HS_LAUNCH_CHECK(ctx);
}

// the scatter of a pass whose histogram run_hist queued
template <typename Src, typename Digit>
void run_scatter(hs_ctx* ctx, SortPlan* plan, Src src, Digit digit, uint64_t* out_keys, uint32_t* out_vals) {
  {
    KernelScope _ks(ctx, "k_seg_scan");
    k_seg_apply<<<(unsigned)plan->nchunks, 1024, 0, ctx->stream>>>(plan->chunks.get(), plan->tile_hist.get(),
                                                                   plan->tile_dst.get(), plan->chunk_sums.get());
    HS_LAUNCH_CHECK(ctx);
  }
  static DeviceOnce attr_once;  // one per (Src, Digit) instantiation
  bool& attr = attr_once(ctx->device);
  if (!attr) {
    HS_CUDA(cudaFuncSetAttribute(k_sort_scatter<Src, Digit>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 (int)sizeof(ScatterShared)));
    attr = true;
  }
  KernelScope _ks(ctx, "k_sort_scatter");
  k_sort_scatter<Src, Digit><<<(unsigned)plan->ntiles, kThreads, sizeof(ScatterShared), ctx->stream>>>(
      plan->tiles.get(), src, digit, plan->tile_dst.get(), out_keys, out_vals);
  HS_LAUNCH_CHECK(ctx);
}

// one whole pass into the scratch pairs, which then hold the sorted pairs
template <typename Src, typename Digit>
void run_pass(hs_ctx* ctx, SortPlan* plan, Src src, Digit digit, SortedRows* s) {
  run_hist(ctx, plan, src, digit, nullptr);
  run_scatter(ctx, plan, src, digit, s->keys_buf[s->cur ^ 1].get(), s->perm_buf[s->cur ^ 1].get());
  s->cur ^= 1;
}

// f(SrcRaw<T>{...}) for the column's type
template <typename F>
void with_raw_source(const KeyColumn& raw, F&& f) {
  switch (raw.type) {
    case HS_TYPE_INT32: f(SrcRaw<HS_TYPE_INT32>{raw.data}); break;
    case HS_TYPE_INT64: f(SrcRaw<HS_TYPE_INT64>{raw.data}); break;
    case HS_TYPE_FLOAT: f(SrcRaw<HS_TYPE_FLOAT>{raw.data}); break;
    case HS_TYPE_DOUBLE: f(SrcRaw<HS_TYPE_DOUBLE>{raw.data}); break;
    default: fail(HS_EUNSUPPORTED, "sort: key type %d", raw.type);
  }
}

// Stable LSD passes on the key bytes that `bits` selects (a byte constant over the input costs nothing).  raw (optional):
// the pairs have not been materialised yet -- the first pass reads the raw key column (position p holds the value of row
// p) and uses p itself as the row index.  bits must then select at least one byte.
void lsd_passes(hs_ctx* ctx, SortPlan* plan, SortedRows* s, uint64_t bits, const KeyColumn* raw) {
  if (plan->ntiles == 0) return;
  bool first = raw != nullptr;
  for (int pass = 0; pass < 8; pass++) {
    if (((bits >> (pass * 8)) & 0xff) == 0) continue;  // digit constant over the whole input
    const DigitShift digit{pass * 8};
    if (first)
      with_raw_source(*raw, [&](auto src) { run_pass(ctx, plan, src, digit, s); });
    else
      run_pass(ctx, plan, SrcPairs{s->keys(), s->perm()}, digit, s);
    first = false;
  }
  if (first) fail(HS_EINVAL, "sort: raw first-pass source given but no pass ran");
}

// The final sorted keys (keys_buf[cur]), allocated on first use: a sort that writes the key pages never needs them.
uint64_t* final_keys(hs_ctx* ctx, SortedRows* s, int64_t n) {
  Buf<uint64_t>& b = s->keys_buf[s->cur];
  if (!b) b.alloc(ctx, std::max<int64_t>(1, n));
  return b.get();
}

// The local sort's destinations: the key pages when key_pages (optional, see sort_rows) gives them, else the final keys.
const KeyPageDest* key_destination(hs_ctx* ctx, const KeyPagesFn* key_pages, SortedRows* s, int64_t n) {
  const KeyPageDest* pages = key_pages ? (*key_pages)() : nullptr;
  if (!pages) final_keys(ctx, s, n);
  s->key_pages_written = pages != nullptr;
  return pages;
}

// Every segment (at most kLocalSortCap rows each) sorted completely on the raw key column in one HBM pass.
void local_sort_segments(hs_ctx* ctx, const SortPlan& plan, const KeyColumn& raw, SortedRows* s,
                         const KeyPagesFn* key_pages) {
  std::vector<LocalSortItem> items;
  for (int g = 0; g < plan.nseg; g++) {
    const uint64_t n = plan.h_seg_start[g + 1] - plan.h_seg_start[g];
    if (n) items.push_back(LocalSortItem{(uint32_t)plan.h_seg_start[g], (uint32_t)n, (uint32_t)g, 0});
  }
  const KeyPageDest* pages = key_destination(ctx, key_pages, s, plan.n);
  with_raw_source(raw, [&](auto src) { launch_local_sort(ctx, items, src, s->keys(), s->perm(), pages); });
}

// Complete sort of the raw key column within every segment in two HBM passes: one stable MSD pass on digit
// (key >> shift) & 255 into the scratch pairs, then k_local_sort of every (segment, digit) sub-bucket back into the sorted
// pairs.  The bits above shift + 7 must be constant over the input.  Returns false, having queued only the MSD histogram,
// when a sub-bucket holds more than kLocalSortCap rows.  Synchronises the stream once.  key_pages (optional, see sort_rows)
// is asked for the page destinations while the MSD scatter runs, so that the caller's host work overlaps it.
bool msd_local_sort(hs_ctx* ctx, SortPlan* plan, const KeyColumn& raw, int shift, SortedRows* s,
                    const KeyPagesFn* key_pages) {
  if (plan->ntiles == 0) return false;
  const size_t nsub = (size_t)plan->nseg * 256;
  Buf<uint32_t> d_base(ctx, nsub);
  const DigitShift digit{shift};
  with_raw_source(raw, [&](auto src) { run_hist(ctx, plan, src, digit, d_base.get()); });
  std::vector<uint32_t> base(nsub + 1);
  copy_d2h(ctx, base.data(), d_base.get(), nsub * 4);
  sync_stream(ctx);
  base[nsub] = (uint32_t)plan->n;
  // work items: consecutive whole sub-buckets of one segment, up to kLocalSortCap rows
  std::vector<LocalSortItem> items;
  for (int g = 0; g < plan->nseg; g++) {
    const uint32_t seg_begin = base[(size_t)g * 256];
    LocalSortItem cur{seg_begin, 0, (uint32_t)g, 0};
    for (size_t d = (size_t)g * 256; d < (size_t)(g + 1) * 256; d++) {
      const uint32_t sz = base[d + 1] - base[d];
      if (sz > (uint32_t)kLocalSortCap) return false;
      if (cur.count + sz > (uint32_t)kLocalSortCap) {
        items.push_back(cur);
        cur = LocalSortItem{base[d], 0, (uint32_t)g, base[d] - seg_begin};
      }
      cur.count += sz;
    }
    if (cur.count) items.push_back(cur);
  }
  uint64_t* keys_alt = s->keys_buf[s->cur ^ 1].get();
  uint32_t* perm_alt = s->perm_buf[s->cur ^ 1].get();
  with_raw_source(raw, [&](auto src) { run_scatter(ctx, plan, src, digit, keys_alt, perm_alt); });
  const KeyPageDest* pages = key_destination(ctx, key_pages, s, plan->n);
  launch_local_sort(ctx, items, SrcPairs{keys_alt, perm_alt}, s->keys(), s->perm(), pages);
  return true;
}

}  // namespace

// tiles of one segment (one CTA per segment): the list has a quarter of a million entries at 1 B rows, so it is generated
// where it is used instead of being built on the host and copied over from pageable memory
__global__ void k_build_tiles(const uint64_t* __restrict__ seg_start, const uint32_t* __restrict__ seg_tile_begin,
                              SortTile* __restrict__ tiles) {
  const uint32_t s = blockIdx.x;
  const uint64_t b = seg_start[s], e = seg_start[s + 1];
  const uint32_t t0 = seg_tile_begin[s], nt = seg_tile_begin[s + 1] - t0;
  for (uint32_t i = threadIdx.x; i < nt; i += blockDim.x) {
    const uint64_t p = b + (uint64_t)i * kSortTile;
    tiles[t0 + i] = SortTile{s, (uint32_t)min((uint64_t)kSortTile, e - p), p};
  }
}

void build_sort_plan(hs_ctx* ctx, const uint64_t* seg_offsets, int nseg, SortPlan* plan) {
  std::vector<uint32_t> stb(nseg + 1), scb(nseg + 1);
  std::vector<uint64_t> sstart(nseg + 1);
  std::vector<SortChunk> chunks;
  uint64_t ntiles = 0;
  for (int s = 0; s < nseg; s++) {
    stb[s] = (uint32_t)ntiles;
    sstart[s] = seg_offsets[s];
    ntiles += ceil_div(seg_offsets[s + 1] - seg_offsets[s], (uint64_t)kSortTile);
    scb[s] = (uint32_t)chunks.size();
    for (uint32_t t = stb[s]; t < ntiles; t += kChunkTiles)
      chunks.push_back(SortChunk{(uint32_t)s, t, (uint32_t)std::min<uint64_t>(t + kChunkTiles, ntiles)});
  }
  stb[nseg] = (uint32_t)ntiles;
  sstart[nseg] = seg_offsets[nseg];
  scb[nseg] = (uint32_t)chunks.size();
  if (seg_offsets[nseg] >= (1ull << 32)) fail(HS_EUNSUPPORTED, "more than 2^32-1 rows per GPU per call");
  plan->n = (int64_t)seg_offsets[nseg];
  plan->ntiles = (int64_t)ntiles;
  plan->nseg = nseg;
  plan->nchunks = (int64_t)chunks.size();
  plan->tiles.alloc(ctx, std::max<size_t>(1, ntiles));
  plan->seg_tile_begin.alloc(ctx, stb.size());
  plan->seg_start.alloc(ctx, sstart.size());
  plan->tile_hist.alloc(ctx, std::max<size_t>(1, ntiles) * 256);
  plan->tile_dst.alloc(ctx, std::max<size_t>(1, ntiles) * 256);
  plan->chunks.alloc(ctx, std::max<size_t>(1, chunks.size()));
  plan->seg_chunk_begin.alloc(ctx, scb.size());
  plan->chunk_sums.alloc(ctx, std::max<size_t>(1, chunks.size()) * 256);
  copy_h2d(ctx, plan->seg_tile_begin.get(), stb.data(), stb.size() * 4);
  copy_h2d(ctx, plan->seg_start.get(), sstart.data(), sstart.size() * 8);
  if (!chunks.empty()) copy_h2d(ctx, plan->chunks.get(), chunks.data(), chunks.size() * sizeof(SortChunk));
  copy_h2d(ctx, plan->seg_chunk_begin.get(), scb.data(), scb.size() * 4);
  if (nseg > 0 && ntiles > 0) {
    k_build_tiles<<<nseg, 256, 0, ctx->stream>>>(plan->seg_start.get(), plan->seg_tile_begin.get(), plan->tiles.get());
    HS_LAUNCH_CHECK(ctx);
  }
  plan->h_seg_tile_begin = std::move(stb);  // (copy_h2d took snapshots of the host vectors)
  plan->h_seg_start = std::move(sstart);
}

void sort_rows(hs_ctx* ctx, SortPlan* plan, const KeyColumn* cols, int ncols, const unsigned long long* last_or_and,
               bool may_defer, SortedRows* out, const KeyPagesFn* key_pages) {
  const int64_t nrows = plan->n;
  const bool lsd_only = getenv("HS_LSD_SORT") != nullptr;
  // only a single null-free integer key can leave its final keys in the pages (sort_decode_int inverts its encoding)
  if (ncols != 1 || cols[0].valid || (cols[0].type != HS_TYPE_INT32 && cols[0].type != HS_TYPE_INT64) || lsd_only)
    key_pages = nullptr;
  // the final keys (keys_buf[0]) are allocated once it is known that the sort does not write the key pages
  out->cur = 0;
  out->keys_buf[1].alloc(ctx, std::max<int64_t>(1, nrows));
  out->keys_buf[0].release();
  auto need_keys = [&] { final_keys(ctx, out, nrows); };
  if (!key_pages) need_keys();
  for (auto& b : out->perm_buf) b.alloc(ctx, std::max<int64_t>(1, nrows));
  out->queued = false;
  out->resort_bits = 0;
  out->key_pages_written = false;
  Buf<unsigned long long> d_or_and(ctx, 2);
  unsigned long long or_and[2] = {0, 0};
  // or_and = OR / AND of the encoded keys that launch(d_or_and) reduces, on the host (synchronises)
  auto reduce = [&](auto launch) {
    const unsigned long long init[2] = {0ull, ~0ull};
    copy_h2d(ctx, d_or_and.get(), init, sizeof init);
    launch(d_or_and.get());
    copy_d2h(ctx, or_and, d_or_and.get(), sizeof or_and);
    sync_stream(ctx);
  };
  uint64_t max_seg = 1;
  for (int g = 0; g < plan->nseg; g++) max_seg = std::max<uint64_t>(max_seg, plan->h_seg_start[g + 1] - plan->h_seg_start[g]);
  // How many high bytes the tie fix-up sorts on: enough that a segment's rows spread over more prefixes than it has rows
  // (expected rows per prefix <= 0.5 for uniformly spread keys), at least 2.  5 M-row segments -> 3 bytes, 125 M-row -> 4.
  int want_bytes = 2;
  while (want_bytes < 8 && (double)max_seg / std::pow(256.0, want_bytes) > 0.5) want_bytes++;
  for (int k = ncols - 1; k >= 0; k--) {
    const KeyColumn& kc = cols[k];
    // The first column sorted (the last key column) starts from rows in input order: its first radix pass reads the raw
    // column and encodes on the fly, so neither the identity permutation nor the encoded keys are written out beforehand;
    // only the OR / AND of the encoded keys is needed to pick the passes.
    const bool from_raw = k == ncols - 1 && kc.type >= HS_TYPE_INT32 && kc.type <= HS_TYPE_DOUBLE;
    if (k == ncols - 1 && !from_raw) launch_iota_u32(ctx, out->perm(), nrows);
    if (kc.type == HS_TYPE_STRING) {
      // A string key is sorted piecewise: stable LSD passes on the length, then on its 8-byte pieces from the last to the
      // first (each piece a big-endian integer; digits that are constant over all rows cost nothing).  Short keys -- the
      // usual case -- take one piece.
      auto sort_piece = [&](int piece) {
        reduce([&](unsigned long long* d) {
          launch_string_piece_keys(ctx, (const uint64_t*)kc.data, out->perm(), nrows, piece, out->keys(), d);
        });
        lsd_passes(ctx, plan, out, or_and[0] ^ or_and[1], nullptr);
      };
      sort_piece(-1);
      const unsigned long long len_or = or_and[0];  // the OR of the lengths bounds the longest key from above
      for (int piece = (int)((len_or + 7) / 8) - 1; piece >= 0; piece--) sort_piece(piece);
    } else {
      if (from_raw && last_or_and) {
        or_and[0] = last_or_and[0];
        or_and[1] = last_or_and[1];
      } else {
        reduce([&](unsigned long long* d) {
          launch_encode_keys(ctx, kc.data, kc.type, from_raw ? nullptr : out->perm(), nrows, from_raw ? nullptr : out->keys(), d);
        });
      }
      const uint64_t varying = nrows ? (or_and[0] ^ or_and[1]) : 0;
      int nbytes = 0, lowest_high_byte = 0;  // varying bytes; the lowest of the top want_bytes of them
      for (int b = 7, seen = 0; b >= 0; b--)
        if ((varying >> (8 * b)) & 0xff) {
          nbytes++;
          if (++seen == want_bytes) lowest_high_byte = b;
        }
      const KeyColumn* raw = from_raw ? &kc : nullptr;
      if (from_raw && varying == 0) {  // nothing to sort on: materialise the pairs as they stand
        need_keys();
        launch_iota_u32(ctx, out->perm(), nrows);
        launch_encode_keys(ctx, kc.data, kc.type, nullptr, nrows, out->keys(), d_or_and.get());
        raw = nullptr;
      }
      // nothing is sorted after a single null-free key column, so the caller need not wait for its sort
      const bool defer = may_defer && ncols == 1 && !kc.valid;
      // A null-free fixed-width first column is sorted completely in shared memory (k_local_sort): straight from the raw
      // column when every segment fits one CTA, else after one MSD pass on the 8 bits below the highest varying bit, as long
      // as the (segment, digit) sub-buckets fit -- two HBM passes instead of one per varying byte.  Segments with more than
      // ~0.85 x 256 x kLocalSortCap rows would rarely pass the sub-bucket check, so they skip the MSD histogram.
      bool local = false;
      if (raw && !kc.valid && !lsd_only) {
        if (max_seg <= (uint64_t)kLocalSortCap) {
          local_sort_segments(ctx, *plan, kc, out, key_pages);
          local = true;
        } else if (nbytes > 2 && max_seg <= (uint64_t)(0.85 * 256 * kLocalSortCap)) {
          local = msd_local_sort(ctx, plan, kc, std::max(0, 63 - __builtin_clzll(varying) - 7), out, key_pages);
        }
      }
      if (!out->key_pages_written) need_keys();
      if (local) {
        out->queued = defer;
      } else if (nbytes > want_bytes) {
        // LSD passes over the top want_bytes varying bytes only, then k_fix_runs sorts the (rare, short) runs of rows that
        // agree on those bytes.  Its verdict travels with the next synchronisation: the caller's when it may wait (the
        // encoder plans its pages on the host meanwhile), else at once, since later passes build on this order.
        const uint64_t high_mask = ~0ull << (8 * lowest_high_byte);
        lsd_passes(ctx, plan, out, varying & high_mask, raw);
        Buf<uint32_t> d_gave_up(ctx, 1);
        fill_bytes(ctx, d_gave_up.get(), 0, 4);
        {
          KernelScope _ks(ctx, "k_fix_runs");
          k_fix_runs<<<(unsigned)plan->ntiles, 256, 0, ctx->stream>>>(plan->tiles.get(), plan->seg_start.get(), out->keys(),
                                                                      out->perm(), high_mask, ~high_mask, kFixMaxRun,
                                                                      d_gave_up.get());
          HS_LAUNCH_CHECK(ctx);
        }
        out->gave_up = 0;
        out->resort_bits = varying;
        out->queued_at = ctx->sync_count;
        out->queued = true;
        copy_d2h(ctx, &out->gave_up, d_gave_up.get(), 4);
        if (!defer) settle_sorted_rows(ctx, plan, out);
      } else {
        lsd_passes(ctx, plan, out, varying, raw);
      }
    }
    if (kc.valid && plan->ntiles)  // nulls first: one more stable pass on the validity byte (0 = null)
      run_pass(ctx, plan, SrcPairs{out->keys(), out->perm()}, DigitTable{kc.valid}, out);
  }
}

bool settle_sorted_rows(hs_ctx* ctx, SortPlan* plan, SortedRows* s) {
  const uint64_t bits = s->resort_bits;
  s->queued = false;
  s->resort_bits = 0;
  if (bits == 0) return false;                            // no fix-up verdict outstanding
  if (ctx->sync_count <= s->queued_at) sync_stream(ctx);  // the verdict has not been delivered yet
  if (!s->gave_up) return false;
  lsd_passes(ctx, plan, s, bits, nullptr);  // a run was too long for k_fix_runs: full passes
  return true;
}

}  // namespace hs
