// hash_partition.cu -- K2 bucket hash + histogram, K3 stable partition into bucket-major order.
//
// Replaces Spark's ShuffleExchangeExec(HashPartitioning(indexedColumns, numBuckets)) behind
// `indexData.repartition(numBuckets, indexedColumns)` (index/covering/CoveringIndex.scala:60): the map side computes
// bucket = pmod(murmur3(keys, seed 42), n) per row; the "shuffle" on one GPU is a stable counting sort of row
// indices by bucket id.  Stability makes the whole build deterministic: rows with equal keys keep source order,
// which is also the oracle's tie order.
//
// K2, every bucket count: k_tile_hist hashes the key columns, keeps every row's bin id (u16) and writes the tile histogram
// M[tile][bin]; k_tile_offsets_* turn M into exclusive per-(tile, bin) destinations (column scan in 3 small kernels).
// K3 up to kFusedMaxBins bins: k_partition_rows ranks each tile's rows and moves every column (the fused partition, below).
// K3 above that, per 4096-row tile (256 threads x 16 rows, each warp owns 512 consecutive rows):
//   k_partition_dest  ranks the tile's rows by bin id (__match_any_sync walk over per-warp counters) and emits dest[row].
//   k_scatter         out[dest[i]] = in[i] for each projected column.
// hash_rows and move_rows at the end of the file are the only entry points: they choose among these.
#include "device_utils.cuh"
#include "kernels.h"

namespace hs {

namespace {

constexpr int kFusedMaxBins = 1024;  // above this the per-warp counters no longer fit next to the exchange buffer

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr int kItems = kFusedTileLocal / kThreads;   // 16 rows per thread
constexpr int kWarpRows = kFusedTileLocal / kWarps;  // 512 consecutive rows per warp

__device__ __forceinline__ uint64_t load_raw(const KeyColumn& k, int64_t row) {
  switch (k.width) {
    case 8: return ((const uint64_t*)k.data)[row];
    case 4: return ((const uint32_t*)k.data)[row];
    default: return ((const uint8_t*)k.data)[row];
  }
}

// Counts the warp's items into its private histogram with match_any aggregation and returns, for every item, its
// rank among the warp's earlier items of the same bin.  cnt = this warp's histogram (nb entries, zeroed).
template <int ITEMS>
__device__ __forceinline__ void warp_rank(const uint16_t (&bin)[ITEMS], const bool (&act)[ITEMS], uint16_t* cnt,
                                          uint16_t (&rank)[ITEMS]) {
  const unsigned lane = threadIdx.x & 31;
  const unsigned lt = (1u << lane) - 1;
#pragma unroll
  for (int j = 0; j < ITEMS; j++) {
    const unsigned amask = __ballot_sync(0xffffffffu, act[j]);
    if (act[j]) {
      const unsigned peers = __match_any_sync(amask, bin[j]);
      const uint16_t pre = cnt[bin[j]];
      rank[j] = (uint16_t)(pre + __popc(peers & lt));
      __syncwarp(amask);
      if ((peers & lt) == 0) cnt[bin[j]] = (uint16_t)(pre + __popc(peers));
    }
    __syncwarp();
  }
}

// ---- column scan of M[ntiles][nb] in chunks of kChunk tiles ---------------------------------------------------------
constexpr int kChunk = 256;

__global__ void k_chunk_sums(const uint32_t* __restrict__ tile_hist, int64_t ntiles, int nb,
                             unsigned long long* __restrict__ chunk_sums) {
  const int64_t chunk = blockIdx.y;
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= nb) return;
  const int64_t t0 = chunk * kChunk, t1 = min(t0 + kChunk, ntiles);
  unsigned long long s = 0;
  for (int64_t t = t0; t < t1; t++) s += tile_hist[t * nb + b];
  chunk_sums[chunk * nb + b] = s;
}

// one thread per bucket: bucket base (exclusive scan over buckets of the global histogram) + prefix over chunks
// explicit_base != nullptr: the destination of bucket b starts at explicit_base[b] (positions in the owner GPU's
// receive buffers, computed on the host from the all-gathered histograms) instead of the local exclusive scan
__global__ void k_chunk_scan(unsigned long long* __restrict__ chunk_sums, int64_t nchunks, int nb,
                             const unsigned long long* __restrict__ global_hist,
                             unsigned long long* __restrict__ bucket_offsets,
                             const unsigned long long* __restrict__ explicit_base) {
  extern __shared__ unsigned long long s_base[];  // nb + 1
  if (threadIdx.x == 0) {
    unsigned long long run = 0;
    for (int b = 0; b < nb; b++) {
      s_base[b] = explicit_base ? explicit_base[b] : run;
      run += global_hist[b];
    }
    s_base[nb] = run;
  }
  __syncthreads();
  if (bucket_offsets)
    for (int b = threadIdx.x; b <= nb; b += blockDim.x) bucket_offsets[b] = s_base[b];
  for (int b = threadIdx.x; b < nb; b += blockDim.x) {
    unsigned long long run = s_base[b];
    for (int64_t c = 0; c < nchunks; c++) {
      unsigned long long v = chunk_sums[c * nb + b];
      chunk_sums[c * nb + b] = run;
      run += v;
    }
  }
}

__global__ void k_chunk_apply(uint32_t* __restrict__ tile_hist, int64_t ntiles, int nb,
                              const unsigned long long* __restrict__ chunk_sums) {
  const int64_t chunk = blockIdx.y;
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= nb) return;
  const int64_t t0 = chunk * kChunk, t1 = min(t0 + kChunk, ntiles);
  unsigned long long run = chunk_sums[chunk * nb + b];
  for (int64_t t = t0; t < t1; t++) {
    uint32_t v = tile_hist[t * nb + b];
    tile_hist[t * nb + b] = (uint32_t)run;  // destinations are < 2^32 (row count checked by the caller)
    run += v;
  }
}

__global__ void __launch_bounds__(kThreads) k_partition_dest(const uint16_t* __restrict__ bucket, int64_t nrows, int nb,
                                                              const uint32_t* __restrict__ tile_offsets,
                                                              uint32_t* __restrict__ dest) {
  extern __shared__ uint16_t s_cnt[];  // [kWarps][nb]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int i = threadIdx.x; i < kWarps * nb; i += kThreads) s_cnt[i] = 0;
  __syncthreads();
  const int64_t tile = blockIdx.x;
  const int64_t wbase = tile * kFusedTileLocal + (int64_t)warp * kWarpRows;
  uint16_t bin[kItems], rank[kItems];
  bool act[kItems];
#pragma unroll
  for (int j = 0; j < kItems; j++) {
    const int64_t row = wbase + j * 32 + lane;
    act[j] = row < nrows;
    bin[j] = act[j] ? bucket[row] : 0;
  }
  warp_rank<kItems>(bin, act, s_cnt + warp * nb, rank);
  __syncthreads();
  // exclusive prefix over warps, in place
  for (int b = threadIdx.x; b < nb; b += kThreads) {
    uint16_t run = 0;
#pragma unroll
    for (int w = 0; w < kWarps; w++) {
      uint16_t v = s_cnt[w * nb + b];
      s_cnt[w * nb + b] = run;
      run = (uint16_t)(run + v);
    }
  }
  __syncthreads();
#pragma unroll
  for (int j = 0; j < kItems; j++) {
    if (act[j]) {
      const int64_t row = wbase + j * 32 + lane;
      dest[row] = tile_offsets[tile * nb + bin[j]] + s_cnt[warp * nb + bin[j]] + rank[j];
    }
  }
}

template <typename T>
__global__ void k_scatter(const T* __restrict__ in, T* __restrict__ out, const uint32_t* __restrict__ dest, int64_t n) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) out[dest[i]] = in[i];
}

__global__ void k_encode_keys(const void* __restrict__ in, int type, int width, const uint32_t* __restrict__ src,
                              int64_t n, uint64_t* __restrict__ out, unsigned long long* __restrict__ or_and) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  uint64_t vor = 0, vand = ~0ull;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const int64_t r = src ? (int64_t)src[i] : i;
    uint64_t raw = width == 8 ? ((const uint64_t*)in)[r] : width == 4 ? ((const uint32_t*)in)[r] : ((const uint8_t*)in)[r];
    uint64_t e = sort_encode(type, raw);
    if (out) out[i] = e;  // out == nullptr: only the OR / AND of the encoded keys is wanted
    vor |= e;
    vand &= e;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    vor |= __shfl_xor_sync(0xffffffffu, (unsigned long long)vor, o);
    vand &= __shfl_xor_sync(0xffffffffu, (unsigned long long)vand, o);
  }
  if ((threadIdx.x & 31) == 0) {
    atomicOr(&or_and[0], (unsigned long long)vor);
    atomicAnd(&or_and[1], (unsigned long long)vand);
  }
}

// One radix-sortable piece of a string key per row: piece < 0 -> the length, else the piece-th 8 bytes as a big-endian
// integer (zero-padded).  Sorting stably by length, then by the pieces from the last to the first, is the byte-wise order
// with a proper prefix first (UTF8String.compareTo).
__global__ void k_string_piece_keys(const uint64_t* __restrict__ refs, const uint32_t* __restrict__ perm, int64_t n, int piece,
                                    uint64_t* __restrict__ out, unsigned long long* __restrict__ or_and) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  uint64_t vor = 0, vand = ~0ull;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const uint64_t r = refs[perm[i]];
    const uint64_t e = piece < 0 ? (uint64_t)ref_len(r) : string_chunk(r, (uint32_t)piece);
    out[i] = e;
    vor |= e;
    vand &= e;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    vor |= __shfl_xor_sync(0xffffffffu, (unsigned long long)vor, o);
    vand &= __shfl_xor_sync(0xffffffffu, (unsigned long long)vand, o);
  }
  if ((threadIdx.x & 31) == 0) {
    atomicOr(&or_and[0], (unsigned long long)vor);
    atomicAnd(&or_and[1], (unsigned long long)vand);
  }
}

__global__ void k_iota(uint32_t* out, int64_t n) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) out[i] = (uint32_t)i;
}

inline int grid_for(hs_ctx* ctx, int64_t n, int threads, int per_sm) {
  int64_t want = ceil_div(n, threads);
  int64_t cap = (int64_t)ctx->sm_count * per_sm;
  return (int)std::max<int64_t>(1, std::min(want, cap));
}

}  // namespace

void launch_tile_offsets(hs_ctx* ctx, uint32_t* tile_hist, int64_t ntiles, int num_buckets,
                         const unsigned long long* global_hist, unsigned long long* bucket_offsets,
                         const unsigned long long* explicit_base) {
  KernelScope _ks(ctx, "k_tile_offsets");
  const int64_t nchunks = std::max<int64_t>(1, ceil_div(ntiles, kChunk));
  Buf<unsigned long long> chunk_sums(ctx, (size_t)nchunks * num_buckets);
  dim3 grid((num_buckets + 127) / 128, (unsigned)nchunks);
  k_chunk_sums<<<grid, 128, 0, ctx->stream>>>(tile_hist, ntiles, num_buckets, chunk_sums.get());
  HS_LAUNCH_CHECK(ctx);
  k_chunk_scan<<<1, 256, (num_buckets + 1) * sizeof(unsigned long long), ctx->stream>>>(
      chunk_sums.get(), nchunks, num_buckets, global_hist, bucket_offsets, explicit_base);
  HS_LAUNCH_CHECK(ctx);
  k_chunk_apply<<<grid, 128, 0, ctx->stream>>>(tile_hist, ntiles, num_buckets, chunk_sums.get());
  HS_LAUNCH_CHECK(ctx);
  // chunk_sums returns to the pool here; the stream order keeps it alive until the kernels above have run because
  // the pool only hands it out again to work enqueued later on the same stream.
}

// dest[row] = stable position of the row in bin-major order (tile_offsets: launch_tile_offsets of the 4096-row tiles)
static void launch_partition_dest(hs_ctx* ctx, const uint16_t* bin_ids, int64_t nrows, int nbins,
                                  const uint32_t* tile_offsets, uint32_t* dest) {
  KernelScope _ks(ctx, "k_partition_dest");
  if (nrows == 0) return;
  const int64_t ntiles = ceil_div(nrows, kFusedTileLocal);
  const size_t smem = (size_t)kWarps * nbins * sizeof(uint16_t);
  static DeviceOnce attr_once;
  bool& attr = attr_once(ctx->device);
  if (!attr) {
    HS_CUDA(cudaFuncSetAttribute(k_partition_dest, cudaFuncAttributeMaxDynamicSharedMemorySize, kWarps * kMaxBuckets * 2));
    attr = true;
  }
  k_partition_dest<<<(unsigned)ntiles, kThreads, smem, ctx->stream>>>(bin_ids, nrows, nbins, tile_offsets, dest);
  HS_LAUNCH_CHECK(ctx);
}

// out[dest[i]] = in[i]
static void launch_scatter_column(hs_ctx* ctx, const void* in, void* out, const uint32_t* dest, int64_t nrows, int width) {
  KernelScope _ks(ctx, "k_scatter_column");
  if (nrows == 0) return;
  const int grid = grid_for(ctx, nrows, 256, 16);
  switch (width) {
    case 8: k_scatter<uint64_t><<<grid, 256, 0, ctx->stream>>>((const uint64_t*)in, (uint64_t*)out, dest, nrows); break;
    case 4: k_scatter<uint32_t><<<grid, 256, 0, ctx->stream>>>((const uint32_t*)in, (uint32_t*)out, dest, nrows); break;
    case 1: k_scatter<uint8_t><<<grid, 256, 0, ctx->stream>>>((const uint8_t*)in, (uint8_t*)out, dest, nrows); break;
    default: fail(HS_EINVAL, "scatter: unsupported width %d", width);
  }
  HS_LAUNCH_CHECK(ctx);
}

void launch_encode_keys(hs_ctx* ctx, const void* in, int type, const uint32_t* src, int64_t nrows, uint64_t* out,
                        unsigned long long* or_and) {
  KernelScope _ks(ctx, "k_encode_keys");
  if (nrows == 0) return;
  k_encode_keys<<<grid_for(ctx, nrows, 256, 16), 256, 0, ctx->stream>>>(in, type, type_width(type), src, nrows, out,
                                                                         or_and);
  HS_LAUNCH_CHECK(ctx);
}

void launch_string_piece_keys(hs_ctx* ctx, const uint64_t* refs, const uint32_t* perm, int64_t nrows, int piece, uint64_t* out,
                              unsigned long long* or_and) {
  KernelScope _ks(ctx, "k_string_piece_keys");
  if (nrows == 0) return;
  k_string_piece_keys<<<grid_for(ctx, nrows, 256, 16), 256, 0, ctx->stream>>>(refs, perm, nrows, piece, out, or_and);
  HS_LAUNCH_CHECK(ctx);
}

void launch_iota_u32(hs_ctx* ctx, uint32_t* out, int64_t n) {
  if (n == 0) return;
  k_iota<<<grid_for(ctx, n, 256, 16), 256, 0, ctx->stream>>>(out, n);
  HS_LAUNCH_CHECK(ctx);
}

}  // namespace hs

// =====================================================================================================================
// Fused partition: one kernel hashes the keys, ranks the tile's rows stably by bucket and moves EVERY column through a
// shared-memory exchange, so each bucket's rows leave the tile as one contiguous run per column (full-sector stores).
// The unfused path above (bucket ids -> dest -> per-column scattered 8-byte stores) issues partial-sector writes, which
// are what HBM + L2 handle worst.
// =====================================================================================================================
namespace hs {
namespace {

// Two tile shapes.  Local: 4096 rows x 256 threads, four CTAs per SM -- the kernel is bound by the latency of its phases
// (hash, rank, one exchange round per column), and four small CTAs overlap them better than two big ones.  Peer: 8192
// rows x 512 threads -- when the runs leave over NVLink, twice as long a run per (tile, bucket) matters more.
template <bool PEER>
struct FusedCfg {
  static constexpr int kTile = PEER ? kFusedTilePeer : kFusedTileLocal;
  static constexpr int kThreads = PEER ? 512 : 256;
  static constexpr int kWarps = kThreads / 32;
  static constexpr int kItems = kTile / kThreads;   // 16
  static constexpr int kWarpRows = kTile / kWarps;  // 512
  static constexpr int kMinCtas = 1024 / kThreads;
};

// CTAs per SM that __launch_bounds__ asks for, i.e. the register budget: 1024 threads per SM = 64 registers per thread.
// Under sm_90a's register allocation the local tile's general-key instantiations spill at 64, so they get three CTAs (up
// to 80 registers).  The peer tile (512 threads) keeps two: one CTA per SM would halve its occupancy.
template <int KT, bool PEER>
constexpr int partition_min_ctas() { return !PEER && KT < 0 ? 3 : FusedCfg<PEER>::kMinCtas; }

// pmod(hash, n) and bucket % world without an integer division per row: Lemire's fastmod (M = 2^64 / n + 1; exact for
// 32-bit operands).  The signed Murmur3 value is shifted into unsigned range first and the shift is taken out again
// modulo n:  pmod(h, n) = ((h + 2^31) mod n - (2^31 mod n)) mod+ n.
struct ModConst {
  uint64_t M;
  uint32_t n;
  uint32_t bias;  // 2^31 mod n
};
__host__ ModConst make_mod_const(uint32_t n) {
  ModConst m;
  m.M = ~0ull / n + 1;  // wraps to 0 for n == 1, which still yields x mod 1 == 0
  m.n = n;
  m.bias = (uint32_t)((1ull << 31) % n);
  return m;
}
__device__ __forceinline__ uint32_t fast_mod(uint32_t x, const ModConst& m) { return (uint32_t)__umul64hi(m.M * x, m.n); }
__device__ __forceinline__ uint32_t fast_pmod(uint32_t h, const ModConst& m) {
  const uint32_t r = fast_mod(h ^ 0x80000000u, m);
  return r >= m.bias ? r - m.bias : r + m.n - m.bias;
}

// last_encoded (optional): receives the sort encoding of the LAST key column's value (0 for a null)
__device__ __forceinline__ uint32_t row_hash(const KeyColumn* keys, int nkeys, int64_t row, uint64_t* last_encoded = nullptr) {
  uint32_t h = 42;
  if (last_encoded) *last_encoded = 0;
  for (int k = 0; k < nkeys; k++) {
    const KeyColumn kc = keys[k];
    if (kc.valid && !kc.valid[row]) continue;  // null leaves the hash unchanged
    const uint64_t raw = load_raw(kc, row);
    if (last_encoded && k == nkeys - 1) *last_encoded = sort_encode(kc.type, raw);
    h = mm3_hash_value(key_hash_kind(kc), raw, h);
  }
  return h;
}

// KT >= 0: exactly one indexed column, of HS_TYPE KT and without nulls -- its descriptor is read once per thread and the
// hash is straight-line code, so a thread's key loads issue back to back.  KT < 0: any number / type of key columns.
// An int32 key may be a decimal(p <= 9), hashed as a long (KeyColumn::hash): read once, a branch uniform over the grid.
// A single-key column may be zero-copy (KeyColumn::tiles): the tile's values then lie in at most two page bodies of the
// source images, addressed by global row through rebased pointers (ZcTile); a decoded column is the same with one "page".
template <int KT>
struct RowHasher {
  const KeyColumn* keys;
  int nkeys;
  const uint8_t *p0, *p1;
  int64_t split;
  bool decimal_hash;
  __device__ __forceinline__ RowHasher(const KeyColumn* k, int n, int64_t tile)
      : keys(k), nkeys(n), p0(nullptr), p1(nullptr), split(INT64_MAX), decimal_hash(false) {
    if (KT >= 0) {
      const KeyColumn kc = k[0];
      decimal_hash = KT == HS_TYPE_INT32 && kc.hash == kHashDecimalInt;
      if (kc.tiles) {
        const ZcTile z = kc.tiles[tile];
        p0 = z.p0;
        p1 = z.p1;
        split = z.split;
      } else {
        p0 = p1 = (const uint8_t*)kc.data;
      }
    }
  }
  __device__ __forceinline__ uint32_t operator()(int64_t row, uint64_t* last_encoded = nullptr) const {
    if (KT >= 0) {
      const uint8_t* b = row < split ? p0 : p1;
      const uint64_t raw = (KT == HS_TYPE_INT64 || KT == HS_TYPE_DOUBLE) ? *(const uint64_t*)(b + row * 8)
                                                                         : (uint64_t) * (const uint32_t*)(b + row * 4);
      if (last_encoded) *last_encoded = sort_encode(KT, raw);
      if (KT == HS_TYPE_INT32 && decimal_hash) return mm3_hash_value(kHashDecimalInt, raw, 42u);
      return mm3_hash_value(KT, raw, 42u);
    }
    return row_hash(keys, nkeys, row, last_encoded);
  }
};

template <int KT, bool PEER>
__global__ void __launch_bounds__(FusedCfg<PEER>::kThreads) k_tile_hist(const KeyColumn* __restrict__ keys, int nkeys, int64_t nrows,
                                                          ModConst bucket_mod, ModConst owner_mod, int use_owner,
                                                          uint32_t* __restrict__ tile_hist,
                                                          unsigned long long* __restrict__ global_hist,
                                                          unsigned long long* __restrict__ key_or_and,
                                                          uint16_t* __restrict__ bin_ids) {
  extern __shared__ uint32_t s_hist[];  // nb
  constexpr int kFThreads = FusedCfg<PEER>::kThreads, kFItems = FusedCfg<PEER>::kItems, kFusedTile = FusedCfg<PEER>::kTile;
  const int nb = use_owner ? (int)owner_mod.n : (int)bucket_mod.n;
  for (int i = threadIdx.x; i < nb; i += kFThreads) s_hist[i] = 0;
  __syncthreads();
  const int64_t base = (int64_t)blockIdx.x * kFusedTile;
  const RowHasher<KT> hasher(keys, nkeys, blockIdx.x);
  uint64_t vor = 0, vand = ~0ull;
#pragma unroll 4
  for (int j = 0; j < kFItems; j++) {
    const int64_t row = base + j * kFThreads + threadIdx.x;
    if (row < nrows) {
      uint64_t e;
      uint32_t b = fast_pmod(hasher(row, &e), bucket_mod);
      if (use_owner) b = fast_mod(b, owner_mod);
      atomicAdd(&s_hist[b], 1u);
      if (bin_ids) bin_ids[row] = (uint16_t)b;  // the partition kernel reads 2 bytes back instead of hashing 8 again
      vor |= e;
      vand &= e;
    }
  }
  if (key_or_and) {  // which bits of the last indexed column vary: picks the radix passes of the sort that follows
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      vor |= __shfl_xor_sync(0xffffffffu, (unsigned long long)vor, o);
      vand &= __shfl_xor_sync(0xffffffffu, (unsigned long long)vand, o);
    }
    // the two accumulators saturate after a few tiles: look first, and only touch them when this warp adds information
    // (millions of atomics on two addresses would serialise in L2)
    if ((threadIdx.x & 31) == 0) {
      const unsigned long long cur_or = *(volatile unsigned long long*)&key_or_and[0];
      const unsigned long long cur_and = *(volatile unsigned long long*)&key_or_and[1];
      if ((vor | cur_or) != cur_or) atomicOr(&key_or_and[0], (unsigned long long)vor);
      if ((vand & cur_and) != cur_and) atomicAnd(&key_or_and[1], (unsigned long long)vand);
    }
  }
  __syncthreads();
  for (int b = threadIdx.x; b < nb; b += kFThreads) {
    const uint32_t s = s_hist[b];
    tile_hist[(size_t)blockIdx.x * nb + b] = s;
    if (s) atomicAdd(&global_hist[b], (unsigned long long)s);
  }
}

// ---- bulk asynchronous stores (TMA engine, 1-D): shared memory -> global / peer memory ----------------------------------
// A bucket's rows leave the tile as ONE cp.async.bulk per column instead of one 8-byte store per row: the copy engine reads
// the run from shared memory and writes it as full-width transactions -- over NVLink that is one packet stream per run
// instead of a sector-sized write per warp slice -- and the issuing thread is free at once.  Both addresses and the size must
// be multiples of 16 bytes: runs are laid out in the exchange buffer with the same 16-byte phase as their destination (see
// the padded layout below); an odd head / tail element goes out as a plain store.
__device__ __forceinline__ void bulk_store_s2g(void* dst, const void* src_smem, uint32_t bytes) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(dst),
               "r"((uint32_t)__cvta_generic_to_shared(src_smem)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
// the shared-memory source of every committed group has been read (the global writes may still be in flight)
__device__ __forceinline__ void bulk_wait_read() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
// generic-proxy writes to shared memory become visible to the async proxy (the copy engine)
__device__ __forceinline__ void fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// dynamic shared memory layout: [exchange buffer XN * 8 B][pos_bin u16 XN][cnt u16 kFWarps*nb][out_adj u32 nb]
// [bin_owner u32 nb][run_start u16 nb][run_len u16 nb][warp_sums 40 u32], XN = kFusedTile + 2 nb + 2
//
// Padded layout of the exchange buffer: bin b's run starts at s_b = P_b + 2 b + ((P_b ^ d_b) & 1), P_b = rows of the bins
// before it, d_b = its destination element index.  Runs never overlap (s_b - end of run b-1 is 1, 2 or 3) and s_b has the
// parity of d_b, so an 8-byte column's run and its destination share their 16-byte phase.
//
// All warp collectives run with the full mask and outside any branch: slots past the end of the last tile carry the
// last bin and, being the last slots of the tile, rank behind every real row of that bin; they are never written out.
//
// PEER: the runs go to the owners' memory over NVLink -- the large tile, and every 8-byte run leaves as a bulk copy; the
// local tile stores row by row into the dense layout.
template <int BITS, int KT, bool PEER>
__global__ void __launch_bounds__(FusedCfg<PEER>::kThreads, partition_min_ctas<KT, PEER>()) k_partition_rows(const KeyColumn* __restrict__ keys, int nkeys, int64_t nrows,
                                                               ModConst bucket_mod, ModConst owner_mod, int use_owner,
                                                               const uint32_t* __restrict__ tile_dst,
                                                               const PartColumn* __restrict__ cols, int ncols,
                                                               void* const* __restrict__ peer_out, int out_world,
                                                               CodePackRound pack, const uint16_t* __restrict__ bin_ids) {
  constexpr bool bulk = PEER;  // compile-time: the plain-store instantiation carries none of the bulk layout's bookkeeping
  extern __shared__ __align__(16) uint8_t smem[];
  constexpr int kFThreads = FusedCfg<PEER>::kThreads, kFItems = FusedCfg<PEER>::kItems, kFusedTile = FusedCfg<PEER>::kTile;
  constexpr int kFWarps = FusedCfg<PEER>::kWarps, kFWarpRows = FusedCfg<PEER>::kWarpRows;
  const int nb = use_owner ? (int)owner_mod.n : (int)bucket_mod.n;
  const uint32_t XN = (uint32_t)kFusedTile + (bulk ? 2u * (uint32_t)nb + 2u : 0u);
  uint64_t* xbuf = reinterpret_cast<uint64_t*>(smem);
  uint16_t* pos_bin = reinterpret_cast<uint16_t*>(smem + (size_t)XN * 8);
  uint16_t* cnt = pos_bin + XN;
  uint32_t* out_adj = reinterpret_cast<uint32_t*>(cnt + (size_t)kFWarps * nb + ((XN + (size_t)kFWarps * nb) & 1));
  uint32_t* bin_owner = out_adj + nb;
  uint16_t* run_start = reinterpret_cast<uint16_t*>(bin_owner + nb);
  uint16_t* run_len = run_start + nb;
  uint32_t* warp_sums = reinterpret_cast<uint32_t*>(run_len + nb);
  const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const unsigned lt = (1u << lane) - 1;
  for (int i = threadIdx.x; i < kFWarps * nb; i += kFThreads) cnt[i] = 0;
  if (bulk)
    for (uint32_t i = threadIdx.x; i < XN; i += kFThreads) pos_bin[i] = 0xffffu;  // padding slots belong to no bin
  const int64_t tile_base = (int64_t)blockIdx.x * kFusedTile;
  const uint32_t first = warp * kFWarpRows + lane;  // tile-relative row of this thread's item 0
  const int64_t wbase = tile_base + first;
  const uint32_t tile_count = (uint32_t)min((int64_t)kFusedTile, nrows - tile_base);
  uint32_t bin[kFItems];  // bin id in the low half; the in-warp rank joins it in the high half; finally the position
  const RowHasher<KT> hasher(keys, nkeys, blockIdx.x);
#pragma unroll
  for (int j = 0; j < kFItems; j++) {
    bin[j] = (uint32_t)nb - 1;
    if (first + j * 32 < tile_count) {
      if (bin_ids) {
        bin[j] = bin_ids[wbase + j * 32];
        continue;
      }
      uint32_t b = fast_pmod(hasher(wbase + j * 32), bucket_mod);
      if (use_owner) b = fast_mod(b, owner_mod);
      bin[j] = b;
    }
  }
  __syncthreads();
  // stable rank inside the warp's 512 consecutive rows
  uint16_t* wcnt = cnt + (size_t)warp * nb;
#pragma unroll
  for (int j = 0; j < kFItems; j++) {
    // (the PTX-spelled vote sequence that pays off in k_sort_scatter made THIS kernel slower -- 16 items per thread
    // instead of 8 -- so the plain form stays here)
    const unsigned peers = match_any_bits<BITS>(0xffffffffu, bin[j]);
    const uint32_t before = __popc(peers & lt);
    const uint32_t pre = wcnt[bin[j]];  // every peer reads the same counter (broadcast)
    __syncwarp();
    if (before == 0) wcnt[bin[j]] = (uint16_t)(pre + __popc(peers));
    __syncwarp();
    bin[j] |= (pre + before) << 16;
  }
  __syncthreads();
  // per bin: exclusive prefix over warps and bins -> first position of every (warp, bin) in the padded exchange buffer
  uint32_t carry = 0;
  for (int b0 = 0; b0 < nb; b0 += kFThreads) {
    const int b = b0 + threadIdx.x;
    uint32_t total = 0;
    if (b < nb) {
#pragma unroll
      for (int w = 0; w < kFWarps; w++) total += cnt[(size_t)w * nb + b];
    }
    uint32_t chunk_total = 0;
    const uint32_t ex = block_exclusive_scan(total, warp_sums, &chunk_total);
    if (b < nb) {
      const uint32_t P = carry + ex;
      const uint32_t dst = tile_dst[(size_t)blockIdx.x * nb + b];
      // padded layout only when the runs leave as bulk copies; plain stores keep the tile dense
      uint32_t run = bulk ? P + 2u * (uint32_t)b + ((P ^ dst) & 1u) : P;
      out_adj[b] = dst - run;
      bin_owner[b] = out_world > 1 ? (uint32_t)b % (uint32_t)out_world : 0u;
      if (bulk) {
        run_start[b] = (uint16_t)run;
        // the phantom slots of a partial last tile sit at the end of the last bin's run
        run_len[b] = (uint16_t)(b == nb - 1 ? total - ((uint32_t)kFusedTile - tile_count) : total);
      }
#pragma unroll
      for (int w = 0; w < kFWarps; w++) {
        const uint16_t c = cnt[(size_t)w * nb + b];
        cnt[(size_t)w * nb + b] = (uint16_t)run;
        run += c;
      }
    }
    carry += chunk_total;
  }
  __syncthreads();
  // positions in use: [0, x_end); the dense layout ends with the tile's last real row
  const uint32_t x_end = bulk ? (uint32_t)run_start[nb - 1] + run_len[nb - 1] : tile_count;
#pragma unroll
  for (int j = 0; j < kFItems; j++) {
    const uint32_t b = bin[j] & 0xffffu;
    bin[j] = wcnt[b] + (bin[j] >> 16);
    if (!bulk || first + j * 32 < tile_count) pos_bin[bin[j]] = (uint16_t)b;
  }
  const uint32_t(&pos)[kFItems] = bin;
  // one bin's run of an 8-byte column: [odd head element] [16-byte aligned body as ONE bulk copy] [odd tail element]
  auto store_runs = [&](void* const* pout, void* local_out) {
    for (int b = threadIdx.x; b < nb; b += kFThreads) {
      const uint32_t n = run_len[b];
      if (n == 0) continue;
      const uint32_t s = run_start[b];
      uint64_t* dst = (uint64_t*)(pout ? pout[bin_owner[b]] : local_out) + (out_adj[b] + s);
      const uint32_t h = (uint32_t)(((uintptr_t)dst >> 3) & 1u);
      if ((h ^ s) & 1u) {  // output base not 16-byte aligned (never the case for pool buffers): plain stores
        for (uint32_t i = 0; i < n; i++) dst[i] = xbuf[s + i];
        continue;
      }
      if (h) dst[0] = xbuf[s];
      const uint32_t body = (n - h) & ~1u;
      if (body) bulk_store_s2g(dst + h, xbuf + s + h, body * 8u);
      if ((n - h) & 1u) dst[n - 1] = xbuf[s + n - 1];
    }
    bulk_commit();
    bulk_wait_read();  // the runs have left shared memory: the next round may overwrite the buffer
  };
  // ---- move every column through the exchange buffer -----------------------------------------------------------
  for (int c = 0; c < ncols; c++) {
    const PartColumn pc = cols[c];
    __syncthreads();  // previous column's readers are done with xbuf (and pos_bin is complete)
    if (pc.tiles) {  // zero-copy column: the tile's values lie in one or two page bodies of the source images
      const ZcTile z = pc.tiles[blockIdx.x];
      if (pc.width == 8) {
#pragma unroll
        for (int j = 0; j < kFItems; j++)
          if (first + j * 32 < tile_count) {
            const int64_t row = wbase + j * 32;
            xbuf[pos[j]] = *(const uint64_t*)((row < z.split ? z.p0 : z.p1) + row * 8);
          }
      } else {
        uint32_t* xb = reinterpret_cast<uint32_t*>(xbuf);
#pragma unroll
        for (int j = 0; j < kFItems; j++)
          if (first + j * 32 < tile_count) {
            const int64_t row = wbase + j * 32;
            xb[pos[j]] = *(const uint32_t*)((row < z.split ? z.p0 : z.p1) + row * 4);
          }
      }
    } else if (pc.width == 8) {
      const uint64_t* in = (const uint64_t*)pc.in + wbase;
#pragma unroll
      for (int j = 0; j < kFItems; j++)
        if (first + j * 32 < tile_count) xbuf[pos[j]] = in[j * 32];
    } else if (pc.width == 4) {
      const uint32_t* in = (const uint32_t*)pc.in + wbase;
      uint32_t* xb = reinterpret_cast<uint32_t*>(xbuf);
#pragma unroll
      for (int j = 0; j < kFItems; j++)
        if (first + j * 32 < tile_count) xb[pos[j]] = in[j * 32];
    } else {
      const uint8_t* in = (const uint8_t*)pc.in + wbase;
      uint8_t* xb = reinterpret_cast<uint8_t*>(xbuf);
#pragma unroll
      for (int j = 0; j < kFItems; j++)
        if (first + j * 32 < tile_count) xb[pos[j]] = in[j * 32];
    }
    if (bulk && pc.width == 8) fence_async_smem();
    __syncthreads();
    // peer_out != nullptr: bucket b lives on GPU (b % out_world); its column c buffer is peer_out[c * out_world + owner]
    // (a peer-mapped pointer: these stores go straight over NVLink into the owner's memory)
    void* const* pout = peer_out ? peer_out + (size_t)c * out_world : nullptr;
    if (pc.width == 8) {
      if (bulk) {
        store_runs(pout, pc.out);
      } else {
#pragma unroll 4
        for (uint32_t i = threadIdx.x; i < x_end; i += kFThreads) {
          const uint32_t b = pos_bin[i];
          uint64_t* out = (uint64_t*)(pout ? pout[bin_owner[b]] : pc.out);
          out[out_adj[b] + i] = xbuf[i];
        }
      }
    } else if (pc.width == 4) {
      const uint32_t* xb = reinterpret_cast<const uint32_t*>(xbuf);
#pragma unroll 4
      for (uint32_t i = threadIdx.x; i < x_end; i += kFThreads) {
        const uint32_t b0 = pos_bin[i];
        const bool real = b0 != 0xffffu;  // padding slot of the bulk layout
        const uint32_t b = real ? b0 : 0u;
        uint32_t* out = (uint32_t*)(pout ? pout[bin_owner[b]] : pc.out);
        const uint32_t v = xb[i];
        if (real) out[out_adj[b] + i] = v;
      }
    } else {
      const uint8_t* xb = reinterpret_cast<const uint8_t*>(xbuf);
      for (uint32_t i = threadIdx.x; i < x_end; i += kFThreads) {
        const uint32_t b0 = pos_bin[i];
        const bool real = b0 != 0xffffu;
        const uint32_t b = real ? b0 : 0u;
        uint8_t* out = (uint8_t*)(pout ? pout[bin_owner[b]] : pc.out);
        const uint8_t v = xb[i];
        if (real) out[out_adj[b] + i] = v;
      }
    }
  }
  // ---- the 16-bit code columns of a row leave as one 8-byte record ---------------------------------------------------
  if (pack.n > 0) {
    __syncthreads();
#pragma unroll
    for (int j = 0; j < kFItems; j++) {
      if (first + j * 32 < tile_count) {
        const int64_t row = wbase + j * 32;
        uint32_t lo = pack.src[0][row], hi = 0;
        if (pack.n > 1) lo |= (uint32_t)pack.src[1][row] << 16;
        if (pack.n > 2) hi = pack.src[2][row];
        if (pack.n > 3) hi |= (uint32_t)pack.src[3][row] << 16;
        xbuf[pos[j]] = (uint64_t)lo | ((uint64_t)hi << 32);
      }
    }
    if (bulk) fence_async_smem();
    __syncthreads();
    // on several GPUs the records go to the bucket's owner like every column: their row of the peer table follows the
    // column rounds'
    void* const* pout = peer_out ? peer_out + (size_t)ncols * out_world : nullptr;
    if (bulk) {
      store_runs(pout, pack.out);
    } else {
#pragma unroll 4
      for (uint32_t i = threadIdx.x; i < x_end; i += kFThreads) {
        const uint32_t b = pos_bin[i];
        uint64_t* out = (uint64_t*)(pout ? pout[bin_owner[b]] : pack.out);
        out[out_adj[b] + i] = xbuf[i];
      }
    }
  }
}


template <bool PEER>
size_t fused_smem_bytes(int nb) {
  const size_t XN = (size_t)FusedCfg<PEER>::kTile + (PEER ? 2 * (size_t)nb + 2 : 0);
  size_t u16s = XN + (size_t)FusedCfg<PEER>::kWarps * nb;
  u16s += u16s & 1;
  return XN * 8 + u16s * 2 + (size_t)nb * 4 * 2 + (size_t)nb * 2 * 2 + 40 * 4;
}

// HS_TYPE_INT32 / HS_TYPE_INT64 when there is exactly one key column, of that type and without nulls (selects the kernels
// with the hash inlined for it); -1 otherwise
int single_key_type_of(const KeyColumn* keys, int nkeys) {
  return nkeys == 1 && keys[0].valid == nullptr && (keys[0].type == HS_TYPE_INT32 || keys[0].type == HS_TYPE_INT64)
             ? keys[0].type
             : -1;
}

template <bool PEER>
void launch_tile_hist(hs_ctx* ctx, const HashedRows& h, unsigned long long* global_hist, unsigned long long* key_or_and) {
  const ModConst bm = make_mod_const((uint32_t)h.num_buckets), om = make_mod_const((uint32_t)std::max(h.owner_mod, 1));
  const int uo = h.owner_mod > 0 ? 1 : 0;
#define HS_HIST(KT)                                                                                                       \
  k_tile_hist<KT, PEER><<<(unsigned)h.ntiles, FusedCfg<PEER>::kThreads, (size_t)h.nbins * 4, ctx->stream>>>(             \
      h.keys.get(), h.nkeys, h.nrows, bm, om, uo, h.tile_hist.get(), global_hist, key_or_and, h.bin_ids.get())
  switch (h.single_key_type) {
    case HS_TYPE_INT32: HS_HIST(HS_TYPE_INT32); break;
    case HS_TYPE_INT64: HS_HIST(HS_TYPE_INT64); break;
    default: HS_HIST(-1); break;
  }
#undef HS_HIST
  HS_LAUNCH_CHECK(ctx);
}

struct PartitionLaunch {
  const KeyColumn* d_keys;
  int nkeys;
  int64_t nrows;
  int num_buckets, owner_mod;
  const uint32_t* tile_dst;
  const PartColumn* d_cols;
  int ncols;
  void* const* d_peer_out;
  int out_world;
  CodePackRound pack;
  const uint16_t* bin_ids;
};

template <int BITS, int KT, bool PEER>
void launch_partition_rows_t(hs_ctx* ctx, const PartitionLaunch& a) {
  const int nb = a.owner_mod > 0 ? a.owner_mod : a.num_buckets;
  const int64_t ntiles = ceil_div(a.nrows, FusedCfg<PEER>::kTile);
  static DeviceOnce attr_once;  // one per instantiation
  bool& attr = attr_once(ctx->device);
  if (!attr) {
    HS_CUDA(cudaFuncSetAttribute(k_partition_rows<BITS, KT, PEER>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 (int)fused_smem_bytes<PEER>(kFusedMaxBins)));
    attr = true;
  }
  k_partition_rows<BITS, KT, PEER><<<(unsigned)ntiles, FusedCfg<PEER>::kThreads, fused_smem_bytes<PEER>(nb), ctx->stream>>>(
      a.d_keys, a.nkeys, a.nrows, make_mod_const((uint32_t)a.num_buckets), make_mod_const((uint32_t)std::max(a.owner_mod, 1)),
      a.owner_mod > 0 ? 1 : 0, a.tile_dst, a.d_cols, a.ncols, a.d_peer_out, a.out_world, a.pack, a.bin_ids);
  HS_LAUNCH_CHECK(ctx);
}

template <int BITS, bool PEER>
void launch_partition_rows_bits(hs_ctx* ctx, const PartitionLaunch& a, int single_key_type) {
  switch (single_key_type) {
    case HS_TYPE_INT32: launch_partition_rows_t<BITS, HS_TYPE_INT32, PEER>(ctx, a); break;
    case HS_TYPE_INT64: launch_partition_rows_t<BITS, HS_TYPE_INT64, PEER>(ctx, a); break;
    default: launch_partition_rows_t<BITS, -1, PEER>(ctx, a);
  }
}

template <bool PEER>
void launch_partition_rows(hs_ctx* ctx, const PartitionLaunch& a, int single_key_type) {
  const int nb = a.owner_mod > 0 ? a.owner_mod : a.num_buckets;
  // the ranking votes once per bin-id bit: 4, 8 or 10 (kFusedMaxBins = 1024)
  if (nb <= 16) launch_partition_rows_bits<4, PEER>(ctx, a, single_key_type);
  else if (nb <= 256) launch_partition_rows_bits<8, PEER>(ctx, a, single_key_type);
  else launch_partition_rows_bits<10, PEER>(ctx, a, single_key_type);
}

}  // namespace

int partition_tile_rows(hs_ctx* ctx, int num_buckets) {
  if (num_buckets > kFusedMaxBins) return 0;
  return ctx->world > 1 ? kFusedTilePeer : kFusedTileLocal;
}

void hash_rows(hs_ctx* ctx, const KeyColumn* keys, int nkeys, int64_t nrows, int num_buckets, int owner_mod, bool to_peers,
               unsigned long long* global_hist, unsigned long long* key_or_and, HashedRows* out) {
  HashedRows& h = *out;
  h.nrows = nrows;
  h.num_buckets = num_buckets;
  h.owner_mod = owner_mod;
  h.nbins = owner_mod > 0 ? owner_mod : num_buckets;
  if (to_peers && h.nbins > kFusedMaxBins) fail(HS_EINVAL, "%d bins: rows go to peer GPUs only up to %d", h.nbins, kFusedMaxBins);
  h.to_peers = to_peers;
  h.single_key_type = single_key_type_of(keys, nkeys);
  h.nkeys = nkeys;
  h.keys.alloc(ctx, nkeys);
  copy_h2d(ctx, h.keys.get(), keys, sizeof(KeyColumn) * nkeys);
  // the unfused partition's tile is the local one: k_partition_dest ranks the rows k_tile_hist counted
  h.ntiles = ceil_div(nrows, to_peers ? kFusedTilePeer : kFusedTileLocal);
  h.tile_hist.alloc(ctx, std::max<int64_t>(1, h.ntiles) * h.nbins);
  if (owner_mod == 0) h.bin_ids.alloc(ctx, std::max<int64_t>(1, nrows));
  KernelScope _ks(ctx, "k_tile_hist");
  if (nrows == 0) return;
  if (to_peers) launch_tile_hist<true>(ctx, h, global_hist, key_or_and);
  else launch_tile_hist<false>(ctx, h, global_hist, key_or_and);
}

void move_rows(hs_ctx* ctx, const HashedRows& h, const PartColumn* cols, int ncols, const CodePackRound* pack,
               void* const* peer_out, int peers) {
  if ((peer_out != nullptr) != h.to_peers) fail(HS_EINVAL, "move_rows: a peer table is needed exactly when rows go to peers");
  if (h.nbins > kFusedMaxBins) {  // bin ids -> destinations -> one scatter per column
    if (pack && pack->n > 0) fail(HS_EINVAL, "%d bins: code records need at most %d bins", h.nbins, kFusedMaxBins);
    for (int c = 0; c < ncols; c++)
      if (cols[c].tiles) fail(HS_EINVAL, "%d bins: columns are read in place only up to %d bins", h.nbins, kFusedMaxBins);
    Buf<uint32_t> dest(ctx, std::max<int64_t>(1, h.nrows));
    launch_partition_dest(ctx, h.bin_ids.get(), h.nrows, h.nbins, h.tile_hist.get(), dest.get());
    for (int c = 0; c < ncols; c++) launch_scatter_column(ctx, cols[c].in, cols[c].out, dest.get(), h.nrows, cols[c].width);
    return;
  }
  Buf<PartColumn> d_cols(ctx, std::max(1, ncols));
  copy_h2d(ctx, d_cols.get(), cols, sizeof(PartColumn) * ncols);
  KernelScope _ks(ctx, "k_partition_rows");
  if (h.nrows == 0) return;
  PartitionLaunch a{h.keys.get(), h.nkeys, h.nrows, h.num_buckets, h.owner_mod, h.tile_hist.get(), d_cols.get(), ncols,
                    peer_out, h.to_peers ? peers : 1, {}, h.bin_ids.get()};
  memset(&a.pack, 0, sizeof a.pack);
  if (pack) a.pack = *pack;
  if (h.to_peers) launch_partition_rows<true>(ctx, a, h.single_key_type);
  else launch_partition_rows<false>(ctx, a, h.single_key_type);
}

}  // namespace hs
