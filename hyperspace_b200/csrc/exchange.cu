// exchange.cu -- the path's only exchange step: rows move to the GPU that owns their bucket.
//
// Replaces Spark's shuffle behind `indexData.repartition(numBuckets, indexedColumns)`
// (index/covering/CoveringIndex.scala:60; on-the-fly variant covering/CoveringIndexRuleUtils.scala:413).
// One process per GPU.  owner(bucket) = bucket % world.  Up to 1024 buckets the partition kernel itself stores every row
// into its owner's memory (exchange_partition_p2p, below).  Above that, each rank partitions its decoded rows by owner
// with the same stable counting sort as K3 (hash_partition.cu), all-gathers the world x world count matrix, and then
// moves every column with ONE grouped ncclSend/ncclRecv all-to-all over NVLink.  NCCL is resolved with dlopen so that a
// single-GPU deployment has no NCCL dependency and so that, inside a torch process, the already-loaded NCCL is used.
#include <dlfcn.h>

#include <map>

#include "device_utils.cuh"
#include "engine.h"

namespace {

struct NcclUniqueId {
  char internal[128];
};
typedef void* ncclComm_t;
enum { kNcclUint8 = 1, kNcclUint64 = 5 };

struct NcclApi {
  void* handle = nullptr;
  int (*GetUniqueId)(NcclUniqueId*) = nullptr;
  int (*CommInitRank)(ncclComm_t*, int, NcclUniqueId, int) = nullptr;
  int (*CommDestroy)(ncclComm_t) = nullptr;
  int (*AllGather)(const void*, void*, size_t, int, ncclComm_t, cudaStream_t) = nullptr;
  int (*Send)(const void*, size_t, int, int, ncclComm_t, cudaStream_t) = nullptr;
  int (*Recv)(void*, size_t, int, int, ncclComm_t, cudaStream_t) = nullptr;
  int (*GroupStart)() = nullptr;
  int (*GroupEnd)() = nullptr;
  const char* (*GetErrorString)(int) = nullptr;
};

NcclApi& nccl() {
  static NcclApi api;
  if (api.handle) return api;
  const char* names[] = {"libnccl.so.2", "libnccl.so"};
  for (const char* n : names) {
    api.handle = dlopen(n, RTLD_NOW | RTLD_GLOBAL);
    if (api.handle) break;
  }
  if (!api.handle) hs::fail(HS_ECOMM, "cannot load libnccl.so.2: %s", dlerror());
#define HS_NCCL_SYM(field, sym)                                          \
  api.field = (decltype(api.field))dlsym(api.handle, sym);               \
  if (!api.field) hs::fail(HS_ECOMM, "libnccl is missing symbol %s", sym);
  HS_NCCL_SYM(GetUniqueId, "ncclGetUniqueId")
  HS_NCCL_SYM(CommInitRank, "ncclCommInitRank")
  HS_NCCL_SYM(CommDestroy, "ncclCommDestroy")
  HS_NCCL_SYM(AllGather, "ncclAllGather")
  HS_NCCL_SYM(Send, "ncclSend")
  HS_NCCL_SYM(Recv, "ncclRecv")
  HS_NCCL_SYM(GroupStart, "ncclGroupStart")
  HS_NCCL_SYM(GroupEnd, "ncclGroupEnd")
  HS_NCCL_SYM(GetErrorString, "ncclGetErrorString")
#undef HS_NCCL_SYM
  return api;
}

#define HS_NCCL(expr)                                                                              \
  do {                                                                                             \
    int _r = (expr);                                                                               \
    if (_r != 0) hs::fail(HS_ECOMM, "%s failed: %s", #expr, nccl().GetErrorString(_r));            \
  } while (0)

}  // namespace

struct hs_comm_state {
  ncclComm_t comm = nullptr;
};

namespace hs {

void close_peer_mappings(hs_ctx* ctx);

void comm_destroy(hs_ctx* ctx) {
  close_peer_mappings(ctx);
  if (ctx->comm) {
    if (ctx->comm->comm) nccl().CommDestroy(ctx->comm->comm);
    delete ctx->comm;
    ctx->comm = nullptr;
  }
}

// All-gather of small host blobs (every rank contributes `bytes`; out = world x bytes, rank-major).  Used for the
// agreement steps around the data path (dictionary unions, flags); the rows themselves never come this way.
void comm_allgather_host(hs_ctx* ctx, const void* in, size_t bytes, void* out) {
  if (ctx->world <= 1) {
    memcpy(out, in, bytes);
    return;
  }
  if (!ctx->comm || !ctx->comm->comm) fail(HS_ECOMM, "hs_comm_init has not been called on this context");
  Buf<uint8_t> d_in(ctx, std::max<size_t>(bytes, 16)), d_out(ctx, std::max<size_t>(bytes, 16) * ctx->world);
  copy_h2d(ctx, d_in.get(), in, bytes);
  HS_NCCL(nccl().AllGather(d_in.get(), d_out.get(), bytes, kNcclUint8, ctx->comm->comm, ctx->stream));
  copy_d2h(ctx, out, d_out.get(), bytes * ctx->world);
  sync_stream(ctx);
}

void exchange_rows(hs_ctx* ctx, Table& table, int nkeys, int num_buckets, hs_stats* stats) {
  const int world = ctx->world;
  if (world <= 1) return;
  if (!ctx->comm || !ctx->comm->comm) fail(HS_ECOMM, "hs_comm_init has not been called on this context");
  const int64_t nrows = table.nrows;
  const int ncols = (int)table.cols.size();
  StageTimer t_part(ctx), t_x(ctx);
  // ---- partition by owner rank (stable) -----------------------------------------------------------------------
  t_part.start();
  std::vector<KeyColumn> h_keys(nkeys);
  for (int k = 0; k < nkeys; k++) h_keys[k] = key_column_of(table.cols[k]);
  Buf<unsigned long long> ghist(ctx, world);
  Buf<uint64_t> d_send_off(ctx, world + 1);
  fill_bytes(ctx, ghist.get(), 0, 8 * world);
  HashedRows owners;  // bins are the owner ranks; the send buffers are local memory
  hash_rows(ctx, h_keys.data(), nkeys, nrows, num_buckets, world, false, ghist.get(), nullptr, &owners);
  launch_tile_offsets(ctx, owners.tile_hist.get(), owners.ntiles, world, ghist.get(), (unsigned long long*)d_send_off.get());
  // ---- count matrix -----------------------------------------------------------------------------------------
  Buf<uint64_t> d_matrix(ctx, (size_t)world * world);  // row r = counts rank r sends to each destination
  HS_NCCL(nccl().AllGather(ghist.get(), d_matrix.get(), world, kNcclUint64, ctx->comm->comm, ctx->stream));
  std::vector<uint64_t> matrix((size_t)world * world), send_off(world + 1);
  copy_d2h(ctx, matrix.data(), d_matrix.get(), 8 * (size_t)world * world);
  copy_d2h(ctx, send_off.data(), d_send_off.get(), 8 * (world + 1));
  sync_stream(ctx);
  std::vector<uint64_t> recv_off(world + 1, 0);
  for (int r = 0; r < world; r++) recv_off[r + 1] = recv_off[r] + matrix[(size_t)r * world + ctx->rank];
  const int64_t n_recv = (int64_t)recv_off[world];
  if (n_recv >= (1ll << 32)) fail(HS_EUNSUPPORTED, "more than 2^32-1 rows land on one GPU");
  // any rank seeing nulls makes the column nullable everywhere
  // (has_nulls flags travel as one more tiny all-gather folded into the matrix would be neater; a second call is fine)
  Buf<uint64_t> d_nulls(ctx, (size_t)ncols), d_nulls_all(ctx, (size_t)ncols * world);
  std::vector<uint64_t> h_nulls(ncols), h_nulls_all((size_t)ncols * world);
  for (int c = 0; c < ncols; c++) h_nulls[c] = table.cols[c].has_nulls ? 1 : 0;
  copy_h2d(ctx, d_nulls.get(), h_nulls.data(), 8 * ncols);
  HS_NCCL(nccl().AllGather(d_nulls.get(), d_nulls_all.get(), ncols, kNcclUint64, ctx->comm->comm, ctx->stream));
  copy_d2h(ctx, h_nulls_all.data(), d_nulls_all.get(), 8 * (size_t)ncols * world);
  sync_stream(ctx);
  // ---- partition into send buffers (rank-major, stable) ---------------------------------------------------------
  std::vector<Buf<uint8_t>> send_data(ncols), send_valid(ncols), recv_data(ncols), recv_valid(ncols);
  std::vector<bool> any_nulls(ncols, false);
  std::vector<PartColumn> h_pc;
  for (int c = 0; c < ncols; c++) {
    for (int r = 0; r < world; r++) any_nulls[c] = any_nulls[c] || h_nulls_all[(size_t)r * ncols + c] != 0;
    DevColumn& col = table.cols[c];
    send_data[c].alloc(ctx, (size_t)nrows * col.width + 16);
    recv_data[c].alloc(ctx, (size_t)n_recv * col.width + 16);
    h_pc.push_back(PartColumn{col.data.get(), send_data[c].get(), col.width, 0, col.zero_copy ? col.zc_tiles.get() : nullptr});
    if (any_nulls[c]) {
      send_valid[c].alloc(ctx, (size_t)nrows + 16);
      recv_valid[c].alloc(ctx, (size_t)n_recv + 16);
      if (col.valid) h_pc.push_back(PartColumn{col.valid.get(), send_valid[c].get(), 1, 0});
      else fill_bytes(ctx, send_valid[c].get(), 1, (size_t)nrows + 16);
    }
  }
  move_rows(ctx, owners, h_pc.data(), (int)h_pc.size());
  sync_stream(ctx);
  for (int c = 0; c < ncols; c++) {
    table.cols[c].data.release();
    table.cols[c].valid.release();
  }
  t_part.stop();
  // ---- the all-to-all -----------------------------------------------------------------------------------------
  t_x.start();
  HS_NCCL(nccl().GroupStart());
  for (int c = 0; c < ncols; c++) {
    const int W = table.cols[c].width;
    for (int peer = 0; peer < world; peer++) {
      const uint64_t scount = send_off[peer + 1] - send_off[peer];
      const uint64_t rcount = recv_off[peer + 1] - recv_off[peer];
      if (scount) {
        HS_NCCL(nccl().Send(send_data[c].get() + send_off[peer] * W, scount * W, kNcclUint8, peer, ctx->comm->comm, ctx->stream));
        if (any_nulls[c])
          HS_NCCL(nccl().Send(send_valid[c].get() + send_off[peer], scount, kNcclUint8, peer, ctx->comm->comm, ctx->stream));
      }
      if (rcount) {
        HS_NCCL(nccl().Recv(recv_data[c].get() + recv_off[peer] * W, rcount * W, kNcclUint8, peer, ctx->comm->comm, ctx->stream));
        if (any_nulls[c])
          HS_NCCL(nccl().Recv(recv_valid[c].get() + recv_off[peer], rcount, kNcclUint8, peer, ctx->comm->comm, ctx->stream));
      }
      if (peer != ctx->rank) stats->bytes_exchanged += (int64_t)(scount * (W + (any_nulls[c] ? 1 : 0)));
    }
  }
  HS_NCCL(nccl().GroupEnd());
  t_x.stop();
  sync_stream(ctx);
  for (int c = 0; c < ncols; c++) {
    table.cols[c].data = std::move(recv_data[c]);
    table.cols[c].zero_copy = false;  // materialised by the exchange
    table.cols[c].zc_tiles.release();
    table.cols[c].has_nulls = any_nulls[c];
    if (any_nulls[c]) table.cols[c].valid = std::move(recv_valid[c]);
  }
  table.nrows = n_recv;
  table.file_row_begin.clear();
  stats->ms_partition += t_part.ms();
  stats->ms_exchange += t_x.ms();
}

}  // namespace hs

extern "C" {

int hs_comm_unique_id(void* out_id128, char* err, size_t errlen) {
  try {
    NcclUniqueId id;
    memset(&id, 0, sizeof id);
    HS_NCCL(nccl().GetUniqueId(&id));
    memcpy(out_id128, &id, 128);
    return HS_OK;
  } catch (const hs::Error& e) {
    if (err && errlen) {
      strncpy(err, e.what(), errlen - 1);
      err[errlen - 1] = 0;
    }
    return e.code;
  }
}

int hs_comm_init(hs_ctx* ctx, int rank, int world_size, const void* id128, char* err, size_t errlen) {
  if (!ctx || world_size < 1 || rank < 0 || rank >= world_size) return HS_EINVAL;
  try {
    HS_CUDA(cudaSetDevice(ctx->device));
    hs::comm_destroy(ctx);
    ctx->rank = rank;
    ctx->world = world_size;
    if (world_size == 1) return HS_OK;
    NcclUniqueId id;
    memcpy(&id, id128, 128);
    ctx->comm = new hs_comm_state();
    HS_NCCL(nccl().CommInitRank(&ctx->comm->comm, world_size, id, rank));
    return HS_OK;
  } catch (const hs::Error& e) {
    if (err && errlen) {
      strncpy(err, e.what(), errlen - 1);
      err[errlen - 1] = 0;
    }
    return e.code;
  }
}

}  // extern "C"

// =====================================================================================================================
// Fused partition + exchange over NVLink peer memory.
//
// The NCCL path above costs a send-buffer pass, the all-to-all and a second (local) partition by bucket.  Here the exchange IS the partition kernel: every rank all-gathers
// the per-bucket histograms, derives for each bucket its final position inside the owner's bucket-major receive buffers
// (source-rank-major inside a bucket, so the result is deterministic and identical to the single-GPU order), maps the
// owners' buffers with CUDA IPC, and k_partition_rows stores each bucket's run straight into peer memory.  One pass over
// the rows, no staging, and the NVLink transfer overlaps the kernel tile by tile.  NCCL is still used for the two tiny
// all-gathers (histograms, IPC handles) and the closing barrier.
// =====================================================================================================================
namespace hs {

namespace {

struct IpcKey {
  unsigned char b[sizeof(cudaIpcMemHandle_t)];
  bool operator<(const IpcKey& o) const { return memcmp(b, o.b, sizeof b) < 0; }
};

std::map<IpcKey, void*>& ipc_cache(hs_ctx* ctx) {
  static std::map<hs_ctx*, std::map<IpcKey, void*>> caches;
  return caches[ctx];
}

void* open_peer(hs_ctx* ctx, const cudaIpcMemHandle_t& h) {
  IpcKey k;
  memcpy(k.b, &h, sizeof h);
  auto& cache = ipc_cache(ctx);
  auto it = cache.find(k);
  if (it != cache.end()) return it->second;
  void* p = nullptr;
  HS_CUDA(cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess));
  cache[k] = p;
  return p;
}

}  // namespace

void close_peer_mappings(hs_ctx* ctx) {
  auto& cache = ipc_cache(ctx);
  for (auto& kv : cache) cudaIpcCloseMemHandle(kv.second);
  cache.clear();
}

void exchange_partition_p2p(hs_ctx* ctx, Table& table, int nkeys, int num_buckets, IndexedRows* out, hs_stats* stats) {
  const int world = ctx->world, me = ctx->rank;
  if (!ctx->comm || !ctx->comm->comm) fail(HS_ECOMM, "hs_comm_init has not been called on this context");
  const int64_t nrows = table.nrows;
  const int ncols = (int)table.cols.size();
  const int nb = num_buckets;
  auto t_hash = std::make_unique<StageTimer>(ctx), t_x = std::make_unique<StageTimer>(ctx);
  t_hash->start();
  std::vector<KeyColumn> h_keys(nkeys);
  for (int k = 0; k < nkeys; k++) h_keys[k] = key_column_of(table.cols[k]);

  // ---- receive buffers, allocated BEFORE the ranks talk ---------------------------------------------------------------
  // Their capacity is a bound derived from the global row count the ranks exchanged while decoding (a uniform hash puts
  // total / world rows on every GPU give or take a per-mille), so that the IPC handles can travel in the SAME all-gather as
  // the bucket histograms; same sizes every call also mean the pool returns the same blocks and the peers' mappings of
  // them stay cached.  Should the bound not hold on some rank (or a column hold nulls somewhere, which needs validity
  // buffers too), every rank sees it in the gathered message and all take the second round below.
  const int64_t total_rows = table.global_rows;
  const int64_t cap_rows = total_rows >= 0 ? (int64_t)((double)ceil_div(nb, world) * ((double)total_rows / nb) * 1.10) + 4096 : 0;
  if (cap_rows >= (1ll << 32)) fail(HS_EUNSUPPORTED, "more than 2^32-1 rows land on one GPU");
  out->part.cols.clear();
  out->part.cols.resize(ncols);
  std::vector<PartColumn> h_pc;          // what the kernel moves (data columns, then validity where needed)
  std::vector<void*> my_recv;            // receive buffer of every moved column on this rank
  CodePackRound pack;                    // late-materialised columns: their codes leave as one record per row
  memset(&pack, 0, sizeof pack);
  for (int c = 0; c < ncols; c++) {
    DevColumn& src = table.cols[c];
    DevColumn& dst = out->part.cols[c];
    dst.name = src.name;
    dst.type = src.type;
    dst.width = src.width;
    dst.schema = src.schema;
    if (src.carried) {  // every rank carries the same columns with the same dictionary (decode_sources agreed on both)
      if (c < nkeys || pack.n >= kMaxCarried) fail(HS_EINVAL, "column '%s' cannot be late-materialised here", src.name.c_str());
      dst.carried = true;
      dst.dict_values = std::move(src.dict_values);
      dst.dict_bw = src.dict_bw;
      dst.carry_slot = pack.n;
      pack.src[pack.n++] = src.codes.get();
      continue;
    }
    if (cap_rows > 0) {
      dst.data.alloc(ctx, (size_t)cap_rows * src.width + 16);
      ctx->pool.mark_exported(dst.data.get());
    }
    h_pc.push_back(PartColumn{src.data.get(), nullptr, src.width, 0, src.zero_copy ? src.zc_tiles.get() : nullptr});
    my_recv.push_back(dst.data.get());
  }
  const int ndata = (int)h_pc.size();
  if (pack.n > 0) {
    if (cap_rows > 0) {
      out->part.rec.alloc(ctx, (size_t)cap_rows * 8 + 16);
      ctx->pool.mark_exported(out->part.rec.get());
    }
    my_recv.push_back(out->part.rec.get());
  }
  const int nfast = (int)my_recv.size();  // buffers whose handles ride in the first message
  constexpr int kHandleWords = (int)(sizeof(cudaIpcMemHandle_t) / 8);
  static_assert(sizeof(cudaIpcMemHandle_t) % 8 == 0, "handle size");

  // ---- ONE message per rank: bucket histogram, has-nulls flags, OR / AND of the encoded key, capacity, IPC handles --------
  const int o_nulls = nb, o_bits = nb + ncols, o_cap = o_bits + 2, o_handles = o_cap + 1;
  const int msg = o_handles + nfast * kHandleWords;
  Buf<unsigned long long> d_mine(ctx, msg), d_all(ctx, (size_t)msg * world);
  std::vector<unsigned long long> h_mine(msg, 0), h_all((size_t)msg * world);
  for (int c = 0; c < ncols; c++) h_mine[o_nulls + c] = table.cols[c].has_nulls ? 1 : 0;
  h_mine[o_bits] = 0ull;
  h_mine[o_bits + 1] = ~0ull;
  h_mine[o_cap] = (unsigned long long)cap_rows;
  if (cap_rows > 0)
    for (int i = 0; i < nfast; i++) {
      cudaIpcMemHandle_t h;
      HS_CUDA(cudaIpcGetMemHandle(&h, my_recv[i]));
      memcpy(&h_mine[o_handles + (size_t)i * kHandleWords], &h, sizeof h);
    }
  copy_h2d(ctx, d_mine.get(), h_mine.data(), 8 * (size_t)msg);
  HashedRows hashed;  // the runs leave over NVLink
  hash_rows(ctx, h_keys.data(), nkeys, nrows, nb, 0, true, d_mine.get(), d_mine.get() + o_bits, &hashed);
  HS_NCCL(nccl().AllGather(d_mine.get(), d_all.get(), msg, kNcclUint64, ctx->comm->comm, ctx->stream));
  copy_d2h(ctx, h_all.data(), d_all.get(), 8 * (size_t)msg * world);
  sync_stream(ctx);
  t_hash->stop();

  // ---- layout of every owner's receive buffers ------------------------------------------------------------------
  t_x->start();
  auto cnt = [&](int r, int b) { return h_all[(size_t)r * msg + b]; };
  std::vector<unsigned long long> my_base(nb, 0);        // where MY rows of bucket b start inside the owner's buffers
  std::vector<uint64_t> my_bucket_offsets(nb + 1, 0);    // bucket-major layout of the rows THIS rank receives
  std::vector<uint64_t> owner_cursor(world, 0);
  for (int b = 0; b < nb; b++) {
    const int o = b % world;
    uint64_t before_me = 0, total = 0;
    for (int r = 0; r < world; r++) {
      if (r < me) before_me += cnt(r, b);
      total += cnt(r, b);
    }
    my_base[b] = owner_cursor[o] + before_me;
    owner_cursor[o] += total;
  }
  {  // non-owned buckets are empty segments: the offsets stay monotone (owned buckets are laid out in increasing b)
    uint64_t run = 0;
    for (int b = 0; b < nb; b++) {
      uint64_t total = 0;
      if ((b % world) == me)
        for (int r = 0; r < world; r++) total += cnt(r, b);
      my_bucket_offsets[b] = run;
      run += total;
    }
    my_bucket_offsets[nb] = run;
  }
  const int64_t n_recv = (int64_t)owner_cursor[me];
  bool second_round = cap_rows <= 0;
  for (int o = 0; o < world; o++) {
    if (owner_cursor[o] >= (1ull << 32)) fail(HS_EUNSUPPORTED, "more than 2^32-1 rows land on one GPU");
    if (owner_cursor[o] > h_all[(size_t)o * msg + o_cap]) second_round = true;  // some rank's bound did not hold
  }
  std::vector<bool> any_nulls(ncols, false);
  unsigned long long key_or = 0ull, key_and = ~0ull;
  for (int r = 0; r < world; r++) {
    for (int c = 0; c < ncols; c++) any_nulls[c] = any_nulls[c] || h_all[(size_t)r * msg + o_nulls + c] != 0;
    key_or |= h_all[(size_t)r * msg + o_bits];
    key_and &= h_all[(size_t)r * msg + o_bits + 1];
  }
  for (int c = 0; c < ncols; c++) second_round = second_round || any_nulls[c];
  // OR / AND of the encoded (last) key over ALL rows of all ranks: a superset of the bits that vary among the rows this rank
  // receives, which is all the sort needs to pick its passes (saves a pass over the received keys and a synchronisation)
  out->key_or_and[0] = key_or;
  out->key_or_and[1] = key_and;
  out->have_key_bits = true;

  out->part.nrows = n_recv;
  std::vector<void*> h_peer;
  int ncolmoved = ndata, nmoved = nfast;
  if (!second_round) {
    h_peer.resize((size_t)nfast * world);
    for (int i = 0; i < nfast; i++)
      for (int r = 0; r < world; r++) {
        if (r == me) {
          h_peer[(size_t)i * world + r] = my_recv[i];
          continue;
        }
        cudaIpcMemHandle_t h;
        memcpy(&h, &h_all[(size_t)r * msg + o_handles + (size_t)i * kHandleWords], sizeof h);
        h_peer[(size_t)i * world + r] = open_peer(ctx, h);
      }
    for (int c = 0; c < ncols; c++) out->part.cols[c].has_nulls = false;
  } else {
    // second round: exact sizes, validity buffers where a column holds nulls on some rank; handles in their own all-gather
    h_pc.clear();
    my_recv.clear();
    for (int c = 0; c < ncols; c++) {
      DevColumn& src = table.cols[c];
      DevColumn& dst = out->part.cols[c];
      dst.has_nulls = any_nulls[c];
      if (dst.carried) continue;
      dst.data.alloc(ctx, (size_t)n_recv * src.width + 16);
      ctx->pool.mark_exported(dst.data.get());
      h_pc.push_back(PartColumn{src.data.get(), nullptr, src.width, 0, src.zero_copy ? src.zc_tiles.get() : nullptr});
      my_recv.push_back(dst.data.get());
      if (any_nulls[c]) {
        dst.valid.alloc(ctx, (size_t)n_recv + 16);
        ctx->pool.mark_exported(dst.valid.get());
        if (!src.valid) {  // this rank saw no nulls in the column but another did: ship all-ones
          src.valid.alloc(ctx, (size_t)nrows + 16);
          fill_bytes(ctx, src.valid.get(), 1, (size_t)nrows + 16);
        }
        h_pc.push_back(PartColumn{src.valid.get(), nullptr, 1, 0});
        my_recv.push_back(dst.valid.get());
      }
    }
    ncolmoved = (int)h_pc.size();  // the kernel's column rounds; the code records (if any) follow them
    if (pack.n > 0) {
      out->part.rec.alloc(ctx, (size_t)n_recv * 8 + 16);
      ctx->pool.mark_exported(out->part.rec.get());
      my_recv.push_back(out->part.rec.get());
    }
    nmoved = (int)my_recv.size();
    std::vector<cudaIpcMemHandle_t> my_handles(nmoved), all_handles((size_t)nmoved * world);
    for (int i = 0; i < nmoved; i++) HS_CUDA(cudaIpcGetMemHandle(&my_handles[i], my_recv[i]));
    const size_t hbytes = sizeof(cudaIpcMemHandle_t) * nmoved;
    Buf<uint8_t> d_h(ctx, hbytes), d_hall(ctx, hbytes * world);
    copy_h2d(ctx, d_h.get(), my_handles.data(), hbytes);
    HS_NCCL(nccl().AllGather(d_h.get(), d_hall.get(), hbytes, kNcclUint8, ctx->comm->comm, ctx->stream));
    copy_d2h(ctx, all_handles.data(), d_hall.get(), hbytes * world);
    sync_stream(ctx);
    h_peer.resize((size_t)nmoved * world);
    for (int i = 0; i < nmoved; i++)
      for (int r = 0; r < world; r++)
        h_peer[(size_t)i * world + r] = (r == me) ? my_recv[i] : open_peer(ctx, all_handles[(size_t)r * nmoved + i]);
  }

  // ---- one kernel: partition + exchange ------------------------------------------------------------------------
  Buf<unsigned long long> d_base(ctx, nb);
  Buf<void*> d_peer(ctx, (size_t)nmoved * world);
  copy_h2d(ctx, d_base.get(), my_base.data(), 8 * nb);
  copy_h2d(ctx, d_peer.get(), h_peer.data(), sizeof(void*) * nmoved * world);
  launch_tile_offsets(ctx, hashed.tile_hist.get(), hashed.ntiles, nb, d_mine.get(), nullptr, d_base.get());
  // the peer table holds one row of `world` pointers per column round, then one row for the code records
  move_rows(ctx, hashed, h_pc.data(), ncolmoved, &pack, (void* const*)d_peer.get(), world);
  // closing barrier: nobody reads its receive buffers before every peer's kernel has completed.  Stream-ordered -- the
  // sort that follows is enqueued behind it, the host does not wait here.
  HS_NCCL(nccl().AllGather(d_mine.get(), d_all.get(), 1, kNcclUint64, ctx->comm->comm, ctx->stream));
  t_x->stop();
  // (the source columns go back to the pool; it hands them out again only to work enqueued later on this stream)
  for (int c = 0; c < ncols; c++) {
    table.cols[c].data.release();
    table.cols[c].valid.release();
    table.cols[c].codes.release();
    table.cols[c].zc_tiles.release();
  }
  out->bucket_offsets = my_bucket_offsets;
  out->d_bucket_offsets.alloc(ctx, nb + 1);
  copy_h2d(ctx, out->d_bucket_offsets.get(), my_bucket_offsets.data(), 8 * (nb + 1));
  for (int r = 0; r < world; r++)
    if (r != me)
      for (int b = r; b < nb; b += world)
        for (int c = 0; c < ncols; c++)
          stats->bytes_exchanged += (int64_t)(cnt(me, b) * ((out->part.cols[c].carried ? 2 : table.cols[c].width) + (any_nulls[c] ? 1 : 0)));
  // the two stage timers are read after the call's next synchronisation (sort_partitioned_rows)
  out->pending_timers.push_back(IndexedRows::DeferredTimer{std::move(t_hash), &hs_stats::ms_hash});
  out->pending_timers.push_back(IndexedRows::DeferredTimer{std::move(t_x), &hs_stats::ms_exchange});
}

}  // namespace hs
