// api.cu -- the C ABI declared in include/hs_gpu.h.
#include <dirent.h>
#include <fcntl.h>
#include <sys/stat.h>
#include <unistd.h>

#include <algorithm>
#include <atomic>
#include <chrono>
#include <exception>
#include <map>
#include <mutex>
#include <thread>

#include "device_utils.cuh"
#include "engine.h"
#include "inflate.h"
#include "lz4_block.h"
#include "predicates.h"

using namespace hs;

#define HS_STR2(x) #x
#define HS_STR(x) HS_STR2(x)

namespace {

void set_err(char* err, size_t errlen, const char* msg) {
  if (err && errlen) {
    strncpy(err, msg, errlen - 1);
    err[errlen - 1] = 0;
  }
}

template <typename F>
int guarded(hs_ctx* ctx, char* err, size_t errlen, F&& f) {
  try {
    if (ctx) {
      cudaError_t e = cudaSetDevice(ctx->device);
      if (e != cudaSuccess) fail(HS_ECUDA, "cudaSetDevice(%d): %s", ctx->device, cudaGetErrorString(e));
      ctx->launches = 0;
    }
    f();
    return HS_OK;
  } catch (const hs::Error& e) {
    set_err(err, errlen, e.what());
    if (ctx) xfer_abort(ctx);
    cudaGetLastError();
    return e.code;
  } catch (const std::exception& e) {
    set_err(err, errlen, e.what());
    if (ctx) xfer_abort(ctx);
    cudaGetLastError();
    return HS_EINVAL;
  }
}

// hs_index_spec.compression -> the codec of the index pages: those Spark 3.1 writes and this engine reads back
int output_codec(int32_t compression) {
  switch (compression) {
    case HS_CODEC_UNCOMPRESSED: return pq::UNCOMPRESSED;
    case HS_CODEC_SNAPPY: return pq::SNAPPY;
    case HS_CODEC_GZIP: return pq::GZIP;
    case HS_CODEC_LZ4: return pq::LZ4;
    default:
      fail(HS_EUNSUPPORTED, "compression codec %d; the GPU path writes UNCOMPRESSED (0), SNAPPY (1), GZIP (2) and LZ4 (5) pages",
           compression);
  }
}
// the file-name extension of parquet-mr's CompressionCodecName
const char* codec_extension(int codec) {
  return codec == pq::SNAPPY ? ".snappy" : codec == pq::GZIP ? ".gz" : codec == pq::LZ4 ? ".lz4" : "";
}

void write_file_atomic(const std::string& dir, const std::string& name, const uint8_t* data, uint64_t size) {
  const std::string tmp = dir + "/." + name + ".tmp";
  const std::string fin = dir + "/" + name;
  int fd = open(tmp.c_str(), O_WRONLY | O_CREAT | O_TRUNC, 0644);
  if (fd < 0) fail(HS_EIO, "cannot create %s", tmp.c_str());
  uint64_t done = 0;
  while (done < size) {
    ssize_t w = write(fd, data + done, size - done);
    if (w <= 0) {
      close(fd);
      unlink(tmp.c_str());
      fail(HS_EIO, "short write on %s", tmp.c_str());
    }
    done += (uint64_t)w;
  }
  close(fd);
  if (rename(tmp.c_str(), fin.c_str()) != 0) {
    unlink(tmp.c_str());
    fail(HS_EIO, "cannot rename %s", tmp.c_str());
  }
}

void mkdirs(const std::string& path) {
  std::string cur;
  for (size_t i = 0; i <= path.size(); i++) {
    if (i == path.size() || path[i] == '/') {
      if (!cur.empty()) mkdir(cur.c_str(), 0755);
    }
    if (i < path.size()) cur += path[i];
  }
}

// Spark's DataPathFilter (util/PathUtils.scala:34-39): names starting with '_' or '.' are not data files
void remove_data_files(const std::string& dir) {
  DIR* d = opendir(dir.c_str());
  if (!d) return;
  while (dirent* e = readdir(d)) {
    if (e->d_name[0] == '.' || e->d_name[0] == '_') continue;
    unlink((dir + "/" + e->d_name).c_str());
  }
  closedir(d);
}

void fill_lineage(hs_ctx* ctx, Table& t, const hs_source_file* files, int n_files);
void drop_deleted_rows(hs_ctx* ctx, Table& t, const int64_t* deleted, int ndeleted);

// gather every column of `t` through idx (n_out rows)
void gather_table(hs_ctx* ctx, Table& t, const uint32_t* d_idx, int64_t n_out) {
  for (DevColumn& c : t.cols) {
    Buf<uint8_t> nd(ctx, (size_t)n_out * c.width + 16);
    launch_gather_plain(ctx, c.data.get(), d_idx, n_out, c.width, nd.get());
    c.data = std::move(nd);
    if (c.valid) {
      Buf<uint8_t> nv(ctx, (size_t)n_out + 16);
      launch_gather_plain(ctx, c.valid.get(), d_idx, n_out, 1, nv.get());
      c.valid = std::move(nv);
    }
  }
  t.nrows = n_out;
}

__global__ void k_fill_u64(uint64_t* out, int64_t n, uint64_t v) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) out[i] = v;
}

// CoveringIndex.createIndexData lineage (index/covering/CoveringIndex.scala:152-186): every row carries the id of the
// source file it came from.
void fill_lineage(hs_ctx* ctx, Table& t, const hs_source_file* files, int n_files) {
  DevColumn dc;
  dc.name = "_data_file_id";
  dc.type = HS_TYPE_INT64;
  dc.width = 8;
  dc.schema.name = dc.name;
  dc.schema.type = pq::INT64;
  dc.schema.repetition = pq::OPTIONAL;
  dc.data.alloc(ctx, (size_t)t.nrows * 8 + 16);
  for (int f = 0; f < n_files; f++) {
    const int64_t b = t.file_row_begin[f], n = t.file_row_begin[f + 1] - b;
    if (n == 0) continue;
    const int grid = (int)std::min<int64_t>(ceil_div(n, 256), ctx->sm_count * 8);
    k_fill_u64<<<grid, 256, 0, ctx->stream>>>((uint64_t*)dc.data.get() + b, n, (uint64_t)files[f].file_id);
    HS_LAUNCH_CHECK(ctx);
  }
  t.cols.push_back(std::move(dc));
}

// Rows whose `_data_file_id` is in `deleted` are dropped (CoveringIndexTrait.refreshIncremental, deleted files branch,
// index/covering/CoveringIndexTrait.scala:78-94).
void drop_deleted_rows(hs_ctx* ctx, Table& t, const int64_t* deleted, int ndeleted) {
  int lc = -1;
  for (size_t c = 0; c < t.cols.size(); c++)
    if (t.cols[c].name == "_data_file_id") lc = (int)c;
  if (lc < 0) fail(HS_EINVAL, "deleted_file_ids given but the source has no _data_file_id column (index built without lineage)");
  if (t.nrows == 0) return;
  Buf<uint32_t> idx;
  const int64_t kept = select_rows(ctx, RowFilter{}, nullptr, t.nrows, (const int64_t*)t.cols[lc].data.get(), deleted, ndeleted, &idx);
  gather_table(ctx, t, idx.get(), kept);
}

std::vector<std::string> names_of(const char* const* a, int na, const char* const* b, int nb) {
  std::vector<std::string> v;
  for (int i = 0; i < na; i++) v.emplace_back(a[i]);
  for (int i = 0; i < nb; i++) v.emplace_back(b[i]);
  return v;
}

// HS_OUT_FILES: the file images in res->h_arena become <out_dir>/<name>, all or nothing
// File-system traffic of the boundary (source files in, bucket files out) runs on a few host threads: one thread alone
// does not saturate the page cache, and the reference's writer runs one task per bucket in parallel as well
// (index/DataFrameWriterExtensions.scala:59-66 under Spark's FileFormatWriter).
int io_threads(size_t n_items) {
  const unsigned hw = std::thread::hardware_concurrency();
  size_t cap = 16;
  if (const char* e = getenv("HS_IO_THREADS")) cap = (size_t)std::max(1, atoi(e));
  return (int)std::max<size_t>(1, std::min<size_t>({cap, n_items, (size_t)std::max(1u, hw / 2)}));
}

// fn(i) for i in [0, n) on io_threads(n) threads; the first exception is rethrown on the caller's thread
template <typename Fn>
void parallel_files(size_t n, Fn fn) {
  const int nt = io_threads(n);
  if (nt <= 1) {
    for (size_t i = 0; i < n; i++) fn(i);
    return;
  }
  std::atomic<size_t> next{0};
  std::atomic<bool> failed{false};
  std::exception_ptr first;
  std::mutex mu;
  std::vector<std::thread> pool;
  for (int t = 0; t < nt; t++)
    pool.emplace_back([&] {
      for (;;) {
        const size_t i = next.fetch_add(1);
        if (i >= n || failed.load()) return;
        try {
          fn(i);
        } catch (...) {
          std::lock_guard<std::mutex> g(mu);
          if (!first) first = std::current_exception();
          failed.store(true);
          return;
        }
      }
    });
  for (auto& th : pool) th.join();
  if (first) std::rethrow_exception(first);
}

void write_result_files(hs_index_result* res, const std::string& dir, int save_mode) {
  if (dir.empty()) fail(HS_EINVAL, "HS_OUT_FILES needs out_dir");
  mkdirs(dir);
  if (save_mode == HS_SAVE_OVERWRITE) remove_data_files(dir);
  std::vector<char> written(res->files.size(), 0);
  try {
    parallel_files(res->files.size(), [&](size_t i) {
      const OutFile& f = res->files[i];
      write_file_atomic(dir, f.name, res->h_arena.get() + f.offset, f.size);
      written[i] = 1;
    });
  } catch (...) {
    for (size_t i = 0; i < written.size(); i++)
      if (written[i]) unlink((dir + "/" + res->files[i].name).c_str());  // all-or-nothing
    throw;
  }
  res->h_arena.release();
}

void finish_result(hs_ctx* ctx, EncodedFiles& enc, int output, const char* out_dir, int save_mode, hs_index_result* res,
                   hs_stats* st) {
  res->ctx = ctx;
  res->output = output;
  res->files = enc.files;
  if (output == HS_OUT_DEVICE) {
    res->d_arena = std::move(enc.arena);
    return;
  }
  StageTimer t(ctx);
  t.start();
  res->h_arena.alloc(ctx, std::max<uint64_t>(enc.arena_bytes, 16), /*pinned=*/true);
  if (enc.arena_bytes)
    copy_d2h(ctx, res->h_arena.get(), enc.arena.get(), enc.arena_bytes);
  t.stop();
  sync_stream(ctx);
  st->ms_d2h += t.ms();
  if (output == HS_OUT_FILES) write_result_files(res, out_dir ? out_dir : "", save_mode);
}

void read_file_into(const char* path, uint8_t* dst, uint64_t size) {
  int fd = open(path, O_RDONLY);
  if (fd < 0) fail(HS_EIO, "cannot open %s", path);
  uint64_t got = 0;
  while (got < size) {
    ssize_t r = read(fd, dst + got, size - got);
    if (r <= 0) {
      close(fd);
      fail(HS_EIO, "short read on %s", path);
    }
    got += (uint64_t)r;
  }
  close(fd);
}

}  // namespace

// =====================================================================================================================
extern "C" {

int hs_abi_version(void) { return HS_ABI_VERSION; }

const char* hs_build_info(void) {
  return "hyperspace_b200 libhs_gpu 0.1.0; arch sm_90a; CUDA " HS_STR(CUDART_VERSION) "; nvcc -O3 -lineinfo";
}

int hs_init(int device_id, void* cuda_stream, hs_ctx** out, char* err, size_t errlen) {
  if (!out) return HS_EINVAL;
  *out = nullptr;
  int count = 0;
  cudaError_t e = cudaGetDeviceCount(&count);
  if (e != cudaSuccess || count == 0) {
    char buf[256];
    snprintf(buf, sizeof buf, "no CUDA device available (%s); libhs_gpu has no CPU fallback",
             e != cudaSuccess ? cudaGetErrorString(e) : "device count is 0");
    set_err(err, errlen, buf);
    cudaGetLastError();
    return HS_ENODEVICE;
  }
  if (device_id < 0 || device_id >= count) {
    set_err(err, errlen, "device id out of range");
    return HS_EINVAL;
  }
  hs_ctx* ctx = new hs_ctx();
  ctx->device = device_id;
  int rc = guarded(nullptr, err, errlen, [&] {
    HS_CUDA(cudaSetDevice(device_id));
    cudaDeviceProp prop;
    HS_CUDA(cudaGetDeviceProperties(&prop, device_id));
    ctx->sm_count = prop.multiProcessorCount;
    // sm_90a code runs on compute capability 9.0 exactly: arch-specific features are not forward compatible
    if (prop.major != 9 || prop.minor != 0)
      fail(HS_ENODEVICE, "device %d is sm_%d%d; this library is built for sm_90a only", device_id, prop.major, prop.minor);
    if (cuda_stream) {
      ctx->stream = (cudaStream_t)cuda_stream;
      ctx->own_stream = false;
    } else {
      HS_CUDA(cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking));
      ctx->own_stream = true;
    }
    HS_CUDA(cudaStreamCreateWithFlags(&ctx->h2d_stream, cudaStreamNonBlocking));
    HS_CUDA(cudaStreamCreateWithFlags(&ctx->d2h_stream, cudaStreamNonBlocking));
  });
  if (rc != HS_OK) {
    delete ctx;
    return rc == HS_ECUDA ? HS_ENODEVICE : rc;
  }
  *out = ctx;
  return HS_OK;
}

void hs_shutdown(hs_ctx* ctx) {
  if (!ctx) return;
  cudaSetDevice(ctx->device);
  xfer_release(ctx);
  if (ctx->decode_cache && ctx->decode_cache_free) ctx->decode_cache_free(ctx->decode_cache);
  ctx->decode_cache = nullptr;
  comm_destroy(ctx);
  if (ctx->own_stream) cudaStreamDestroy(ctx->stream);
  if (ctx->h2d_stream) {
    cudaStreamSynchronize(ctx->h2d_stream);
    cudaStreamDestroy(ctx->h2d_stream);
  }
  if (ctx->d2h_stream) {
    cudaStreamSynchronize(ctx->d2h_stream);
    cudaStreamDestroy(ctx->d2h_stream);
  }
  delete ctx;
}

void hs_trim(hs_ctx* ctx) {
  if (!ctx) return;
  cudaSetDevice(ctx->device);
  cudaStreamSynchronize(ctx->stream);
  ctx->pool.trim();
}

void hs_profile_enable(hs_ctx* ctx, int on) {
  if (!ctx) return;
  cudaSetDevice(ctx->device);
  cudaStreamSynchronize(ctx->stream);
  for (auto& k : ctx->kevents) {
    ctx->event_pool.push_back(k.a);
    ctx->event_pool.push_back(k.b);
  }
  ctx->kevents.clear();
  ctx->profile = on != 0;
}

int hs_profile_report(hs_ctx* ctx, char* out, size_t outlen) {
  if (!ctx || !out || !outlen) return HS_EINVAL;
  cudaSetDevice(ctx->device);
  cudaStreamSynchronize(ctx->stream);
  struct Acc {
    int launches = 0;
    double ms = 0;
    int64_t items = 0;
  };
  std::map<std::string, Acc> acc;
  for (auto& k : ctx->kevents) {
    float ms = 0;
    if (cudaEventElapsedTime(&ms, k.a, k.b) != cudaSuccess) {
      cudaGetLastError();
      continue;
    }
    Acc& e = acc[k.name];
    e.launches++;
    e.ms += ms;
    e.items += k.items;
  }
  std::string s = "{";
  bool first = true;
  for (auto& kv : acc) {
    char buf[256];
    snprintf(buf, sizeof buf, "%s\"%s\": {\"launches\": %d, \"ms\": %.6f", first ? "" : ", ", kv.first.c_str(), kv.second.launches,
             kv.second.ms);
    s += buf;
    if (kv.second.items) s += ", \"items\": " + std::to_string(kv.second.items);
    s += "}";
    first = false;
  }
  s += "}";
  if (s.size() + 1 > outlen) return HS_ENOMEM;
  memcpy(out, s.c_str(), s.size() + 1);
  for (auto& k : ctx->kevents) {
    ctx->event_pool.push_back(k.a);
    ctx->event_pool.push_back(k.b);
  }
  ctx->kevents.clear();
  return HS_OK;
}

void* hs_host_alloc(hs_ctx* ctx, size_t bytes) {
  if (!ctx) return nullptr;
  try {
    cudaSetDevice(ctx->device);
    return ctx->pool.get(bytes, true);
  } catch (...) {
    return nullptr;
  }
}

void hs_host_free(hs_ctx* ctx, void* p) {
  if (ctx && p) ctx->pool.put(p);
}

// ---- staging: host file images -> device, asynchronously on the H2D copy stream -----------------------------------------

int hs_stage_sources(hs_ctx* ctx, const hs_source_file* files, int32_t n_files, hs_staged** out, char* err, size_t errlen) {
  if (!ctx || !out || n_files < 0 || (n_files > 0 && !files)) return HS_EINVAL;
  *out = nullptr;
  std::unique_ptr<hs_staged> sg(new hs_staged());
  sg->ctx = ctx;
  int rc = guarded(ctx, err, errlen, [&] {
    const int launches_before = ctx->launches;
    std::vector<uint64_t> sizes(n_files), off(n_files);
    uint64_t total = 0;
    for (int f = 0; f < n_files; f++) {
      const hs_source_file& sf = files[f];
      if (sf.data && sf.on_device) fail(HS_EINVAL, "source file %d is already on the device", f);
      if (sf.data) {
        sizes[f] = sf.size;
      } else {
        if (!sf.path) fail(HS_EINVAL, "source file %d has neither data nor path", f);
        struct stat st;
        if (stat(sf.path, &st) != 0) fail(HS_EIO, "cannot stat %s", sf.path);
        sizes[f] = (uint64_t)st.st_size;
      }
      if (sizes[f] < 12) fail(HS_EFORMAT, "source file %d: too small to be a Parquet file", f);
      off[f] = total;
      total += round_up(sizes[f], 16) + 16;
    }
    sg->d_images.alloc(ctx, std::max<uint64_t>(total, 16));
    HS_CUDA(cudaEventCreate(&sg->begin));
    HS_CUDA(cudaEventRecord(sg->begin, ctx->h2d_stream));
    sg->files.resize(n_files);
    sg->names.resize(n_files);
    sg->metas.resize(n_files);
    // file system sources are read into pinned memory first (kept until the copy has completed): the buffers come from the
    // pool on this thread, the reads run on a few threads, and each file's H2D copy is queued as soon as its read is done
    std::vector<uint8_t*> pinned(n_files, nullptr);
    std::vector<size_t> disk;
    for (int f = 0; f < n_files; f++)
      if (!files[f].data) {
        sg->staging.emplace_back(ctx, sizes[f], /*pinned=*/true);
        pinned[f] = sg->staging.back().get();
        disk.push_back((size_t)f);
      }
    std::vector<std::atomic<int>> read_done(n_files);
    for (auto& d : read_done) d.store(0);
    std::exception_ptr read_error;
    std::thread reader;
    if (!disk.empty())
      reader = std::thread([&] {
        try {
          parallel_files(disk.size(), [&](size_t j) {
            const size_t f = disk[j];
            read_file_into(files[f].path, pinned[f], sizes[f]);
            read_done[f].store(1, std::memory_order_release);
          });
        } catch (...) {
          read_error = std::current_exception();
        }
        for (size_t f : disk)  // wake the consumer whatever happened
          if (!read_done[f].load()) read_done[f].store(-1, std::memory_order_release);
      });
    struct Joiner {
      std::thread& t;
      ~Joiner() {
        if (t.joinable()) t.join();
      }
    } joiner{reader};
    for (int f = 0; f < n_files; f++) {
      const hs_source_file& sf = files[f];
      sg->names[f] = sf.path ? sf.path : ("<memory file " + std::to_string(f) + ">");
      const uint8_t* host = (const uint8_t*)sf.data;
      if (!host) {
        int st;
        while ((st = read_done[f].load(std::memory_order_acquire)) == 0) std::this_thread::yield();
        if (st < 0) {
          if (reader.joinable()) reader.join();
          if (read_error) std::rethrow_exception(read_error);
          fail(HS_EIO, "cannot read %s", sf.path);
        }
        host = pinned[f];
      }
      // the footer is parsed here, from host memory, so that the build never has to fetch it back from the device
      sg->metas[f] = std::make_shared<hs::pq::FileMeta>(hs::pq::parse_footer(host, sizes[f], sg->names[f].c_str()));
      HS_CUDA(cudaMemcpyAsync(sg->d_images.get() + off[f], host, sizes[f], cudaMemcpyHostToDevice, ctx->h2d_stream));
      hs_source_file& o = sg->files[f];
      o.path = nullptr;  // patched to names[f].c_str() by hs_staged_file (the vector may still move here)
      o.data = sg->d_images.get() + off[f];
      o.size = sizes[f];
      o.file_id = sf.file_id;
      o.on_device = 1;
      o.reserved = 0;
      sg->bytes += sizes[f];
    }
    HS_CUDA(cudaEventCreate(&sg->ready));
    HS_CUDA(cudaEventRecord(sg->ready, ctx->h2d_stream));
    for (int f = 0; f < n_files; f++) ctx->staged[sg->files[f].data] = hs_ctx::StagedImage{sg->metas[f], sg->ready};
    ctx->launches = launches_before;
  });
  if (rc == HS_OK) *out = sg.release();
  return rc;
}

int32_t hs_staged_num_files(const hs_staged* s) { return s ? (int32_t)s->files.size() : 0; }

int hs_staged_file(const hs_staged* s, int32_t i, hs_source_file* out) {
  if (!s || !out || i < 0 || i >= (int32_t)s->files.size()) return HS_EINVAL;
  *out = s->files[i];
  out->path = s->names[i].c_str();
  return HS_OK;
}

// HS_TIMELINE=1: begin / end of every staged copy, build and drain relative to the first event seen, on stderr
static void timeline(hs_ctx* ctx, const char* what, cudaEvent_t a, cudaEvent_t b) {
  static const bool on = getenv("HS_TIMELINE") != nullptr;
  if (!on || !a || !b) return;
  static cudaEvent_t base = nullptr;
  if (!base) base = a;  // (leaks one reference to an event that may be destroyed later: diagnostics only, first event kept alive)
  float t0 = 0, t1 = 0;
  if (cudaEventElapsedTime(&t0, base, a) != cudaSuccess || cudaEventElapsedTime(&t1, base, b) != cudaSuccess) {
    cudaGetLastError();
    return;
  }
  fprintf(stderr, "[hs timeline] %-8s %10.2f -> %10.2f  (%8.2f ms)\n", what, t0, t1, t1 - t0);
}

int hs_staged_wait(hs_staged* s, float* ms_copy) {
  if (!s) return HS_EINVAL;
  cudaSetDevice(s->ctx->device);
  if (cudaEventSynchronize(s->ready) != cudaSuccess) return HS_ECUDA;
  if (ms_copy && cudaEventElapsedTime(ms_copy, s->begin, s->ready) != cudaSuccess) *ms_copy = 0;
  timeline(s->ctx, "H2D", s->begin, s->ready);
  return HS_OK;
}

void hs_staged_free(hs_staged* s) {
  if (!s) return;
  hs_ctx* ctx = s->ctx;
  cudaSetDevice(ctx->device);
  if (s->ready) {
    cudaEventSynchronize(s->ready);  // the copies read caller memory / pinned staging and write d_images
    cudaEventDestroy(s->ready);
  }
  if (s->begin && !getenv("HS_TIMELINE")) cudaEventDestroy(s->begin);  // (the timeline's base event is one of these)
  for (const hs_source_file& f : s->files) ctx->staged.erase(f.data);
  cudaStreamSynchronize(ctx->stream);  // a build that decodes these images may still be running
  delete s;
}

// ---- createIndex -----------------------------------------------------------------------------------------------------

int hs_create_index_async(hs_ctx* ctx, const hs_index_spec* spec, hs_pending** out, char* err, size_t errlen) {
  if (!ctx || !spec || !out) return HS_EINVAL;
  *out = nullptr;
  std::unique_ptr<hs_pending> pd(new hs_pending());
  pd->ctx = ctx;
  pd->res.reset(new hs_index_result());
  hs_stats& st = pd->st;
  memset(&st, 0, sizeof st);
  hs_index_result* res = pd->res.get();
  int rc = guarded(ctx, err, errlen, [&] {
    if (spec->n_indexed < 1) fail(HS_EINVAL, "at least one indexed column is required");
    if (spec->n_files < 0 || (spec->n_files > 0 && !spec->files)) fail(HS_EINVAL, "bad source file list");
    if (spec->output == HS_OUT_FILES && !spec->out_dir) fail(HS_EINVAL, "HS_OUT_FILES needs out_dir");
    HS_CUDA(cudaEventCreate(&pd->t_begin));
    HS_CUDA(cudaEventCreate(&pd->t_compute_end));
    HS_CUDA(cudaEventRecord(pd->t_begin, ctx->stream));
    std::vector<std::string> cols = names_of(spec->indexed_columns, spec->n_indexed, spec->included_columns, spec->n_included);
    for (size_t i = 0; i < cols.size(); i++)
      for (size_t j = i + 1; j < cols.size(); j++)
        if (cols[i] == cols[j]) fail(HS_EINVAL, "duplicate column '%s' in index config", cols[i].c_str());
    EncodedFiles enc;
    {
      Table table;
      // Included columns whose source pages are all dictionary-encoded travel through the build as 16-bit dictionary codes
      // (late materialisation).  Only where nothing between decode and encode needs their values: the fused partition (on
      // one GPU, or writing straight into the owners' memory on several), no rows to drop.  HS_NO_CARRY=1 switches it off
      // (A/B measurements; on several GPUs every rank must be given the same setting).
      const bool no_carry = getenv("HS_NO_CARRY") != nullptr;
      // 0 above 1024 buckets: the partition there moves materialised columns only
      const int part_tile_rows = partition_tile_rows(ctx, spec->num_buckets);
      CarryOptions carry;
      if (part_tile_rows > 0 && !spec->disable_dictionary && spec->n_deleted_file_ids == 0 && !no_carry) {
        carry.first_col = spec->n_indexed;
        carry.num_segments = spec->num_buckets;
      }
      // PLAIN, null-free, value-aligned columns are not decoded either: hash and partition read them in place from the file
      // images (zero copy), which therefore stay alive until the rows have been partitioned.  HS_NO_ZEROCOPY=1: A/B switch.
      if (part_tile_rows > 0 && spec->n_deleted_file_ids == 0 && !getenv("HS_NO_ZEROCOPY")) {
        carry.zc_tile_rows = part_tile_rows;
        carry.zc_first_col = spec->n_indexed;
        carry.zc_key = spec->n_indexed == 1;
      }
      SourceSet src;
      open_sources(ctx, spec->files, spec->n_files, &src, &st);
      refuse_boolean_keys(src, std::vector<std::string>(cols.begin(), cols.begin() + spec->n_indexed));
      decode_sources(ctx, src, cols, nullptr, &table, &st, &carry);
      const bool has_strings = table.has_strings;
      if (has_strings && ctx->world > 1)
        fail(HS_EUNSUPPORTED, "string / binary columns are not exchanged between GPUs yet: build this index on one GPU");
      if (spec->lineage) fill_lineage(ctx, table, spec->files, spec->n_files);
      if (spec->n_deleted_file_ids > 0) drop_deleted_rows(ctx, table, spec->deleted_file_ids, spec->n_deleted_file_ids);
      IndexedRows rows;
      EncodeRequest req;
      req.table = &rows.part;
      req.key_sorted = true;
      req.plan = &rows.plan;
      req.rows_per_page = spec->rows_per_page;
      req.rows_per_row_group = spec->rows_per_row_group;
      req.use_dictionary = spec->disable_dictionary == 0;
      req.codec = output_codec(spec->compression);
      const std::string uuid = spec->job_uuid ? spec->job_uuid : make_uuid();
      req.seg_names.resize(spec->num_buckets);
      for (int b = 0; b < spec->num_buckets; b++) {
        // Spark FileFormatWriter: part-<task>-<jobUUID>_<bucket>.c000<codec ext>.parquet ; bucket id parsed back by
        // BucketingUtils.getBucketId (relied on by actions/OptimizeAction.scala:110)
        char nm[160];
        snprintf(nm, sizeof nm, "part-%05d-%s_%05d.c000%s.parquet", b, uuid.c_str(), b, codec_extension(req.codec));
        req.seg_names[b] = nm;
      }
      // The files are laid out before the sort when their layout does not depend on the sorted order: a local sort of a
      // single integer key then stores the key straight into its pages (the sort calls this while its MSD scatter runs).
      // Otherwise the host lays the pages out below, while the GPU still sorts.
      EncodeLayout lay;
      const KeyPagesFn layout_before_sort = [&]() -> const KeyPageDest* {
        if (layout_needs_sorted_rows(rows.part)) return nullptr;
        req.seg_offsets = rows.bucket_offsets;
        req.probe = rows.probe.get();
        layout_segments(ctx, req, &lay, &enc, &st);
        return key_page_dest(lay, req, &enc);
      };
      if (ctx->world > 1 && part_tile_rows > 0) {
        // partition + exchange fused over NVLink peer memory, then the local sort
        exchange_partition_p2p(ctx, table, spec->n_indexed, spec->num_buckets, &rows, &st);
        sort_partitioned_rows(ctx, spec->n_indexed, spec->num_buckets, &rows, &st, /*defer_settle=*/true, &layout_before_sort);
      } else {
        if (ctx->world > 1) exchange_rows(ctx, table, spec->n_indexed, spec->num_buckets, &st);  // NCCL all-to-all
        index_rows(ctx, table, spec->n_indexed, spec->num_buckets, &rows, &st, /*defer_settle=*/true, &layout_before_sort);
      }
      // From here to the end of write_segments the host does not wait for the GPU unless it has to: the sort kernels are
      // queued and the verdict of the tie fix-up is on its way (settle_sort below).
      if (!has_strings) src.release_images();  // every column is materialised bucket-major now (string
                                                         // references keep pointing into the images until the encode)
      req.d_perm = rows.sorted.perm();
      if (!rows.sorted.key_pages_written) req.d_sorted_keys = rows.sorted.keys();
      if (!lay.impl) {
        req.seg_offsets = rows.bucket_offsets;
        req.probe = rows.probe.get();
        layout_segments(ctx, req, &lay, &enc, &st);
      }
      write_segments(ctx, req, lay, rows.sorted.key_pages_written, &enc, &st);  // synchronises the stream before it returns
      if (settle_sort(ctx, &rows, &st)) {    // (rare) the fix-up gave up on a long run of equal key prefixes: the rows were sorted
        req.probe = nullptr;                 // again with full passes, so the pages are gathered again
        req.d_perm = rows.sorted.perm();
        req.d_sorted_keys = rows.sorted.keys();
        enc = EncodedFiles();
        encode_segments(ctx, req, &enc, &st);
      }
      st.rows_out = rows.part.nrows;
      // the decoded / partitioned / sorted intermediates go back to the pool here: while this call's index files drain to
      // the host, the next call can already build in the same memory
    }
    HS_CUDA(cudaEventRecord(pd->t_compute_end, ctx->stream));
    res->ctx = ctx;
    res->output = spec->output;
    res->files = enc.files;
    pd->save_mode = spec->save_mode;
    if (spec->out_dir) pd->out_dir = spec->out_dir;
    st.gpu_launches = ctx->launches;
    if (spec->output == HS_OUT_DEVICE) {
      res->d_arena = std::move(enc.arena);
      return;
    }
    // device -> host on the D2H copy stream; hs_pending_wait picks it up
    pd->d_arena = std::move(enc.arena);
    res->h_arena.alloc(ctx, std::max<uint64_t>(enc.arena_bytes, 16), /*pinned=*/true);
    HS_CUDA(cudaEventCreate(&pd->t_d2h_begin));
    HS_CUDA(cudaEventCreate(&pd->t_d2h_end));
    HS_CUDA(cudaStreamWaitEvent(ctx->d2h_stream, pd->t_compute_end, 0));
    HS_CUDA(cudaEventRecord(pd->t_d2h_begin, ctx->d2h_stream));
    if (enc.arena_bytes)
      HS_CUDA(cudaMemcpyAsync(res->h_arena.get(), pd->d_arena.get(), enc.arena_bytes, cudaMemcpyDeviceToHost, ctx->d2h_stream));
    HS_CUDA(cudaEventRecord(pd->t_d2h_end, ctx->d2h_stream));
    pd->has_d2h = true;
  });
  if (rc == HS_OK) *out = pd.release();
  return rc;
}

int hs_pending_wait(hs_pending* p, hs_index_result** out, hs_stats* stats, char* err, size_t errlen) {
  if (!p || !out) return HS_EINVAL;
  *out = nullptr;
  std::unique_ptr<hs_pending> pd(p);  // consumed either way
  hs_ctx* ctx = pd->ctx;
  const int launches = ctx->launches;
  int rc = guarded(ctx, err, errlen, [&] {
    hs_stats& st = pd->st;
    float ms = 0;
    if (pd->has_d2h) {
      HS_CUDA(cudaEventSynchronize(pd->t_d2h_end));
      HS_CUDA(cudaEventElapsedTime(&ms, pd->t_d2h_begin, pd->t_d2h_end));
      st.ms_d2h += ms;
      HS_CUDA(cudaEventElapsedTime(&ms, pd->t_begin, pd->t_d2h_end));
      st.ms_total = ms;
      timeline(ctx, "build", pd->t_begin, pd->t_compute_end);
      timeline(ctx, "D2H", pd->t_d2h_begin, pd->t_d2h_end);
      pd->d_arena.release();
    } else {
      HS_CUDA(cudaEventSynchronize(pd->t_compute_end));
      HS_CUDA(cudaEventElapsedTime(&ms, pd->t_begin, pd->t_compute_end));
      st.ms_total = ms;
    }
    if (pd->res->output == HS_OUT_FILES) {
      const auto w0 = std::chrono::steady_clock::now();
      write_result_files(pd->res.get(), pd->out_dir, pd->save_mode);
      st.ms_write += std::chrono::duration<float, std::milli>(std::chrono::steady_clock::now() - w0).count();
    }
  });
  ctx->launches = launches;
  if (stats) *stats = pd->st;
  if (rc == HS_OK) *out = pd->res.release();
  return rc;
}

void hs_pending_cancel(hs_pending* p) {
  if (!p) return;
  cudaSetDevice(p->ctx->device);
  if (p->has_d2h) cudaEventSynchronize(p->t_d2h_end);
  delete p;
}

int hs_create_index(hs_ctx* ctx, const hs_index_spec* spec, hs_index_result** out, hs_stats* stats, char* err,
                    size_t errlen) {
  if (!ctx || !spec || !out) return HS_EINVAL;
  *out = nullptr;
  if (stats) memset(stats, 0, sizeof *stats);
  hs_pending* pd = nullptr;
  int rc = hs_create_index_async(ctx, spec, &pd, err, errlen);
  if (rc != HS_OK) return rc;
  const int launches = ctx->launches;
  rc = hs_pending_wait(pd, out, stats, err, errlen);
  if (stats) stats->gpu_launches = launches;
  return rc;
}

int32_t hs_result_num_files(const hs_index_result* r) { return r ? (int32_t)r->files.size() : 0; }

int hs_result_file(const hs_index_result* r, int32_t i, int32_t* bucket, const char** name, const void** data,
                   uint64_t* size, int64_t* rows) {
  if (!r || i < 0 || i >= (int32_t)r->files.size()) return HS_EINVAL;
  const OutFile& f = r->files[i];
  if (bucket) *bucket = f.bucket;
  if (name) *name = f.name.c_str();
  if (data) {
    if (r->output == HS_OUT_DEVICE) *data = r->d_arena.get() + f.offset;
    else if (r->output == HS_OUT_HOST) *data = r->h_arena.get() + f.offset;
    else *data = nullptr;
  }
  if (size) *size = f.size;
  if (rows) *rows = f.rows;
  return HS_OK;
}

void hs_result_free(hs_index_result* r) {
  if (!r) return;
  if (r->ctx) {
    cudaSetDevice(r->ctx->device);
    cudaStreamSynchronize(r->ctx->stream);
  }
  delete r;
}

// ---------------------------------------------------------------------------------------------------------------------
// read side
// ---------------------------------------------------------------------------------------------------------------------

// padded: d_idx may hold kNoRow (an outer join's null-supplying side), which gives a null; every column then has a
// validity vector
static void batch_from_gather(hs_ctx* ctx, const Table& t, const std::vector<int>& col_idx, const uint32_t* d_idx,
                              int64_t n_out, hs_batch* b, bool padded = false) {
  // all gathers first, then all copies, one synchronisation at the end
  std::vector<Buf<uint8_t>> d_data, d_valid;
  std::vector<Buf<uint64_t>> d_offsets(col_idx.size());
  std::vector<uint64_t> str_bytes(col_idx.size(), 0);
  for (size_t k = 0; k < col_idx.size(); k++) {
    const int ci = col_idx[k];
    const DevColumn& c = t.cols[ci];
    if (padded) {
      const uint8_t* valid = c.has_nulls ? c.valid.get() : nullptr;
      d_valid.emplace_back(ctx, (size_t)std::max<int64_t>(1, n_out));
      if (c.type == HS_TYPE_STRING) {
        Buf<uint32_t> lens(ctx, (size_t)std::max<int64_t>(1, n_out));
        d_offsets[k].alloc(ctx, (size_t)n_out + 1);
        launch_string_lengths_padded(ctx, (const uint64_t*)c.data.get(), valid, d_idx, n_out, lens.get(), d_valid.back().get());
        exclusive_scan_u32_u64(ctx, lens.get(), n_out, d_offsets[k].get());
        copy_d2h(ctx, &str_bytes[k], d_offsets[k].get() + n_out, 8);
        sync_stream(ctx);
        d_data.emplace_back(ctx, std::max<uint64_t>(1, str_bytes[k]));
        launch_copy_strings_padded(ctx, (const uint64_t*)c.data.get(), valid, d_idx, n_out, d_offsets[k].get(), d_data.back().get());
      } else {
        d_data.emplace_back(ctx, (size_t)std::max<int64_t>(1, n_out) * c.width);
        launch_gather_padded(ctx, c.data.get(), valid, d_idx, n_out, c.width, d_data.back().get(), d_valid.back().get());
      }
      continue;
    }
    if (c.type == HS_TYPE_STRING) {
      // values are references into the source images (still alive here): lengths -> offsets -> one copy of the bytes
      const uint8_t* valid = c.has_nulls ? c.valid.get() : nullptr;
      Buf<uint32_t> lens(ctx, (size_t)std::max<int64_t>(1, n_out));
      d_offsets[k].alloc(ctx, (size_t)n_out + 1);
      launch_string_lengths(ctx, (const uint64_t*)c.data.get(), valid, d_idx, n_out, lens.get());
      exclusive_scan_u32_u64(ctx, lens.get(), n_out, d_offsets[k].get());
      copy_d2h(ctx, &str_bytes[k], d_offsets[k].get() + n_out, 8);
      sync_stream(ctx);
      d_data.emplace_back(ctx, std::max<uint64_t>(1, str_bytes[k]));
      launch_copy_strings(ctx, (const uint64_t*)c.data.get(), valid, d_idx, n_out, d_offsets[k].get(), d_data.back().get());
      d_valid.emplace_back();
      if (c.has_nulls) {
        d_valid.back().alloc(ctx, (size_t)std::max<int64_t>(1, n_out));
        launch_gather_plain(ctx, c.valid.get(), d_idx, n_out, 1, d_valid.back().get());
      }
      continue;
    }
    d_data.emplace_back(ctx, (size_t)std::max<int64_t>(1, n_out) * c.width);
    launch_gather_plain(ctx, c.data.get(), d_idx, n_out, c.width, d_data.back().get());
    d_valid.emplace_back();
    if (c.has_nulls) {
      d_valid.back().alloc(ctx, (size_t)std::max<int64_t>(1, n_out));
      launch_gather_plain(ctx, c.valid.get(), d_idx, n_out, 1, d_valid.back().get());
    }
  }
  for (size_t i = 0; i < col_idx.size(); i++) {
    const DevColumn& c = t.cols[col_idx[i]];
    hs_batch::Col bc;
    bc.name = c.name;
    bc.type = c.type;
    bc.has_valid = c.has_nulls || padded;
    const bool is_str = c.type == HS_TYPE_STRING;
    const size_t data_bytes = is_str ? (size_t)str_bytes[i] : (size_t)n_out * c.width;
    bc.total_bytes = is_str ? str_bytes[i] : 0;
    if (b->on_device) {  // the next GPU operator consumes the columns where they are
      bc.data = std::move(d_data[i]);
      if (is_str) bc.offsets = std::move(d_offsets[i]);
      if (bc.has_valid) bc.valid = std::move(d_valid[i]);
    } else {
      // result columns go straight to their pinned buffers on the copy engine (the ring of copy_d2h would stage results of
      // up to 16 MB through a host memcpy)
      bc.data.alloc(ctx, std::max<size_t>(1, data_bytes), true);
      if (data_bytes) copy_d2h_engine(ctx, bc.data.get(), d_data[i].get(), data_bytes);
      if (is_str) {
        bc.offsets.alloc(ctx, (size_t)n_out + 1, true);
        copy_d2h_engine(ctx, bc.offsets.get(), d_offsets[i].get(), 8 * ((size_t)n_out + 1));
      }
      if (bc.has_valid) {
        bc.valid.alloc(ctx, (size_t)std::max<int64_t>(1, n_out), true);
        if (n_out) copy_d2h_engine(ctx, bc.valid.get(), d_valid[i].get(), (size_t)n_out);
      }
    }
    b->cols.push_back(std::move(bc));
  }
  sync_stream(ctx);
  b->nrows = n_out;
}

}  // extern "C"

// ---- predicates: resolved on the host (predicates.h), uploaded here -------------------------------------------------

// Device memory that uploaded descriptors point into: string bound bytes and set-form range arrays, with the host
// arrays their copies read from (a large copy reads its source until the stream is synchronised).  Kept until the
// kernels that read them have run.
struct PredUploads {
  std::vector<Buf<uint8_t>> bytes;
  std::vector<Buf<PredRange>> sets;
  std::vector<Buf<uint16_t>> items;
  std::vector<Buf<int32_t>> fails;
  std::vector<Buf<PatSeg>> segs;
  std::vector<std::vector<uint8_t>> staged_bytes;
  std::vector<std::vector<PredRange>> staged_sets;
};

// The PredRanges of a set on a column of type `type`: the one place string bounds go to the device (one copy of their
// bytes, referenced by the ranges).  Returns them; as_array: uploads them instead, to up->sets.back(), for the set form
// and the window search.
static std::vector<PredRange> upload_set(hs_ctx* ctx, int type, const RangeSet& s, PredUploads* up, bool as_array) {
  std::vector<PredRange> h(std::max<size_t>(1, s.size()));
  uint8_t* bytes = nullptr;
  if (type == HS_TYPE_STRING) {
    std::vector<uint8_t> hb;
    for (const SetRange& r : s) hb.insert(hb.end(), r.lo_b.begin(), r.lo_b.end()), hb.insert(hb.end(), r.hi_b.begin(), r.hi_b.end());
    up->bytes.emplace_back(ctx, hb.size() + 16);
    bytes = up->bytes.back().get();
    if (!hb.empty()) copy_h2d(ctx, bytes, hb.data(), hb.size());
    up->staged_bytes.push_back(std::move(hb));
  }
  uint64_t off = 0;
  for (size_t i = 0; i < s.size(); i++) {
    const SetRange& r = s[i];
    PredRange& d = h[i];
    d = PredRange{};
    d.type = type;
    d.has_lo = r.has_lo, d.has_hi = r.has_hi, d.lo_strict = r.lo_strict, d.hi_strict = r.hi_strict;
    if (type == HS_TYPE_STRING) {
      d.lo = string_ref(bytes + off, (uint32_t)r.lo_b.size());
      off += r.lo_b.size();
      d.hi = string_ref(bytes + off, (uint32_t)r.hi_b.size());
      off += r.hi_b.size();
    } else {
      d.lo = r.lo, d.hi = r.hi;
    }
  }
  if (!as_array) return h;
  up->sets.emplace_back(ctx, h.size());
  copy_h2d(ctx, up->sets.back().get(), h.data(), sizeof(PredRange) * h.size());
  up->staged_sets.push_back(std::move(h));
  return {};
}

static PredColumn pred_column(const DevColumn& c) { return PredColumn{c.type, c.schema, c.name}; }

// Every term's resolution (predicates.h: resolve_any), computed once per side of a call: the key's windows and the
// residual share it.  A term resolves against its own column, which is the same column before and after decoding.
struct TermResolutions {
  const hs_predicate_any* anys = nullptr;
  std::vector<std::unique_ptr<ResolvedTerm>> r;
  TermResolutions() = default;
  TermResolutions(const hs_predicate_any* a, int n) : anys(a), r(n) {}
  const ResolvedTerm& operator()(int i, const DevColumn& c) {
    if (!r[i]) r[i].reset(new ResolvedTerm(resolve_any(anys[i], pred_column(c))));
    return *r[i];
  }
};

// The compiled pattern of term a on the string column c, uploaded for k_pattern_mask.  cp lives in the term's resolution,
// which outlasts the copies that read it.
static PatternDesc upload_pattern(hs_ctx* ctx, const DevColumn& c, const hs_predicate_any& a, const CompiledPattern& cp, PredUploads* up) {
  up->items.emplace_back(ctx, std::max<size_t>(1, cp.items.size()));
  up->fails.emplace_back(ctx, std::max<size_t>(1, cp.fail.size()));
  up->segs.emplace_back(ctx, cp.segs.size());
  if (!cp.items.empty()) {
    copy_h2d(ctx, up->items.back().get(), cp.items.data(), 2 * cp.items.size());
    copy_h2d(ctx, up->fails.back().get(), cp.fail.data(), 4 * cp.fail.size());
  }
  copy_h2d(ctx, up->segs.back().get(), cp.segs.data(), sizeof(PatSeg) * cp.segs.size());
  PatternDesc d{};
  d.refs = (const uint64_t*)c.data.get(), d.valid = c.has_nulls ? c.valid.get() : nullptr;
  d.items = up->items.back().get(), d.fail = up->fails.back().get(), d.segs = up->segs.back().get();
  d.nseg = (int32_t)cp.segs.size(), d.whole = cp.whole, d.negate = (a.flags & HS_TERM_NOT) != 0;
  d.null_true = term_null_selects(a.flags);
  return d;
}

// the index of column nm in cols, appended when it is not there yet
static int column_index(std::vector<std::string>* cols, const std::string& nm) {
  auto it = std::find(cols->begin(), cols->end(), nm);
  if (it != cols->end()) return (int)(it - cols->begin());
  cols->push_back(nm);
  return (int)cols->size() - 1;
}

// A filter bound to the columns a call decodes: the column of every predicate and term, the two columns of every
// comparison, the column of every COLUMN node of each expression comparison, and the terms' resolutions
struct BoundFilter {
  Filter f;
  std::vector<int> pred_col, any_col;
  std::vector<std::pair<int, int>> cmp_col;
  TermResolutions terms;
  std::vector<std::vector<int>> expr_col;  // per expression comparison: its COLUMN nodes' columns, the left side's first
};

// f bound to the columns cols, which gains those not in it yet: the predicates' columns, the terms', each comparison's
// left and right column, then each expression comparison's columns (after the others, so that a call without
// expressions decodes what it always has)
static BoundFilter bind_filter(const Filter& f, std::vector<std::string>* cols) {
  BoundFilter b{f, {}, {}, {}, TermResolutions(f.anys, f.n_anys)};
  for (int i = 0; i < f.n_preds; i++) b.pred_col.push_back(column_index(cols, f.preds[i].column));
  for (int i = 0; i < f.n_anys; i++) b.any_col.push_back(column_index(cols, f.anys[i].column));
  for (int i = 0; i < f.n_cmps; i++)
    b.cmp_col.push_back({column_index(cols, f.cmps[i].left), column_index(cols, f.cmps[i].right)});
  for (int i = 0; i < f.n_exprs; i++) {
    const hs_expr_compare& e = f.exprs[i];
    std::vector<int> ec;
    for (int s = 0; s < 2; s++)
      for (int k = 0; k < (s ? e.n_right : e.n_left); k++) {
        const hs_expr_node& x = (s ? e.right : e.left)[k];
        if (x.kind == HS_EXPR_COLUMN) ec.push_back(column_index(cols, x.column));
      }
    b.expr_col.push_back(std::move(ec));
  }
  return b;
}

// A host array copied to a new device buffer of up->bytes; the host copy is kept in up->staged_bytes until the copy has run
template <typename T>
static const T* upload_array(hs_ctx* ctx, const std::vector<T>& h, PredUploads* up) {
  const size_t nb = sizeof(T) * h.size();
  up->staged_bytes.emplace_back((const uint8_t*)h.data(), (const uint8_t*)h.data() + nb);
  up->bytes.emplace_back(ctx, std::max<size_t>(16, nb));
  if (nb) copy_h2d(ctx, up->bytes.back().get(), up->staged_bytes.back().data(), nb);
  return (const T*)up->bytes.back().get();
}

// The expression comparisons of filter b on the columns of t, resolved (predicates.h: resolve_expr) into one program per
// comparison and uploaded in one set: the descriptors, every instruction, every column they read and the bytes of their
// string literals.  *funcs: some program uses a function or a string, date or timestamp value, so the set runs in
// k_func_mask.
static ExprSet upload_exprs(hs_ctx* ctx, const Table& t, const BoundFilter& b, PredUploads* up, bool* funcs) {
  std::vector<ExprDesc> descs;
  std::vector<ExprInst> insts;
  std::vector<ExprColumn> ecols;
  std::vector<uint8_t> pool;
  *funcs = false;
  for (size_t i = 0; i < b.expr_col.size(); i++) {
    std::vector<PredColumn> pcs;
    for (int c : b.expr_col[i]) pcs.push_back(pred_column(t.cols[c]));
    const ExprProgram pg = resolve_expr(b.f.exprs[i], pcs);
    *funcs = *funcs || pg.funcs;
    const int32_t base = (int32_t)ecols.size(), pool_base = (int32_t)pool.size();
    pool.insert(pool.end(), pg.pool.begin(), pg.pool.end());
    for (int c : b.expr_col[i]) {
      const DevColumn& dc = t.cols[c];
      ecols.push_back(ExprColumn{dc.data.get(), dc.has_nulls ? dc.valid.get() : nullptr, dc.type});
    }
    ExprDesc d{(int32_t)insts.size(), 0, pg.domain, pg.op, pg.negate};
    for (ExprInst in : pg.insts) {
      if (in.op == kXLoad) in.arg += base;
      if (in.op == kXStringConst) in.arg += pool_base;
      insts.push_back(in);
    }
    d.end = (int32_t)insts.size();
    descs.push_back(d);
  }
  // every kXStringConst becomes a kXConst, also when every string literal is empty: upload_array allocates at least
  // 16 bytes, so the pool has an address
  relocate_strings(&insts, upload_array(ctx, pool, up));
  ExprSet es;
  es.descs = upload_array(ctx, descs, up);
  es.insts = upload_array(ctx, insts, up);
  es.cols = upload_array(ctx, ecols, up);
  es.n = (int)descs.size();
  return es;
}

// Appends to rf the descriptors of filter b on the columns of t, skipping those on column skip_col that its windows
// already decide: a predicate in scalar form and a term in set form.  A pattern term that is not a prefix goes to
// rf->pats (on skip_col too: the windows only bound its values), every comparison to rf->cmps, and the expression
// comparisons to rf->exprs, or to rf->funcs when they use functions.
static void add_filter(hs_ctx* ctx, const Table& t, BoundFilter& b, int skip_col, RowFilter* rf, PredUploads* up) {
  PredSet* ps = &rf->preds;
  for (size_t i = 0; i < b.pred_col.size(); i++) {
    if (b.pred_col[i] == skip_col) continue;
    const DevColumn& c = t.cols[b.pred_col[i]];
    const RangeSet one{resolve_range(b.f.preds[i], pred_column(c))};
    ps->p[ps->n++] = PredDesc{c.data.get(), c.has_nulls ? c.valid.get() : nullptr, upload_set(ctx, c.type, one, up, false)[0]};
  }
  for (size_t i = 0; i < b.any_col.size(); i++) {
    const DevColumn& c = t.cols[b.any_col[i]];
    const ResolvedTerm& rt = b.terms((int)i, c);
    const RangeSet& s = rt.set;
    if (!rt.exact) {
      rf->pats.p[rf->pats.n++] = upload_pattern(ctx, c, b.f.anys[i], rt.pattern, up);
      continue;
    }
    if (b.any_col[i] == skip_col) continue;
    upload_set(ctx, c.type, s, up, true);
    PredDesc d{c.data.get(), c.has_nulls ? c.valid.get() : nullptr, PredRange{}};
    d.r.type = c.type;
    d.set = up->sets.back().get();
    d.n_set = (int64_t)s.size();
    d.null_true = term_null_selects(b.f.anys[i].flags);
    ps->p[ps->n++] = d;
  }
  for (size_t i = 0; i < b.cmp_col.size(); i++) {
    const DevColumn& l = t.cols[b.cmp_col[i].first];
    const DevColumn& r = t.cols[b.cmp_col[i].second];
    CompareDesc d = resolve_compare(b.f.cmps[i], pred_column(l), pred_column(r));
    d.col[0] = l.data.get(), d.col[1] = r.data.get();
    d.valid[0] = l.has_nulls ? l.valid.get() : nullptr, d.valid[1] = r.has_nulls ? r.valid.get() : nullptr;
    rf->cmps.p[rf->cmps.n++] = d;
  }
  if (!b.expr_col.empty()) {
    bool funcs;
    const ExprSet es = upload_exprs(ctx, t, b, up, &funcs);
    (funcs ? rf->funcs : rf->exprs) = es;
  }
}

// the bucket of every point of a key set, by the hash the build used (hash_rows over a column of the key's storage type
// and schema: key_column_of gives a decimal(p <= 9) the hashLong kind)
static std::vector<int> point_buckets(hs_ctx* ctx, const DevColumn& key, const RangeSet& pts, int num_buckets) {
  const int64_t n = (int64_t)pts.size();
  std::vector<int> out(n);
  if (n == 0) return out;
  DevColumn c;
  c.name = key.name;
  c.type = key.type;
  c.width = key.width;
  c.schema = key.schema;
  c.data.alloc(ctx, (size_t)n * c.width + 16);
  Buf<uint8_t> bytes;
  std::vector<uint8_t> raw((size_t)n * c.width);
  if (key.type == HS_TYPE_STRING) {  // references into one device copy of the points' bytes
    std::vector<uint8_t> hb;
    for (const SetRange& r : pts) hb.insert(hb.end(), r.lo_b.begin(), r.lo_b.end());
    bytes.alloc(ctx, hb.size() + 16);
    if (!hb.empty()) copy_h2d(ctx, bytes.get(), hb.data(), hb.size());
    uint64_t off = 0;
    for (int64_t i = 0; i < n; i++) {
      const uint64_t ref = string_ref(bytes.get() + off, (uint32_t)pts[i].lo_b.size());
      memcpy(raw.data() + 8 * i, &ref, 8);
      off += pts[i].lo_b.size();
    }
  } else {
    for (int64_t i = 0; i < n; i++) {
      if (key.width == 4) {
        const uint32_t v = (uint32_t)pts[i].lo ^ 0x80000000u;
        memcpy(raw.data() + 4 * i, &v, 4);
      } else {
        const uint64_t v = pts[i].lo ^ 0x8000000000000000ull;
        memcpy(raw.data() + 8 * i, &v, 8);
      }
    }
  }
  copy_h2d(ctx, c.data.get(), raw.data(), raw.size());
  const KeyColumn kc = key_column_of(c);
  Buf<unsigned long long> ghist(ctx, num_buckets);
  fill_bytes(ctx, ghist.get(), 0, 8 * num_buckets);
  HashedRows hashed;
  hash_rows(ctx, &kc, 1, n, num_buckets, 0, false, ghist.get(), nullptr, &hashed);
  std::vector<uint16_t> hb(n);
  copy_d2h(ctx, hb.data(), hashed.bin_ids.get(), 2 * n);
  sync_stream(ctx);
  for (int64_t i = 0; i < n; i++) out[i] = hb[i];
  return out;
}

// The one filter scan: the sorted path binary-searches the key column's windows and decodes the other columns only inside
// them, then evaluates the predicates on other columns over the window rows; the unsorted path (source files, Hybrid
// Scan's appended files, the lineage NOT-IN) evaluates every predicate over all rows.
// legacy (hs_filter_scan): predicates may have no bound (the row's key must then not be null, as that call always did),
// literal types follow the column, and floating-point keys are refused (the call's bounds are int64).
// The filter's terms: on the key column they turn the key's one window per file into one window per range of the key's
// set; elsewhere they are set-form residual predicates.  Its comparisons between two columns are always residual (they
// make no window, so a key that appears only in them is read whole).  file_buckets (optional): see hs_filter_scan_any.
static int filter_scan_core(hs_ctx* ctx, const hs_scan_spec* spec, const Filter& filter, bool legacy, const int32_t* file_buckets,
                            int num_buckets, hs_batch** out, hs_stats* stats, char* err, size_t errlen) {
  *out = nullptr;
  hs_stats st;
  memset(&st, 0, sizeof st);
  std::unique_ptr<hs_batch> res(new hs_batch());
  res->ctx = ctx;
  res->on_device = spec->output == HS_OUT_DEVICE;
  int rc = guarded(ctx, err, errlen, [&] {
    StageTimer total(ctx);
    total.start();
    const bool try_sorted = spec->sorted_on_key && spec->n_deleted_file_ids == 0;
    if (try_sorted && !spec->key_column) fail(HS_EINVAL, "key_column is required");
    // columns to decode: the key first (sorted path), then the projection, the predicate columns, and lineage when
    // deletes must be filtered
    std::vector<std::string> cols;
    if (try_sorted) column_index(&cols, spec->key_column);
    std::vector<int> proj_idx;
    for (int i = 0; i < spec->n_projected; i++) proj_idx.push_back(column_index(&cols, spec->projected_columns[i]));
    BoundFilter bf = bind_filter(filter, &cols);
    const int lineage_col = spec->n_deleted_file_ids > 0 ? column_index(&cols, "_data_file_id") : -1;
    PredUploads uploads;
    // The key's set (when a term is on the key, or for pruning): the predicates on the key and every term on it,
    // intersected.
    auto on_key_name = [&](const char* column) { return spec->key_column && strcmp(column, spec->key_column) == 0; };
    // a term that selects null keys (IS NULL, NOT (k <=> v)) finds them in the null key's bucket: no pruning then
    bool key_terms = false, key_nulls = false;
    for (int i = 0; i < filter.n_anys; i++) {
      key_terms = key_terms || on_key_name(filter.anys[i].column);
      key_nulls = key_nulls || (on_key_name(filter.anys[i].column) && term_null_selects(filter.anys[i].flags));
    }
    auto key_set_of = [&](const DevColumn& kc) {
      const bool str = kc.type == HS_TYPE_STRING;
      RangeSet s{SetRange{}};  // every value
      for (int i = 0; i < filter.n_preds; i++)
        if (on_key_name(filter.preds[i].column)) s = intersect_sets(str, s, RangeSet{resolve_range(filter.preds[i], pred_column(kc))});
      for (int i = 0; i < filter.n_anys; i++)
        if (on_key_name(filter.anys[i].column)) s = intersect_sets(str, s, bf.terms(i, kc).set);
      return s;
    };
    // Bucket pruning: a key whose windows are points lives in the files of the points' buckets only
    const hs_source_file* files = spec->files;
    int n_files = spec->n_files;
    std::vector<hs_source_file> kept;
    std::vector<int> kept_bucket, point_bucket;
    RangeSet key_set;
    bool have_key_set = false;
    if (file_buckets && num_buckets > 0 && spec->key_column && n_files > 0) {
      for (int f = 0; f < n_files; f++)
        if (file_buckets[f] < 0 || file_buckets[f] >= num_buckets) fail(HS_EINVAL, "bucket id %d out of range", file_buckets[f]);
      const DevColumn kc = source_column_type(ctx, files[0], spec->key_column);
      const bool hashable = kc.type == HS_TYPE_INT32 || kc.type == HS_TYPE_INT64 || kc.type == HS_TYPE_STRING;
      bool keyed = key_terms;
      for (int i = 0; i < filter.n_preds; i++) keyed = keyed || on_key_name(filter.preds[i].column);
      if (hashable && keyed && !key_nulls) {
        key_set = key_set_of(kc);
        have_key_set = true;
        if (set_is_points(kc.type == HS_TYPE_STRING, key_set)) {
          point_bucket = point_buckets(ctx, kc, key_set, num_buckets);
          std::vector<char> hit(num_buckets, 0);
          for (int b : point_bucket) hit[b] = 1;
          for (int f = 0; f < n_files; f++)
            if (hit[file_buckets[f]]) kept.push_back(files[f]), kept_bucket.push_back(file_buckets[f]);
          // no file can hold a row: the first one is opened to give the result its columns, and searched for nothing
          if (kept.empty()) kept.push_back(files[0]), kept_bucket.push_back(-1);
          files = kept.data();
          n_files = (int)kept.size();
        }
      }
    }
    const bool pruned = !kept.empty();
    SourceSet src;
    open_sources(ctx, files, n_files, &src, &st);
    Table t;
    // phase 1 (sorted path): only the key column; the other columns are decoded after the binary search, restricted to
    // the pages that hold rows inside the windows
    if (try_sorted) decode_sources(ctx, src, {cols[0]}, nullptr, &t, &st);
    else decode_sources(ctx, src, cols, nullptr, &t, &st);
    if (legacy && try_sorted && t.cols[0].type != HS_TYPE_STRING && t.cols[0].type != HS_TYPE_INT64 && t.cols[0].type != HS_TYPE_INT32)
      fail(HS_EUNSUPPORTED, "filter scan: key column must be int32 / int64 / string");
    const int64_t n = t.nrows;
    StageTimer t_scan(ctx);
    t_scan.start();
    Buf<uint32_t> idx;
    int64_t n_out = 0;
    bool sorted = try_sorted && !t.cols[0].has_nulls;
    if (try_sorted && !sorted) {  // nulls in the key: fall back to the predicate scan over all columns
      Table full;
      decode_sources(ctx, src, cols, nullptr, &full, &st);
      t = std::move(full);
    }
    if (sorted) {
      // K7: two binary searches per (file, range of the key)
      const int ktype = t.cols[0].type;
      if (ktype < HS_TYPE_INT32 || ktype > HS_TYPE_STRING || ktype == HS_TYPE_BOOL)
        fail(HS_EUNSUPPORTED, "filter scan: the sorted key column '%s' must be int32 / int64 / float / double / string", cols[0].c_str());
      int on_key = 0;  // the predicates and terms the windows decide (a pattern that is not a prefix stays residual)
      for (int i = 0; i < filter.n_preds; i++) on_key += bf.pred_col[i] == 0;
      for (int i = 0; i < filter.n_anys; i++) on_key += bf.any_col[i] == 0 && bf.terms(i, t.cols[0]).exact;
      const int nseg = n_files;
      std::vector<uint64_t> seg(nseg + 1);
      for (int f = 0; f <= nseg; f++) seg[f] = (uint64_t)t.file_row_begin[f];
      Buf<uint64_t> d_seg(ctx, nseg + 1);
      copy_h2d(ctx, d_seg.get(), seg.data(), 8 * (nseg + 1));
      // The key's ranges: its set when a term is on the key or the files are pruned; otherwise the intersection of the
      // predicates on the key, one range kept even when it is empty, so that every file still decodes the page its
      // empty window falls on (below)
      if (!(key_terms || pruned)) {
        SetRange r;
        for (int i = 0; i < filter.n_preds; i++)
          if (bf.pred_col[i] == 0) r = intersect_range(ktype == HS_TYPE_STRING, r, resolve_range(filter.preds[i], pred_column(t.cols[0])));
        key_set = RangeSet{r};
      } else if (!have_key_set) {
        key_set = key_set_of(t.cols[0]);
      }
      upload_set(ctx, ktype, key_set, &uploads, true);
      const PredRange* d_ranges = uploads.sets.back().get();
      std::vector<uint2> work;
      work.reserve((size_t)nseg * (pruned ? 1 : key_set.size()));
      for (int f = 0; f < nseg; f++)
        for (size_t r = 0; r < key_set.size(); r++)
          if (!pruned || point_bucket[r] == kept_bucket[f]) work.push_back(make_uint2((unsigned)f, (unsigned)r));
      const int64_t nwork = (int64_t)work.size();
      Buf<uint2> d_work(ctx, std::max<int64_t>(1, nwork));
      Buf<int64_t> d_bounds(ctx, 2 * std::max<int64_t>(1, nwork));
      if (nwork) copy_h2d(ctx, d_work.get(), work.data(), sizeof(uint2) * nwork);
      launch_range_bounds(ctx, t.cols[0].data.get(), ktype, d_ranges, d_seg.get(), d_work.get(), nwork, d_bounds.get());
      std::vector<int64_t> bounds(2 * std::max<int64_t>(1, nwork));
      if (nwork) copy_d2h(ctx, bounds.data(), d_bounds.get(), 16 * nwork);
      sync_stream(ctx);
      // The windows, file by file and ascending inside a file (the ranges are), touching ones merged.  The pages to decode
      // keep the empty windows too: an empty window still decodes the page it falls inside, as the one-range scan always
      // has (so a nullable column keeps its validity array when no row qualifies); the candidate rows need only the
      // non-empty ones.
      FileWindows fw;
      fw.offsets.assign(nseg + 1, 0);
      std::vector<int64_t> win;         // non-empty windows: [lo, hi) global rows
      std::vector<uint64_t> oo(1, 0);   // output offset of every non-empty window
      int prev_f = -1, prev_win_f = -1;
      for (int64_t w = 0; w < nwork; w++) {
        const int f = (int)work[w].x;
        const int64_t first = bounds[2 * w], last = bounds[2 * w + 1];
        if (prev_f == f && fw.windows.back().second >= first) {
          fw.windows.back().second = std::max(fw.windows.back().second, last);
        } else {
          fw.windows.push_back({first, last});
          fw.offsets[f + 1]++;
        }
        prev_f = f;
        if (last <= first) continue;
        if (prev_win_f == f && win.back() == (int64_t)seg[f] + first) {
          win.back() = (int64_t)seg[f] + last;
        } else {
          win.push_back((int64_t)seg[f] + first);
          win.push_back((int64_t)seg[f] + last);
          oo.push_back(oo.back());
        }
        prev_win_f = f;
        oo.back() += (uint64_t)(last - first);
      }
      for (int f = 0; f < nseg; f++) fw.offsets[f + 1] += fw.offsets[f];
      const int64_t nwin = (int64_t)win.size() / 2;
      if (cols.size() > 1) {  // phase 2: decode the other columns, only the pages inside the windows
        std::vector<std::string> rest(cols.begin() + 1, cols.end());
        Table others;
        decode_sources(ctx, src, rest, &fw, &others, &st);
        for (auto& c : others.cols) t.cols.push_back(std::move(c));
      }
      const int64_t n_cand = (int64_t)oo.back();
      Buf<int64_t> d_win(ctx, std::max<size_t>(2, win.size()));
      Buf<uint64_t> d_oo(ctx, oo.size());
      if (nwin) copy_h2d(ctx, d_win.get(), win.data(), 8 * win.size());
      copy_h2d(ctx, d_oo.get(), oo.data(), 8 * oo.size());
      idx.alloc(ctx, std::max<int64_t>(1, n_cand));
      if (nseg) launch_windows_to_indices(ctx, d_win.get(), d_oo.get(), nwin, n_cand, idx.get());
      n_out = n_cand;
      if (on_key < filter.n_preds + filter.n_anys || filter.n_cmps > 0 || filter.n_exprs > 0) {
        // residual: the predicates on other columns, the comparisons and the expression comparisons, over the window
        // rows, compacted through the candidate list
        RowFilter residual;
        add_filter(ctx, t, bf, 0, &residual, &uploads);
        Buf<uint32_t> kept_rows;
        n_out = select_rows(ctx, residual, idx.get(), n_cand, nullptr, nullptr, 0, &kept_rows);
        idx = std::move(kept_rows);
      }
    } else {
      // full predicate scan (source files, appended source files under Hybrid Scan, or lineage NOT-IN filter)
      RowFilter rf;
      add_filter(ctx, t, bf, -1, &rf, &uploads);
      const int64_t* file_ids = lineage_col >= 0 ? (const int64_t*)t.cols[lineage_col].data.get() : nullptr;
      n_out = select_rows(ctx, rf, nullptr, n, file_ids, spec->deleted_file_ids, spec->n_deleted_file_ids, &idx);
    }
    sync_stream(ctx);
    t_scan.stop();
    StageTimer t_gather(ctx);
    t_gather.start();
    batch_from_gather(ctx, t, proj_idx, idx.get(), n_out, res.get());
    t_gather.stop();
    total.stop();
    sync_stream(ctx);
    st.ms_sort += t_scan.ms();
    st.ms_gather += t_gather.ms();
    st.rows_out = n_out;
    st.ms_total = total.ms();
    st.gpu_launches = ctx->launches;
  });
  if (stats) *stats = st;
  if (rc == HS_OK) *out = res.release();
  return rc;
}

extern "C" {

int hs_filter_scan(hs_ctx* ctx, const hs_scan_spec* spec, hs_batch** out, hs_stats* stats, char* err, size_t errlen) {
  if (!ctx || !spec || !out) return HS_EINVAL;
  *out = nullptr;
  if (!spec->key_column) return refuse(HS_EINVAL, stats, err, errlen, "key_column is required");
  // one predicate on the key, its literal type following the column
  hs_predicate p;
  memset(&p, 0, sizeof p);
  p.column = spec->key_column;
  p.literal_type = -1;
  p.has_lo = spec->has_lo, p.has_hi = spec->has_hi;
  p.lo_i = spec->lo, p.hi_i = spec->hi;
  p.lo_bytes = spec->lo_bytes, p.hi_bytes = spec->hi_bytes;
  p.lo_len = spec->lo_len, p.hi_len = spec->hi_len;
  const Filter f{&p, 1};
  return filter_scan_core(ctx, spec, f, true, nullptr, 0, out, stats, err, errlen);
}

int hs_filter_scan_where(hs_ctx* ctx, const hs_scan_spec* spec, const hs_predicate* preds, int32_t n_preds, hs_batch** out,
                         hs_stats* stats, char* err, size_t errlen) {
  return hs_filter_scan_any(ctx, spec, preds, n_preds, nullptr, 0, nullptr, 0, out, stats, err, errlen);
}

int hs_filter_scan_any(hs_ctx* ctx, const hs_scan_spec* spec, const hs_predicate* preds, int32_t n_preds,
                       const hs_predicate_any* anys, int32_t n_anys, const int32_t* file_buckets, int32_t num_buckets,
                       hs_batch** out, hs_stats* stats, char* err, size_t errlen) {
  return hs_filter_scan_cmp(ctx, spec, preds, n_preds, anys, n_anys, nullptr, 0, file_buckets, num_buckets, out, stats, err, errlen);
}

int hs_filter_scan_cmp(hs_ctx* ctx, const hs_scan_spec* spec, const hs_predicate* preds, int32_t n_preds,
                       const hs_predicate_any* anys, int32_t n_anys, const hs_column_compare* cmps, int32_t n_cmps,
                       const int32_t* file_buckets, int32_t num_buckets, hs_batch** out, hs_stats* stats, char* err,
                       size_t errlen) {
  return hs_filter_scan_expr(ctx, spec, preds, n_preds, anys, n_anys, cmps, n_cmps, nullptr, 0, file_buckets, num_buckets, out, stats,
                             err, errlen);
}

int hs_filter_scan_expr(hs_ctx* ctx, const hs_scan_spec* spec, const hs_predicate* preds, int32_t n_preds,
                        const hs_predicate_any* anys, int32_t n_anys, const hs_column_compare* cmps, int32_t n_cmps,
                        const hs_expr_compare* exprs, int32_t n_exprs, const int32_t* file_buckets, int32_t num_buckets,
                        hs_batch** out, hs_stats* stats, char* err, size_t errlen) {
  if (!ctx || !spec || !out || n_preds < 0 || (n_preds > 0 && !preds) || num_buckets < 0 || (num_buckets > 0 && !file_buckets))
    return HS_EINVAL;
  *out = nullptr;
  const Filter f{preds, n_preds, anys, n_anys, cmps, n_cmps, exprs, n_exprs};
  const int rc = check_filters(&f, 1, spec->has_lo || spec->has_hi, stats, err, errlen);
  if (rc != HS_OK) return rc;
  if (num_buckets > kMaxBuckets) return refuse(HS_EUNSUPPORTED, stats, err, errlen, "numBuckets must be in 1..%d", kMaxBuckets);
  return filter_scan_core(ctx, spec, f, false, num_buckets > 0 ? file_buckets : nullptr, num_buckets, out, stats, err, errlen);
}

}  // extern "C"

// One side of a bucket join: its rows bucket-major and ascending on the key columns.  perm maps a sorted position to a
// row of t (nullptr: the identity, every bucket is one index file); after the side selection it lists only the rows
// that can take part in the join, still in sorted order, and seg holds the buckets' new boundaries.
struct JoinSide {
  SourceSet src;  // string values are references into the file images: kept alive until the result batch exists
  Table t;
  IndexedRows rows;
  std::vector<uint64_t> seg;  // nb+1 sorted positions
  const uint32_t* perm = nullptr;
  Buf<uint32_t> kept;
  int64_t n = 0;  // rows in sorted order
  std::vector<int> proj;  // the projected columns of t
  BoundFilter filter;
  RowFilter sel;  // the side selection: IS NOT NULL on the nullable key columns (not on a preserved side), then the filter
  // FullOuter: the selected positions with no null key, the ones the other side's probe searches (a binary search over
  // positions with a null key would not be over sorted data: a null sorts first only at its own column).  The same as
  // the above when no key column has nulls.
  const uint32_t* nn_perm = nullptr;
  Buf<uint32_t> nn_kept;
  int64_t nn_n = 0;
  std::vector<uint64_t> nn_seg;
};

// Orders the decoded rows of one join side bucket-major and key-sorted.  When every bucket holds exactly one file the
// files are already sorted (they are index files) and only need to be visited in bucket order; otherwise the rows go
// through K2-K4 again on all n_keys key columns, which is what Spark's SortExec does for multi-file buckets.
// cols: the n_keys key columns first, then the projected and the predicate columns.
static void prepare_join_side(hs_ctx* ctx, JoinSide* side, const hs_source_file* files, int n_files, const int32_t* buckets, int nb,
                              const std::vector<std::string>& cols, int n_keys, bool nulls_refused, hs_stats* st) {
  // reorder files by bucket so the decoded table is bucket-major
  std::vector<int> order(n_files);
  for (int i = 0; i < n_files; i++) order[i] = i;
  std::stable_sort(order.begin(), order.end(), [&](int a, int b) { return buckets[a] < buckets[b]; });
  std::vector<hs_source_file> sorted_files(n_files);
  std::vector<int> per_bucket(nb, 0);
  for (int i = 0; i < n_files; i++) {
    sorted_files[i] = files[order[i]];
    if (buckets[order[i]] < 0 || buckets[order[i]] >= nb) fail(HS_EINVAL, "bucket id %d out of range", buckets[order[i]]);
    per_bucket[buckets[order[i]]]++;
  }
  Table* t = &side->t;
  open_sources(ctx, sorted_files.data(), n_files, &side->src, st);
  decode_sources(ctx, side->src, cols, nullptr, t, st);
  if (!t->has_strings) side->src.release_images();
  for (int k = 0; k < n_keys; k++) {
    const int ty = t->cols[k].type;
    if (ty != HS_TYPE_STRING && ty != HS_TYPE_INT64 && ty != HS_TYPE_INT32)
      fail(HS_EUNSUPPORTED, "bucket join: key column must be int32, int64 or string");
    if (nulls_refused && t->cols[k].has_nulls) fail(HS_EUNSUPPORTED, "bucket join: null join keys are not handled yet");
  }
  const bool single = std::all_of(per_bucket.begin(), per_bucket.end(), [](int c) { return c <= 1; });
  if (single) {
    side->seg.assign(nb + 1, 0);
    int fi = 0;
    for (int b = 0; b < nb; b++) {
      side->seg[b] = (uint64_t)t->file_row_begin[fi];
      if (per_bucket[b]) fi++;
    }
    side->seg[nb] = (uint64_t)t->nrows;
  } else {
    IndexedRows* rows = &side->rows;
    index_rows(ctx, *t, n_keys, nb, rows, st);
    side->seg = rows->bucket_offsets;
    rows->sorted.keys_buf[rows->sorted.cur ^ 1].release();  // the sort's scratch keys
    t->cols.clear();
    t->cols = std::move(rows->part.cols);
    t->nrows = rows->part.nrows;
    side->perm = rows->sorted.perm();
  }
  side->n = t->nrows;
}

// Side selection: keeps the rows that pass side->sel.  It runs over the sorted positions as its candidate list, so the
// compacted rows stay in sorted order and a bucket's new boundaries are the scan's values at the old ones.  Launches
// nothing when side->sel is empty.
// d_out[b] = d_scan[seg[b]] for the nb + 1 bucket boundaries seg (< 2^32: the caller checked the side's size)
static void at_bucket_bounds(hs_ctx* ctx, const uint64_t* d_scan, const std::vector<uint64_t>& seg, int nb, Buf<uint64_t>* d_out) {
  std::vector<uint32_t> bounds(nb + 1);
  for (int b = 0; b <= nb; b++) bounds[b] = (uint32_t)seg[b];
  Buf<uint32_t> d_bounds(ctx, nb + 1);
  d_out->alloc(ctx, nb + 1);
  copy_h2d(ctx, d_bounds.get(), bounds.data(), 4 * (nb + 1));
  launch_gather_plain(ctx, d_scan, d_bounds.get(), nb + 1, 8, d_out->get());
}

// Keeps the sorted positions (*perm, *n, *seg) that pass sel: compacted into *kept, which *perm then points into
static void select_positions(hs_ctx* ctx, const RowFilter& sel, int nb, Buf<uint32_t>* kept, const uint32_t** perm, int64_t* n,
                             std::vector<uint64_t>* seg) {
  Buf<uint64_t> offs;
  *n = select_rows(ctx, sel, *perm, *n, nullptr, nullptr, 0, kept, &offs);
  *perm = kept->get();
  Buf<uint64_t> d_seg;
  at_bucket_bounds(ctx, offs.get(), *seg, nb, &d_seg);
  copy_d2h(ctx, seg->data(), d_seg.get(), 8 * (nb + 1));
  sync_stream(ctx);
}

static void select_join_side(hs_ctx* ctx, JoinSide* side, int nb) {
  if (side->sel.empty()) return;
  select_positions(ctx, side->sel, nb, &side->kept, &side->perm, &side->n, &side->seg);
}

// bucket_join_core's join_type for the inner join (include/hs_gpu.h numbers the semi and anti joins from 1, the outer
// joins from 3)
constexpr int kJoinInner = HS_JOIN_INNER;

static bool is_outer_join(int join_type) {
  return join_type == HS_JOIN_LEFT_OUTER || join_type == HS_JOIN_RIGHT_OUTER || join_type == HS_JOIN_FULL_OUTER;
}

// The one bucket join of the sides' filters (left, right).  legacy (hs_bucket_join): one key per side, no filters, null
// keys refused.  k_join_count (inner), k_join_exists (join_type HS_JOIN_LEFT_SEMI / HS_JOIN_LEFT_ANTI) or
// k_join_count_outer (HS_JOIN_*_OUTER) probes on the key columns where they lie: the decoded columns, or their gather
// through the side's permutation.
static int bucket_join_core(hs_ctx* ctx, const hs_join_spec* spec, const char* const* left_keys, const char* const* right_keys,
                            int n_keys, const Filter filters[2], bool legacy, int join_type, hs_batch** out, hs_stats* stats,
                            char* err, size_t errlen) {
  hs_stats st;
  memset(&st, 0, sizeof st);
  std::unique_ptr<hs_batch> res(new hs_batch());
  res->ctx = ctx;
  res->on_device = spec->output == HS_OUT_DEVICE;
  int rc = guarded(ctx, err, errlen, [&] {
    StageTimer total(ctx);
    total.start();
    const int nb = spec->num_buckets;
    if (nb < 1) fail(HS_EINVAL, "num_buckets must be positive");
    JoinSide side[2];
    JoinSide &L = side[0], &R = side[1];
    // columns to decode: the keys first, then the projection, then the filter's columns
    std::vector<std::string> cols[2];
    for (int s = 0; s < 2; s++) {
      const char* const* keys = s == 0 ? left_keys : right_keys;
      for (int k = 0; k < n_keys; k++) {
        if (!keys[k]) fail(HS_EINVAL, "bucket join: missing key column");
        if (std::find(cols[s].begin(), cols[s].end(), keys[k]) != cols[s].end())
          fail(HS_EINVAL, "bucket join: key column '%s' given twice", keys[k]);
        cols[s].push_back(keys[k]);
      }
      const char* const* proj = s == 0 ? spec->left_columns : spec->right_columns;
      const int n_proj = s == 0 ? spec->n_left_columns : spec->n_right_columns;
      for (int i = 0; i < n_proj; i++) side[s].proj.push_back(column_index(&cols[s], proj[i]));
      side[s].filter = bind_filter(filters[s], &cols[s]);
    }
    prepare_join_side(ctx, &L, spec->left_files, spec->n_left, spec->left_buckets, nb, cols[0], n_keys, legacy, &st);
    prepare_join_side(ctx, &R, spec->right_files, spec->n_right, spec->right_buckets, nb, cols[1], n_keys, legacy, &st);
    // hashInt and hashLong put equal values into different buckets: both sides must have been bucketed on the same types
    // (JoinIndexRule only pairs indexes whose indexed columns have the same data types)
    // the same holds for the decimals and timestamps riding on them: decimal(p <= 9) hashes as a long, an int32 as an int,
    // and a decimal(9,2) equals a decimal(9,3) only after rescaling (other int32 / int64 / string pairs bucket alike)
    auto spark_typed = [](const pq::SchemaColumn& s) { return is_decimal(s) || is_timestamp(s); };
    for (int k = 0; k < n_keys; k++)
      if (L.t.cols[k].type != R.t.cols[k].type ||
          ((spark_typed(L.t.cols[k].schema) || spark_typed(R.t.cols[k].schema)) &&
           pq::spark_type_name(L.t.cols[k].schema) != pq::spark_type_name(R.t.cols[k].schema))) {
        if (n_keys == 1) fail(HS_EUNSUPPORTED, "bucket join: key columns have different types");
        fail(HS_EUNSUPPORTED, "bucket join: key columns '%s' and '%s' have different types", left_keys[k], right_keys[k]);
      }
    if (R.n >= (1ll << 32) || L.n >= (1ll << 32)) fail(HS_EUNSUPPORTED, "join side larger than 2^32-1 rows");
    // side selection: IS NOT NULL on the nullable key columns, then the side's filter.  A preserved side -- the left side
    // of an anti join, the output sides of an outer join -- keeps the rows with a null key (they match nothing, so they
    // are output): its probe reads their validity instead.
    const bool anti = join_type == HS_JOIN_LEFT_ANTI, outer = is_outer_join(join_type), full = join_type == HS_JOIN_FULL_OUTER;
    const bool preserved[2] = {anti || join_type == HS_JOIN_LEFT_OUTER || full, join_type == HS_JOIN_RIGHT_OUTER || full};
    PredUploads uploads;
    RowFilter not_null[2];  // FullOuter: IS NOT NULL on the side's nullable key columns, for its searched positions
    for (int s = 0; s < 2; s++) {
      PredSet& ps = (preserved[s] ? not_null[s] : side[s].sel).preds;
      for (int k = 0; k < n_keys; k++) {
        const DevColumn& c = side[s].t.cols[k];
        if (c.has_nulls) {
          PredDesc d{};
          d.data = c.data.get(), d.valid = c.valid.get(), d.r.type = c.type;
          ps.p[ps.n++] = d;
        }
      }
      add_filter(ctx, side[s].t, side[s].filter, -1, &side[s].sel, &uploads);
    }
    StageTimer t_sel(ctx);
    t_sel.start();
    for (JoinSide& s : side) select_join_side(ctx, &s, nb);
    if (full) {  // the searched positions: the selected ones again, through IS NOT NULL alone
      for (int s = 0; s < 2; s++) {
        JoinSide& S = side[s];
        S.nn_perm = S.perm, S.nn_n = S.n, S.nn_seg = S.seg;
        if (!not_null[s].empty()) select_positions(ctx, not_null[s], nb, &S.nn_kept, &S.nn_perm, &S.nn_n, &S.nn_seg);
      }
    }
    t_sel.stop();
    // the key columns in (selected) sorted order
    std::vector<Buf<uint8_t>> key_bufs;
    auto sorted_column = [&](const uint32_t* perm, int64_t n, const uint8_t* data, int width) {
      if (!perm) return data;
      key_bufs.emplace_back(ctx, (size_t)std::max<int64_t>(1, n) * width);
      launch_gather_plain(ctx, data, perm, n, width, key_bufs.back().get());
      return (const uint8_t*)key_bufs.back().get();
    };
    auto key_cols_at = [&](const JoinSide& s, const uint32_t* perm, int64_t n) {
      JoinKeyCols kc{};
      kc.n = n_keys;
      for (int k = 0; k < n_keys; k++) {
        const DevColumn& c = s.t.cols[k];
        kc.type[k] = c.type;
        kc.col[k] = sorted_column(perm, n, c.data.get(), c.width);
      }
      return kc;
    };
    auto key_cols = [&](const JoinSide& s) { return key_cols_at(s, s.perm, s.n); };
    // the validity of a preserved side's nullable key columns, in its selected sorted order
    auto key_valid = [&](const JoinSide& s) {
      JoinKeyValid kv{};
      kv.n = n_keys;
      for (int k = 0; k < n_keys; k++) {
        const DevColumn& c = s.t.cols[k];
        if (c.has_nulls) kv.valid[k] = sorted_column(s.perm, s.n, c.valid.get(), 1);
      }
      return kv;
    };
    const int64_t nl = L.n;
    StageTimer t_join(ctx);
    t_join.start();
    Buf<uint64_t> d_lseg(ctx, nb + 1), d_rseg(ctx, nb + 1);
    copy_h2d(ctx, d_lseg.get(), L.seg.data(), 8 * (nb + 1));
    copy_h2d(ctx, d_rseg.get(), R.seg.data(), 8 * (nb + 1));
    const JoinKeyCols lk = key_cols(L), rk = key_cols(R);
    uint64_t total_out = 0;
    if (outer) {
      // the probing side p is the preserved one (the left side of FullOuter), q the side it searches: RightOuter is
      // LeftOuter with the roles swapped, the batch still the left columns, then the right ones
      const int p = join_type == HS_JOIN_RIGHT_OUTER ? 1 : 0, q = 1 - p;
      const JoinSide& P = side[p];
      const JoinKeyCols kc[2] = {lk, rk};
      const uint64_t* d_seg[2] = {d_lseg.get(), d_rseg.get()};
      // the searched positions: FullOuter's non-null ones where a side has them apart
      JoinKeyCols sk[2] = {lk, rk};
      const uint64_t* d_sseg[2] = {d_seg[0], d_seg[1]};
      const uint32_t* sperm[2] = {L.perm, R.perm};
      Buf<uint64_t> d_nn_seg[2];
      for (int s = 0; s < 2 && full; s++) {
        const JoinSide& S = side[s];
        sperm[s] = S.nn_perm;
        if (S.nn_perm == S.perm) continue;
        sk[s] = key_cols_at(S, S.nn_perm, S.nn_n);
        d_nn_seg[s].alloc(ctx, nb + 1);
        copy_h2d(ctx, d_nn_seg[s].get(), S.nn_seg.data(), 8 * (nb + 1));
        d_sseg[s] = d_nn_seg[s].get();
      }
      const int64_t np = P.n;
      Buf<uint32_t> counts(ctx, std::max<int64_t>(1, np)), first(ctx, std::max<int64_t>(1, np));
      Buf<uint64_t> offs(ctx, np + 1);
      launch_join_count_outer(ctx, kc[p], key_valid(P), d_seg[p], sk[q], d_sseg[q], nb, np, counts.get(), first.get());
      exclusive_scan_u32_u64(ctx, counts.get(), np, offs.get());
      copy_d2h(ctx, &total_out, offs.get() + np, 8);
      sync_stream(ctx);
      // FullOuter: the right positions that match nothing (k_join_exists in anti mode into the left side's searched
      // positions), compacted into right rows; ranks[i] = how many of them come before right position i
      Buf<uint32_t> urow;
      Buf<uint64_t> ranks;
      int64_t nu = 0;
      if (full) {
        Buf<uint32_t> keep(ctx, std::max<int64_t>(1, R.n));
        launch_join_exists(ctx, rk, key_valid(R), d_rseg.get(), sk[0], d_sseg[0], nb, R.n, false, keep.get());
        nu = compact_rows(ctx, keep.get(), R.n, R.perm, &urow, &ranks);
        total_out += (uint64_t)nu;
      }
      if (total_out >= (1ull << 32)) fail(HS_EUNSUPPORTED, "join output larger than 2^32-1 rows per call");
      Buf<uint32_t> lrow(ctx, std::max<uint64_t>(1, total_out)), rrow(ctx, std::max<uint64_t>(1, total_out));
      uint32_t* out_row[2] = {lrow.get(), rrow.get()};
      // FullOuter's placement: bucket b's left-outer rows move up by the unmatched right rows of the buckets before it
      // (ucum[b]); its unmatched right rows follow its left-outer rows (the scan of counts at the next bucket's start)
      Buf<uint64_t> ucum, lcum;
      if (full) {
        at_bucket_bounds(ctx, ranks.get(), R.seg, nb, &ucum);
        at_bucket_bounds(ctx, offs.get(), L.seg, nb, &lcum);
        launch_join_place_unmatched(ctx, urow.get(), nu, ucum.get(), lcum.get() + 1, nb, lrow.get(), rrow.get());
      }
      launch_join_emit_outer(ctx, counts.get(), first.get(), offs.get(), d_seg[p], full ? ucum.get() : nullptr, nb, np, P.perm,
                             sperm[q], out_row[p], out_row[q]);
      t_join.stop();
      batch_from_gather(ctx, L.t, L.proj, lrow.get(), (int64_t)total_out, res.get(), preserved[1]);
      batch_from_gather(ctx, R.t, R.proj, rrow.get(), (int64_t)total_out, res.get(), preserved[0]);
    } else if (join_type != kJoinInner) {
      // semi / anti: one keep mask over the left sorted positions, compacted through L.perm into left rows
      JoinKeyValid lv{};
      if (anti) lv = key_valid(L);
      Buf<uint32_t> keep(ctx, std::max<int64_t>(1, nl)), lrow;
      launch_join_exists(ctx, lk, lv, d_lseg.get(), rk, d_rseg.get(), nb, nl, !anti, keep.get());
      total_out = (uint64_t)compact_rows(ctx, keep.get(), nl, L.perm, &lrow);
      t_join.stop();
      batch_from_gather(ctx, L.t, L.proj, lrow.get(), (int64_t)total_out, res.get());
    } else {
      Buf<uint32_t> counts(ctx, std::max<int64_t>(1, nl)), first(ctx, std::max<int64_t>(1, nl));
      Buf<uint64_t> offs(ctx, nl + 1);
      launch_join_count(ctx, lk, d_lseg.get(), rk, d_rseg.get(), nb, nl, counts.get(), first.get());
      exclusive_scan_u32_u64(ctx, counts.get(), nl, offs.get());
      copy_d2h(ctx, &total_out, offs.get() + nl, 8);
      sync_stream(ctx);
      if (total_out >= (1ull << 32)) fail(HS_EUNSUPPORTED, "join output larger than 2^32-1 rows per call");
      Buf<uint32_t> lrow(ctx, std::max<uint64_t>(1, total_out)), rrow(ctx, std::max<uint64_t>(1, total_out));
      launch_join_emit(ctx, counts.get(), first.get(), offs.get(), nl, L.perm, R.perm, lrow.get(), rrow.get());
      t_join.stop();
      batch_from_gather(ctx, L.t, L.proj, lrow.get(), (int64_t)total_out, res.get());
      batch_from_gather(ctx, R.t, R.proj, rrow.get(), (int64_t)total_out, res.get());
    }
    total.stop();
    sync_stream(ctx);
    st.ms_sort += t_join.ms();
    if (!L.sel.empty() || !R.sel.empty() || (full && (!not_null[0].empty() || !not_null[1].empty()))) st.ms_exchange += t_sel.ms();
    st.rows_out = (int64_t)total_out;
    st.ms_total = total.ms();
    st.gpu_launches = ctx->launches;
  });
  if (stats) *stats = st;
  if (rc == HS_OK) *out = res.release();
  return rc;
}

extern "C" {

int hs_bucket_join(hs_ctx* ctx, const hs_join_spec* spec, hs_batch** out, hs_stats* stats, char* err, size_t errlen) {
  if (!ctx || !spec || !out) return HS_EINVAL;
  *out = nullptr;
  const Filter none[2];
  return bucket_join_core(ctx, spec, &spec->left_key, &spec->right_key, 1, none, true, kJoinInner, out, stats, err, errlen);
}

int hs_bucket_join_where(hs_ctx* ctx, const hs_join_spec* spec, const char* const* left_keys, const char* const* right_keys,
                         int32_t n_keys, const hs_predicate* left_preds, int32_t n_left_preds, const hs_predicate* right_preds,
                         int32_t n_right_preds, hs_batch** out, hs_stats* stats, char* err, size_t errlen) {
  return hs_bucket_join_any(ctx, spec, left_keys, right_keys, n_keys, left_preds, n_left_preds, nullptr, 0, right_preds, n_right_preds,
                            nullptr, 0, out, stats, err, errlen);
}

int hs_bucket_join_any(hs_ctx* ctx, const hs_join_spec* spec, const char* const* left_keys, const char* const* right_keys,
                       int32_t n_keys, const hs_predicate* left_preds, int32_t n_left_preds, const hs_predicate_any* left_anys,
                       int32_t n_left_anys, const hs_predicate* right_preds, int32_t n_right_preds,
                       const hs_predicate_any* right_anys, int32_t n_right_anys, hs_batch** out, hs_stats* stats, char* err,
                       size_t errlen) {
  return hs_bucket_join_cmp(ctx, spec, left_keys, right_keys, n_keys, left_preds, n_left_preds, left_anys, n_left_anys, nullptr, 0,
                            right_preds, n_right_preds, right_anys, n_right_anys, nullptr, 0, out, stats, err, errlen);
}

}  // extern "C"

// bucket_join_checked's join_type for a join_type hs_bucket_join_exists / hs_bucket_join_outer / hs_bucket_join_expr does
// not take
constexpr int kBadExistsJoin = -1, kBadOuterJoin = -2, kBadJoin = -3;

// hs_bucket_join_cmp's, hs_bucket_join_exists's and hs_bucket_join_outer's checks that need no data, then the join of the
// sides' filters
static int bucket_join_checked(hs_ctx* ctx, const hs_join_spec* spec, int join_type, const char* const* left_keys,
                               const char* const* right_keys, int n_keys, const Filter filters[2], hs_batch** out, hs_stats* stats,
                               char* err, size_t errlen) {
  if (!ctx || !spec || !out || !left_keys || !right_keys) return HS_EINVAL;
  for (int s = 0; s < 2; s++)
    if (filters[s].n_preds < 0 || (filters[s].n_preds > 0 && !filters[s].preds)) return HS_EINVAL;
  *out = nullptr;
  if (join_type == kBadExistsJoin)
    return refuse(HS_EINVAL, stats, err, errlen, "bucket join: join_type must be HS_JOIN_LEFT_SEMI or HS_JOIN_LEFT_ANTI");
  if (join_type == kBadOuterJoin)
    return refuse(HS_EINVAL, stats, err, errlen,
                  "bucket join: join_type must be HS_JOIN_LEFT_OUTER, HS_JOIN_RIGHT_OUTER or HS_JOIN_FULL_OUTER");
  if (join_type == kBadJoin)
    return refuse(HS_EINVAL, stats, err, errlen,
                  "bucket join: join_type must be HS_JOIN_INNER, HS_JOIN_LEFT_SEMI, HS_JOIN_LEFT_ANTI or an HS_JOIN_*_OUTER");
  if ((join_type == HS_JOIN_LEFT_SEMI || join_type == HS_JOIN_LEFT_ANTI) && spec->n_right_columns != 0)
    return refuse(HS_EINVAL, stats, err, errlen, "bucket join: a semi or anti join outputs left columns only (n_right_columns must be 0)");
  if (n_keys < 1) return refuse(HS_EINVAL, stats, err, errlen, "bucket join: at least one key column per side");
  if (n_keys > kMaxJoinKeys) return refuse(HS_EUNSUPPORTED, stats, err, errlen, "bucket join: more than 8 key columns");
  if (spec->left_key || spec->right_key) return refuse(HS_EINVAL, stats, err, errlen, "bucket join: the keys go in left_keys / right_keys");
  const int rc = check_filters(filters, 2, false, stats, err, errlen);
  if (rc != HS_OK) return rc;
  return bucket_join_core(ctx, spec, left_keys, right_keys, n_keys, filters, false, join_type, out, stats, err, errlen);
}

extern "C" {

int hs_bucket_join_cmp(hs_ctx* ctx, const hs_join_spec* spec, const char* const* left_keys, const char* const* right_keys,
                       int32_t n_keys, const hs_predicate* left_preds, int32_t n_left_preds, const hs_predicate_any* left_anys,
                       int32_t n_left_anys, const hs_column_compare* left_cmps, int32_t n_left_cmps, const hs_predicate* right_preds,
                       int32_t n_right_preds, const hs_predicate_any* right_anys, int32_t n_right_anys,
                       const hs_column_compare* right_cmps, int32_t n_right_cmps, hs_batch** out, hs_stats* stats, char* err,
                       size_t errlen) {
  const Filter filters[2] = {{left_preds, n_left_preds, left_anys, n_left_anys, left_cmps, n_left_cmps},
                             {right_preds, n_right_preds, right_anys, n_right_anys, right_cmps, n_right_cmps}};
  return bucket_join_checked(ctx, spec, kJoinInner, left_keys, right_keys, n_keys, filters, out, stats, err, errlen);
}

int hs_bucket_join_exists(hs_ctx* ctx, const hs_join_spec* spec, int32_t join_type, const char* const* left_keys,
                          const char* const* right_keys, int32_t n_keys, const hs_predicate* left_preds, int32_t n_left_preds,
                          const hs_predicate_any* left_anys, int32_t n_left_anys, const hs_column_compare* left_cmps,
                          int32_t n_left_cmps, const hs_predicate* right_preds, int32_t n_right_preds,
                          const hs_predicate_any* right_anys, int32_t n_right_anys, const hs_column_compare* right_cmps,
                          int32_t n_right_cmps, hs_batch** out, hs_stats* stats, char* err, size_t errlen) {
  const Filter filters[2] = {{left_preds, n_left_preds, left_anys, n_left_anys, left_cmps, n_left_cmps},
                             {right_preds, n_right_preds, right_anys, n_right_anys, right_cmps, n_right_cmps}};
  // an inner join is hs_bucket_join_cmp's: kJoinInner (0) is refused like any other value outside the two
  const bool ok = join_type == HS_JOIN_LEFT_SEMI || join_type == HS_JOIN_LEFT_ANTI;
  return bucket_join_checked(ctx, spec, ok ? join_type : kBadExistsJoin, left_keys, right_keys, n_keys, filters, out, stats, err,
                             errlen);
}

int hs_bucket_join_outer(hs_ctx* ctx, const hs_join_spec* spec, int32_t join_type, const char* const* left_keys,
                         const char* const* right_keys, int32_t n_keys, const hs_predicate* left_preds, int32_t n_left_preds,
                         const hs_predicate_any* left_anys, int32_t n_left_anys, const hs_column_compare* left_cmps,
                         int32_t n_left_cmps, const hs_predicate* right_preds, int32_t n_right_preds,
                         const hs_predicate_any* right_anys, int32_t n_right_anys, const hs_column_compare* right_cmps,
                         int32_t n_right_cmps, hs_batch** out, hs_stats* stats, char* err, size_t errlen) {
  const Filter filters[2] = {{left_preds, n_left_preds, left_anys, n_left_anys, left_cmps, n_left_cmps},
                             {right_preds, n_right_preds, right_anys, n_right_anys, right_cmps, n_right_cmps}};
  return bucket_join_checked(ctx, spec, is_outer_join(join_type) ? join_type : kBadOuterJoin, left_keys, right_keys, n_keys, filters,
                             out, stats, err, errlen);
}

int hs_bucket_join_expr(hs_ctx* ctx, const hs_join_spec* spec, int32_t join_type, const char* const* left_keys,
                        const char* const* right_keys, int32_t n_keys, const hs_predicate* left_preds, int32_t n_left_preds,
                        const hs_predicate_any* left_anys, int32_t n_left_anys, const hs_column_compare* left_cmps,
                        int32_t n_left_cmps, const hs_expr_compare* left_exprs, int32_t n_left_exprs,
                        const hs_predicate* right_preds, int32_t n_right_preds, const hs_predicate_any* right_anys,
                        int32_t n_right_anys, const hs_column_compare* right_cmps, int32_t n_right_cmps,
                        const hs_expr_compare* right_exprs, int32_t n_right_exprs, hs_batch** out, hs_stats* stats, char* err,
                        size_t errlen) {
  const Filter filters[2] = {{left_preds, n_left_preds, left_anys, n_left_anys, left_cmps, n_left_cmps, left_exprs, n_left_exprs},
                             {right_preds, n_right_preds, right_anys, n_right_anys, right_cmps, n_right_cmps, right_exprs, n_right_exprs}};
  const bool ok = join_type == HS_JOIN_INNER || join_type == HS_JOIN_LEFT_SEMI || join_type == HS_JOIN_LEFT_ANTI || is_outer_join(join_type);
  return bucket_join_checked(ctx, spec, ok ? join_type : kBadJoin, left_keys, right_keys, n_keys, filters, out, stats, err, errlen);
}

int64_t hs_batch_num_rows(const hs_batch* b) { return b ? b->nrows : 0; }
int32_t hs_batch_on_device(const hs_batch* b) { return b && b->on_device ? 1 : 0; }
int32_t hs_batch_num_columns(const hs_batch* b) { return b ? (int32_t)b->cols.size() : 0; }
int hs_batch_column(const hs_batch* b, int32_t i, const char** name, int32_t* type, const void** data,
                    const uint8_t** valid) {
  if (!b || i < 0 || i >= (int32_t)b->cols.size()) return HS_EINVAL;
  const hs_batch::Col& c = b->cols[i];
  if (name) *name = c.name.c_str();
  if (type) *type = c.type;
  if (data) *data = c.data.get();
  if (valid) *valid = c.has_valid ? c.valid.get() : nullptr;
  return HS_OK;
}
int hs_batch_string_offsets(const hs_batch* b, int32_t i, const uint64_t** offsets, uint64_t* total_bytes) {
  if (!b || i < 0 || i >= (int32_t)b->cols.size() || b->cols[i].type != HS_TYPE_STRING) return HS_EINVAL;
  if (offsets) *offsets = b->cols[i].offsets.get();
  if (total_bytes) *total_bytes = b->cols[i].total_bytes;
  return HS_OK;
}

void hs_batch_free(hs_batch* b) {
  if (!b) return;
  if (b->ctx) {
    cudaSetDevice(b->ctx->device);
    if (b->on_device) cudaStreamSynchronize(b->ctx->stream);
  }
  delete b;
}

// ---------------------------------------------------------------------------------------------------------------------
// kernel-level entry points
// ---------------------------------------------------------------------------------------------------------------------

static void upload_table(hs_ctx* ctx, const hs_host_column* keys, int nkeys, int64_t nrows, Table* t) {
  t->nrows = nrows;
  t->cols.resize(nkeys);
  for (int k = 0; k < nkeys; k++) {
    DevColumn& c = t->cols[k];
    c.name = "k" + std::to_string(k);
    c.type = keys[k].type;
    c.width = type_width(c.type);
    if (c.width == 0) fail(HS_EUNSUPPORTED, "key type %d is not handled by the GPU path", c.type);
    c.data.alloc(ctx, (size_t)nrows * c.width + 16);
    if (nrows) copy_h2d(ctx, c.data.get(), keys[k].data, (size_t)nrows * c.width);
    if (keys[k].valid) {
      c.valid.alloc(ctx, (size_t)nrows + 16);
      if (nrows) copy_h2d(ctx, c.valid.get(), keys[k].valid, (size_t)nrows);
      c.has_nulls = true;
    }
    if (keys[k].reserved == HS_KEY_DECIMAL) {  // hashed as the build hashes a decimal source column (key_column_of)
      if (c.type != HS_TYPE_INT32 && c.type != HS_TYPE_INT64) fail(HS_EINVAL, "a decimal key is an int32 or int64 column");
      c.schema.converted_type = pq::CT_DECIMAL;
      c.schema.precision = c.type == HS_TYPE_INT32 ? 9 : 18;
      c.schema.scale = 0;
    } else if (keys[k].reserved != 0) {
      fail(HS_EINVAL, "key column %d: unknown flags %d", k, keys[k].reserved);
    }
  }
  sync_stream(ctx);
}

int hs_k_bucket_ids(hs_ctx* ctx, const hs_host_column* keys, int32_t nkeys, int64_t nrows, int32_t num_buckets,
                    int32_t* out_bucket, int64_t* out_hist, char* err, size_t errlen) {
  if (!ctx) return HS_EINVAL;
  return guarded(ctx, err, errlen, [&] {
    if (num_buckets < 1 || num_buckets > kMaxBuckets) fail(HS_EUNSUPPORTED, "numBuckets must be in 1..%d", kMaxBuckets);
    Table t;
    upload_table(ctx, keys, nkeys, nrows, &t);
    std::vector<KeyColumn> h_keys(nkeys);
    for (int k = 0; k < nkeys; k++)
      h_keys[k] = key_column_of(t.cols[k]);
    Buf<unsigned long long> ghist(ctx, num_buckets);
    fill_bytes(ctx, ghist.get(), 0, 8 * num_buckets);
    HashedRows hashed;  // the hash step of index_rows
    hash_rows(ctx, h_keys.data(), nkeys, nrows, num_buckets, 0, false, ghist.get(), nullptr, &hashed);
    std::vector<uint16_t> hb(nrows);
    if (nrows) copy_d2h(ctx, hb.data(), hashed.bin_ids.get(), 2 * nrows);
    if (out_hist) copy_d2h(ctx, out_hist, ghist.get(), 8 * num_buckets);
    sync_stream(ctx);
    if (out_bucket) for (int64_t i = 0; i < nrows; i++) out_bucket[i] = hb[i];
  });
}

int hs_k_sort_perm(hs_ctx* ctx, const hs_host_column* keys, int32_t nkeys, int64_t nrows, int32_t num_buckets,
                   int64_t* out_perm, int64_t* out_bucket_offsets, char* err, size_t errlen) {
  if (!ctx) return HS_EINVAL;
  return guarded(ctx, err, errlen, [&] {
    Table t;
    upload_table(ctx, keys, nkeys, nrows, &t);
    // carry the original row index through the partition as an extra column
    DevColumn rid;
    rid.name = "__row";
    rid.type = HS_TYPE_INT32;
    rid.width = 4;
    rid.data.alloc(ctx, (size_t)nrows * 4 + 16);
    launch_iota_u32(ctx, (uint32_t*)rid.data.get(), nrows);
    t.cols.push_back(std::move(rid));
    IndexedRows rows;
    hs_stats st;
    memset(&st, 0, sizeof st);
    index_rows(ctx, t, nkeys, num_buckets, &rows, &st);
    Buf<uint8_t> orig(ctx, (size_t)std::max<int64_t>(1, nrows) * 4);
    launch_gather_plain(ctx, rows.part.cols[nkeys].data.get(), rows.sorted.perm(), nrows, 4, orig.get());
    std::vector<uint32_t> h(nrows);
    if (nrows) copy_d2h(ctx, h.data(), orig.get(), 4 * nrows);
    sync_stream(ctx);
    for (int64_t i = 0; i < nrows; i++) out_perm[i] = h[i];
    for (int b = 0; b <= num_buckets; b++) out_bucket_offsets[b] = (int64_t)rows.bucket_offsets[b];
  });
}

int hs_k_partition(hs_ctx* ctx, const hs_host_column* keys, int32_t nkeys, int64_t nrows, int32_t num_buckets,
                   const hs_host_column* payload, int32_t npayload, const uint16_t* const* codes, int32_t ncodes,
                   int32_t mode, int32_t world, const uint64_t* peer_base, const uint64_t* owner_rows,
                   const int32_t* owner_shift, int32_t fill, void* const* out_payload, void* const* out_records,
                   uint64_t* out_offsets, uint64_t* out_key_or_and, char* err, size_t errlen) {
  if (!ctx) return HS_EINVAL;
  return guarded(ctx, err, errlen, [&] {
    if (num_buckets < 1 || num_buckets > kMaxBuckets) fail(HS_EUNSUPPORTED, "numBuckets must be in 1..%d", kMaxBuckets);
    if (nkeys < 1 || !keys || nrows < 0 || nrows >= (1ll << 32)) fail(HS_EINVAL, "bad keys or row count");
    if (mode != HS_PART_LOCAL && mode != HS_PART_OWNER && mode != HS_PART_PEER) fail(HS_EINVAL, "unknown mode %d", mode);
    if (world < 1 || world > 64) fail(HS_EINVAL, "world = %d: 1..64 owners", world);
    if (npayload < 0 || (npayload && (!payload || !out_payload))) fail(HS_EINVAL, "bad payload columns");
    if (ncodes < 0 || ncodes > 4 || (ncodes && (!codes || !out_records))) fail(HS_EINVAL, "bad code columns");
    if (peer_base && !owner_rows) fail(HS_EINVAL, "a peer layout needs every owner's buffer size");
    Table t;
    upload_table(ctx, keys, nkeys, nrows, &t);
    std::vector<KeyColumn> h_keys(nkeys);
    for (int k = 0; k < nkeys; k++) h_keys[k] = key_column_of(t.cols[k]);
    const int owner_mod = mode == HS_PART_OWNER ? world : 0;
    const int nbins = owner_mod > 0 ? owner_mod : num_buckets;
    // output buffers: one per column, or one per (column, owner) with a peer layout; `shift` bytes before the first row
    const int owners = peer_base ? world : 1;
    auto rows_of = [&](int o) { return peer_base ? (size_t)owner_rows[o] : (size_t)nrows; };
    auto shift_of = [&](int o) -> size_t {
      const int s = peer_base && owner_shift ? owner_shift[o] : 0;
      if (s != 0 && s != 8) fail(HS_EINVAL, "owner %d: shift %d bytes, 0 or 8 expected", o, s);
      return (size_t)s;
    };
    std::vector<Buf<uint8_t>> in(npayload), out((size_t)(npayload + 1) * owners);
    std::vector<size_t> out_bytes((size_t)(npayload + 1) * owners, 0);
    std::vector<void*> table((size_t)(npayload + 1) * owners, nullptr);  // the peer table: a row of owners per round
    std::vector<PartColumn> h_pc(npayload);
    auto alloc_out = [&](size_t i, int o, int width) {
      out_bytes[i] = shift_of(o) + rows_of(o) * width + 16;
      out[i].alloc(ctx, out_bytes[i]);
      fill_bytes(ctx, out[i].get(), fill & 0xff, out_bytes[i]);
      table[i] = out[i].get() + shift_of(o);
    };
    for (int c = 0; c < npayload; c++) {
      const int width = payload[c].type == HS_TYPE_STRING ? 0 : type_width(payload[c].type);
      if (width != 1 && width != 4 && width != 8) fail(HS_EINVAL, "payload column %d: type %d", c, payload[c].type);
      in[c].alloc(ctx, (size_t)nrows * width + 16);
      if (nrows) copy_h2d(ctx, in[c].get(), payload[c].data, (size_t)nrows * width);
      for (int o = 0; o < owners; o++) alloc_out((size_t)c * owners + o, o, width);
      h_pc[c] = PartColumn{in[c].get(), peer_base ? nullptr : table[(size_t)c * owners], width, 0};
    }
    std::vector<Buf<uint16_t>> code_in(ncodes);
    CodePackRound pack;
    memset(&pack, 0, sizeof pack);
    for (int j = 0; j < ncodes; j++) {
      code_in[j].alloc(ctx, (size_t)nrows + 16);
      if (nrows) copy_h2d(ctx, code_in[j].get(), codes[j], (size_t)nrows * 2);
      pack.src[j] = code_in[j].get();
    }
    pack.n = ncodes;
    if (ncodes) {
      for (int o = 0; o < owners; o++) alloc_out((size_t)npayload * owners + o, o, 8);
      if (!peer_base) pack.out = table[(size_t)npayload * owners];
    }
    Buf<unsigned long long> ghist(ctx, nbins), offsets(ctx, nbins + 1), key_bits(ctx, 2), base;
    fill_bytes(ctx, ghist.get(), 0, 8 * (size_t)nbins);
    const unsigned long long init[2] = {0ull, ~0ull};
    copy_h2d(ctx, key_bits.get(), init, sizeof init);
    if (peer_base) {
      base.alloc(ctx, std::max(nbins, num_buckets));
      fill_bytes(ctx, base.get(), 0, 8 * (size_t)std::max(nbins, num_buckets));
      copy_h2d(ctx, base.get(), peer_base, 8 * (size_t)num_buckets);
    }
    Buf<void*> d_table(ctx, table.size());
    copy_h2d(ctx, d_table.get(), table.data(), sizeof(void*) * table.size());
    // the three steps of index_rows (one GPU) and exchange_partition_p2p (the owners' buffers over NVLink)
    HashedRows hashed;
    hash_rows(ctx, h_keys.data(), nkeys, nrows, num_buckets, owner_mod, mode == HS_PART_PEER, ghist.get(), key_bits.get(),
              &hashed);
    launch_tile_offsets(ctx, hashed.tile_hist.get(), hashed.ntiles, nbins, ghist.get(), peer_base ? nullptr : offsets.get(),
                        peer_base ? base.get() : nullptr);
    move_rows(ctx, hashed, h_pc.data(), npayload, &pack, peer_base ? d_table.get() : nullptr, world);
    for (int c = 0; c < npayload; c++)
      for (int o = 0; o < owners; o++) {
        const size_t i = (size_t)c * owners + o;
        copy_d2h(ctx, out_payload[i], out[i].get(), out_bytes[i]);
      }
    for (int o = 0; ncodes && o < owners; o++) {
      const size_t i = (size_t)npayload * owners + o;
      copy_d2h(ctx, out_records[o], out[i].get(), out_bytes[i]);
    }
    if (out_offsets && !peer_base) copy_d2h(ctx, out_offsets, offsets.get(), 8 * (size_t)(nbins + 1));
    if (out_key_or_and) copy_d2h(ctx, out_key_or_and, key_bits.get(), sizeof init);
    sync_stream(ctx);
  });
}

int hs_synth_table(hs_ctx* ctx, int64_t first_row, int64_t nrows, int32_t ncols, int32_t n_files,
                   int32_t row_groups_per_file, int32_t dictionary, int32_t output, hs_index_result** out, char* err,
                   size_t errlen) {
  return hs_synth_table_ex(ctx, first_row, nrows, ncols, n_files, row_groups_per_file, dictionary, HS_CODEC_UNCOMPRESSED, output, out,
                           err, errlen);
}

namespace {
// one page body through compress_bodies, as the encoder compresses it: preamble, pieces, trailer
int compress_one_body(hs_ctx* ctx, int codec, const void* in, uint64_t n, void* out_buf, uint64_t cap, uint64_t* out_len,
                      char* err, size_t errlen) {
  return guarded(ctx, err, errlen, [&] {
    Buf<uint8_t> d_in(ctx, std::max<uint64_t>(n, 16) + 16);
    if (n) copy_h2d(ctx, d_in.get(), in, n);
    CompressedBodies packed;
    compress_bodies(ctx, codec, d_in.get(), {{0, n}}, &packed);
    std::vector<uint8_t> stream;
    packed.append_preamble(0, stream);
    std::vector<BlobCopy> pieces;
    uint64_t end = stream.size();
    packed.place(0, pieces, &end);
    stream.resize(end);
    for (const BlobCopy& pc : pieces)
      HS_CUDA(cudaMemcpy(stream.data() + pc.dst, packed.slots.get() + pc.src, pc.len, cudaMemcpyDeviceToHost));
    packed.append_trailer(0, stream);
    *out_len = stream.size();
    if (stream.size() > cap) fail(HS_ENOMEM, "output buffer too small: %zu bytes needed", stream.size());
    if (out_buf) memcpy(out_buf, stream.data(), stream.size());
  });
}
}  // namespace

int hs_k_snappy_compress(hs_ctx* ctx, const void* in, uint64_t n, void* out_buf, uint64_t cap, uint64_t* out_len, char* err,
                         size_t errlen) {
  if (!ctx || !out_len || (n && !in)) return HS_EINVAL;
  return compress_one_body(ctx, pq::SNAPPY, in, n, out_buf, cap, out_len, err, errlen);
}

int hs_k_compress(hs_ctx* ctx, int32_t codec, const void* in, uint64_t n, void* out_buf, uint64_t cap, uint64_t* out_len,
                  char* err, size_t errlen) {
  if (!ctx || !out_len || (n && !in) || (codec != HS_CODEC_GZIP && codec != HS_CODEC_LZ4)) return HS_EINVAL;
  return compress_one_body(ctx, codec, in, n, out_buf, cap, out_len, err, errlen);
}

namespace {
// Blobs of one host buffer through decompress_blobs, in one launch as decompress_pages makes it: each blob's `src` holds
// its offset in `in` on entry.  The whole scratch is pre-filled with `fill` and copied back to `out`, gaps included, so a
// caller sees any byte a decoder wrote outside its blob.  sequential (optional): per blob in the caller's order, 1 where
// a snappy stream was decoded front to back.
void decompress_host_blobs(hs_ctx* ctx, const void* in, uint64_t n_in, std::vector<PageBlob> blobs, int fill, void* out,
                           uint64_t out_len, int32_t* sequential) {
  // decoders read up to 8 bytes past a stream and one aligned word past a page
  Buf<uint8_t> d_in(ctx, n_in + 16), d_out(ctx, out_len + 32);
  if (n_in) copy_h2d(ctx, d_in.get(), in, n_in);
  fill_bytes(ctx, d_out.get(), fill, out_len + 32);
  Buf<uint32_t> d_error(ctx, 1);
  fill_bytes(ctx, d_error.get(), 0, 4);
  std::vector<uint32_t> codecs(blobs.size());
  for (size_t i = 0; i < blobs.size(); i++) {
    blobs[i].src = d_in.get() + (uintptr_t)blobs[i].src;
    codecs[i] = blobs[i].codec;
  }
  std::vector<uint32_t> seq;
  decompress_blobs(ctx, blobs, d_out.get(), d_error.get(), &seq);
  uint32_t error = 0;
  copy_d2h(ctx, &error, d_error.get(), 4);
  sync_stream(ctx);
  const uint32_t check = error & 0xffffffu;
  if ((error >> 24) == DERR_SNAPPY) fail(HS_EFORMAT, "corrupt snappy stream (check %u)", check);
  if ((error >> 24) == DERR_GZIP) fail(HS_EFORMAT, "corrupt gzip stream: %s (check %u)", gz::inflate_error_text(check), check);
  if ((error >> 24) == DERR_LZ4) fail(HS_EFORMAT, "corrupt lz4 block: %s (check %u)", lz4::lz4_error_text(check), check);
  if (error) fail(HS_EFORMAT, "page decompression failed (code %u, check %u)", error >> 24, check);
  if (out_len) HS_CUDA(cudaMemcpy(out, d_out.get(), out_len, cudaMemcpyDeviceToHost));
  if (sequential) {  // decompress_blobs puts the snappy blobs first, in the caller's order
    size_t k = 0;
    for (size_t i = 0; i < codecs.size(); i++) sequential[i] = codecs[i] == (uint32_t)pq::SNAPPY ? (int32_t)seq[k++] : 0;
  }
}

PageBlob one_blob(uint64_t n, uint64_t out_len, int codec) {
  return PageBlob{nullptr, 0, (uint32_t)n, (uint32_t)out_len, 0u, 1u, 0u, (uint32_t)codec};
}
}  // namespace

int hs_k_decompress_blobs(hs_ctx* ctx, const void* in, uint64_t n_in, int32_t n_blobs, const uint64_t* src_off,
                          const uint32_t* src_len, const uint64_t* dst_off, const uint32_t* dst_len, const uint32_t* prefix,
                          const int32_t* compressed, const int32_t* codec, int32_t fill, void* out, uint64_t out_len,
                          int32_t* sequential, char* err, size_t errlen) {
  if (!ctx || n_blobs < 0 || (n_in && !in) || (out_len && !out) ||
      (n_blobs && (!src_off || !src_len || !dst_off || !dst_len || !prefix || !compressed || !codec)))
    return HS_EINVAL;
  return guarded(ctx, err, errlen, [&] {
    if (n_in > 0xffffffffull || out_len > 0xfffffff0ull) fail(HS_EINVAL, "buffers above 4 GB");
    std::vector<PageBlob> blobs;
    std::vector<std::pair<uint64_t, uint64_t>> dst;  // (offset, length) of every blob's decoded bytes
    for (int32_t i = 0; i < n_blobs; i++) {
      const int c = codec[i];
      if (c != pq::SNAPPY && c != pq::GZIP && c != pq::LZ4 && c != pq::LZ4_RAW) fail(HS_EINVAL, "blob %d: codec %d", i, c);
      if (compressed[i] != 0 && compressed[i] != 1) fail(HS_EINVAL, "blob %d: compressed must be 0 or 1", i);
      if (src_off[i] > n_in || src_len[i] > n_in - src_off[i]) fail(HS_EINVAL, "blob %d: source range beyond the input", i);
      if (dst_off[i] > out_len || dst_len[i] > out_len - dst_off[i]) fail(HS_EINVAL, "blob %d: destination range beyond the output", i);
      if (prefix[i] > src_len[i] || prefix[i] > dst_len[i]) fail(HS_EINVAL, "blob %d: prefix beyond the blob", i);
      blobs.push_back(PageBlob{(const uint8_t*)(uintptr_t)src_off[i], dst_off[i], src_len[i], dst_len[i], prefix[i],
                               (uint32_t)compressed[i], 0u, (uint32_t)c});
      dst.emplace_back(dst_off[i], dst_len[i]);
    }
    std::sort(dst.begin(), dst.end());
    for (size_t i = 1; i < dst.size(); i++)
      if (dst[i - 1].first + dst[i - 1].second > dst[i].first) fail(HS_EINVAL, "destination ranges overlap");
    decompress_host_blobs(ctx, in, n_in, std::move(blobs), fill, out, out_len, sequential);
  });
}

int hs_k_snappy_decompress(hs_ctx* ctx, const void* in, uint64_t n, void* out_buf, uint64_t out_len, int32_t* sequential,
                           char* err, size_t errlen) {
  if (!ctx || !in || n == 0 || n > 0xffffffffull || out_len > 0xfffffff0ull || (out_len && !out_buf)) return HS_EINVAL;
  return guarded(ctx, err, errlen,
                 [&] { decompress_host_blobs(ctx, in, n, {one_blob(n, out_len, pq::SNAPPY)}, 0, out_buf, out_len, sequential); });
}

int hs_k_inflate(hs_ctx* ctx, const void* in, uint64_t n, void* out_buf, uint64_t out_len, char* err, size_t errlen) {
  if (!ctx || (n && !in) || n > 0xffffffffull || out_len > 0xfffffff0ull || (out_len && !out_buf)) return HS_EINVAL;
  return guarded(ctx, err, errlen,
                 [&] { decompress_host_blobs(ctx, in, n, {one_blob(n, out_len, pq::GZIP)}, 0, out_buf, out_len, nullptr); });
}

int hs_k_lz4(hs_ctx* ctx, int32_t codec, const void* in, uint64_t n, void* out_buf, uint64_t out_len, char* err, size_t errlen) {
  if (!ctx || (codec != pq::LZ4 && codec != pq::LZ4_RAW) || (n && !in) || n > 0xffffffffull || out_len > 0xfffffff0ull ||
      (out_len && !out_buf))
    return HS_EINVAL;
  return guarded(ctx, err, errlen,
                 [&] { decompress_host_blobs(ctx, in, n, {one_blob(n, out_len, codec)}, 0, out_buf, out_len, nullptr); });
}

int hs_synth_table_ex(hs_ctx* ctx, int64_t first_row, int64_t nrows, int32_t ncols, int32_t n_files,
                      int32_t row_groups_per_file, int32_t dictionary, int32_t compression, int32_t output,
                      hs_index_result** out, char* err, size_t errlen) {
  if (!ctx || !out) return HS_EINVAL;
  *out = nullptr;
  std::unique_ptr<hs_index_result> res(new hs_index_result());
  int rc = guarded(ctx, err, errlen, [&] {
    if (ncols < 1 || ncols > 5 || n_files < 1 || row_groups_per_file < 1 || nrows < 0) fail(HS_EINVAL, "bad synthetic table shape");
    if (output != HS_OUT_HOST && output != HS_OUT_DEVICE) fail(HS_EINVAL, "synthetic tables are returned in memory");
    static const char* names[5] = {"k", "v1", "v2", "v3", "v4"};
    static const int types[5] = {HS_TYPE_INT64, HS_TYPE_INT64, HS_TYPE_DOUBLE, HS_TYPE_INT32, HS_TYPE_FLOAT};
    static const int ptypes[5] = {pq::INT64, pq::INT64, pq::DOUBLE, pq::INT32, pq::FLOAT};
    Table t;
    t.nrows = nrows;
    t.cols.resize(ncols);
    for (int c = 0; c < ncols; c++) {
      DevColumn& dc = t.cols[c];
      dc.name = names[c];
      dc.type = types[c];
      dc.width = type_width(types[c]);
      dc.schema.name = names[c];
      dc.schema.type = ptypes[c];
      dc.schema.repetition = pq::OPTIONAL;
      dc.data.alloc(ctx, (size_t)nrows * dc.width + 16);
      launch_synth_column(ctx, c, first_row, nrows, dc.data.get());
    }
    // files are the segments; rows split evenly, row groups per file likewise (multiples of the page size)
    const int64_t P = 131072;
    std::vector<uint64_t> seg(n_files + 1, 0);
    const int64_t per_file = ceil_div(nrows, n_files);
    for (int f = 0; f < n_files; f++) seg[f + 1] = (uint64_t)std::min<int64_t>(nrows, (int64_t)(f + 1) * per_file);
    SortPlan plan;
    build_sort_plan(ctx, seg.data(), n_files, &plan);
    Buf<uint32_t> iota(ctx, std::max<int64_t>(1, nrows));
    launch_iota_u32(ctx, iota.get(), nrows);
    EncodeRequest req;
    req.table = &t;
    req.d_perm = iota.get();
    req.plan = &plan;
    req.seg_offsets = seg;
    req.rows_per_page = P;
    req.use_dictionary = dictionary != 0;
    if (compression != HS_CODEC_UNCOMPRESSED && compression != HS_CODEC_SNAPPY) fail(HS_EUNSUPPORTED, "compression codec %d", compression);
    req.codec = compression == HS_CODEC_SNAPPY ? pq::SNAPPY : pq::UNCOMPRESSED;
    req.rows_per_row_group = std::max<int64_t>(P, (int64_t)round_up((size_t)ceil_div(per_file, row_groups_per_file), (size_t)P));
    req.seg_names.resize(n_files);
    for (int f = 0; f < n_files; f++) {
      char nm[64];
      snprintf(nm, sizeof nm, "part-%05d.parquet", f);
      req.seg_names[f] = nm;
    }
    EncodedFiles enc;
    hs_stats st;
    memset(&st, 0, sizeof st);
    encode_segments(ctx, req, &enc, &st);
    finish_result(ctx, enc, output, nullptr, HS_SAVE_OVERWRITE, res.get(), &st);
  });
  if (rc == HS_OK) *out = res.release();
  return rc;
}

}  // extern "C"
