// verify.cu -- whole-index consistency checks on the GPU (hs_verify_index, hs_synth_checksum).
//
// The reference pins the written index through three properties (T/index/DataFrameWriterExtensionsTest.scala:93-158):
// every row of a bucket file hashes to that file's bucket id (Spark's HashPartitioning.partitionIdExpression), every file
// is sorted on the indexed columns, and the files together hold exactly the source's rows.  hs_verify_index evaluates the
// same three on index files of any size -- the 1 B-row benchmark output is checked this way after every bench run:
//   * bucket_mismatches  rows whose pmod(murmur3(keys, 42), numBuckets) differs from the bucket of their file
//   * order_violations   adjacent rows of one file whose key tuples are not ascending (nulls first)
//   * row_checksum       sum over rows (mod 2^64) of a 64-bit mix of ALL the row's column values: independent of row
//                        order, but a value that moved to another row changes it; equal to the same sum over the source
//                        rows (hs_synth_checksum for the synthetic table) iff the row multiset survived
//   * column_checksum[c] the same per column (tells which column broke)
#include "device_utils.cuh"
#include "engine.h"

namespace hs {
namespace {

constexpr int kMaxVerifyCols = 16;

struct VerifyCols {
  const void* data[kMaxVerifyCols];
  const uint8_t* valid[kMaxVerifyCols];
  int32_t width[kMaxVerifyCols];
  int32_t type[kMaxVerifyCols];
  int32_t ncols;
};

// what a string contributes to the checksums: a 64-bit digest of its bytes and its length (never its address)
__device__ __forceinline__ uint64_t string_digest(uint64_t ref) {
  const uint8_t* p = ref_ptr(ref);
  const uint32_t len = ref_len(ref);
  uint64_t h = 0xCBF29CE484222325ull ^ len;
  for (uint32_t i = 0; i < len; i++) h = (h ^ p[i]) * 0x100000001B3ull;
  return h;
}

__host__ __device__ __forceinline__ uint64_t mix64(uint64_t z) {
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}

__device__ __forceinline__ uint64_t raw_value(const void* data, int width, int64_t row) {
  switch (width) {
    case 8: return ((const uint64_t*)data)[row];
    case 4: return ((const uint32_t*)data)[row];
    default: return ((const uint8_t*)data)[row];
  }
}

// sums[0] = row checksum, sums[1 + c] = checksum of column c
__global__ void __launch_bounds__(256) k_row_checksums(VerifyCols cols, int64_t nrows, unsigned long long* __restrict__ sums) {
  uint64_t acc[1 + kMaxVerifyCols];
#pragma unroll
  for (int c = 0; c <= kMaxVerifyCols; c++) acc[c] = 0;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < nrows; i += stride) {
    uint64_t h = 0x9E3779B97F4A7C15ull;
#pragma unroll
    for (int c = 0; c < kMaxVerifyCols; c++) {
      if (c < cols.ncols) {
        const bool null = cols.valid[c] && !cols.valid[c][i];
        uint64_t v = null ? 0x6C6C756E6C6C756Eull : raw_value(cols.data[c], cols.width[c], i);
        if (!null && cols.type[c] == HS_TYPE_STRING) v = string_digest(v);
        const uint64_t salted = v + (uint64_t)(c + 1) * 0xD6E8FEB86659FD93ull + (null ? 1ull : 0ull);
        acc[1 + c] += mix64(salted);
        h = mix64(h ^ salted);
      }
    }
    acc[0] += h;
  }
#pragma unroll
  for (int c = 0; c <= kMaxVerifyCols; c++) {
    if (c > cols.ncols) break;
    unsigned long long v = acc[c];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if ((threadIdx.x & 31) == 0) atomicAdd(&sums[c], v);
  }
}

// -1 / 0 / +1: key tuple of row a against row b, ascending nulls first (Spark's SortOrder on the indexed columns)
__device__ __forceinline__ int compare_rows(const KeyColumn* keys, int nkeys, int64_t a, int64_t b) {
  for (int k = 0; k < nkeys; k++) {
    const KeyColumn kc = keys[k];
    const bool va = !kc.valid || kc.valid[a], vb = !kc.valid || kc.valid[b];
    if (va != vb) return va ? 1 : -1;
    if (!va) continue;
    if (kc.type == HS_TYPE_STRING) {
      const int r = string_compare(raw_value(kc.data, 8, a), raw_value(kc.data, 8, b));
      if (r) return r;
      continue;
    }
    const uint64_t ea = sort_encode(kc.type, raw_value(kc.data, kc.width, a));
    const uint64_t eb = sort_encode(kc.type, raw_value(kc.data, kc.width, b));
    if (ea != eb) return ea < eb ? -1 : 1;
  }
  return 0;
}

// counters[0] = bucket mismatches, counters[1] = order violations
__global__ void __launch_bounds__(256) k_check_rows(const KeyColumn* __restrict__ keys, int nkeys, int64_t nrows, int nb,
                                                     const int64_t* __restrict__ file_row_begin,
                                                     const int32_t* __restrict__ file_bucket, int nfiles,
                                                     unsigned long long* __restrict__ counters) {
  unsigned long long bad_bucket = 0, bad_order = 0;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < nrows; i += stride) {
    int lo = 0, hi = nfiles;  // last file whose first row is <= i
    while (hi - lo > 1) {
      const int mid = (lo + hi) >> 1;
      if (file_row_begin[mid] <= i) lo = mid;
      else hi = mid;
    }
    uint32_t h = 42;
    for (int k = 0; k < nkeys; k++) {
      const KeyColumn kc = keys[k];
      if (kc.valid && !kc.valid[i]) continue;
      h = mm3_hash_value(key_hash_kind(kc), raw_value(kc.data, kc.width, i), h);
    }
    if (spark_pmod(h, nb) != file_bucket[lo]) bad_bucket++;
    if (i > file_row_begin[lo] && compare_rows(keys, nkeys, i - 1, i) > 0) bad_order++;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    bad_bucket += __shfl_xor_sync(0xffffffffu, bad_bucket, o);
    bad_order += __shfl_xor_sync(0xffffffffu, bad_order, o);
  }
  if ((threadIdx.x & 31) == 0) {
    if (bad_bucket) atomicAdd(&counters[0], bad_bucket);
    if (bad_order) atomicAdd(&counters[1], bad_order);
  }
}

void checksum_table(hs_ctx* ctx, const Table& t, unsigned long long* d_sums) {
  const int ncols = (int)t.cols.size();
  if (ncols > kMaxVerifyCols) fail(HS_EUNSUPPORTED, "verification handles up to %d columns", kMaxVerifyCols);
  if (t.nrows == 0) return;
  VerifyCols vc;
  memset(&vc, 0, sizeof vc);
  vc.ncols = ncols;
  for (int c = 0; c < ncols; c++) {
    vc.data[c] = t.cols[c].data.get();
    vc.valid[c] = t.cols[c].has_nulls ? t.cols[c].valid.get() : nullptr;
    vc.width[c] = t.cols[c].width;
    vc.type[c] = t.cols[c].type;
  }
  const int grid = (int)std::min<int64_t>(ceil_div(t.nrows, 256), (int64_t)ctx->sm_count * 8);
  k_row_checksums<<<grid, 256, 0, ctx->stream>>>(vc, t.nrows, d_sums);
  HS_LAUNCH_CHECK(ctx);
}

template <typename F>
int guarded_call(hs_ctx* ctx, char* err, size_t errlen, F&& f) {
  try {
    cudaError_t e = cudaSetDevice(ctx->device);
    if (e != cudaSuccess) fail(HS_ECUDA, "cudaSetDevice(%d): %s", ctx->device, cudaGetErrorString(e));
    ctx->launches = 0;
    f();
    return HS_OK;
  } catch (const hs::Error& e) {
    if (err && errlen) {
      strncpy(err, e.what(), errlen - 1);
      err[errlen - 1] = 0;
    }
    xfer_abort(ctx);
    cudaGetLastError();
    return e.code;
  }
}

}  // namespace
}  // namespace hs

using namespace hs;

extern "C" {

int hs_verify_index(hs_ctx* ctx, const hs_source_file* files, const int32_t* buckets, int32_t n_files,
                    const char* const* indexed_columns, int32_t n_indexed, const char* const* included_columns,
                    int32_t n_included, int32_t num_buckets, hs_verify_report* out, char* err, size_t errlen) {
  if (!ctx || !out || n_files < 0 || (n_files > 0 && (!files || !buckets)) || n_indexed < 1) return HS_EINVAL;
  memset(out, 0, sizeof *out);
  return guarded_call(ctx, err, errlen, [&] {
    if (num_buckets < 1) fail(HS_EINVAL, "num_buckets must be positive");
    std::vector<std::string> cols;
    for (int i = 0; i < n_indexed; i++) cols.emplace_back(indexed_columns[i]);
    for (int i = 0; i < n_included; i++) cols.emplace_back(included_columns[i]);
    if ((int)cols.size() > kMaxVerifyCols) fail(HS_EUNSUPPORTED, "verification handles up to %d columns", kMaxVerifyCols);
    out->n_columns = (int32_t)cols.size();
    if (n_files == 0) return;
    for (int f = 0; f < n_files; f++)
      if (buckets[f] < 0 || buckets[f] >= num_buckets) fail(HS_EINVAL, "bucket id %d out of range", buckets[f]);
    hs_stats st;
    memset(&st, 0, sizeof st);
    Table t;
    SourceSet src;  // outlives the kernels below: string columns hold references into its images
    open_sources(ctx, files, n_files, &src, &st);
    decode_sources(ctx, src, cols, nullptr, &t, &st);
    out->rows = t.nrows;
    Buf<unsigned long long> d_sums(ctx, 2 + 1 + kMaxVerifyCols);
    fill_bytes(ctx, d_sums.get(), 0, 8 * (3 + kMaxVerifyCols));
    checksum_table(ctx, t, d_sums.get() + 2);
    std::vector<KeyColumn> h_keys(n_indexed);
    for (int k = 0; k < n_indexed; k++) {
      h_keys[k] = key_column_of(t.cols[k]);
    }
    Buf<KeyColumn> d_keys(ctx, n_indexed);
    Buf<int64_t> d_frb(ctx, n_files + 1);
    Buf<int32_t> d_fb(ctx, n_files);
    copy_h2d(ctx, d_keys.get(), h_keys.data(), sizeof(KeyColumn) * n_indexed);
    copy_h2d(ctx, d_frb.get(), t.file_row_begin.data(), 8 * (size_t)(n_files + 1));
    copy_h2d(ctx, d_fb.get(), buckets, 4 * (size_t)n_files);
    if (t.nrows) {
      const int grid = (int)std::min<int64_t>(ceil_div(t.nrows, 256), (int64_t)ctx->sm_count * 8);
      k_check_rows<<<grid, 256, 0, ctx->stream>>>(d_keys.get(), n_indexed, t.nrows, num_buckets, d_frb.get(), d_fb.get(), n_files,
                                                  d_sums.get());
      HS_LAUNCH_CHECK(ctx);
    }
    unsigned long long h[3 + kMaxVerifyCols];
    copy_d2h(ctx, h, d_sums.get(), sizeof h);
    sync_stream(ctx);
    out->bucket_mismatches = (int64_t)h[0];
    out->order_violations = (int64_t)h[1];
    out->row_checksum = h[2];
    for (int c = 0; c < out->n_columns; c++) out->column_checksum[c] = h[3 + c];
  });
}

int hs_synth_checksum(hs_ctx* ctx, int64_t first_row, int64_t nrows, int32_t ncols, hs_verify_report* out, char* err,
                      size_t errlen) {
  if (!ctx || !out || ncols < 1 || ncols > 5 || nrows < 0) return HS_EINVAL;
  memset(out, 0, sizeof *out);
  return guarded_call(ctx, err, errlen, [&] {
    static const int types[5] = {HS_TYPE_INT64, HS_TYPE_INT64, HS_TYPE_DOUBLE, HS_TYPE_INT32, HS_TYPE_FLOAT};
    out->n_columns = ncols;
    out->rows = nrows;
    Buf<unsigned long long> d_sums(ctx, 1 + kMaxVerifyCols);
    fill_bytes(ctx, d_sums.get(), 0, 8 * (1 + kMaxVerifyCols));
    const int64_t chunk = 1ll << 26;  // generated and summed 64 M rows at a time: no table-sized allocation
    Table t;
    t.cols.resize(ncols);
    for (int c = 0; c < ncols; c++) {
      t.cols[c].type = types[c];
      t.cols[c].width = type_width(types[c]);
      t.cols[c].data.alloc(ctx, (size_t)std::min(chunk, std::max<int64_t>(1, nrows)) * t.cols[c].width + 16);
    }
    for (int64_t r0 = 0; r0 < nrows; r0 += chunk) {
      t.nrows = std::min(chunk, nrows - r0);
      for (int c = 0; c < ncols; c++) launch_synth_column(ctx, c, first_row + r0, t.nrows, t.cols[c].data.get());
      checksum_table(ctx, t, d_sums.get());
    }
    unsigned long long h[1 + kMaxVerifyCols];
    copy_d2h(ctx, h, d_sums.get(), sizeof h);
    sync_stream(ctx);
    out->row_checksum = h[0];
    for (int c = 0; c < ncols; c++) out->column_checksum[c] = h[1 + c];
  });
}

}  // extern "C"
