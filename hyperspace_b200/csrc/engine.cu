// engine.cu -- host orchestration of the covering-index data path on one GPU:
//   load_sources   (H2D of file images, footer parse, K1 page walk + decode)
//   index_rows     (K2 hash + histogram, K3 stable partition, K4 segmented radix sort)
//   encode_segments(K5 gather fused with K6 PLAIN page encode into one file image per bucket)
// Together they are the body of CoveringIndex.write (index/covering/CoveringIndex.scala:56-71) as executed by Spark
// for the reference: scan -> project -> repartition(numBuckets, indexedColumns) -> sort within bucket -> bucketed
// Parquet write (index/DataFrameWriterExtensions.scala:50-68).
#include <fcntl.h>
#include <sys/stat.h>
#include <unistd.h>

#include <algorithm>
#include <array>
#include <map>
#include <random>

#include "device_utils.cuh"
#include "engine.h"
#include "inflate.h"
#include "lz4_block.h"
#include "spark_types.h"

namespace hs {

std::string make_uuid() {
  std::random_device rd;
  std::mt19937_64 gen(((uint64_t)rd() << 32) ^ rd());
  uint64_t a = gen(), b = gen();
  char buf[40];
  snprintf(buf, sizeof buf, "%08x-%04x-4%03x-%04x-%012llx", (unsigned)(a >> 32), (unsigned)((a >> 16) & 0xffff),
           (unsigned)(a & 0xfff), (unsigned)(0x8000 | ((b >> 48) & 0x3fff)), (unsigned long long)(b & 0xffffffffffffull));
  return buf;
}

namespace {

bool iequals(const std::string& a, const std::string& b) {
  if (a.size() != b.size()) return false;
  for (size_t i = 0; i < a.size(); i++)
    if (tolower((unsigned char)a[i]) != tolower((unsigned char)b[i])) return false;
  return true;
}

int find_column(const pq::FileMeta& fm, const std::string& name) {
  for (size_t i = 0; i < fm.columns.size(); i++)
    if (fm.columns[i].name == name) return (int)i;
  for (size_t i = 0; i < fm.columns.size(); i++)  // Spark resolves names case-insensitively by default
    if (iequals(fm.columns[i].name, name)) return (int)i;
  return -1;
}

const char* decode_error_text(uint32_t code) {
  switch (code) {
    case DERR_BAD_HEADER: return "malformed page header";
    case DERR_UNSUPPORTED_ENCODING: return "unsupported page encoding (PLAIN, PLAIN_/RLE_DICTIONARY and RLE for BOOLEAN are handled)";
    case DERR_VALUE_COUNT: return "page value counts do not add up to the column chunk's num_values";
    case DERR_COMPRESSED: return "page sizes disagree in an UNCOMPRESSED chunk";
    case DERR_OVERRUN: return "page data shorter than its header claims";
    case DERR_DICT_INDEX: return "dictionary index out of range or missing dictionary page";
    case DERR_UNSUPPORTED_TYPE: return "unsupported physical type";
    case DERR_SNAPPY: return "corrupt snappy stream";
    case DERR_STRING_TOO_LONG: return "string / binary value longer than 65535 bytes";
    case DERR_SPARK_RANGE: return "timestamp that Spark 3.1 does not read (an INT96 value before 1900-01-01T00:00:00Z, or millis beyond the int64 micros range)";
    case DERR_DECIMAL_WIDTH: return "decimal value wider than its precision allows";
    case DERR_GZIP: return "corrupt gzip stream";
    case DERR_LZ4: return "corrupt lz4 block";
  }
  return "unknown decode error";
}

struct FileImage {
  std::string what;
  const uint8_t* dev = nullptr;
  uint64_t size = 0;
  pq::FileMeta meta;
};

void read_whole_file(const char* path, uint8_t* dst, uint64_t size) {
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

struct SourceSet::Impl {
  std::vector<FileImage> imgs;
  Buf<uint8_t> d_images;
  Buf<uint8_t> d_scratch;  // decompressed pages: string references may point into them, like into the images
};
SourceSet::SourceSet() : impl(new Impl()) {}
SourceSet::~SourceSet() { delete impl; }
void SourceSet::release_images() {
  impl->d_images.release();
  impl->d_scratch.release();
}

void load_sources(hs_ctx* ctx, const hs_source_file* files, int n_files, const std::vector<std::string>& columns,
                  Table* out, hs_stats* stats, const CarryOptions* carry) {
  SourceSet src;
  open_sources(ctx, files, n_files, &src, stats);
  decode_sources(ctx, src, columns, nullptr, out, stats, carry);
  // string columns hold references into the file images, which die with `src`: callers that handle strings keep their own
  // SourceSet (hs_create_index, hs_verify_index)
  for (const DevColumn& c : out->cols)
    if (c.type == HS_TYPE_STRING)
      fail(HS_EUNSUPPORTED, "column '%s' is a string / binary column; the index scans and joins of the GPU path do not read those yet",
           c.name.c_str());
}

// ---- dictionary helpers shared by the decoder (late-materialised columns) and the page encoder -------------------------

// Column order first, raw bits second: values that compare equal (-0.0 / 0.0, NaN payloads) still get one fixed order, so
// every rank -- and every run -- numbers the same dictionary the same way.
static void sort_dictionary(std::vector<uint64_t>& values, int type) {
  std::sort(values.begin(), values.end(), [type](uint64_t a, uint64_t b) {
    const uint64_t ea = sort_encode(type, a), eb = sort_encode(type, b);
    return ea != eb ? ea < eb : a < b;
  });
}

// The distinct values of a device hash set (state[0] of them, plus the empty marker when state[2] is set), sorted in the
// column's order.  Synchronises the stream.
static std::vector<uint64_t> sorted_dictionary(hs_ctx* ctx, const unsigned long long* keys, const uint32_t* state, int type) {
  const uint32_t ntab = state[0];
  Buf<unsigned long long> d_list(ctx, std::max<uint32_t>(1, ntab) + 1);
  Buf<uint32_t> d_counter(ctx, 1);
  fill_bytes(ctx, d_counter.get(), 0, 4);
  launch_dict_collect(ctx, keys, kDictCapacity, d_list.get(), d_counter.get());
  std::vector<uint64_t> values(ntab);
  if (ntab) copy_d2h(ctx, values.data(), d_list.get(), 8 * (size_t)ntab);
  sync_stream(ctx);
  if (state[2]) values.push_back(~0ull);
  sort_dictionary(values, type);
  return values;
}

// parquet-mr's choice, restated: dictionary-encode when the bit-packed codes plus one dictionary page per output file are
// clearly smaller than the PLAIN values
static bool dictionary_pays_off(uint32_t ndict, uint32_t bw, int width, int64_t total_rows, int nseg) {
  const double plain_bytes = (double)total_rows * width;
  const double dict_bytes = (double)total_rows * bw / 8.0 + (double)ndict * width * std::max(1, nseg);
  return ndict > 0 && ndict <= kMaxDictEntries && dict_bytes <= 0.9 * plain_bytes;
}

static uint32_t bits_for(uint32_t ndict) {
  uint32_t bw = 1;
  while ((1u << bw) < ndict) bw++;
  return bw;
}

// value -> code look-up table (open addressing, linear probing, 16-byte {key lo, key hi, code, 0} entries), built on the
// host (<= 65536 inserts) and sized to the dictionary (load <= 0.5) so that it stays resident in L1 while rows stream
// through it.  The empty marker ~0 cannot be stored: *empty_index receives its code instead.
static void upload_lookup_table(hs_ctx* ctx, const std::vector<uint64_t>& values, Buf<uint8_t>* entries, uint32_t* mask,
                                uint32_t* empty_index) {
  const uint32_t ndict = (uint32_t)values.size();
  uint32_t cap = 256;
  while (cap < 2 * ndict) cap <<= 1;
  *mask = cap - 1;
  *empty_index = 0;
  std::vector<uint32_t> tab((size_t)cap * 4, 0u);
  for (uint32_t s2 = 0; s2 < cap; s2++) tab[(size_t)s2 * 4] = tab[(size_t)s2 * 4 + 1] = 0xffffffffu;
  for (uint32_t i = 0; i < ndict; i++) {
    const uint64_t v = values[i];
    if (v == ~0ull) {
      *empty_index = i;
      continue;
    }
    uint32_t h = dict_hash_u64(v) & *mask;
    while (tab[(size_t)h * 4] != 0xffffffffu || tab[(size_t)h * 4 + 1] != 0xffffffffu) h = (h + 1) & *mask;
    tab[(size_t)h * 4] = (uint32_t)v;
    tab[(size_t)h * 4 + 1] = (uint32_t)(v >> 32);
    tab[(size_t)h * 4 + 2] = i;
  }
  entries->alloc(ctx, (size_t)cap * 16);
  copy_h2d(ctx, entries->get(), tab.data(), (size_t)cap * 16);  // snapshot: tab may go out of scope
}

// out[dst_off .. dst_off + len) = src[0 .. len): gathers the tails / footers of device-resident file images into one
// buffer so that they reach the host with a single copy.  One CTA per span.
struct SpanCopy {
  const uint8_t* src;
  uint64_t dst_off;
  uint32_t len;
};
__global__ void k_gather_spans(const SpanCopy* __restrict__ spans, uint8_t* __restrict__ out) {
  const SpanCopy sp = spans[blockIdx.x];
  for (uint32_t i = threadIdx.x; i < sp.len; i += blockDim.x) out[sp.dst_off + i] = sp.src[i];
}

void open_sources(hs_ctx* ctx, const hs_source_file* files, int n_files, SourceSet* set, hs_stats* stats) {
  StageTimer t_h2d(ctx);
  set->n_files = n_files;
  std::vector<FileImage>& imgs = set->impl->imgs;
  Buf<uint8_t>& d_images = set->impl->d_images;
  imgs.assign(n_files, FileImage());
  // ---- sizes + device arena for host-supplied images --------------------------------------------------------
  std::vector<uint64_t> sizes(n_files), dev_off(n_files, 0);
  uint64_t arena_bytes = 0;
  for (int f = 0; f < n_files; f++) {
    const hs_source_file& sf = files[f];
    if (sf.data == nullptr) {
      if (!sf.path) fail(HS_EINVAL, "source file %d has neither data nor path", f);
      struct stat st;
      if (stat(sf.path, &st) != 0) fail(HS_EIO, "cannot stat %s", sf.path);
      sizes[f] = (uint64_t)st.st_size;
      imgs[f].what = sf.path;
    } else {
      sizes[f] = sf.size;
      imgs[f].what = sf.path ? sf.path : ("<memory file " + std::to_string(f) + ">");
    }
    if (sizes[f] < 12) fail(HS_EFORMAT, "%s: too small to be a Parquet file", imgs[f].what.c_str());
    imgs[f].size = sizes[f];
    if (!(sf.data && sf.on_device)) {
      dev_off[f] = arena_bytes;
      arena_bytes += round_up(sizes[f], 16) + 16;
    }
  }
  if (arena_bytes) d_images.alloc(ctx, arena_bytes);
  // ---- H2D + footers -----------------------------------------------------------------------------------------
  t_h2d.start();
  std::vector<Buf<uint8_t>> staging;  // pinned buffers for path-based files; kept until the copies have completed
  // device-resident images: fetch all 8-byte tails into ONE pinned buffer with one sync, then all footers likewise
  // (a D2H copy into pageable memory blocks the host once per copy, i.e. once per file)
  std::vector<uint64_t> footer_off(n_files + 1, 0);
  Buf<uint8_t> pinned_tails, pinned_footers;
  bool any_dev = false;
  for (int f = 0; f < n_files; f++) any_dev = any_dev || (files[f].data && files[f].on_device);
  // images staged by hs_stage_sources may still be on their way: everything this call enqueues waits for THEIR copies (and
  // only theirs: the images of the next call are being staged at this very moment); their footers were parsed from host
  // memory when they were staged
  std::vector<std::shared_ptr<pq::FileMeta>> cached(n_files);
  bool fetch_footers = false;
  {
    cudaEvent_t last_ev = nullptr;
    for (int f = 0; f < n_files; f++) {
      if (!(files[f].data && files[f].on_device)) continue;
      auto it = ctx->staged.find(files[f].data);
      if (it == ctx->staged.end()) {
        fetch_footers = true;
        continue;
      }
      cached[f] = it->second.meta;
      if (it->second.ready != last_ev) {
        last_ev = it->second.ready;
        HS_CUDA(cudaStreamWaitEvent(ctx->stream, last_ev, 0));
      }
    }
  }
  if (any_dev && !fetch_footers) {
    for (int f = 0; f < n_files; f++)
      if (cached[f]) {
        if (((uintptr_t)files[f].data & 15) != 0) fail(HS_EINVAL, "%s: device images must be 16-byte aligned", imgs[f].what.c_str());
        imgs[f].dev = (const uint8_t*)files[f].data;
      }
  }
  if (any_dev && fetch_footers) {
    // one gather kernel + one copy per round instead of one small copy per file (each costs ~4.5 us of launch overhead)
    pinned_tails.alloc(ctx, (size_t)n_files * 8, /*pinned=*/true);
    Buf<SpanCopy> h_spans(ctx, n_files, /*pinned=*/true);
    Buf<SpanCopy> d_spans(ctx, n_files);
    Buf<uint8_t> d_gathered(ctx, (size_t)n_files * 8);
    int nspans = 0;
    for (int f = 0; f < n_files; f++) {
      const hs_source_file& sf = files[f];
      if (!(sf.data && sf.on_device)) continue;
      if (((uintptr_t)sf.data & 15) != 0) fail(HS_EINVAL, "%s: device images must be 16-byte aligned", imgs[f].what.c_str());
      imgs[f].dev = (const uint8_t*)sf.data;
      h_spans.get()[nspans++] = SpanCopy{imgs[f].dev + sizes[f] - 8, (uint64_t)f * 8, 8};
    }
    copy_h2d(ctx, d_spans.get(), h_spans.get(), sizeof(SpanCopy) * nspans);
    k_gather_spans<<<nspans, 128, 0, ctx->stream>>>(d_spans.get(), d_gathered.get());
    HS_LAUNCH_CHECK(ctx);
    copy_d2h(ctx, pinned_tails.get(), d_gathered.get(), (size_t)n_files * 8);
    sync_stream(ctx);
    for (int f = 0; f < n_files; f++) {
      const hs_source_file& sf = files[f];
      footer_off[f + 1] = footer_off[f];
      if (!(sf.data && sf.on_device)) continue;
      uint32_t flen;
      memcpy(&flen, pinned_tails.get() + (size_t)f * 8, 4);
      if (memcmp(pinned_tails.get() + (size_t)f * 8 + 4, "PAR1", 4) != 0 || (uint64_t)flen + 12 > sizes[f])
        fail(HS_EFORMAT, "%s: not a Parquet file", imgs[f].what.c_str());
      footer_off[f + 1] = footer_off[f] + flen;
    }
    pinned_footers.alloc(ctx, std::max<uint64_t>(1, footer_off[n_files]), /*pinned=*/true);
    Buf<uint8_t> d_footers(ctx, std::max<uint64_t>(1, footer_off[n_files]));
    nspans = 0;
    for (int f = 0; f < n_files; f++) {
      const uint64_t flen = footer_off[f + 1] - footer_off[f];
      if (flen) h_spans.get()[nspans++] = SpanCopy{imgs[f].dev + sizes[f] - 8 - flen, footer_off[f], (uint32_t)flen};
    }
    if (nspans) {
      copy_h2d(ctx, d_spans.get(), h_spans.get(), sizeof(SpanCopy) * nspans);
      k_gather_spans<<<nspans, 128, 0, ctx->stream>>>(d_spans.get(), d_footers.get());
      HS_LAUNCH_CHECK(ctx);
      copy_d2h(ctx, pinned_footers.get(), d_footers.get(), footer_off[n_files]);
    }
    sync_stream(ctx);
  }
  for (int f = 0; f < n_files; f++) {
    const hs_source_file& sf = files[f];
    const uint8_t* host = nullptr;
    if (sf.data && sf.on_device) {
      if (!fetch_footers) imgs[f].meta = *cached[f];
      else
        imgs[f].meta = pq::parse_footer_bytes(pinned_footers.get() + footer_off[f], (uint32_t)(footer_off[f + 1] - footer_off[f]),
                                              imgs[f].what.c_str());
    } else {
      if (sf.data) host = (const uint8_t*)sf.data;
      else {
        staging.emplace_back(ctx, sizes[f], /*pinned=*/true);
        read_whole_file(sf.path, staging.back().get(), sizes[f]);
        host = staging.back().get();
      }
      imgs[f].meta = pq::parse_footer(host, sizes[f], imgs[f].what.c_str());
      imgs[f].dev = d_images.get() + dev_off[f];
      copy_h2d(ctx, d_images.get() + dev_off[f], host, sizes[f]);
    }
    stats->bytes_in += (int64_t)sizes[f];
  }
  t_h2d.stop();
  sync_stream(ctx);  // pinned staging buffers and caller memory are free to go
  stats->ms_h2d += t_h2d.ms();
}

// The outcome of the late-materialisation agreement for one gathered message: which columns travel as codes, their merged
// dictionaries and the device look-up tables.  Builds over the same sources (a refresh cycle, a benchmark loop) gather the
// same message again; comparing the message costs far less host time than merging every rank's dictionaries and
// rebuilding the tables.  The key is the message itself (content, not identity): nothing stale can match.
struct DecodeCache {
  struct Column {
    int col = -1;
    std::vector<uint64_t> values;
    uint32_t bw = 0, mask = 0, empty_index = 0;
    Buf<uint8_t> table;
  };
  std::vector<uint64_t> message;
  int num_segments = 0, first_col = 0;
  int64_t total_rows = 0;
  std::vector<Column> carried;
};
static void free_decode_cache(void* p) { delete static_cast<DecodeCache*>(p); }

DevColumn source_column_type(hs_ctx* ctx, const hs_source_file& sf, const std::string& name) {
  const std::string what = sf.path ? sf.path : "source file";
  uint64_t size = sf.size;
  std::vector<uint8_t> tail(8), footer;
  auto read_at = [&](uint64_t off, uint8_t* dst, uint64_t n) {
    if (sf.data && sf.on_device) HS_CUDA(cudaMemcpy(dst, (const uint8_t*)sf.data + off, n, cudaMemcpyDeviceToHost));
    else if (sf.data) memcpy(dst, (const uint8_t*)sf.data + off, n);
    else {
      int fd = open(sf.path, O_RDONLY);
      if (fd < 0) fail(HS_EIO, "cannot open %s", sf.path);
      const ssize_t r = pread(fd, dst, n, (off_t)off);
      close(fd);
      if (r != (ssize_t)n) fail(HS_EIO, "short read on %s", sf.path);
    }
  };
  if (!sf.data) {
    if (!sf.path) fail(HS_EINVAL, "source file without path or data");
    struct stat stt;
    if (stat(sf.path, &stt) != 0) fail(HS_EIO, "cannot stat %s", sf.path);
    size = (uint64_t)stt.st_size;
  }
  if (size < 12) fail(HS_EFORMAT, "%s: not a Parquet file", what.c_str());
  read_at(size - 8, tail.data(), 8);
  uint32_t flen;
  memcpy(&flen, tail.data(), 4);
  if (memcmp(tail.data() + 4, "PAR1", 4) != 0 || (uint64_t)flen + 12 > size) fail(HS_EFORMAT, "%s: not a Parquet file", what.c_str());
  footer.resize(flen);
  read_at(size - 8 - flen, footer.data(), flen);
  const pq::FileMeta fm = pq::parse_footer_bytes(footer.data(), flen, what.c_str());
  const int idx = find_column(fm, name);
  if (idx < 0) fail(HS_EINVAL, "%s: column '%s' not found", what.c_str(), name.c_str());
  const SourceType st = source_type_of(fm.columns[idx], what.c_str());
  DevColumn dc;
  dc.name = name;
  dc.type = st.type;
  dc.width = type_width(st.type);
  dc.schema = st.schema;
  dc.schema.name = name;
  return dc;
}

void decode_sources(hs_ctx* ctx, SourceSet& set, const std::vector<std::string>& columns, const FileWindows* file_windows,
                    Table* out, hs_stats* stats, const CarryOptions* carry) {
  StageTimer t_plan(ctx), t_dec(ctx);
  const int n_files = set.n_files;
  std::vector<FileImage>& imgs = set.impl->imgs;
  // ---- resolve columns, build chunk descriptors -----------------------------------------------------------------
  t_plan.start();
  const int ncols = (int)columns.size();
  out->cols.clear();
  out->cols.resize(ncols);
  out->file_row_begin.assign(n_files + 1, 0);
  std::vector<ChunkDesc> chunks;
  bool any_compressed = false;
  std::vector<bool> col_optional(ncols, false);
  std::vector<bool> col_converted(ncols, false);  // some chunk's values are converted (ValueConv): the value path only
  int64_t nrows = 0;
  for (int f = 0; f < n_files; f++) {
    const pq::FileMeta& fm = imgs[f].meta;
    const char* what = imgs[f].what.c_str();
    std::vector<int> idx(ncols), conv(ncols);
    for (int c = 0; c < ncols; c++) {
      idx[c] = find_column(fm, columns[c]);
      if (idx[c] < 0) fail(HS_EINVAL, "%s: column '%s' not found", what, columns[c].c_str());
      const pq::SchemaColumn& sc = fm.columns[idx[c]];
      if (fm.nested) fail(HS_EUNSUPPORTED, "%s: nested schemas are not handled by the GPU path", what);
      const SourceType st = source_type_of(sc, what);
      DevColumn& dc = out->cols[c];
      if (dc.type < 0) {
        dc.name = columns[c];
        dc.type = st.type;
        dc.width = type_width(st.type);
        dc.schema = st.schema;
        dc.schema.name = columns[c];
      } else if (dc.type != st.type ||
                 ((is_decimal(dc.schema) || is_decimal(st.schema) || is_timestamp(dc.schema) || is_timestamp(st.schema)) &&
                  pq::spark_type_name(dc.schema) != pq::spark_type_name(st.schema))) {
        fail(HS_EINVAL, "%s: column '%s' changes type between source files", what, columns[c].c_str());
      }
      conv[c] = st.conv;
      col_converted[c] = col_converted[c] || st.conv != CONV_NONE;
      if (sc.repetition == pq::OPTIONAL) col_optional[c] = true;
    }
    out->file_row_begin[f] = nrows;
    for (const pq::RowGroupMeta& rg : fm.row_groups) {
      if (rg.num_rows == 0) continue;  // writers emit an empty row group for an empty table
      for (int c = 0; c < ncols; c++) {
        const pq::ColumnChunkMeta& cm = rg.columns[idx[c]];
        if (cm.codec != pq::UNCOMPRESSED && cm.codec != pq::SNAPPY && cm.codec != pq::GZIP && cm.codec != pq::LZ4 &&
            cm.codec != pq::LZ4_RAW)
          fail(HS_EUNSUPPORTED,
               "%s: column '%s' uses compression codec %d; the GPU path reads UNCOMPRESSED, SNAPPY, GZIP, LZ4 and LZ4_RAW pages",
               what, columns[c].c_str(), cm.codec);
        any_compressed = any_compressed || cm.codec != pq::UNCOMPRESSED;
        if (cm.num_values != rg.num_rows)
          fail(HS_EFORMAT, "%s: column '%s' has %lld values for %lld rows", what, columns[c].c_str(), (long long)cm.num_values,
               (long long)rg.num_rows);
        const int64_t start = cm.start();
        if (start < 4 || (uint64_t)(start + cm.total_compressed_size) > imgs[f].size)
          fail(HS_EFORMAT, "%s: column chunk of '%s' lies outside the file", what, columns[c].c_str());
        ChunkDesc cd;
        cd.data = imgs[f].dev + start;
        cd.size = (uint64_t)cm.total_compressed_size;
        cd.num_values = cm.num_values;
        cd.row_base = nrows;
        cd.col = c;
        cd.phys_type = fm.columns[idx[c]].type;
        cd.max_def = fm.columns[idx[c]].repetition == pq::OPTIONAL ? 1 : 0;
        cd.file_index = f;
        cd.codec = cm.codec;
        cd.conv = conv[c];
        cd.type_length = fm.columns[idx[c]].type_length;
        cd.pad = 0;
        chunks.push_back(cd);
      }
      nrows += rg.num_rows;
    }
  }
  out->file_row_begin[n_files] = nrows;
  out->nrows = nrows;
  if (nrows >= (1ll << 32)) fail(HS_EUNSUPPORTED, "more than 2^32-1 rows per GPU per call");
  stats->rows_in += nrows;

  std::vector<ColumnOut> h_cols(ncols);
  // destinations are allocated once the late-materialised columns are known (they get 2-byte codes, not values)
  auto alloc_destinations = [&]() {
    for (int c = 0; c < ncols; c++) {
      DevColumn& dc = out->cols[c];
      if (dc.carried || dc.zero_copy) continue;
      dc.data.alloc(ctx, (size_t)nrows * dc.width + 16);
      if (col_optional[c]) {
        dc.valid.alloc(ctx, (size_t)nrows + 16);
        fill_bytes(ctx, dc.valid.get(), 1, (size_t)nrows + 16);
      }
      h_cols[c] = ColumnOut{dc.data.get(), col_optional[c] ? dc.valid.get() : nullptr, dc.width, dc.type, nullptr, 0u, 0u, 0, 0};
    }
  };
  const int n_chunks = (int)chunks.size();
  t_plan.stop();
  const bool want_carry = carry && carry->first_col >= 0 && !file_windows;
  // (with several GPUs a rank without rows still takes part in the agreement on the late-materialised columns below)
  if ((n_chunks == 0 || nrows == 0) && !(want_carry && ctx->world > 1)) {
    alloc_destinations();
    sync_stream(ctx);
    return;
  }
  // ---- page walk -----------------------------------------------------------------------------------------
  t_dec.start();
  Buf<ChunkDesc> d_chunks(ctx, std::max(1, n_chunks));
  Buf<int32_t> d_counts(ctx, std::max(1, n_chunks));
  Buf<int64_t> d_offsets(ctx, std::max(1, n_chunks));
  Buf<uint32_t> d_flags(ctx, 1 + ncols);  // [0] error word, [1..] per-column has-nulls
  Buf<ColumnOut> d_cols(ctx, ncols);
  copy_h2d(ctx, d_chunks.get(), chunks.data(), sizeof(ChunkDesc) * n_chunks);
  fill_bytes(ctx, d_flags.get(), 0, sizeof(uint32_t) * (1 + ncols));
  launch_walk_pages(ctx, d_chunks.get(), n_chunks, d_counts.get(), nullptr, nullptr, d_flags.get(), 0);
  std::vector<int32_t> counts(n_chunks);
  copy_d2h(ctx, counts.data(), d_counts.get(), sizeof(int32_t) * n_chunks);
  sync_stream(ctx);
  std::vector<int64_t> offsets(n_chunks);
  int64_t n_pages = 0;
  for (int i = 0; i < n_chunks; i++) {
    offsets[i] = n_pages;
    n_pages += counts[i];
  }
  Buf<PageDesc> d_pages(ctx, std::max<int64_t>(1, n_pages));
  copy_h2d(ctx, d_offsets.get(), offsets.data(), sizeof(int64_t) * n_chunks);
  launch_walk_pages(ctx, d_chunks.get(), n_chunks, d_counts.get(), d_offsets.get(), d_pages.get(), d_flags.get(), 1);
  // a chunk whose page headers do not add up must not reach the decoder (its pages would write outside the columns): the
  // error word is read back with the next results the host needs anyway, and checked before any page is decoded
  uint32_t walk_error = 0;
  bool walk_checked = false;
  copy_d2h(ctx, &walk_error, d_flags.get(), sizeof walk_error);
  auto check_walk = [&]() {
    if (walk_checked) return;
    walk_checked = true;
    if (walk_error) {
      const uint32_t code = walk_error >> 24, detail = walk_error & 0xffffffu;
      fail(code == DERR_COMPRESSED ? HS_EUNSUPPORTED : HS_EFORMAT, "Parquet page walk failed: %s (column chunk %u)",
           decode_error_text(code), detail);
    }
  };
  // ---- compressed pages (and dictionary pages) are decompressed into a scratch buffer and the pages repointed at it ----
  if (any_compressed && n_pages > 0) {
    std::vector<PageDesc> h_pages((size_t)n_pages);
    copy_d2h(ctx, h_pages.data(), d_pages.get(), sizeof(PageDesc) * (size_t)n_pages);
    sync_stream(ctx);
    check_walk();
    decompress_pages(ctx, h_pages, d_pages.get(), &set.impl->d_scratch, d_flags.get());
  }
  // ---- strings: the dictionary pages of BYTE_ARRAY columns become tables of references --------------------------------------
  Buf<uint64_t> d_string_dicts;
  bool any_string = false;
  for (int c = 0; c < ncols; c++) any_string = any_string || out->cols[c].type == HS_TYPE_STRING;
  out->has_strings = any_string;
  if (any_string && n_pages > 0) {
    std::vector<PageDesc> h_pages((size_t)n_pages);
    copy_d2h(ctx, h_pages.data(), d_pages.get(), sizeof(PageDesc) * (size_t)n_pages);
    sync_stream(ctx);
    check_walk();
    std::map<const uint8_t*, size_t> job_of;  // dictionary page -> job
    std::vector<StringDictJob> jobs;
    std::vector<size_t> job_off;
    size_t total = 0;
    for (PageDesc& pg : h_pages) {
      if (pg.phys_type != pq::BYTE_ARRAY || !pg.dict || pg.encoding == pq::ENC_PLAIN) continue;
      auto it = job_of.find(pg.dict);
      if (it == job_of.end()) {
        it = job_of.emplace(pg.dict, jobs.size()).first;
        jobs.push_back(StringDictJob{pg.dict, nullptr, pg.dict_size, pg.dict_count});
        job_off.push_back(total);
        total += (size_t)std::max(0, pg.dict_count);
      }
    }
    if (!jobs.empty()) {
      d_string_dicts.alloc(ctx, std::max<size_t>(1, total));
      for (size_t j = 0; j < jobs.size(); j++) jobs[j].refs = d_string_dicts.get() + job_off[j];
      for (PageDesc& pg : h_pages) {
        if (pg.phys_type != pq::BYTE_ARRAY || !pg.dict || pg.encoding == pq::ENC_PLAIN) continue;
        const StringDictJob& job = jobs[job_of[pg.dict]];
        pg.dict = (const uint8_t*)job.refs;  // decodes as a dictionary of 8-byte values from here on
        pg.dict_size = job.count * 8;
      }
      Buf<StringDictJob> d_jobs(ctx, jobs.size());
      copy_h2d(ctx, d_jobs.get(), jobs.data(), sizeof(StringDictJob) * jobs.size());
      launch_build_string_dicts(ctx, d_jobs.get(), (int64_t)jobs.size(), d_flags.get());
      copy_h2d(ctx, d_pages.get(), h_pages.data(), sizeof(PageDesc) * (size_t)n_pages);
      if (sizeof(PageDesc) * (size_t)n_pages > (16u << 20)) sync_stream(ctx);  // too big for a snapshot: keep h_pages alive
    }
  }
  // ---- late-materialised dictionary columns --------------------------------------------------------------------------
  // A candidate column whose every page is dictionary-encoded and free of nulls, and whose chunk dictionaries unite to a
  // dictionary that pays off, is decoded to 16-bit codes of that dictionary: its values are never written to HBM, the
  // partition moves 2 bytes per row instead of 4 or 8, and the page encoder finds its codes ready-made.  On several GPUs
  // the ranks agree on the columns and on one dictionary per column (unions all-gathered and merged), so that codes mean
  // the same everywhere and can cross NVLink in place of the values.
  //
  // One device round and ONE all-gather: the page classification and, speculatively, the dictionary union of every
  // candidate column are computed back to back and fetched with a single synchronisation; each rank then contributes one
  // fixed-size message (flags, row count, per candidate its type and up to kAgreeCap dictionary values) and every rank
  // derives the same decisions from the gathered messages.  (The first version took a host round trip per step and per
  // candidate: 2 + 2 x candidates all-gathers, each with its own synchronisation -- a quarter of an 8-GPU build.)
  const bool want_zc = carry && carry->zc_tile_rows > 0 && !file_windows && n_pages > 0 && nrows > 0;
  std::vector<uint32_t> local_cls(ncols, 0u);  // classification of this rank's own pages, per column
  constexpr uint32_t kAgreeCap = 8192;  // dictionary values per candidate carried by the message (larger unions: no carry)
  constexpr int kMaxSpec = 6;           // candidates examined (kMaxCarried of them can be carried)
  std::vector<int> spec;                // candidate columns, the same list on every rank
  if (want_carry)
    for (int c = carry->first_col; c < ncols && (int)spec.size() < kMaxSpec; c++) spec.push_back(c);
  const int nspec = (int)spec.size();
  std::vector<uint32_t> spec_state(4 * (size_t)std::max(1, nspec), 0u), spec_count(std::max(1, nspec), 0u);
  std::vector<uint64_t> spec_vals((size_t)std::max(1, nspec) * kAgreeCap);
  if ((want_carry || want_zc) && n_pages > 0) {
    Buf<uint32_t> d_class(ctx, ncols);
    fill_bytes(ctx, d_class.get(), 0, 4 * (size_t)ncols);
    launch_classify_pages(ctx, d_pages.get(), n_pages, d_class.get(), want_zc ? carry->zc_tile_rows : 0);
    copy_d2h(ctx, local_cls.data(), d_class.get(), 4 * (size_t)ncols);
    Buf<uint32_t> d_states(ctx, 4 * (size_t)std::max(1, nspec)), d_cnt(ctx, std::max(1, nspec));
    Buf<unsigned long long> d_vals(ctx, (size_t)std::max(1, nspec) * kAgreeCap);
    std::vector<Buf<unsigned long long>> sets(nspec);
    if (nspec) {
      fill_bytes(ctx, d_states.get(), 0, 16 * (size_t)nspec);
      fill_bytes(ctx, d_cnt.get(), 0, 4 * (size_t)nspec);
      for (int i = 0; i < nspec; i++) {
        const DevColumn& dc = out->cols[spec[i]];
        if ((dc.width != 4 && dc.width != 8) || dc.type == HS_TYPE_STRING || col_converted[spec[i]]) continue;
        sets[i].alloc(ctx, kDictCapacity);
        fill_bytes(ctx, sets[i].get(), 0xFF, sizeof(unsigned long long) * kDictCapacity);
        launch_dict_build_from_pages(ctx, d_pages.get(), n_pages, spec[i], dc.width, sets[i].get(), kDictCapacity, kMaxDictEntries,
                                     d_states.get() + 4 * i);
        launch_dict_collect(ctx, sets[i].get(), kDictCapacity, d_vals.get() + (size_t)i * kAgreeCap, d_cnt.get() + i, kAgreeCap);
      }
      copy_d2h(ctx, spec_state.data(), d_states.get(), 16 * (size_t)nspec);
      copy_d2h(ctx, spec_count.data(), d_cnt.get(), 4 * (size_t)nspec);
      copy_d2h(ctx, spec_vals.data(), d_vals.get(), 8 * (size_t)nspec * kAgreeCap);
    }
    sync_stream(ctx);
  } else {
    sync_stream(ctx);
  }
  check_walk();
  if (want_carry) {
    const int W = ctx->world;
    // message: [ncols class flags][rows][per candidate: type, width, distinct count, overflow, holds ~0, values...]
    const size_t per_cand = 5 + kAgreeCap, words = (size_t)ncols + 1 + (size_t)nspec * per_cand;
    std::vector<uint64_t> mine(words, 0ull), all(words * W);
    for (int c = 0; c < ncols; c++) mine[c] = local_cls[c] & (PAGECLASS_NOT_DICT | PAGECLASS_MAYBE_NULLS);
    mine[ncols] = (uint64_t)nrows;
    for (int i = 0; i < nspec; i++) {
      const DevColumn& dc = out->cols[spec[i]];
      uint64_t* m = &mine[(size_t)ncols + 1 + (size_t)i * per_cand];
      m[0] = (uint64_t)(int64_t)dc.type;
      m[1] = dc.type == HS_TYPE_STRING ? 0ull : (uint64_t)dc.width;  // string references are not values: never carried
      m[2] = spec_state[4 * i];                                                    // distinct values in the set (excl. ~0)
      // overflow, or a converted column (its dictionary pages hold stored values, not the engine's): no carry for this column
      m[3] = (spec_state[4 * i + 1] || spec_count[i] > kAgreeCap || col_converted[spec[i]]) ? 1 : 0;
      m[4] = spec_state[4 * i + 2];                                                // the value ~0 occurs
      const uint32_t nv = std::min<uint32_t>(spec_count[i], kAgreeCap);
      for (uint32_t j = 0; j < nv; j++) m[5 + j] = spec_vals[(size_t)i * kAgreeCap + j];
      std::sort(m + 5, m + 5 + nv);  // the hash set yields them in no particular order: a canonical message can be cached
      m[2] = nv;
    }
    comm_allgather_host(ctx, mine.data(), 8 * words, all.data());
    DecodeCache* cache = static_cast<DecodeCache*>(ctx->decode_cache);
    const bool hit = cache && cache->num_segments == carry->num_segments && cache->first_col == carry->first_col &&
                     cache->message.size() == all.size() && memcmp(cache->message.data(), all.data(), 8 * all.size()) == 0;
    std::vector<uint32_t> cls(ncols, 0u);
    int64_t total_rows = 0;
    if (hit) {
      total_rows = cache->total_rows;
      for (DecodeCache::Column& cc : cache->carried) {
        DevColumn& dc = out->cols[cc.col];
        dc.carried = true;
        dc.dict_values = cc.values;
        dc.dict_bw = cc.bw;
        dc.codes.alloc(ctx, (size_t)std::max<int64_t>(1, nrows) + 16);
        h_cols[cc.col] = ColumnOut{dc.codes.get(), nullptr, dc.width, dc.type, cc.table.get(), cc.mask, cc.empty_index, 1, 0};
      }
    } else {
      for (int r = 0; r < W; r++) {
        const uint64_t* a = &all[(size_t)r * words];
        for (int c = 0; c < ncols; c++) cls[c] |= (uint32_t)a[c];
        total_rows += (int64_t)a[ncols];
      }
      if (!cache) {
        cache = new DecodeCache();
        ctx->decode_cache = cache;
        ctx->decode_cache_free = free_decode_cache;
      }
      cache->carried.clear();  // (the previous entry's tables were last read by kernels of an earlier, completed call)
      cache->message = all;
      cache->num_segments = carry->num_segments;
      cache->first_col = carry->first_col;
      cache->total_rows = total_rows;
    }
    out->global_rows = total_rows;
    int ncarried = 0;
    for (int i = 0; !hit && i < nspec && ncarried < kMaxCarried && total_rows > 0; i++) {
      const int c = spec[i];
      DevColumn& dc = out->cols[c];
      if (cls[c] != 0) continue;
      int type = -1, width = 0;
      bool overflow = false, has_empty = false;
      std::vector<uint64_t> values;
      for (int r = 0; r < W; r++) {
        const uint64_t* m = &all[(size_t)r * words + (size_t)ncols + 1 + (size_t)i * per_cand];
        if ((int64_t)m[0] >= 0) type = (int)(int64_t)m[0];
        width = std::max(width, (int)m[1]);
        overflow = overflow || m[3] != 0;
        has_empty = has_empty || m[4] != 0;
        values.insert(values.end(), m + 5, m + 5 + m[2]);
      }
      if (overflow || type < 0 || (width != 4 && width != 8)) continue;
      if (has_empty) values.push_back(~0ull);
      sort_dictionary(values, type);
      values.erase(std::unique(values.begin(), values.end()), values.end());
      const uint32_t bw = bits_for((uint32_t)values.size());
      if (!dictionary_pays_off((uint32_t)values.size(), bw, width, total_rows, carry->num_segments)) continue;
      cache->carried.emplace_back();
      DecodeCache::Column& cc = cache->carried.back();
      cc.col = c;
      cc.bw = bw;
      upload_lookup_table(ctx, values, &cc.table, &cc.mask, &cc.empty_index);
      cc.values = values;
      dc.carried = true;
      dc.dict_values = std::move(values);
      dc.dict_bw = bw;
      dc.codes.alloc(ctx, (size_t)std::max<int64_t>(1, nrows) + 16);
      h_cols[c] = ColumnOut{dc.codes.get(), nullptr, dc.width, dc.type, cc.table.get(), cc.mask, cc.empty_index, 1, 0};
      ncarried++;
    }
  }
  // ---- zero-copy PLAIN columns -------------------------------------------------------------------------------------
  // A column whose every page is PLAIN, stored, free of nulls, value-aligned and at least one partition tile long is not
  // decoded at all: the hash and partition kernels read its values where they lie (a local decision: it only changes where
  // this rank's kernels load from).  For table T that is k and v2: 32 of the 42 GB the decoder used to move per 1 B rows.
  Buf<ZcTile*> d_tile_src;
  if (want_zc) {
    std::vector<ZcTile*> h_tile_src(ncols, nullptr);
    const int64_t T = carry->zc_tile_rows;
    bool any = false;
    for (int c = 0; c < ncols; c++) {
      DevColumn& dc = out->cols[c];
      const bool candidate = c >= carry->zc_first_col || (c == 0 && carry->zc_key && (dc.type == HS_TYPE_INT32 || dc.type == HS_TYPE_INT64));
      if (!candidate || dc.carried || col_converted[c] || (dc.width != 4 && dc.width != 8)) continue;
      if (local_cls[c] & (PAGECLASS_NOT_IN_PLACE | PAGECLASS_MAYBE_NULLS)) continue;
      dc.zero_copy = true;
      dc.zc_tiles.alloc(ctx, (size_t)ceil_div(nrows, T));
      h_tile_src[c] = dc.zc_tiles.get();
      h_cols[c] = ColumnOut{nullptr, nullptr, dc.width, dc.type, nullptr, 0u, 0u, 0, 1};
      any = true;
    }
    if (any) {
      d_tile_src.alloc(ctx, ncols);
      copy_h2d(ctx, d_tile_src.get(), h_tile_src.data(), sizeof(ZcTile*) * ncols);
      launch_fill_zc_tiles(ctx, d_pages.get(), n_pages, d_tile_src.get(), (int)T, nrows);
    }
  }
  alloc_destinations();
  copy_h2d(ctx, d_cols.get(), h_cols.data(), sizeof(ColumnOut) * ncols);
  // ---- decode -----------------------------------------------------------------------------------------
  // optional per-file row windows (file-relative -> global): pages that intersect none of their file's windows are skipped
  Buf<int64_t> d_window, d_window_offsets;
  if (file_windows) {
    const FileWindows& fw = *file_windows;
    std::vector<int64_t> w(2 * std::max<size_t>(1, fw.windows.size()));
    for (int f = 0; f < n_files; f++)
      for (int64_t i = fw.offsets[f]; i < fw.offsets[f + 1]; i++) {
        w[2 * i] = out->file_row_begin[f] + fw.windows[i].first;
        w[2 * i + 1] = out->file_row_begin[f] + fw.windows[i].second;
      }
    d_window.alloc(ctx, w.size());
    d_window_offsets.alloc(ctx, n_files + 1);
    copy_h2d(ctx, d_window.get(), w.data(), 8 * w.size());
    copy_h2d(ctx, d_window_offsets.get(), fw.offsets.data(), 8 * ((size_t)n_files + 1));
    sync_stream(ctx);
  }
  launch_decode_pages(ctx, d_pages.get(), n_pages, d_cols.get(), d_flags.get() + 1, file_windows ? d_window.get() : nullptr,
                      d_window_offsets.get(), d_flags.get(),
                      std::find(col_converted.begin(), col_converted.end(), true) != col_converted.end());
  std::vector<uint32_t> flags(1 + ncols);
  copy_d2h(ctx, flags.data(), d_flags.get(), sizeof(uint32_t) * (1 + ncols));
  t_dec.stop();
  sync_stream(ctx);
  if (flags[0]) {
    const uint32_t code = flags[0] >> 24, detail = flags[0] & 0xffffffu;
    const int ecode = (code == DERR_COMPRESSED || code == DERR_UNSUPPORTED_ENCODING || code == DERR_UNSUPPORTED_TYPE ||
                       code == DERR_STRING_TOO_LONG || code == DERR_SPARK_RANGE)
                          ? HS_EUNSUPPORTED
                          : HS_EFORMAT;
    if (code == DERR_GZIP) fail(ecode, "Parquet decode failed: %s: %s", decode_error_text(code), gz::inflate_error_text(detail));
    if (code == DERR_LZ4) fail(ecode, "Parquet decode failed: %s: %s", decode_error_text(code), lz4::lz4_error_text(detail));
    if ((code == DERR_SPARK_RANGE || code == DERR_DECIMAL_WIDTH) && detail < (uint32_t)ncols)
      fail(ecode, "Parquet decode failed: column '%s' holds a %s", columns[detail].c_str(), decode_error_text(code));
    fail(ecode, "Parquet decode failed: %s (detail %u)", decode_error_text(code), detail);
  }
  for (int c = 0; c < ncols; c++) out->cols[c].has_nulls = (flags[1 + c] & 1u) != 0;
  // columns whose every page was dictionary-encoded: the union of the chunk dictionaries becomes the encoder's hash set
  if (!file_windows && ctx->world == 1) {
    std::vector<int> cand;
    Buf<uint32_t> d_states(ctx, 4 * (size_t)std::max(1, ncols));
    fill_bytes(ctx, d_states.get(), 0, 16 * (size_t)std::max(1, ncols));
    for (int c = 0; c < ncols; c++) {
      DevColumn& dc = out->cols[c];
      if (dc.carried || dc.zero_copy || dc.type == HS_TYPE_STRING || col_converted[c] || (flags[1 + c] & 2u) || (dc.width != 4 && dc.width != 8))
        continue;
      dc.dict_keys.alloc(ctx, kDictCapacity);
      fill_bytes(ctx, dc.dict_keys.get(), 0xFF, sizeof(unsigned long long) * kDictCapacity);
      launch_dict_build_from_pages(ctx, d_pages.get(), n_pages, c, dc.width, dc.dict_keys.get(), kDictCapacity, kMaxDictEntries,
                                   d_states.get() + 4 * c);
      cand.push_back(c);
    }
    if (!cand.empty()) {
      std::vector<uint32_t> h_states(4 * (size_t)ncols);
      copy_d2h(ctx, h_states.data(), d_states.get(), 16 * (size_t)ncols);
      sync_stream(ctx);
      for (int c : cand) {
        DevColumn& dc = out->cols[c];
        memcpy(dc.dict_state, &h_states[4 * c], 16);
        dc.dict_ready = dc.dict_state[1] == 0 && dc.dict_state[0] <= kMaxDictEntries;  // (the count can pass it unflagged)
        if (!dc.dict_ready) dc.dict_keys.release();
      }
    }
  }
  stats->ms_plan += t_plan.ms();
  stats->ms_decode += t_dec.ms();
}

// ---------------------------------------------------------------------------------------------------------------------

void index_rows(hs_ctx* ctx, Table& table, int nkeys, int num_buckets, IndexedRows* out, hs_stats* stats, bool defer_settle,
                const KeyPagesFn* key_pages) {
  const int64_t nrows = table.nrows;
  const int ncols = (int)table.cols.size();
  if (num_buckets < 1 || num_buckets > kMaxBuckets)
    fail(HS_EUNSUPPORTED, "numBuckets = %d; the GPU path handles 1..%d buckets", num_buckets, kMaxBuckets);
  if (nkeys < 1 || nkeys > ncols) fail(HS_EINVAL, "bad number of indexed columns");
  if (nrows >= (1ll << 32)) fail(HS_EUNSUPPORTED, "more than 2^32-1 rows per GPU per call");
  StageTimer t_hash(ctx), t_part(ctx);

  // ---- K2: bucket ids + histograms -----------------------------------------------------------------------------
  t_hash.start();
  std::vector<KeyColumn> h_keys(nkeys);
  for (int k = 0; k < nkeys; k++) {
    h_keys[k] = key_column_of(table.cols[k]);
  }
  Buf<unsigned long long> ghist(ctx, num_buckets);
  out->d_bucket_offsets.alloc(ctx, num_buckets + 1);
  fill_bytes(ctx, ghist.get(), 0, sizeof(unsigned long long) * num_buckets);
  Buf<unsigned long long> d_key_bits(ctx, 2);
  const unsigned long long init[2] = {0ull, ~0ull};
  copy_h2d(ctx, d_key_bits.get(), init, sizeof init);
  HashedRows hashed;
  hash_rows(ctx, h_keys.data(), nkeys, nrows, num_buckets, 0, false, ghist.get(), d_key_bits.get(), &hashed);
  copy_d2h(ctx, out->key_or_and, d_key_bits.get(), sizeof out->key_or_and);
  out->have_key_bits = true;  // valid after the stream synchronisation below
  launch_tile_offsets(ctx, hashed.tile_hist.get(), hashed.ntiles, num_buckets, ghist.get(),
                      (unsigned long long*)out->d_bucket_offsets.get());
  out->bucket_offsets.assign(num_buckets + 1, 0);
  copy_d2h(ctx, out->bucket_offsets.data(), out->d_bucket_offsets.get(), sizeof(uint64_t) * (num_buckets + 1));
  t_hash.stop();

  // ---- K3: stable partition -----------------------------------------------------------------------------------
  t_part.start();
  out->part.nrows = nrows;
  out->part.cols.clear();
  out->part.cols.resize(ncols);
  std::vector<PartColumn> h_pc;
  CodePackRound pack;
  memset(&pack, 0, sizeof pack);
  for (int c = 0; c < ncols; c++) {
    DevColumn& src = table.cols[c];
    DevColumn& dst = out->part.cols[c];
    dst.name = src.name;
    dst.type = src.type;
    dst.width = src.width;
    dst.schema = src.schema;
    dst.has_nulls = src.has_nulls;
    dst.dict_keys = std::move(src.dict_keys);
    memcpy(dst.dict_state, src.dict_state, sizeof dst.dict_state);
    dst.dict_ready = src.dict_ready;
    if (src.carried) {  // travels as a 16-bit code inside the row's code record
      if (c < nkeys || pack.n >= kMaxCarried) fail(HS_EINVAL, "column '%s' cannot be late-materialised here", src.name.c_str());
      dst.carried = true;
      dst.dict_values = std::move(src.dict_values);
      dst.dict_bw = src.dict_bw;
      dst.carry_slot = pack.n;
      pack.src[pack.n++] = src.codes.get();
      continue;
    }
    dst.data.alloc(ctx, (size_t)nrows * src.width + 16);
    h_pc.push_back(PartColumn{src.data.get(), dst.data.get(), src.width, 0, src.zero_copy ? src.zc_tiles.get() : nullptr});
    if (src.has_nulls) {
      dst.valid.alloc(ctx, (size_t)nrows + 16);
      h_pc.push_back(PartColumn{src.valid.get(), dst.valid.get(), 1, 0});
    }
  }
  if (pack.n > 0) {
    out->part.rec.alloc(ctx, (size_t)nrows * 8 + 16);
    pack.out = out->part.rec.get();
  }
  move_rows(ctx, hashed, h_pc.data(), (int)h_pc.size(), &pack);
  t_part.stop();
  if (defer_settle) launch_dictionary_probes(ctx, out->part, true, &out->probe);  // results ride on the synchronisation below
  sync_stream(ctx);  // h_pc is read by the async copy; bucket_offsets now valid on the host
  for (int c = 0; c < ncols; c++) {
    table.cols[c].data.release();
    table.cols[c].valid.release();
    table.cols[c].codes.release();
    table.cols[c].zc_tiles.release();
  }

  stats->ms_hash += t_hash.ms();
  stats->ms_partition += t_part.ms();
  sort_partitioned_rows(ctx, nkeys, num_buckets, out, stats, defer_settle, key_pages);
}

void sort_partitioned_rows(hs_ctx* ctx, int nkeys, int num_buckets, IndexedRows* out, hs_stats* stats, bool defer_settle,
                           const KeyPagesFn* key_pages) {
  auto t_sort = std::make_unique<StageTimer>(ctx);
  // ---- K4: segmented sort on the indexed columns (radix_sort.cu) -----------------------------------------------
  if (defer_settle && !out->probe) {
    // rows that arrived through the fused exchange: the probes need the peers' rows (i.e. the closing barrier), and their
    // results must be on the host before the sort is queued if the encoder is to plan while the GPU sorts -- one
    // synchronisation here (the ranks are in step anyway) buys the overlap
    launch_dictionary_probes(ctx, out->part, true, &out->probe);
    if (out->probe) sync_stream(ctx);
  }
  t_sort->start();
  build_sort_plan(ctx, out->bucket_offsets.data(), num_buckets, &out->plan);
  std::vector<KeyColumn> keys(nkeys);
  for (int k = 0; k < nkeys; k++) keys[k] = key_column_of(out->part.cols[k]);
  sort_rows(ctx, &out->plan, keys.data(), nkeys, out->have_key_bits ? out->key_or_and : nullptr, defer_settle, &out->sorted,
            key_pages);
  t_sort->stop();
  if (out->sorted.queued) {  // no synchronisation here: the stage timers are read in settle_sort
    out->pending_timers.push_back(IndexedRows::DeferredTimer{std::move(t_sort), &hs_stats::ms_sort});
    return;
  }
  sync_stream(ctx);
  stats->ms_sort += t_sort->ms();
  for (auto& d : out->pending_timers) stats->*(d.field) += d.t->ms();
  out->pending_timers.clear();
}

bool settle_sort(hs_ctx* ctx, IndexedRows* out, hs_stats* stats) {
  StageTimer t(ctx);
  t.start();
  const bool again = settle_sorted_rows(ctx, &out->plan, &out->sorted);
  t.stop();
  if (again) {
    sync_stream(ctx);
    stats->ms_sort += t.ms();
  }
  for (auto& d : out->pending_timers) stats->*(d.field) += d.t->ms();
  out->pending_timers.clear();
  return again;
}

// see DictProbe
void launch_dictionary_probes(hs_ctx* ctx, const Table& part, bool use_dictionary, std::unique_ptr<DictProbe>* out) {
  out->reset();
  const int ncols = (int)part.cols.size();
  if (!use_dictionary || part.nrows == 0) return;
  auto pr = std::make_unique<DictProbe>();
  pr->mini = std::min<int64_t>(part.nrows, 1 << 14);
  pr->d_states.alloc(ctx, 4 * (size_t)ncols);
  pr->h_states.assign(4 * (size_t)ncols, 0u);
  pr->keys.resize(ncols);
  fill_bytes(ctx, pr->d_states.get(), 0, 16 * (size_t)ncols);
  bool any = false;
  for (int c = 0; c < ncols; c++) {
    const DevColumn& dc = part.cols[c];
    if (dc.has_nulls || dc.carried || dc.type == HS_TYPE_STRING || (dc.dict_ready && dc.dict_keys)) continue;
    if (dc.width != 4 && dc.width != 8) continue;
    pr->keys[c].alloc(ctx, kDictCapacity);
    fill_bytes(ctx, pr->keys[c].get(), 0xFF, sizeof(unsigned long long) * kDictCapacity);
    launch_dict_build(ctx, dc.data.get(), dc.width, 0, pr->mini, pr->keys[c].get(), kDictCapacity, kMaxDictEntries,
                      pr->d_states.get() + 4 * c);
    copy_d2h(ctx, &pr->h_states[4 * (size_t)c], pr->d_states.get() + 4 * c, 16);
    any = true;
  }
  if (!any) return;
  pr->queued_at = ctx->sync_count;
  *out = std::move(pr);
}

// ---------------------------------------------------------------------------------------------------------------------

namespace {

struct ColDict {
  bool use = false;
  uint32_t bw = 0, ndict = 0, empty_index = 0, mask = 0;
  Buf<unsigned long long> keys;       // owned when the set was built here
  const unsigned long long* keys_ptr = nullptr;  // the hash set in use (own or the column's ready-made one)
  Buf<uint8_t> entries;               // value -> code look-up table, 16-byte entries (upload_lookup_table)
  size_t skel_off = 0, skel_len = 0;  // [dictionary page header][PLAIN values] inside the skeleton
  std::vector<uint64_t> values;       // sorted dictionary (raw bits)
};
// every page of every file, in file order (needed only when the pages are compressed afterwards)
struct PagePlan {
  uint64_t hdr_off;   // arena offset of the page header
  uint32_t hdr_len;   // Thrift header bytes
  uint32_t body_len;  // page bytes behind the header
  int32_t page_type;  // what the header says: pq::PageType, the number of values and their pq::Encoding
  int32_t num_values, encoding;
};
struct FilePlan {
  int seg = 0;
  int64_t rows = 0;
  std::vector<pq::OutRowGroup> rgs;
  std::vector<std::pair<size_t, size_t>> chunk_pages;  // per (row group, column): first page, page count
};
// Appends the end of a file to `skeleton`: the footer, its length and the magic.  `at` is the arena offset the footer goes
// to and seg_begin the sorted position of the file's first row: the min / max placeholders of the sorted key in the footer
// become one StatPatch per row group.
void append_file_end(const std::vector<pq::SchemaColumn>& schema, const std::vector<pq::OutRowGroup>& rgs, int64_t rows,
                     const std::string& schema_json, uint64_t seg_begin, uint64_t at, std::vector<uint8_t>& skeleton,
                     std::vector<StatPatch>& patches) {
  std::vector<pq::StatSlot> slots;
  std::vector<uint8_t> footer = pq::write_footer(schema, rgs, rows, schema_json, &slots);
  for (const pq::StatSlot& sl : slots) {
    StatPatch sp;
    int64_t row0 = 0;
    for (int g = 0; g < sl.row_group; g++) row0 += rgs[g].num_rows;
    sp.first_pos = seg_begin + (uint64_t)row0;
    sp.last_pos = sp.first_pos + (uint64_t)rgs[sl.row_group].num_rows - 1;
    for (int j = 0; j < 2; j++) {
      sp.min_off[j] = at + sl.min_off[j];
      sp.max_off[j] = at + sl.max_off[j];
    }
    sp.width = sl.width;
    sp.pad = 0;
    patches.push_back(sp);
  }
  skeleton.insert(skeleton.end(), footer.begin(), footer.end());
  const uint32_t flen = (uint32_t)footer.size();
  const uint8_t* lp = (const uint8_t*)&flen;
  skeleton.insert(skeleton.end(), lp, lp + 4);
  skeleton.insert(skeleton.end(), {'P', 'A', 'R', '1'});
}

}  // namespace

// what layout_segments decided and uploaded, for write_segments
struct EncodeLayout::Impl {
  explicit Impl(hs_ctx* ctx) : t_plan(ctx) {}
  StageTimer t_plan;  // read at the end of write_segments (reading it synchronises)
  int64_t P = 0;      // rows per page
  std::vector<pq::SchemaColumn> schema;
  std::string schema_json;
  std::vector<std::vector<uint64_t>> tile_val_off, tile_def_off;  // nullable and string columns
  std::vector<ColDict> dicts;
  std::vector<int> carried_cols;  // by record slot
  std::vector<StatPatch> stat_patches;
  std::vector<uint8_t> skeleton;
  std::vector<ByteCopy> copies;
  bool compress = false;
  std::vector<PagePlan> page_plans;
  std::vector<FilePlan> file_plans;
  uint64_t cursor = 0;
  uint32_t page_counter = 0;
  Buf<uint8_t> d_skel;
  Buf<ByteCopy> d_copies;
  Buf<uint32_t> d_page_begin;
  Buf<uint64_t> d_pvo;  // ncols x page_counter
  KeyPageDest key_dest{};
};

bool layout_needs_sorted_rows(const Table& table) {
  for (const DevColumn& dc : table.cols)
    if (dc.has_nulls || dc.type == HS_TYPE_STRING) return true;
  return false;
}

void encode_segments(hs_ctx* ctx, const EncodeRequest& req, EncodedFiles* out, hs_stats* stats) {
  EncodeLayout lay;
  layout_segments(ctx, req, &lay, out, stats);
  write_segments(ctx, req, lay, false, out, stats);
}

const KeyPageDest* key_page_dest(EncodeLayout& lay, const EncodeRequest& req, EncodedFiles* out) {
  EncodeLayout::Impl& L = *lay.impl;
  const DevColumn& dc = req.table->cols[0];
  if (dc.has_nulls || L.dicts[0].use || (dc.type != HS_TYPE_INT32 && dc.type != HS_TYPE_INT64) || L.P > (int64_t)UINT32_MAX)
    return nullptr;
  L.key_dest = KeyPageDest{out->arena.get(), L.d_page_begin.get(), L.d_pvo.get(), (uint32_t)L.P, dc.width, dc.type};
  return &L.key_dest;
}

void layout_segments(hs_ctx* ctx, const EncodeRequest& req, EncodeLayout* lay, EncodedFiles* out, hs_stats* stats) {
  (void)stats;
  lay->impl = std::make_shared<EncodeLayout::Impl>(ctx);
  EncodeLayout::Impl& L = *lay->impl;
  const Table& table = *req.table;
  const int ncols = (int)table.cols.size();
  const int nseg = (int)req.seg_offsets.size() - 1;
  int64_t P = req.rows_per_page > 0 ? req.rows_per_page : 131072;
  P = (int64_t)round_up((size_t)P, kSortTile);
  L.P = P;
  L.t_plan.start();
  for (int c = 0; c < ncols; c++) {
    const DevColumn& dc = table.cols[c];
    if (dc.type == HS_TYPE_BOOL ? P > INT32_MAX : dc.width != 4 && dc.width != 8)  // (a boolean's schema type is the source's)
      fail(HS_EUNSUPPORTED, dc.type == HS_TYPE_BOOL ? "column '%s': boolean pages hold at most 2^31 - 1 rows" : "column '%s': %d-byte values cannot be written by the GPU encoder yet", dc.name.c_str(), dc.width);
  }
  std::vector<pq::SchemaColumn>& schema = L.schema;
  schema.resize(ncols);
  for (int c = 0; c < ncols; c++) {
    schema[c] = table.cols[c].schema;
    schema[c].repetition = pq::OPTIONAL;  // Spark writes every column of a DataFrame read from Parquet as optional
    schema[c].num_children = 0;
    switch (table.cols[c].type) {
      case HS_TYPE_INT32: schema[c].type = pq::INT32; break;
      case HS_TYPE_INT64: schema[c].type = pq::INT64; break;
      case HS_TYPE_FLOAT: schema[c].type = pq::FLOAT; break;
      case HS_TYPE_DOUBLE: schema[c].type = pq::DOUBLE; break;
      case HS_TYPE_STRING: schema[c].type = pq::BYTE_ARRAY; break;  // converted type (UTF8 or none) comes from the source
    }
  }
  L.schema_json = pq::spark_schema_json(schema);
  const std::string& schema_json = L.schema_json;

  // nullable columns: per-tile non-null counts (tiles are kSortTile-aligned inside a segment and P is a multiple of
  // kSortTile, so a tile never straddles a page)
  const int64_t ntiles = req.plan->ntiles;
  std::vector<std::vector<uint32_t>> tile_valid(ncols), tile_bytes(ncols);  // tile_bytes: string columns only
  std::vector<std::vector<uint64_t>>& tile_val_off = L.tile_val_off;
  std::vector<std::vector<uint64_t>>& tile_def_off = L.tile_def_off;
  tile_val_off.resize(ncols);
  tile_def_off.resize(ncols);
  {
    std::vector<Buf<uint32_t>> d_counts(ncols), d_bytes(ncols);
    bool any = false;
    for (int c = 0; c < ncols; c++) {
      if (table.cols[c].type == HS_TYPE_STRING) {  // always laid out tile by tile: the value sizes are data
        any = true;
        d_counts[c].alloc(ctx, std::max<int64_t>(1, ntiles));
        d_bytes[c].alloc(ctx, std::max<int64_t>(1, ntiles));
        launch_tile_string_sizes(ctx, req.plan->tiles.get(), ntiles, req.d_perm, (const uint64_t*)table.cols[c].data.get(),
                                 table.cols[c].has_nulls ? table.cols[c].valid.get() : nullptr, d_bytes[c].get(), d_counts[c].get());
        tile_valid[c].resize(ntiles);
        tile_bytes[c].resize(ntiles);
        tile_val_off[c].assign(ntiles, 0);
        tile_def_off[c].assign(ntiles, 0);
        if (ntiles) {
          copy_d2h(ctx, tile_valid[c].data(), d_counts[c].get(), sizeof(uint32_t) * ntiles);
          copy_d2h(ctx, tile_bytes[c].data(), d_bytes[c].get(), sizeof(uint32_t) * ntiles);
        }
        continue;
      }
      if (!table.cols[c].has_nulls) continue;
      any = true;
      d_counts[c].alloc(ctx, std::max<int64_t>(1, ntiles));
      launch_tile_valid_counts(ctx, req.plan->tiles.get(), ntiles, req.d_perm, table.cols[c].valid.get(), d_counts[c].get());
      tile_valid[c].resize(ntiles);
      tile_val_off[c].assign(ntiles, 0);
      tile_def_off[c].assign(ntiles, 0);
      if (ntiles)
        copy_d2h(ctx, tile_valid[c].data(), d_counts[c].get(), sizeof(uint32_t) * ntiles);
    }
    if (any) sync_stream(ctx);
  }
  const std::vector<uint32_t>& seg_tile_begin = req.plan->h_seg_tile_begin;

  // ---- dictionary analysis: distinct values of every non-null column, capped at kMaxDictEntries ---------------------
  std::vector<ColDict>& dicts = L.dicts;
  dicts.resize(ncols);
  const int64_t total_rows = table.nrows;
  std::vector<int>& carried_cols = L.carried_cols;
  carried_cols.assign(kMaxCarried, -1);
  for (int c = 0; c < ncols; c++) {
    const DevColumn& dc = table.cols[c];
    if (!dc.carried) continue;  // late-materialised: the dictionary and the codes were fixed when the sources were decoded
    if (dc.carry_slot < 0 || dc.carry_slot >= kMaxCarried || !table.rec) fail(HS_EINVAL, "column '%s': code record missing", dc.name.c_str());
    ColDict& cd = dicts[c];
    cd.values = dc.dict_values;
    cd.ndict = (uint32_t)cd.values.size();
    cd.bw = dc.dict_bw;
    cd.use = true;
    carried_cols[dc.carry_slot] = c;
  }
  if (req.use_dictionary && total_rows > 0) {
    // staged sampling: 16 K rows that are (nearly) all distinct mark a key-like column at once; a 256 K-row sample then
    // lets the remaining high-cardinality columns overflow cheaply (the overflow path serialises on one counter).  The
    // first stage runs for ALL columns before the host looks at any result: one synchronisation instead of one per column.
    DictProbe* early = req.probe;  // first stage already launched behind the partition (see DictProbe)?
    if (early && ((int)early->keys.size() != ncols || early->mini != std::min<int64_t>(total_rows, 1 << 14))) early = nullptr;
    if (early && !early->delivered(ctx)) sync_stream(ctx);
    Buf<uint32_t> own_states;
    if (early) own_states = std::move(early->d_states);
    else own_states.alloc(ctx, 4 * (size_t)ncols);
    Buf<uint32_t>& d_states = own_states;
    std::vector<uint32_t> h_states(4 * (size_t)ncols, 0u);
    if (early) h_states = early->h_states;
    else fill_bytes(ctx, d_states.get(), 0, 16 * (size_t)ncols);
    const int64_t mini = std::min<int64_t>(total_rows, 1 << 14);
    bool any_sampled = false;
    for (int c = 0; c < ncols; c++) {
      const DevColumn& dc = table.cols[c];
      if (dc.has_nulls || dc.carried || dc.type == HS_TYPE_STRING || dc.width == 1) continue;  // booleans: PLAIN, as parquet-mr
      ColDict& cd = dicts[c];
      if (dc.dict_ready && dc.dict_keys) {
        cd.keys_ptr = dc.dict_keys.get();
        memcpy(&h_states[4 * (size_t)c], dc.dict_state, 16);
        continue;
      }
      if (early && early->keys[c]) {
        cd.keys = std::move(early->keys[c]);
        cd.keys_ptr = cd.keys.get();
        continue;
      }
      cd.keys.alloc(ctx, kDictCapacity);
      cd.keys_ptr = cd.keys.get();
      fill_bytes(ctx, cd.keys.get(), 0xFF, sizeof(unsigned long long) * kDictCapacity);
      launch_dict_build(ctx, dc.data.get(), dc.width, 0, mini, cd.keys.get(), kDictCapacity, kMaxDictEntries, d_states.get() + 4 * c);
      copy_d2h(ctx, &h_states[4 * (size_t)c], d_states.get() + 4 * c, 16);
      any_sampled = true;
    }
    if (any_sampled) sync_stream(ctx);
    for (int c = 0; c < ncols; c++) {
      const DevColumn& dc = table.cols[c];
      if (dc.has_nulls || dc.carried || dc.type == HS_TYPE_STRING || dc.width == 1) continue;
      ColDict& cd = dicts[c];
      uint32_t* st = &h_states[4 * (size_t)c];
      const bool ready = dc.dict_ready && dc.dict_keys;
      if (!ready) {
        uint32_t* d_state = d_states.get() + 4 * c;
        if (total_rows > (1 << 20) && st[0] + st[2] > 0.95 * mini) {
          cd.keys.release();
          continue;
        }
        const int64_t sample = std::min<int64_t>(total_rows, 1 << 18);
        if (sample > mini) {
          launch_dict_build(ctx, dc.data.get(), dc.width, mini, sample, cd.keys.get(), kDictCapacity, kMaxDictEntries, d_state);
          copy_d2h(ctx, st, d_state, 16);
          sync_stream(ctx);
        }
        if (!st[1] && sample < total_rows) {
          launch_dict_build(ctx, dc.data.get(), dc.width, sample, total_rows, cd.keys.get(), kDictCapacity, kMaxDictEntries, d_state);
          copy_d2h(ctx, st, d_state, 16);
          sync_stream(ctx);
        }
      }
      if (st[1]) {
        cd.keys.release();
        continue;
      }
      // distinct values: compacted on the device, sorted on the host (<= 65536 of them)
      cd.values = sorted_dictionary(ctx, cd.keys_ptr, st, dc.type);
      cd.ndict = (uint32_t)cd.values.size();
      cd.bw = bits_for(cd.ndict);
      if (!dictionary_pays_off(cd.ndict, cd.bw, dc.width, total_rows, nseg)) {
        cd.keys.release();
        continue;
      }
      upload_lookup_table(ctx, cd.values, &cd.entries, &cd.mask, &cd.empty_index);
      cd.use = true;
    }
  }

  const bool stats_on_key = req.key_sorted && !table.cols[0].has_nulls &&
                            (table.cols[0].type == HS_TYPE_INT32 || table.cols[0].type == HS_TYPE_INT64);
  std::vector<StatPatch>& stat_patches = L.stat_patches;
  std::vector<uint8_t>& skeleton = L.skeleton;
  std::vector<ByteCopy>& copies = L.copies;
  L.compress = req.codec != pq::UNCOMPRESSED;
  const bool compress = L.compress;
  std::vector<PagePlan>& page_plans = L.page_plans;
  std::vector<FilePlan>& file_plans = L.file_plans;
  auto header_len_at = [&](size_t skel_pos) -> uint32_t {  // length of the Thrift struct (page header) that starts there
    thrift::Reader r(skeleton.data() + skel_pos, skeleton.data() + skeleton.size());
    r.skip(thrift::T_STRUCT);
    if (r.bad) fail(HS_EINVAL, "internal: page header does not parse");
    return (uint32_t)(r.p - (skeleton.data() + skel_pos));
  };
  std::vector<uint32_t> seg_page_begin(nseg + 1, 0);
  std::vector<std::vector<uint64_t>> page_value_offset(ncols);
  uint64_t& cursor = L.cursor;
  uint32_t& page_counter = L.page_counter;
  auto emit = [&](uint64_t dst, size_t skel_begin) {
    copies.push_back(ByteCopy{dst, (uint32_t)skel_begin, (uint32_t)(skeleton.size() - skel_begin)});
  };
  for (int c = 0; c < ncols; c++) {
    ColDict& cd = dicts[c];
    if (!cd.use) continue;
    const int W = table.cols[c].width;
    cd.skel_off = skeleton.size();
    pq::write_dict_page_header(skeleton, (int32_t)(cd.ndict * W), (int32_t)cd.ndict);
    for (uint64_t v : cd.values) {
      const uint8_t* vp = (const uint8_t*)&v;
      skeleton.insert(skeleton.end(), vp, vp + W);
    }
    cd.skel_len = skeleton.size() - cd.skel_off;
  }
  out->files.clear();
  for (int s = 0; s < nseg; s++) {
    seg_page_begin[s] = page_counter;
    const int64_t n = (int64_t)(req.seg_offsets[s + 1] - req.seg_offsets[s]);
    if (n == 0) continue;  // no file for an empty bucket
    int64_t RG = !req.seg_rows_per_row_group.empty() ? req.seg_rows_per_row_group[s]
                                                     : (req.rows_per_row_group > 0 ? req.rows_per_row_group : 4194304);
    RG = std::max<int64_t>(P, RG / P * P);
    const uint64_t file_off = round_up(cursor, 64);
    cursor = file_off;
    {
      size_t b = skeleton.size();
      skeleton.insert(skeleton.end(), {'P', 'A', 'R', '1'});
      emit(cursor, b);
      cursor += 4;
    }
    const int64_t npages = ceil_div(n, P);
    for (int c = 0; c < ncols; c++) page_value_offset[c].resize(page_counter + npages);
    std::vector<pq::OutRowGroup> rgs;
    for (int64_t r0 = 0; r0 < n; r0 += RG) {
      const int64_t r1 = std::min(n, r0 + RG);
      pq::OutRowGroup g;
      g.num_rows = r1 - r0;
      g.file_offset = (int64_t)(cursor - file_off);
      const uint64_t rg_begin = cursor;
      for (int c = 0; c < ncols; c++) {
        const int W = table.cols[c].width;
        pq::OutChunk ch;
        ch.type = schema[c].type;
        ch.num_values = r1 - r0;
        ch.data_page_offset = (int64_t)(cursor - file_off);
        ch.null_count = 0;
        ch.value_width = W;
        // the indexed column is sorted inside a bucket: min / max of a row group are its first / last key (filled in on the
        // GPU after the sort); this is what lets a Spark reader prune row groups on the key (SURVEY.md 8a, row a7)
        ch.has_minmax = stats_on_key && c == 0;
        const uint64_t chunk_begin = cursor;
        const size_t chunk_first_page = page_plans.size();
        if (dicts[c].use) {  // every chunk of the column carries the same (global) dictionary page
          ch.has_dictionary = true;
          ch.dictionary_page_offset = (int64_t)(cursor - file_off);
          copies.push_back(ByteCopy{cursor, (uint32_t)dicts[c].skel_off, (uint32_t)dicts[c].skel_len});
          if (compress) {
            const uint32_t hl = header_len_at(dicts[c].skel_off);
            page_plans.push_back(PagePlan{cursor, hl, (uint32_t)(dicts[c].skel_len - hl), pq::DICTIONARY_PAGE,
                                          (int32_t)dicts[c].ndict, pq::ENC_PLAIN_DICTIONARY});
          }
          cursor += dicts[c].skel_len;
          ch.data_page_offset = (int64_t)(cursor - file_off);
        }
        for (int64_t p0 = r0; p0 < r1; p0 += P) {
          const int64_t np = std::min(P, r1 - p0);
          const size_t b = skeleton.size();
          const uint64_t page_begin = cursor;
          if (dicts[c].use) {
            pq::write_dict_data_page_prefix(skeleton, np, dicts[c].bw);
            emit(cursor, b);
            cursor += skeleton.size() - b;
            page_value_offset[c][page_counter + (p0 / P)] = cursor;
            cursor += (uint64_t)((np + 7) / 8) * dicts[c].bw;
          } else if (table.cols[c].type == HS_TYPE_STRING) {
            // PLAIN BYTE_ARRAY: definition bits for every row, then [u32 length][bytes] per non-null value, tile by tile
            const int64_t t0 = seg_tile_begin[s] + p0 / kSortTile, t1 = seg_tile_begin[s] + ceil_div(p0 + np, (int64_t)kSortTile);
            int64_t non_null = 0;
            uint64_t value_bytes = 0;
            for (int64_t t = t0; t < t1; t++) {
              non_null += tile_valid[c][t];
              value_bytes += tile_bytes[c][t];
            }
            if (value_bytes + (uint64_t)np / 8 + 64 >= (1ull << 31)) fail(HS_EUNSUPPORTED, "column '%s': a page of strings exceeds 2 GiB", table.cols[c].name.c_str());
            pq::write_nullable_page_prefix_bytes(skeleton, np, value_bytes);
            emit(cursor, b);
            cursor += skeleton.size() - b;
            const uint64_t def_bits = cursor;
            cursor += (uint64_t)((np + 7) / 8);
            page_value_offset[c][page_counter + (p0 / P)] = cursor;
            uint64_t voff = cursor;
            for (int64_t t = t0; t < t1; t++) {
              tile_def_off[c][t] = def_bits + (uint64_t)(t - t0) * (kSortTile / 8);
              tile_val_off[c][t] = voff;
              voff += tile_bytes[c][t];
            }
            cursor += value_bytes;
            ch.null_count += np - non_null;
          } else if (!table.cols[c].has_nulls) {
            W == 1 ? pq::write_bool_page_prefix(skeleton, np) : pq::write_plain_page_prefix(skeleton, cursor, np, W);  // (arena: 64-byte aligned files)
            emit(cursor, b);
            cursor += skeleton.size() - b;
            page_value_offset[c][page_counter + (p0 / P)] = cursor;
            cursor += W == 1 ? (uint64_t)(np + 7) / 8 : (uint64_t)np * W;  // booleans bit-packed
          } else {
            // tiles of this page: [t0, t1) in the segment's tile list
            const int64_t t0 = seg_tile_begin[s] + p0 / kSortTile, t1 = seg_tile_begin[s] + ceil_div(p0 + np, (int64_t)kSortTile);
            int64_t non_null = 0;
            for (int64_t t = t0; t < t1; t++) non_null += tile_valid[c][t];
            pq::write_nullable_page_prefix_bytes(skeleton, np, W == 1 ? (uint64_t)(non_null + 7) / 8 : (uint64_t)non_null * W);
            emit(cursor, b);
            cursor += skeleton.size() - b;
            const uint64_t def_bits = cursor;
            cursor += (uint64_t)((np + 7) / 8);
            page_value_offset[c][page_counter + (p0 / P)] = cursor;
            uint64_t voff = cursor;
            for (int64_t t = t0; t < t1; t++) {
              tile_def_off[c][t] = def_bits + (uint64_t)(t - t0) * (kSortTile / 8);
              tile_val_off[c][t] = voff;
              voff += (uint64_t)tile_valid[c][t] * W;
            }
            cursor += W == 1 ? (uint64_t)(non_null + 7) / 8 : (uint64_t)non_null * W;  // (booleans: one CTA per page, see k_gather_encode_bool_nullable)
            ch.null_count += np - non_null;
          }
          if (compress) {
            const uint32_t hl = header_len_at(b);
            page_plans.push_back(PagePlan{page_begin, hl, (uint32_t)(cursor - page_begin - hl), pq::DATA_PAGE, (int32_t)np,
                                          dicts[c].use ? pq::ENC_PLAIN_DICTIONARY : pq::ENC_PLAIN});
          }
        }
        ch.total_size = (int64_t)(cursor - chunk_begin);
        g.chunks.push_back(ch);
        if (compress) {
          if (file_plans.empty() || file_plans.back().seg != s) {
            file_plans.emplace_back();
            file_plans.back().seg = s;
            file_plans.back().rows = n;
          }
          file_plans.back().chunk_pages.emplace_back(chunk_first_page, page_plans.size() - chunk_first_page);
        }
      }
      g.total_byte_size = (int64_t)(cursor - rg_begin);
      rgs.push_back(std::move(g));
    }
    {
      const size_t b = skeleton.size();
      append_file_end(schema, rgs, n, schema_json, req.seg_offsets[s], cursor, skeleton, stat_patches);
      if (compress) file_plans.back().rgs = rgs;
      emit(cursor, b);
      cursor += skeleton.size() - b;
    }
    OutFile of;
    of.bucket = req.seg_ids.empty() ? s : req.seg_ids[s];
    of.name = req.seg_names[s];
    of.offset = file_off;
    of.size = cursor - file_off;
    of.rows = n;
    out->files.push_back(std::move(of));
    page_counter += (uint32_t)npages;
  }
  seg_page_begin[nseg] = page_counter;
  if (skeleton.size() >= (1ull << 32)) fail(HS_EUNSUPPORTED, "index metadata exceeds 4 GiB");
  out->arena_bytes = cursor;
  out->arena.alloc(ctx, std::max<uint64_t>(cursor, 16) + 64);

  // upload the plan
  L.d_skel.alloc(ctx, std::max<size_t>(1, skeleton.size()));
  L.d_copies.alloc(ctx, std::max<size_t>(1, copies.size()));
  L.d_page_begin.alloc(ctx, seg_page_begin.size());
  L.d_pvo.alloc(ctx, std::max<size_t>(1, (size_t)ncols * page_counter));
  if (!skeleton.empty())
    copy_h2d(ctx, L.d_skel.get(), skeleton.data(), skeleton.size());
  if (!copies.empty())
    copy_h2d(ctx, L.d_copies.get(), copies.data(), copies.size() * sizeof(ByteCopy));
  copy_h2d(ctx, L.d_page_begin.get(), seg_page_begin.data(), seg_page_begin.size() * 4);
  for (int c = 0; c < ncols; c++)
    if (page_counter)
      copy_h2d(ctx, L.d_pvo.get() + (size_t)c * page_counter, page_value_offset[c].data(), (size_t)page_counter * 8);
  L.t_plan.stop();
}

void write_segments(hs_ctx* ctx, const EncodeRequest& req, EncodeLayout& lay, bool key_pages_written, EncodedFiles* out,
                    hs_stats* stats) {
  EncodeLayout::Impl& L = *lay.impl;
  const Table& table = *req.table;
  const int ncols = (int)table.cols.size();
  const int64_t ntiles = req.plan->ntiles;
  const int64_t P = L.P;
  const std::vector<pq::SchemaColumn>& schema = L.schema;
  const std::string& schema_json = L.schema_json;
  const std::vector<std::vector<uint64_t>>& tile_val_off = L.tile_val_off;
  const std::vector<std::vector<uint64_t>>& tile_def_off = L.tile_def_off;
  const std::vector<ColDict>& dicts = L.dicts;
  const std::vector<int>& carried_cols = L.carried_cols;
  const std::vector<StatPatch>& stat_patches = L.stat_patches;
  const std::vector<ByteCopy>& copies = L.copies;
  const bool compress = L.compress;
  const std::vector<PagePlan>& page_plans = L.page_plans;
  std::vector<FilePlan>& file_plans = L.file_plans;
  uint64_t& cursor = L.cursor;
  const uint32_t page_counter = L.page_counter;
  const Buf<uint8_t>& d_skel = L.d_skel;
  const Buf<ByteCopy>& d_copies = L.d_copies;
  const Buf<uint32_t>& d_page_begin = L.d_page_begin;
  const Buf<uint64_t>& d_pvo = L.d_pvo;
  StageTimer t_enc(ctx);

  // ---- K5+K6 -----------------------------------------------------------------------------------------
  t_enc.start();
  launch_scatter_bytes(ctx, d_copies.get(), (int64_t)copies.size(), d_skel.get(), out->arena.get());
  for (int c = 0; c < ncols; c++) {
    const DevColumn& dc = table.cols[c];
    GatherColumn gc;
    gc.src = dc.data.get();
    gc.sorted_keys = nullptr;
    gc.key_type = dc.type;
    gc.width = dc.width;
    gc.page_value_offset = d_pvo.get() + (size_t)c * page_counter;
    if (dicts[c].use) continue;  // handled below, all dictionary columns together
    if (dc.type == HS_TYPE_STRING) {
      Buf<uint64_t> d_voff(ctx, std::max<int64_t>(1, ntiles)), d_doff(ctx, std::max<int64_t>(1, ntiles));
      if (ntiles) {
        copy_h2d(ctx, d_voff.get(), tile_val_off[c].data(), 8 * ntiles);
        copy_h2d(ctx, d_doff.get(), tile_def_off[c].data(), 8 * ntiles);
      }
      launch_gather_encode_strings(ctx, req.plan->tiles.get(), ntiles, req.d_perm, (const uint64_t*)dc.data.get(),
                                   dc.has_nulls ? dc.valid.get() : nullptr, d_voff.get(), d_doff.get(), out->arena.get());
      continue;
    }
    if (dc.has_nulls) {
      Buf<uint64_t> d_voff(ctx, std::max<int64_t>(1, ntiles)), d_doff(ctx, std::max<int64_t>(1, ntiles));
      if (ntiles) {
        copy_h2d(ctx, d_voff.get(), tile_val_off[c].data(), 8 * ntiles);
        copy_h2d(ctx, d_doff.get(), tile_def_off[c].data(), 8 * ntiles);
      }
      launch_gather_encode_nullable(ctx, req.plan->tiles.get(), ntiles, req.d_perm, dc.data.get(), dc.valid.get(), dc.width,
                                    d_voff.get(), d_doff.get(), out->arena.get());
      continue;
    }
    if (c == 0 && key_pages_written) continue;  // the sort stored the key into its pages
    if (c == 0 && req.d_sorted_keys && (dc.type == HS_TYPE_INT32 || dc.type == HS_TYPE_INT64)) gc.sorted_keys = req.d_sorted_keys;
    launch_gather_encode(ctx, req.plan->tiles.get(), req.plan->ntiles, req.plan->seg_start.get(), req.d_perm, gc,
                         d_page_begin.get(), P, out->arena.get());
  }
  if (!stat_patches.empty()) {
    Buf<StatPatch> d_sp(ctx, stat_patches.size());
    copy_h2d(ctx, d_sp.get(), stat_patches.data(), sizeof(StatPatch) * stat_patches.size());
    launch_patch_key_stats(ctx, d_sp.get(), (int64_t)stat_patches.size(), req.d_perm, table.cols[0].data.get(), out->arena.get());
  }
  {  // dictionary columns, up to 8 per launch pair
    std::vector<int> dcols;
    for (int c = 0; c < ncols; c++)
      if (dicts[c].use && !table.cols[c].carried) dcols.push_back(c);
    if (carried_cols[0] >= 0) {  // codes are already in the partitioned records: bit-pack only
      DictPackArgs pa;
      memset(&pa, 0, sizeof pa);
      for (int slot = 0; slot < kMaxCarried && carried_cols[slot] >= 0; slot++) {
        const int c = carried_cols[slot];
        pa.page_value_offset[slot] = d_pvo.get() + (size_t)c * page_counter;
        pa.bw[slot] = dicts[c].bw;
        pa.ncols = slot + 1;
      }
      launch_dict_pack(ctx, req.plan->tiles.get(), ntiles, req.plan->seg_start.get(), req.d_perm, pa, 4,
                       (const uint16_t*)table.rec.get(), d_page_begin.get(), P, out->arena.get());
    }
    for (size_t b0 = 0; b0 < dcols.size(); b0 += 8) {
      DictMapArgs ma;
      DictPackArgs pa;
      memset(&ma, 0, sizeof ma);
      memset(&pa, 0, sizeof pa);
      const int nd = (int)std::min<size_t>(8, dcols.size() - b0);
      ma.ncols = pa.ncols = nd;
      for (int j = 0; j < nd; j++) {
        const int c = dcols[b0 + j];
        ma.src[j] = table.cols[c].data.get();
        ma.width[j] = table.cols[c].width;
        ma.entries[j] = dicts[c].entries.get();
        ma.mask[j] = dicts[c].mask;
        ma.empty_index[j] = dicts[c].empty_index;
        pa.page_value_offset[j] = d_pvo.get() + (size_t)c * page_counter;
        pa.bw[j] = dicts[c].bw;
      }
      Buf<uint16_t> rec(ctx, (size_t)std::max<int64_t>(1, table.nrows) * (nd <= 4 ? 4 : 8));
      launch_dict_encode_all(ctx, req.plan->tiles.get(), ntiles, req.plan->seg_start.get(), req.d_perm, ma, pa, table.nrows,
                             kDictCapacity, rec.get(), d_page_begin.get(), P, out->arena.get());
    }
  }
  // ---- SNAPPY, GZIP, LZ4: the pages just written are compressed and the files laid out again -----------------------------
  // Compressed sizes are data: the files cannot be laid out before the pages exist.  So the uncompressed images above serve
  // as the compressor's input; the compressed sizes of the page bodies come back to the host, which lays the files out
  // again (new page headers, new footers, the codec in every chunk) and a copy kernel moves the compressed pieces into place.
  if (compress && !page_plans.empty()) {
    std::vector<std::pair<uint64_t, uint64_t>> bodies;
    for (const PagePlan& pp : page_plans) bodies.emplace_back(pp.hdr_off + pp.hdr_len, pp.body_len);
    CompressedBodies packed;
    compress_bodies(ctx, req.codec, out->arena.get(), bodies, &packed);
    // second layout
    std::vector<uint8_t> skel2;
    std::vector<ByteCopy> copies2;
    std::vector<BlobCopy> blobs;
    std::vector<StatPatch> patches2;
    uint64_t cur2 = 0;
    auto emit2 = [&](size_t skel_begin) {
      copies2.push_back(ByteCopy{cur2, (uint32_t)skel_begin, (uint32_t)(skel2.size() - skel_begin)});
      cur2 += skel2.size() - skel_begin;
    };
    std::vector<OutFile> files2;
    for (size_t fi = 0; fi < file_plans.size(); fi++) {
      FilePlan& fp = file_plans[fi];
      const uint64_t file_off = round_up(cur2, 64);
      cur2 = file_off;
      {
        const size_t b0 = skel2.size();
        skel2.insert(skel2.end(), {'P', 'A', 'R', '1'});
        emit2(b0);
      }
      size_t chunk_i = 0;
      for (pq::OutRowGroup& g : fp.rgs) {
        g.file_offset = (int64_t)(cur2 - file_off);
        int64_t rg_comp = 0, rg_uncomp = 0;
        for (pq::OutChunk& ch : g.chunks) {
          const auto range = fp.chunk_pages[chunk_i++];
          const uint64_t chunk_begin = cur2;
          int64_t uncomp = 0;
          bool first_data = true;
          for (size_t pi = range.first; pi < range.first + range.second; pi++) {
            const PagePlan& pp = page_plans[pi];
            const uint64_t comp = packed.size(pi);
            if (comp >= (1ull << 31)) fail(HS_EUNSUPPORTED, "a compressed page exceeds 2 GiB");
            const size_t b0 = skel2.size();
            if (pp.page_type == pq::DICTIONARY_PAGE) {
              ch.dictionary_page_offset = (int64_t)(cur2 - file_off);
              pq::write_dict_page_header(skel2, (int32_t)pp.body_len, pp.num_values, (int32_t)comp);
            } else {
              if (first_data) ch.data_page_offset = (int64_t)(cur2 - file_off);
              first_data = false;
              pq::write_data_page_header(skel2, (int32_t)pp.body_len, pp.num_values, pp.encoding, (int32_t)comp);
            }
            uncomp += (int64_t)(skel2.size() - b0) + pp.body_len;
            packed.append_preamble(pi, skel2);
            emit2(b0);
            packed.place(pi, blobs, &cur2);
            const size_t t0 = skel2.size();
            packed.append_trailer(pi, skel2);
            if (skel2.size() > t0) emit2(t0);
          }
          ch.total_size = (int64_t)(cur2 - chunk_begin);
          ch.total_uncompressed = uncomp;
          ch.codec = req.codec;
          rg_comp += ch.total_size;
          rg_uncomp += uncomp;
        }
        g.total_byte_size = rg_uncomp;
        g.total_compressed = rg_comp;
      }
      {
        const size_t b0 = skel2.size();
        append_file_end(schema, fp.rgs, fp.rows, schema_json, req.seg_offsets[fp.seg], cur2, skel2, patches2);
        emit2(b0);
      }
      OutFile of = out->files[fi];
      of.offset = file_off;
      of.size = cur2 - file_off;
      files2.push_back(std::move(of));
    }
    if (skel2.size() >= (1ull << 32)) fail(HS_EUNSUPPORTED, "index metadata exceeds 4 GiB");
    Buf<uint8_t> arena2(ctx, std::max<uint64_t>(cur2, 16) + 64);
    Buf<uint8_t> d_skel2(ctx, std::max<size_t>(1, skel2.size()));
    Buf<ByteCopy> d_copies2(ctx, std::max<size_t>(1, copies2.size()));
    Buf<BlobCopy> d_blobs(ctx, std::max<size_t>(1, blobs.size()));
    copy_h2d(ctx, d_skel2.get(), skel2.data(), skel2.size());
    copy_h2d(ctx, d_copies2.get(), copies2.data(), copies2.size() * sizeof(ByteCopy));
    copy_h2d(ctx, d_blobs.get(), blobs.data(), blobs.size() * sizeof(BlobCopy));
    launch_scatter_bytes(ctx, d_copies2.get(), (int64_t)copies2.size(), d_skel2.get(), arena2.get());
    launch_copy_blobs(ctx, d_blobs.get(), (int64_t)blobs.size(), packed.slots.get(), arena2.get());
    if (!patches2.empty()) {
      Buf<StatPatch> d_sp(ctx, patches2.size());
      copy_h2d(ctx, d_sp.get(), patches2.data(), sizeof(StatPatch) * patches2.size());
      launch_patch_key_stats(ctx, d_sp.get(), (int64_t)patches2.size(), req.d_perm, table.cols[0].data.get(), arena2.get());
    }
    sync_stream(ctx);  // (large plan arrays may have gone through cudaMemcpyAsync: keep them alive until here)
    out->arena = std::move(arena2);
    out->arena_bytes = cur2;
    out->files = std::move(files2);
    cursor = cur2;
  }
  t_enc.stop();
  sync_stream(ctx);  // host plan vectors are about to go out of scope
  stats->ms_plan += L.t_plan.ms();
  stats->ms_encode += t_enc.ms();
  stats->bytes_out += (int64_t)cursor;
  stats->files_out += (int32_t)out->files.size();
  lay.impl.reset();
}

void refuse_boolean_keys(const SourceSet& set, const std::vector<std::string>& keys) {
  for (const FileImage& img : set.impl->imgs)
    for (const std::string& k : keys) {
      const int idx = find_column(img.meta, k);
      if (idx >= 0 && img.meta.columns[idx].type == pq::BOOLEAN)
        fail(HS_EUNSUPPORTED, "column '%s' is boolean: boolean columns can be included in an index but not indexed", k.c_str());
    }
}

}  // namespace hs
