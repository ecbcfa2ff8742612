// parquet_decode.cu -- K1: Parquet page walk + page decode on the GPU.
//
// Replaces the map stage Spark runs for the reference's createIndex (SURVEY.md section 3.1, HOT LOOP 1):
// FileSourceScanExec -> VectorizedParquetRecordReader, reached from `spark.read.parquet` upstream of
// CreateAction (actions/CreateAction.scala:31) and from CoveringIndexTrait.scala:82-84,132 for refresh / optimize.
//
// Layout: whole Parquet file images live in HBM.  One thread per column chunk walks the Thrift page headers
// (k_walk_pages) and emits a PageDesc per data page; one CTA per data page then decodes it (k_decode_pages):
//   PLAIN fixed-width            unaligned little-endian loads -> coalesced stores
//   PLAIN_/RLE_DICTIONARY        RLE/bit-packed hybrid index stream expanded warp-per-run, dictionary in smem
//   definition levels (optional) same hybrid decoder at bit width 1, block scan -> dense value positions
//   converted values (ValueConv) INT96 / MILLIS timestamps -> int64 micros, FIXED_LEN_BYTE_ARRAY / INT64 decimals -> their
//                                unscaled int32 / int64, value by value (dictionary entries once, into the smem cache)
//   RLE BOOLEAN                  [4-byte length] + hybrid stream at bit width 1, through the dictionary-index reader
// Supported: data page v1 and v2, UNCOMPRESSED codec, BOOLEAN/INT32/INT64/FLOAT/DOUBLE, flat schemas.
#include "device_utils.cuh"
#include "kernels.h"
#include "parquet_meta.h"
#include "thrift_compact.h"

namespace hs {

namespace {

struct PageHeaderInfo {
  int32_t type = -1;
  int32_t uncompressed_size = 0;
  int32_t compressed_size = 0;
  int32_t num_values = 0;
  int32_t encoding = 0;
  int32_t def_bytes = -1;
  int32_t rep_bytes = 0;
  int32_t is_compressed = 1;  // v2 default
};

// Parses one PageHeader; returns false on malformed input.  r.p is left at the first byte of the page body.
__device__ bool parse_page_header(thrift::Reader& r, PageHeaderInfo& h) {
  int16_t fid = 0;
  for (;;) {
    uint8_t t = r.field(fid);
    if (r.bad) return false;
    if (t == thrift::T_STOP) break;
    switch (fid) {
      case 1: h.type = (int32_t)r.zigzag(); break;
      case 2: h.uncompressed_size = (int32_t)r.zigzag(); break;
      case 3: h.compressed_size = (int32_t)r.zigzag(); break;
      case 5:    // DataPageHeader
      case 7:    // DictionaryPageHeader
      case 8: {  // DataPageHeaderV2
        if (t != thrift::T_STRUCT) return false;
        int16_t f2 = 0;
        for (;;) {
          uint8_t t2 = r.field(f2);
          if (r.bad) return false;
          if (t2 == thrift::T_STOP) break;
          if (fid == 5 || fid == 7) {
            if (f2 == 1) h.num_values = (int32_t)r.zigzag();
            else if (f2 == 2) h.encoding = (int32_t)r.zigzag();
            else r.skip(t2);
          } else {
            if (f2 == 1) h.num_values = (int32_t)r.zigzag();
            else if (f2 == 4) h.encoding = (int32_t)r.zigzag();
            else if (f2 == 5) h.def_bytes = (int32_t)r.zigzag();
            else if (f2 == 6) h.rep_bytes = (int32_t)r.zigzag();
            else if (f2 == 7) h.is_compressed = (t2 == thrift::T_TRUE) ? 1 : 0;
            else r.skip(t2);
          }
        }
        break;
      }
      default: r.skip(t);
    }
  }
  return !r.bad;
}

__device__ void set_error(uint32_t* d_error, uint32_t code, uint32_t detail) {
  atomicCAS(d_error, 0u, (code << 24) | (detail & 0xffffffu));
}

__global__ void k_walk_pages(const ChunkDesc* __restrict__ chunks, int n_chunks, int32_t* __restrict__ page_counts,
                             const int64_t* __restrict__ page_offsets, PageDesc* __restrict__ pages,
                             uint32_t* d_error, int mode) {
  int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= n_chunks) return;
  const ChunkDesc ch = chunks[c];
  thrift::Reader r(ch.data, ch.data + ch.size);
  const uint8_t* dict = nullptr;
  int32_t dict_count = 0, dict_size = 0, dict_usize = 0;
  int64_t values_seen = 0;
  int32_t n_pages = 0;
  int64_t out = mode ? page_offsets[c] : 0;
  while (r.p < r.end && values_seen < ch.num_values) {
    PageHeaderInfo h;
    if (!parse_page_header(r, h) || h.compressed_size < 0 || h.uncompressed_size < 0 || h.num_values < 0 ||
        (int64_t)(r.end - r.p) < h.compressed_size) {
      set_error(d_error, DERR_BAD_HEADER, (uint32_t)c);
      break;
    }
    const uint8_t* body = r.p;
    // Every field a decoder will index with is range-checked HERE, before any page is decoded: a page header is
    // untrusted input, and a chunk that fails stops the whole call (decode_sources reads the error word first).
    if (h.type == pq::DATA_PAGE || h.type == pq::DATA_PAGE_V2) {
      bool ok = values_seen + h.num_values <= ch.num_values;  // a page never writes past its chunk's rows
      if (h.type == pq::DATA_PAGE_V2)
        ok = ok && h.rep_bytes >= 0 && h.def_bytes >= 0 && (int64_t)h.rep_bytes + h.def_bytes <= h.compressed_size &&
             (int64_t)h.rep_bytes + h.def_bytes <= h.uncompressed_size;
      if (!ok) {
        set_error(d_error, DERR_BAD_HEADER, (uint32_t)c);
        break;
      }
    } else if (h.type == pq::DICTIONARY_PAGE) {
      // dictionary entries are PLAIN values: all of them must lie inside the (decompressed) page
      const int64_t vw = ch.phys_type == pq::INT96 ? 12
                         : ch.phys_type == pq::FIXED_LEN_BYTE_ARRAY ? ch.type_length
                         : (ch.phys_type == pq::INT64 || ch.phys_type == pq::DOUBLE) ? 8 : (ch.phys_type == pq::BOOLEAN ? 0 : 4);
      const int64_t need = vw ? (int64_t)h.num_values * vw : ((int64_t)h.num_values + 7) / 8;
      if (need > h.uncompressed_size) {
        set_error(d_error, DERR_BAD_HEADER, (uint32_t)c);
        break;
      }
    }
    if (h.type == pq::DICTIONARY_PAGE) {
      dict = body;
      dict_count = h.num_values;
      dict_size = h.compressed_size;
      dict_usize = h.uncompressed_size;
      if (ch.codec == pq::UNCOMPRESSED && h.compressed_size != h.uncompressed_size) set_error(d_error, DERR_COMPRESSED, (uint32_t)c);
    } else if (h.type == pq::DATA_PAGE || h.type == pq::DATA_PAGE_V2) {
      if (mode) {
        PageDesc pd;
        pd.data = body;
        pd.dict = dict;
        pd.first_row = ch.row_base + values_seen;
        pd.dict_count = dict_count;
        pd.size = h.compressed_size;
        pd.num_values = h.num_values;
        pd.encoding = h.encoding;
        pd.page_type = h.type;
        pd.def_bytes = h.type == pq::DATA_PAGE_V2 ? h.def_bytes : -1;
        pd.rep_bytes = h.type == pq::DATA_PAGE_V2 ? h.rep_bytes : 0;
        pd.col = ch.col;
        pd.phys_type = ch.phys_type;
        pd.max_def = ch.max_def;
        pd.file_index = ch.file_index;
        pd.uncompressed_size = h.uncompressed_size;
        pd.dict_size = dict_size;
        pd.dict_uncompressed_size = dict_usize;
        pd.codec = ch.codec;
        // v1 pages of a compressed chunk are always compressed; v2 pages say so in their header
        pd.is_compressed = ch.codec != pq::UNCOMPRESSED && (h.type == pq::DATA_PAGE || h.is_compressed) ? 1 : 0;
        pd.chunk = c;
        pd.conv = ch.conv;
        pd.type_length = ch.type_length;
        pages[out + n_pages] = pd;
      }
      if (ch.codec == pq::UNCOMPRESSED && h.compressed_size != h.uncompressed_size) set_error(d_error, DERR_COMPRESSED, (uint32_t)c);
      values_seen += h.num_values;
      n_pages++;
    }  // index pages and unknown page types are skipped
    r.p = body + h.compressed_size;
  }
  if (values_seen != ch.num_values) set_error(d_error, DERR_VALUE_COUNT, (uint32_t)c);
  if (!mode) page_counts[c] = n_pages;
}

// ---- RLE / bit-packed hybrid decoder, resumable, CTA-cooperative -----------------------------------------------------
constexpr int kDecodeThreads = 256;
constexpr int kRunTable = 128;      // run-table entries per refill
constexpr int kMaxPerEntry = 256;   // values per entry (a warp expands one entry)
constexpr int kTileRows = 2048;     // rows per tile on the nullable / dictionary paths
constexpr int kSmemDict = 2048;     // dictionary entries cached in shared memory (8 B each)

struct HybridState {  // lives in shared memory; mutated by thread 0 only
  const uint8_t* p;
  const uint8_t* end;
  const uint8_t* run_data;  // bit-packed run: first byte
  uint32_t bw;
  uint32_t run_left;        // values left in the current run
  uint32_t run_pos;         // values of the current bit-packed run already consumed
  uint32_t run_value;       // RLE value
  uint32_t run_is_rle;
  uint32_t bad;
};

struct RunEntry {
  const uint8_t* data;
  uint32_t out_start;
  uint32_t count;
  uint32_t first;     // first value index inside the bit-packed run, or the RLE value
  uint32_t is_rle;
};

struct HybridShared {
  HybridState st;
  RunEntry tab[kRunTable];
  uint32_t n_runs;
  uint32_t produced;
};

__device__ void hybrid_init(HybridState& st, const uint8_t* p, const uint8_t* end, uint32_t bw) {
  st.p = p;
  st.end = end;
  st.bw = bw;
  st.run_left = 0;
  st.run_pos = 0;
  st.run_value = 0;
  st.run_is_rle = 1;
  st.run_data = p;
  st.bad = 0;
}

// thread 0: extend the run table to cover up to `want` more values
__device__ void hybrid_fill_table(HybridShared& hs, uint32_t want) {
  HybridState& st = hs.st;
  uint32_t produced = 0, nr = 0;
  while (produced < want && nr < kRunTable) {
    if (st.run_left == 0) {
      if (st.p >= st.end) {
        st.bad = 1;
        break;
      }
      // varint run header
      uint32_t h = 0;
      int shift = 0;
      while (st.p < st.end) {
        uint8_t b = *st.p++;
        h |= (uint32_t)(b & 0x7f) << shift;
        if (!(b & 0x80)) break;
        shift += 7;
        if (shift > 28) break;
      }
      if (h & 1) {  // bit-packed: (h >> 1) groups of 8 values
        uint32_t groups = h >> 1;
        // a run header may claim more groups than the stream holds: only what is there is decoded (the caller then
        // sees the stream end early and reports DERR_OVERRUN), nothing past `end` is read
        const uint64_t avail = st.bw ? (uint64_t)(st.end - st.p) / st.bw : 0xffffffffu / 8;
        const bool claimed = groups > 0;
        if (groups > avail) groups = (uint32_t)avail;
        if (groups > 0xffffffffu / 8) groups = 0xffffffffu / 8;
        st.run_is_rle = 0;
        st.run_left = groups * 8;
        st.run_pos = 0;
        st.run_data = st.p;
        st.p += (size_t)groups * st.bw;
        if (claimed && groups == 0) {  // nothing decodable is left
          st.bad = 1;
          break;
        }
      } else {
        st.run_is_rle = 1;
        st.run_left = h >> 1;
        uint32_t nbytes = (st.bw + 7) >> 3, v = 0;
        for (uint32_t i = 0; i < nbytes && st.p < st.end; i++) v |= (uint32_t)(*st.p++) << (8 * i);
        st.run_value = v;
      }
      if (st.run_left == 0) continue;  // empty run: legal but useless
    }
    uint32_t take = min(min(st.run_left, want - produced), (uint32_t)kMaxPerEntry);
    RunEntry& e = hs.tab[nr++];
    e.out_start = produced;
    e.count = take;
    e.is_rle = st.run_is_rle;
    e.data = st.run_data;
    e.first = st.run_is_rle ? st.run_value : st.run_pos;
    st.run_left -= take;
    st.run_pos += take;
    produced += take;
  }
  hs.n_runs = nr;
  hs.produced = produced;
}

// All threads: decode the next `count` values of the stream, calling sink(i, value) for i in [0, count).
// Returns false when the stream ended early.
template <typename Sink>
__device__ bool hybrid_decode_next(HybridShared& hs, uint32_t count, Sink sink) {
  uint32_t done = 0;
  const unsigned warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarps = blockDim.x >> 5;
  while (done < count) {
    __syncthreads();
    if (threadIdx.x == 0) hybrid_fill_table(hs, count - done);
    __syncthreads();
    const uint32_t nr = hs.n_runs, produced = hs.produced, bw = hs.st.bw;
    for (uint32_t e = warp; e < nr; e += nwarps) {
      const RunEntry en = hs.tab[e];
      for (uint32_t j = lane; j < en.count; j += 32) {
        uint32_t v = en.is_rle ? en.first : extract_bits(en.data, (uint64_t)en.first + j, bw);
        sink(done + en.out_start + j, v);
      }
    }
    if (produced == 0) return false;
    done += produced;
  }
  return true;
}

// all-valid when the definition-level block is nothing but RLE runs of the value 1 that cover the page (writers emit one
// such run; this engine's own encoder emits a few, see write_plain_page_prefix)
__device__ bool def_levels_all_valid(const uint8_t* def_p, const uint8_t* def_end, uint32_t n) {
  const uint8_t* q = def_p;
  uint32_t covered = 0;
  bool all_ones = true;
  for (int r = 0; r < 64 && covered < n && all_ones; r++) {
    uint32_t h = 0;
    int shift = 0;
    while (q < def_end) {
      uint8_t b = *q++;
      h |= (uint32_t)(b & 0x7f) << shift;
      if (!(b & 0x80)) break;
      shift += 7;
      if (shift > 28) break;
    }
    if ((h & 1) || q >= def_end || !(*q & 1) || (h >> 1) == 0) all_ones = false;
    else {
      covered += h >> 1;
      q++;
    }
  }
  return all_ones && covered >= n;
}

// An RLE BOOLEAN stream [q, end) whose runs, up to the first that reaches value n, all lie inside it: every run header,
// every RLE run's value byte and every bit-packed run's bytes (the hybrid reader would decode a run cut short by the end
// of the stream as far as it goes; a stream that holds too few values is caught while decoding)
__device__ bool rle_bool_stream_ok(const uint8_t* q, const uint8_t* end, uint32_t n) {
  uint64_t covered = 0;
  while (covered < n && q < end) {
    uint32_t h = 0;
    int shift = 0;
    uint8_t b;
    do {
      if (q >= end || shift > 28) return false;
      b = *q++;
      h |= (uint32_t)(b & 0x7f) << shift;
      shift += 7;
    } while (b & 0x80);
    const uint64_t len = h & 1 ? (uint64_t)(h >> 1) : 1;  // bytes behind the header: groups of 8 bits, or the value
    if (len > (uint64_t)(end - q)) return false;
    q += len;
    covered += h & 1 ? 8ull * (h >> 1) : (uint64_t)(h >> 1);
  }
  return true;
}

// where the definition levels of a page sit; returns false when the page is malformed
__device__ __forceinline__ bool locate_def_levels(const PageDesc& pg, const uint8_t*& p, const uint8_t*& def_p,
                                                  const uint8_t*& def_end) {
  const uint8_t* pend = pg.data + pg.size;
  def_p = def_end = nullptr;
  if (pg.page_type == pq::DATA_PAGE_V2) {
    p += pg.rep_bytes;
    if (pg.max_def > 0) {
      def_p = p;
      def_end = p + pg.def_bytes;
    }
    p += pg.def_bytes > 0 ? pg.def_bytes : 0;
  } else if (pg.max_def > 0) {
    if (pend - p < 4) return false;
    uint32_t len = load_le32_unaligned(p);
    if ((uint64_t)len > (uint64_t)(pend - p - 4)) return false;
    def_p = p + 4;
    def_end = def_p + len;
    p = def_end;
  }
  return p <= pend;
}

// One thread per data page: is it dictionary-encoded, and can it hold nulls?
__global__ void k_classify_pages(const PageDesc* __restrict__ pages, int64_t n_pages, uint32_t* __restrict__ col_flags,
                                 int zc_tile_rows) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_pages) return;
  const PageDesc pg = pages[i];
  uint32_t f = 0;
  if (pg.encoding != pq::ENC_PLAIN_DICTIONARY && pg.encoding != pq::ENC_RLE_DICTIONARY) f |= PAGECLASS_NOT_DICT;
  if (pg.max_def > 0) {
    const uint8_t* p = pg.data;
    const uint8_t *def_p, *def_end;
    if (!locate_def_levels(pg, p, def_p, def_end) || !def_levels_all_valid(def_p, def_end, (uint32_t)pg.num_values))
      f |= PAGECLASS_MAYBE_NULLS;
  }
  // readable in place?
  {
    const int W = (pg.phys_type == pq::INT64 || pg.phys_type == pq::DOUBLE) ? 8 : ((pg.phys_type == pq::INT32 || pg.phys_type == pq::FLOAT) ? 4 : 0);
    bool in_place = W != 0 && pg.conv == CONV_NONE && pg.encoding == pq::ENC_PLAIN && !pg.is_compressed && pg.size == pg.uncompressed_size &&
                    (f & PAGECLASS_MAYBE_NULLS) == 0 && zc_tile_rows > 0 && pg.num_values >= zc_tile_rows;
    if (in_place) {
      const uint8_t* p = pg.data;
      const uint8_t *def_p, *def_end;
      in_place = locate_def_levels(pg, p, def_p, def_end) && ((uintptr_t)p % W) == 0 &&
                 (int64_t)(pg.data + pg.size - p) >= (int64_t)pg.num_values * W;
    }
    if (!in_place) f |= PAGECLASS_NOT_IN_PLACE;
  }
  if (f) atomicOr(&col_flags[pg.col], f);
}

// one CTA per page: the page's share of the tile table (see ZcTile)
__global__ void k_fill_zc_tiles(const PageDesc* __restrict__ pages, ZcTile* const* __restrict__ tile_src, int T, int64_t nrows) {
  const PageDesc pg = pages[blockIdx.x];
  ZcTile* dst = tile_src[pg.col];
  if (!dst || pg.num_values <= 0) return;
  const int W = (pg.phys_type == pq::INT64 || pg.phys_type == pq::DOUBLE) ? 8 : 4;
  const uint8_t* p = pg.data;
  const uint8_t *def_p, *def_end;
  locate_def_levels(pg, p, def_p, def_end);  // validated by k_classify_pages
  const int64_t r0 = pg.first_row, r1 = pg.first_row + pg.num_values;  // rows [r0, r1)
  const uint8_t* rebased = p - (size_t)r0 * W;
  for (int64_t t = r0 / T + threadIdx.x; t * T < r1; t += blockDim.x) {
    const int64_t first = t * T, last = min(first + T, nrows) - 1;
    if (first >= r0) {  // the tile starts in this page
      dst[t].p0 = rebased;
      if (last < r1) {  // ... and ends in it
        dst[t].p1 = rebased;
        dst[t].split = INT64_MAX;
      }
    }
    if (last < r1 && first < r0) {  // the tile started in the page before
      dst[t].p1 = rebased;
      dst[t].split = r0;
    }
  }
}

// value -> code of a late-materialised dictionary column (same table layout and probing as k_dict_map_all)
__device__ __forceinline__ uint32_t carry_code(const ColumnOut& co, uint64_t v, uint32_t* d_error) {
  if (v == ~0ull) return co.carry_empty_index;
  const uint4* tab = reinterpret_cast<const uint4*>(co.carry_entries);
  const uint32_t mask = co.carry_mask, vlo = (uint32_t)v, vhi = (uint32_t)(v >> 32);
  uint32_t h = dict_hash_u64(v) & mask;
  for (uint32_t probes = 0; probes <= mask; probes++) {
    const uint4 e = tab[h];
    if (e.x == vlo && e.y == vhi) return e.z;
    if (e.x == 0xffffffffu && e.y == 0xffffffffu) break;
    h = (h + 1) & mask;
  }
  set_error(d_error, DERR_DICT_INDEX, 0xffffffu);  // a chunk dictionary holds a value the union does not
  return 0;
}

template <int W>
__device__ __forceinline__ uint64_t load_value(const uint8_t* p) {
  if (W == 8) return load_le64_unaligned(p);
  if (W == 4) return load_le32_unaligned(p);
  return *p;
}
template <int W>
__device__ __forceinline__ void store_value(void* base, int64_t row, uint64_t v) {
  if (W == 8) ((uint64_t*)base)[row] = v;
  else if (W == 4) ((uint32_t*)base)[row] = (uint32_t)v;
  else ((uint8_t*)base)[row] = (uint8_t)v;
}

// ---- converted values (ValueConv) ------------------------------------------------------------------------------------
// bytes one stored value of a converted page takes
__device__ __forceinline__ int conv_src_width(const PageDesc& pg) {
  return pg.conv == CONV_INT96 ? 12 : (pg.conv == CONV_FLBA ? pg.type_length : 8);
}

constexpr int64_t kJulianDayOfEpoch = 2440588;          // DateTimeUtils.JULIAN_DAY_OF_EPOCH
constexpr int64_t kMicrosPerDay = 86400000000ll;
constexpr int64_t kMicros1900 = -2208988800000000ll;    // 1900-01-01T00:00:00Z: Spark 3.1 fails to load INT96 before it

// The stored value at p as the engine keeps it (W bytes: int32 for a decimal(p <= 9), else int64).  A value Spark would
// refuse, or that does not fit W, raises the conversion's error (detail: the column) and yields 0.
template <int W>
__device__ __forceinline__ uint64_t convert_value(const PageDesc& pg, const uint8_t* p, uint32_t* d_error) {
  int64_t v;
  switch (pg.conv) {
    case CONV_INT96: {  // DateTimeUtils.fromJulianDay: (day - 2440588) * MICROS_PER_DAY + nanos / 1000 (truncating)
      const int64_t nanos = (int64_t)load_le64_unaligned(p);
      const int32_t day = (int32_t)load_le32_unaligned(p + 8);
      v = (int64_t)((uint64_t)((int64_t)day - kJulianDayOfEpoch) * (uint64_t)kMicrosPerDay) + nanos / 1000;
      if (v < kMicros1900) {
        set_error(d_error, DERR_SPARK_RANGE, (uint32_t)pg.col);
        return 0;
      }
      return (uint64_t)v;
    }
    case CONV_MILLIS: {  // Math.multiplyExact(millis, 1000)
      const int64_t ms = (int64_t)load_le64_unaligned(p);
      if (ms > INT64_MAX / 1000 || ms < INT64_MIN / 1000) {
        set_error(d_error, DERR_SPARK_RANGE, (uint32_t)pg.col);
        return 0;
      }
      return (uint64_t)(ms * 1000);
    }
    case CONV_FLBA: {  // big-endian two's complement of type_length bytes; the bytes above the low 8 only extend the sign
      const int L = pg.type_length;
      const int first = L > 8 ? L - 8 : 0;
      uint64_t u = (p[first] & 0x80) ? ~0ull : 0ull;
      for (int i = first; i < L; i++) u = (u << 8) | p[i];
      v = (int64_t)u;
      const uint8_t ext = v < 0 ? 0xff : 0x00;
      bool ok = true;
      for (int i = 0; i < first; i++) ok = ok && p[i] == ext;
      if (!ok || (W == 4 && (v < INT32_MIN || v > INT32_MAX))) {
        set_error(d_error, DERR_DECIMAL_WIDTH, (uint32_t)pg.col);
        return 0;
      }
      return W == 4 ? (uint64_t)(uint32_t)(int32_t)v : (uint64_t)v;
    }
    default: {  // CONV_NARROW: INT64 decimal(p <= 9) -> int32
      v = (int64_t)load_le64_unaligned(p);
      if (v < INT32_MIN || v > INT32_MAX) {
        set_error(d_error, DERR_DECIMAL_WIDTH, (uint32_t)pg.col);
        return 0;
      }
      return (uint64_t)(uint32_t)(int32_t)v;
    }
  }
}

struct DecodeShared {
  HybridShared def;
  HybridShared idx;
  uint64_t dict[kSmemDict];
  uint32_t tile_idx[kTileRows];
  uint32_t tile_pos[kTileRows];
  uint8_t tile_valid[kTileRows];
  uint32_t warp_sums[40];
  uint32_t flag;
};

// W = value width in bytes (8, 4) or 1 for BOOLEAN (bit-packed PLAIN, one output byte per row)
// CONV: the page's values are converted (pg.conv): W is the width kept, the stored values take conv_src_width bytes each
template <int W, bool CONV = false>
__device__ void decode_page(const PageDesc& pg, const ColumnOut& co, uint32_t* col_has_nulls, uint32_t* d_error,
                            DecodeShared& sm) {
  static_assert(!CONV || W == 4 || W == 8, "converted values are int32 / int64");
  const int SW = CONV ? conv_src_width(pg) : W;  // bytes per stored value
  // stored value i of the PLAIN run at base, as the column keeps it
  auto load_at = [&](const uint8_t* base, int64_t i) -> uint64_t {
    if (CONV) return convert_value<W>(pg, base + i * SW, d_error);
    return load_value<W>(base + i * W);
  };
  const int n = pg.num_values;
  const uint8_t* p = pg.data;
  const uint8_t* pend = pg.data + pg.size;  // from the values on: the end of their bytes
  const bool is_dict = pg.encoding == pq::ENC_PLAIN_DICTIONARY || pg.encoding == pq::ENC_RLE_DICTIONARY;
  // RLE BOOLEAN: the values are a hybrid stream of bit width 1, read like dictionary indices that are their own values
  const bool rle_bool = W == 1 && pg.encoding == pq::ENC_RLE;
  const bool hybrid_values = is_dict || rle_bool;
  if (!hybrid_values && pg.encoding != pq::ENC_PLAIN) {
    if (threadIdx.x == 0) set_error(d_error, DERR_UNSUPPORTED_ENCODING, (uint32_t)pg.encoding);
    return;
  }
  const bool carry = W != 1 && !CONV && co.carry != 0;  // emit 16-bit codes of the column-wide dictionary instead of values
  if (carry && !is_dict) {  // the column was classified dictionary-only before decoding
    if (threadIdx.x == 0) set_error(d_error, DERR_UNSUPPORTED_ENCODING, (uint32_t)pg.encoding);
    return;
  }
  // bit 1 of the column's flag word: a page that is NOT dictionary-encoded was seen (when it stays clear, the union of the
  // chunk dictionaries is a superset of the column's distinct values and the encoder can skip its full-column scan)
  if (!is_dict && threadIdx.x == 0) atomicOr(col_has_nulls, 2u);
  // ---- definition levels -----------------------------------------------------------------------------------
  const uint8_t* def_p = nullptr;
  const uint8_t* def_end = nullptr;
  if (n < 0 || pg.size < 0 || !locate_def_levels(pg, p, def_p, def_end)) {  // level bytes reach past the page
    if (threadIdx.x == 0) set_error(d_error, DERR_OVERRUN, (uint32_t)pg.col);
    return;
  }
  // all-valid fast check: a single RLE run of ones covering the page
  bool has_def = def_p != nullptr;
  if (has_def) {
    if (threadIdx.x == 0) sm.flag = def_levels_all_valid(def_p, def_end, (uint32_t)n) ? 1u : 0u;
    __syncthreads();
    if (sm.flag) has_def = false;
    __syncthreads();
  }
  // ---- dictionary -----------------------------------------------------------------------------------
  uint32_t idx_bw = 0;
  // carry mode keeps 16-bit codes in the same shared array: four times as many entries fit
  uint16_t* const dict16 = reinterpret_cast<uint16_t*>(sm.dict);
  const bool dict_in_smem = is_dict && pg.dict_count <= (carry ? kSmemDict * 4 : kSmemDict);
  if (is_dict) {
    if (pg.dict == nullptr) {
      if (threadIdx.x == 0) set_error(d_error, DERR_DICT_INDEX, 0);
      return;
    }
    if (n > 0 && p >= pend) {  // no room for the bit-width byte
      if (threadIdx.x == 0) set_error(d_error, DERR_OVERRUN, (uint32_t)pg.col);
      return;
    }
    idx_bw = n > 0 ? *p : 0;
    if (n > 0) p += 1;
    if (idx_bw > 32) {
      if (threadIdx.x == 0) set_error(d_error, DERR_UNSUPPORTED_ENCODING, idx_bw);
      return;
    }
    if (dict_in_smem) {
      for (int i = threadIdx.x; i < pg.dict_count; i += blockDim.x) {
        uint64_t v;
        if (W == 1) v = (pg.dict[i >> 3] >> (i & 7)) & 1;
        else v = load_at(pg.dict, i);
        if (carry) dict16[i] = (uint16_t)carry_code(co, v, d_error);
        else sm.dict[i] = v;
      }
    }
    if (threadIdx.x == 0) hybrid_init(sm.idx.st, p, pend, idx_bw);
  }
  if (rle_bool) {  // [4-byte length][stream], in v1 and v2 pages alike
    const uint32_t len = pend - p >= 4 ? load_le32_unaligned(p) : 0xffffffffu;
    if ((int64_t)len > (int64_t)(pend - p) - 4) {
      if (threadIdx.x == 0) set_error(d_error, DERR_OVERRUN, (uint32_t)pg.col);
      return;
    }
    p += 4;
    pend = p + len;
    if (threadIdx.x == 0) sm.flag = rle_bool_stream_ok(p, pend, (uint32_t)n) ? 1u : 0u;
    __syncthreads();
    if (!sm.flag) {
      if (threadIdx.x == 0) set_error(d_error, DERR_OVERRUN, (uint32_t)pg.col);
      return;
    }
    idx_bw = 1;
    if (threadIdx.x == 0) hybrid_init(sm.idx.st, p, pend, 1);
  }
  if (has_def && threadIdx.x == 0) hybrid_init(sm.def.st, def_p, def_end, 1);
  __syncthreads();
  const int64_t row0 = pg.first_row;
  const uint32_t dict_count = (uint32_t)pg.dict_count;
  auto dict_lookup = [&](uint32_t ix) -> uint64_t {
    if (rle_bool) return ix & 1u;
    if (ix >= dict_count) {
      set_error(d_error, DERR_DICT_INDEX, ix);
      return 0;
    }
    if (carry) return dict_in_smem ? (uint64_t)dict16[ix] : (uint64_t)carry_code(co, load_value<W>(pg.dict + (size_t)ix * W), d_error);
    if (dict_in_smem) return sm.dict[ix];
    if (W == 1) return (pg.dict[ix >> 3] >> (ix & 7)) & 1;
    return load_at(pg.dict, ix);
  };
  auto emit = [&](int64_t row, uint64_t v) {
    if (carry) ((uint16_t*)co.data)[row] = (uint16_t)v;
    else store_value<W>(co.data, row, v);
  };
  if (carry && has_def) {  // classified free of nulls before decoding
    if (threadIdx.x == 0) set_error(d_error, DERR_VALUE_COUNT, (uint32_t)pg.col);
    return;
  }

  // ---- fast paths: no nulls in this page -----------------------------------------------------------------------
  if (!has_def) {
    if (!hybrid_values) {
      if (W == 1) {
        if ((int64_t)(pend - p) < ((int64_t)n + 7) / 8) {
          if (threadIdx.x == 0) set_error(d_error, DERR_OVERRUN, (uint32_t)pg.col);
          return;
        }
        for (int i = threadIdx.x; i < n; i += blockDim.x) store_value<1>(co.data, row0 + i, (p[i >> 3] >> (i & 7)) & 1);
      } else if (CONV) {
        if ((int64_t)(pend - p) < (int64_t)n * SW) {
          if (threadIdx.x == 0) set_error(d_error, DERR_OVERRUN, (uint32_t)pg.col);
          return;
        }
        for (int i = threadIdx.x; i < n; i += kDecodeThreads) store_value<W>(co.data, row0 + i, load_at(p, i));
      } else {
        if ((int64_t)(pend - p) < (int64_t)n * W) {
          if (threadIdx.x == 0) set_error(d_error, DERR_OVERRUN, (uint32_t)pg.col);
          return;
        }
        // A straight copy.  Both variants keep a thread's loads free of branches so that eight of them are in flight
        // at once: naturally aligned bodies (this engine's own files) take plain vector loads; any other alignment
        // assembles each value from the two aligned words around it (the second word of the page's last value may
        // lie past the page but never past the file: a footer and the magic follow every page).
        if (W == 8) {
          uint64_t* dst = (uint64_t*)co.data + row0;
          if (((uintptr_t)p & 7) == 0) {
            const uint64_t* src = (const uint64_t*)p;
#pragma unroll 8
            for (int i = threadIdx.x; i < n; i += kDecodeThreads) dst[i] = __ldg(src + i);
          } else {
            const uint64_t* w = (const uint64_t*)((uintptr_t)p & ~(uintptr_t)7);
            const unsigned sh = (unsigned)((uintptr_t)p & 7) * 8;
#pragma unroll 8
            for (int i = threadIdx.x; i < n; i += kDecodeThreads) dst[i] = (__ldg(w + i) >> sh) | (__ldg(w + i + 1) << (64 - sh));
          }
        } else {
          uint32_t* dst = (uint32_t*)co.data + row0;
          if (((uintptr_t)p & 3) == 0) {
            const uint32_t* src = (const uint32_t*)p;
#pragma unroll 8
            for (int i = threadIdx.x; i < n; i += kDecodeThreads) dst[i] = __ldg(src + i);
          } else {
            const uint32_t* w = (const uint32_t*)((uintptr_t)p & ~(uintptr_t)3);
            const unsigned sh = (unsigned)((uintptr_t)p & 3) * 8;
#pragma unroll 8
            for (int i = threadIdx.x; i < n; i += kDecodeThreads) dst[i] = __funnelshift_r(__ldg(w + i), __ldg(w + i + 1), sh);
          }
        }
      }
    } else {
      // Fast path: the whole index stream is ONE bit-packed run (what this engine's encoder writes, and what parquet-mr /
      // pyarrow write for pages without long repeats): every index sits at a fixed bit offset, so all threads extract
      // in parallel with no run table and no barriers.
      if (threadIdx.x == 0) {
        uint32_t h = 0;
        int shift = 0;
        const uint8_t* q = p;
        while (q < pend) {
          const uint8_t b = *q++;
          h |= (uint32_t)(b & 0x7f) << shift;
          if (!(b & 0x80)) break;
          shift += 7;
          if (shift > 28) break;
        }
        const uint64_t groups = h >> 1;
        const bool single = (h & 1) && groups * 8 >= (uint64_t)n && q + groups * idx_bw <= pend;
        sm.flag = single ? (uint32_t)(q - p) : 0u;
      }
      __syncthreads();
      const uint32_t hdr_len = sm.flag;
      if (hdr_len) {
        const uint8_t* run = p + hdr_len;
        int done = 0;
        if (idx_bw >= 1 && idx_bw <= 16 && dict_in_smem && W != 1) {
          // One bit-packed group (8 indices = idx_bw bytes) per thread: five aligned words cover the group wherever it
          // starts, the eight indices come out of registers, the eight look-ups hit shared memory, and -- when the page
          // starts on a multiple of eight rows -- the eight 16-bit codes leave as one 16-byte store.  The per-value loop
          // below spends about 40 instructions and one exposed load latency per value.
          // The last two groups are left to it: a group's words may reach 19 bytes past its first byte.
          const int ngroups = n / 8 - 2;
          const uint64_t mask = (1ull << idx_bw) - 1;
          const bool wide_store = carry && ((row0 & 7) == 0);
          bool bad = false;
          for (int g = threadIdx.x; g < ngroups; g += kDecodeThreads) {
            const uint8_t* gp = run + (size_t)g * idx_bw;
            const uint32_t* w = (const uint32_t*)((uintptr_t)gp & ~(uintptr_t)3);
            const unsigned sh = (unsigned)((uintptr_t)gp & 3) * 8;
            const uint32_t x0 = __ldg(w), x1 = __ldg(w + 1), x2 = __ldg(w + 2), x3 = __ldg(w + 3), x4 = __ldg(w + 4);
            const uint64_t lo = (uint64_t)__funnelshift_r(x0, x1, sh) | ((uint64_t)__funnelshift_r(x1, x2, sh) << 32);
            const uint64_t hi = (uint64_t)__funnelshift_r(x2, x3, sh) | ((uint64_t)__funnelshift_r(x3, x4, sh) << 32);
            uint32_t code[8];
#pragma unroll
            for (int j = 0; j < 8; j++) {
              const uint32_t bit = (uint32_t)j * idx_bw;  // < 128
              uint64_t v;
              if (bit >= 64) v = hi >> (bit - 64);
              else v = (lo >> bit) | (bit ? (hi << (64 - bit)) : 0ull);
              const uint32_t ix = (uint32_t)(v & mask);
              bad = bad || ix >= dict_count;
              const uint32_t safe = ix < dict_count ? ix : 0u;
              code[j] = carry ? (uint32_t)dict16[safe] : 0u;
              if (!carry) store_value<W>(co.data, row0 + (int64_t)g * 8 + j, sm.dict[safe]);
            }
            if (carry) {
              uint16_t* out16 = (uint16_t*)co.data + row0 + (int64_t)g * 8;
              if (wide_store) {
                *reinterpret_cast<uint4*>(out16) = make_uint4(code[0] | (code[1] << 16), code[2] | (code[3] << 16),
                                                              code[4] | (code[5] << 16), code[6] | (code[7] << 16));
              } else {
#pragma unroll
                for (int j = 0; j < 8; j++) out16[j] = (uint16_t)code[j];
              }
            }
          }
          if (bad) set_error(d_error, DERR_DICT_INDEX, 0xfffffeu);
          done = ngroups > 0 ? ngroups * 8 : 0;
        }
#pragma unroll 8
        for (int i = done + threadIdx.x; i < n; i += kDecodeThreads)
          emit(row0 + i, dict_lookup(extract_bits(run, (uint64_t)i, idx_bw)));
        return;
      }
      for (int base = 0; base < n; base += kTileRows) {
        const uint32_t cnt = (uint32_t)min(kTileRows, n - base);
        bool ok = hybrid_decode_next(sm.idx, cnt, [&](uint32_t i, uint32_t v) {
          emit(row0 + base + i, dict_lookup(v));
        });
        if (!ok) {
          if (threadIdx.x == 0) set_error(d_error, DERR_OVERRUN, (uint32_t)pg.col);
          return;
        }
      }
    }
    return;
  }

  // ---- general path: definition levels select which rows carry a value ---------------------------------------------
  int64_t val_cursor = 0;  // dense values consumed so far
  for (int base = 0; base < n; base += kTileRows) {
    const uint32_t cnt = (uint32_t)min(kTileRows, n - base);
    bool ok = hybrid_decode_next(sm.def, cnt, [&](uint32_t i, uint32_t v) { sm.tile_valid[i] = (uint8_t)(v != 0); });
    __syncthreads();
    if (!ok) {
      if (threadIdx.x == 0) set_error(d_error, DERR_OVERRUN, (uint32_t)pg.col);
      return;
    }
    // exclusive positions of the valid rows: each thread owns kTileRows / blockDim consecutive rows
    constexpr int kPer = kTileRows / kDecodeThreads;
    uint32_t local = 0;
    const uint32_t t0 = threadIdx.x * kPer;
#pragma unroll
    for (int k = 0; k < kPer; k++) local += (t0 + k < cnt) ? sm.tile_valid[t0 + k] : 0;
    uint32_t total = 0;
    uint32_t pre = block_exclusive_scan(local, sm.warp_sums, &total);
    if (threadIdx.x == 0 && total < cnt) atomicOr(col_has_nulls, 1u);  // an actual null, not just a level stream
#pragma unroll
    for (int k = 0; k < kPer; k++) {
      if (t0 + k < cnt) {
        sm.tile_pos[t0 + k] = pre;
        pre += sm.tile_valid[t0 + k];
      }
    }
    __syncthreads();
    if (hybrid_values) {
      ok = hybrid_decode_next(sm.idx, total, [&](uint32_t j, uint32_t v) { sm.tile_idx[j] = v; });
      __syncthreads();
      if (!ok) {
        if (threadIdx.x == 0) set_error(d_error, DERR_OVERRUN, (uint32_t)pg.col);
        return;
      }
    } else {  // the tile's dense PLAIN values must lie inside the page
      const int64_t have = (int64_t)(pend - p), upto = val_cursor + total;
      if (W == 1 ? (upto + 7) / 8 > have : upto * SW > have) {
        if (threadIdx.x == 0) set_error(d_error, DERR_OVERRUN, (uint32_t)pg.col);
        return;
      }
    }
    for (uint32_t i = threadIdx.x; i < cnt; i += blockDim.x) {
      const bool valid = sm.tile_valid[i] != 0;
      uint64_t v = 0;
      if (valid) {
        const uint32_t pos = sm.tile_pos[i];
        if (hybrid_values) v = dict_lookup(sm.tile_idx[pos]);
        else if (W == 1) {
          const int64_t bit = val_cursor + pos;
          v = (p[bit >> 3] >> (bit & 7)) & 1;
        } else v = load_at(p, val_cursor + pos);
      }
      store_value<W>(co.data, row0 + base + i, v);
      co.valid[row0 + base + i] = valid ? 1 : 0;
    }
    val_cursor += total;
    __syncthreads();
  }
}

// ---- strings ---------------------------------------------------------------------------------------------------------
// PLAIN BYTE_ARRAY values are length-prefixed: where value i starts is known only after values 0..i-1 have been walked.  One
// thread walks a page (pages are walked in parallel with each other); every row gets a reference to its bytes inside the
// page -- the bytes themselves are not copied anywhere until the index pages are written.
__device__ __forceinline__ uint32_t load_u32_bytes(const uint8_t* p) {
  return (uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) | ((uint32_t)p[3] << 24);
}

__device__ void decode_byte_array_plain(const PageDesc& pg, const ColumnOut& co, uint32_t* col_has_nulls, uint32_t* d_error) {
  if (threadIdx.x != 0) return;
  atomicOr(col_has_nulls, 2u);  // not a dictionary page
  const int n = pg.num_values;
  const uint8_t* p = pg.data;
  const uint8_t* pend = pg.data + pg.size;
  const uint8_t *def_p = nullptr, *def_end = nullptr;
  if (n < 0 || pg.size < 0 || !locate_def_levels(pg, p, def_p, def_end)) {
    set_error(d_error, DERR_OVERRUN, (uint32_t)pg.col);
    return;
  }
  uint64_t* out = (uint64_t*)co.data + pg.first_row;
  uint8_t* valid = co.valid ? co.valid + pg.first_row : nullptr;
  // definition levels (bit width 1), walked serially alongside the values: run_left values of the current run remain
  uint32_t run_left = 0, run_val = 1, bit_pos = 0;
  const uint8_t* bits = nullptr;
  bool run_rle = true, saw_null = false;
  for (int i = 0; i < n; i++) {
    bool is_valid = true;
    if (def_p) {
      if (run_left == 0) {
        if (def_p >= def_end) {
          set_error(d_error, DERR_OVERRUN, (uint32_t)pg.col);
          return;
        }
        uint32_t h = 0;
        int shift = 0;
        while (def_p < def_end) {
          const uint8_t b = *def_p++;
          h |= (uint32_t)(b & 0x7f) << shift;
          if (!(b & 0x80)) break;
          shift += 7;
          if (shift > 28) break;
        }
        if (h & 1) {
          uint32_t groups = h >> 1;
          if ((uint64_t)groups > (uint64_t)(def_end - def_p)) groups = (uint32_t)(def_end - def_p);
          run_rle = false;
          run_left = groups * 8;
          bits = def_p;
          bit_pos = 0;
          def_p += groups;
        } else {
          run_rle = true;
          run_left = h >> 1;
          run_val = def_p < def_end ? (*def_p++ & 1u) : 0u;
        }
        if (run_left == 0) {
          set_error(d_error, DERR_OVERRUN, (uint32_t)pg.col);
          return;
        }
      }
      is_valid = run_rle ? run_val != 0 : ((bits[bit_pos >> 3] >> (bit_pos & 7)) & 1u) != 0;
      bit_pos++;
      run_left--;
    }
    uint64_t ref = 0;
    if (is_valid) {
      if (pend - p < 4) {
        set_error(d_error, DERR_OVERRUN, (uint32_t)pg.col);
        return;
      }
      const uint32_t len = load_u32_bytes(p);
      if ((uint64_t)len > (uint64_t)(pend - p - 4)) {
        set_error(d_error, DERR_OVERRUN, (uint32_t)pg.col);
        return;
      }
      if (len > kMaxStringLen) {
        set_error(d_error, DERR_STRING_TOO_LONG, (uint32_t)pg.col);
        return;
      }
      ref = string_ref(p + 4, len);
      p += 4 + (size_t)len;
    } else {
      saw_null = true;
    }
    out[i] = ref;
    if (valid) valid[i] = is_valid ? 1 : 0;
  }
  if (saw_null) atomicOr(col_has_nulls, 1u);
}

__global__ void k_build_string_dicts(const StringDictJob* __restrict__ jobs, int64_t n, uint32_t* d_error) {
  const int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  const StringDictJob job = jobs[j];
  const uint8_t* p = job.page;
  const uint8_t* pend = job.page + job.size;
  for (int i = 0; i < job.count; i++) {
    if (pend - p < 4) {
      set_error(d_error, DERR_OVERRUN, 0xfffffdu);
      return;
    }
    const uint32_t len = load_u32_bytes(p);
    if ((uint64_t)len > (uint64_t)(pend - p - 4)) {
      set_error(d_error, DERR_OVERRUN, 0xfffffdu);
      return;
    }
    if (len > kMaxStringLen) {
      set_error(d_error, DERR_STRING_TOO_LONG, 0xfffffdu);
      return;
    }
    job.refs[i] = string_ref(p + 4, len);
    p += 4 + (size_t)len;
  }
}

// a page lies outside every window of its file (launch_decode_pages): one binary search for the first window ending after
// the page's first row
__device__ __forceinline__ bool page_outside_windows(const PageDesc& pg, const int64_t* __restrict__ windows,
                                                     const int64_t* __restrict__ window_offsets) {
  int64_t lo = window_offsets[pg.file_index], hi = window_offsets[pg.file_index + 1];
  while (lo < hi) {
    const int64_t mid = lo + ((hi - lo) >> 1);
    if (windows[2 * mid + 1] <= pg.first_row) lo = mid + 1;
    else hi = mid;
  }
  return lo == window_offsets[pg.file_index + 1] || windows[2 * lo] >= pg.first_row + pg.num_values;
}

__global__ void __launch_bounds__(kDecodeThreads) k_decode_pages(const PageDesc* __restrict__ pages,
                                                                 const ColumnOut* __restrict__ cols,
                                                                 uint32_t* col_has_nulls,
                                                                 const int64_t* __restrict__ windows,
                                                                 const int64_t* __restrict__ window_offsets,
                                                                 uint32_t* d_error) {
  extern __shared__ __align__(16) uint8_t smem_raw[];
  DecodeShared& sm = *reinterpret_cast<DecodeShared*>(smem_raw);
  const PageDesc pg = pages[blockIdx.x];
  if (windows && page_outside_windows(pg, windows, window_offsets)) return;
  const ColumnOut co = cols[pg.col];
  if (co.skip || pg.conv != CONV_NONE) return;  // zero-copy column: read in place by the partition; converted: below
  switch (pg.phys_type) {
    case pq::INT64:
    case pq::DOUBLE: decode_page<8>(pg, co, col_has_nulls + pg.col, d_error, sm); break;
    case pq::INT32:
    case pq::FLOAT: decode_page<4>(pg, co, col_has_nulls + pg.col, d_error, sm); break;
    case pq::BOOLEAN: decode_page<1>(pg, co, col_has_nulls + pg.col, d_error, sm); break;
    case pq::BYTE_ARRAY:
      // dictionary-encoded strings: the dictionary has been turned into a table of 8-byte references (decode_sources), so
      // the page decodes like any dictionary page of 8-byte values; PLAIN pages are walked
      if (pg.encoding == pq::ENC_PLAIN) decode_byte_array_plain(pg, co, col_has_nulls + pg.col, d_error);
      else decode_page<8>(pg, co, col_has_nulls + pg.col, d_error, sm);
      break;
    default:
      if (threadIdx.x == 0) set_error(d_error, DERR_UNSUPPORTED_TYPE, (uint32_t)pg.phys_type);
  }
}

// The pages whose values are converted (Spark timestamps and decimals, ValueConv), one CTA per page as above.  A kernel of
// its own: the conversions inlined into k_decode_pages would raise its register count from 64 to 80 for every page.
__global__ void __launch_bounds__(kDecodeThreads) k_decode_converted_pages(const PageDesc* __restrict__ pages,
                                                                           const ColumnOut* __restrict__ cols,
                                                                           uint32_t* col_has_nulls,
                                                                           const int64_t* __restrict__ windows,
                                                                           const int64_t* __restrict__ window_offsets,
                                                                           uint32_t* d_error) {
  extern __shared__ __align__(16) uint8_t smem_raw[];
  DecodeShared& sm = *reinterpret_cast<DecodeShared*>(smem_raw);
  const PageDesc pg = pages[blockIdx.x];
  if (pg.conv == CONV_NONE) return;
  if (windows && page_outside_windows(pg, windows, window_offsets)) return;
  const ColumnOut co = cols[pg.col];
  // the column's width, whatever the stored type
  if (co.width == 8) decode_page<8, true>(pg, co, col_has_nulls + pg.col, d_error, sm);
  else decode_page<4, true>(pg, co, col_has_nulls + pg.col, d_error, sm);
}

}  // namespace

void launch_walk_pages(hs_ctx* ctx, const ChunkDesc* chunks, int n_chunks, int32_t* page_counts,
                       const int64_t* page_offsets, PageDesc* pages, uint32_t* d_error, int mode) {
  KernelScope _ks(ctx, "k_walk_pages");
  if (n_chunks == 0) return;
  const int threads = 64;
  k_walk_pages<<<(n_chunks + threads - 1) / threads, threads, 0, ctx->stream>>>(chunks, n_chunks, page_counts,
                                                                                page_offsets, pages, d_error, mode);
  HS_LAUNCH_CHECK(ctx);
}

void launch_classify_pages(hs_ctx* ctx, const PageDesc* pages, int64_t n_pages, uint32_t* col_flags, int zc_tile_rows) {
  KernelScope _ks(ctx, "k_classify_pages");
  if (n_pages == 0) return;
  k_classify_pages<<<(unsigned)ceil_div(n_pages, 128), 128, 0, ctx->stream>>>(pages, n_pages, col_flags, zc_tile_rows);
  HS_LAUNCH_CHECK(ctx);
}

void launch_build_string_dicts(hs_ctx* ctx, const StringDictJob* jobs, int64_t n, uint32_t* d_error) {
  KernelScope _ks(ctx, "k_build_string_dicts");
  if (n == 0) return;
  k_build_string_dicts<<<(unsigned)ceil_div(n, 64), 64, 0, ctx->stream>>>(jobs, n, d_error);
  HS_LAUNCH_CHECK(ctx);
}

void launch_fill_zc_tiles(hs_ctx* ctx, const PageDesc* pages, int64_t n_pages, ZcTile* const* tile_src, int zc_tile_rows,
                          int64_t nrows) {
  KernelScope _ks(ctx, "k_fill_zc_tiles");
  if (n_pages == 0) return;
  k_fill_zc_tiles<<<(unsigned)n_pages, 32, 0, ctx->stream>>>(pages, tile_src, zc_tile_rows, nrows);
  HS_LAUNCH_CHECK(ctx);
}

void launch_decode_pages(hs_ctx* ctx, const PageDesc* pages, int64_t n_pages, const ColumnOut* cols,
                         uint32_t* col_has_nulls, const int64_t* windows, const int64_t* window_offsets, uint32_t* d_error,
                         bool any_converted) {
  if (n_pages == 0) return;
  static DeviceOnce attr_set_once;
  bool& attr_set = attr_set_once(ctx->device);
  if (!attr_set) {
    HS_CUDA(cudaFuncSetAttribute(k_decode_pages, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(DecodeShared)));
    HS_CUDA(cudaFuncSetAttribute(k_decode_converted_pages, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(DecodeShared)));
    attr_set = true;
  }
  {
    KernelScope _ks(ctx, "k_decode_pages");
    k_decode_pages<<<(unsigned)n_pages, kDecodeThreads, sizeof(DecodeShared), ctx->stream>>>(pages, cols, col_has_nulls,
                                                                                             windows, window_offsets, d_error);
    HS_LAUNCH_CHECK(ctx);
  }
  if (any_converted) {
    KernelScope _ks(ctx, "k_decode_converted_pages");
    k_decode_converted_pages<<<(unsigned)n_pages, kDecodeThreads, sizeof(DecodeShared), ctx->stream>>>(pages, cols, col_has_nulls,
                                                                                                       windows, window_offsets,
                                                                                                       d_error);
    HS_LAUNCH_CHECK(ctx);
  }
}

}  // namespace hs
