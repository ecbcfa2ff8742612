// parquet_meta.h -- host-side Parquet metadata: footer parse (source tables, index files) and footer / page-header
// serialisation (index files).  Format per apache/parquet-format parquet.thrift; the reference delegates all of this
// to parquet-mr through Spark (index/DataFrameWriterExtensions.scala:58-67 on the write side,
// covering/CoveringIndexTrait.scala:82-84 and CoveringIndexRuleUtils.scala:113-123 on the read side).
#pragma once
#include <cstdint>
#include <map>
#include <string>
#include <vector>

#include "hs_common.h"
#include "thrift_compact.h"

namespace hs {
namespace pq {

enum PhysType : int32_t { BOOLEAN = 0, INT32 = 1, INT64 = 2, INT96 = 3, FLOAT = 4, DOUBLE = 5, BYTE_ARRAY = 6, FIXED_LEN_BYTE_ARRAY = 7 };
enum Repetition : int32_t { REQUIRED = 0, OPTIONAL = 1, REPEATED = 2 };
enum Encoding : int32_t { ENC_PLAIN = 0, ENC_PLAIN_DICTIONARY = 2, ENC_RLE = 3, ENC_BIT_PACKED = 4, ENC_RLE_DICTIONARY = 8 };
enum Codec : int32_t { UNCOMPRESSED = 0, SNAPPY = 1, GZIP = 2, LZ4 = 5, LZ4_RAW = 7 };
enum PageType : int32_t { DATA_PAGE = 0, INDEX_PAGE = 1, DICTIONARY_PAGE = 2, DATA_PAGE_V2 = 3 };

struct SchemaColumn {
  std::string name;
  int32_t type = -1;          // PhysType
  int32_t type_length = 0;
  int32_t repetition = REQUIRED;
  int32_t converted_type = -1;  // carried through to the index file so Spark sees the same SQL type
  int32_t scale = -1, precision = -1;
  int32_t num_children = 0;
  // LogicalType TIMESTAMP's unit (SchemaElement field 10): 1 millis, 2 micros, 3 nanos; 0 when the leaf has none.  NANOS
  // has no converted type, so this is the only place it shows.
  int32_t time_unit = 0;
};

// ConvertedType values the engine reads
enum Converted : int32_t { CT_DECIMAL = 5, CT_DATE = 6, CT_TIMESTAMP_MILLIS = 9, CT_TIMESTAMP_MICROS = 10 };

struct ColumnChunkMeta {
  int32_t type = -1;
  int32_t codec = 0;
  int64_t num_values = 0;
  int64_t total_uncompressed_size = 0;
  int64_t total_compressed_size = 0;
  int64_t data_page_offset = 0;
  int64_t dictionary_page_offset = -1;
  // byte range of the chunk in the file
  int64_t start() const {
    return (dictionary_page_offset > 0 && dictionary_page_offset < data_page_offset) ? dictionary_page_offset
                                                                                      : data_page_offset;
  }
};

struct RowGroupMeta {
  int64_t num_rows = 0;
  std::vector<ColumnChunkMeta> columns;
};

struct FileMeta {
  int64_t num_rows = 0;
  std::vector<SchemaColumn> columns;  // flat leaf columns (root stripped)
  bool nested = false;                // any column with children -> only flat columns are addressable
  std::vector<RowGroupMeta> row_groups;
  std::string created_by;
  std::vector<std::pair<std::string, std::string>> key_values;
};

// A list header read from an untrusted footer: every element occupies at least one byte, so a count larger than what is
// left of the buffer is corrupt (a mutated footer must not make the parser allocate billions of elements).
inline uint32_t read_list_header(thrift::Reader& r, uint8_t& etype) {
  const uint32_t n = r.list(etype);
  if (r.bad || (uint64_t)n > (uint64_t)(r.end - r.p)) {
    r.bad = true;
    return 0;
  }
  return n;
}

inline std::string read_string(thrift::Reader& r) {
  uint64_t n = r.varint();
  if ((uint64_t)(r.end - r.p) < n) {
    r.bad = true;
    return std::string();
  }
  std::string s((const char*)r.p, (size_t)n);
  r.p += n;
  return s;
}

// LogicalType union (SchemaElement field 10): DECIMAL and TIMESTAMP are mapped onto the converted type they stand for, so
// that a leaf written with the logical type only reads like one written with both (pyarrow writes both, except for NANOS)
inline void parse_logical_type(thrift::Reader& r, SchemaColumn& c) {
  int16_t fid = 0;
  for (;;) {
    uint8_t t = r.field(fid);
    if (t == thrift::T_STOP || r.bad) break;
    if (t != thrift::T_STRUCT || (fid != 5 && fid != 8)) {
      r.skip(t);
      continue;
    }
    int32_t scale = 0, precision = -1, unit = 0;
    int16_t f2 = 0;
    for (;;) {
      uint8_t t2 = r.field(f2);
      if (t2 == thrift::T_STOP || r.bad) break;
      if (fid == 5 && f2 == 1) scale = (int32_t)r.zigzag();
      else if (fid == 5 && f2 == 2) precision = (int32_t)r.zigzag();
      else if (fid == 8 && f2 == 2 && t2 == thrift::T_STRUCT) {  // TimeUnit union: the set member's id is the unit
        int16_t f3 = 0;
        for (;;) {
          uint8_t t3 = r.field(f3);
          if (t3 == thrift::T_STOP || r.bad) break;
          unit = f3;
          r.skip(t3);
        }
      } else r.skip(t2);
    }
    if (fid == 5) {
      if (c.converted_type < 0) c.converted_type = CT_DECIMAL;
      if (c.precision < 0) c.precision = precision, c.scale = scale;
    } else {
      c.time_unit = unit;
      if (c.converted_type < 0 && unit == 1) c.converted_type = CT_TIMESTAMP_MILLIS;
      if (c.converted_type < 0 && unit == 2) c.converted_type = CT_TIMESTAMP_MICROS;
    }
  }
}

inline void parse_schema_element(thrift::Reader& r, SchemaColumn& c) {
  int16_t fid = 0;
  for (;;) {
    uint8_t t = r.field(fid);
    if (t == thrift::T_STOP || r.bad) break;
    switch (fid) {
      case 1: c.type = (int32_t)r.zigzag(); break;
      case 2: c.type_length = (int32_t)r.zigzag(); break;
      case 3: c.repetition = (int32_t)r.zigzag(); break;
      case 4: c.name = read_string(r); break;
      case 5: c.num_children = (int32_t)r.zigzag(); break;
      case 6: c.converted_type = (int32_t)r.zigzag(); break;
      case 7: c.scale = (int32_t)r.zigzag(); break;
      case 8: c.precision = (int32_t)r.zigzag(); break;
      case 10:
        if (t == thrift::T_STRUCT) parse_logical_type(r, c);
        else r.skip(t);
        break;
      default: r.skip(t);
    }
  }
}

inline void parse_column_meta(thrift::Reader& r, ColumnChunkMeta& m) {
  int16_t fid = 0;
  for (;;) {
    uint8_t t = r.field(fid);
    if (t == thrift::T_STOP || r.bad) break;
    switch (fid) {
      case 1: m.type = (int32_t)r.zigzag(); break;
      case 4: m.codec = (int32_t)r.zigzag(); break;
      case 5: m.num_values = r.zigzag(); break;
      case 6: m.total_uncompressed_size = r.zigzag(); break;
      case 7: m.total_compressed_size = r.zigzag(); break;
      case 9: m.data_page_offset = r.zigzag(); break;
      case 11: m.dictionary_page_offset = r.zigzag(); break;
      default: r.skip(t);
    }
  }
}

inline void parse_column_chunk(thrift::Reader& r, ColumnChunkMeta& m) {
  int16_t fid = 0;
  for (;;) {
    uint8_t t = r.field(fid);
    if (t == thrift::T_STOP || r.bad) break;
    if (fid == 3 && t == thrift::T_STRUCT) parse_column_meta(r, m);
    else r.skip(t);
  }
}

inline void parse_row_group(thrift::Reader& r, RowGroupMeta& g) {
  int16_t fid = 0;
  for (;;) {
    uint8_t t = r.field(fid);
    if (t == thrift::T_STOP || r.bad) break;
    if (fid == 1 && t == thrift::T_LIST) {
      uint8_t et;
      uint32_t n = read_list_header(r, et);
      g.columns.resize(n);
      for (uint32_t i = 0; i < n && !r.bad; i++) parse_column_chunk(r, g.columns[i]);
    } else if (fid == 3) {
      g.num_rows = r.zigzag();
    } else {
      r.skip(t);
    }
  }
}

// Parses a serialised FileMetaData (the `flen` bytes that precede the trailing length + magic).
inline FileMeta parse_footer_bytes(const uint8_t* footer, uint32_t flen, const char* what) {
  thrift::Reader r(footer, footer + flen);
  FileMeta fm;
  std::vector<SchemaColumn> elems;
  int16_t fid = 0;
  for (;;) {
    uint8_t t = r.field(fid);
    if (t == thrift::T_STOP || r.bad) break;
    switch (fid) {
      case 2: {
        uint8_t et;
        uint32_t n = read_list_header(r, et);
        elems.resize(n);
        for (uint32_t i = 0; i < n && !r.bad; i++) parse_schema_element(r, elems[i]);
        break;
      }
      case 3: fm.num_rows = r.zigzag(); break;
      case 4: {
        uint8_t et;
        uint32_t n = read_list_header(r, et);
        fm.row_groups.resize(n);
        for (uint32_t i = 0; i < n && !r.bad; i++) parse_row_group(r, fm.row_groups[i]);
        break;
      }
      case 5: {
        uint8_t et;
        uint32_t n = read_list_header(r, et);
        for (uint32_t i = 0; i < n && !r.bad; i++) {
          std::string k, v;
          int16_t f2 = 0;
          for (;;) {
            uint8_t t2 = r.field(f2);
            if (t2 == thrift::T_STOP || r.bad) break;
            if (f2 == 1) k = read_string(r);
            else if (f2 == 2) v = read_string(r);
            else r.skip(t2);
          }
          fm.key_values.emplace_back(std::move(k), std::move(v));
        }
        break;
      }
      case 6: fm.created_by = read_string(r); break;
      default: r.skip(t);
    }
  }
  if (r.bad || elems.empty()) fail(HS_EFORMAT, "%s: corrupt Parquet footer", what);
  // flatten: root element then leaves; a child with children marks the schema nested
  for (size_t i = 1; i < elems.size(); i++) {
    if (elems[i].num_children > 0) fm.nested = true;
    fm.columns.push_back(elems[i]);
  }
  if (!fm.nested) {
    for (auto& g : fm.row_groups)
      if (g.columns.size() != fm.columns.size())
        fail(HS_EFORMAT, "%s: row group has %zu column chunks for %zu columns", what, g.columns.size(),
             fm.columns.size());
  }
  return fm;
}

// Parses the footer of a whole-file image (host memory).  `what` names the file in error messages.
inline FileMeta parse_footer(const uint8_t* file, uint64_t size, const char* what) {
  if (size < 12 || memcmp(file, "PAR1", 4) != 0 || memcmp(file + size - 4, "PAR1", 4) != 0)
    fail(HS_EFORMAT, "%s: not a Parquet file (bad magic or encrypted footer)", what);
  uint32_t flen;
  memcpy(&flen, file + size - 8, 4);
  if ((uint64_t)flen + 12 > size) fail(HS_EFORMAT, "%s: footer length %u exceeds file size", what, flen);
  return parse_footer_bytes(file + size - 8 - flen, flen, what);
}

// ---- writing ---------------------------------------------------------------------------------------------

// v1 data page header for `num_values` values: PLAIN (or dictionary) values, RLE definition levels.
// compressed_bytes < 0: the page is stored as it is (compressed size == uncompressed size)
inline void write_data_page_header(std::vector<uint8_t>& out, int32_t page_bytes, int32_t num_values, int32_t encoding,
                                   int32_t compressed_bytes = -1) {
  thrift::Writer w;
  w.struct_begin();
  w.f_i32(1, DATA_PAGE);
  w.f_i32(2, page_bytes);
  w.f_i32(3, compressed_bytes < 0 ? page_bytes : compressed_bytes);
  w.f_struct_begin(5);
  w.f_i32(1, num_values);
  w.f_i32(2, encoding);
  w.f_i32(3, ENC_RLE);
  w.f_i32(4, ENC_RLE);  // parquet-mr writes BIT_PACKED here for flat schemas; unused either way (max rep level 0)
  w.struct_end();
  w.struct_end();
  out.insert(out.end(), w.buf.begin(), w.buf.end());
}

inline void write_dict_page_header(std::vector<uint8_t>& out, int32_t page_bytes, int32_t num_values, int32_t compressed_bytes = -1) {
  thrift::Writer w;
  w.struct_begin();
  w.f_i32(1, DICTIONARY_PAGE);
  w.f_i32(2, page_bytes);
  w.f_i32(3, compressed_bytes < 0 ? page_bytes : compressed_bytes);
  w.f_struct_begin(7);
  w.f_i32(1, num_values);
  w.f_i32(2, ENC_PLAIN_DICTIONARY);
  w.struct_end();
  w.struct_end();
  out.insert(out.end(), w.buf.begin(), w.buf.end());
}

// RLE/bit-packed hybrid block for `n` definition levels all equal to 1, with the v1 4-byte length prefix.
inline void write_all_valid_def_levels(std::vector<uint8_t>& out, int64_t n) {
  uint8_t tmp[16];
  int len = 0;
  uint64_t h = (uint64_t)n << 1;  // RLE run header
  while (h >= 0x80) {
    tmp[len++] = (uint8_t)(h | 0x80);
    h >>= 7;
  }
  tmp[len++] = (uint8_t)h;
  tmp[len++] = 1;  // run value, bit width 1 -> one byte
  uint32_t l32 = (uint32_t)len;
  const uint8_t* lp = (const uint8_t*)&l32;
  out.insert(out.end(), lp, lp + 4);
  out.insert(out.end(), tmp, tmp + len);
}

// Definition levels for `n` non-null values as several RLE runs of ones.  Splitting the single run (n ones) into extra
// runs is a legal RLE/bit-packed hybrid encoding; each extra run of 1 value costs 2 bytes and each extra run of 64
// values costs 3 bytes, which lets the writer choose the block length so that the values that follow start 8-byte
// aligned in the file image (the GPU then writes page bodies with full-width aligned stores).
inline void write_def_levels_runs(std::vector<uint8_t>& out, int64_t n, int small_runs, int medium_runs) {
  std::vector<uint8_t> body;
  auto run = [&](uint64_t count) {
    uint64_t h = count << 1;
    while (h >= 0x80) {
      body.push_back((uint8_t)(h | 0x80));
      h >>= 7;
    }
    body.push_back((uint8_t)h);
    body.push_back(1);
  };
  run((uint64_t)(n - small_runs - 64 * (int64_t)medium_runs));
  for (int i = 0; i < small_runs; i++) run(1);
  for (int i = 0; i < medium_runs; i++) run(64);
  uint32_t l32 = (uint32_t)body.size();
  const uint8_t* lp = (const uint8_t*)&l32;
  out.insert(out.end(), lp, lp + 4);
  out.insert(out.end(), body.begin(), body.end());
}

// Appends [page header][definition levels] for a PLAIN v1 data page of `n` non-null W-byte values that starts at file
// offset `page_offset`, choosing the run split so that the values start 8-byte aligned when n allows it.
inline void write_plain_page_prefix(std::vector<uint8_t>& out, uint64_t page_offset, int64_t n, int W) {
  // the winning split depends only on (n, W, page_offset mod 8): memoised, since an index has ~40 k pages of a few shapes
  struct Key {
    int64_t n;
    int w, mod;
    bool operator<(const Key& o) const { return n != o.n ? n < o.n : (w != o.w ? w < o.w : mod < o.mod); }
  };
  static thread_local std::map<Key, std::pair<int, int>> memo;  // -> (small, medium), (-1,-1) = no aligned split
  const Key key{n, W, (int)(page_offset % 8)};
  auto it = memo.find(key);
  if (it == memo.end()) {
    std::pair<int, int> best{-1, -1};
    for (int extra = 0; extra <= 24 && best.first < 0; extra++) {  // extra bytes over the single-run encoding
      for (int medium = 0; 3 * medium <= extra; medium++) {
        const int rest = extra - 3 * medium;
        if (rest % 2) continue;
        const int small = rest / 2;
        if (n - small - 64 * (int64_t)medium < 1) continue;
        std::vector<uint8_t> defs, hdr;
        write_def_levels_runs(defs, n, small, medium);
        write_data_page_header(hdr, (int32_t)(defs.size() + (size_t)n * W), (int32_t)n, ENC_PLAIN);
        if ((page_offset + hdr.size() + defs.size()) % 8 == 0) {
          best = {small, medium};
          break;
        }
      }
    }
    it = memo.emplace(key, best).first;
  }
  // the serialised prefix itself is cached too: an index has tens of thousands of identical full pages
  static thread_local std::map<Key, std::vector<uint8_t>> bytes_memo;
  auto bt = bytes_memo.find(key);
  if (bt == bytes_memo.end()) {
    std::vector<uint8_t> pre, defs;
    if (it->second.first >= 0) write_def_levels_runs(defs, n, it->second.first, it->second.second);
    else write_all_valid_def_levels(defs, n);  // tiny page: the GPU falls back to its unaligned store path
    write_data_page_header(pre, (int32_t)(defs.size() + (size_t)n * W), (int32_t)n, ENC_PLAIN);
    pre.insert(pre.end(), defs.begin(), defs.end());
    bt = bytes_memo.emplace(key, std::move(pre)).first;
  }
  out.insert(out.end(), bt->second.begin(), bt->second.end());
}

// [page header][definition levels] for a PLAIN v1 BOOLEAN data page of `n` non-null values, as parquet-mr writes it: one
// RLE run of ones, then ceil(n / 8) bytes of values bit-packed LSB first (written by the GPU)
inline void write_bool_page_prefix(std::vector<uint8_t>& out, int64_t n) {
  std::vector<uint8_t> defs;
  write_all_valid_def_levels(defs, n);
  write_data_page_header(out, (int32_t)(defs.size() + (size_t)(n + 7) / 8), (int32_t)n, ENC_PLAIN);
  out.insert(out.end(), defs.begin(), defs.end());
}

// [page header][4-byte length][bit-packed run header] for a v1 data page of `n` rows whose definition levels are written as
// ONE bit-packed run of ceil(n/8) groups (the bits themselves are written by the GPU right after this prefix) followed by
// `non_null` dense PLAIN values.
inline void write_nullable_page_prefix(std::vector<uint8_t>& out, int64_t n, int64_t non_null, int W) {
  const uint64_t groups = (uint64_t)(n + 7) / 8;
  uint8_t hv[10];
  int hl = 0;
  uint64_t h = (groups << 1) | 1;
  while (h >= 0x80) {
    hv[hl++] = (uint8_t)(h | 0x80);
    h >>= 7;
  }
  hv[hl++] = (uint8_t)h;
  const uint32_t def_len = (uint32_t)(hl + groups);
  write_data_page_header(out, (int32_t)(4 + def_len + (size_t)non_null * W), (int32_t)n, ENC_PLAIN);
  const uint8_t* lp = (const uint8_t*)&def_len;
  out.insert(out.end(), lp, lp + 4);
  out.insert(out.end(), hv, hv + hl);
}

// the same for a page whose values take `value_bytes` bytes in all (PLAIN BYTE_ARRAY: [u32 length][bytes] per non-null value)
inline void write_nullable_page_prefix_bytes(std::vector<uint8_t>& out, int64_t n, uint64_t value_bytes) {
  const uint64_t groups = (uint64_t)(n + 7) / 8;
  uint8_t hv[10];
  int hl = 0;
  uint64_t h = (groups << 1) | 1;
  while (h >= 0x80) {
    hv[hl++] = (uint8_t)(h | 0x80);
    h >>= 7;
  }
  hv[hl++] = (uint8_t)h;
  const uint32_t def_len = (uint32_t)(hl + groups);
  write_data_page_header(out, (int32_t)(4 + def_len + value_bytes), (int32_t)n, ENC_PLAIN);
  const uint8_t* lp = (const uint8_t*)&def_len;
  out.insert(out.end(), lp, lp + 4);
  out.insert(out.end(), hv, hv + hl);
}

// [page header][all-valid definition levels][bit width byte][bit-packed run header] of a PLAIN_DICTIONARY v1 data page of
// `n` non-null values whose indices are written as ONE bit-packed run of ceil(n/8) groups of `bw` bits (the packed bytes
// follow this prefix).
inline void write_dict_data_page_prefix(std::vector<uint8_t>& real_out, int64_t n, uint32_t bw) {
  static thread_local std::map<std::pair<int64_t, uint32_t>, std::vector<uint8_t>> memo;
  auto it = memo.find({n, bw});
  if (it != memo.end()) {
    real_out.insert(real_out.end(), it->second.begin(), it->second.end());
    return;
  }
  std::vector<uint8_t> out;
  std::vector<uint8_t> defs;
  write_all_valid_def_levels(defs, n);
  const uint64_t groups = (uint64_t)(n + 7) / 8;
  uint8_t hv[10];
  int hl = 0;
  uint64_t h = (groups << 1) | 1;
  while (h >= 0x80) {
    hv[hl++] = (uint8_t)(h | 0x80);
    h >>= 7;
  }
  hv[hl++] = (uint8_t)h;
  write_data_page_header(out, (int32_t)(defs.size() + 1 + hl + groups * bw), (int32_t)n, ENC_PLAIN_DICTIONARY);
  out.insert(out.end(), defs.begin(), defs.end());
  out.push_back((uint8_t)bw);
  out.insert(out.end(), hv, hv + hl);
  real_out.insert(real_out.end(), out.begin(), out.end());
  memo.emplace(std::make_pair(n, bw), std::move(out));
}

struct OutChunk {
  int32_t type;
  int64_t num_values;
  int64_t total_size;       // bytes of all pages incl. headers, as stored (compressed)
  int64_t total_uncompressed = -1;  // the same with every page uncompressed (-1: equal to total_size)
  int32_t codec = UNCOMPRESSED;
  int64_t data_page_offset; // absolute file offset of the first data page header
  int64_t dictionary_page_offset = -1;
  bool has_dictionary = false;
  int64_t null_count = -1;
  bool has_minmax = false;
  uint8_t min_le[8] = {0}, max_le[8] = {0};  // little-endian plain-encoded min/max (fixed-width types)
  int32_t value_width = 0;
};

struct OutRowGroup {
  int64_t num_rows;
  int64_t total_byte_size;        // uncompressed
  int64_t total_compressed = -1;  // -1: equal to total_byte_size
  int64_t file_offset;
  std::vector<OutChunk> chunks;
};

// Where the min / max statistics of a chunk sit inside the serialised footer (deprecated max/min + max_value/min_value).
struct StatSlot {
  int32_t row_group, column, width;
  size_t max_off[2], min_off[2];
};

// Serialises FileMetaData.  `spark_schema_json` is stored under org.apache.spark.sql.parquet.row.metadata exactly as
// Spark's ParquetWriteSupport does, so Spark reads the index with the same StructType it was built from.
inline std::vector<uint8_t> write_footer(const std::vector<SchemaColumn>& cols, const std::vector<OutRowGroup>& rgs,
                                         int64_t num_rows, const std::string& spark_schema_json,
                                         std::vector<StatSlot>* stat_slots = nullptr) {
  thrift::Writer w;
  w.struct_begin();
  w.f_i32(1, 1);  // version
  w.f_list_begin(2, thrift::T_STRUCT, (uint32_t)cols.size() + 1);
  w.struct_begin();  // root
  w.f_string(4, "spark_schema");
  w.f_i32(5, (int32_t)cols.size());
  w.struct_end();
  for (auto& c : cols) {
    w.struct_begin();
    w.f_i32(1, c.type);
    if (c.type == FIXED_LEN_BYTE_ARRAY) w.f_i32(2, c.type_length);
    w.f_i32(3, c.repetition);
    w.f_string(4, c.name);
    if (c.converted_type >= 0) w.f_i32(6, c.converted_type);
    if (c.scale >= 0) w.f_i32(7, c.scale);
    if (c.precision >= 0) w.f_i32(8, c.precision);
    w.struct_end();
  }
  w.f_i64(3, num_rows);
  w.f_list_begin(4, thrift::T_STRUCT, (uint32_t)rgs.size());
  for (size_t gi = 0; gi < rgs.size(); gi++) {
    auto& g = rgs[gi];
    w.struct_begin();
    w.f_list_begin(1, thrift::T_STRUCT, (uint32_t)g.chunks.size());
    for (size_t ci = 0; ci < g.chunks.size(); ci++) {
      auto& ch = g.chunks[ci];
      w.struct_begin();
      w.f_i64(2, ch.has_dictionary ? ch.dictionary_page_offset : ch.data_page_offset);  // file_offset
      w.f_struct_begin(3);
      w.f_i32(1, ch.type);
      if (ch.has_dictionary) {
        w.f_list_begin(2, thrift::T_I32, 3);
        w.zigzag(ENC_PLAIN_DICTIONARY);
        w.zigzag(ENC_PLAIN);
        w.zigzag(ENC_RLE);
      } else {
        w.f_list_begin(2, thrift::T_I32, 2);
        w.zigzag(ENC_PLAIN);
        w.zigzag(ENC_RLE);
      }
      w.f_list_begin(3, thrift::T_BINARY, 1);
      w.string_elem(cols[ci].name);
      w.f_i32(4, ch.codec);
      w.f_i64(5, ch.num_values);
      w.f_i64(6, ch.total_uncompressed >= 0 ? ch.total_uncompressed : ch.total_size);
      w.f_i64(7, ch.total_size);
      w.f_i64(9, ch.data_page_offset);
      if (ch.has_dictionary) w.f_i64(11, ch.dictionary_page_offset);
      if (ch.null_count >= 0 || ch.has_minmax) {
        w.f_struct_begin(12);
        StatSlot slot;
        slot.row_group = (int32_t)gi;
        slot.column = (int32_t)ci;
        slot.width = ch.value_width;
        if (ch.has_minmax) {
          slot.max_off[0] = w.f_binary(1, ch.max_le, ch.value_width);
          slot.min_off[0] = w.f_binary(2, ch.min_le, ch.value_width);
        }
        if (ch.null_count >= 0) w.f_i64(3, ch.null_count);
        if (ch.has_minmax) {
          slot.max_off[1] = w.f_binary(5, ch.max_le, ch.value_width);
          slot.min_off[1] = w.f_binary(6, ch.min_le, ch.value_width);
          if (stat_slots) stat_slots->push_back(slot);
        }
        w.struct_end();
      }
      w.struct_end();
      w.struct_end();
    }
    w.f_i64(2, g.total_byte_size);
    w.f_i64(3, g.num_rows);
    w.f_i64(5, g.file_offset);
    w.f_i64(6, g.total_compressed >= 0 ? g.total_compressed : g.total_byte_size);
    w.struct_end();
  }
  w.f_list_begin(5, thrift::T_STRUCT, 2);
  w.struct_begin();
  w.f_string(1, "org.apache.spark.version");
  w.f_string(2, "3.1.1");
  w.struct_end();
  w.struct_begin();
  w.f_string(1, "org.apache.spark.sql.parquet.row.metadata");
  w.f_string(2, spark_schema_json);
  w.struct_end();
  w.f_string(6, "hyperspace_b200 version 0.1.0 (build sm_90a)");
  w.struct_end();
  return std::move(w.buf);
}

// Spark SQL type name of a Parquet leaf (ParquetToSparkSchemaConverter) for the row.metadata JSON.
inline std::string spark_type_name(const SchemaColumn& c) {
  if (c.converted_type == CT_DECIMAL)
    return "decimal(" + std::to_string(c.precision) + "," + std::to_string(c.scale < 0 ? 0 : c.scale) + ")";
  switch (c.type) {
    case BOOLEAN: return "boolean";
    case INT96: return "timestamp";
    case INT32:
      if (c.converted_type == 6) return "date";
      if (c.converted_type == 15) return "byte";
      if (c.converted_type == 16) return "short";
      return "integer";
    case INT64:
      if (c.converted_type == 9 || c.converted_type == 10) return "timestamp";
      return "long";
    case FLOAT: return "float";
    case DOUBLE: return "double";
    case BYTE_ARRAY: return c.converted_type == 0 ? "string" : "binary";
    default: return "binary";
  }
}

inline std::string spark_schema_json(const std::vector<SchemaColumn>& cols) {
  std::string s = "{\"type\":\"struct\",\"fields\":[";
  for (size_t i = 0; i < cols.size(); i++) {
    if (i) s += ",";
    s += "{\"name\":\"";
    for (char ch : cols[i].name) {
      if (ch == '"' || ch == '\\') s += '\\';
      s += ch;
    }
    s += "\",\"type\":\"";
    s += spark_type_name(cols[i]);
    s += "\",\"nullable\":true,\"metadata\":{}}";
  }
  s += "]}";
  return s;
}

}  // namespace pq
}  // namespace hs
