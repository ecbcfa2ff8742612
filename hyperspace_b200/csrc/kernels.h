// kernels.h -- host-callable launchers of the CUDA kernels (one .cu per stage).
#pragma once
#include <functional>

#include "column_compare.h"
#include "hs_common.h"
#include "string_match.h"

namespace hs {

// ---- Parquet decode (parquet_decode.cu) ---------------------------------------------------------------------------
// How the decoder turns a stored value into the value the engine keeps for Spark's TimestampType / DecimalType
// (engine.cu: source_type_of decides it per source column chunk).  Converted pages take the value path: never read in
// place, never late-materialised.
enum ValueConv : int32_t {
  CONV_NONE = 0,
  CONV_INT96 = 1,   // INT96 (8 B nanos of day, 4 B Julian day) -> int64 micros since the epoch; before 1900: DERR_SPARK_RANGE
  CONV_MILLIS = 2,  // INT64 TIMESTAMP_MILLIS -> micros (x 1000); overflow: DERR_SPARK_RANGE
  CONV_FLBA = 3,    // FIXED_LEN_BYTE_ARRAY decimal: big-endian two's complement -> int32 / int64 unscaled; DERR_DECIMAL_WIDTH
  CONV_NARROW = 4,  // INT64 decimal(p <= 9) -> int32 unscaled; DERR_DECIMAL_WIDTH when it does not fit
};
struct ChunkDesc {          // one per (file, row group, projected column)
  const uint8_t* data;      // device pointer to the first page header of the chunk
  uint64_t size;            // chunk bytes
  int64_t num_values;       // values (rows) in the chunk
  int64_t row_base;         // global row index of the row group's first row
  int32_t col;              // projected column index
  int32_t phys_type;        // pq::PhysType
  int32_t max_def;          // 0 (required) or 1 (optional)
  int32_t file_index;
  int32_t codec;            // pq::Codec of the chunk (UNCOMPRESSED, SNAPPY, GZIP, LZ4 or LZ4_RAW)
  int32_t conv;             // ValueConv
  int32_t type_length;      // FIXED_LEN_BYTE_ARRAY: bytes per value
  int32_t pad;
};

struct PageDesc {           // one per data page
  const uint8_t* data;      // page body
  const uint8_t* dict;      // dictionary page body (PLAIN values) or nullptr
  int64_t first_row;        // global row index of the page's first value
  int32_t dict_count;
  int32_t size;             // body bytes
  int32_t num_values;
  int32_t encoding;         // pq::Encoding of the values
  int32_t page_type;        // DATA_PAGE / DATA_PAGE_V2
  int32_t def_bytes;        // v2: definition_levels_byte_length, v1: -1 (length-prefixed block)
  int32_t rep_bytes;        // v2
  int32_t col, phys_type, max_def;
  int32_t file_index;
  int32_t uncompressed_size;  // body bytes after decompression (== size for stored pages)
  // compressed chunks only: the chunk's dictionary page as stored, and whether this page / the dictionary is compressed
  int32_t dict_size, dict_uncompressed_size;
  int32_t is_compressed;      // this page's values are compressed with the chunk's codec
  int32_t codec;
  int32_t chunk;              // index of the column chunk (ChunkDesc) the page belongs to
  int32_t conv;               // ValueConv of the chunk
  int32_t type_length;        // FIXED_LEN_BYTE_ARRAY: bytes per value
};

struct ColumnOut {          // decoded column destination
  void* data;               // num_rows values of `width` bytes (row order); carry != 0: one uint16 code per row
  uint8_t* valid;           // one byte per row (pre-set to 1) or nullptr for required columns
  int32_t width;
  int32_t type;             // HS_TYPE_*
  // Late-materialised dictionary column (carry != 0): every page of the column is dictionary-encoded and free of nulls, and
  // the union of the chunk dictionaries is already final.  The decoder then translates each chunk-local index into the
  // code of the value in that global dictionary (look-up table `carry_entries`, see DictMapArgs) and never writes values.
  const void* carry_entries;
  uint32_t carry_mask;
  uint32_t carry_empty_index;  // code of the value 0xFFFF...F, which the look-up table cannot hold
  int32_t carry;
  int32_t skip;                // != 0: zero-copy column, its pages are not decoded at all
};

// Per-column OR over the column's data pages (k_classify_pages), read before decoding to pick late-materialised columns
// PAGECLASS_NOT_IN_PLACE: the page cannot be read where it lies -- it is not a PLAIN, stored (uncompressed), null-free
// page of 4- or 8-byte values whose body is value-aligned, large enough, and at least one partition tile long
enum : uint32_t { PAGECLASS_NOT_DICT = 1u, PAGECLASS_MAYBE_NULLS = 2u, PAGECLASS_NOT_IN_PLACE = 4u };
void launch_classify_pages(hs_ctx* ctx, const PageDesc* pages, int64_t n_pages, uint32_t* col_flags, int zc_tile_rows);
// Zero-copy PLAIN columns: a column whose every page passes the PAGECLASS_NOT_IN_PLACE test is never decoded.  Its values
// are read by the hash and partition kernels straight from the page bodies inside the source file images.  Per partition
// tile (zc_tile_rows rows: 4096, or 8192 when the rows leave over NVLink) they need to know where the tile's values lie:
// pages are at least one tile long, so a tile touches at most two of them.
struct ZcTile {
  const uint8_t* p0;  // page body of the tile's first row, rebased: the value of GLOBAL row r is at p0 + r * width ...
  const uint8_t* p1;  // ... for r < split, and at p1 + r * width from row `split` on (the next page)
  int64_t split;
};
// entries of every page of a column with tile_src[col] != nullptr
void launch_fill_zc_tiles(hs_ctx* ctx, const PageDesc* pages, int64_t n_pages, ZcTile* const* tile_src, int zc_tile_rows,
                          int64_t nrows);

// device error word: 0 = ok, else (code << 24 | detail)
enum DecodeError : uint32_t {
  DERR_NONE = 0, DERR_BAD_HEADER = 1, DERR_UNSUPPORTED_ENCODING = 2, DERR_VALUE_COUNT = 3, DERR_COMPRESSED = 4,
  DERR_OVERRUN = 5, DERR_DICT_INDEX = 6, DERR_UNSUPPORTED_TYPE = 7, DERR_SNAPPY = 8, DERR_STRING_TOO_LONG = 9,
  DERR_SPARK_RANGE = 10,    // a timestamp Spark 3.1 refuses to read: INT96 before 1900, MILLIS beyond int64 micros (detail: column)
  DERR_DECIMAL_WIDTH = 11,  // a decimal value wider than its precision's int32 / int64 (detail: column)
  DERR_GZIP = 12,           // a GZIP page body fails a check of inflate.h (detail: gz::InflateError)
  DERR_LZ4 = 13             // an LZ4 / LZ4_RAW page body fails a check of lz4_block.h (detail: lz4::Lz4Error)
};
// BYTE_ARRAY dictionary pages -> tables of string references (device_utils.cuh: string_ref): one job per dictionary page,
// walked by one thread (the entries are length-prefixed, so their positions are only found sequentially)
struct StringDictJob {
  const uint8_t* page;   // PLAIN byte arrays: [u32 length][bytes] ...
  uint64_t* refs;        // count references out
  int32_t size, count;
};
void launch_build_string_dicts(hs_ctx* ctx, const StringDictJob* jobs, int64_t n, uint32_t* d_error);

// ---- compressed pages (page_codec.cu; the kernels of each codec: snappy.cu, inflate.cu, lz4.cu) -----------------------
// Decompresses every compressed data page and dictionary page of `pages` (host copy of d_pages) into *scratch, repoints
// the descriptors at the decompressed bytes and uploads them to d_pages.  A dictionary page shared by several data pages
// is decompressed once.  A failed check sets d_error (DERR_SNAPPY / DERR_GZIP / DERR_LZ4).  Synchronises the stream once.
void decompress_pages(hs_ctx* ctx, std::vector<PageDesc>& pages, PageDesc* d_pages, Buf<uint8_t>* scratch, uint32_t* d_error);
// one per compressed page (or dictionary page) of a call: where it lies, where its decompressed copy goes
struct PageBlob {
  const uint8_t* src;   // stored bytes (device)
  uint64_t dst_off;     // offset of the decompressed bytes in the scratch buffer
  uint32_t src_len;
  uint32_t dst_len;     // prefix + decompressed length
  uint32_t prefix;      // leading bytes copied verbatim (v2 level bytes)
  uint32_t compressed;  // 0: copy, 1: compressed with `codec`
  uint32_t first_block; // filled by decompress_blobs (snappy: the page's first 64 KB output block in the block table)
  uint32_t codec;       // pq::Codec of the page's chunk: SNAPPY, GZIP, LZ4 or LZ4_RAW
};
// Decompresses the blobs into `scratch`: chooses and launches the kernels of each codec (the blobs are reordered by
// codec).  sequential (optional, host): per blob in its new order, 1 where a snappy stream was decoded front to back.
// Synchronises the stream once.
void decompress_blobs(hs_ctx* ctx, std::vector<PageBlob>& blobs, uint8_t* scratch, uint32_t* d_error,
                      std::vector<uint32_t>* sequential = nullptr);

// Walks the page headers of every chunk.  mode 0: page_counts[chunk] = number of data pages.
// mode 1: fills pages[page_offsets[chunk] ...].
void launch_walk_pages(hs_ctx* ctx, const ChunkDesc* chunks, int n_chunks, int32_t* page_counts,
                       const int64_t* page_offsets, PageDesc* pages, uint32_t* d_error, int mode);
// Decodes all pages into the column arrays.  windows (optional, device): [lo, hi) global rows, ascending and disjoint
// within a file; the windows of file f are windows[window_offsets[f] .. window_offsets[f+1]) (pairs).  A page is decoded
// only when it intersects one of its file's windows.  any_converted: some page has a ValueConv (those are decoded by
// k_decode_converted_pages, launched right after k_decode_pages).
void launch_decode_pages(hs_ctx* ctx, const PageDesc* pages, int64_t n_pages, const ColumnOut* cols,
                         uint32_t* col_has_nulls, const int64_t* windows, const int64_t* window_offsets, uint32_t* d_error,
                         bool any_converted);

// ---- hash / partition (hash_partition.cu) ---------------------------------------------------------------------------
struct KeyColumn {
  const void* data;
  const uint8_t* valid;  // nullptr -> no nulls
  int32_t type;
  int32_t width;
  // zero-copy column (data == nullptr): where each partition tile's values lie inside the source images.  Only a single
  // int32 / int64 key without nulls may come this way (the specialised hash kernels handle it).
  const ZcTile* tiles = nullptr;
  // kind mm3_hash_value hashes the value as: kHashDecimalInt for a decimal(p <= 9) column, else the type (engine.h:
  // key_column_of sets it; every site that buckets a row reads it through key_hash_kind)
  int32_t hash = -1;
};
// -1 (a descriptor built without key_column_of) hashes by the type, as before decimals existed
__host__ __device__ __forceinline__ int key_hash_kind(const KeyColumn& k) { return k.hash >= 0 ? k.hash : k.type; }

constexpr int kMaxBuckets = 4096;

// The hash partition (K2 + K3): every row's bucket is pmod(murmur3(keys, seed 42), num_buckets); its bin is the bucket, or
// the owner rank bucket % owner_mod.  The rows then move stably into bin-major order.  hash_rows and move_rows choose the
// kernels: up to 1024 bins one kernel moves every column through shared memory (the fused partition, which can also read
// columns in place and carry dictionary codes); above that, a destination per row and a scatter per column.
//
// Rows per tile of the partition that runs on ctx for num_buckets buckets, i.e. the tile a column read in place
// (ZcTile) is laid out for: 8192 when the runs go to peer GPUs (world > 1), else 4096.  0: the unfused partition, which
// takes neither carried nor in-place columns.
constexpr int kFusedTileLocal = 4096;  // rows per tile when the partition writes local memory (256 threads x 16)
constexpr int kFusedTilePeer = 8192;   // ... and when it writes peer GPUs' memory over NVLink (512 threads x 16)
int partition_tile_rows(hs_ctx* ctx, int num_buckets);
struct HashedRows {
  int64_t nrows = 0, ntiles = 0;
  int num_buckets = 0, owner_mod = 0, nbins = 0;
  bool to_peers = false;    // the runs go to the owners' memory (move_rows with a peer table)
  int single_key_type = -1;
  int nkeys = 0;
  Buf<KeyColumn> keys;      // device copy of the key descriptors
  Buf<uint32_t> tile_hist;  // ntiles x nbins; launch_tile_offsets turns the counts into destinations in place
  Buf<uint16_t> bin_ids;    // every row's bin; not kept by the owner pass (owner_mod > 0), whose partition hashes again
};
// K2: hashes the key columns (host descriptors from key_column_of), counts the tile and global histograms
// (global_hist: nbins entries, zero on entry) and keeps every row's bin.  key_or_and (optional, {0, ~0} on entry):
// accumulates OR / AND of the sort-encoded values of the last key column.
void hash_rows(hs_ctx* ctx, const KeyColumn* keys, int nkeys, int64_t nrows, int num_buckets, int owner_mod, bool to_peers,
               unsigned long long* global_hist, unsigned long long* key_or_and, HashedRows* out);
// in-place: tile_hist[t][b] <- bucket_base[b] + sum_{t'<t} tile_hist[t'][b]   (bucket_base = exclusive scan of global hist)
// explicit_base (optional, device, nb entries): start of every bucket's destination instead of the local scan
void launch_tile_offsets(hs_ctx* ctx, uint32_t* tile_hist, int64_t ntiles, int num_buckets,
                         const unsigned long long* global_hist, unsigned long long* bucket_offsets /* nb+1 or null */,
                         const unsigned long long* explicit_base = nullptr);
struct PartColumn {
  const void* in;
  void* out;
  int32_t width;  // 8, 4 or 1 (validity bytes travel as width-1 columns)
  int32_t pad;
  const ZcTile* tiles = nullptr;  // zero-copy source (in == nullptr), see KeyColumn::tiles
};
// pack: one more round that reads up to four 16-bit code columns and writes them as ONE 8-byte record per row (slot s in
// bits [16 s, 16 s + 16)) -- the layout k_dict_pack_all gathers from
struct CodePackRound {
  const uint16_t* src[4];
  void* out;   // nrows x 8 bytes
  int32_t n;   // code columns in use (0: no such round)
  int32_t pad;
};
// K3, after launch_tile_offsets(h.tile_hist): moves the columns (host descriptors, read until the caller's next
// synchronisation) into bin-major order, stable.  pack (optional): the code records, fused partition only.
// peer_out (to_peers only): device table of peer-mapped output pointers, one row of `peers` per column round and then
// one for the code records; bucket b is written to owner b % peers (exchange.cu: the GPU of that rank, peers = world).
void move_rows(hs_ctx* ctx, const HashedRows& h, const PartColumn* cols, int ncols, const CodePackRound* pack = nullptr,
               void* const* peer_out = nullptr, int peers = 1);
// out[i] = sort_encode(in[src ? src[i] : i])  (+ global OR / AND reduction into or_and[0], or_and[1])
void launch_encode_keys(hs_ctx* ctx, const void* in, int type, const uint32_t* src, int64_t nrows, uint64_t* out,
                        unsigned long long* or_and);
void launch_iota_u32(hs_ctx* ctx, uint32_t* out, int64_t n);
// out[i] = piece of the string refs[perm[i]]: its length (piece < 0) or its piece-th 8 bytes, big-endian, zero-padded
// (+ OR / AND reduction); see k_string_piece_keys
void launch_string_piece_keys(hs_ctx* ctx, const uint64_t* refs, const uint32_t* perm, int64_t nrows, int piece, uint64_t* out,
                              unsigned long long* or_and);

// ---- segmented radix sort (radix_sort.cu) ---------------------------------------------------------------------------
constexpr int kSortTile = 4096;  // pairs per tile (256 threads x 16)
struct SortTile {
  uint32_t seg;
  uint32_t count;
  uint64_t start;  // global position of the tile's first pair
};
struct SortChunk;  // radix_sort.cu
struct SortPlan {
  int64_t n = 0;
  int64_t ntiles = 0;
  int32_t nseg = 0;
  Buf<SortTile> tiles;          // device
  Buf<uint32_t> seg_tile_begin; // device, nseg+1: first tile of each segment
  Buf<uint64_t> seg_start;      // device, nseg+1: global start of each segment
  Buf<uint32_t> tile_hist;      // device, ntiles x 256
  Buf<uint32_t> tile_dst;       // device, ntiles x 256: destination of every (tile, digit) for the current pass
  std::vector<uint32_t> h_seg_tile_begin;  // host mirror of seg_tile_begin
  std::vector<uint64_t> h_seg_start;       // host mirror of seg_start
  int64_t nchunks = 0;          // the per-segment scan of a pass works on chunks of up to 128 tiles of one segment:
  Buf<SortChunk> chunks;        // device, nchunks
  Buf<uint32_t> seg_chunk_begin;// device, nseg+1: first chunk of each segment
  Buf<uint32_t> chunk_sums;     // device, nchunks x 256
};
// seg_offsets: host array of nseg+1 global offsets
void build_sort_plan(hs_ctx* ctx, const uint64_t* seg_offsets, int nseg, SortPlan* plan);
// Where the PLAIN page bodies of a single int32 / int64 key column lie in the encoder's arena, laid out before the sort:
// the value at position lr of segment s goes to arena + page_value_offset[seg_page_begin[s] + lr / rows_per_page]
// + (lr % rows_per_page) * width.  The local sort writes the decoded keys there itself (see sort_rows).
struct KeyPageDest {
  uint8_t* arena;
  const uint32_t* seg_page_begin;     // device, per segment: its first page
  const uint64_t* page_value_offset;  // device, per page: arena offset of the first value byte
  uint32_t rows_per_page;             // a multiple of kSortTile
  int32_t width;                      // 4 or 8
  int32_t type;                       // HS_TYPE_INT32 / HS_TYPE_INT64
};
// The rows of a SortPlan in sorted order: at sorted position p, keys()[p] is the sort encoding of the first key column and
// perm()[p] the row (the position in the plan's input order).  When the sort wrote the key pages (key_pages_written),
// the final keys are not materialised and keys() is not valid.
struct SortedRows {
  Buf<uint64_t> keys_buf[2];  // the pairs and scratch pairs of the same size: the sort passes move them back and forth
  Buf<uint32_t> perm_buf[2];
  int cur = 0;                // the pairs are in keys_buf[cur] / perm_buf[cur]
  uint64_t* keys() const { return keys_buf[cur].get(); }
  uint32_t* perm() const { return perm_buf[cur].get(); }
  // queued, not yet settled (sort_rows with may_defer): the sort may still be running, and settle_sorted_rows() says
  // whether the rows had to be sorted again
  bool queued = false;
  // the tie fix-up's verdict while it is outstanding (resort_bits != 0): gave_up arrives with the first synchronisation
  // after ctx->sync_count was queued_at; if it is set, the rows are sorted again on resort_bits
  uint64_t resort_bits = 0, queued_at = 0;
  uint32_t gave_up = 0;
  bool key_pages_written = false;  // the sort stored the key into the pages of a KeyPageDest
};
// Lays the key's pages out on request: called at most once, by a sort that can store the key into its pages, as soon as
// the sort has queued the work that does not depend on them.  Returns the destinations, or nullptr to have the sort
// write keys() as usual.
using KeyPagesFn = std::function<const KeyPageDest*()>;
// Sorts the rows within every segment of `plan` stably by cols[0], then cols[1], ... (nulls first); row r of a column
// is the row at position r of the plan's input.  Chooses the sort path (radix_sort.cu).  last_or_and (optional): OR / AND
// of the sort encoding of cols[ncols - 1], when the caller has them already.  may_defer: the sort of a single null-free
// key column may be left queued (out->queued) -- the host does not wait for it, and settle_sorted_rows() must run before
// out is read, best after the caller's next synchronisation.  Otherwise the result is final in stream order.
// key_pages (optional): a single null-free int32 / int64 key that takes k_local_sort asks it for the key's page
// destinations and stores the decoded keys there instead of into keys() (out->key_pages_written).
void sort_rows(hs_ctx* ctx, SortPlan* plan, const KeyColumn* cols, int ncols, const unsigned long long* last_or_and,
               bool may_defer, SortedRows* out, const KeyPagesFn* key_pages = nullptr);
// Settles a queued sort (a no-op otherwise).  True when the rows had to be sorted again: whatever was derived from
// keys() / perm() must be redone.
bool settle_sorted_rows(hs_ctx* ctx, SortPlan* plan, SortedRows* s);

// ---- gather + Parquet encode (gather_encode.cu) -----------------------------------------------------------------
struct GatherColumn {
  const void* src;        // partitioned column values
  const uint64_t* sorted_keys;  // when non-null: take the value from the sorted encoded keys (decode with key_type)
  int32_t key_type;
  int32_t width;
  const uint64_t* page_value_offset;  // device: arena offset of the first value byte of each (bucket, page)
};
// For every sorted position p (tile by tile): value = src[perm[p]] written PLAIN into its page body (width 1: bit-packed).
// page index of local row lr in bucket b = bucket_page_begin[b] + lr / rows_per_page.
void launch_gather_encode(hs_ctx* ctx, const SortTile* tiles, int64_t ntiles, const uint64_t* seg_start,
                          const uint32_t* perm, const GatherColumn& col, const uint32_t* bucket_page_begin,
                          int64_t rows_per_page, uint8_t* arena);
// nullable columns: per-tile non-null counts, then bit-packed definition levels + dense values per tile (width 1: per page)
void launch_tile_valid_counts(hs_ctx* ctx, const SortTile* tiles, int64_t ntiles, const uint32_t* perm,
                              const uint8_t* valid, uint32_t* counts);
void launch_gather_encode_nullable(hs_ctx* ctx, const SortTile* tiles, int64_t ntiles, const uint32_t* perm,
                                   const void* src, const uint8_t* valid, int width, const uint64_t* tile_value_offset,
                                   const uint64_t* tile_def_offset, uint8_t* arena);
// string columns (8-byte references, device_utils.cuh): per tile the bytes its non-null values take as PLAIN BYTE_ARRAY
// ([u32 length][bytes] each) and their number; then definition bits + values per tile.  valid == nullptr: no nulls
void launch_tile_string_sizes(hs_ctx* ctx, const SortTile* tiles, int64_t ntiles, const uint32_t* perm, const uint64_t* refs,
                              const uint8_t* valid, uint32_t* bytes, uint32_t* counts);
void launch_gather_encode_strings(hs_ctx* ctx, const SortTile* tiles, int64_t ntiles, const uint32_t* perm, const uint64_t* refs,
                                  const uint8_t* valid, const uint64_t* tile_value_offset, const uint64_t* tile_def_offset,
                                  uint8_t* arena);
// ---- dictionary encoding (dict_encode.cu) -------------------------------------------------------------------------
constexpr uint32_t kMaxDictEntries = 65536;          // bit width <= 16
constexpr uint32_t kDictCapacity = 8 * kMaxDictEntries;  // open-addressing slots (power of two)
// inserts the distinct raw values of src[begin, end) into the hash set `keys` (capacity slots preset to all-ones);
// state[0] = distinct count, state[1] = 1 when more than max_distinct values were seen, state[2] = the all-ones value occurs
void launch_dict_build(hs_ctx* ctx, const void* src, int width, int64_t begin, int64_t end, unsigned long long* keys,
                       uint32_t capacity, uint32_t max_distinct, uint32_t* state);
// same hash set, filled from the dictionary pages of the decoded source chunks of projected column `col`
void launch_dict_build_from_pages(hs_ctx* ctx, const PageDesc* pages, int64_t n_pages, int col, int width,
                                  unsigned long long* keys, uint32_t capacity, uint32_t max_distinct, uint32_t* state);
// compacts the distinct values out of the hash set (counter must be zeroed); then slot -> rank in the sorted dictionary
// (at most max_out values are written; the counter still counts all of them)
void launch_dict_collect(hs_ctx* ctx, const unsigned long long* keys, uint32_t capacity, unsigned long long* out,
                         uint32_t* counter, uint32_t max_out = 0xffffffffu);
// entries: capacity x 16 bytes {key lo, key hi, dictionary index, 0}
// all dictionary columns of a table in one map + one pack launch (up to 8 columns per call)
struct DictMapArgs {
  const void* src[8];
  const void* entries[8];  // 16-byte {key, index} hash-table entries (open addressing, linear probing, dict_hash_u64)
  uint32_t mask[8];        // table capacity - 1 (a power of two sized to the dictionary, so that the table stays in L1)
  uint32_t empty_index[8];
  int32_t width[8];
  int32_t ncols;
};
struct DictPackArgs {
  const uint64_t* page_value_offset[8];
  uint32_t bw[8];
  int32_t ncols;
};
// rec_scratch: nrows records of 4 (ncols <= 4) or 8 uint16 indices
// bit-packs the codes of already mapped records (4 or 8 uint16 slots per row) into the dictionary-encoded data pages
void launch_dict_pack(hs_ctx* ctx, const SortTile* tiles, int64_t ntiles, const uint64_t* seg_start, const uint32_t* perm,
                      const DictPackArgs& pack_args, int slots, const uint16_t* rec, const uint32_t* bucket_page_begin,
                      int64_t rows_per_page, uint8_t* arena);
void launch_dict_encode_all(hs_ctx* ctx, const SortTile* tiles, int64_t ntiles, const uint64_t* seg_start, const uint32_t* perm,
                            const DictMapArgs& map_args, const DictPackArgs& pack_args, int64_t nrows, uint32_t capacity,
                            uint16_t* rec_scratch, const uint32_t* bucket_page_begin, int64_t rows_per_page, uint8_t* arena);
// Plain gather: out[i] = src[perm[i]]
void launch_gather_plain(hs_ctx* ctx, const void* src, const uint32_t* perm, int64_t n, int width, void* out);
struct StatPatch {        // min/max of the sorted key column of one row group
  uint64_t first_pos, last_pos;  // sorted positions of the row group's first and last row
  uint64_t min_off[2], max_off[2];  // arena offsets of the footer placeholders
  int32_t width, pad;
};
// min / max = the key values (width bytes each, in `keys`) of the rows perm[first_pos] and perm[last_pos]
void launch_patch_key_stats(hs_ctx* ctx, const StatPatch* patches, int64_t n, const uint32_t* perm, const void* keys,
                            uint8_t* arena);
struct ByteCopy {
  uint64_t dst;  // arena offset
  uint32_t src;  // offset into the skeleton byte stream
  uint32_t len;
};
void launch_scatter_bytes(hs_ctx* ctx, const ByteCopy* copies, int64_t n, const uint8_t* skeleton, uint8_t* arena);
// larger pieces at any alignment (compressed page fragments moving into their place in the file): one CTA per blob
struct BlobCopy {
  uint64_t src, dst;  // byte offsets into src_base / dst_base
  uint32_t len, pad;
};
void launch_copy_blobs(hs_ctx* ctx, const BlobCopy* blobs, int64_t n, const uint8_t* src_base, uint8_t* dst_base);
// Page bodies compressed with a page codec (page_codec.cu): SNAPPY, GZIP or LZ4 (Hadoop-framed).  A body's compressed form
// is its preamble and its trailer, which the host writes (snappy's length varint; the gzip member's header, and its final
// block, CRC-32 and ISIZE), around its pieces, which lie in `slots` on the device.
struct CompressedBodies {
  int codec = 0;                     // pq::Codec
  Buf<uint8_t> slots;
  std::vector<uint64_t> raw_len;     // per body: uncompressed bytes
  std::vector<uint32_t> crc;         // GZIP, per body: CRC-32 of the uncompressed bytes
  std::vector<size_t> first_piece;   // per body (+1): its pieces
  std::vector<BlobCopy> pieces;      // src: offset in slots, len: compressed bytes
  uint64_t size(size_t body) const;  // compressed bytes of the body: preamble + pieces + trailer
  void append_preamble(size_t body, std::vector<uint8_t>& out) const;
  void append_trailer(size_t body, std::vector<uint8_t>& out) const;
  // appends the body's pieces to `copies` with consecutive destinations from *dst on; advances *dst
  void place(size_t body, std::vector<BlobCopy>& copies, uint64_t* dst) const;
};
// Compresses the bodies (offset, length) of `raw` (device), each on its own, with `codec` (pq::SNAPPY, GZIP or LZ4).
// Synchronises the stream once: the compressed sizes are data.
void compress_bodies(hs_ctx* ctx, int codec, const uint8_t* raw, const std::vector<std::pair<uint64_t, uint64_t>>& bodies,
                     CompressedBodies* out);
// Synthetic table generator: rows [first_row, first_row+n) of column `col` (0..4) of table T (SURVEY.md section 8d)
void launch_synth_column(hs_ctx* ctx, int col, int64_t first_row, int64_t n, void* out);

// ---- read side (read_side.cu) ---------------------------------------------------------------------------
// A filter scan's comparisons (api.cu resolves Spark's coercion into these ranges).  One range on one column of type `type`:
// numeric columns compare sort_encode(type, value) with the inclusive encoded bounds lo / hi (lo_strict = hi_strict = 0;
// lo > hi is an empty range); string / binary columns compare the value with the references lo / hi (device copies of the
// bound bytes) in UTF8String byte order, strictly where lo_strict / hi_strict say so.
constexpr int kMaxPredicates = 16;
constexpr int kMaxJoinKeys = 8;
struct PredRange {
  int32_t type;
  int32_t has_lo, has_hi, lo_strict, hi_strict;
  uint64_t lo, hi;
};
struct PredDesc {
  const void* data;      // column values (string references for strings)
  const uint8_t* valid;  // nullptr: no nulls; a null row qualifies only when null_true is set
  PredRange r;           // neither bound: the row only has to be non-null (a join side's key columns)
  // set form (a disjunction on the column): when set is not nullptr the value must lie in one of the n_set ranges at set
  // (device; ascending and disjoint, of type r.type), and r's bounds are not used
  const PredRange* set = nullptr;
  int64_t n_set = 0;
  int32_t null_true = 0;  // a null row makes the predicate true (IS NULL, NOT (c <=> v)): predicates.h term_null_selects
};
struct PredSet {
  PredDesc p[kMaxPredicates + kMaxJoinKeys];  // a join side: its predicates plus one IS NOT NULL per nullable key column
  int n = 0;
};
// A string pattern term the ranges cannot express (EndsWith, Contains, a LIKE that is not a prefix), compiled on the host
// (predicates.h: compile_pattern) for pattern_matches (string_match.h): items and segs are device copies.  A non-null row
// qualifies when the match, inverted under negate, holds; a null row when null_true is set.
struct PatternDesc {
  const uint64_t* refs;  // string references of the column
  const uint8_t* valid;  // nullptr: no nulls
  const uint16_t* items;
  const int32_t* fail;
  const PatSeg* segs;
  int32_t nseg, whole, negate, null_true;
};
struct PatternSet {
  PatternDesc p[kMaxPredicates];
  int n = 0;
};
// The comparisons between two columns of a scan or join side (predicates.h: resolve_compare), evaluated by compare_holds
// (column_compare.h).
struct CompareSet {
  CompareDesc p[kMaxPredicates];
  int n = 0;
};
struct ExprDesc;  // column_expr.h
struct ExprInst;
struct ExprColumn;
// The expression comparisons of a scan or join side (predicates.h: resolve_expr), evaluated by expr_holds
// (column_expr.h).  Device arrays, uploaded once per call: descs[n], the instructions they index and the columns those
// read.  Pointers and a count only, so that the kernel's parameter block stays small whatever the programs' length.
struct ExprSet {
  const ExprDesc* descs = nullptr;
  const ExprInst* insts = nullptr;
  const ExprColumn* cols = nullptr;
  int n = 0;
};
// The row filter of a scan or join side: a row is kept when every predicate, pattern, comparison and expression
// comparison holds.  A side's expression comparisons are in exprs when they are arithmetic only, in funcs (k_func_mask)
// when one of them uses a function, a string, date or timestamp value.
struct RowFilter {
  PredSet preds;
  PatternSet pats;
  CompareSet cmps;
  ExprSet exprs;
  ExprSet funcs;
  bool empty() const { return preds.n == 0 && pats.n == 0 && cmps.n == 0 && exprs.n == 0 && funcs.n == 0; }
};
// The window search over sorted segments (each ascending on `keys`), one pair (segment, range) per work item:
// work[w] = {s, r} with r indexing `ranges` (device); bounds[2w] = first row of s inside ranges[r], bounds[2w+1] = first
// row above it (segment-relative).  All ranges are of type ranges_type.
void launch_range_bounds(hs_ctx* ctx, const void* keys, int ranges_type, const PredRange* ranges, const uint64_t* seg_offsets,
                         const uint2* work, int64_t nwork, int64_t* bounds);
// the candidate rows of sorted windows: out_idx[o] = win[2w] + (o - out_offsets[w]) for out_offsets[w] <= o <
// out_offsets[w+1] (win: [lo, hi) global rows, out_offsets: nwin + 1 entries).  One thread per output row.
void launch_windows_to_indices(hs_ctx* ctx, const int64_t* win, const uint64_t* out_offsets, int64_t nwin, int64_t n_out,
                               uint32_t* out_idx);
// mask[i] = every predicate of `preds` holds for row cand[i] (row i when cand is nullptr)
void launch_predicate_mask(hs_ctx* ctx, const PredSet& preds, const uint32_t* cand, int64_t n, uint32_t* mask);
// mask[i] = 0 where a pattern of `pats` does not hold for row cand[i] (row i when cand is nullptr); launches nothing when
// pats is empty
void launch_pattern_mask(hs_ctx* ctx, const PatternSet& pats, const uint32_t* cand, int64_t n, uint32_t* mask);
// mask[i] = 0 where a comparison of `cmps` does not hold for row cand[i] (row i when cand is nullptr); launches nothing when
// cmps is empty
void launch_compare_mask(hs_ctx* ctx, const CompareSet& cmps, const uint32_t* cand, int64_t n, uint32_t* mask);
// mask[i] = 0 where an expression comparison of `exprs` does not hold for row cand[i] (row i when cand is nullptr);
// launches nothing when exprs is empty
void launch_expr_mask(hs_ctx* ctx, const ExprSet& exprs, const uint32_t* cand, int64_t n, uint32_t* mask);
// the same for expression comparisons with functions (k_func_mask)
void launch_func_mask(hs_ctx* ctx, const ExprSet& funcs, const uint32_t* cand, int64_t n, uint32_t* mask);
// The n key columns of one join side in sorted order: col[k] holds key column k at sorted position p, read at its
// type's width (type[k]: HS_TYPE_INT32 / HS_TYPE_INT64, or HS_TYPE_STRING for string references).  The tuples compare
// column by column, integers as signed values, strings in byte order.
struct JoinKeyCols {
  const void* col[kMaxJoinKeys];
  int32_t type[kMaxJoinKeys];
  int32_t n;
};
// match counts of every left position against the right positions of the same bucket (k_join_count)
void launch_join_count(hs_ctx* ctx, const JoinKeyCols& lkeys, const uint64_t* lseg, const JoinKeyCols& rkeys,
                       const uint64_t* rseg, int nseg, int64_t nl, uint32_t* counts, uint32_t* first_match);
// the (left row, right row) pairs at out_offsets (the scan of counts); a sorted position p is row perm[p] of its side
// (perm nullptr: row p)
void launch_join_emit(hs_ctx* ctx, const uint32_t* counts, const uint32_t* first_match, const uint64_t* out_offsets,
                      int64_t nl, const uint32_t* lperm, const uint32_t* rperm, uint32_t* out_lrow, uint32_t* out_rrow);
// The validity of the n key columns of the probing side in sorted order, one byte per position (valid[k] nullptr: key
// column k has no nulls): a position with a null in any of them matches nothing.
struct JoinKeyValid {
  const uint8_t* valid[kMaxJoinKeys];
  int32_t n;
};
// The semi / anti join's probe (k_join_exists): keep[i] = 1 when left position i has an equal key tuple among the right
// positions of its bucket and keep_match is set (semi), or has none and keep_match is clear (anti); 0 otherwise
void launch_join_exists(hs_ctx* ctx, const JoinKeyCols& lkeys, const JoinKeyValid& lvalid, const uint64_t* lseg,
                        const JoinKeyCols& rkeys, const uint64_t* rseg, int nseg, int64_t nl, bool keep_match, uint32_t* keep);
// The outer joins' "no row": the row an output pair holds for a side padded with nulls.  Never a real row: a join side
// has fewer than 2^32 - 1 rows.
constexpr uint32_t kNoRow = 0xFFFFFFFFu;
// The outer joins' probe (k_join_count_outer), from the np positions of the preserved side p into the searched side t:
// k_join_count's counts and first matches, except that a position with a null in a key column (pvalid) or with no match
// gets count 1 and first_match kNoRow
void launch_join_count_outer(hs_ctx* ctx, const JoinKeyCols& pkeys, const JoinKeyValid& pvalid, const uint64_t* pseg,
                             const JoinKeyCols& tkeys, const uint64_t* tseg, int nseg, int64_t np, uint32_t* counts,
                             uint32_t* first_match);
// The outer joins' (preserved row, searched row) pairs at out_offsets (the scan of counts), the searched row kNoRow where
// first_match is; shift (nseg + 1 entries, or nullptr) moves every output position of bucket b up by shift[b]
void launch_join_emit_outer(hs_ctx* ctx, const uint32_t* counts, const uint32_t* first_match, const uint64_t* out_offsets,
                            const uint64_t* pseg, const uint64_t* shift, int nseg, int64_t np, const uint32_t* pperm,
                            const uint32_t* tperm, uint32_t* out_prow, uint32_t* out_trow);
// FullOuter: the right row urow[r] (rank r; ucum: the ranks at which the nseg buckets start, nseg + 1 entries) goes to
// output position base[b] + r of the bucket b holding r, its left row kNoRow
void launch_join_place_unmatched(hs_ctx* ctx, const uint32_t* urow, int64_t nu, const uint64_t* ucum, const uint64_t* base,
                                 int nseg, uint32_t* out_lrow, uint32_t* out_rrow);
// launch_gather_plain for a padded side: out[i] = src[idx[i]] and out_valid[i] = valid[idx[i]] (1 when valid is nullptr),
// 0 and 0 where idx[i] is kNoRow
void launch_gather_padded(hs_ctx* ctx, const void* src, const uint8_t* valid, const uint32_t* idx, int64_t n, int width, void* out,
                          uint8_t* out_valid);
// launch_string_lengths / launch_copy_strings for a padded side: a kNoRow value is a null of length 0; the lengths pass
// also writes every value's validity
void launch_string_lengths_padded(hs_ctx* ctx, const uint64_t* refs, const uint8_t* valid, const uint32_t* idx, int64_t n,
                                  uint32_t* lens, uint8_t* out_valid);
void launch_copy_strings_padded(hs_ctx* ctx, const uint64_t* refs, const uint8_t* valid, const uint32_t* idx, int64_t n,
                                const uint64_t* offsets, uint8_t* out);
// exclusive scan of uint32 counts into uint64 offsets (n+1 entries; last = total)
void exclusive_scan_u32_u64(hs_ctx* ctx, const uint32_t* in, int64_t n, uint64_t* out);
// lens[i] = length of refs[idx[i]] (0 for a null);  then, with offsets = exclusive scan of lens: out[offsets[i] ..] = bytes
void launch_string_lengths(hs_ctx* ctx, const uint64_t* refs, const uint8_t* valid, const uint32_t* idx, int64_t n,
                           uint32_t* lens);
void launch_copy_strings(hs_ctx* ctx, const uint64_t* refs, const uint8_t* valid, const uint32_t* idx, int64_t n,
                         const uint64_t* offsets, uint8_t* out);
// Row selection over n candidates (cand[i], or row i when cand is nullptr): keeps those that pass `filter` and, when
// ndeleted > 0, whose file_ids[i] is not in the host array `deleted`.  The kept candidates go to *kept in their order;
// returns how many there are (after a stream synchronisation).  offsets, when given, receives the exclusive scan of the
// keep mask (n+1 entries): offsets[i] is the number of kept candidates before i.
int64_t select_rows(hs_ctx* ctx, const RowFilter& filter, const uint32_t* cand, int64_t n, const int64_t* file_ids,
                    const int64_t* deleted, int ndeleted, Buf<uint32_t>* kept, Buf<uint64_t>* offsets = nullptr);
// The compaction select_rows ends with, over a keep mask of n candidates (1 / 0): the kept cand[i] (i when cand is
// nullptr) go to *kept in their order; returns how many there are (after a stream synchronisation); offsets as in
// select_rows.
int64_t compact_rows(hs_ctx* ctx, const uint32_t* mask, int64_t n, const uint32_t* cand, Buf<uint32_t>* kept,
                     Buf<uint64_t>* offsets = nullptr);

}  // namespace hs
