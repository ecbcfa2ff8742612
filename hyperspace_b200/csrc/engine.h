// engine.h -- host-side orchestration types shared by api.cu / engine.cu / exchange.cu.
#pragma once
#include <memory>
#include <string>
#include <vector>

#include "device_utils.cuh"
#include "hs_common.h"
#include "kernels.h"
#include "parquet_meta.h"
#include "spark_types.h"

namespace hs {

// A decoded (or partitioned) column resident in HBM.
struct DevColumn {
  std::string name;
  int32_t type = -1;          // HS_TYPE_*
  int32_t width = 0;
  pq::SchemaColumn schema;    // Parquet leaf it came from (converted type carried into the index file)
  Buf<uint8_t> data;          // nrows * width
  Buf<uint8_t> valid;         // nrows bytes, only for optional columns
  bool has_nulls = false;
  // Optional superset of the column's distinct values as a ready-made hash set (built from the source chunks' dictionary
  // pages when every page was dictionary-encoded); lets the encoder skip its full-column distinct scan.
  Buf<unsigned long long> dict_keys;
  uint32_t dict_state[4] = {0, 0, 0, 0};
  bool dict_ready = false;
  // Late-materialised dictionary column (index builds on one GPU): every source page was dictionary-encoded and free of
  // nulls, so the column travels as 16-bit codes of one column-wide sorted dictionary and its values are never written
  // to HBM.  `data` stays empty.  Before the partition `codes` holds one code per row; the partition packs the codes of
  // all carried columns of a row into one 8-byte record (Table::rec, slot `carry_slot`) that the page encoder bit-packs.
  // Zero-copy PLAIN column: never decoded; the hash and partition kernels read its values in place from the page bodies
  // inside the source file images (`data` stays empty until the partition has materialised the column bucket-major).
  bool zero_copy = false;
  Buf<ZcTile> zc_tiles;
  bool carried = false;
  Buf<uint16_t> codes;
  std::vector<uint64_t> dict_values;  // sorted dictionary, raw value bits; code = position
  uint32_t dict_bw = 0;               // bits per code
  int carry_slot = -1;
};

constexpr int kMaxCarried = 4;  // codes per record

// The hash and partition kernels' view of a key column.  The one place that decides how a key value is hashed: Spark
// hashes a decimal(p <= 9) -- an int32 here -- as hashLong of the sign-extended unscaled value.
inline KeyColumn key_column_of(const DevColumn& c) {
  KeyColumn k{c.data.get(), c.has_nulls ? c.valid.get() : nullptr, c.type, c.width, c.zero_copy ? c.zc_tiles.get() : nullptr};
  k.hash = c.type == HS_TYPE_INT32 && is_decimal(c.schema) ? kHashDecimalInt : c.type;
  return k;
}

struct Table {
  int64_t nrows = 0;
  std::vector<DevColumn> cols;
  std::vector<int64_t> file_row_begin;  // nfiles+1: row range of every source file
  int64_t global_rows = -1;             // rows of all ranks together, when the ranks exchanged that while decoding
  bool has_strings = false;             // some column holds string references into the source images (keep those alive)
  Buf<uint8_t> rec;                     // nrows x 4 uint16 codes of the carried columns (after the partition)
};

// Which columns may be late-materialised while decoding (nullptr / first_col < 0: none).
struct CarryOptions {
  int first_col = -1;   // columns [first_col, ncols) are candidates (the indexed columns never are)
  int num_segments = 1; // output files: every one repeats the dictionary page, which enters the size criterion
  // zero-copy PLAIN columns (0 = off): rows per tile of the partition kernel that will read them; the included columns
  // [zc_first_col, ncols) are candidates, and column 0 too when zc_key is set (a single int32 / int64 key)
  int zc_tile_rows = 0;
  int zc_first_col = 0;
  bool zc_key = false;
};

// Rows in bucket-major, key-sorted order (result of K2-K4).
// First stage of the encoder's dictionary analysis (a 16 K-row probe per column that is neither late-materialised nor
// nullable), launched as soon as the partitioned columns exist so that its results reach the host with a synchronisation
// the path performs anyway -- the encoder's page-layout plan can then run on the host while the GPU still sorts.
struct DictProbe {
  int64_t mini = 0;
  Buf<uint32_t> d_states;                             // 4 words per column
  std::vector<uint32_t> h_states;                     // valid once delivered()
  std::vector<Buf<unsigned long long>> keys;          // per column: the hash set the probe filled (empty: not probed)
  uint64_t queued_at = 0;
  bool delivered(const hs_ctx* ctx) const { return ctx->sync_count > queued_at; }
};

struct IndexedRows {
  Table part;                         // partitioned columns (bucket-major, source order inside a bucket)
  std::vector<uint64_t> bucket_offsets;  // host, nb+1
  Buf<uint64_t> d_bucket_offsets;     // device copy
  SortPlan plan;
  // sorted.perm()[p] = partitioned row at sorted position p.  radix_sort.cu (sort_rows) chooses how the rows are sorted
  // and keeps what a sort left queued needs; settle_sort() settles it
  SortedRows sorted;
  // OR / AND of the sort-encoded last indexed column, when the partition's histogram pass already computed them
  bool have_key_bits = false;
  unsigned long long key_or_and[2] = {0, ~0ull};
  // stage timers whose events are read at the call's next synchronisation (reading one synchronises)
  struct DeferredTimer {
    std::unique_ptr<StageTimer> t;
    float hs_stats::*field;
  };
  std::vector<DeferredTimer> pending_timers;
  std::unique_ptr<DictProbe> probe;   // see DictProbe
};

struct OutFile {
  int32_t bucket = 0;
  std::string name;
  uint64_t offset = 0;  // arena offset
  uint64_t size = 0;
  int64_t rows = 0;
};

struct StageTimes;

// Source handling ----------------------------------------------------------------------------------------------
struct LoadOptions {
  const int64_t* d_row_window = nullptr;  // optional per-file [lo,hi) window (device)
  bool allow_missing_lineage = true;
};
// Loads the projected columns of the source files into HBM (H2D of the file images when needed, footer parse on the
// host, page walk + decode on the GPU).
void load_sources(hs_ctx* ctx, const hs_source_file* files, int n_files, const std::vector<std::string>& columns,
                  Table* out, hs_stats* stats, const CarryOptions* carry = nullptr);
// The same in two steps, so that a query can decode the key column first and then only the pages of the other columns
// that intersect the qualifying row range of each file.
struct SourceSet {
  struct Impl;
  Impl* impl;
  int n_files = 0;
  SourceSet();
  ~SourceSet();
  void release_images();  // frees the device copies of host-supplied images (zero-copy columns point into them until then)
  SourceSet(const SourceSet&) = delete;
  SourceSet& operator=(const SourceSet&) = delete;
};
void open_sources(hs_ctx* ctx, const hs_source_file* files, int n_files, SourceSet* set, hs_stats* stats);
// The rows of each file that must be decoded: windows[offsets[f] .. offsets[f+1]) are file f's half-open ranges of
// file-relative rows, ascending and disjoint (offsets: n_files + 1 entries).
struct FileWindows {
  std::vector<int64_t> offsets;
  std::vector<std::pair<int64_t, int64_t>> windows;
};
// file_windows (optional): only the pages that intersect one of their file's windows are decoded
void decode_sources(hs_ctx* ctx, SourceSet& set, const std::vector<std::string>& columns, const FileWindows* file_windows,
                    Table* out, hs_stats* stats, const CarryOptions* carry = nullptr);
// HS_EUNSUPPORTED when one of `keys` is a BOOLEAN column of any opened file: a boolean indexed column could never be read
// back (filters and join keys on booleans are refused), so an index build refuses it before it decodes anything
void refuse_boolean_keys(const SourceSet& set, const std::vector<std::string>& keys);
// type, width and schema of column `name` as decode_sources would decode it, read from the footer of `file` alone
DevColumn source_column_type(hs_ctx* ctx, const hs_source_file& file, const std::string& name);

// K2-K4 on a decoded table whose first nkeys columns are the indexed columns.
// defer_settle: the sort may be left queued (sort_rows' may_defer) -- the caller must call settle_sort() after its next
// synchronisation.  key_pages (optional): passed on to sort_rows (kernels.h)
void index_rows(hs_ctx* ctx, Table& table, int nkeys, int num_buckets, IndexedRows* out, hs_stats* stats, bool defer_settle = false,
                const KeyPagesFn* key_pages = nullptr);

// K5+K6: encode every segment (bucket or source file) as one Parquet file image inside one device arena.
struct EncodeRequest {
  const Table* table = nullptr;            // column values (indexed by perm)
  const uint32_t* d_perm = nullptr;        // sorted position -> row of `table`
  // optional: sorted encoded values of column 0 (integer key), streamed into its pages instead of gathered through d_perm
  const uint64_t* d_sorted_keys = nullptr;
  bool key_sorted = false;                 // column 0 is sorted inside every segment: its row groups carry min / max
  const SortPlan* plan = nullptr;          // tiles over the segments
  std::vector<uint64_t> seg_offsets;       // host, nseg+1
  std::vector<std::string> seg_names;      // file name per segment (empty segments produce no file)
  std::vector<int32_t> seg_ids;            // bucket id per segment
  int64_t rows_per_page = 0;
  int64_t rows_per_row_group = 0;
  std::vector<int64_t> seg_rows_per_row_group;  // optional per-segment override
  bool use_dictionary = true;                   // dictionary-encode columns whose distinct values fit (like parquet-mr)
  int codec = 0;                                // pq::Codec of the written pages: UNCOMPRESSED, SNAPPY, GZIP or LZ4
  DictProbe* probe = nullptr;                   // optional: first-stage dictionary probes already launched (consumed)
};
struct EncodedFiles {
  Buf<uint8_t> arena;       // device
  uint64_t arena_bytes = 0;
  std::vector<OutFile> files;
};
void encode_segments(hs_ctx* ctx, const EncodeRequest& req, EncodedFiles* out, hs_stats* stats);
// encode_segments in two halves, so that an index build can lay its files out before it sorts and let the sort store the
// key into its pages.  layout_segments: the dictionary decisions, the host page plan and skeleton, the arena (out->arena,
// out->files) and the upload of the page tables; it needs the bucket sizes and req.plan, and the sorted rows (req.d_perm)
// only for a table where layout_needs_sorted_rows() holds (nullable or string columns: their page sizes depend on the
// order).  write_segments: the kernels that fill the pages, footer statistics and the page codec; key_pages_written: the sort
// has stored column 0 already (to key_page_dest()).
struct EncodeLayout {
  struct Impl;  // engine.cu
  std::shared_ptr<Impl> impl;
};
bool layout_needs_sorted_rows(const Table& table);
void layout_segments(hs_ctx* ctx, const EncodeRequest& req, EncodeLayout* lay, EncodedFiles* out, hs_stats* stats);
// where column 0's PLAIN page bodies lie, or nullptr when it has none to store into (nulls, a dictionary, not an integer)
const KeyPageDest* key_page_dest(EncodeLayout& lay, const EncodeRequest& req, EncodedFiles* out);
void write_segments(hs_ctx* ctx, const EncodeRequest& req, EncodeLayout& lay, bool key_pages_written, EncodedFiles* out,
                    hs_stats* stats);

// multi-GPU exchange (exchange.cu): redistributes the rows of `table` so that this rank holds exactly the rows of
// the buckets it owns (owner(b) = b % world), with an NCCL all-to-all; index_rows partitions them by bucket afterwards.
// The path above 1024 buckets.  No-op when world == 1.
void exchange_rows(hs_ctx* ctx, Table& table, int nkeys, int num_buckets, hs_stats* stats);
void comm_destroy(hs_ctx* ctx);
// all-gather of a small host blob (out: world x bytes, rank-major); a plain copy on one GPU
void comm_allgather_host(hs_ctx* ctx, const void* in, size_t bytes, void* out);
// Up to 1024 buckets (partition_tile_rows() > 0), over NVLink peer memory: partitions by bucket and delivers every row
// to its final bucket-major position on the owner GPU in one kernel; fills out->part / bucket_offsets so that
// sort_partitioned_rows can run next.
void exchange_partition_p2p(hs_ctx* ctx, Table& table, int nkeys, int num_buckets, IndexedRows* out, hs_stats* stats);
// K4 only: sorts out->part (already bucket-major, offsets in out->bucket_offsets) on the first nkeys columns.
void sort_partitioned_rows(hs_ctx* ctx, int nkeys, int num_buckets, IndexedRows* out, hs_stats* stats, bool defer_settle = false,
                           const KeyPagesFn* key_pages = nullptr);
// settle_sorted_rows() plus the stage timers: true when the rows had to be sorted again (whatever was derived from
// sorted.keys() / sorted.perm() must be redone)
bool settle_sort(hs_ctx* ctx, IndexedRows* out, hs_stats* stats);
void launch_dictionary_probes(hs_ctx* ctx, const Table& part, bool use_dictionary, std::unique_ptr<DictProbe>* out);

std::string make_uuid();

}  // namespace hs

struct hs_index_result {
  hs_ctx* ctx = nullptr;
  int output = HS_OUT_FILES;
  hs::Buf<uint8_t> d_arena;
  hs::Buf<uint8_t> h_arena;
  std::vector<hs::OutFile> files;
};

// Source file images on their way to (or already in) device memory: hs_stage_sources.
struct hs_staged {
  hs_ctx* ctx = nullptr;
  hs::Buf<uint8_t> d_images;
  std::vector<hs_source_file> files;   // on_device descriptors pointing into d_images
  std::vector<std::string> names;
  std::vector<std::shared_ptr<hs::pq::FileMeta>> metas;
  std::vector<hs::Buf<uint8_t>> staging;  // pinned copies of file-system sources
  cudaEvent_t begin = nullptr, ready = nullptr;  // recorded on ctx->h2d_stream around the copies
  uint64_t bytes = 0;
};

// A createIndex whose kernels have run and whose index files are draining to the host: hs_create_index_async.
struct hs_pending {
  hs_ctx* ctx = nullptr;
  std::unique_ptr<hs_index_result> res;
  hs_stats st;
  hs::Buf<uint8_t> d_arena;             // device file images until the copy has completed
  cudaEvent_t t_begin = nullptr, t_compute_end = nullptr, t_d2h_begin = nullptr, t_d2h_end = nullptr;
  bool has_d2h = false;
  std::string out_dir;
  int save_mode = 0;
  ~hs_pending() {
    if (getenv("HS_TIMELINE")) return;  // diagnostics: the timeline's base event may be one of these
    for (cudaEvent_t e : {t_begin, t_compute_end, t_d2h_begin, t_d2h_end})
      if (e) cudaEventDestroy(e);
  }
};

struct hs_batch {
  hs_ctx* ctx = nullptr;
  int64_t nrows = 0;
  bool on_device = false;
  struct Col {
    std::string name;
    int32_t type;
    hs::Buf<uint8_t> data;
    hs::Buf<uint8_t> valid;
    bool has_valid = false;
    hs::Buf<uint64_t> offsets;  // HS_TYPE_STRING: nrows + 1 byte offsets into data
    uint64_t total_bytes = 0;
  };
  std::vector<Col> cols;
};
