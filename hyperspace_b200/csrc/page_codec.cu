// page_codec.cu -- page compression behind one entry point each way: decompress_pages for the readers (under it
// decompress_blobs, which the kernel tests reach too) and compress_bodies for the encoder.  The callers say which bytes
// are compressed and where the result goes; what a codec's kernels need besides that -- how the work is cut up, their
// scratch tables, which of them run -- is decided here.  The kernels are in snappy.cu (SNAPPY, both ways), inflate.cu
// (GZIP, reading), deflate.cu (GZIP, writing) and lz4.cu (LZ4 and LZ4_RAW reading, LZ4 writing).
#include <algorithm>
#include <map>
#include <set>

#include "deflate.h"
#include "lz4_block.h"
#include "page_codec_kernels.h"
#include "parquet_meta.h"

namespace hs {

void decompress_blobs(hs_ctx* ctx, std::vector<PageBlob>& blobs, uint8_t* scratch, uint32_t* d_error,
                      std::vector<uint32_t>* sequential) {
  // each codec's kernels run over its own blobs: the snappy ones first, in page order, then the GZIP ones, then the LZ4
  // ones of both framings
  const size_t n_snappy = (size_t)(std::stable_partition(blobs.begin(), blobs.end(),
                                                         [](const PageBlob& b) { return b.codec == pq::SNAPPY; }) -
                                   blobs.begin());
  const size_t n_gzip = (size_t)(std::stable_partition(blobs.begin() + n_snappy, blobs.end(),
                                                       [](const PageBlob& b) { return b.codec == pq::GZIP; }) -
                                 blobs.begin()) - n_snappy;
  uint64_t total_blocks = 0;  // 64 KB output blocks, the unit of the snappy decoder's parallelism
  bool any_verbatim = false;
  for (size_t i = 0; i < n_snappy; i++) {
    PageBlob& b = blobs[i];
    any_verbatim = any_verbatim || b.prefix != 0 || !b.compressed;
    b.first_block = (uint32_t)total_blocks;
    total_blocks += snappy_blocks_of(b.dst_len, b.prefix);
  }
  if (total_blocks >= 0xffffffffull) fail(HS_EUNSUPPORTED, "more than 256 TB of compressed pages in one call");
  Buf<PageBlob> d_blobs(ctx, std::max<size_t>(1, blobs.size()));
  Buf<uint32_t> d_block_in(ctx, (size_t)total_blocks + 1), d_sequential(ctx, std::max<size_t>(1, n_snappy));
  copy_h2d(ctx, d_blobs.get(), blobs.data(), sizeof(PageBlob) * blobs.size());
  launch_snappy_decompress(ctx, d_blobs.get(), (int64_t)n_snappy, (int64_t)total_blocks, any_verbatim, d_block_in.get(),
                           d_sequential.get(), scratch, d_error);
  launch_inflate(ctx, d_blobs.get() + n_snappy, (int64_t)n_gzip, scratch, d_error);
  launch_lz4(ctx, d_blobs.get() + n_snappy + n_gzip, (int64_t)(blobs.size() - n_snappy - n_gzip), scratch, d_error);
  if (sequential) {
    sequential->assign(blobs.size(), 0u);
    copy_d2h(ctx, sequential->data(), d_sequential.get(), sizeof(uint32_t) * n_snappy);
  }
  sync_stream(ctx);  // the blobs (and whatever else the caller uploaded from host vectors) may go out of scope
}

void decompress_pages(hs_ctx* ctx, std::vector<PageDesc>& pages, PageDesc* d_pages, Buf<uint8_t>* scratch, uint32_t* d_error) {
  // a page is decompressed (or, stored inside a compressed chunk, copied) when its stored bytes are not its decoded bytes
  auto relocated = [](const PageDesc& pg) { return pg.is_compressed || pg.size != pg.uncompressed_size; };
  auto level_bytes = [](const PageDesc& pg) {  // v2: the levels in front of the values are stored verbatim
    return pg.page_type == pq::DATA_PAGE_V2 ? (uint32_t)(pg.rep_bytes + std::max(0, pg.def_bytes)) : 0u;
  };
  auto room = [](int32_t bytes) { return (uint64_t)round_up((size_t)bytes, 16) + 16; };
  // every size is in the descriptors: the scratch bytes first, then real pointers.  The dictionary page of a compressed
  // chunk is compressed too, and all data pages of the chunk name the same one.
  std::set<const uint8_t*> dicts_seen;
  uint64_t total = 0;
  for (const PageDesc& pg : pages) {
    if (pg.codec == pq::UNCOMPRESSED) continue;
    if (pg.dict && dicts_seen.insert(pg.dict).second) total += room(pg.dict_uncompressed_size);
    if (!relocated(pg)) continue;
    if (level_bytes(pg) > (uint32_t)pg.size || level_bytes(pg) > (uint32_t)pg.uncompressed_size)
      fail(HS_EFORMAT, "compressed page has level bytes beyond its size");
    total += room(pg.uncompressed_size);
  }
  scratch->alloc(ctx, std::max<uint64_t>(total, 16) + 16);  // decoders may read one aligned word past a page
  std::vector<PageBlob> blobs;
  std::map<const uint8_t*, uint64_t> dict_off;  // stored dictionary page -> scratch offset of its decompressed copy
  uint64_t cursor = 0;
  for (PageDesc& pg : pages) {
    if (pg.codec == pq::UNCOMPRESSED) continue;
    if (pg.dict) {
      auto it = dict_off.find(pg.dict);
      if (it == dict_off.end()) {
        it = dict_off.emplace(pg.dict, cursor).first;
        blobs.push_back(PageBlob{pg.dict, cursor, (uint32_t)pg.dict_size, (uint32_t)pg.dict_uncompressed_size, 0u, 1u, 0u,
                                 (uint32_t)pg.codec});
        cursor += room(pg.dict_uncompressed_size);
      }
      pg.dict = scratch->get() + it->second;
      pg.dict_size = pg.dict_uncompressed_size;
    }
    if (relocated(pg)) {
      blobs.push_back(PageBlob{pg.data, cursor, (uint32_t)pg.size, (uint32_t)pg.uncompressed_size, level_bytes(pg),
                               (uint32_t)(pg.is_compressed ? 1 : 0), 0u, (uint32_t)pg.codec});
      pg.data = scratch->get() + cursor;
      pg.size = pg.uncompressed_size;
      cursor += room(pg.uncompressed_size);
    }
  }
  copy_h2d(ctx, d_pages, pages.data(), sizeof(PageDesc) * pages.size());
  decompress_blobs(ctx, blobs, scratch->get(), d_error);
}

void compress_bodies(hs_ctx* ctx, int codec, const uint8_t* raw, const std::vector<std::pair<uint64_t, uint64_t>>& bodies,
                     CompressedBodies* out) {
  if (codec != pq::SNAPPY && codec != pq::GZIP && codec != pq::LZ4) fail(HS_EINVAL, "internal: no compressor for codec %d", codec);
  // A body is cut into 64 KB fragments that compress in parallel, each into a slot of its codec's worst-case size.
  auto slot_bytes = [codec](uint32_t len) -> uint64_t {
    const uint64_t bound = codec == pq::SNAPPY ? snappy_max_compressed(len)
                           : codec == pq::GZIP ? gz::deflate_fragment_bound(len) + 4
                                               : lz4::kHadoopGroupHeader + lz4::block_bound(len);
    return round_up(bound, 16);
  };
  std::vector<PageFragment> frags;
  out->codec = codec;
  out->raw_len.clear();
  out->first_piece.clear();
  uint64_t slot_cursor = 0;
  for (const auto& body : bodies) {
    out->raw_len.push_back(body.second);
    out->first_piece.push_back(frags.size());
    for (uint64_t o = 0; o < body.second; o += kCompressFragment) {
      const uint32_t len = (uint32_t)std::min<uint64_t>(kCompressFragment, body.second - o);
      frags.push_back(PageFragment{body.first + o, slot_cursor, len, 0});
      slot_cursor += slot_bytes(len);
    }
  }
  out->first_piece.push_back(frags.size());
  out->slots.alloc(ctx, std::max<uint64_t>(slot_cursor, 16));
  Buf<PageFragment> d_frags(ctx, std::max<size_t>(1, frags.size()));
  Buf<uint32_t> d_flen(ctx, std::max<size_t>(1, frags.size())), d_fcrc(ctx, std::max<size_t>(1, frags.size()));
  std::vector<uint32_t> flen(frags.size()), fcrc(frags.size());
  copy_h2d(ctx, d_frags.get(), frags.data(), sizeof(PageFragment) * frags.size());
  if (codec == pq::SNAPPY) {
    launch_snappy_compress(ctx, d_frags.get(), (int64_t)frags.size(), raw, out->slots.get(), d_flen.get());
  } else if (codec == pq::GZIP) {
    launch_deflate_compress(ctx, d_frags.get(), (int64_t)frags.size(), raw, out->slots.get(), d_flen.get(), d_fcrc.get());
    copy_d2h(ctx, fcrc.data(), d_fcrc.get(), 4 * frags.size());
  } else {
    launch_lz4_compress(ctx, d_frags.get(), (int64_t)frags.size(), raw, out->slots.get(), d_flen.get());
  }
  copy_d2h(ctx, flen.data(), d_flen.get(), 4 * frags.size());
  sync_stream(ctx);
  out->pieces.resize(frags.size());
  for (size_t f = 0; f < frags.size(); f++) out->pieces[f] = BlobCopy{frags[f].dst_off, 0, flen[f], 0};
  out->crc.assign(bodies.size(), 0u);
  if (codec == pq::GZIP) {
    // the member's CRC-32 from its fragments': each is shifted past the bytes after it (gz::crc32_piece's combination)
    for (size_t b = 0; b < bodies.size(); b++) {
      uint32_t x = 0;
      for (size_t f = out->first_piece[b]; f < out->first_piece[b + 1]; f++) {
        const uint64_t after = bodies[b].first + bodies[b].second - frags[f].src_off - frags[f].len;
        x ^= gz::crc32_multmodp(gz::crc32_x8n(after), fcrc[f]);
      }
      out->crc[b] = x;
    }
  }
}

// snappy's preamble is the uncompressed length, as the varint Thrift writes too; the gzip member's is its header
void CompressedBodies::append_preamble(size_t body, std::vector<uint8_t>& out) const {
  if (codec == pq::SNAPPY) {
    thrift::Writer w;
    w.varint(raw_len[body]);
    out.insert(out.end(), w.buf.begin(), w.buf.end());
  } else if (codec == pq::GZIP) {
    out.insert(out.end(), std::begin(gz::kGzipHeader), std::end(gz::kGzipHeader));
  }
}

// the gzip member's final block, CRC-32 and ISIZE
void CompressedBodies::append_trailer(size_t body, std::vector<uint8_t>& out) const {
  if (codec != pq::GZIP) return;
  uint8_t t[10];
  gz::gzip_trailer(crc[body], raw_len[body], t);
  out.insert(out.end(), t, t + sizeof t);
}

uint64_t CompressedBodies::size(size_t body) const {
  std::vector<uint8_t> ends;
  append_preamble(body, ends);
  append_trailer(body, ends);
  uint64_t bytes = ends.size();
  for (size_t f = first_piece[body]; f < first_piece[body + 1]; f++) bytes += pieces[f].len;
  return bytes;
}

void CompressedBodies::place(size_t body, std::vector<BlobCopy>& copies, uint64_t* dst) const {
  for (size_t f = first_piece[body]; f < first_piece[body + 1]; f++) {
    copies.push_back(BlobCopy{pieces[f].src, *dst, pieces[f].len, 0});
    *dst += pieces[f].len;
  }
}

}  // namespace hs
