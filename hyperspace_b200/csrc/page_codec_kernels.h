// page_codec_kernels.h -- what page_codec.cu and the codec kernel files (snappy.cu, inflate.cu, lz4.cu) share.  Private to
// those four translation units: everyone else goes through decompress_pages / decompress_blobs / compress_bodies (kernels.h).
#pragma once
#include "kernels.h"

namespace hs {

// snappy: 64 KB output blocks of a blob, the unit of the decoder's parallelism
__host__ __device__ inline uint32_t snappy_blocks_of(uint32_t dst_len, uint32_t prefix) {
  const uint32_t body = dst_len - prefix;
  return body == 0 ? 1u : (body + 65535u) / 65536u;
}
// The n blobs are snappy's, with first_block filled; total_blocks is their sum of snappy_blocks_of.
// block_in: one uint32 per block (+1), sequential: one uint32 per blob -- scratch of the two launches
// any_verbatim: some blob has a prefix or is stored uncompressed
void launch_snappy_decompress(hs_ctx* ctx, const PageBlob* blobs, int64_t n, int64_t total_blocks, bool any_verbatim,
                              uint32_t* block_in, uint32_t* sequential, uint8_t* scratch, uint32_t* d_error);

// GZIP page bodies, one warp per blob: copies what is stored verbatim (prefix, or the whole page when !compressed) and
// inflates the rest; a failed check sets (DERR_GZIP << 24 | gz::InflateError) in d_error
void launch_inflate(hs_ctx* ctx, const PageBlob* blobs, int64_t n, uint8_t* scratch, uint32_t* d_error);

// LZ4 (codec 5, Hadoop-framed) and LZ4_RAW (codec 7) page bodies, one warp per blob: copies what is stored verbatim and
// decodes the rest; a failed check sets (DERR_LZ4 << 24 | lz4::Lz4Error) in d_error
void launch_lz4(hs_ctx* ctx, const PageBlob* blobs, int64_t n, uint8_t* scratch, uint32_t* d_error);

// Compression of page bodies: one warp per fragment (<= 65536 bytes) of a page; fragment f of raw bytes [src_off, src_off +
// len) is written to scratch at dst_off (room for the codec's bound below), its compressed length to out_len[f].
struct PageFragment {
  uint64_t src_off, dst_off;
  uint32_t len, pad;
};
constexpr uint32_t kCompressFragment = 65536;
// SNAPPY: the fragment's element stream (the body's varint preamble is the host's)
inline uint64_t snappy_max_compressed(uint64_t len) { return 32 + len + len / 6; }
void launch_snappy_compress(hs_ctx* ctx, const PageFragment* frags, int64_t n, const uint8_t* raw, uint8_t* scratch,
                            uint32_t* out_len);
// GZIP: the fragment's DEFLATE blocks, ending in a sync flush (room: gz::deflate_fragment_bound + 4, as the last word is
// stored whole), and out_crc[f], its CRC-32 without pre- and post-inversion (the member around it is the host's)
void launch_deflate_compress(hs_ctx* ctx, const PageFragment* frags, int64_t n, const uint8_t* raw, uint8_t* scratch,
                             uint32_t* out_len, uint32_t* out_crc);
// LZ4: the fragment as one block in a Hadoop group of one chunk (room: lz4::kHadoopGroupHeader + lz4::block_bound)
void launch_lz4_compress(hs_ctx* ctx, const PageFragment* frags, int64_t n, const uint8_t* raw, uint8_t* scratch,
                         uint32_t* out_len);

}  // namespace hs
