// Host-only driver of the LZ4 page decoder's per-stream code (hyperspace_b200/csrc/lz4_block.h), for tests/test_lz4_host.py.
//   lz4 <records> <results>
// records: [u32 codec (5 or 7)][u32 compressed length][u32 uncompressed length][compressed bytes] ...
// results: per record [u32 Lz4Error][u32 output length][output bytes when the error is 0]
// Every stream is copied into a buffer of exactly its length, and decoded into one of exactly the uncompressed length, so a
// build with -fsanitize=address fails on any access outside them.  nvcc compiles it as host code; it makes no CUDA call.
#include <cstdio>

#include "../../hyperspace_b200/csrc/lz4_block.h"

using namespace hs;

int main(int argc, char** argv) {
  if (argc != 3) {
    fprintf(stderr, "usage: lz4 <records> <results>\n");
    return 2;
  }
  FILE* in = fopen(argv[1], "rb");
  FILE* out = fopen(argv[2], "wb");
  if (!in || !out) return 2;
  uint32_t hdr[3];
  while (fread(hdr, 4, 3, in) == 3) {
    uint8_t* src = new uint8_t[hdr[1] ? hdr[1] : 1];
    uint8_t* dst = new uint8_t[hdr[2] ? hdr[2] : 1];
    if (hdr[1] && fread(src, 1, hdr[1], in) != hdr[1]) return 2;
    const uint32_t e = lz4::decode_page_serial(hdr[0], src, hdr[1], dst, hdr[2]);
    const uint32_t res[2] = {e, e ? 0u : hdr[2]};
    fwrite(res, 4, 2, out);
    if (!e) fwrite(dst, 1, hdr[2], out);
    delete[] src;
    delete[] dst;
  }
  fclose(in);
  fclose(out);
  return 0;
}
