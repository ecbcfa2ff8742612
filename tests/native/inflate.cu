// Host-only driver of the GZIP page decoder's per-stream code (hyperspace_b200/csrc/inflate.h), for
// tests/test_inflate_host.py.
//   inflate <records> <results>
// records: [u32 compressed length][u32 uncompressed length][compressed bytes] ...
// results: per record [u32 InflateError][u32 output length][output bytes when the error is 0]
// Every stream is copied into a buffer of exactly its length, and decoded into one of exactly the uncompressed length, so a
// build with -fsanitize=address fails on any access outside them.  The member CRC is computed in 32 pieces, as a warp does.
// nvcc compiles it as host code; it makes no CUDA call.
#include <cstdio>
#include <cstring>
#include <vector>

#include "../../hyperspace_b200/csrc/inflate.h"

using namespace hs;

int main(int argc, char** argv) {
  if (argc != 3) {
    fprintf(stderr, "usage: inflate <records> <results>\n");
    return 2;
  }
  FILE* in = fopen(argv[1], "rb");
  FILE* out = fopen(argv[2], "wb");
  if (!in || !out) return 2;
  uint32_t table[256];
  for (uint32_t i = 0; i < 256; i++) table[i] = gz::crc32_table_entry(i);
  gz::InflateTables* t = new gz::InflateTables();
  uint32_t hdr[2];
  while (fread(hdr, 4, 2, in) == 2) {
    uint8_t* src = new uint8_t[hdr[0] ? hdr[0] : 1];
    uint8_t* dst = new uint8_t[hdr[1] ? hdr[1] : 1];
    if (hdr[0] && fread(src, 1, hdr[0], in) != hdr[0]) return 2;
    const uint32_t e = gz::inflate_gzip_serial(src, hdr[0], dst, hdr[1], *t, table, 32);
    const uint32_t res[2] = {e, e ? 0u : hdr[1]};
    fwrite(res, 4, 2, out);
    if (!e) fwrite(dst, 1, hdr[1], out);
    delete[] src;
    delete[] dst;
  }
  delete t;
  fclose(in);
  fclose(out);
  return 0;
}
