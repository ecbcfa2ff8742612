// Host-only driver of the index page compressors' per-stream code (hyperspace_b200/csrc/deflate.h and the encoder half of
// lz4_block.h), for tests/test_index_codecs_host.py.  nvcc compiles it as host code; it makes no CUDA call.
//   index_codecs lengths <records> <results>: records [u32 n][u32 limit][n x u32 frequency]; results [n x u8 length] each
//   index_codecs gzip <raw> <results>: one gzip member of stored fragments around raw, built with deflate.h's header,
//       sync-flush and trailer code, then decoded by inflate.h; results [u64 bound][u32 InflateError][member]
//   index_codecs lz4 <raw> <results>: raw in Hadoop groups of one block per 64 KB, sequences found by a serial hash parse
//       under the end-of-block rules and written by lz4_block.h's encoder, then decoded by lz4_block.h;
//       results [u64 bound][u32 Lz4Error][stream]
// Buffers are allocated at their exact sizes, so a build with -fsanitize=address fails on any access outside them.
#include <cstdio>
#include <cstring>
#include <vector>

#include "../../hyperspace_b200/csrc/deflate.h"
#include "../../hyperspace_b200/csrc/lz4_block.h"

using namespace hs;

static std::vector<uint8_t> read_all(const char* path) {
  std::vector<uint8_t> v;
  FILE* f = fopen(path, "rb");
  if (!f) return v;
  uint8_t buf[65536];
  size_t k;
  while ((k = fread(buf, 1, sizeof buf, f)) > 0) v.insert(v.end(), buf, buf + k);
  fclose(f);
  return v;
}

static constexpr uint32_t kFragment = 65536;

static std::vector<uint8_t> gzip_stored(const std::vector<uint8_t>& raw) {
  std::vector<uint8_t> m(std::begin(gz::kGzipHeader), std::end(gz::kGzipHeader));
  uint32_t table[256];
  for (uint32_t i = 0; i < 256; i++) table[i] = gz::crc32_table_entry(i);
  uint32_t x = 0;
  for (uint64_t o = 0; o < raw.size(); o += kFragment) {
    const uint32_t len = (uint32_t)std::min<uint64_t>(kFragment, raw.size() - o);
    for (uint32_t b = 0; b < len; b += 65535) {
      const uint32_t bl = std::min(65535u, len - b);
      uint8_t h[5];
      gz::put_stored_header(h, bl);
      m.insert(m.end(), h, h + 5);
      m.insert(m.end(), raw.begin() + o + b, raw.begin() + o + b + bl);
    }
    uint8_t flush[5];
    gz::put_stored_header(flush, 0);
    m.insert(m.end(), flush, flush + 5);
    x ^= gz::crc32_multmodp(gz::crc32_x8n(raw.size() - o - len), gz::crc32_raw(table, 0u, raw.data() + o, len));
  }
  uint8_t t[10];
  gz::gzip_trailer(x, raw.size(), t);
  m.insert(m.end(), t, t + 10);
  return m;
}

static std::vector<uint8_t> lz4_hadoop(const std::vector<uint8_t>& raw) {
  std::vector<uint8_t> s;
  for (uint64_t o = 0; o < raw.size(); o += kFragment) {
    const uint32_t len = (uint32_t)std::min<uint64_t>(kFragment, raw.size() - o);
    const uint8_t* in = raw.data() + o;
    std::vector<uint8_t> blk(lz4::block_bound(len));
    std::vector<int32_t> table(4096, -1);
    uint32_t op = 0, lit = 0;
    for (uint32_t ip = 0; ip + lz4::kMatchStartMargin <= len;) {
      uint32_t w;
      memcpy(&w, in + ip, 4);
      const uint32_t h = (w * 2654435761u) >> 20;
      const int32_t c = table[h];
      table[h] = (int32_t)ip;
      uint32_t cw = 0;
      if (c >= 0) memcpy(&cw, in + c, 4);
      if (c < 0 || ip - (uint32_t)c > 65535 || cw != w) {
        ip++;
        continue;
      }
      uint32_t m = 4;
      while (ip + m < len - lz4::kLastLiterals && in[ip + m] == in[c + m]) m++;
      op = lz4::put_sequence_head(blk.data(), op, ip - lit, m, true);
      memcpy(blk.data() + op, in + lit, ip - lit);
      op += ip - lit;
      op = lz4::put_match(blk.data(), op, ip - (uint32_t)c, m, true);
      ip += m;
      lit = ip;
    }
    op = lz4::put_sequence_head(blk.data(), op, len - lit, 0, true);
    memcpy(blk.data() + op, in + lit, len - lit);
    op += len - lit;
    uint8_t g[lz4::kHadoopGroupHeader];
    lz4::put_be32(g, len);
    lz4::put_be32(g + 4, op);
    s.insert(s.end(), g, g + sizeof g);
    s.insert(s.end(), blk.begin(), blk.begin() + op);
  }
  return s;
}

int main(int argc, char** argv) {
  if (argc != 4) {
    fprintf(stderr, "usage: index_codecs lengths|gzip|lz4 <in> <out>\n");
    return 2;
  }
  const std::vector<uint8_t> in = read_all(argv[2]);
  FILE* out = fopen(argv[3], "wb");
  if (!out) return 2;
  if (!strcmp(argv[1], "lengths")) {
    for (size_t p = 0; p + 8 <= in.size();) {
      uint32_t n, limit;
      memcpy(&n, in.data() + p, 4);
      memcpy(&limit, in.data() + p + 4, 4);
      p += 8;
      std::vector<uint32_t> freq(n), work(5 * n);
      memcpy(freq.data(), in.data() + p, 4 * n);
      p += 4 * n;
      std::vector<uint8_t> lens(n);
      gz::huffman_lengths(freq.data(), (int)n, (int)limit, lens.data(), work.data());
      fwrite(lens.data(), 1, n, out);
    }
  } else if (!strcmp(argv[1], "gzip")) {
    const std::vector<uint8_t> m = gzip_stored(in);
    const uint64_t bound = gz::gzip_body_bound(in.size(), kFragment);
    std::vector<uint8_t> src(m), dst(in.size());
    gz::InflateTables t;
    uint32_t table[256];
    for (uint32_t i = 0; i < 256; i++) table[i] = gz::crc32_table_entry(i);
    uint8_t none = 0;
    const uint32_t e = gz::inflate_gzip_serial(src.data(), (uint32_t)src.size(), dst.empty() ? &none : dst.data(),
                                               (uint32_t)dst.size(), t, table, 7);
    const uint32_t err = e ? e : (dst == in ? 0u : 0xffffffffu);
    fwrite(&bound, 8, 1, out);
    fwrite(&err, 4, 1, out);
    fwrite(m.data(), 1, m.size(), out);
  } else if (!strcmp(argv[1], "lz4")) {
    const std::vector<uint8_t> s = lz4_hadoop(in);
    uint64_t bound = 0;
    for (uint64_t o = 0; o < in.size(); o += kFragment)
      bound += lz4::kHadoopGroupHeader + lz4::block_bound(std::min<uint64_t>(kFragment, in.size() - o));
    std::vector<uint8_t> src(s), dst(in.size());
    uint8_t none = 0;
    const uint32_t e = lz4::decode_page_serial(lz4::kCodecLz4, src.empty() ? &none : src.data(), (uint32_t)src.size(),
                                               dst.empty() ? &none : dst.data(), (uint32_t)dst.size());
    const uint32_t err = e ? e : (dst == in ? 0u : 0xffffffffu);
    fwrite(&bound, 8, 1, out);
    fwrite(&err, 4, 1, out);
    fwrite(s.data(), 1, s.size(), out);
  } else {
    return 2;
  }
  fclose(out);
  return 0;
}
