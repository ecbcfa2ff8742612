// Host-only driver of the engine's Spark type rules (hyperspace_b200/csrc/spark_types.h), for tests/test_spark_types_host.py.
//   spark_types footer <file.parquet>   per column: what the footer reader parsed (converted and logical type) and what
//                                       source_type_of makes of it -- or the refusal's code and message
//   spark_types compare                 compare_scaled(a, sa, b, sb) over a grid of values and scales, one line each
//   spark_types grid <cs> <ls>          compare_scaled of column values -300..300 (scale cs) with literals (scale ls)
// nvcc compiles it as host code; it makes no CUDA call.
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "../../hyperspace_b200/csrc/spark_types.h"

using namespace hs;

static std::vector<uint8_t> read_file(const char* path) {
  FILE* f = fopen(path, "rb");
  if (!f) return {};
  std::vector<uint8_t> b;
  uint8_t buf[65536];
  size_t n;
  while ((n = fread(buf, 1, sizeof buf, f)) > 0) b.insert(b.end(), buf, buf + n);
  fclose(f);
  return b;
}

int main(int argc, char** argv) {
  if (argc >= 3 && strcmp(argv[1], "footer") == 0) {
    std::vector<uint8_t> img = read_file(argv[2]);
    pq::FileMeta fm = pq::parse_footer(img.data(), img.size(), argv[2]);
    for (const pq::SchemaColumn& c : fm.columns) {
      printf("column %s parsed type=%d length=%d converted=%d precision=%d scale=%d unit=%d", c.name.c_str(), c.type,
             c.type_length, c.converted_type, c.precision, c.scale, c.time_unit);
      try {
        const SourceType st = source_type_of(c, argv[2]);
        printf(" -> hs_type=%d conv=%d type=%d converted=%d precision=%d scale=%d spark=%s\n", st.type, st.conv, st.schema.type,
               st.schema.converted_type, st.schema.precision, st.schema.scale, pq::spark_type_name(st.schema).c_str());
      } catch (const Error& e) {
        printf(" -> refused code=%d %s\n", e.code, e.what());
      }
    }
    return 0;
  }
  if (argc >= 2 && strcmp(argv[1], "compare") == 0) {
    const int64_t vals[] = {INT64_MIN, -1000000000000000007ll, -1001, -100, -15, -1, 0, 1, 15, 99, 100, 101,
                            1000000000000000003ll, INT64_MAX};
    const int sa[] = {0, 1, 2, 18}, sb[] = {0, 1, 3, 18, 19, 20, 25, 38};
    for (int64_t a : vals)
      for (int64_t b : vals)
        for (int x : sa)
          for (int y : sb) printf("%lld %d %lld %d %d\n", (long long)a, x, (long long)b, y, compare_scaled(a, x, b, y));
    return 0;
  }
  if (argc >= 4 && strcmp(argv[1], "grid") == 0) {  // column values -300..300 of scale argv[2] against literals of scale argv[3]
    const int cs = atoi(argv[2]), ls = atoi(argv[3]);
    for (int64_t v = -300; v <= 300; v++)
      for (int64_t lit = -250; lit <= 250; lit += 7) printf("%lld %lld %d\n", (long long)v, (long long)lit, compare_scaled(v, cs, lit, ls));
    return 0;
  }
  fprintf(stderr, "usage: spark_types footer <file> | compare | grid <column scale> <literal scale>\n");
  return 2;
}
