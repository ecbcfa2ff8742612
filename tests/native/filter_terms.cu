// Host-only driver of the filter terms' NOT, null and pattern handling (predicates.h: resolve_any, complement_set,
// prefix_range, parse_like, compile_pattern, check_anys) and of the matcher (string_match.h), for
// tests/test_filter_terms_host.py.  One case per line on stdin, one line out per case.
//   tset <column> <flags> T        resolve_any: "ok <exact>" and the ranges (tests/native/predicates.cu's format), or "refused"
//   checkt <flags> T               check_anys: "ok" or "refused <code> <message>"
//   prefix <hex>                   prefix_range: the range
//   like <hex>                     parse_like: "ok" and the items (bytes in hex, _ for any character, % for any run)
//   match <kind> <hex pattern> <n> <hex value>...   pattern_matches of the compiled pattern: one 0 / 1 per value
// <column> and T are as in tests/native/predicates.cu ('-' is the empty string).  nvcc compiles it as host code.
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <deque>
#include <iostream>
#include <sstream>
#include <string>
#include <vector>

#include "../../hyperspace_b200/csrc/predicates.h"

using namespace hs;

namespace {

struct Input {
  std::istringstream in;
  std::deque<std::string> keep;
  std::string tok() {
    std::string t;
    if (!(in >> t)) throw std::runtime_error("truncated case");
    return t;
  }
  long long i() { return std::stoll(tok()); }
  std::string bytes() {
    const std::string h = tok();
    std::string b;
    if (h != "-")
      for (size_t k = 0; k + 1 < h.size(); k += 2) b.push_back((char)std::stoi(h.substr(k, 2), nullptr, 16));
    return b;
  }
};

struct Term {
  hs_predicate_any a;
  std::vector<int64_t> vi;
  std::vector<double> vf;
  std::vector<uint64_t> offs{0};
  std::string bytes;
  std::vector<hs_predicate> ranges;
};

void read_value(Input& in, int lit, int64_t* vi, double* vf, const void** b, uint32_t* len) {
  if (lit == HS_TYPE_STRING) {
    in.keep.push_back(in.bytes());
    *b = in.keep.back().data(), *len = (uint32_t)in.keep.back().size();
  } else if (lit == HS_TYPE_DOUBLE) {
    *vf = strtod(in.tok().c_str(), nullptr);
  } else {
    *vi = in.i();
  }
}

void read_term(Input& in, Term* t) {
  memset(&t->a, 0, sizeof t->a);
  t->a.column = "c";
  t->a.literal_type = (int)in.i();
  t->a.scale = (int)in.i();
  t->a.n_values = in.i();
  for (int64_t k = 0; k < t->a.n_values; k++) {
    if (t->a.literal_type == HS_TYPE_STRING) t->bytes += in.bytes(), t->offs.push_back(t->bytes.size());
    else if (t->a.literal_type == HS_TYPE_DOUBLE) t->vf.push_back(strtod(in.tok().c_str(), nullptr));
    else t->vi.push_back(in.i());
  }
  t->a.n_ranges = (int32_t)in.i();
  for (int32_t r = 0; r < t->a.n_ranges; r++) {
    hs_predicate p;
    memset(&p, 0, sizeof p);
    p.column = "c";
    p.literal_type = (int)in.i();
    p.scale = (int)in.i();
    p.has_lo = (int)in.i(), p.lo_strict = (int)in.i();
    read_value(in, p.literal_type, &p.lo_i, &p.lo_f, (const void**)&p.lo_bytes, &p.lo_len);
    p.has_hi = (int)in.i(), p.hi_strict = (int)in.i();
    read_value(in, p.literal_type, &p.hi_i, &p.hi_f, (const void**)&p.hi_bytes, &p.hi_len);
    t->ranges.push_back(p);
  }
  t->a.values_i = t->vi.data(), t->a.values_f = t->vf.data();
  t->a.values_bytes = (const uint8_t*)t->bytes.data(), t->a.values_offsets = t->offs.data();
  t->a.ranges = t->ranges.data();
}

void print_range(bool str, const SetRange& r) {
  auto bound = [&](uint64_t v, const std::string& b) {
    if (!str) return printf(" %llu", (unsigned long long)v), void();
    printf(" %s", b.empty() ? "-" : "");
    for (unsigned char c : b) printf("%02x", c);
  };
  printf(" [%d %d", r.has_lo, r.lo_strict);
  bound(r.lo, r.lo_b);
  printf(" %d %d", r.has_hi, r.hi_strict);
  bound(r.hi, r.hi_b);
  printf("]");
}

void run(const std::string& line) {
  Input in;
  in.in.str(line);
  const std::string op = in.tok();
  try {
    if (op == "tset") {
      const int type = (int)in.i();
      const std::string kind = in.tok();
      const int scale = (int)in.i();
      pq::SchemaColumn schema;
      if (kind == "d") schema.converted_type = pq::CT_DECIMAL, schema.precision = 18, schema.scale = scale;
      if (kind == "t") schema.type = pq::INT64, schema.converted_type = pq::CT_TIMESTAMP_MICROS;
      const std::string name = "c";
      const int flags = (int)in.i();
      Term t;
      read_term(in, &t);
      t.a.flags = flags;
      const ResolvedTerm rt = resolve_any(t.a, PredColumn{type, schema, name});
      printf("ok %d", rt.exact ? 1 : 0);
      for (const SetRange& r : rt.set) print_range(type == HS_TYPE_STRING, r);
      printf("\n");
    } else if (op == "checkt") {
      const int flags = (int)in.i();
      Term t;
      read_term(in, &t);
      t.a.flags = flags;
      char err[256] = "";
      const int rc = check_anys(&t.a, 1, 0, nullptr, err, sizeof err);
      if (rc == HS_OK) printf("ok\n");
      else printf("refused %d %s\n", rc, err);
    } else if (op == "prefix") {
      printf("ok");
      print_range(true, prefix_range(in.bytes()));
      printf("\n");
    } else if (op == "like") {
      const std::vector<uint16_t> items = parse_like(in.bytes());
      printf("ok");
      for (uint16_t it : items) it == kAnyChar ? printf(" _") : (it == kAnyRun ? printf(" %%") : printf(" %02x", it));
      printf("\n");
    } else if (op == "match") {
      const int kind = (int)in.i();
      const CompiledPattern cp = compile_pattern(kind, in.bytes());
      printf("ok");
      for (long long n = in.i(); n > 0; n--) {
        const std::string v = in.bytes();
        printf(" %d", pattern_matches((const uint8_t*)v.data(), (int64_t)v.size(), cp.items.data(), cp.fail.data(), cp.segs.data(),
                                      (int)cp.segs.size(), cp.whole) ? 1 : 0);
      }
      printf("\n");
    } else {
      throw std::runtime_error("unknown op " + op);
    }
  } catch (const Error& e) {
    printf("refused %d %s\n", e.code, e.what());
  }
}

}  // namespace

int main(int argc, char**) {
  if (argc > 1) {
    fprintf(stderr, "usage: filter_terms < cases\n");
    return 2;
  }
  std::string line;
  while (std::getline(std::cin, line))
    if (!line.empty()) run(line);
  return 0;
}
