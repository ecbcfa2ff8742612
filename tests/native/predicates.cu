// Host-only driver of the engine's predicate resolution (hyperspace_b200/csrc/predicates.h), for tests/test_predicates_host.py.
// Reads one case per line from stdin and prints one line per case: "ok" and the resulting ranges, or "refused <code> <message>".
//   <op> <column> <args>
//   column    <hs type> <p | d | t> <scale>    plain, decimal (of that scale) or timestamp
//   range C P                                  resolve_range
//   term C T                                   resolve_term
//   inter C T T                                intersect_sets of two resolved terms
//   fold C n P...                              intersect_range over n resolved predicates, from the open range
//   norm C n R...                              normalise_set of n ranges given as they are
//   checkp P / checkt T                        check_predicates / check_anys
//   P: <literal type> <scale> <has_lo> <lo_strict> <lo> <has_hi> <hi_strict> <hi>
//      values by literal type: integers in decimal, doubles as C hex floats (or nan / inf / -inf), strings as hex bytes
//      ('-' for none); literal type -1 follows the column
//   T: <literal type> <scale> <n values> <value>... <n ranges> P...
//   R: <has_lo> <lo_strict> <lo> <has_hi> <hi_strict> <hi>  (numeric bounds as encoded values)
// A range prints as [has_lo lo_strict lo has_hi hi_strict hi]: encoded values, or hex bytes for strings.
// nvcc compiles it as host code; it makes no CUDA call.
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
  std::deque<std::string> keep;  // bytes and names the predicates point into
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

struct Column {
  int type;
  pq::SchemaColumn schema;
  std::string name = "c";
  PredColumn view() const { return PredColumn{type, schema, name}; }
};

Column read_column(Input& in) {
  Column c;
  c.type = (int)in.i();
  const std::string kind = in.tok();
  const int scale = (int)in.i();
  if (kind == "d") c.schema.converted_type = pq::CT_DECIMAL, c.schema.precision = 18, c.schema.scale = scale;
  if (kind == "t") c.schema.type = pq::INT64, c.schema.converted_type = pq::CT_TIMESTAMP_MICROS;
  return c;
}

// one bound of a predicate, by its literal type (-1: the column's)
void read_value(Input& in, int lit, int col_type, int64_t* vi, double* vf, const void** b, uint32_t* len) {
  if (lit == HS_TYPE_STRING || (lit < 0 && col_type == HS_TYPE_STRING)) {
    in.keep.push_back(in.bytes());
    *b = in.keep.back().data(), *len = (uint32_t)in.keep.back().size();
  } else if (lit == HS_TYPE_DOUBLE) {
    *vf = strtod(in.tok().c_str(), nullptr);
  } else {
    *vi = in.i();
  }
}

hs_predicate read_pred(Input& in, int col_type) {
  hs_predicate p;
  memset(&p, 0, sizeof p);
  p.column = "c";
  p.literal_type = (int)in.i();
  p.scale = (int)in.i();
  p.has_lo = (int)in.i(), p.lo_strict = (int)in.i();
  read_value(in, p.literal_type, col_type, &p.lo_i, &p.lo_f, (const void**)&p.lo_bytes, &p.lo_len);
  p.has_hi = (int)in.i(), p.hi_strict = (int)in.i();
  read_value(in, p.literal_type, col_type, &p.hi_i, &p.hi_f, (const void**)&p.hi_bytes, &p.hi_len);
  return p;
}

struct Term {
  hs_predicate_any a;
  std::vector<int64_t> vi;
  std::vector<double> vf;
  std::vector<uint64_t> offs{0};
  std::string bytes;
  std::vector<hs_predicate> ranges;
};

void read_term(Input& in, int col_type, Term* t) {
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
  for (int32_t r = 0; r < t->a.n_ranges; r++) t->ranges.push_back(read_pred(in, col_type));
  t->a.values_i = t->vi.data(), t->a.values_f = t->vf.data();
  t->a.values_bytes = (const uint8_t*)t->bytes.data(), t->a.values_offsets = t->offs.data();
  t->a.ranges = t->ranges.data();
}

void print_ranges(bool str, const RangeSet& s) {
  auto bound = [&](uint64_t v, const std::string& b) {
    if (!str) return printf(" %llu", (unsigned long long)v), void();
    printf(" %s", b.empty() ? "-" : "");
    for (unsigned char c : b) printf("%02x", c);
  };
  printf("ok");
  for (const SetRange& r : s) {
    printf(" [%d %d", r.has_lo, r.lo_strict);
    bound(r.lo, r.lo_b);
    printf(" %d %d", r.has_hi, r.hi_strict);
    bound(r.hi, r.hi_b);
    printf("]");
  }
  printf("\n");
}

void run(const std::string& line) {
  Input in;
  in.in.str(line);
  const std::string op = in.tok();
  char err[256] = "";
  if (op == "checkp" || op == "checkt") {
    int rc;
    if (op == "checkp") {
      const hs_predicate p = read_pred(in, -1);
      rc = check_predicates(&p, 1, false, nullptr, err, sizeof err);
    } else {
      Term t;
      read_term(in, -1, &t);
      rc = check_anys(&t.a, 1, 0, nullptr, err, sizeof err);
    }
    if (rc == HS_OK) printf("ok\n");
    else printf("refused %d %s\n", rc, err);
    return;
  }
  const Column c = read_column(in);
  const bool str = c.type == HS_TYPE_STRING;
  try {
    RangeSet out;
    if (op == "range") {
      out.push_back(resolve_range(read_pred(in, c.type), c.view()));
    } else if (op == "term") {
      Term t;
      read_term(in, c.type, &t);
      out = resolve_term(t.a, c.view());
    } else if (op == "inter") {
      Term a, b;
      read_term(in, c.type, &a);
      read_term(in, c.type, &b);
      out = intersect_sets(str, resolve_term(a.a, c.view()), resolve_term(b.a, c.view()));
    } else if (op == "fold") {
      SetRange r;
      for (long long k = in.i(); k > 0; k--) r = intersect_range(str, r, resolve_range(read_pred(in, c.type), c.view()));
      out.push_back(r);
    } else if (op == "norm") {
      for (long long k = in.i(); k > 0; k--) {
        SetRange r;
        r.has_lo = in.i(), r.lo_strict = in.i();
        if (str) r.lo_b = in.bytes();
        else r.lo = std::stoull(in.tok());
        r.has_hi = in.i(), r.hi_strict = in.i();
        if (str) r.hi_b = in.bytes();
        else r.hi = std::stoull(in.tok());
        out.push_back(r);
      }
      normalise_set(str, &out);
    } else {
      throw std::runtime_error("unknown op " + op);
    }
    print_ranges(str, out);
  } catch (const Error& e) {
    printf("refused %d %s\n", e.code, e.what());
  }
}

}  // namespace

int main(int argc, char**) {
  if (argc > 1) {
    fprintf(stderr, "usage: predicates < cases\n");
    return 2;
  }
  std::string line;
  while (std::getline(std::cin, line))
    if (!line.empty()) run(line);
  return 0;
}
