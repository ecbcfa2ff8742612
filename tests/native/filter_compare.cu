// Host-only driver of the comparisons between two columns: their coercion (predicates.h: resolve_compare, check_compares)
// and the scalar comparison (column_compare.h: compare_holds, decimal_to_double), for tests/test_filter_compare_host.py.
// One case per line on stdin, one line out per case.
//   resolve L R <op> <flags>         resolve_compare: "ok <domain> <factor0> <factor1>", or "refused <code> <message>"
//   check <left|-> <right|-> <op> <flags> <n_others>   check_compares of one comparison: "ok" or "refused <code> <message>"
//   sides <left op> <left pred ok> <right op> <right pred ok>   check_filters of two sides, each with the comparison a OP b
//                                    and one predicate on a, without a column when "pred ok" is 0: as check
//   rows L R <op> <flags> <n> then n times: <lnull> <lvalue> <rnull> <rvalue>    compare_holds per row: "ok" and 0 / 1 each
//   d2d <unscaled> <scale>           decimal_to_double: "ok" and the double's bits in hex
// A column L / R is "<kind> <precision> <scale>": kind one of integer long float double string binary date timestamp decimal
// boolean byte.  Values: integers (unscaled for decimals, days for dates, micros for timestamps) in decimal, floating point
// as strtod reads it (nan, inf, -0), strings in hex ('-' is the empty string).  nvcc compiles it as host code.
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
  std::string tok() {
    std::string t;
    if (!(in >> t)) throw std::runtime_error("truncated case");
    return t;
  }
  long long i() { return std::stoll(tok()); }
};

struct Col {
  int type = HS_TYPE_INT32;
  pq::SchemaColumn schema;
  std::string name;
  std::vector<int32_t> i32;
  std::vector<int64_t> i64;
  std::vector<float> f32;
  std::vector<double> f64;
  std::deque<std::string> bytes;
  std::vector<uint64_t> refs;
  std::vector<uint8_t> valid;
  bool has_nulls = false;

  const void* data() const {
    switch (type) {
      case HS_TYPE_INT32: return i32.data();
      case HS_TYPE_INT64: return i64.data();
      case HS_TYPE_FLOAT: return f32.data();
      case HS_TYPE_DOUBLE: return f64.data();
      default: return refs.data();
    }
  }
  void push(Input& in) {
    const bool null = in.i() != 0;
    const std::string v = in.tok();
    valid.push_back(null ? 0 : 1);
    has_nulls = has_nulls || null;
    switch (type) {
      case HS_TYPE_INT32: i32.push_back(null ? 0 : (int32_t)std::stoll(v)); break;
      case HS_TYPE_INT64: i64.push_back(null ? 0 : (int64_t)std::stoll(v)); break;
      case HS_TYPE_FLOAT: f32.push_back(null ? 0.f : strtof(v.c_str(), nullptr)); break;
      case HS_TYPE_DOUBLE: f64.push_back(null ? 0.0 : strtod(v.c_str(), nullptr)); break;
      default: {
        std::string b;
        if (v != "-")
          for (size_t k = 0; k + 1 < v.size(); k += 2) b.push_back((char)std::stoi(v.substr(k, 2), nullptr, 16));
        bytes.push_back(b);
        refs.push_back(0);
      }
    }
  }
  void finish() {  // string references into the deque's (stable) strings
    for (size_t k = 0; k < bytes.size(); k++) refs[k] = string_ref(bytes[k].data(), (uint32_t)bytes[k].size());
  }
};

void read_col(Input& in, Col* c, const char* name) {
  const std::string kind = in.tok();
  const int precision = (int)in.i(), scale = (int)in.i();
  c->name = name;
  pq::SchemaColumn& s = c->schema;
  s.converted_type = -1;
  if (kind == "integer" || kind == "byte" || kind == "date") {
    c->type = HS_TYPE_INT32, s.type = pq::INT32;
    if (kind == "date") s.converted_type = pq::CT_DATE;
    if (kind == "byte") s.converted_type = 15;
  } else if (kind == "long" || kind == "timestamp") {
    c->type = HS_TYPE_INT64, s.type = pq::INT64;
    if (kind == "timestamp") s.converted_type = pq::CT_TIMESTAMP_MICROS;
  } else if (kind == "float") {
    c->type = HS_TYPE_FLOAT, s.type = pq::FLOAT;
  } else if (kind == "double") {
    c->type = HS_TYPE_DOUBLE, s.type = pq::DOUBLE;
  } else if (kind == "string" || kind == "binary") {
    c->type = HS_TYPE_STRING, s.type = pq::BYTE_ARRAY;
    if (kind == "string") s.converted_type = 0;
  } else if (kind == "decimal") {
    c->type = precision <= 9 ? HS_TYPE_INT32 : HS_TYPE_INT64;
    s.type = precision <= 9 ? pq::INT32 : pq::INT64;
    s.converted_type = pq::CT_DECIMAL, s.precision = precision, s.scale = scale;
  } else if (kind == "boolean") {
    c->type = HS_TYPE_BOOL, s.type = pq::BOOLEAN;
  } else {
    throw std::runtime_error("unknown column kind " + kind);
  }
}

void run(const std::string& line) {
  Input in;
  in.in.str(line);
  const std::string op = in.tok();
  try {
    if (op == "resolve" || op == "rows") {
      Col l, r;
      read_col(in, &l, "a");
      read_col(in, &r, "b");
      hs_column_compare cc{"a", "b", (int32_t)in.i(), (int32_t)in.i()};
      CompareDesc d = resolve_compare(cc, PredColumn{l.type, l.schema, l.name}, PredColumn{r.type, r.schema, r.name});
      if (op == "resolve") {
        printf("ok %d %lld %lld\n", d.domain, (long long)d.factor[0], (long long)d.factor[1]);
        return;
      }
      const long long n = in.i();
      for (long long k = 0; k < n; k++) l.push(in), r.push(in);
      l.finish(), r.finish();
      d.col[0] = l.data(), d.col[1] = r.data();
      d.valid[0] = l.has_nulls ? l.valid.data() : nullptr, d.valid[1] = r.has_nulls ? r.valid.data() : nullptr;
      printf("ok");
      for (long long k = 0; k < n; k++) printf(" %d", compare_holds(d, k) ? 1 : 0);
      printf("\n");
    } else if (op == "check") {
      const std::string a = in.tok(), b = in.tok();
      hs_column_compare cc{a == "-" ? nullptr : a.c_str(), b == "-" ? nullptr : b.c_str(), (int32_t)in.i(), (int32_t)in.i()};
      const int n_others = (int)in.i();
      char err[256] = "";
      const int rc = check_compares(&cc, 1, n_others, nullptr, err, sizeof err);
      if (rc == HS_OK) printf("ok\n");
      else printf("refused %d %s\n", rc, err);
    } else if (op == "sides") {
      hs_column_compare cc[2];
      hs_predicate p[2];
      Filter f[2];
      for (int s = 0; s < 2; s++) {
        cc[s] = hs_column_compare{"a", "b", (int32_t)in.i(), 0};
        p[s] = hs_predicate{};
        p[s].column = in.i() ? "a" : nullptr, p[s].has_lo = 1, p[s].literal_type = HS_TYPE_INT64;
        f[s].preds = &p[s], f[s].n_preds = 1, f[s].cmps = &cc[s], f[s].n_cmps = 1;
      }
      char err[256] = "";
      const int rc = check_filters(f, 2, false, nullptr, err, sizeof err);
      if (rc == HS_OK) printf("ok\n");
      else printf("refused %d %s\n", rc, err);
    } else if (op == "d2d") {
      const int64_t u = (int64_t)in.i();
      const int s = (int)in.i();
      const double d = decimal_to_double(u, pow10_i64(s));
      uint64_t b;
      memcpy(&b, &d, 8);
      printf("ok %016llx\n", (unsigned long long)b);
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
    fprintf(stderr, "usage: filter_compare < cases\n");
    return 2;
  }
  std::string line;
  while (std::getline(std::cin, line))
    if (!line.empty()) run(line);
  return 0;
}
