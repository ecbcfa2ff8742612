// Host-only driver of the Spark functions inside expression comparisons (`year(d) = 1995`, `substring(s, 1, 2) = '13'`):
// their typing (predicates.h: resolve_expr, check_exprs) and the evaluator (column_expr.h: expr_holds<true>, date_part),
// for tests/test_filter_func_host.py.  One case per line on stdin, one line out per case.
//   resolve <n> <column>... <op> <flags> <left> | <right>     resolve_expr: "ok <domain> <funcs> <instruction ops...>", or
//                                                              "refused <code> <message>"
//   rows <n> <column>... <op> <flags> <left> | <right> ; <rows> then, per row, per column: <null> <value>
//                                                              expr_holds<true> per row: "ok" and 0 / 1 each
//   check <n_others> <op> <flags> <left> | <right>             check_exprs of one comparison: "ok" or "refused ..."
//   calendar <lo> <hi>                                         date_part of every day in [lo, hi]: one line per day,
//                                                              year quarter month dayofmonth dayofweek dayofyear weekofyear
// A column is "<name> <kind> <precision> <scale>" as in filter_expr.cu.  A side is filter_expr.cu's tokens plus s:<hex> (a
// string literal, its bytes in hex), D:<days>, T:<micros>, the functions by their Spark names (year .. abs) and
// coalesce:<n>.  A string or binary value is h<hex>.  nvcc compiles it as host code.
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
  std::deque<std::string> str;  // the bytes the references point to (a deque: they stay where they are)
  std::vector<uint64_t> refs;
  std::vector<uint8_t> valid;
  bool has_nulls = false;

  const void* data() const {
    switch (type) {
      case HS_TYPE_INT32: return i32.data();
      case HS_TYPE_INT64: return i64.data();
      case HS_TYPE_FLOAT: return f32.data();
      case HS_TYPE_STRING: return refs.data();
      default: return f64.data();
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
      case HS_TYPE_STRING:
        str.push_back(null ? std::string() : unhex(v.substr(1)));
        refs.push_back(string_ref(str.back().data(), (uint32_t)str.back().size()));
        break;
      default: f64.push_back(null ? 0.0 : strtod(v.c_str(), nullptr)); break;
    }
  }
  static std::string unhex(const std::string& h) {
    std::string out;
    for (size_t k = 0; k + 1 < h.size(); k += 2) out.push_back((char)std::stoi(h.substr(k, 2), nullptr, 16));
    return out;
  }
};

void read_col(Input& in, Col* c) {
  c->name = in.tok();
  const std::string kind = in.tok();
  const int precision = (int)in.i(), scale = (int)in.i();
  pq::SchemaColumn& s = c->schema;
  s.converted_type = -1;
  if (kind == "integer" || kind == "byte" || kind == "short" || kind == "date") {
    c->type = HS_TYPE_INT32, s.type = pq::INT32;
    if (kind == "date") s.converted_type = pq::CT_DATE;
    if (kind == "byte") s.converted_type = 15;
    if (kind == "short") s.converted_type = 16;
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

// One side's tokens up to `end` ("|", ";" or the end of the line) as nodes; names stays the owner of the column names
const char* const kFuncs[] = {"year", "quarter", "month", "dayofmonth", "dayofweek", "dayofyear", "weekofyear", "hour", "minute",
                              "second", "date_add", "date_sub", "datediff", "length", "substring", "abs"};

std::vector<hs_expr_node> read_side(Input& in, const char* end, std::deque<std::string>* names) {
  std::vector<hs_expr_node> out;
  std::string t;
  while (in.in >> t && t != end) {
    hs_expr_node x{};
    int fn = -1;
    for (int k = 0; k < 16; k++)
      if (t == kFuncs[k]) fn = k;
    if (fn >= 0) {
      x.kind = HS_EXPR_YEAR + fn;
    } else if (t.rfind("coalesce:", 0) == 0) {
      x.kind = HS_EXPR_COALESCE, x.value_i = std::stoll(t.substr(9));
    } else if (t.rfind("s:", 0) == 0) {
      names->push_back(Col::unhex(t.substr(2)));
      x.kind = HS_EXPR_LITERAL, x.literal_type = HS_TYPE_STRING, x.column = names->back().c_str(), x.value_i = (int64_t)names->back().size();
    } else if (t == "+" || t == "-" || t == "*" || t == "/" || t == "%" || t == "neg") {
      x.kind = t == "+" ? HS_EXPR_ADD : t == "-" ? HS_EXPR_SUB : t == "*" ? HS_EXPR_MUL : t == "/" ? HS_EXPR_DIV : t == "%" ? HS_EXPR_REM : HS_EXPR_NEG;
    } else if (t.size() > 2 && t[1] == ':') {
      const std::string v = t.substr(2);
      switch (t[0]) {
        case 'c':
          x.kind = HS_EXPR_COLUMN;
          if (v != "-") names->push_back(v), x.column = names->back().c_str();
          break;
        case 'i': x.kind = HS_EXPR_LITERAL, x.literal_type = HS_TYPE_INT32, x.value_i = std::stoll(v); break;
        case 'l': x.kind = HS_EXPR_LITERAL, x.literal_type = HS_TYPE_INT64, x.value_i = std::stoll(v); break;
        case 'd': x.kind = HS_EXPR_LITERAL, x.literal_type = HS_TYPE_DOUBLE, x.value_f = strtod(v.c_str(), nullptr); break;
        case 'm': {
          const size_t colon = v.find(':');
          x.kind = HS_EXPR_LITERAL, x.literal_type = HS_TYPE_DECIMAL;
          x.value_i = std::stoll(v.substr(0, colon)), x.scale = std::stoi(v.substr(colon + 1));
          break;
        }
        case 't': {
          const size_t colon = v.find(':');
          x.kind = HS_EXPR_LITERAL, x.literal_type = std::stoi(v.substr(0, colon)), x.value_i = std::stoll(v.substr(colon + 1));
          break;
        }
        case 'k': x.kind = std::stoi(v); break;
        case 'D': x.kind = HS_EXPR_LITERAL, x.literal_type = HS_TYPE_DATE, x.value_i = std::stoll(v); break;
        case 'T': x.kind = HS_EXPR_LITERAL, x.literal_type = HS_TYPE_TIMESTAMP, x.value_i = std::stoll(v); break;
        default: throw std::runtime_error("unknown token " + t);
      }
    } else {
      throw std::runtime_error("unknown token " + t);
    }
    out.push_back(x);
  }
  return out;
}

void run(const std::string& line) {
  Input in;
  in.in.str(line);
  const std::string what = in.tok();
  try {
    if (what == "resolve" || what == "rows") {
      const int n = (int)in.i();
      std::deque<Col> cols(n);
      for (Col& c : cols) read_col(in, &c);
      const int op = (int)in.i(), flags = (int)in.i();
      std::deque<std::string> names;
      const std::vector<hs_expr_node> l = read_side(in, "|", &names), r = read_side(in, ";", &names);
      const hs_expr_compare e{l.data(), (int32_t)l.size(), r.data(), (int32_t)r.size(), op, flags};
      char err[256] = "";
      const int rc = check_exprs(&e, 1, 0, nullptr, err, sizeof err);
      if (rc != HS_OK) {
        printf("refused %d %s\n", rc, err);
        return;
      }
      // the columns of the COLUMN nodes, left side first, as api.cu binds them
      std::vector<PredColumn> pcs;
      std::vector<const Col*> used;
      for (const std::vector<hs_expr_node>* side : {&l, &r})
        for (const hs_expr_node& x : *side) {
          if (x.kind != HS_EXPR_COLUMN) continue;
          const Col* c = nullptr;
          for (const Col& k : cols)
            if (k.name == x.column) c = &k;
          if (!c) throw std::runtime_error(std::string("unknown column ") + x.column);
          pcs.push_back(PredColumn{c->type, c->schema, c->name});
          used.push_back(c);
        }
      ExprProgram pg = resolve_expr(e, pcs);
      // the pool placed as api.cu's upload_exprs places it: an allocation of at least 16 bytes, relocated even when empty
      std::vector<uint8_t> pool(std::max<size_t>(16, pg.pool.size()));
      std::copy(pg.pool.begin(), pg.pool.end(), pool.begin());
      relocate_strings(&pg.insts, pool.data());
      if (what == "resolve") {
        printf("ok %d %d", pg.domain, pg.funcs ? 1 : 0);
        for (const ExprInst& i : pg.insts) printf(" %d", i.op);
        printf("\n");
        return;
      }
      const long long rows = in.i();
      for (long long k = 0; k < rows; k++)
        for (Col& c : cols) c.push(in);
      std::vector<ExprColumn> ecols;
      for (const Col* c : used) ecols.push_back(ExprColumn{c->data(), c->has_nulls ? c->valid.data() : nullptr, c->type});
      const ExprDesc d{0, (int32_t)pg.insts.size(), pg.domain, pg.op, pg.negate};
      printf("ok");
      for (long long k = 0; k < rows; k++) printf(" %d", expr_holds<true>(d, pg.insts.data(), ecols.data(), k) ? 1 : 0);
      printf("\n");
    } else if (what == "check") {
      const int n_others = (int)in.i(), op = (int)in.i(), flags = (int)in.i();
      std::deque<std::string> names;
      const std::vector<hs_expr_node> l = read_side(in, "|", &names), r = read_side(in, ";", &names);
      const hs_expr_compare e{l.empty() ? nullptr : l.data(), (int32_t)l.size(), r.empty() ? nullptr : r.data(), (int32_t)r.size(), op, flags};
      char err[256] = "";
      const int rc = check_exprs(&e, 1, n_others, nullptr, err, sizeof err);
      if (rc == HS_OK) printf("ok\n");
      else printf("refused %d %s\n", rc, err);
    } else if (what == "calendar") {
      const long long lo = in.i(), hi = in.i();
      std::string out;
      char buf[96];
      for (long long d = lo; d <= hi; d++) {
        snprintf(buf, sizeof buf, "%d %d %d %d %d %d %d\n", date_part(d, kPartYear), date_part(d, kPartQuarter), date_part(d, kPartMonth),
                 date_part(d, kPartDayOfMonth), date_part(d, kPartDayOfWeek), date_part(d, kPartDayOfYear), date_part(d, kPartWeekOfYear));
        out += buf;
      }
      fwrite(out.data(), 1, out.size(), stdout);
    } else {
      throw std::runtime_error("unknown op " + what);
    }
  } catch (const Error& e) {
    printf("refused %d %s\n", e.code, e.what());
  }
}

}  // namespace

int main(int argc, char**) {
  if (argc > 1) {
    fprintf(stderr, "usage: filter_func < cases\n");
    return 2;
  }
  std::string line;
  while (std::getline(std::cin, line))
    if (!line.empty()) run(line);
  return 0;
}
