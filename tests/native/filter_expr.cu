// Host-only driver of the expression comparisons: their typing (predicates.h: resolve_expr, check_exprs, check_filters)
// and the evaluator (column_expr.h: expr_holds), for tests/test_filter_expr_host.py.  One case per line on stdin, one
// line out per case.
//   resolve <n> <column>... <op> <flags> <left> | <right>     resolve_expr: "ok <domain> <instruction ops...>", or
//                                                              "refused <code> <message>"
//   rows <n> <column>... <op> <flags> <left> | <right> ; <rows> then, per row, per column: <null> <value>
//                                                              expr_holds per row: "ok" and 0 / 1 each
//   check <n_others> <op> <flags> <left> | <right>             check_exprs of one comparison: "ok" or "refused ..."
//   sides <left pred ok> <left op> <right pred ok> <right op>  check_filters of two sides, each with one predicate on a
//                                                              (without a column when "pred ok" is 0) and `(a + 1) OP b`
// A column is "<name> <kind> <precision> <scale>", kind one of integer long float double decimal string binary date
// timestamp boolean byte short.  A side is postfix tokens: c:<name> (c:- a column without a name), i:<int32>, l:<int64>,
// d:<double>, m:<unscaled>:<scale> literals, t:<type>:<value> an integer literal of any literal_type, the operators
// + - * / % neg, and k:<kind> a node of that kind.  Values: integers (unscaled for decimals) in decimal, floating point
// as strtod reads it (nan, inf, -0).  nvcc compiles it as host code.
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
  std::vector<uint8_t> valid;
  bool has_nulls = false;

  const void* data() const {
    switch (type) {
      case HS_TYPE_INT32: return i32.data();
      case HS_TYPE_INT64: return i64.data();
      case HS_TYPE_FLOAT: return f32.data();
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
      default: f64.push_back(null ? 0.0 : strtod(v.c_str(), nullptr)); break;
    }
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
std::vector<hs_expr_node> read_side(Input& in, const char* end, std::deque<std::string>* names) {
  std::vector<hs_expr_node> out;
  std::string t;
  while (in.in >> t && t != end) {
    hs_expr_node x{};
    if (t == "+" || t == "-" || t == "*" || t == "/" || t == "%" || t == "neg") {
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
      const ExprProgram pg = resolve_expr(e, pcs);
      if (what == "resolve") {
        printf("ok %d", pg.domain);
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
      for (long long k = 0; k < rows; k++) printf(" %d", expr_holds(d, pg.insts.data(), ecols.data(), k) ? 1 : 0);
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
    } else if (what == "sides") {
      hs_expr_node nodes[2][4];
      hs_expr_compare ec[2];
      hs_predicate p[2];
      Filter f[2];
      for (int s = 0; s < 2; s++) {
        const bool pred_ok = in.i() != 0;
        const int op = (int)in.i();
        nodes[s][0] = hs_expr_node{HS_EXPR_COLUMN, "a", 0, 0, 0, 0.0};
        nodes[s][1] = hs_expr_node{HS_EXPR_LITERAL, nullptr, HS_TYPE_INT32, 0, 1, 0.0};
        nodes[s][2] = hs_expr_node{HS_EXPR_ADD, nullptr, 0, 0, 0, 0.0};
        nodes[s][3] = hs_expr_node{HS_EXPR_COLUMN, "b", 0, 0, 0, 0.0};
        ec[s] = hs_expr_compare{nodes[s], 3, nodes[s] + 3, 1, op, 0};
        p[s] = hs_predicate{};
        p[s].column = pred_ok ? "a" : nullptr, p[s].has_lo = 1, p[s].literal_type = HS_TYPE_INT64;
        f[s].preds = &p[s], f[s].n_preds = 1, f[s].exprs = &ec[s], f[s].n_exprs = 1;
      }
      char err[256] = "";
      const int rc = check_filters(f, 2, false, nullptr, err, sizeof err);
      if (rc == HS_OK) printf("ok\n");
      else printf("refused %d %s\n", rc, err);
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
    fprintf(stderr, "usage: filter_expr < cases\n");
    return 2;
  }
  std::string line;
  while (std::getline(std::cin, line))
    if (!line.empty()) run(line);
  return 0;
}
