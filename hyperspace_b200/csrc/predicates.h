// predicates.h -- filter predicates resolved on the host, with Spark 3.1's binary-comparison coercion: every predicate
// (hs_predicate) and disjunction term (hs_predicate_any) on a column becomes ranges of the column's values (SetRange),
// which api.cu uploads as the kernels' PredRanges.  Host code only: no CUDA call; tests/native/predicates.cu runs it.
//
// Numeric columns get inclusive ranges of sort_encode values, found by binary search over the encoded domain with the
// comparison Spark would evaluate -- in the wider of the column's and the literal's types (int < long < float < double),
// with SQLOrderingUtil's order (NaN == NaN, NaN above +inf, -0.0 == 0.0).  Every cast on the way (int/long -> double,
// float -> double, long -> float) is monotone, so the rows satisfying a bound are one end of the encoded order, and
// rounding casts (long -> double beyond 2^53) are followed exactly.  String columns keep the bounds' bytes and strictness.
// A term's flags (HS_TERM_*) add NOT -- the complement of the set over the column's domain --, a null outcome, and string
// patterns: a prefix is one range; other patterns are compiled for the matcher of string_match.h, their literal prefix
// bounding the values they can match.  A comparison between two columns (hs_column_compare) resolves to the one domain both
// sides are compared in (resolve_compare); column_compare.h evaluates it.  An expression comparison (hs_expr_compare)
// resolves to a typed postfix program with every implicit cast explicit (resolve_expr); column_expr.h evaluates it.
#pragma once
#include <algorithm>
#include <cstdarg>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <initializer_list>
#include <string>
#include <vector>

#include "device_utils.cuh"
#include "column_compare.h"
#include "column_expr.h"
#include "spark_types.h"
#include "string_match.h"

namespace hs {

// A column as the predicates see it: HS storage type, the leaf the index file declares (decimal scale, timestamp), name.
struct PredColumn {
  int type;
  const pq::SchemaColumn& schema;
  const std::string& name;
};

template <typename F>
inline int spark_compare(F a, F b) {  // SQLOrderingUtil.compareDoubles / compareFloats
  const bool na = a != a, nb = b != b;
  if (na || nb) return na == nb ? 0 : (na ? 1 : -1);
  return a < b ? -1 : (a > b ? 1 : 0);
}

// the column value whose sort_encode is e, compared with the literal (lit_i when lit_type is HS_TYPE_INT64 or
// HS_TYPE_DECIMAL, else lit_f).  Integer columns and integer / decimal literals compare as decimals of their scales
// (col_scale: the column's, 0 unless it is a decimal; lit_scale: the literal's, 0 for HS_TYPE_INT64).
inline int compare_encoded(int col_type, uint64_t e, int lit_type, int64_t lit_i, double lit_f, int col_scale, int lit_scale) {
  const bool lit_long = lit_type == HS_TYPE_INT64 || lit_type == HS_TYPE_DECIMAL;
  switch (col_type) {
    case HS_TYPE_INT32:
    case HS_TYPE_INT64: {
      const int64_t v = col_type == HS_TYPE_INT32 ? (int64_t)(int32_t)((uint32_t)e ^ 0x80000000u) : (int64_t)(e ^ 0x8000000000000000ull);
      if (lit_long) return compare_scaled(v, col_scale, lit_i, lit_scale);
      return spark_compare((double)v, lit_f);
    }
    case HS_TYPE_FLOAT: {
      const uint32_t u = (uint32_t)e, bits = (u & 0x80000000u) ? (u & 0x7fffffffu) : ~u;
      float f;
      memcpy(&f, &bits, 4);
      return lit_long ? spark_compare(f, (float)lit_i) : spark_compare((double)f, lit_f);
    }
    default: {
      const uint64_t bits = (e & 0x8000000000000000ull) ? (e & 0x7fffffffffffffffull) : ~e;
      double d;
      memcpy(&d, &bits, 8);
      return spark_compare(d, lit_long ? (double)lit_i : lit_f);
    }
  }
}

// encoded values of a column type, lowest to highest (floating point: -inf .. the NaNs above +inf)
inline void encoded_domain(int col_type, uint64_t* lo, uint64_t* hi) {
  switch (col_type) {
    case HS_TYPE_INT32: *lo = 0, *hi = 0xffffffffull; return;
    case HS_TYPE_INT64: *lo = 0, *hi = ~0ull; return;
    case HS_TYPE_FLOAT: *lo = 0x007fffffull, *hi = 0xffffffffull; return;   // ~bits(-inf)
    default: *lo = 0x000fffffffffffffull, *hi = ~0ull; return;             // ~bits(-inf)
  }
}

// One range of a column's values.  Numeric: inclusive sort_encode bounds (the strictness is resolved into them; lo > hi
// is empty); strings: the bounds' bytes with their strictness.  A missing bound is open.
struct SetRange {
  bool has_lo = false, has_hi = false, lo_strict = false, hi_strict = false;
  uint64_t lo = 0, hi = 0;
  std::string lo_b, hi_b;
};
// a term's ranges; normalised (normalise_set): sorted, disjoint, none empty
using RangeSet = std::vector<SetRange>;

// One predicate on column c as one range, possibly empty (numeric: lo = 1, hi = 0).  p.literal_type < 0 (hs_filter_scan):
// the literal type follows the column -- int64 bounds on an integer column, bytes on a string column.
inline SetRange resolve_range(const hs_predicate& p, const PredColumn& c) {
  const bool str_col = c.type == HS_TYPE_STRING;
  int lit = p.literal_type;
  if (lit < 0) {
    if (!str_col && c.type != HS_TYPE_INT32 && c.type != HS_TYPE_INT64) fail(HS_EUNSUPPORTED, "filter scan: key column must be int32 / int64 / string");
    lit = str_col ? HS_TYPE_STRING : HS_TYPE_INT64;
  }
  if (c.type == HS_TYPE_BOOL) fail(HS_EUNSUPPORTED, "filter scan: predicates on the boolean column '%s' are not handled", c.name.c_str());
  if (c.type < HS_TYPE_INT32 || c.type > HS_TYPE_STRING) fail(HS_EUNSUPPORTED, "filter scan: column '%s' has an unhandled type", c.name.c_str());
  if (str_col != (lit == HS_TYPE_STRING))
    fail(HS_EUNSUPPORTED, "filter scan: a %s literal cannot be compared with the %s column '%s'", lit == HS_TYPE_STRING ? "string" : "numeric",
         str_col ? "string" : "numeric", c.name.c_str());
  // Spark compares these in double: the caller keeps the conjunct in a Filter of its own
  const bool dec_col = is_decimal(c.schema), ts_col = is_timestamp(c.schema);
  if (lit == HS_TYPE_DOUBLE && (dec_col || ts_col))
    fail(HS_EUNSUPPORTED, "filter scan: a double literal cannot be compared with the %s column '%s'", dec_col ? "decimal" : "timestamp",
         c.name.c_str());
  if (lit == HS_TYPE_DECIMAL && (ts_col || (c.type != HS_TYPE_INT32 && c.type != HS_TYPE_INT64)))
    fail(HS_EUNSUPPORTED, "filter scan: a decimal literal cannot be compared with the %s column '%s'",
         ts_col ? "timestamp" : (c.type == HS_TYPE_STRING ? "string" : "floating-point"), c.name.c_str());
  if (lit == HS_TYPE_DECIMAL && (p.scale < 0 || p.scale > 38))
    fail(HS_EINVAL, "filter scan: decimal literal on '%s' has scale %d", c.name.c_str(), p.scale);
  const int col_scale = dec_col ? c.schema.scale : 0, lit_scale = lit == HS_TYPE_DECIMAL ? p.scale : 0;
  SetRange r;
  r.has_lo = p.has_lo != 0;
  r.has_hi = p.has_hi != 0;
  if (str_col) {
    if ((p.has_lo && p.lo_len && !p.lo_bytes) || (p.has_hi && p.hi_len && !p.hi_bytes))
      fail(HS_EINVAL, "filter scan: string column '%s' needs lo_bytes / hi_bytes", c.name.c_str());
    if (p.lo_len > kMaxStringLen || p.hi_len > kMaxStringLen) fail(HS_EUNSUPPORTED, "string bound longer than 65535 bytes");
    if (r.has_lo && p.lo_len) r.lo_b.assign((const char*)p.lo_bytes, p.lo_len);
    if (r.has_hi && p.hi_len) r.hi_b.assign((const char*)p.hi_bytes, p.hi_len);
    r.lo_strict = r.has_lo && p.lo_strict;
    r.hi_strict = r.has_hi && p.hi_strict;
    return r;
  }
  uint64_t emin, emax;
  encoded_domain(c.type, &emin, &emax);
  auto cmp = [&](uint64_t e, bool hi_side) {
    return compare_encoded(c.type, e, lit, hi_side ? p.hi_i : p.lo_i, hi_side ? p.hi_f : p.lo_f, col_scale, lit_scale);
  };
  bool empty = false;
  if (r.has_lo) {  // smallest e with value >= lo (> lo when strict)
    const int t = p.lo_strict ? 1 : 0;
    if (cmp(emax, false) < t) {
      empty = true;
    } else {
      uint64_t a = emin, b = emax;
      while (a < b) {
        const uint64_t mid = a + ((b - a) >> 1);
        if (cmp(mid, false) >= t) b = mid;
        else a = mid + 1;
      }
      r.lo = a;
    }
  }
  if (r.has_hi) {  // largest e with value <= hi (< hi when strict)
    const int t = p.hi_strict ? -1 : 0;
    if (cmp(emin, true) > t) {
      empty = true;
    } else {
      uint64_t a = emin, b = emax;
      while (a < b) {
        const uint64_t mid = b - ((b - a) >> 1);
        if (cmp(mid, true) <= t) a = mid;
        else b = mid - 1;
      }
      r.hi = a;
    }
  }
  if (empty) r.has_lo = r.has_hi = true, r.lo = 1, r.hi = 0;
  return r;
}

inline int host_string_compare(const uint8_t* a, uint32_t la, const uint8_t* b, uint32_t lb) {
  const int c = memcmp(a, b, std::min(la, lb));
  if (c) return c < 0 ? -1 : 1;
  return la == lb ? 0 : (la < lb ? -1 : 1);
}
inline int set_bound_cmp(bool str, uint64_t a, const std::string& as, uint64_t b, const std::string& bs) {
  if (str) return host_string_compare((const uint8_t*)as.data(), (uint32_t)as.size(), (const uint8_t*)bs.data(), (uint32_t)bs.size());
  return a < b ? -1 : (a > b ? 1 : 0);
}
inline bool set_range_empty(bool str, const SetRange& r) {
  if (!r.has_lo || !r.has_hi) return false;
  const int c = set_bound_cmp(str, r.lo, r.lo_b, r.hi, r.hi_b);
  return c > 0 || (c == 0 && (r.lo_strict || r.hi_strict));
}
inline bool lo_before(bool str, const SetRange& a, const SetRange& b) {  // a starts below b
  if (!a.has_lo || !b.has_lo) return !a.has_lo && b.has_lo;
  const int c = set_bound_cmp(str, a.lo, a.lo_b, b.lo, b.lo_b);
  return c < 0 || (c == 0 && !a.lo_strict && b.lo_strict);
}
inline bool hi_before(bool str, const SetRange& a, const SetRange& b) {  // a ends below b
  if (!a.has_hi || !b.has_hi) return a.has_hi && !b.has_hi;
  const int c = set_bound_cmp(str, a.hi, a.hi_b, b.hi, b.hi_b);
  return c < 0 || (c == 0 && a.hi_strict && !b.hi_strict);
}

// the values in both a and b: the later lower bound and the earlier upper bound; the result may be empty
inline SetRange intersect_range(bool str, const SetRange& a, const SetRange& b) {
  const SetRange& lo = lo_before(str, a, b) ? b : a;
  const SetRange& hi = hi_before(str, a, b) ? a : b;
  SetRange r;
  r.has_lo = lo.has_lo, r.lo = lo.lo, r.lo_b = lo.lo_b, r.lo_strict = lo.lo_strict;
  r.has_hi = hi.has_hi, r.hi = hi.hi, r.hi_b = hi.hi_b, r.hi_strict = hi.hi_strict;
  return r;
}

// sorts, drops empty ranges and merges overlapping and adjacent ones
inline void normalise_set(bool str, RangeSet* rs) {
  rs->erase(std::remove_if(rs->begin(), rs->end(), [&](const SetRange& r) { return set_range_empty(str, r); }), rs->end());
  std::sort(rs->begin(), rs->end(), [&](const SetRange& a, const SetRange& b) { return lo_before(str, a, b); });
  RangeSet out;
  for (SetRange& r : *rs) {
    bool joins = false;
    if (!out.empty()) {
      const SetRange& cur = out.back();
      if (!cur.has_hi || !r.has_lo) joins = true;
      else if (!str) joins = r.lo <= cur.hi || r.lo - 1 == cur.hi;  // r.lo > cur.hi >= 0 in the second test
      else {
        const int c = set_bound_cmp(true, r.lo, r.lo_b, cur.hi, cur.hi_b);
        joins = c < 0 || (c == 0 && !(r.lo_strict && cur.hi_strict));
      }
    }
    if (!joins) {
      out.push_back(std::move(r));
    } else if (hi_before(str, out.back(), r)) {
      SetRange& cur = out.back();
      cur.has_hi = r.has_hi, cur.hi = r.hi, cur.hi_b = std::move(r.hi_b), cur.hi_strict = r.hi_strict;
    }
  }
  *rs = std::move(out);
}

// the values in both normalised sets, normalised
inline RangeSet intersect_sets(bool str, const RangeSet& a, const RangeSet& b) {
  RangeSet out;
  size_t i = 0, j = 0;
  while (i < a.size() && j < b.size()) {
    SetRange r = intersect_range(str, a[i], b[j]);
    if (!set_range_empty(str, r)) out.push_back(std::move(r));
    if (hi_before(str, a[i], b[j])) i++;
    else j++;
  }
  return out;
}

// Every value and range of the term on column c, as one normalised set; values that match nothing (int_col IN (2.5))
// are dropped.  The refusals are resolve_range's, for the list's literal type and for every range.
inline RangeSet resolve_term(const hs_predicate_any& a, const PredColumn& c) {
  const bool str = c.type == HS_TYPE_STRING;
  RangeSet out;
  hs_predicate p;
  memset(&p, 0, sizeof p);
  p.column = a.column;
  p.literal_type = a.literal_type;
  p.scale = a.scale;
  p.has_lo = p.has_hi = 1;
  const bool lit_long = a.literal_type == HS_TYPE_INT64 || a.literal_type == HS_TYPE_DECIMAL;
  const int col_scale = is_decimal(c.schema) ? c.schema.scale : 0, lit_scale = a.literal_type == HS_TYPE_DECIMAL ? a.scale : 0;
  if (a.n_values > 0) resolve_range(p, c);  // the list's refusals, once
  out.reserve((size_t)a.n_values + a.n_ranges);
  for (int64_t k = 0; k < a.n_values; k++) {
    SetRange s;
    if (str) {
      const uint64_t b = a.values_offsets[k], e = a.values_offsets[k + 1];
      s.has_lo = s.has_hi = true;
      s.lo_b.assign((const char*)a.values_bytes + b, e - b);
      s.hi_b = s.lo_b;
      out.push_back(std::move(s));
      continue;
    }
    // an integer column against an integer literal at its own scale equals at most one value: the literal's own encoding,
    // confirmed by the comparison; everything else goes through the binary searches of resolve_range
    if (lit_long && col_scale == lit_scale && (c.type == HS_TYPE_INT64 || (c.type == HS_TYPE_INT32 && a.values_i[k] == (int32_t)a.values_i[k]))) {
      const uint64_t e = c.type == HS_TYPE_INT32 ? (uint64_t)((uint32_t)(int32_t)a.values_i[k] ^ 0x80000000u)
                                                 : (uint64_t)a.values_i[k] ^ 0x8000000000000000ull;
      if (compare_encoded(c.type, e, a.literal_type, a.values_i[k], 0.0, col_scale, lit_scale) == 0) {
        s.has_lo = s.has_hi = true;
        s.lo = s.hi = e;
        out.push_back(std::move(s));
        continue;
      }
    }
    if (lit_long) p.lo_i = p.hi_i = a.values_i[k];
    else p.lo_f = p.hi_f = a.values_f[k];
    out.push_back(resolve_range(p, c));
  }
  for (int32_t r = 0; r < a.n_ranges; r++) {
    hs_predicate q = a.ranges[r];
    q.column = a.column;
    out.push_back(resolve_range(q, c));
  }
  normalise_set(str, &out);
  return out;
}

inline bool set_is_points(bool str, const RangeSet& s) {
  for (const SetRange& r : s) {
    if (!r.has_lo || !r.has_hi) return false;
    if (str ? (r.lo_b != r.hi_b || r.lo_strict || r.hi_strict) : r.lo != r.hi) return false;
  }
  return true;
}

// ---- NOT, null tests and string patterns (hs_predicate_any.flags) -------------------------------------------------------

constexpr int kTermPatterns = HS_TERM_STARTS_WITH | HS_TERM_ENDS_WITH | HS_TERM_CONTAINS | HS_TERM_LIKE;
constexpr int kTermFlags = HS_TERM_NOT | HS_TERM_NULL_TRUE | HS_TERM_NULL_FALSE | kTermPatterns;
constexpr uint16_t kAnyRun = 257;  // LIKE's `%` in a parsed pattern (string_match.h: kAnyChar is `_`)

// Whether a null row qualifies under the term: only when the term is true there -- NULL_TRUE, or NULL_FALSE under NOT
// (NOT keeps unknown unknown).
inline bool term_null_selects(int flags) {
  return (flags & HS_TERM_NOT) ? (flags & HS_TERM_NULL_FALSE) != 0 : (flags & HS_TERM_NULL_TRUE) != 0;
}

// The values of a column of type col_type outside the normalised set s, normalised.  Numeric: the gaps of the encoded
// domain (encoded_domain); strings: the gaps between the bounds, each bound's strictness flipped, from "" up.
inline RangeSet complement_set(int col_type, const RangeSet& s) {
  RangeSet out;
  if (col_type == HS_TYPE_STRING) {
    SetRange gap;
    gap.has_lo = true;  // from "" inclusive: every value
    for (const SetRange& r : s) {
      if (r.has_lo) {
        SetRange g = gap;
        g.has_hi = true, g.hi_b = r.lo_b, g.hi_strict = !r.lo_strict;
        if (!set_range_empty(true, g)) out.push_back(std::move(g));
      }
      if (!r.has_hi) return out;
      gap = SetRange{};
      gap.has_lo = true, gap.lo_b = r.hi_b, gap.lo_strict = !r.hi_strict;
    }
    out.push_back(std::move(gap));
    return out;
  }
  uint64_t emin, emax;
  encoded_domain(col_type, &emin, &emax);
  auto push = [&](uint64_t lo, uint64_t hi) {
    SetRange g;
    g.has_lo = g.has_hi = true, g.lo = lo, g.hi = hi;
    out.push_back(g);
  };
  uint64_t next = emin;  // the lowest value not yet covered by s or a gap
  for (const SetRange& r : s) {
    const uint64_t lo = r.has_lo ? r.lo : emin, hi = r.has_hi ? r.hi : emax;
    if (lo > next) push(next, lo - 1);
    if (hi >= emax) return out;
    next = std::max(next, hi + 1);
  }
  push(next, emax);
  return out;
}

// The strings that start with p: [p, succ(p)), succ(p) being p without its trailing 0xff bytes and the last byte left
// incremented; open above when nothing is left (p empty or all 0xff).
inline SetRange prefix_range(const std::string& p) {
  SetRange r;
  r.has_lo = true, r.lo_b = p;
  std::string hi = p;
  while (!hi.empty() && (uint8_t)hi.back() == 0xff) hi.pop_back();
  if (!hi.empty()) {
    hi.back() = (char)((uint8_t)hi.back() + 1);
    r.has_hi = r.hi_strict = true, r.hi_b = std::move(hi);
  }
  return r;
}

// A LIKE pattern with the escape character '\' as items: literal bytes, kAnyChar (`_`) and kAnyRun (`%`).  Spark's
// refusals (StringUtils.escapeLikeRegex): HS_EINVAL.
inline std::vector<uint16_t> parse_like(const std::string& pat) {
  std::vector<uint16_t> out;
  out.reserve(pat.size());
  for (size_t i = 0; i < pat.size(); i++) {
    const uint8_t ch = (uint8_t)pat[i];
    if (ch == '\\') {
      if (i + 1 == pat.size()) fail(HS_EINVAL, "the pattern '%s' is invalid, it is not allowed to end with the escape character", pat.c_str());
      const uint8_t nx = (uint8_t)pat[++i];
      if (nx != '_' && nx != '%' && nx != '\\') {
        const std::string c = pat.substr(i, utf8_char_len(nx));
        fail(HS_EINVAL, "the pattern '%s' is invalid, the escape character is not allowed to precede '%s'", pat.c_str(), c.c_str());
      }
      out.push_back(nx);
    } else {
      out.push_back(ch == '_' ? kAnyChar : (ch == '%' ? kAnyRun : ch));
    }
  }
  return out;
}

// A pattern term compiled for pattern_matches (string_match.h), and what the host can say of it without a matcher.
struct CompiledPattern {
  std::vector<uint16_t> items;  // literal bytes and kAnyChar
  std::vector<int32_t> fail;    // per item: the KMP failure function of its segment (string_match.h: find_literal)
  std::vector<PatSeg> segs;     // the runs between `%`s
  bool whole = false;           // no `%`: the one segment spans the value
  std::string prefix;           // the literal bytes before the first wildcard
  bool prefix_only = false;     // no wildcard but `%` after the prefix: the pattern is a prefix range, or an equality when whole
};

// kind: one of HS_TERM_STARTS_WITH / ENDS_WITH / CONTAINS / LIKE
inline CompiledPattern compile_pattern(int kind, const std::string& pat) {
  std::vector<uint16_t> seq;
  if (kind == HS_TERM_LIKE) {
    seq = parse_like(pat);
  } else {
    if (kind != HS_TERM_STARTS_WITH) seq.push_back(kAnyRun);
    for (unsigned char ch : pat) seq.push_back(ch);
    if (kind != HS_TERM_ENDS_WITH) seq.push_back(kAnyRun);
  }
  CompiledPattern cp;
  size_t k = 0;
  while (k < seq.size() && seq[k] < kAnyChar) cp.prefix.push_back((char)seq[k++]);
  cp.prefix_only = std::all_of(seq.begin() + k, seq.end(), [](uint16_t it) { return it == kAnyRun; });
  PatSeg cur{0, 0, 0};
  for (uint16_t it : seq) {
    if (it == kAnyRun) {
      cp.segs.push_back(cur);
      cur = PatSeg{(uint32_t)cp.items.size(), 0, 0};
      continue;
    }
    cp.items.push_back(it);
    cur.len++;
    cur.any_char |= it == kAnyChar;
  }
  cp.segs.push_back(cur);
  cp.whole = cp.segs.size() == 1;
  // fail[off + j]: the longest proper prefix of the segment's first j + 1 items that is also their suffix
  cp.fail.assign(cp.items.size(), 0);
  for (const PatSeg& g : cp.segs) {
    const uint16_t* it = cp.items.data() + g.off;
    int32_t* f = cp.fail.data() + g.off;
    for (uint32_t j = 1, k = 0; j < g.len; j++) {
      while (k > 0 && it[j] != it[k]) k = f[k - 1];
      if (it[j] == it[k]) k++;
      f[j] = (int32_t)k;
    }
  }
  return cp;
}

// the pattern of a pattern term (check_anys has checked its shape)
inline std::string term_pattern(const hs_predicate_any& a) {
  const uint64_t b = a.values_offsets[0], e = a.values_offsets[1];
  return e > b ? std::string((const char*)a.values_bytes + b, e - b) : std::string();
}

// A term resolved once for both uses: the key's windows and the residual.
struct ResolvedTerm {
  // the values of non-null rows for which the term is true, normalised: resolve_term's set, a pattern's prefix range (an
  // equality for a LIKE without wildcards), complemented under NOT
  RangeSet set;
  // false for a pattern that is not a prefix: `set` then only bounds the values it can match (its literal prefix; every
  // value under NOT), and `pattern` is what the matcher runs
  bool exact = true;
  CompiledPattern pattern;
};

// Patterns on other than string columns, and any flag on a boolean column: HS_EUNSUPPORTED.
inline ResolvedTerm resolve_any(const hs_predicate_any& a, const PredColumn& c) {
  ResolvedTerm rt;
  if (const int kind = a.flags & kTermPatterns) {
    if (c.type != HS_TYPE_STRING)
      fail(HS_EUNSUPPORTED, "filter scan: a string pattern cannot be applied to the %s column '%s'", c.type == HS_TYPE_BOOL ? "boolean" : "numeric",
           c.name.c_str());
    rt.pattern = compile_pattern(kind, term_pattern(a));
    const CompiledPattern& cp = rt.pattern;
    if (cp.prefix_only && cp.whole) {
      SetRange r;
      r.has_lo = r.has_hi = true, r.lo_b = r.hi_b = cp.prefix;
      rt.set.push_back(std::move(r));
    } else {
      rt.set.push_back(prefix_range(cp.prefix));
    }
    rt.exact = cp.prefix_only;
  } else {
    if (a.flags && c.type == HS_TYPE_BOOL) fail(HS_EUNSUPPORTED, "filter scan: predicates on the boolean column '%s' are not handled", c.name.c_str());
    rt.set = resolve_term(a, c);
  }
  if (a.flags & HS_TERM_NOT) rt.set = rt.exact ? complement_set(c.type, rt.set) : RangeSet{SetRange{}};
  return rt;
}

// A call refused before it runs: stats zeroed, the message in err.  Returns code.
__attribute__((format(printf, 5, 6))) inline int refuse(int code, hs_stats* stats, char* err, size_t errlen, const char* fmt, ...) {
  if (stats) memset(stats, 0, sizeof *stats);
  if (err && errlen) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(err, errlen, fmt, ap);
    va_end(ap);
  }
  return code;
}

// The refusals of a predicate list that need no data: HS_OK or the code, with stats zeroed and the message in err.
// bounds_in_spec: hs_filter_scan_where was also given the bounds of hs_filter_scan.
inline int check_predicates(const hs_predicate* preds, int n_preds, bool bounds_in_spec, hs_stats* stats, char* err, size_t errlen) {
  if (n_preds > kMaxPredicates) return refuse(HS_EUNSUPPORTED, stats, err, errlen, "filter scan: more than 16 predicates");
  if (bounds_in_spec) return refuse(HS_EINVAL, stats, err, errlen, "filter scan: the bounds go in the predicates");
  for (int i = 0; i < n_preds; i++) {
    const hs_predicate& p = preds[i];
    if (!p.column) return refuse(HS_EINVAL, stats, err, errlen, "filter scan: predicate without a column");
    if (!p.has_lo && !p.has_hi) return refuse(HS_EINVAL, stats, err, errlen, "filter scan: predicate on '%s' has no bound", p.column);
    if (p.literal_type != HS_TYPE_INT64 && p.literal_type != HS_TYPE_DOUBLE && p.literal_type != HS_TYPE_STRING &&
        p.literal_type != HS_TYPE_DECIMAL)
      return refuse(HS_EINVAL, stats, err, errlen, "filter scan: predicate on '%s' has an unknown literal type", p.column);
  }
  return HS_OK;
}

// The same for the disjunction terms beside n_preds predicates: their counts, arrays, offsets and string lengths.
inline int check_anys(const hs_predicate_any* anys, int n_anys, int n_preds, hs_stats* stats, char* err, size_t errlen) {
  if (n_anys < 0 || (n_anys > 0 && !anys)) return refuse(HS_EINVAL, stats, err, errlen, "filter scan: bad term array");
  if (n_preds + n_anys > kMaxPredicates)
    return refuse(HS_EUNSUPPORTED, stats, err, errlen, "filter scan: more than 16 predicates and terms");
  for (int i = 0; i < n_anys; i++) {
    const hs_predicate_any& a = anys[i];
    if (!a.column) return refuse(HS_EINVAL, stats, err, errlen, "filter scan: term without a column");
    const char* c = a.column;
    if (a.n_values < 0 || a.n_ranges < 0 || (a.n_ranges > 0 && !a.ranges))
      return refuse(HS_EINVAL, stats, err, errlen, "filter scan: term on '%s' has a bad value or range array", c);
    if (a.n_values + a.n_ranges > (1ll << 24))
      return refuse(HS_EUNSUPPORTED, stats, err, errlen, "filter scan: term on '%s' has more than 2^24 values and ranges", c);
    if (a.literal_type != HS_TYPE_INT64 && a.literal_type != HS_TYPE_DOUBLE && a.literal_type != HS_TYPE_STRING &&
        a.literal_type != HS_TYPE_DECIMAL)
      return refuse(HS_EINVAL, stats, err, errlen, "filter scan: term on '%s' has an unknown literal type", c);
    const int kind = a.flags & kTermPatterns;
    if (a.flags & ~kTermFlags) return refuse(HS_EINVAL, stats, err, errlen, "filter scan: term on '%s' has unknown flags 0x%x", c, a.flags);
    if ((a.flags & HS_TERM_NULL_TRUE) && (a.flags & HS_TERM_NULL_FALSE))
      return refuse(HS_EINVAL, stats, err, errlen, "filter scan: term on '%s' has two null outcomes", c);
    if (kind & (kind - 1)) return refuse(HS_EINVAL, stats, err, errlen, "filter scan: term on '%s' has more than one pattern kind", c);
    if (kind && (a.literal_type != HS_TYPE_STRING || a.n_values != 1 || a.n_ranges != 0))
      return refuse(HS_EINVAL, stats, err, errlen, "filter scan: the pattern term on '%s' needs one string value and no ranges", c);
    if (a.n_values > 0) {
      const bool missing = a.literal_type == HS_TYPE_STRING ? (!a.values_offsets || (!a.values_bytes && a.values_offsets[a.n_values] != a.values_offsets[0]))
                                                            : (a.literal_type == HS_TYPE_DOUBLE ? !a.values_f : !a.values_i);
      if (missing) return refuse(HS_EINVAL, stats, err, errlen, "filter scan: term on '%s' has no value array", c);
      if (a.literal_type == HS_TYPE_STRING)
        for (int64_t k = 0; k < a.n_values; k++) {
          if (a.values_offsets[k + 1] < a.values_offsets[k])
            return refuse(HS_EINVAL, stats, err, errlen, "filter scan: term on '%s' has descending value offsets", c);
          if (a.values_offsets[k + 1] - a.values_offsets[k] > kMaxStringLen)
            return refuse(HS_EUNSUPPORTED, stats, err, errlen, "filter scan: a value of the term on '%s' is longer than 65535 bytes", c);
        }
    }
    if (kind == HS_TERM_LIKE) {
      try {
        parse_like(term_pattern(a));
      } catch (const Error& e) {
        return refuse(e.code, stats, err, errlen, "%s", e.what());
      }
    }
    for (int r = 0; r < a.n_ranges; r++) {
      if (a.ranges[r].column && strcmp(a.ranges[r].column, c) != 0)
        return refuse(HS_EINVAL, stats, err, errlen, "filter scan: a range of the term on '%s' names another column", c);
      hs_predicate q = a.ranges[r];
      q.column = c;
      const int rc = check_predicates(&q, 1, false, stats, err, errlen);
      if (rc != HS_OK) return rc;
    }
  }
  return HS_OK;
}


// ---- comparisons between two columns (hs_column_compare) ----------------------------------------------------------------

// A column's Spark type as the comparison coercion sees it
enum CompareKind { kKindInt, kKindLong, kKindFloat, kKindDouble, kKindDecimal, kKindString, kKindBinary, kKindDate, kKindTimestamp, kKindOther };

inline int compare_kind(const PredColumn& c) {
  if (is_decimal(c.schema)) return kKindDecimal;
  switch (c.type) {
    case HS_TYPE_INT32: return c.schema.converted_type == pq::CT_DATE ? kKindDate : kKindInt;  // byte and short count as int
    case HS_TYPE_INT64: return is_timestamp(c.schema) ? kKindTimestamp : kKindLong;
    case HS_TYPE_FLOAT: return kKindFloat;
    case HS_TYPE_DOUBLE: return kKindDouble;
    case HS_TYPE_STRING: return pq::spark_type_name(c.schema) == "binary" ? kKindBinary : kKindString;
    default: return kKindOther;  // boolean
  }
}

inline int64_t pow10_i64(int k) {
  int64_t p = 1;
  while (k-- > 0) p *= 10;
  return p;
}

// The comparison `l OP r` (check_compares has checked cc) in its domain, column pointers left for the caller.  Spark 3.1's
// coercion of BinaryComparison(attribute, attribute), as include/hs_gpu.h states it; other pairs are HS_EUNSUPPORTED.
inline CompareDesc resolve_compare(const hs_column_compare& cc, const PredColumn& l, const PredColumn& r) {
  CompareDesc d{};
  d.type[0] = l.type, d.type[1] = r.type;
  d.factor[0] = d.factor[1] = 1;
  d.op = cc.op;
  d.negate = (cc.flags & HS_TERM_NOT) != 0;
  const int k[2] = {compare_kind(l), compare_kind(r)};
  auto has = [&](int kind) { return k[0] == kind || k[1] == kind; };
  auto all_of_kinds = [&](std::initializer_list<int> kinds) {
    for (int s = 0; s < 2; s++)
      if (std::find(kinds.begin(), kinds.end(), k[s]) == kinds.end()) return false;
    return true;
  };
  const int scale[2] = {k[0] == kKindDecimal ? l.schema.scale : 0, k[1] == kKindDecimal ? r.schema.scale : 0};
  if (all_of_kinds({kKindInt, kKindLong})) {
    d.domain = kCmpInt;
  } else if ((k[0] == k[1] && (k[0] == kKindDate || k[0] == kKindTimestamp)) || all_of_kinds({kKindDate, kKindTimestamp})) {
    d.domain = kCmpInt;
    for (int s = 0; s < 2; s++)
      if (k[s] == kKindDate && k[s ^ 1] == kKindTimestamp) d.factor[s] = 86400000000ll;
  } else if (k[0] == k[1] && (k[0] == kKindString || k[0] == kKindBinary)) {
    d.domain = kCmpString;
  } else if (has(kKindDecimal) && all_of_kinds({kKindDecimal, kKindInt, kKindLong})) {
    d.domain = kCmpInt;  // exact: the side of the smaller scale is rescaled
    const int lo = scale[0] < scale[1] ? 0 : 1;
    d.factor[lo] = pow10_i64(scale[lo ^ 1] - scale[lo]);
  } else if (all_of_kinds({kKindInt, kKindLong, kKindFloat, kKindDouble, kKindDecimal})) {
    if (has(kKindDouble) || has(kKindDecimal)) {
      d.domain = kCmpDouble;
      for (int s = 0; s < 2; s++)
        if (k[s] == kKindDecimal) d.factor[s] = pow10_i64(scale[s]);
    } else {
      d.domain = kCmpFloat;
    }
  } else {
    fail(HS_EUNSUPPORTED, "filter scan: the columns '%s' (%s) and '%s' (%s) cannot be compared", l.name.c_str(),
         pq::spark_type_name(l.schema).c_str(), r.name.c_str(), pq::spark_type_name(r.schema).c_str());
  }
  return d;
}

// The refusals of a comparison list that need no data, beside n_others predicates and terms: as check_anys.
inline int check_compares(const hs_column_compare* cmps, int n_cmps, int n_others, hs_stats* stats, char* err, size_t errlen) {
  if (n_cmps < 0 || (n_cmps > 0 && !cmps)) return refuse(HS_EINVAL, stats, err, errlen, "filter scan: bad comparison array");
  if (n_others + n_cmps > kMaxPredicates)
    return refuse(HS_EUNSUPPORTED, stats, err, errlen, "filter scan: more than 16 predicates and terms");
  for (int i = 0; i < n_cmps; i++) {
    const hs_column_compare& c = cmps[i];
    if (!c.left || !c.right) return refuse(HS_EINVAL, stats, err, errlen, "filter scan: comparison without a column");
    if (c.op < HS_CMP_LT || c.op > HS_CMP_EQ_NULL_SAFE)
      return refuse(HS_EINVAL, stats, err, errlen, "filter scan: comparison of '%s' and '%s' has an unknown operator %d", c.left,
                    c.right, c.op);
    if (c.flags & ~HS_TERM_NOT)
      return refuse(HS_EINVAL, stats, err, errlen, "filter scan: comparison of '%s' and '%s' has unknown flags 0x%x", c.left,
                    c.right, c.flags);
  }
  return HS_OK;
}

// ---- arithmetic expressions compared (hs_expr_compare) ------------------------------------------------------------------

// The refusals of one side's postfix program that need no data: HS_OK or the code (message in err, stats zeroed)
inline int check_expr_side(const hs_expr_node* nodes, int n, int i, const char* side, hs_stats* stats, char* err, size_t errlen) {
  if (n < 1 || !nodes) return refuse(HS_EINVAL, stats, err, errlen, "filter scan: expression comparison %d has an empty %s side", i, side);
  if (n > kMaxExprNodes)
    return refuse(HS_EUNSUPPORTED, stats, err, errlen, "filter scan: the %s side of expression comparison %d has more than %d nodes", side,
                  i, kMaxExprNodes);
  int depth = 0;
  for (int k = 0; k < n; k++) {
    const hs_expr_node& x = nodes[k];
    switch (x.kind) {
      case HS_EXPR_COLUMN:
        if (!x.column) return refuse(HS_EINVAL, stats, err, errlen, "filter scan: expression comparison %d has a column node without a name", i);
        depth++;
        break;
      case HS_EXPR_LITERAL:
        if (x.literal_type != HS_TYPE_INT32 && x.literal_type != HS_TYPE_INT64 && x.literal_type != HS_TYPE_DOUBLE &&
            x.literal_type != HS_TYPE_DECIMAL && x.literal_type != HS_TYPE_STRING && x.literal_type != HS_TYPE_DATE &&
            x.literal_type != HS_TYPE_TIMESTAMP)
          return refuse(HS_EINVAL, stats, err, errlen, "filter scan: expression comparison %d has a literal of unknown type %d", i,
                        x.literal_type);
        if ((x.literal_type == HS_TYPE_INT32 || x.literal_type == HS_TYPE_DATE) && x.value_i != (int32_t)x.value_i)
          return refuse(HS_EINVAL, stats, err, errlen, "filter scan: expression comparison %d has %s literal outside int32", i,
                        x.literal_type == HS_TYPE_DATE ? "a date" : "an int");
        if (x.literal_type == HS_TYPE_DECIMAL && (x.scale < 0 || x.scale > 38))
          return refuse(HS_EINVAL, stats, err, errlen, "filter scan: expression comparison %d has a decimal literal of scale %d", i, x.scale);
        if (x.literal_type == HS_TYPE_STRING && (x.value_i < 0 || x.value_i > (int64_t)kMaxStringLen || (x.value_i > 0 && !x.column)))
          return refuse(HS_EINVAL, stats, err, errlen, "filter scan: expression comparison %d has a string literal of %lld bytes%s", i,
                        (long long)x.value_i, x.value_i < 0 || x.value_i > (int64_t)kMaxStringLen ? ", not 0..65535" : " and no bytes");
        depth++;
        break;
      case HS_EXPR_NEG:
      case HS_EXPR_YEAR:
      case HS_EXPR_QUARTER:
      case HS_EXPR_MONTH:
      case HS_EXPR_DAYOFMONTH:
      case HS_EXPR_DAYOFWEEK:
      case HS_EXPR_DAYOFYEAR:
      case HS_EXPR_WEEKOFYEAR:
      case HS_EXPR_HOUR:
      case HS_EXPR_MINUTE:
      case HS_EXPR_SECOND:
      case HS_EXPR_LENGTH:
      case HS_EXPR_ABS:
        if (depth < 1) return refuse(HS_EINVAL, stats, err, errlen, "filter scan: the %s side of expression comparison %d underflows its stack", side, i);
        break;
      case HS_EXPR_ADD:
      case HS_EXPR_SUB:
      case HS_EXPR_MUL:
      case HS_EXPR_DIV:
      case HS_EXPR_REM:
      case HS_EXPR_DATE_ADD:
      case HS_EXPR_DATE_SUB:
      case HS_EXPR_DATEDIFF:
        if (depth < 2) return refuse(HS_EINVAL, stats, err, errlen, "filter scan: the %s side of expression comparison %d underflows its stack", side, i);
        depth--;
        break;
      case HS_EXPR_SUBSTRING: {
        auto int_literal = [&](int at) { return at >= 0 && nodes[at].kind == HS_EXPR_LITERAL && nodes[at].literal_type == HS_TYPE_INT32; };
        if (depth < 3) return refuse(HS_EINVAL, stats, err, errlen, "filter scan: the %s side of expression comparison %d underflows its stack", side, i);
        if (!int_literal(k - 1) || !int_literal(k - 2))
          return refuse(HS_EINVAL, stats, err, errlen, "filter scan: expression comparison %d has a SUBSTRING whose pos and len are not int literals", i);
        depth -= 2;
        break;
      }
      case HS_EXPR_COALESCE:
        if (x.value_i < 2 || x.value_i > 8 || x.value_i > depth)
          return refuse(HS_EINVAL, stats, err, errlen, "filter scan: expression comparison %d has a COALESCE of %lld arguments over %d values", i,
                        (long long)x.value_i, depth);
        depth -= (int)x.value_i - 1;
        break;
      default: return refuse(HS_EINVAL, stats, err, errlen, "filter scan: expression comparison %d has a node of unknown kind %d", i, x.kind);
    }
    if (depth > kMaxExprDepth)
      return refuse(HS_EUNSUPPORTED, stats, err, errlen, "filter scan: the %s side of expression comparison %d is deeper than %d values", side,
                    i, kMaxExprDepth);
  }
  if (depth != 1)
    return refuse(HS_EINVAL, stats, err, errlen, "filter scan: the %s side of expression comparison %d leaves %d values", side, i, depth);
  return HS_OK;
}

// The refusals of an expression comparison list that need no data, beside n_others predicates, terms and comparisons: as
// check_compares, then each side's postfix shape, kinds, literals and names
inline int check_exprs(const hs_expr_compare* exprs, int n_exprs, int n_others, hs_stats* stats, char* err, size_t errlen) {
  if (n_exprs < 0 || (n_exprs > 0 && !exprs)) return refuse(HS_EINVAL, stats, err, errlen, "filter scan: bad expression array");
  if (n_others + n_exprs > kMaxPredicates)
    return refuse(HS_EUNSUPPORTED, stats, err, errlen, "filter scan: more than 16 predicates and terms");
  for (int i = 0; i < n_exprs; i++) {
    const hs_expr_compare& e = exprs[i];
    if (e.op < HS_CMP_LT || e.op > HS_CMP_EQ_NULL_SAFE)
      return refuse(HS_EINVAL, stats, err, errlen, "filter scan: expression comparison %d has an unknown operator %d", i, e.op);
    if (e.flags & ~HS_TERM_NOT)
      return refuse(HS_EINVAL, stats, err, errlen, "filter scan: expression comparison %d has unknown flags 0x%x", i, e.flags);
    int rc = check_expr_side(e.left, e.n_left, i, "left", stats, err, errlen);
    if (rc == HS_OK) rc = check_expr_side(e.right, e.n_right, i, "right", stats, err, errlen);
    if (rc != HS_OK) return rc;
  }
  return HS_OK;
}

// An operand's Spark type as the coercion sees it: kind (kKindInt / Long / Float / Double / Decimal, and for the
// functions kKindString / Binary / Date / Timestamp; kKindOther is a boolean), a decimal's precision and scale, and, for
// an integer literal, its digits (DecimalType.fromLiteral)
struct ExprType {
  int kind;
  int p = 0, s = 0;
  int lit_digits = 0;  // > 0: an integer literal
  bool narrow = false;  // a byte or short column: Spark's arithmetic between two of them wraps at their width
};

inline int decimal_digits(uint64_t v) {
  int d = 1;
  while (v >= 10) v /= 10, d++;
  return d;
}

inline __int128 pow10_i128(int k) {
  __int128 p = 1;
  while (k-- > 0) p *= 10;
  return p;
}

// the decimal type an integral or decimal operand takes beside a decimal: int column decimal(10,0), long column
// decimal(20,0), integer literal decimal(its digits, 0)
inline void as_decimal(const ExprType& t, int* p, int* s) {
  if (t.kind == kKindDecimal) *p = t.p, *s = t.s;
  else *p = t.lit_digits ? t.lit_digits : (t.kind == kKindInt ? 10 : 20), *s = 0;
}

inline bool numeric_kind(int k) { return k == kKindInt || k == kKindLong || k == kKindFloat || k == kKindDouble || k == kKindDecimal; }
inline bool datetime_kind(int k) { return k == kKindDate || k == kKindTimestamp; }

// Spark's simpleString of an operand's type, for messages
inline std::string expr_type_text(const ExprType& t) {
  switch (t.kind) {
    case kKindInt: return "int";
    case kKindLong: return "bigint";
    case kKindFloat: return "float";
    case kKindDouble: return "double";
    case kKindDecimal: return "decimal(" + std::to_string(t.p) + "," + std::to_string(t.s) + ")";
    case kKindString: return "string";
    case kKindBinary: return "binary";
    case kKindDate: return "date";
    case kKindTimestamp: return "timestamp";
    default: return "boolean";
  }
}

// Whether two operand kinds compare without arithmetic coercion: string with string, binary with binary, dates and
// timestamps with each other
inline bool comparable_kinds(int a, int b) {
  return (datetime_kind(a) && datetime_kind(b)) || (a == b && (a == kKindString || a == kKindBinary));
}

// A resolved expression comparison: the program of column_expr.h (kXLoad's arg: the ordinal of the COLUMN node, left side
// first), the comparison's domain, op and NOT.  funcs: the program holds a function, or a string, binary, date or
// timestamp value, and runs in k_func_mask.  String literals are kXStringConst instructions into `pool`, which the caller
// places (relocate_strings) before the program runs.
struct ExprProgram {
  std::vector<ExprInst> insts;
  int32_t domain = kCmpInt, op = 0, negate = 0;
  bool funcs = false;
  std::string pool;
};

// kXStringConst instructions (arg: offset into the pool, v.i: length) to kXConst of a reference into the pool at base
inline void relocate_strings(std::vector<ExprInst>* insts, const uint8_t* base) {
  for (ExprInst& in : *insts)
    if (in.op == kXStringConst) {
      const uint32_t len = (uint32_t)in.v.i;
      in.v.i = (__int128)string_ref(base + in.arg, len);
      in.op = kXConst, in.arg = 0;
    }
}

// the node kinds that existed before the functions, and their literal types: a comparison of such sides is refused
// exactly as it was when a column of another type is used
inline bool arithmetic_only(const hs_expr_node* nodes, int n) {
  for (int k = 0; k < n; k++) {
    if (nodes[k].kind > HS_EXPR_NEG) return false;
    if (nodes[k].kind == HS_EXPR_LITERAL && nodes[k].literal_type > HS_TYPE_DOUBLE && nodes[k].literal_type != HS_TYPE_DECIMAL) return false;
  }
  return true;
}

// the values node x takes from the stack: its operator's or function's arguments, none for a column or a literal
inline int expr_arity(const hs_expr_node& x) {
  switch (x.kind) {
    case HS_EXPR_COLUMN:
    case HS_EXPR_LITERAL: return 0;
    case HS_EXPR_COALESCE: return (int)x.value_i;
    case HS_EXPR_SUBSTRING: return 3;
    case HS_EXPR_ADD:
    case HS_EXPR_SUB:
    case HS_EXPR_MUL:
    case HS_EXPR_DIV:
    case HS_EXPR_REM:
    case HS_EXPR_DATE_ADD:
    case HS_EXPR_DATE_SUB:
    case HS_EXPR_DATEDIFF: return 2;
    default: return 1;
  }
}

// whether the value node k of a checked side pushes is an argument of a function, rather than of arithmetic or the
// comparison
inline bool consumed_by_function(const hs_expr_node* nodes, int n, int k) {
  for (int above = 0, j = k + 1; j < n; j++) {  // above: the values pushed after node k's that are still on the stack
    const int pops = expr_arity(nodes[j]);
    if (pops > above) return nodes[j].kind > HS_EXPR_NEG;
    above += 1 - pops;
  }
  return false;
}

inline std::string date_text(int64_t days) {
  char buf[48];
  snprintf(buf, sizeof buf, "DATE '%04d-%02d-%02d'", date_part(days, kPartYear), date_part(days, kPartMonth), date_part(days, kPartDayOfMonth));
  return buf;
}

// The expression comparison e (check_exprs has checked it) typed and lowered to column_expr.h's instructions, every
// implicit cast explicit.  cols: one column per COLUMN node, the left side's first.  Spark 3.1's coercion, as
// include/hs_gpu.h states it; what it cannot evaluate exactly as Spark would is HS_EUNSUPPORTED.
inline ExprProgram resolve_expr(const hs_expr_compare& e, const std::vector<PredColumn>& cols) {
  ExprProgram pg;
  pg.op = e.op;
  pg.negate = (e.flags & HS_TERM_NOT) != 0;
  std::vector<ExprType> ts;    // the type stack
  std::vector<std::string> txt;  // the nodes' SQL text, for messages
  std::vector<int> bare;       // per stack value: the COLUMN node's ordinal when the value is a bare column, else -1
  auto emit = [&](int op, int arg, __int128 v = 0) {
    ExprInst in{};
    in.op = op, in.arg = arg, in.v.i = v;
    pg.insts.push_back(in);
  };
  auto column_refused = [&](int ord) {
    const PredColumn& c = cols[ord];
    fail(HS_EUNSUPPORTED, "filter scan: the column '%s' (%s) cannot be used in arithmetic", c.name.c_str(), pq::spark_type_name(c.schema).c_str());
  };
  // an arithmetic operand at stack index at: numeric, or refused -- a bare column with arithmetic's own message
  auto arith_operand = [&](size_t at) {
    if (numeric_kind(ts[at].kind)) return;
    if (bare[at] >= 0) column_refused(bare[at]);
    fail(HS_EUNSUPPORTED, "filter scan: %s (%s) cannot be used in arithmetic", txt[at].c_str(), expr_type_text(ts[at]).c_str());
  };
  auto to_double = [&](int at, ExprType& t, const std::string& what) {
    switch (t.kind) {
      case kKindInt:
      case kKindLong: emit(kXIntToDouble, at); break;
      case kKindFloat: emit(kXFloatToDouble, at); break;
      case kKindDecimal:
        if (t.p > 18) fail(HS_EUNSUPPORTED, "filter scan: %s turns a decimal of more than 18 digits into a double", what.c_str());
        emit(kXDecToDouble, at, pow10_i128(t.s));
        break;
      default: break;
    }
    t = ExprType{kKindDouble};
  };
  auto to_float = [&](int at, ExprType& t) {
    if (t.kind == kKindInt || t.kind == kKindLong) emit(kXIntToFloat, at);
    t = ExprType{kKindFloat};
  };
  // both operands (a at slot 1, b at slot 0) to one domain for `what`: kXInt / kXLong / kXDec / kXFloat / kXDouble.
  // Decimals: to the scale `scale_to` when >= 0 (rescaling the smaller), returned in *p / *s as each side's decimal type.
  auto is_dec = [](const ExprType& t) { return t.kind == kKindDecimal; };
  auto is_fp = [](const ExprType& t) { return t.kind == kKindFloat || t.kind == kKindDouble; };
  auto unify = [&](ExprType& a, ExprType& b, const std::string& what, bool rescale) {
    if ((is_dec(a) || is_dec(b)) && !is_fp(a) && !is_fp(b)) {
      int pa, sa, pb, sb;
      as_decimal(a, &pa, &sa);
      as_decimal(b, &pb, &sb);
      const int s = std::max(sa, sb), wider = std::max(pa - sa, pb - sb) + s;
      if (wider > 38) fail(HS_EUNSUPPORTED, "filter scan: %s needs a decimal of more than 38 digits", what.c_str());
      if (rescale) {
        if (sa < s) emit(kXRescale, 1, pow10_i128(s - sa));
        if (sb < s) emit(kXRescale, 0, pow10_i128(s - sb));
      }
      a = ExprType{kKindDecimal, pa, sa}, b = ExprType{kKindDecimal, pb, sb};
      return (int)kXDec;
    }
    if (a.kind == kKindDouble || b.kind == kKindDouble || is_dec(a) || is_dec(b)) {
      to_double(1, a, what), to_double(0, b, what);
      return (int)kXDouble;
    }
    if (a.kind == kKindFloat || b.kind == kKindFloat) {
      to_float(1, a), to_float(0, b);
      return (int)kXFloat;
    }
    return (a.kind == kKindLong || b.kind == kKindLong) ? (int)kXLong : (int)kXInt;
  };
  auto domain_of = [](const ExprType& t) {
    return t.kind == kKindInt ? kXInt : t.kind == kKindLong ? kXLong : t.kind == kKindDecimal ? kXDec : t.kind == kKindFloat ? kXFloat : kXDouble;
  };
  // COALESCE's findWiderCommonType over the n values at the top, each cast to it in its slot
  auto coalesce = [&](int n, const std::string& what) {
    const size_t base = ts.size() - n;
    ExprType w = ts[base];
    w.lit_digits = 0;
    for (int j = 0; j < n; j++) {
      ExprType t = ts[base + j];
      t.lit_digits = 0;
      t.narrow = false;
      const bool ok = j == 0 ? (numeric_kind(t.kind) || comparable_kinds(t.kind, t.kind))
                             : (numeric_kind(t.kind) && numeric_kind(w.kind)) || comparable_kinds(t.kind, w.kind);
      if (!ok) fail(HS_EUNSUPPORTED, "filter scan: %s mixes %s (%s) with %s", what.c_str(), txt[base + j].c_str(), expr_type_text(t).c_str(),
                    j ? expr_type_text(w).c_str() : "nothing it widens with");
      if (j == 0) { w = t; continue; }
      if (datetime_kind(w.kind)) {
        w.kind = w.kind == kKindTimestamp || t.kind == kKindTimestamp ? kKindTimestamp : kKindDate;
      } else if (numeric_kind(w.kind)) {
        if ((is_dec(w) || is_dec(t)) && !is_fp(w) && !is_fp(t)) {
          int pa, sa, pb, sb;
          as_decimal(w, &pa, &sa);
          as_decimal(t, &pb, &sb);
          const int s = std::max(sa, sb), p = std::max(pa - sa, pb - sb) + s;
          if (p > 38) fail(HS_EUNSUPPORTED, "filter scan: %s needs a decimal of more than 38 digits", what.c_str());
          w = ExprType{kKindDecimal, p, s};
        } else if (w.kind == kKindDouble || t.kind == kKindDouble || is_dec(w) || is_dec(t)) {
          w = ExprType{kKindDouble};
        } else if (w.kind == kKindFloat || t.kind == kKindFloat) {
          w = ExprType{kKindFloat};
        } else {
          w = ExprType{w.kind == kKindLong || t.kind == kKindLong ? kKindLong : kKindInt};
        }
      }
    }
    for (int j = 0; j < n; j++) {
      ExprType t = ts[base + j];
      const int slot = n - 1 - j;
      if (w.kind == kKindTimestamp && t.kind == kKindDate) emit(kXRescale, slot, (__int128)86400000000ll);
      else if (w.kind == kKindDouble && t.kind != kKindDouble) to_double(slot, t, what);
      else if (w.kind == kKindFloat && t.kind != kKindFloat) to_float(slot, t);
      else if (w.kind == kKindDecimal) {
        int p, s;
        as_decimal(ExprType{t.kind, t.p, t.s}, &p, &s);
        if (s < w.s) emit(kXRescale, slot, pow10_i128(w.s - s));
      }
    }
    emit(kXCoalesce, n);
    return w;
  };
  static const char* const kOpText[] = {"", "", "", "+", "-", "*", "/", "%"};
  static const char* const kFuncText[] = {"year", "quarter", "month", "dayofmonth", "dayofweek", "dayofyear", "weekofyear", "hour", "minute",
                                          "second", "date_add", "date_sub", "datediff", "length", "substring", "abs", "coalesce"};
  int col_ord = 0;
  auto side = [&](const hs_expr_node* nodes, int n, const hs_expr_node* other, int n_other, int other_bare_kind) {
    for (int k = 0; k < n; k++) {
      const hs_expr_node& x = nodes[k];
      if (x.kind == HS_EXPR_COLUMN) {
        const PredColumn& c = cols[col_ord];
        const int kind = compare_kind(c);
        if (!numeric_kind(kind)) {
          // A boolean never serves.  A column of another type serves as a function's argument, or as a bare side beside a
          // side it compares with -- decided after that side, unless the comparison is arithmetic only: then it is
          // refused here, as it always was, unless the other side is a bare column it compares with.
          const bool deferred = n == 1 && (!arithmetic_only(other, n_other) || comparable_kinds(kind, other_bare_kind));
          if (kind == kKindOther || (!deferred && !consumed_by_function(nodes, n, k))) column_refused(col_ord);
          pg.funcs = true;
        }
        ExprType t{kind};
        if (kind == kKindDecimal) t.p = c.schema.precision, t.s = c.schema.scale;
        t.narrow = c.schema.converted_type == 15 || c.schema.converted_type == 16;  // INT_8, INT_16
        bare.push_back(col_ord);
        emit(kXLoad, col_ord++);
        ts.push_back(t);
        txt.push_back(c.name);
      } else if (x.kind == HS_EXPR_LITERAL) {
        ExprType t{kKindInt};
        char buf[64];
        switch (x.literal_type) {
          case HS_TYPE_INT32:
          case HS_TYPE_INT64:
            t.kind = x.literal_type == HS_TYPE_INT32 ? kKindInt : kKindLong;
            t.lit_digits = decimal_digits(x.value_i < 0 ? 0ull - (uint64_t)x.value_i : (uint64_t)x.value_i);
            emit(kXConst, 0, x.value_i);
            snprintf(buf, sizeof buf, "%lld", (long long)x.value_i);
            break;
          case HS_TYPE_DOUBLE: {
            t.kind = kKindDouble;
            ExprInst in{};
            in.op = kXConst, in.v.d = x.value_f;
            pg.insts.push_back(in);
            snprintf(buf, sizeof buf, "%.17g", x.value_f);
            break;
          }
          case HS_TYPE_STRING:
            t.kind = kKindString;
            emit(kXStringConst, (int32_t)pg.pool.size(), x.value_i);
            pg.pool.append(x.value_i ? x.column : "", (size_t)x.value_i);
            snprintf(buf, sizeof buf, "%.*s", (int)std::min<int64_t>(x.value_i, 40), x.value_i ? x.column : "");
            pg.funcs = true;
            break;
          case HS_TYPE_DATE:
            t.kind = kKindDate;
            emit(kXConst, 0, x.value_i);
            snprintf(buf, sizeof buf, "%s", date_text(x.value_i).c_str());
            pg.funcs = true;
            break;
          case HS_TYPE_TIMESTAMP:
            t.kind = kKindTimestamp;
            emit(kXConst, 0, x.value_i);
            snprintf(buf, sizeof buf, "TIMESTAMP_MICROS(%lld)", (long long)x.value_i);
            pg.funcs = true;
            break;
          default: {  // HS_TYPE_DECIMAL: DecimalType(max(digits, scale), scale)
            t.kind = kKindDecimal, t.s = x.scale;
            t.p = std::max(decimal_digits(x.value_i < 0 ? 0ull - (uint64_t)x.value_i : (uint64_t)x.value_i), x.scale);
            emit(kXConst, 0, x.value_i);
            snprintf(buf, sizeof buf, "%lldE-%d", (long long)x.value_i, x.scale);
            break;
          }
        }
        ts.push_back(t);
        txt.push_back(buf);
        bare.push_back(-1);
      } else if (x.kind == HS_EXPR_NEG) {
        arith_operand(ts.size() - 1);
        const ExprType& t = ts.back();
        if (t.narrow) fail(HS_EUNSUPPORTED, "filter scan: (- %s) is byte or short arithmetic, which wraps at its width: not handled", txt.back().c_str());
        emit(domain_of(t) + kXNeg, 0);
        ts.back().lit_digits = 0;
        txt.back() = "(- " + txt.back() + ")";
        bare.back() = -1;
      } else if (x.kind <= HS_EXPR_REM) {
        arith_operand(ts.size() - 2);
        arith_operand(ts.size() - 1);
        ExprType b = ts.back();
        ts.pop_back();
        ExprType a = ts.back();
        ts.pop_back();
        const std::string what = "(" + txt[txt.size() - 2] + " " + kOpText[x.kind] + " " + txt.back() + ")";
        txt.pop_back();
        txt.back() = what;
        bare.pop_back();
        bare.back() = -1;
        if (a.narrow && b.narrow) fail(HS_EUNSUPPORTED, "filter scan: %s is byte or short arithmetic, which wraps at its width: not handled", what.c_str());
        ExprType r;
        int dom;
        if (x.kind == HS_EXPR_DIV) {  // TypeCoercion.Division: double, unless DecimalPrecision made it a decimal division
          if ((is_dec(a) || is_dec(b)) && !is_fp(a) && !is_fp(b))
            fail(HS_EUNSUPPORTED, "filter scan: decimal division is not handled: %s", what.c_str());
          to_double(1, a, what), to_double(0, b, what);
          dom = kXDouble, r = ExprType{kKindDouble};
        } else {
          dom = unify(a, b, what, x.kind != HS_EXPR_MUL);
          if (dom == kXDec) {  // DecimalPrecision's result types
            const int s = std::max(a.s, b.s), range = std::max(a.p - a.s, b.p - b.s);
            switch (x.kind) {
              case HS_EXPR_ADD:
              case HS_EXPR_SUB: r = ExprType{kKindDecimal, range + s + 1, s}; break;
              case HS_EXPR_MUL: r = ExprType{kKindDecimal, a.p + b.p + 1, a.s + b.s}; break;
              default: r = ExprType{kKindDecimal, std::min(a.p - a.s, b.p - b.s) + s, s}; break;  // HS_EXPR_REM
            }
            if (r.p > 38) fail(HS_EUNSUPPORTED, "filter scan: %s needs a decimal of more than 38 digits", what.c_str());
          } else {
            r = ExprType{dom == kXInt ? kKindInt : dom == kXLong ? kKindLong : dom == kXFloat ? kKindFloat : kKindDouble};
          }
        }
        emit(dom + (x.kind - HS_EXPR_ADD), 0);
        ts.push_back(r);
      } else {  // a function (check_exprs: HS_EXPR_YEAR .. HS_EXPR_COALESCE)
        pg.funcs = true;
        const int nargs = expr_arity(x);
        const size_t base = ts.size() - nargs;
        std::string what = std::string(kFuncText[x.kind - HS_EXPR_YEAR]) + "(";
        for (int j = 0; j < nargs; j++) what += (j ? ", " : "") + txt[base + j];
        what += ")";
        auto need = [&](int j, bool ok, const char* kinds) {
          if (!ok) fail(HS_EUNSUPPORTED, "filter scan: %s: %s (%s) is not %s", what.c_str(), txt[base + j].c_str(),
                        expr_type_text(ts[base + j]).c_str(), kinds);
        };
        ExprType r{kKindInt};
        switch (x.kind) {
          case HS_EXPR_HOUR:
          case HS_EXPR_MINUTE:
          case HS_EXPR_SECOND:
            need(0, ts[base].kind == kKindTimestamp, "a timestamp");
            emit(kXTimePart, kPartHour + (x.kind - HS_EXPR_HOUR));
            break;
          case HS_EXPR_DATE_ADD:
          case HS_EXPR_DATE_SUB:
          case HS_EXPR_DATEDIFF: {
            need(0, datetime_kind(ts[base].kind), "a date or timestamp");
            if (x.kind == HS_EXPR_DATEDIFF) need(1, datetime_kind(ts[base + 1].kind), "a date or timestamp");
            else need(1, ts[base + 1].kind == kKindInt, "an int, short or byte");  // days: Spark would cast anything else
            if (ts[base].kind == kKindTimestamp) emit(kXTsToDate, 1);
            if (ts[base + 1].kind == kKindTimestamp) emit(kXTsToDate, 0);
            emit(kXInt + (x.kind == HS_EXPR_DATE_ADD ? kXAdd : kXSub), 0);
            if (x.kind != HS_EXPR_DATEDIFF) r = ExprType{kKindDate};
            break;
          }
          case HS_EXPR_LENGTH:
            need(0, ts[base].kind == kKindString || ts[base].kind == kKindBinary, "a string or binary");
            emit(kXLength, ts[base].kind == kKindBinary);
            break;
          case HS_EXPR_SUBSTRING: {
            need(0, ts[base].kind == kKindString || ts[base].kind == kKindBinary, "a string or binary");
            pg.insts.pop_back(), pg.insts.pop_back();  // the pos and len literals' kXConst: check_exprs made them literals
            const uint64_t pos = (uint32_t)(int32_t)nodes[k - 2].value_i, len = (uint32_t)(int32_t)nodes[k - 1].value_i;
            emit(kXSubstr, ts[base].kind == kKindBinary, (__int128)(pos | len << 32));
            r = ExprType{ts[base].kind};
            break;
          }
          case HS_EXPR_ABS:
            need(0, numeric_kind(ts[base].kind), "a number");
            if (ts[base].narrow) fail(HS_EUNSUPPORTED, "filter scan: %s is byte or short arithmetic, which wraps at its width: not handled", what.c_str());
            emit(kXAbs, domain_of(ts[base]));
            r = ts[base];
            r.lit_digits = 0;
            break;
          case HS_EXPR_COALESCE: r = coalesce(nargs, what); break;
          default:  // HS_EXPR_YEAR .. HS_EXPR_WEEKOFYEAR
            need(0, datetime_kind(ts[base].kind), "a date or timestamp");
            if (ts[base].kind == kKindTimestamp) emit(kXTsToDate, 0);
            emit(kXDatePart, kPartYear + (x.kind - HS_EXPR_YEAR));
            break;
        }
        ts.resize(base), txt.resize(base), bare.resize(base);
        ts.push_back(r), txt.push_back(what), bare.push_back(-1);
      }
    }
  };
  // the kind of each side that is one COLUMN node (-1 otherwise); the right side's column follows the left side's columns
  int n_left_cols = 0;
  for (int k = 0; k < e.n_left; k++) n_left_cols += e.left[k].kind == HS_EXPR_COLUMN;
  const int left_bare = e.n_left == 1 && e.left[0].kind == HS_EXPR_COLUMN ? compare_kind(cols[0]) : -1;
  const int right_bare = e.n_right == 1 && e.right[0].kind == HS_EXPR_COLUMN ? compare_kind(cols[n_left_cols]) : -1;
  side(e.left, e.n_left, e.right, e.n_right, right_bare);
  side(e.right, e.n_right, e.left, e.n_left, left_bare);
  ExprType b = ts.back(), a = ts[0];
  static const char* const kCmpText[] = {"", "<", "<=", ">", ">=", "=", "<=>"};
  const std::string what = "(" + txt[0] + " " + kCmpText[e.op] + " " + txt[1] + ")";
  if (numeric_kind(a.kind) && numeric_kind(b.kind)) {
    const int dom = unify(a, b, what, true);  // resolve_compare's table, decimals widened to 38 digits
    pg.domain = dom == kXFloat ? kCmpFloat : (dom == kXDouble ? kCmpDouble : kCmpInt);
  } else if (comparable_kinds(a.kind, b.kind)) {
    pg.domain = datetime_kind(a.kind) ? kCmpInt : kCmpString;
    if (a.kind == kKindDate && b.kind == kKindTimestamp) emit(kXRescale, 1, (__int128)86400000000ll);
    if (b.kind == kKindDate && a.kind == kKindTimestamp) emit(kXRescale, 0, (__int128)86400000000ll);
  } else {
    for (int s = 0; s < 2; s++)
      if (bare[s] >= 0 && !numeric_kind((s ? b : a).kind)) column_refused(bare[s]);
    fail(HS_EUNSUPPORTED, "filter scan: %s (%s) and %s (%s) cannot be compared", txt[0].c_str(), expr_type_text(a).c_str(), txt[1].c_str(),
         expr_type_text(b).c_str());
  }
  return pg;
}

// The filter of a filter scan or of one join side, as its entry point was given it: predicates, disjunction terms,
// comparisons between two columns and expression comparisons, all AND-ed.
struct Filter {
  const hs_predicate* preds = nullptr;
  int n_preds = 0;
  const hs_predicate_any* anys = nullptr;
  int n_anys = 0;
  const hs_column_compare* cmps = nullptr;
  int n_cmps = 0;
  const hs_expr_compare* exprs = nullptr;
  int n_exprs = 0;
};

// The refusals of the filters of a call's n_sides sides that need no data, in one order whatever side a fault is on:
// every side's predicates, then every side's terms, then every side's comparisons, then every side's expression
// comparisons.  bounds_in_spec: as check_predicates.
inline int check_filters(const Filter* sides, int n_sides, bool bounds_in_spec, hs_stats* stats, char* err, size_t errlen) {
  int rc = HS_OK;
  for (int s = 0; s < n_sides && rc == HS_OK; s++)
    rc = check_predicates(sides[s].preds, sides[s].n_preds, bounds_in_spec, stats, err, errlen);
  for (int s = 0; s < n_sides && rc == HS_OK; s++)
    rc = check_anys(sides[s].anys, sides[s].n_anys, sides[s].n_preds, stats, err, errlen);
  for (int s = 0; s < n_sides && rc == HS_OK; s++)
    rc = check_compares(sides[s].cmps, sides[s].n_cmps, sides[s].n_preds + sides[s].n_anys, stats, err, errlen);
  for (int s = 0; s < n_sides && rc == HS_OK; s++)
    rc = check_exprs(sides[s].exprs, sides[s].n_exprs, sides[s].n_preds + sides[s].n_anys + sides[s].n_cmps, stats, err, errlen);
  return rc;
}

}  // namespace hs
