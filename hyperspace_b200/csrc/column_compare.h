// column_compare.h -- a comparison between two columns of the same row (`a < b`, `a = b`, `a <=> b`), evaluated in the
// one domain the host resolved for the pair (predicates.h: resolve_compare, with Spark 3.1's TypeCoercion and
// DecimalPrecision).  __host__ __device__ like string_match.h: k_compare_mask (read_side.cu) runs it one thread per row,
// and tests/native/filter_compare.cu runs the same code on the CPU against a Python restatement.
//
// Domains:
//   kCmpInt     both sides as signed integers (int32 sign-extended): integers, dates, timestamps, decimals of one scale.
//               A side with factor != 1 is multiplied by it in 128 bits first: 10^k rescales the decimal of the smaller
//               scale, 86 400 000 000 turns a date's days into a timestamp's micros.  The comparison is exact.
//   kCmpFloat   both sides as float: an integer rounds to nearest (__int2float_rn / __ll2float_rn).
//   kCmpDouble  both sides as double: an integer rounds to nearest, a float widens exactly, and a decimal (factor =
//               10^scale) is its unscaled value over 10^scale rounded to nearest, ties to even, as Decimal.toDouble.
//   kCmpString  UTF8String byte order over the string references.
// Floating point follows SQLOrderingUtil: NaN equals NaN and sorts above +inf, -0.0 equals 0.0.
#pragma once
#include <cstdint>
#include <cstring>

#include "device_utils.cuh"
#include "hs_common.h"

namespace hs {

enum CompareDomain : int32_t { kCmpInt = 0, kCmpFloat = 1, kCmpDouble = 2, kCmpString = 3 };

// One resolved comparison `side 0 OP side 1`.  op is HS_CMP_*; negate: NOT over it.  col[s] is read at its storage type
// type[s] (HS_TYPE_INT32 / INT64 / FLOAT / DOUBLE, or STRING references); valid[s] nullptr: no nulls.
struct CompareDesc {
  const void* col[2];
  const uint8_t* valid[2];
  int64_t factor[2];  // kCmpInt: the multiplier of the side (1: none); kCmpDouble: 10^scale of a decimal side (1 otherwise)
  int32_t type[2];
  int32_t domain, op, negate;
};

template <typename F>
HS_HD int order_floating(F a, F b) {  // SQLOrderingUtil.compareDoubles / compareFloats
  const bool na = a != a, nb = b != b;
  if (na || nb) return na == nb ? 0 : (na ? 1 : -1);
  return a < b ? -1 : (a > b ? 1 : 0);
}

HS_HD int64_t read_integer(const void* col, int type, int64_t row) {
  return type == HS_TYPE_INT32 ? (int64_t)((const int32_t*)col)[row] : ((const int64_t*)col)[row];
}

HS_HD double bits_double(uint64_t b) {
  double d;
  memcpy(&d, &b, 8);
  return d;
}

// sign(u / p - n * 2^e) for u >= 0, 0 < p <= 10^18, 0 < n < 2^55 and -62 <= e <= 10: exact in 128 bits
HS_HD int cmp_quotient_dyadic(int64_t u, int64_t p, int64_t n, int e) {
  __int128 lhs = u, rhs = (__int128)n * p;
  if (e >= 0) rhs <<= e;
  else lhs <<= -e;
  return lhs < rhs ? -1 : (lhs > rhs ? 1 : 0);
}

// u / p rounded to the nearest double, ties to even (p = 10^scale, 1 <= p <= 10^18).  Below 2^53 u and p are exact
// doubles and one division rounds once.  Above it (decimals of 16 digits or more) the conversion of u rounds first, so the
// quotient may sit one ulp off; the midpoints to both neighbours are then tested exactly.
HS_HD double decimal_to_double(int64_t u, int64_t p) {
  const double q = (double)u / (double)p;
  if (p == 1 || (u > -(1ll << 53) && u < (1ll << 53))) return q;
  const bool neg = u < 0;
  const int64_t a = neg ? -u : u;  // |u| < 2^63: a decimal of at most 18 digits
  double d = neg ? -q : q;
  uint64_t b;
  memcpy(&b, &d, 8);
  const int ex = (int)(b >> 52) - 1075;                      // d = m * 2^ex; d >= 2^53 / 10^18 is normal
  const int64_t m = (int64_t)((b & 0xfffffffffffffull) | (1ull << 52));
  const int up = cmp_quotient_dyadic(a, p, 2 * m + 1, ex - 1);
  if (up > 0 || (up == 0 && (m & 1))) {
    d = bits_double(b + 1);
  } else {
    // the midpoint below d: half an ulp lower, or a quarter when d is a power of two (the binade below is finer)
    const int down = m == (1ll << 52) ? cmp_quotient_dyadic(a, p, 4 * m - 1, ex - 2) : cmp_quotient_dyadic(a, p, 2 * m - 1, ex - 1);
    if (down < 0 || (down == 0 && (m & 1))) d = bits_double(b - 1);
  }
  return neg ? -d : d;
}

HS_HD float side_float(const CompareDesc& d, int s, int64_t row) {
  switch (d.type[s]) {
#ifdef __CUDA_ARCH__
    case HS_TYPE_INT32: return __int2float_rn(((const int32_t*)d.col[s])[row]);
    case HS_TYPE_INT64: return __ll2float_rn(((const int64_t*)d.col[s])[row]);
#else
    case HS_TYPE_INT32: return (float)((const int32_t*)d.col[s])[row];
    case HS_TYPE_INT64: return (float)((const int64_t*)d.col[s])[row];
#endif
    default: return ((const float*)d.col[s])[row];
  }
}

HS_HD double side_double(const CompareDesc& d, int s, int64_t row) {
  switch (d.type[s]) {
    case HS_TYPE_INT32:
    case HS_TYPE_INT64: return decimal_to_double(read_integer(d.col[s], d.type[s], row), d.factor[s]);
    case HS_TYPE_FLOAT: return (double)((const float*)d.col[s])[row];
    default: return ((const double*)d.col[s])[row];
  }
}

// -1 / 0 / +1: side 0 against side 1 on a row where neither is null
HS_HD int compare_sides(const CompareDesc& d, int64_t row) {
  switch (d.domain) {
    case kCmpInt: {
      const int64_t a = read_integer(d.col[0], d.type[0], row), b = read_integer(d.col[1], d.type[1], row);
      if (d.factor[0] == 1 && d.factor[1] == 1) return a < b ? -1 : (a > b ? 1 : 0);
      const __int128 x = (__int128)a * d.factor[0], y = (__int128)b * d.factor[1];
      return x < y ? -1 : (x > y ? 1 : 0);
    }
    case kCmpFloat: return order_floating(side_float(d, 0, row), side_float(d, 1, row));
    case kCmpDouble: return order_floating(side_double(d, 0, row), side_double(d, 1, row));
    default: return string_compare(((const uint64_t*)d.col[0])[row], ((const uint64_t*)d.col[1])[row]);
  }
}

// Whether the comparison is true on the row (three-valued logic: unknown does not qualify).  A null on either side makes
// `<`, `<=`, `>`, `>=` and `=` unknown, under NOT too; `<=>` is true on two nulls and false on one, and NOT flips that.
HS_HD bool compare_holds(const CompareDesc& d, int64_t row) {
  const bool n0 = d.valid[0] && !d.valid[0][row], n1 = d.valid[1] && !d.valid[1][row];
  bool r;
  if (n0 || n1) {
    if (d.op != HS_CMP_EQ_NULL_SAFE) return false;
    r = n0 && n1;
  } else {
    const int c = compare_sides(d, row);
    switch (d.op) {
      case HS_CMP_LT: r = c < 0; break;
      case HS_CMP_LE: r = c <= 0; break;
      case HS_CMP_GT: r = c > 0; break;
      case HS_CMP_GE: r = c >= 0; break;
      default: r = c == 0; break;  // HS_CMP_EQ, HS_CMP_EQ_NULL_SAFE
    }
  }
  return r != (d.negate != 0);
}

}  // namespace hs
