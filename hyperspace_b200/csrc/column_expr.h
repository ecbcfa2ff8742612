// column_expr.h -- arithmetic and Spark functions over the columns of a row, compared (`a + b < c`,
// `price * (1 - discount) > 100`, `k % 7 = 0`, `year(d) = 1995`, `substring(s, 1, 2) = '13'`), evaluated as the flat
// typed program the host resolved (predicates.h: resolve_expr, with Spark 3.1's TypeCoercion and DecimalPrecision).
// __host__ __device__ like column_compare.h, whose order_floating, read_integer and decimal_to_double it uses:
// k_expr_mask (read_side.cu) runs arithmetic-only programs one thread per row and k_func_mask those with functions, and
// tests/native/filter_expr.cu and filter_func.cu run the same code on the CPU against Python restatements.
//
// The program is postfix over a stack of at most kMaxExprStack values, one side's result staying below the other side
// while it is computed.  Integers and decimals live in the value's 128-bit integer (an int or a long sign-extended, a
// decimal as its unscaled value), floats and doubles in their own fields; the host has inserted every cast, so each
// instruction knows the representation of its operands.  Every floating-point operation rounds on its own (__fadd_rn and
// friends: nvcc would otherwise fuse a multiply into an add, and Java never does).
#pragma once
#include <cmath>
#include <cstdint>

#include "column_compare.h"
#include "string_match.h"

namespace hs {

constexpr int kMaxExprNodes = 32;                 // per side
constexpr int kMaxExprDepth = 8;                  // stack depth per side
constexpr int kMaxExprStack = kMaxExprDepth + 1;  // the left side's value stays below the right side's stack

// ExprInst.op: stack instructions below kXArith; then one group of eight per arithmetic domain, op = domain + ExprArith
enum ExprOp : int32_t {
  kXLoad = 0,         // push the column cols[arg] at the row (its storage type: ExprColumn.type)
  kXConst = 1,        // push v
  kXRescale = 2,      // the value `arg` slots below the top (0: the top) times v.i (10^k: a decimal to a larger scale)
  kXIntToFloat = 3,   // an int or long at slot arg to float, rounded to nearest
  kXIntToDouble = 4,  // an int or long to double, rounded to nearest
  kXFloatToDouble = 5,
  kXDecToDouble = 6,  // a decimal of at most 18 digits to double (v.i = 10^scale), rounded to nearest as Decimal.toDouble
  kXArith = 8,
  kXInt = 8, kXLong = 16, kXDec = 24, kXFloat = 32, kXDouble = 40,
  // Spark functions (include/hs_gpu.h), run by expr_holds<true> only.  Dates are int days, timestamps long micros,
  // strings and binaries 64-bit references (device_utils.cuh: string_ref) in the value's integer.
  kXFunc = 64,
  kXDatePart = 64,  // the top (days) to the calendar field arg (DatePart)
  kXTimePart = 65,  // the top (micros) to the UTC wall-clock field arg (kPartHour / kPartMinute / kPartSecond)
  kXTsToDate = 66,  // the timestamp at slot arg to its UTC date: floorDiv(micros, 86 400 000 000)
  kXLength = 67,    // the top (a reference) to its length: characters, or bytes when arg is 1 (binary)
  kXSubstr = 68,    // the top (a reference) to substringSQL(pos = low 32 bits of v.i, len = the next 32); arg 1: binary
  kXAbs = 69,       // the top to its absolute value in the arithmetic domain arg (kXInt .. kXDouble)
  kXCoalesce = 70,  // the arg values at the top to the first non-null one
  kXStringConst = 127,  // host only: a string literal in the program's pool, relocated to kXConst before it runs
};
enum ExprArith : int32_t { kXAdd = 0, kXSub = 1, kXMul = 2, kXDiv = 3, kXRem = 4, kXNeg = 5 };
enum DatePart : int32_t { kPartYear, kPartQuarter, kPartMonth, kPartDayOfMonth, kPartDayOfWeek, kPartDayOfYear, kPartWeekOfYear,
                          kPartHour, kPartMinute, kPartSecond };

union ExprValue {
  __int128 i;
  double d;
  float f;
};

struct ExprInst {
  int32_t op, arg;
  int64_t reserved;
  ExprValue v;
};

// one column an expression reads: values at its storage type (HS_TYPE_INT32 / INT64 / FLOAT / DOUBLE, and HS_TYPE_STRING
// references for the functions); valid nullptr: no nulls
struct ExprColumn {
  const void* data;
  const uint8_t* valid;
  int32_t type;
};

// One resolved expression comparison: instructions [begin, end) leave the left side's value and the right side's value
// on the stack, in the comparison's domain (kCmpInt: 128-bit integers, decimals at one scale, dates and timestamps;
// kCmpFloat; kCmpDouble; kCmpString, string references, with functions only).
// op is HS_CMP_*; negate: NOT over it.
struct ExprDesc {
  int32_t begin, end;
  int32_t domain, op, negate;
};

HS_HD float x_fadd(float a, float b) {
#ifdef __CUDA_ARCH__
  return __fadd_rn(a, b);
#else
  return a + b;
#endif
}
HS_HD float x_fsub(float a, float b) {
#ifdef __CUDA_ARCH__
  return __fsub_rn(a, b);
#else
  return a - b;
#endif
}
HS_HD float x_fmul(float a, float b) {
#ifdef __CUDA_ARCH__
  return __fmul_rn(a, b);
#else
  return a * b;
#endif
}
HS_HD double x_dadd(double a, double b) {
#ifdef __CUDA_ARCH__
  return __dadd_rn(a, b);
#else
  return a + b;
#endif
}
HS_HD double x_dsub(double a, double b) {
#ifdef __CUDA_ARCH__
  return __dsub_rn(a, b);
#else
  return a - b;
#endif
}
HS_HD double x_dmul(double a, double b) {
#ifdef __CUDA_ARCH__
  return __dmul_rn(a, b);
#else
  return a * b;
#endif
}
HS_HD double x_ddiv(double a, double b) {
#ifdef __CUDA_ARCH__
  return __ddiv_rn(a, b);
#else
  return a / b;
#endif
}
HS_HD float x_int_to_float(int64_t v) {
#ifdef __CUDA_ARCH__
  return __ll2float_rn(v);
#else
  return (float)v;
#endif
}
HS_HD double x_int_to_double(int64_t v) {
#ifdef __CUDA_ARCH__
  return __ll2double_rn(v);
#else
  return (double)v;
#endif
}

// a = a OP b in the domain dom (b unused by kXNeg).  Returns false where Spark gives null: a zero divisor of DIV or REM.
HS_HD bool expr_arith(int dom, int ar, ExprValue& a, const ExprValue& b) {
  switch (dom) {
    case kXInt: {  // wraps at 2^31: the arithmetic of uint32
      const int32_t x = (int32_t)(int64_t)a.i, y = (int32_t)(int64_t)b.i;
      int32_t r;
      switch (ar) {
        case kXAdd: r = (int32_t)((uint32_t)x + (uint32_t)y); break;
        case kXSub: r = (int32_t)((uint32_t)x - (uint32_t)y); break;
        case kXMul: r = (int32_t)((uint32_t)x * (uint32_t)y); break;
        case kXRem:
          if (y == 0) return false;
          r = y == -1 ? 0 : x % y;  // MIN % -1 is 0 in Java, undefined in C++
          break;
        default: r = (int32_t)(0u - (uint32_t)x); break;
      }
      a.i = r;
      return true;
    }
    case kXLong: {
      const int64_t x = (int64_t)a.i, y = (int64_t)b.i;
      int64_t r;
      switch (ar) {
        case kXAdd: r = (int64_t)((uint64_t)x + (uint64_t)y); break;
        case kXSub: r = (int64_t)((uint64_t)x - (uint64_t)y); break;
        case kXMul: r = (int64_t)((uint64_t)x * (uint64_t)y); break;
        case kXRem:
          if (y == 0) return false;
          r = y == -1 ? 0 : x % y;
          break;
        default: r = (int64_t)(0ull - (uint64_t)x); break;
      }
      a.i = r;
      return true;
    }
    case kXDec:  // exact: the host refused every node that could leave 38 digits
      switch (ar) {
        case kXAdd: a.i = a.i + b.i; return true;
        case kXSub: a.i = a.i - b.i; return true;
        case kXMul: a.i = a.i * b.i; return true;
        case kXRem:
          if (b.i == 0) return false;
          a.i = a.i % b.i;  // truncated, the dividend's sign: BigDecimal.remainder
          return true;
        default: a.i = -a.i; return true;
      }
    case kXFloat:
      switch (ar) {
        case kXAdd: a.f = x_fadd(a.f, b.f); return true;
        case kXSub: a.f = x_fsub(a.f, b.f); return true;
        case kXMul: a.f = x_fmul(a.f, b.f); return true;
        case kXRem:
          if (b.f == 0.0f) return false;  // -0.0 too: Spark tests isZero before IEEE does
          a.f = fmodf(a.f, b.f);
          return true;
        default: a.f = -a.f; return true;
      }
    default:  // kXDouble
      switch (ar) {
        case kXAdd: a.d = x_dadd(a.d, b.d); return true;
        case kXSub: a.d = x_dsub(a.d, b.d); return true;
        case kXMul: a.d = x_dmul(a.d, b.d); return true;
        case kXDiv:
          if (b.d == 0.0) return false;
          a.d = x_ddiv(a.d, b.d);
          return true;
        case kXRem:
          if (b.d == 0.0) return false;
          a.d = fmod(a.d, b.d);
          return true;
        default: a.d = -a.d; return true;
      }
  }
}

// ---- functions -----------------------------------------------------------------------------------------------------------

HS_HD int64_t floor_div(int64_t a, int64_t b) {  // b > 0
  const int64_t q = a / b;
  return q - ((a % b) < 0 ? 1 : 0);
}
// floor_div of a timestamp's micros, which are 128-bit when COALESCE promoted a date beyond the int64 micros range (a
// date of more than 106 751 991 days from the epoch, which Spark's cast would refuse): exact for every value
#ifdef __CUDA_ARCH__
__host__ __device__ __noinline__
#else
inline
#endif
__int128 floor_div_128(__int128 a, int64_t b) {  // out of line: the common 64-bit case keeps k_func_mask's registers
  const __int128 q = a / b;
  return q - ((a % b) < 0 ? 1 : 0);
}
HS_HD __int128 floor_div_wide(__int128 a, int64_t b) {
  return a == (__int128)(int64_t)a ? (__int128)floor_div((int64_t)a, b) : floor_div_128(a, b);
}
HS_HD bool leap_year(int64_t y) { return (y % 4 == 0 && y % 100 != 0) || y % 400 == 0; }

// days since the epoch of a proleptic Gregorian date (H. Hinnant's days_from_civil), exact for any int32 day's year
HS_HD int64_t days_from_civil(int64_t y, int64_t m, int64_t d) {
  y -= m <= 2;
  const int64_t era = floor_div(y, 400);
  const int64_t yoe = y - era * 400;
  const int64_t doy = (153 * (m + (m > 2 ? -3 : 9)) + 2) / 5 + d - 1;
  return era * 146097 + yoe * 365 + yoe / 4 - yoe / 100 + doy - 719468;
}

// Calendar field `part` of the date `days` (LocalDate.ofEpochDay): civil_from_days, with only divisions by constants
HS_HD int32_t date_part(int64_t days, int part) {
  const int64_t z = days + 719468;
  const int64_t era = floor_div(z, 146097);
  const int64_t doe = z - era * 146097;                                 // [0, 146096]
  const int64_t yoe = (doe - doe / 1460 + doe / 36524 - doe / 146096) / 365;  // [0, 399]
  const int64_t doy_mar = doe - (365 * yoe + yoe / 4 - yoe / 100);       // [0, 365], from March 1
  const int64_t mp = (5 * doy_mar + 2) / 153;
  const int64_t m = mp < 10 ? mp + 3 : mp - 9;
  const int64_t y = yoe + era * 400 + (m <= 2);
  switch (part) {
    case kPartYear: return (int32_t)y;
    case kPartQuarter: return (int32_t)((m - 1) / 3 + 1);
    case kPartMonth: return (int32_t)m;
    case kPartDayOfMonth: return (int32_t)(doy_mar - (153 * mp + 2) / 5 + 1);
    case kPartDayOfWeek: return (int32_t)(days - floor_div(days + 4, 7) * 7 + 4) % 7 + 1;  // 1 = Sunday; 1970-01-01 a Thursday
    default: break;
  }
  // day of the year from January 1, 0-based: January 1 is day 306 of the March-based year before it
  const int64_t doy = m <= 2 ? doy_mar - 306 : doy_mar + 59 + leap_year(y);
  if (part == kPartDayOfYear) return (int32_t)(doy + 1);
  // ISO week: week 1 holds the first Thursday; dow 0 = Monday
  const int64_t dow = days + 3 - floor_div(days + 3, 7) * 7;
  const int64_t w = (doy - dow + 10) / 7;  // doy 1-based is doy + 1: (doy + 1 - (dow + 1) + 10) / 7
  auto weeks_in = [](int64_t yr, int64_t jan1_dow) {  // 53 when January 1 is a Thursday, or a Wednesday in a leap year
    return (jan1_dow == 3 || (jan1_dow == 2 && leap_year(yr))) ? 53 : 52;
  };
  const int64_t jan1 = days - doy;
  const int64_t jan1_dow = jan1 + 3 - floor_div(jan1 + 3, 7) * 7;
  if (w < 1) {
    const int64_t py = y - 1, pjan1 = jan1 - 365 - leap_year(py);
    return weeks_in(py, pjan1 + 3 - floor_div(pjan1 + 3, 7) * 7);
  }
  if (w > weeks_in(y, jan1_dow)) return 1;
  return (int32_t)w;
}

// substringSQL over a reference (include/hs_gpu.h): a new reference into the same bytes
HS_HD uint64_t substring_ref(uint64_t ref, int32_t pos, int32_t len, bool binary) {
  const uint8_t* s = ref_ptr(ref);
  const int64_t nb = ref_len(ref);
  int64_t n = nb;  // characters
  if (!binary) {
    n = 0;
    for (int64_t i = 0; i < nb; i += utf8_char_len(s[i])) n++;
  }
  int64_t start = pos > 0 ? (int64_t)pos - 1 : (pos < 0 ? n + pos : 0);
  int64_t end = start + len;
  end = end > 2147483647 ? 2147483647 : (end < -2147483647 - 1 ? -2147483647 - 1 : end);
  start = start < 0 ? 0 : start;
  if (start >= end || start >= n) return string_ref(s, 0);
  if (end > n) end = n;
  if (binary) return string_ref(s + start, (uint32_t)(end - start));
  int64_t i = 0, c = 0;
  while (i < nb && c < start) i += utf8_char_len(s[i]), c++;
  int64_t j = i;
  while (j < nb && c < end) j += utf8_char_len(s[j]), c++;
  if (j > nb) j = nb;
  return string_ref(s + i, (uint32_t)(j - i));
}

// Function instruction `in` over the stack st[0, *sp) with its null bits (kXFunc <= in.op)
HS_HD void expr_func(const ExprInst& in, ExprValue* st, uint32_t& nulls, int& sp) {
  ExprValue& x = st[sp - 1];
  switch (in.op) {
    case kXDatePart: x.i = date_part((int64_t)x.i, in.arg); break;
    case kXTimePart: {
      const int64_t unit = in.arg == kPartHour ? 3600000000ll : (in.arg == kPartMinute ? 60000000ll : 1000000ll);
      const int64_t wrap = in.arg == kPartHour ? 24 : 60;
      const int64_t q = (int64_t)floor_div_wide(x.i, unit);  // 64 bits: a promoted date's micros are below 2^68
      x.i = q - floor_div(q, wrap) * wrap;
      break;
    }
    case kXTsToDate: {
      ExprValue& t = st[sp - 1 - in.arg];
      t.i = floor_div_wide(t.i, 86400000000ll);
      break;
    }
    case kXLength: {
      const uint64_t ref = (uint64_t)x.i;
      int64_t n = ref_len(ref);
      if (!in.arg) {
        const uint8_t* s = ref_ptr(ref);
        const int64_t nb = n;
        n = 0;
        for (int64_t i = 0; i < nb; i += utf8_char_len(s[i])) n++;
      }
      x.i = n;
      break;
    }
    case kXSubstr:
      x.i = substring_ref((uint64_t)x.i, (int32_t)(uint32_t)(uint64_t)in.v.i, (int32_t)(uint32_t)((uint64_t)in.v.i >> 32), in.arg != 0);
      break;
    case kXAbs:
      switch (in.arg) {
        case kXInt: {
          const int32_t v = (int32_t)(int64_t)x.i;
          x.i = v < 0 ? (int32_t)(0u - (uint32_t)v) : v;
          break;
        }
        case kXLong: {
          const int64_t v = (int64_t)x.i;
          x.i = v < 0 ? (int64_t)(0ull - (uint64_t)v) : v;
          break;
        }
        case kXDec: x.i = x.i < 0 ? -x.i : x.i; break;
        case kXFloat: x.f = fabsf(x.f); break;
        default: x.d = fabs(x.d); break;
      }
      break;
    default: {  // kXCoalesce
      const int n = in.arg, base = sp - n;
      int k = 0;
      while (k < n - 1 && ((nulls >> (base + k)) & 1u)) k++;
      st[base] = st[base + k];
      const uint32_t null = (nulls >> (base + k)) & 1u;
      nulls = (nulls & ~(1u << base)) | (null << base);
      sp = base + 1;
      break;
    }
  }
}

// Whether the expression comparison e is true on the row (three-valued logic, as compare_holds: a null side makes `<`,
// `<=`, `>`, `>=` and `=` unknown, under NOT too; `<=>` is true on two null sides and false on one).  kFuncs: the program
// may hold function instructions, string columns and the string domain (k_func_mask); without, exactly the arithmetic
// evaluator k_expr_mask runs.
template <bool kFuncs = false>
HS_HD bool expr_holds(const ExprDesc& e, const ExprInst* insts, const ExprColumn* cols, int64_t row) {
  ExprValue st[kMaxExprStack];
  uint32_t nulls = 0;  // bit k: slot k is null
  int sp = 0;
  for (int pc = e.begin; pc < e.end; pc++) {
    const ExprInst& in = insts[pc];
    const int op = in.op;
    if (op == kXLoad) {
      const ExprColumn& c = cols[in.arg];
      ExprValue v;
      if (kFuncs && c.type == HS_TYPE_STRING) v.i = ((const uint64_t*)c.data)[row];
      else switch (c.type) {
        case HS_TYPE_INT32:
        case HS_TYPE_INT64: v.i = read_integer(c.data, c.type, row); break;
        case HS_TYPE_FLOAT: v.f = ((const float*)c.data)[row]; break;
        default: v.d = ((const double*)c.data)[row]; break;
      }
      const uint32_t null = c.valid && !c.valid[row] ? 1u : 0u;
      nulls = (nulls & ~(1u << sp)) | (null << sp);
      st[sp++] = v;
    } else if (op == kXConst) {
      nulls &= ~(1u << sp);
      st[sp++] = in.v;
    } else if (kFuncs && op >= kXFunc) {
      expr_func(in, st, nulls, sp);
    } else if (op < kXArith) {
      ExprValue& x = st[sp - 1 - in.arg];
      switch (op) {
        case kXRescale: x.i = x.i * in.v.i; break;
        case kXIntToFloat: x.f = x_int_to_float((int64_t)x.i); break;
        case kXIntToDouble: x.d = x_int_to_double((int64_t)x.i); break;
        case kXFloatToDouble: x.d = (double)x.f; break;
        default: x.d = decimal_to_double((int64_t)x.i, (int64_t)in.v.i); break;  // kXDecToDouble
      }
    } else {
      const int dom = op & ~7, ar = op & 7;
      if (ar == kXNeg) {
        expr_arith(dom, ar, st[sp - 1], st[sp - 1]);
        continue;
      }
      sp--;
      uint32_t null = ((nulls >> (sp - 1)) | (nulls >> sp)) & 1u;
      if (!null && !expr_arith(dom, ar, st[sp - 1], st[sp])) null = 1;
      nulls = (nulls & ~(1u << (sp - 1))) | (null << (sp - 1));
    }
  }
  const bool n0 = nulls & 1u, n1 = (nulls >> 1) & 1u;
  bool r;
  if (n0 || n1) {
    if (e.op != HS_CMP_EQ_NULL_SAFE) return false;
    r = n0 && n1;
  } else {
    int c;
    if (kFuncs && e.domain == kCmpString) c = string_compare((uint64_t)st[0].i, (uint64_t)st[1].i);
    else switch (e.domain) {
      case kCmpInt: c = st[0].i < st[1].i ? -1 : (st[0].i > st[1].i ? 1 : 0); break;
      case kCmpFloat: c = order_floating(st[0].f, st[1].f); break;
      default: c = order_floating(st[0].d, st[1].d); break;
    }
    switch (e.op) {
      case HS_CMP_LT: r = c < 0; break;
      case HS_CMP_LE: r = c <= 0; break;
      case HS_CMP_GT: r = c > 0; break;
      case HS_CMP_GE: r = c >= 0; break;
      default: r = c == 0; break;  // HS_CMP_EQ, HS_CMP_EQ_NULL_SAFE
    }
  }
  return r != (e.negate != 0);
}

}  // namespace hs
