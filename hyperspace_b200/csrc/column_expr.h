// column_expr.h -- arithmetic over the columns of a row, compared (`a + b < c`, `price * (1 - discount) > 100`,
// `k % 7 = 0`), evaluated as the flat typed program the host resolved (predicates.h: resolve_expr, with Spark 3.1's
// TypeCoercion and DecimalPrecision).  __host__ __device__ like column_compare.h, whose order_floating, read_integer and
// decimal_to_double it uses: k_expr_mask (read_side.cu) runs it one thread per row, and tests/native/filter_expr.cu runs
// the same code on the CPU against a Python restatement.
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
};
enum ExprArith : int32_t { kXAdd = 0, kXSub = 1, kXMul = 2, kXDiv = 3, kXRem = 4, kXNeg = 5 };

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

// one column an expression reads: values at its storage type (HS_TYPE_INT32 / INT64 / FLOAT / DOUBLE); valid nullptr: no
// nulls
struct ExprColumn {
  const void* data;
  const uint8_t* valid;
  int32_t type;
};

// One resolved expression comparison: instructions [begin, end) leave the left side's value and the right side's value
// on the stack, in the comparison's domain (kCmpInt: 128-bit integers, decimals at one scale; kCmpFloat; kCmpDouble).
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

// Whether the expression comparison e is true on the row (three-valued logic, as compare_holds: a null side makes `<`,
// `<=`, `>`, `>=` and `=` unknown, under NOT too; `<=>` is true on two null sides and false on one).
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
      switch (c.type) {
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
    switch (e.domain) {
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
