"""Python restatement of Spark 3.1's arithmetic in filters (spark.sql.ansi.enabled=false), as include/hs_gpu.h states it
beside hs_expr_compare: the types of Add, Subtract, Multiply, Divide, Remainder and UnaryMinus over attributes and
literals, their values, and the comparison of the two sides.  Integers are exact Python ints wrapped at their width,
decimals exact unscaled ints, floats numpy float32 / float64 scalars (each operation rounds on its own, never fused).

The rules come from:
  * TypeCoercion.ImplicitTypeCasts / findTightestCommonType -- int with long is long, with float float, with double double
  * TypeCoercion.Division -- Divide casts non-decimal operands to double
  * DecimalPrecision -- decimal result types (Add/Subtract, Multiply, Remainder), nondecimalAndDecimal (an int column as
    decimal(10,0), a long as decimal(20,0), an integer literal as DecimalType.fromLiteral: its digits), decimal with
    float / double as double, BinaryComparison of two decimals in widerDecimalType
  * Literal / Decimal.set -- a Python Decimal is DecimalType(max(digits, scale), scale)
  * Divide / Remainder (DivModLike) -- a zero divisor gives null (isZero: -0.0 too); Java's % truncates; MIN % -1 = 0
  * SQLOrderingUtil.compareDoubles / compareFloats -- NaN equals NaN and sorts above +inf, -0.0 equals 0.0
A node the library refuses raises Refused.
"""
import decimal
import math
from fractions import Fraction

import numpy as np

INT, LONG, FLOAT, DOUBLE, DEC = "int", "long", "float", "double", "decimal"
OPS = ("+", "-", "*", "/", "%")


class Refused(Exception):
    pass


class T:
    """An operand's type: kind, a decimal's (p, s), an integer literal's digits, a byte / short column (narrow)."""

    def __init__(self, kind, p=0, s=0, lit_digits=0, narrow=False):
        self.kind, self.p, self.s, self.lit_digits, self.narrow = kind, p, s, lit_digits, narrow

    def __eq__(self, o):
        return (self.kind, self.p, self.s) == (o.kind, o.p, o.s)

    def __repr__(self):
        return f"decimal({self.p},{self.s})" if self.kind == DEC else self.kind


def column_type(spark_type):
    """The operand type of a column of a Spark type name; other types are refused."""
    if spark_type.startswith("decimal("):
        p, s = (int(x) for x in spark_type[len("decimal("):-1].split(","))
        return T(DEC, p, s)
    kinds = {"integer": INT, "byte": INT, "short": INT, "long": LONG, "float": FLOAT, "double": DOUBLE}
    if spark_type not in kinds:
        raise Refused(f"the column ({spark_type}) cannot be used in arithmetic")
    return T(kinds[spark_type], narrow=spark_type in ("byte", "short"))


def digits(v):
    return len(str(abs(int(v))))


def literal_type(v):
    """py4j's typing of a Python literal: int (32 bits) / long, double, decimal(max(digits, scale), scale)."""
    if isinstance(v, decimal.Decimal):
        _, ds, exp = v.as_tuple()
        s = max(0, -exp)
        return T(DEC, max(digits(int(v.scaleb(s))), s), s)
    if isinstance(v, float):
        return T(DOUBLE)
    return T(INT if -2**31 <= v < 2**31 else LONG, lit_digits=digits(v))


def as_decimal(t):
    if t.kind == DEC:
        return t.p, t.s
    return (t.lit_digits or (10 if t.kind == INT else 20)), 0


def _is_fp(t):
    return t.kind in (FLOAT, DOUBLE)


def common(a, b):
    """The domain two operands (or the two compared sides) meet in: (kind, decimal scale or None)."""
    if (a.kind == DEC or b.kind == DEC) and not _is_fp(a) and not _is_fp(b):
        (pa, sa), (pb, sb) = as_decimal(a), as_decimal(b)
        s = max(sa, sb)
        if max(pa - sa, pb - sb) + s > 38:
            raise Refused("needs a decimal of more than 38 digits")
        return DEC, s
    if DOUBLE in (a.kind, b.kind) or DEC in (a.kind, b.kind):
        for t in (a, b):
            if t.kind == DEC and t.p > 18:
                raise Refused("turns a decimal of more than 18 digits into a double")
        return DOUBLE, None
    if FLOAT in (a.kind, b.kind):
        return FLOAT, None
    return (LONG if LONG in (a.kind, b.kind) else INT), None


def result_type(op, a, b=None):
    """The type of `a op b` (or of `- a` when op is "neg")."""
    if op == "neg":
        if a.narrow:
            raise Refused("is byte or short arithmetic")
        return T(a.kind, a.p, a.s)
    if a.narrow and b.narrow:
        raise Refused("is byte or short arithmetic")
    if op == "/":
        if (a.kind == DEC or b.kind == DEC) and not _is_fp(a) and not _is_fp(b):
            raise Refused("decimal division is not handled")
        common(T(DOUBLE), a), common(T(DOUBLE), b)  # the decimal -> double refusals
        return T(DOUBLE)
    kind, _ = common(a, b)
    if kind != DEC:
        return T(kind)
    (p1, s1), (p2, s2) = as_decimal(a), as_decimal(b)
    s = max(s1, s2)
    if op in ("+", "-"):
        r = T(DEC, max(p1 - s1, p2 - s2) + s + 1, s)
    elif op == "*":
        r = T(DEC, p1 + p2 + 1, s1 + s2)
    else:
        r = T(DEC, min(p1 - s1, p2 - s2) + s, s)
    if r.p > 38:
        raise Refused("needs a decimal of more than 38 digits")
    return r


def _wrap(v, bits):
    v &= (1 << bits) - 1
    return v - (1 << bits) if v >> (bits - 1) else v


def int_to_f32(x):
    """An integer to float, rounded to nearest, ties to even, in one rounding."""
    x = int(x)
    if abs(x) < 2**53:
        return np.float32(float(x))
    a = abs(x)
    shift = a.bit_length() - 24
    q, r = divmod(a, 1 << shift)
    half = 1 << (shift - 1)
    if r > half or (r == half and q & 1):
        q += 1
    return np.float32(math.copysign(math.ldexp(q, shift), x))


def to_kind(v, t, kind, scale=None):
    """Value v of type t in the domain kind (DEC: the unscaled value at `scale`)."""
    if kind == DEC:
        s = t.s if t.kind == DEC else 0
        return int(v) * 10**(scale - s)
    if kind == DOUBLE:
        if t.kind == DEC:
            return np.float64(float(Fraction(int(v), 10**t.s)))
        if t.kind in (INT, LONG):
            return np.float64(float(int(v)))
        return np.float64(v)
    if kind == FLOAT:
        return int_to_f32(v) if t.kind in (INT, LONG) else np.float32(v)
    return int(v)


def arith(op, t, a, b):
    """a op b in the result type t (operands already in t's domain; decimals: +, -, % at t's scale, * at their own)."""
    if t.kind in (INT, LONG):
        bits = 32 if t.kind == INT else 64
        if op == "%":
            if b == 0:
                return None
            r = abs(a) % abs(b)
            return _wrap(-r if a < 0 else r, bits)
        return _wrap({"+": a + b, "-": a - b, "*": a * b}[op], bits)
    if t.kind == DEC:
        if op == "%":
            if b == 0:
                return None
            r = abs(a) % abs(b)
            return -r if a < 0 else r
        return {"+": a + b, "-": a - b, "*": a * b}[op]
    if op in ("/", "%") and b == 0:
        return None
    with np.errstate(all="ignore"):
        if op == "%":
            return np.fmod(a, b)
        return {"+": a + b, "-": a - b, "*": a * b, "/": a / b}[op]


def evaluate(nodes, row):
    """One side (postfix nodes: ("column", name), ("literal", v), (op,)) on a row {name: (spark type, value or None)}:
    (type, value or None)."""
    st = []
    for n in nodes:
        if n[0] == "column":
            spark_type, v = row[n[1]]
            t = column_type(spark_type)
            st.append((t, None if v is None else to_kind(v, t, t.kind) if t.kind in (FLOAT, DOUBLE) else int(v)))
        elif n[0] == "literal":
            t = literal_type(n[1])
            v = n[1]
            if t.kind == DEC:
                v = int(v.scaleb(t.s))
            elif t.kind == DOUBLE:
                v = np.float64(v)
            st.append((t, v))
        elif n[0] == "neg":
            t, v = st.pop()
            r = result_type("neg", t)
            if v is None:
                st.append((r, None))
            elif r.kind in (INT, LONG):
                st.append((r, _wrap(-v, 32 if r.kind == INT else 64)))
            else:
                st.append((r, -v))
        else:
            op = n[0]
            tb, b = st.pop()
            ta, a = st.pop()
            r = result_type(op, ta, tb)
            if a is None or b is None:
                st.append((r, None))
                continue
            if op == "/":
                st.append((r, arith(op, r, to_kind(a, ta, DOUBLE), to_kind(b, tb, DOUBLE))))
            elif r.kind == DEC and op == "*":
                st.append((r, arith(op, r, to_kind(a, ta, DEC, as_decimal(ta)[1]), to_kind(b, tb, DEC, as_decimal(tb)[1]))))
            else:
                st.append((r, arith(op, r, to_kind(a, ta, r.kind, r.s), to_kind(b, tb, r.kind, r.s))))
    (t, v), = st
    return t, v


def _order(a, b):
    na, nb = a != a, b != b
    if na or nb:
        return 0 if na == nb else (1 if na else -1)
    return -1 if a < b else (1 if a > b else 0)


def holds(left, op, right, negated, row):
    """Whether `left op right` (under NOT when negated) is true on the row."""
    (ta, a), (tb, b) = evaluate(left, row), evaluate(right, row)
    kind, scale = common(ta, tb)
    if a is None or b is None:
        if op != "<=>":
            return False
        r = a is None and b is None
    else:
        c = _order(to_kind(a, ta, kind, scale), to_kind(b, tb, kind, scale))
        r = {"<": c < 0, "<=": c <= 0, ">": c > 0, ">=": c >= 0, "=": c == 0, "<=>": c == 0}[op]
    return r != negated


def side_type(nodes, types):
    """The type of one side over columns of the given Spark types (refusals raise Refused)."""
    row = {n: (t, None) for n, t in types.items()}
    return evaluate(nodes, row)[0]


def mask(left, op, right, negated, columns, n):
    """holds() over n rows of columns {name: (spark type, values, valid or None)}."""
    out = np.zeros(n, dtype=bool)
    for i in range(n):
        row = {c: (t, None if valid is not None and not valid[i] else vals[i]) for c, (t, vals, valid) in columns.items()}
        out[i] = holds(left, op, right, negated, row)
    return out
