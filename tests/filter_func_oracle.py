"""Python restatement of the Spark 3.1 functions in filters (spark.sql.ansi.enabled=false), as include/hs_gpu.h states them
beside the HS_EXPR_YEAR .. HS_EXPR_COALESCE kinds: their types, their values and the comparison of the two sides.  The
arithmetic is filter_expr_oracle's.  Dates are int days since the epoch, timestamps int micros, strings and binaries
bytes.

The rules come from:
  * Year, Quarter, Month, DayOfMonth, DayOfWeek, DayOfYear, WeekOfYear -- LocalDate.ofEpochDay (proleptic Gregorian),
    restated here with numpy.datetime64; DayOfWeek 1 = Sunday; WeekOfYear IsoFields.WEEK_OF_WEEK_BASED_YEAR
  * Hour, Minute, Second -- the UTC wall clock; a timestamp argument of a date function is cast to a date in UTC
    (floorDiv by a day's micros)
  * DateAdd, DateSub, DateDiff -- int arithmetic wrapping at 2^31
  * Length -- UTF8String.numChars (by the length each first byte announces) / the bytes of a binary
  * Substring -- UTF8String.substringSQL / ByteArray.subStringSQL
  * Abs -- wrapping for int and long, the sign cleared for float and double, exact for decimals
  * Coalesce -- findWiderCommonType of the arguments, the first non-null one
A node the library refuses raises Refused.
"""
import datetime

import numpy as np

import filter_expr_oracle as FX
from filter_expr_oracle import DEC, DOUBLE, FLOAT, INT, LONG, Refused, T

STR, BIN, DATE, TS, BOOL = "string", "binary", "date", "timestamp", "boolean"
DATE_PARTS = ("year", "quarter", "month", "dayofmonth", "dayofweek", "dayofyear", "weekofyear")
TIME_PARTS = ("hour", "minute", "second")
FUNCS = DATE_PARTS + TIME_PARTS + ("date_add", "date_sub", "datediff", "length", "substring", "abs", "coalesce")
DAY_US = 86_400_000_000
NUMERIC = (INT, LONG, FLOAT, DOUBLE, DEC)


def arity(node):
    f = node[0]
    if f == "coalesce":
        return node[1]
    if f == "substring":
        return 3
    return 2 if f in ("date_add", "date_sub", "datediff") or f in FX.OPS else 1


def column_type(spark_type):
    if spark_type in (STR, BIN, DATE, TS, BOOL):
        return T(spark_type)
    return FX.column_type(spark_type)


def literal_type(v):
    if isinstance(v, (str, bytes)):
        return T(STR)
    if isinstance(v, datetime.datetime):
        return T(TS)
    if isinstance(v, datetime.date):
        return T(DATE)
    return FX.literal_type(v)


def literal_value(v):
    if isinstance(v, str):
        return v.encode()
    if isinstance(v, bytes):
        return v
    if isinstance(v, datetime.datetime):
        v = v if v.tzinfo else v.replace(tzinfo=datetime.timezone.utc)
        return (v - datetime.datetime(1970, 1, 1, tzinfo=datetime.timezone.utc)) // datetime.timedelta(microseconds=1)
    if isinstance(v, datetime.date):
        return (v - datetime.date(1970, 1, 1)).days
    return v


def _wrap32(v):
    return FX._wrap(v, 32)


# ---- calendar ---------------------------------------------------------------------------------------------------------------

def calendar(days):
    """The seven date parts of every day of an int64 array, restated with numpy.datetime64: a dict of arrays."""
    days = np.asarray(days, dtype=np.int64)
    d = days.astype("datetime64[D]")
    y = d.astype("datetime64[Y]").astype(np.int64) + 1970
    m = d.astype("datetime64[M]").astype(np.int64) % 12 + 1
    dom = (d - d.astype("datetime64[M]").astype("datetime64[D]")).astype(np.int64) + 1
    doy = (d - d.astype("datetime64[Y]").astype("datetime64[D]")).astype(np.int64) + 1
    iso_dow = (days + 3) % 7  # 0 = Monday
    thursday = (days - iso_dow + 3).astype("datetime64[D]")  # the ISO week's year is its Thursday's
    woy = (thursday - thursday.astype("datetime64[Y]").astype("datetime64[D]")).astype(np.int64) // 7 + 1
    return {"year": y, "quarter": (m - 1) // 3 + 1, "month": m, "dayofmonth": dom, "dayofweek": (days + 4) % 7 + 1,
            "dayofyear": doy, "weekofyear": woy}


def date_part(part, days):
    return int(calendar([days])[part][0])


def time_part(part, micros):
    unit, wrap = {"hour": (3_600_000_000, 24), "minute": (60_000_000, 60), "second": (1_000_000, 60)}[part]
    return (micros // unit) % wrap


# ---- strings ----------------------------------------------------------------------------------------------------------------

def _char_len(b):
    return 1 if b < 0xC0 else 2 if b < 0xE0 else 3 if b < 0xF0 else 4


def char_starts(s):
    """The byte offset of every character, then len(s)."""
    out, i = [], 0
    while i < len(s):
        out.append(i)
        i += _char_len(s[i])
    return out + [len(s)]


def num_chars(s):
    return len(char_starts(s)) - 1


def substring(s, pos, length, binary):
    n = len(s) if binary else num_chars(s)
    start = pos - 1 if pos > 0 else (n + pos if pos < 0 else 0)
    end = max(min(start + length, 2**31 - 1), -2**31)
    start = max(start, 0)
    if start >= end or start >= n:
        return b""
    end = min(end, n)
    if binary:
        return s[start:end]
    cs = char_starts(s)
    return s[cs[start]:cs[end]]


# ---- types --------------------------------------------------------------------------------------------------------------------

def wider(a, b, what="coalesce"):
    """findWiderCommonType of two argument types, as the library restates it."""
    if a.kind in NUMERIC and b.kind in NUMERIC:
        a, b = T(a.kind, a.p, a.s), T(b.kind, b.p, b.s)  # an integer literal counts as int / long
        if (a.kind == DEC or b.kind == DEC) and a.kind not in (FLOAT, DOUBLE) and b.kind not in (FLOAT, DOUBLE):
            (pa, sa), (pb, sb) = FX.as_decimal(a), FX.as_decimal(b)
            s = max(sa, sb)
            p = max(pa - sa, pb - sb) + s
            if p > 38:
                raise Refused("needs a decimal of more than 38 digits")
            return T(DEC, p, s)
        if DOUBLE in (a.kind, b.kind) or DEC in (a.kind, b.kind):
            for t in (a, b):
                if t.kind == DEC and t.p > 18:
                    raise Refused("turns a decimal of more than 18 digits into a double")
            return T(DOUBLE)
        if FLOAT in (a.kind, b.kind):
            return T(FLOAT)
        return T(LONG if LONG in (a.kind, b.kind) else INT)
    if a.kind in (DATE, TS) and b.kind in (DATE, TS):
        return T(TS if TS in (a.kind, b.kind) else DATE)
    if a.kind == b.kind and a.kind in (STR, BIN):
        return T(a.kind)
    raise Refused(f"{what} mixes {a} with {b}")


def func_type(f, args):
    """The result type of function f over argument types (refusals raise Refused)."""
    a = args[0]
    if f in DATE_PARTS:
        if a.kind not in (DATE, TS):
            raise Refused("is not a date or timestamp")
        return T(INT)
    if f in TIME_PARTS:
        if a.kind != TS:
            raise Refused("is not a timestamp")
        return T(INT)
    if f in ("date_add", "date_sub", "datediff"):
        if a.kind not in (DATE, TS):
            raise Refused("is not a date or timestamp")
        if f == "datediff":
            if args[1].kind not in (DATE, TS):
                raise Refused("is not a date or timestamp")
            return T(INT)
        if args[1].kind != INT:
            raise Refused("is not an int, short or byte")
        return T(DATE)
    if f in ("length", "substring"):
        if a.kind not in (STR, BIN):
            raise Refused("is not a string or binary")
        return T(INT) if f == "length" else T(a.kind)
    if f == "abs":
        if a.kind not in NUMERIC:
            raise Refused("is not a number")
        if a.narrow:
            raise Refused("is byte or short arithmetic")
        return T(a.kind, a.p, a.s)
    w = args[0]
    if w.kind == BOOL:
        raise Refused("boolean")
    for t in args[1:]:
        w = wider(w, t)
    return w


def _to_wide(v, t, w):
    """An argument value of type t in the coalesce type w (the library's explicit casts)."""
    if v is None:
        return None
    if w.kind == TS and t.kind == DATE:
        return v * DAY_US
    if w.kind in NUMERIC:
        return FX.to_kind(v, T(t.kind, t.p, t.s), w.kind, w.s)
    return v


def evaluate(nodes, row):
    """One side on a row {name: (spark type, value or None)}: (type, value or None).  Arithmetic is filter_expr_oracle's,
    with the refusal of non-numeric operands."""
    st = []
    for n in nodes:
        tag = n[0]
        if tag == "column":
            spark_type, v = row[n[1]]
            t = column_type(spark_type)
            if t.kind == BOOL:
                raise Refused("boolean column")
            if v is not None:
                v = FX.to_kind(v, t, t.kind) if t.kind in (FLOAT, DOUBLE) else (v if t.kind in (STR, BIN) else int(v))
            st.append((t, v))
        elif tag == "literal":
            t = literal_type(n[1])
            v = literal_value(n[1])
            if t.kind == DEC:
                v = int(v.scaleb(t.s))
            elif t.kind == DOUBLE:
                v = np.float64(v)
            st.append((t, v))
        elif tag in FUNCS:
            k = arity(n)
            args = st[-k:]
            del st[-k:]
            if tag == "substring":
                types = [args[0][0]]
            else:
                types = [t for t, _ in args]
            r = func_type(tag, types)
            vals = [v for _, v in args]
            if tag == "coalesce":
                vals = [_to_wide(v, t, r) for t, v in args]
                st.append((r, next((v for v in vals if v is not None), None)))
                continue
            if any(v is None for v in vals):
                st.append((r, None))
                continue
            if tag in DATE_PARTS:
                d = vals[0] // DAY_US if types[0].kind == TS else vals[0]
                st.append((r, date_part(tag, d)))
            elif tag in TIME_PARTS:
                st.append((r, time_part(tag, vals[0])))
            elif tag in ("date_add", "date_sub", "datediff"):
                a, b = (v // DAY_US if t.kind == TS else v for t, v in args)
                st.append((r, _wrap32(a + b if tag == "date_add" else a - b)))
            elif tag == "length":
                st.append((r, len(vals[0]) if types[0].kind == BIN else num_chars(vals[0])))
            elif tag == "substring":
                st.append((r, substring(vals[0], vals[1], vals[2], types[0].kind == BIN)))
            else:  # abs
                t, v = args[0]
                if t.kind in (INT, LONG):
                    st.append((r, FX._wrap(abs(v), 32 if t.kind == INT else 64)))
                else:
                    st.append((r, abs(v)))
        elif tag == "neg" or tag in FX.OPS:
            k = arity(n) if tag != "neg" else 1
            args = st[-k:]
            del st[-k:]
            for t, _ in args:
                if t.kind not in NUMERIC:
                    raise Refused(f"({t.kind}) cannot be used in arithmetic")
            sub = [("column", f"_{i}") for i in range(k)] + [n]
            t, v = FX.evaluate(sub, {f"_{i}": (_spark_name(t), v) for i, (t, v) in enumerate(args)}) if all(
                t.lit_digits == 0 for t, _ in args) else _literal_arith(n, args)
            st.append((t, v))
        else:
            raise ValueError(n)
    (t, v), = st
    return t, v


def _spark_name(t):
    if t.narrow:
        return "byte"
    return {INT: "integer", LONG: "long", FLOAT: "float", DOUBLE: "double"}.get(t.kind) or f"decimal({t.p},{t.s})"


def _literal_arith(n, args):
    """Arithmetic with an integer literal operand, which keeps its digits (DecimalType.fromLiteral)."""
    nodes, row = [], {}
    for i, (t, v) in enumerate(args):
        if t.lit_digits:
            nodes.append(("literal", v))
        else:
            nodes.append(("column", f"_{i}"))
            row[f"_{i}"] = (_spark_name(t), v)
    return FX.evaluate(nodes + [n], row)


def compare_domain(a, b):
    """The domain the two sides compare in: a filter_expr_oracle domain, "string" or "days_or_micros"."""
    if a.kind in NUMERIC and b.kind in NUMERIC:
        return FX.common(a, b)
    if a.kind in (DATE, TS) and b.kind in (DATE, TS):
        return "micros" if TS in (a.kind, b.kind) else "days", None
    if a.kind == b.kind and a.kind in (STR, BIN):
        return "string", None
    raise Refused(f"{a} and {b} cannot be compared")


def holds(left, op, right, negated, row):
    (ta, a), (tb, b) = evaluate(left, row), evaluate(right, row)
    kind, scale = compare_domain(ta, tb)
    if a is None or b is None:
        if op != "<=>":
            return False
        r = a is None and b is None
    else:
        if kind == "micros":
            a, b = (v * DAY_US if t.kind == DATE else v for t, v in ((ta, a), (tb, b)))
            c = (a > b) - (a < b)
        elif kind in ("days", "string"):
            c = (a > b) - (a < b)
        else:
            c = FX._order(FX.to_kind(a, ta, kind, scale), FX.to_kind(b, tb, kind, scale))
        r = {"<": c < 0, "<=": c <= 0, ">": c > 0, ">=": c >= 0, "=": c == 0, "<=>": c == 0}[op]
    return r != negated


def side_type(nodes, types):
    return evaluate(nodes, {n: (t, None) for n, t in types.items()})[0]


def mask(left, op, right, negated, columns, n):
    """holds() over n rows of columns {name: (spark type, values, valid or None)}."""
    out = np.zeros(n, dtype=bool)
    for i in range(n):
        row = {c: (t, None if valid is not None and not valid[i] else vals[i]) for c, (t, vals, valid) in columns.items()}
        out[i] = holds(left, op, right, negated, row)
    return out
