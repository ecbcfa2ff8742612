"""numpy restatement of the comparisons between two columns (Spark 3.1's BinaryComparison of two attributes), with
three-valued logic over validity masks: the oracle of tests/test_filter_compare_host.py and tests/test_gpu_filter_compare.py.

A column is ``(spark_type, values, valid)``: values as the engine stores them (int32 / int64 numpy arrays for integers,
dates (days), timestamps (micros) and decimals (unscaled); float32 / float64; bytes objects for strings), valid a bool
array or None.  Spark types are names: integer, long, float, double, string, binary, date, timestamp, decimal(p,s)."""
import re

import numpy as np

OPS = ("<", "<=", ">", ">=", "=", "<=>")
DAY_MICROS = 86_400_000_000


def _decimal(t):
    m = re.fullmatch(r"decimal\((\d+),(\d+)\)", t)
    return (int(m.group(1)), int(m.group(2))) if m else None


def kind(t):
    if _decimal(t):
        return "decimal"
    return {"byte": "integer", "short": "integer"}.get(t, t)


def domain(lt, rt):
    """("int", lfactor, rfactor) / ("float",) / ("double", ldivisor, rdivisor) / ("string",), or None when Spark's coercion
    leaves the pair without a comparison the GPU path runs."""
    lk, rk = kind(lt), kind(rt)
    ints = {"integer", "long"}
    if {lk, rk} <= ints:
        return ("int", 1, 1)
    if {lk, rk} <= {"date", "timestamp"}:
        return ("int", DAY_MICROS if (lk, rk) == ("date", "timestamp") else 1, DAY_MICROS if (lk, rk) == ("timestamp", "date") else 1)
    if lk == rk and lk in ("string", "binary"):
        return ("string",)
    ls = _decimal(lt)[1] if lk == "decimal" else 0
    rs = _decimal(rt)[1] if rk == "decimal" else 0
    if "decimal" in (lk, rk) and {lk, rk} <= ints | {"decimal"}:
        s = max(ls, rs)
        return ("int", 10 ** (s - ls), 10 ** (s - rs))
    if {lk, rk} <= ints | {"float", "double", "decimal"}:
        if "double" in (lk, rk) or "decimal" in (lk, rk):
            return ("double", 10 ** ls, 10 ** rs)
        return ("float",)
    return None


def _as_float32(v, t):
    v = np.asarray(v)
    return v.astype(np.float32) if v.dtype != np.float32 else v  # int64 -> float32 rounds once, to nearest


def _as_double(v, divisor):
    v = np.asarray(v)
    if v.dtype.kind == "f":
        return v.astype(np.float64)
    if divisor == 1:
        return v.astype(np.float64)
    return np.array([int(u) / divisor for u in v.tolist()], dtype=np.float64)  # correctly rounded, as Decimal.toDouble


def _order_floating(a, b):
    na, nb = np.isnan(a), np.isnan(b)
    c = np.where(a < b, -1, np.where(a > b, 1, 0))
    return np.where(na | nb, np.where(na & nb, 0, np.where(na, 1, -1)), c)


def order(lt, lv, rt, rv):
    """-1 / 0 / +1 per row, side against side, ignoring nulls."""
    d = domain(lt, rt)
    if d is None:
        raise ValueError(f"{lt} and {rt} cannot be compared")
    if d[0] == "int":
        a = [int(x) * d[1] for x in np.asarray(lv).tolist()]
        b = [int(x) * d[2] for x in np.asarray(rv).tolist()]
        return np.array([(x > y) - (x < y) for x, y in zip(a, b)], dtype=np.int64)
    if d[0] == "string":
        return np.array([(bytes(x) > bytes(y)) - (bytes(x) < bytes(y)) for x, y in zip(lv, rv)], dtype=np.int64)
    if d[0] == "float":
        return _order_floating(_as_float32(lv, lt), _as_float32(rv, rt))
    return _order_floating(_as_double(lv, d[1]), _as_double(rv, d[2]))


def mask(left, right, op, negated=False):
    """Rows where `left op right` (NOT of it when negated) is true; left / right are (spark_type, values, valid)."""
    (lt, lv, lval), (rt, rv, rval) = left, right
    n = len(lv)
    lnull = np.zeros(n, bool) if lval is None else ~np.asarray(lval, bool)
    rnull = np.zeros(n, bool) if rval is None else ~np.asarray(rval, bool)
    c = order(lt, lv, rt, rv)
    r = {"<": c < 0, "<=": c <= 0, ">": c > 0, ">=": c >= 0, "=": c == 0, "<=>": c == 0}[op]
    any_null = lnull | rnull
    if op == "<=>":
        r = np.where(any_null, lnull & rnull, r)
        return r != negated
    return np.where(any_null, False, r != negated)
