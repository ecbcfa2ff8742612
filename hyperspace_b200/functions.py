"""The Spark SQL functions a filter can apply on the GPU path, mirroring pyspark.sql.functions:

    from hyperspace_b200.functions import col, year, substring, datediff
    df.filter(year(col("o_orderdate")) == 1995)
    df.filter(substring(col("c_phone"), 1, 2) == "13")
    df.filter(datediff("l_receiptdate", "l_commitdate") > 30)

Each function takes a Column, an Expr or a column name and returns an Expr, which compares into an expression
comparison (session.ExprCompare) like arithmetic does; the engine types it as Spark 3.1 does (include/hs_gpu.h).  A
function that reads a timestamp is refused when spark.sql.session.timeZone is set to a zone other than UTC.
"""
from typing import Union

import numpy as np

from . import log_entry as LE
from .session import Column, Expr, col

__all__ = ["col", "lit", "year", "quarter", "month", "dayofmonth", "dayofweek", "dayofyear", "weekofyear", "hour", "minute",
           "second", "date_add", "date_sub", "datediff", "length", "substring", "abs", "coalesce"]

ColumnOrName = Union[Column, Expr, str]


def _arg(c: ColumnOrName) -> Expr:
    """A function argument: a Column, an Expr, or a column name (as in pyspark.sql.functions)."""
    if isinstance(c, str):
        return Expr("column", value=c)
    if isinstance(c, (Column, Expr)):
        return Expr.of(c)
    raise LE.HyperspaceException(f"a function argument must be a Column, an expression or a column name, not {c!r}")


def _int(v, what: str) -> int:
    if isinstance(v, (bool, np.bool_)) or not isinstance(v, (int, np.integer)) or not -2**31 <= int(v) < 2**31:
        raise LE.HyperspaceException(f"{what} must be an int literal on the GPU path, not {v!r}")
    return int(v)


def lit(v) -> Expr:
    """A literal: an int, float, Decimal, str, bytes, datetime.date or datetime.datetime."""
    return Expr.operand(v)


def _unary(name: str):
    def f(c: ColumnOrName) -> Expr:
        return Expr(name, (_arg(c),))

    f.__name__ = name
    f.__doc__ = f"Spark's {name}() of a column or expression (include/hs_gpu.h states its type and value)."
    return f


year = _unary("year")
quarter = _unary("quarter")
month = _unary("month")
dayofmonth = _unary("dayofmonth")
dayofweek = _unary("dayofweek")
dayofyear = _unary("dayofyear")
weekofyear = _unary("weekofyear")
hour = _unary("hour")
minute = _unary("minute")
second = _unary("second")
length = _unary("length")
abs = _unary("abs")  # noqa: A001 -- pyspark.sql.functions.abs


def date_add(start: ColumnOrName, days) -> Expr:
    """start + days (an int literal, or a byte, short or int column): a date."""
    return Expr("date_add", (_arg(start), _arg(days) if isinstance(days, (str, Column, Expr)) else Expr.of(_int(days, "date_add's days"))))


def date_sub(start: ColumnOrName, days) -> Expr:
    """start - days: a date."""
    return Expr("date_sub", (_arg(start), _arg(days) if isinstance(days, (str, Column, Expr)) else Expr.of(_int(days, "date_sub's days"))))


def datediff(end: ColumnOrName, start: ColumnOrName) -> Expr:
    """end - start in days: an int."""
    return Expr("datediff", (_arg(end), _arg(start)))


def substring(str: ColumnOrName, pos: int, len: int) -> Expr:  # noqa: A002 -- pyspark.sql.functions' parameter names
    """substring(str, pos, len) as Spark's Substring: pos 1-based (0 counts as 1, a negative pos from the end), at most
    len characters of a string or bytes of a binary."""
    return Expr("substring", (_arg(str), Expr.of(_int(pos, "substring's pos")), Expr.of(_int(len, "substring's len"))))


def coalesce(*cols) -> Expr:
    """The first non-null argument, in the arguments' wider type; literals go in as lit(v)."""
    if len(cols) < 2:
        raise LE.HyperspaceException("coalesce on the GPU path takes at least two arguments")
    if len(cols) > 8:
        raise LE.HyperspaceException("coalesce on the GPU path takes at most eight arguments")
    return Expr("coalesce", tuple(_arg(c) for c in cols))
