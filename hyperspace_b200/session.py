"""Minimal session / DataFrame layer the Hyperspace API needs around the GPU engine.

The reference plugs into Spark: ``spark.read.parquet`` gives the source relation, the optimizer hook
(``ApplyHyperspace``, src/main/scala/com/microsoft/hyperspace/index/rules/ApplyHyperspace.scala:45-66) swaps relations for
index scans, Spark executes.  Spark is not available here, so this module provides just enough of that surface for
notebooks of the shape used in the reference's docs/tests to run unchanged against the GPU engine:

    session = HyperspaceSession()
    df = session.read.parquet("/data/t")
    hs = Hyperspace(session); hs.createIndex(df, IndexConfig("idx", ["k"], ["v1"]))
    session.enableHyperspace()
    df.filter(col("k").between(0, 100)).select("k", "v1").collect()
    a.join(b, on="k").select(...).collect()
    a.filter(col("v") > 0).join(b, on=[("k1", "k1"), ("k2", "key2")]).collect()

Every scan, filter and join runs on the GPU through the C ABI (no CPU fallback); the plan layer only decides which
files the native call reads -- the same decision FilterIndexRule / JoinIndexRule make (hyperspace_b200/rules.py).
"""
from __future__ import annotations

import dataclasses
import datetime
import decimal
import math
import os
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np

from . import log_entry as LE

# conf keys and defaults: src/main/scala/com/microsoft/hyperspace/index/IndexConstants.scala:21-170
INDEX_SYSTEM_PATH = "spark.hyperspace.system.path"
INDEX_NUM_BUCKETS = "spark.hyperspace.index.numBuckets"
INDEX_NUM_BUCKETS_LEGACY = "spark.hyperspace.index.num.buckets"
INDEX_NUM_BUCKETS_DEFAULT = 200
INDEX_LINEAGE_ENABLED = "spark.hyperspace.index.lineage.enabled"
INDEX_HYBRID_SCAN_ENABLED = "spark.hyperspace.index.hybridscan.enabled"
INDEX_HYBRID_SCAN_APPENDED_RATIO_THRESHOLD = "spark.hyperspace.index.hybridscan.maxAppendedRatio"
INDEX_HYBRID_SCAN_DELETED_RATIO_THRESHOLD = "spark.hyperspace.index.hybridscan.maxDeletedRatio"
OPTIMIZE_FILE_SIZE_THRESHOLD = "spark.hyperspace.index.optimize.fileSizeThreshold"
OPTIMIZE_FILE_SIZE_THRESHOLD_DEFAULT = 256 * 1024 * 1024
HYPERSPACE_ENABLED = "spark.hyperspace.enabled"  # session flag toggled by enableHyperspace()/disableHyperspace()
PARQUET_COMPRESSION_CODEC = "spark.sql.parquet.compression.codec"
# the codecs of spark.sql.parquet.compression.codec that index files are written with -> Parquet's codec ids (HS_CODEC_*)
PARQUET_OUTPUT_CODECS = {"none": 0, "uncompressed": 0, "snappy": 1, "gzip": 2, "lz4": 5}


class RuntimeConf:
    """String key/value conf like ``spark.conf`` (typed getters: util/HyperspaceConf.scala:27-238)."""

    def __init__(self, values: Optional[Dict[str, str]] = None):
        self._v: Dict[str, str] = dict(values or {})

    def set(self, key: str, value) -> None:
        self._v[key] = str(value).lower() if isinstance(value, bool) else str(value)

    def get(self, key: str, default=None):
        return self._v.get(key, default)

    def unset(self, key: str) -> None:
        self._v.pop(key, None)

    def get_bool(self, key: str, default: bool) -> bool:
        return str(self._v.get(key, default)).lower() == "true"

    @property
    def num_buckets(self) -> int:
        """HyperspaceConf.numBucketsForIndex (util/HyperspaceConf.scala:88-93): new key, legacy key, then 200."""
        return int(self._v.get(INDEX_NUM_BUCKETS, self._v.get(INDEX_NUM_BUCKETS_LEGACY, INDEX_NUM_BUCKETS_DEFAULT)))

    @property
    def lineage_enabled(self) -> bool:
        return self.get_bool(INDEX_LINEAGE_ENABLED, False)

    @property
    def hybrid_scan_enabled(self) -> bool:
        return self.get_bool(INDEX_HYBRID_SCAN_ENABLED, False)

    @property
    def hybrid_scan_appended_ratio(self) -> float:
        return float(self._v.get(INDEX_HYBRID_SCAN_APPENDED_RATIO_THRESHOLD, 0.3))

    @property
    def hybrid_scan_deleted_ratio(self) -> float:
        return float(self._v.get(INDEX_HYBRID_SCAN_DELETED_RATIO_THRESHOLD, 0.2))

    @property
    def parquet_compression_codec(self) -> int:
        """The codec of the index files' pages (HS_CODEC_*), from spark.sql.parquet.compression.codec, case-insensitive as
        Spark's ParquetOptions reads it.  Unset: UNCOMPRESSED.  A codec the engine does not write raises."""
        name = self._v.get(PARQUET_COMPRESSION_CODEC)
        if name is None:
            return 0
        codec = PARQUET_OUTPUT_CODECS.get(str(name).lower())
        if codec is None:
            raise LE.HyperspaceException(f"Index files cannot be written with {PARQUET_COMPRESSION_CODEC}={name}: "
                                         f"the codecs written are {', '.join(PARQUET_OUTPUT_CODECS)}.")
        return codec

    @property
    def optimize_file_size_threshold(self) -> int:
        return int(self._v.get(OPTIMIZE_FILE_SIZE_THRESHOLD, OPTIMIZE_FILE_SIZE_THRESHOLD_DEFAULT))


# ---------------------------------------------------------------------------------------------------------------------
# expressions
# ---------------------------------------------------------------------------------------------------------------------

# comparison operator of a term -> (lower bound?, strict?) sides it sets
_TERM_SIDES = {">=": ((False,), ()), ">": ((True,), ()), "<=": ((), (False,)), "<": ((), (True,)), "==": ((False,), (False,))}


# string patterns of a term -> (explain() form, hs_predicate_any flag)
_PATTERNS = {"startswith": ("StartsWith", 8), "endswith": ("EndsWith", 16), "contains": ("Contains", 32), "like": ("LIKE", 64)}
_TERM_NOT, _TERM_NULL_TRUE, _TERM_NULL_FALSE = 1, 2, 4  # hs_predicate_any.flags (include/hs_gpu.h)


@dataclass
class AnyTerm:
    """A disjunction on one column (Spark's In / InSet, or an Or of comparisons on that column): the value equals one of
    ``values`` (a list, or a numpy array) or lies in one of ``ranges``, each ``(lo, lo_strict, hi, hi_strict)`` with None
    for an open side.  In three-valued logic: ``null`` is what a null row gives (True: IsNull; False: EqualNullSafe; None:
    unknown); ``null_in_list``: the isin list held a None, so a value outside the list gives unknown rather than false;
    ``pattern``: a string pattern (startswith / endswith / contains / like) whose one value is the pattern; ``negated``:
    Not of all that."""
    column: str
    values: object = field(default_factory=list)
    ranges: List[Tuple[object, bool, object, bool]] = field(default_factory=list)
    null: Optional[bool] = None
    negated: bool = False
    pattern: Optional[str] = None
    null_in_list: bool = False

    def _inner(self) -> str:
        c = self.column
        if self.pattern:
            name = _PATTERNS[self.pattern][0]
            return f"{c} LIKE {self.values[0]!r}" if self.pattern == "like" else f"{name}({c}, {self.values[0]!r})"
        vals = self.values.tolist() if isinstance(self.values, np.ndarray) else list(self.values)
        if not vals and not self.ranges and self.null is True:
            return f"{c} IS NULL"
        if self.null is False:
            parts = [f"{c} <=> {v!r}" for v in vals[:3]] + ([f"... {len(vals) - 3} more"] if len(vals) > 3 else [])
        else:
            shown = ", ".join(repr(v) for v in vals[:3]) + (f", ... {len(vals) - 3} more" if len(vals) > 3 else "")
            parts = [f"{c} IN ({shown})"] if vals or not self.ranges else []
        for lo, ls, hi, hs in self.ranges:
            side = [f"{c} {'>' if ls else '>='} {lo!r}"] if lo is not None else []
            side += [f"{c} {'<' if hs else '<='} {hi!r}"] if hi is not None else []
            parts.append(" AND ".join(side))
        if self.null is True:
            parts.append(f"{c} IS NULL")
        return " OR ".join(f"({p})" if " AND " in p and len(parts) > 1 else p for p in parts)

    def __str__(self) -> str:
        if not self.negated:
            return self._inner()
        if not self.pattern and self.null is True and not len(self.values) and not self.ranges:
            return f"{self.column} IS NOT NULL"
        return f"NOT ({self._inner()})"

    def as_native(self) -> tuple:
        """(column, values, ranges), with the HS_TERM_* flags as a fourth element when there are any, for
        Context.filter_scan_any / bucket_join_any."""
        if self.negated and self.null_in_list:  # NOT (k IN (..., NULL)): false or unknown on every row
            return self.column, [], []
        flags = (_TERM_NOT if self.negated else 0) | (_PATTERNS[self.pattern][1] if self.pattern else 0)
        flags |= {True: _TERM_NULL_TRUE, False: _TERM_NULL_FALSE, None: 0}[self.null]
        if not flags:
            return self.column, self.values, list(self.ranges)
        return self.column, self.values, list(self.ranges), flags


@dataclass
class ColumnCompare:
    """A comparison between two columns of the same row (Spark's BinaryComparison of two attributes): ``left op right`` with
    op one of <, <=, >, >=, = and <=> (EqualNullSafe), under Not when ``negated``.  The engine coerces the two columns'
    types as Spark does; a null on either side makes it unknown, except for <=>."""
    left: str
    op: str
    right: str
    negated: bool = False

    def __str__(self) -> str:
        inner = f"({self.left} {self.op} {self.right})"
        return f"NOT {inner}" if self.negated else inner

    def as_native(self) -> tuple:
        """(left, op, right, HS_TERM_* flags) for Context.filter_scan_cmp / bucket_join_cmp."""
        return self.left, self.op, self.right, _TERM_NOT if self.negated else 0


class Expr:
    """Arithmetic over columns and literals (Spark's Add, Subtract, Multiply, Divide, Remainder and UnaryMinus over
    attributes and literals): a column (``op`` "column", ``value`` its name), a literal (``op`` "literal"), a unary minus
    (``op`` "neg", one argument), a binary operation (``op`` one of + - * / %, two arguments) or a Spark function
    (``op`` one of FUNCTIONS, its arguments; hyperspace_b200.functions builds them).  Its comparison operators,
    ``eqNullSafe`` and ``between`` give a Predicate holding an ExprCompare; the engine types the arithmetic and the
    functions as Spark 3.1 does (include/hs_gpu.h)."""
    __hash__ = None  # == builds a comparison

    def __init__(self, op: str, args: Tuple["Expr", ...] = (), value=None):
        self.op, self.args, self.value = op, tuple(args), value

    @staticmethod
    def of(v) -> "Expr":
        """A Column, an Expr or a literal as an Expr; a literal must be an int, a float or a Decimal."""
        if isinstance(v, Expr):
            return v
        if isinstance(v, Column):
            return Expr("column", value=v.name)
        if isinstance(v, (bool, np.bool_)) or not isinstance(v, (int, float, decimal.Decimal, np.integer, np.floating)):
            raise LE.HyperspaceException(f"the literal {v!r} cannot be used in arithmetic on the GPU path")
        return Expr("literal", value=v)

    @staticmethod
    def operand(v) -> "Expr":
        """Expr.of, which also takes the literals a comparison or a function argument may hold: str and bytes (a string),
        datetime.date (a date) and datetime.datetime (a timestamp; naive is UTC)."""
        if isinstance(v, (str, bytes, datetime.date)):
            return Expr("literal", value=v)
        return Expr.of(v)

    def __str__(self) -> str:
        if self.op == "column":
            return self.value
        if self.op == "literal":
            return self.value.decode("utf-8", "replace") if isinstance(self.value, bytes) else str(self.value)
        if self.op == "neg":
            return f"(- {self.args[0]})"
        if self.op in FUNCTIONS:
            return f"{self.op}({', '.join(str(a) for a in self.args)})"
        return f"({self.args[0]} {self.op} {self.args[1]})"

    def postfix(self) -> List[tuple]:
        """The nodes in postfix order, as Context.filter_scan_expr takes them."""
        if self.op in ("column", "literal"):
            return [(self.op, self.value)]
        tail = ("coalesce", len(self.args)) if self.op == "coalesce" else (self.op,)
        return [n for a in self.args for n in a.postfix()] + [tail]

    @property
    def columns(self) -> List[str]:
        if self.op == "column":
            return [self.value]
        out = []
        for a in self.args:
            out += [c for c in a.columns if c not in out]
        return out

    def renamed(self, fn) -> "Expr":
        """The expression with every column name passed through fn."""
        if self.op == "column":
            return Expr("column", value=fn(self.value))
        if self.op == "literal":
            return self
        return Expr(self.op, tuple(a.renamed(fn) for a in self.args))

    def _bin(self, op, other, reflected=False) -> "Expr":
        other = Expr.of(other)
        return Expr(op, (other, self) if reflected else (self, other))

    def __add__(self, o): return self._bin("+", o)
    def __radd__(self, o): return self._bin("+", o, True)
    def __sub__(self, o): return self._bin("-", o)
    def __rsub__(self, o): return self._bin("-", o, True)
    def __mul__(self, o): return self._bin("*", o)
    def __rmul__(self, o): return self._bin("*", o, True)
    def __truediv__(self, o): return self._bin("/", o)
    def __rtruediv__(self, o): return self._bin("/", o, True)
    def __mod__(self, o): return self._bin("%", o)
    def __rmod__(self, o): return self._bin("%", o, True)
    def __neg__(self): return Expr("neg", (self,))

    def _compare(self, op: str, other, negated: bool = False) -> "Predicate":
        return Predicate({}, [], [], [], [ExprCompare(self, op, Expr.operand(other), negated)])

    def __lt__(self, o): return self._compare("<", o)
    def __le__(self, o): return self._compare("<=", o)
    def __gt__(self, o): return self._compare(">", o)
    def __ge__(self, o): return self._compare(">=", o)
    def __eq__(self, o): return self._compare("=", o)  # noqa: A003
    def __ne__(self, o): return self._compare("=", o, negated=True)  # noqa: A003

    def eqNullSafe(self, o) -> "Predicate":
        return self._compare("<=>", o)

    def between(self, lo, hi) -> "Predicate":
        return (self >= lo) & (self <= hi)

    def isin(self, *values):
        raise LE.HyperspaceException(f"isin on the expression {self} is an OR across columns, which is not handled by the GPU path")

    def __bool__(self):
        raise LE.HyperspaceException(f"the expression {self} is not a filter: compare it")


# The Spark functions an Expr may apply (hyperspace_b200.functions), by their SQL names
FUNCTIONS = ("year", "quarter", "month", "dayofmonth", "dayofweek", "dayofyear", "weekofyear", "hour", "minute", "second",
             "date_add", "date_sub", "datediff", "length", "substring", "abs", "coalesce")
# the functions whose argument may be a timestamp, which they read in the session time zone
_TIME_ZONE_FUNCTIONS = ("year", "quarter", "month", "dayofmonth", "dayofweek", "dayofyear", "weekofyear", "hour", "minute",
                        "second", "date_add", "date_sub", "datediff")
_UTC_ZONES = ("UTC", "GMT", "Z", "+00:00", "-00:00")


def _static_type(e: Expr, types: Dict[str, str]) -> Optional[str]:
    """The Spark type name of an expression as far as the time-zone rule needs it: a column's, a date / timestamp
    literal's, and the date or timestamp a function gives; None otherwise."""
    if e.op == "column":
        return types.get(e.value.lower())
    if e.op == "literal":
        return "timestamp" if isinstance(e.value, datetime.datetime) else ("date" if isinstance(e.value, datetime.date) else None)
    if e.op in ("date_add", "date_sub"):
        return "date"
    if e.op == "coalesce":
        kinds = [_static_type(a, types) for a in e.args]
        return "timestamp" if "timestamp" in kinds else ("date" if "date" in kinds else None)
    return None


def _refuse_time_zone(e: Expr, types: Dict[str, str], zone: str) -> None:
    """A function of a timestamp in a session time zone other than UTC: the engine reads timestamps in UTC."""
    if e.op in _TIME_ZONE_FUNCTIONS and any(_static_type(a, types) == "timestamp" for a in e.args):
        raise LE.HyperspaceException(f"{e} reads a timestamp in the session time zone {zone}, and the GPU path reads timestamps in "
                                     "UTC only: keep it in a Spark Filter")
    for a in e.args:
        _refuse_time_zone(a, types, zone)


@dataclass
class ExprCompare:
    """A comparison of two arithmetic expressions of the same row (Spark's BinaryComparison over Add, Subtract, Multiply,
    Divide, Remainder, UnaryMinus, attributes and literals): ``left op right``, op as in ColumnCompare, under Not when
    ``negated``.  A null side makes it unknown, except for <=>."""
    left: Expr
    op: str
    right: Expr
    negated: bool = False

    def __str__(self) -> str:
        inner = f"({self.left} {self.op} {self.right})"
        return f"NOT {inner}" if self.negated else inner

    @property
    def columns(self) -> List[str]:
        return self.left.columns + [c for c in self.right.columns if c not in self.left.columns]

    def as_native(self) -> tuple:
        """(left nodes, op, right nodes, HS_TERM_* flags) for Context.filter_scan_expr / bucket_join_expr."""
        return self.left.postfix(), self.op, self.right.postfix(), _TERM_NOT if self.negated else 0


def _prefix_range(p) -> Tuple[object, bool, object, bool]:
    """The values that start with p, as a range: [p, succ(p)), succ(p) being p without its trailing 0xff bytes and its
    last byte incremented; open above when nothing is left."""
    b = _as_bytes(p).rstrip(b"\xff")
    return (p, False, b[:-1] + bytes([b[-1] + 1]), True) if b else (p, False, None, False)


def _merge_values(a, b):
    if isinstance(a, np.ndarray) and isinstance(b, np.ndarray) and a.dtype.kind == b.dtype.kind:
        return np.concatenate([a, b])
    return (a.tolist() if isinstance(a, np.ndarray) else list(a)) + (b.tolist() if isinstance(b, np.ndarray) else list(b))


@dataclass
class Predicate:
    """Conjunction of comparisons with literals.  ``bounds`` is the inclusive integer (or byte-string) range per column, which
    the plan layer uses to pick an index; ``terms`` are the comparisons as written -- (column, operator, literal) with the
    operator one of >=, >, <=, <, == -- which the engine evaluates with Spark's type coercion.  ``anys`` are AND-ed
    disjunctions on one column each (``isin`` and ``|``); ``compares`` are AND-ed comparisons between two columns;
    ``exprs`` are AND-ed comparisons of arithmetic expressions."""
    bounds: Dict[str, Tuple[Optional[int], Optional[int]]]
    terms: List[Tuple[str, str, object]] = field(default_factory=list)
    anys: List[AnyTerm] = field(default_factory=list, repr=False)  # explain() shows them by their SQL form
    compares: List[ColumnCompare] = field(default_factory=list, repr=False)
    exprs: List[ExprCompare] = field(default_factory=list, repr=False)

    def __and__(self, other: "Predicate") -> "Predicate":
        out = dict(self.bounds)
        for c, (lo, hi) in other.bounds.items():
            if c in out:
                l0, h0 = out[c]
                lo = l0 if lo is None else (lo if l0 is None else max(lo, l0))
                hi = h0 if hi is None else (hi if h0 is None else min(hi, h0))
            out[c] = (lo, hi)
        return Predicate(out, self._as_terms() + other._as_terms(), self.anys + other.anys, self.compares + other.compares,
                         self.exprs + other.exprs)

    def __or__(self, other: "Predicate") -> "Predicate":
        """An Or of branches on one and the same column, each a comparison, a conjunction of comparisons that is one range
        (at most one lower and one upper bound), or an isin / Or on that column; anything else raises."""
        for branch in (self, other):
            if branch.compares:
                raise LE.HyperspaceException(f"an OR across columns ({branch.compares[0]}) is not handled by the GPU path")
            if branch.exprs:
                raise LE.HyperspaceException(f"an OR across columns ({branch.exprs[0]}) is not handled by the GPU path")
        c = self._single_column()
        if other._single_column().lower() != c.lower():
            raise LE.HyperspaceException(f"an OR across columns ({c}, {other._single_column()}) is not handled by the GPU path")
        merged = AnyTerm(c)
        nulls = []  # what a null row gives in each branch
        for branch in (self, other):
            a = branch.anys[0] if branch.anys else None
            if a is not None and a.negated:
                raise LE.HyperspaceException("a NOT inside an OR is not handled by the GPU path")
            if a is not None and a.pattern not in (None, "startswith"):
                raise LE.HyperspaceException(f"a {a.pattern} pattern inside an OR is not handled by the GPU path")
            if a is None or a.pattern:
                merged.ranges.append(_prefix_range(a.values[0]) if a is not None else branch._one_range())
                nulls.append(None)
            else:
                merged.values = _merge_values(merged.values, a.values)
                merged.ranges += a.ranges
                merged.null_in_list = merged.null_in_list or a.null_in_list
                nulls.append(a.null)
        merged.null = True if True in nulls else (False if all(n is False for n in nulls) else None)
        return Predicate({}, [], [merged])

    def __invert__(self) -> "Predicate":
        """Not of a filter on one column: of one comparison or range, or of one isin, OR, null test or pattern; or of one
        comparison between two columns."""
        cols = {c.lower(): c for c in self.columns}
        if self.compares and len(self.compares) == 1 and not self.anys and not self._as_terms() and not self.exprs:
            return Predicate({}, [], [], [dataclasses.replace(self.compares[0], negated=not self.compares[0].negated)])
        if self.exprs and len(self.exprs) == 1 and not self.anys and not self._as_terms() and not self.compares:
            return Predicate({}, [], [], [], [dataclasses.replace(self.exprs[0], negated=not self.exprs[0].negated)])
        if len(cols) != 1 or self.compares or self.exprs:
            raise LE.HyperspaceException(f"a NOT over several columns ({', '.join(cols.values())}) is not handled by the GPU "
                                         "path: it would be an OR across columns")
        if self.anys:
            if len(self.anys) > 1 or self._as_terms():
                raise LE.HyperspaceException("a NOT must cover one comparison, range, isin, OR, null test or pattern")
            return Predicate({}, [], [dataclasses.replace(self.anys[0], negated=not self.anys[0].negated)])
        try:
            rng = self._one_range()
        except LE.HyperspaceException:
            raise LE.HyperspaceException("a NOT must cover one range: at most one lower and one upper bound") from None
        return Predicate({}, [], [AnyTerm(next(iter(cols.values())), [], [rng], negated=True)])

    def _single_column(self) -> str:
        cols = {c.lower(): c for c in self.columns}
        if len(cols) != 1 or len(self.anys) > 1 or (self.anys and self._as_terms()):
            raise LE.HyperspaceException("an OR branch must compare one column, the same one in every branch")
        return next(iter(cols.values()))

    def _one_range(self) -> Tuple[object, bool, object, bool]:
        lo = hi = None
        lo_s = hi_s = False
        for c, v_lo, ls, v_hi, hs in self.conjuncts():
            if (v_lo is not None and lo is not None) or (v_hi is not None and hi is not None):
                raise LE.HyperspaceException("an OR branch must be one range: at most one lower and one upper bound")
            if v_lo is not None:
                lo, lo_s = v_lo, ls
            if v_hi is not None:
                hi, hi_s = v_hi, hs
        return lo, lo_s, hi, hi_s

    def disjunctions(self) -> List[AnyTerm]:
        """The AND-ed disjunction terms (isin, |), which conjuncts() does not list."""
        return list(self.anys)

    def _as_terms(self) -> List[Tuple[str, str, object]]:
        """The comparisons; a Predicate built from bounds alone states them as inclusive bounds, so that a conjunction with
        one that has terms keeps both sides' conditions."""
        if self.terms:
            return list(self.terms)
        out = []
        for c, (lo, hi) in self.bounds.items():
            if lo is not None:
                out.append((c, ">=", lo))
            if hi is not None:
                out.append((c, "<=", hi))
        return out

    def comparisons(self) -> List[ColumnCompare]:
        """The AND-ed comparisons between two columns, which conjuncts() and disjunctions() do not list."""
        return list(self.compares)

    def expressions(self) -> List[ExprCompare]:
        """The AND-ed comparisons of arithmetic expressions, which the other accessors do not list."""
        return list(self.exprs)

    @property
    def columns(self) -> List[str]:
        out = list(self.bounds)
        for c in ([a.column for a in self.anys] + [n for cc in self.compares for n in (cc.left, cc.right)] +
                  [n for e in self.exprs for n in e.columns]):
            if c not in out:
                out.append(c)
        return out

    def conjuncts(self) -> List[Tuple[str, object, bool, object, bool]]:
        """The comparisons as (column, lo, lo_strict, hi, hi_strict) ranges for Context.filter_scan_where (a Predicate
        built from bounds alone gives its inclusive bounds)."""
        out = []
        for c, op, v in self._as_terms():
            lo_side, hi_side = _TERM_SIDES[op]
            out.append((c, v if lo_side else None, lo_side[0] if lo_side else False, v if hi_side else None,
                        hi_side[0] if hi_side else False))
        return out


def _number(v):
    """A literal as a number for the bounds: a datetime is a timestamp's micros since the epoch (naive = UTC), a date its
    days since the epoch (DataFrame.filter restates a date's bounds in the column's own unit)."""
    if isinstance(v, datetime.datetime):
        from ._native import timestamp_micros

        return timestamp_micros(v)
    if _is_date(v):
        return (v - datetime.date(1970, 1, 1)).days
    return v


def _is_date(v) -> bool:
    return isinstance(v, datetime.date) and not isinstance(v, datetime.datetime)


_DAY_MICROS = 86_400_000_000


def _date_literal(column: str, spark_type: Optional[str], v):
    """A datetime.date literal compared with a column, as Spark casts it: the days on a date column, the day's UTC
    midnight in micros on a timestamp column; any other column raises.  Other literals pass as they are."""
    if not _is_date(v):
        return v
    days = (v - datetime.date(1970, 1, 1)).days
    if spark_type == "date":
        return days
    if spark_type == "timestamp":
        return days * _DAY_MICROS
    raise LE.HyperspaceException(f"the date literal {v} cannot be compared with the {spark_type} column '{column}' on the GPU path")


def _term_bounds(op: str, v) -> Tuple[object, object]:
    """The inclusive integer bounds of one comparison with a number, as Column's comparison operators give them."""
    return {">=": (_ceil(v), None), ">": (_floor(v) + 1, None), "<=": (None, _floor(v)), "<": (None, _ceil(v) - 1), "==": (v, v)}[op]


def _ceil(v):  # NaN and infinities (floating-point columns) stay as they are in the bounds
    v = _number(v)
    return math.ceil(v) if math.isfinite(v) else v


def _floor(v):
    v = _number(v)
    return math.floor(v) if math.isfinite(v) else v


def _as_bytes(v) -> bytes:
    return v.encode("utf-8") if isinstance(v, str) else bytes(v)


class Column:
    def __init__(self, name: str):
        self.name = name

    # integer key columns: a non-integral literal is rounded in the direction that keeps the predicate's meaning
    # (k < 1.5  <=>  k <= 1;  k >= 1.5  <=>  k >= 2).  String / binary literals give byte bounds in UTF8String order --
    # `col("Query") == "facebook"` is the predicate of the reference's own filter-rule tests (T/index/E2EHyperspaceRulesTest.scala).
    def _compare(self, op: str, other: "Column", negated: bool = False) -> Predicate:
        return Predicate({}, [], [], [ColumnCompare(self.name, op, other.name, negated)])

    def substr(self, startPos: int, length: int) -> Expr:
        """Column.substr with int arguments: substring(self, startPos, length)."""
        from .functions import substring

        return substring(self, startPos, length)

    # arithmetic: an Expr, which compares into an expression comparison
    def __add__(self, o): return Expr.of(self) + o
    def __radd__(self, o): return Expr.of(o) + Expr.of(self)
    def __sub__(self, o): return Expr.of(self) - o
    def __rsub__(self, o): return Expr.of(o) - Expr.of(self)
    def __mul__(self, o): return Expr.of(self) * o
    def __rmul__(self, o): return Expr.of(o) * Expr.of(self)
    def __truediv__(self, o): return Expr.of(self) / o
    def __rtruediv__(self, o): return Expr.of(o) / Expr.of(self)
    def __mod__(self, o): return Expr.of(self) % o
    def __rmod__(self, o): return Expr.of(o) % Expr.of(self)
    def __neg__(self): return -Expr.of(self)

    def __ge__(self, v):
        if isinstance(v, Expr):
            return Expr.of(self) >= v
        if isinstance(v, Column):
            return self._compare(">=", v)
        if isinstance(v, (str, bytes)):
            return Predicate({self.name: (_as_bytes(v), None)}, [(self.name, ">=", v)])
        return Predicate({self.name: (_ceil(v), None)}, [(self.name, ">=", v)])

    def __gt__(self, v):
        if isinstance(v, Expr):
            return Expr.of(self) > v
        if isinstance(v, Column):
            return self._compare(">", v)
        if isinstance(v, (str, bytes)):
            return Predicate({self.name: (_as_bytes(v) + b"\x00", None)}, [(self.name, ">", v)])  # the smallest value above v
        return Predicate({self.name: (_floor(v) + 1, None)}, [(self.name, ">", v)])

    def __le__(self, v):
        if isinstance(v, Expr):
            return Expr.of(self) <= v
        if isinstance(v, Column):
            return self._compare("<=", v)
        if isinstance(v, (str, bytes)):
            return Predicate({self.name: (None, _as_bytes(v))}, [(self.name, "<=", v)])
        return Predicate({self.name: (None, _floor(v))}, [(self.name, "<=", v)])

    def __lt__(self, v):
        if isinstance(v, Expr):
            return Expr.of(self) < v
        if isinstance(v, Column):
            return self._compare("<", v)
        if isinstance(v, (str, bytes)):
            raise ValueError("a strict upper bound on a string column has no inclusive form: use <= or between")
        return Predicate({self.name: (None, _ceil(v) - 1)}, [(self.name, "<", v)])

    def __eq__(self, v):  # noqa: A003
        if isinstance(v, Expr):
            return Expr.of(self) == v
        if isinstance(v, Column):
            return self._compare("=", v)
        if isinstance(v, (str, bytes)):
            return Predicate({self.name: (_as_bytes(v), _as_bytes(v))}, [(self.name, "==", v)])
        n = _number(v)
        if not math.isfinite(n) or n != math.floor(n):
            return Predicate({self.name: (1, 0)}, [(self.name, "==", v)])  # an integer never equals a fraction: empty range
        return Predicate({self.name: (int(n), int(n))}, [(self.name, "==", v)])

    def __ne__(self, v):  # noqa: A003
        """Not(EqualTo): a null row, or a None literal, gives unknown."""
        if isinstance(v, Expr):
            return Expr.of(self) != v
        if isinstance(v, Column):
            return self._compare("=", v, negated=True)
        return ~self.isin([v])

    def isin(self, *values) -> Predicate:
        """PySpark's Column.isin: varargs, or one list / tuple / set / numpy array.  None is dropped (it never makes a row
        qualify; under ~ it makes every row unknown); ints, floats, Decimals, datetimes, str and bytes are accepted, and the
        list is cast as Spark casts it (a float makes every value a double, Decimals share one scale).  Strings mixed with
        numbers raise."""
        vals = values[0] if len(values) == 1 and isinstance(values[0], (list, tuple, set, frozenset, np.ndarray)) else values
        if not isinstance(vals, np.ndarray) and any(isinstance(v, (Column, Expr)) for v in vals):
            raise LE.HyperspaceException(f"isin on '{self.name}' with a column value is an OR across columns, which is not "
                                         "handled by the GPU path")
        had_none = not isinstance(vals, np.ndarray) and any(v is None for v in vals)
        vals = vals if isinstance(vals, np.ndarray) else [v for v in vals if v is not None]
        return Predicate({}, [], [AnyTerm(self.name, self._checked(vals, "isin"), null_in_list=had_none)])

    def _checked(self, vals, what):
        from ._native import any_values

        try:
            any_values(vals)
        except ValueError as e:
            raise LE.HyperspaceException(f"{what} on '{self.name}': {e}") from None
        return vals

    def isNull(self) -> Predicate:
        return Predicate({}, [], [AnyTerm(self.name, [], null=True)])

    def isNotNull(self) -> Predicate:
        return Predicate({}, [], [AnyTerm(self.name, [], null=True, negated=True)])

    def eqNullSafe(self, v) -> Predicate:
        """EqualNullSafe (`<=>`): a null row gives false, and `eqNullSafe(None)` is isNull()."""
        if v is None:
            return self.isNull()
        if isinstance(v, Expr):
            return Expr.of(self).eqNullSafe(v)
        if isinstance(v, Column):
            return self._compare("<=>", v)
        return Predicate({}, [], [AnyTerm(self.name, self._checked([v], "eqNullSafe"), null=False)])

    def _pattern(self, kind, p) -> Predicate:
        if not isinstance(p, (str, bytes)):
            raise LE.HyperspaceException(f"{kind} on '{self.name}' takes a string pattern, not {p!r}")
        return Predicate({}, [], [AnyTerm(self.name, [p], pattern=kind)])

    def startswith(self, p) -> Predicate:
        """StartsWith, in bytes: the range [p, succ(p))."""
        return self._pattern("startswith", p)

    def endswith(self, s) -> Predicate:
        return self._pattern("endswith", s)

    def contains(self, s) -> Predicate:
        return self._pattern("contains", s)

    def like(self, pattern) -> Predicate:
        """Like with the escape character '\\': '%' matches any run of characters, '_' one character, and the whole value
        must match.  Values that are not valid UTF-8 are not covered (Spark matches the decoded string)."""
        return self._pattern("like", pattern)

    def between(self, lo, hi):
        if isinstance(lo, (Column, Expr)) or isinstance(hi, (Column, Expr)):  # two conjuncts: lo <= self AND self <= hi
            return (self >= lo) & (self <= hi)
        terms = [(self.name, ">=", lo), (self.name, "<=", hi)]
        if isinstance(lo, (str, bytes)) or isinstance(hi, (str, bytes)):
            return Predicate({self.name: (_as_bytes(lo), _as_bytes(hi))}, terms)
        return Predicate({self.name: (_ceil(lo), _floor(hi))}, terms)


def col(name: str) -> Column:
    return Column(name)


# ---------------------------------------------------------------------------------------------------------------------
# logical plan
# ---------------------------------------------------------------------------------------------------------------------

@dataclass
class RelationNode:
    """A file-based Parquet relation (DefaultFileBasedRelation, index/sources/default/DefaultFileBasedRelation.scala:38-242)."""
    root_paths: List[str]
    files: List[Tuple[str, int, int]]  # (uri, size, mtime) of every data file, DataPathFilter applied
    schema: List[Tuple[str, str]]      # (name, spark type name)

    @property
    def signature(self) -> str:
        """md5 fold over len + mtime + path of the files sorted by path (DefaultFileBasedRelation.scala:45-53,193-196)."""
        acc = ""
        for uri, size, mtime in sorted(self.files, key=lambda f: f[0]):
            acc = LE.md5_hex(acc + f"{size}{mtime}{uri}")
        return acc

    @property
    def column_names(self) -> List[str]:
        return [n for n, _ in self.schema]


@dataclass
class FilterNode:
    child: object
    predicate: Predicate


@dataclass
class ProjectNode:
    child: object
    columns: List[str]


@dataclass
class JoinNode:
    """Equi-join on the AND of ``left column == right column`` for every pair (a pair may name its columns in either
    order; rules.join_key_pairs orients them).  ``how`` is "inner", "leftsemi" or "leftanti" (normalise_join_type), or
    "leftouter", "rightouter" or "fullouter" -- the canonical names of Spark's JoinType.apply -- for an outer join."""
    left: object
    right: object
    pairs: List[Tuple[str, str]]
    how: str = "inner"


# The join types the GPU path runs, under the spellings JoinType.apply accepts once lower-cased with "_" removed:
# EXISTS / IN-subquery (LeftSemi) and NOT EXISTS (LeftAnti) besides the inner join.  The outer joins run from a JoinNode
# whose how is "leftouter", "rightouter" or "fullouter"; DataFrame.join does not take their spellings yet.
_JOIN_TYPES = {"inner": "inner", "leftsemi": "leftsemi", "semi": "leftsemi", "leftanti": "leftanti", "anti": "leftanti"}


def normalise_join_type(how: str) -> str:
    """Spark's JoinType.apply normalisation (lower case, "_" removed) onto "inner", "leftsemi" or "leftanti"; any other
    join type raises HyperspaceException."""
    key = str(how).lower().replace("_", "")
    if key not in _JOIN_TYPES:
        raise LE.HyperspaceException(f"join type '{how}' is not handled by the GPU path: only inner, left semi and left anti "
                                     "equi-joins are")
    return _JOIN_TYPES[key]


_SPARK_TYPE_OF_ARROW = {"int32": "integer", "int64": "long", "float": "float", "double": "double", "bool": "boolean",
                        "string": "string", "large_string": "string", "date32[day]": "date", "timestamp[us]": "timestamp",
                        "int8": "byte", "int16": "short"}


def spark_type_of_arrow(t) -> str:
    """Spark SQL type name of a pyarrow field type, as ParquetToSparkSchemaConverter names the Parquet leaf: a timestamp of
    any unit (INT96 included) is `timestamp`, a decimal `decimal(p,s)`."""
    import pyarrow as pa

    if pa.types.is_timestamp(t):
        return "timestamp"
    if pa.types.is_decimal(t):
        return f"decimal({t.precision},{t.scale})"
    return _SPARK_TYPE_OF_ARROW.get(str(t), str(t))


def spark_values(d: np.ndarray, spark_type: Optional[str]) -> np.ndarray:
    """A result column as the engine returns it (timestamps: int64 micros; decimals: unscaled int32 / int64) in the Python
    form of its Spark type: datetime64[us], or an object array of decimal.Decimal."""
    if spark_type == "timestamp" and d.dtype == np.int64:
        return d.view("datetime64[us]")
    if spark_type and spark_type.startswith("decimal(") and d.dtype in (np.int32, np.int64):
        scale = int(spark_type[len("decimal("):-1].split(",")[1])
        out = np.empty(len(d), dtype=object)
        out[:] = [decimal.Decimal(int(v)).scaleb(-scale) for v in d.tolist()]
        return out
    return d


def list_data_files(path: str) -> List[Tuple[str, int, int]]:
    p = LE.from_uri(path)
    out = []
    if os.path.isdir(p):
        for dirpath, dirnames, filenames in os.walk(p):
            dirnames[:] = sorted(d for d in dirnames if not d.startswith("_") and not d.startswith("."))
            for fn in sorted(filenames):
                if fn.startswith("_") or fn.startswith("."):
                    continue
                out.append(LE.file_status(os.path.join(dirpath, fn)))
    elif os.path.isfile(p):
        out.append(LE.file_status(p))
    else:
        raise LE.HyperspaceException(f"Path does not exist: {path}")
    return out


def read_parquet_schema(path: str) -> List[Tuple[str, str]]:
    """Footer-only read (driver-side metadata, like Spark's schema inference)."""
    import pyarrow.parquet as pq

    sch = pq.ParquetFile(LE.from_uri(path)).schema_arrow
    return [(f.name, spark_type_of_arrow(f.type)) for f in sch]


class DataFrameReader:
    def __init__(self, session: "HyperspaceSession"):
        self._s = session

    def parquet(self, *paths: str) -> "DataFrame":
        files: List[Tuple[str, int, int]] = []
        for p in paths:
            files.extend(list_data_files(p))
        if not files:
            raise LE.HyperspaceException(f"No Parquet data files under {paths}")
        schema = read_parquet_schema(files[0][0])
        return DataFrame(self._s, RelationNode([LE.to_uri(p) for p in paths], files, schema))


class DataFrame:
    def __init__(self, session: "HyperspaceSession", plan):
        self.session = session
        self.plan = plan

    # ---- transformations ------------------------------------------------------------------------------------
    def _resolve(self, name: str) -> str:
        """Column names resolve case-insensitively (Spark's default, spark.sql.caseSensitive=false; the reference does the
        same for index configs in util/ResolverUtils.scala) and come out in the schema's own spelling."""
        hits = [c for c in self.columns if c.lower() == name.lower()]
        if not hits:
            raise LE.HyperspaceException(f"cannot resolve column '{name}' among ({', '.join(self.columns)})")
        if len(hits) > 1 and name not in hits:
            raise LE.HyperspaceException(f"Reference '{name}' is ambiguous, could be: {', '.join(hits)}")
        return name if name in hits else hits[0]

    def filter(self, predicate: Predicate) -> "DataFrame":
        if isinstance(predicate, Expr):
            raise LE.HyperspaceException(f"the expression {predicate} is not a filter: compare it (a boolean column is not "
                                         "handled by the GPU path)")
        self._refuse_join_compares(predicate)
        zone = self.session.conf.get("spark.sql.session.timeZone")
        if zone is not None and str(zone).upper() not in _UTC_ZONES and predicate.exprs:
            types = {n.lower(): t for n, t in _schema_types(self.plan)}
            for e in predicate.exprs:
                _refuse_time_zone(e.left, types, zone)
                _refuse_time_zone(e.right, types, zone)
        bounds = {self._resolve(c): b for c, b in predicate.bounds.items()}
        terms = [(self._resolve(c), op, v) for c, op, v in predicate.terms]
        dated = {c for c, _, v in terms if _is_date(v)}
        if dated:  # a date literal in the unit of its column; that column's bounds restated from its terms
            types = {n.lower(): t for n, t in _schema_types(self.plan)}
            terms = [(c, op, _date_literal(c, types.get(c.lower()), v)) for c, op, v in terms]
            for c in dated:
                los, his = zip(*[_term_bounds(op, v) for t, op, v in terms if t == c])
                lo, hi = [x for x in los if x is not None], [x for x in his if x is not None]
                bounds[c] = (max(lo) if lo else None, min(hi) if hi else None)
        resolved = Predicate(bounds, terms,
                             [dataclasses.replace(a, column=self._resolve(a.column), ranges=list(a.ranges)) for a in predicate.anys],
                             [dataclasses.replace(c, left=self._resolve(c.left), right=self._resolve(c.right)) for c in predicate.compares],
                             [dataclasses.replace(e, left=e.left.renamed(self._resolve), right=e.right.renamed(self._resolve))
                              for e in predicate.exprs])
        return DataFrame(self.session, FilterNode(self.plan, resolved))

    def _refuse_join_compares(self, predicate: Predicate) -> None:
        """A comparison between a column of each side of a join is a non-equi join condition, not a filter of one side."""
        node = self.plan.child if isinstance(self.plan, ProjectNode) else self.plan
        if not isinstance(node, JoinNode):
            return
        sides = [{c.lower() for c in output_columns(node.left)}, {c.lower() for c in output_columns(node.right)}]
        for c in predicate.compares:
            in_sides = [{i for i, side in enumerate(sides) if n.lower() in side} for n in (c.left, c.right)]
            if in_sides[0] and in_sides[1] and not (in_sides[0] & in_sides[1]):
                raise LE.HyperspaceException(f"{c} compares columns of the two sides of a join: a non-equi join condition, "
                                             "which the GPU path does not handle")
        for e in predicate.exprs:  # an expression over columns of both sides is a join condition too
            in_sides = [x for x in ({i for i, side in enumerate(sides) if n.lower() in side} for n in e.columns) if x]
            if in_sides and not set.intersection(*in_sides):
                raise LE.HyperspaceException(f"{e} compares columns of the two sides of a join: a non-equi join condition, "
                                             "which the GPU path does not handle")

    where = filter

    def select(self, *columns: str) -> "DataFrame":
        cols = list(columns[0]) if len(columns) == 1 and isinstance(columns[0], (list, tuple)) else list(columns)
        return DataFrame(self.session, ProjectNode(self.plan, [self._resolve(c) for c in cols]))

    def join(self, other: "DataFrame", on, how: str = "inner") -> "DataFrame":
        how = normalise_join_type(how)
        if isinstance(on, Predicate):
            shown = ", ".join([str(c) for c in on.compares] + [str(e) for e in on.exprs]) or "a filter"
            raise LE.HyperspaceException(f"join `on` {shown}: a non-equi join condition, which the GPU path does not handle; "
                                         "join on column names")
        if isinstance(on, str):
            pairs = [(on, on)]
        elif isinstance(on, tuple) and len(on) == 2 and all(isinstance(c, str) for c in on):
            pairs = [on]
        else:
            pairs = list(on)
            if not pairs or not all(isinstance(p, (tuple, list)) and len(p) == 2 for p in pairs):
                raise LE.HyperspaceException("join `on` takes a column name, a (left, right) pair or a list of such pairs")
        return DataFrame(self.session, JoinNode(self.plan, other.plan, [self._join_pair(other, a, b) for a, b in pairs], how))

    def _join_pair(self, other: "DataFrame", a: str, b: str) -> Tuple[str, str]:
        """Resolves one equality of a join condition: (this side, other side) when it reads so, else swapped, else (for a
        pair whose columns are on the same side, which no index can serve) both on the side that has them."""
        def has(df, c):
            return any(x.lower() == c.lower() for x in df.columns)

        if has(self, a) and has(other, b):
            return self._resolve(a), other._resolve(b)
        if has(other, a) and has(self, b):
            return self._resolve(b), other._resolve(a)
        side = self if has(self, a) and has(self, b) else other
        return side._resolve(a), side._resolve(b)

    # ---- introspection ------------------------------------------------------------------------------------
    @property
    def columns(self) -> List[str]:
        return output_columns(self.plan)

    def explain(self) -> str:
        from .rules import plan_query

        return plan_query(self.session, self.plan).describe()

    # ---- actions ------------------------------------------------------------------------------------
    def collect(self) -> Dict[str, np.ndarray]:
        """Executes the plan on the GPU and returns the result columns as numpy arrays (row order unspecified).  Under an
        outer join a column that can hold nulls comes back as a numpy.ma.MaskedArray, masked where the value is null."""
        from .rules import plan_query

        return plan_query(self.session, self.plan).execute()

    def count(self) -> int:
        res = self.collect()
        return len(next(iter(res.values()))) if res else 0


def _schema_types(plan) -> List[Tuple[str, str]]:
    """(name, Spark type name) of every column of the relations under a plan."""
    if isinstance(plan, RelationNode):
        return list(plan.schema)
    if isinstance(plan, (FilterNode, ProjectNode)):
        return _schema_types(plan.child)
    if isinstance(plan, JoinNode):
        return _schema_types(plan.left) + _schema_types(plan.right)
    return []


def output_columns(plan) -> List[str]:
    if isinstance(plan, RelationNode):
        return plan.column_names
    if isinstance(plan, FilterNode):
        return output_columns(plan.child)
    if isinstance(plan, ProjectNode):
        return list(plan.columns)
    if isinstance(plan, JoinNode):
        if plan.how in ("leftsemi", "leftanti"):  # a semi or anti join outputs the left side's columns only
            return output_columns(plan.left)
        return output_columns(plan.left) + [c for c in output_columns(plan.right)]
    raise TypeError(plan)


class HyperspaceSession:
    """Stand-in for the SparkSession a Hyperspace object is constructed with (src/main/scala/.../Hyperspace.scala:27)."""

    def __init__(self, conf: Optional[Dict[str, str]] = None, device: int = 0):
        self.conf = RuntimeConf(conf)
        self.device = device
        self._ctx = None

    @property
    def read(self) -> DataFrameReader:
        return DataFrameReader(self)

    @property
    def gpu(self):
        """The native context (created on first use; raises without a CUDA device -- there is no CPU fallback)."""
        if self._ctx is None:
            from . import _native

            self._ctx = _native.Context(self.device)
        return self._ctx

    # S/package.scala:40-93
    def enableHyperspace(self) -> "HyperspaceSession":
        self.conf.set(HYPERSPACE_ENABLED, True)
        return self

    def disableHyperspace(self) -> "HyperspaceSession":
        self.conf.set(HYPERSPACE_ENABLED, False)
        return self

    def isHyperspaceEnabled(self) -> bool:
        return self.conf.get_bool(HYPERSPACE_ENABLED, False)

    def stop(self) -> None:
        if self._ctx is not None:
            self._ctx.close()
            self._ctx = None
