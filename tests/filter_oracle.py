"""numpy restatement of Spark 3.1's evaluation of a conjunction of range comparisons with literals -- what the GPU filter
scans (hs_filter_scan_where) are compared against.

Written independently of the engine's host code (which binary-searches an encoded domain): here every row is compared
directly, after the promotion Spark's binary-comparison coercion applies.
  * The comparison happens in the wider of the column's and the literal's types, precedence int < long < float < double:
    an int / long column against a double literal compares (double)k (rounded beyond 2^53); a float column against a
    double literal compares (double)f; a float column against a long literal compares with (float)literal.
  * Floating-point order is SQLOrderingUtil.compareDoubles: NaN == NaN, NaN above +inf, -0.0 == 0.0.
  * Strings and binary compare as unsigned bytes, a proper prefix first (UTF8String.compareTo).
  * A null never satisfies a comparison.
A predicate is (column, lo, lo_strict, hi, hi_strict) with None for a missing bound, the shape Context.filter_scan_where
takes.
"""
import numpy as np


def _compare_floats(a: np.ndarray, b) -> np.ndarray:
    """compareDoubles(a[i], b) in {-1, 0, 1}; a is a float array (float32 or float64), b a scalar of the same width."""
    an = np.isnan(a)
    if np.isnan(b):
        return np.where(an, 0, -1).astype(np.int8)
    out = np.where(a < b, -1, np.where(a > b, 1, 0)).astype(np.int8)
    out[an] = 1
    return out


def _compare_ints(a: np.ndarray, b: int) -> np.ndarray:
    a = a.astype(np.int64)
    return np.where(a < b, -1, np.where(a > b, 1, 0)).astype(np.int8)


def long_to_float32(v: int) -> np.float32:
    """(float) of a long as Java and C cast it: ONE rounding to nearest, ties to even (np.float32(v) rounds through double
    first, which differs for some values beyond 2^53)."""
    a = abs(int(v))
    shift = max(0, a.bit_length() - 24)
    q, r = divmod(a, 1 << shift)
    half = (1 << shift) >> 1
    if shift and (r > half or (r == half and q & 1)):
        q += 1
    m = q << shift  # at most 25 significant bits when q overflowed to 2^24: still a power of two times 2^24, exact in float
    return np.float32(-m if v < 0 else m)


def compare(values: np.ndarray, literal) -> np.ndarray:
    """Spark's comparison of every value of a column with one literal, after type coercion: -1 / 0 / +1 per row."""
    if values.dtype == object:
        if not isinstance(literal, (str, bytes)):
            raise TypeError("a string column takes string literals")
        lit = literal.encode("utf-8") if isinstance(literal, str) else bytes(literal)
        return np.array([(v > lit) - (v < lit) for v in values], dtype=np.int8)
    if isinstance(literal, (str, bytes)):
        raise TypeError("a numeric column takes numeric literals")
    is_long = isinstance(literal, (int, np.integer)) and not isinstance(literal, bool)
    kind = values.dtype
    if kind in (np.int32, np.int64):
        if is_long:
            return _compare_ints(values, int(literal))
        return _compare_floats(values.astype(np.float64), np.float64(literal))  # (double)k, rounded like a C cast
    if kind == np.float32:
        if is_long:
            return _compare_floats(values, long_to_float32(int(literal)))  # the literal is cast to float
        return _compare_floats(values.astype(np.float64), np.float64(literal))
    if kind == np.float64:
        return _compare_floats(values, np.float64(int(literal)) if is_long else np.float64(literal))
    raise TypeError(f"unhandled column type {kind}")


def predicate_mask(columns, predicates, valids=None) -> np.ndarray:
    """Rows where every predicate holds.  columns: {name: numpy array (object arrays of bytes for strings)}; valids:
    {name: bool array} for nullable columns."""
    valids = valids or {}
    n = len(next(iter(columns.values())))
    mask = np.ones(n, dtype=bool)
    for name, lo, lo_strict, hi, hi_strict in predicates:
        v = columns[name]
        if name in valids:
            mask &= np.asarray(valids[name], dtype=bool)
        if lo is not None:
            c = compare(v, lo)
            mask &= (c > 0) if lo_strict else (c >= 0)
        if hi is not None:
            c = compare(v, hi)
            mask &= (c < 0) if hi_strict else (c <= 0)
    return mask
