"""Spark's values of timestamp and decimal columns, restated for the oracle.

Spark hashes, sorts and compares a TimestampType as its int64 microseconds since the epoch and a DecimalType of precision
<= 18 as its unscaled value, hashed with hashLong at every precision (Murmur3Hash).  These helpers turn pyarrow arrays
into those int64 values, so that the oracle's bucket ids and sort order (which hash an int64 column with hashLong) are
Spark's.  pyarrow reads INT96 with coerce_int96_timestamp_unit="us".

It also builds the source files pyarrow does not write, with tests/parquet_shapes.py's writer: INT96 in parquet-mr's
shape, INT64-stored decimal(p <= 9), FIXED_LEN_BYTE_ARRAY of any length, a decimal with a logical type only.
"""
import decimal
import struct
from unittest import mock

import numpy as np
import pyarrow as pa
import pyarrow.compute as pc

JULIAN_DAY_OF_EPOCH = 2440588
MICROS_PER_DAY = 86_400_000_000
MICROS_1900 = -2_208_988_800_000_000  # 1900-01-01T00:00:00Z


def int96_to_micros(julian_day: int, nanos_of_day: int) -> int:
    """DateTimeUtils.fromJulianDay: (day - 2440588) * MICROS_PER_DAY + nanos / 1000, the division truncating."""
    q = abs(nanos_of_day) // 1000
    return (julian_day - JULIAN_DAY_OF_EPOCH) * MICROS_PER_DAY + (q if nanos_of_day >= 0 else -q)


def int96_of_nanos(ns: int):
    """(Julian day, nanos of day) the way parquet writers store a timestamp of `ns` nanoseconds since the epoch."""
    day, nanos = divmod(ns, MICROS_PER_DAY * 1000)
    return day + JULIAN_DAY_OF_EPOCH, nanos


def spark_int64(arr) -> tuple:
    """(int64 values with nulls as 0, validity or None) of a pyarrow timestamp / decimal / integer array."""
    if isinstance(arr, pa.ChunkedArray):
        arr = arr.combine_chunks()
    valid = np.asarray(arr.is_valid()) if arr.null_count else None
    t = arr.type
    if pa.types.is_timestamp(t):
        vals = pc.cast(arr, pa.timestamp("us", tz=t.tz)).cast(pa.int64()).fill_null(0)
        return np.asarray(vals).astype(np.int64), valid
    if pa.types.is_decimal(t):
        out = np.zeros(len(arr), dtype=np.int64)
        for i, v in enumerate(arr.to_pylist()):
            if v is not None:
                out[i] = int(v.scaleb(t.scale).to_integral_exact())
        return out, valid
    return np.asarray(arr.fill_null(0)).astype(np.int64), valid


def unscaled(v: decimal.Decimal, scale: int) -> int:
    return int(v.scaleb(scale).to_integral_exact())


def int96_bytes(micros) -> np.ndarray:
    """12-byte INT96 values (8 B little-endian nanos of day, 4 B Julian day) of timestamps given in micros."""
    out = np.zeros(len(micros), dtype=[("nanos", "<i8"), ("day", "<i4")])
    day, rem = np.divmod(np.asarray(micros, dtype=np.int64), MICROS_PER_DAY)
    out["nanos"], out["day"] = rem * 1000, day + JULIAN_DAY_OF_EPOCH
    return out.view("V12")


def flba_bytes(unscaled, length: int) -> np.ndarray:
    """Big-endian two's complement FIXED_LEN_BYTE_ARRAY values of `length` bytes."""
    return np.array([int(u).to_bytes(length, "big", signed=True) for u in unscaled], dtype=f"V{length}")


def write_shapes_file(spec, ptype_widths) -> bytes:
    """parquet_shapes.write_file for physical types its writer has no width for: ptype_widths {ptype: bytes per value}."""
    import parquet_shapes as P

    with mock.patch.dict(P.DTYPE, {t: np.dtype(f"V{w}") for t, w in ptype_widths.items()}):
        return P.write_file(spec)


def annotate_leaf(image: bytes, name: str, ptype: int, optional: bool, type_length=None, converted=None, precision=None,
                  scale=None, logical_decimal=None) -> bytes:
    """The file with the schema element of leaf `name` re-serialised with a type length, a converted type (+ precision /
    scale) and / or a LogicalType DECIMAL (precision, scale) -- what parquet_shapes' writer leaves out."""
    import parquet_shapes as P

    def element(extra: bool) -> bytes:
        w = P.ThriftWriter().elem_begin().i32(1, ptype)
        if extra and type_length is not None:
            w.i32(2, type_length)
        w.i32(3, 1 if optional else 0).binary(4, name.encode())
        if extra and converted is not None:
            w.i32(6, converted)
            if scale is not None:
                w.i32(7, scale)
            if precision is not None:
                w.i32(8, precision)
        if extra and logical_decimal is not None:
            w.begin(10).begin(5).i32(1, logical_decimal[1]).i32(2, logical_decimal[0]).end().end()
        return bytes(w.end().b)

    flen = struct.unpack("<I", image[-8:-4])[0]
    body, footer = image[:-8 - flen], image[-8 - flen:-8]
    old, new = element(False), element(True)
    assert footer.count(old) == 1, name
    footer = footer.replace(old, new)
    return body + footer + struct.pack("<I", len(footer)) + b"PAR1"


# ---- hand-built source files (parquet_shapes' writer) -----------------------------------------------------------------
INT96, FIXED_LEN_BYTE_ARRAY, CT_DECIMAL = 3, 7, 5


def _v_column(n, rows_per_group):
    import parquet_shapes as P

    v = np.arange(n, dtype=np.int64)
    chunks, r = [], 0
    for g in rows_per_group:
        chunks.append(P.Chunk([P.Page(rows=g, values=v[r:r + g])]))
        r += g
    return P.Col("v", P.INT64, False, chunks), v


def parquet_mr_int96(seed=7):
    """An INT96 column in parquet-mr's shape (Spark 3.1's default timestamp output): v1 pages, a PLAIN_DICTIONARY
    dictionary page and data pages with page statistics, then -- the dictionary grown too large -- a PLAIN fallback page;
    a second row group that is PLAIN from the start.  Returns (image, expected micros of column ts, column v)."""
    import parquet_shapes as P

    rng = np.random.default_rng(seed)
    dict_micros = rng.integers(MICROS_1900, 4_102_444_800_000_000, 300)
    dict_micros[:3] = [MICROS_1900, -1, 0]  # 1900-01-01 exactly, the last micro before the epoch, the epoch
    idx = [rng.integers(0, 300, 3000), rng.integers(0, 300, 1000)]
    fallback = rng.integers(MICROS_1900, 4_102_444_800_000_000, 1500)
    second = rng.integers(MICROS_1900, 4_102_444_800_000_000, 2500)
    pages = [P.Page(rows=len(i), enc=P.PLAIN_DICTIONARY, idx=[P.packed(i)], stats=True) for i in idx]
    pages.append(P.Page(rows=len(fallback), enc=P.PLAIN, values=int96_bytes(fallback), stats=True))
    ts = P.Col("ts", INT96, False, [P.Chunk(pages, dict=int96_bytes(dict_micros), dict_enc=P.PLAIN_DICTIONARY),
                                    P.Chunk([P.Page(rows=len(second), enc=P.PLAIN, values=int96_bytes(second))])])
    vcol, v = _v_column(8000, [5500, 2500])
    image = write_shapes_file(P.FileSpec([ts, vcol]), {INT96: 12})
    return image, np.concatenate([dict_micros[idx[0]], dict_micros[idx[1]], fallback, second]), v


def decimal_file(ptype, unscaled, precision, scale, length=None, optional=False, logical_only=False, rows_per_page=None):
    """A column d of decimal(precision, scale) stored as INT32 / INT64 / FIXED_LEN_BYTE_ARRAY(length) PLAIN pages
    (converted type DECIMAL, or only the LogicalType when logical_only), and a column v.  Returns the image."""
    import parquet_shapes as P

    u = np.asarray(unscaled, dtype=np.int64)
    n = len(u)
    per = rows_per_page or n
    if ptype == FIXED_LEN_BYTE_ARRAY:
        vals, widths = flba_bytes(u, length), {FIXED_LEN_BYTE_ARRAY: length}
    else:
        vals, widths = u.astype(np.int32 if ptype == P.INT32 else np.int64), {}
    pages = [P.Page(rows=min(per, n - r), values=vals[r:r + per]) for r in range(0, n, per)]
    d = P.Col("d", ptype, optional, [P.Chunk(pages)])
    vcol, _ = _v_column(n, [n])
    image = write_shapes_file(P.FileSpec([d, vcol]), widths)
    if logical_only:
        return annotate_leaf(image, "d", ptype, optional, type_length=length, logical_decimal=(precision, scale))
    return annotate_leaf(image, "d", ptype, optional, type_length=length, converted=CT_DECIMAL, precision=precision, scale=scale)
