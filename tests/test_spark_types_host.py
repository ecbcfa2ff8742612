"""Host-side tests of Spark timestamp and decimal columns: the INT96 -> micros restatement against pyarrow, the Spark type
names the session reads from Parquet footers, and the exact decimal comparison behind literal bounds."""
import datetime
import decimal
import io
import os
import shutil
import subprocess
from fractions import Fraction

import numpy as np
import pyarrow as pa
import pyarrow.parquet as pq
import pytest

import spark_types_oracle as S
from hyperspace_b200 import _native as N
from hyperspace_b200 import session as SE

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _image(table, **kw):
    sink = io.BytesIO()
    pq.write_table(table, sink, **kw)
    return sink.getvalue()


def _ns(dt: datetime.datetime) -> int:
    return (dt.replace(tzinfo=datetime.timezone.utc) - datetime.datetime(1970, 1, 1, tzinfo=datetime.timezone.utc)) \
        // datetime.timedelta(microseconds=1) * 1000


CASES_NS = [
    _ns(datetime.datetime(1900, 1, 1)),                     # the first instant Spark 3.1 loads from INT96
    _ns(datetime.datetime(1900, 1, 1)) + 999,               # truncation inside the first microsecond
    _ns(datetime.datetime(1950, 6, 30, 12, 0, 0, 123456)) + 789,  # before the epoch
    0,                                                      # the epoch
    -1,                                                     # the last nanosecond before it
    _ns(datetime.datetime(1999, 12, 31)) + 86_400 * 10**9 - 1,  # the last nanosecond of a day
    _ns(datetime.datetime(2262, 4, 11)),
]


def test_int96_restatement_matches_pyarrow():
    t = pa.table({"ts": pa.array(CASES_NS, pa.timestamp("ns"))})
    sink = io.BytesIO()
    pq.write_table(t, sink, use_deprecated_int96_timestamps=True)
    back = pq.read_table(io.BytesIO(sink.getvalue()), coerce_int96_timestamp_unit="us").column("ts")
    got, _ = S.spark_int64(back)
    want = [S.int96_to_micros(*S.int96_of_nanos(ns)) for ns in CASES_NS]
    assert got.tolist() == want
    # pre-epoch values truncate toward zero inside the day's nanos, which are never negative
    assert S.int96_of_nanos(-1) == (S.JULIAN_DAY_OF_EPOCH - 1, 86_400 * 10**9 - 1)
    assert S.int96_to_micros(*S.int96_of_nanos(_ns(datetime.datetime(1900, 1, 1)))) == S.MICROS_1900


def _schema_of(table, **kw):
    sink = io.BytesIO()
    pq.write_table(table, sink, **kw)
    path = io.BytesIO(sink.getvalue())
    return [(f.name, SE.spark_type_of_arrow(f.type)) for f in pq.ParquetFile(path).schema_arrow]


@pytest.mark.parametrize("kw", [dict(use_deprecated_int96_timestamps=True), dict(coerce_timestamps="ms"),
                                dict(coerce_timestamps="us"), dict(version="2.6", coerce_timestamps=None)])
def test_session_names_timestamps(kw):
    t = pa.table({"t": pa.array([1000, 2000], pa.timestamp("ns" if "version" in kw else "us")), "u": pa.array([1, 1], pa.int64())})
    assert _schema_of(t, **kw) == [("t", "timestamp"), ("u", "long")]


@pytest.mark.parametrize("as_int", [True, False])
def test_session_names_decimals(as_int):
    t = pa.table({"a": pa.array([decimal.Decimal("1.25")], pa.decimal128(9, 2)),
                  "b": pa.array([decimal.Decimal("-3.5")], pa.decimal128(12, 1)),
                  "c": pa.array([decimal.Decimal("1")], pa.decimal128(18, 0)),
                  "d": pa.array([decimal.Decimal("1")], pa.decimal128(20, 0))})
    assert _schema_of(t, store_decimal_as_integer=as_int) == [
        ("a", "decimal(9,2)"), ("b", "decimal(12,1)"), ("c", "decimal(18,0)"), ("d", "decimal(20,0)")]


def test_spark_values_of_results():
    ts = SE.spark_values(np.array([0, 1_500_000], np.int64), "timestamp")
    assert ts.dtype == np.dtype("datetime64[us]") and ts[1] == np.datetime64("1970-01-01T00:00:01.5")
    d = SE.spark_values(np.array([-125, 7], np.int32), "decimal(9,2)")
    assert d.tolist() == [decimal.Decimal("-1.25"), decimal.Decimal("0.07")]
    assert SE.spark_values(np.array([3], np.int64), "long").tolist() == [3]


def test_literals_become_predicate_fields():
    preds, n = N._predicate_array([("c", decimal.Decimal("1.50"), True, decimal.Decimal("2.25"), False)])
    assert n == 1 and preds[0].literal_type == N.HS_TYPE_DECIMAL
    assert (preds[0].lo_i, preds[0].hi_i, preds[0].scale) == (150, 225, 2)
    # bounds of two scales, or a decimal beside an int / float, are two comparisons
    preds, n = N._predicate_array([("c", decimal.Decimal("1.5"), False, decimal.Decimal("2.25"), False)])
    assert n == 2 and (preds[0].lo_i, preds[0].scale, preds[1].hi_i, preds[1].scale) == (15, 1, 225, 2)
    preds, n = N._predicate_array([("c", 1, False, decimal.Decimal("2.25"), False)])
    assert n == 2 and preds[0].literal_type == N.HS_TYPE_INT64 and preds[1].literal_type == N.HS_TYPE_DECIMAL
    preds, n = N._predicate_array([("t", datetime.datetime(1970, 1, 1, 0, 0, 1), False, None, False)])
    assert n == 1 and preds[0].literal_type == N.HS_TYPE_INT64 and preds[0].lo_i == 1_000_000
    assert N.timestamp_micros(datetime.datetime(1969, 12, 31, 23, 59, 59, 999999)) == -1
    assert N.decimal_unscaled(decimal.Decimal("1E+3")) == (1000, 0)
    with pytest.raises(ValueError):
        N.decimal_unscaled(decimal.Decimal("0.1234567890123456789012"))
    # the bounds the plan layer picks an index by
    p = SE.col("t") >= datetime.datetime(1970, 1, 1, 0, 0, 2)
    assert p.bounds == {"t": (2_000_000, None)}
    assert (SE.col("d") > decimal.Decimal("1.5")).bounds == {"d": (2, None)}


@pytest.fixture(scope="module")
def native(tmp_path_factory):
    """tests/native/spark_types.cu: the engine's own source_type_of, footer reader and compare_scaled, built as host code."""
    if shutil.which("nvcc") is None:
        pytest.skip("nvcc not on PATH")
    exe = str(tmp_path_factory.mktemp("spark_types") / "spark_types")
    subprocess.check_call(["nvcc", "-std=c++17", "-O1", "-Wno-deprecated-gpu-targets", "-I", os.path.join(ROOT, "include"), "-o", exe,
                           os.path.join(ROOT, "tests", "native", "spark_types.cu")])
    return exe


def _footer(native, tmp_path, name, image):
    path = tmp_path / name
    path.write_bytes(image)
    out = {}
    for line in subprocess.check_output([native, "footer", str(path)], text=True).splitlines():
        col, rest = line.split()[1], line.split(" -> ")[1]
        out[col] = rest if rest.startswith("refused") else dict(kv.split("=") for kv in rest.split())
    return out


def test_source_types_of_every_row_of_the_table(native, tmp_path):
    """Every row of the type table through the engine's footer reader and source_type_of: storage type, conversion,
    the leaf the index file declares and its Spark name -- or the refusal."""
    ts = pa.array([0, 1000], pa.timestamp("us"))
    files = {
        "int96": _image(pa.table({"c": ts}), use_deprecated_int96_timestamps=True),
        "micros": _image(pa.table({"c": ts}), coerce_timestamps="us"),      # logical type only (not adjusted to UTC)
        "millis": _image(pa.table({"c": ts}), coerce_timestamps="ms"),
        "nanos": _image(pa.table({"c": pa.array([1], pa.timestamp("ns"))}), version="2.6", coerce_timestamps=None),
        "d9_int32": _image(pa.table({"c": pa.array([decimal.Decimal("1.25")], pa.decimal128(9, 2))}), store_decimal_as_integer=True),
        "d9_flba": _image(pa.table({"c": pa.array([decimal.Decimal("1.25")], pa.decimal128(9, 2))})),
        "d12_int64": _image(pa.table({"c": pa.array([decimal.Decimal("1.25")], pa.decimal128(12, 2))}), store_decimal_as_integer=True),
        "d18_flba": _image(pa.table({"c": pa.array([decimal.Decimal("1.25")], pa.decimal128(18, 2))})),
        "d19": _image(pa.table({"c": pa.array([decimal.Decimal("1")], pa.decimal128(19, 0))})),
    }
    got = {k: _footer(native, tmp_path, k + ".parquet", im)["c"] for k, im in files.items()}
    ts_row = dict(hs_type="1", type="2", converted="10", precision="-1", scale="-1", spark="timestamp")
    assert got["int96"] == dict(ts_row, conv="1")
    assert got["micros"] == dict(ts_row, conv="0")
    assert got["millis"] == dict(ts_row, conv="2")
    assert got["nanos"].startswith("refused code=-6") and "NANOS" in got["nanos"]
    assert got["d9_int32"] == dict(hs_type="0", conv="0", type="1", converted="5", precision="9", scale="2", spark="decimal(9,2)")
    assert got["d9_flba"] == dict(got["d9_int32"], conv="3")
    assert got["d12_int64"] == dict(hs_type="1", conv="0", type="2", converted="5", precision="12", scale="2", spark="decimal(12,2)")
    assert got["d18_flba"] == dict(hs_type="1", conv="3", type="2", converted="5", precision="18", scale="2", spark="decimal(18,2)")
    assert got["d19"].startswith("refused code=-6") and "decimal(19,0)" in got["d19"]
    # what pyarrow does not write: an INT64 decimal(9,2), FLBA lengths of 5 and 16, a decimal with only its logical type,
    # a BYTE_ARRAY decimal
    hand = {
        "d9_int64": S.decimal_file(2, [1, -5], 9, 2),
        "d9_flba5": S.decimal_file(S.FIXED_LEN_BYTE_ARRAY, [1, -5], 9, 2, length=5),
        "d18_flba16": S.decimal_file(S.FIXED_LEN_BYTE_ARRAY, [1, -5], 18, 3, length=16),
        "d_logical": S.decimal_file(1, [1, -5], 7, 3, logical_only=True),
    }
    got = {k: _footer(native, tmp_path, k + ".parquet", im)["d"] for k, im in hand.items()}
    assert got["d9_int64"] == dict(hs_type="0", conv="4", type="1", converted="5", precision="9", scale="2", spark="decimal(9,2)")
    assert got["d9_flba5"] == dict(got["d9_int64"], conv="3")
    assert got["d18_flba16"] == dict(hs_type="1", conv="3", type="2", converted="5", precision="18", scale="3", spark="decimal(18,3)")
    assert got["d_logical"] == dict(hs_type="0", conv="0", type="1", converted="5", precision="7", scale="3", spark="decimal(7,3)")
    import parquet_shapes as P
    image = S.write_shapes_file(P.FileSpec([P.Col("b", P.BYTE_ARRAY, False, [P.Chunk([P.Page(rows=1, values=[b"\x01"])])])]), {})
    image = S.annotate_leaf(image, "b", P.BYTE_ARRAY, False, converted=S.CT_DECIMAL, precision=5, scale=1)
    got = _footer(native, tmp_path, "bytes.parquet", image)["b"]
    assert got.startswith("refused code=-6") and "BYTE_ARRAY" in got


def test_compare_scaled_is_exact(native):
    """api.cu's comparison of a / 10^sa with b / 10^sb (the engine's code, built for the host) against exact fractions,
    including the 128-bit products and the scale differences past 10^19."""
    lines = subprocess.check_output([native, "compare"], text=True).split("\n")
    n = 0
    for line in lines:
        if not line:
            continue
        a, sa, b, sb, r = map(int, line.split())
        fa, fb = Fraction(a, 10**sa), Fraction(b, 10**sb)
        assert r == (fa > fb) - (fa < fb), line
        n += 1
    assert n == 14 * 14 * 4 * 8


@pytest.mark.parametrize("col_scale", [0, 2])
@pytest.mark.parametrize("lit_scale", [0, 1, 2, 4])
def test_decimal_bounds_brute_force(native, col_scale, lit_scale):
    """Over small unscaled ranges, the column values the engine's comparison keeps for each operator are exactly those
    at or past the literal's ceiling / floor in the column's scale, with the right strictness -- which is what the binary
    search over the encoded domain returns as the range's bound."""
    out = subprocess.check_output([native, "grid", str(col_scale), str(lit_scale)], text=True)
    cmp = {}
    for line in out.splitlines():
        v, lit, r = map(int, line.split())
        cmp[(v, lit)] = r
    domain = range(-300, 301)
    for lit in range(-250, 251, 7):
        q = Fraction(lit, 10**lit_scale) * 10**col_scale  # the literal in the column's units
        for strict in (False, True):
            lo_ok = [v for v in domain if (cmp[(v, lit)] > 0 if strict else cmp[(v, lit)] >= 0)]
            hi_ok = [v for v in domain if (cmp[(v, lit)] < 0 if strict else cmp[(v, lit)] <= 0)]
            want_lo = (q.__floor__() + 1) if strict else q.__ceil__()
            want_hi = (q.__ceil__() - 1) if strict else q.__floor__()
            assert lo_ok == list(range(max(want_lo, -300), 301))
            assert hi_ok == list(range(-300, min(want_hi, 300) + 1))
