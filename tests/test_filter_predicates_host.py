"""CPU tests of multi-column filter predicates: the numpy oracle's Spark semantics on hand-written cases, the comparison
terms a Predicate records and their conjunction, FilterIndexRule on a conjunction, and the new C entry point's export."""
import math
import os

import numpy as np

import filter_oracle as F


def _sel(values, *pred, valid=None):
    cols = {"x": values}
    return np.flatnonzero(F.predicate_mask(cols, [("x",) + pred], {"x": valid} if valid is not None else None)).tolist()


def test_nan_is_greatest_and_equals_itself():
    x = np.array([1.0, np.nan, np.inf, -np.inf, 0.5], dtype=np.float64)
    assert _sel(x, 1.0, False, None, False) == [0, 1, 2]          # x >= 1.0 selects the NaN row
    assert _sel(x, np.nan, False, np.nan, False) == [1]           # x == NaN
    assert _sel(x, np.nan, True, None, False) == []               # nothing is above NaN
    assert _sel(x, None, False, np.inf, False) == [0, 2, 3, 4]    # NaN > +inf
    assert _sel(x, None, False, np.nan, True) == [0, 2, 3, 4]     # x < NaN: every number


def test_negative_zero_equals_zero():
    x = np.array([-0.0, 0.0, -1e-300, 5e-324], dtype=np.float64)
    assert _sel(x, 0.0, False, 0.0, False) == [0, 1]
    assert _sel(x, -0.0, True, None, False) == [3]                # x > -0.0 excludes 0.0 and -0.0
    assert _sel(x, None, False, 0.0, True) == [2]                 # x < 0.0 excludes -0.0
    f = x.astype(np.float32)                                      # -1e-300 and 5e-324 become -0.0 / 0.0 in float
    assert _sel(f, 0.0, False, 0.0, False) == [0, 1, 2, 3]


def test_float_column_against_double_and_long_literals():
    f = np.array([0.1, 0.2, 16777216.0], dtype=np.float32)
    # f32 > 0.1 compares (double)f with 0.1: float(0.1f) = 0.100000001490116... is above the double 0.1
    assert _sel(f, 0.1, True, None, False) == [0, 1, 2]
    assert _sel(f, float(np.float32(0.1)), True, None, False) == [1, 2]
    # a long literal is cast to float: 16777217 -> 16777216.0f
    assert _sel(f, 16777217, False, None, False) == [2]
    assert _sel(f, 16777217.0, False, None, False) == []          # a double literal is not rounded


def test_integer_column_against_a_double_literal():
    k = np.array([0, 1, 2, 3, -1, -2], dtype=np.int64)
    assert _sel(k, 1.5, True, None, False) == [2, 3]              # k > 1.5 is k >= 2
    assert _sel(k, None, False, -1.5, False) == [5]
    assert _sel(k, 1.5, False, 1.5, False) == []                  # k == 1.5 matches nothing
    assert _sel(k.astype(np.int32), 0.5, False, 2.5, False) == [1, 2]


def test_int64_near_two_to_the_53():
    t = 2**53
    k = np.array([t - 1, t, t + 1, t + 2, t + 3], dtype=np.int64)
    assert _sel(k, t + 1, False, None, False) == [2, 3, 4]        # long literal: exact
    # double literal: (double)(2^53 + 1) rounds to 2^53, (double)(2^53 + 3) to 2^53 + 4
    assert _sel(k, float(t), True, None, False) == [3, 4]
    assert _sel(k, float(t), False, float(t), False) == [1, 2]
    assert _sel(k, None, False, float(t + 2), True) == [0, 1, 2]
    big = np.array([2**60 - 1, 2**60, 2**63 - 1], dtype=np.int64)
    assert _sel(big, float(2**60), False, float(2**60), False) == [0, 1]  # 2^60 - 1 rounds up to 2^60
    assert _sel(big, 1e30, False, None, False) == []
    assert _sel(big, None, False, 1e30, False) == [0, 1, 2]


def test_integer_literal_outside_the_column_range():
    k = np.array([np.iinfo(np.int32).min, 0, np.iinfo(np.int32).max], dtype=np.int32)
    assert _sel(k, 2**40, False, None, False) == []
    assert _sel(k, -(2**40), False, None, False) == [0, 1, 2]
    assert _sel(k, None, False, 2**62, True) == [0, 1, 2]


def test_nulls_never_match():
    k = np.array([5, 5, 7], dtype=np.int64)
    valid = np.array([True, False, True])
    assert _sel(k, 5, False, None, False, valid=valid) == [0, 2]
    s = np.array([b"a", b"", b"b"], dtype=object)
    assert _sel(s, "", False, None, False, valid=valid) == [0, 2]


def test_strings_compare_as_unsigned_bytes_with_strict_bounds():
    s = np.array([b"abc", b"abd", b"ab", "é".encode(), b"\xff"], dtype=object)
    assert _sel(s, "abc", True, None, False) == [1, 3, 4]
    assert _sel(s, None, False, "abc", True) == [2]
    assert _sel(s, "ab", False, b"\xc3", False) == [0, 1, 2]


def test_conjunction_of_several_columns():
    cols = {"k": np.arange(10, dtype=np.int64), "v": np.arange(10, dtype=np.float64)[::-1].copy()}
    m = F.predicate_mask(cols, [("k", 2, False, None, False), ("v", None, False, 4.5, False), ("k", None, False, 8, True)])
    assert np.flatnonzero(m).tolist() == [5, 6, 7]


def test_predicate_records_terms_and_keeps_bounds():
    from hyperspace_b200.session import col

    p = col("k").between(100, 300) & (col("v1") >= 500) & (col("v2") > 0.5)
    assert p.bounds == {"k": (100, 300), "v1": (500, None), "v2": (1, None)}    # unchanged integer rounding
    assert p.terms == [("k", ">=", 100), ("k", "<=", 300), ("v1", ">=", 500), ("v2", ">", 0.5)]
    assert p.conjuncts() == [("k", 100, False, None, False), ("k", None, False, 300, False), ("v1", 500, False, None, False),
                             ("v2", 0.5, True, None, False)]
    assert (col("x") < 2.5).conjuncts() == [("x", None, False, 2.5, True)]
    assert (col("q") == "facebook").conjuncts() == [("q", "facebook", False, "facebook", False)]
    assert (col("q") > "abc").conjuncts() == [("q", "abc", True, None, False)]
    nan = (col("d") >= math.nan).conjuncts()[0]                                   # non-finite literals are kept as written
    assert nan[0] == "d" and math.isnan(nan[1]) and (col("d") <= math.inf).terms == [("d", "<=", math.inf)]


def test_filter_resolves_term_column_names(tmp_path):
    import pyarrow as pa
    import pyarrow.parquet as pq

    from hyperspace_b200.session import HyperspaceSession, col

    pq.write_table(pa.table({"Key": pa.array([1], pa.int64()), "Val": pa.array([1.0])}), str(tmp_path / "a.parquet"))
    df = HyperspaceSession().read.parquet(str(tmp_path))
    f = df.filter((col("key") >= 1) & (col("VAL") < 2.0)).plan
    assert f.predicate.terms == [("Key", ">=", 1), ("Val", "<", 2.0)] and set(f.predicate.bounds) == {"Key", "Val"}


def test_filter_index_rule_accepts_a_conjunction(tmp_path):
    """FilterIndexRule: the first indexed column in the filter and every column covered -> the index is used for a conjunction
    over several columns; a filter without the first indexed column stays a source scan."""
    from hyperspace_b200 import log_entry as LE
    from hyperspace_b200 import rules
    from hyperspace_b200.session import DataFrame, HyperspaceSession, RelationNode, col

    s = HyperspaceSession({"spark.hyperspace.system.path": str(tmp_path / "ix")}).enableHyperspace()
    rel = RelationNode([f"file:{tmp_path}/t"], [(f"file:{tmp_path}/t/a.parquet", 100, 1)],
                       [("k", "long"), ("v1", "long"), ("v2", "double"), ("v3", "integer")])
    tracker = LE.FileIdTracker()
    idx_files = [(f"file:{tmp_path}/ix/idx/v__=0/part-00000-x_{b:05d}.c000.parquet", 10, 1) for b in range(2)]
    e = LE.IndexLogEntry(
        name="idx", indexedColumns=["k"], includedColumns=["v1", "v2"], schema={"type": "struct", "fields": []}, numBuckets=2,
        derived_properties={"lineage": "false"}, content=LE.Content.from_leaf_files(idx_files, LE.FileIdTracker()),
        relations=[LE.Relation(rel.root_paths, LE.Content.from_leaf_files(rel.files, tracker), {"type": "struct", "fields": []}, "parquet")],
        signatures=[LE.Signature(LE.INDEX_SIGNATURE_PROVIDER, rules.index_signature(rel))], state="ACTIVE", id=1)
    lm = LE.IndexLogManager(str(tmp_path / "ix" / "idx"))
    lm.write_log(1, e)
    lm.create_latest_stable_log(1)
    df = DataFrame(s, rel)
    assert "Name: idx" in df.filter(col("k").between(100, 300) & (col("v1") >= 500)).select("k", "v2").explain()
    assert "Name: idx" in df.filter((col("v1") >= 500) & (col("k") > 1.5) & (col("v2") < 0.5)).select("k").explain()
    assert "GpuSourceScan" in df.filter((col("v1") >= 500) & (col("v2") < 0.5)).select("k").explain()   # no first column
    assert "GpuSourceScan" in df.filter((col("k") >= 1) & (col("v3") < 5)).select("k").explain()       # v3 not covered


def test_filter_scan_where_is_exported():
    from hyperspace_b200 import _native as N

    assert "hs_filter_scan_where" in N.EXPORTED_SYMBOLS
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    with open(os.path.join(root, "include", "hs_gpu.h")) as f:
        header = f.read()
    assert "int hs_filter_scan_where(" in header and "} hs_predicate;" in header
    if os.path.exists(N.LIB_PATH):
        import ctypes

        assert hasattr(ctypes.CDLL(N.LIB_PATH), "hs_filter_scan_where")


def test_literal_types_of_predicates():
    import pytest

    from hyperspace_b200 import _native as N

    assert N._literal_type(1, None) == N.HS_TYPE_INT64
    assert N._literal_type(None, 2.5) == N.HS_TYPE_DOUBLE
    assert N._literal_type("a", b"b") == N.HS_TYPE_STRING
    for bad in ((True, None), (None, None), ("a", 1), (2**63, None)):
        with pytest.raises(ValueError):
            N._literal_type(*bad)


def test_conjunction_with_a_predicate_built_from_bounds_keeps_both():
    from hyperspace_b200.session import Predicate, col

    p = Predicate({"k": (1, 5)}) & (col("v") > 0.5)
    assert p.conjuncts() == [("k", 1, False, None, False), ("k", None, False, 5, False), ("v", 0.5, True, None, False)]
    q = (col("v") > 0.5) & Predicate({"k": (None, 7)})
    assert q.conjuncts() == [("v", 0.5, True, None, False), ("k", None, False, 7, False)]
    assert Predicate({"k": (2, None)}).conjuncts() == [("k", 2, False, None, False)]


def test_long_literal_is_cast_to_float_with_one_rounding():
    v = 2**60 + 2**36 + 1                      # np.float32(v) goes through double and lands on 2^60
    assert F.long_to_float32(v) == np.float32(2.0**60 + 2.0**37)
    assert F.long_to_float32(-v) == -np.float32(2.0**60 + 2.0**37)
    assert F.long_to_float32(16777217) == np.float32(16777216.0) and F.long_to_float32(16777219) == np.float32(16777220.0)
    f = np.array([2.0**60, 2.0**60 + 2.0**37], dtype=np.float32)
    assert _sel(f, v, False, None, False) == [1]
