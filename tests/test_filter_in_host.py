"""CPU tests of the disjunctions on one column: Column.isin and Predicate.__or__, the ctypes arrays they become, the filter
rule's choice of an index for them, and their explain() text."""
import datetime
import decimal

import numpy as np
import pytest

import filter_in_oracle as FI


def test_isin_forms_and_none():
    from hyperspace_b200.session import col

    for p in (col("k").isin(1, 2, None, 3), col("k").isin([1, 2, None, 3]), col("k").isin((1, 2, 3)), col("k").isin({1, 2, 3})):
        assert p.columns == ["k"] and p.conjuncts() == [] and len(p.disjunctions()) == 1
        assert sorted(p.disjunctions()[0].values) == [1, 2, 3]
    arr = np.arange(5, dtype=np.int64)
    a = col("k").isin(arr).disjunctions()[0]
    assert a.values is arr
    assert col("k").isin().disjunctions()[0].values == []


def test_isin_refusals():
    from hyperspace_b200 import log_entry as LE
    from hyperspace_b200.session import col

    with pytest.raises(LE.HyperspaceException, match="mix string and numeric"):
        col("k").isin("a", 1)
    with pytest.raises(LE.HyperspaceException, match="boolean"):
        col("k").isin(True)


def test_or_on_one_column_and_refusals():
    from hyperspace_b200 import log_entry as LE
    from hyperspace_b200.session import col

    p = (col("k") < 10) | (col("k") > 100)
    a = p.disjunctions()[0]
    assert a.column == "k" and a.values == [] and a.ranges == [(None, False, 10, True), (100, True, None, False)]
    q = (p | col("k").isin(50, 51) | col("k").between(60, 70)) & (col("v") > 0.5)
    assert q.columns == ["v", "k"] and q.conjuncts() == [("v", 0.5, True, None, False)]
    b = q.disjunctions()[0]
    assert b.values == [50, 51] and (60, False, 70, False) in b.ranges and len(b.ranges) == 3
    with pytest.raises(LE.HyperspaceException, match="across columns"):
        (col("k") < 1) | (col("v") > 2)
    with pytest.raises(LE.HyperspaceException, match="one column"):
        ((col("k") < 1) & (col("v") > 2)) | (col("k") > 5)
    with pytest.raises(LE.HyperspaceException, match="one range"):
        ((col("k") > 1) & (col("k") > 2)) | (col("k") > 5)


def test_ctypes_arrays_for_each_literal_kind():
    from hyperspace_b200 import _native as N

    assert N.any_values([1, 2, datetime.datetime(1970, 1, 1, 0, 0, 1)])[0] == N.HS_TYPE_INT64
    lt, sc, v = N.any_values([1, 2.5])
    assert lt == N.HS_TYPE_DOUBLE and v.dtype == np.float64 and v.tolist() == [1.0, 2.5]
    lt, sc, v = N.any_values([decimal.Decimal("1.5"), 2, decimal.Decimal("0.125")])
    assert (lt, sc, v.tolist()) == (N.HS_TYPE_DECIMAL, 3, [1500, 2000, 125])
    lt, sc, v = N.any_values(np.array([3, 4], dtype=np.int32))
    assert lt == N.HS_TYPE_INT64 and v.dtype == np.int64
    f = np.array([1.0, np.nan])
    assert N.any_values(f)[2] is f  # no copy, no Python object per value
    arr, n, keep = N._any_array([("s", ["ab", b"", "é"], [(b"x", False, None, False)])])
    a = arr[0]
    assert n == 1 and a.literal_type == N.HS_TYPE_STRING and a.n_values == 3 and a.n_ranges == 1
    offs = np.ctypeslib.as_array((np.ctypeslib.ctypes.c_uint64 * 4).from_address(a.values_offsets))
    assert offs.tolist() == [0, 2, 2, 4]
    assert a.ranges[0].literal_type == N.HS_TYPE_STRING and a.ranges[0].lo_len == 1
    arr, _, _ = N._any_array([("d", [], [(decimal.Decimal("-1.005"), False, decimal.Decimal("1.5"), True)])])
    r = arr[0].ranges[0]
    assert (r.lo_i, r.hi_i, r.scale, r.hi_strict) == (-1005, 1500, 3, 1)
    with pytest.raises(ValueError):
        N._any_array([("x", [], [(1, False, 2.5, False)])])
    assert "hs_filter_scan_any" in N.EXPORTED_SYMBOLS and "hs_bucket_join_any" in N.EXPORTED_SYMBOLS


def test_oracle_follows_in_semantics():
    cols = {"f": np.array([0.0, -0.0, np.nan, 1.0, 2.0]), "i": np.array([1, 2, 3, 4, 5], dtype=np.int32)}
    assert FI.term_mask(cols, ("f", [-0.0, np.nan], [])).tolist() == [True, True, True, False, False]
    assert FI.term_mask(cols, ("i", [2.5, 3.0, None], [(5, False, None, False)])).tolist() == [False, False, True, False, True]
    assert FI.term_mask(cols, ("i", [1], []), {"i": np.array([0, 1, 1, 1, 1], bool)}).tolist() == [False] * 5


def _fabricated(tmp_path, indexed):
    from hyperspace_b200 import log_entry as LE
    from hyperspace_b200 import rules
    from hyperspace_b200.session import DataFrame, HyperspaceSession, RelationNode

    s = HyperspaceSession({"spark.hyperspace.system.path": str(tmp_path / "ix")}).enableHyperspace()
    rel = RelationNode([f"file:{tmp_path}/t"], [(f"file:{tmp_path}/t/a.parquet", 100, 1)],
                       [("k", "long"), ("v1", "long"), ("v2", "double")])
    tracker = LE.FileIdTracker()
    idx_files = [(f"file:{tmp_path}/ix/idx/v__=0/part-00000-x_{b:05d}.c000.parquet", 10, 1) for b in range(2)]
    e = LE.IndexLogEntry(
        name="idx", indexedColumns=indexed, includedColumns=[c for c in ["k", "v1", "v2"] if c not in indexed],
        schema={"type": "struct", "fields": []}, numBuckets=2, derived_properties={"lineage": "false"},
        content=LE.Content.from_leaf_files(idx_files, LE.FileIdTracker()),
        relations=[LE.Relation(rel.root_paths, LE.Content.from_leaf_files(rel.files, tracker), {"type": "struct", "fields": []}, "parquet")],
        signatures=[LE.Signature(LE.INDEX_SIGNATURE_PROVIDER, rules.index_signature(rel))], state="ACTIVE", id=1)
    lm = LE.IndexLogManager(str(tmp_path / "ix" / "idx"))
    lm.write_log(1, e)
    lm.create_latest_stable_log(1)
    return DataFrame(s, rel)


def test_filter_index_rule_takes_isin_on_the_first_indexed_column(tmp_path):
    from hyperspace_b200.session import col

    df = _fabricated(tmp_path, ["k", "v1"])
    assert "Name: idx" in df.filter(col("k").isin(1, 2, 3)).select("k", "v2").explain()
    assert "Name: idx" in df.filter((col("k") < 1) | (col("k") > 9)).select("k").explain()
    assert "Name: idx" in df.filter(((col("k") < 1) | (col("k") > 9)) & (col("v2") > 0)).select("k").explain()
    assert "GpuSourceScan" in df.filter(col("v1").isin(1, 2)).select("k").explain()   # a later indexed column


def test_explain_shows_the_terms(tmp_path):
    from hyperspace_b200.session import col

    df = _fabricated(tmp_path, ["k"])
    plan = df.filter(col("k").isin(list(range(1000)))).select("k").explain()
    assert "Name: idx" in plan and "where=(k IN (0, 1, 2, ... 997 more))" in plan
    plan = df.filter((col("k") < 10) | col("k").between(20, 30)).select("k").explain()
    assert "where=(k < 10 OR (k >= 20 AND k <= 30))" in plan
    plan = df.filter(col("v1").isin("a")).select("k").explain()
    assert plan.startswith("GpuSourceScan") and "where=(v1 IN ('a'))" in plan
