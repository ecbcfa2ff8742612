"""Left semi / left anti bucket joins without a GPU: hand-written cases that pin tests/join_exists_oracle.py (null keys on
either side, partial nulls in a composite key, duplicates, empty right buckets, filters), DataFrame.join's join types,
the output columns and explain() of such joins, and index selection for a right side that is only probed."""
import numpy as np
import pytest

import join_exists_oracle as JE
from hyperspace_b200.log_entry import HyperspaceException
from oracle import oracle as O
from test_join_rule_composite_host import FIVE, _fixture, _uses


def _both(L, R, nb, lkeys, rkeys, **kw):
    return (JE.exists_join(L, R, nb, lkeys, rkeys, "semi", **kw).tolist(),
            JE.exists_join(L, R, nb, lkeys, rkeys, "anti", **kw).tolist())


def test_null_left_key_never_matches_zero_or_empty_string():
    # nulls decode to 0 / the empty string: a null left key must not match a right 0 or "", and an anti join keeps it
    L = {"k": np.array([0, 5, 0, 7], dtype=np.int64), "lid": np.arange(4)}
    R = {"k": np.array([0, 5, 9, 7], dtype=np.int64)}
    lv, rv = {"k": np.array([False, True, True, True])}, {"k": np.array([True, True, True, False])}
    # one bucket, sorted nulls first: rows 0 (null), 2 (0), 1 (5), 3 (7); the right 7 is null and matches nothing
    assert _both(L, R, 1, ["k"], ["k"], left_valids=lv, right_valids=rv) == ([2, 1], [0, 3])
    Ls = {"s": np.array([b"", b"a", b"", b"b"], dtype=object)}
    Rs = {"s": np.array([b"", b"a"], dtype=object)}
    assert _both(Ls, Rs, 1, ["s"], ["s"], left_valids={"s": lv["k"]}) == ([2, 1], [0, 3])
    # no nulls on the left: the same rows match, and nothing null is kept by anti
    assert _both(L, R, 1, ["k"], ["k"], right_valids=rv) == ([0, 2, 1], [3])


def test_partial_nulls_in_a_three_column_key():
    L = {"a": np.array([1, 1, 1, 2, 1]), "b": np.array([2, 2, 0, 2, 2]), "c": np.array([3, 0, 3, 2, 3])}
    lv = {"b": np.array([True, True, False, True, True]), "c": np.array([True, False, True, True, True])}
    R = {"a": np.array([1, 1, 2]), "b": np.array([2, 2, 0]), "c": np.array([3, 3, 2])}
    rv = {"b": np.array([True, True, False])}
    # sorted: (1, null, 3) row 2, (1, 2, null) row 1, (1, 2, 3) rows 0 and 4, (2, 2, 2) row 3 -- whose right twin has a
    # null b, so it matches nothing
    assert _both(L, R, 1, ["a", "b", "c"], ["a", "b", "c"], left_valids=lv, right_valids=rv) == ([0, 4], [2, 1, 3])


def test_duplicates_on_both_sides_give_each_left_row_once():
    L = {"k": np.array([3, 3, 4, 3], dtype=np.int32)}
    R = {"k": np.array([3, 3, 3, 5], dtype=np.int32)}
    assert _both(L, R, 1, ["k"], ["k"]) == ([0, 1, 3], [2])


def test_empty_right_buckets():
    nb = 4
    L = {"k": np.arange(40, dtype=np.int64) % 20}
    R = {"k": np.array([6, 6], dtype=np.int64)}
    bucket = O.np_pmod(O.np_hash_long(L["k"]), nb)
    semi, anti = _both(L, R, nb, ["k"], ["k"])
    assert semi == [6, 26]
    assert sorted(anti) == [i for i in range(40) if L["k"][i] != 6]
    # anti keeps whole buckets the right side leaves empty, in (bucket, key, row) order
    assert anti == sorted(anti, key=lambda i: (bucket[i], L["k"][i], i))
    assert {int(bucket[i]) for i in anti} == set(range(nb))
    # no right rows at all
    assert _both(L, {"k": np.empty(0, dtype=np.int64)}, nb, ["k"], ["k"]) == ([], sorted(range(40), key=lambda i: (bucket[i], L["k"][i], i)))


def test_filters_below_either_side():
    L = {"k": np.array([1, 2, 3, 4]), "v": np.array([10, 20, 30, 40])}
    R = {"k": np.array([1, 2, 3]), "w": np.array([5, 50, 500])}
    # a right filter that empties the bucket: semi keeps nothing, anti everything
    assert _both(L, R, 1, ["k"], ["k"], right_predicates=[("w", 1000, False, None, False)]) == ([], [0, 1, 2, 3])
    # a right filter drops its failing rows from the match set
    assert _both(L, R, 1, ["k"], ["k"], right_predicates=[("w", 40, False, None, False)]) == ([1, 2], [0, 3])
    # left rows failing the left filter are never output, semi or anti
    assert _both(L, R, 1, ["k"], ["k"], left_predicates=[("v", 20, False, None, False)]) == ([1, 2], [3])
    assert _both(L, R, 1, ["k"], ["k"], left_mask=np.array([True, False, True, True]),
                 right_mask=np.array([False, True, True])) == ([2], [0, 3])


# ---- the host layer ----------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("how, want", [("leftsemi", "leftsemi"), ("semi", "leftsemi"), ("left_semi", "leftsemi"),
                                       ("LeftSemi", "leftsemi"), ("leftanti", "leftanti"), ("anti", "leftanti"),
                                       ("left_anti", "leftanti"), ("LEFT_ANTI", "leftanti"), ("inner", "inner")])
def test_join_type_spellings(tmp_path, how, want):
    s, t1, t2 = _fixture(tmp_path, FIVE)
    j = t1.join(t2, on=("t1c1", "t2c1"), how=how)
    assert j.plan.how == want
    assert j.columns == (t1.columns + t2.columns if want == "inner" else t1.columns)


@pytest.mark.parametrize("how", ["left", "outer", "right", "full", "left_outer", "cross", "semi_left"])
def test_other_join_types_still_raise(tmp_path, how):
    s, t1, t2 = _fixture(tmp_path, FIVE)
    with pytest.raises(HyperspaceException, match="not handled"):
        t1.join(t2, on=("t1c1", "t2c1"), how=how)


def test_join_node_defaults_to_inner(tmp_path):
    from hyperspace_b200.session import JoinNode

    s, t1, t2 = _fixture(tmp_path, FIVE)
    assert JoinNode(t1.plan, t2.plan, [("t1c1", "t2c1")]).how == "inner"
    assert t1.join(t2, on=("t1c1", "t2c1")).plan.how == "inner"


def test_explain_names_the_join_type_only_for_semi_and_anti(tmp_path):
    from hyperspace_b200.session import col

    s, t1, t2 = _fixture(tmp_path, FIVE)
    inner = t1.filter(col("t1c3") >= 1).join(t2, on=("t1c1", "t2c1")).select("t1c1", "t1c3", "t2c3").explain()
    assert "joinType" not in inner
    for how, name in (("leftsemi", "LeftSemi"), ("anti", "LeftAnti")):
        plan = t1.filter(col("t1c3") >= 1).join(t2.filter(col("t2c3") >= 1), on=("t1c1", "t2c1"), how=how).select("t1c3").explain()
        assert _uses(plan, "t1i1", "t2i1")
        assert f"keys=[t1c1 = t2c1], joinType={name}, leftFilter=" in plan and "rightFilter=" in plan and "exchange=none" in plan
        assert plan.startswith("Project(['t1c3']) <- GpuBucketJoin(")
    # a semi / anti join outputs no right column
    with pytest.raises(HyperspaceException):
        t1.join(t2, on=("t1c1", "t2c1"), how="semi").select("t2c3")
    from hyperspace_b200.rules import plan_query
    from hyperspace_b200.session import DataFrame, ProjectNode

    bad = DataFrame(s, ProjectNode(t1.join(t2, on=("t1c1", "t2c1"), how="anti").plan, ["t1c3", "t2c1"]))
    with pytest.raises(HyperspaceException, match="left columns only"):
        plan_query(s, bad.plan)


def test_right_index_needs_to_cover_only_keys_and_filter_columns(tmp_path):
    """The right side of a semi / anti join is only probed: an index holding its key and filter columns serves it,
    where an inner join that projects another right column cannot use that index."""
    from hyperspace_b200.session import col

    idx = [("t1i1", "t1", ["t1c1"], ["t1c3"]), ("t2k", "t2", ["t2c1"], ["t2c2"])]
    s, t1, t2 = _fixture(tmp_path, idx)
    for how in ("leftsemi", "leftanti"):
        plan = t1.join(t2.filter(col("t2c2") >= 1), on=("t1c1", "t2c1"), how=how).select("t1c1", "t1c3").explain()
        assert _uses(plan, "t1i1", "t2k"), plan
        plan = t1.select("t1c1", "t1c3").join(t2, on=("t1c1", "t2c1"), how=how).explain()  # no projection above the join
        assert _uses(plan, "t1i1", "t2k") and not plan.startswith("Project")
    inner = t1.join(t2.filter(col("t2c2") >= 1), on=("t1c1", "t2c1")).select("t1c1", "t1c3", "t2c3").explain()
    assert "Name:" not in inner
    # a right filter on a column the index does not hold keeps it off, for semi as for inner
    plan = t1.join(t2.filter(col("t2c4") >= 1), on=("t1c1", "t2c1"), how="semi").select("t1c1", "t1c3").explain()
    assert "Name: t2k," not in plan
