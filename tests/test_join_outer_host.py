"""Left, right and full outer bucket joins without a GPU: hand-written cases that pin tests/join_outer_oracle.py (null keys
on either side, a null in the second of two key columns, duplicate groups, buckets empty on one side, filters on the
preserved and on the null-supplying side, where FullOuter puts unmatched right rows), a cross-check of the oracle
against the inner and anti join oracles, and the plan layer: output columns, explain() and the index pair chosen."""
import numpy as np
import pytest

import join_exists_oracle as JE
import join_oracle as J
import join_outer_oracle as JO
from oracle import oracle as O
from test_join_rule_composite_host import FIVE, _fixture, _uses


def _pairs(L, R, nb, lkeys, rkeys, how, **kw):
    lrow, rrow = JO.outer_join(L, R, nb, lkeys, rkeys, how, **kw)
    return list(zip(lrow.tolist(), rrow.tolist()))


def test_null_keys_on_each_side_and_in_the_second_key_column():
    L = {"a": np.array([1, 1, 1, 2]), "b": np.array([2, 0, 2, 5])}
    lv = {"b": np.array([True, False, True, True])}
    R = {"a": np.array([1, 1, 2]), "b": np.array([2, 2, 0])}
    rv = {"b": np.array([True, True, False])}
    kw = dict(left_valids=lv, right_valids=rv)
    # left sorted: (1, null) row 1, (1, 2) rows 0 and 2, (2, 5) row 3; right: (1, 2) rows 0 and 1, (2, null) row 2
    assert _pairs(L, R, 1, ["a", "b"], ["a", "b"], "left", **kw) == [(1, -1), (0, 0), (0, 1), (2, 0), (2, 1), (3, -1)]
    assert _pairs(L, R, 1, ["a", "b"], ["a", "b"], "right", **kw) == [(0, 0), (2, 0), (0, 1), (2, 1), (-1, 2)]
    assert _pairs(L, R, 1, ["a", "b"], ["a", "b"], "full", **kw) == [(1, -1), (0, 0), (0, 1), (2, 0), (2, 1), (3, -1), (-1, 2)]


def test_null_key_never_matches_zero_or_empty_string():
    L = {"k": np.array([0, 5, 0], dtype=np.int64)}
    R = {"k": np.array([0, 5, 0], dtype=np.int64)}
    lv, rv = {"k": np.array([False, True, True])}, {"k": np.array([True, True, False])}
    # sorted nulls first: left 0 (null), 2 (0), 1 (5); right 2 (null), 0 (0), 1 (5)
    assert _pairs(L, R, 1, ["k"], ["k"], "full", left_valids=lv, right_valids=rv) == [(0, -1), (2, 0), (1, 1), (-1, 2)]
    Ls, Rs = {"s": np.array([b"", b"a", b""], dtype=object)}, {"s": np.array([b"", b"a", b""], dtype=object)}
    assert _pairs(Ls, Rs, 1, ["s"], ["s"], "full", left_valids={"s": lv["k"]}, right_valids={"s": rv["k"]}) == \
        [(0, -1), (2, 0), (1, 1), (-1, 2)]


def test_duplicate_groups():
    L = {"k": np.array([3, 3, 4], dtype=np.int32)}
    R = {"k": np.array([3, 3, 5], dtype=np.int32)}
    assert _pairs(L, R, 1, ["k"], ["k"], "left") == [(0, 0), (0, 1), (1, 0), (1, 1), (2, -1)]
    assert _pairs(L, R, 1, ["k"], ["k"], "right") == [(0, 0), (1, 0), (0, 1), (1, 1), (-1, 2)]
    assert _pairs(L, R, 1, ["k"], ["k"], "full") == [(0, 0), (0, 1), (1, 0), (1, 1), (2, -1), (-1, 2)]


def test_buckets_empty_on_one_side_and_where_unmatched_right_rows_go():
    nb = 4
    L = {"k": np.arange(8, dtype=np.int64)}
    R = {"k": np.array([6, 6, 100, 101, 102], dtype=np.int64)}
    lb, rb = O.np_pmod(O.np_hash_long(L["k"]), nb), O.np_pmod(O.np_hash_long(R["k"]), nb)
    left = _pairs(L, R, nb, ["k"], ["k"], "left")
    assert sorted(l for l, _ in left) == [0, 1, 2, 3, 4, 5, 6, 6, 7]
    assert [r for l, r in left if l == 6] == [0, 1] and all(r == -1 for l, r in left if l != 6)
    right = _pairs(L, R, nb, ["k"], ["k"], "right")
    assert sorted(r for l, r in right if l == -1) == [2, 3, 4] and [p for p in right if p[0] >= 0] == [(6, 0), (6, 1)]
    full = _pairs(L, R, nb, ["k"], ["k"], "full")
    assert len(full) == 9 + 3
    # bucket-major: every output row's bucket, with a right row's bucket for the unmatched ones
    buckets = [int(lb[l]) if l >= 0 else int(rb[r]) for l, r in full]
    assert buckets == sorted(buckets)
    for b in range(nb):  # inside a bucket the left-outer rows come first, then the unmatched right rows
        rows = [p for p, x in zip(full, buckets) if x == b]
        kinds = [p[0] == -1 for p in rows]
        assert kinds == sorted(kinds)
        assert [p for p in rows if p[0] >= 0] == [p for p in left if int(lb[p[0]]) == b]
    # a side with no rows at all
    none = {"k": np.empty(0, dtype=np.int64)}
    assert [r for _, r in _pairs(L, none, nb, ["k"], ["k"], "left")] == [-1] * 8
    assert _pairs(L, none, nb, ["k"], ["k"], "right") == []
    assert [l for l, _ in _pairs(none, R, nb, ["k"], ["k"], "full")] == [-1] * 5


def test_filters_on_the_preserved_and_the_null_supplying_side():
    L = {"k": np.array([1, 2, 3, 4]), "v": np.array([10, 20, 30, 40])}
    R = {"k": np.array([1, 2, 3]), "w": np.array([5, 50, 500])}
    # a preserved row that fails its filter is not output
    assert _pairs(L, R, 1, ["k"], ["k"], "left", left_predicates=[("v", 20, False, None, False)]) == [(1, 1), (2, 2), (3, -1)]
    # a null-supplying row that fails its filter matches nothing
    assert _pairs(L, R, 1, ["k"], ["k"], "left", right_predicates=[("w", 40, False, None, False)]) == \
        [(0, -1), (1, 1), (2, 2), (3, -1)]
    assert _pairs(L, R, 1, ["k"], ["k"], "right", right_predicates=[("w", 40, False, None, False)]) == [(1, 1), (2, 2)]
    assert _pairs(L, R, 1, ["k"], ["k"], "right", left_predicates=[("v", 30, False, None, False)]) == [(-1, 0), (-1, 1), (2, 2)]
    # both sides are preserved under FullOuter: a row failing its filter is not output, the other side's twin unmatched
    assert _pairs(L, R, 1, ["k"], ["k"], "full", left_predicates=[("v", 30, False, None, False)]) == \
        [(2, 2), (3, -1), (-1, 0), (-1, 1)]
    assert _pairs(L, R, 1, ["k"], ["k"], "full", left_mask=np.array([True, False, True, True]),
                  right_mask=np.array([False, True, True])) == [(0, -1), (2, 2), (3, -1), (-1, 1)]
    # a right filter that empties the bucket: every left row, padded
    assert _pairs(L, R, 1, ["k"], ["k"], "left", right_predicates=[("w", 1000, False, None, False)]) == [(i, -1) for i in range(4)]


def _random(seed, nl, nr):
    rng = np.random.default_rng(seed)
    L = {"a": rng.integers(0, 6, nl).astype(np.int64), "b": rng.integers(0, 5, nl).astype(np.int64)}
    R = {"a": rng.integers(0, 6, nr).astype(np.int64), "b": rng.integers(0, 5, nr).astype(np.int64)}
    lv = {"b": rng.random(nl) >= 0.15}
    rv = {"a": rng.random(nr) >= 0.1, "b": rng.random(nr) >= 0.1}
    return L, R, lv, rv


@pytest.mark.parametrize("nb", [1, 5])
def test_left_outer_is_inner_plus_anti(nb):
    """The rows of LeftOuter with a right row are the inner join's, in the same order; its padded rows are the anti join's."""
    L, R, lv, rv = _random(1, 400, 300)
    kw = dict(left_valids=lv, right_valids=rv, left_predicates=[("a", 1, False, None, False)],
              right_predicates=[("b", None, False, 3, False)])
    lrow, rrow = JO.outer_join(L, R, nb, ["a", "b"], ["a", "b"], "left", **kw)
    il, ir = J.bucket_join(L, R, nb, ["a", "b"], ["a", "b"], **kw)
    matched = rrow >= 0
    assert np.array_equal(lrow[matched], il) and np.array_equal(rrow[matched], ir) and len(il) > 0
    anti = JE.exists_join(L, R, nb, ["a", "b"], ["a", "b"], "anti", **kw)
    assert np.array_equal(lrow[~matched], anti) and len(anti) > 0
    # RightOuter is LeftOuter with the sides swapped
    swapped = dict(left_valids=rv, right_valids=lv, left_predicates=kw["right_predicates"], right_predicates=kw["left_predicates"])
    rl, rr = JO.outer_join(L, R, nb, ["a", "b"], ["a", "b"], "right", **kw)
    sl, sr = JO.outer_join(R, L, nb, ["a", "b"], ["a", "b"], "left", **swapped)
    assert np.array_equal(rl, sr) and np.array_equal(rr, sl)
    # FullOuter: LeftOuter's rows, plus the right side's anti join rows
    fl, fr = JO.outer_join(L, R, nb, ["a", "b"], ["a", "b"], "full", **kw)
    assert sorted(zip(fl[fl >= 0].tolist(), fr[fl >= 0].tolist())) == sorted(zip(lrow.tolist(), rrow.tolist()))
    ranti = JE.exists_join(R, L, nb, ["a", "b"], ["a", "b"], "anti", **swapped)
    assert sorted(fr[fl < 0].tolist()) == sorted(ranti.tolist()) and len(ranti) > 0


# ---- the host layer ----------------------------------------------------------------------------------------------------

OUTER = [("leftouter", "LeftOuter"), ("rightouter", "RightOuter"), ("fullouter", "FullOuter")]


def _join(s, a, b, pairs, how):
    from hyperspace_b200.session import DataFrame, JoinNode

    return DataFrame(s, JoinNode(a.plan, b.plan, pairs, how))


@pytest.mark.parametrize("how", [h for h, _ in OUTER])
def test_output_columns_are_both_sides(tmp_path, how):
    s, t1, t2 = _fixture(tmp_path, FIVE)
    assert _join(s, t1, t2, [("t1c1", "t2c1")], how).columns == t1.columns + t2.columns
    assert _join(s, t1, t2, [("t1c1", "t2c1")], "leftanti").columns == t1.columns


@pytest.mark.parametrize("how, name", OUTER)
def test_explain_and_the_index_pair(tmp_path, how, name):
    from hyperspace_b200.session import DataFrame, ProjectNode, col

    s, t1, t2 = _fixture(tmp_path, FIVE)
    a, b = t1.filter(col("t1c3") >= 1), t2.filter(col("t2c3") >= 1)
    for pairs, names in (([("t1c1", "t2c1")], ("t1i1", "t2i1")), ([("t1c2", "t2c2"), ("t1c1", "t2c1")], ("t1i2", "t2i2"))):
        inner = a.join(b, on=pairs).select("t1c1", "t1c3", "t2c3").explain()
        plan = DataFrame(s, ProjectNode(_join(s, a, b, pairs, how).plan, ["t1c1", "t1c3", "t2c3"])).explain()
        assert _uses(inner, *names) and _uses(plan, *names), plan
        assert plan == inner.replace("], leftFilter=", f"], joinType={name}, leftFilter=")
        assert plan.startswith("Project(['t1c1', 't1c3', 't2c3']) <- GpuBucketJoin(") and "exchange=none" in plan
    assert "joinType" not in inner
    # an index that does not cover a referenced right column serves neither an inner nor an outer join
    plan = _join(s, t1, t2.filter(col("t2c4") >= 1), [("t1c1", "t2c1")], how).explain()
    assert "Name: t2i1," not in plan and f"joinType={name}" in plan


def test_outer_join_type_strings_of_the_binding():
    from hyperspace_b200 import _native

    assert _native.OUTER_JOIN_TYPES == {"left": _native.HS_JOIN_LEFT_OUTER, "right": _native.HS_JOIN_RIGHT_OUTER,
                                        "full": _native.HS_JOIN_FULL_OUTER} == {"left": 3, "right": 4, "full": 5}
    for bad in ("outer", "leftouter", "semi", "inner"):
        with pytest.raises(ValueError, match="join_type"):
            _native.Context.bucket_join_outer(None, [], [], [], [], 1, ["k"], ["k"], [], [], bad)
    assert "left" not in _native.JOIN_TYPES
