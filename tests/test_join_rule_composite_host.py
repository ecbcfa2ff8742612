"""JoinIndexRule over AND-ed equi-joins on several columns, restated from T/index/covering/JoinIndexRuleTest.scala:420-550
over the same five indexes as its fixture (t1i1, t1i2, t1i3, t2i1, t2i2), plus JoinRankFilter.isCompatible, the plan of
E2EHyperspaceRulesTest.scala:376-405 and the forms DataFrame.join's `on` takes.  Plans only: no GPU needed."""
import os

import pytest

from hyperspace_b200 import log_entry as LE
from hyperspace_b200.log_entry import FileIdTracker, HyperspaceException


def _entry():
    e = LE.IndexLogEntry.from_json(open(os.path.join(os.path.dirname(__file__), "golden", "index_log_entry_spec.json")).read())
    e.state = "ACTIVE"
    return e


def _fixture(tmp_path, indexes, types=None):
    from hyperspace_b200 import rules as R
    from hyperspace_b200.session import DataFrame, HyperspaceSession, RelationNode

    s = HyperspaceSession({"spark.hyperspace.system.path": str(tmp_path / "indexes")}).enableHyperspace()
    types = types or {}

    def rel(t):
        return RelationNode([f"file:{tmp_path}/{t}"], [(f"file:{tmp_path}/{t}/f1", 100, 1)],
                            [(f"{t}c{i}", types.get(f"{t}c{i}", "long")) for i in (1, 2, 3, 4)])

    rels = {"t1": rel("t1"), "t2": rel("t2")}
    for name, t, indexed, included in indexes:
        r = rels[t]
        e = _entry()
        e.name, e.indexedColumns, e.includedColumns, e.id = name, indexed, included, 1
        e.content = LE.Content.from_leaf_files([(f"file:{tmp_path}/indexes/{name}/v__=0/part-00000-x_00000.c000.parquet", 10, 1)],
                                               FileIdTracker())
        e.relations = [LE.Relation(r.root_paths, LE.Content.from_leaf_files(r.files, FileIdTracker()),
                                   {"type": "struct", "fields": []}, "parquet")]
        e.signatures = [LE.Signature(LE.INDEX_SIGNATURE_PROVIDER, R.index_signature(r))]
        lm = LE.IndexLogManager(os.path.join(str(tmp_path / "indexes"), name))
        assert lm.write_log(1, e) and lm.create_latest_stable_log(1)
    return s, DataFrame(s, rels["t1"]), DataFrame(s, rels["t2"])


FIVE = [("t1i1", "t1", ["t1c1"], ["t1c3"]), ("t1i2", "t1", ["t1c1", "t1c2"], ["t1c3"]), ("t1i3", "t1", ["t1c2"], ["t1c3"]),
        ("t2i1", "t2", ["t2c1"], ["t2c3"]), ("t2i2", "t2", ["t2c1", "t2c2"], ["t2c3"])]


def _plan(t1, t2, on, cols=("t1c1", "t1c2", "t1c3", "t2c1", "t2c2", "t2c3")):
    from hyperspace_b200.session import col

    # the reference's fixture puts a Filter under both sides (JoinIndexRuleTest.scala:84-95)
    return t1.filter(col("t1c3") >= 1).join(t2.filter(col("t2c3") >= 1), on=on).select(*cols).explain()


def _uses(plan, *names):
    return all(f"Name: {n}," in plan for n in names) and plan.count("Name: ") == len(names)


def test_composite_condition(tmp_path):
    s, t1, t2 = _fixture(tmp_path, FIVE)
    # 'Join rule updates plan for composite query (AND based Equi-Join).'
    assert _uses(_plan(t1, t2, [("t1c1", "t2c1"), ("t1c2", "t2c2")]), "t1i2", "t2i2")
    # '... with order of predicates changed.'
    plan = _plan(t1, t2, [("t1c2", "t2c2"), ("t1c1", "t2c1")])
    assert _uses(plan, "t1i2", "t2i2")
    assert "keys=[t1c1 = t2c1, t1c2 = t2c2]" in plan  # both sides in the left index's column order
    # '... with swapped attributes.'
    assert _uses(_plan(t1, t2, [("t1c1", "t2c1"), ("t2c2", "t1c2")]), "t1i2", "t2i2")


def test_no_one_to_one_mapping(tmp_path):
    s, t1, t2 = _fixture(tmp_path, FIVE)
    # "Join rule doesn't update plan if columns don't have one-to-one mapping."
    assert "Name:" not in _plan(t1, t2, [("t1c1", "t2c1"), ("t1c1", "t2c2")])   # t1c1 against t2c1 and t2c2
    assert "Name:" not in _plan(t1, t2, [("t1c1", "t2c1"), ("t1c2", "t2c1")])   # t2c1 against t1c1 and t1c2
    from hyperspace_b200.rules import plan_query

    with pytest.raises(HyperspaceException, match="one-to-one"):  # and the GPU join does not run such a condition
        plan_query(s, t1.join(t2, on=[("t1c1", "t2c1"), ("t1c1", "t2c2")]).plan).execute()


def test_repeated_predicates(tmp_path):
    s, t1, t2 = _fixture(tmp_path, FIVE)
    # '... one-to-one mapping with repeated case-insensitive predicates.'
    plan = _plan(t1, t2, [("t1c1", "t2c1"), ("T1C1", "T2C1")], cols=("t1c1", "t1c3", "t2c1", "t2c3"))
    assert _uses(plan, "t1i1", "t2i1") and "keys=[t1c1 = t2c1]" in plan
    # '... composite query for repeated predicates.'
    assert _uses(_plan(t1, t2, [("t1c1", "t2c1"), ("t1c2", "t2c2"), ("t1c1", "t2c1")]), "t1i2", "t2i2")


def test_columns_of_one_side_compared_with_each_other(tmp_path):
    s, t1, t2 = _fixture(tmp_path, FIVE)
    # "Join rule doesn't update plan if columns don't belong to either side of join node."
    plan = _plan(t1, t2, [("t1c1", "t1c2"), ("t1c2", "t2c2")])
    assert "Name:" not in plan and "GpuShuffle" in plan


def test_is_compatible(tmp_path):
    """JoinRankFilter.isCompatible: (A, C) on the left pairs with (B, D) on the right when A = B and C = D, not with (D, B)."""
    idx = [("l_ac", "t1", ["t1c1", "t1c3"], ["t1c4"]), ("r_bd", "t2", ["t2c2", "t2c4"], ["t2c3"]),
           ("r_db", "t2", ["t2c4", "t2c2"], ["t2c3"])]
    s, t1, t2 = _fixture(tmp_path, idx)
    on = [("t1c1", "t2c2"), ("t1c3", "t2c4")]
    plan = _plan(t1, t2, on, cols=("t1c1", "t1c3", "t1c4", "t2c2", "t2c3", "t2c4"))
    assert _uses(plan, "l_ac", "r_bd")
    from hyperspace_b200 import rules as R
    from hyperspace_b200.rules import Linear, _linear

    l = Linear(_linear(t1.plan).relation, None, ["t1c1", "t1c3", "t1c4"])
    r = Linear(_linear(t2.plan).relation, None, ["t2c2", "t2c3", "t2c4"])
    keys = R.join_key_pairs(l, r, on)
    assert R.join_index_rule(s, l, r, keys)[1].entry.name == "r_bd"
    # without r_bd, the incompatible order leaves the join without indexes
    s2, u1, u2 = _fixture(tmp_path / "b", [idx[0], idx[2]])
    assert "Name:" not in _plan(u1, u2, on, cols=("t1c1", "t1c3", "t1c4", "t2c2", "t2c3", "t2c4"))


def test_key_types_must_match_per_position(tmp_path):
    s, t1, t2 = _fixture(tmp_path, FIVE, types={"t2c2": "integer"})
    assert "Name:" not in _plan(t1, t2, [("t1c1", "t2c1"), ("t1c2", "t2c2")])
    assert _uses(_plan(t1, t2, [("t1c1", "t2c1")], cols=("t1c1", "t1c3", "t2c3")), "t1i1", "t2i1")


def test_filter_columns_must_be_covered(tmp_path):
    from hyperspace_b200.session import col

    s, t1, t2 = _fixture(tmp_path, FIVE)
    on = [("t1c1", "t2c1"), ("t1c2", "t2c2")]
    plan = t1.filter(col("t1c4") >= 1).join(t2, on=on).select("t1c3", "t2c3").explain()
    assert "Name:" not in plan  # t1c4 is read by the filter, and no t1 index includes it
    plan = t1.filter(col("t1c3") >= 1).join(t2, on=on).select("t1c1", "t2c3").explain()
    assert _uses(plan, "t1i2", "t2i2") and "leftFilter=[('t1c3', 1, False, None, False)]" in plan
    assert "rightFilter" not in plan


def test_e2e_filtered_sides_choose_the_join_indexes(tmp_path):
    """E2EHyperspaceRulesTest.scala:376-405: join and filter indexes on both sides; the join indexes are chosen."""
    from hyperspace_b200.session import col

    idx = [("leftJoinIndex", "t1", ["t1c3"], ["t1c4"]), ("leftDfFilterIndex", "t1", ["t1c4"], ["t1c3"]),
           ("rightDfJoinIndex", "t2", ["t2c3"], ["t2c1"]), ("rightDfFilterIndex", "t2", ["t2c1"], ["t2c3"])]
    s, t1, t2 = _fixture(tmp_path, idx)
    left = t1.filter(col("t1c4") == 2).select("t1c4", "t1c3")
    right = t2.filter(col("t2c1") == 3000).select("t2c1", "t2c3")
    plan = left.join(right, on=("t1c3", "t2c3")).select("t1c3", "t1c4", "t2c1").explain()
    assert _uses(plan, "leftJoinIndex", "rightDfJoinIndex") and "exchange=none" in plan


def test_join_on_forms(tmp_path):
    from hyperspace_b200.session import JoinNode

    s, t1, t2 = _fixture(tmp_path, FIVE)
    assert t1.join(t2, on=("T1C1", "t2c1")).plan.pairs == [("t1c1", "t2c1")]
    assert t1.join(t2, on=[("t1c1", "t2c1"), ("t2c2", "t1c2")]).plan.pairs == [("t1c1", "t2c1"), ("t1c2", "t2c2")]
    assert t1.join(t2, on=[["t1c1", "t2c1"]]).plan.pairs == [("t1c1", "t2c1")]
    assert t1.join(t2, on=[("t1c1", "t1c2")]).plan.pairs == [("t1c1", "t1c2")]  # kept: the rule turns it down
    both = t1.join(t1, on="t1c1").plan
    assert isinstance(both, JoinNode) and both.pairs == [("t1c1", "t1c1")]
    for bad in ([], [("t1c1",)], ["t1c1"]):
        with pytest.raises(HyperspaceException):
            t1.join(t2, on=bad)
    with pytest.raises(HyperspaceException):
        t1.join(t2, on=[("t1c1", "t2c1"), ("t1c2", "t2c2")], how="left")
    with pytest.raises(HyperspaceException):
        t1.join(t2, on=[("t1c1", "nope")])
