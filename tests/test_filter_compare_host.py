"""Host-side tests of comparisons between two columns (`a < b`, `a = b`, `a <=> b`): the coercion in
hyperspace_b200/csrc/predicates.h (resolve_compare, check_compares) and the scalar comparison in column_compare.h, built as
host code under AddressSanitizer where the compiler has it, against tests/filter_compare_oracle.py; and the Python forms of
the session layer."""
import itertools
import os
import shutil
import subprocess

import numpy as np
import pytest

import filter_compare_oracle as FC

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OPS = {"<": 1, "<=": 2, ">": 3, ">=": 4, "=": 5, "<=>": 6}
NOT = 1
INT, FLOAT, DOUBLE, STRING = 0, 1, 2, 3  # CompareDomain
I64_MIN, I64_MAX = -2**63, 2**63 - 1


@pytest.fixture(scope="module")
def native(tmp_path_factory):
    if shutil.which("nvcc") is None:
        pytest.skip("nvcc not on PATH")
    exe = str(tmp_path_factory.mktemp("filter_compare") / "filter_compare")
    base = ["nvcc", "-std=c++17", "-O1", "-g", "-Wno-deprecated-gpu-targets", "-o", exe,
            os.path.join(ROOT, "tests", "native", "filter_compare.cu")]
    try:
        subprocess.check_call(base + ["-Xcompiler", "-fsanitize=address,-fno-omit-frame-pointer"], stderr=subprocess.DEVNULL)
        asan = subprocess.run([exe, "x"], capture_output=True).returncode == 2
    except subprocess.CalledProcessError:
        asan = False
    if not asan:
        subprocess.check_call(base)
    return exe


def run(native, lines):
    out = subprocess.run([native], input="\n".join(lines) + "\n", capture_output=True, text=True, check=True).stdout
    got = out.splitlines()
    assert len(got) == len(lines)
    return got


def spec(t):
    """A Spark type name as the driver's column: kind, precision, scale."""
    d = FC._decimal(t)
    if d:
        return f"decimal {d[0]} {d[1]}"
    return f"{t} 0 0"


# ---- coercion: every cell of the table and every refusal -------------------------------------------------------------

CELLS = [  # (left, right, domain, factor0, factor1)
    ("integer", "integer", INT, 1, 1), ("long", "long", INT, 1, 1), ("float", "float", FLOAT, 1, 1),
    ("double", "double", DOUBLE, 1, 1), ("string", "string", STRING, 1, 1), ("binary", "binary", STRING, 1, 1),
    ("timestamp", "timestamp", INT, 1, 1), ("date", "date", INT, 1, 1), ("decimal(12,2)", "decimal(12,2)", INT, 1, 1),
    ("integer", "long", INT, 1, 1), ("long", "integer", INT, 1, 1), ("byte", "long", INT, 1, 1),
    ("integer", "float", FLOAT, 1, 1), ("float", "long", FLOAT, 1, 1),
    ("integer", "double", DOUBLE, 1, 1), ("double", "long", DOUBLE, 1, 1), ("float", "double", DOUBLE, 1, 1),
    ("decimal(9,2)", "decimal(12,2)", INT, 1, 1), ("decimal(9,2)", "decimal(18,5)", INT, 1000, 1),
    ("decimal(18,18)", "decimal(5,0)", INT, 1, 10**18), ("decimal(18,4)", "integer", INT, 1, 10**4),
    ("long", "decimal(18,18)", INT, 10**18, 1), ("decimal(7,0)", "long", INT, 1, 1),
    ("decimal(9,3)", "float", DOUBLE, 1000, 1), ("double", "decimal(18,6)", DOUBLE, 1, 10**6),
    ("date", "timestamp", INT, FC.DAY_MICROS, 1), ("timestamp", "date", INT, 1, FC.DAY_MICROS),
]

REFUSED = [("string", "integer"), ("long", "string"), ("string", "date"), ("timestamp", "string"), ("string", "binary"),
           ("date", "integer"), ("long", "timestamp"), ("timestamp", "double"), ("decimal(9,2)", "date"),
           ("boolean", "boolean"), ("boolean", "integer"), ("string", "decimal(9,2)"), ("float", "date")]


def test_coercion_table(native):
    got = run(native, [f"resolve {spec(l)} {spec(r)} 1 0" for l, r, *_ in CELLS])
    for (l, r, dom, f0, f1), line in zip(CELLS, got):
        assert line == f"ok {dom} {f0} {f1}", (l, r, line)
        want = FC.domain(l, r)
        assert want is not None and {"int": INT, "float": FLOAT, "double": DOUBLE, "string": STRING}[want[0]] == dom
        if want[0] in ("int", "double"):
            assert (want[1], want[2]) == (f0, f1), (l, r)


def test_coercion_refusals_name_both_columns(native):
    got = run(native, [f"resolve {spec(l)} {spec(r)} 5 0" for l, r in REFUSED])
    for (l, r), line in zip(REFUSED, got):
        assert line == f"refused -6 filter scan: the columns 'a' ({l}) and 'b' ({r}) cannot be compared", line
        assert FC.domain(l, r) is None


def test_check_compares(native):
    got = run(native, ["check a b 1 0 0", "check a b 6 1 15", "check - b 1 0 0", "check a - 1 0 0", "check a b 0 0 0",
                       "check a b 7 0 0", "check a b 1 2 0", "check a b 1 0 16", "check a a 5 1 0"])
    assert got[0] == "ok" and got[1] == "ok" and got[8] == "ok"
    assert got[2] == got[3] == "refused -1 filter scan: comparison without a column"
    assert got[4] == "refused -1 filter scan: comparison of 'a' and 'b' has an unknown operator 0"
    assert got[5] == "refused -1 filter scan: comparison of 'a' and 'b' has an unknown operator 7"
    assert got[6] == "refused -1 filter scan: comparison of 'a' and 'b' has unknown flags 0x2"
    assert got[7] == "refused -6 filter scan: more than 16 predicates and terms"


def test_check_filters_order_across_sides(native):
    # every side's predicates before any side's comparisons, and the left side before the right one
    got = run(native, ["sides 1 1 5 1", "sides 7 1 1 0", "sides 7 1 9 1", "sides 1 1 9 1", "sides 1 0 7 0"])
    assert got[0] == "ok"
    assert got[1] == got[4] == "refused -1 filter scan: predicate without a column"
    assert got[2] == "refused -1 filter scan: comparison of 'a' and 'b' has an unknown operator 7"
    assert got[3] == "refused -1 filter scan: comparison of 'a' and 'b' has an unknown operator 9"


# ---- the scalar comparison on hard values -------------------------------------------------------------------------------

def _fmt(t, v):
    if isinstance(v, (bytes, bytearray)):
        return v.hex() or "-"
    if isinstance(v, (float, np.floating)):
        return repr(float(v)) if np.isfinite(v) else ("nan" if np.isnan(v) else ("inf" if v > 0 else "-inf"))
    return str(int(v))


def _arr(t, vals):
    k = FC.kind(t)
    if k in ("string", "binary"):
        return list(vals)
    if k == "float":
        return np.array(vals, dtype=np.float32)
    if k == "double":
        return np.array(vals, dtype=np.float64)
    d = FC._decimal(t)
    narrow = k in ("integer", "date") or (d is not None and d[0] <= 9)
    return np.array(vals, dtype=np.int32 if narrow else np.int64)


def check_pairs(native, lt, rt, pairs):
    """Every pair of (left value | None, right value | None) under all six ops, with and without NOT, against the oracle."""
    lv = [0 if a is None else a for a, _ in pairs]
    rv = [0 if b is None else b for _, b in pairs]
    if FC.kind(lt) in ("string", "binary"):
        lv = [b"" if a is None else a for a, _ in pairs]
    if FC.kind(rt) in ("string", "binary"):
        rv = [b"" if b is None else b for _, b in pairs]
    lval = np.array([a is not None for a, _ in pairs])
    rval = np.array([b is not None for _, b in pairs])
    rows = " ".join(f"{int(a is None)} {_fmt(lt, x)} {int(b is None)} {_fmt(rt, y)}" for (a, b), x, y in zip(pairs, lv, rv))
    cases = [(op, neg) for op in OPS for neg in (False, True)]
    got = run(native, [f"rows {spec(lt)} {spec(rt)} {OPS[op]} {NOT if neg else 0} {len(pairs)} {rows}" for op, neg in cases])
    L, R = (lt, _arr(lt, lv), lval), (rt, _arr(rt, rv), rval)
    for (op, neg), line in zip(cases, got):
        want = FC.mask(L, R, op, neg)
        assert line.split()[1:] == [str(int(x)) for x in want], (lt, rt, op, neg)


FLOATS = [float("nan"), -0.0, 0.0, float("inf"), float("-inf"), 1.5, -2.0, 16777216.0, 3.4028234663852886e38]


def test_floating_point_edges(native):
    pairs = list(itertools.product(FLOATS, FLOATS)) + [(None, 1.0), (1.0, None), (None, None), (float("nan"), None)]
    check_pairs(native, "double", "double", pairs)
    check_pairs(native, "float", "float", pairs)
    check_pairs(native, "float", "double", [(np.float32(0.1), 0.1), (np.float32(0.1), float(np.float32(0.1)))] + pairs)


def test_integers_against_floating_point_round_to_nearest(native):
    t24, t53 = 2**24, 2**53
    ints = [t24, t24 + 1, t24 + 2, t24 + 3, -(t24 + 1), 2**31 - 1, -2**31]
    check_pairs(native, "integer", "float", [(i, float(np.float32(f))) for i in ints for f in (t24, t24 + 2, t24 + 4, 2**31, -2**31)])
    longs = [t53, t53 + 1, t53 + 2, t53 + 3, I64_MAX, I64_MIN, 2**60 + 2**36 + 1, 2**60 + 2**36, t24 + 1]
    check_pairs(native, "long", "float", [(i, f) for i in longs for f in (float(t24), 2.0**60, 2.0**60 + 2**37, 2.0**63, -2.0**63, float("nan"))])
    check_pairs(native, "long", "double", [(i, f) for i in longs for f in (float(t53), float(t53 + 2), 2.0**63, -2.0**63, float("inf"))])
    check_pairs(native, "integer", "double", [(i, float(f)) for i in ints for f in (t24, t24 + 1, 2**31 - 1, -2**31)])
    check_pairs(native, "integer", "long", [(i, j) for i in (-2**31, 2**31 - 1, 0) for j in (-2**31, 2**31 - 1, 2**31, I64_MIN, I64_MAX)])


@pytest.mark.parametrize("scale", range(19))
def test_int64_extremes_against_decimal18(native, scale):
    dmax = 10**18 - 1
    decs = [dmax, -dmax, 0, 1, -1, 10**scale, -(10**scale), 9223372036854775 * 10**min(scale, 3) % 10**18]
    longs = [I64_MIN, I64_MAX, 0, 1, -1, 999999999999999999, -999999999999999999]
    t = f"decimal(18,{scale})"
    check_pairs(native, "long", t, [(a, b) for a in longs for b in decs])
    check_pairs(native, t, "integer", [(b, a) for b in decs for a in (-2**31, 2**31 - 1, 0, 1, -1)])


def test_decimals_of_unequal_scale(native):
    check_pairs(native, "decimal(9,2)", "decimal(18,5)", [(150, 1500000 // 10), (150, 1500), (150, 1501), (-1, -10), (999999999, 9999999990000),
                                                           (-999999999, -9999999990001), (None, 1), (None, None)])
    check_pairs(native, "decimal(18,18)", "decimal(5,0)", [(10**18 - 1, 1), (10**18 - 1, 0), (-(10**18) + 1, -1), (0, 0), (5 * 10**17, 0)])
    check_pairs(native, "decimal(12,2)", "decimal(12,2)", [(1, 2), (2, 1), (5, 5), (None, 5)])


def test_decimal_to_double_is_correctly_rounded(native):
    cases = [(9007199254740993, 1), (10**18 - 1, 18), (999999999999999999, 2), (-999999999999999999, 17), (9007199254740993, 0),
             (123456789012345678, 9), (2**53 + 1, 3), (2**60, 18), (2**59 + 1, 1), (3, 1), (-7, 18), (2**53 * 5 + 5, 1)]
    import random
    rng = random.Random(5)
    cases += [(rng.randrange(-10**18 + 1, 10**18), rng.randrange(0, 19)) for _ in range(3000)]
    cases += [(rng.randrange(2**53, 2**60) * rng.choice((1, -1)), rng.randrange(1, 19)) for _ in range(3000)]
    got = run(native, [f"d2d {u} {s}" for u, s in cases])
    for (u, s), line in zip(cases, got):
        want = np.float64(u / 10**s).view(np.uint64)
        assert line == f"ok {int(want):016x}", (u, s)
    check_pairs(native, "decimal(18,1)", "double", [(9007199254740993, 900719925474099.2), (9007199254740993, 900719925474099.3),
                                                     (1, 0.1), (-1, -0.1), (1, float("nan")), (None, 0.0)])
    check_pairs(native, "decimal(9,1)", "float", [(1, float(np.float32(0.1))), (15, 1.5), (-0, -0.0)])


def test_date_against_timestamp_at_day_edges(native):
    day = FC.DAY_MICROS
    pairs = [(d, d * day + k) for d in (0, 1, -1, 19000, -719162, 2932896) for k in (-1, 0, 1, day - 1, day)]
    check_pairs(native, "date", "timestamp", pairs + [(None, 0), (0, None)])
    check_pairs(native, "timestamp", "date", [(b, a) for a, b in pairs])
    check_pairs(native, "date", "date", [(1, 2), (2, 1), (3, 3)])


def test_strings_in_byte_order(native):
    words = [b"", b"a", b"ab", b"abc", b"ab\x00", b"\x80", b"\xff", b"\xff\xff", "é".encode(), b"b"]
    check_pairs(native, "string", "string", list(itertools.product(words, words)) + [(None, b"a"), (b"", None), (None, None)])


# ---- the Python forms ----------------------------------------------------------------------------------------------------

def test_python_forms():
    from hyperspace_b200.session import col

    cases = [(col("a") < col("b"), "(a < b)", ("a", "<", "b", 0)), (col("a") <= col("b"), "(a <= b)", ("a", "<=", "b", 0)),
             (col("a") > col("b"), "(a > b)", ("a", ">", "b", 0)), (col("a") >= col("b"), "(a >= b)", ("a", ">=", "b", 0)),
             (col("a") == col("b"), "(a = b)", ("a", "=", "b", 0)), (col("a") != col("b"), "NOT (a = b)", ("a", "=", "b", NOT)),
             (col("a").eqNullSafe(col("b")), "(a <=> b)", ("a", "<=>", "b", 0)),
             (~col("a").eqNullSafe(col("b")), "NOT (a <=> b)", ("a", "<=>", "b", NOT)),
             (~(col("a") < col("b")), "NOT (a < b)", ("a", "<", "b", NOT)), (~(col("a") != col("b")), "(a = b)", ("a", "=", "b", 0)),
             (col("k") < col("k"), "(k < k)", ("k", "<", "k", 0))]
    for p, text, native_form in cases:
        c, = p.compares
        assert str(c) == text and c.as_native() == native_form
        assert not p.bounds and not p.anys
    p = col("k").between(col("lo"), col("hi"))
    assert [str(c) for c in p.compares] == ["(k >= lo)", "(k <= hi)"] and p.columns == ["k", "lo", "hi"]
    p = (col("a") < col("b")) & (col("k") > 5) & col("s").isNull()
    assert [str(c) for c in p.compares] == ["(a < b)"] and p.terms == [("k", ">", 5)] and len(p.anys) == 1
    assert set(p.columns) == {"a", "b", "k", "s"}
    p = col("k").between(col("lo"), 9)
    assert [str(c) for c in p.compares] == ["(k >= lo)"] and p.terms == [("k", "<=", 9)]


def test_python_refusals():
    from hyperspace_b200 import log_entry as LE
    from hyperspace_b200.session import col

    with pytest.raises(LE.HyperspaceException, match="OR across columns"):
        (col("a") < col("b")) | (col("a") > 5)
    with pytest.raises(LE.HyperspaceException, match="OR across columns"):
        (col("a") > 5) | (col("a") < col("a"))
    with pytest.raises(LE.HyperspaceException, match="OR across columns"):
        col("k").isin(1, col("v"))
    with pytest.raises(LE.HyperspaceException, match="a NOT over several columns"):
        ~((col("a") < col("b")) & (col("a") > 1))
    with pytest.raises(LE.HyperspaceException, match="a NOT over several columns"):
        ~((col("a") < col("b")) & (col("c") < col("d")))


def _fabricated(tmp_path, indexed, included, schema):
    from hyperspace_b200 import log_entry as LE
    from hyperspace_b200 import rules
    from hyperspace_b200.session import DataFrame, HyperspaceSession, RelationNode

    s = HyperspaceSession({"spark.hyperspace.system.path": str(tmp_path / "ix")}).enableHyperspace()
    rel = RelationNode([f"file:{tmp_path}/t"], [(f"file:{tmp_path}/t/a.parquet", 100, 1)], schema)
    tracker = LE.FileIdTracker()
    idx_files = [(f"file:{tmp_path}/ix/idx/v__=0/part-00000-x_{b:05d}.c000.parquet", 10, 1) for b in range(2)]
    e = LE.IndexLogEntry(
        name="idx", indexedColumns=indexed, includedColumns=included, schema={"type": "struct", "fields": []}, numBuckets=2,
        derived_properties={"lineage": "false"}, content=LE.Content.from_leaf_files(idx_files, LE.FileIdTracker()),
        relations=[LE.Relation(rel.root_paths, LE.Content.from_leaf_files(rel.files, tracker), {"type": "struct", "fields": []}, "parquet")],
        signatures=[LE.Signature(LE.INDEX_SIGNATURE_PROVIDER, rules.index_signature(rel))], state="ACTIVE", id=1)
    lm = LE.IndexLogManager(str(tmp_path / "ix" / "idx"))
    lm.write_log(1, e)
    lm.create_latest_stable_log(1)
    return DataFrame(s, rel)


def test_filter_rule_and_explain(tmp_path):
    from hyperspace_b200.session import col

    df = _fabricated(tmp_path, ["k"], ["v1", "v2"], [("k", "long"), ("v1", "long"), ("v2", "double"), ("w", "long")])
    # the first indexed column only inside a comparison: the index serves, the whole comparison is the residual
    plan = df.filter(col("K") < col("V1")).select("k", "v2").explain()
    assert "Name: idx" in plan and "where=((k < v1))" in plan, plan
    plan = df.filter(col("v1") != col("k")).select("k").explain()
    assert "Name: idx" in plan and "where=(NOT (v1 = k))" in plan, plan
    plan = df.filter((col("k") > 5) & col("k").eqNullSafe(col("v2"))).select("v1").explain()
    assert "Name: idx" in plan and "where=((k <=> v2))" in plan, plan
    # the index does not cover w: no index
    plan = df.filter(col("k") < col("w")).select("k").explain()
    assert plan.startswith("GpuSourceScan") and "where=((k < w))" in plan, plan
    # the first indexed column is not in the filter: no index
    assert df.filter(col("v1") < col("v2")).select("k").explain().startswith("GpuSourceScan")
    # filter() resolves both names case-insensitively
    c, = df.filter(col("V2") >= col("K")).plan.predicate.compares
    assert (c.left, c.op, c.right) == ("v2", ">=", "k")


def test_comparison_across_join_sides_is_refused(tmp_path):
    from hyperspace_b200 import log_entry as LE
    from hyperspace_b200.session import DataFrame, RelationNode, col

    a = _fabricated(tmp_path, ["k"], ["v1", "v2"], [("k", "long"), ("v1", "long"), ("v2", "double"), ("w", "long")])
    b = DataFrame(a.session, RelationNode([f"file:{tmp_path}/u"], [(f"file:{tmp_path}/u/a.parquet", 100, 1)], [("k2", "long"), ("x", "long")]))
    j = a.join(b, on=("k", "k2"))
    with pytest.raises(LE.HyperspaceException, match="non-equi join condition"):
        j.filter(col("v1") < col("x"))
    with pytest.raises(LE.HyperspaceException, match="non-equi join condition"):
        a.join(b, on=col("v1") < col("x"))
    # a comparison inside one side stays that side's filter
    plan = a.filter(col("v1") < col("w")).join(b.filter(col("k2") <= col("x")), on=("k", "k2")).explain()
    assert "where=((v1 < w))" in plan and "where=((k2 <= x))" in plan, plan
