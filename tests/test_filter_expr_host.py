"""Host-side tests of expression comparisons (`a + b < c`, `k % 7 = 0`): the typing in hyperspace_b200/csrc/predicates.h
(resolve_expr, check_exprs) and the evaluator in column_expr.h, built as host code under AddressSanitizer where the
compiler has it, against tests/filter_expr_oracle.py; and the Python forms of the session layer."""
import decimal
import itertools
import os
import random
import shutil
import subprocess
from fractions import Fraction

import numpy as np
import pytest

import filter_expr_oracle as FX
from test_filter_compare_host import _fabricated

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OPS = {"<": 1, "<=": 2, ">": 3, ">=": 4, "=": 5, "<=>": 6}
INT, FLOAT, DOUBLE = 0, 1, 2  # CompareDomain
# ExprOp domains (column_expr.h)
XINT, XLONG, XDEC, XFLOAT, XDOUBLE = 8, 16, 24, 32, 40


@pytest.fixture(scope="module")
def native(tmp_path_factory):
    if shutil.which("nvcc") is None:
        pytest.skip("nvcc not on PATH")
    exe = str(tmp_path_factory.mktemp("filter_expr") / "filter_expr")
    base = ["nvcc", "-std=c++17", "-O1", "-g", "-Wno-deprecated-gpu-targets", "-o", exe, os.path.join(ROOT, "tests", "native", "filter_expr.cu")]
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


def colspec(name, t):
    if t.startswith("decimal("):
        p, s = t[len("decimal("):-1].split(",")
        return f"{name} decimal {p} {s}"
    return f"{name} {t} 0 0"


def tok(node):
    if node[0] == "column":
        return f"c:{node[1]}"
    if node[0] == "literal":
        v = node[1]
        if isinstance(v, decimal.Decimal):
            s = max(0, -v.as_tuple()[2])
            return f"m:{int(v.scaleb(s))}:{s}"
        if isinstance(v, float):
            return f"d:{v!r}"
        return f"i:{v}" if -2**31 <= v < 2**31 else f"l:{v}"
    return node[0]


def case(types, left, op, right, negated=False):
    cols = " ".join(colspec(n, t) for n, t in types.items())
    return (f"{len(types)} {cols} {OPS[op]} {int(negated)} " + " ".join(tok(n) for n in left) + " | " +
            " ".join(tok(n) for n in right) + " ;")


def fmt(v):
    if isinstance(v, (float, np.floating)):
        return "nan" if v != v else ("inf" if v == float("inf") else ("-inf" if v == float("-inf") else repr(float(v))))
    return str(int(v))


def check_rows(native, types, exprs, rows):
    """Every expression (left, op, right) under NOT and without, over the rows (dicts of column -> value or None),
    against the oracle."""
    names = list(types)
    data = " ".join(f"{int(r[n] is None)} {0 if r[n] is None else fmt(r[n])}" for r in rows for n in names)
    lines, want = [], []
    for (left, op, right), neg in itertools.product(exprs, (False, True)):
        lines.append(f"rows {case(types, left, op, right, neg)} {len(rows)} {data}")
        orow = [{n: (types[n], r[n]) for n in names} for r in rows]
        want.append("ok" + "".join(f" {int(FX.holds(left, op, right, neg, o))}" for o in orow))
    for line, w, e in zip(run(native, lines), want, [e for e in exprs for _ in (0, 1)]):
        assert line == w, (e, line, w)


def C(n):
    return ("column", n)


def L(v):
    return ("literal", v)


# ---- typing: the operand-type x operator table, and the refusals ---------------------------------------------------------

TYPES = ["integer", "long", "float", "double", "decimal(9,2)", "decimal(18,4)"]


def test_result_type_table(native):
    lines, want = [], []
    for ta, tb, op in itertools.product(TYPES, TYPES, FX.OPS):
        types = {"a": ta, "b": tb}
        left = [C("a"), C("b"), (op,)]
        try:
            r = FX.side_type(left, types)
            FX.common(r, FX.T(FX.INT))
        except FX.Refused:
            r = None
        lines.append(f"resolve {case(types, left, '<', [L(0)])}")
        want.append(r)
    for line, r, (ta, tb, op) in zip(run(native, lines), want, itertools.product(TYPES, TYPES, FX.OPS)):
        if r is None:
            assert line.startswith("refused -6"), (ta, tb, op, line)
            continue
        ops = [int(x) for x in line.split()[2:]]
        arith = [o for o in ops if o >= 8]
        dom = {FX.INT: XINT, FX.LONG: XLONG, FX.DEC: XDEC, FX.FLOAT: XFLOAT, FX.DOUBLE: XDOUBLE}[r.kind]
        assert arith == [dom + "+-*/%".index(op)], (ta, tb, op, r, line)


def test_refusals_name_what_they_refuse(native):
    got = run(native, [
        "resolve " + case({"s": "string"}, [C("s"), L(1), ("+",)], "<", [L(1)]),
        "resolve " + case({"d": "date"}, [C("d")], "<", [L(1)]),
        "resolve " + case({"t": "timestamp"}, [C("t"), ("neg",)], "<", [L(1)]),
        "resolve " + case({"b": "boolean"}, [C("b")], "=", [L(1)]),
        "resolve " + case({"a": "decimal(9,2)", "b": "integer"}, [C("a"), C("b"), ("/",)], "<", [L(1)]),
        "resolve " + case({"a": "byte", "b": "short"}, [C("a"), C("b"), ("+",)], "<", [L(1)]),
        "resolve " + case({"a": "byte"}, [C("a"), L(1), ("+",)], "<", [L(1)]),
        "resolve " + case({"a": "decimal(18,2)", "b": "decimal(18,2)"}, [C("a"), C("b"), ("*",)], "<", [L(1.5)]),
    ])
    assert got[0] == "refused -6 filter scan: the column 's' (string) cannot be used in arithmetic"
    assert got[1] == "refused -6 filter scan: the column 'd' (date) cannot be used in arithmetic"
    assert got[2] == "refused -6 filter scan: the column 't' (timestamp) cannot be used in arithmetic"
    assert got[3] == "refused -6 filter scan: the column 'b' (boolean) cannot be used in arithmetic"
    assert got[4] == "refused -6 filter scan: decimal division is not handled: (a / b)"
    assert got[5] == "refused -6 filter scan: (a + b) is byte or short arithmetic, which wraps at its width: not handled"
    assert got[6].startswith("ok")  # byte + int literal is int arithmetic
    assert got[7] == "refused -6 filter scan: ((a * b) < 1.5) turns a decimal of more than 18 digits into a double"


def test_decimal_38_digit_boundary(native):
    # decimal(18,0) * decimal(18,0) is decimal(37,0); times decimal(1,0) once more: 37 + 1 + 1 = 39
    t = {"a": "decimal(18,0)", "b": "decimal(18,0)", "c": "decimal(1,0)"}
    t2 = {"a": "decimal(18,0)", "b": "decimal(18,0)", "c": "decimal(1,0)"}
    got = run(native, ["resolve " + case(t, [C("a"), C("b"), ("*",)], "<", [L(0)]),
                       "resolve " + case(t2, [C("a"), C("b"), ("*",), C("c"), ("*",)], "<", [L(0)]),
                       # add: max(p-s) + s + 1: decimal(37,0) + decimal(1,0) is decimal(38,0), one more is 39
                       "resolve " + case(t, [C("a"), C("b"), ("*",), C("c"), ("+",)], "<", [L(0)]),
                       "resolve " + case(t, [C("a"), C("b"), ("*",), C("c"), ("+",), C("c"), ("+",)], "<", [L(0)])])
    assert got[0].startswith("ok") and got[2].startswith("ok"), got
    assert got[1] == "refused -6 filter scan: ((a * b) * c) needs a decimal of more than 38 digits", got[1]
    assert got[3] == "refused -6 filter scan: (((a * b) + c) + c) needs a decimal of more than 38 digits", got[3]
    with pytest.raises(FX.Refused):
        FX.side_type([C("a"), C("b"), ("*",), C("c"), ("*",)], t2)
    assert FX.side_type([C("a"), C("b"), ("*",), C("c"), ("+",)], t) == FX.T(FX.DEC, 38, 0)


def test_integer_literal_minimum_precision(native):
    # decimal(18,18) + 5: the literal is decimal(1,0), so (max(0, 1) + 18 + 1) = 20 digits; a long column would be 39
    got = run(native, ["resolve " + case({"a": "decimal(18,18)"}, [C("a"), L(5), ("+",)], "<", [L(0)]),
                       "resolve " + case({"a": "decimal(18,18)", "k": "long"}, [C("a"), C("k"), ("+",)], "<", [L(0)])])
    assert got[0].startswith("ok")
    assert got[1] == "refused -6 filter scan: (a + k) needs a decimal of more than 38 digits"
    assert FX.side_type([C("a"), L(5), ("+",)], {"a": "decimal(18,18)"}) == FX.T(FX.DEC, 20, 18)


def test_check_exprs(native):
    got = run(native, ["check 0 1 0 c:a | i:1", "check 15 1 1 c:a c:b + | c:c", "check 16 1 0 c:a | i:1",
                       "check 0 0 0 c:a | i:1", "check 0 1 2 c:a | i:1", "check 0 1 0 | i:1", "check 0 1 0 c:a +  | i:1",
                       "check 0 1 0 c:a c:b | i:1", "check 0 1 0 k:99 | i:1", "check 0 1 0 c:- | i:1", "check 0 1 0 t:9:1 | i:1",
                       "check 0 1 0 t:0:3000000000 | i:1", "check 0 1 0 m:1:39 | i:1",
                       "check 0 1 0 " + " ".join(["c:a"] * 9) + " " + " ".join(["+"] * 8) + " | i:1",
                       "check 0 1 0 " + " ".join(["c:a"] * 8) + " " + " ".join(["+"] * 7) + " | i:1",
                       "check 0 1 0 c:a " + " ".join(["neg"] * 32) + " | i:1"])
    assert got[0] == got[1] == got[14] == "ok"
    assert got[2] == "refused -6 filter scan: more than 16 predicates and terms"
    assert got[3] == "refused -1 filter scan: expression comparison 0 has an unknown operator 0"
    assert got[4] == "refused -1 filter scan: expression comparison 0 has unknown flags 0x2"
    assert got[5] == "refused -1 filter scan: expression comparison 0 has an empty left side"
    assert got[6] == "refused -1 filter scan: the left side of expression comparison 0 underflows its stack"
    assert got[7] == "refused -1 filter scan: the left side of expression comparison 0 leaves 2 values"
    assert got[8] == "refused -1 filter scan: expression comparison 0 has a node of unknown kind 99"
    assert got[9] == "refused -1 filter scan: expression comparison 0 has a column node without a name"
    assert got[10] == "refused -1 filter scan: expression comparison 0 has a literal of unknown type 9"
    assert got[11] == "refused -1 filter scan: expression comparison 0 has an int literal outside int32"
    assert got[12] == "refused -1 filter scan: expression comparison 0 has a decimal literal of scale 39"
    assert got[13] == "refused -6 filter scan: the left side of expression comparison 0 is deeper than 8 values"
    assert got[15] == "refused -6 filter scan: the left side of expression comparison 0 has more than 32 nodes"


def test_check_filters_order_with_expressions_on_both_sides(native):
    # every side's predicates before any side's expression comparisons, the left side before the right one
    got = run(native, ["sides 1 1 1 5", "sides 1 9 0 1", "sides 1 9 1 8", "sides 1 1 1 0"])
    assert got[0] == "ok"
    assert got[1] == "refused -1 filter scan: predicate without a column"
    assert got[2] == "refused -1 filter scan: expression comparison 0 has an unknown operator 9"
    assert got[3] == "refused -1 filter scan: expression comparison 0 has an unknown operator 0"


# ---- values ----------------------------------------------------------------------------------------------------------------

I32_MIN, I32_MAX, I64_MIN, I64_MAX = -2**31, 2**31 - 1, -2**63, 2**63 - 1


def test_int_wrap_and_remainder(native):
    ints = [0, 1, -1, 7, -7, 3, -3, 65536, 46341, I32_MIN, I32_MAX]
    rows = [{"a": a, "b": b} for a in ints for b in ints] + [{"a": None, "b": 1}, {"a": 1, "b": None}]
    exprs = [([C("a"), C("b"), (op,)], cmp, [L(v)]) for op in ("+", "-", "*", "%") for cmp, v in (("=", 0), ("<", 0), (">", 1))]
    exprs += [([C("a"), ("neg",)], "=", [C("a")]), ([C("a"), C("b"), ("%",)], "=", [C("a")]),
              ([C("a"), C("b"), ("*",)], "=", [L(2**31 + 1)])]  # int * int wraps before it meets the long literal
    check_rows(native, {"a": "integer", "b": "integer"}, exprs, rows)
    longs = [0, 1, -1, 7, -7, 2**32, I64_MIN, I64_MAX]
    rows = [{"a": a, "b": b} for a in longs for b in longs]
    check_rows(native, {"a": "long", "b": "long"}, [([C("a"), C("b"), (op,)], "<", [L(0)]) for op in ("+", "-", "*", "%")], rows)
    check_rows(native, {"a": "integer", "b": "long"}, [([C("a"), C("b"), ("*",)], ">", [L(2**40)])],
               [{"a": I32_MAX, "b": 2**20}, {"a": 3, "b": I64_MAX}])
    assert FX.holds([C("a"), C("b"), ("%",)], "=", [L(0)], False, {"a": ("integer", I32_MIN), "b": ("integer", -1)})
    assert FX.holds([C("a"), L(3), ("%",)], "=", [L(-1)], False, {"a": ("integer", -7)})


def test_division_and_remainder_by_zero_are_null(native):
    zs = [0.0, -0.0, 1.0, float("nan"), float("inf")]
    rows = [{"a": a, "b": b} for a in [1.0, -1.0, 0.0, float("nan")] for b in zs]
    exprs = [([C("a"), C("b"), (op,)], cmp, [L(0.0)]) for op in ("/", "%") for cmp in ("<", "<=>", ">=")]
    exprs += [([C("a"), C("b"), ("/",)], "<=>", [C("a"), C("b"), ("%",)])]
    check_rows(native, {"a": "double", "b": "double"}, exprs, rows)
    check_rows(native, {"a": "float", "b": "float"}, exprs, rows)
    rows = [{"a": a, "b": b} for a in [5, -5, 0] for b in [0, 2, -2]]
    check_rows(native, {"a": "integer", "b": "integer"}, [([C("a"), C("b"), ("/",)], "<=>", [L(2.5)]),
                                                         ([C("a"), C("b"), ("%",)], "<=>", [L(1)])], rows)
    check_rows(native, {"a": "decimal(9,2)", "b": "decimal(5,1)"}, [([C("a"), C("b"), ("%",)], "<=>", [L(decimal.Decimal("0.5"))])],
               [{"a": a, "b": b} for a in [150, -150, 5] for b in [0, 10, -10, 3]])


def test_decimal_results_and_scales(native):
    t = {"a": "decimal(9,2)", "b": "decimal(5,1)", "k": "integer", "l": "long"}
    vals = [0, 1, -1, 999999999, -999999999, 12345, 50]
    rows = [{"a": a, "b": b, "k": k, "l": l} for a in vals for b in [0, 1, -99999, 25] for k in [0, 3, I32_MIN] for l in [0, -7, I64_MAX]]
    exprs = [([C("a"), C("b"), (op,)], "<", [L(decimal.Decimal("0.123"))]) for op in ("+", "-", "*", "%")]
    exprs += [([C("a"), C("k"), ("*",)], ">=", [C("b"), C("l"), ("-",)]), ([C("a"), L(3), ("%",)], "=", [L(decimal.Decimal("0.5"))]),
              ([C("a"), ("neg",)], "<=>", [C("b"), C("b"), ("+",)]), ([C("a"), C("b"), ("*",)], "=", [L(0.25)])]
    check_rows(native, t, exprs, rows)


def test_double_operations_are_not_fused(native):
    # cases where a * b + c rounded once (fused) differs from rounding the product first
    rng = random.Random(7)
    rows = []
    while len(rows) < 40:
        a, b = rng.uniform(-1e3, 1e3), rng.uniform(-1e3, 1e3)
        c = -float(np.float64(a) * np.float64(b))
        unfused = float(np.float64(a) * np.float64(b) + np.float64(c))
        fused = float(Fraction(a) * Fraction(b) + Fraction(c))
        if unfused != fused:
            rows.append({"a": a, "b": b, "c": c})
    assert rows
    check_rows(native, {"a": "double", "b": "double", "c": "double"},
               [([C("a"), C("b"), ("*",), C("c"), ("+",)], "=", [L(0.0)]), ([C("a"), C("b"), ("*",), C("c"), ("-",)], "<", [L(0.0)])], rows)
    for r in rows:  # the unfused product plus c is exactly 0; the fused one is not
        assert FX.holds([C("a"), C("b"), ("*",), C("c"), ("+",)], "=", [L(0.0)], False, {k: ("double", v) for k, v in r.items()})
    frows = []
    while len(frows) < 40:
        a, b = np.float32(rng.uniform(-1e3, 1e3)), np.float32(rng.uniform(-1e3, 1e3))
        frows.append({"a": float(a), "b": float(b), "c": float(-(a * b))})
    check_rows(native, {"a": "float", "b": "float", "c": "float"}, [([C("a"), C("b"), ("*",), C("c"), ("+",)], "=", [L(0)])], frows)


def test_nan_negative_zero_nulls_and_null_safe(native):
    fl = [float("nan"), -0.0, 0.0, 1.0, float("inf"), float("-inf"), None]
    rows = [{"a": a, "b": b} for a in fl for b in fl]
    exprs = [([C("a"), L(0.0), ("+",)], op, [C("b"), ("neg",)]) for op in OPS]
    check_rows(native, {"a": "double", "b": "double"}, exprs, rows)
    check_rows(native, {"a": "float", "b": "integer"}, [([C("a"), C("b"), ("+",)], op, [C("b")]) for op in OPS],
               [{"a": a, "b": b} for a in fl for b in [0, 16777217, None]])


def test_random_programs_against_the_oracle(native):
    rng = random.Random(3)
    types = {"i": "integer", "l": "long", "f": "float", "d": "double", "m": "decimal(9,2)", "n": "decimal(18,3)"}
    gen = {"i": lambda: rng.choice([0, 1, -1, rng.randrange(-2**31, 2**31)]), "l": lambda: rng.choice([0, -3, rng.randrange(-2**63, 2**63)]),
           "f": lambda: float(np.float32(rng.uniform(-1e4, 1e4))), "d": lambda: rng.choice([0.0, -0.0, rng.uniform(-1e6, 1e6)]),
           "m": lambda: rng.randrange(-10**9 + 1, 10**9), "n": lambda: rng.choice([0, rng.randrange(-10**18 + 1, 10**18)])}
    rows = [{c: (None if rng.random() < 0.1 else g()) for c, g in gen.items()} for _ in range(40)]
    lits = [1, -2, 7, 2**40, 0.5, -1.25, decimal.Decimal("0.05"), decimal.Decimal("-12.5")]

    def side(depth):
        if depth == 0 or rng.random() < 0.3:
            return [C(rng.choice(list(types)))] if rng.random() < 0.7 else [L(rng.choice(lits))]
        if rng.random() < 0.15:
            return side(depth - 1) + [("neg",)]
        return side(depth - 1) + side(depth - 1) + [(rng.choice(FX.OPS),)]

    exprs = []
    while len(exprs) < 120:
        e = (side(3), rng.choice(list(OPS)), side(2))
        try:
            FX.holds(e[0], e[1], e[2], False, {c: (t, None) for c, t in types.items()})
        except FX.Refused:
            continue
        exprs.append(e)
    check_rows(native, types, exprs, rows)


# ---- the Python forms ------------------------------------------------------------------------------------------------------

def test_python_forms():
    from hyperspace_b200.session import col

    cases = [(col("a") + col("b") < col("c"), "((a + b) < c)"), (col("p") * (1 - col("d")) > 100, "((p * (1 - d)) > 100)"),
             (col("k") % 7 == 0, "((k % 7) = 0)"), (col("v2") / col("v4") > 1.5, "((v2 / v4) > 1.5)"),
             (2 * col("a") <= col("b") - 1, "((2 * a) <= (b - 1))"), (10 / col("a") >= 1, "((10 / a) >= 1)"),
             (5 % col("a") != 0, "NOT ((5 % a) = 0)"), (-col("a") == col("b"), "((- a) = b)"),
             (col("a") + 1 - col("b") < 3, "(((a + 1) - b) < 3)"), ((col("a") + 1).eqNullSafe(col("b")), "((a + 1) <=> b)"),
             (~(col("a") * 2 > 1), "NOT ((a * 2) > 1)"), (col("a") > col("b") + decimal.Decimal("0.05"), "(a > (b + 0.05))"),
             (100 < col("a") * 3, "((a * 3) > 100)")]
    for p, text in cases:
        e, = p.exprs
        assert str(e) == text
        assert not p.bounds and not p.anys and not p.compares
    e, = (col("a") + col("b") < col("c")).exprs
    assert e.as_native() == ([("column", "a"), ("column", "b"), ("+",)], "<", [("column", "c")], 0)
    p = col("k").between(col("a") + 1, 9)
    assert [str(x) for x in p.exprs] == ["(k >= (a + 1))"] and p.terms == [("k", "<=", 9)] and p.columns == ["k", "a"]
    p = (col("a") * 2 < col("b")) & (col("k") > 5) & (col("a") < col("c"))
    assert len(p.exprs) == 1 and len(p.compares) == 1 and set(p.columns) == {"a", "b", "k", "c"}
    assert (col("x") + 1).between(0, 2).exprs[1].op == "<="


def test_python_refusals(tmp_path):
    from hyperspace_b200 import log_entry as LE
    from hyperspace_b200.session import col

    with pytest.raises(LE.HyperspaceException, match="OR across columns"):
        (col("a") + 1 < 3) | (col("a") > 5)
    with pytest.raises(LE.HyperspaceException, match="OR across columns"):
        (col("a") > 5) | (col("a") % 2 == 0)
    with pytest.raises(LE.HyperspaceException, match="OR across columns"):
        (col("a") + 1).isin(1, 2)
    with pytest.raises(LE.HyperspaceException, match="OR across columns"):
        col("k").isin(1, col("a") + 1)
    with pytest.raises(LE.HyperspaceException, match="a NOT over several columns"):
        ~((col("a") + 1 < 3) & (col("a") > 1))
    with pytest.raises(LE.HyperspaceException, match="cannot be used in arithmetic"):
        col("a") + "x"
    df = _fabricated(tmp_path, ["k"], ["v1", "v2"], [("k", "long"), ("v1", "long"), ("v2", "double"), ("w", "long")])
    with pytest.raises(LE.HyperspaceException, match="is not a filter"):
        df.filter(col("v1") + 1)


def test_filter_rule_and_explain(tmp_path):
    from hyperspace_b200.session import col

    df = _fabricated(tmp_path, ["k"], ["v1", "v2"], [("k", "long"), ("v1", "long"), ("v2", "double"), ("w", "long")])
    plan = df.filter((col("K") > 3) & (col("V1") + col("v2") < col("k"))).select("k", "v2").explain()
    assert "Name: idx" in plan and "where=(((v1 + v2) < k))" in plan, plan
    # the key only inside an expression: the index still serves
    plan = df.filter(col("k") % 7 == 0).select("k").explain()
    assert "Name: idx" in plan and "where=(((k % 7) = 0))" in plan, plan
    # w is not covered: no index
    assert df.filter(col("k") * 2 < col("w")).select("k").explain().startswith("GpuSourceScan")
    e, = df.filter(col("V2") / col("V1") > 1.5).plan.predicate.exprs
    assert str(e) == "((v2 / v1) > 1.5)"


def test_expression_across_join_sides_is_refused(tmp_path):
    from hyperspace_b200 import log_entry as LE
    from hyperspace_b200.session import DataFrame, RelationNode, col

    a = _fabricated(tmp_path, ["k"], ["v1", "v2"], [("k", "long"), ("v1", "long"), ("v2", "double"), ("w", "long")])
    b = DataFrame(a.session, RelationNode([f"file:{tmp_path}/u"], [(f"file:{tmp_path}/u/a.parquet", 100, 1)], [("k2", "long"), ("x", "long")]))
    j = a.join(b, on=("k", "k2"))
    with pytest.raises(LE.HyperspaceException, match="non-equi join condition"):
        j.filter(col("v1") + col("x") > 3)
    with pytest.raises(LE.HyperspaceException, match="non-equi join condition"):
        a.join(b, on=col("v1") + 1 < col("x"))
    plan = a.filter(col("v1") * 2 < col("w")).join(b.filter(col("k2") % 3 == 1), on=("k", "k2")).explain()
    assert "where=(((v1 * 2) < w))" in plan and "where=(((k2 % 3) = 1))" in plan, plan
