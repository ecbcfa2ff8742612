"""Host-side tests of NOT, null tests, null-safe equality and string patterns in filter terms: the resolution in
hyperspace_b200/csrc/predicates.h and the matcher in string_match.h, built as host code under AddressSanitizer where the
compiler has it, and the Python forms of the session layer."""
import os
import random
import re
import shutil
import subprocess

import numpy as np
import pytest

import filter_terms_oracle as FT
import test_predicates_host as PH

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INT32, INT64, FLOAT, DOUBLE, BOOL, STRING, DECIMAL = range(7)
NOT, NULL_TRUE, NULL_FALSE, STARTS, ENDS, CONTAINS, LIKE = 1, 2, 4, 8, 16, 32, 64


@pytest.fixture(scope="module")
def native(tmp_path_factory):
    if shutil.which("nvcc") is None:
        pytest.skip("nvcc not on PATH")
    exe = str(tmp_path_factory.mktemp("filter_terms") / "filter_terms")
    base = ["nvcc", "-std=c++17", "-O1", "-g", "-Wno-deprecated-gpu-targets", "-o", exe,
            os.path.join(ROOT, "tests", "native", "filter_terms.cu")]
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


def tsets(native, column, cases):
    """resolve_any of (flags, term) cases: (exact, ranges) or (code, message)."""
    out = []
    for line in run(native, [f"tset {column} {flags} {t}" for flags, t in cases]):
        if line.startswith("refused"):
            out.append(PH._parse(line))
        else:
            _, exact, rest = (line + " ").split(" ", 2)
            out.append((exact == "1", PH._parse("ok " + rest.strip())))
    return out


HARD = [(f"{INT32} p 0", PH.I32, [5, -2**31, 2**31 - 1, 16777217, 2.5]),
        (f"{INT64} p 0", PH.I64, [PH.T53 + 1, -2**63, 2**63 - 1, float(PH.T53), 0]),
        (f"{FLOAT} p 0", PH.F32, [float("nan"), -0.0, float("inf"), 16777217, 0.1]),
        (f"{DOUBLE} p 0", PH.F64, [float("nan"), -0.0, float("-inf"), PH.T53 + 1, 1.5]),
        (f"{STRING} p 0", PH.STR, [b"", b"a", b"ab", b"\xff", b"\xff\xff", b"a\x00"])]


@pytest.mark.parametrize("column,values,lits", HARD, ids=["int32", "int64", "float", "double", "string"])
def test_complement_partitions_the_domain(native, column, values, lits):
    """A set and its NOT: their union is every value, and they are disjoint -- for points, lists, one-sided and two-sided
    ranges over the hard values."""
    terms = [PH.term([v], []) for v in lits] + [PH.term(lits[:3], []), PH.term([], [])]
    lo, hi = lits[1], lits[2]
    if isinstance(lo, bytes) == isinstance(hi, bytes) and type(lo) is type(hi):
        terms += [PH.term([], [(lo, False, None, False)]), PH.term([], [(None, False, hi, True)]),
                  PH.term([], [(lo, True, hi, False), (lits[0], False, lits[0], False)])]
    got = tsets(native, column, [(f, t) for t in terms for f in (0, NOT)])
    for k in range(0, len(got), 2):
        (e0, s0), (e1, s1) = got[k], got[k + 1]
        assert e0 and e1
        m0, m1 = PH.select(values, s0), PH.select(values, s1)
        assert (m0 | m1).all() and not (m0 & m1).any(), terms[k // 2]


def test_not_of_a_point_is_two_ranges(native):
    (_, s), = tsets(native, f"{INT64} p 0", [(NOT, PH.term([5], []))])
    assert len(s) == 2
    (_, s), = tsets(native, f"{DOUBLE} p 0", [(NOT, PH.term([-0.0], []))])  # both zeros go
    assert PH.select(PH.F64, s).tolist() == [not (x == 0.0) for x in PH.F64]


@pytest.mark.parametrize("p", [b"", b"a", b"ab", b"a\xff", b"\xff", b"\xff\xff", b"\x00", "é".encode()])
def test_prefix_range_selects_the_prefixed_values(native, p):
    values = np.array(list(PH.STR) + [b"a\xff\x00", b"b\x00", b"\xfe\xff", "é!".encode(), b"\x00\x01"], dtype=object)
    line, = run(native, [f"prefix {p.hex() or '-'}"])
    ranges = PH._parse(line)
    assert PH.select(values, ranges).tolist() == [v.startswith(p) for v in values]
    (exact, s), = tsets(native, f"{STRING} p 0", [(STARTS, PH.term([p], []))])
    assert exact and PH.select(values, s).tolist() == [v.startswith(p) for v in values]


def test_like_prefixes_and_equalities_are_ranges(native):
    got = tsets(native, f"{STRING} p 0", [(LIKE, PH.term([b"abc%"], [])), (LIKE, PH.term([b"abc"], [])),
                                          (LIKE, PH.term([b"a_c%"], [])), (LIKE, PH.term([b"a\\%%"], [])),
                                          (ENDS, PH.term([b""], [])), (CONTAINS, PH.term([b"x"], [])),
                                          (LIKE | NOT, PH.term([b"a%b"], []))])
    assert got[0] == (True, [(True, False, "616263", True, True, "616264")])
    assert got[1] == (True, [(True, False, "616263", True, False, "616263")])
    assert got[2] == (False, [(True, False, "61", True, True, "62")])        # bounds only: the matcher decides
    assert got[3] == (True, [(True, False, "6125", True, True, "6126")])       # an escaped % is a literal byte
    assert got[4][0] and got[5] == (False, [(True, False, "-", False, False, "-")])
    assert got[6] == (False, [(False, False, "-", False, False, "-")])


def test_like_refusals_carry_sparks_messages(native):
    got = run(native, ["like " + b"ab\\".hex(), "like " + b"a\\b".hex(), "like " + "a\\é".encode().hex(),
                       "like " + b"a\\%\\_\\\\%_".hex()])
    assert got[0] == "refused -1 the pattern 'ab\\' is invalid, it is not allowed to end with the escape character"
    assert got[1] == "refused -1 the pattern 'a\\b' is invalid, the escape character is not allowed to precede 'b'"
    assert got[2] == "refused -1 the pattern 'a\\é' is invalid, the escape character is not allowed to precede 'é'"
    assert got[3] == "ok 61 25 5f 5c % _"
    for pat in ("ab\\", "a\\b"):
        with pytest.raises(ValueError) as e:
            FT.like_regex(pat)
        assert str(e.value) in got[0] + got[1]


def test_check_anys_flags(native):
    s1 = PH.term([b"ab"], [])
    got = run(native, [f"checkt {f} {t}" for f, t in [
        (128, s1), (NULL_TRUE | NULL_FALSE, s1), (STARTS | ENDS, s1), (LIKE, PH.term([b"a", b"b"], [])),
        (LIKE, PH.term([5], [])), (CONTAINS, PH.term([b"a"], [(b"a", False, None, False)])), (LIKE, PH.term([b"a\\"], [])),
        (LIKE | NOT | NULL_FALSE, s1), (NOT | NULL_TRUE, PH.term([], []))]])
    assert [g.split(" ")[1] if g != "ok" else "ok" for g in got] == ["-1"] * 7 + ["ok", "ok"]
    assert "unknown flags" in got[0] and "two null outcomes" in got[1] and "more than one pattern" in got[2]
    assert "one string value and no ranges" in got[3] and "escape character" in got[6]


def test_patterns_and_flags_refused_on_other_columns(native):
    got = tsets(native, f"{INT64} p 0", [(CONTAINS, PH.term([b"1"], []))])
    assert got[0][0] == -6 and "string pattern" in got[0][1]
    got = tsets(native, f"{BOOL} p 0", [(NULL_TRUE, PH.term([], [])), (0, PH.term([], []))])
    assert got[0][0] == -6 and got[1] == (True, [])


# ---- the matcher against Python's re -----------------------------------------------------------------------------------

ALPHABET = ["a", "b", "_", "%", "\\", "é", "€", "𝄞", "\n", "ab"]


def _random_text(rng, n):
    return "".join(rng.choice(ALPHABET) for _ in range(n))


def _random_like(rng):
    out = []
    for _ in range(rng.randint(0, 6)):
        r = rng.random()
        out.append("%" if r < 0.25 else "_" if r < 0.45 else ("\\" + rng.choice("%_\\")) if r < 0.55 else rng.choice(ALPHABET[:2] + ALPHABET[5:9]))
    return "".join(out)


def test_matcher_agrees_with_re_on_random_utf8(native):
    rng = random.Random(7)
    values = [_random_text(rng, rng.randint(0, 12)) for _ in range(60)] + ["", "a", "ab", "𝄞𝄞"]
    lines, want = [], []
    for _ in range(400):
        kind = rng.choice([LIKE, LIKE, ENDS, CONTAINS])
        pat = _random_like(rng) if kind == LIKE else _random_text(rng, rng.randint(0, 3))
        enc = [v.encode() for v in values]
        lines.append(f"match {kind} {pat.encode().hex() or '-'} {len(enc)} " + " ".join(e.hex() or "-" for e in enc))
        if kind == LIKE:
            rx = re.compile(FT.like_regex(pat))
            want.append([rx.fullmatch(v) is not None for v in values])
        else:
            p = pat.encode()
            want.append([e.endswith(p) if kind == ENDS else p in e for e in enc])
    for line, w, case in zip(run(native, lines), want, lines):
        assert line.split()[1:] == [str(int(x)) for x in w], case


def test_matcher_on_repetitive_segments(native):
    """every pattern over {a, b} of up to 5 letters against every value of up to 8: the KMP search of literal segments
    (borders, restarts after a partial match) as Contains, EndsWith and LIKE '%p%q' / '%p%' / 'p%q%r'"""
    import itertools

    words = [""] + ["".join(w) for n in range(1, 9) for w in itertools.product("ab", repeat=n)]
    pats = ["".join(w) for n in range(1, 6) for w in itertools.product("ab", repeat=n)]
    enc = " ".join(w.encode().hex() or "-" for w in words)
    lines, want = [], []
    for p in pats:
        for kind, like in ((CONTAINS, None), (ENDS, None), (LIKE, f"%{p}%"), (LIKE, f"%{p}%{p[::-1]}"), (LIKE, f"{p[:1]}%{p}%{p[-1:]}")):
            pat = like if like is not None else p
            lines.append(f"match {kind} {pat.encode().hex()} {len(words)} {enc}")
            if kind == CONTAINS:
                want.append([p in w for w in words])
            elif kind == ENDS:
                want.append([w.endswith(p) for w in words])
            else:
                rx = re.compile(FT.like_regex(pat))
                want.append([rx.fullmatch(w) is not None for w in words])
    for line, w, case in zip(run(native, lines), want, lines):
        assert line.split()[1:] == [str(int(x)) for x in w], case.split()[:3]


# ---- the Python forms ----------------------------------------------------------------------------------------------------

def test_python_forms():
    from hyperspace_b200.session import Predicate, col

    assert isinstance(col("k") != 5, Predicate)
    cases = [(col("k") != 5, "NOT (k IN (5))", ("k", [5], [], NOT)),
             (col("k").isNull(), "k IS NULL", ("k", [], [], NULL_TRUE)),
             (col("k").isNotNull(), "k IS NOT NULL", ("k", [], [], NOT | NULL_TRUE)),
             (col("k").eqNullSafe(5), "k <=> 5", ("k", [5], [], NULL_FALSE)),
             (~col("k").eqNullSafe(5), "NOT (k <=> 5)", ("k", [5], [], NOT | NULL_FALSE)),
             (col("k").eqNullSafe(None), "k IS NULL", ("k", [], [], NULL_TRUE)),
             (~col("k").isin(1, None), "NOT (k IN (1))", ("k", [], [])),
             (~col("k").isin(1, 2), "NOT (k IN (1, 2))", ("k", [1, 2], [], NOT)),
             (~(col("k") >= 3), "NOT (k >= 3)", ("k", [], [(3, False, None, False)], NOT)),
             (col("s").startswith("ab"), "StartsWith(s, 'ab')", ("s", ["ab"], [], STARTS)),
             (col("s").endswith("ab"), "EndsWith(s, 'ab')", ("s", ["ab"], [], ENDS)),
             (col("s").contains("ab"), "Contains(s, 'ab')", ("s", ["ab"], [], CONTAINS)),
             (col("s").like("a%b"), "s LIKE 'a%b'", ("s", ["a%b"], [], LIKE)),
             (~col("s").like("a%b"), "NOT (s LIKE 'a%b')", ("s", ["a%b"], [], LIKE | NOT)),
             (col("k").isNull() | (col("k") > 5), "k > 5 OR k IS NULL", ("k", [], [(5, True, None, False)], NULL_TRUE)),
             (col("k").eqNullSafe(1) | col("k").eqNullSafe(2), "k <=> 1 OR k <=> 2", ("k", [1, 2], [], NULL_FALSE)),
             (col("s").startswith("a\xff") | (col("s") == "z"), None, ("s", [], [("a\xff", False, b"a\xc3\xc0", True), ("z", False, "z", False)])),
             (~(col("k").isin(1, None) | col("k").isNull()), None, ("k", [], []))]
    for p, text, native_form in cases:
        a, = p.anys
        if text is not None:
            assert str(a) == text
        assert a.as_native() == native_form, text


def test_python_refusals():
    from hyperspace_b200 import log_entry as LE
    from hyperspace_b200.session import col

    with pytest.raises(LE.HyperspaceException, match="several columns"):
        ~((col("a") > 1) & (col("b") > 1))
    with pytest.raises(LE.HyperspaceException, match="NOT inside an OR"):
        (col("k") != 1) | (col("k") > 5)
    with pytest.raises(LE.HyperspaceException, match="like pattern inside an OR"):
        col("s").like("a%b") | col("s").isNull()
    with pytest.raises(LE.HyperspaceException, match="OR across columns"):
        col("a").isNull() | col("b").isNull()
    with pytest.raises(LE.HyperspaceException, match="one range"):
        ~((col("k") > 1) & (col("k") > 2))
    with pytest.raises(LE.HyperspaceException, match="string pattern"):
        col("s").startswith(5)


def test_filter_rule_takes_the_new_terms_on_the_first_indexed_column(tmp_path):
    from hyperspace_b200.session import col
    from test_filter_in_host import _fabricated

    df = _fabricated(tmp_path, ["k"])
    for p, text in [(col("k") != 5, "NOT (k IN (5))"), (col("k").isNull(), "k IS NULL"), (col("k").eqNullSafe(5), "k <=> 5"),
                    (~col("k").isin(1, 2), "NOT (k IN (1, 2))"), (col("k").isNotNull(), "k IS NOT NULL")]:
        plan = df.filter(p).select("k", "v1").explain()
        assert "Name: idx" in plan and f"where=({text})" in plan, plan
    plan = df.filter(col("v1").isNull()).select("k").explain()
    assert plan.startswith("GpuSourceScan") and "where=(v1 IS NULL)" in plan
    # filter() keeps the new fields when it resolves the column's spelling
    a, = df.filter(~col("K").eqNullSafe(5)).plan.predicate.anys
    assert (a.column, a.null, a.negated) == ("k", False, True)


def test_oracle_three_valued_logic():
    cols = {"k": np.array([1, 2, 3, 0], dtype=np.int64), "s": np.array([b"ab", b"xb", "é".encode(), b""], dtype=object)}
    valids = {"k": np.array([1, 1, 1, 0], bool), "s": np.array([1, 1, 1, 0], bool)}
    m = lambda *t: FT.mask(cols, list(t), valids).tolist()  # noqa: E731
    assert m(("not", ("in", "k", [1]))) == [False, True, True, False]
    assert m(("not", ("in", "k", [1, None]))) == [False] * 4
    assert m(("not", ("eqns", "k", 1))) == [False, True, True, True]
    assert m(("isnull", "k")) == [False, False, False, True]
    assert m(("or", [("isnull", "k"), ("range", "k", 3, False, None, False)])) == [False, False, True, True]
    assert m(("like", "s", "_b")) == [True, True, False, False]
    assert m(("not", ("endswith", "s", b"b"))) == [False, False, True, False]
