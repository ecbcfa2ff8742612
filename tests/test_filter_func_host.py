"""Host-side tests of the Spark functions in expression comparisons (`year(d) = 1995`, `substring(s, 1, 2) = '13'`,
`datediff(a, b) > 30`, `abs`, `coalesce`): the typing in hyperspace_b200/csrc/predicates.h (resolve_expr, check_exprs) and
the evaluator in column_expr.h (expr_holds<true>, date_part), built as host code under AddressSanitizer where the compiler
has it, against tests/filter_func_oracle.py; and the Python forms of hyperspace_b200/functions.py."""
import datetime
import decimal
import itertools
import os
import random
import shutil
import subprocess

import numpy as np
import pytest

import filter_func_oracle as FF
from test_filter_compare_host import _fabricated

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OPS = {"<": 1, "<=": 2, ">": 3, ">=": 4, "=": 5, "<=>": 6}
I32_MIN, I32_MAX, I64_MIN, I64_MAX = -2**31, 2**31 - 1, -2**63, 2**63 - 1
DAY_US = FF.DAY_US


@pytest.fixture(scope="module")
def native(tmp_path_factory):
    if shutil.which("nvcc") is None:
        pytest.skip("nvcc not on PATH")
    exe = str(tmp_path_factory.mktemp("filter_func") / "filter_func")
    base = ["nvcc", "-std=c++17", "-O1", "-g", "-Wno-deprecated-gpu-targets", "-o", exe, os.path.join(ROOT, "tests", "native", "filter_func.cu")]
    try:
        subprocess.check_call(base + ["-Xcompiler", "-fsanitize=address,-fno-omit-frame-pointer"], stderr=subprocess.DEVNULL)
        asan = subprocess.run([exe, "x"], capture_output=True).returncode == 2
    except subprocess.CalledProcessError:
        asan = False
    if not asan:
        subprocess.check_call(base)
    return exe


def run(native, lines, n_out=None):
    out = subprocess.run([native], input="\n".join(lines) + "\n", capture_output=True, text=True, check=True).stdout
    got = out.splitlines()
    assert len(got) == (len(lines) if n_out is None else n_out)
    return got


def colspec(name, t):
    if t.startswith("decimal("):
        p, s = t[len("decimal("):-1].split(",")
        return f"{name} decimal {p} {s}"
    return f"{name} {t} 0 0"


def tok(node):
    tag = node[0]
    if tag == "column":
        return f"c:{node[1]}"
    if tag == "literal":
        v = node[1]
        if isinstance(v, (str, bytes)):
            return "s:" + (v.encode() if isinstance(v, str) else v).hex()
        if isinstance(v, datetime.datetime):
            return f"T:{FF.literal_value(v)}"
        if isinstance(v, datetime.date):
            return f"D:{FF.literal_value(v)}"
        if isinstance(v, decimal.Decimal):
            s = max(0, -v.as_tuple()[2])
            return f"m:{int(v.scaleb(s))}:{s}"
        if isinstance(v, float):
            return f"d:{v!r}"
        return f"i:{v}" if -2**31 <= v < 2**31 else f"l:{v}"
    if tag == "coalesce":
        return f"coalesce:{node[1]}"
    return tag


def case(types, left, op, right, negated=False):
    cols = " ".join(colspec(n, t) for n, t in types.items())
    return (f"{len(types)} {cols} {OPS[op]} {int(negated)} " + " ".join(tok(n) for n in left) + " | " +
            " ".join(tok(n) for n in right) + " ;")


def fmt(v):
    if isinstance(v, (bytes, bytearray)):
        return "h" + bytes(v).hex()
    if isinstance(v, (float, np.floating)):
        return "nan" if v != v else ("inf" if v == float("inf") else ("-inf" if v == float("-inf") else repr(float(v))))
    return str(int(v))


def check_rows(native, types, exprs, rows, negations=(False, True)):
    """Every expression (left, op, right) under NOT and without, over the rows (dicts of column -> value or None), against
    the oracle."""
    names = list(types)
    null_token = {"string": "h", "binary": "h"}
    data = " ".join(f"{int(r[n] is None)} {null_token.get(types[n], '0') if r[n] is None else fmt(r[n])}" for r in rows for n in names)
    lines, want, which = [], [], []
    for (left, op, right), neg in itertools.product(exprs, negations):
        lines.append(f"rows {case(types, left, op, right, neg)} {len(rows)} {data}")
        orow = [{n: (types[n], r[n]) for n in names} for r in rows]
        want.append("ok" + "".join(f" {int(FF.holds(left, op, right, neg, o))}" for o in orow))
        which.append((left, op, right, neg))
    for line, w, e in zip(run(native, lines), want, which):
        assert line == w, (e, line, w)


def C(n):
    return ("column", n)


def L(v):
    return ("literal", v)


def F(name, *args):
    """A function node over argument sides (each a list of nodes)."""
    out = [n for a in args for n in a]
    return out + [("coalesce", len(args)) if name == "coalesce" else (name,)]


# ---- typing -------------------------------------------------------------------------------------------------------------------

ARG_TYPES = ["integer", "long", "float", "double", "decimal(9,2)", "decimal(20,2)", "string", "binary", "date", "timestamp",
             "boolean", "byte"]


def _signature_lines(side, types):
    """Lines whose outcomes pin a side's type: itself compared, plus an int addition, a string literal and a date literal."""
    return ["resolve " + case(types, side, "<=>", side), "resolve " + case(types, side + [L(1), ("+",)], "<", [L(0)]),
            "resolve " + case(types, side, "=", [L("x")]), "resolve " + case(types, side, "=", [L(datetime.date(2000, 1, 1))])]


def _expect_signature(t, got, what):
    """The outcomes _signature_lines gives for a side of type t (None: refused)."""
    if t is None:
        assert got[0].startswith("refused -6"), (what, got[0])
        return
    domain = {FF.FLOAT: 1, FF.DOUBLE: 2, FF.STR: 3, FF.BIN: 3}.get(t.kind, 0)
    assert got[0].split()[:2] == ["ok", str(domain)], (what, t, got[0])
    if t.kind in FF.NUMERIC:
        arith = {FF.INT: 8, FF.LONG: 16, FF.DEC: 24, FF.FLOAT: 32, FF.DOUBLE: 40}[t.kind]
        assert got[1].startswith("ok") and str(arith) in got[1].split()[3:], (what, t, got[1])
    else:
        assert got[1].startswith("refused -6") and "cannot be used in arithmetic" in got[1], (what, t, got[1])
    assert got[2].startswith("ok") == (t.kind == FF.STR), (what, t, got[2])
    assert got[3].startswith("ok") == (t.kind in (FF.DATE, FF.TS)), (what, t, got[3])
    if t.kind in (FF.DATE, FF.TS):  # a timestamp side rescales the date literal (instruction 2)
        assert ("2" in got[3].split()[3:]) == (t.kind == FF.TS), (what, t, got[3])


def test_result_types_of_every_function_over_every_argument_type(native):
    lines, want = [], []
    sides = []
    for f in FF.DATE_PARTS + FF.TIME_PARTS + ("length", "abs"):
        for ta in ARG_TYPES:
            sides.append((F(f, [C("a")]), {"a": ta}))
    for f in ("date_add", "date_sub", "datediff"):
        for ta, tb in itertools.product(["date", "timestamp", "integer", "string"], ["integer", "byte", "long", "date", "timestamp", "double"]):
            sides.append((F(f, [C("a")], [C("b")]), {"a": ta, "b": tb}))
        sides.append((F(f, [C("a")], [L(3)]), {"a": "date"}))
        sides.append((F(f, [C("a")], [L(2**40)]), {"a": "date"}))
    for ta in ARG_TYPES:
        sides.append((F("substring", [C("a")], [L(1)], [L(2)]), {"a": ta}))
    for ta, tb in itertools.product(ARG_TYPES[:-2], ARG_TYPES[:-2]):
        sides.append((F("coalesce", [C("a")], [C("b")]), {"a": ta, "b": tb}))
    sides.append((F("coalesce", [C("a")], [L(0)]), {"a": "decimal(9,2)"}))
    sides.append((F("coalesce", [C("a")], [C("b")], [L(1.5)]), {"a": "integer", "b": "long"}))
    for side, types in sides:
        try:
            t = FF.side_type(side, types)
        except FF.Refused:
            t = None
        lines += _signature_lines(side, types)
        want.append((t, side, types))
    got = run(native, lines)
    for k, (t, side, types) in enumerate(want):
        _expect_signature(t, got[4 * k:4 * k + 4], (side, types))
    # spot checks of the restatement itself
    assert FF.side_type(F("coalesce", [C("a")], [L(0)]), {"a": "decimal(9,2)"}) == FF.T(FF.DEC, 12, 2)
    assert FF.side_type(F("coalesce", [C("a")], [C("b")]), {"a": "date", "b": "timestamp"}).kind == FF.TS
    assert FF.side_type(F("date_add", [C("a")], [C("b")]), {"a": "timestamp", "b": "short"}).kind == FF.DATE


def test_new_refusals_name_what_they_refuse(native):
    got = run(native, [
        "resolve " + case({"d": "date"}, F("hour", [C("d")]), "<", [L(1)]),
        "resolve " + case({"a": "integer"}, F("year", [C("a")]), "<", [L(1)]),
        "resolve " + case({"d": "date"}, F("date_add", [C("d")], [L(2**40)]), "<", [C("d")]),
        "resolve " + case({"a": "byte"}, F("abs", [C("a")]), "<", [L(1)]),
        "resolve " + case({"s": "string", "k": "integer"}, F("coalesce", [C("s")], [C("k")]), "<", [L(1)]),
        "resolve " + case({"s": "string", "b": "binary"}, F("substring", [C("s")], [L(1)], [L(2)]), "=", F("substring", [C("b")], [L(1)], [L(2)])),
        "resolve " + case({"d": "date"}, F("year", [C("d")]), "=", [L("1995")]),
        "resolve " + case({"d": "date"}, F("date_add", [C("d")], [L(1)]), "<", [L(5)]),
        "resolve " + case({"d": "date"}, F("date_add", [C("d")], [L(1)]) + [L(1), ("+",)], "<", [L(5)]),
        "resolve " + case({"s": "string"}, F("length", [C("s")]), "=", [L("3")]),
        "check 0 1 0 c:s i:1 c:n substring | s:",
        "check 0 1 0 c:s i:1 l:2 substring | s:",
        "check 0 1 0 c:s coalesce:1 | s:",
        "check 0 1 0 c:s c:t coalesce:3 | s:",
        "check 0 1 0 " + " ".join(["c:a"] * 9) + " coalesce:9 | i:1",
        "check 0 1 0 year | i:1",
        "check 0 1 0 c:a i:1 substring | i:1",
        "check 0 1 0 t:5:70000 | i:1",
        "check 0 1 0 t:7:3000000000 | i:1",
    ])
    assert got[0] == "refused -6 filter scan: hour(d): d (date) is not a timestamp"
    assert got[1] == "refused -6 filter scan: year(a): a (int) is not a date or timestamp"
    assert got[2] == "refused -6 filter scan: date_add(d, 1099511627776): 1099511627776 (bigint) is not an int, short or byte"
    assert got[3] == "refused -6 filter scan: abs(a) is byte or short arithmetic, which wraps at its width: not handled"
    assert got[4] == "refused -6 filter scan: coalesce(s, k) mixes k (int) with string"
    assert got[5] == "refused -6 filter scan: substring(s, 1, 2) (string) and substring(b, 1, 2) (binary) cannot be compared"
    assert got[6] == "refused -6 filter scan: year(d) (int) and 1995 (string) cannot be compared"
    assert got[7] == "refused -6 filter scan: date_add(d, 1) (date) and 5 (int) cannot be compared"
    assert got[8] == "refused -6 filter scan: date_add(d, 1) (date) cannot be used in arithmetic"
    assert got[9] == "refused -6 filter scan: length(s) (int) and 3 (string) cannot be compared"
    assert got[10] == got[11] == "refused -1 filter scan: expression comparison 0 has a SUBSTRING whose pos and len are not int literals"
    assert got[12] == "refused -1 filter scan: expression comparison 0 has a COALESCE of 1 arguments over 1 values"
    assert got[13] == "refused -1 filter scan: expression comparison 0 has a COALESCE of 3 arguments over 2 values"
    assert got[14] == "refused -6 filter scan: the left side of expression comparison 0 is deeper than 8 values"
    assert got[15] == "refused -1 filter scan: the left side of expression comparison 0 underflows its stack"
    assert got[16] == "refused -1 filter scan: the left side of expression comparison 0 underflows its stack"
    assert got[17] == "refused -1 filter scan: expression comparison 0 has a string literal of 70000 bytes, not 0..65535"
    assert got[18] == "refused -1 filter scan: expression comparison 0 has a date literal outside int32"


def test_old_messages_are_unchanged(native):
    # the arithmetic change's refusals, byte for byte, through the function driver
    got = run(native, [
        "resolve " + case({"s": "string"}, [C("s"), L(1), ("+",)], "<", [L(1)]),
        "resolve " + case({"d": "date"}, [C("d")], "<", [L(1)]),
        "resolve " + case({"d": "date"}, [C("d"), L(1), ("+",)], "<", [L(1)]),
        "resolve " + case({"t": "timestamp"}, [C("t"), ("neg",)], "<", [L(1)]),
        "resolve " + case({"t": "timestamp"}, [C("t")], "<", [L(1)]),
        "resolve " + case({"s": "string"}, [C("s")], "<", [L(1)]),
        "resolve " + case({"b": "boolean"}, [C("b")], "=", [L(1)]),
        "resolve " + case({"b": "boolean"}, [C("b")], "=", [C("b")]),
        "resolve " + case({"s": "string", "b": "binary"}, [C("s")], "=", [C("b")]),
        "resolve " + case({"d": "date", "a": "byte", "b": "short"}, [C("d")], "<", [C("a"), C("b"), ("+",)]),
        "check 0 1 0 k:99 | i:1", "check 0 1 0 t:9:1 | i:1", "check 0 1 0 t:0:3000000000 | i:1",
        "check 0 1 0 " + " ".join(["c:a"] * 9) + " " + " ".join(["+"] * 8) + " | i:1",
        "check 0 1 0 c:a " + " ".join(["year"] * 32) + " | i:1",
        "check 17 1 0 c:a | i:1",
    ])
    assert got[0] == "refused -6 filter scan: the column 's' (string) cannot be used in arithmetic"
    assert got[1] == got[2] == "refused -6 filter scan: the column 'd' (date) cannot be used in arithmetic"
    assert got[3] == got[4] == "refused -6 filter scan: the column 't' (timestamp) cannot be used in arithmetic"
    assert got[5] == "refused -6 filter scan: the column 's' (string) cannot be used in arithmetic"
    assert got[6] == got[7] == "refused -6 filter scan: the column 'b' (boolean) cannot be used in arithmetic"
    assert got[8] == "refused -6 filter scan: the column 's' (string) cannot be used in arithmetic"
    assert got[9] == "refused -6 filter scan: the column 'd' (date) cannot be used in arithmetic"
    assert got[10] == "refused -1 filter scan: expression comparison 0 has a node of unknown kind 99"
    assert got[11] == "refused -1 filter scan: expression comparison 0 has a literal of unknown type 9"
    assert got[12] == "refused -1 filter scan: expression comparison 0 has an int literal outside int32"
    assert got[13] == "refused -6 filter scan: the left side of expression comparison 0 is deeper than 8 values"
    assert got[14] == "refused -6 filter scan: the left side of expression comparison 0 has more than 32 nodes"
    assert got[15] == "refused -6 filter scan: more than 16 predicates and terms"


def test_bare_date_timestamp_and_string_sides_compare(native):
    got = run(native, ["resolve " + case({"a": "date", "b": "date"}, [C("a")], "<", [C("b")]),
                       "resolve " + case({"a": "date", "t": "timestamp"}, [C("a")], "<", [C("t")]),
                       "resolve " + case({"s": "string", "u": "string"}, [C("s")], "=", [C("u")]),
                       "resolve " + case({"d": "date"}, [C("d")], ">=", [L(datetime.date(1995, 1, 1))]),
                       "resolve " + case({"d": "date"}, [C("d")], ">=", F("date_add", [C("d")], [L(1)]))])
    assert got[0] == "ok 0 1 0 0"
    assert got[1] == "ok 0 1 0 0 2"  # the date side at slot 1 rescaled to micros
    assert got[2] == "ok 3 1 0 0"
    assert got[3] == "ok 0 1 0 1"
    assert got[4].startswith("ok 0 1")


# ---- calendar -----------------------------------------------------------------------------------------------------------------

def _calendar(native, lo, hi):
    out = subprocess.run([native], input=f"calendar {lo} {hi}\n", capture_output=True, text=True, check=True).stdout
    return np.array(out.split(), dtype=np.int64).reshape(-1, 7)


def test_calendar_against_numpy(native):
    lo, hi = -800_000, 800_000
    got = _calendar(native, lo, hi)
    want = FF.calendar(np.arange(lo, hi + 1))
    for k, part in enumerate(FF.DATE_PARTS):
        bad = np.nonzero(got[:, k] != want[part])[0]
        assert bad.size == 0, (part, lo + bad[:5], got[bad[:5], k], want[part][bad[:5]])


def test_calendar_edges(native):
    days = [I32_MIN, I32_MIN + 1, I32_MAX - 1, I32_MAX]
    days += [(datetime.date(y, 1, 1) - datetime.date(1970, 1, 1)).days + k for y in (1900, 2000, 2100) for k in (-1, 0, 59, 60)]
    days += [-719528, -719529, -719528 + 59, -719528 + 60]  # year 0 (a leap year) and its neighbours
    days += [(datetime.date(1582, 10, 4) - datetime.date(1970, 1, 1)).days, (datetime.date(1582, 10, 15) - datetime.date(1970, 1, 1)).days]
    for d in days:
        row = _calendar(native, d, d)[0]
        want = FF.calendar([d])
        assert [int(x) for x in row] == [int(want[p][0]) for p in FF.DATE_PARTS], d
    # 1582-10-04 and 1582-10-15 are eleven days apart in the proleptic calendar, not one as in the Julian switch
    a = _calendar(native, days[-2], days[-1])
    assert len(a) == 12 and list(a[0][:4]) == [1582, 4, 10, 4] and list(a[-1][:4]) == [1582, 4, 10, 15]
    assert list(_calendar(native, 0, 0)[0]) == [1970, 1, 1, 1, 5, 1, 1]  # a Thursday


def test_weekofyear_at_every_year_edge_against_isocalendar(native):
    lo = (datetime.date(1, 1, 1) - datetime.date(1970, 1, 1)).days
    hi = (datetime.date(9999, 12, 31) - datetime.date(1970, 1, 1)).days
    got = _calendar(native, lo, hi)
    for y in range(1, 10000):
        for d in (datetime.date(y, 1, 1), datetime.date(y, 12, 31)):
            k = (d - datetime.date(1970, 1, 1)).days - lo
            assert got[k, 6] == d.isocalendar()[1], d
            assert got[k, 0] == y and got[k, 4] == d.isoweekday() % 7 + 1 and got[k, 5] == d.timetuple().tm_yday, d


def test_timestamps_around_midnights_and_at_the_limits(native):
    ts = [I64_MIN, I64_MAX, 0, -1, 1]
    for day in (-719528, -1, 0, 1, 9131, 2932896):
        ts += [day * DAY_US - 1, day * DAY_US, day * DAY_US + 1]
    rows = [{"t": t, "w": None} for t in ts] + [{"t": None, "w": None}]
    exprs = [(F(f, [C("t")]), op, [L(v)]) for f in FF.DATE_PARTS + FF.TIME_PARTS for op, v in (("=", 1), (">", 30), ("<", 1970))]
    exprs += [(F("datediff", [C("t")], [L(datetime.date(1970, 1, 1))]), "<", [L(0)]),
              (F("date_add", [C("t")], [L(1)]), ">", [L(datetime.datetime(1970, 1, 1, 23, 59, 59))]),
              ([C("t")], "<", [L(datetime.date(1970, 1, 1))]), ([C("t")], "<=>", [L(datetime.date(1970, 1, 2))])]
    check_rows(native, {"t": "timestamp", "w": "timestamp"}, exprs, rows)
    # the values themselves, one expected column per part
    for f in FF.DATE_PARTS + FF.TIME_PARTS:
        want = [None if t is None else (FF.date_part(f, t // DAY_US) if f in FF.DATE_PARTS else FF.time_part(f, t)) for t in ts + [None]]
        check_rows(native, {"t": "timestamp", "w": "integer"}, [(F(f, [C("t")]), "<=>", [C("w")])],
                   [{"t": t, "w": w} for t, w in zip(ts + [None], want)], negations=(False,))
        assert all(FF.holds(F(f, [C("t")]), "<=>", [C("w")], False, {"t": ("timestamp", t), "w": ("integer", w)})
                   for t, w in zip(ts, want))


def test_date_add_and_datediff_wrap(native):
    rows = [{"a": a, "b": b} for a in (I32_MIN, I32_MAX, 0, -1, 9131) for b in (I32_MIN, I32_MAX, 0, 1, -1)]
    exprs = [(F("date_add", [C("a")], [C("b")]), op, [L(datetime.date(1970, 1, 1))]) for op in ("<", "=")]
    exprs += [(F("date_sub", [C("a")], [C("b")]), op, [L(datetime.date(1970, 1, 1))]) for op in ("<", ">")]
    check_rows(native, {"a": "date", "b": "integer"}, exprs, rows)
    check_rows(native, {"a": "date", "b": "date"}, [(F("datediff", [C("a")], [C("b")]), op, [L(v)]) for op, v in (("<", 0), (">", 30), ("=", -1))], rows)
    assert FF.evaluate(F("date_add", [C("a")], [C("b")]), {"a": ("date", I32_MAX), "b": ("integer", 1)})[1] == I32_MIN
    assert FF.evaluate(F("datediff", [C("a")], [C("b")]), {"a": ("date", I32_MIN), "b": ("date", 1)})[1] == I32_MAX


# ---- strings ------------------------------------------------------------------------------------------------------------------

STRINGS = ["", "a", "abc", "hello world", "é", "aé€😀z", "€€€", "😀😀", "日本語テキスト", "13-555-0100"]


def test_substring_grid(native):
    values = [s.encode() for s in STRINGS]
    positions = list(range(-8, 9)) + [I32_MIN, I32_MAX]
    lengths = list(range(-8, 9)) + [I32_MIN, I32_MAX]
    for kind in ("string", "binary"):
        rows_all = []
        lines, want = [], []
        for p in positions:
            for ln in lengths:
                rows = [{"s": v, "w": FF.substring(v, p, ln, kind == "binary")} for v in values] + [{"s": None, "w": None}]
                names = ["s", "w"]
                data = " ".join(f"{int(r[n] is None)} {'h' if r[n] is None else fmt(r[n])}" for r in rows for n in names)
                side = F("substring", [C("s")], [L(p)], [L(ln)])
                lines.append(f"rows {case({'s': kind, 'w': kind}, side, '<=>', [C('w')])} {len(rows)} {data}")
                want.append("ok" + " 1" * len(rows))
                rows_all.append((p, ln))
        for line, w, pl in zip(run(native, lines), want, rows_all):
            assert line == w, (kind, pl, line)
    assert FF.substring("aé€😀z".encode(), -3, 2, False) == "€😀".encode()
    assert FF.substring(b"abc", 0, 2, True) == b"ab" and FF.substring(b"abc", -5, 3, True) == b"a"


def test_length_and_string_comparisons(native):
    rows = [{"s": s.encode(), "u": u.encode()} for s in STRINGS for u in ("", "a", "é", "13")] + [{"s": None, "u": b"a"}]
    exprs = [(F("length", [C("s")]), op, [L(v)]) for op, v in (("=", 0), ("=", 3), (">", 2), ("<=>", 7))]
    exprs += [(F("substring", [C("s")], [L(1)], [L(2)]), "=", [L("13")]), ([C("s")], "<", [C("u")]),
              (F("substring", [C("s")], [L(-1)], [L(1)]), ">=", [C("u")]), ([C("s")], "<=>", [L("abc")])]
    check_rows(native, {"s": "string", "u": "string"}, exprs, rows)
    check_rows(native, {"s": "binary", "u": "binary"}, [(F("length", [C("s")]), ">", [L(3)]),
                                                        (F("substring", [C("s")], [L(2)], [L(3)]), "<", [C("u")])], rows)


# ---- abs and coalesce -----------------------------------------------------------------------------------------------------------

def test_abs(native):
    check_rows(native, {"a": "integer"}, [(F("abs", [C("a")]), op, [L(v)]) for op, v in (("<", 0), ("=", I32_MIN), ("=", 5))],
               [{"a": v} for v in (I32_MIN, I32_MAX, -5, 5, 0, None)])
    check_rows(native, {"a": "long"}, [(F("abs", [C("a")]), op, [L(v)]) for op, v in (("<", 0), ("=", I64_MIN), ("=", 5))],
               [{"a": v} for v in (I64_MIN, I64_MAX, -5, 0, None)])
    for t in ("double", "float"):
        check_rows(native, {"a": t}, [(F("abs", [C("a")]), op, [L(v)]) for op, v in (("<", 0.0), ("=", 0.0), ("=", float("nan")), ("=", 2.5))],
                   [{"a": v} for v in (-0.0, 0.0, float("nan"), -2.5, float("-inf"), None)])
    check_rows(native, {"a": "decimal(18,4)"}, [(F("abs", [C("a")]), op, [L(decimal.Decimal(v))]) for op, v in (("=", "12.5"), ("<", "0"))],
               [{"a": v} for v in (-125000, 125000, -(10**18 - 1), 0, None)])
    check_rows(native, {"a": "integer", "b": "integer"}, [(F("abs", [C("a"), C("b"), ("-",)]), "<", [L(5)])],
               [{"a": a, "b": b} for a in (0, 3, -3, I32_MIN) for b in (0, 7, I32_MAX)])


def test_coalesce(native):
    types = {"a": "integer", "b": "long", "f": "float", "d": "double", "m": "decimal(9,2)", "x": "date", "t": "timestamp", "s": "string", "u": "string"}
    vals = {"a": [None, 7, -1], "b": [None, 2**40], "f": [None, 1.5], "d": [None, -0.25], "m": [None, 1234], "x": [None, 9131],
            "t": [None, 9131 * DAY_US + 1], "s": [None, b"ab"], "u": [None, b""]}
    rng = random.Random(5)
    rows = [{c: rng.choice(v) for c, v in vals.items()} for _ in range(40)] + [{c: None for c in vals}]
    exprs = [(F("coalesce", [C("a")], [C("b")]), ">", [L(5)]), (F("coalesce", [C("a")], [C("f")]), "<=>", [L(1.5)]),
             (F("coalesce", [C("m")], [C("a")], [L(0)]), ">", [L(decimal.Decimal("0.05"))]),
             (F("coalesce", [C("d")], [C("m")]), "<", [L(0)]), (F("coalesce", [C("f")], [C("b")], [C("d")]), ">=", [L(0)]),
             (F("coalesce", [C("x")], [C("t")]), "<", [L(datetime.datetime(1995, 1, 1, 0, 0, 0, 1))]),
             (F("coalesce", [C("x")], [L(datetime.date(1995, 1, 2))]), "=", [L(datetime.date(1995, 1, 2))]),
             (F("coalesce", [C("s")], [C("u")]), "<=>", [L("")]), (F("coalesce", [C("s")], [C("u")], [L("z")]), ">", [L("a")])]
    check_rows(native, types, exprs, rows)


def test_empty_string_literals(native):
    # a program whose only string literals are empty still has its literals placed (no kXStringConst, 127, is left)
    types = {"s": "string", "u": "string"}
    exprs = [(F("coalesce", [C("s")], [C("u")]), "<=>", [L("")]), (F("substring", [C("s")], [L(1)], [L(2)]), "=", [L("")]),
             ([C("s")], "<", [L("")]), (F("length", [C("s")]), "=", F("length", [L("")]))]
    got = run(native, ["resolve " + case(types, l, op, r) for l, op, r in exprs])
    for line in got:
        assert line.startswith("ok 3 1") or line.startswith("ok 0 1"), line
        assert "127" not in line.split()[3:] and "1" in line.split()[3:], line
    rows = [{"s": s, "u": u} for s in (None, b"", b"x", b"xyz") for u in (None, b"", b"xy")]
    check_rows(native, types, exprs, rows)
    assert FF.holds(exprs[0][0], "<=>", [L("")], False, {"s": ("string", b""), "u": ("string", b"xy")})


def test_dates_promoted_to_timestamps_beyond_the_long_range(native):
    # coalesce(date, timestamp) promotes the date to micros in 128 bits: a date beyond 106 751 991 days keeps its fields
    types = {"x": "date", "t": "timestamp"}
    rows = [{"x": x, "t": None} for x in (I32_MIN, I32_MAX, -106_751_992, 106_751_992, 9131)] + [{"x": None, "t": -1}]
    promoted = F("coalesce", [C("x")], [C("t")])
    exprs = [(F(f, promoted), op, [L(v)]) for f in ("hour", "minute", "second") for op, v in (("=", 0), ("=", 59))]
    exprs += [(F(f, promoted), "=", [L(v)]) for f, v in (("year", 5881580), ("year", -5877641), ("month", 1), ("dayofmonth", 31))]
    exprs += [(F("datediff", promoted, [C("x")]), "=", [L(0)]), (F("date_add", promoted, [L(1)]), ">", [C("x")]), (promoted, ">", [C("t")])]
    check_rows(native, types, exprs, rows)
    assert FF.evaluate(F("year", promoted), {"x": ("date", I32_MAX), "t": ("timestamp", None)})[1] == 5881580


def test_random_function_programs_against_the_oracle(native):
    rng = random.Random(11)
    types = {"i": "integer", "l": "long", "d": "double", "m": "decimal(9,2)", "x": "date", "t": "timestamp", "s": "string"}
    gen = {"i": lambda: rng.randrange(-2**31, 2**31), "l": lambda: rng.randrange(-2**40, 2**40), "d": lambda: rng.uniform(-1e3, 1e3),
           "m": lambda: rng.randrange(-10**9 + 1, 10**9), "x": lambda: rng.randrange(-100_000, 100_000),
           "t": lambda: rng.randrange(-2**50, 2**50), "s": lambda: rng.choice(STRINGS).encode()}
    rows = [{c: (None if rng.random() < 0.1 else g()) for c, g in gen.items()} for _ in range(30)]
    fns = [lambda: F(rng.choice(FF.DATE_PARTS), [C(rng.choice("xt"))]), lambda: F(rng.choice(FF.TIME_PARTS), [C("t")]),
           lambda: F("datediff", [C(rng.choice("xt"))], [C(rng.choice("xt"))]), lambda: F("length", [C("s")]),
           lambda: F("abs", [C(rng.choice("ildm"))]), lambda: F("coalesce", [C(rng.choice("ildm"))], [C(rng.choice("ildm"))]),
           lambda: F("abs", F("length", F("substring", [C("s")], [L(rng.randrange(-4, 5))], [L(rng.randrange(-2, 5))])) + [C("i"), ("-",)])]
    exprs = []
    while len(exprs) < 60:
        e = (rng.choice(fns)(), rng.choice(list(OPS)), rng.choice(fns)() if rng.random() < 0.5 else [L(rng.choice([0, 1, 7, 1995, 2.5]))])
        try:
            FF.holds(e[0], e[1], e[2], False, {c: (t, None) for c, t in types.items()})
        except FF.Refused:
            continue
        exprs.append(e)
    check_rows(native, types, exprs, rows)


# ---- the Python forms -----------------------------------------------------------------------------------------------------------

def test_python_functions_build_expressions():
    from hyperspace_b200 import functions as Fn
    from hyperspace_b200.session import Expr, col

    cases = [(Fn.year(col("d")) == 1995, "(year(d) = 1995)"), (Fn.substring(col("s"), 1, 2) == "13", "(substring(s, 1, 2) = 13)"),
             (Fn.datediff(col("a"), "b") > 30, "(datediff(a, b) > 30)"), (Fn.abs(col("a") - col("b")) < 5, "(abs((a - b)) < 5)"),
             (Fn.coalesce("x", Fn.lit(0)) > 0.05, "(coalesce(x, 0) > 0.05)"), (~(Fn.month("d") == 3), "NOT (month(d) = 3)"),
             (Fn.date_add("d", 7) <= Fn.col("e"), "(date_add(d, 7) <= e)"), (Fn.date_sub(Fn.col("d"), 1) >= "e", None),
             (Fn.length("s").eqNullSafe(3), "(length(s) <=> 3)"), (col("s").substr(2, 3) != "ab", "NOT (substring(s, 2, 3) = ab)"),
             (Fn.hour("t") == 23, "(hour(t) = 23)"), (Fn.weekofyear("d") == 1, "(weekofyear(d) = 1)")]
    for p, text in cases:
        e, = p.exprs
        if text:
            assert str(e) == text
    for name in ("year", "quarter", "month", "dayofmonth", "dayofweek", "dayofyear", "weekofyear", "hour", "minute", "second", "length", "abs"):
        e = getattr(Fn, name)("c")
        assert isinstance(e, Expr) and e.postfix() == [("column", "c"), (name,)] and str(e) == f"{name}(c)"
    assert Fn.substring("s", 1, 2).postfix() == [("column", "s"), ("literal", 1), ("literal", 2), ("substring",)]
    assert Fn.coalesce("a", "b", Fn.lit(0)).postfix() == [("column", "a"), ("column", "b"), ("literal", 0), ("coalesce", 3)]
    assert Fn.datediff("a", "b").columns == ["a", "b"]
    e, = (Fn.year("d") == datetime.date(1995, 1, 1)).exprs
    assert e.as_native()[2] == [("literal", datetime.date(1995, 1, 1))]
    p = col("d") >= datetime.date(1995, 1, 1)  # the date stays a date until DataFrame.filter knows its column's type
    assert p.bounds == {"d": (9131, None)} and p.terms == [("d", ">=", datetime.date(1995, 1, 1))]


def test_python_refusals_that_still_raise():
    from hyperspace_b200 import functions as Fn
    from hyperspace_b200 import log_entry as LE
    from hyperspace_b200.session import col

    with pytest.raises(LE.HyperspaceException, match="OR across columns"):
        (Fn.year("d") == 1995) | (col("a") > 5)
    with pytest.raises(LE.HyperspaceException, match="OR across columns"):
        Fn.year("d").isin(1995, 1996)
    for bad in ("x", b"x", datetime.date(1995, 1, 1), datetime.datetime(1995, 1, 1)):
        with pytest.raises(LE.HyperspaceException, match="cannot be used in arithmetic"):
            Fn.year("d") + bad
    with pytest.raises(LE.HyperspaceException, match="int"):
        Fn.substring("s", col("p"), 2)
    with pytest.raises(LE.HyperspaceException, match="at least two"):
        Fn.coalesce("a")
    with pytest.raises(LE.HyperspaceException, match="not a filter"):
        bool(Fn.year("d"))


def test_date_literals_take_their_columns_unit(tmp_path):
    from hyperspace_b200 import log_entry as LE
    from hyperspace_b200.session import col

    df = _fabricated(tmp_path, ["k"], ["d", "t"], [("k", "long"), ("d", "date"), ("t", "timestamp"), ("w", "long")])
    day, nxt = datetime.date(1995, 1, 1), datetime.date(1995, 1, 2)
    cases = [(col("d") >= day, {"d": (9131, None)}, [("d", ">=", 9131)]),
             (col("T") >= day, {"t": (9131 * DAY_US, None)}, [("t", ">=", 9131 * DAY_US)]),  # the day's UTC midnight
             ((col("t") > day) & (col("t") <= nxt), {"t": (9131 * DAY_US + 1, 9132 * DAY_US)}, [("t", ">", 9131 * DAY_US), ("t", "<=", 9132 * DAY_US)]),
             (col("t") < day, {"t": (None, 9131 * DAY_US - 1)}, [("t", "<", 9131 * DAY_US)]),
             (col("t") == day, {"t": (9131 * DAY_US, 9131 * DAY_US)}, [("t", "==", 9131 * DAY_US)]),
             (col("d").between(day, nxt), {"d": (9131, 9132)}, [("d", ">=", 9131), ("d", "<=", 9132)]),
             ((col("k") > 3) & (col("t") >= day), {"k": (4, None), "t": (9131 * DAY_US, None)}, [("k", ">", 3), ("t", ">=", 9131 * DAY_US)])]
    for p, bounds, terms in cases:
        r = df.filter(p).plan.predicate
        assert r.bounds == bounds and r.terms == terms, (r.bounds, r.terms)
    with pytest.raises(LE.HyperspaceException, match="date literal 1995-01-01 cannot be compared with the long column 'w'"):
        df.filter(col("w") >= day)


def test_session_time_zone_refuses_timestamp_functions(tmp_path):
    from hyperspace_b200 import functions as Fn
    from hyperspace_b200 import log_entry as LE

    df = _fabricated(tmp_path, ["k"], ["d", "t"], [("k", "long"), ("d", "date"), ("t", "timestamp"), ("w", "long")])
    for zone in (None, "UTC", "GMT", "Z", "+00:00", "-00:00"):
        if zone is None:
            df.session.conf.unset("spark.sql.session.timeZone")
        else:
            df.session.conf.set("spark.sql.session.timeZone", zone)
        df.filter(Fn.hour("t") == 1)
    df.session.conf.set("spark.sql.session.timeZone", "America/Los_Angeles")
    for p in (Fn.hour("t") == 1, Fn.year(Fn.col("T")) == 1995, Fn.datediff("d", "t") > 3, Fn.year(Fn.coalesce("d", "t")) > 1):
        with pytest.raises(LE.HyperspaceException, match="America/Los_Angeles"):
            df.filter(p)
    df.filter(Fn.year("d") == 1995)  # a date needs no time zone
    df.session.conf.unset("spark.sql.session.timeZone")


def test_filter_rule_and_explain_with_functions(tmp_path):
    from hyperspace_b200 import functions as Fn
    from hyperspace_b200.session import col

    df = _fabricated(tmp_path, ["k"], ["d", "s"], [("k", "long"), ("d", "date"), ("s", "string"), ("w", "long")])
    plan = df.filter((col("K") > 3) & (Fn.year(col("D")) == 1995)).select("k", "s").explain()
    assert "Name: idx" in plan and "where=((year(d) = 1995))" in plan, plan
    # the index serves a filter on its key: the function alone leaves the source scan, with the same residual
    plan = df.filter(Fn.substring(col("s"), 1, 2) == "13").select("k").explain()
    assert plan.startswith("GpuSourceScan") and "where=((substring(s, 1, 2) = 13))" in plan, plan
    plan = df.filter(Fn.datediff(col("d"), Fn.date_sub("d", 3)) > col("k")).select("k").explain()
    assert "Name: idx" in plan and "where=((datediff(d, date_sub(d, 3)) > k))" in plan, plan
    assert df.filter(Fn.length(col("w")) > 1).select("k").explain().startswith("GpuSourceScan")
