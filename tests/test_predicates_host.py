"""Host-side tests of the engine's predicate resolution (hyperspace_b200/csrc/predicates.h), built as host code under
AddressSanitizer where the compiler has it: the ranges it resolves select, over columns of hard values encoded as the
kernels see them, exactly the rows the numpy oracles select; normalise_set and intersect_sets keep their shapes; and
the refusals keep their codes and messages."""
import math
import os
import shutil
import subprocess
from fractions import Fraction

import numpy as np
import pytest

import filter_in_oracle as FI
import filter_oracle as F
import sort_edge_cases as E

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INT32, INT64, FLOAT, DOUBLE, BOOL, STRING, DECIMAL = range(7)


@pytest.fixture(scope="module")
def native(tmp_path_factory):
    if shutil.which("nvcc") is None:
        pytest.skip("nvcc not on PATH")
    exe = str(tmp_path_factory.mktemp("predicates") / "predicates")
    base = ["nvcc", "-std=c++17", "-O1", "-g", "-Wno-deprecated-gpu-targets", "-o", exe,
            os.path.join(ROOT, "tests", "native", "predicates.cu")]
    try:
        subprocess.check_call(base + ["-Xcompiler", "-fsanitize=address,-fno-omit-frame-pointer"], stderr=subprocess.DEVNULL)
        asan = subprocess.run([exe, "x"], capture_output=True).returncode == 2  # usage error, sanitizer runtime loaded
    except subprocess.CalledProcessError:
        asan = False
    if not asan:
        subprocess.check_call(base)
    return exe


def run(native, lines):
    out = subprocess.run([native], input="\n".join(lines) + "\n", capture_output=True, text=True, check=True).stdout
    got = out.splitlines()
    assert len(got) == len(lines)
    return [_parse(line) for line in got]


def _parse(line):
    if line.startswith("refused"):
        _, code, msg = line.split(" ", 2)
        return int(code), msg
    ranges = []
    for r in line[3:].split("]")[:-1]:
        hl, ls, lo, hh, hs, hi = r.strip(" [").split()
        ranges.append((hl == "1", ls == "1", lo, hh == "1", hs == "1", hi))
    return ranges


# ---- case encoding ----------------------------------------------------------------------------------------------------

def _lit(v):
    """(literal type, scale, token) of a literal as Context marshals it."""
    if isinstance(v, bytes):
        return STRING, 0, v.hex() or "-"
    if isinstance(v, float):
        return DOUBLE, 0, "nan" if math.isnan(v) else v.hex()
    if isinstance(v, tuple):  # (unscaled, scale): a decimal literal
        return DECIMAL, v[1], str(v[0])
    return INT64, 0, str(v)


def pred(lo, ls, hi, hs):
    kinds = {_lit(v)[:2] for v in (lo, hi) if v is not None}
    assert len(kinds) == 1
    lt, sc = kinds.pop()
    tok = lambda v: _lit(v)[2] if v is not None else ("-" if lt == STRING else "0")  # noqa: E731
    return f"{lt} {sc} {int(lo is not None)} {int(ls)} {tok(lo)} {int(hi is not None)} {int(hs)} {tok(hi)}"


def term(values, ranges):
    lt, sc = _lit(values[0])[:2] if values else (INT64, 0)
    toks = " ".join(_lit(v)[2] for v in values)
    rs = " ".join(pred(*r) for r in ranges)
    return f"{lt} {sc} {len(values)} {toks} {len(ranges)} {rs}".replace("  ", " ")


# ---- applying resolved ranges ----------------------------------------------------------------------------------------

def select(values, ranges):
    """Rows inside any of the resolved ranges: numeric bounds against sort_encode, string bounds as bytes."""
    m = np.zeros(len(values), dtype=bool)
    strings = values.dtype == object
    enc = None if strings else E.encode(values)
    for hl, ls, lo, hh, hs, hi in ranges:
        if strings:
            lo_b = b"" if lo == "-" else bytes.fromhex(lo)
            hi_b = b"" if hi == "-" else bytes.fromhex(hi)
            r = np.array([(not hl or (v > lo_b if ls else v >= lo_b)) and (not hh or (v < hi_b if hs else v <= hi_b))
                          for v in values], dtype=bool)
        else:
            r = np.ones(len(values), dtype=bool)
            if hl:
                r &= enc >= np.uint64(int(lo))
            if hh:
                r &= enc <= np.uint64(int(hi))
        m |= r
    return m


I32 = np.array([-2**31, -2**31 + 1, -16777217, -2, -1, 0, 1, 2, 3, 16777216, 16777217, 2**31 - 2, 2**31 - 1], np.int32)
T53 = 2**53
I64 = np.array([-2**63, -2**63 + 1, -T53 - 2, -T53 - 1, -T53, -1, 0, 1, T53 - 1, T53, T53 + 1, T53 + 2, T53 + 3, T53 + 4,
                2**62, 2**63 - 2, 2**63 - 1], np.int64)
F32 = np.array([np.nan, -np.inf, np.inf, -0.0, 0.0, 0.1, -0.1, 1.5, 16777215.0, 16777216.0, 16777218.0, 3.4e38, -3.4e38,
                1e-45, np.float32(T53)], np.float32)
F64 = np.array([np.nan, -np.inf, np.inf, -0.0, 0.0, 5e-324, -5e-324, 0.1, 1.5, -1.5, float(T53), float(T53 + 2),
                float(T53 - 1), 1.7e308, -1.7e308, float(2**63)], np.float64)
STR = np.array([b"", b"a", b"a\x00", b"ab", b"abc", b"abd", b"b", b"\x7f", b"\x80", b"\xff", b"\xff\xff"], dtype=object)

INT_LITS = [-2**63, -2**63 + 1, -2**31 - 1, -2**31, -16777217, -1, 0, 1, 2, 16777217, 16777218, 2**31 - 1, 2**31, T53 - 1,
            T53, T53 + 1, T53 + 2, T53 + 3, 2**63 - 1]
DBL_LITS = [float("nan"), float("inf"), float("-inf"), -0.0, 0.0, 0.1, 1.5, -1.5, 2.5, 5e-324, float(T53), float(T53 + 2),
            float(2**31), float(2**31 - 1) + 0.5, float(2**63), -float(2**63), 1e300, float(np.float32(0.1)), 16777217.0]
STR_LITS = [b"", b"a", b"a\x00", b"ab", b"abc", b"abcd", b"b", b"\x80", b"\xff", b"\xff\xff\xff"]

NUMERIC = [(INT32, I32, INT_LITS + DBL_LITS), (INT64, I64, INT_LITS + DBL_LITS), (FLOAT, F32, INT_LITS + DBL_LITS),
           (DOUBLE, F64, INT_LITS + DBL_LITS)]


def _bounds(lits):
    """Every one-sided predicate on each literal, and two-sided ones on neighbouring literals."""
    out = []
    for v in lits:
        for s in (False, True):
            out += [(v, s, None, False), (None, False, v, s)]
    for a, b in zip(lits, lits[1:] + lits[:1]):
        if type(a) is type(b):
            out += [(a, False, b, False), (b, True, a, True)]
    return out


def test_single_predicates_select_the_oracle_rows(native):
    """resolve_range on int32 / int64 / float / double / string columns: the 2^31 and 2^63 extremes, 2^53 +- k as long
    and double literals, long -> float rounding, NaN, +-inf and -0.0, and strings that are proper prefixes of each other."""
    cases = [(t, vals, b) for t, vals, lits in NUMERIC for b in _bounds(lits)]
    cases += [(STRING, STR, b) for b in _bounds(STR_LITS)]
    got = run(native, [f"range {t} p 0 {pred(*b)}" for t, vals, b in cases])
    for (t, vals, (lo, ls, hi, hs)), ranges in zip(cases, got):
        assert isinstance(ranges, list) and len(ranges) == 1, (t, lo, hi, ranges)
        want = F.predicate_mask({"x": vals}, [("x", lo, ls, hi, hs)])
        assert select(vals, ranges).tolist() == want.tolist(), (t, lo, ls, hi, hs, ranges)


def test_empty_and_open_ranges_keep_their_shape(native):
    lines = [f"range {INT64} p 0 {pred(2**63 - 1, True, None, False)}",  # nothing above: lo = 1, hi = 0
             f"range {INT64} p 0 {pred(None, False, 7, False)}",    # open below
             f"range {DOUBLE} p 0 {pred(float('nan'), True, None, False)}",
             f"range {STRING} p 0 {pred(b'ab', True, None, False)}"]
    empty, open_lo, above_nan, s = run(native, lines)
    assert empty == [(True, False, "1", True, False, "0")]
    assert open_lo[0][0] is False and open_lo[0][3] is True
    assert above_nan == [(True, False, "1", True, False, "0")]
    assert s == [(True, True, "6162", False, False, "-")]


@pytest.mark.parametrize("col_scale", [0, 2, 9, 18])
def test_decimal_columns_against_long_and_decimal_literals(native, col_scale):
    """An int64 decimal(18, s) column against long literals and decimal literals of scales 0-18, compared exactly."""
    vals = np.array([-2**63, -10**18 + 1, -10**col_scale - 1, -10**col_scale, -1, 0, 1, 5 * 10**max(col_scale - 1, 0), 10**col_scale,
                     10**col_scale + 1, 10**18 - 1, 2**63 - 1], np.int64)
    lits = [-2**63, -1, 0, 1, 2, 10**18]
    for ls in (0, 1, 2, 9, 17, 18):
        lits += [(-1, ls), (0, ls), (1, ls), (15, ls), (10**ls, ls), (10**18 - 1, ls), (-(10**18) + 1, ls)]
    cases = []
    for v in lits:
        for s in (False, True):
            cases += [(v, s, None, False), (None, False, v, s)]
    got = run(native, [f"range {INT64} d {col_scale} {pred(*b)}" for b in cases])
    exact = [Fraction(int(v), 10**col_scale) for v in vals]
    for (lo, ls, hi, hs), ranges in zip(cases, got):
        lit = lo if lo is not None else hi
        q = Fraction(lit[0], 10**lit[1]) if isinstance(lit, tuple) else Fraction(lit)
        if lo is not None:
            want = [x > q if ls else x >= q for x in exact]
        else:
            want = [x < q if hs else x <= q for x in exact]
        assert select(vals, ranges).tolist() == want, (col_scale, lo, ls, hi, hs, ranges)


def test_terms_select_the_oracle_rows(native):
    """resolve_term: IN lists and OR-ed ranges, merged into one sorted disjoint set."""
    cases = [
        (INT64, I64, [T53, T53 + 1, -1, 2**63 - 1], []),
        (INT64, I64, [float(T53), 1.5, float("nan")], []),
        (INT64, I64, [], [(None, False, -1, True), (T53, False, None, False)]),
        (INT64, I64, [0, 1, 2], [(T53 - 1, False, T53 + 1, False), (1, True, 3, False)]),
        (INT32, I32, [2**31, -2**31, 16777217, 3], [(2**31 - 2, False, None, False)]),
        (INT32, I32, [0.5, -0.0, float(2**31 - 1)], []),
        (FLOAT, F32, [16777217, 0, 2**63 - 1], []),
        (FLOAT, F32, [float("nan"), -0.0, float(np.float32(0.1)), 0.1], [(None, False, float("-inf"), False)]),
        (DOUBLE, F64, [float("nan"), 0.0, float(T53 + 2)], [(-1.5, True, 1.5, True)]),
        (DOUBLE, F64, [T53 + 1, 1], []),
        (STRING, STR, [b"a", b"ab", b"", b"zz"], [(b"abc", False, b"b", True)]),
        (STRING, STR, [], [(None, False, b"a", False), (b"a\x00", True, None, False)]),
    ]
    got = run(native, [f"term {t} p 0 {term(v, r)}" for t, _, v, r in cases])
    for (t, vals, values, ranges), res in zip(cases, got):
        want = FI.term_mask({"x": vals}, ("x", values, ranges))
        assert select(vals, res).tolist() == want.tolist(), (t, values, ranges, res)
        _assert_normalised(t == STRING, res)


def _key(t, b):
    return (b"" if b == "-" else bytes.fromhex(b)) if t else int(b)


def _assert_normalised(str_, ranges):
    """Sorted, disjoint, none empty, and not adjacent (adjacent ranges are merged)."""
    for hl, ls, lo, hh, hs, hi in ranges:
        if hl and hh:
            a, b = _key(str_, lo), _key(str_, hi)
            assert a < b or (a == b and not ls and not hs)
    for (_, _, _, hh, hs, hi), (hl, ls, lo, _, _, _) in zip(ranges, ranges[1:]):
        assert hh and hl
        a, b = _key(str_, hi), _key(str_, lo)
        if str_:
            assert a < b or (a == b and hs and ls)
        else:
            assert b > a + 1


def test_normalise_set_on_random_sets(native):
    rng = np.random.default_rng(11)
    lines, sets = [], []
    for k in range(300):
        rs = []
        for _ in range(int(rng.integers(0, 9))):
            lo, hi = sorted(int(x) for x in rng.integers(0, 40, 2))
            if rng.random() < 0.2:
                lo, hi = hi + 1, lo  # empty
            rs.append((int(rng.random() > 0.15), lo, int(rng.random() > 0.15), hi))
        sets.append(rs)
        lines.append(f"norm {INT64} p 0 {len(rs)} " + " ".join(f"{hl} 0 {lo + 2**63} {hh} 0 {hi + 2**63}" for hl, lo, hh, hi in rs))
    strs = []
    for k in range(200):
        rs = []
        for _ in range(int(rng.integers(0, 7))):
            lo, hi = (bytes(rng.integers(97, 100, int(rng.integers(0, 3))).astype(np.uint8)) for _ in range(2))
            rs.append((int(rng.random() > 0.15), int(rng.random() < 0.5), lo, int(rng.random() > 0.15), int(rng.random() < 0.5), hi))
        strs.append(rs)
        lines.append(f"norm {STRING} p 0 {len(rs)} " + " ".join(f"{a} {b} {c.hex() or '-'} {d} {e} {f.hex() or '-'}" for a, b, c, d, e, f in rs))
    got = run(native, lines)
    domain = np.arange(-2, 43, dtype=np.int64)
    universe = np.array([bytes(97 + c for c in x) for n in range(4) for x in np.ndindex(*(3,) * n)], dtype=object)
    for rs, res in zip(sets, got[:300]):
        raw = [(bool(hl), False, str(lo + 2**63), bool(hh), False, str(hi + 2**63)) for hl, lo, hh, hi in rs]
        assert select(domain, res).tolist() == select(domain, raw).tolist()
        _assert_normalised(False, res)
    for rs, res in zip(strs, got[300:]):
        raw = [(bool(a), bool(b), c.hex() or "-", bool(d), bool(e), f.hex() or "-") for a, b, c, d, e, f in rs]
        assert select(universe, res).tolist() == select(universe, raw).tolist()
        _assert_normalised(True, res)


def test_intersections_match_the_masks(native):
    """intersect_sets of two terms, and the key's one-range fold of intersect_range over its predicates."""
    cases = [
        (INT64, I64, ([0, 1, T53], [(T53 + 2, False, None, False)]), ([], [(None, False, T53, False), (T53 + 3, False, None, False)])),
        (DOUBLE, F64, ([float("nan"), 0.0], [(None, False, -1.5, False)]), ([-0.0, float("nan")], [(float("-inf"), False, 0.1, True)])),
        (STRING, STR, ([b"a", b"ab"], [(b"abc", False, None, False)]), ([], [(b"a", True, b"abd", False)])),
        (INT32, I32, ([], [(None, False, 0, False)]), ([], [(0, True, None, False)])),
    ]
    lines = [f"inter {t} p 0 {term(*a)} {term(*b)}" for t, _, a, b in cases]
    folds = [
        (INT64, I64, [(0, False, None, False), (None, False, T53, True), (-1, True, T53 + 4, False)]),
        (INT64, I64, [(10, False, None, False), (None, False, 5, False)]),  # empty, kept
        (FLOAT, F32, [(1.5, True, None, False), (None, False, 16777217, False)]),
        (STRING, STR, [(b"a", False, None, False), (b"a", True, None, False), (None, False, b"abd", True)]),
        (STRING, STR, []),
    ]
    lines += [f"fold {t} p 0 {len(ps)} " + " ".join(pred(*p) for p in ps) for t, _, ps in folds]
    got = run(native, lines)
    for (t, vals, a, b), res in zip(cases, got):
        want = FI.term_mask({"x": vals}, ("x",) + a) & FI.term_mask({"x": vals}, ("x",) + b)
        assert select(vals, res).tolist() == want.tolist(), (t, a, b, res)
        _assert_normalised(t == STRING, res)
    for (t, vals, ps), res in zip(folds, got[len(cases):]):
        assert len(res) == 1
        want = F.predicate_mask({"x": vals}, [("x",) + p for p in ps])
        assert select(vals, res).tolist() == want.tolist(), (t, ps, res)
    assert got[len(cases) + 1][0][0] and got[len(cases) + 1][0][3]  # the empty intersection keeps both bounds
    assert got[-1] == [(False, False, "-", False, False, "-")]


EUNSUPPORTED, EINVAL = -6, -1


def test_refusals_keep_their_codes_and_messages(native):
    """The refusals the GPU suites expect, with their codes and the column they name."""
    big = "78" * 65536
    lines = [
        f"range {STRING} p 0 {pred(1, False, None, False)}",
        f"range {DOUBLE} p 0 {pred(b'a', False, None, False)}",
        f"range {BOOL} p 0 {pred(0, False, None, False)}",
        f"range {INT64} d 2 {pred(1.5, False, None, False)}",
        f"range {INT64} t 0 {pred(1.5, False, None, False)}",
        f"range {INT64} t 0 {pred((15, 1), False, None, False)}",
        f"range {DOUBLE} p 0 {pred((15, 1), False, None, False)}",
        f"range {INT64} d 2 {DECIMAL} 39 1 0 1 0 0 0",
        f"range {STRING} p 0 {STRING} 0 1 0 {big} 0 0 -",
        f"range {DOUBLE} p 0 -1 0 1 0 0 0 0 0",
        f"term {INT64} p 0 {term([b'abc'], [])}",
        f"term {INT64} d 2 {term([1.5], [])}",
        f"term {STRING} p 0 {term([1], [])}",
        f"checkp {pred(1, False, None, False).replace('1 0 1 0 1', '1 0 0 0 1')}",
        f"checkp 9 0 1 0 0 0 0 0",
        f"checkt {STRING} 0 1 {big} 0",
        f"checkt 9 0 0 0",
        f"checkt {INT64} 0 0 1 {INT64} 0 0 0 0 0 0 0",
    ]
    got = run(native, lines)
    want = [
        (EUNSUPPORTED, "filter scan: a numeric literal cannot be compared with the string column 'c'"),
        (EUNSUPPORTED, "filter scan: a string literal cannot be compared with the numeric column 'c'"),
        (EUNSUPPORTED, "filter scan: predicates on the boolean column 'c' are not handled"),
        (EUNSUPPORTED, "filter scan: a double literal cannot be compared with the decimal column 'c'"),
        (EUNSUPPORTED, "filter scan: a double literal cannot be compared with the timestamp column 'c'"),
        (EUNSUPPORTED, "filter scan: a decimal literal cannot be compared with the timestamp column 'c'"),
        (EUNSUPPORTED, "filter scan: a decimal literal cannot be compared with the floating-point column 'c'"),
        (EINVAL, "filter scan: decimal literal on 'c' has scale 39"),
        (EUNSUPPORTED, "string bound longer than 65535 bytes"),
        (EUNSUPPORTED, "filter scan: key column must be int32 / int64 / string"),
        (EUNSUPPORTED, "filter scan: a string literal cannot be compared with the numeric column 'c'"),
        (EUNSUPPORTED, "filter scan: a double literal cannot be compared with the decimal column 'c'"),
        (EUNSUPPORTED, "filter scan: a numeric literal cannot be compared with the string column 'c'"),
        (EINVAL, "filter scan: predicate on 'c' has no bound"),
        (EINVAL, "filter scan: predicate on 'c' has an unknown literal type"),
        (EUNSUPPORTED, "filter scan: a value of the term on 'c' is longer than 65535 bytes"),
        (EINVAL, "filter scan: term on 'c' has an unknown literal type"),
        (EINVAL, "filter scan: predicate on 'c' has no bound"),
    ]
    assert got == want
