"""GPU filter scans with disjunctions on one column (hs_filter_scan_any, hs_bucket_join_any): IN lists and OR-ed ranges on
every key type, on sorted index files and on unsorted source files, bucket pruning of point lookups, and the Hyperspace
API's isin / |.  Answers are compared with tests/filter_in_oracle.py as exact sequences of row ids (file, then row)."""
import ctypes as C
import datetime
import decimal
import io
import os

import numpy as np
import pyarrow as pa
import pyarrow.parquet as pq
import pytest

import filter_in_oracle as FI
import filter_oracle as F
import parquet_shapes as S

pytestmark = pytest.mark.gpu

N_ROWS = 60_000
NB = 16
KEYS = ["i32", "i64", "f32", "f64", "s", "ts", "d9", "d18"]
WORDS = [b"", b"a", b"ab", b"abc", b"abd", b"b", "été".encode(), b"facebook", b"zz", b"\xff", b"\xff\x00", b"donde"]
EPOCH = datetime.datetime(1970, 1, 1)


def _make_columns(seed=11):
    rng = np.random.default_rng(seed)
    n = N_ROWS
    i32 = rng.integers(-3000, 3000, n).astype(np.int32)
    i32[:2] = [np.iinfo(np.int32).min, np.iinfo(np.int32).max]
    i64 = rng.integers(-10**5, 10**5, n).astype(np.int64)
    i64[:3] = [2**53 + 1, np.iinfo(np.int64).max, np.iinfo(np.int64).min]
    special = [np.nan, -np.nan, np.inf, -np.inf, 0.0, -0.0, 0.1, 12.5]
    f64 = np.round(rng.normal(0, 100, n), 1)
    f64[100:100 + len(special)] = special
    f64[rng.random(n) < 0.01] = -0.0
    f64[rng.random(n) < 0.01] = np.nan
    f32 = np.round(rng.normal(0, 100, n), 1).astype(np.float32)
    f32[200:200 + len(special)] = np.array(special).astype(np.float32)
    f32[rng.random(n) < 0.01] = 0.0
    s = np.array([WORDS[i] for i in rng.integers(0, len(WORDS), n)], dtype=object)
    ts = rng.integers(0, 5000, n).astype(np.int64) * 1_000_000
    d9 = rng.integers(-5000, 5000, n).astype(np.int64)        # unscaled, scale 2
    d18 = rng.integers(-10**7, 10**7, n).astype(np.int64)
    n64 = rng.integers(0, 300, n).astype(np.int64)
    n64_valid = rng.random(n) >= 0.2
    ids = np.arange(n, dtype=np.int64)
    cols = {"i32": i32, "i64": i64, "f32": f32, "f64": f64, "s": s, "ts": ts, "d9": d9, "d18": d18, "n64": n64, "id": ids}
    return cols, {"n64": n64_valid}


def _arrow(cols, valids, rows):
    out = {}
    for name, v in cols.items():
        v = v[rows]
        mask = ~valids[name][rows] if name in valids else None
        if name == "s":
            out[name] = pa.array(list(v), pa.binary())
        elif name == "ts":
            out[name] = pa.array(v, pa.timestamp("us"))
        elif name in ("d9", "d18"):
            t = pa.decimal128(9, 2) if name == "d9" else pa.decimal128(18, 2)
            out[name] = pa.array([decimal.Decimal(int(x)).scaleb(-2) for x in v], t)
        else:
            out[name] = pa.array(v, mask=mask)
    return pa.table(out)


def _parquet_bytes(table):
    sink = io.BytesIO()
    pq.write_table(table, sink, compression="NONE", data_page_size=16 << 10, row_group_size=20_000)
    return sink.getvalue()


@pytest.fixture(scope="module")
def data():
    from hyperspace_b200 import _native as N

    ctx = N.Context(0)
    cols, valids = _make_columns()
    halves = [np.arange(0, N_ROWS // 2), np.arange(N_ROWS // 2, N_ROWS)]
    sources = [N.FileImage(path=f"src{i}.parquet", data=_parquet_bytes(_arrow(cols, valids, r)), file_id=i)
               for i, r in enumerate(halves)]
    others = list(cols)
    indexes = {k: ctx.create_index(sources, [k], [c for c in others if c != k], NB, output=N.HS_OUT_HOST)[0] for k in KEYS}
    two = [ctx.create_index([s], ["i64"], [c for c in others if c != "i64"], NB, output=N.HS_OUT_HOST)[0] for s in sources]
    yield {"ctx": ctx, "cols": cols, "valids": valids, "sources": sources, "indexes": indexes, "two": two}
    for r in list(indexes.values()) + two:
        r.free()
    ctx.close()


def _file_ids(res):
    return [pq.read_table(pa.BufferReader(res.host_bytes(i)), columns=["id"]).column("id").to_numpy() for i in range(len(res.files))]


def _decimal_unscaled_at(v, scale):
    """the unscaled value of a literal at the column's scale, or None when it has more fractional digits"""
    q = decimal.Decimal(v).scaleb(scale)
    return int(q) if q == q.to_integral_value() else None


def _term_mask(d, key, values, ranges=()):
    """filter_in_oracle's mask, vectorised for long lists (np.isin after Spark's coercion of the list)."""
    v = d["cols"][key]
    if ranges or len(values) <= 64:
        if key in ("d9", "d18"):  # decimals compare exactly at the column's scale
            want = {_decimal_unscaled_at(x, 2) for x in values} - {None}
            return np.isin(v, np.array(sorted(want), dtype=np.int64))
        if key == "ts":
            values = [int((x - EPOCH) / datetime.timedelta(microseconds=1)) for x in values]
        return FI.term_mask(d["cols"], (key, list(values), list(ranges)), d["valids"])
    if key == "s":
        want = set(values)
        return np.array([x in want for x in v])
    if key in ("d9", "d18"):
        want = {_decimal_unscaled_at(x, 2) for x in values} - {None}
        return np.isin(v, np.array(sorted(want), dtype=np.int64))
    if key == "ts":
        return np.isin(v, np.array([int((x - EPOCH) / datetime.timedelta(microseconds=1)) for x in values], dtype=np.int64))
    vals = np.asarray(values)
    if vals.dtype.kind in "iu" and v.dtype.kind == "i":
        return np.isin(v.astype(np.int64), vals.astype(np.int64))
    if v.dtype == np.float32 and vals.dtype.kind in "iu":
        a, b = v, np.array([F.long_to_float32(int(x)) for x in vals], dtype=np.float32)
    elif vals.dtype.kind in "iu":
        a, b = v.astype(np.float64), vals.astype(np.float64)
    else:
        a, b = v.astype(np.float64), vals.astype(np.float64)
    return np.isin(a, b[~np.isnan(b)]) | (np.isnan(a) & bool(np.isnan(b).any()))


def _ids(batch):
    out = next(v.copy() for n, v, _ in batch.columns if n == "id")
    batch.free()
    return out


def _scan(d, files, key, preds, terms, sorted_on_key=True, buckets=None, projected=("id",)):
    b, st = d["ctx"].filter_scan_any(files, key, list(projected), preds, terms, sorted_on_key=sorted_on_key,
                                     file_buckets=buckets, num_buckets=NB if buckets is not None else 0)
    return _ids(b), st


def _check_both_paths(d, key, values, ranges=()):
    m = _term_mask(d, key, values, ranges)
    res = d["indexes"][key]
    want = np.concatenate([ids[m[ids]] for ids in _file_ids(res)])
    got, _ = _scan(d, res.as_sources(), key, [], [(key, values, list(ranges))])
    assert np.array_equal(got, want), (key, len(got), len(want))
    got, _ = _scan(d, d["sources"], None, [], [(key, values, list(ranges))], sorted_on_key=False)
    assert np.array_equal(got, np.flatnonzero(m)), (key, "unsorted")


def _values(d, key, size, rng):
    """size values, about half present in the column and half absent, with duplicates and the type's edge literals"""
    col = d["cols"][key]
    present = col[rng.integers(0, len(col), max(1, size // 2))]
    if key == "s":
        extra = [b"", b"ab", b"abz", b"\xff", b"\xfe\xff", b"zzz", "été".encode() + b"!", b"faceboo"]
        absent = [b"k%d" % i for i in range(size)]
        vals = list(present) + extra + absent
    elif key == "ts":
        vals = [EPOCH + datetime.timedelta(microseconds=int(x)) for x in present] + \
               [EPOCH + datetime.timedelta(microseconds=int(x) * 1_000_000 + 1) for x in range(size)]
    elif key in ("d9", "d18"):
        vals = [decimal.Decimal(int(x)).scaleb(-2) for x in present]
        vals += [decimal.Decimal("1.5"), decimal.Decimal("-3"), decimal.Decimal("0.505"), decimal.Decimal("12.3400")]
        vals += [decimal.Decimal(10**8 + i) for i in range(size)]
    elif key in ("f32", "f64"):
        vals = [float(x) for x in present] + [np.nan, -0.0, 0.0, np.inf, -np.inf, 12.5, 0.1] + [1e9 + i for i in range(size)]
    else:
        vals = [int(x) for x in present] + [2**40, -2**40, 2**63 - 1, -3000, 2999] + [10**7 + i for i in range(size)]
    vals = vals[:max(0, size - 2)] + vals[:2]  # duplicates
    return vals[:size] if size else []


@pytest.mark.parametrize("key", KEYS)
@pytest.mark.parametrize("size", [0, 1, 7, 1000, 100_000])
def test_in_lists_on_every_key_type(data, key, size):
    rng = np.random.default_rng(size + len(key))
    _check_both_paths(data, key, _values(data, key, size, rng))


@pytest.mark.parametrize("key", ["i32", "i64", "f32"])
def test_fractional_and_mixed_literals_on_numeric_keys(data, key):
    """a float in the list casts the whole list to double (int_col IN (2.5) matches nothing, 3.0 matches 3)"""
    col = data["cols"][key]
    _check_both_paths(data, key, [2.5, float(col[5]), int(col[6]), 2.0**40, np.nan, -0.0])
    _check_both_paths(data, key, np.array([col[7], col[8], 123456789], dtype=np.int64))


@pytest.mark.parametrize("key,ranges", [
    ("i64", [(None, False, -50_000, True), (50_000, True, None, False)]),
    ("i64", [(0, False, 100, False), (50, False, 200, True), (200, False, 300, False), (10, False, 20, False)]),  # overlap, adjacent, nested
    ("i32", [(-10, True, 10, True), (10, False, 10, False), (1000, False, None, False)]),
    ("f64", [(None, False, -0.0, False), (100.0, True, None, False)]),  # -0.0 == 0.0, NaN above +inf
    ("f32", [(-1.5, False, 1.5, True), (1.5, False, 2.5, False)]),
    ("s", [(b"a", True, b"abd", False), (b"abd", True, b"b", True), (b"facebook", False, None, False)]),
    ("s", [(None, False, b"", False), (b"\xff", False, b"\xff", False)]),
    ("d9", [(decimal.Decimal("-1.005"), False, decimal.Decimal("1.5"), True), (decimal.Decimal("20"), False, None, False)]),
])
def test_ored_ranges(data, key, ranges):
    d = data
    if key == "d9":  # the oracle's decimal comparison: exact, on the unscaled values at scale 2
        v = d["cols"]["d9"]
        m = ((v * 10 >= -1005) & (v < 150)) | (v >= 2000)  # -1.005 <= x < 1.5 or x >= 20
        res = d["indexes"][key]
        want = np.concatenate([ids[m[ids]] for ids in _file_ids(res)])
        got, _ = _scan(d, res.as_sources(), key, [], [(key, [], ranges)])
        assert np.array_equal(got, want)
        return
    _check_both_paths(d, key, [b"zz"] if key == "s" else [17], ranges)


def test_terms_on_nullable_and_non_key_columns(data):
    d = data
    term = ("n64", [0, 5, 7, 299, 1000], [(250, True, 260, False)])
    for key, preds in (("i64", []), ("i64", [("i64", -20_000, False, 30_000, True)]), ("f64", [("f64", 0.0, False, None, False)])):
        m = FI.mask(d["cols"], preds, [term], d["valids"])
        res = d["indexes"][key]
        want = np.concatenate([ids[m[ids]] for ids in _file_ids(res)])
        got, _ = _scan(d, res.as_sources(), key, preds, [term])
        assert np.array_equal(got, want)
        got, _ = _scan(d, d["sources"], None, preds, [term], sorted_on_key=False)
        assert np.array_equal(got, np.flatnonzero(m))
    # a key term AND-ed with a key range and a term on another column
    key_term = ("i64", [int(x) for x in d["cols"]["i64"][:500]], [])
    preds = [("i64", -50_000, False, None, False)]
    m = FI.mask(d["cols"], preds, [key_term, term], d["valids"])
    res = d["indexes"]["i64"]
    got, _ = _scan(d, res.as_sources(), "i64", preds, [key_term, term])
    assert np.array_equal(got, np.concatenate([ids[m[ids]] for ids in _file_ids(res)]))


def test_windows_on_page_edges():
    """k = 6 r in file 0 and 6 r + 3 in file 1: lists that hit the first and last rows of pages, many windows in one page and
    whole pages between windows."""
    from hyperspace_b200 import _native as N

    images, expected, _ = S.case_data("windows_on_page_edges")
    files = [N.FileImage(data=img) for img in images]
    w = S.WINDOW_PAGES[0]
    edges = set()
    for sizes in (w["a"], w["b"], w["c"]):
        edges |= set(np.cumsum(sizes)[:-1].tolist())
    rows = sorted({e + dd for e in edges for dd in (-1, 0, 1)} | {0, w["n"] - 1})
    cols = ["k", "a", "b", "c"]
    with N.Context(0) as ctx:
        for sel in (rows, rows[::3], list(range(100, 140)) + [w["n"] - 1], [0] + list(range(2000, 2003, 2))):
            values = [6 * r for r in sel] + [6 * r + 3 for r in sel[::2]] + [6 * r + 1 for r in sel]  # the last: absent
            term = ("k", values, [])
            batch, _ = ctx.filter_scan_any(files, "k", cols, [], [term], sorted_on_key=True)
            m = FI.term_mask({"k": expected["k"][0]}, term)
            sel_rows = np.flatnonzero(m)
            assert batch.num_rows == len(sel_rows)
            for cname, got, got_valid in batch.columns:
                values_c, v = expected[cname]
                want = values_c[sel_rows]
                if want.dtype == object:
                    ok = [i for i in range(len(want)) if (v is None or v[sel_rows][i]) and got[i] != want[i]]
                    assert not ok, cname
                else:
                    keep = np.ones(len(want), bool) if v is None else v[sel_rows].astype(bool)
                    assert np.array_equal(np.asarray(got)[keep], want[keep]), cname
            batch.free()


def _bucket_of(ctx, keys):
    return ctx.k_bucket_ids([np.asarray(keys, dtype=np.int64)], NB)[0]


def test_bucket_pruning_point_lookups(data):
    d, ctx = data, data["ctx"]
    res = d["indexes"]["i64"]
    files = res.as_sources()
    buckets = [f.bucket for f in res.files]
    sizes = [len(res.host_bytes(i)) for i in range(len(res.files))]
    keys = [int(d["cols"]["i64"][i]) for i in (10, 20_000, 45_000)]
    hit = set(_bucket_of(ctx, keys).tolist())
    terms = [("i64", keys, [])]
    full, st_full = _scan(d, files, "i64", [], terms)
    pruned, st = _scan(d, files, "i64", [], terms, buckets=buckets)
    assert np.array_equal(pruned, full) and len(full) >= 3
    assert st["bytes_in"] == sum(s for s, b in zip(sizes, buckets) if b in hit) < st_full["bytes_in"]
    # an equality in the predicates is a point too; with many columns projected the rows are byte-identical
    proj = ["id", "i32", "f64", "s", "n64"]
    b1, _ = ctx.filter_scan_any(files, "i64", proj, [("i64", keys[0], False, keys[0], False)], [("n64", [], [(0, False, None, False)])])
    b2, st2 = ctx.filter_scan_any(files, "i64", proj, [("i64", keys[0], False, keys[0], False)], [("n64", [], [(0, False, None, False)])],
                                  file_buckets=buckets, num_buckets=NB)
    for (n1, v1, m1), (n2, v2, m2) in zip(b1.columns, b2.columns):
        same = list(v1) == list(v2) if v1.dtype == object else v1.tobytes() == v2.tobytes()
        assert n1 == n2 and same and (m1 is None) == (m2 is None)
        assert m1 is None or m1.tobytes() == m2.tobytes()
    b1.free()
    b2.free()
    assert st2["bytes_in"] == sum(s for s, b in zip(sizes, buckets) if b == _bucket_of(ctx, keys[:1])[0])


def test_bucket_pruning_searches_every_file_of_a_bucket(data):
    d = data
    files = d["two"][0].as_sources() + d["two"][1].as_sources()
    buckets = [f.bucket for f in d["two"][0].files] + [f.bucket for f in d["two"][1].files]
    sizes = [len(r.host_bytes(i)) for r in d["two"] for i in range(len(r.files))]
    keys = [int(d["cols"]["i64"][i]) for i in (5, 31_000, 59_000)]
    hit = set(_bucket_of(d["ctx"], keys).tolist())
    full, _ = _scan(d, files, "i64", [], [("i64", keys, [])])
    pruned, st = _scan(d, files, "i64", [], [("i64", keys, [])], buckets=buckets)
    assert np.array_equal(pruned, full)
    assert set(np.flatnonzero(np.isin(d["cols"]["i64"], keys))) == set(full.tolist())
    assert st["bytes_in"] == sum(s for s, b in zip(sizes, buckets) if b in hit)


def test_bucket_pruning_decimal_and_double_keys(data):
    d = data
    res = d["indexes"]["d9"]
    files, buckets = res.as_sources(), [f.bucket for f in res.files]
    sizes = [len(res.host_bytes(i)) for i in range(len(res.files))]
    unscaled = [int(d["cols"]["d9"][i]) for i in (3, 300, 30_003)]
    values = [decimal.Decimal(u).scaleb(-2) for u in unscaled]
    hit = set(_bucket_of(d["ctx"], unscaled).tolist())  # decimal(p <= 9) hashes its unscaled value as a long
    full, _ = _scan(d, files, "d9", [], [("d9", values, [])])
    pruned, st = _scan(d, files, "d9", [], [("d9", values, [])], buckets=buckets)
    assert np.array_equal(pruned, full) and len(full) >= 3
    assert st["bytes_in"] == sum(s for s, b in zip(sizes, buckets) if b in hit)
    res = d["indexes"]["f64"]
    files, buckets = res.as_sources(), [f.bucket for f in res.files]
    vals = [float(d["cols"]["f64"][i]) for i in (1, 2, 3)]
    full, st_full = _scan(d, files, "f64", [], [("f64", vals, [])])
    pruned, st = _scan(d, files, "f64", [], [("f64", vals, [])], buckets=buckets)
    assert np.array_equal(pruned, full) and st["bytes_in"] == st_full["bytes_in"] == sum(len(res.host_bytes(i)) for i in range(len(res.files)))


def test_without_terms_equals_the_where_calls(data):
    d, ctx = data, data["ctx"]
    res = d["indexes"]["i64"]
    preds = [("i64", -1000, False, 5000, True), ("n64", 10, False, None, False)]
    b1, s1 = ctx.filter_scan_where(res.as_sources(), "i64", ["id", "s"], preds)
    b2, s2 = ctx.filter_scan_any(res.as_sources(), "i64", ["id", "s"], preds, [])
    assert np.array_equal(_ids(b1), _ids(b2)) and s1["gpu_launches"] == s2["gpu_launches"] and s1["rows_out"] == s2["rows_out"]
    r = d["indexes"]["i64"]
    args = (r.as_sources(), [f.bucket for f in r.files], r.as_sources(), [f.bucket for f in r.files], NB, ["i64"], ["i64"], ["id"], ["id"])
    j1, t1 = ctx.bucket_join_where(*args, [("n64", 5, False, None, False)], [])
    j2, t2 = ctx.bucket_join_any(*args, [("n64", 5, False, None, False)], [])
    c1, c2 = [v.copy() for _, v, _ in j1.columns], [v.copy() for _, v, _ in j2.columns]
    j1.free()
    j2.free()
    assert all(np.array_equal(a, b) for a, b in zip(c1, c2)) and t1["gpu_launches"] == t2["gpu_launches"]
    # isin below the left side, a range term below the right side: the join of the filtered sides
    lterm, rterm = ("n64", [1, 2, 3, 250], []), ("f64", [], [(0.0, False, None, False)])
    j, _ = ctx.bucket_join_any(*args, [], [], [lterm], [rterm])
    got = sorted(zip(*[v.tolist() for _, v, _ in j.columns]))
    j.free()
    lm = FI.term_mask(d["cols"], lterm, d["valids"])
    rm = FI.term_mask(d["cols"], rterm, d["valids"])
    by_key = {}
    for i in np.flatnonzero(rm):
        by_key.setdefault(int(d["cols"]["i64"][i]), []).append(int(i))
    want = sorted((int(i), j) for i in np.flatnonzero(lm) for j in by_key.get(int(d["cols"]["i64"][i]), []))
    assert got == want and len(want) > 0


def test_refusals_and_the_context_keeps_working(data):
    from hyperspace_b200 import _native as N

    d, ctx = data, data["ctx"]
    files = d["indexes"]["i64"].as_sources()

    def refused(code, column, *args, **kw):
        with pytest.raises(N.HyperspaceGpuError) as e:
            ctx.filter_scan_any(*args, **kw)
        assert e.value.code == code, e.value.message
        if column:
            assert f"'{column}'" in e.value.message, e.value.message

    refused(N.HS_EUNSUPPORTED, None, files, "i64", ["id"], [], [("i64", [i], []) for i in range(17)])
    refused(N.HS_EUNSUPPORTED, "i64", files, "i64", ["id"], [], [("i64", np.zeros(2**24 + 1, np.int64), [])])
    refused(N.HS_EUNSUPPORTED, "s", d["indexes"]["s"].as_sources(), "s", ["id"], [], [("s", [b"x" * 65536], [])])
    refused(N.HS_EUNSUPPORTED, "i64", files, "i64", ["id"], [], [("i64", [b"abc"], [])])
    refused(N.HS_EUNSUPPORTED, "n64", files, "i64", ["id"], [], [("n64", ["abc"], [])])
    refused(N.HS_EUNSUPPORTED, "d9", d["indexes"]["d9"].as_sources(), "d9", ["id"], [], [("d9", [1.5], [])])
    refused(N.HS_EUNSUPPORTED, "ts", d["indexes"]["ts"].as_sources(), "ts", ["id"], [], [("ts", [1.5], [])])
    # malformed arrays, built by hand
    L = N.load_library()
    src, keep = N._source_array(files)
    spec = N.ScanSpec()
    spec.files, spec.n_files, spec.sorted_on_key, spec.key_column = src, len(files), 1, b"i64"
    pc = N._cstr_array(["id"])
    spec.projected_columns, spec.n_projected = pc, 1
    blob = np.frombuffer(b"abcdefgh", dtype=np.uint8)
    for offs, n_values, values_i in ((np.array([0, 5, 2], np.uint64), 2, None), (None, 1, None), (np.array([0, 1], np.uint64), 1, "i")):
        a = (N.PredicateAnySpec * 1)()
        a[0].column, a[0].n_values = b"i64" if values_i else b"s", n_values
        a[0].literal_type = N.HS_TYPE_INT64 if values_i else N.HS_TYPE_STRING
        a[0].values_bytes = blob.ctypes.data
        a[0].values_offsets = offs.ctypes.data if offs is not None else None
        res, st, err = C.c_void_p(), N.Stats(), C.create_string_buffer(512)
        rc = L.hs_filter_scan_any(ctx._h, C.byref(spec), None, 0, a, 1, None, 0, C.byref(res), C.byref(st), err, 512)
        assert rc == N.HS_EINVAL, err.value
    got, _ = _scan(d, files, "i64", [], [("i64", [int(d["cols"]["i64"][0])], [])])
    assert sorted(got.tolist()) == np.flatnonzero(d["cols"]["i64"] == d["cols"]["i64"][0]).tolist()


SAMPLE = [
    ("2017-09-03", "810a20a2baa24ff3ad493bfbf064569a", "donde", 2, 1000),
    ("2017-09-03", "fd093f8a05604515957083e70cb3dceb", "facebook", 1, 3000),
    ("2017-09-03", "af3ed6a197a8447cba8bc8ea21fad208", "facebook", 1, 3000),
    ("2017-09-03", "975134eca06c4711a0406d0464cbe7d6", "facebook", 1, 4000),
    ("2018-09-03", "e90a6028e15b4f4593eef557daf5166d", "ibraco", 2, 3000),
    ("2018-09-03", "576ed96b0d5340aa98a47de15c9f87ce", "facebook", 2, 3000),
    ("2018-09-03", "50d690516ca641438166049a6303650c", "ibraco", 2, 1000),
    ("2019-10-03", "380786e6495d4cd8a5dd4cc8d3d12917", "facebook", 2, 3000),
    ("2019-10-03", "ff60e4838b92421eafc3e6ee59a9e9f1", "miperro", 2, 2000),
    ("2019-10-03", "187696fe0a6a40cc9516bc6e47c70bc1", "facebook", 4, 3000),
]


@pytest.fixture()
def env(tmp_path):
    from hyperspace_b200.hyperspace import Hyperspace
    from hyperspace_b200.session import HyperspaceSession

    s = HyperspaceSession({"spark.hyperspace.system.path": str(tmp_path / "indexes"), "spark.hyperspace.index.numBuckets": "8"})
    yield s, Hyperspace(s), tmp_path
    s.stop()


def _write(dirpath, name, cols):
    os.makedirs(dirpath, exist_ok=True)
    pq.write_table(pa.table(cols), os.path.join(dirpath, name), compression="snappy")


def _same_answers(s, q, cols):
    s.enableHyperspace()
    got = q.collect()
    s.disableHyperspace()
    base = q.collect()
    s.enableHyperspace()
    key = lambda r: sorted(zip(*[[x if not isinstance(x, float) else repr(x) for x in r[c].tolist()] for c in cols]))  # noqa: E731
    assert key(got) == key(base)
    return got


def test_hyperspace_api_isin_and_or(env):
    from hyperspace_b200.index_config import IndexConfig
    from hyperspace_b200.session import col

    s, hs, tmp = env
    rng = np.random.default_rng(3)
    for i in range(3):
        _write(tmp / "t", f"f{i}.parquet", {"k": rng.integers(0, 2000, 5000).astype(np.int64), "v": rng.normal(size=5000)})
    df = s.read.parquet(str(tmp / "t"))
    hs.createIndex(df, IndexConfig("kidx", ["k"], ["v"]))
    s.enableHyperspace()
    q = df.filter(col("k").isin(list(range(0, 2000, 37)) + [None, 5000])).select("k", "v")
    assert "Name: kidx" in q.explain() and "k IN (0, 37, 74, ... " in q.explain()
    got = _same_answers(s, q, ["k", "v"])
    assert len(got["k"]) > 0 and set(got["k"].tolist()) <= set(range(0, 2000, 37))
    q = df.filter((col("k") < 10) | (col("k") > 1990)).select("k", "v")
    assert "Name: kidx" in q.explain()
    got = _same_answers(s, q, ["k", "v"])
    assert all(k < 10 or k > 1990 for k in got["k"].tolist()) and len(got["k"]) > 0
    q = df.filter(((col("k") < 100) | col("k").isin(1500, 1501)) & (col("v") > 0)).select("k", "v")
    _same_answers(s, q, ["k", "v"])
    # Hybrid Scan: an appended file, then a deleted one with lineage
    s.conf.set("spark.hyperspace.index.hybridscan.enabled", True)
    _write(tmp / "t", "f3.parquet", {"k": np.arange(0, 400, dtype=np.int64), "v": np.ones(400)})
    q = s.read.parquet(str(tmp / "t")).filter(col("k").isin(3, 37, 399)).select("k", "v")
    assert "hybridScan(appended=1" in q.explain() and "Name: kidx" in q.explain()
    _same_answers(s, q, ["k", "v"])


def test_hyperspace_api_isin_with_deleted_lineage_ids(env):
    from hyperspace_b200.index_config import IndexConfig
    from hyperspace_b200.session import col

    s, hs, tmp = env
    s.conf.set("spark.hyperspace.index.lineage.enabled", True)
    for i in range(6):
        _write(tmp / "t", f"f{i}.parquet", {"k": np.arange(i * 1000, i * 1000 + 1000, dtype=np.int64) % 1500, "v": np.arange(1000.0)})
    hs.createIndex(s.read.parquet(str(tmp / "t")), IndexConfig("idx", ["k"], ["v"]))
    os.remove(tmp / "t" / "f5.parquet")
    s.enableHyperspace()
    s.conf.set("spark.hyperspace.index.hybridscan.enabled", True)
    q = s.read.parquet(str(tmp / "t")).filter(col("k").isin(1, 2, 1200, 1499)).select("k", "v")
    assert "deletedIds=[5]" in q.explain() and "Name: idx" in q.explain()
    _same_answers(s, q, ["k", "v"])


def test_hyperspace_api_string_isin_over_sample_data(env):
    from hyperspace_b200.index_config import IndexConfig
    from hyperspace_b200.session import col

    s, hs, tmp = env
    cols = list(zip(*SAMPLE))
    _write(tmp / "sample", "a.parquet", {"Date": pa.array(cols[0]), "RGUID": pa.array(cols[1]), "Query": pa.array(cols[2]),
                                          "imprs": pa.array(cols[3], pa.int32()), "clicks": pa.array(cols[4], pa.int32())})
    df = s.read.parquet(str(tmp / "sample"))
    hs.createIndex(df, IndexConfig("filterIndex", ["Query"], ["clicks"]))
    s.enableHyperspace()
    q = df.filter(col("Query").isin("facebook", "donde")).select("Query", "clicks")
    assert "Name: filterIndex" in q.explain()
    got = _same_answers(s, q, ["Query", "clicks"])
    assert sorted(zip(got["Query"].tolist(), got["clicks"].tolist())) == \
        sorted((r[2], r[4]) for r in SAMPLE if r[2] in ("facebook", "donde"))
