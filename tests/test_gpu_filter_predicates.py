"""GPU filter scans over conjunctions of range predicates on several columns (hs_filter_scan_where), with int32, int64,
float, double and string keys, compared with the numpy restatement of Spark's semantics (tests/filter_oracle.py).

Every answer is checked as the exact sequence of row ids: the scans keep the files' order and each file's row order, so
on an index the rows of every file come out ascending on the key, on both the sorted and the unsorted paths."""
import io
import os

import numpy as np
import pyarrow as pa
import pyarrow.parquet as pq
import pytest

import filter_oracle as F

pytestmark = pytest.mark.gpu

N_ROWS = 200_000
NB = 16
KEYS = ["i32", "i64", "f32", "f64", "t"]
ALL = ["i32", "i64", "f32", "f64", "t", "s", "n64", "b", "id"]
INDEXED = [c for c in ALL if c != "b"]  # the index writer does not take boolean columns


def _make_columns(seed=7):
    rng = np.random.default_rng(seed)
    n = N_ROWS
    i32 = rng.integers(-1000, 1000, n).astype(np.int32)
    i32[:4] = [np.iinfo(np.int32).min, np.iinfo(np.int32).max, 0, -1]
    i64 = rng.integers(-10**6, 10**6, n).astype(np.int64)
    t53 = 2**53
    i64[:12] = [t53 - 1, t53, t53 + 1, t53 + 2, t53 + 3, 2**60 - 1, 2**60, 2**60 + 1, np.iinfo(np.int64).max,
                np.iinfo(np.int64).min, -t53 - 1, -t53]
    f64 = rng.normal(0, 100, n)
    f64[rng.random(n) < 0.02] = np.nan
    special = [np.nan, -np.nan, np.inf, -np.inf, 0.0, -0.0, 5e-324, -5e-324, 2.2e-308, 0.1, 12.5, 20.0, 1.0]
    f64[100:100 + len(special)] = special
    f64[rng.random(n) < 0.01] = -0.0
    f64[rng.random(n) < 0.01] = 0.0
    f32 = rng.normal(0, 10, n).astype(np.float32)
    f32[rng.random(n) < 0.02] = np.nan
    f32[200:200 + len(special)] = np.array(special, dtype=np.float64).astype(np.float32)
    f32[300:305] = [np.float32(0.1), np.float32(1e-45), 16777216.0, 2.0**60, 2.0**60 + 2.0**37]
    f32[rng.random(n) < 0.01] = -0.0
    words = [b"", b"a", b"ab", b"abc", b"abd", b"b", "été".encode(), b"facebook", b"zz", b"\xff"]
    t = np.array([words[i] for i in rng.integers(0, len(words), n)], dtype=object)
    s = np.array([words[i] for i in rng.integers(0, len(words), n)], dtype=object)
    s_valid = rng.random(n) >= 0.2
    n64 = rng.integers(0, 1000, n).astype(np.int64)
    n64_valid = rng.random(n) >= 0.15
    b = rng.random(n) < 0.5
    ids = np.arange(n, dtype=np.int64)
    cols = {"i32": i32, "i64": i64, "f32": f32, "f64": f64, "t": t, "s": s, "n64": n64, "b": b, "id": ids}
    return cols, {"s": s_valid, "n64": n64_valid}


def _arrow(cols, valids, rows):
    arrs = {}
    for name in ALL:
        v = cols[name][rows]
        mask = ~valids[name][rows] if name in valids else None
        if v.dtype == object:
            arrs[name] = pa.array(list(v), pa.binary(), mask=mask)
        else:
            arrs[name] = pa.array(v, mask=mask)
    return pa.table(arrs)


def _parquet_bytes(table):
    sink = io.BytesIO()
    pq.write_table(table, sink, compression="NONE", data_page_size=32 << 10, row_group_size=60_000)
    return sink.getvalue()


@pytest.fixture(scope="module")
def data():
    from hyperspace_b200 import _native as N

    ctx = N.Context(0)
    cols, valids = _make_columns()
    halves = [np.arange(0, N_ROWS // 2), np.arange(N_ROWS // 2, N_ROWS)]
    src_bytes = [_parquet_bytes(_arrow(cols, valids, r)) for r in halves]
    sources = [N.FileImage(path=f"src{i}.parquet", data=b, file_id=i) for i, b in enumerate(src_bytes)]
    indexes = {}
    for key in KEYS:
        res, _ = ctx.create_index(sources, [key], [c for c in INDEXED if c != key], NB, output=N.HS_OUT_HOST, lineage=True)
        indexes[key] = res
    # the same data as two halves indexed separately: every bucket of the union holds two files
    two = [ctx.create_index([s], ["f64"], [c for c in INDEXED if c != "f64"], NB, output=N.HS_OUT_HOST)[0] for s in sources]
    yield {"ctx": ctx, "cols": cols, "valids": valids, "sources": sources, "indexes": indexes, "two": two}
    for r in list(indexes.values()) + two:
        r.free()
    ctx.close()


def _file_ids(res):
    """Row ids of every index file, in file order."""
    return [pq.read_table(pa.BufferReader(res.host_bytes(i)), columns=["id"]).column("id").to_numpy() for i in range(len(res.files))]


def _expected(d, file_ids, preds, deleted_src=()):
    m = F.predicate_mask(d["cols"], preds, d["valids"])
    if deleted_src:
        m = m & ~np.isin(d["cols"]["id"] // (N_ROWS // 2), list(deleted_src))
    return np.concatenate([ids[m[ids]] for ids in file_ids]) if file_ids else np.empty(0, np.int64)


def _run(d, files, key, projected, preds, sorted_on_key, deleted=()):
    b, st = d["ctx"].filter_scan_where(files, key, projected, preds, sorted_on_key=sorted_on_key, deleted_file_ids=list(deleted))
    out = {n: (v.copy(), None if val is None else val.copy()) for n, v, val in b.columns}
    rows = b.num_rows
    b.free()
    return out, rows


def _check(d, key, preds, projected=("id",), file_ids=None, files=None):
    if files is None:
        files, file_ids = d["indexes"][key].as_sources(), _file_ids(d["indexes"][key])
    want = _expected(d, file_ids, preds)
    proj = list(projected)
    for sorted_on_key in (True, False):
        out, rows = _run(d, files, key, proj + ["id"] if "id" not in proj else proj, preds, sorted_on_key)
        got = out["id"][0]
        assert rows == len(want), (key, preds, sorted_on_key)
        assert np.array_equal(got, want), (key, preds, sorted_on_key)
        for c in proj:  # projected values are the rows' own values
            v, valid = out[c]
            src = d["cols"][c][got]
            if c in d["valids"]:
                assert np.array_equal(valid.astype(bool), d["valids"][c][got])
                keep = valid.astype(bool)
                v, src = v[keep], src[keep]
            if v.dtype == object:
                assert list(v) == list(src)
            else:
                assert np.array_equal(v.view(np.uint8), np.ascontiguousarray(src).view(np.uint8)) or np.array_equal(v, src, equal_nan=True)
    return want


def _literal(rng, col, d):
    v = d["cols"][col]
    if v.dtype == object:
        return bytes(v[rng.integers(0, len(v))]).decode("utf-8", "replace") if rng.random() < 0.5 else bytes(v[rng.integers(0, len(v))])
    x = v[rng.integers(0, len(v))]
    if v.dtype.kind == "i":
        r = rng.random()
        return int(x) if r < 0.5 else (float(x) + 0.5 if r < 0.8 else float(x))
    r = rng.random()
    if r < 0.1:
        return float(rng.choice([np.nan, np.inf, -np.inf, 0.0, -0.0]))
    if r < 0.3:
        return int(np.nan_to_num(x, nan=0, posinf=0, neginf=0))
    return float(x)


def _random_conjunction(rng, d):
    out = []
    for _ in range(int(rng.integers(1, 5))):
        c = str(rng.choice(["i32", "i64", "f32", "f64", "t", "s", "n64"]))
        kind = rng.integers(0, 3)
        lo = _literal(rng, c, d) if kind != 1 else None
        hi = _literal(rng, c, d) if kind != 0 else None
        out.append((c, lo, bool(rng.random() < 0.4), hi, bool(rng.random() < 0.4)))
    return out


@pytest.mark.parametrize("seed", range(32))
def test_random_conjunctions_match_the_oracle(data, seed):
    rng = np.random.default_rng(1000 + seed)
    preds = _random_conjunction(rng, data)
    key = KEYS[seed % len(KEYS)]
    if rng.random() < 0.7:  # mostly with a predicate on the key, so the window search does work
        preds.append((key, _literal(rng, key, data), False, None, False))
    _check(data, key, preds, projected=("id",) if seed % 3 == 0 else (key, "s", "n64", "f32"))


EDGE_CASES = [
    ("f64", [("f64", 1.0, False, None, False)]),                       # NaN is above every number
    ("f64", [("f64", float("nan"), False, float("nan"), False)]),      # == NaN
    ("f64", [("f64", float("nan"), True, None, False)]),               # nothing above NaN
    ("f64", [("f64", None, False, float("nan"), True)]),               # every number
    ("f64", [("f64", -0.0, False, 0.0, False)]),                       # -0.0 == 0.0
    ("f64", [("f64", 0.0, True, None, False), ("f64", None, False, 1e-300, False)]),  # subnormals only
    ("f64", [("f64", None, False, -0.0, True)]),
    ("f64", [("f64", float("-inf"), False, float("-inf"), False)]),
    ("f64", [("f64", float("inf"), True, None, False)]),
    ("f64", [("f64", 12.5, True, None, False), ("f64", None, False, 20, True)]),
    ("f32", [("f32", 0.1, True, None, False)]),                        # (double)f > 0.1, not f > 0.1f
    ("f32", [("f32", 16777217, False, None, False)]),                  # long literal cast to float
    ("f32", [("f32", 2**60 + 2**36 + 1, False, None, False)]),         # ... rounded once: 2^60 + 2^37, not 2^60
    ("f32", [("f32", 0, True, 1, False)]),
    ("f32", [("f32", -0.0, False, -0.0, False)]),
    ("f32", [("f32", float("nan"), False, None, False)]),
    ("i64", [("i64", 1.5, True, None, False)]),                        # k > 1.5 is k >= 2
    ("i64", [("i64", float(2**53), True, None, False)]),               # rounded comparison beyond 2^53
    ("i64", [("i64", float(2**53), False, float(2**53), False)]),
    ("i64", [("i64", float(2**60), False, float(2**60), False)]),
    ("i64", [("i64", 2**53 + 1, False, 2**53 + 2, False)]),
    ("i64", [("i64", 2**63 - 1, True, None, False)]),                  # empty, no wrap-around
    ("i64", [("i64", None, False, -2**63, True)]),
    ("i64", [("i64", 1e30, False, None, False)]),
    ("i64", [("i64", None, False, 1e30, False)]),
    ("i64", [("i64", float("nan"), False, None, False)]),
    ("i32", [("i32", 2**40, False, None, False)]),                     # beyond the int32 range: empty
    ("i32", [("i32", -2**40, False, None, False)]),                    # every row
    ("i32", [("i32", None, False, 2**62, True)]),
    ("i32", [("i32", -0.5, True, 0.5, True)]),
    ("t", [("t", "abc", True, None, False)]),                          # strict string bounds
    ("t", [("t", None, False, "abc", True)]),
    ("t", [("t", "ab", True, "abd", True)]),
    ("t", [("t", b"\xff", False, None, False)]),
    ("t", [("t", "", False, "", False)]),
]


@pytest.mark.parametrize("case", range(len(EDGE_CASES)))
def test_edge_cases_of_spark_comparison(data, case):
    key, preds = EDGE_CASES[case]
    _check(data, key, preds, projected=("id", key))


def test_two_predicates_on_the_key_and_residuals_out_of_the_projection(data):
    _check(data, "i64", [("i64", -5000, False, None, False), ("i64", None, False, 90_000, True), ("i64", 0, True, None, False)])
    # predicate columns left out of the projection; a string residual; nulls never match
    _check(data, "i32", [("i32", -100, False, 500, False), ("s", "ab", False, "b", False), ("n64", None, False, 700, False)],
           projected=("id", "f64"))
    _check(data, "f64", [("t", "facebook", False, "facebook", False), ("f32", 0.0, True, None, False)], projected=("i32",))


def test_empty_results(data):
    for key in KEYS:
        want = _check(data, key, [("i64", 5, False, 4, False)])
        assert len(want) == 0
    want = _check(data, "i64", [("i64", 0, False, 10, False), ("n64", 5000, False, None, False)])
    assert len(want) == 0


def test_nullable_key_falls_back_and_nulls_never_match(data):
    """An index on a nullable column is scanned by the predicate path; null keys match no bound."""
    from hyperspace_b200 import _native as N

    d = data
    res, _ = d["ctx"].create_index(d["sources"], ["n64"], ["id", "s"], NB, output=N.HS_OUT_HOST)
    try:
        for preds in ([("n64", 0, False, None, False)], [("n64", None, False, 100.5, True), ("s", "", False, None, False)]):
            _check(d, "n64", preds, files=res.as_sources(), file_ids=_file_ids(res))
    finally:
        res.free()


def test_deleted_file_ids_with_residuals(data):
    d = data
    res = d["indexes"]["i64"]
    preds = [("i64", -10_000, False, 10_000, False), ("f64", 0.0, True, None, False), ("s", None, False, "b", False)]
    for deleted in ([0], [1], [0, 1]):
        want = _expected(d, _file_ids(res), preds, deleted_src=deleted)
        out, rows = _run(d, res.as_sources(), "i64", ["id", "f64"], preds, True, deleted)
        assert rows == len(want) and np.array_equal(out["id"][0], want), deleted


def test_buckets_with_two_files(data):
    d = data
    files, ids = [], []
    for res in d["two"]:
        files += res.as_sources()
        ids += _file_ids(res)
    for preds in ([("f64", -50.0, False, 50.0, True)], [("f64", 0.0, False, None, False), ("i32", None, False, 0, False)],
                  [("f64", float("nan"), False, None, False)]):
        _check(d, "f64", preds, projected=("id", "f64"), files=files, file_ids=ids)


def test_hs_filter_scan_is_a_one_predicate_call(data):
    """hs_filter_scan and hs_filter_scan_where with that predicate give byte-identical batches."""
    d = data
    ctx = d["ctx"]
    cases = {"i32": [(-100, 100), (None, 0), (5, None), (2000, 3000), (None, None)],
             "i64": [(-5000, 5000), (2**53, None), (None, -10**6), (10, 9)],
             "t": [("ab", "abd"), ("facebook", "facebook"), (None, "b"), ("zz", None)]}
    for key, bounds in cases.items():
        files = d["indexes"][key].as_sources()
        proj = [key, "s", "f64", "id", "t"] if key != "t" else ["t", "s", "id"]
        for lo, hi in bounds:
            for sorted_on_key in (True, False):
                a, _ = ctx.filter_scan(files, key, proj, lo=lo, hi=hi, sorted_on_key=sorted_on_key)
                preds = [(key, lo, False, hi, False)] if (lo is not None or hi is not None) else []
                b, _ = ctx.filter_scan_where(files, key, proj, preds, sorted_on_key=sorted_on_key)
                assert a.num_rows == b.num_rows
                for (na, va, ma), (nb, vb, mb) in zip(a.columns, b.columns):
                    assert na == nb and va.dtype == vb.dtype
                    if va.dtype == object:
                        assert list(va) == list(vb)
                    else:
                        assert va.tobytes() == vb.tobytes()
                    assert (ma is None) == (mb is None) and (ma is None or ma.tobytes() == mb.tobytes())
                a.free()
                b.free()


def test_refusals(data):
    from hyperspace_b200 import _native as N

    d = data
    files = d["indexes"]["i64"].as_sources()

    def code(preds, key="i64"):
        with pytest.raises(N.HyperspaceGpuError) as e:
            d["ctx"].filter_scan_where(files, key, ["id"], preds)
        return e.value.code

    assert code([("t", 1, False, None, False)]) == N.HS_EUNSUPPORTED          # numeric literal, string column
    assert code([("f64", "a", False, None, False)]) == N.HS_EUNSUPPORTED      # string literal, numeric column
    assert code([("i64", "a", False, None, False)]) == N.HS_EUNSUPPORTED      # ... also on the key
    with pytest.raises(N.HyperspaceGpuError) as e:                            # boolean column (source files)
        d["ctx"].filter_scan_where(d["sources"], None, ["id"], [("b", 0, False, None, False)], sorted_on_key=False)
    assert e.value.code == N.HS_EUNSUPPORTED
    assert code([("i64", i, False, None, False) for i in range(17)]) == N.HS_EUNSUPPORTED
    assert code([("nope", 1, False, None, False)]) in (N.HS_EINVAL, N.HS_EUNSUPPORTED)
    assert code([("t", "x" * 70_000, False, None, False)]) in (N.HS_EINVAL, N.HS_EUNSUPPORTED)
    # hs_filter_scan keeps refusing floating-point keys (its bounds are int64)
    with pytest.raises(N.HyperspaceGpuError) as e:
        d["ctx"].filter_scan(d["indexes"]["f64"].as_sources(), "f64", ["id"], lo=0, hi=1)
    assert e.value.code == N.HS_EUNSUPPORTED


# ---- through the Hyperspace API ----------------------------------------------------------------------------------------

def _write(dirpath, name, cols):
    os.makedirs(dirpath, exist_ok=True)
    pq.write_table(pa.table(cols), os.path.join(dirpath, name), compression="snappy")


def _table(first, n):
    rng = np.random.default_rng(first)
    return {"k": np.arange(first, first + n, dtype=np.int64) % 5000, "v1": rng.integers(0, 1000, n).astype(np.int64),
            "v2": rng.normal(15, 10, n), "v3": rng.integers(0, 100, n).astype(np.int32)}


def _sorted_rows(res, cols):
    return sorted(zip(*[np.asarray(res[c]).tolist() for c in cols]), key=repr)


@pytest.fixture()
def env(tmp_path):
    from hyperspace_b200.hyperspace import Hyperspace
    from hyperspace_b200.session import HyperspaceSession

    s = HyperspaceSession({"spark.hyperspace.system.path": str(tmp_path / "indexes"), "spark.hyperspace.index.numBuckets": "8"})
    yield s, Hyperspace(s), tmp_path
    s.stop()


def test_conjunction_through_the_api_with_and_without_the_index(env):
    from hyperspace_b200.index_config import IndexConfig
    from hyperspace_b200.session import col

    s, hs, tmp = env
    parts = [_table(0, 30_000), _table(30_000, 20_000)]
    for i, p in enumerate(parts):
        _write(tmp / "t", f"p{i}.parquet", p)
    df = s.read.parquet(str(tmp / "t"))
    hs.createIndex(df, IndexConfig("kidx", ["k"], ["v1", "v2"]))
    allc = {c: np.concatenate([p[c] for p in parts]) for c in parts[0]}
    q = df.filter(col("k").between(100, 300) & (col("v1") >= 500)).select("k", "v2")
    s.disableHyperspace()
    assert "GpuSourceScan" in q.explain()
    base = q.collect()
    s.enableHyperspace()
    assert "Name: kidx" in q.explain()
    got = q.collect()
    m = (allc["k"] >= 100) & (allc["k"] <= 300) & (allc["v1"] >= 500)
    assert len(got["k"]) == int(m.sum()) > 0
    assert _sorted_rows(got, ["k", "v2"]) == _sorted_rows(base, ["k", "v2"])
    # no first indexed column in the filter: a source scan that still answers
    q2 = df.filter((col("v1") >= 990) & (col("v2") > 12.5)).select("k", "v1")
    assert "GpuSourceScan" in q2.explain()
    assert len(q2.collect()["k"]) == int(((allc["v1"] >= 990) & (allc["v2"] > 12.5)).sum())
    # Hybrid Scan: an appended file is scanned raw with the same conjunction and unioned
    extra = _table(50_000, 5_000)
    _write(tmp / "t", "p9.parquet", extra)
    s.conf.set("spark.hyperspace.index.hybridscan.enabled", True)
    df2 = s.read.parquet(str(tmp / "t"))
    q3 = df2.filter(col("k").between(100, 300) & (col("v1") >= 500) & (col("v2") < 20)).select("k", "v1", "v2")
    assert "hybridScan(appended=1" in q3.explain()
    allc2 = {c: np.concatenate([allc[c], extra[c]]) for c in allc}
    m3 = (allc2["k"] >= 100) & (allc2["k"] <= 300) & (allc2["v1"] >= 500) & (allc2["v2"] < 20)
    got3 = q3.collect()
    assert _sorted_rows(got3, ["k", "v1", "v2"]) == sorted(zip(allc2["k"][m3].tolist(), allc2["v1"][m3].tolist(), allc2["v2"][m3].tolist()), key=repr)


def test_index_on_a_double_column(env):
    from hyperspace_b200.index_config import IndexConfig
    from hyperspace_b200.session import col

    s, hs, tmp = env
    t = _table(0, 40_000)
    t["v2"][:5] = [np.nan, -0.0, 0.0, np.inf, 12.5]
    _write(tmp / "d", "a.parquet", t)
    df = s.read.parquet(str(tmp / "d"))
    hs.createIndex(df, IndexConfig("didx", ["v2"], ["k"]))
    s.enableHyperspace()
    q = df.filter((col("v2") > 12.5) & (col("v2") < 20)).select("v2", "k")
    assert "Name: didx" in q.explain()
    got = q.collect()
    m = (t["v2"] > 12.5) & (t["v2"] < 20)
    assert _sorted_rows(got, ["v2", "k"]) == sorted(zip(t["v2"][m].tolist(), t["k"][m].tolist()), key=repr)
    nan_rows = df.filter(col("v2") >= 1.0).select("v2").collect()["v2"]  # NaN sorts above every number
    assert int(np.isnan(nan_rows).sum()) == 1 and len(nan_rows) == int((t["v2"] >= 1.0).sum()) + 1


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


def test_sample_data_conjunctions(env):
    from hyperspace_b200.index_config import IndexConfig
    from hyperspace_b200.session import col

    s, hs, tmp = env
    cols = list(zip(*SAMPLE))
    _write(tmp / "sample", "a.parquet", {"Date": pa.array(cols[0]), "RGUID": pa.array(cols[1]), "Query": pa.array(cols[2]),
                                          "imprs": pa.array(cols[3], pa.int32()), "clicks": pa.array(cols[4], pa.int32())})
    df = s.read.parquet(str(tmp / "sample"))
    hs.createIndex(df, IndexConfig("qidx", ["Query"], ["clicks", "Date"]))
    hs.createIndex(df, IndexConfig("didx", ["Date"], ["Query", "clicks"]))
    s.enableHyperspace()
    q = df.filter((col("Query") == "facebook") & (col("clicks") >= 3000)).select("Query", "clicks")
    assert "Name: qidx" in q.explain()
    assert sorted(q.collect()["clicks"].tolist()) == [3000, 3000, 3000, 3000, 3000, 4000]
    q2 = df.filter(col("Date") >= "2018-09-03").select("Date", "Query")
    assert "Name: didx" in q2.explain()
    got = sorted(zip(q2.collect()["Date"].tolist(), q2.collect()["Query"].tolist()))
    assert got == sorted((d, q) for d, _, q, _, _ in SAMPLE if d >= "2018-09-03")


def test_source_scan_without_a_filter_keeps_rows_with_nulls(env):
    """No filter: every row comes back, also those whose first column is null (Spark's scan drops nothing)."""
    from hyperspace_b200.session import col

    s, _, tmp = env
    k = pa.array([1, None, 3, None, 5], pa.int64())
    v = pa.array([10, 20, 30, 40, 50], pa.int64())
    os.makedirs(tmp / "n", exist_ok=True)
    pq.write_table(pa.table({"k": k, "v": v}), str(tmp / "n" / "a.parquet"))
    df = s.read.parquet(str(tmp / "n"))
    assert sorted(df.select("v").collect()["v"].tolist()) == [10, 20, 30, 40, 50]
    assert sorted(df.select("k", "v").collect()["v"].tolist()) == [10, 20, 30, 40, 50]
    assert sorted(df.filter(col("v") >= 30).select("v").collect()["v"].tolist()) == [30, 40, 50]
