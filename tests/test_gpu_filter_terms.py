"""GPU filter scans and join sides with NOT, IS [NOT] NULL, null-safe equality and string patterns (hs_predicate_any flags):
every form on every key type, on sorted index files and unsorted source files, on the key and on other (nullable) columns,
on a nullable key, on both join sides, and through the Hyperspace API with Hybrid Scan and lineage.  Answers are compared
with tests/filter_terms_oracle.py as exact sequences of row ids (file, then row)."""
import decimal
import io
import os

import numpy as np
import pyarrow as pa
import pyarrow.parquet as pq
import pytest

import filter_terms_oracle as FT

pytestmark = pytest.mark.gpu

N_ROWS = 40_000
NB = 16
KEYS = ["i32", "i64", "f32", "f64", "s", "ts", "d9"]
WORDS = ["", "a", "ab", "abc", "abd", "b", "été", "facebook", "zz", "ÿ", "ÿÿ", "donde", "€uro", "𝄞 clef", "a%b", "a_b", "x\\y"]


def _make_columns(seed=5):
    rng = np.random.default_rng(seed)
    n = N_ROWS
    i32 = rng.integers(-300, 300, n).astype(np.int32)
    i32[:2] = [np.iinfo(np.int32).min, np.iinfo(np.int32).max]
    i64 = rng.integers(-2000, 2000, n).astype(np.int64)
    i64[:2] = [np.iinfo(np.int64).max, np.iinfo(np.int64).min]
    f64 = np.round(rng.normal(0, 10, n), 0)
    f64[100:106] = [np.nan, np.inf, -np.inf, 0.0, -0.0, 5.0]
    f32 = np.round(rng.normal(0, 10, n), 0).astype(np.float32)
    f32[200:206] = np.array([np.nan, np.inf, -np.inf, 0.0, -0.0, 5.0], np.float32)
    words = [w.encode() for w in WORDS]
    s = np.array([words[i] for i in rng.integers(0, len(words), n)], dtype=object)
    long_rows = rng.random(n) < 0.02  # values of 1-2 KB
    for i in np.flatnonzero(long_rows):
        s[i] = ("€" * int(rng.integers(300, 700)) + WORDS[int(rng.integers(0, len(WORDS)))]).encode()
    ts = rng.integers(0, 3000, n).astype(np.int64) * 1_000_000
    d9 = rng.integers(-3000, 3000, n).astype(np.int64)  # unscaled, scale 2
    n64 = rng.integers(0, 300, n).astype(np.int64)
    ns = np.array([words[i] for i in rng.integers(0, len(words), n)], dtype=object)
    ids = np.arange(n, dtype=np.int64)
    cols = {"i32": i32, "i64": i64, "f32": f32, "f64": f64, "s": s, "ts": ts, "d9": d9, "n64": n64, "ns": ns, "id": ids}
    return cols, {"n64": rng.random(n) >= 0.2, "ns": rng.random(n) >= 0.2}


def _arrow(cols, valids, rows):
    out = {}
    for name, v in cols.items():
        v = v[rows]
        mask = ~valids[name][rows] if name in valids else None
        if name in ("s", "ns"):
            out[name] = pa.array([x.decode() for x in v], pa.string(), mask=mask)
        elif name == "ts":
            out[name] = pa.array(v, pa.timestamp("us"))
        elif name == "d9":
            out[name] = pa.array([decimal.Decimal(int(x)).scaleb(-2) for x in v], pa.decimal128(9, 2))
        else:
            out[name] = pa.array(v, mask=mask)
    return pa.table(out)


def _parquet_bytes(table):
    sink = io.BytesIO()
    pq.write_table(table, sink, compression="NONE", data_page_size=16 << 10, row_group_size=10_000)
    return sink.getvalue()


@pytest.fixture(scope="module")
def data():
    from hyperspace_b200 import _native as N

    ctx = N.Context(0)
    cols, valids = _make_columns()
    halves = [np.arange(0, N_ROWS // 2), np.arange(N_ROWS // 2, N_ROWS)]
    sources = [N.FileImage(path=f"src{i}.parquet", data=_parquet_bytes(_arrow(cols, valids, r)), file_id=i)
               for i, r in enumerate(halves)]
    indexes = {k: ctx.create_index(sources, [k], [c for c in cols if c != k], NB, output=N.HS_OUT_HOST)[0] for k in KEYS + ["n64", "ns"]}
    yield {"ctx": ctx, "cols": cols, "valids": valids, "sources": sources, "indexes": indexes}
    for r in indexes.values():
        r.free()
    ctx.close()


def _file_ids(res):
    return [pq.read_table(pa.BufferReader(res.host_bytes(i)), columns=["id"]).column("id").to_numpy() for i in range(len(res.files))]


def _ids(batch):
    out = next(v.copy() for n, v, _ in batch.columns if n == "id")
    batch.free()
    return out


def _scan(d, files, key, terms, sorted_on_key=True, buckets=None, preds=()):
    b, st = d["ctx"].filter_scan_any(files, key, ["id"], list(preds), terms, sorted_on_key=sorted_on_key, file_buckets=buckets,
                                     num_buckets=NB if buckets is not None else 0)
    return _ids(b), st


def _check(d, index_key, terms, oterms, preds=()):
    """the terms over the index on index_key (sorted path) and over the source files (unsorted path)"""
    m = FT.mask(d["cols"], oterms, d["valids"], preds)
    res = d["indexes"][index_key]
    want = np.concatenate([ids[m[ids]] for ids in _file_ids(res)])
    got, _ = _scan(d, res.as_sources(), index_key, terms, preds=preds)
    assert np.array_equal(got, want), (index_key, oterms, len(got), len(want))
    got, _ = _scan(d, d["sources"], None, terms, sorted_on_key=False, preds=preds)
    assert np.array_equal(got, np.flatnonzero(m)), (index_key, oterms, "unsorted")
    return m


def _literal(d, key, row):
    """(Python literal for the engine, literal for the oracle) of the value at row"""
    v = d["cols"][key][row]
    if key == "d9":
        return decimal.Decimal(int(v)).scaleb(-2), int(v)
    if key in ("s", "ns"):
        return v.decode(), v
    if key in ("f32", "f64"):
        return float(v), float(v)
    return int(v), int(v)


def _forms(d, key):
    """(Predicate, oracle term) of every non-pattern form on column key"""
    from hyperspace_b200.session import col

    (a, oa), (b, ob) = sorted([_literal(d, key, 7), _literal(d, key, 11)], key=lambda x: x[1], reverse=True)  # b <= a
    c = col(key)
    return [(c != a, ("not", ("in", key, [oa]))),
            (~c.isin(a, b), ("not", ("in", key, [oa, ob]))),
            (~c.isin(a, None), ("not", ("in", key, [oa, None]))),
            (c.isNull(), ("isnull", key)),
            (c.isNotNull(), ("isnotnull", key)),
            (c.eqNullSafe(a), ("eqns", key, oa)),
            (~c.eqNullSafe(a), ("not", ("eqns", key, oa))),
            (~(c >= a), ("not", ("range", key, oa, False, None, False))),
            (~c.between(b, a) if key not in ("s", "ns") else ~((c >= b) & (c <= a)), ("not", ("range", key, ob, False, oa, False))),
            (c.isNull() | (c > a), ("or", [("isnull", key), ("range", key, oa, True, None, False)])),
            (c.eqNullSafe(a) | c.eqNullSafe(b), ("or", [("eqns", key, oa), ("eqns", key, ob)]))]


def _native(p):
    return [t.as_native() for t in p.anys]


@pytest.mark.parametrize("key", KEYS)
def test_forms_on_every_key_type(data, key):
    for p, o in _forms(data, key):
        m = _check(data, key, _native(p), [o])
        assert 0 < m.sum() < N_ROWS or o[0] in ("isnull", "isnotnull") or o[1][0] == "in" and None in o[1][2], o


def test_not_equal_on_special_floats(data):
    from hyperspace_b200.session import col

    for key in ("f32", "f64"):
        for lit in (-0.0, float("nan"), float("inf")):
            _check(data, key, _native(col(key) != lit), [("not", ("in", key, [lit]))])


def _patterns(key):
    from hyperspace_b200.session import col

    c = col(key)
    out = []
    for p in ["a", "", "ÿ", "€", "fa", "zz"]:
        out += [(c.startswith(p), ("startswith", key, p.encode())), (~c.startswith(p), ("not", ("startswith", key, p.encode())))]
    for p in ["b", "", "€", "clef", "€€€b", "ook"]:
        out += [(c.endswith(p), ("endswith", key, p.encode())), (c.contains(p), ("contains", key, p.encode())),
                (~c.contains(p), ("not", ("contains", key, p.encode())))]
    for p in ["a%", "a%b", "%b", "_b", "a_", "%€%b", "%_%", "abc", "a\\%b", "a\\_b", "x\\\\y", "%é_", "_", "%", "€%€%€",
              "𝄞%", "_ clef", "%o_d%"]:
        out += [(c.like(p), ("like", key, p)), (~c.like(p), ("not", ("like", key, p)))]
    out.append((c.startswith("ab") | c.isNull(), ("or", [("startswith", key, b"ab"), ("isnull", key)])))
    return out


@pytest.mark.parametrize("key", ["s", "ns"])
def test_patterns_on_the_key_and_on_a_nullable_column(data, key):
    for p, o in _patterns(key):
        _check(data, "s", _native(p), [o])          # key "s": on the sorted key; "ns": a residual column
        if key == "ns":
            _check(data, "ns", _native(p), [o])     # nullable key: the predicate scan over every row


def test_terms_on_other_and_nullable_columns(data):
    from hyperspace_b200.session import col

    for key in ("n64", "ns", "f64"):
        for p, o in _forms(data, key):
            _check(data, "i64", _native(p), [o], preds=[("i64", -1000, False, 1000, False)])
    for p, o in _forms(data, "n64"):
        _check(data, "n64", _native(p), [o])   # the nullable key
    # several terms AND-ed, on the key and elsewhere
    p = (col("s") != "ab") & col("ns").like("%b") & ~col("n64").eqNullSafe(3) & (col("i32") != 0)
    _check(data, "s", _native(p), [("not", ("in", "s", [b"ab"])), ("like", "ns", "%b"), ("not", ("eqns", "n64", 3)),
                                    ("not", ("in", "i32", [0]))])


def _profiled(d, files, key, terms):
    """(ids, stats, per-kernel profile) of one sorted scan"""
    ctx = d["ctx"]
    ctx.profile_enable(True)
    ctx.profile_report()
    try:
        ids, st = _scan(d, files, key, terms)
        return ids, st, ctx.profile_report()
    finally:
        ctx.profile_enable(False)


def test_key_terms_fold_into_windows(data):
    """NOT, NOT IN and prefixes on the sorted key are windows, not a residual: k_range_bounds searches 2 work items per
    file for `k != v`, n + 1 for NOT IN of n values, 1 for a prefix and 2 for its NOT, and no mask kernel runs; a
    pattern that is not a prefix searches its prefix's window and leaves the rest to k_pattern_mask."""
    from hyperspace_b200.session import col

    d = data
    cases = []
    vals = sorted({int(v) for v in d["cols"]["i64"][5:40] if abs(v) < 1500})[:6]
    cases += [("i64", col("i64") != vals[0], 2, ("not", ("in", "i64", [vals[0]]))),
              ("i64", ~col("i64").isin(*vals), len(vals) + 1, ("not", ("in", "i64", vals))),
              ("i64", col("i64").isNotNull(), 1, ("isnotnull", "i64")),
              ("f64", col("f64") != -0.0, 2, ("not", ("in", "f64", [-0.0]))),
              ("s", col("s").startswith("ab"), 1, ("startswith", "s", b"ab")),
              ("s", ~col("s").startswith("ab"), 2, ("not", ("startswith", "s", b"ab"))),
              ("s", col("s").like("fa%"), 1, ("like", "s", "fa%")),
              ("s", col("s") != "ab", 2, ("not", ("in", "s", [b"ab"])))]
    for key, p, per_file, o in cases:
        res = d["indexes"][key]
        ids, st, rep = _profiled(d, res.as_sources(), key, _native(p))
        m = FT.mask(d["cols"], [o], d["valids"])
        assert np.array_equal(ids, np.concatenate([x[m[x]] for x in _file_ids(res)])), o
        assert rep["k_range_bounds"]["items"] == per_file * len(res.files), (o, rep["k_range_bounds"])
        assert "k_predicate_mask" not in rep and "k_pattern_mask" not in rep, (o, rep)
    # the key's window of a LIKE prefix, then the matcher over it
    res = d["indexes"]["s"]
    ids, st, rep = _profiled(d, res.as_sources(), "s", _native(col("s").like("a%b")))
    m = FT.mask(d["cols"], [("like", "s", "a%b")], d["valids"])
    assert np.array_equal(ids, np.concatenate([x[m[x]] for x in _file_ids(res)]))
    assert rep["k_range_bounds"]["items"] == len(res.files) and rep["k_pattern_mask"]["launches"] == 1
    # IS NULL on a null-free key: the empty set, no window searched
    ids, st, rep = _profiled(d, res.as_sources(), "s", _native(col("s").isNull()))
    assert len(ids) == 0 and rep.get("k_range_bounds", {}).get("items", 0) == 0


def test_null_safe_equality_prunes_like_equality(data):
    from hyperspace_b200.session import col

    d = data
    for key in ("i64", "s"):
        res = d["indexes"][key]
        files, buckets = res.as_sources(), [f.bucket for f in res.files]
        a, _ = _literal(d, key, 7)
        got, st = _scan(d, files, key, _native(col(key).eqNullSafe(a)), buckets=buckets)
        want, st_eq = _scan(d, files, key, [(key, [a], [])], buckets=buckets)
        _, st_full = _scan(d, files, key, _native(col(key).eqNullSafe(a)))
        assert np.array_equal(got, want) and len(got) > 0
        assert st["bytes_in"] == st_eq["bytes_in"] < st_full["bytes_in"]
    # IS NULL on a nullable key reads every file: the nulls are in the null key's bucket
    res = d["indexes"]["n64"]
    got, st = _scan(d, res.as_sources(), "n64", _native(col("n64").isNull()), buckets=[f.bucket for f in res.files])
    assert len(got) == int((~d["valids"]["n64"]).sum())


def test_refusals(data):
    from hyperspace_b200 import _native as N

    d, ctx = data, data["ctx"]
    files = d["indexes"]["i64"].as_sources()

    def refused(code, text, terms):
        with pytest.raises(N.HyperspaceGpuError) as e:
            ctx.filter_scan_any(files, "i64", ["id"], [], terms)
        assert e.value.code == code and text in e.value.message, e.value.message

    refused(N.HS_EUNSUPPORTED, "string pattern", [("n64", ["1"], [], N.HS_TERM_CONTAINS)])
    refused(N.HS_EINVAL, "it is not allowed to end with the escape character", [("ns", ["ab\\"], [], N.HS_TERM_LIKE)])
    refused(N.HS_EINVAL, "not allowed to precede 'x'", [("ns", ["a\\x"], [], N.HS_TERM_LIKE)])
    refused(N.HS_EINVAL, "unknown flags", [("ns", ["a"], [], 1 << 9)])
    refused(N.HS_EINVAL, "one string value", [("ns", ["a", "b"], [], N.HS_TERM_ENDS_WITH)])
    refused(N.HS_EUNSUPPORTED, "decimal", [("d9", [1.5], [], N.HS_TERM_NOT)])
    got, _ = _scan(d, files, "i64", [("i64", [int(d["cols"]["i64"][3])], [])])
    assert len(got) > 0


def test_join_sides_with_terms(data):
    from hyperspace_b200.session import col

    d, ctx = data, data["ctx"]
    r = d["indexes"]["i64"]
    args = (r.as_sources(), [f.bucket for f in r.files], r.as_sources(), [f.bucket for f in r.files], NB, ["i64"], ["i64"], ["id"], ["id"])
    lp, lo = ~col("ns").like("%b"), ("not", ("like", "ns", "%b"))
    rp, ro = ~col("n64").eqNullSafe(5), ("not", ("eqns", "n64", 5))
    lp2, lo2 = col("s").contains("€"), ("contains", "s", "€".encode())
    j, _ = ctx.bucket_join_any(*args, [], [], _native(lp) + _native(lp2), _native(rp))
    got = sorted(zip(*[v.tolist() for _, v, _ in j.columns]))
    j.free()
    lm = FT.mask(d["cols"], [lo, lo2], d["valids"])
    rm = FT.mask(d["cols"], [ro], d["valids"])
    by_key = {}
    for i in np.flatnonzero(rm):
        by_key.setdefault(int(d["cols"]["i64"][i]), []).append(int(i))
    want = sorted((int(i), j) for i in np.flatnonzero(lm) for j in by_key.get(int(d["cols"]["i64"][i]), []))
    assert got == want and len(want) > 0


# ---- the Hyperspace API --------------------------------------------------------------------------------------------------

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
    key = lambda r: sorted(zip(*[[repr(x) for x in r[c].tolist()] for c in cols]))  # noqa: E731
    assert key(got) == key(base)
    return got


def _table(rng, n, base=0):
    words = ["apple", "apricot", "banana", "été", "€uro", "grape", "", "a_b"]
    k = rng.integers(0, 500, n).astype(np.int64) + base
    s = [words[i] for i in rng.integers(0, len(words), n)]
    v = pa.array(rng.normal(size=n), mask=rng.random(n) < 0.1)
    return {"k": k, "s": pa.array(s, mask=rng.random(n) < 0.1), "v": v}


def test_hyperspace_api_with_and_without_hyperspace(env):
    from hyperspace_b200.index_config import IndexConfig
    from hyperspace_b200.session import col

    s, hs, tmp = env
    rng = np.random.default_rng(9)
    for i in range(3):
        _write(tmp / "t", f"f{i}.parquet", _table(rng, 4000))
    df = s.read.parquet(str(tmp / "t"))
    hs.createIndex(df, IndexConfig("kidx", ["k"], ["s", "v"]))
    hs.createIndex(df, IndexConfig("sidx", ["s"], ["k", "v"]))
    s.enableHyperspace()
    queries = [(df.filter(col("k") != 7).select("k", "v"), "kidx", "NOT (k IN (7))"),
               (df.filter(~col("k").isin(1, 2, 3) & (col("k") < 50)).select("k", "s"), "kidx", None),
               (df.filter(col("k").eqNullSafe(42)).select("k", "v"), "kidx", "k <=> 42"),
               (df.filter(col("s").isNull()).select("s", "k"), "sidx", "s IS NULL"),
               (df.filter(col("s").isNotNull() & (col("k") < 3)).select("s", "k"), None, "s IS NOT NULL"),
               (df.filter(col("s").startswith("ap")).select("s", "k"), "sidx", "StartsWith(s, 'ap')"),
               (df.filter(col("s").like("%a_a%")).select("s", "k"), "sidx", "s LIKE '%a_a%'"),
               (df.filter(~col("s").endswith("e") & col("v").isNotNull()).select("s", "v"), "sidx", None),
               (df.filter(col("s").startswith("€") | col("s").isNull()).select("s", "k"), "sidx", None)]
    for q, idx, text in queries:
        plan = q.explain()
        assert idx is None or f"Name: {idx}" in plan, plan
        assert text is None or text in plan, plan
        _same_answers(s, q, q.columns)
    # Hybrid Scan: an appended file
    s.conf.set("spark.hyperspace.index.hybridscan.enabled", True)
    _write(tmp / "t", "f3.parquet", _table(rng, 400, base=450))
    df = s.read.parquet(str(tmp / "t"))
    for q in (df.filter(col("k") != 460).select("k", "v"), df.filter(col("s").like("_p%")).select("s", "k")):
        assert "hybridScan(appended=1" in q.explain()
        _same_answers(s, q, q.columns)


def test_hyperspace_api_with_deleted_lineage_ids(env):
    from hyperspace_b200.index_config import IndexConfig
    from hyperspace_b200.session import col

    s, hs, tmp = env
    s.conf.set("spark.hyperspace.index.lineage.enabled", True)
    rng = np.random.default_rng(4)
    for i in range(6):
        _write(tmp / "t", f"f{i}.parquet", _table(rng, 1000))
    hs.createIndex(s.read.parquet(str(tmp / "t")), IndexConfig("idx", ["s"], ["k", "v"]))
    os.remove(tmp / "t" / "f5.parquet")
    s.enableHyperspace()
    s.conf.set("spark.hyperspace.index.hybridscan.enabled", True)
    df = s.read.parquet(str(tmp / "t"))
    for q in (df.filter(col("s") != "apple").select("s", "k"), df.filter(col("s").endswith("a")).select("s", "k"),
              df.filter(~col("s").eqNullSafe("grape")).select("s", "v")):
        assert "deletedIds=[5]" in q.explain() and "Name: idx" in q.explain()
        _same_answers(s, q, q.columns)
