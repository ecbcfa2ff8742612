"""GPU filter scans and join sides with Spark functions in expression comparisons (year, substring, datediff, abs,
coalesce, ...): over pyarrow-written sources with date32, timestamp (INT64 micros and INT96), PLAIN and dictionary strings
and binary columns with nulls; sorted index scans with key windows and unsorted source scans; NOT and <=>; below one side
of every join type; the Hyperspace API; and profiled calls showing that calls without functions launch what they did
before, and calls with them k_func_mask once per filtered side.  Answers are compared with tests/filter_func_oracle.py as
exact sequences of row ids."""
import datetime
import io

import numpy as np
import pyarrow as pa
import pyarrow.parquet as pq
import pytest

import filter_func_oracle as FF

pytestmark = pytest.mark.gpu

N_ROWS = 6_000
NB = 8
DAY_US = FF.DAY_US
TYPES = {"id": "long", "k": "integer", "d": "date", "d2": "date", "ts": "timestamp", "s": "string", "sd": "string",
         "b": "binary", "i": "integer", "x": "double"}
PHONES = ["13-555-0100", "31-555-0101", "13-9", "", "é€😀-13", "1", "日本-13", "23-0000"]


def _make_columns(seed=9):
    rng = np.random.default_rng(seed)
    n = N_ROWS
    cols = {"id": np.arange(n, dtype=np.int64), "k": rng.integers(0, 400, n).astype(np.int32),
            "d": rng.integers(8000, 11000, n).astype(np.int32),  # 1991 .. 2000
            "ts": rng.integers(-2_000_000_000, 4_000_000_000, n).astype(np.int64) * 1_000_000 + rng.integers(0, 1_000_000, n),
            "i": rng.integers(-40, 40, n).astype(np.int32), "x": rng.normal(0, 1, n)}
    cols["d2"] = (cols["d"] + rng.integers(-10, 60, n)).astype(np.int32)
    cols["ts"][:6] = [0, -1, DAY_US - 1, DAY_US, -DAY_US, -DAY_US - 1]
    cols["s"] = [PHONES[j].encode() for j in rng.integers(0, len(PHONES), n)]
    cols["sd"] = [PHONES[j].encode() for j in rng.integers(0, 3, n)]
    cols["b"] = [bytes(rng.integers(0, 256, int(m)).astype(np.uint8)) for m in rng.integers(0, 6, n)]
    valids = {c: rng.random(n) >= 0.1 for c in TYPES if c not in ("id", "k")}
    for v in valids.values():
        v[:6] = True
    return cols, valids


def _arrow(cols, valids, rows):
    out = {}
    arrow_types = {"id": pa.int64(), "k": pa.int32(), "d": pa.date32(), "d2": pa.date32(), "ts": pa.timestamp("us"), "s": pa.string(),
                   "sd": pa.string(), "b": pa.binary(), "i": pa.int32(), "x": pa.float64()}
    for name, t in arrow_types.items():
        v = cols[name]
        vals = [v[r] for r in rows] if isinstance(v, list) else v[rows]
        if name in ("s", "sd"):
            vals = [x.decode() for x in vals]
        mask = ~valids[name][rows] if name in valids else None
        out[name] = pa.array(vals, t, mask=mask)
    return pa.table(out)


def _parquet_bytes(table, int96=False):
    sink = io.BytesIO()
    pq.write_table(table, sink, compression="NONE", data_page_size=16 << 10, row_group_size=2_000, use_dictionary=["sd"],
                   use_deprecated_int96_timestamps=int96)
    return sink.getvalue()


@pytest.fixture(scope="module")
def data():
    from hyperspace_b200 import _native as N

    ctx = N.Context(0)
    cols, valids = _make_columns()
    halves = [np.arange(0, N_ROWS // 2), np.arange(N_ROWS // 2, N_ROWS)]
    sources = [N.FileImage(path=f"src{i}.parquet", data=_parquet_bytes(_arrow(cols, valids, r)), file_id=i) for i, r in enumerate(halves)]
    int96 = [N.FileImage(path=f"int96_{i}.parquet", data=_parquet_bytes(_arrow(cols, valids, r), int96=True), file_id=i)
             for i, r in enumerate(halves)]
    idx = ctx.create_index(sources, ["id"], [c for c in TYPES if c != "id"], NB, output=N.HS_OUT_HOST)[0]
    yield {"ctx": ctx, "cols": cols, "valids": valids, "sources": sources, "int96": int96, "index": idx}
    idx.free()
    ctx.close()


def C(n):
    return ("column", n)


def L(v):
    return ("literal", v)


def F(name, *args):
    out = [n for a in args for n in a]
    return out + [("coalesce", len(args)) if name == "coalesce" else (name,)]


def _mask(d, exprs, preds=()):
    columns = {c: (TYPES[c], list(d["cols"][c]) if isinstance(d["cols"][c], list) else d["cols"][c].tolist(), d["valids"].get(c))
               for c in TYPES}
    m = np.ones(N_ROWS, bool)
    for left, op, right, *neg in exprs:
        m &= FF.mask(left, op, right, bool(neg and neg[0]), columns, N_ROWS)
    for c, lo, ls, hi, hs in preds:
        v = d["cols"][c]
        if lo is not None:
            m &= (v > lo) if ls else (v >= lo)
        if hi is not None:
            m &= (v < hi) if hs else (v <= hi)
    return m


def _native(exprs):
    return [(l, op, r, 1 if (neg and neg[0]) else 0) for l, op, r, *neg in exprs]


def _file_ids(res):
    return [pq.read_table(pa.BufferReader(res.host_bytes(i)), columns=["id"]).column("id").to_numpy() for i in range(len(res.files))]


def _ids(batch):
    out = next(v.copy() for n, v, _ in batch.columns if n == "id")
    batch.free()
    return out


def _check(d, exprs, preds=()):
    ctx = d["ctx"]
    m = _mask(d, exprs, preds)
    want = np.concatenate([ids[m[ids]] for ids in _file_ids(d["index"])])
    b, _ = ctx.filter_scan_expr(d["index"].as_sources(), "id", ["id"], list(preds), [], [], _native(exprs), sorted_on_key=True)
    got = _ids(b)
    assert np.array_equal(got, want), (exprs, preds, len(got), len(want))
    for files in (d["sources"], d["int96"]):
        b, _ = ctx.filter_scan_expr(files, None, ["id"], list(preds), [], [], _native(exprs), sorted_on_key=False)
        assert np.array_equal(_ids(b), np.flatnonzero(m)), (exprs, preds, "unsorted", files[0].path)
    return m


EXPRS = [
    (F("year", [C("d")]), "=", [L(1995)]),
    (F("substring", [C("s")], [L(1)], [L(2)]), "=", [L("13")]),            # TPC-H Q22's country code, PLAIN strings
    (F("substring", [C("sd")], [L(-2)], [L(2)]), "=", [L("13")]),           # dictionary strings, from the end
    (F("datediff", [C("d2")], [C("d")]), ">", [L(30)]),
    (F("month", [C("ts")]), "<=", F("quarter", [C("d")]) + [L(3), ("*",)]),
    (F("dayofweek", [C("d")]), "=", [L(1)]),
    (F("weekofyear", [C("ts")]), ">=", [L(52)]),
    (F("dayofyear", [C("d")]), "<", F("dayofmonth", [C("d2")])),
    (F("hour", [C("ts")]), "=", [L(0)]),
    (F("minute", [C("ts")]) + F("second", [C("ts")]) + [("+",)], ">", [L(90)]),
    (F("date_add", [C("d")], [C("i")]), "<", [C("d2")]),
    (F("date_sub", [C("ts")], [L(3)]), "<=", [L(datetime.date(1995, 6, 1))]),
    ([C("ts")], "<", [C("d")]),                                            # a timestamp with a date: its UTC midnight
    ([C("d")], ">=", [L(datetime.date(1996, 2, 29))]),
    (F("length", [C("s")]), "=", [L(11)]),
    (F("length", [C("b")]), ">", [L(3)]),
    (F("substring", [C("b")], [L(2)], [L(2)]), "<", F("substring", [C("b")], [L(1)], [L(1)])),
    (F("abs", [C("i"), L(7), ("-",)]), "<", [L(5)]),
    (F("abs", [C("x")]), ">", [L(1.5)]),
    (F("coalesce", [C("x")], [L(0)]), ">", [L(0.05)]),
    (F("coalesce", [C("s")], [C("sd")]), "<=>", [L("13-9")]),
    (F("coalesce", [C("d")], [C("ts")]), "<", [L(datetime.datetime(1990, 1, 1))]),
    (F("coalesce", [C("s")], [C("sd")]), "<=>", [L("")]),                   # only empty string literals in the program
    (F("substring", [C("s")], [L(1)], [L(2)]), "=", [L("")]),
]


@pytest.mark.parametrize("k", range(len(EXPRS)))
def test_scans_against_the_oracle(data, k):
    left, op, right = EXPRS[k]
    hits = 0
    for neg in (False, True):
        hits += int(_check(data, [(left, op, right, neg)]).sum() > 0)
    assert hits >= 1
    _check(data, [(left, "<=>", right)])  # null-safe equality of the same two sides


def test_key_windows_with_function_conjuncts(data):
    preds = [("id", 500, False, 4000, True)]
    for exprs in ([EXPRS[0]], [EXPRS[1], EXPRS[3]], [(EXPRS[8][0], "=", EXPRS[8][2], True), EXPRS[17]],
                  [([C("id"), L(7), ("%",)], "=", [L(3)]), EXPRS[14]]):  # an arithmetic conjunct beside a function
        assert _check(data, exprs, preds).sum() > 0
    assert _check(data, [(F("abs", [C("id"), L(3000), ("-",)]), "<", [L(10)])]).sum() == 19  # the key inside a function


def test_refusals(data):
    from hyperspace_b200 import _native as N

    ctx, files = data["ctx"], data["sources"]

    def refused(code, text, exprs):
        with pytest.raises(N.HyperspaceGpuError) as e:
            ctx.filter_scan_expr(files, None, ["id"], [], [], [], exprs, sorted_on_key=False)
        assert e.value.code == code and text in str(e.value), str(e.value)

    refused(N.HS_EUNSUPPORTED, "hour(d): d (date) is not a timestamp", [(F("hour", [C("d")]), "<", [L(1)])])
    refused(N.HS_EUNSUPPORTED, "the column 'd' (date) cannot be used in arithmetic", [([C("d")], "<", [L(1)])])
    refused(N.HS_EUNSUPPORTED, "(string) and substring(b, 1, 2) (binary) cannot be compared",
            [(F("substring", [C("s")], [L(1)], [L(2)]), "=", F("substring", [C("b")], [L(1)], [L(2)]))])
    refused(N.HS_EINVAL, "whose pos and len are not int literals", [([C("s"), L(1), C("i"), ("substring",)], "=", [L("x")])])


def test_launches(data):
    """calls without functions launch the kernels they did before and no k_func_mask; a call with functions launches
    k_func_mask once per filtered side"""
    ctx = data["ctx"]
    r = data["index"]
    preds = [("id", 100, False, 4000, False)]
    arith = [([C("k"), L(7), ("%",)], "=", [L(0)], 0)]
    ctx.profile_enable(True)
    ctx.profile_report()
    a, _ = ctx.filter_scan_expr(r.as_sources(), "id", ["id"], preds, [], [], arith)
    ka = ctx.profile_report()
    assert ka["k_expr_mask"]["launches"] == 1 and "k_func_mask" not in ka
    b, _ = ctx.filter_scan_expr(r.as_sources(), "id", ["id"], preds, [], [], [])
    kb = ctx.profile_report()
    assert "k_func_mask" not in kb and "k_expr_mask" not in kb
    c, _ = ctx.filter_scan_expr(r.as_sources(), "id", ["id"], preds, [], [], _native([EXPRS[0], EXPRS[1]]))
    kc = ctx.profile_report()
    assert kc["k_func_mask"]["launches"] == 1 and "k_expr_mask" not in kc
    # the rest of the call is what an arithmetic residual launches: the same decodes, masks and compaction
    assert ({k: v["launches"] for k, v in kc.items() if k != "k_func_mask"} ==
            {k: v["launches"] for k, v in ka.items() if k != "k_expr_mask"})
    for x in (a, b, c):
        x.free()
    args = (r.as_sources(), [f.bucket for f in r.files], r.as_sources(), [f.bucket for f in r.files], NB, ["id"], ["id"], ["id"], ["k"])
    j, _ = ctx.bucket_join_expr(*args, "inner", left_exprs=_native([EXPRS[0]]), right_exprs=_native([EXPRS[3]]))
    kj = ctx.profile_report()
    assert kj["k_func_mask"]["launches"] == 2
    j.free()
    ctx.profile_enable(False)


JOINS = ["inner", "semi", "anti", "left", "right", "full"]


@pytest.mark.parametrize("jt", JOINS)
def test_every_join_type_with_a_function_below_a_side(data, jt):
    """bucket_join_expr with a function conjunct on each side: the rows each side keeps are the oracle's"""
    from hyperspace_b200 import _native as N

    d, ctx = data, data["ctx"]
    idx = ctx.create_index(d["sources"], ["k"], [c for c in TYPES if c != "k"], NB, output=N.HS_OUT_HOST)[0]
    files, buckets = idx.as_sources(), [f.bucket for f in idx.files]
    le, re_ = [EXPRS[0]], [EXPRS[1]]
    rcols = [] if jt in ("semi", "anti") else ["id"]
    j, _ = ctx.bucket_join_expr(files, buckets, files, buckets, NB, ["k"], ["k"], ["id"], rcols, jt, left_exprs=_native(le),
                                right_exprs=_native(re_))
    got = [(v.tolist(), None if m is None else np.asarray(m).tolist()) for _, v, m in j.columns]
    j.free()
    idx.free()
    lm, rm = _mask(d, le), _mask(d, re_)
    key = d["cols"]["k"]
    lsel, rsel = set(np.flatnonzero(lm).tolist()), set(np.flatnonzero(rm).tolist())
    by_key = {}
    for i in rsel:
        by_key.setdefault(int(key[i]), []).append(i)
    matches = {i: by_key.get(int(key[i]), []) for i in lsel}
    lid = got[0][0]
    if jt == "semi":
        assert sorted(lid) == sorted(i for i in lsel if matches[i])
        return
    if jt == "anti":
        assert sorted(lid) == sorted(i for i in lsel if not matches[i])
        return
    rid = got[1][0]
    lvalid = got[0][1] or [1] * len(lid)
    rvalid = got[1][1] or [1] * len(rid)
    pairs = [(l if lv else None, r if rv else None) for l, r, lv, rv in zip(lid, rid, lvalid, rvalid)]
    want = [(i, j) for i in lsel for j in matches[i]]
    matched_r = {j for i in lsel for j in matches[i]}
    if jt in ("left", "full"):
        want += [(i, None) for i in lsel if not matches[i]]
    if jt in ("right", "full"):
        want += [(None, j) for j in rsel if j not in matched_r]
    if jt == "right":
        want = [p for p in want if p[1] is not None]
    key_of = lambda p: (p[0] if p[0] is not None else -1, p[1] if p[1] is not None else -1)  # noqa: E731
    assert sorted(pairs, key=key_of) == sorted(want, key=key_of) and len(want) > 0


def test_hyperspace_api(tmp_path):
    import os

    from hyperspace_b200.functions import col, datediff, substring, year
    from hyperspace_b200.hyperspace import Hyperspace
    from hyperspace_b200.index_config import IndexConfig
    from hyperspace_b200.session import HyperspaceSession

    s = HyperspaceSession({"spark.hyperspace.system.path": str(tmp_path / "indexes"), "spark.hyperspace.index.numBuckets": "8"})
    hs = Hyperspace(s)
    rng = np.random.default_rng(4)
    os.makedirs(tmp_path / "orders")
    os.makedirs(tmp_path / "customer")
    for i in range(3):
        n = 3000
        od = rng.integers(8000, 11000, n).astype(np.int32)
        pq.write_table(pa.table({"o_orderkey": np.arange(i * n, (i + 1) * n, dtype=np.int64), "o_orderdate": pa.array(od, pa.date32()),
                                 "o_shipdate": pa.array(od + rng.integers(0, 60, n).astype(np.int32), pa.date32(), mask=rng.random(n) < 0.1),
                                 "o_total": rng.uniform(0, 1000, n),
                                 "o_ts": pa.array(od.astype(np.int64) * DAY_US + rng.integers(-DAY_US, DAY_US, n), pa.timestamp("us"))}),
                       str(tmp_path / "orders" / f"f{i}.parquet"))
        phones = [f"{rng.integers(10, 35)}-{rng.integers(100, 999)}-{rng.integers(1000, 9999)}" for _ in range(n)]
        pq.write_table(pa.table({"c_custkey": np.arange(i * n, (i + 1) * n, dtype=np.int64), "c_phone": pa.array(phones, pa.string()),
                                 "c_acctbal": rng.uniform(-1000, 10000, n)}), str(tmp_path / "customer" / f"f{i}.parquet"))
    orders = s.read.parquet(str(tmp_path / "orders"))
    customer = s.read.parquet(str(tmp_path / "customer"))
    hs.createIndex(orders, IndexConfig("odate", ["o_orderdate"], ["o_orderkey", "o_shipdate", "o_total", "o_ts"]))
    hs.createIndex(customer, IndexConfig("cphone", ["c_phone"], ["c_custkey", "c_acctbal"]))
    queries = [(orders.filter(year(col("o_orderdate")) == 1995).select("o_orderkey", "o_total"), "odate", "(year(o_orderdate) = 1995)"),
               (orders.filter(datediff(col("o_shipdate"), col("o_orderdate")) > 30).select("o_orderkey"), "odate",
                "(datediff(o_shipdate, o_orderdate) > 30)"),
               (customer.filter(substring(col("c_phone"), 1, 2) == "13").select("c_custkey", "c_phone"), "cphone",
                "(substring(c_phone, 1, 2) = 13)")]
    try:
        for q, idx, text in queries:
            s.enableHyperspace()
            plan = q.explain()
            assert f"Name: {idx}" in plan and text in plan, plan
            got = q.collect()
            s.disableHyperspace()
            base = q.collect()
            key = lambda r: sorted(zip(*[[repr(x) for x in r[c].tolist()] for c in q.columns]))  # noqa: E731
            assert key(got) == key(base) and len(key(got)) > 0
        # the oracle for the first and last queries, from the files themselves
        t = pq.read_table(str(tmp_path / "orders"))
        od = t.column("o_orderdate").cast(pa.int32()).to_numpy()
        want = t.column("o_orderkey").to_numpy()[FF.calendar(od)["year"] == 1995]
        s.enableHyperspace()
        assert sorted(queries[0][0].collect()["o_orderkey"].tolist()) == sorted(want.tolist())
        c = pq.read_table(str(tmp_path / "customer"))
        want = [k for k, p in zip(c.column("c_custkey").to_pylist(), c.column("c_phone").to_pylist()) if p[:2] == "13"]
        assert sorted(queries[2][0].collect()["c_custkey"].tolist()) == sorted(want)
        # a date literal on a timestamp column is that day's UTC midnight, on a date column its days
        ts = t.column("o_ts").cast(pa.int64()).to_numpy()
        day, midnight = datetime.date(1995, 3, 1), 9190 * DAY_US
        for q, m in ((orders.filter((col("o_orderdate") >= datetime.date(1995, 1, 1)) & (col("o_ts") < day)), (od >= 9131) & (ts < midnight)),
                     (orders.filter((col("o_orderdate") > 0) & (col("o_ts") >= day)), (od > 0) & (ts >= midnight))):
            q = q.select("o_orderkey")
            assert "Name: odate" in q.explain()
            assert sorted(q.collect()["o_orderkey"].tolist()) == sorted(t.column("o_orderkey").to_numpy()[m].tolist()) and m.sum() > 0
    finally:
        s.stop()
