"""GPU filter scans and join sides with expression comparisons (hs_expr_compare): on sorted index files (key windows from
literal predicates with an expression residual, and the key inside an expression alone), on raw sources with nulls, the
decimal and int / float mixes and a division by zero; below both sides of every join type; the Hyperspace API; and a
profiled call showing that calls without expressions launch no k_expr_mask and the kernels of their _cmp call.  Answers
are compared with tests/filter_expr_oracle.py as exact sequences of row ids (file, then row)."""
import decimal
import io

import numpy as np
import pyarrow as pa
import pyarrow.parquet as pq
import pytest

import filter_expr_oracle as FX

pytestmark = pytest.mark.gpu

N_ROWS = 6_000
NB = 8
TYPES = {"i32": "integer", "i32b": "integer", "i64": "long", "f32": "float", "f64": "double", "d92": "decimal(9,2)",
         "d185": "decimal(18,5)", "id": "long"}


def _make_columns(seed=5):
    rng = np.random.default_rng(seed)
    n = N_ROWS
    cols = {"i32": rng.integers(-50, 50, n).astype(np.int32), "i32b": rng.integers(-5, 5, n).astype(np.int32),
            "i64": rng.integers(-1000, 1000, n).astype(np.int64), "f32": rng.integers(-40, 40, n).astype(np.float32) / 4,
            "f64": rng.normal(0, 20, n), "d92": rng.integers(-5000, 5000, n).astype(np.int64),
            "d185": rng.integers(-10**9, 10**9, n).astype(np.int64), "id": np.arange(n, dtype=np.int64)}
    cols["i32"][:4] = [2**31 - 1, -2**31, 46341, 65536]
    cols["i32b"][:4] = [2, -1, 46341, 65536]
    cols["f64"][:6] = [np.nan, -0.0, 0.0, np.inf, -np.inf, 1e308]
    valids = {c: rng.random(n) >= 0.1 for c in TYPES if c != "id"}
    for v in valids.values():
        v[:6] = True
    return cols, valids


def _arrow(cols, valids, rows):
    out = {}
    for name, v in cols.items():
        v = v[rows]
        mask = ~valids[name][rows] if name in valids else None
        t = TYPES[name]
        if t.startswith("decimal"):
            p, s = (int(x) for x in t[len("decimal("):-1].split(","))
            out[name] = pa.array([decimal.Decimal(int(x)).scaleb(-s) for x in v], pa.decimal128(p, s), mask=mask)
        else:
            out[name] = pa.array(v, mask=mask)
    return pa.table(out)


def _parquet_bytes(table):
    sink = io.BytesIO()
    pq.write_table(table, sink, compression="NONE", data_page_size=16 << 10, row_group_size=2_000)
    return sink.getvalue()


@pytest.fixture(scope="module")
def data():
    from hyperspace_b200 import _native as N

    ctx = N.Context(0)
    cols, valids = _make_columns()
    halves = [np.arange(0, N_ROWS // 2), np.arange(N_ROWS // 2, N_ROWS)]
    sources = [N.FileImage(path=f"src{i}.parquet", data=_parquet_bytes(_arrow(cols, valids, r)), file_id=i) for i, r in enumerate(halves)]
    idx = ctx.create_index(sources, ["id"], [c for c in cols if c != "id"], NB, output=N.HS_OUT_HOST)[0]
    yield {"ctx": ctx, "cols": cols, "valids": valids, "sources": sources, "index": idx}
    idx.free()
    ctx.close()


def C(n):
    return ("column", n)


def L(v):
    return ("literal", v)


def _mask(d, exprs, preds=()):
    columns = {c: (TYPES[c], d["cols"][c].tolist(), d["valids"].get(c)) for c in TYPES}
    m = np.ones(N_ROWS, bool)
    for left, op, right, *neg in exprs:
        m &= FX.mask(left, op, right, bool(neg and neg[0]), columns, N_ROWS)
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
    b, _ = ctx.filter_scan_expr(d["sources"], None, ["id"], list(preds), [], [], _native(exprs), sorted_on_key=False)
    assert np.array_equal(_ids(b), np.flatnonzero(m)), (exprs, preds, "unsorted")
    return m


EXPRS = [
    ([C("i32"), C("i32b"), ("*",)], "=", [L(0)]),                       # int * int wraps at 2^31
    ([C("i32"), L(7), ("%",)], "=", [L(0)]),
    ([C("i32"), C("i32b"), ("%",)], "<", [L(0)]),                        # remainder signs, MIN % -1, % 0 is null
    ([C("i64"), L(3), ("*",), C("i32"), ("+",)], "<", [L(1500)]),
    ([C("f64"), C("i32b"), ("/",)], ">", [L(2.0)]),                      # / 0 is null
    ([C("f32"), C("i32"), ("*",)], "<=", [C("f64")]),                    # int * float is float
    ([C("d92"), C("i32"), ("+",)], ">=", [L(decimal.Decimal("1.25"))]),   # decimal + int column
    ([C("d92"), C("d185"), ("*",)], "<", [C("d185"), L(3), ("-",)]),
    ([C("d92"), L(7), ("%",)], "=", [L(decimal.Decimal("0.50"))]),
    ([C("d185"), C("f32"), ("-",)], ">", [L(0.5)]),                       # decimal with float is double
    ([C("i32"), ("neg",)], "<=>", [C("i32b")]),
    ([L(1), C("f64"), ("-",)], "=", [C("f64"), L(0.0), ("*",)]),
]


@pytest.mark.parametrize("k", range(len(EXPRS)))
def test_scans_against_the_oracle(data, k):
    left, op, right = EXPRS[k]
    hits = 0
    for neg in (False, True):
        hits += int(_check(data, [(left, op, right, neg)]).sum() > 0)
    assert hits >= 1


def test_key_windows_with_an_expression_residual(data):
    preds = [("id", 500, False, 4000, True)]
    for exprs in ([EXPRS[3]], [EXPRS[4], EXPRS[6]], [(EXPRS[8][0], "=", EXPRS[8][2], True)]):
        assert _check(data, exprs, preds).sum() > 0
    # the key inside an expression alone: every row read
    assert _check(data, [([C("id"), L(7), ("%",)], "=", [L(3)])]).sum() > 0
    assert _check(data, [([C("id"), C("i64"), ("+",)], "<", [L(2000)])], [("id", None, False, 100, False)]).sum() > 0


def test_refusals(data):
    from hyperspace_b200 import _native as N

    ctx, files = data["ctx"], data["sources"]

    def refused(code, text, exprs):
        with pytest.raises(N.HyperspaceGpuError) as e:
            ctx.filter_scan_expr(files, None, ["id"], [], [], [], exprs, sorted_on_key=False)
        assert e.value.code == code and text in str(e.value), str(e.value)

    refused(N.HS_EUNSUPPORTED, "decimal division is not handled: (d92 / i32)", [([C("d92"), C("i32"), ("/",)], "<", [L(1)])])
    refused(N.HS_EUNSUPPORTED, "needs a decimal of more than 38 digits",
            [([C("d185"), C("d185"), ("*",), C("d185"), ("*",)], "<", [L(1)])])
    refused(N.HS_EINVAL, "underflows its stack", [([C("i32"), ("+",)], "<", [L(1)])])
    refused(N.HS_EUNSUPPORTED, "more than 16 predicates and terms", [([C("i32")], "<", [L(1)])] * 17)


def test_without_expressions_the_cmp_calls_run_unchanged(data):
    """the _expr calls with no expressions launch the kernels of the _cmp calls, and no k_expr_mask"""
    ctx = data["ctx"]
    r = data["index"]
    preds, cmps = [("id", 100, False, 4000, False)], [("i32", "<", "i64")]
    ctx.profile_enable(True)
    ctx.profile_report()
    a, sa = ctx.filter_scan_cmp(r.as_sources(), "id", ["id", "f64"], preds, [], cmps)
    ka = ctx.profile_report()
    b, sb = ctx.filter_scan_expr(r.as_sources(), "id", ["id", "f64"], preds, [], cmps, [])
    kb = ctx.profile_report()
    assert sorted(ka) == sorted(kb) and "k_expr_mask" not in kb and sa["rows_out"] == sb["rows_out"] > 0
    assert {k: v["launches"] for k, v in ka.items()} == {k: v["launches"] for k, v in kb.items()}
    assert _ids(a).tolist() == _ids(b).tolist()
    args = (r.as_sources(), [f.bucket for f in r.files], r.as_sources(), [f.bucket for f in r.files], NB, ["id"], ["id"], ["id"], ["i64"])
    j1, s1 = ctx.bucket_join_cmp(*args, preds, [], [], [], cmps, [])
    k1 = ctx.profile_report()
    j2, s2 = ctx.bucket_join_expr(*args, "inner", preds, [], [], [], cmps, [], [], [])
    k2 = ctx.profile_report()
    assert {k: v["launches"] for k, v in k1.items()} == {k: v["launches"] for k, v in k2.items()} and "k_expr_mask" not in k2
    assert s1["rows_out"] == s2["rows_out"] > 0
    j1.free()
    j2.free()
    c, _ = ctx.filter_scan_expr(r.as_sources(), "id", ["id"], preds, [], [], [EXPRS[3]])
    kc = ctx.profile_report()
    assert kc["k_expr_mask"]["launches"] == 1
    c.free()
    ctx.profile_enable(False)


JOINS = {"inner": None, "semi": None, "anti": None, "left": "left", "right": "right", "full": "full"}


@pytest.mark.parametrize("jt", list(JOINS))
def test_every_join_type_with_expressions_below_each_side(data, jt):
    """bucket_join_expr with an expression on each side against bucket_join_cmp / _exists / _outer over the same rows
    filtered on the host: the rows each side keeps are the oracle's."""
    from hyperspace_b200 import _native as N

    d, ctx = data, data["ctx"]
    idx = ctx.create_index(d["sources"], ["i32b"], [c for c in d["cols"] if c != "i32b"], NB, output=N.HS_OUT_HOST)[0]
    files, buckets = idx.as_sources(), [f.bucket for f in idx.files]
    le, re_ = [EXPRS[3]], [EXPRS[6]]
    rcols = [] if jt in ("semi", "anti") else ["id"]
    j, _ = ctx.bucket_join_expr(files, buckets, files, buckets, NB, ["i32b"], ["i32b"], ["id"], rcols, jt, left_exprs=_native(le),
                                right_exprs=_native(re_))
    got = [(v.tolist(), None if m is None else np.asarray(m).tolist()) for _, v, m in j.columns]
    j.free()
    idx.free()
    lm, rm = _mask(d, le), _mask(d, re_)
    key, kv = d["cols"]["i32b"], d["valids"]["i32b"]
    lsel, rsel = set(np.flatnonzero(lm).tolist()), set(np.flatnonzero(rm).tolist())
    by_key = {}
    for i in rsel:
        if kv[i]:
            by_key.setdefault(int(key[i]), []).append(i)
    matches = {i: by_key.get(int(key[i]), []) if kv[i] else [] for i in lsel}
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

    from hyperspace_b200.hyperspace import Hyperspace
    from hyperspace_b200.index_config import IndexConfig
    from hyperspace_b200.session import HyperspaceSession, col

    s = HyperspaceSession({"spark.hyperspace.system.path": str(tmp_path / "indexes"), "spark.hyperspace.index.numBuckets": "8"})
    hs = Hyperspace(s)
    rng = np.random.default_rng(4)
    os.makedirs(tmp_path / "t")
    for i in range(3):
        n = 3000
        pq.write_table(pa.table({"k": rng.integers(0, 300, n).astype(np.int64), "v": pa.array(rng.integers(-50, 50, n).astype(np.int32)),
                                 "price": pa.array(rng.uniform(0, 200, n), mask=rng.random(n) < 0.1),
                                 "disc": pa.array([decimal.Decimal(int(x)).scaleb(-2) for x in rng.integers(0, 10, n)], pa.decimal128(4, 2))}),
                       str(tmp_path / "t" / f"f{i}.parquet"))
    df = s.read.parquet(str(tmp_path / "t"))
    hs.createIndex(df, IndexConfig("kidx", ["k"], ["v", "price", "disc"]))
    queries = [(df.filter((col("k") < 100) & (col("price") * (1 - col("disc")) > 100)).select("k", "price"), "kidx",
                "(((price * (1 - disc)) > 100)"),
               (df.filter(col("k") % 7 == 0).select("k", "v"), "kidx", "((k % 7) = 0)"),
               (df.filter(col("v") + col("k") < col("price")).select("k", "v"), "kidx", "((v + k) < price)"),
               (df.filter(col("v") * 2 >= 10).select("v"), None, "((v * 2) >= 10)")]
    try:
        for q, idx, text in queries:
            s.enableHyperspace()
            plan = q.explain()
            assert (idx is None and plan.startswith("GpuSourceScan")) or f"Name: {idx}" in plan, plan
            assert text in plan, plan
            got = q.collect()
            s.disableHyperspace()
            base = q.collect()
            key = lambda r: sorted(zip(*[[repr(x) for x in r[c].tolist()] for c in q.columns]))  # noqa: E731
            assert key(got) == key(base) and len(key(got)) > 0
    finally:
        s.stop()
