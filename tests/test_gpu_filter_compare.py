"""GPU filter scans and join sides with comparisons between two columns (hs_column_compare): every operator, with and
without NOT, over every type pair of the coercion table, with nulls on either side or both; on sorted index files (with key
windows from literal predicates, and with the key inside the comparison) and on raw sources; on both join sides; device
output; the n_cmps = 0 calls against the _any calls; and the Hyperspace API with Hybrid Scan and lineage.  Answers are
compared with tests/filter_compare_oracle.py as exact sequences of row ids (file, then row)."""
import datetime
import decimal
import io
import os

import numpy as np
import pyarrow as pa
import pyarrow.parquet as pq
import pytest

import filter_compare_oracle as FC

pytestmark = pytest.mark.gpu

N_ROWS = 30_000
NB = 8
DAY = FC.DAY_MICROS
TYPES = {"i32": "integer", "i32b": "integer", "i64": "long", "i64b": "long", "f32": "float", "f32b": "float", "f64": "double",
         "f64b": "double", "s": "string", "s2": "string", "dt": "date", "dt2": "date", "ts": "timestamp", "ts2": "timestamp",
         "d92": "decimal(9,2)", "d92b": "decimal(9,2)", "d185": "decimal(18,5)"}
PAIRS = [("i32", "i32b"), ("i64", "i64b"), ("f32", "f32b"), ("f64", "f64b"), ("s", "s2"), ("ts", "ts2"), ("dt", "dt2"),
         ("d92", "d92b"), ("i32", "i64"), ("i32", "f32"), ("i64", "f32"), ("i32", "f64"), ("i64", "f64"), ("f32", "f64"),
         ("d92", "d185"), ("d185", "i64"), ("i32", "d92"), ("d92", "f64"), ("f32", "d185"), ("dt", "ts"), ("i32", "i32")]
OPS = ["<", "<=", ">", ">=", "=", "<=>"]


def _make_columns(seed=11):
    rng = np.random.default_rng(seed)
    n = N_ROWS
    small = lambda: rng.integers(-20, 20, n)  # noqa: E731  (small ranges: equal values are common)
    cols = {"i32": small().astype(np.int32), "i32b": small().astype(np.int32), "i64": small().astype(np.int64),
            "i64b": small().astype(np.int64), "f32": small().astype(np.float32), "f32b": small().astype(np.float32),
            "f64": small().astype(np.float64), "f64b": small().astype(np.float64)}
    cols["i32"][:4] = [16777217, -2**31, 2**31 - 1, 16777217]
    cols["f32"][:4] = [16777216, -2**31, 2**31, np.nan]
    cols["i64"][:4] = [2**53 + 1, 2**63 - 1, -2**63, 2**53 + 1]
    cols["f64"][:4] = [2**53, 2.0**63, -2.0**63, np.nan]
    for c in ("f32", "f32b", "f64", "f64b"):
        cols[c][10:16] = np.array([np.nan, np.inf, -np.inf, 0.0, -0.0, np.nan], cols[c].dtype)
    cols["f32b"][10:16] = np.array([np.nan, np.inf, 0.0, -0.0, 0.0, 1.0], np.float32)
    words = [w.encode() for w in ["", "a", "ab", "abc", "b", "é", "ÿ", "ab\x00"]]
    cols["s"] = np.array([words[i] for i in rng.integers(0, len(words), n)], dtype=object)
    cols["s2"] = np.array([words[i] for i in rng.integers(0, len(words), n)], dtype=object)
    cols["dt"] = rng.integers(-3, 3, n).astype(np.int32)
    cols["dt2"] = rng.integers(-3, 3, n).astype(np.int32)
    cols["ts"] = rng.integers(-3, 3, n).astype(np.int64) * DAY + rng.choice([0, 0, 1, -1, DAY - 1], n)
    cols["ts2"] = rng.integers(-3, 3, n).astype(np.int64) * DAY + rng.choice([0, 0, 1, -1], n)
    cols["d92"] = (rng.integers(-20, 20, n) * 100 + rng.choice([0, 0, 50], n)).astype(np.int64)      # unscaled, scale 2
    cols["d92b"] = (rng.integers(-20, 20, n) * 100 + rng.choice([0, 0, 50], n)).astype(np.int64)
    cols["d185"] = (rng.integers(-20, 20, n) * 100000 + rng.choice([0, 0, 50000, 1], n)).astype(np.int64)  # scale 5
    cols["id"] = np.arange(n, dtype=np.int64)
    valids = {c: rng.random(n) >= 0.15 for c in TYPES}
    for v in valids.values():
        v[:16] = True  # the hand-placed edge values above
    return cols, valids


def _arrow(cols, valids, rows):
    out = {}
    for name, v in cols.items():
        v = v[rows]
        mask = ~valids[name][rows] if name in valids else None
        t = TYPES.get(name)
        if t == "string":
            out[name] = pa.array([x.decode() for x in v], pa.string(), mask=mask)
        elif t == "date":
            out[name] = pa.array(v, pa.date32(), mask=mask)
        elif t == "timestamp":
            out[name] = pa.array(v, pa.timestamp("us"), mask=mask)
        elif t and t.startswith("decimal"):
            p, s = FC._decimal(t)
            out[name] = pa.array([decimal.Decimal(int(x)).scaleb(-s) for x in v], pa.decimal128(p, s), mask=mask)
        else:
            out[name] = pa.array(v, mask=mask)
    return pa.table(out)


def _parquet_bytes(table):
    sink = io.BytesIO()
    pq.write_table(table, sink, compression="NONE", data_page_size=16 << 10, row_group_size=5_000)
    return sink.getvalue()


@pytest.fixture(scope="module")
def data():
    from hyperspace_b200 import _native as N

    ctx = N.Context(0)
    cols, valids = _make_columns()
    halves = [np.arange(0, N_ROWS // 2), np.arange(N_ROWS // 2, N_ROWS)]
    sources = [N.FileImage(path=f"src{i}.parquet", data=_parquet_bytes(_arrow(cols, valids, r)), file_id=i)
               for i, r in enumerate(halves)]
    # an index sorted on the non-null id column: literal predicates on id make the key windows
    idx = ctx.create_index(sources, ["id"], [c for c in cols if c != "id"], NB, output=N.HS_OUT_HOST)[0]
    yield {"ctx": ctx, "cols": cols, "valids": valids, "sources": sources, "index": idx}
    idx.free()
    ctx.close()


def _file_ids(res):
    return [pq.read_table(pa.BufferReader(res.host_bytes(i)), columns=["id"]).column("id").to_numpy() for i in range(len(res.files))]


def _ids(batch):
    out = next(v.copy() for n, v, _ in batch.columns if n == "id")
    batch.free()
    return out


def _side(d, c):
    return TYPES.get(c, "long"), d["cols"][c], d["valids"].get(c)  # id: a non-null long


def _mask(d, cmps, preds=()):
    m = np.ones(N_ROWS, bool)
    for l, op, r, *neg in cmps:
        m &= FC.mask(_side(d, l), _side(d, r), op, bool(neg and neg[0]))
    for c, lo, ls, hi, hs in preds:
        v = d["cols"][c]
        if lo is not None:
            m &= (v > lo) if ls else (v >= lo)
        if hi is not None:
            m &= (v < hi) if hs else (v <= hi)
    return m


def _cmp_native(cmps):
    return [(l, op, r, 1 if (neg and neg[0]) else 0) for l, op, r, *neg in cmps]


def _check(d, cmps, preds=()):
    """the comparisons over the index (sorted on id) and over the source files; returns the oracle's mask"""
    ctx = d["ctx"]
    m = _mask(d, cmps, preds)
    want = np.concatenate([ids[m[ids]] for ids in _file_ids(d["index"])])
    b, _ = ctx.filter_scan_cmp(d["index"].as_sources(), "id", ["id"], list(preds), [], _cmp_native(cmps), sorted_on_key=True)
    got = _ids(b)
    assert np.array_equal(got, want), (cmps, preds, len(got), len(want))
    b, _ = ctx.filter_scan_cmp(d["sources"], None, ["id"], list(preds), [], _cmp_native(cmps), sorted_on_key=False)
    assert np.array_equal(_ids(b), np.flatnonzero(m)), (cmps, preds, "unsorted")
    return m


@pytest.mark.parametrize("pair", PAIRS, ids=[f"{a}-{b}" for a, b in PAIRS])
def test_every_op_over_every_type_pair(data, pair):
    l, r = pair
    hits = 0
    for op in OPS:
        for neg in (False, True):
            hits += int(_check(data, [(l, op, r, neg)]).sum() > 0)
    assert hits >= 6  # the data exercise the operators


def test_rounding_rows(data):
    """2^24 + 1 (int32) equals 16777216f; 2^53 + 1 (int64) equals 2^53 as a double; NaN equals NaN."""
    assert _check(data, [("i32", "=", "f32")])[0]
    assert _check(data, [("i64", "=", "f64")])[0]
    assert _check(data, [("f32", "=", "f32b")])[10]  # NaN = NaN


def test_key_windows_with_a_comparison_residual(data):
    """the index is sorted on id: literal predicates on id make windows, the comparison runs over their rows; and the key
    inside a comparison alone reads every row."""
    preds = [("id", 1000, False, 20000, True)]
    for cmps in ([("i32", "<", "i64")], [("f64", ">=", "d92")], [("s", "<=>", "s2", True)], [("dt", "<", "ts"), ("i32", "=", "i32b", True)]):
        assert _check(data, cmps, preds).sum() > 0
    assert _check(data, [("id", ">", "i64")]).sum() > 0
    assert _check(data, [("id", "<", "i32"), ("i32", "<", "i64b")], [("id", None, False, 5, False)]).sum() >= 0


class _Dev:
    """A device array for torch.as_tensor (__cuda_array_interface__)."""

    def __init__(self, ptr, n, typestr):
        self.__cuda_array_interface__ = {"shape": (n,), "typestr": typestr, "data": (ptr, False), "version": 2}


def test_device_output(data):
    import torch

    from hyperspace_b200 import _native as N

    ctx = data["ctx"]
    cmps = [("i64", "<", "f32"), ("s", "=", "s2", True)]
    host, _ = ctx.filter_scan_cmp(data["index"].as_sources(), "id", ["id", "i64"], [], [], _cmp_native(cmps))
    dev, _ = ctx.filter_scan_cmp(data["index"].as_sources(), "id", ["id", "i64"], [], [], _cmp_native(cmps), output=N.HS_OUT_DEVICE)
    assert dev.on_device and dev.num_rows == host.num_rows > 0
    for (name, ty, ptr), (hname, hdata, _) in zip(dev.device_columns, host.columns):
        assert name == hname and ty == N.HS_TYPE_INT64
        got = torch.as_tensor(_Dev(ptr, dev.num_rows, "<i8"), device="cuda").cpu().numpy()
        assert np.array_equal(got, hdata)
    host.free()
    dev.free()


def test_no_comparisons_is_the_any_call(data):
    ctx = data["ctx"]
    for files, key, srt in ((data["index"].as_sources(), "id", True), (data["sources"], None, False)):
        preds, terms = [("id", 100, False, 9000, False)], [("i32", [1, 2, 3], [])]
        a, sa = ctx.filter_scan_any(files, key, ["id", "s", "f64"], preds, terms, sorted_on_key=srt)
        b, sb = ctx.filter_scan_cmp(files, key, ["id", "s", "f64"], preds, terms, [], sorted_on_key=srt)
        assert sa["gpu_launches"] == sb["gpu_launches"] and sa["rows_out"] == sb["rows_out"] > 0
        for (n1, v1, m1), (n2, v2, m2) in zip(a.columns, b.columns):
            assert n1 == n2 and list(v1) == list(v2) and (m1 is None) == (m2 is None)
        a.free()
        b.free()
    r = data["index"]
    args = (r.as_sources(), [f.bucket for f in r.files], r.as_sources(), [f.bucket for f in r.files], NB, ["id"], ["id"], ["id", "s"], ["i64"])
    a, sa = ctx.bucket_join_any(*args, [("i32", 0, False, None, False)], [], [("i64", [1, 5], [])], [])
    b, sb = ctx.bucket_join_cmp(*args, [("i32", 0, False, None, False)], [], [("i64", [1, 5], [])], [], [], [])
    assert sa["gpu_launches"] == sb["gpu_launches"] and sa["rows_out"] == sb["rows_out"] > 0
    for (n1, v1, _), (n2, v2, _) in zip(a.columns, b.columns):
        assert n1 == n2 and list(v1) == list(v2)
    a.free()
    b.free()


def test_refusals(data):
    from hyperspace_b200 import _native as N

    ctx, files = data["ctx"], data["sources"]

    def refused(code, text, cmps, preds=()):
        with pytest.raises(N.HyperspaceGpuError) as e:
            ctx.filter_scan_cmp(files, None, ["id"], list(preds), [], cmps, sorted_on_key=False)
        assert e.value.code == code and text in str(e.value), str(e.value)

    refused(N.HS_EUNSUPPORTED, "the columns 's' (string) and 'i32' (integer) cannot be compared", [("s", "<", "i32")])
    refused(N.HS_EUNSUPPORTED, "the columns 'ts' (timestamp) and 'i64' (long) cannot be compared", [("ts", "=", "i64")])
    refused(N.HS_EINVAL, "unknown operator", [("i32", 9, "i64")])
    refused(N.HS_EINVAL, "unknown flags", [("i32", "<", "i64", 4)])
    refused(N.HS_EUNSUPPORTED, "more than 16 predicates and terms", [("i32", "<", "i64")] * 10, [("i32", -5, False, None, False)] * 7)
    with pytest.raises(N.HyperspaceGpuError) as e:
        ctx.filter_scan_cmp(files, None, ["id"], [], [], [("nope", "<", "i64")], sorted_on_key=False)
    with pytest.raises(N.HyperspaceGpuError) as e2:
        ctx.filter_scan_cmp(files, None, ["id"], [("nope", 1, False, None, False)], [], [], sorted_on_key=False)
    assert e.value.code == e2.value.code


def test_join_sides_with_comparisons(data):
    d, ctx = data, data["ctx"]
    from hyperspace_b200 import _native as N

    idx = ctx.create_index(d["sources"], ["i64b"], [c for c in d["cols"] if c != "i64b"], NB, output=N.HS_OUT_HOST)[0]
    args = (idx.as_sources(), [f.bucket for f in idx.files], idx.as_sources(), [f.bucket for f in idx.files], NB, ["i64b"], ["i64b"],
            ["id"], ["id"])
    lc, rc = [("i32", "<", "f64"), ("s", "<=>", "s2", True)], [("dt", ">=", "ts")]
    j, st = ctx.bucket_join_cmp(*args, [], [], [], [], _cmp_native(lc), _cmp_native(rc))
    got = sorted(zip(*[v.tolist() for _, v, _ in j.columns]))
    j.free()
    idx.free()
    lm, rm = _mask(d, lc), _mask(d, rc)
    key, kv = d["cols"]["i64b"], d["valids"]["i64b"]
    by_key = {}
    for i in np.flatnonzero(rm & kv):
        by_key.setdefault(int(key[i]), []).append(int(i))
    want = sorted((int(i), j) for i in np.flatnonzero(lm & kv) for j in by_key.get(int(key[i]), []))
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
    k = rng.integers(0, 300, n).astype(np.int64) + base
    ship = rng.integers(0, 60, n)
    commit = ship + rng.integers(-5, 5, n)
    epoch = datetime.date(1995, 1, 1)
    dates = lambda v: pa.array([epoch + datetime.timedelta(days=int(x)) for x in v], pa.date32(), mask=rng.random(n) < 0.1)  # noqa: E731
    return {"k": k, "ship": dates(ship), "commit": dates(commit), "v": pa.array(rng.integers(-50, 50, n).astype(np.int32)),
            "f": pa.array(rng.normal(0, 30, n), mask=rng.random(n) < 0.1)}


def test_hyperspace_api_with_and_without_hyperspace(env):
    from hyperspace_b200.index_config import IndexConfig
    from hyperspace_b200.session import col

    s, hs, tmp = env
    rng = np.random.default_rng(3)
    for i in range(3):
        _write(tmp / "t", f"f{i}.parquet", _table(rng, 3000))
    df = s.read.parquet(str(tmp / "t"))
    hs.createIndex(df, IndexConfig("kidx", ["k"], ["ship", "commit", "v", "f"]))
    s.enableHyperspace()
    queries = [(df.filter(col("ship") < col("commit")).select("k", "ship"), None, "(ship < commit)"),
               (df.filter((col("k") < 100) & (col("ship") < col("commit"))).select("k", "v"), "kidx", "(ship < commit)"),
               (df.filter(col("k") > col("v")).select("k", "v"), "kidx", "(k > v)"),
               (df.filter(col("k") != col("v")).select("k", "f"), "kidx", "NOT (k = v)"),
               (df.filter(col("f") >= col("v")).select("k", "f"), None, "(f >= v)"),
               (df.filter((col("k") < 50) & ~col("ship").eqNullSafe(col("commit"))).select("k", "ship", "commit"), "kidx", "NOT (ship <=> commit)"),
               (df.filter(col("v").between(col("k"), col("f"))).select("k", "v", "f"), None, "(v >= k)")]
    for q, idx, text in queries:
        plan = q.explain()
        assert idx is None or f"Name: {idx}" in plan, plan
        assert text in plan, plan
        got = _same_answers(s, q, q.columns)
        assert len(next(iter(got.values()))) > 0
    # Hybrid Scan: an appended file
    s.conf.set("spark.hyperspace.index.hybridscan.enabled", True)
    _write(tmp / "t", "f3.parquet", _table(rng, 300, base=250))
    df = s.read.parquet(str(tmp / "t"))
    for q in (df.filter((col("k") > 200) & (col("ship") <= col("commit"))).select("k", "commit"), df.filter(col("k") < col("v")).select("k", "v")):
        assert "hybridScan(appended=1" in q.explain()
        _same_answers(s, q, q.columns)


def test_hyperspace_api_with_deleted_lineage_ids(env):
    from hyperspace_b200.index_config import IndexConfig
    from hyperspace_b200.session import col

    s, hs, tmp = env
    s.conf.set("spark.hyperspace.index.lineage.enabled", True)
    rng = np.random.default_rng(8)
    for i in range(6):
        _write(tmp / "t", f"f{i}.parquet", _table(rng, 800))
    hs.createIndex(s.read.parquet(str(tmp / "t")), IndexConfig("idx", ["k"], ["ship", "commit", "v"]))
    os.remove(tmp / "t" / "f5.parquet")
    s.enableHyperspace()
    s.conf.set("spark.hyperspace.index.hybridscan.enabled", True)
    df = s.read.parquet(str(tmp / "t"))
    for q in (df.filter((col("k") < 150) & (col("ship") > col("commit"))).select("k", "ship"),
              df.filter(col("k") >= col("v")).select("k", "v")):
        assert "deletedIds=[5]" in q.explain() and "Name: idx" in q.explain()
        _same_answers(s, q, q.columns)
