"""GPU bucket joins on several key columns, with null keys and a filter below either side (hs_bucket_join_where),
compared with the numpy restatement in tests/join_oracle.py as exact row sequences: the engine emits the pairs in
(bucket, left sorted position, right sorted position) order, and so does the oracle."""
import io
import os

import numpy as np
import pyarrow as pa
import pyarrow.parquet as pq
import pytest

import join_oracle as J

pytestmark = pytest.mark.gpu

WORDS = [b"", b"a", b"ab", b"abc", b"abd", b"b", "été".encode(), b"facebook", b"zz", b"\xff"]


@pytest.fixture(scope="module")
def ctx():
    from hyperspace_b200 import _native

    c = _native.Context(0)
    yield c
    c.close()


def _arrow_column(v, valid):
    mask = None if valid is None else ~np.asarray(valid, dtype=bool)
    if v.dtype == object:
        return pa.array([None if (mask is not None and mask[i]) else x for i, x in enumerate(v.tolist())], pa.binary())
    return pa.array(v, mask=mask)


def _index(ctx, cols, valids, keys, nb, uuid):
    """createIndex over the columns (in memory): indexed = keys, included = every other column."""
    from hyperspace_b200 import _native

    sink = io.BytesIO()
    pq.write_table(pa.table({c: _arrow_column(v, (valids or {}).get(c)) for c, v in cols.items()}), sink, compression="NONE")
    res, _ = ctx.create_index([_native.FileImage(data=sink.getvalue())], list(keys), [c for c in cols if c not in keys], nb,
                              output=_native.HS_OUT_HOST, job_uuid=uuid)
    return res


def _sides(res_list):
    files, buckets = [], []
    for r in res_list:
        files += r.as_sources()
        buckets += [f.bucket for f in r.files]
    return files, buckets


def _run(ctx, lres, rres, nb, lkeys, rkeys, lpreds=(), rpreds=(), output=None):
    from hyperspace_b200 import _native

    lf, lb = _sides(lres)
    rf, rb = _sides(rres)
    kw = {} if output is None else {"output": output}
    return ctx.bucket_join_where(lf, lb, rf, rb, nb, lkeys, rkeys, ["lid"], ["rid"], lpreds, rpreds, **kw)


def _check(ctx, L, R, nb, lkeys, rkeys, lpreds=(), rpreds=(), lvalid=None, rvalid=None, lsplit=None, rsplit=None):
    """Indexes both tables (in two createIndex calls where a split is given: multi-file buckets), joins them on the GPU
    and compares the (left id, right id) sequence with the oracle's."""
    def build(cols, valids, keys, split, tag):
        if split is None:
            return [_index(ctx, cols, valids, keys, nb, tag)]
        parts = []
        for j, (a, b) in enumerate(((0, split), (split, len(cols["lid" if "lid" in cols else "rid"])))):
            parts.append(_index(ctx, {c: v[a:b] for c, v in cols.items()}, {c: v[a:b] for c, v in (valids or {}).items()}, keys,
                                nb, f"{tag}{j}"))
        return parts

    lres, rres = build(L, lvalid, lkeys, lsplit, "l"), build(R, rvalid, rkeys, rsplit, "r")
    batch, st = _run(ctx, lres, rres, nb, lkeys, rkeys, lpreds, rpreds)
    li, ri = J.bucket_join(L, R, nb, lkeys, rkeys, lpreds, rpreds, lvalid, rvalid)
    assert batch.num_rows == len(li) == st["rows_out"]
    assert np.array_equal(batch.column("lid"), L["lid"][li])
    assert np.array_equal(batch.column("rid"), R["rid"][ri])
    batch.free()
    for r in lres + rres:
        r.free()
    return len(li), st


def _tables(kind, nl, nr, seed):
    rng = np.random.default_rng(seed)

    def one(n, idname):
        if kind == "i64_i32":
            cols = {"a": rng.integers(0, 60, n).astype(np.int64), "b": rng.integers(-20, 20, n).astype(np.int32)}
        elif kind == "i64_i32_extremes":  # signed order at both ends of each range and around zero
            i64, i32 = np.iinfo(np.int64), np.iinfo(np.int32)
            a = np.concatenate([[i64.min, i64.min + 1, -1, 0, 1, i64.max - 1, i64.max], rng.integers(-2**62, 2**62, 33)])
            b = np.concatenate([[i32.min, i32.min + 1, -1, 0, 1, i32.max - 1, i32.max], rng.integers(-2**30, 2**30, 33)])
            cols = {"a": a.astype(np.int64)[rng.integers(0, len(a), n)], "b": b.astype(np.int32)[rng.integers(0, len(b), n)]}
        elif kind == "i32_str":  # the reference fixture's types: (int, string)
            cols = {"a": rng.integers(0, 40, n).astype(np.int32),
                    "b": np.array([WORDS[i] for i in rng.integers(0, len(WORDS), n)], dtype=object)}
        else:  # three longs, the first with heavy ties: matches depend on the later columns
            cols = {"a": rng.integers(0, 3, n).astype(np.int64), "b": rng.integers(0, 25, n).astype(np.int64),
                    "c": rng.integers(0, 25, n).astype(np.int64) * 10**12}
        cols["f32"] = rng.normal(0, 10, n).astype(np.float32)
        cols["f64"] = rng.normal(0, 100, n)
        cols["f64"][rng.random(n) < 0.05] = np.nan
        cols["i"] = rng.integers(0, 1000, n).astype(np.int64)
        cols["s"] = np.array([WORDS[i] for i in rng.integers(0, len(WORDS), n)], dtype=object)
        cols[idname] = np.arange(n, dtype=np.int64)
        return cols

    L, R = one(nl, "lid"), one(nr, "rid")
    keys = ["a", "b"] if kind != "i64_3" else ["a", "b", "c"]
    return L, R, keys


KINDS = ["i64_i32", "i32_str", "i64_3"]


@pytest.mark.parametrize("nb", [12, 200])
@pytest.mark.parametrize("kind", KINDS + ["i64_i32_extremes"])
def test_composite_keys(ctx, kind, nb):
    L, R, keys = _tables(kind, 12_000, 9_000, 1)
    n, _ = _check(ctx, L, R, nb, keys, keys)
    assert n > 0
    if kind == "i64_i32_extremes":  # each key alone: the int64 and the int32 extremes on both sides
        for k in keys:
            assert _check(ctx, L, R, nb, [k], [k])[0] > 0


@pytest.mark.parametrize("kind", KINDS)
def test_null_keys_at_every_position_on_both_sides(ctx, kind):
    L, R, keys = _tables(kind, 10_000, 8_000, 2)
    rng = np.random.default_rng(3)
    for pos in range(len(keys)):
        lvalid = {keys[pos]: rng.random(len(L["lid"])) >= 0.1}
        rvalid = {keys[pos]: rng.random(len(R["rid"])) >= 0.1}
        n, _ = _check(ctx, L, R, 12, keys, keys, lvalid=lvalid, rvalid=rvalid)
        assert n > 0
    # nulls in every key column at once, and one key joins with nulls too
    lvalid = {k: rng.random(len(L["lid"])) >= 0.05 for k in keys}
    rvalid = {k: rng.random(len(R["rid"])) >= 0.05 for k in keys}
    _check(ctx, L, R, 12, keys, keys, lvalid=lvalid, rvalid=rvalid)
    _check(ctx, L, R, 12, keys[:1], keys[:1], lvalid={keys[0]: lvalid[keys[0]]}, rvalid=None)


@pytest.mark.parametrize("kind", KINDS)
def test_multi_file_buckets(ctx, kind):
    L, R, keys = _tables(kind, 10_000, 8_000, 4)
    _check(ctx, L, R, 12, keys, keys, lsplit=6_000)                  # one side
    _check(ctx, L, R, 12, keys, keys, lsplit=3_000, rsplit=5_000)    # both sides
    rng = np.random.default_rng(5)
    lvalid = {keys[-1]: rng.random(len(L["lid"])) >= 0.1}
    _check(ctx, L, R, 12, keys, keys, lpreds=[("i", 100, False, 800, True)], lvalid=lvalid, lsplit=4_000, rsplit=2_000)


PREDICATE_CASES = {
    "int_inclusive": ([("i", 100, False, 600, False)], [("i", None, False, 500, False)]),
    "int_strict_with_float_literal": ([("i", 99.5, True, 700, True)], [("i", 10, True, None, False)]),
    "float": ([("f32", -5.0, False, 5.0, True)], [("f32", 0.1, True, None, False)]),
    "double_nan_literal": ([("f64", None, False, float("nan"), True)], [("f64", -50.0, False, None, False)]),
    "double_is_nan": ([("f64", float("nan"), False, None, False)], []),
    "string": ([("s", b"ab", False, b"facebook", True)], [("s", "a", True, None, False)]),
    "on_keys": ([("a", 1, False, 30, False)], [("b", None, False, 10, True)]),
    "left_only": ([("i", 200, False, None, False), ("s", None, False, b"b", False)], []),
    "right_only": ([], [("f64", -10.0, False, 10.0, False), ("i", 0, False, 900, True)]),
}


@pytest.mark.parametrize("case", sorted(PREDICATE_CASES))
@pytest.mark.parametrize("kind", ["i64_i32", "i32_str"])
def test_side_predicates(ctx, kind, case):
    L, R, keys = _tables(kind, 10_000, 8_000, 6)
    lp, rp = PREDICATE_CASES[case]
    if kind == "i32_str" and case == "on_keys":
        rp = [("b", None, False, b"b", True)]
    n, st = _check(ctx, L, R, 12, keys, keys, lp, rp)
    assert n > 0 or case == "double_is_nan"
    assert st["ms_exchange"] > 0  # the side selection's time


def test_one_key_with_predicates(ctx):
    L, R, _ = _tables("i64_i32", 10_000, 8_000, 7)
    _check(ctx, L, R, 12, ["a"], ["a"], [("f64", -20.0, False, 30.0, False)], [("s", b"abc", False, None, False)])
    L, R, _ = _tables("i32_str", 10_000, 8_000, 7)
    _check(ctx, L, R, 12, ["b"], ["b"], [("i", 500, True, None, False)], [])


def test_a_predicate_that_keeps_nothing_gives_a_valid_empty_batch(ctx):
    from hyperspace_b200 import _native

    L, R, keys = _tables("i32_str", 5_000, 5_000, 8)
    lres, rres = [_index(ctx, L, None, keys, 12, "l")], [_index(ctx, R, None, keys, 12, "r")]
    for output in (_native.HS_OUT_HOST, _native.HS_OUT_DEVICE):
        batch, st = _run(ctx, lres, rres, 12, keys, keys, [("i", 5000, False, None, False)], [], output=output)
        assert batch.num_rows == 0 and st["rows_out"] == 0
        if output == _native.HS_OUT_HOST:
            assert [n for n, _, _ in batch.columns] == ["lid", "rid"]
            assert all(len(d) == 0 for _, d, _ in batch.columns)
        else:
            assert [n for n, _, _ in batch.device_columns] == ["lid", "rid"]
        batch.free()
    for r in lres + rres:
        r.free()


class _Dev:
    """A device array for torch.as_tensor (__cuda_array_interface__)."""

    def __init__(self, ptr, n, typestr):
        self.__cuda_array_interface__ = {"shape": (n,), "typestr": typestr, "data": (ptr, False), "version": 2}


def test_device_output(ctx):
    import torch

    from hyperspace_b200 import _native

    L, R, keys = _tables("i64_3", 8_000, 8_000, 9)
    lres, rres = [_index(ctx, L, None, keys, 12, "l")], [_index(ctx, R, None, keys, 12, "r")]
    lp, rp = [("i", 100, False, None, False)], [("f32", None, False, 3.0, True)]
    host, _ = _run(ctx, lres, rres, 12, keys, keys, lp, rp)
    dev, _ = _run(ctx, lres, rres, 12, keys, keys, lp, rp, output=_native.HS_OUT_DEVICE)
    assert dev.on_device and dev.num_rows == host.num_rows > 0
    for (name, ty, ptr), (hname, hdata, _) in zip(dev.device_columns, host.columns):
        assert name == hname and ty == _native.HS_TYPE_INT64
        got = torch.as_tensor(_Dev(ptr, dev.num_rows, "<i8"), device="cuda").cpu().numpy()
        assert np.array_equal(got, hdata)
    host.free()
    dev.free()
    for r in lres + rres:
        r.free()


# ---- one key, no predicates: exactly hs_bucket_join ------------------------------------------------------------------

def _profile(ctx):
    return {k: v["launches"] for k, v in ctx.profile_report().items()}


@pytest.mark.parametrize("ktype", ["int32", "int64", "string"])
def test_one_key_without_predicates_is_hs_bucket_join(ctx, ktype):
    rng = np.random.default_rng(10)
    nl, nr, nb = 30_000, 20_000, 16

    def table(n, idname):
        if ktype == "string":
            k = np.array([WORDS[i] + str(j).encode() for i, j in zip(rng.integers(0, len(WORDS), n), rng.integers(0, 300, n))],
                         dtype=object)
        else:
            k = rng.integers(-3000, 3000, n).astype(np.int32 if ktype == "int32" else np.int64)
        return {"k": k, "v": rng.normal(0, 1, n), "s": np.array([WORDS[i] for i in rng.integers(0, len(WORDS), n)], dtype=object),
                idname: np.arange(n, dtype=np.int64)}

    L, R = table(nl, "lid"), table(nr, "rid")
    for split in (None, 12_000):  # single-file buckets, then multi-file buckets on the left
        if split is None:
            lres = [_index(ctx, L, None, ["k"], nb, "l")]
        else:
            lres = [_index(ctx, {c: v[:split] for c, v in L.items()}, None, ["k"], nb, "l0"),
                    _index(ctx, {c: v[split:] for c, v in L.items()}, None, ["k"], nb, "l1")]
        rres = [_index(ctx, R, None, ["k"], nb, "r")]
        lf, lb = _sides(lres)
        rf, rb = _sides(rres)
        ctx.profile_enable(True)
        ctx.profile_report()
        a, sa = ctx.bucket_join(lf, lb, rf, rb, nb, "k", "k", ["k", "lid", "s"], ["v", "rid"])
        pa_ = _profile(ctx)
        b, sb = ctx.bucket_join_where(lf, lb, rf, rb, nb, ["k"], ["k"], ["k", "lid", "s"], ["v", "rid"])
        pb = _profile(ctx)
        ctx.profile_enable(False)
        assert pa_ == pb and pb.get("k_join_count") == 1 and "k_predicate_mask" not in pb
        assert split is not None or "k_encode_keys" not in pb  # (multi-file buckets are re-sorted, which may encode keys)
        assert sa["gpu_launches"] == sb["gpu_launches"]
        assert a.num_rows == b.num_rows > 0
        for (na, va, ma), (nb_, vb, mb) in zip(a.columns, b.columns):
            assert na == nb_ and va.dtype == vb.dtype
            if va.dtype == object:
                assert list(va) == list(vb)
            else:
                assert va.tobytes() == vb.tobytes()
            assert (ma is None) == (mb is None) and (ma is None or ma.tobytes() == mb.tobytes())
        a.free()
        b.free()
        for r in lres + rres:
            r.free()


def test_composite_join_runs_one_probe_without_key_encoding(ctx):
    L, R, keys = _tables("i64_i32", 5_000, 5_000, 11)
    lres, rres = [_index(ctx, L, None, keys, 12, "l")], [_index(ctx, R, None, keys, 12, "r")]
    ctx.profile_enable(True)
    ctx.profile_report()
    batch, _ = _run(ctx, lres, rres, 12, keys, keys)  # the join alone: createIndex encodes keys for its sort
    prof = _profile(ctx)
    ctx.profile_enable(False)
    li, ri = J.bucket_join(L, R, 12, keys, keys)
    assert np.array_equal(batch.column("lid"), L["lid"][li]) and np.array_equal(batch.column("rid"), R["rid"][ri])
    assert prof.get("k_join_count") == 1 and "k_encode_keys" not in prof and "k_predicate_mask" not in prof
    batch.free()
    for r in lres + rres:
        r.free()


# ---- refusals ----------------------------------------------------------------------------------------------------------

def _raw_side(cols):
    """One Parquet file as a one-bucket side (enough for the refusals, which come before any join)."""
    from hyperspace_b200 import _native

    sink = io.BytesIO()
    pq.write_table(pa.table(cols), sink, compression="NONE")
    return [_native.FileImage(data=sink.getvalue())], [0]


def test_refusals(ctx):
    from hyperspace_b200 import _native as N

    n = 100
    cols = {f"k{i}": np.arange(n, dtype=np.int64) for i in range(9)}
    cols.update({"i32": np.arange(n, dtype=np.int32), "f": np.arange(n, dtype=np.float32), "d": np.arange(n, dtype=np.float64),
                 "b": np.arange(n) % 2 == 0, "t": np.array([b"x"] * n, dtype=object), "lid": np.arange(n, dtype=np.int64)})
    cols["t"] = pa.array(cols["t"].tolist(), pa.binary())
    f, b = _raw_side(cols)

    def err(lkeys, rkeys, lpreds=(), rpreds=()):
        with pytest.raises(N.HyperspaceGpuError) as e:
            ctx.bucket_join_where(f, b, f, b, 1, lkeys, rkeys, ["lid"], ["lid"], lpreds, rpreds)
        return e.value

    assert err([], []).code == N.HS_EINVAL
    assert err([f"k{i}" for i in range(9)], [f"k{i}" for i in range(9)]).code == N.HS_EUNSUPPORTED
    e = err(["k0", "k1"], ["k0", "i32"])
    assert e.code == N.HS_EUNSUPPORTED and "different types" in e.message
    e = err(["i32"], ["k0"])
    assert e.code == N.HS_EUNSUPPORTED and "different types" in e.message
    for key in ("f", "d", "b"):
        assert err(["k0", key], ["k0", key]).code == N.HS_EUNSUPPORTED
        assert err([key], [key]).code == N.HS_EUNSUPPORTED
    # a bad predicate: the codes and messages of hs_filter_scan_where
    for preds in ([("t", 1, False, None, False)], [("d", "a", False, None, False)], [("k0", i, False, None, False) for i in range(17)],
                  [("b", 0, False, None, False)], [("nope", 1, False, None, False)]):
        with pytest.raises(N.HyperspaceGpuError) as want:
            ctx.filter_scan_where(f, None, ["lid"], preds, sorted_on_key=False)
        for side in ("left", "right"):
            got = err(["k0"], ["k0"], preds, ()) if side == "left" else err(["k0"], ["k0"], (), preds)
            assert (got.code, got.message) == (want.value.code, want.value.message)
    # hs_bucket_join keeps refusing null keys
    nullable = {"k": pa.array([1, None, 3], pa.int64()), "lid": pa.array([0, 1, 2], pa.int64())}
    g, gb = _raw_side(nullable)
    with pytest.raises(N.HyperspaceGpuError) as e:
        ctx.bucket_join(g, gb, g, gb, 1, "k", "k", ["lid"], ["lid"])
    assert e.value.code == N.HS_EUNSUPPORTED
    batch, _ = ctx.bucket_join_where(g, gb, g, gb, 1, ["k"], ["k"], ["lid"], ["lid"])  # ... which an inner join drops
    assert batch.column("lid").tolist() == [0, 2]
    batch.free()


# ---- through the Hyperspace API ----------------------------------------------------------------------------------------

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


def _rows(res, cols):
    return sorted(zip(*[np.asarray(res[c]).tolist() for c in cols]), key=repr)


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


def test_e2e_join_of_filtered_sides_uses_the_join_indexes(env):
    """E2EHyperspaceRulesTest.scala:376-405: two filtered sub-queries joined on their join indexes, over SampleData."""
    from hyperspace_b200.index_config import IndexConfig
    from hyperspace_b200.session import col

    s, hs, tmp = env
    cols = list(zip(*SAMPLE))
    _write(tmp / "sample", "a.parquet", {"Date": pa.array(cols[0]), "RGUID": pa.array(cols[1]), "Query": pa.array(cols[2]),
                                          "imprs": pa.array(cols[3], pa.int32()), "clicks": pa.array(cols[4], pa.int32())})
    df = s.read.parquet(str(tmp / "sample"))
    hs.createIndex(df, IndexConfig("leftJoinIndex", ["clicks"], ["Query"]))
    hs.createIndex(df, IndexConfig("leftFilterIndex", ["Query"], ["clicks"]))
    hs.createIndex(df, IndexConfig("rightJoinIndex", ["clicks"], ["imprs"]))
    hs.createIndex(df, IndexConfig("rightFilterIndex", ["imprs"], ["clicks"]))
    left = df.filter(col("Query") == "facebook").select("clicks", "Query")
    right = df.filter(col("imprs") >= 2).select("clicks", "imprs")
    q = left.join(right, on="clicks")
    s.disableHyperspace()
    base = q.collect()
    s.enableHyperspace()
    plan = q.explain()
    assert "Name: leftJoinIndex" in plan and "Name: rightJoinIndex" in plan and "FilterIndex" not in plan
    assert "exchange=none" in plan and "leftFilter=" in plan and "rightFilter=" in plan
    got = q.collect()
    want = sorted(((c1, q1, c2, i2) for _, _, q1, _, c1 in SAMPLE for _, _, _, i2, c2 in SAMPLE
                   if q1 == "facebook" and i2 >= 2 and c1 == c2), key=repr)
    assert _rows(got, ["clicks", "Query", "clicks_right", "imprs"]) == want == _rows(base, ["clicks", "Query", "clicks_right", "imprs"])


def _kv_table(first, n, seed, other=("c3", "c4")):
    """c1 int, c2 string (the reference fixture's key types), and two more columns under the names `other`."""
    rng = np.random.default_rng(seed)
    return {"c1": (np.arange(first, first + n) % 97).astype(np.int32),
            "c2": np.array([WORDS[i] for i in rng.integers(0, 6, n)], dtype=object).astype(str),
            other[0]: rng.integers(0, 1000, n).astype(np.int64), other[1]: rng.normal(0, 1, n)}


def test_composite_index_join_refresh_and_hybrid_scan(env):
    from hyperspace_b200.index_config import IndexConfig
    from hyperspace_b200.session import col

    s, hs, tmp = env
    t1 = _kv_table(0, 4_000, 1)
    t2 = _kv_table(50, 3_000, 2, ("d3", "d4"))
    _write(tmp / "t1", "a.parquet", t1)
    _write(tmp / "t2", "a.parquet", t2)
    s.conf.set("spark.hyperspace.index.lineage.enabled", True)
    d1, d2 = s.read.parquet(str(tmp / "t1")), s.read.parquet(str(tmp / "t2"))
    hs.createIndex(d1, IndexConfig("t1i2", ["c1", "c2"], ["c3"]))
    hs.createIndex(d2, IndexConfig("t2i2", ["c1", "c2"], ["d4"]))

    def query(a, b):
        return a.filter(col("c3") >= 100).join(b, on=[("c2", "c2"), ("c1", "c1")]).select("c1", "c2", "c3", "d4")

    def want(a, b):
        out = []
        from collections import defaultdict

        idx = defaultdict(list)
        for c1, c2, c4 in zip(b["c1"].tolist(), b["c2"].tolist(), b["d4"].tolist()):
            idx[(c1, c2)].append(c4)
        for c1, c2, c3 in zip(a["c1"].tolist(), a["c2"].tolist(), a["c3"].tolist()):
            if c3 >= 100:
                out += [(c1, c2, c3, c4) for c4 in idx[(c1, c2)]]
        return sorted(out, key=repr)

    s.enableHyperspace()
    q = query(d1, d2)
    plan = q.explain()
    assert "Name: t1i2" in plan and "Name: t2i2" in plan
    assert _rows(q.collect(), ["c1", "c2", "c3", "d4"]) == want(t1, t2)
    s.disableHyperspace()
    assert _rows(q.collect(), ["c1", "c2", "c3", "d4"]) == want(t1, t2)
    # appended files: incremental refresh (multi-file buckets), then Hybrid Scan over a further unindexed file
    extra = _kv_table(10, 1_500, 3)
    _write(tmp / "t1", "b.parquet", extra)
    d1 = s.read.parquet(str(tmp / "t1"))
    hs.refreshIndex("t1i2", "incremental")
    s.enableHyperspace()
    t1b = {c: np.concatenate([t1[c], extra[c]]) for c in t1}
    q = query(d1, d2)
    assert "Name: t1i2" in q.explain()
    assert _rows(q.collect(), ["c1", "c2", "c3", "d4"]) == want(t1b, t2)
    more = _kv_table(20, 800, 4, ("d3", "d4"))
    _write(tmp / "t2", "b.parquet", more)
    s.conf.set("spark.hyperspace.index.hybridscan.enabled", True)
    s.conf.set("spark.hyperspace.index.hybridscan.maxAppendedRatio", "0.9")
    d2 = s.read.parquet(str(tmp / "t2"))
    q = query(d1, d2)
    plan = q.explain()
    assert "Name: t1i2" in plan and "Name: t2i2" in plan
    t2b = {c: np.concatenate([t2[c], more[c]]) for c in t2}
    assert _rows(q.collect(), ["c1", "c2", "c3", "d4"]) == want(t1b, t2b)
