"""GPU left semi / left anti bucket joins (hs_bucket_join_exists), compared with the numpy restatement in
tests/join_exists_oracle.py as exact row sequences: the engine outputs the kept left rows in (bucket, left sorted
position) order, and so does the oracle.  Key types int32 / int64 / string / timestamp / decimal, 1-3 key columns,
nullable keys, filters below either side, multi-file buckets, a grid-stride-sized probe, the refusals, the kernels a
call launches, and the Hyperspace API (TPC-H Q4- and Q22-shaped queries, Hybrid Scan)."""
import ctypes as C
import decimal
import io
import os

import numpy as np
import pyarrow as pa
import pyarrow.parquet as pq
import pytest

import join_exists_oracle as JE
import join_oracle as J

pytestmark = pytest.mark.gpu

WORDS = [b"", b"a", b"ab", b"abc", b"abd", b"b", "été".encode(), b"facebook", b"zz", b"\xff"]
HOWS = ["semi", "anti"]


@pytest.fixture(scope="module")
def ctx():
    from hyperspace_b200 import _native

    c = _native.Context(0)
    yield c
    c.close()


def _arrow_column(v, valid, kind):
    mask = None if valid is None else ~np.asarray(valid, dtype=bool)
    if kind == "ts":
        return pa.array(v, pa.timestamp("us"), mask=mask)
    if kind == "dec":
        return pa.array([None if (mask is not None and mask[i]) else decimal.Decimal(int(x)).scaleb(-2) for i, x in enumerate(v)],
                        pa.decimal128(12, 2))
    if v.dtype == object:
        return pa.array([None if (mask is not None and mask[i]) else x for i, x in enumerate(v.tolist())], pa.binary())
    return pa.array(v, mask=mask)


def _index(ctx, cols, valids, keys, nb, uuid, kinds):
    """createIndex over the columns (in memory): indexed = keys, included = every other column."""
    from hyperspace_b200 import _native

    sink = io.BytesIO()
    pq.write_table(pa.table({c: _arrow_column(v, (valids or {}).get(c), kinds.get(c)) for c, v in cols.items()}), sink,
                   compression="NONE")
    res, _ = ctx.create_index([_native.FileImage(data=sink.getvalue())], list(keys), [c for c in cols if c not in keys], nb,
                              output=_native.HS_OUT_HOST, job_uuid=uuid)
    return res


def _sides(res_list):
    files, buckets = [], []
    for r in res_list:
        files += r.as_sources()
        buckets += [f.bucket for f in r.files]
    return files, buckets


def _tables(kind, nl, nr, seed):
    """Two tables with heavy key ties and partial overlap, their key names and the Spark kinds of typed columns."""
    rng = np.random.default_rng(seed)

    def one(n, idname):
        kinds = {}
        if kind == "i32":
            cols = {"a": rng.integers(-40, 40, n).astype(np.int32)}
        elif kind == "i64_2":
            cols = {"a": rng.integers(0, 30, n).astype(np.int64) * 10**12, "b": rng.integers(-5, 5, n).astype(np.int64)}
        elif kind == "str":
            cols = {"a": np.array([WORDS[i] + str(j).encode() for i, j in zip(rng.integers(0, len(WORDS), n),
                                                                                rng.integers(0, 20, n))], dtype=object)}
        elif kind == "ts_dec":  # a timestamp and a decimal(12,2): both int64 here, hashed as Spark hashes them
            cols = {"a": (rng.integers(0, 40, n) * 1_000_000 + 1_600_000_000_000_000).astype(np.int64),
                    "b": rng.integers(-4, 4, n).astype(np.int64)}
            kinds = {"a": "ts", "b": "dec"}
        elif kind == "i32_str":
            cols = {"a": rng.integers(0, 20, n).astype(np.int32),
                    "b": np.array([WORDS[i] for i in rng.integers(0, len(WORDS), n)], dtype=object)}
        else:  # three longs, the first with heavy ties: a match depends on the later columns
            cols = {"a": rng.integers(0, 3, n).astype(np.int64), "b": rng.integers(0, 12, n).astype(np.int64),
                    "c": rng.integers(0, 12, n).astype(np.int64)}
        cols["i"] = rng.integers(0, 1000, n).astype(np.int64)
        cols["j"] = rng.integers(0, 1000, n).astype(np.int64)
        cols["s"] = np.array([WORDS[i] for i in rng.integers(0, len(WORDS), n)], dtype=object)
        cols[idname] = np.arange(n, dtype=np.int64)
        return cols, kinds

    (L, kinds), (R, _) = one(nl, "lid"), one(nr, "rid")
    keys = [k for k in ("a", "b", "c") if k in L]
    # the right side lacks every fourth value of the first key, so that every kind has left rows without a match
    keep = J.tuple_codes([R["a"]]) % 4 != 0
    R = {c: v[keep] for c, v in R.items()}
    R["rid"] = np.arange(len(R["rid"]), dtype=np.int64)
    return L, R, keys, kinds


# filters below a side: (predicates, terms, compares) and the rows they keep, restated in numpy
def _filter(case, cols):
    n = len(cols["i"])
    if case == "none":
        return ((), (), ()), np.ones(n, bool)
    if case == "pred":
        return (([("i", 150, False, 800, True)], (), ())), (cols["i"] >= 150) & (cols["i"] < 800)
    if case == "isin":
        vals = list(range(0, 1000, 3))
        return (((), [("i", vals, [])], ())), np.isin(cols["i"], vals)
    if case == "cmp":
        return (((), (), [("i", "<", "j")])), cols["i"] < cols["j"]
    # all three at once
    vals = [b"a", b"ab", b"zz", b""]
    s_in = np.array([v in vals for v in cols["s"].tolist()])
    return (([("j", 100, False, None, False)], [("s", vals, [])], [("i", "<=", "j")]),
            (cols["j"] >= 100) & s_in & (cols["i"] <= cols["j"]))


def _run(ctx, lres, rres, nb, lkeys, rkeys, how, lf_=((), (), ()), rf_=((), (), ()), **kw):
    lf, lb = _sides(lres)
    rf, rb = _sides(rres)
    return ctx.bucket_join_exists(lf, lb, rf, rb, nb, lkeys, rkeys, ["lid"], how, lf_[0], rf_[0], lf_[1], rf_[1], lf_[2],
                                  rf_[2], **kw)


def _check(ctx, kind, L, R, nb, keys, kinds, lvalid=None, rvalid=None, lcase="none", rcase="none", lsplit=None, rsplit=None):
    """Indexes both tables (in two createIndex calls where a split is given: multi-file buckets), runs the semi and the
    anti join on the GPU and compares each left-id sequence with the oracle's.  Returns the two row counts."""
    def build(cols, valids, split, tag):
        if split is None:
            return [_index(ctx, cols, valids, keys, nb, tag, kinds)]
        n = len(next(iter(cols.values())))
        return [_index(ctx, {c: v[a:b] for c, v in cols.items()}, {c: v[a:b] for c, v in (valids or {}).items()}, keys, nb,
                       f"{tag}{j}", kinds) for j, (a, b) in enumerate(((0, split), (split, n)))]

    lres, rres = build(L, lvalid, lsplit, "l"), build(R, rvalid, rsplit, "r")
    lf_, lmask = _filter(lcase, L)
    rf_, rmask = _filter(rcase, R)
    counts = []
    for how in HOWS:
        batch, st = _run(ctx, lres, rres, nb, keys, keys, how, lf_, rf_)
        want = JE.exists_join(L, R, nb, keys, keys, how, left_valids=lvalid, right_valids=rvalid, left_mask=lmask, right_mask=rmask)
        assert batch.num_rows == len(want) == st["rows_out"], (kind, how)
        assert [n for n, _, _ in batch.columns] == ["lid"]
        assert np.array_equal(batch.column("lid"), L["lid"][want]), (kind, how)
        counts.append(len(want))
        batch.free()
    for r in lres + rres:
        r.free()
    return counts


KINDS = ["i32", "i64_2", "str", "ts_dec", "i32_str", "i64_3"]


@pytest.mark.parametrize("nb", [1, 16])
@pytest.mark.parametrize("kind", KINDS)
def test_against_the_oracle(ctx, kind, nb):
    L, R, keys, kinds = _tables(kind, 9_000, 6_000, 1)
    semi, anti = _check(ctx, kind, L, R, nb, keys, kinds)
    assert semi > 0 and anti > 0 and semi + anti == 9_000


@pytest.mark.parametrize("kind", KINDS)
def test_nullable_keys(ctx, kind):
    """Nulls in each key column on both sides, then in every key column at once: semi drops null-key left rows, anti keeps
    them, and a null never matches a right 0 or empty string."""
    L, R, keys, kinds = _tables(kind, 8_000, 6_000, 2)
    rng = np.random.default_rng(3)
    for pos in range(len(keys)):
        lvalid = {keys[pos]: rng.random(8_000) >= 0.1}
        rvalid = {keys[pos]: rng.random(len(R["rid"])) >= 0.1}
        semi, anti = _check(ctx, kind, L, R, 12, keys, kinds, lvalid, rvalid)
        assert semi + anti == 8_000
    lvalid = {k: rng.random(8_000) >= 0.05 for k in keys}
    rvalid = {k: rng.random(len(R["rid"])) >= 0.05 for k in keys}
    _check(ctx, kind, L, R, 12, keys, kinds, lvalid, rvalid)
    _check(ctx, kind, L, R, 12, keys, kinds, lvalid, None)


def test_null_left_key_against_right_zero_and_empty_string(ctx):
    """The values a null decodes to (0, the empty string) sit on the right side: semi must not match them, anti must keep
    the null-key rows."""
    for kind, zero in (("i32", 0), ("str", b"")):
        L, R, keys, kinds = _tables(kind, 2_000, 1_000, 4)
        L["a"][:200] = zero
        R["a"][:50] = zero
        lvalid = {"a": np.arange(2_000) >= 100}  # rows 0-99 null, rows 100-199 a real zero
        semi, anti = _check(ctx, kind, L, R, 4, keys, kinds, lvalid, None)
        assert semi >= 100 and anti >= 100


@pytest.mark.parametrize("case", ["pred", "isin", "cmp", "all"])
@pytest.mark.parametrize("kind", ["i64_2", "i32_str", "ts_dec"])
def test_filters_below_either_side(ctx, kind, case):
    L, R, keys, kinds = _tables(kind, 8_000, 6_000, 5)
    rng = np.random.default_rng(6)
    lvalid = {keys[0]: rng.random(8_000) >= 0.08}
    rvalid = {keys[-1]: rng.random(len(R["rid"])) >= 0.08}
    _check(ctx, kind, L, R, 12, keys, kinds, lvalid, rvalid, lcase=case)
    _check(ctx, kind, L, R, 12, keys, kinds, lvalid, rvalid, rcase=case)
    _check(ctx, kind, L, R, 12, keys, kinds, lvalid, rvalid, lcase=case, rcase=case)


def test_a_right_filter_that_empties_every_bucket(ctx):
    L, R, keys, kinds = _tables("i64_2", 4_000, 3_000, 7)
    lres, rres = [_index(ctx, L, None, keys, 8, "l", kinds)], [_index(ctx, R, None, keys, 8, "r", kinds)]
    none = ([("i", 5000, False, None, False)], (), ())
    semi, _ = _run(ctx, lres, rres, 8, keys, keys, "semi", rf_=none)
    anti, _ = _run(ctx, lres, rres, 8, keys, keys, "anti", rf_=none)
    assert semi.num_rows == 0 and semi.column("lid").size == 0
    assert np.array_equal(anti.column("lid"), L["lid"][JE.exists_join(L, R, 8, keys, keys, "anti", right_mask=np.zeros(len(R["rid"]), bool))])
    assert anti.num_rows == 4_000
    for b in (semi, anti):
        b.free()
    for r in lres + rres:
        r.free()


@pytest.mark.parametrize("kind", ["i64_2", "str", "i64_3"])
def test_multi_file_buckets(ctx, kind):
    """Two index versions per side, as an incremental refresh leaves them: the engine re-sorts each bucket's rows."""
    L, R, keys, kinds = _tables(kind, 9_000, 7_000, 8)
    rng = np.random.default_rng(9)
    lvalid = {keys[-1]: rng.random(9_000) >= 0.1}
    _check(ctx, kind, L, R, 12, keys, kinds, lsplit=5_000)
    _check(ctx, kind, L, R, 12, keys, kinds, rsplit=2_000)
    _check(ctx, kind, L, R, 12, keys, kinds, lvalid, None, lcase="pred", rcase="cmp", lsplit=3_000, rsplit=4_000)


def test_device_output(ctx):
    import torch

    from hyperspace_b200 import _native

    L, R, keys, kinds = _tables("i64_3", 6_000, 6_000, 10)
    lres, rres = [_index(ctx, L, None, keys, 12, "l", kinds)], [_index(ctx, R, None, keys, 12, "r", kinds)]
    for how in HOWS:
        host, _ = _run(ctx, lres, rres, 12, keys, keys, how)
        dev, _ = _run(ctx, lres, rres, 12, keys, keys, how, output=_native.HS_OUT_DEVICE)
        assert dev.on_device and dev.num_rows == host.num_rows > 0
        (name, ty, ptr), = dev.device_columns
        arr = {"shape": (dev.num_rows,), "typestr": "<i8", "data": (ptr, False), "version": 2}
        got = torch.as_tensor(type("D", (), {"__cuda_array_interface__": arr})(), device="cuda").cpu().numpy()
        assert name == "lid" and ty == _native.HS_TYPE_INT64 and np.array_equal(got, host.column("lid"))
        host.free()
        dev.free()
    for r in lres + rres:
        r.free()


def test_grid_stride_probe(ctx):
    """20 M left rows (more than one thread per row of the capped grid) against the synthetic table's overlapping half:
    k is a bijection of the row, so semi keeps exactly rows [N/2, N) and anti rows [0, N/2), in (bucket, k) order."""
    from hyperspace_b200 import _native as N
    from oracle import oracle as O

    n, nb = 20_000_000, 64

    def build(first, included):
        src = ctx.synth_table(first, n, 5, n_files=16, row_groups_per_file=2, output=N.HS_OUT_DEVICE)
        idx, _ = ctx.create_index(src.as_sources(), ["k"], included, nb, output=N.HS_OUT_DEVICE, job_uuid="g")
        src.free()
        return idx

    L, R = build(0, ["v1", "v3"]), build(n // 2, [])
    lf, lb, rf, rb = L.as_sources(), [f.bucket for f in L.files], R.as_sources(), [f.bucket for f in R.files]
    try:
        for how, rows in (("semi", np.arange(n // 2, n)), ("anti", np.arange(0, n // 2))):
            batch, st = ctx.bucket_join_exists(lf, lb, rf, rb, nb, ["k"], ["k"], ["k", "v3"], how)
            k, v3 = batch.column("k"), batch.column("v3")
            batch.free()
            assert len(k) == len(rows) == st["rows_out"]
            want = O.synthetic_rows_at(rows)
            assert np.array_equal(np.sort(k), np.sort(want["k"]))
            assert int(v3.astype(np.int64).sum()) == int(want["v3"].astype(np.int64).sum())
            b = O.np_pmod(O.np_hash_long(k), nb)
            assert np.all(np.diff(b) >= 0)                                   # bucket-major
            same = b[1:] == b[:-1]
            assert np.all(k[1:][same] > k[:-1][same])                        # ascending keys inside a bucket
    finally:
        L.free()
        R.free()
        ctx.trim()


# ---- the kernels a call launches ---------------------------------------------------------------------------------------

def _profile(ctx):
    return {k: v["launches"] for k, v in ctx.profile_report().items()}


def test_one_probe_and_no_emit(ctx):
    L, R, keys, kinds = _tables("i32_str", 6_000, 5_000, 11)
    rng = np.random.default_rng(12)
    lvalid = {"b": rng.random(6_000) >= 0.1}
    lres, rres = [_index(ctx, L, lvalid, keys, 12, "l", kinds)], [_index(ctx, R, None, keys, 12, "r", kinds)]
    lf, lb = _sides(lres)
    rf, rb = _sides(rres)
    ctx.profile_enable(True)
    ctx.profile_report()
    try:
        for how in HOWS:
            b, _ = ctx.bucket_join_exists(lf, lb, rf, rb, 12, keys, keys, ["lid", "s"], how)
            prof = _profile(ctx)
            assert prof.get("k_join_exists") == 1 and "k_join_emit" not in prof and "k_join_count" not in prof, prof
            # the anti join keeps null-key rows: no IS NOT NULL selection on the left, so no mask kernel at all
            assert ("k_predicate_mask" in prof) == (how == "semi"), prof
            b.free()
        b, _ = ctx.bucket_join_where(lf, lb, rf, rb, 12, keys, keys, ["lid", "s"], ["rid"])
        prof = _profile(ctx)
        assert prof.get("k_join_count") == 1 and prof.get("k_join_emit") == 1 and "k_join_exists" not in prof, prof
        b.free()
    finally:
        ctx.profile_enable(False)
        for r in lres + rres:
            r.free()


# ---- refusals ----------------------------------------------------------------------------------------------------------

def _raw_side(cols):
    from hyperspace_b200 import _native

    sink = io.BytesIO()
    pq.write_table(pa.table(cols), sink, compression="NONE")
    return [_native.FileImage(data=sink.getvalue())], [0]


def test_refusals(ctx):
    from hyperspace_b200 import _native as N

    n = 100
    cols = {"k0": np.arange(n, dtype=np.int64), "k1": np.arange(n, dtype=np.int64), "i32": np.arange(n, dtype=np.int32),
            "f": np.arange(n, dtype=np.float32), "d": np.arange(n, dtype=np.float64), "b": np.arange(n) % 2 == 0,
            "lid": np.arange(n, dtype=np.int64)}
    f, b = _raw_side(cols)

    def both(lkeys, rkeys, how="semi"):
        with pytest.raises(N.HyperspaceGpuError) as want:
            ctx.bucket_join_where(f, b, f, b, 1, lkeys, rkeys, ["lid"], ["lid"])
        with pytest.raises(N.HyperspaceGpuError) as got:
            ctx.bucket_join_exists(f, b, f, b, 1, lkeys, rkeys, ["lid"], how)
        assert (got.value.code, got.value.message) == (want.value.code, want.value.message)
        return got.value

    for how in HOWS:
        for key in ("f", "d", "b"):  # float, double and boolean keys: the inner join's code and message
            assert both([key], [key], how).code == N.HS_EUNSUPPORTED
            assert both(["k0", key], ["k0", key], how).code == N.HS_EUNSUPPORTED
        e = both(["i32"], ["k0"], how)
        assert e.code == N.HS_EUNSUPPORTED and "different types" in e.message
        e = both(["k0", "k1"], ["k0", "i32"], how)
        assert e.code == N.HS_EUNSUPPORTED and "different types" in e.message
        assert both([], [], how).code == N.HS_EINVAL
        assert both([f"k{i % 2}" for i in range(9)], [f"k{i % 2}" for i in range(9)], how).code == N.HS_EUNSUPPORTED
    # join_type outside HS_JOIN_LEFT_SEMI / HS_JOIN_LEFT_ANTI, the inner join's 0 included
    for jt in (0, 3, -1):
        with pytest.raises(N.HyperspaceGpuError) as e:
            ctx.bucket_join_exists(f, b, f, b, 1, ["k0"], ["k0"], ["lid"], jt)
        assert e.value.code == N.HS_EINVAL and "join_type" in e.value.message
    with pytest.raises(ValueError):
        ctx.bucket_join_exists(f, b, f, b, 1, ["k0"], ["k0"], ["lid"], "left")
    # a right projection: the C entry point refuses it
    L = N.load_library()
    spec, keep, lk, rk, (lp, nlp), (rp, nrp) = ctx._join_where_args(f, b, f, b, 1, ["k0"], ["k0"], ["lid"], ["lid"], (), (), N.HS_OUT_HOST)
    res, st, err = C.c_void_p(), N.Stats(), C.create_string_buffer(1024)
    rc = L.hs_bucket_join_exists(ctx._h, C.byref(spec), N.HS_JOIN_LEFT_SEMI, lk, rk, 1, lp, nlp, None, 0, None, 0, rp, nrp, None, 0,
                                 None, 0, C.byref(res), C.byref(st), err, len(err))
    assert rc == N.HS_EINVAL and b"n_right_columns" in err.value and not res.value
    # the same call without the projection runs
    spec.n_right_columns = 0
    rc = L.hs_bucket_join_exists(ctx._h, C.byref(spec), N.HS_JOIN_LEFT_ANTI, lk, rk, 1, lp, nlp, None, 0, None, 0, rp, nrp, None, 0,
                                 None, 0, C.byref(res), C.byref(st), err, len(err))
    assert rc == N.HS_OK and L.hs_batch_num_rows(res) == 0
    L.hs_batch_free(res)
    del keep


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


def _orders(first, n, seed):
    rng = np.random.default_rng(seed)
    return {"o_orderkey": np.arange(first, first + n, dtype=np.int64),
            "o_custkey": rng.integers(0, 900, n).astype(np.int64),
            "o_orderdate": rng.integers(8000, 10000, n).astype(np.int32),  # days since the epoch
            "o_orderpriority": np.array([f"{p}-X" for p in rng.integers(1, 6, n)], dtype=object).astype(str)}


def _lineitem(n, max_order, seed):
    rng = np.random.default_rng(seed)
    commit = rng.integers(8000, 10000, n).astype(np.int32)
    return {"l_orderkey": rng.integers(0, max_order, n).astype(np.int64), "l_commitdate": commit,
            "l_receiptdate": (commit + rng.integers(-30, 30, n)).astype(np.int32), "l_quantity": rng.integers(1, 50, n).astype(np.int64)}


def _both_ways(s, q, cols):
    s.disableHyperspace()
    base = q.collect()
    s.enableHyperspace()
    plan = q.explain()
    got = q.collect()
    assert _rows(got, cols) == _rows(base, cols)
    return got, plan


def test_q4_shaped_semi_join(env):
    """TPC-H Q4: orders in a date range for which some lineitem has l_commitdate < l_receiptdate (EXISTS)."""
    from hyperspace_b200.index_config import IndexConfig
    from hyperspace_b200.session import col

    s, hs, tmp = env
    orders, li = _orders(0, 6_000, 1), _lineitem(20_000, 7_000, 2)
    _write(tmp / "orders", "a.parquet", orders)
    _write(tmp / "lineitem", "a.parquet", li)
    o, l = s.read.parquet(str(tmp / "orders")), s.read.parquet(str(tmp / "lineitem"))
    hs.createIndex(o, IndexConfig("ordersIdx", ["o_orderkey"], ["o_orderdate", "o_orderpriority"]))
    hs.createIndex(l, IndexConfig("lineitemIdx", ["l_orderkey"], ["l_commitdate", "l_receiptdate"]))
    q = (o.filter((col("o_orderdate") >= 8500) & (col("o_orderdate") < 8600))
         .join(l.filter(col("l_commitdate") < col("l_receiptdate")), on=("o_orderkey", "l_orderkey"), how="left_semi")
         .select("o_orderkey", "o_orderpriority"))
    got, plan = _both_ways(s, q, ["o_orderkey", "o_orderpriority"])
    assert "Name: ordersIdx" in plan and "Name: lineitemIdx" in plan and "joinType=LeftSemi" in plan
    late = {k for k, c, r in zip(li["l_orderkey"].tolist(), li["l_commitdate"].tolist(), li["l_receiptdate"].tolist()) if c < r}
    want = sorted(((k, p) for k, d, p in zip(orders["o_orderkey"].tolist(), orders["o_orderdate"].tolist(),
                                             orders["o_orderpriority"].tolist()) if 8500 <= d < 8600 and k in late), key=repr)
    assert _rows(got, ["o_orderkey", "o_orderpriority"]) == want and want
    assert list(got) == ["o_orderkey", "o_orderpriority"]


def test_q22_shaped_anti_join(env):
    """TPC-H Q22's NOT EXISTS: customers without orders, some with a null key (kept, as Spark's LeftAnti keeps them)."""
    from hyperspace_b200.index_config import IndexConfig
    from hyperspace_b200.session import col

    s, hs, tmp = env
    rng = np.random.default_rng(3)
    ckey = np.arange(1_200, dtype=np.int64)
    null = rng.random(1_200) < 0.05
    cust = {"c_custkey": pa.array(ckey, mask=null), "c_acctbal": pa.array(rng.integers(-1000, 10000, 1_200).astype(np.int64)),
            "c_phone": pa.array([f"{13 + i % 20}-555" for i in range(1_200)])}
    orders = _orders(0, 5_000, 4)
    _write(tmp / "customer", "a.parquet", cust)
    _write(tmp / "orders", "a.parquet", orders)
    c, o = s.read.parquet(str(tmp / "customer")), s.read.parquet(str(tmp / "orders"))
    hs.createIndex(c, IndexConfig("custIdx", ["c_custkey"], ["c_acctbal", "c_phone"]))
    hs.createIndex(o, IndexConfig("ordCustIdx", ["o_custkey"], []))
    q = c.filter(col("c_acctbal") > 0).join(o, on=("c_custkey", "o_custkey"), how="anti").select("c_custkey", "c_phone")
    got, plan = _both_ways(s, q, ["c_custkey", "c_phone"])
    assert "Name: custIdx" in plan and "Name: ordCustIdx" in plan and "joinType=LeftAnti" in plan
    has = set(orders["o_custkey"].tolist())
    bal = cust["c_acctbal"].to_numpy()
    want = sorted(((0 if null[i] else i, cust["c_phone"][i].as_py()) for i in range(1_200)
                   if bal[i] > 0 and (null[i] or i not in has)), key=repr)
    assert _rows(got, ["c_custkey", "c_phone"]) == want
    assert sum(null[i] and bal[i] > 0 for i in range(1_200)) > 0 and len(want) > 0


def test_hybrid_scan_with_appended_files_on_each_side(env):
    from hyperspace_b200.index_config import IndexConfig
    from hyperspace_b200.session import col

    s, hs, tmp = env
    orders, li = _orders(0, 4_000, 5), _lineitem(12_000, 5_000, 6)
    _write(tmp / "orders", "a.parquet", orders)
    _write(tmp / "lineitem", "a.parquet", li)
    o, l = s.read.parquet(str(tmp / "orders")), s.read.parquet(str(tmp / "lineitem"))
    hs.createIndex(o, IndexConfig("oi", ["o_orderkey"], ["o_orderdate"]))
    hs.createIndex(l, IndexConfig("li", ["l_orderkey"], ["l_commitdate", "l_receiptdate"]))
    more_o, more_l = _orders(4_000, 800, 7), _lineitem(2_000, 5_000, 8)
    _write(tmp / "orders", "b.parquet", more_o)
    _write(tmp / "lineitem", "b.parquet", more_l)
    s.conf.set("spark.hyperspace.index.hybridscan.enabled", True)
    s.conf.set("spark.hyperspace.index.hybridscan.maxAppendedRatio", "0.9")
    o, l = s.read.parquet(str(tmp / "orders")), s.read.parquet(str(tmp / "lineitem"))
    allo = {c: np.concatenate([orders[c], more_o[c]]) for c in ("o_orderkey", "o_orderdate")}
    alll = {c: np.concatenate([li[c], more_l[c]]) for c in li}
    late = {k for k, c, r in zip(alll["l_orderkey"].tolist(), alll["l_commitdate"].tolist(), alll["l_receiptdate"].tolist()) if c < r}
    for how, name in (("semi", "LeftSemi"), ("leftanti", "LeftAnti")):
        q = (o.filter(col("o_orderdate") >= 9000).join(l.filter(col("l_commitdate") < col("l_receiptdate")),
                                                      on=("o_orderkey", "l_orderkey"), how=how).select("o_orderkey", "o_orderdate"))
        got, plan = _both_ways(s, q, ["o_orderkey", "o_orderdate"])
        assert "Name: oi" in plan and "Name: li" in plan and f"joinType={name}" in plan
        want = sorted(((k, d) for k, d in zip(allo["o_orderkey"].tolist(), allo["o_orderdate"].tolist())
                       if d >= 9000 and ((k in late) == (how == "semi"))), key=repr)
        assert _rows(got, ["o_orderkey", "o_orderdate"]) == want and want
    # after an incremental refresh the appended rows sit in second files of the buckets (multi-file buckets)
    hs.refreshIndex("oi", "incremental")
    hs.refreshIndex("li", "incremental")
    s.conf.set("spark.hyperspace.index.hybridscan.enabled", False)
    q = o.join(l, on=("o_orderkey", "l_orderkey"), how="semi").select("o_orderkey")
    got, plan = _both_ways(s, q, ["o_orderkey"])
    assert "Name: oi" in plan and "Name: li" in plan
    keys = set(alll["l_orderkey"].tolist())
    assert _rows(got, ["o_orderkey"]) == sorted(((k,) for k in allo["o_orderkey"].tolist() if k in keys), key=repr)
