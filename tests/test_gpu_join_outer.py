"""GPU left, right and full outer bucket joins (hs_bucket_join_outer), compared with the numpy restatement in
tests/join_outer_oracle.py as exact row sequences with their validity.  Key types int32 / int64 / string / timestamp /
decimal, 1-3 key columns, nullable keys on either side (non-leading columns included), filters below either side,
multi-file buckets, padded string columns, device output, a grid-stride-sized probe, the refusals, the kernels a call
launches, and the Hyperspace API (a TPC-H Q13-shaped query, FullOuter, Hybrid Scan, masked collect())."""
import ctypes as C

import numpy as np
import pyarrow as pa
import pytest

import join_outer_oracle as JO
from test_gpu_join_exists import KINDS, _filter, _index, _raw_side, _sides, _tables, _write

pytestmark = pytest.mark.gpu

HOWS = ["left", "right", "full"]


@pytest.fixture(scope="module")
def ctx():
    from hyperspace_b200 import _native

    c = _native.Context(0)
    yield c
    c.close()


def _run(ctx, lres, rres, nb, keys, how, lf_=((), (), ()), rf_=((), (), ()), lcols=("lid", "s"), rcols=("rid", "i"), **kw):
    lf, lb = _sides(lres)
    rf, rb = _sides(rres)
    return ctx.bucket_join_outer(lf, lb, rf, rb, nb, keys, keys, list(lcols), list(rcols), how, lf_[0], rf_[0], lf_[1], rf_[1],
                                 lf_[2], rf_[2], **kw)


def _expect_side(batch, cols, table, rows, padded_side):
    """Each column of one side equals table[c][rows] where rows >= 0, is padded (value 0 / empty, validity 0) where rows
    is -1, and has a validity vector exactly when the side may be padded."""
    pad = rows < 0
    got = {n: (d, v) for n, d, v in batch.columns}
    for c in cols:
        d, v = got[c]
        assert (v is not None) == padded_side, c
        if v is not None:
            assert np.array_equal(v.astype(bool), ~pad), c
        want = table[c][np.where(pad, 0, rows)]
        if d.dtype == object:
            assert all(x == b"" for x in d[pad]), c
            assert list(d[~pad]) == list(want[~pad]), c
        else:
            assert np.all(d[pad] == 0), c
            assert np.array_equal(d[~pad], want[~pad]), c


def _check(ctx, L, R, nb, keys, kinds, lvalid=None, rvalid=None, lcase="none", rcase="none", lsplit=None, rsplit=None,
           hows=HOWS):
    """Indexes both tables (two createIndex calls per side where a split is given: multi-file buckets), runs each outer
    join and compares the row sequences and validity with the oracle's.  Returns {how: (rows, padded left, padded right)}."""
    def build(cols, valids, split, tag):
        if split is None:
            return [_index(ctx, cols, valids, keys, nb, tag, kinds)]
        n = len(next(iter(cols.values())))
        return [_index(ctx, {c: v[a:b] for c, v in cols.items()}, {c: v[a:b] for c, v in (valids or {}).items()}, keys, nb,
                       f"{tag}{j}", kinds) for j, (a, b) in enumerate(((0, split), (split, n)))]

    lres, rres = build(L, lvalid, lsplit, "l"), build(R, rvalid, rsplit, "r")
    lf_, lmask = _filter(lcase, L)
    rf_, rmask = _filter(rcase, R)
    out = {}
    try:
        for how in hows:
            batch, st = _run(ctx, lres, rres, nb, keys, how, lf_, rf_)
            lrow, rrow = JO.outer_join(L, R, nb, keys, keys, how, left_valids=lvalid, right_valids=rvalid, left_mask=lmask,
                                       right_mask=rmask)
            assert batch.num_rows == len(lrow) == st["rows_out"], how
            assert [n for n, _, _ in batch.columns] == ["lid", "s", "rid", "i"]
            _expect_side(batch, ["lid", "s"], L, lrow, how != "left")
            _expect_side(batch, ["rid", "i"], R, rrow, how != "right")
            out[how] = (len(lrow), int((lrow < 0).sum()), int((rrow < 0).sum()))
            batch.free()
    finally:
        for r in lres + rres:
            r.free()
    return out


@pytest.mark.parametrize("nb", [1, 16])
@pytest.mark.parametrize("kind", KINDS)
def test_against_the_oracle(ctx, kind, nb):
    L, R, keys, kinds = _tables(kind, 9_000, 6_000, 1)
    got = _check(ctx, L, R, nb, keys, kinds)
    assert got["left"][2] > 0 and got["right"][1] == 0 and got["full"][1] + got["full"][2] > 0


@pytest.mark.parametrize("kind", KINDS)
def test_nullable_keys(ctx, kind):
    """Nulls in each key column on both sides (a null in a later column sits inside its leading column's group), then in
    every key column at once, then on one side only."""
    L, R, keys, kinds = _tables(kind, 8_000, 6_000, 2)
    rng = np.random.default_rng(3)
    nr = len(R["rid"])
    for pos in range(len(keys)):
        lvalid = {keys[pos]: rng.random(8_000) >= 0.1}
        rvalid = {keys[pos]: rng.random(nr) >= 0.1}
        got = _check(ctx, L, R, 12, keys, kinds, lvalid, rvalid)
        assert got["full"][1] > 0 and got["full"][2] > 0
    lvalid = {k: rng.random(8_000) >= 0.05 for k in keys}
    rvalid = {k: rng.random(nr) >= 0.05 for k in keys}
    _check(ctx, L, R, 12, keys, kinds, lvalid, rvalid)
    _check(ctx, L, R, 12, keys, kinds, lvalid, None)
    _check(ctx, L, R, 12, keys, kinds, None, rvalid)


def test_null_key_against_zero_and_empty_string(ctx):
    for kind, zero in (("i32", 0), ("str", b"")):
        L, R, keys, kinds = _tables(kind, 2_000, 1_000, 4)
        L["a"][:200] = zero
        R["a"][:100] = zero
        lvalid = {"a": np.arange(2_000) >= 100}  # rows 0-99 null, rows 100-199 a real zero
        rvalid = {"a": np.arange(len(R["rid"])) >= 50}
        _check(ctx, L, R, 4, keys, kinds, lvalid, rvalid)


@pytest.mark.parametrize("case", ["pred", "isin", "cmp", "all"])
@pytest.mark.parametrize("kind", ["i64_2", "i32_str", "ts_dec"])
def test_filters_below_either_side(ctx, kind, case):
    L, R, keys, kinds = _tables(kind, 8_000, 6_000, 5)
    rng = np.random.default_rng(6)
    lvalid = {keys[-1]: rng.random(8_000) >= 0.08}
    rvalid = {keys[-1]: rng.random(len(R["rid"])) >= 0.08}
    _check(ctx, L, R, 12, keys, kinds, lvalid, rvalid, lcase=case)
    _check(ctx, L, R, 12, keys, kinds, lvalid, rvalid, rcase=case)
    _check(ctx, L, R, 12, keys, kinds, lvalid, rvalid, lcase=case, rcase=case)


@pytest.mark.parametrize("kind", ["i64_2", "str", "i64_3"])
def test_multi_file_buckets(ctx, kind):
    L, R, keys, kinds = _tables(kind, 9_000, 7_000, 8)
    rng = np.random.default_rng(9)
    lvalid = {keys[-1]: rng.random(9_000) >= 0.1}
    rvalid = {keys[-1]: rng.random(7_000)[:len(R["rid"])] >= 0.1}
    _check(ctx, L, R, 12, keys, kinds, lsplit=5_000)
    _check(ctx, L, R, 12, keys, kinds, rsplit=2_000)
    _check(ctx, L, R, 12, keys, kinds, lvalid, rvalid, lcase="pred", rcase="cmp", lsplit=3_000, rsplit=4_000)


def test_a_right_filter_that_empties_every_bucket(ctx):
    L, R, keys, kinds = _tables("i64_2", 4_000, 3_000, 7)
    none = np.zeros(len(R["rid"]), bool)
    lres, rres = [_index(ctx, L, None, keys, 8, "l", kinds)], [_index(ctx, R, None, keys, 8, "r", kinds)]
    try:
        batch, _ = _run(ctx, lres, rres, 8, keys, "left", rf_=([("i", 5000, False, None, False)], (), ()))
        lrow, rrow = JO.outer_join(L, R, 8, keys, keys, "left", right_mask=none)
        assert batch.num_rows == 4_000 and np.all(rrow == -1)
        assert np.array_equal(batch.column("lid"), L["lid"][lrow])
        _expect_side(batch, ["rid", "i"], R, rrow, True)
        batch.free()
    finally:
        for r in lres + rres:
            r.free()


def test_padded_string_columns(ctx):
    """A padded string is a null of length 0: its offset repeats and its validity is 0; a real empty string is valid."""
    from hyperspace_b200 import _native as N

    L, R, keys, kinds = _tables("i32", 3_000, 2_000, 13)
    L["s"][::7] = b""
    R["a"][:50] = 1_000  # right rows without a left match: their left columns are padded
    lres, rres = [_index(ctx, L, None, keys, 4, "l", kinds)], [_index(ctx, R, None, keys, 4, "r", kinds)]
    lf, lb = _sides(lres)
    rf, rb = _sides(rres)
    lib = N.load_library()
    try:
        for how in ("right", "full"):
            batch, _ = ctx.bucket_join_outer(lf, lb, rf, rb, 4, keys, keys, ["s"], ["rid"], how)
            lrow, _ = JO.outer_join(L, R, 4, keys, keys, how)
            off_p, total = C.c_void_p(), C.c_uint64()
            assert lib.hs_batch_string_offsets(batch._h, 0, C.byref(off_p), C.byref(total)) == N.HS_OK
            offs = np.ctypeslib.as_array((C.c_uint64 * (batch.num_rows + 1)).from_address(off_p.value)).copy()
            pad = lrow < 0
            assert pad.any()
            assert np.all(offs[1:][pad] == offs[:-1][pad])
            (_, d, v), _ = batch.columns
            assert np.array_equal(v.astype(bool), ~pad)
            assert total.value == sum(len(x) for x in L["s"][lrow[~pad]])
            assert any(x == b"" for x in L["s"][lrow[~pad]])
            batch.free()
    finally:
        for r in lres + rres:
            r.free()


def test_device_output(ctx):
    import torch

    from hyperspace_b200 import _native

    L, R, keys, kinds = _tables("i64_3", 6_000, 6_000, 10)
    lres, rres = [_index(ctx, L, None, keys, 12, "l", kinds)], [_index(ctx, R, None, keys, 12, "r", kinds)]
    lib = _native.load_library()
    try:
        for how in HOWS:
            host, _ = _run(ctx, lres, rres, 12, keys, how, lcols=["lid"], rcols=["rid"])
            dev, _ = _run(ctx, lres, rres, 12, keys, how, lcols=["lid"], rcols=["rid"], output=_native.HS_OUT_DEVICE)
            assert dev.on_device and dev.num_rows == host.num_rows > 0
            for i, (name, ty, ptr) in enumerate(dev.device_columns):
                arr = {"shape": (dev.num_rows,), "typestr": "<i8", "data": (ptr, False), "version": 2}
                got = torch.as_tensor(type("D", (), {"__cuda_array_interface__": arr})(), device="cuda").cpu().numpy()
                hn, hd, hv = host.columns[i]
                assert name == hn and ty == _native.HS_TYPE_INT64 and np.array_equal(got, hd)
                nm, t, d = C.c_char_p(), C.c_int32(), C.c_void_p()
                vp = C.c_void_p()
                lib.hs_batch_column(dev._h, i, C.byref(nm), C.byref(t), C.byref(d), C.byref(vp))
                assert (vp.value is not None) == (hv is not None)
                if hv is not None:
                    varr = {"shape": (dev.num_rows,), "typestr": "|u1", "data": (vp.value, False), "version": 2}
                    gv = torch.as_tensor(type("D", (), {"__cuda_array_interface__": varr})(), device="cuda").cpu().numpy()
                    assert np.array_equal(gv, hv)
            host.free()
            dev.free()
    finally:
        for r in lres + rres:
            r.free()


def test_grid_stride_probe(ctx):
    """20 M rows per side, R = rows [N/2, 3N/2) of the synthetic table against L = rows [0, N): k is a bijection of the
    row, so LeftOuter pads exactly rows [0, N/2), RightOuter rows [N, 3N/2), and FullOuter both."""
    from hyperspace_b200 import _native as N
    from oracle import oracle as O

    n, nb = 20_000_000, 64

    def build(first, included):
        src = ctx.synth_table(first, n, 5, n_files=16, row_groups_per_file=2, output=N.HS_OUT_DEVICE)
        idx, _ = ctx.create_index(src.as_sources(), ["k"], included, nb, output=N.HS_OUT_DEVICE, job_uuid="g")
        src.free()
        return idx

    L, R = build(0, ["v1"]), build(n // 2, ["v3"])
    lf, lb, rf, rb = L.as_sources(), [f.bucket for f in L.files], R.as_sources(), [f.bucket for f in R.files]
    try:
        for how, nrows in (("left", n), ("right", n), ("full", n + n // 2)):
            batch, st = ctx.bucket_join_outer(lf, lb, rf, rb, nb, ["k"], ["k"], ["k", "v1"], ["k", "v3"], how)
            (_, lk, lv), (_, lv1, _), (_, rk, rv), (_, rv2, _) = batch.columns
            lk, rk = lk.copy(), rk.copy()
            lvalid = np.ones(len(lk), bool) if lv is None else lv.astype(bool)
            rvalid = np.ones(len(rk), bool) if rv is None else rv.astype(bool)
            lsum = int(lv1.astype(np.int64)[lvalid].sum())
            rsum = int(rv2.astype(np.int64)[rvalid].sum())
            batch.free()
            assert len(lk) == nrows == st["rows_out"]
            both = lvalid & rvalid
            assert np.array_equal(lk[both], rk[both]) and both.sum() == n // 2
            want_l = O.synthetic_rows_at(np.arange(0, n))
            want_r = O.synthetic_rows_at(np.arange(n // 2, n // 2 + n))
            if how != "right":
                assert lvalid.sum() == n and np.array_equal(np.sort(lk[lvalid]), np.sort(want_l["k"]))
                assert lsum == int(want_l["v1"].astype(np.int64).sum())
            if how != "left":
                assert rvalid.sum() == n and np.array_equal(np.sort(rk[rvalid]), np.sort(want_r["k"]))
                assert rsum == int(want_r["v3"].astype(np.int64).sum())
            key = np.where(lvalid, lk, rk)
            b = O.np_pmod(O.np_hash_long(key), nb)
            assert np.all(np.diff(b) >= 0)  # bucket-major
    finally:
        L.free()
        R.free()
        ctx.trim()


# ---- the kernels a call launches ---------------------------------------------------------------------------------------

def _profile(ctx):
    return {k: v["launches"] for k, v in ctx.profile_report().items()}


def test_launched_kernels(ctx):
    L, R, keys, kinds = _tables("i32_str", 6_000, 5_000, 11)
    rng = np.random.default_rng(12)
    lvalid = {"b": rng.random(6_000) >= 0.1}
    rvalid = {"b": rng.random(len(R["rid"])) >= 0.1}
    lres, rres = [_index(ctx, L, lvalid, keys, 12, "l", kinds)], [_index(ctx, R, rvalid, keys, 12, "r", kinds)]
    clean_l, clean_r = [_index(ctx, L, None, keys, 12, "cl", kinds)], [_index(ctx, R, None, keys, 12, "cr", kinds)]
    lf, lb = _sides(lres)
    rf, rb = _sides(rres)
    ctx.profile_enable(True)
    ctx.profile_report()
    try:
        for how in HOWS:
            b, _ = ctx.bucket_join_outer(lf, lb, rf, rb, 12, keys, keys, ["lid", "s"], ["rid", "s"], how)
            prof = _profile(ctx)
            assert prof.get("k_join_count_outer") == 1 and prof.get("k_join_emit_outer") == 1, prof
            assert "k_join_count" not in prof and "k_join_emit" not in prof, prof
            assert prof.get("k_join_exists", 0) == (how == "full") and prof.get("k_join_place_unmatched", 0) == (how == "full"), prof
            # nullable keys: the null-supplying side gets IS NOT NULL, FullOuter one per side for its searched positions
            assert prof.get("k_predicate_mask") == (2 if how == "full" else 1), prof
            b.free()
        # a preserved side with no filter and no null keys launches no mask kernel
        cf, cb = _sides(clean_l)
        crf, crb = _sides(clean_r)
        for how in HOWS:
            b, _ = ctx.bucket_join_outer(cf, cb, crf, crb, 12, keys, keys, ["lid"], ["rid"], how)
            prof = _profile(ctx)
            assert "k_predicate_mask" not in prof and prof.get("k_join_count_outer") == 1, prof
            b.free()
        # inner, semi and anti launch what they launched before
        b, _ = ctx.bucket_join_where(lf, lb, rf, rb, 12, keys, keys, ["lid", "s"], ["rid"])
        prof = _profile(ctx)
        assert prof.get("k_join_count") == 1 and prof.get("k_join_emit") == 1 and not any("outer" in k or "padded" in k for k in prof), prof
        b.free()
        for how in ("semi", "anti"):
            b, _ = ctx.bucket_join_exists(lf, lb, rf, rb, 12, keys, keys, ["lid", "s"], how)
            prof = _profile(ctx)
            assert prof.get("k_join_exists") == 1 and "k_join_count" not in prof and not any("outer" in k or "padded" in k for k in prof), prof
            b.free()
    finally:
        ctx.profile_enable(False)
        for r in lres + rres + clean_l + clean_r:
            r.free()


# ---- refusals ----------------------------------------------------------------------------------------------------------

def test_refusals(ctx):
    from hyperspace_b200 import _native as N

    n = 100
    cols = {"k0": np.arange(n, dtype=np.int64), "k1": np.arange(n, dtype=np.int64), "i32": np.arange(n, dtype=np.int32),
            "f": np.arange(n, dtype=np.float32), "d": np.arange(n, dtype=np.float64), "b": np.arange(n) % 2 == 0,
            "lid": np.arange(n, dtype=np.int64)}
    f, b = _raw_side(cols)

    def both(lkeys, rkeys, how):
        with pytest.raises(N.HyperspaceGpuError) as want:
            ctx.bucket_join_where(f, b, f, b, 1, lkeys, rkeys, ["lid"], ["lid"])
        with pytest.raises(N.HyperspaceGpuError) as got:
            ctx.bucket_join_outer(f, b, f, b, 1, lkeys, rkeys, ["lid"], ["lid"], how)
        assert (got.value.code, got.value.message) == (want.value.code, want.value.message)
        return got.value

    for how in HOWS:
        for key in ("f", "d", "b"):
            assert both([key], [key], how).code == N.HS_EUNSUPPORTED
            assert both(["k0", key], ["k0", key], how).code == N.HS_EUNSUPPORTED
        e = both(["i32"], ["k0"], how)
        assert e.code == N.HS_EUNSUPPORTED and "different types" in e.message
        e = both(["k0", "k1"], ["k0", "i32"], how)
        assert e.code == N.HS_EUNSUPPORTED and "different types" in e.message
        assert both([], [], how).code == N.HS_EINVAL
        assert both([f"k{i % 2}" for i in range(9)], [f"k{i % 2}" for i in range(9)], how).code == N.HS_EUNSUPPORTED
    for jt in (0, 1, 2, 6, -1):
        with pytest.raises(N.HyperspaceGpuError) as e:
            ctx.bucket_join_outer(f, b, f, b, 1, ["k0"], ["k0"], ["lid"], ["lid"], jt)
        assert e.value.code == N.HS_EINVAL and "join_type" in e.value.message
    for jt in (3, 4, 5):  # the outer types stay outside hs_bucket_join_exists
        with pytest.raises(N.HyperspaceGpuError) as e:
            ctx.bucket_join_exists(f, b, f, b, 1, ["k0"], ["k0"], ["lid"], jt)
        assert e.value.code == N.HS_EINVAL and "join_type" in e.value.message
    with pytest.raises(ValueError):
        ctx.bucket_join_outer(f, b, f, b, 1, ["k0"], ["k0"], ["lid"], ["lid"], "outer")
    # either projection may be empty
    for lc, rc in (([], ["lid"]), (["lid"], []), ([], [])):
        batch, st = ctx.bucket_join_outer(f, b, f, b, 1, ["k0"], ["k0"], lc, rc, "full")
        assert batch.num_rows == n == st["rows_out"] and len(batch.columns) == len(lc) + len(rc)
        batch.free()


# ---- through the Hyperspace API ----------------------------------------------------------------------------------------

@pytest.fixture()
def env(tmp_path):
    from hyperspace_b200.hyperspace import Hyperspace
    from hyperspace_b200.session import HyperspaceSession

    s = HyperspaceSession({"spark.hyperspace.system.path": str(tmp_path / "indexes"), "spark.hyperspace.index.numBuckets": "8"})
    yield s, Hyperspace(s), tmp_path
    s.stop()


def _outer(a, b, pairs, how):
    from hyperspace_b200.session import DataFrame, JoinNode

    return DataFrame(a.session, JoinNode(a.plan, b.plan, pairs, how))


def _rows(res, cols):
    """The result rows as tuples, a masked (null) value as None."""
    def values(c):
        a = res[c]
        if isinstance(a, np.ma.MaskedArray):
            return [None if m else v for v, m in zip(np.asarray(a.data).tolist(), np.ma.getmaskarray(a).tolist())]
        return np.asarray(a).tolist()

    return sorted(zip(*[values(c) for c in cols]), key=repr)


def _both_ways(s, q, cols):
    s.disableHyperspace()
    base = q.collect()
    s.enableHyperspace()
    plan = q.explain()
    got = q.collect()
    assert _rows(got, cols) == _rows(base, cols)
    return got, plan


def test_q13_shaped_left_outer_join(env):
    """TPC-H Q13's join: customer LEFT OUTER JOIN orders ON c_custkey = o_custkey AND o_comment NOT LIKE
    '%special%requests%', the NOT LIKE below the orders side."""
    from hyperspace_b200.index_config import IndexConfig
    from hyperspace_b200.session import ProjectNode, DataFrame, col

    s, hs, tmp = env
    rng = np.random.default_rng(1)
    nc, no = 1_500, 12_000
    cust = {"c_custkey": np.arange(nc, dtype=np.int64), "c_name": np.array([f"Customer#{i:09d}" for i in range(nc)])}
    words = ["special requests", "special packages requests", "regular deposits", "pending requests", "special"]
    orders = {"o_orderkey": np.arange(no, dtype=np.int64), "o_custkey": (rng.integers(0, nc // 3, no) * 3).astype(np.int64),
              "o_comment": np.array([f"x {words[i]} y" for i in rng.integers(0, len(words), no)])}
    _write(tmp / "customer", "a.parquet", cust)
    _write(tmp / "orders", "a.parquet", orders)
    c, o = s.read.parquet(str(tmp / "customer")), s.read.parquet(str(tmp / "orders"))
    hs.createIndex(c, IndexConfig("custIdx", ["c_custkey"], ["c_name"]))
    hs.createIndex(o, IndexConfig("ordCustIdx", ["o_custkey"], ["o_orderkey", "o_comment"]))
    j = _outer(c, o.filter(~col("o_comment").like("%special%requests%")), [("c_custkey", "o_custkey")], "leftouter")
    q = DataFrame(s, ProjectNode(j.plan, ["c_custkey", "o_orderkey"]))
    got, plan = _both_ways(s, q, ["c_custkey", "o_orderkey"])
    assert "Name: custIdx" in plan and "Name: ordCustIdx" in plan and "joinType=LeftOuter" in plan
    import re

    keep = [not re.search("special.*requests", t) for t in orders["o_comment"].tolist()]
    by_cust = {}
    for k, ok_, ck in zip(orders["o_orderkey"].tolist(), keep, orders["o_custkey"].tolist()):
        if ok_:
            by_cust.setdefault(ck, []).append(k)
    want = sorted(((ck, ok_) for ck in range(nc) for ok_ in (by_cust.get(ck) or [None])), key=repr)
    assert _rows(got, ["c_custkey", "o_orderkey"]) == want
    assert isinstance(got["o_orderkey"], np.ma.MaskedArray) and np.ma.getmaskarray(got["o_orderkey"]).any()
    assert not isinstance(got["c_custkey"], np.ma.MaskedArray)
    # Q13's count per customer: customers without qualifying orders count 0
    counts = {}
    for ck, ok_ in _rows(got, ["c_custkey", "o_orderkey"]):
        counts[ck] = counts.get(ck, 0) + (ok_ is not None)
    assert sum(1 for v in counts.values() if v == 0) > nc // 2 and len(counts) == nc


def test_full_outer_with_unmatched_rows_on_both_sides(env):
    from hyperspace_b200.index_config import IndexConfig
    from hyperspace_b200.session import col

    s, hs, tmp = env
    rng = np.random.default_rng(2)
    a = {"ak": rng.integers(0, 600, 3_000).astype(np.int64), "ax": np.arange(3_000, dtype=np.int64),
         "as": np.array([f"a{i}" for i in range(3_000)])}
    null = rng.random(2_000) < 0.05
    bk = rng.integers(300, 900, 2_000).astype(np.int64)
    b = {"bk": pa.array(bk, mask=null), "by": pa.array(np.arange(2_000, dtype=np.int64))}
    _write(tmp / "a", "a.parquet", a)
    _write(tmp / "b", "a.parquet", b)
    A, B = s.read.parquet(str(tmp / "a")), s.read.parquet(str(tmp / "b"))
    hs.createIndex(A, IndexConfig("aIdx", ["ak"], ["ax", "as"]))
    hs.createIndex(B, IndexConfig("bIdx", ["bk"], ["by"]))
    q = _outer(A.filter(col("ax") >= 100), B, [("ak", "bk")], "fullouter")
    cols = ["ak", "ax", "as", "bk", "by"]
    got, plan = _both_ways(s, q, cols)
    assert "Name: aIdx" in plan and "Name: bIdx" in plan and "joinType=FullOuter" in plan
    assert list(got) == cols and all(isinstance(got[c], np.ma.MaskedArray) for c in cols)
    arows = [(k, x, t) for k, x, t in zip(a["ak"].tolist(), a["ax"].tolist(), a["as"].tolist()) if x >= 100]
    brows = [(None if null[i] else int(bk[i]), i) for i in range(2_000)]
    want, bmatched = [], set()
    for k, x, t in arows:
        m = [(bk_, y) for bk_, y in brows if bk_ == k]
        bmatched |= {y for _, y in m}
        want += [(k, x, t, bk_, y) for bk_, y in m] or [(k, x, t, None, None)]
    want += [(None, None, None, bk_, y) for bk_, y in brows if y not in bmatched]
    assert _rows(got, cols) == sorted(want, key=repr)
    assert any(r[0] is None for r in want) and any(r[3] is None for r in want) and any(r[0] is None and r[3] is None for r in want)


def test_hybrid_scan_with_appended_files_on_each_side(env):
    from hyperspace_b200.index_config import IndexConfig
    from hyperspace_b200.session import DataFrame, ProjectNode, col

    s, hs, tmp = env
    rng = np.random.default_rng(5)

    def part(first, n):
        return ({"lk": np.arange(first, first + n, dtype=np.int64), "lv": rng.integers(0, 100, n).astype(np.int64)},
                {"rk": rng.integers(first // 2, first + n, n).astype(np.int64), "rv": rng.integers(0, 100, n).astype(np.int64)})

    (l1, r1), (l2, r2) = part(0, 3_000), part(3_000, 600)
    _write(tmp / "l", "a.parquet", l1)
    _write(tmp / "r", "a.parquet", r1)
    Lf, Rf = s.read.parquet(str(tmp / "l")), s.read.parquet(str(tmp / "r"))
    hs.createIndex(Lf, IndexConfig("li", ["lk"], ["lv"]))
    hs.createIndex(Rf, IndexConfig("ri", ["rk"], ["rv"]))
    _write(tmp / "l", "b.parquet", l2)
    _write(tmp / "r", "b.parquet", r2)
    s.conf.set("spark.hyperspace.index.hybridscan.enabled", True)
    s.conf.set("spark.hyperspace.index.hybridscan.maxAppendedRatio", "0.9")
    Lf, Rf = s.read.parquet(str(tmp / "l")), s.read.parquet(str(tmp / "r"))
    L = {c: np.concatenate([l1[c], l2[c]]) for c in l1}
    R = {c: np.concatenate([r1[c], r2[c]]) for c in r1}
    for how, name in (("leftouter", "LeftOuter"), ("rightouter", "RightOuter"), ("fullouter", "FullOuter")):
        j = _outer(Lf.filter(col("lv") >= 20), Rf.filter(col("rv") < 80), [("lk", "rk")], how)
        q = DataFrame(s, ProjectNode(j.plan, ["lk", "lv", "rk", "rv"]))
        got, plan = _both_ways(s, q, ["lk", "lv", "rk", "rv"])
        assert "Name: li" in plan and "Name: ri" in plan and f"joinType={name}" in plan
        ls = [(k, v) for k, v in zip(L["lk"].tolist(), L["lv"].tolist()) if v >= 20]
        rs = [(k, v) for k, v in zip(R["rk"].tolist(), R["rv"].tolist()) if v < 80]
        rby = {}
        for k, v in rs:
            rby.setdefault(k, []).append(v)
        want = []
        if how != "rightouter":
            want += [(k, v, k, w) for k, v in ls for w in rby.get(k, [])]
            want += [(k, v, None, None) for k, v in ls if k not in rby]
        if how != "leftouter":
            lkeys = {k for k, _ in ls}
            if how == "rightouter":
                want += [(k, v, k, w) for k, v in ls for w in rby.get(k, [])]
            want += [(None, None, k, w) for k, w in rs if k not in lkeys]
        assert _rows(got, ["lk", "lv", "rk", "rv"]) == sorted(want, key=repr) and want
