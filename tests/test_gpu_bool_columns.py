"""Boolean included columns on the GPU: index pages against the numpy restatement (bool_pages.py) and the CPU oracle, build
invariance, PLAIN and RLE boolean sources, the read side over the new indexes, and the refusals."""
import os

import numpy as np
import pyarrow as pa
import pyarrow.parquet as pq
import pytest

import bool_pages as B
import parquet_shapes as S
from oracle import oracle as O

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    from hyperspace_b200 import _native

    c = _native.Context(0)
    yield c
    c.close()


def _table(n, seed, *, bool_cols=(("b1", 0.0), ("b2", 0.1)), key=None, extra=True, valid_of=None):
    """k (int64 key) plus boolean columns (name, null fraction), and int / double / string / decimal / dictionary columns."""
    rng = np.random.default_rng(seed)
    cols = {"k": pa.array(key if key is not None else rng.integers(0, max(1, n // 3), n, dtype=np.int64))}
    for name, nf in bool_cols:
        v = rng.random(n) < 0.5
        valid = valid_of[name] if valid_of and name in valid_of else (rng.random(n) >= nf if nf else None)
        cols[name] = pa.array(v, mask=None if valid is None else ~valid)
    if extra:
        cols["i"] = pa.array(rng.integers(-1000, 1000, n, dtype=np.int32))
        cols["d"] = pa.array(rng.random(n))
        cols["s"] = pa.array([f"s{x}" for x in rng.integers(0, 50, n)])
        cols["dec"] = pa.array([None if x % 7 == 0 else int(x) for x in rng.integers(0, 10**6, n)], pa.decimal128(10, 2)).cast(pa.decimal128(10, 2))
        for j in range(5):  # low-cardinality: dictionary-encoded at the source, carried through the build
            cols[f"c{j}"] = pa.array(rng.integers(0, 5 + j, n, dtype=np.int64))
    return pa.table(cols)


def _np(table):
    cols, valid = {}, {}
    for name in table.column_names:
        c = table.column(name).combine_chunks()
        if pa.types.is_string(c.type):
            cols[name] = np.array([x or "" for x in c.to_pylist()], dtype=object)
        elif pa.types.is_decimal(c.type):
            cols[name] = np.array([0 if x is None else int(x.scaleb(2)) for x in c.to_pylist()], dtype=np.int64)
        else:
            cols[name] = c.fill_null(False if pa.types.is_boolean(c.type) else 0).to_numpy(zero_copy_only=False)
        if c.null_count:
            valid[name] = np.asarray(c.is_valid())
    return cols, valid


def _images(tmp_path, tables, **kw):
    from hyperspace_b200 import _native

    out = []
    for i, t in enumerate(tables):
        p = str(tmp_path / f"src{i}_{abs(hash(str(kw))) % 1000}.parquet")
        pq.write_table(t, p, **kw)
        out.append(_native.FileImage(path=p))
    return out


def _build(ctx, files, indexed, included, nb, **kw):
    from hyperspace_b200 import _native

    res, st = ctx.create_index(files, indexed, included, nb, output=_native.HS_OUT_HOST, job_uuid="bool", **kw)
    out = {f.bucket: res.host_bytes(i) for i, f in enumerate(res.files)}
    res.free()
    return out, st


def _check(files_by_bucket, table, indexed, included, nb, rows_per_page=131072):
    """Every bucket file against the oracle row by row; every boolean page body byte for byte against the restatement."""
    cols, valid = _np(table)
    perm, offs, order = O.index_rows(cols, indexed, included, nb, valids=valid or None)
    for b in range(nb):
        lo, hi = int(offs[b]), int(offs[b + 1])
        if lo == hi:
            assert b not in files_by_bucket
            continue
        img = files_by_bucket[b]
        t = pq.ParquetFile(pa.BufferReader(img)).read()
        assert t.column_names == order
        rows = perm[lo:hi]
        for name in order:
            got = t.column(name).combine_chunks()
            if name in valid:
                assert np.array_equal(np.asarray(got.is_valid()), valid[name][rows]), (name, b)
            if pa.types.is_boolean(got.type):
                ok = np.asarray(got.is_valid())
                assert np.array_equal(got.fill_null(False).to_numpy(zero_copy_only=False)[ok], cols[name][rows][ok]), (name, b)
                pages = B.data_pages(img, name)
                vv = valid.get(name)
                want = B.page_bodies(cols[name][rows], None if vv is None else vv[rows], rows_per_page)
                assert [p["body"] for p in pages] == want, (name, b)
                assert all(p["enc"] == S.PLAIN for p in pages)
    return perm, offs, order


def test_create_index_against_the_oracle(ctx, tmp_path):
    t = _table(60_000, 1)
    inc = [c for c in t.column_names if c != "k"]
    files = _images(tmp_path, [t.slice(0, 30_000), t.slice(30_000)], compression="snappy")
    out, st = _build(ctx, files, ["k"], inc, 16)
    _check(out, t, ["k"], inc, 16)
    md = pq.ParquetFile(pa.BufferReader(next(iter(out.values())))).metadata
    assert b'"name":"b1","type":"boolean"' in md.metadata[b"org.apache.spark.sql.parquet.row.metadata"]
    leaf = md.schema.column(1)
    assert leaf.physical_type == "BOOLEAN" and leaf.converted_type == "NONE" and leaf.max_definition_level == 1
    assert md.row_group(0).column(1).statistics is None or not md.row_group(0).column(1).statistics.has_min_max


@pytest.mark.parametrize("case", ["null_free", "nullable", "all_null", "no_nulls_in_a_file"])
def test_null_shapes(ctx, tmp_path, case):
    n = 20_000
    rng = np.random.default_rng(3)
    vo = {"null_free": {}, "nullable": {"b1": rng.random(n) >= 0.5}, "all_null": {"b1": np.zeros(n, bool)},
          "no_nulls_in_a_file": {"b1": np.concatenate([np.ones(n // 2, bool), rng.random(n - n // 2) >= 0.3])}}[case]
    t = _table(n, 4, bool_cols=(("b1", 0.0), ("b3", 0.0)), valid_of=vo, extra=False)
    files = _images(tmp_path, [t.slice(0, n // 2), t.slice(n // 2)])
    out, _ = _build(ctx, files, ["k"], ["b1", "b3"], 8)
    _check(out, t, ["k"], ["b1", "b3"], 8)


@pytest.mark.parametrize("rows", [0, 1, 7, 8, 9, 4095, 4096, 4097])
@pytest.mark.parametrize("nullable", [False, True])
def test_bucket_sizes(ctx, tmp_path, rows, nullable):
    t = _table(rows, rows + 10, bool_cols=(("b1", 0.3 if nullable else 0.0),), key=np.arange(rows, dtype=np.int64), extra=False)
    out, _ = _build(ctx, _images(tmp_path, [t]), ["k"], ["b1"], 1)
    _check(out, t, ["k"], ["b1"], 1)


@pytest.mark.parametrize("P", [4096, 8192])
@pytest.mark.parametrize("delta", [-1, 0, 1])
def test_pages(ctx, tmp_path, P, delta):
    n = 3 * P + delta
    t = _table(n, P + delta, bool_cols=(("b1", 0.0), ("b2", 0.25)), key=np.arange(n, dtype=np.int64), extra=False)
    out, _ = _build(ctx, _images(tmp_path, [t]), ["k"], ["b1", "b2"], 1, rows_per_page=P)
    _check(out, t, ["k"], ["b1", "b2"], 1, rows_per_page=P)


def test_tile_boundaries_at_every_bit_offset(ctx, tmp_path):
    """4001 non-null rows per 4096-row tile: the value bits of tile t start at bit 4001 t, i.e. at every offset mod 8."""
    n = 9 * 4096 + 100
    rng = np.random.default_rng(5)
    valid = np.zeros(n, bool)
    for t0 in range(0, n, 4096):
        m = min(4096, n - t0)
        valid[t0 + rng.choice(m, min(4001, m), replace=False)] = True
    t = _table(n, 6, bool_cols=(("b1", 0.0),), key=np.arange(n, dtype=np.int64), valid_of={"b1": valid}, extra=False)
    out, _ = _build(ctx, _images(tmp_path, [t]), ["k"], ["b1"], 1)
    _check(out, t, ["k"], ["b1"], 1)


def test_invariance_codecs_and_verify(ctx, tmp_path, monkeypatch):
    from hyperspace_b200 import _native

    t = _table(50_000, 7)
    inc = [c for c in t.column_names if c != "k"]
    files = _images(tmp_path, [t.slice(0, 25_000), t.slice(25_000)])
    a, _ = _build(ctx, files, ["k"], inc, 8)
    b, _ = _build(ctx, files, ["k"], inc, 8)
    assert a == b
    for var in ("HS_NO_CARRY", "HS_NO_ZEROCOPY"):
        monkeypatch.setenv(var, "1")
        c, _ = _build(ctx, files, ["k"], inc, 8)
        monkeypatch.delenv(var)
        assert c == a, var
    for codec in (_native.HS_CODEC_SNAPPY, _native.HS_CODEC_GZIP, _native.HS_CODEC_LZ4):
        c, _ = _build(ctx, files, ["k"], inc, 8, compression=codec)
        for bk in a:
            for name in ("b1", "b2"):
                if codec == _native.HS_CODEC_LZ4:
                    import page_encoder_cases as PE

                    got = [p["body"] for p in PE.walk(c[bk])[1] if p["col"] == name]
                else:
                    got = [p["body"] for p in B.data_pages(c[bk], name)]
                assert got == [p["body"] for p in B.data_pages(a[bk], name)], (codec, bk, name)
    for bk, img in a.items():
        rep = ctx.verify_index([_native.FileImage(data=np.frombuffer(img, np.uint8))], [bk], ["k"], ["b1", "b2", "i", "d"], 8)
        assert rep["rows"] == pq.ParquetFile(pa.BufferReader(img)).metadata.num_rows
        assert rep["bucket_mismatches"] == 0 and rep["order_violations"] == 0


@pytest.mark.parametrize("version", ["1.0", "2.0"])
@pytest.mark.parametrize("codec", ["NONE", "SNAPPY"])
@pytest.mark.parametrize("nulls", [0.0, 0.15])
def test_plain_and_rle_sources_give_identical_indexes(ctx, tmp_path, version, codec, nulls):
    t = _table(40_000, 8, bool_cols=(("b1", nulls), ("b2", 0.1)), extra=False)
    outs = []
    for enc in ("PLAIN", "RLE"):
        files = _images(tmp_path, [t.slice(0, 20_000), t.slice(20_000)], use_dictionary=False, compression=codec,
                        data_page_version=version, column_encoding={"b1": enc, "b2": enc, "k": "PLAIN"}, data_page_size=1 << 13)
        outs.append(_build(ctx, files, ["k"], ["b1", "b2"], 8)[0])
    assert outs[0] == outs[1]
    _check(outs[1], t, ["k"], ["b1", "b2"], 8)


def _rle_file(tmp_path, name, bool_bytes, ptype=S.BOOLEAN):
    """A 64-row file: k = 0..63 and one required column whose single page has encoding RLE and body `bool_bytes`."""
    from hyperspace_b200 import _native

    n = len(bool_bytes) * 8
    vals = np.unpackbits(np.frombuffer(bool_bytes, np.uint8), bitorder="little") if ptype == S.BOOLEAN else \
        np.frombuffer(bool_bytes, np.int64)
    n = len(vals)
    spec = S.FileSpec([S.Col("k", S.INT64, False, [S.Chunk([S.Page(rows=n, values=np.arange(n, dtype=np.int64))])]),
                       S.Col("b", ptype, False, [S.Chunk([S.Page(rows=n, enc=S.RLE, values=vals)])])])
    img = S.write_file(spec)
    img = img[0] if isinstance(img, tuple) else img
    p = str(tmp_path / name)
    open(p, "wb").write(bytes(img))
    return [_native.FileImage(path=p)]


def test_damaged_rle_pages_are_refused(ctx, tmp_path):
    from hyperspace_b200 import _native

    good = (4).to_bytes(4, "little") + bytes([0x80, 0x01, 0x01, 0x00])  # one RLE run of 64 trues
    out, _ = _build(ctx, _rle_file(tmp_path, "good.parquet", good), ["k"], ["b"], 1)
    assert pq.ParquetFile(pa.BufferReader(out[0])).read().column("b").to_pylist() == [True] * 64
    cases = {"truncated_length": bytes([4, 0]),
             "length_past_the_page": (100).to_bytes(4, "little") + bytes([0x80, 0x01, 0x01, 0x00]),
             "run_past_the_page": (4).to_bytes(4, "little") + bytes([(10 << 1) | 1, 0xff, 0xff, 0xff])}
    for name, body in cases.items():
        with pytest.raises(_native.HyperspaceGpuError) as e:
            _build(ctx, _rle_file(tmp_path, name + ".parquet", body), ["k"], ["b"], 1)
        assert e.value.code == _native.HS_EFORMAT, name
    with pytest.raises(_native.HyperspaceGpuError) as e:
        _build(ctx, _rle_file(tmp_path, "int64.parquet", np.arange(8, dtype=np.int64).tobytes(), S.INT64), ["k"], ["b"], 1)
    assert e.value.code == _native.HS_EUNSUPPORTED


def test_filter_scan_and_joins_project_booleans(ctx, tmp_path):
    from hyperspace_b200 import _native

    nb = 8
    L = _table(30_000, 9, bool_cols=(("lb", 0.0), ("ln", 0.2)), extra=False)
    R = _table(20_000, 10, bool_cols=(("rb", 0.0), ("rn", 0.3)), extra=False)
    li, _ = _build(ctx, _images(tmp_path, [L]), ["k"], ["lb", "ln"], nb)
    ri, _ = _build(ctx, _images(tmp_path, [R]), ["k"], ["rb", "rn"], nb)
    lf = [_native.FileImage(data=np.frombuffer(v, np.uint8)) for v in li.values()]
    rf = [_native.FileImage(data=np.frombuffer(v, np.uint8)) for v in ri.values()]
    lc, lv = _np(L)
    rc, rv = _np(R)
    # filter scan: k <= 2000, projecting both booleans
    batch, _ = ctx.filter_scan_where(lf, "k", ["k", "lb", "ln"], [("k", None, False, 2000, False)])
    sel = lc["k"] <= 2000
    want = sorted(zip(lc["k"][sel].tolist(), lc["lb"][sel].tolist(), np.where(lv["ln"][sel], lc["ln"][sel], 2).tolist()))
    got_ln = np.where(batch.columns[2][2].astype(bool), batch.column("ln"), 2)
    got = sorted(zip(batch.column("k").tolist(), batch.column("lb").astype(bool).tolist(), got_ln.tolist()))
    assert got == want
    batch.free()
    lb, rb = list(li.keys()), list(ri.keys())

    def rows(batch):
        out = []
        for name, d, v in batch.columns:
            out.append([None if v is not None and not v[i] else int(d[i]) for i in range(batch.num_rows)])
        return sorted(zip(*out), key=lambda r: tuple((x is None, x) for x in r))

    def oracle(how):
        ri_by_k = {}
        for j, k in enumerate(rc["k"].tolist()):
            ri_by_k.setdefault(k, []).append(j)
        lval = lambda i: (int(lc["lb"][i]), int(lc["ln"][i]) if lv["ln"][i] else None)
        rval = lambda j: (int(rc["rb"][j]), int(rc["rn"][j]) if rv["rn"][j] else None)
        out, matched = [], set()
        for i, k in enumerate(lc["k"].tolist()):
            js = ri_by_k.get(k, [])
            if how in ("inner", "left", "full"):
                out += [lval(i) + rval(j) for j in js]
                matched.update(js)
                if not js and how in ("left", "full"):
                    out.append(lval(i) + (None, None))
            elif how == "semi" and js:
                out.append(lval(i))
            elif how == "anti" and not js:
                out.append(lval(i))
        if how == "full":
            out += [(None, None) + rval(j) for j in range(len(rc["k"])) if j not in matched]
        if how == "right":
            for j, k in enumerate(rc["k"].tolist()):
                is_ = [i for i in np.flatnonzero(lc["k"] == k)]
                out += [lval(i) + rval(j) for i in is_] or [(None, None) + rval(j)]
        return sorted(out, key=lambda r: tuple((x is None, x) for x in r))

    args = (lf, lb, rf, rb, nb, ["k"], ["k"])
    b, _ = ctx.bucket_join(lf, lb, rf, rb, nb, "k", "k", ["lb", "ln"], ["rb", "rn"])
    assert rows(b) == oracle("inner")
    for how in ("semi", "anti"):
        b, _ = ctx.bucket_join_exists(*args, ["lb", "ln"], join_type=how)
        assert rows(b) == oracle(how), how
    for how in ("left", "right", "full"):
        b, _ = ctx.bucket_join_outer(*args, ["lb", "ln"], ["rb", "rn"], join_type=how)
        assert rows(b) == oracle(how), how


@pytest.mark.parametrize("indexed", [["b1"], ["k", "b1"]])
def test_boolean_indexed_column_refused(ctx, tmp_path, indexed):
    from hyperspace_b200 import _native

    t = _table(1000, 11, extra=False)
    out_dir = tmp_path / "out"
    with pytest.raises(_native.HyperspaceGpuError) as e:
        ctx.create_index(_images(tmp_path, [t]), indexed, ["b2"], 4, out_dir=str(out_dir), output=_native.HS_OUT_FILES)
    assert e.value.code == _native.HS_EUNSUPPORTED and "'b1'" in e.value.message and "not indexed" in e.value.message
    assert not out_dir.exists() or not os.listdir(out_dir)


def test_launches(ctx, tmp_path):
    t = _table(30_000, 12, bool_cols=(("b1", 0.0), ("b2", 0.2)), extra=False)
    plain = t.drop(["b1", "b2"]).append_column("v", pa.array(np.arange(30_000, dtype=np.int64)))
    new = {"k_gather_encode_bool", "k_gather_encode_bool_nullable"}
    ctx.profile_enable(True)
    try:
        ctx.profile_report()
        _build(ctx, _images(tmp_path, [plain]), ["k"], ["v"], 8)
        without = set(ctx.profile_report())
        _build(ctx, _images(tmp_path, [t]), ["k"], ["b1", "b2"], 8)
        with_bools = set(ctx.profile_report())
    finally:
        ctx.profile_enable(False)
    assert not (without & new) and new <= with_bools


def test_hyperspace_api_with_boolean_columns(tmp_path):
    from hyperspace_b200.hyperspace import Hyperspace
    from hyperspace_b200.index_config import IndexConfig
    from hyperspace_b200.session import HyperspaceSession, col

    s = HyperspaceSession({"spark.hyperspace.system.path": str(tmp_path / "indexes"), "spark.hyperspace.index.numBuckets": "8"})
    hs = Hyperspace(s)
    os.makedirs(tmp_path / "t")
    tabs = [_table(8000, 20 + i, extra=False) for i in range(4)]
    for i in range(2):
        pq.write_table(tabs[i], str(tmp_path / "t" / f"f{i}.parquet"), compression="snappy")

    def same(q):
        s.disableHyperspace()
        base = q.collect()
        s.enableHyperspace()
        got = q.collect()
        key = lambda r: [np.asarray(r[c]).astype(np.int64) for c in ("k", "b1", "b2")]
        mk = lambda r: sorted(zip(*[x.tolist() for x in key(r)]) if len(r["k"]) else [])
        assert len(got["k"]) == len(base["k"]) and mk(got) == mk(base)
        return got

    hs.createIndex(s.read.parquet(str(tmp_path / "t")), IndexConfig("idx", ["k"], ["b1", "b2"]))
    q = lambda: s.read.parquet(str(tmp_path / "t")).filter(col("k") <= 1000).select("k", "b1", "b2")
    s.enableHyperspace()
    assert "Name: idx" in q().explain()
    same(q())
    pq.write_table(tabs[2], str(tmp_path / "t" / "f2.parquet"))
    hs.refreshIndex("idx", "incremental")
    same(q())
    hs.optimizeIndex("idx", "full")
    same(q())
    pq.write_table(tabs[3], str(tmp_path / "t" / "f3.parquet"), use_dictionary=False, column_encoding={"b1": "RLE", "b2": "RLE"})
    s.conf.set("spark.hyperspace.index.hybridscan.enabled", True)
    assert "hybridScan(appended=1" in q().explain()
    same(q())
    s.stop()
