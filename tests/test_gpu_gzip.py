"""GZIP-compressed Parquet on the GPU: the page decompressor (k_inflate) against zlib on the corpus of tests/gzip_corpus.py,
createIndex over GZIP sources written by pyarrow -- index files byte-identical to those built from the same table written
UNCOMPRESSED and SNAPPY --, codecs mixed in one call, the unsorted scan, and the Hyperspace API over a GZIP lake."""
import decimal
import io
import os

import numpy as np
import pyarrow as pa
import pyarrow.parquet as pq
import pytest

import gzip_corpus as G
from oracle import oracle as O

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    from hyperspace_b200 import _native

    c = _native.Context(0)
    yield c
    c.close()


def _image(table, **kw):
    sink = io.BytesIO()
    pq.write_table(table, sink, **kw)
    return sink.getvalue()


def _files(images):
    from hyperspace_b200 import _native

    return [_native.FileImage(data=img) for img in images]


# ---- the kernel on its own --------------------------------------------------------------------------------------------------
def test_inflate_matches_zlib_on_the_corpus(ctx):
    bad = []
    for name, stream, data in G.valid():
        if ctx.k_inflate(stream, len(data)) != data:
            bad.append(name)
    assert not bad, bad[:10]


def test_damaged_streams_are_format_errors_and_the_context_keeps_working(ctx):
    from hyperspace_b200 import _native as N

    texts = {G.TRUNCATED: "runs past", G.CRC: "CRC-32", G.ISIZE: "ISIZE", G.TRAILING: "trailing", G.BAD_MAGIC: "magic",
             G.BLOCK_TYPE: "block type", G.STORED_LEN: "NLEN", G.BAD_LENGTHS: "code-length", G.FAR_DISTANCE: "before the start",
             G.BAD_SYMBOL: "symbol", G.OUTPUT_OVERRUN: "longer", G.OUTPUT_SHORT: "shorter", G.BAD_METHOD: "method",
             G.BAD_FLAGS: "reserved", G.HEADER_CRC: "CRC-16"}
    for name, stream, n, check in G.damaged():
        with pytest.raises(N.HyperspaceGpuError) as e:
            ctx.k_inflate(stream, n)
        assert e.value.code == N.HS_EFORMAT, name
        assert texts[check] in str(e.value), (name, str(e.value))
    data = b"still working " * 1000
    assert ctx.k_inflate(G.gzip_compress(data), len(data)) == data


# ---- createIndex over GZIP sources ------------------------------------------------------------------------------------------
def _typed_table(n, seed):
    rng = np.random.default_rng(seed)
    nulls = rng.random(n) < 0.1
    base = np.datetime64("2001-02-03T04:05:06", "us").astype(np.int64)
    return pa.table({
        "i32": pa.array(rng.integers(-5000, 5000, n, dtype=np.int32), mask=nulls),
        "i64": pa.array(rng.integers(-2**40, 2**40, n, dtype=np.int64)),
        "f32": pa.array((rng.integers(0, 1000, n) * 0.25).astype(np.float32)),
        "f64": pa.array(rng.normal(size=n)),
        "s": pa.array([f"key-{v}" for v in rng.integers(0, 3000, n)], mask=rng.random(n) < 0.05),
        "ts": pa.array((base + rng.integers(0, 10**12, n)).astype("datetime64[us]"), pa.timestamp("us")),
        "dec": pa.array([None if m else decimal.Decimal(int(v)).scaleb(-2) for v, m in
                         zip(rng.integers(-10**10, 10**10, n), rng.random(n) < 0.1)], pa.decimal128(12, 2)),
    })


WRITES = {
    "dict_v1": dict(),
    "plain_v1": dict(use_dictionary=False),
    "dict_v2": dict(data_page_version="2.0"),
    "plain_v2_small_pages": dict(use_dictionary=False, data_page_version="2.0", data_page_size=8 << 10),
    "level1": dict(compression_level=1),
    "level9_small_pages": dict(compression_level=9, data_page_size=16 << 10),
}
KEYS = ["i32", "i64", "f32", "f64", "s", "ts", "dec"]


def _build(ctx, images, key, included, nb=8, profile=False):
    from hyperspace_b200 import _native as N

    ctx.profile_enable(profile)
    try:
        res, st = ctx.create_index(_files(images), [key], included, nb, output=N.HS_OUT_HOST, job_uuid="gz")
        kernels = ctx.profile_report() if profile else {}
    finally:
        ctx.profile_enable(False)
    out = [(f.name, f.bucket, res.host_bytes(i)) for i, f in enumerate(res.files)]
    res.free()
    return out, st, kernels


@pytest.mark.parametrize("write", list(WRITES))
@pytest.mark.parametrize("key", KEYS)
def test_gzip_sources_index_like_uncompressed_and_snappy(ctx, monkeypatch, write, key):
    t = _typed_table(30_000, 3)
    kw = WRITES[write]
    imgs = {}
    for c in ("gzip", "none", "snappy"):  # the level only applies to gzip
        kc = dict(kw, use_deprecated_int96_timestamps=True) if c == "gzip" else \
            {k: v for k, v in kw.items() if k != "compression_level"} | {"use_deprecated_int96_timestamps": True}
        imgs[c] = [_image(t.slice(0, 17_000), compression=c, **kc), _image(t.slice(17_000), compression=c, **kc)]
    md = pq.ParquetFile(io.BytesIO(imgs["gzip"][0])).metadata
    assert md.row_group(0).column(0).compression == "GZIP"
    included = [c for c in t.column_names if c != key]
    gz, st_gz, kern = _build(ctx, imgs["gzip"], key, included, profile=True)
    assert "k_inflate" in kern
    plain, st_plain, kern_plain = _build(ctx, imgs["none"], key, included, profile=True)
    assert "k_inflate" not in kern_plain
    snap, _, _ = _build(ctx, imgs["snappy"], key, included)
    assert gz == plain == snap  # the source codec does not leak into the index files
    monkeypatch.setenv("HS_NO_CARRY", "1")
    nc, _, _ = _build(ctx, imgs["gzip"], key, included)
    monkeypatch.delenv("HS_NO_CARRY")
    assert nc == gz
    # every row lands in its Spark bucket, in key order (the engine's own decoder re-reads the files)
    from hyperspace_b200 import _native as N

    rep = ctx.verify_index([N.FileImage(data=d) for _, _, d in gz], [b for _, b, _ in gz], [key], included, 8)
    assert rep["rows"] == t.num_rows and rep["bucket_mismatches"] == 0 and rep["order_violations"] == 0


def test_gzip_index_matches_the_oracle_and_no_inflate_without_gzip(ctx):
    cols = O.synthetic_table(0, 200_000, 5)
    t = pa.table(cols)
    order = ["k", "v1", "v2", "v3", "v4"]
    gz, _, kern = _build(ctx, [_image(t, compression="gzip", data_page_size=64 << 10)], "k", order[1:], nb=16, profile=True)
    perm, offs, oorder = O.index_rows(cols, ["k"], order[1:], 16)
    for _, b, data in gz:
        got = pq.ParquetFile(pa.BufferReader(data)).read()
        for c in oorder:
            assert got.column(c).to_numpy().tobytes() == cols[c][perm[int(offs[b]):int(offs[b + 1])]].tobytes(), (c, b)
    assert kern["k_inflate"]["launches"] == 1
    _, _, kern_snap = _build(ctx, [_image(t, compression="snappy")], "k", order[1:], nb=16, profile=True)
    _, _, kern_none = _build(ctx, [_image(t, compression="none")], "k", order[1:], nb=16, profile=True)
    assert "k_inflate" not in kern_snap and "k_inflate" not in kern_none


def test_all_null_v2_page(ctx):
    n = 5000
    t = pa.table({"k": np.arange(n, dtype=np.int64), "v": pa.nulls(n, pa.int64())})
    a, _, _ = _build(ctx, [_image(t, compression="gzip", data_page_version="2.0")], "k", ["v"])
    b, _, _ = _build(ctx, [_image(t, compression="none", data_page_version="2.0")], "k", ["v"])
    assert a == b
    assert sum(pq.ParquetFile(pa.BufferReader(d)).read().column("v").null_count for _, _, d in a) == n


def test_mixed_codecs_in_one_call(ctx):
    from hyperspace_b200 import _native as N

    cols = O.synthetic_table(0, 90_000, 5)
    t = pa.table(cols)
    parts = [t.slice(0, 30_000), t.slice(30_000, 30_000), t.slice(60_000)]
    mixed = [_image(parts[0], compression="gzip"), _image(parts[1], compression="snappy"),
             _image(parts[2], compression={"k": "gzip", "v1": "snappy", "v2": "none", "v3": "gzip", "v4": "snappy"})]
    plain = [_image(p, compression="none") for p in parts]
    inc = ["v1", "v2", "v3", "v4"]
    a, _, kern = _build(ctx, mixed, "k", inc, profile=True)
    b, _, _ = _build(ctx, plain, "k", inc)
    assert a == b
    assert "k_inflate" in kern and "k_snappy_blocks" in kern
    # a file that mixes GZIP and ZSTD columns is refused, naming the ZSTD column
    bad = _image(parts[0], compression={"k": "gzip", "v1": "gzip", "v2": "zstd", "v3": "gzip", "v4": "gzip"})
    with pytest.raises(N.HyperspaceGpuError) as e:
        ctx.create_index(_files([bad]), ["k"], inc, 4, output=N.HS_OUT_HOST)
    assert e.value.code == N.HS_EUNSUPPORTED and "'v2'" in str(e.value) and "codec 6" in str(e.value)


def test_each_codec_kernel_runs_once_over_mixed_sources(ctx):
    n = 60_000
    rng = np.random.default_rng(11)
    t = pa.table({"k": rng.integers(0, 1 << 40, n, dtype=np.int64),
                  "v": pa.array(rng.integers(0, 1000, n, dtype=np.int64), mask=rng.random(n) < 0.2)})
    parts = [t.slice(0, 20_000), t.slice(20_000, 20_000), t.slice(40_000)]
    # v2 pages keep their (here non-empty) definition levels uncompressed in front of the values: the snappy decoder
    # copies them with a kernel of its own, which runs only when some page needs it.  PLAIN values, so that the pages
    # shrink and pyarrow does store them compressed.
    v2 = _image(parts[0], compression="snappy", data_page_version="2.0", use_dictionary=False)
    v1 = _image(parts[0], compression="snappy", use_dictionary=False)
    rest = [_image(parts[1], compression="gzip"), _image(parts[2], compression="none")]
    plain, _, _ = _build(ctx, [_image(p, compression="none") for p in parts], "k", ["v"])
    a, _, kern = _build(ctx, [v2] + rest, "k", ["v"], profile=True)
    assert a == plain
    assert {k: kern[k]["launches"] for k in kern if k.startswith("k_snappy") or k == "k_inflate"} == \
        {"k_snappy_levels": 1, "k_snappy_index": 1, "k_snappy_blocks": 1, "k_inflate": 1}
    b, _, kern = _build(ctx, [v1] + rest, "k", ["v"], profile=True)
    assert b == plain
    assert {k: kern[k]["launches"] for k in kern if k.startswith("k_snappy") or k == "k_inflate"} == \
        {"k_snappy_index": 1, "k_snappy_blocks": 1, "k_inflate": 1}
    _, _, kern = _build(ctx, rest, "k", ["v"], profile=True)
    assert [k for k in kern if k.startswith("k_snappy")] == [] and kern["k_inflate"]["launches"] == 1


def test_corrupt_gzip_page_is_a_format_error(ctx):
    from hyperspace_b200 import _native as N

    t = pa.table({"k": np.arange(50_000, dtype=np.int64), "v": np.arange(50_000, dtype=np.int64) * 3})
    img = bytearray(_image(t, compression="gzip", use_dictionary=False))
    md = pq.ParquetFile(io.BytesIO(bytes(img))).metadata
    start = md.row_group(0).column(1).data_page_offset
    img[start + md.row_group(0).column(1).total_compressed_size - 6] ^= 0x55  # inside the last page's trailer
    with pytest.raises(N.HyperspaceGpuError) as e:
        ctx.create_index(_files([bytes(img)]), ["k"], ["v"], 4, output=N.HS_OUT_HOST)
    assert e.value.code == N.HS_EFORMAT and "gzip" in str(e.value)
    ok, _, _ = _build(ctx, [_image(t, compression="gzip")], "k", ["v"])  # the context keeps working
    assert len(ok) > 0


def test_unsorted_scan_over_gzip_sources(ctx):
    t = _typed_table(40_000, 5)
    imgs = [_image(t.slice(0, 25_000), compression="gzip", data_page_version="2.0", use_deprecated_int96_timestamps=True),
            _image(t.slice(25_000), compression="gzip", use_deprecated_int96_timestamps=True)]
    plain = [_image(t.slice(0, 25_000), compression="none", data_page_version="2.0", use_deprecated_int96_timestamps=True),
             _image(t.slice(25_000), compression="none", use_deprecated_int96_timestamps=True)]
    cols = ["i32", "i64", "f64", "s"]
    preds = [("i32", -1000, False, 2000, True)]
    a, _ = ctx.filter_scan_where(_files(imgs), None, cols, preds, sorted_on_key=False)
    b, _ = ctx.filter_scan_where(_files(plain), None, cols, preds, sorted_on_key=False)
    want = int(np.sum(np.asarray(t.column("i32").fill_null(-99999)) >= -1000) -
               np.sum(np.asarray(t.column("i32").fill_null(-99999)) >= 2000))
    assert a.num_rows == b.num_rows == want
    for (na, da, va), (nb_, db, vb) in zip(a.columns, b.columns):
        assert na == nb_
        assert list(da) == list(db), na
        assert (va is None and vb is None) or np.array_equal(np.asarray(va), np.asarray(vb)), na
    a.free()
    b.free()


# ---- the Hyperspace API over a GZIP lake ------------------------------------------------------------------------------------
def _write(dirpath, name, cols):
    os.makedirs(dirpath, exist_ok=True)
    pq.write_table(pa.table(cols), os.path.join(dirpath, name), compression="gzip")


def _table(first, n):
    c = O.synthetic_table(first, n, 3)
    c["k"] = (c["k"] % 5000).astype(np.int64)
    return c


def _rows(res, cols):
    return np.sort(np.rec.fromarrays([np.asarray(res[c]).view(np.int64) if np.asarray(res[c]).dtype.itemsize == 8
                                      else np.asarray(res[c]) for c in cols]))


def test_hyperspace_api_over_a_gzip_lake(tmp_path):
    from hyperspace_b200.hyperspace import Hyperspace
    from hyperspace_b200.index_config import IndexConfig
    from hyperspace_b200.session import HyperspaceSession, col

    s = HyperspaceSession({"spark.hyperspace.system.path": str(tmp_path / "indexes"), "spark.hyperspace.index.numBuckets": "8"})
    try:
        hs = Hyperspace(s)
        L, R = _table(0, 30_000), _table(100_000, 25_000)
        R = {"k": R["k"], "w": R["v1"]}
        _write(tmp_path / "l", "a.parquet", L)
        _write(tmp_path / "r", "a.parquet", R)
        dl, dr = s.read.parquet(str(tmp_path / "l")), s.read.parquet(str(tmp_path / "r"))
        hs.createIndex(dl, IndexConfig("lidx", ["k"], ["v1", "v2"]))
        hs.createIndex(dr, IndexConfig("ridx", ["k"], ["w"]))
        q = dl.filter(col("k").between(100, 300)).select("k", "v2")
        s.disableHyperspace()
        base = q.collect()
        s.enableHyperspace()
        assert "Name: lidx" in q.explain()
        got = q.collect()
        assert len(got["k"]) == int(((L["k"] >= 100) & (L["k"] <= 300)).sum())
        assert np.array_equal(_rows(got, ["k", "v2"]), _rows(base, ["k", "v2"]))
        j = dl.join(dr, on="k").select("v1", "w")
        s.disableHyperspace()
        jb = j.collect()
        s.enableHyperspace()
        assert "Name: lidx" in j.explain() and "Name: ridx" in j.explain()
        jg = j.collect()
        assert len(jg["v1"]) == len(jb["v1"]) > 0
        assert np.array_equal(_rows(jg, ["v1", "w"]), _rows(jb, ["v1", "w"]))
        # appended GZIP file: Hybrid Scan answers without a refresh, then an incremental refresh takes it in
        _write(tmp_path / "l", "b.parquet", _table(50_000, 5_000))
        cur = np.concatenate([L["k"], _table(50_000, 5_000)["k"]])
        s.conf.set("spark.hyperspace.index.hybridscan.enabled", True)
        dl = s.read.parquet(str(tmp_path / "l"))
        q = dl.filter(col("k") <= 50).select("k", "v1")
        assert "hybridScan(appended=1" in q.explain()
        assert len(q.collect()["k"]) == int((cur <= 50).sum())
        s.conf.set("spark.hyperspace.index.hybridscan.enabled", False)
        hs.refreshIndex("lidx", "incremental")
        dl = s.read.parquet(str(tmp_path / "l"))
        q = dl.filter(col("k") <= 50).select("k", "v1")
        assert "Name: lidx" in q.explain()
        assert len(q.collect()["k"]) == int((cur <= 50).sum())
    finally:
        s.stop()
