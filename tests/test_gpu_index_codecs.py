"""GZIP and LZ4 index files on the GPU (spark.sql.parquet.compression.codec=gzip / lz4, as Spark 3.1 writes them through
DataFrameWriter, index/DataFrameWriterExtensions.scala:59-66): the page compressors on a corpus, createIndex with each
codec, the snappy compressor unchanged by the parse they now share, and the Hyperspace API under the conf."""
import gzip
import hashlib
import os
import struct

import numpy as np
import pyarrow as pa
import pyarrow.parquet as pq
import pytest

import parquet_shapes as S
from oracle import oracle as O

pytestmark = pytest.mark.gpu

GZIP, LZ4 = 2, 5
FRAG = 65536


@pytest.fixture(scope="module")
def ctx():
    from hyperspace_b200 import _native

    c = _native.Context(0)
    yield c
    c.close()


def _corpus():
    rng = np.random.default_rng(29)
    for n in (0, 1, 4, 5, 12, 13, 65_535, 65_536, 65_537, (1 << 20) + 4321):
        yield f"zeros{n}", bytes(n)
        yield f"random{n}", rng.integers(0, 256, size=n, dtype=np.uint8).tobytes()
    for p in range(1, 41):
        yield f"period{p}", (rng.integers(0, 256, size=p, dtype=np.uint8).tobytes() * (150_000 // p + 1))[:150_000]
    t = O.synthetic_table(0, 200_000, 5)
    for c in ("k", "v1", "v2", "v3", "v4"):  # table T's columns as PLAIN page bytes, and sorted
        yield f"T.{c}", t[c].tobytes()
        yield f"T.{c}.sorted", np.sort(t[c]).tobytes()
    yield "strings", b"".join(struct.pack("<I", len(s)) + s for s in (f"key-{v}".encode() for v in rng.integers(0, 3000, 40_000)))
    yield "text", (b"the quick brown fox jumps over the lazy dog. " * 5000)[:200_001]


def _gzip_bound(n):
    frag = lambda m: m + 5 * (2 if m > 65535 else 1) + 5
    return 10 + (n // FRAG) * frag(FRAG) + (frag(n % FRAG) if n % FRAG else 0) + 10


def _lz4_groups(stream):
    p, out = 0, []
    while p < len(stream):
        u, c = struct.unpack_from(">II", stream, p)
        out.append((u, stream[p + 8:p + 8 + c]))
        p += 8 + c
    assert p == len(stream)
    return out


def test_k_compress_gzip_round_trips(ctx):
    for name, data in _corpus():
        comp = ctx.k_compress(data, GZIP)
        assert gzip.decompress(comp) == data, name
        assert ctx.k_inflate(comp, len(data)) == data, name
        assert len(comp) <= _gzip_bound(len(data)), name
        if name.startswith(("zeros", "period")) and len(data) > 1000:
            assert len(comp) < 0.2 * len(data), (name, len(comp))
        if name.startswith("T.") and name.endswith("sorted"):
            assert len(comp) < len(data), name
        if len(data) > 100_000:
            assert ctx.k_compress(data, GZIP) == comp, name  # the same on every run


def test_k_compress_lz4_round_trips(ctx):
    raw = pa.Codec("lz4_raw")
    for name, data in _corpus():
        comp = ctx.k_compress(data, LZ4)
        groups = _lz4_groups(comp)
        assert [u for u, _ in groups] == [min(FRAG, len(data) - o) for o in range(0, len(data), FRAG)], name
        back = b"".join(raw.decompress(b, decompressed_size=u).to_pybytes() for u, b in groups)
        assert back == data, name
        assert ctx.k_lz4(comp, len(data), codec=5) == data, name
        bound = sum(8 + u + u // 255 + 16 for u, _ in groups)
        assert len(comp) <= bound, name
        for u, b in groups:  # the end-of-block rule the writer keeps: the last 5 bytes are literals
            if u >= 13:
                assert len(b) >= 6
        if name.startswith(("zeros", "period")) and len(data) > 1000:
            assert len(comp) < 0.2 * len(data), (name, len(comp))
        if len(data) > 100_000:
            assert ctx.k_compress(data, LZ4) == comp, name


def test_k_compress_refuses_other_codecs(ctx):
    from hyperspace_b200._native import HyperspaceGpuError

    for codec in (0, 1, 3, 4, 6, 7):
        with pytest.raises(HyperspaceGpuError):
            ctx.k_compress(b"abc", codec)


# digests of k_snappy_compress's output on a seeded corpus, taken with the compressor as it was before the LZ77 parse was
# shared with the GZIP and LZ4 compressors: the snappy index files must not change
SNAPPY_DIGESTS = {
    "zeros": "f315524d13865d987922ea75779bfef8",
    "random": "a7ce4dc7b2df221a80108d4a2eca2f46",
    "text": "ec33aa3faa5358b6f94d282f565975eb",
    "arange": "593818295613fc7ece76af60c7bede51",
    "floats": "31fa70b6967bd8b6f525dc9c67c06072",
    "low65535": "3c42d9fa554e55d2a90bce3300ea6f85",
    "low65536": "16f0e1b346b056282baf5617e2880aff",
    "low65537": "dd528fded7f03aa50b9d74a201010939",
    "low131077": "a58d92e68c532fba4f18c861cb3dec73",
    "T.k": "a0c6f1caf933566f058a033d63a91a86",
    "T.k.sorted": "41bb855a34d57d4710e47856c3bce4e8",
    "T.v1": "85011e6b0d145b3db092771778110d3b",
    "T.v1.sorted": "2a4e44c574ea0b3d7d39c0cc241dde41",
    "T.v2": "31fa70b6967bd8b6f525dc9c67c06072",
    "T.v2.sorted": "31fa70b6967bd8b6f525dc9c67c06072",
    "T.v3": "016f54b5b5855affbe38ec64204aea14",
    "T.v3.sorted": "1639decb70d972706134231359e927ff",
    "T.v4": "286229c458f04a6bebab0d113413c96e",
    "T.v4.sorted": "160513d7c075f9c736fe1508fc17e6ab",
}


def _snappy_corpus():
    rng = np.random.default_rng(5)
    yield "zeros", bytes(100_000)
    yield "random", rng.integers(0, 256, size=200_000, dtype=np.uint8).tobytes()
    yield "text", (b"the quick brown fox jumps over the lazy dog. " * 5000)[:200_001]
    yield "arange", np.arange(50_000, dtype=np.int64).tobytes()
    yield "floats", (np.arange(300_000, dtype=np.float64) * 1e-3).tobytes()
    for n in (65_535, 65_536, 65_537, 131_077):
        yield f"low{n}", rng.integers(0, 4, size=n, dtype=np.uint8).tobytes()
    t = O.synthetic_table(0, 300_000, 5)
    for c in ("k", "v1", "v2", "v3", "v4"):
        yield f"T.{c}", t[c].tobytes()
        yield f"T.{c}.sorted", np.sort(t[c]).tobytes()


def test_snappy_output_unchanged(ctx):
    got = {name: hashlib.sha256(ctx.k_snappy_compress(data)).hexdigest()[:32] for name, data in _snappy_corpus()}
    assert got == SNAPPY_DIGESTS


# ---- createIndex with each codec -------------------------------------------------------------------------------------------
def _footer_codecs(data):
    """the codec ids of every column chunk in the footer (pyarrow names codec 5 UNKNOWN)"""
    footer, _ = S.read_struct(data, len(data) - 8 - int.from_bytes(data[-8:-4], "little"))
    return {cc[3][4] for rg in footer[4] for cc in rg[1]}


def _build(ctx, sources, key, included, nb, compression, **kw):
    from hyperspace_b200 import _native as N

    res, _ = ctx.create_index(sources, key, included, nb, output=N.HS_OUT_HOST, job_uuid="codecs", compression=compression, **kw)
    out = [(f.name, f.bucket, res.host_bytes(i)) for i, f in enumerate(res.files)]
    res.free()
    return out


EXT = {0: ".c000.parquet", 1: ".c000.snappy.parquet", GZIP: ".c000.gz.parquet", LZ4: ".c000.lz4.parquet"}


@pytest.mark.parametrize("lsd", [False, True])
@pytest.mark.parametrize("dictionary", [True, False])
def test_create_index_over_table_t(ctx, monkeypatch, dictionary, lsd):
    from hyperspace_b200 import _native as N

    if lsd:
        monkeypatch.setenv("HS_LSD_SORT", "1")
    n, nb = 400_000, 16
    src = ctx.synth_table(0, n, 5, n_files=3, row_groups_per_file=2, output=N.HS_OUT_DEVICE, dictionary=dictionary)
    inc = ["v1", "v2", "v3", "v4"]
    try:
        builds = {c: _build(ctx, src.as_sources(), ["k"], inc, nb, c, dictionary=dictionary) for c in (0, 1, GZIP, LZ4)}
        gen = ctx.synth_checksum(0, n, 5)
        for codec in (GZIP, LZ4):
            files = builds[codec]
            assert all(name.endswith(EXT[codec]) for name, _, _ in files)
            assert _build(ctx, src.as_sources(), ["k"], inc, nb, codec, dictionary=dictionary) == files  # byte-identical
            for (name, b, data), (_, b0, plain) in zip(files, builds[0]):
                assert b == b0
                assert _footer_codecs(data) == {codec}
                got = pq.ParquetFile(pa.BufferReader(data)).read()
                assert got.equals(pq.ParquetFile(pa.BufferReader(plain)).read()), name
                st = pq.ParquetFile(pa.BufferReader(data)).metadata.row_group(0).column(0).statistics
                assert st is not None and st.min == got.column("k")[0].as_py()  # key statistics survive
            rep = ctx.verify_index([N.FileImage(data=d) for _, _, d in files], [b for _, b, _ in files], ["k"], inc, nb)
            assert rep["rows"] == n and rep["bucket_mismatches"] == 0 and rep["order_violations"] == 0
            assert rep["row_checksum"] == gen["row_checksum"]
        assert sum(len(d) for _, _, d in builds[GZIP]) <= sum(len(d) for _, _, d in builds[1])
    finally:
        src.free()


def _typed_table(n, seed):
    import decimal

    rng = np.random.default_rng(seed)
    base = np.datetime64("2001-02-03T04:05:06", "us").astype(np.int64)
    return pa.table({
        "i64": pa.array(np.sort(rng.integers(-2**40, 2**40, n, dtype=np.int64))),
        "i32": pa.array(rng.integers(-5000, 5000, n, dtype=np.int32), mask=rng.random(n) < 0.1),
        "s": pa.array([f"key-{v}" for v in rng.integers(0, 3000, n)], mask=rng.random(n) < 0.05),
        "ts": pa.array((base + rng.integers(0, 10**12, n)).astype("datetime64[us]"), pa.timestamp("us")),
        "dec": pa.array([None if m else decimal.Decimal(int(v)).scaleb(-2) for v, m in
                         zip(rng.integers(-10**10, 10**10, n), rng.random(n) < 0.1)], pa.decimal128(12, 2)),
    })


@pytest.mark.parametrize("key", ["i64", "s", "ts", "dec"])
@pytest.mark.parametrize("codec", [GZIP, LZ4])
def test_create_index_typed_nullable_columns(ctx, key, codec):
    from hyperspace_b200 import _native as N

    t = _typed_table(60_000, 4)
    imgs = []
    for part in (t.slice(0, 35_000), t.slice(35_000)):
        sink = pa.BufferOutputStream()
        pq.write_table(part, sink, compression="snappy", use_deprecated_int96_timestamps=True)
        imgs.append(N.FileImage(data=sink.getvalue().to_pybytes()))
    inc = [c for c in t.column_names if c != key]
    plain = _build(ctx, imgs, [key], inc, 8, 0)
    files = _build(ctx, imgs, [key], inc, 8, codec)
    assert files == _build(ctx, imgs, [key], inc, 8, codec)
    for (name, b, data), (_, _, p) in zip(files, plain):
        assert name.endswith(EXT[codec]) and _footer_codecs(data) == {codec}
        assert pq.ParquetFile(pa.BufferReader(data)).read().equals(pq.ParquetFile(pa.BufferReader(p)).read())
    rep = ctx.verify_index([N.FileImage(data=d) for _, _, d in files], [b for _, b, _ in files], [key], inc, 8)
    assert rep["rows"] == t.num_rows and rep["bucket_mismatches"] == 0 and rep["order_violations"] == 0
    # the engine re-reads its own files (optimize, refresh): an index built from them is the uncompressed build
    again = _build(ctx, [N.FileImage(data=d) for _, _, d in files], [key], inc, 8, 0)
    assert [pq.ParquetFile(pa.BufferReader(d)).read() for _, _, d in again] == \
           [pq.ParquetFile(pa.BufferReader(d)).read() for _, _, d in plain]


def test_other_spec_codecs_are_refused(ctx):
    from hyperspace_b200 import _native as N

    src = ctx.synth_table(0, 1000, 2, output=N.HS_OUT_DEVICE)
    try:
        for codec in (3, 4, 6, 7, -1):
            with pytest.raises(N.HyperspaceGpuError) as e:
                ctx.create_index(src.as_sources(), ["k"], ["v1"], 4, output=N.HS_OUT_HOST, compression=codec)
            assert e.value.code == N.HS_EUNSUPPORTED and f"codec {codec}" in str(e.value)
    finally:
        src.free()


# ---- the Hyperspace API under spark.sql.parquet.compression.codec --------------------------------------------------------------
def _write(dirpath, name, cols):
    os.makedirs(dirpath, exist_ok=True)
    pq.write_table(pa.table(cols), os.path.join(dirpath, name), compression="snappy")


def _table(first, n):
    c = O.synthetic_table(first, n, 3)
    c["k"] = (c["k"] % 5000).astype(np.int64)
    return c


def _rows(res, cols):
    return np.sort(np.rec.fromarrays([np.asarray(res[c]).view(np.int64) if np.asarray(res[c]).dtype.itemsize == 8
                                      else np.asarray(res[c]) for c in cols]))


def _index_files(root, name):
    out = []
    for d, _, fs in os.walk(os.path.join(root, name)):
        out += [os.path.join(d, f) for f in fs if f.endswith(".parquet")]
    return sorted(out)


@pytest.mark.parametrize("conf,refresh_conf", [("gzip", "lz4"), ("LZ4", "GZIP")])
def test_hyperspace_api_with_the_codec_conf(tmp_path, conf, refresh_conf):
    from hyperspace_b200.hyperspace import Hyperspace
    from hyperspace_b200.index_config import IndexConfig
    from hyperspace_b200.log_entry import HyperspaceException
    from hyperspace_b200.session import HyperspaceSession, col

    root = str(tmp_path / "indexes")
    s = HyperspaceSession({"spark.hyperspace.system.path": root, "spark.hyperspace.index.numBuckets": "8",
                           "spark.sql.parquet.compression.codec": conf})
    ext = {"gzip": ".gz.parquet", "lz4": ".lz4.parquet"}
    try:
        hs = Hyperspace(s)
        L_, R = _table(0, 30_000), _table(100_000, 25_000)
        R = {"k": R["k"], "w": R["v1"]}
        _write(tmp_path / "l", "a.parquet", L_)
        _write(tmp_path / "r", "a.parquet", R)
        dl, dr = s.read.parquet(str(tmp_path / "l")), s.read.parquet(str(tmp_path / "r"))
        hs.createIndex(dl, IndexConfig("lidx", ["k"], ["v1", "v2"]))
        hs.createIndex(dr, IndexConfig("ridx", ["k"], ["w"]))
        assert all(f.endswith(ext[conf.lower()]) for f in _index_files(root, "lidx"))
        q = dl.filter(col("k").between(100, 300)).select("k", "v2")
        s.disableHyperspace()
        base = q.collect()
        s.enableHyperspace()
        assert "Name: lidx" in q.explain()
        assert np.array_equal(_rows(q.collect(), ["k", "v2"]), _rows(base, ["k", "v2"]))
        j = dl.join(dr, on="k").select("v1", "w")
        s.disableHyperspace()
        jb = j.collect()
        s.enableHyperspace()
        assert "Name: lidx" in j.explain() and "Name: ridx" in j.explain()
        assert np.array_equal(_rows(j.collect(), ["v1", "w"]), _rows(jb, ["v1", "w"]))

        # codecs the engine does not write: refused before any log entry, the index left as it was
        _write(tmp_path / "l", "b.parquet", _table(50_000, 5_000))
        before = sorted(os.listdir(os.path.join(root, "lidx", "_hyperspace_log")))
        for bad in ("zstd", "brotli", "lzo", "Snappy2"):
            s.conf.set("spark.sql.parquet.compression.codec", bad)
            with pytest.raises(HyperspaceException, match=bad):
                hs.refreshIndex("lidx", "incremental")
            assert sorted(os.listdir(os.path.join(root, "lidx", "_hyperspace_log"))) == before
        # an incremental refresh under another codec: an index of mixed-codec files
        s.conf.set("spark.sql.parquet.compression.codec", refresh_conf)
        cur = np.concatenate([L_["k"], _table(50_000, 5_000)["k"]])
        dl = s.read.parquet(str(tmp_path / "l"))
        s.conf.set("spark.hyperspace.index.hybridscan.enabled", True)
        q = dl.filter(col("k") <= 50).select("k", "v1")
        assert "hybridScan(appended=1" in q.explain()
        assert len(q.collect()["k"]) == int((cur <= 50).sum())
        s.conf.set("spark.hyperspace.index.hybridscan.enabled", False)
        hs.refreshIndex("lidx", "incremental")
        files = _index_files(root, "lidx")
        assert any(f.endswith(ext[conf.lower()]) for f in files) and any(f.endswith(ext[refresh_conf.lower()]) for f in files)
        dl = s.read.parquet(str(tmp_path / "l"))
        q = dl.filter(col("k") <= 50).select("k", "v1")
        assert "Name: lidx" in q.explain()
        assert len(q.collect()["k"]) == int((cur <= 50).sum())
        j = dl.join(dr, on="k").select("v1", "w")
        s.disableHyperspace()
        jb = j.collect()
        s.enableHyperspace()
        assert np.array_equal(_rows(j.collect(), ["v1", "w"]), _rows(jb, ["v1", "w"]))
        # optimize rewrites the small files in the current codec
        s.conf.set("spark.sql.parquet.compression.codec", conf)
        hs.optimizeIndex("lidx", "full")
        latest = max(os.listdir(os.path.join(root, "lidx")), key=lambda d: (d.startswith("v__="), d))
        new = [f for f in _index_files(root, "lidx") if f"/{latest}/" in f]
        assert new and all(f.endswith(ext[conf.lower()]) for f in new)
        q = dl.filter(col("k") <= 50).select("k", "v1")
        assert len(q.collect()["k"]) == int((cur <= 50).sum())
    finally:
        s.stop()


@pytest.mark.parametrize("conf,suffix", [(None, ".c000.parquet"), ("none", ".c000.parquet"), ("uncompressed", ".c000.parquet"),
                                         ("snappy", ".c000.snappy.parquet")])
def test_unset_none_and_snappy_keep_todays_names(tmp_path, conf, suffix):
    from hyperspace_b200.hyperspace import Hyperspace
    from hyperspace_b200.index_config import IndexConfig
    from hyperspace_b200.session import HyperspaceSession

    root = str(tmp_path / "indexes")
    confs = {"spark.hyperspace.system.path": root, "spark.hyperspace.index.numBuckets": "4"}
    if conf:
        confs["spark.sql.parquet.compression.codec"] = conf
    s = HyperspaceSession(confs)
    try:
        _write(tmp_path / "l", "a.parquet", _table(0, 5_000))
        Hyperspace(s).createIndex(s.read.parquet(str(tmp_path / "l")), IndexConfig("idx", ["k"], ["v1"]))
        files = _index_files(root, "idx")
        assert files and all(f.endswith(suffix) for f in files)
    finally:
        s.stop()
