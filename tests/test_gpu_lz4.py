"""LZ4-compressed Parquet on the GPU: the page decompressor (k_lz4) against pyarrow on the corpus and the mutations of
tests/lz4_corpus.py, createIndex over LZ4_RAW sources written by pyarrow and over hand-built LZ4 (Hadoop-framed) sources --
index files byte-identical to those built from the same rows written UNCOMPRESSED --, codecs mixed in one call, the
unsorted scan, and the Hyperspace API over an LZ4 lake."""
import copy
import decimal
import io
import os
import struct

import numpy as np
import pyarrow as pa
import pyarrow.parquet as pq
import pytest

import lz4_corpus as L
import parquet_shapes as S
from oracle import oracle as O

pytestmark = pytest.mark.gpu

TEXTS = {L.TRUNCATED: "inside a sequence", L.OFFSET_ZERO: "offset 0", L.BEFORE_START: "before the start",
         L.OUTPUT_OVERRUN: "longer", L.OUTPUT_SHORT: "shorter", L.END_OF_BLOCK: "end-of-block"}


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


def _codecs(img):
    """{column: codec id in the footer} of the first row group"""
    footer, _ = S.read_struct(img, len(img) - 8 - int.from_bytes(img[-8:-4], "little"))
    return {cc[3][3][0].decode(): cc[3][4] for cc in footer[4][0][1]}


# ---- the kernel on its own --------------------------------------------------------------------------------------------------
def test_k_lz4_decodes_the_corpus(ctx):
    bad = []
    for name, codec, stream, data in L.valid():
        if ctx.k_lz4(stream, len(data), codec) != data:
            bad.append(name)
    assert not bad, bad[:10]


def test_k_lz4_agrees_with_pyarrow_on_every_mutation(ctx):
    from hyperspace_b200 import _native as N

    disagree = []
    for name, stream, n in L.mutations():
        theirs = L.pyarrow_accepts(stream, n)
        try:
            got, check = ctx.k_lz4(stream, n), None
        except N.HyperspaceGpuError as e:
            assert e.code == N.HS_EFORMAT and "corrupt lz4 block" in str(e), (name, str(e))
            got, check = None, str(e)
        if theirs and check is not None and TEXTS[L.OFFSET_ZERO] in check:
            continue  # pyarrow's LZ4 takes a match offset of 0; the block format does not
        if (check is None) != theirs or (theirs and got != L.pyarrow_decode(stream, n)):
            disagree.append((name, check, theirs))
    assert not disagree, disagree[:10]


def test_damaged_streams_are_format_errors_and_the_context_keeps_working(ctx):
    from hyperspace_b200 import _native as N

    for name, codec, stream, n, check in L.damaged():
        with pytest.raises(N.HyperspaceGpuError) as e:
            ctx.k_lz4(stream, n, codec)
        assert e.value.code == N.HS_EFORMAT, name
        assert TEXTS[check] in str(e.value), (name, str(e.value))
    with pytest.raises(N.HyperspaceGpuError) as e:
        ctx.k_lz4(L.compress(b"abc" * 100), 300, codec=6)
    assert e.value.code == N.HS_EINVAL
    data = b"still working " * 1000
    assert ctx.k_lz4(L.compress(data), len(data)) == data


# ---- createIndex over LZ4 sources -------------------------------------------------------------------------------------------
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
    "level12_small_pages": dict(compression_level=12, data_page_size=16 << 10),
}
KEYS = ["i32", "i64", "f32", "f64", "s", "ts", "dec"]


def _build(ctx, images, key, included, nb=8, profile=False):
    from hyperspace_b200 import _native as N

    ctx.profile_enable(profile)
    try:
        res, st = ctx.create_index(_files(images), [key], included, nb, output=N.HS_OUT_HOST, job_uuid="lz4")
        kernels = ctx.profile_report() if profile else {}
    finally:
        ctx.profile_enable(False)
    out = [(f.name, f.bucket, res.host_bytes(i)) for i, f in enumerate(res.files)]
    res.free()
    return out, st, kernels


@pytest.mark.parametrize("write", list(WRITES))
@pytest.mark.parametrize("key", KEYS)
def test_lz4_sources_index_like_uncompressed(ctx, write, key):
    from hyperspace_b200 import _native as N

    t = _typed_table(30_000, 3)
    kw = dict(WRITES[write], use_deprecated_int96_timestamps=True)
    plain_kw = {k: v for k, v in kw.items() if k != "compression_level"}
    lz = [_image(t.slice(0, 17_000), compression="lz4", **kw), _image(t.slice(17_000), compression="lz4", **kw)]
    none = [_image(t.slice(0, 17_000), compression="none", **plain_kw), _image(t.slice(17_000), compression="none", **plain_kw)]
    assert set(_codecs(lz[0]).values()) == {7}  # pyarrow's "lz4" is LZ4_RAW
    included = [c for c in t.column_names if c != key]
    a, _, kern = _build(ctx, lz, key, included, profile=True)
    assert kern["k_lz4"]["launches"] == 1
    b, _, kern_plain = _build(ctx, none, key, included, profile=True)
    assert "k_lz4" not in kern_plain
    assert a == b  # the source codec does not leak into the index files
    rep = ctx.verify_index([N.FileImage(data=d) for _, _, d in a], [bk for _, bk, _ in a], [key], included, 8)
    assert rep["rows"] == t.num_rows and rep["bucket_mismatches"] == 0 and rep["order_violations"] == 0


# ---- codec-5 files from the writer of tests/parquet_shapes.py -----------------------------------------------------------
def _hadoop_block(data: bytes) -> bytes:
    """Hadoop's Lz4Codec framing: one group (big-endian uncompressed length) of one chunk (big-endian compressed length)"""
    block = L.compress(data)
    return struct.pack(">II", len(data), len(block)) + block


def _codec_positions(img):
    """file offsets of the codec field value of every ColumnMetaData (FileMetaData.row_groups[].columns[].meta_data.codec)"""
    out = []

    def walk(p, path):  # a compact-protocol struct at p; returns the position after it
        last = 0
        while True:
            x = img[p]
            p += 1
            if x == 0:
                return p
            t, d = x & 0x0F, x >> 4
            if d:
                fid = last + d
            else:
                v, p = S._read_varint(img, p)
                fid = S._unzz(v)
            last = fid
            here = path + (fid,)
            if here == (4, 1, 3, 4):
                out.append(p)
            if t == S.T_STRUCT:
                p = walk(p, here)
            elif t == S.T_LIST and here in ((4,), (4, 1)):
                h = img[p]
                p += 1
                n = h >> 4
                if n == 15:
                    n, p = S._read_varint(img, p)
                for _ in range(n):
                    p = walk(p, here)
            else:
                _, p = S._read_value(img, p, t)

    walk(len(img) - 8 - int.from_bytes(img[-8:-4], "little"), ())
    return out


def _codec5_files(monkeypatch, specs, compress):
    """The files of parquet_shapes specs with every chunk compressed by `compress` and marked codec 5 (LZ4).  The writer
    compresses SNAPPY chunks with its `_snappy`, so the chunks are written as SNAPPY with `compress` in its place, and the
    footer's codec ids are then rewritten (1 and 5 are both one-byte varints).  A compressed page is decoded from an
    aligned scratch copy, so where its values start in the file is not asked for."""
    specs = copy.deepcopy(specs)
    for s in specs:
        for col in s.cols:
            for ch in col.chunks:
                ch.codec = S.SNAPPY
                for pg in ch.pages:
                    pg.align = None
    with monkeypatch.context() as m:
        m.setattr(S, "_snappy", compress)
        images = [bytearray(S.write_file(s)) for s in specs]
    for img in images:
        for pos in _codec_positions(img):
            assert img[pos] == S._zz(S.SNAPPY)
            img[pos] = S._zz(L.LZ4_HADOOP)
    return [bytes(img) for img in images]


SHAPES = ["v2_pages_stored_uncompressed_in_snappy_chunks", "dict_2049_entries_in_global_memory",
          "strings_null_at_every_position", "levels_nulls_at_tile_edges_dictionary", "index_bit_widths_1_to_20",
          "parquet_mr_v1_plain_dictionary_with_statistics"]


@pytest.mark.parametrize("framing", ["hadoop", "raw_fallback"])
@pytest.mark.parametrize("name", SHAPES)
def test_codec5_files_read_like_the_case_as_written(ctx, monkeypatch, name, framing):
    specs, _ = S.CASES[name]()
    # older Parquet C++ wrote raw blocks under codec 5
    lz = _codec5_files(monkeypatch, specs, _hadoop_block if framing == "hadoop" else L.compress)
    plain = S.case_data(name)[0]  # the case as written (UNCOMPRESSED, or SNAPPY where it says so)
    assert lz != plain and set(_codecs(lz[0]).values()) == {5}
    cols = [c.name for c in specs[0].cols]
    a, _ = ctx.filter_scan_where(_files(lz), None, cols, [], sorted_on_key=False)
    b, _ = ctx.filter_scan_where(_files(plain), None, cols, [], sorted_on_key=False)
    assert a.num_rows == b.num_rows > 0
    for (na, da, va), (nb_, db, vb) in zip(a.columns, b.columns):
        assert na == nb_
        assert list(da) == list(db), na
        assert (va is None and vb is None) or np.array_equal(np.asarray(va), np.asarray(vb)), na
    a.free()
    b.free()
    fixed = [c.name for c in specs[0].cols if c.ptype in S.FIXED and c.name != "k"]
    if fixed:
        x, _, kern = _build(ctx, lz, "k", fixed, nb=4, profile=True)
        y, _, _ = _build(ctx, plain, "k", fixed, nb=4)
        assert x == y and kern["k_lz4"]["launches"] == 1


def test_lz4_index_matches_the_oracle(ctx):
    cols = O.synthetic_table(0, 200_000, 5)
    t = pa.table(cols)
    order = ["k", "v1", "v2", "v3", "v4"]
    got, _, kern = _build(ctx, [_image(t, compression="lz4", data_page_size=64 << 10)], "k", order[1:], nb=16, profile=True)
    perm, offs, oorder = O.index_rows(cols, ["k"], order[1:], 16)
    for _, b, data in got:
        f = pq.ParquetFile(pa.BufferReader(data)).read()
        for c in oorder:
            assert f.column(c).to_numpy().tobytes() == cols[c][perm[int(offs[b]):int(offs[b + 1])]].tobytes(), (c, b)
    assert kern["k_lz4"]["launches"] == 1


def test_all_null_v2_page(ctx):
    n = 5000
    t = pa.table({"k": np.arange(n, dtype=np.int64), "v": pa.nulls(n, pa.int64())})
    a, _, _ = _build(ctx, [_image(t, compression="lz4", data_page_version="2.0")], "k", ["v"])
    b, _, _ = _build(ctx, [_image(t, compression="none", data_page_version="2.0")], "k", ["v"])
    assert a == b
    assert sum(pq.ParquetFile(pa.BufferReader(d)).read().column("v").null_count for _, _, d in a) == n


def _codec_kernels(kern):
    return {k: kern[k]["launches"] for k in kern if k.startswith("k_snappy") or k in ("k_inflate", "k_lz4")}


def test_mixed_codecs_in_one_call(ctx, monkeypatch):
    from hyperspace_b200 import _native as N

    cols = O.synthetic_table(0, 90_000, 5)
    t = pa.table(cols)
    parts = [t.slice(0, 30_000), t.slice(30_000, 30_000), t.slice(60_000)]
    per_column = {"k": "snappy", "v1": "gzip", "v2": "lz4", "v3": "none", "v4": "lz4"}
    mixed = [_image(parts[0], compression="lz4"), _image(parts[1], compression="gzip"),
             _image(parts[2], compression=per_column)]
    # and a hand-built codec-5 file of the same rows as the first part
    p0 = {c: parts[0].column(c).to_numpy() for c in t.column_names}
    ptype = {np.dtype(np.int64): S.INT64, np.dtype(np.float64): S.DOUBLE, np.dtype(np.int32): S.INT32,
             np.dtype(np.float32): S.FLOAT}
    spec = S.FileSpec([S.Col(c, ptype[v.dtype], False, [S.Chunk([S.Page(rows=10_000, values=v[i:i + 10_000])
                                                                  for i in range(0, 30_000, 10_000)])])
                       for c, v in p0.items()])
    hadoop, = _codec5_files(monkeypatch, [spec], _hadoop_block)
    assert set(_codecs(hadoop).values()) == {5} and _codecs(mixed[2]) == {"k": 1, "v1": 2, "v2": 7, "v3": 0, "v4": 7}
    plain = [_image(p, compression="none") for p in parts]
    inc = ["v1", "v2", "v3", "v4"]
    a, _, kern = _build(ctx, mixed + [hadoop], "k", inc, profile=True)
    b, _, _ = _build(ctx, plain + [plain[0]], "k", inc)
    assert a == b
    assert _codec_kernels(kern) == {"k_snappy_index": 1, "k_snappy_blocks": 1, "k_inflate": 1, "k_lz4": 1}
    _, _, kern = _build(ctx, [_image(p, compression="snappy") for p in parts] + [_image(parts[0], compression="gzip")], "k", inc,
                        profile=True)
    assert "k_lz4" not in kern and kern["k_inflate"]["launches"] == 1
    # a file that mixes LZ4 and ZSTD columns is refused, naming the ZSTD column
    bad = _image(parts[0], compression={"k": "lz4", "v1": "lz4", "v2": "zstd", "v3": "lz4", "v4": "lz4"})
    with pytest.raises(N.HyperspaceGpuError) as e:
        ctx.create_index(_files([bad]), ["k"], inc, 4, output=N.HS_OUT_HOST)
    assert e.value.code == N.HS_EUNSUPPORTED and "'v2'" in str(e.value) and "codec 6" in str(e.value)
    assert "LZ4_RAW" in str(e.value)


def test_corrupt_lz4_page_is_a_format_error(ctx):
    from hyperspace_b200 import _native as N

    t = pa.table({"k": np.arange(50_000, dtype=np.int64), "v": np.arange(50_000, dtype=np.int64) * 3})
    img = bytearray(_image(t, compression="lz4", use_dictionary=False))
    cm = pq.ParquetFile(io.BytesIO(bytes(img))).metadata.row_group(0).column(1)
    p, end, last_body = cm.data_page_offset, cm.data_page_offset + cm.total_compressed_size, None
    while p < end:  # the last data page's body
        h, p = S.read_struct(img, p)
        last_body = p
        p += h[3]
    img[last_body] = 0x0F  # its first token: no literals, then a match before any output
    with pytest.raises(N.HyperspaceGpuError) as e:
        ctx.create_index(_files([bytes(img)]), ["k"], ["v"], 4, output=N.HS_OUT_HOST)
    assert e.value.code == N.HS_EFORMAT and "corrupt lz4 block: match reaches before the start" in str(e.value)
    ok, _, _ = _build(ctx, [_image(t, compression="lz4")], "k", ["v"])  # the context keeps working
    assert len(ok) > 0


def test_unsorted_scan_over_lz4_sources(ctx):
    t = _typed_table(40_000, 5)
    kw = dict(use_deprecated_int96_timestamps=True)
    imgs = [_image(t.slice(0, 25_000), compression="lz4", data_page_version="2.0", **kw),
            _image(t.slice(25_000), compression="lz4", **kw)]
    plain = [_image(t.slice(0, 25_000), compression="none", data_page_version="2.0", **kw),
             _image(t.slice(25_000), compression="none", **kw)]
    cols = ["i32", "i64", "f64", "s", "ts", "dec"]
    preds = [("i32", -1000, False, 2000, True)]
    a, _ = ctx.filter_scan_where(_files(imgs), None, cols, preds, sorted_on_key=False)
    b, _ = ctx.filter_scan_where(_files(plain), None, cols, preds, sorted_on_key=False)
    i32 = np.asarray(t.column("i32").fill_null(-99999))
    assert a.num_rows == b.num_rows == int(np.sum((i32 >= -1000) & (i32 < 2000)))
    for (na, da, va), (nb_, db, vb) in zip(a.columns, b.columns):
        assert na == nb_
        assert list(da) == list(db), na
        assert (va is None and vb is None) or np.array_equal(np.asarray(va), np.asarray(vb)), na
    a.free()
    b.free()


# ---- the Hyperspace API over an LZ4 lake ------------------------------------------------------------------------------------
def _write(dirpath, name, cols):
    os.makedirs(dirpath, exist_ok=True)
    pq.write_table(pa.table(cols), os.path.join(dirpath, name), compression="lz4")


def _table(first, n):
    c = O.synthetic_table(first, n, 3)
    c["k"] = (c["k"] % 5000).astype(np.int64)
    return c


def _rows(res, cols):
    return np.sort(np.rec.fromarrays([np.asarray(res[c]).view(np.int64) if np.asarray(res[c]).dtype.itemsize == 8
                                      else np.asarray(res[c]) for c in cols]))


def test_hyperspace_api_over_an_lz4_lake(tmp_path):
    from hyperspace_b200.hyperspace import Hyperspace
    from hyperspace_b200.index_config import IndexConfig
    from hyperspace_b200.session import HyperspaceSession, col

    s = HyperspaceSession({"spark.hyperspace.system.path": str(tmp_path / "indexes"), "spark.hyperspace.index.numBuckets": "8"})
    try:
        hs = Hyperspace(s)
        L_, R = _table(0, 30_000), _table(100_000, 25_000)
        R = {"k": R["k"], "w": R["v1"]}
        _write(tmp_path / "l", "a.parquet", L_)
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
        assert len(got["k"]) == int(((L_["k"] >= 100) & (L_["k"] <= 300)).sum())
        assert np.array_equal(_rows(got, ["k", "v2"]), _rows(base, ["k", "v2"]))
        j = dl.join(dr, on="k").select("v1", "w")
        s.disableHyperspace()
        jb = j.collect()
        s.enableHyperspace()
        assert "Name: lidx" in j.explain() and "Name: ridx" in j.explain()
        jg = j.collect()
        assert len(jg["v1"]) == len(jb["v1"]) > 0
        assert np.array_equal(_rows(jg, ["v1", "w"]), _rows(jb, ["v1", "w"]))
        # appended LZ4 file: Hybrid Scan answers without a refresh, then an incremental refresh takes it in
        _write(tmp_path / "l", "b.parquet", _table(50_000, 5_000))
        cur = np.concatenate([L_["k"], _table(50_000, 5_000)["k"]])
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
