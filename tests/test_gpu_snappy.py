"""SNAPPY pages both ways on the GPU: the page compressor (any Snappy decoder must give its input back), index files
written as Spark writes them by default (`...c000.snappy.parquet`, T/index/VacuumOutdatedActionTest.scala:67; codec via
index/DataFrameWriterExtensions.scala:59-66) read by pyarrow and by the engine's own decoder, and snappy-compressed sources."""
import numpy as np
import pyarrow as pa
import pyarrow.parquet as pq
import pytest

import snappy_corpus as S
from oracle import oracle as O

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    from hyperspace_b200 import _native

    c = _native.Context(0)
    yield c
    c.close()


def test_page_compressor_round_trips_through_a_reference_decoder(ctx):
    codec = pa.Codec("snappy")
    for data in S.inputs():
        comp = ctx.k_snappy_compress(data)
        back = codec.decompress(comp, decompressed_size=len(data)) if data else b""
        assert bytes(back) == data, len(data)
        if len(data) > 1000 and len(set(data[:1000])) < 8:
            assert len(comp) < 0.8 * len(data), (len(data), len(comp))  # low-entropy inputs do shrink
    # the output is the same on every run (the hash table takes atomicMax updates)
    d = next(x for x in S.inputs() if len(x) > 150_000)
    assert ctx.k_snappy_compress(d) == ctx.k_snappy_compress(d)


@pytest.mark.parametrize("dictionary", [True, False])
def test_snappy_index_files_like_spark_writes_them(ctx, tmp_path, dictionary):
    from hyperspace_b200 import _native as N

    n, nb = 400_000, 16
    src = ctx.synth_table(0, n, 5, n_files=3, row_groups_per_file=2, output=N.HS_OUT_DEVICE, dictionary=dictionary)
    plain, _ = ctx.create_index(src.as_sources(), ["k"], ["v1", "v2", "v3", "v4"], nb, output=N.HS_OUT_HOST, job_uuid="u",
                                dictionary=dictionary)
    out_dir = str(tmp_path / "idx")
    snap, st = ctx.create_index(src.as_sources(), ["k"], ["v1", "v2", "v3", "v4"], nb, out_dir=out_dir, output=N.HS_OUT_FILES,
                                job_uuid="u", dictionary=dictionary, compression=N.HS_CODEC_SNAPPY)
    assert all(f.name.endswith(".c000.snappy.parquet") for f in snap.files)
    total_plain = sum(f.size for f in plain.files)
    total_snap = sum(f.size for f in snap.files)
    assert total_snap < total_plain * 1.02  # random keys do not compress; nothing may blow up either
    for i, f in enumerate(snap.files):
        pf = pq.ParquetFile(f"{out_dir}/{f.name}")
        md = pf.metadata
        assert all(md.row_group(g).column(c).compression == "SNAPPY" for g in range(md.num_row_groups) for c in range(md.num_columns))
        got = pf.read()
        want = pq.ParquetFile(pa.BufferReader(plain.host_bytes(i))).read()
        assert got.equals(want), f.name
        st_k = md.row_group(0).column(0).statistics
        assert st_k.min == got.column("k")[0].as_py()  # key statistics survive the second layout
    # the engine's own decoder reads its snappy files (optimize / refresh re-read index files)
    files = [N.FileImage(path=f"{out_dir}/{f.name}") for f in snap.files]
    rep = ctx.verify_index(files, [f.bucket for f in snap.files], ["k"], ["v1", "v2", "v3", "v4"], nb)
    gen = ctx.synth_checksum(0, n, 5)
    assert rep["rows"] == n and rep["bucket_mismatches"] == 0 and rep["order_violations"] == 0
    assert rep["row_checksum"] == gen["row_checksum"]
    plain.free()
    snap.free()
    src.free()


def test_snappy_source_table_and_compressible_columns(ctx):
    from hyperspace_b200 import _native as N

    n, nb = 300_000, 8
    ssrc = ctx.synth_table(5, n, 5, n_files=2, row_groups_per_file=2, output=N.HS_OUT_HOST, compression=N.HS_CODEC_SNAPPY)
    usrc = ctx.synth_table(5, n, 5, n_files=2, row_groups_per_file=2, output=N.HS_OUT_HOST)
    for i in range(2):  # pyarrow reads the GPU-written snappy source and finds the same table
        a = pq.ParquetFile(pa.BufferReader(ssrc.host_bytes(i))).read()
        b = pq.ParquetFile(pa.BufferReader(usrc.host_bytes(i))).read()
        assert a.equals(b)
    ri, _ = ctx.create_index(ssrc.as_sources(), ["k"], ["v1", "v2", "v3", "v4"], nb, output=N.HS_OUT_HOST, job_uuid="x")
    rj, _ = ctx.create_index(usrc.as_sources(), ["k"], ["v1", "v2", "v3", "v4"], nb, output=N.HS_OUT_HOST, job_uuid="x")
    assert [ri.host_bytes(i) for i in range(len(ri.files))] == [rj.host_bytes(i) for i in range(len(rj.files))]
    ri.free()
    rj.free()
    ssrc.free()
    usrc.free()
    # a table that does compress: sorted keys, a constant column -> the snappy index is much smaller and still right
    k = np.arange(200_000, dtype=np.int64)
    t = pa.table({"k": k, "c": np.full(200_000, 7, dtype=np.int64), "d": (k // 1000).astype(np.float64)})
    sink = pa.BufferOutputStream()
    pq.write_table(t, sink, compression="SNAPPY")
    img = [N.FileImage(data=sink.getvalue().to_pybytes())]
    plain, _ = ctx.create_index(img, ["k"], ["c", "d"], 4, output=N.HS_OUT_HOST, dictionary=False)
    snap, _ = ctx.create_index(img, ["k"], ["c", "d"], 4, output=N.HS_OUT_HOST, dictionary=False, compression=N.HS_CODEC_SNAPPY)
    assert sum(f.size for f in snap.files) < 0.5 * sum(f.size for f in plain.files)
    cols = {"k": k, "c": t.column("c").to_numpy(), "d": t.column("d").to_numpy()}
    perm, offs, order = O.index_rows(cols, ["k"], ["c", "d"], 4)
    for i, f in enumerate(snap.files):
        got = pq.ParquetFile(pa.BufferReader(snap.host_bytes(i))).read()
        for c in order:
            assert got.column(c).to_numpy().tobytes() == cols[c][perm[int(offs[f.bucket]):int(offs[f.bucket + 1])]].tobytes()
    plain.free()
    snap.free()


def test_page_decompressor_on_reference_streams_block_by_block(ctx):
    """Streams of the C++ snappy library (pyarrow's codec, the one behind snappy-java): 64 KB blocks are independent, so
    the decoder takes one warp per block; the result is the input."""
    codec = pa.Codec("snappy")
    for data in S.inputs():
        comp = codec.compress(data, asbytes=True)
        back, sequential = ctx.k_snappy_decompress(comp, len(data))
        assert back == data, len(data)
        assert not sequential
        mine = ctx.k_snappy_compress(data)  # and the engine's own compressor's streams
        back, sequential = ctx.k_snappy_decompress(mine, len(data))
        assert back == data and not sequential


def test_page_decompressor_falls_back_for_streams_whose_blocks_depend_on_each_other(ctx):
    """Legal snappy that no mainstream writer produces: a back-reference reaching into the previous 64 KB block, an element
    straddling a block boundary, an overlapping (run-length) copy.  Decoded front to back by one warp, same bytes."""
    rng = np.random.default_rng(5)
    a = rng.integers(0, 256, size=70_000, dtype=np.uint8).tobytes()
    # 70 000 literal bytes (straddles 65 536), then 64 bytes copied from 69 000 back (crosses the boundary), then a run
    want = a + a[1000:1064]
    want += want[-3:] * 20
    stream = S.varint(len(want)) + S.literal(a) + S.copy4(69_000, 64) + S.copy4(3, 60)
    back, sequential = ctx.k_snappy_decompress(stream, len(want))
    assert sequential and back == want
    # blocks aligned by construction but the second one copies from the first
    b0, b1 = a[:65_536], a[:1000]
    want = b0 + b1[:64] + b1
    stream = S.varint(len(want)) + S.literal(b0) + S.copy4(65_536, 64) + S.literal(b1)
    back, sequential = ctx.k_snappy_decompress(stream, len(want))
    assert sequential and back == want


def test_page_decompressor_rejects_damaged_streams(ctx):
    from hyperspace_b200 import _native as N

    codec = pa.Codec("snappy")
    data = (b"0123456789abcdef" * 20_000)[:300_000]
    comp = codec.compress(data, asbytes=True)
    bad = [
        comp[:len(comp) // 2],                                  # truncated
        S.varint(len(data) + 1) + comp[len(S.varint(len(data))):],  # preamble disagrees with the page header
        S.varint(100) + S.copy4(50, 60) + S.literal(b"x" * 40),     # back-reference before the start of the output
        S.varint(10) + S.literal(b"y" * 30),                      # element longer than the output
        S.varint(50) + S.literal(b"z" * 10),                      # stream ends early
    ]
    lens = [len(data), len(data), 100, 10, 50]
    for stream, n in zip(bad, lens):
        with pytest.raises(N.HyperspaceGpuError) as e:
            ctx.k_snappy_decompress(stream, n)
        assert e.value.code == N.HS_EFORMAT
