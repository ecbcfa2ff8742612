"""GPU parity tests: the CUDA path, called through the C ABI, against the CPU oracle on the same seeded inputs.

Integer / byte / index work is compared bit-exactly; floating-point included columns are pass-through copies and are
compared bit-exactly too (tolerance required by the north star: 1e-6 relative).
Mirrors the reference's hot-path tests: T/index/DataFrameWriterExtensionsTest.scala:93-158 (bucket id per row, per-file
sortedness, row multiset), T/index/BucketUnionTest.scala:101-123 (golden vector), T/index/E2EHyperspaceRulesTest.scala
:1079-1094 (same answers with and without the index).
"""
import io
import os

import numpy as np
import pyarrow as pa
import pyarrow.parquet as pq
import pytest

from oracle import oracle as O

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    from hyperspace_b200 import _native

    c = _native.Context(0)
    yield c
    c.close()


def _bits(a):
    a = np.asarray(a)
    return a.view({4: np.int32, 8: np.int64, 1: np.uint8}[a.dtype.itemsize])


# ---------------------------------------------------------------------------------------------------------------------
# K2: bucket ids
# ---------------------------------------------------------------------------------------------------------------------

def test_golden_vectors_on_gpu(ctx):
    b, _ = ctx.k_bucket_ids([np.array([2, 3], dtype=np.int32)], 10)
    assert b.tolist() == [4, 1]  # BucketUnionTest.scala:122
    ks = np.array([0, 1, 2, 3, -1], dtype=np.int64)
    b, h = ctx.k_bucket_ids([ks], 200)
    assert b.tolist() == [5, 69, 128, 107, 193]
    assert h.sum() == 5


@pytest.mark.parametrize("nb", [1, 7, 200, 1000, 1024, 1025, 4096])
def test_bucket_ids_match_oracle(ctx, nb):
    rng = np.random.default_rng(nb)
    n = 300_000
    k64 = rng.integers(-2**63, 2**63 - 1, size=n, dtype=np.int64)
    k32 = rng.integers(-2**31, 2**31 - 1, size=n, dtype=np.int32)
    f64 = rng.standard_normal(n)
    f64[:4] = [0.0, -0.0, np.nan, np.inf]
    f32 = f64.astype(np.float32)
    for cols in ([k64], [k32], [k32, k64], [f64], [f32, k64]):
        got, hist = ctx.k_bucket_ids(cols, nb)
        want = O.bucket_ids(cols, nb)
        assert np.array_equal(got, want)
        assert np.array_equal(hist, np.bincount(want, minlength=nb))


def test_bucket_ids_null_keys(ctx):
    rng = np.random.default_rng(3)
    k = rng.integers(-1000, 1000, size=50_000, dtype=np.int64)
    valid = (rng.random(50_000) > 0.2).astype(np.uint8)
    got, _ = ctx.k_bucket_ids([k], 200, [valid])
    assert np.array_equal(got, O.bucket_ids([k], 200, [valid]))


def test_bucket_ids_come_from_the_build_kernel(ctx):
    """hs_k_bucket_ids runs the hash step of createIndex (k_tile_hist) on both sides of the fused partition's 1024 bins."""
    rng = np.random.default_rng(4)
    n = 20_000
    k64 = rng.integers(-2**63, 2**63 - 1, size=n, dtype=np.int64)
    k32 = rng.integers(-2**31, 2**31 - 1, size=n, dtype=np.int32)
    valids = [(rng.random(n) > 0.2).astype(np.uint8), (rng.random(n) > 0.5).astype(np.uint8)]
    for cols, vs in (([k64], None), ([k32, k64], valids)):
        for nb in (200, 2048):
            ctx.profile_enable(True)
            try:
                got, _ = ctx.k_bucket_ids(cols, nb, vs)
                kernels = ctx.profile_report()
            finally:
                ctx.profile_enable(False)
            assert "k_tile_hist" in kernels and "k_bucket_hist" not in kernels, kernels
            assert np.array_equal(got, O.bucket_ids(cols, nb, vs))


# ---------------------------------------------------------------------------------------------------------------------
# K3 + K4: partition + segmented sort
# ---------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("n,nb,lo,hi", [(1, 200, -5, 5), (100, 3, -5, 5), (4096, 1, 0, 50), (4097, 200, -2**63, 2**63 - 1),
                                         (250_000, 200, -2**63, 2**63 - 1), (250_000, 13, -50, 50),
                                         (1_000_000, 200, 0, 2**31), (250_000, 1024, -2**63, 2**63 - 1),
                                         (250_000, 1025, -2**63, 2**63 - 1), (300_000, 4096, 0, 2**31)])
def test_sort_perm_matches_oracle_exactly(ctx, n, nb, lo, hi):
    rng = np.random.default_rng(n + nb)
    k = rng.integers(lo, hi, size=n, dtype=np.int64)
    perm, offs = ctx.k_sort_perm([k], nb)
    b = O.bucket_ids([k], nb)
    want_perm, want_offs = O.sort_perm([k], nb, b)
    assert np.array_equal(offs, want_offs)
    assert np.array_equal(perm, want_perm)  # stable: ties keep source order, like the oracle


def test_sort_tie_run_fixup_and_fallback(ctx):
    """Keys with > 4 varying bytes are sorted on their top four varying bytes and short tie runs are fixed up in place;
    long runs (low-entropy high bytes) must fall back to full passes.  Both must equal the oracle's stable order."""
    rng = np.random.default_rng(77)
    n = 300_000
    hi = rng.integers(0, 1 << 16, size=n, dtype=np.int64) << 44      # 65536 distinct values in the top bytes
    lo = rng.integers(0, 5, size=n, dtype=np.int64) << 8             # few distinct low parts -> ties on the full key too
    for keys in (hi | lo,                                             # short runs: fix-up path
                 (rng.integers(0, 3, size=n, dtype=np.int64) << 60) | rng.integers(0, 1 << 30, size=n, dtype=np.int64),  # long runs
                 -(hi | lo)):                                         # negative keys
        for nb in (1, 8):
            perm, offs = ctx.k_sort_perm([keys], nb)
            b = O.bucket_ids([keys], nb)
            want_perm, want_offs = O.sort_perm([keys], nb, b)
            assert np.array_equal(offs, want_offs)
            assert np.array_equal(perm, want_perm)


def test_sort_perm_other_key_types(ctx):
    rng = np.random.default_rng(5)
    n = 100_000
    k32 = rng.integers(-1000, 1000, size=n, dtype=np.int32)
    f64 = np.round(rng.standard_normal(n), 2)
    f64[:6] = [0.0, -0.0, np.nan, np.inf, -np.inf, np.nan]
    f32 = f64.astype(np.float32)
    k64 = rng.integers(-3, 3, size=n, dtype=np.int64)
    for cols in ([k32], [f64], [f32], [k64, k32], [k32, f64, k64]):
        perm, offs = ctx.k_sort_perm(cols, 16)
        b = O.bucket_ids(cols, 16)
        want_perm, want_offs = O.sort_perm(cols, 16, b)
        assert np.array_equal(offs, want_offs)
        assert np.array_equal(perm, want_perm)


def test_sort_perm_nulls_first(ctx):
    rng = np.random.default_rng(9)
    n = 60_000
    k = rng.integers(-100, 100, size=n, dtype=np.int64)
    valid = (rng.random(n) > 0.1).astype(np.uint8)
    k = np.where(valid.astype(bool), k, 0)  # decoded nulls hold 0
    for nb in (8, 2000):  # 2000: the unfused partition scatters the validity bytes as a width-1 column
        perm, offs = ctx.k_sort_perm([k], nb, [valid])
        b = O.bucket_ids([k], nb, [valid])
        want_perm, want_offs = O.sort_perm([k], nb, b, [valid])
        assert np.array_equal(offs, want_offs)
        assert np.array_equal(perm, want_perm)


# ---------------------------------------------------------------------------------------------------------------------
# K6 via the synthetic table: GPU-encoded Parquet must read back (pyarrow) as the oracle's table
# ---------------------------------------------------------------------------------------------------------------------

def _read_image(buf: bytes) -> pa.Table:
    return pq.ParquetFile(pa.BufferReader(buf)).read()


def test_synth_table_round_trips_through_pyarrow(ctx):
    n = 300_001
    res = ctx.synth_table(1000, n, ncols=5, n_files=3, row_groups_per_file=2)
    got = pa.concat_tables([_read_image(res.host_bytes(i)) for i in range(len(res.files))])
    want = O.synthetic_table(1000, n, 5)
    assert got.column_names == list(want)
    assert got.num_rows == n
    for name, arr in want.items():
        assert np.array_equal(_bits(got.column(name).to_numpy()), _bits(arr)), name
    md = pq.ParquetFile(pa.BufferReader(res.host_bytes(0))).metadata
    assert md.num_row_groups == 1 or md.num_row_groups == 2
    res.free()


# ---------------------------------------------------------------------------------------------------------------------
# whole write path: K1 decode of pyarrow-written sources -> K2..K6 -> files that pyarrow reads back
# ---------------------------------------------------------------------------------------------------------------------

def _write_sources(tmp_path, cols, n_files, **kw):
    n = len(next(iter(cols.values())))
    paths = []
    per = (n + n_files - 1) // n_files
    for f in range(n_files):
        part = {k: v[f * per:(f + 1) * per] for k, v in cols.items()}
        p = str(tmp_path / f"src-{f}.parquet")
        pq.write_table(pa.table(part), p, **{"compression": "NONE", **kw})
        paths.append(p)
    return paths


def _check_index(res, cols, indexed, included, nb, job_uuid):
    perm, offs, order = O.index_rows(cols, indexed, included, nb)
    seen = set()
    for i, f in enumerate(res.files):
        assert f.name == O.bucket_file_name(f.bucket, job_uuid)
        lo, hi = int(offs[f.bucket]), int(offs[f.bucket + 1])
        assert f.rows == hi - lo and f.rows > 0
        t = _read_image(res.host_bytes(i))
        assert t.column_names == order
        for name in order:
            got = t.column(name).to_numpy()
            want = cols[name][perm[lo:hi]]
            assert got.dtype == want.dtype, name
            assert np.array_equal(_bits(got), _bits(want)), (name, f.bucket)
        seen.add(f.bucket)
    nonempty = {b for b in range(nb) if offs[b + 1] > offs[b]}
    assert seen == nonempty  # one file per non-empty bucket, none for empty ones


@pytest.mark.parametrize("variant", ["plain_v1", "dict_v1", "dict_v2", "plain_v2_small_pages", "snappy_v1", "snappy_dict_v2",
                                     "snappy_small_pages"])
def test_create_index_matches_oracle(ctx, tmp_path, variant):
    from hyperspace_b200 import _native

    n = 200_000
    cols = O.synthetic_table(0, n, 5)
    kw = {
        "plain_v1": dict(use_dictionary=False, data_page_version="1.0"),
        "dict_v1": dict(use_dictionary=True, data_page_version="1.0"),
        "dict_v2": dict(use_dictionary=True, data_page_version="2.0", row_group_size=30_000),
        "plain_v2_small_pages": dict(use_dictionary=False, data_page_version="2.0", data_page_size=4096, row_group_size=50_000),
        # Spark's default codec: snappy pages (v1: whole page compressed; v2: levels stored, values compressed)
        "snappy_v1": dict(use_dictionary=False, data_page_version="1.0", compression="snappy"),
        "snappy_dict_v2": dict(use_dictionary=True, data_page_version="2.0", compression="snappy", row_group_size=30_000),
        "snappy_small_pages": dict(use_dictionary=["v1", "v3"], data_page_version="1.0", compression="snappy", data_page_size=2048),
    }[variant]
    paths = _write_sources(tmp_path, cols, 3, **kw)
    files = [_native.FileImage(path=p) for p in paths]
    res, st = ctx.create_index(files, ["k"], ["v1", "v2", "v3", "v4"], 200, output=_native.HS_OUT_HOST, job_uuid="uuid-1",
                               rows_per_page=4096, rows_per_row_group=8192)
    assert st["rows_in"] == n and st["rows_out"] == n and st["gpu_launches"] > 0
    _check_index(res, cols, ["k"], ["v1", "v2", "v3", "v4"], 200, "uuid-1")
    res.free()


def test_create_index_when_the_tie_fixup_gives_up(ctx):
    """createIndex does not wait for the verdict of the tie fix-up before it lays out and gathers the pages; when the fix-up
    gives up (long runs of equal key prefixes) the rows are sorted again with full passes and the pages are written again.
    Keys: three values in the top byte, 30 random low bits -> runs of ~n/3/256 rows on the sorted top bytes."""
    rng = np.random.default_rng(78)
    n = 300_000
    cols = {"k": (rng.integers(0, 3, size=n, dtype=np.int64) << 60) | rng.integers(0, 1 << 30, size=n, dtype=np.int64),
            "v": rng.integers(0, 50, size=n, dtype=np.int32), "w": rng.standard_normal(n)}
    for nb in (1, 8):
        res = _index_in_memory(ctx, cols, ["k"], ["v", "w"], nb, "u")
        _check_index(res, cols, ["k"], ["v", "w"], nb, "u")
        res.free()
    short = dict(cols, k=(rng.integers(0, 1 << 16, size=n, dtype=np.int64) << 44) | (rng.integers(0, 5, size=n, dtype=np.int64) << 8))
    res = _index_in_memory(ctx, short, ["k"], ["v", "w"], 8, "u")   # the usual case: short runs, nothing to redo
    _check_index(res, short, ["k"], ["v", "w"], 8, "u")
    res.free()


def test_create_index_c1_config_and_files_on_disk(ctx, tmp_path):
    """BASELINE.json configs[0]: 10k rows x 3 columns; written to disk like the reference does."""
    from hyperspace_b200 import _native

    cols = O.synthetic_table(0, 10_000, 3)
    paths = _write_sources(tmp_path, cols, 1)
    out_dir = str(tmp_path / "idx" / "v__=0")
    res, st = ctx.create_index([_native.FileImage(path=paths[0])], ["k"], ["v1", "v2"], 200, out_dir=out_dir,
                               output=_native.HS_OUT_FILES, job_uuid="u")
    perm, offs, order = O.index_rows(cols, ["k"], ["v1", "v2"], 200)
    names = sorted(os.listdir(out_dir))
    assert names == sorted(f.name for f in res.files)
    total = 0
    for name in names:
        assert name.startswith("part-0")  # T/index/IndexManagerTest.scala:259,738
        bucket = int(name.rsplit("_", 1)[1].split(".")[0])
        t = pq.ParquetFile(os.path.join(out_dir, name)).read()
        k = t.column("k").to_numpy()
        assert np.all(O.np_bucket_ids([k], 200) == bucket)
        assert np.all(k[:-1] <= k[1:])
        lo, hi = int(offs[bucket]), int(offs[bucket + 1])
        assert np.array_equal(k, cols["k"][perm[lo:hi]])
        total += len(k)
    assert total == 10_000
    res.free()


def test_create_index_int32_and_multi_key(ctx, tmp_path):
    from hyperspace_b200 import _native

    rng = np.random.default_rng(21)
    n = 50_000
    cols = {"a": rng.integers(-50, 50, size=n, dtype=np.int32), "b": rng.integers(-3, 3, size=n, dtype=np.int64),
            "x": rng.standard_normal(n), "y": rng.standard_normal(n).astype(np.float32)}
    paths = _write_sources(tmp_path, cols, 2)
    files = [_native.FileImage(path=p) for p in paths]
    for indexed, included in ((["a"], ["x", "y", "b"]), (["a", "b"], ["x"]), (["b", "a"], ["y"])):
        res, _ = ctx.create_index(files, indexed, included, 10, output=_native.HS_OUT_HOST, job_uuid="u2")
        _check_index(res, cols, indexed, included, 10, "u2")
        res.free()


def test_create_index_required_columns_and_in_memory_images(ctx, tmp_path):
    from hyperspace_b200 import _native

    cols = O.synthetic_table(5, 30_000, 3)
    schema = pa.schema([pa.field("k", pa.int64(), nullable=False), pa.field("v1", pa.int64(), nullable=False),
                        pa.field("v2", pa.float64(), nullable=True)])
    sink = io.BytesIO()
    pq.write_table(pa.table(cols, schema=schema), sink, compression="NONE")
    img = sink.getvalue()
    res, _ = ctx.create_index([_native.FileImage(data=img)], ["k"], ["v2", "v1"], 7, output=_native.HS_OUT_HOST, job_uuid="m")
    _check_index(res, cols, ["k"], ["v2", "v1"], 7, "m")
    res.free()


def test_create_index_is_deterministic_and_device_resident_inputs_work(ctx):
    from hyperspace_b200 import _native

    src = ctx.synth_table(0, 100_000, 5, n_files=2, row_groups_per_file=2, output=_native.HS_OUT_DEVICE)
    r1, _ = ctx.create_index(src.as_sources(), ["k"], ["v1", "v2", "v3", "v4"], 50, output=_native.HS_OUT_HOST, job_uuid="d")
    r2, _ = ctx.create_index(src.as_sources(), ["k"], ["v1", "v2", "v3", "v4"], 50, output=_native.HS_OUT_HOST, job_uuid="d")
    assert [f.name for f in r1.files] == [f.name for f in r2.files]
    for i in range(len(r1.files)):
        assert r1.host_bytes(i) == r2.host_bytes(i)
    _check_index(r1, O.synthetic_table(0, 100_000, 5), ["k"], ["v1", "v2", "v3", "v4"], 50, "d")
    for r in (r1, r2, src):
        r.free()


def test_dictionary_encoding_applied_and_optional(ctx):
    """Low-cardinality columns are PLAIN_DICTIONARY-encoded (as parquet-mr does); high-cardinality ones stay PLAIN."""
    from hyperspace_b200 import _native

    n = 150_000
    cols = O.synthetic_table(0, n, 5)
    src = ctx.synth_table(0, n, 5, n_files=2, row_groups_per_file=2, output=_native.HS_OUT_HOST, dictionary=True)
    md = pq.ParquetFile(pa.BufferReader(src.host_bytes(0))).metadata
    enc = {md.schema.column(i).name: md.row_group(0).column(i) for i in range(5)}
    assert enc["v1"].has_dictionary_page and enc["v3"].has_dictionary_page and enc["v4"].has_dictionary_page
    assert not enc["k"].has_dictionary_page and not enc["v2"].has_dictionary_page
    assert enc["v1"].total_compressed_size < enc["k"].total_compressed_size // 4   # 10 bits vs 64 bits per value
    got = pa.concat_tables([_read_image(src.host_bytes(i)) for i in range(2)])
    for name, arr in cols.items():
        assert np.array_equal(_bits(got.column(name).to_numpy()), _bits(arr)), name
    plain = ctx.synth_table(0, n, 5, n_files=2, row_groups_per_file=2, output=_native.HS_OUT_HOST, dictionary=False)
    assert sum(f.size for f in src.files) < 0.7 * sum(f.size for f in plain.files)
    for dictionary in (True, False):
        res, st = ctx.create_index(src.as_sources(), ["k"], ["v1", "v2", "v3", "v4"], 20, output=_native.HS_OUT_HOST, job_uuid="dd",
                                   dictionary=dictionary)
        _check_index(res, cols, ["k"], ["v1", "v2", "v3", "v4"], 20, "dd")
        m = pq.ParquetFile(pa.BufferReader(res.host_bytes(0))).metadata.row_group(0)
        assert m.column(1).has_dictionary_page == dictionary and not m.column(0).has_dictionary_page
        res.free()
    # values equal to the hash set's empty marker (all ones) and a single-value column
    sink = io.BytesIO()
    odd = {"k": np.arange(5000, dtype=np.int64), "a": np.where(np.arange(5000) % 3 == 0, -1, 7).astype(np.int64),
           "b": np.full(5000, 3, dtype=np.int32)}
    pq.write_table(pa.table(odd), sink, compression="NONE")
    res, _ = ctx.create_index([_native.FileImage(data=sink.getvalue())], ["k"], ["a", "b"], 4, output=_native.HS_OUT_HOST, job_uuid="o")
    _check_index(res, odd, ["k"], ["a", "b"], 4, "o")
    res.free()
    src.free()
    plain.free()


def test_lineage_column(ctx, tmp_path):
    from hyperspace_b200 import _native

    cols = O.synthetic_table(0, 20_000, 2)
    paths = _write_sources(tmp_path, cols, 4)
    files = [_native.FileImage(path=p, file_id=10 + i) for i, p in enumerate(paths)]
    res, _ = ctx.create_index(files, ["k"], ["v1"], 5, output=_native.HS_OUT_HOST, job_uuid="l", lineage=True)
    want = dict(cols)
    want["_data_file_id"] = np.repeat(np.arange(10, 14, dtype=np.int64), 5000)
    _check_index(res, want, ["k"], ["v1", "_data_file_id"], 5, "l")
    # refreshIncremental's delete branch: drop rows of deleted source files from the old index and rewrite it
    res2, st2 = ctx.create_index(res.as_sources(), ["k"], ["v1", "_data_file_id"], 5, output=_native.HS_OUT_HOST, job_uuid="l2",
                                 deleted_file_ids=[11, 13])
    keep = np.isin(want["_data_file_id"], [10, 12])
    kept = {k: v[keep] for k, v in want.items()}
    assert st2["rows_out"] == keep.sum()
    _check_index(res2, kept, ["k"], ["v1", "_data_file_id"], 5, "l2")
    res.free()
    res2.free()


def test_create_index_with_nulls(ctx, tmp_path):
    """Nulls in the indexed column (hash unchanged -> bucket pmod(42, n); sorted first) and in included columns."""
    from hyperspace_b200 import _native

    rng = np.random.default_rng(31)
    n = 70_000
    k = rng.integers(-500, 500, size=n, dtype=np.int64)
    kvalid = rng.random(n) > 0.05
    v1 = rng.integers(0, 100, size=n, dtype=np.int32)
    v1valid = rng.random(n) > 0.3
    v2 = rng.standard_normal(n)
    v2valid = rng.random(n) > 0.9          # mostly null
    v3 = rng.standard_normal(n).astype(np.float32)
    tbl = pa.table({"k": pa.array(k, mask=~kvalid), "v1": pa.array(v1, mask=~v1valid), "v2": pa.array(v2, mask=~v2valid),
                    "v3": pa.array(v3)})
    for variant, kw in (("plain", dict(use_dictionary=False)), ("dict", dict(use_dictionary=True, data_page_size=8192)),
                        ("snappy", dict(use_dictionary=True, compression="snappy", data_page_version="2.0"))):
        p = str(tmp_path / f"n-{variant}.parquet")
        pq.write_table(tbl, p, **{"compression": "NONE", "row_group_size": 25_000, **kw})
        res, st = ctx.create_index([_native.FileImage(path=p)], ["k"], ["v1", "v2", "v3"], 16, output=_native.HS_OUT_HOST,
                                   job_uuid="nn", rows_per_page=8192, rows_per_row_group=16384)
        kz = np.where(kvalid, k, 0)
        perm, offs, order = O.index_rows({"k": kz, "v1": v1, "v2": v2, "v3": v3}, ["k"], ["v1", "v2", "v3"], 16,
                                         valids={"k": kvalid.astype(np.uint8)})
        masks = {"k": kvalid, "v1": v1valid, "v2": v2valid, "v3": np.ones(n, bool)}
        vals = {"k": k, "v1": v1, "v2": v2, "v3": v3}
        total = 0
        for i, f in enumerate(res.files):
            t = _read_image(res.host_bytes(i))
            lo, hi = int(offs[f.bucket]), int(offs[f.bucket + 1])
            assert t.num_rows == hi - lo
            for name in order:
                arr = t.column(name).combine_chunks()
                got_valid = np.asarray(arr.is_valid())
                want_valid = masks[name][perm[lo:hi]]
                assert np.array_equal(got_valid, want_valid), (variant, name, f.bucket)
                got = np.asarray(arr.fill_null(0))
                want = np.where(want_valid, vals[name][perm[lo:hi]], 0).astype(got.dtype)
                assert np.array_equal(_bits(got), _bits(want)), (variant, name, f.bucket)
            total += t.num_rows
        assert total == n
        # the GPU reads its own nullable files back: filter scan over the index == numpy
        batch, _ = ctx.filter_scan(res.as_sources(), "k", ["k", "v1"], lo=-10, hi=10, sorted_on_key=False)
        m = kvalid & (k >= -10) & (k <= 10)
        assert batch.num_rows == int(m.sum())
        res.free()


@pytest.mark.parametrize("nb", [1024, 1025, 4096])
def test_create_index_on_both_sides_of_the_fused_partition(ctx, tmp_path, nb):
    """Up to 1024 buckets k_partition_rows moves the rows; above, k_partition_dest + k_scatter at widths 8, 4 and 1."""
    from hyperspace_b200 import _native

    rng = np.random.default_rng(nb)
    n = 300_000
    cols = {"k": rng.integers(-2**63, 2**63 - 1, size=n, dtype=np.int64), "a": rng.integers(-2**40, 2**40, size=n, dtype=np.int64),
            "d": rng.standard_normal(n), "i": rng.integers(-1000, 1000, size=n, dtype=np.int32),
            "f": rng.standard_normal(n).astype(np.float32)}
    ivalid = rng.random(n) > 0.3
    p = str(tmp_path / "s.parquet")
    pq.write_table(pa.table({**cols, "i": pa.array(cols["i"], mask=~ivalid)}), p, compression="NONE", use_dictionary=False)
    ctx.profile_enable(True)
    try:
        res, st = ctx.create_index([_native.FileImage(path=p)], ["k"], ["a", "d", "i", "f"], nb, output=_native.HS_OUT_HOST,
                                   job_uuid="fp")
        kernels = ctx.profile_report()
    finally:
        ctx.profile_enable(False)
    assert ("k_partition_dest" in kernels) == (nb > 1024) and ("k_partition_rows" in kernels) == (nb <= 1024), kernels
    assert st["rows_out"] == n
    perm, offs, order = O.index_rows(cols, ["k"], ["a", "d", "i", "f"], nb)
    masks = {name: np.ones(n, bool) for name in order}
    masks["i"] = ivalid
    total = 0
    for i, f in enumerate(res.files):
        assert f.name == O.bucket_file_name(f.bucket, "fp")
        t = _read_image(res.host_bytes(i))
        lo, hi = int(offs[f.bucket]), int(offs[f.bucket + 1])
        assert t.num_rows == hi - lo and t.column_names == order
        for name in order:
            arr = t.column(name).combine_chunks()
            want_valid = masks[name][perm[lo:hi]]
            assert np.array_equal(np.asarray(arr.is_valid()), want_valid), (name, f.bucket)
            got = np.asarray(arr.fill_null(0))
            want = np.where(want_valid, cols[name][perm[lo:hi]], 0).astype(got.dtype)
            assert np.array_equal(_bits(got), _bits(want)), (name, f.bucket)
        total += t.num_rows
    assert total == n
    res.free()


def test_errors_are_loud(ctx, tmp_path):
    from hyperspace_b200 import _native

    cols = O.synthetic_table(0, 1000, 2)
    p = str(tmp_path / "s.parquet")
    pq.write_table(pa.table(cols), p, compression="zstd")
    with pytest.raises(_native.HyperspaceGpuError) as e:
        ctx.create_index([_native.FileImage(path=p)], ["k"], ["v1"], 4, output=_native.HS_OUT_HOST)
    assert e.value.code == _native.HS_EUNSUPPORTED
    p2 = str(tmp_path / "u.parquet")
    pq.write_table(pa.table(cols), p2, compression="NONE")
    with pytest.raises(_native.HyperspaceGpuError) as e:
        ctx.create_index([_native.FileImage(path=p2)], ["nope"], ["v1"], 4, output=_native.HS_OUT_HOST)
    assert e.value.code == _native.HS_EINVAL
    with pytest.raises(_native.HyperspaceGpuError) as e:
        ctx.create_index([_native.FileImage(path=str(tmp_path / "missing.parquet"))], ["k"], [], 4, output=_native.HS_OUT_HOST)
    assert e.value.code == _native.HS_EIO
    with pytest.raises(_native.HyperspaceGpuError):
        ctx.create_index([_native.FileImage(data=b"PAR1 this is not parquet PAR1")], ["k"], [], 4, output=_native.HS_OUT_HOST)
    # the context survives errors
    b, _ = ctx.k_bucket_ids([np.array([1], dtype=np.int64)], 200)
    assert b.tolist() == [69]


def test_empty_source(ctx, tmp_path):
    from hyperspace_b200 import _native

    p = str(tmp_path / "e.parquet")
    pq.write_table(pa.table({"k": np.empty(0, np.int64), "v1": np.empty(0, np.int64)}), p, compression="NONE")
    res, st = ctx.create_index([_native.FileImage(path=p)], ["k"], ["v1"], 8, output=_native.HS_OUT_HOST)
    assert st["rows_out"] == 0 and len(res.files) == 0
    res.free()


# ---------------------------------------------------------------------------------------------------------------------
# read side
# ---------------------------------------------------------------------------------------------------------------------

def _index_in_memory(ctx, cols, indexed, included, nb, uuid):
    from hyperspace_b200 import _native

    sink = io.BytesIO()
    pq.write_table(pa.table(cols), sink, compression="NONE")
    res, _ = ctx.create_index([_native.FileImage(data=sink.getvalue())], indexed, included, nb, output=_native.HS_OUT_HOST,
                              job_uuid=uuid)
    return res


def test_filter_scan_matches_unindexed_answer(ctx):
    rng = np.random.default_rng(17)
    n = 150_000
    cols = {"k": rng.integers(-10_000, 10_000, size=n, dtype=np.int64), "v1": rng.integers(0, 1000, size=n, dtype=np.int64),
            "v2": rng.standard_normal(n)}
    res = _index_in_memory(ctx, cols, ["k"], ["v1", "v2"], 20, "f")
    for lo, hi in ((-100, 100), (None, -9_990), (9_000, None), (5, 5), (20_000, 30_000)):
        batch, st = ctx.filter_scan(res.as_sources(), "k", ["k", "v2", "v1"], lo=lo, hi=hi)
        m = np.ones(n, bool)
        if lo is not None:
            m &= cols["k"] >= lo
        if hi is not None:
            m &= cols["k"] <= hi
        assert batch.num_rows == m.sum()
        got = np.rec.fromarrays([batch.column("k"), batch.column("v1"), _bits(batch.column("v2"))])
        want = np.rec.fromarrays([cols["k"][m], cols["v1"][m], _bits(cols["v2"][m])])
        assert np.array_equal(np.sort(got), np.sort(want))  # verifyIndexUsage: sorted rows identical
        # unsorted (source-file) scan path gives the same answer
        batch2, _ = ctx.filter_scan(res.as_sources(), "k", ["k", "v2", "v1"], lo=lo, hi=hi, sorted_on_key=False)
        got2 = np.rec.fromarrays([batch2.column("k"), batch2.column("v1"), _bits(batch2.column("v2"))])
        assert np.array_equal(np.sort(got2), np.sort(want))
    res.free()


def test_bucket_join_matches_oracle(ctx):
    rng = np.random.default_rng(23)
    nl, nr, nb = 80_000, 60_000, 16
    L = {"k": rng.integers(0, 40_000, size=nl, dtype=np.int64), "v1": np.arange(nl, dtype=np.int64)}
    R = {"k": rng.integers(0, 40_000, size=nr, dtype=np.int64), "v2": np.arange(nr, dtype=np.float64) * 0.5}
    li = _index_in_memory(ctx, L, ["k"], ["v1"], nb, "L")
    ri = _index_in_memory(ctx, R, ["k"], ["v2"], nb, "R")
    batch, st = ctx.bucket_join(li.as_sources(), [f.bucket for f in li.files], ri.as_sources(), [f.bucket for f in ri.files],
                                nb, "k", "k", ["k", "v1"], ["v2"])
    # oracle: per bucket merge join of the sorted buckets
    want = []
    lperm, loffs, _ = O.index_rows(L, ["k"], ["v1"], nb)
    rperm, roffs, _ = O.index_rows(R, ["k"], ["v2"], nb)
    for b in range(nb):
        lp, rp = lperm[loffs[b]:loffs[b + 1]], rperm[roffs[b]:roffs[b + 1]]
        a, c = O.merge_join(L["k"][lp], R["k"][rp])
        want.append(np.rec.fromarrays([L["k"][lp][a], L["v1"][lp][a], _bits(R["v2"][rp][c])]))
    want = np.concatenate(want)
    got = np.rec.fromarrays([batch.column("k"), batch.column("v1"), _bits(batch.column("v2"))])
    assert batch.num_rows == len(want)
    assert np.array_equal(got, want)  # same (bucket, left row, right row) order as the oracle
    li.free()
    ri.free()


def test_bucket_join_with_multi_file_buckets(ctx):
    """After an incremental refresh a bucket holds several files; the join re-sorts them (Spark adds a SortExec)."""
    from hyperspace_b200 import _native

    rng = np.random.default_rng(29)
    nb = 8
    L1 = {"k": rng.integers(0, 5_000, size=20_000, dtype=np.int64), "v1": np.arange(20_000, dtype=np.int64)}
    L2 = {"k": rng.integers(0, 5_000, size=7_000, dtype=np.int64), "v1": np.arange(20_000, 27_000, dtype=np.int64)}
    R = {"k": rng.integers(0, 5_000, size=15_000, dtype=np.int64), "v2": np.arange(15_000, dtype=np.float64)}
    a, b2, r = (_index_in_memory(ctx, t, ["k"], [c], nb, u) for t, c, u in ((L1, "v1", "a"), (L2, "v1", "b"), (R, "v2", "r")))
    left = a.as_sources() + b2.as_sources()
    lb = [f.bucket for f in a.files] + [f.bucket for f in b2.files]
    batch, _ = ctx.bucket_join(left, lb, r.as_sources(), [f.bucket for f in r.files], nb, "k", "k", ["v1"], ["v2"])
    Lk = np.concatenate([L1["k"], L2["k"]])
    Lv = np.concatenate([L1["v1"], L2["v1"]])
    order = np.argsort(R["k"], kind="stable")
    pos_lo = np.searchsorted(R["k"][order], Lk, "left")
    pos_hi = np.searchsorted(R["k"][order], Lk, "right")
    want = sorted((int(Lv[i]), float(R["v2"][order[j]])) for i in range(len(Lk)) for j in range(pos_lo[i], pos_hi[i]))
    got = sorted(zip(batch.column("v1").tolist(), batch.column("v2").tolist()))
    assert got == want
    for x in (a, b2, r):
        x.free()


def test_read_side_with_int32_keys(ctx):
    """IntegerType keys (hashInt buckets): filter scan and bucket join widen the key on the GPU."""
    rng = np.random.default_rng(31)
    nl, nr, nb = 50_000, 30_000, 12
    L = {"k": rng.integers(-20_000, 20_000, size=nl, dtype=np.int32), "v1": np.arange(nl, dtype=np.int64)}
    R = {"k": rng.integers(-20_000, 20_000, size=nr, dtype=np.int32), "v2": np.arange(nr, dtype=np.float64)}
    li = _index_in_memory(ctx, L, ["k"], ["v1"], nb, "L")
    ri = _index_in_memory(ctx, R, ["k"], ["v2"], nb, "R")
    for lo, hi in ((-50, 50), (None, -19_900), (7, 7)):
        for sorted_on_key in (True, False):
            batch, _ = ctx.filter_scan(li.as_sources(), "k", ["k", "v1"], lo=lo, hi=hi, sorted_on_key=sorted_on_key)
            m = np.ones(nl, bool)
            if lo is not None:
                m &= L["k"] >= lo
            if hi is not None:
                m &= L["k"] <= hi
            assert batch.column("k").dtype == np.int32
            got = np.rec.fromarrays([batch.column("k"), batch.column("v1")])
            assert np.array_equal(np.sort(got), np.sort(np.rec.fromarrays([L["k"][m], L["v1"][m]])))
    batch, _ = ctx.bucket_join(li.as_sources(), [f.bucket for f in li.files], ri.as_sources(), [f.bucket for f in ri.files],
                               nb, "k", "k", ["k", "v1"], ["v2"])
    want = []
    lperm, loffs, _ = O.index_rows(L, ["k"], ["v1"], nb)
    rperm, roffs, _ = O.index_rows(R, ["k"], ["v2"], nb)
    for b in range(nb):
        lp, rp = lperm[loffs[b]:loffs[b + 1]], rperm[roffs[b]:roffs[b + 1]]
        a, c = O.merge_join(L["k"][lp].astype(np.int64), R["k"][rp].astype(np.int64))
        want.append(np.rec.fromarrays([L["k"][lp][a], L["v1"][lp][a], _bits(R["v2"][rp][c])]))
    want = np.concatenate(want)
    got = np.rec.fromarrays([batch.column("k"), batch.column("v1"), _bits(batch.column("v2"))])
    assert np.array_equal(got, want)
    # a long-keyed index is bucketed with hashLong: pairing it with an int-keyed one must be refused
    R64 = {"k": R["k"].astype(np.int64), "v2": R["v2"]}
    r64 = _index_in_memory(ctx, R64, ["k"], ["v2"], nb, "R64")
    with pytest.raises(Exception, match="different types"):
        ctx.bucket_join(li.as_sources(), [f.bucket for f in li.files], r64.as_sources(), [f.bucket for f in r64.files],
                        nb, "k", "k", ["v1"], ["v2"])
    for x in (li, ri, r64):
        x.free()


def test_key_statistics_in_index_files(ctx):
    """Every row group of an index file carries min / max of the (sorted) indexed column, so a Parquet reader can prune."""
    rng = np.random.default_rng(37)
    n = 60_000
    for dtype in (np.int64, np.int32):
        cols = {"k": rng.integers(-1_000_000, 1_000_000, size=n).astype(dtype), "v": rng.integers(0, 9, size=n, dtype=np.int64)}
        from hyperspace_b200 import _native

        sink = io.BytesIO()
        pq.write_table(pa.table(cols), sink, compression="NONE")
        res, _ = ctx.create_index([_native.FileImage(data=sink.getvalue())], ["k"], ["v"], 5, output=_native.HS_OUT_HOST,
                                  job_uuid="s", rows_per_row_group=2_000, rows_per_page=500)
        seen = 0
        for i in range(len(res.files)):
            image = res.host_bytes(i)
            pf = pq.ParquetFile(io.BytesIO(image))
            assert pf.metadata.num_row_groups > 1
            tbl = pf.read()
            r0 = 0
            for g in range(pf.metadata.num_row_groups):
                rg = pf.metadata.row_group(g)
                st = rg.column(0).statistics
                assert st is not None and st.has_min_max and st.null_count == 0
                k = tbl.column("k").to_numpy()[r0:r0 + rg.num_rows]
                assert st.min == k.min() == k[0] and st.max == k.max() == k[-1]
                r0 += rg.num_rows
                seen += rg.num_rows
            # the statistics drive row-group pruning in any Parquet reader
            probe = int(tbl.column("k")[len(tbl) // 2].as_py())
            hit = pq.read_table(io.BytesIO(image), filters=[("k", "==", probe)])
            assert len(hit) == int((tbl.column("k").to_numpy() == probe).sum())
        assert seen == n
        res.free()


# ---------------------------------------------------------------------------------------------------------------------
# late-materialised dictionary columns (codes instead of values between decode and encode)
# ---------------------------------------------------------------------------------------------------------------------

def _index_images(ctx, files, indexed, included, nb, uuid, **kw):
    from hyperspace_b200 import _native

    res, st = ctx.create_index(files, indexed, included, nb, output=_native.HS_OUT_HOST, job_uuid=uuid, **kw)
    images = {f.name: res.host_bytes(i) for i, f in enumerate(res.files)}
    return res, images, st


def test_late_materialised_columns_give_identical_files(ctx, tmp_path, monkeypatch):
    """The code-carrying path and the value path must produce byte-identical index files (HS_NO_CARRY switches it off)."""
    from hyperspace_b200 import _native

    rng = np.random.default_rng(41)
    n = 120_000
    cols = {
        "k": rng.integers(-2**62, 2**62, size=n, dtype=np.int64),
        "a": rng.integers(0, 900, size=n, dtype=np.int64) - 1,          # contains -1 == the hash sets' empty marker
        "b": rng.integers(-3, 60, size=n).astype(np.int32),
        "c": (rng.integers(0, 2000, size=n) * 0.5).astype(np.float64),
        "d": np.where(rng.integers(0, 4, size=n) == 0, np.float32("nan"), rng.integers(0, 7, size=n).astype(np.float32)),
        "e": rng.integers(0, 3, size=n, dtype=np.int64),                 # fifth and sixth dictionary columns: more than one
        "f": rng.integers(0, 300, size=n).astype(np.int32),              # record holds -> mapped by the encoder instead
        "g": rng.standard_normal(n),                                      # high cardinality: pyarrow falls back to PLAIN pages
    }
    included = ["a", "b", "c", "d", "e", "f", "g"]
    paths = _write_sources(tmp_path, cols, 3, use_dictionary=True, data_page_version="1.0", row_group_size=25_000,
                           dictionary_pagesize_limit=256 * 1024)
    files = [_native.FileImage(path=p) for p in paths]
    res1, img1, st1 = _index_images(ctx, files, ["k"], included, 16, "lm", rows_per_page=4096, rows_per_row_group=8192)
    _check_index(res1, cols, ["k"], included, 16, "lm")
    md = pq.ParquetFile(pa.BufferReader(next(iter(img1.values())))).metadata.row_group(0)
    assert all(md.column(i).has_dictionary_page for i in range(1, 7)) and not md.column(7).has_dictionary_page
    monkeypatch.setenv("HS_NO_CARRY", "1")
    res2, img2, st2 = _index_images(ctx, files, ["k"], included, 16, "lm", rows_per_page=4096, rows_per_row_group=8192)
    monkeypatch.delenv("HS_NO_CARRY")
    assert img1.keys() == img2.keys()
    for name in img1:
        assert img1[name] == img2[name], name
    res1.free()
    res2.free()


def test_late_materialisation_falls_back_when_pages_differ(ctx, tmp_path):
    """A column that is dictionary-encoded in one source file and PLAIN (or nullable) in another takes the value path."""
    from hyperspace_b200 import _native

    rng = np.random.default_rng(43)
    n = 30_000
    cols = {"k": rng.integers(0, 10**9, size=n, dtype=np.int64), "a": rng.integers(0, 50, size=n, dtype=np.int64),
            "b": rng.integers(0, 9, size=n).astype(np.int32)}
    p1, p2 = str(tmp_path / "s1.parquet"), str(tmp_path / "s2.parquet")
    half = n // 2
    pq.write_table(pa.table({k: v[:half] for k, v in cols.items()}), p1, compression="NONE", use_dictionary=True)
    pq.write_table(pa.table({k: v[half:] for k, v in cols.items()}), p2, compression="NONE", use_dictionary=["b"])
    res, _ = ctx.create_index([_native.FileImage(path=p1), _native.FileImage(path=p2)], ["k"], ["a", "b"], 8,
                              output=_native.HS_OUT_HOST, job_uuid="fb")
    _check_index(res, cols, ["k"], ["a", "b"], 8, "fb")
    res.free()
    # nulls in a dictionary-encoded column: not carried, still correct (checked against pyarrow's own reading)
    a = pa.array([None if i % 7 == 0 else int(i % 5) for i in range(n)], type=pa.int64())
    t = pa.table({"k": cols["k"], "a": a})
    p3 = str(tmp_path / "s3.parquet")
    pq.write_table(t, p3, compression="NONE", use_dictionary=True)
    res, _ = ctx.create_index([_native.FileImage(path=p3)], ["k"], ["a"], 4, output=_native.HS_OUT_HOST, job_uuid="nn")
    got = pa.concat_tables([_read_image(res.host_bytes(i)) for i in range(len(res.files))]).sort_by("k")
    want = t.sort_by("k")
    assert got.column("a").to_pylist() == want.column("a").to_pylist()
    res.free()
