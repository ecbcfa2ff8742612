"""GPU tests of the key pages that the local sort writes itself.

For a single null-free int32 / int64 key the index files are laid out before the sort, and k_local_sort stores every
sorted key, decoded, straight into its PLAIN page body: k_gather_encode then runs for the included columns only.
HS_LSD_SORT=1 takes the LSD passes, after which k_gather_encode writes the key as before.  Both must give byte-identical
files, in every page layout: work items that cross page boundaries (4096-row pages), tiny pages whose bodies are not
8-byte aligned, several row groups with min / max statistics, SNAPPY pages, and a table with a nullable included column,
whose pages are laid out after the sort."""
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


def _build(ctx, table, nb, lsd, **kw):
    """Index files of `table` on column k (name -> bytes) and the kernels that ran."""
    from hyperspace_b200 import _native as N

    sink = io.BytesIO()
    pq.write_table(table, sink, compression="NONE")
    included = [c for c in table.column_names if c != "k"]
    if lsd:
        os.environ["HS_LSD_SORT"] = "1"
    try:
        ctx.profile_enable(True)
        res, _ = ctx.create_index([N.FileImage(data=sink.getvalue())], ["k"], included, nb, output=N.HS_OUT_HOST,
                                  job_uuid="kp", **kw)
        kernels = ctx.profile_report()
    finally:
        ctx.profile_enable(False)
        os.environ.pop("HS_LSD_SORT", None)
    files = {f.name: res.host_bytes(i) for i, f in enumerate(res.files)}
    buckets = {f.name: f.bucket for f in res.files}
    res.free()
    return files, buckets, kernels


def _check_files(files, buckets, cols, nb):
    """pyarrow reads every file as the oracle's rows, and every row group's key statistics are its first / last key."""
    perm, offs, order = O.index_rows(cols, ["k"], [c for c in cols if c != "k"], nb)
    for name, image in files.items():
        b = buckets[name]
        lo, hi = int(offs[b]), int(offs[b + 1])
        pf = pq.ParquetFile(io.BytesIO(image))
        t = pf.read()
        assert t.column_names == order
        for c in order:
            assert np.array_equal(t.column(c).to_numpy(), cols[c][perm[lo:hi]]), (c, b)
        k = t.column("k").to_numpy()
        r0 = 0
        for g in range(pf.metadata.num_row_groups):
            rg = pf.metadata.row_group(g)
            st = rg.column(0).statistics
            assert st is not None and st.has_min_max
            assert st.min == k[r0] == k[r0:r0 + rg.num_rows].min()
            assert st.max == k[r0 + rg.num_rows - 1] == k[r0:r0 + rg.num_rows].max()
            r0 += rg.num_rows
        assert r0 == hi - lo


# (rows, buckets, create_index keywords)
LAYOUTS = {
    # one bucket of 49 x 4096 + 1 rows: the MSD pass + local sort, work items of up to 12 288 rows across 4096-row pages,
    # a last page of one row (its body is not 8-byte aligned)
    "msd_4096_row_pages": (49 * 4096 + 1, 1, dict(rows_per_page=4096, rows_per_row_group=3 * 4096)),
    # ~15 rows per bucket: whole buckets sorted from the raw column, every page tiny and most bodies unaligned
    "tiny_pages": (3_000, 200, dict(rows_per_page=4096, dictionary=False)),
    # several buckets on the MSD path with several row groups each, then the default page size
    "msd_buckets": (1_000_000, 16, dict(rows_per_page=4096, rows_per_row_group=5 * 4096)),
    "default_pages": (1_000_000, 7, dict()),
    # the files laid out again after compression: statistics are patched into the second layout
    "snappy": (300_000, 5, dict(rows_per_page=4096, rows_per_row_group=4 * 4096, compression="snappy")),
}


@pytest.mark.parametrize("dtype", [np.int64, np.int32])
@pytest.mark.parametrize("layout", list(LAYOUTS))
def test_sort_written_key_pages_equal_gathered_ones(ctx, layout, dtype):
    from hyperspace_b200 import _native as N

    n, nb, kw = LAYOUTS[layout]
    if kw.get("compression") == "snappy":
        kw = dict(kw, compression=N.HS_CODEC_SNAPPY)
    rng = np.random.default_rng(n + nb)
    info = np.iinfo(dtype)
    cols = {"k": rng.integers(info.min, info.max, size=n, dtype=dtype, endpoint=True),
            "v": rng.integers(0, 50, size=n, dtype=np.int64), "w": rng.standard_normal(n)}
    cols["k"][:4] = [info.min, info.max, 0, -1]
    table = pa.table(cols)
    local, buckets, k_local = _build(ctx, table, nb, lsd=False, **kw)
    lsd, _, k_lsd = _build(ctx, table, nb, lsd=True, **kw)
    assert "k_local_sort" in k_local and "k_local_sort" not in k_lsd
    # the key's pages came from the sort: one gather launch less
    assert k_local["k_gather_encode"]["launches"] == k_lsd["k_gather_encode"]["launches"] - 1
    assert local == lsd
    _check_files(local, buckets, cols, nb)


def test_nullable_included_column_lays_out_after_the_sort(ctx):
    """A nullable column's page sizes depend on the sorted order: the files are laid out after the sort, which keeps its
    keys, and the key is written by k_gather_encode."""
    n, nb = 400_000, 9
    rng = np.random.default_rng(5)
    k = rng.integers(-2**63, 2**63 - 1, size=n, dtype=np.int64)
    v = rng.integers(0, 1 << 40, size=n, dtype=np.int64)
    v_valid = rng.random(n) > 0.2
    table = pa.table({"k": k, "v": pa.array(v, mask=~v_valid), "w": rng.standard_normal(n)})
    kw = dict(rows_per_page=4096, rows_per_row_group=8 * 4096)
    local, buckets, k_local = _build(ctx, table, nb, lsd=False, **kw)
    lsd, _, k_lsd = _build(ctx, table, nb, lsd=True, **kw)
    assert "k_local_sort" in k_local
    assert k_local["k_gather_encode"]["launches"] == k_lsd["k_gather_encode"]["launches"]
    assert local == lsd
    perm, offs, _ = O.index_rows({"k": k}, ["k"], [], nb)
    for name, image in local.items():
        b = buckets[name]
        lo, hi = int(offs[b]), int(offs[b + 1])
        pf = pq.ParquetFile(io.BytesIO(image))
        t = pf.read()
        assert np.array_equal(t.column("k").to_numpy(), k[perm[lo:hi]])
        got_v = t.column("v")
        assert np.array_equal(got_v.is_valid().to_numpy(zero_copy_only=False), v_valid[perm[lo:hi]])
        assert np.array_equal(got_v.fill_null(0).to_numpy(), np.where(v_valid, v, 0)[perm[lo:hi]])
        r0 = 0
        for g in range(pf.metadata.num_row_groups):
            rg = pf.metadata.row_group(g)
            st = rg.column(0).statistics
            assert st.min == t.column("k")[r0].as_py() and st.max == t.column("k")[r0 + rg.num_rows - 1].as_py()
            r0 += rg.num_rows
