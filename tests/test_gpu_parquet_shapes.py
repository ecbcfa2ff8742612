"""GPU tests of the Parquet page decoder on hand-built files (tests/parquet_shapes.py), each placed where the decoder
changes path: every case decoded in full by the unsorted scan, bit for bit with its validity; createIndex on every case
with fixed-width columns against the oracle, byte-identical with late materialisation and zero copy switched off; sorted
scans whose row windows start and end on page edges; and the refusal of an unsupported encoding and of a nested column."""
import numpy as np
import pyarrow as pa
import pyarrow.parquet as pq
import pytest

import filter_oracle as F
import parquet_shapes as S
from oracle import oracle as O

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    from hyperspace_b200 import _native

    c = _native.Context(0)
    yield c
    c.close()


def _files(images):
    from hyperspace_b200 import _native

    return [_native.FileImage(data=img) for img in images]


def _bits(a):
    a = np.ascontiguousarray(a)
    return a.view({1: np.uint8, 4: np.uint32, 8: np.uint64}[a.dtype.itemsize])


def _check_column(name, got, got_valid, values, valid):
    n = len(values)
    assert len(got) == n, (name, len(got), n)
    want_valid = np.ones(n, bool) if valid is None else valid
    have_valid = np.ones(n, bool) if got_valid is None else np.asarray(got_valid).astype(bool)
    bad = np.flatnonzero(have_valid != want_valid)
    assert not len(bad), f"{name}: validity differs at {len(bad)} rows, first at row {bad[0]}"
    if values.dtype == object:
        diff = [i for i in np.flatnonzero(want_valid) if got[i] != values[i]]
        assert not diff, f"{name}: {len(diff)} strings differ, first at row {diff[0]}"
        return
    g, w = _bits(np.asarray(got).astype(values.dtype)), _bits(values)
    bad = np.flatnonzero((g != w) & want_valid)
    assert not len(bad), f"{name}: {len(bad)} values differ, first at row {bad[0]}: {g[bad[0]]:#x} != {w[bad[0]]:#x}"


@pytest.mark.parametrize("name", list(S.CASES))
def test_scan_decodes_every_row(ctx, name):
    images, expected, specs = S.case_data(name)
    cols = [c.name for c in specs[0].cols]
    batch, st = ctx.filter_scan_where(_files(images), None, cols, [], sorted_on_key=False)
    assert batch.num_rows == len(expected["k"][0])
    for cname, data, valid in batch.columns:
        _check_column(cname, data, valid, *expected[cname])
    batch.free()


def _build(ctx, images, included, nb):
    from hyperspace_b200 import _native

    ctx.profile_enable(True)
    try:
        res, _ = ctx.create_index(_files(images), ["k"], included, nb, output=_native.HS_OUT_HOST, job_uuid="shapes")
        kernels = ctx.profile_report()
    finally:
        ctx.profile_enable(False)
    files = {f.name: (f.bucket, res.host_bytes(i)) for i, f in enumerate(res.files)}
    res.free()
    return files, kernels


INDEXED_CASES = [n for n in S.CASES if S.index_columns(n)]


@pytest.mark.parametrize("name", INDEXED_CASES)
def test_create_index_matches_oracle(ctx, monkeypatch, name):
    images, expected, _ = S.case_data(name)
    a = S.analyse(name)
    included = S.index_columns(name)
    nb = S.CLAIMS[name].get("nb", 4)
    files, kernels = _build(ctx, images, included, nb)
    perm, offs, order = O.index_rows({c: expected[c][0] for c in ["k"] + included}, ["k"], included, nb)
    assert sorted(b for b, _ in files.values()) == [b for b in range(nb) if offs[b + 1] > offs[b]]
    for bucket, data in files.values():
        t = pq.ParquetFile(pa.BufferReader(data)).read()
        lo, hi = int(offs[bucket]), int(offs[bucket + 1])
        assert t.column_names == order and t.num_rows == hi - lo
        for c in order:
            arr = t.column(c).combine_chunks()
            values, valid = expected[c]
            got = arr.fill_null(values.dtype.type(0)).to_numpy(zero_copy_only=False).astype(values.dtype)
            _check_column(f"{c} (bucket {bucket})", got, np.asarray(arr.is_valid()), values[perm[lo:hi]],
                          None if valid is None else valid[perm[lo:hi]])
    # the paths the profile shows: tiles for in-place columns exactly when a column is read in place; no dictionary
    # mapping pass when the only dictionary column travels as codes
    assert ("k_fill_zc_tiles" in kernels) == bool(a["zero_copy"]), (a["zero_copy"], sorted(kernels))
    if S.CLAIMS[name].get("no_dict_map"):
        assert a["carried"] and "k_dict_map" not in kernels, sorted(kernels)
    for switch in ("HS_NO_CARRY", "HS_NO_ZEROCOPY"):
        monkeypatch.setenv(switch, "1")
        other, kern = _build(ctx, images, included, nb)
        monkeypatch.delenv(switch)
        assert other == files, f"{name}: index files differ under {switch}=1"
        if switch == "HS_NO_ZEROCOPY":
            assert "k_fill_zc_tiles" not in kern


@pytest.fixture(scope="module")
def window_case():
    return S.case_data("windows_on_page_edges")


@pytest.mark.parametrize("lo_row,hi_row", S.window_queries())
def test_sorted_scan_windows_on_page_edges(ctx, window_case, lo_row, hi_row):
    """k = 6 r in file 0 and 6 r + 3 in file 1: [6 lo, 6 hi) selects rows [lo, hi) of both files."""
    images, expected, specs = window_case
    cols = ["k", "a", "b", "c"]
    preds = [("k", 6 * lo_row, False, 6 * hi_row, True)]
    batch, _ = ctx.filter_scan_where(_files(images), "k", cols, preds, sorted_on_key=True)
    mask = F.predicate_mask({c: expected[c][0] for c in cols}, preds,
                            {c: expected[c][1] for c in cols if expected[c][1] is not None})
    rows = np.flatnonzero(mask)
    assert batch.num_rows == len(rows)
    for cname, data, valid in batch.columns:
        values, v = expected[cname]
        _check_column(cname, data, valid, values[rows], None if v is None else v[rows])
    batch.free()


@pytest.mark.parametrize("name", list(S.REFUSALS))
def test_unsupported_shapes_are_refused(ctx, name):
    from hyperspace_b200 import _native

    specs, cols, word = S.REFUSALS[name]()
    files = _files([S.write_file(s) for s in specs])
    with pytest.raises(_native.HyperspaceGpuError) as e:
        ctx.filter_scan_where(files, None, list(cols), [], sorted_on_key=False)
    assert e.value.code == _native.HS_EUNSUPPORTED and word in e.value.message.lower(), e.value.message
    with pytest.raises(_native.HyperspaceGpuError) as e:
        ctx.create_index(files, ["k"], [c for c in cols if c != "k"], 4, output=_native.HS_OUT_HOST, job_uuid="r")
    assert e.value.code == _native.HS_EUNSUPPORTED and word in e.value.message.lower(), e.value.message
