"""GPU tests of the shared-memory local sort (k_local_sort) and of the choice between it and the LSD passes.

A null-free fixed-width first key column is sorted straight from the raw column when every bucket fits one CTA, after
one MSD pass on the 8 bits below the highest varying bit when the (bucket, digit) sub-buckets fit, and with the LSD
passes + tie-run fix-up otherwise.  Every case must equal the oracle's stable order exactly, and the kernels that ran
show which path it took."""
import os

import numpy as np
import pytest

from oracle import oracle as O

pytestmark = pytest.mark.gpu

LOCAL_CAP = 12288  # kLocalSortCap


@pytest.fixture(scope="module")
def ctx():
    from hyperspace_b200 import _native

    c = _native.Context(0)
    yield c
    c.close()


def _sorted_and_kernels(ctx, cols, nb):
    ctx.profile_enable(True)
    try:
        perm, offs = ctx.k_sort_perm(cols, nb)
        kernels = ctx.profile_report()
    finally:
        ctx.profile_enable(False)
    b = O.bucket_ids(cols, nb)
    want_perm, want_offs = O.sort_perm(cols, nb, b)
    assert np.array_equal(offs, want_offs)
    assert np.array_equal(perm, want_perm)
    return offs, kernels


def _specials(a):
    a = a.copy()
    a[:7] = [0.0, -0.0, np.nan, np.inf, -np.inf, -0.0, np.nan]
    return a


N_BIG = 4_000_000  # 8 buckets of ~500 K rows: above the local sort's capacity, below one MSD level's


def _big_keys():
    rng = np.random.default_rng(11)
    n = N_BIG
    uniform = rng.integers(-2**63, 2**63 - 1, size=n, dtype=np.int64)
    # floating-point keys with magnitudes spread over most exponents (the MSD digit is the sign and the exponent's top bits)
    f64 = rng.standard_normal(n) * 10.0 ** rng.uniform(-300, 300, size=n)
    f32 = (rng.standard_normal(n) * 10.0 ** rng.uniform(-30, 30, size=n)).astype(np.float32)
    return {
        "uniform_int64": [uniform],
        "sequential_ids": [np.arange(n, dtype=np.int64)],
        "negative_int64": [-rng.integers(1, 2**40, size=n, dtype=np.int64)],
        "int32": [rng.integers(-2**31, 2**31 - 1, size=n, dtype=np.int32)],
        "float64": [_specials(f64)],
        "float32": [_specials(f32)],
        "two_columns": [rng.integers(-3, 3, size=n, dtype=np.int32), uniform],
        # the top byte spreads the rows over the MSD digit; under it only 50 values (in three bytes): runs of equal prefixes
        # far longer than the insertion sort takes, and ties on the whole key
        "heavy_ties": [(rng.integers(0, 256, size=n, dtype=np.int64) << 56) | (rng.integers(0, 50, size=n, dtype=np.int64) * 0x10101)],
    }


@pytest.mark.parametrize("case", list(_big_keys()))
def test_msd_then_local_sort_matches_oracle(ctx, case):
    cols = _big_keys()[case]
    offs, kernels = _sorted_and_kernels(ctx, cols, 8)
    assert np.diff(offs).max() > LOCAL_CAP
    assert "k_local_sort" in kernels, sorted(kernels)
    if len(cols) == 1:  # one MSD scatter; an earlier key column is sorted with its own LSD passes (+ fix-up)
        assert "k_fix_runs" not in kernels, sorted(kernels)
        assert kernels["k_sort_scatter"]["launches"] == 1, kernels["k_sort_scatter"]


def test_skewed_msd_digit_falls_back_to_lsd_passes(ctx):
    """A third of the rows share one value of the MSD digit, so that digit's sub-bucket of every bucket is larger than the
    local sort's capacity: the rows are sorted with the LSD passes + tie-run fix-up instead."""
    rng = np.random.default_rng(12)
    n = N_BIG
    k = rng.integers(0, 2**62, size=n, dtype=np.int64)
    k[rng.random(n) < 1 / 3] &= ~(np.int64(0xff) << 54)  # bits 54..61: the digit under the highest varying bit (61)
    offs, kernels = _sorted_and_kernels(ctx, [k], 8)
    assert "k_local_sort" not in kernels, sorted(kernels)
    assert "k_fix_runs" in kernels, sorted(kernels)


@pytest.mark.parametrize("n,nb", [(100_000, 16), (12_288, 1), (50_000, 200)])
def test_small_buckets_are_sorted_from_the_raw_column(ctx, n, nb):
    rng = np.random.default_rng(n)
    for cols in ([rng.integers(-2**63, 2**63 - 1, size=n, dtype=np.int64)], [_specials(rng.standard_normal(n))],
                 [_specials(rng.standard_normal(n).astype(np.float32))], [rng.integers(0, 1000, size=n, dtype=np.int32)]):
        offs, kernels = _sorted_and_kernels(ctx, cols, nb)
        assert np.diff(offs).max() <= LOCAL_CAP
        assert "k_local_sort" in kernels, sorted(kernels)
        assert "k_sort_scatter" not in kernels and "k_sort_hist" not in kernels, sorted(kernels)


def test_lsd_switch_gives_byte_identical_files(ctx):
    """The benchmark's shape: 64 M rows in 200 buckets take the MSD pass + local sort; HS_LSD_SORT=1 forces the LSD passes
    + tie-run fix-up.  The index files must be byte-identical."""
    from hyperspace_b200 import _native as N

    rows, nb = 64_000_000, 200
    src = ctx.synth_table(0, rows, 5, n_files=64, row_groups_per_file=2, output=N.HS_OUT_DEVICE)
    built = {}
    for lsd in (False, True):
        if lsd:
            os.environ["HS_LSD_SORT"] = "1"
        try:
            ctx.profile_enable(True)
            res, _ = ctx.create_index(src.as_sources(), ["k"], ["v1", "v2", "v3", "v4"], nb, output=N.HS_OUT_HOST,
                                      job_uuid="lsd")
            kernels = ctx.profile_report()
            ctx.profile_enable(False)
        finally:
            os.environ.pop("HS_LSD_SORT", None)
        assert ("k_local_sort" in kernels) != lsd, sorted(kernels)
        assert ("k_fix_runs" in kernels) == lsd, sorted(kernels)
        built[lsd] = {f.name: res.host_bytes(i) for i, f in enumerate(res.files)}
        res.free()
    src.free()
    assert len(built[False]) == nb
    assert built[False] == built[True]
    ctx.trim()
