"""GPU tests of the key sort at the limits where it changes path (tests/sort_edge_cases.py): every case must give the
oracle's stable order exactly, through the path the case names, with the default settings and with HS_LSD_SORT=1.
Then createIndex end to end on float and double keys and columns holding NaN payloads and -0.0, which must reach the
index files bit for bit, and a fix-up case through createIndex (the only caller that defers the fix-up's verdict)."""
import numpy as np
import pyarrow as pa
import pyarrow.parquet as pq
import pytest

import sort_edge_cases as S
from oracle import oracle as O

pytestmark = pytest.mark.gpu

SORT_KERNELS = ("k_sort_hist", "k_sort_scatter", "k_local_sort", "k_fix_runs")


@pytest.fixture(scope="module")
def ctx():
    from hyperspace_b200 import _native

    c = _native.Context(0)
    yield c
    c.close()


def _path_problem(path, kernels, plain):
    """Why the kernels that ran do not fit `path`, or None.  plain: one null-free key column; otherwise the other columns'
    passes and the validity pass add LSD passes of their own, and only the last column's choice is checked."""
    ran = set(kernels)
    if path in ("raw_local", "msd_local"):
        if "k_local_sort" not in ran:
            return "no k_local_sort"
        if plain and "k_fix_runs" in ran:
            return "k_fix_runs ran"
        if plain and path == "raw_local" and ran & {"k_sort_hist", "k_sort_scatter"}:
            return "a radix pass ran"
        if plain and path == "msd_local" and kernels.get("k_sort_scatter", {}).get("launches") != 1:
            return "not exactly one k_sort_scatter launch"
    elif path == "lsd_fixup":
        if "k_fix_runs" not in ran or "k_local_sort" in ran:
            return "no k_fix_runs, or k_local_sort ran"
    elif path == "lsd_full":
        if "k_sort_scatter" not in ran or ran & {"k_fix_runs", "k_local_sort"}:
            return "no k_sort_scatter, or k_fix_runs / k_local_sort ran"
    elif path == "materialise":
        if ran & set(SORT_KERNELS):
            return "a sort kernel ran"
    return None


@pytest.mark.parametrize("lsd", [False, True], ids=["default", "HS_LSD_SORT"])
@pytest.mark.parametrize("name", list(S.CASES))
def test_sort_edge_case(ctx, monkeypatch, name, lsd):
    cols, valids, nb, expected = S.case_data(name)
    a = S.analyse(name)
    if lsd:
        monkeypatch.setenv("HS_LSD_SORT", "1")
        expected = a["lsd_path"]
    ctx.profile_enable(True)
    try:
        perm, offs = ctx.k_sort_perm(cols, nb, valids)
        kernels = ctx.profile_report()
    finally:
        ctx.profile_enable(False)
    ran = {k: v.get("launches") for k, v in kernels.items() if k in SORT_KERNELS}
    assert np.array_equal(offs, a["offs"]), f"{name}: bucket offsets differ"
    if not np.array_equal(perm, a["perm"]):
        bad = np.flatnonzero(perm != a["perm"])
        pytest.fail(f"{name} ({expected}, sort kernels {ran}): {len(bad)} rows out of place, first at sorted position "
                    f"{bad[0]}")
    plain = len(cols) == 1 and (valids is None or valids[0] is None)
    problem = _path_problem(expected, kernels, plain)
    assert problem is None, f"{name}: expected {expected}, but {problem}; sort kernels {ran}"
    if lsd:
        assert "k_local_sort" not in kernels, f"{name}: k_local_sort ran under HS_LSD_SORT=1; sort kernels {ran}"


# ---------------------------------------------------------------------------------------------------------------------
# createIndex: float keys and float columns, bit for bit
# ---------------------------------------------------------------------------------------------------------------------

def _bits(a):
    a = np.asarray(a)
    return a.view({4: np.uint32, 8: np.uint64}[a.dtype.itemsize])


def _float_source(tmp_path, n=200_000):
    rng = np.random.default_rng(90)

    def sprinkle(values, special):
        values[rng.choice(n, 40 * len(special), replace=False)] = np.repeat(special, 40)
        return values

    kd = sprinkle(rng.standard_normal(n) * 10.0 ** rng.uniform(-20, 20, size=n), S._F64_SPECIAL)
    kf = sprinkle((rng.standard_normal(n) * 10.0 ** rng.uniform(-20, 20, size=n)).astype(np.float32), S._F32_SPECIAL)
    # low cardinality: NaN payloads of both signs, both zeros and two numbers -- dictionary-encoded by the GPU
    ld_vals = S._F64_SPECIAL[[0, 1, 2, 3, 4, 8, 9]].tolist() + [1.5, -2.5]
    lf_vals = S._F32_SPECIAL[[0, 1, 2, 3, 4, 8, 9]].tolist() + [1.5, -2.5]
    cols = {"kd": kd, "kf": kf,
            "ld": np.array(ld_vals, dtype=np.float64)[rng.integers(0, len(ld_vals), size=n)],
            "lf": np.array(lf_vals, dtype=np.float32)[rng.integers(0, len(lf_vals), size=n)],
            "hd": rng.standard_normal(n)}
    path = str(tmp_path / "floats.parquet")
    pq.write_table(pa.table(cols), path, use_dictionary=False, compression="NONE", row_group_size=60_000)
    back = pq.read_table(path)
    # the values as the source holds them, read back (NaN payloads and -0.0 included)
    return path, {name: back.column(name).to_numpy() for name in cols}


@pytest.mark.parametrize("key", ["kd", "kf"])
def test_create_index_float_keys_bit_exact(ctx, tmp_path, key):
    from hyperspace_b200 import _native

    path, src = _float_source(tmp_path)
    assert np.isin(_bits(S._F64_SPECIAL), _bits(src["kd"])).all()  # the writer kept every payload
    nb = 8
    included = [c for c in ("kd", "kf", "ld", "lf", "hd") if c != key]
    res, st = ctx.create_index([_native.FileImage(path=path)], [key], included, nb, output=_native.HS_OUT_HOST,
                               job_uuid="fl")
    perm, offs, order = O.index_rows(src, [key], included, nb)
    rows = 0
    for i, f in enumerate(res.files):
        pf = pq.ParquetFile(pa.BufferReader(res.host_bytes(i)))
        t = pf.read()
        lo, hi = int(offs[f.bucket]), int(offs[f.bucket + 1])
        assert t.num_rows == hi - lo
        for name in order:
            got = t.column(name).to_numpy()
            assert np.array_equal(_bits(got), _bits(src[name][perm[lo:hi]])), (key, name, f.bucket)
        names = [pf.metadata.schema.column(j).name for j in range(len(order))]
        md = pf.metadata.row_group(0)
        assert md.column(names.index("ld")).has_dictionary_page and md.column(names.index("lf")).has_dictionary_page
        assert not md.column(names.index("hd")).has_dictionary_page
        rows += t.num_rows
    assert rows == len(src[key])
    rep = ctx.verify_index(res.as_sources(), [f.bucket for f in res.files], [key], included, nb)
    assert rep["rows"] == rows and rep["bucket_mismatches"] == 0 and rep["order_violations"] == 0, rep
    res.free()


@pytest.mark.parametrize("name", ["fix_run_of_64_across_tiles", "fix_run_of_65_across_tiles"])
def test_create_index_fixup_runs_lsd_switch(ctx, tmp_path, monkeypatch, name):
    """createIndex defers the fix-up's verdict to its next synchronisation; a run across a tile edge, sorted in place or
    given up on, must give the same files with and without HS_LSD_SORT=1, in the oracle's order."""
    from hyperspace_b200 import _native

    (k,), _, nb, expected = S.case_data(name)
    assert expected == "lsd_fixup"
    v = np.arange(len(k), dtype=np.int64)
    path = str(tmp_path / "fix.parquet")
    pq.write_table(pa.table({"k": k, "v": v}), path, use_dictionary=False, compression="NONE")
    built = {}
    for lsd in (False, True):
        if lsd:
            monkeypatch.setenv("HS_LSD_SORT", "1")
        ctx.profile_enable(True)
        try:
            res, _ = ctx.create_index([_native.FileImage(path=path)], ["k"], ["v"], nb, output=_native.HS_OUT_HOST,
                                      job_uuid="fx")
            kernels = ctx.profile_report()
        finally:
            ctx.profile_enable(False)
        assert "k_fix_runs" in kernels and "k_local_sort" not in kernels, sorted(kernels)
        built[lsd] = {f.name: res.host_bytes(i) for i, f in enumerate(res.files)}
        if not lsd:
            perm, offs, _ = O.index_rows({"k": k, "v": v}, ["k"], ["v"], nb)
            for i, f in enumerate(res.files):
                t = pq.ParquetFile(pa.BufferReader(res.host_bytes(i))).read()
                lo, hi = int(offs[f.bucket]), int(offs[f.bucket + 1])
                assert np.array_equal(t.column("v").to_numpy(), perm[lo:hi]), f.bucket
        res.free()
    assert built[False] == built[True]
