"""GPU tests of the hash partition at the limits where it changes path (tests/partition_cases.py): every case through
hs_k_partition, compared byte for byte with the numpy restatement -- the moved columns and code records, the bin offsets
and the OR / AND of the last key -- with every byte outside the expected runs still holding the sentinel.  Then the
kernels each side of the fused limit, the refusals, and createIndex at the vote-width edges against the oracle.

The peer cases write `world` buffers on this one GPU: they check the owners' layout and the bulk-copy arithmetic of the
multi-GPU partition, not NVLink (tests/multi_gpu_check.py runs the real exchange)."""
import numpy as np
import pyarrow as pa
import pyarrow.parquet as pq
import pytest

import partition_cases as P
from oracle import oracle as O

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    from hyperspace_b200 import _native

    c = _native.Context(0)
    yield c
    c.close()


def _run(ctx, c, a=None, **over):
    kw = dict(valids=c.valids, decimal=c.decimal, payload=c.payload, codes=c.codes, mode=c.mode, world=c.world,
              fill=P.SENTINEL)
    if a is not None and c.mode == "peer":
        kw.update(peer_base=a["base"], owner_rows=a["owner_rows"], owner_shift=a["shift"])
    kw.update(over)
    return ctx.k_partition(c.keys, c.nb, **kw)


def _diff(name, cname, o, got, want, mask, width):
    """None, or what is wrong with one output buffer: bytes written outside the runs, or rows that differ inside."""
    if np.array_equal(got, want):
        return None
    bad = np.flatnonzero(got != want)
    outside = bad[~mask[bad]]
    if len(outside):
        return f"{name} {cname} owner {o}: {len(outside)} bytes outside the runs overwritten, first at byte {outside[0]}"
    return f"{name} {cname} owner {o}: {len(bad)} bytes differ inside the runs, first at byte {bad[0]} (element " \
           f"{bad[0] // width})"


@pytest.mark.parametrize("name", list(P.CASES))
def test_partition_case(ctx, name):
    c, a = P.case_data(name), P.analyse(name)
    ctx.profile_enable(True)
    try:
        out = _run(ctx, c, a)
        kernels = ctx.profile_report()
    finally:
        ctx.profile_enable(False)
    want = P.expected(name)
    got = {cn: out["payload"][i] for i, (cn, _) in enumerate(P.moved_columns(c)[:len(c.payload)])}
    if c.codes:
        got["records"] = out["records"]
    problems = []
    for cname, col in P.moved_columns(c):
        bufs = got[cname] if c.mode == "peer" else [got[cname]]
        assert len(bufs) == len(want[cname])
        for o, (g, (w, m)) in enumerate(zip(bufs, want[cname])):
            p = _diff(name, cname, o, g, w, m, col.dtype.itemsize)
            if p:
                problems.append(p)
    assert not problems, "\n".join(problems)
    if c.mode != "peer":
        assert np.array_equal(out["offsets"], a["offsets"]), f"{name}: bin offsets differ"
    assert out["key_or_and"] == a["key_or_and"], (name, [hex(v) for v in out["key_or_and"]],
                                                  [hex(v) for v in a["key_or_and"]])
    if a["n"]:
        fused = P.vote_bits(a["nbins"]) is not None
        ran = sorted(k for k in kernels if k.startswith("k_"))
        if fused:
            assert "k_partition_rows" in kernels and "k_partition_dest" not in kernels, ran
        else:
            assert {"k_partition_dest", "k_scatter_column"} <= set(kernels) and "k_partition_rows" not in kernels, ran


def test_decimal_flag_changes_the_buckets(ctx):
    """The same int32 keys bucket differently as an int and as a decimal's unscaled value (hashInt vs hashLong)."""
    k = P.keys_in("int32", 64, np.arange(64), 5)
    b_int, _ = ctx.k_bucket_ids([k], 64)
    assert np.array_equal(b_int, np.arange(64))
    c = P.Case([k], 64, decimal=[True])
    out = _run(ctx, c)
    want = P.bucket_ids([k], [None], [True], 64)
    assert np.array_equal(out["offsets"], np.concatenate([[0], np.cumsum(np.bincount(want, minlength=64))]))


def _refused(ctx, c, code, **over):
    from hyperspace_b200 import _native

    with pytest.raises(_native.HyperspaceGpuError) as e:
        _run(ctx, c, **over)
    assert e.value.code == code, e.value.message
    return e.value.message


def test_refusals(ctx):
    from hyperspace_b200 import _native

    n = 5000
    k = P._random_keys(n, 2000, seed=50)
    codes = [np.arange(n, dtype=np.uint16)]
    # code records need the fused partition
    msg = _refused(ctx, P.Case([k], 1025, codes=codes), _native.HS_EINVAL)
    assert "code records" in msg
    # the runs go to the owners' buffers only up to the fused limit
    base = np.zeros(1025, np.uint64)
    msg = _refused(ctx, P.Case([k], 1025, mode="peer", world=2), _native.HS_EINVAL, peer_base=base, owner_rows=[n, n])
    assert "peer" in msg
    # a peer layout without rows going to peers, and rows going to peers without one
    msg = _refused(ctx, P.Case([k], 100), _native.HS_EINVAL, world=2, peer_base=np.zeros(100, np.uint64), owner_rows=[n, n])
    assert "peer table" in msg
    msg = _refused(ctx, P.Case([k], 100, mode="peer", world=2), _native.HS_EINVAL)
    assert "peer table" in msg
    # the context still works after the refusals
    c = P.case_data("rows_4097")
    out = _run(ctx, c)
    assert np.array_equal(out["offsets"], P.analyse("rows_4097")["offsets"])


# ---------------------------------------------------------------------------------------------------------------------
# createIndex at the vote-width edges: four dictionary-carried columns and a nullable one
# ---------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("nb", [16, 17, 256, 257])
def test_create_index_vote_width_edges(ctx, tmp_path, nb):
    from hyperspace_b200 import _native

    n = 40_000
    rng = np.random.default_rng(nb)
    cols = {"k": P._random_keys(n, nb, seed=nb + 60),
            "c0": rng.integers(0, 5, size=n).astype(np.int64) * 1_000_003,
            "c1": rng.integers(-3, 4, size=n).astype(np.int32),
            "c2": np.array([1.5, -0.0, 7.25], dtype=np.float64)[rng.integers(0, 3, size=n)],
            "c3": rng.integers(0, 9, size=n).astype(np.int32) - 4,
            "v": rng.standard_normal(n)}
    valid_v = rng.random(n) >= 0.2
    path = str(tmp_path / "t.parquet")
    table = pa.table({**{c: cols[c] for c in ("k", "c0", "c1", "c2", "c3")},
                      "v": pa.array(cols["v"], mask=~valid_v)})
    pq.write_table(table, path, compression="NONE", use_dictionary=["c0", "c1", "c2", "c3"], row_group_size=15_000)
    included = ["c0", "c1", "c2", "c3", "v"]
    ctx.profile_enable(True)
    try:
        res, _ = ctx.create_index([_native.FileImage(path=path)], ["k"], included, nb, output=_native.HS_OUT_HOST,
                                  job_uuid="pv")
        kernels = ctx.profile_report()
    finally:
        ctx.profile_enable(False)
    assert "k_partition_rows" in kernels and "k_dict_pack" in kernels, sorted(kernels)
    perm, offs, order = O.index_rows(cols, ["k"], included, nb)
    rows = 0
    for i, f in enumerate(res.files):
        t = pq.ParquetFile(pa.BufferReader(res.host_bytes(i))).read()
        lo, hi = int(offs[f.bucket]), int(offs[f.bucket + 1])
        assert t.num_rows == hi - lo, f.bucket
        for name in order:
            col = t.column(name)
            if name == "v":
                assert np.array_equal(col.is_valid().to_numpy(zero_copy_only=False), valid_v[perm[lo:hi]]), f.bucket
                got = col.to_numpy(zero_copy_only=False)[valid_v[perm[lo:hi]]]
                want = cols["v"][perm[lo:hi]][valid_v[perm[lo:hi]]]
            else:
                got, want = col.to_numpy(), cols[name][perm[lo:hi]]
            assert got.tobytes() == want.tobytes(), (nb, name, f.bucket)
        rows += t.num_rows
    assert rows == n
    res.free()
