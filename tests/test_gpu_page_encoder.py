"""GPU tests of the index page encoder on the cases of tests/page_encoder_cases.py: every page of every index file
against the bytes the walker expects from the oracle's rows, pyarrow's reading against the oracle, the kernels that ran
against the path the restatement claims, byte-identical files with carrying switched off, and compressed files whose
page bodies decompress to the uncompressed build's."""
import numpy as np
import pyarrow as pa
import pyarrow.parquet as pq
import pytest

import page_encoder_cases as C
from oracle import oracle as O

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    from hyperspace_b200 import _native

    c = _native.Context(0)
    yield c
    c.close()


def _build(ctx, name, codec=0):
    """{bucket: (file name, image)} of the case's index and the kernels that ran."""
    from hyperspace_b200 import _native as N

    c = C.case_data(name)
    ctx.profile_enable(True)
    try:
        res, _ = ctx.create_index([N.FileImage(data=img) for img in c.images], ["k"], c.included, c.nb,
                                  output=N.HS_OUT_HOST, job_uuid="pe", compression=codec, **c.kw)
        kernels = ctx.profile_report()
    finally:
        ctx.profile_enable(False)
    files = {f.bucket: (f.name, res.host_bytes(i)) for i, f in enumerate(res.files)}
    res.free()
    return files, kernels


def _launches(kernels, name):
    return int(kernels.get(name, {}).get("launches", 0))


def _check_values(c, files, perm, offs):
    """pyarrow reads every file as the oracle's rows (bits, validity, strings)."""
    for b, (fname, img) in files.items():
        rows = perm[offs[b]:offs[b + 1]]
        t = pq.ParquetFile(pa.BufferReader(img)).read()
        assert t.column_names == ["k"] + c.included and t.num_rows == len(rows), fname
        for col in t.column_names:
            arr = t.column(col).combine_chunks()
            want_valid = c.valids[col][rows] if col in c.valids else np.ones(len(rows), bool)
            assert np.array_equal(np.asarray(arr.is_valid()), want_valid), (fname, col)
            want = c.cols[col][rows]
            if want.dtype == object:
                got = [x.encode() if x is not None else b"" for x in arr.to_pylist()]
                assert got == list(want), (fname, col)
            else:
                got = arr.fill_null(0).to_numpy(zero_copy_only=False).astype(want.dtype)
                assert got.tobytes() == want.tobytes(), (fname, col)


@pytest.mark.parametrize("name", list(C.CASES))
def test_index_pages_match_the_walker(ctx, monkeypatch, name):
    c = C.case_data(name)
    files, kernels = _build(ctx, name)
    perm, offs, _ = O.index_rows({"k": c.cols["k"]}, ["k"], [], c.nb)
    assert sorted(files) == [b for b in range(c.nb) if offs[b + 1] > offs[b]]  # no file for an empty bucket
    walked = []
    for b, (fname, img) in files.items():
        walked += C.check_file(img, name, perm[offs[b]:offs[b + 1]], fname)
    _check_values(c, files, perm, offs)
    # the path the restatement claims, from the kernels that ran
    want = C.expected_launches(name)
    lo, hi = want["k_dict_build"]
    assert lo <= _launches(kernels, "k_dict_build") <= hi, (want, {k: v["launches"] for k, v in kernels.items()})
    assert _launches(kernels, "k_dict_map") == want["k_dict_map"]
    assert _launches(kernels, "k_dict_pack") == want["k_dict_pack"]
    if want["from_pages"]:
        assert _launches(kernels, "k_dict_build_from_pages") > 0
    cl = C.CLAIMS[name]
    if "plain_page_offsets_mod8" in cl:
        plain = [p for p in walked if p.get("can_align") is not None]
        assert cl["plain_page_offsets_mod8"] <= {p["offset"] % 8 for p in plain}
        assert any(not p["can_align"] and not p["aligned"] for p in plain)
    # carrying switched off: the same dictionaries (see test_dictionaries_do_not_depend_on_carrying), the same bytes
    if any(p["dictionary"] for p in C.plan(name).values()):
        monkeypatch.setenv("HS_NO_CARRY", "1")
        other, _ = _build(ctx, name)
        monkeypatch.delenv("HS_NO_CARRY")
        assert other.keys() == files.keys()
        for b in files:
            if other[b][1] != files[b][1]:
                C.check_file(other[b][1], name, perm[offs[b]:offs[b + 1]], other[b][0] + " (HS_NO_CARRY=1)", carry=False)
            assert other[b][1] == files[b][1], f"{files[b][0]} differs with HS_NO_CARRY=1"


@pytest.mark.parametrize("codec", ["snappy", "gzip", "lz4"])
@pytest.mark.parametrize("name", C.COMPRESSED_CASES)
def test_compressed_pages_hold_the_uncompressed_bodies(ctx, name, codec):
    from hyperspace_b200 import _native as N

    code = {"snappy": N.HS_CODEC_SNAPPY, "gzip": N.HS_CODEC_GZIP, "lz4": N.HS_CODEC_LZ4}[codec]
    c = C.case_data(name)
    plain, _ = _build(ctx, name)
    packed, _ = _build(ctx, name, code)
    perm, offs, _ = O.index_rows({"k": c.cols["k"]}, ["k"], [], c.nb)
    assert packed.keys() == plain.keys()
    for b, (fname, img) in packed.items():
        pages = C.check_file(img, name, perm[offs[b]:offs[b + 1]], fname, codec=code)
        _, ref = C.walk(plain[b][1], plain[b][0])
        assert [(p["rg"], p["col"], p["kind"], p["hdr"][2]) for p in pages] == \
               [(p["rg"], p["col"], p["kind"], p["hdr"][2]) for p in ref], fname
        for p, r in zip(pages, ref):
            assert p["body"] == r["body"], p["where"]
    _check_values(c, packed, perm, offs)
