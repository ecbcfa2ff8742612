"""CPU self-checks of the sort edge cases (tests/sort_edge_cases.py): every case must really sit where it claims to --
its bucket, sub-bucket, item and run sizes, where its runs lie relative to tiles, items and buckets, its varying bytes and
the path sort_rows takes for it -- measured from the oracle's order.  A case that drifts off its boundary would still
pass on the GPU and test nothing."""
import os
import re

import numpy as np
import pytest

import sort_edge_cases as S

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_limits_match_the_sort_source():
    with open(os.path.join(ROOT, "hyperspace_b200", "csrc", "radix_sort.cu")) as f:
        src = f.read()
    with open(os.path.join(ROOT, "hyperspace_b200", "csrc", "kernels.h")) as f:
        hdr = f.read()

    def const(text, name):
        return int(re.search(rf"constexpr (?:int|uint32_t) {name} = (\d+);", text).group(1))

    assert const(src, "kLocalSortCap") == S.LOCAL_CAP
    assert const(src, "kLocalMaxRun") == S.MAX_RUN and const(src, "kFixMaxRun") == S.MAX_RUN
    assert const(hdr, "kSortTile") == S.SORT_TILE
    assert "max_seg <= (uint64_t)(0.85 * 256 * kLocalSortCap)" in src
    assert "63 - __builtin_clzll(varying) - 7" in src
    assert S.MSD_MAX_SEG == 2_673_868


def test_restated_rules():
    assert [S.want_bytes(m) for m in (1, 32_768, 32_769, 8_388_608, 8_388_609)] == [2, 2, 3, 3, 4]
    assert S.local_prefix_low(8000, 1 << 63) == 48 and S.local_prefix_low(8000, 1 << 55) == 40
    assert S.local_prefix_low(S.LOCAL_CAP, 1 << 63) == 48      # 2 x 12 288 rows need 15 bits: two digits
    assert S.local_prefix_low(100, (1 << 20) - 1) == 12        # one digit under the top varying bit
    assert S.local_prefix_low(100, 0xF) == 0
    assert S.msd_shift(1 << 63) == 56 and S.msd_shift(0xFFFFFF) == 16 and S.msd_shift(0x3F) == 0
    assert S.fix_low_bit(~0 & (2**64 - 1), 20_000) == 48 and S.fix_low_bit((1 << 56) | 0xFFFFFF, 20_000) == 16
    enc = S.encode(np.array([-0.0, 0.0, float("nan"), -float("nan"), -float("inf"), float("inf"), -1.0, 1.0]))
    assert enc[0] == enc[1] and enc[2] == enc[3]
    assert enc[4] < enc[6] < enc[0] < enc[7] < enc[5] < enc[2]
    assert S.encode(np.array([-2**63, 2**63 - 1], dtype=np.int64)).tolist() == [0, 2**64 - 1]
    assert S.encode(np.array([-2**31, 2**31 - 1], dtype=np.int32)).tolist() == [0, 2**32 - 1]


def _check_runs(runs, claims, key):
    for ln, where in claims:
        field = "where" if key == "local" else "kinds"
        hits = [r for r in runs if r["len"] == ln and (r[field] == where if key == "local" else where in r[field])]
        assert hits, f"no {key} run of {ln} rows ({where}); runs of 60+: " + str([r for r in runs if r["len"] >= 60])


@pytest.mark.parametrize("name", list(S.CASES))
def test_case_sits_on_its_boundary(name):
    cols, valids, nb, expected = S.case_data(name)
    claims = S.CLAIMS[name]
    a = S.analyse(name)
    assert expected in S.PATHS
    assert a["path"] == expected, (name, a["path"], a["max_seg"], a["nbytes"])
    assert a["lsd_path"] in ("lsd_fixup", "lsd_full", "materialise")
    if "n" in claims:
        assert a["n"] == claims["n"]
    if "max_bucket" in claims:
        assert int(a["sizes"].max()) == claims["max_bucket"], sorted(a["sizes"])[-3:]
    if claims.get("empty_between"):
        ne = np.flatnonzero(a["sizes"])
        assert any(a["sizes"][g] == 0 for g in range(ne[0], ne[-1]))
    if "max_sub" in claims:
        assert int(a["sub_sizes"].max()) == claims["max_sub"]
    if "item_sizes" in claims:
        got = [c for _, c in a["items"]]
        for size in set(claims["item_sizes"]):
            assert got.count(size) >= claims["item_sizes"].count(size), (size, sorted(got)[-5:])
    if "nbytes" in claims:
        assert a["nbytes"] == claims["nbytes"]
    if "constant_items" in claims:
        assert a["constant_items"] == claims["constant_items"]
    if "local_runs" in claims:
        _check_runs(a["local_runs"], claims["local_runs"], "local")
        if not claims.get("ties"):  # every placed run has to be reversed by the sort
            placed = [r for r in a["local_runs"] if r["len"] in {ln for ln, _ in claims["local_runs"]}]
            assert all(r["reversed"] for r in placed)
        else:  # the placed run holds equal whole keys, whose order only the row index decides
            assert any(r["ties"] for r in a["local_runs"] if r["len"] == claims["local_runs"][0][0])
    if "max_local_run" in claims:
        assert max(r["len"] for r in a["local_runs"]) == claims["max_local_run"]
    if "fix_runs" in claims:
        _check_runs(a["fix_runs"], claims["fix_runs"], "fix")
        placed = [r for r in a["fix_runs"] if r["len"] in {ln for ln, _ in claims["fix_runs"]}]
        assert all(r["reversed"] for r in placed)
    if "max_fix_run" in claims:
        assert max(r["len"] for r in a["fix_runs"]) == claims["max_fix_run"]
    if claims.get("specials"):
        col = next(c for c in cols if c.dtype.kind == "f") if any(c.dtype.kind == "f" for c in cols) else cols[0]
        special = {np.dtype(np.int64): S._I64_SPECIAL, np.dtype(np.int32): S._I32_SPECIAL,
                   np.dtype(np.float64): S._F64_SPECIAL, np.dtype(np.float32): S._F32_SPECIAL}[col.dtype]
        bits = {np.dtype(np.float64): np.uint64, np.dtype(np.float32): np.uint32}.get(col.dtype, col.dtype)
        have = np.unique(col.view(bits))
        assert np.isin(special.view(bits), have).all()


def test_boundary_pairs_straddle_their_limits():
    """The cases on either side of one limit differ by one row, and take different paths."""
    for below, above, measure in (("raw_bucket_at_cap", "raw_bucket_over_cap", lambda a: int(a["sizes"].max())),
                                  ("msd_sub_bucket_at_cap", "msd_sub_bucket_over_cap", lambda a: int(a["sub_sizes"].max())),
                                  ("msd_bucket_at_ceiling", "msd_bucket_over_ceiling", lambda a: int(a["sizes"].max()))):
        lo, hi = S.analyse(below), S.analyse(above)
        assert measure(hi) == measure(lo) + 1
        assert lo["path"] != hi["path"]
    assert S.analyse("raw_bucket_at_cap")["max_seg"] == S.LOCAL_CAP
    assert S.analyse("msd_bucket_at_ceiling")["max_seg"] == S.MSD_MAX_SEG
    assert S.analyse("two_varying_bytes")["path"] == "lsd_full" and S.analyse("three_varying_bytes")["path"] == "msd_local"
    # one row more in the third sub-bucket moves the first item's end from row 12 288 to row 8192
    full, over = S.analyse("msd_items_exactly_full"), S.analyse("msd_items_one_row_over")
    assert full["items"][0] == (0, S.LOCAL_CAP) and over["items"][0] == (0, 8192)
    assert over["items"][1][0] == 8192 and over["items"][1][0] + over["items"][1][1] > S.LOCAL_CAP
