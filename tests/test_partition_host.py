"""CPU self-checks of the partition cases (tests/partition_cases.py): the restated limits still match hash_partition.cu and
kernels.h, and every case really has the shape it claims -- its vote width, row count, tail, run lengths, number of scan
chunks, the parities of its runs in the owners' buffers -- measured from the oracle's buckets.  A case that drifts off
its boundary would still pass on the GPU and test nothing."""
import os
import re

import numpy as np
import pytest

import partition_cases as P

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _source(name):
    with open(os.path.join(ROOT, "hyperspace_b200", "csrc", name)) as f:
        return f.read()


def test_limits_match_the_partition_source():
    src, hdr = _source("hash_partition.cu"), _source("kernels.h")

    def const(text, name):
        return int(re.search(rf"constexpr int {name} = (\d+);", text).group(1))

    assert const(src, "kFusedMaxBins") == P.FUSED_MAX_BINS
    assert const(src, "kChunk") == P.CHUNK
    assert const(hdr, "kFusedTileLocal") == P.TILE_LOCAL and const(hdr, "kFusedTilePeer") == P.TILE_PEER
    assert const(hdr, "kMaxBuckets") == P.MAX_BUCKETS
    assert const(src, "kThreads") == 256 and P.TILE_LOCAL // 256 == 16 and P.TILE_LOCAL // (256 // 32) == P.WARP_ROWS
    assert P.TILE_PEER // (512 // 32) == P.WARP_ROWS  # FusedCfg<true>: 512 threads, 16 warps of 512 rows
    # the vote widths, in the order launch_partition_rows tries them
    bands = re.findall(r"(?:else )?if \(nb <= (\d+)\) launch_partition_rows_bits<(\d+), PEER>", src)
    assert [(int(a), int(b)) for a, b in bands] == [b for b in P.BITS_BANDS[:2]]
    assert "else launch_partition_rows_bits<10, PEER>" in src and P.BITS_BANDS[2] == (P.FUSED_MAX_BINS, 10)
    assert "return ctx->world > 1 ? kFusedTilePeer : kFusedTileLocal;" in src
    assert "h.ntiles = ceil_div(nrows, to_peers ? kFusedTilePeer : kFusedTileLocal);" in src
    assert ("nkeys == 1 && keys[0].valid == nullptr && (keys[0].type == HS_TYPE_INT32 || keys[0].type == HS_TYPE_INT64)"
            in src)


def test_restated_rules():
    assert [P.vote_bits(n) for n in (1, 16, 17, 256, 257, 1024, 1025, 4096)] == [4, 4, 8, 8, 10, 10, None, None]
    assert P.tile_rows("local") == P.tile_rows("owner") == 4096 and P.tile_rows("peer") == 8192
    c = P.Case([np.arange(5, dtype=np.int32)], 4)
    assert P.single_key_type(c) == "int32"
    c = P.Case([np.arange(5, dtype=np.int32)], 4, valids=[np.ones(5, np.uint8)])
    assert P.single_key_type(c) is None
    assert P.single_key_type(P.Case([np.zeros(5)], 4)) is None
    # records: code j in bits [16 j, 16 j + 16)
    c = P.Case([np.arange(2, dtype=np.int64)], 4, codes=[np.array([1, 0xFFFF], np.uint16), np.array([2, 3], np.uint16),
                                                         np.array([4, 5], np.uint16)])
    assert P.records(c).tolist() == [1 | 2 << 16 | 4 << 32, 0xFFFF | 3 << 16 | 5 << 32]


def test_pool_places_keys_in_their_buckets():
    for kind in ("int64", "int32", "decimal"):
        want = np.array([0, 4095, 17, 17, 1000])
        k = P.keys_in(kind, 4096, want, 1)
        assert np.array_equal(P.bucket_ids([k], [None], [kind == "decimal"], 4096), want), kind
    # a decimal int32 is not bucketed like an int32
    k = P.keys_in("int32", 4096, np.arange(64), 2)
    assert not np.array_equal(P.bucket_ids([k], [None], [True], 4096), np.arange(64))


@pytest.mark.parametrize("name", list(P.CASES))
def test_case_has_its_shape(name):
    c, a, claims = P.case_data(name), P.analyse(name), P.CLAIMS[name]
    n, t = a["n"], P.tile_rows(c.mode)
    assert 1 <= c.nb <= P.MAX_BUCKETS and len(c.codes) <= 4
    assert {p.dtype.itemsize for p in c.payload} == {8, 4, 1}
    if len(c.codes):
        assert a["nbins"] <= P.FUSED_MAX_BINS, "code records need the fused partition"
    if "bits" in claims:
        assert P.vote_bits(a["nbins"]) == claims["bits"]
        # rows in a bin past the narrower vote below, which would take that bin for a lower one
        lower = {4: 0, 8: 16, 10: 256, None: P.FUSED_MAX_BINS}[claims["bits"]]
        assert np.flatnonzero(a["counts"]).max() >= lower
    if "split_round" in claims:
        lo, hi = claims["split_round"]
        assert lo ^ hi == 16 and set(a["bins"][:32].tolist()) == {lo, hi}
    if "n" in claims:
        assert n == claims["n"]
        if n > t * P.CHUNK:
            assert a["ntiles"] == P.CHUNK + 1, "one tile past a whole chunk"
        elif n >= t * P.CHUNK - 1:
            assert a["ntiles"] == P.CHUNK
    if "tail" in claims:
        assert a["tail"] == claims["tail"]
    if "max_run" in claims:
        assert int(a["tile_bin"].max()) == claims["max_run"]
        warp_bins = a["bins"][:(n // P.WARP_ROWS) * P.WARP_ROWS].reshape(-1, P.WARP_ROWS)
        assert (warp_bins == warp_bins[:, :1]).all(axis=1).any(), "512 rows of one warp in one bin"
    if claims.get("last_bin_only"):
        assert (a["bins"] == a["nbins"] - 1).all()
    if claims.get("tail_in_last_bin"):
        tail_bins = a["bins"][(a["ntiles"] - 1) * t:]
        assert (tail_bins == a["nbins"] - 1).all() and (a["bins"][:(a["ntiles"] - 1) * t] != a["nbins"] - 1).all()
    if claims.get("empty_between"):
        used = np.flatnonzero(a["counts"])
        assert (a["counts"][used[0]:used[-1]] == 0).any() and used[0] == 0 and used[-1] == a["nbins"] - 1
    if claims.get("one_per_bin"):
        assert (a["counts"] == 1).all()
    if "kt" in claims:
        assert a["kt"] == claims["kt"]
    if claims.get("specials"):
        col = c.keys[-1]
        bits = np.uint64 if col.dtype == np.float64 else np.uint32
        special = P.E._F64_SPECIAL if col.dtype == np.float64 else P.E._F32_SPECIAL
        assert np.isin(special.view(bits), col.view(bits)).all()
    if "ncodes" in claims:
        assert len(c.codes) == claims["ncodes"]
    if c.mode == "peer":
        _check_peer_layout(name, c, a, claims)


def _check_peer_layout(name, c, a, claims):
    # every owner's runs lie inside its buffer, apart from each other, in increasing bucket order
    for o in range(c.world):
        mine = [b for b in range(c.nb) if b % c.world == o]
        ends = [(int(a["base"][b]), int(a["base"][b]) + int(a["counts"][b])) for b in mine]
        assert all(e0[1] <= e1[0] for e0, e1 in zip(ends, ends[1:]))
        assert not ends or ends[-1][1] <= int(a["owner_rows"][o])
    assert any(int(a["base"][b + c.world]) > int(a["base"][b]) + int(a["counts"][b]) for b in range(c.nb - c.world)) or \
        c.nb <= c.world, "no gap between two runs of one owner"
    runs = [r for r in P.runs(name) if r[3] not in c.shifted]
    if claims.get("parity"):
        pairs = {(p & 1, d & 1) for p, d, _, _ in runs}
        assert pairs == {(0, 0), (0, 1), (1, 0), (1, 1)}, pairs
        assert any(d & 1 for _, d, _, _ in runs), "no odd head element"
        assert any((ln - (d & 1)) & 1 for _, d, ln, _ in runs), "no odd tail element"
        assert any(ln - (d & 1) >= 2 for _, d, ln, _ in runs), "no bulk body"
    if claims.get("shifted"):
        assert [o for o in range(c.world) if a["shift"][o]] == list(claims["shifted"])
        assert any(r[3] in claims["shifted"] for r in P.runs(name))
