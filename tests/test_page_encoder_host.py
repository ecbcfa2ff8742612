"""CPU self-checks of the index page encoder cases (tests/page_encoder_cases.py): the restated limits still stand on the
source lines they cite, every case has the shape it claims -- measured from the data in the partition order the
encoder samples, with the oracle's bucket ids -- the boundary cases straddle their limits in pairs, and the page
walker accepts a hand-built file in the encoder's page shapes and rejects it after one corrupted byte."""
import os
import struct

import numpy as np
import pyarrow as pa
import pyarrow.parquet as pq
import pytest

import page_encoder_cases as C
import parquet_shapes as S
from oracle import oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _line(fname, lineno):
    with open(os.path.join(ROOT, "hyperspace_b200", "csrc", fname)) as f:
        return f.read().split("\n")[lineno - 1]


@pytest.mark.parametrize("value,fname,lineno,text", C.SOURCE_LINES, ids=[f"{f}:{n}" for _, f, n, _ in C.SOURCE_LINES])
def test_limits_match_the_encoder_source(value, fname, lineno, text):
    placeholder = "{}" in text or "{0}" in text
    want = text.format(value) if placeholder else text
    assert want in _line(fname, lineno), f"{fname}:{lineno} no longer reads {want!r}"
    if value is not None and not placeholder:  # the constant is spelled out in the cited text
        assert str(value) in want or f"1 << {int(value).bit_length() - 1}" in want


def test_restated_rules():
    assert [C.bits_for(m) for m in (1, 2, 3, 4, 5, 65536, 65537)] == [1, 1, 2, 2, 3, 16, 17]
    # the 0.9 rule, by parquet_shapes' restatement, at its edge: 10 rows of 8 bytes, one segment
    assert S.dictionary_pays_off(1, 8, 10, 1) and not S.dictionary_pays_off(2, 8, 2, 1)
    assert not S.dictionary_pays_off(C.MAX_DICT_ENTRIES + 1, 8, 10**9, 1)
    # sort_dictionary: -0.0 before 0.0 (equal in the column's order, raw bits decide), NaNs last by raw bits
    d = np.array([0x7FF8000000000000, 0, 0xFFFFFFFFFFFFFFFF, 0x8000000000000000, 0x3FF0000000000000], dtype=np.uint64)
    assert C.sort_dictionary(d, np.float64).tolist() == [0, 0x8000000000000000, 0x3FF0000000000000,
                                                          0x7FF8000000000000, 0xFFFFFFFFFFFFFFFF]
    assert C.layout_sizes({}) == (131072, 4194304)
    assert C.layout_sizes(dict(rows_per_page=5000, rows_per_row_group=20_000)) == (8192, 16384)
    assert C.layout_sizes(dict(rows_per_page=4096, rows_per_row_group=3000)) == (4096, 4096)
    # a one-row page admits no run split: its values are aligned only where the page happens to start
    assert sum(C.plain_alignment_possible(m, 1, 8) for m in range(8)) < 8
    assert all(C.plain_alignment_possible(m, 4096, 8) for m in range(8))


def _first_seen(raw_in_order, values):
    """Row (partition order) at which any of `values` first appears."""
    hit = np.isin(raw_in_order, np.asarray(list(values), dtype=np.uint64))
    return int(np.flatnonzero(hit)[0])


@pytest.mark.parametrize("name", list(C.CASES))
def test_case_has_its_claimed_shape(name):
    c = C.case_data(name)
    cl = C.CLAIMS[name]
    pl = C.plan(name)
    n = len(c.cols["k"])
    order = C.partition_order(c.cols["k"], c.nb)
    sizes = np.bincount(O.bucket_ids([c.cols["k"]], c.nb), minlength=c.nb)
    # pyarrow reads the sources back as the case's columns
    t = pa.concat_tables([pq.ParquetFile(pa.BufferReader(img)).read() for img in c.images])
    for col in ["k"] + c.included:
        arr = t.column(col).combine_chunks()
        valid = np.asarray(arr.is_valid())
        assert np.array_equal(valid, c.valids.get(col, np.ones(n, bool))), col
        if c.cols[col].dtype == object:
            assert [x.encode() if x is not None else b"" for x in arr.to_pylist()] == list(c.cols[col]), col
        else:
            got = arr.fill_null(0).to_numpy(zero_copy_only=False).astype(c.cols[col].dtype)
            assert got.tobytes() == c.cols[col].tobytes(), col
    for col, m in cl.get("distinct", {}).items():
        assert len(np.unique(C.raw_bits(c.cols[col]))) == m, col
    for col, at in cl.get("first_new", {}).items():
        raw = C.raw_bits(c.cols[col])[order]
        new = set(np.unique(raw).tolist()) - set(np.unique(raw[:at]).tolist())
        assert new and _first_seen(raw, new) == at, col
        stage = 2 if at < C.STAGE2_ROWS else 3
        assert (C.STAGE1_ROWS <= at < C.STAGE2_ROWS) if stage == 2 else (C.STAGE2_ROWS <= at < n)
    if "burst" in cl:
        col, quiet = cl["burst"]
        raw = C.raw_bits(c.cols[col])[order]
        assert len(np.unique(raw[:quiet])) < 10 and len(np.unique(raw[quiet:])) > C.MAX_DICT_ENTRIES + 100_000
    for col in cl.get("empty_marker", []):
        assert (C.raw_bits(c.cols[col]) == np.uint64(C.EMPTY)).any(), col
    if "rows_over" in cl:
        assert n > cl["rows_over"]
    for col, m in cl.get("stage1_distinct", {}).items():
        assert len(np.unique(C.raw_bits(c.cols[col])[order][:C.STAGE1_ROWS])) == m, col
        assert len(np.unique(c.cols[col])) == m, col
    if "dict_columns" in cl:
        assert sum(p["dictionary"] for p in pl.values()) == cl["dict_columns"]
    if "map_launches" in cl:
        assert C.expected_launches(name)["k_dict_map"] == cl["map_launches"]
    if "mapped" in cl:
        assert sum(p["dictionary"] and not p["carried"] for p in pl.values()) == cl["mapped"]
        assert sum(p["carried"] for p in pl.values()) == cl["carried"]
    if isinstance(cl.get("carried"), list):
        assert [col for col, p in pl.items() if p["carried"]] == cl["carried"]
    srcd, _ = C.source_dictionaries_of(name)
    for col, m in cl.get("union", {}).items():
        assert srcd[col]["all_dict"] and len(srcd[col]["union"]) == m, col
    for col, m in cl.get("used", {}).items():
        assert len(np.unique(c.cols[col])) == m, col
    if "null_rows_in_bucket0" in cl:
        perm, offs, _ = O.index_rows({"k": c.cols["k"]}, ["k"], [], c.nb)
        assert not c.valids["ne"][perm[offs[0] + np.array(cl["null_rows_in_bucket0"])]].any()
        b, page = cl["all_null_page"]
        assert not c.valids["ne"][perm[offs[b] + 4096 * page:offs[b] + 4096 * (page + 1)]].any()
        assert offs[b + 1] - offs[b] > 4096 * (page + 1)
        assert not c.valids[cl["all_null_column"]].any()
    if "bucket_rows" in cl:
        assert sizes.tolist() == cl["bucket_rows"]
        P, _ = C.layout_sizes(c.kw)
        assert {P - 1, P, P + 1, 0} <= set(sizes.tolist())
        assert cl["last_group_rows"] <= {int(s % P) % 8 for s in sizes if s % P}
    if "page_rows" in cl:
        assert C.layout_sizes(c.kw) == (cl["page_rows"], cl["rg_rows"])
        assert c.kw["rows_per_page"] % C.SORT_TILE or c.kw["rows_per_row_group"] < c.kw["rows_per_page"]
        assert sizes.max() > cl["rg_rows"] or c.kw["rows_per_row_group"] < c.kw["rows_per_page"]
    if cl.get("default_layout"):
        assert not c.kw and sizes.min() > C.DEFAULT_PAGE_ROWS
    if cl.get("specials"):
        bits = set(C.raw_bits(c.cols["f64"]).tolist())
        assert {0, 0x8000000000000000, C.EMPTY, 0x7FF8000000000000, 0xFFF8000000000000} <= bits
        assert len({b for b in bits if (b & 0x7FFFFFFFFFFFFFFF) > 0x7FF0000000000000}) >= 4
    if cl.get("unaligned_pages"):
        assert sizes.min() < 8 and sizes.max() < 64


def test_plans_pin_the_rules():
    """What the restatement decides at each limit -- the GPU test then requires the files to agree."""
    p = C.plan("bit_widths_1_to_13")
    for col, pc in p.items():
        if col.startswith("d"):
            m = int(col[1:])
            assert pc["dictionary"] and pc["bw"] == C.bits_for(m) and len(pc["values"]) == m, col
    assert {C.bits_for(int(c[1:])) for c in p if c.startswith("d")} == set(range(1, 14))
    assert p["m1"]["bw"] == 4 and 0xFFFFFFFF in p["m1"]["values"].tolist() and p["m1"]["rule"] == "pays_off"
    assert p["k"]["rule"] == "overflow"  # 200 K distinct keys
    q = C.plan("bit_widths_14_to_16_limits_and_stages")
    assert {C.bits_for(int(c[1:])) for c in q if c.startswith("d") and q[c]["dictionary"]} == {13, 14, 15, 16}
    assert q["d65536"]["dictionary"] and q["d65536"]["bw"] == 16
    assert q["e65535"]["dictionary"] and C.EMPTY in q["e65535"]["values"].tolist()
    for col in ("d65537", "burst"):
        assert q[col]["rule"] == "overflow" and not q[col]["dictionary"], col
    # 65 536 values fill the hash set without overflowing it; ~0 (tracked beside the set) makes 65 537 entries, which
    # dictionary_pays_off refuses
    assert q["e65536"]["rule"] == "no_pay" and len(q["e65536"]["values"]) == C.MAX_DICT_ENTRIES + 1
    assert q["burst"]["launches"] == (3, 3)   # quiet first 256 K rows: the burst overflows in stage 3
    assert q["d65537"]["launches"] == (3, 3)  # its first 256 K rows hold fewer than 65 537 of its values
    assert q["k"]["launches"] == (2, 3)  # overflows in stage 2: the flag may be left clear (dict_encode.cu:51-53)
    for col in ("s2", "s3", "late_empty"):
        assert q[col]["dictionary"] and q[col]["launches"] == (3, 3), col
    assert C.EMPTY in q["late_empty"]["values"].tolist()
    e = C.plan("early_drop_over_2_20_rows")
    assert e["drop"]["rule"] == "early_drop" and e["drop"]["launches"] == (1, 1)
    assert e["keep"]["dictionary"] and e["keep"]["bw"] == 14 and e["keep"]["launches"] == (3, 3)
    # the early drop is the stage-1 rule alone: the dropped column would have paid off
    assert S.dictionary_pays_off(15565, 8, 1_100_000, 4)
    s = C.plan("source_dictionaries")
    assert s["u"]["source"] == "carried" and len(s["u"]["values"]) == 300 and s["u"]["bw"] == 9
    assert s["w"]["source"] == "pages" and s["w"]["dictionary"] and s["w"]["bw"] == 14
    assert s["z"]["source"] == "pages" and s["z"]["rule"] == "no_pay" and s["z"]["launches"] == (0, 0)
    assert s["x"]["source"] == "data" and s["x"]["dictionary"] and len(s["x"]["values"]) == 300
    f = C.plan("float_specials")
    assert len(f["f64"]["values"]) == 12 and len(f["f32"]["values"]) == 9
    n = C.plan("nullable_and_strings")
    assert n["d"]["dictionary"] and {n[c]["rule"] for c in ("nv", "ne", "allnull")} == {"nullable"}
    assert {n[c]["rule"] for c in ("s", "ns")} == {"string"}


def test_boundary_pairs_straddle_their_limits():
    q = C.plan("bit_widths_14_to_16_limits_and_stages")
    assert (q["d65536"]["dictionary"], q["d65537"]["dictionary"]) == (True, False)
    assert (q["e65535"]["dictionary"], q["e65536"]["dictionary"]) == (True, False)
    e = C.plan("early_drop_over_2_20_rows")
    assert (e["keep"]["dictionary"], e["drop"]["dictionary"]) == (True, False)
    assert 15564 <= C.EARLY_DROP_FRACTION * C.STAGE1_ROWS < 15565
    p = C.plan("bit_widths_1_to_13")
    for k in range(1, 13):
        assert p[f"d{1 << k}"]["bw"] + 1 == p[f"d{(1 << k) + 1}"]["bw"], k
    s = C.plan("source_dictionaries")
    assert len(C.source_dictionaries_of("source_dictionaries")[0]["w"]["union"]) == C.AGREE_CAP + 1
    assert (s["z"]["source"], s["x"]["source"]) == ("pages", "data")  # 65 536 vs 65 537 union entries
    pe = C.plan("pays_off_edge")
    assert (pe["pay5226"]["rule"], pe["pay5227"]["rule"]) == ("pays_off", "no_pay")
    assert pe["pay5226"]["bw"] == pe["pay5227"]["bw"] == 13
    counts = {nd: C.expected_launches(f"dict_columns_{nd}")["k_dict_map"] for nd in (1, 4, 5, 8, 9, 12)}
    assert counts == {1: 1, 4: 1, 5: 1, 8: 1, 9: 2, 12: 2}


@pytest.mark.parametrize("name", list(C.CASES))
def test_dictionaries_do_not_depend_on_carrying(name):
    """On one GPU a carried column's dictionary is the union its pages give the uncarried path too: the files must be
    byte-identical with carrying switched off."""
    a, b = C.plan(name, True), C.plan(name, False)
    for col in a:
        assert a[col]["dictionary"] == b[col]["dictionary"], col
        if a[col]["dictionary"]:
            assert a[col]["values"].tolist() == b[col]["values"].tolist(), col


# ---- the walker on a hand-built file ------------------------------------------------------------------------------------
def _encoder_shaped_file():
    """One row group, k PLAIN and d dictionary-encoded as the encoder writes it: PLAIN_DICTIONARY pages, all-valid
    levels as one RLE run, one bit-packed index run whose last group is padded (101 rows)."""
    rng = np.random.default_rng(0)
    n = 101
    d = np.array([5, -3, 8, 13, 21], dtype=np.int64)
    ix = rng.integers(0, 5, size=n)
    k = np.arange(n, dtype=np.int64)
    cols = [S.Col("k", S.INT64, True, [S.Chunk([S.Page(rows=n, values=k)])]),
            S.Col("d", S.INT64, True, [S.Chunk([S.Page(rows=n, enc=S.PLAIN_DICTIONARY, idx=[S.packed(ix)], bw=3)],
                                               dict=d, dict_enc=S.PLAIN_DICTIONARY)])]
    return S.write_file(S.FileSpec(cols)), d, ix


def test_walker_reads_a_hand_built_file():
    img, d, ix = _encoder_shaped_file()
    _, pages = C.walk(img)
    dp = [p for p in pages if p["col"] == "d"]
    assert dp[0]["kind"] == "dict" and dp[0]["values"].view(np.int64).tolist() == d.tolist()
    assert dp[1]["bw"] == 3 and dp[1]["indices"].tolist() == ix.tolist()
    kp = [p for p in pages if p["col"] == "k"]
    assert np.frombuffer(kp[0]["values"], np.int64).tolist() == list(range(101))


def _corrupt(img, at, fn):
    b = bytearray(img)
    b[at] = fn(b[at])
    return bytes(b)


def test_walker_rejects_single_byte_corruptions():
    img, _, _ = _encoder_shaped_file()
    _, pages = C.walk(img)
    p = [x for x in pages if x["col"] == "d" and x["kind"] == "data"][0]
    bw_at = p["body_offset"] + p["values_at"]
    run_at = bw_at + 1
    last = p["body_offset"] + len(p["body"]) - 1  # the last packed byte: 101 rows leave 3 padding slots of 3 bits
    with pytest.raises(C.PageError, match="bit width byte"):
        C.walk(_corrupt(img, bw_at, lambda x: x + 1))
    with pytest.raises(C.PageError, match="run header"):
        C.walk(_corrupt(img, run_at, lambda x: x + 2))
    with pytest.raises(C.PageError, match="padding"):
        C.walk(_corrupt(img, last, lambda x: x | 0x80))
    # the unchanged file still passes, and a change inside the used bits is a value change, not a structural one
    C.walk(img)
    assert struct.unpack_from("<I", img, len(img) - 8)[0] > 0
