"""CPU self-checks of the hand-built Parquet shapes (tests/parquet_shapes.py): the restated decoder limits still match
the CUDA source, pyarrow reads every file to the case's expected columns bit for bit (an independent check of the
writer), and every case has the shape it claims -- measured from the bytes, not from the case's description -- and takes
the decoder path it claims.  A case that drifted off its boundary would still pass on the GPU and test nothing."""
import os
import re

import numpy as np
import pyarrow as pa
import pyarrow.parquet as pq
import pytest

import parquet_shapes as S

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _src(*parts):
    with open(os.path.join(ROOT, "hyperspace_b200", "csrc", *parts)) as f:
        return f.read()


def test_limits_match_the_decoder_source():
    dec, eng, ker, hdr = _src("parquet_decode.cu"), _src("engine.cu"), _src("kernels.h"), _src("engine.h")

    def const(text, name):
        return int(re.search(rf"constexpr (?:int|uint32_t) {name} = (\d+);", text).group(1))

    assert const(dec, "kSmemDict") == S.SMEM_DICT
    assert "pg.dict_count <= (carry ? kSmemDict * 4 : kSmemDict)" in dec and S.SMEM_DICT_CARRIED == 4 * S.SMEM_DICT
    assert const(dec, "kRunTable") == S.RUN_TABLE
    assert const(dec, "kMaxPerEntry") == S.MAX_PER_ENTRY
    assert const(dec, "kTileRows") == S.TILE_ROWS
    assert f"for (int r = 0; r < {S.ALL_VALID_RUNS} && covered < n && all_ones; r++)" in dec
    assert f"idx_bw >= 1 && idx_bw <= {S.GROUP_MAX_BW} && dict_in_smem && W != 1" in dec
    assert f"const int ngroups = n / 8 - {S.GROUP_TAIL};" in dec
    assert "pg.num_values >= zc_tile_rows" in dec
    assert const(ker, "kFusedTileLocal") == S.ZC_TILE
    assert const(eng, "kAgreeCap") == S.AGREE_CAP
    assert const(eng, "kMaxSpec") == S.MAX_SPEC
    assert const(hdr, "kMaxCarried") == S.MAX_CARRIED
    assert const(ker, "kMaxDictEntries") == S.MAX_DICT_ENTRIES
    assert "dict_bytes <= 0.9 * plain_bytes" in eng


def test_thrift_round_trip():
    w = S.ThriftWriter()
    w.i32(1, -5).i64(20, 2**40).binary(21, b"xy").boolean(22, False).begin(40).i32(1, 7).end()
    w.list(41, S.T_I32, 20).raw(b"".join(S.varint(S._zz(i)) for i in range(20)))
    w.end()
    got, end = S.read_struct(bytes(w.b))
    assert end == len(w.b)
    assert got == {1: -5, 20: 2**40, 21: b"xy", 22: False, 40: {1: 7}, 41: list(range(20))}


def test_run_encoding_reads_back():
    rng = np.random.default_rng(0)
    for bw in (0, 1, 3, 8, 9, 17, 25, 32):
        vals = rng.integers(0, 1 << bw, size=37) if bw else np.zeros(37, np.int64)
        runs = [S.rle(5, (1 << bw) - 1 if bw else 0), S.packed(vals), S.rle(300, 0)]
        b = S.encode_runs(runs, bw)
        parsed = S.parse_runs(b, 0, len(b), bw, 5 + 40 + 300)
        assert [(k, c) for k, c, _, _ in parsed] == [("rle", 5), ("packed", 40), ("rle", 300)]
        assert np.array_equal(S.run_values(runs, 45)[5:42], vals)


def _arrow_values(arr, ptype):
    arr = arr.combine_chunks() if hasattr(arr, "combine_chunks") else arr
    valid = np.asarray(arr.is_valid())
    if ptype == S.BYTE_ARRAY:
        return np.array([x if x is not None else b"" for x in arr.to_pylist()], dtype=object), valid
    if ptype == S.BOOLEAN:
        return np.array([bool(x) if x is not None else False for x in arr.to_pylist()], dtype=np.uint8), valid
    dt = S.DTYPE[ptype]
    return arr.fill_null(dt(0)).to_numpy(zero_copy_only=False).astype(dt), valid


def _same(a, b):
    if a.dtype == object:
        return list(a) == list(b)
    return a.tobytes() == b.tobytes()


@pytest.mark.parametrize("name", list(S.CASES))
def test_pyarrow_reads_the_expected_columns(name):
    images, expected, specs = S.case_data(name)
    tables = [pq.ParquetFile(pa.BufferReader(img)).read() for img in images]
    t = pa.concat_tables(tables)
    for col in specs[0].cols:
        values, valid = expected[col.name]
        got, got_valid = _arrow_values(t.column(col.name), col.ptype)
        want_valid = np.ones(len(values), bool) if valid is None else valid
        assert np.array_equal(got_valid, want_valid), col.name
        if col.ptype != S.BYTE_ARRAY:
            values = np.where(want_valid, values, 0).astype(values.dtype)
        assert _same(got, values), col.name


@pytest.mark.parametrize("name", list(S.REFUSALS))
def test_pyarrow_reads_the_refused_files(name):
    specs, cols, _ = S.REFUSALS[name]()
    for img in (S.write_file(s) for s in specs):
        t = pq.ParquetFile(pa.BufferReader(img)).read()
        assert t.num_rows == sum(p.rows for p in specs[0].cols[0].chunks[0].pages)
    if name == "delta_binary_packed_page":
        assert t.column("x").to_pylist() == list(range(100, 300))


def _matches(path, page, want, carried):
    for k, v in want.items():
        if k == "col":
            if page["col"] != v:
                return False
        elif k == "carried":
            if (page["col"] in carried) != v:
                return False
        elif path[k] != v:
            return False
    return True


def _tile_crossing_packed(pg):
    at = 0
    for kind, count, _, _ in pg.get("idx_runs", []):
        if kind == "packed" and at // S.TILE_ROWS != (at + count - 1) // S.TILE_ROWS and count:
            return True
        at += count
    return False


@pytest.mark.parametrize("name", list(S.CASES))
def test_case_has_its_claimed_shape(name):
    images, expected, specs = S.case_data(name)
    a = S.analyse(name)
    pages, other, paths = a["pages"], a["other"], a["paths"]
    cl = S.CLAIMS[name]
    dpages = [p for p in pages if p["enc"] in (S.PLAIN_DICTIONARY, S.RLE_DICTIONARY)]
    ppages = [p for p in pages if p["enc"] == S.PLAIN and p["ptype"] in S.FIXED]
    assert sum(p["n"] for p in pages if p["col"] == "k") == len(expected["k"][0])
    for want in cl.get("paths", []):
        assert any(_matches(path, pg, want, a["carried"]) for pg, path in zip(pages, paths)), \
            (want, sorted({(pg["col"], tuple(sorted(path.items()))) for pg, path in zip(pages, paths) if pg["col"] == want.get("col")}))
    if "carried" in cl:
        assert a["carried"] == cl["carried"]
    if "zero_copy" in cl:
        assert a["zero_copy"] == cl["zero_copy"]
    if "dict_sizes" in cl:
        assert set(cl["dict_sizes"]) <= {d[1] for d in other["dict"]}, other["dict"]
    if "dict_encodings" in cl:
        assert cl["dict_encodings"] == {d[2] for d in other["dict"]} == {p["enc"] for p in dpages}
    if "bws" in cl:
        assert cl["bws"] <= {p["bw"] for p in dpages}
    if "page_rows" in cl:
        for c, rows in cl["page_rows"].items():
            assert [p["n"] for p in pages if p["col"] == c] == rows
    if "first_row_mod8" in cl:
        assert cl["first_row_mod8"] <= {p["first_row"] % 8 for p in dpages}
    if "run_data_mod4" in cl:
        assert cl["run_data_mod4"] <= {p["run_data_mod"] % 4 for p in dpages if p["single_run"]}
    if "value_mod4" in cl:
        assert cl["value_mod4"] <= {p["value_mod"] % 4 for p in ppages if S.WIDTH[p["ptype"]] == 4}
    if "value_mod8" in cl:
        assert cl["value_mod8"] <= {p["value_mod"] for p in ppages if S.WIDTH[p["ptype"]] == 8}
    if cl.get("claimed_groups_over_rows"):
        firsts = [p["idx_runs"][0] for p in dpages if p["idx_runs"]]
        full = [p for p in dpages if p["single_run"] and p["idx_runs"][0][3] * 8 > p["n"]]
        assert firsts and len(full) == len(dpages)
    if "max_idx_runs_min" in cl:
        in_tile = [sum(1 for _ in _runs_starting_before(p["idx_runs"], S.TILE_ROWS)) for p in dpages]
        assert max(in_tile) > S.RUN_TABLE and max(len(p["idx_runs"]) for p in dpages) >= cl["max_idx_runs_min"]
    if "idx_run_lengths" in cl:
        assert cl["idx_run_lengths"] <= {(k, c) for p in dpages for k, c, _, _ in p["idx_runs"]}
    if cl.get("packed_run_across_tile"):
        assert any(_tile_crossing_packed(p) for p in dpages)
    if "rle_value_bytes" in cl:
        assert cl["rle_value_bytes"] <= {(p["bw"] + 7) // 8 for p in dpages if any(r[0] == "rle" for r in p["idx_runs"])}
    if "multibyte_headers" in cl:
        assert cl["multibyte_headers"] <= {hl for p in dpages for _, _, hl, _ in p["idx_runs"]}
    if "def_runs_per_page" in cl:
        assert set(cl["def_runs_per_page"]) <= {len(p["def_runs"]) for p in pages if p["def_runs"]}
    if cl.get("packed_all_ones"):
        assert any(p["levels"] == "general" and S._level_values(p["def_runs"], p["n"]).all() for p in pages if p["def_runs"])
    if "null_rows" in cl:
        nulls = set()
        for p in pages:
            if p["def_runs"]:
                nulls |= set(np.flatnonzero(S._level_values(p["def_runs"], p["n"]) == 0).tolist())
        assert cl["null_rows"] <= nulls
    if "index_pages" in cl:
        assert other["index"] == cl["index_pages"]
    if cl.get("v2_uncompressed_in_snappy"):
        v2s = [p for p in pages if p["v2"] and p["codec"] == S.SNAPPY]
        assert any(p["compressed"] for p in v2s) and any(not p["compressed"] for p in v2s)
    if cl.get("page_stats"):
        assert dpages and all(p["stats"] for p in dpages)
    if cl.get("fallback"):
        f = [p["enc"] for p in pages if p["col"] == "f"]
        assert f[0] == S.PLAIN_DICTIONARY and f[-1] == S.PLAIN and f == sorted(f, reverse=True)
    if "union" in cl:
        assert {c: len(a["unions"][c]) for c in cl["union"]} == cl["union"]
    if cl.get("all_ones_values"):
        assert (expected["m"][0] == -1).any()
        assert (expected["n"][0].view(np.uint64) == np.uint64(0xFFFFFFFFFFFFFFFF)).any()
    if "page_edges_mod_tile" in cl:
        edges = np.cumsum([p["n"] for p in pages if p["col"] == "a"])[:-1]
        assert cl["page_edges_mod_tile"] <= set((edges % S.ZC_TILE).tolist())
    if "file_rows" in cl:
        assert other["file_rows"] == cl["file_rows"]
    if cl.get("windows"):
        edges = set()
        for c in ("a", "b", "c"):
            edges |= set(np.cumsum([p["n"] for p in pages if p["col"] == c and p["file"] == 0])[:-1].tolist())
        starts = {lo for lo, _ in S.window_queries()}
        ends = {hi for _, hi in S.window_queries()}
        for e in edges:
            assert {e - 1, e, e + 1} <= starts and {e - 1, e, e + 1} <= ends


def _runs_starting_before(runs, limit):
    at = 0
    for r in runs:
        if at >= limit:
            return
        yield r
        at += r[1]


def test_boundary_pairs_straddle_their_limits():
    """The cases on either side of one limit differ by one unit and take different paths."""
    def dict_path(name):
        a = S.analyse(name)
        return {path["dict"] for pg, path in zip(a["pages"], a["paths"]) if pg["col"] == "d"}
    assert dict_path("dict_2048_entries_in_shared_memory") == {"smem"}
    assert dict_path("dict_2049_entries_in_global_memory") == {"global"}
    assert dict_path("dict_8192_entries_carried_in_shared_memory") == {"smem"}
    assert dict_path("dict_8193_entries_not_carried") == {"global"}
    lv = {n: {p["levels"] for p in S.analyse(n)["pages"] if p["col"] == "o"}
          for n in ("levels_all_valid_as_64_rle_runs", "levels_all_valid_as_65_rle_runs")}
    assert lv == {"levels_all_valid_as_64_rle_runs": {"all_valid"}, "levels_all_valid_as_65_rle_runs": {"general"}}
    assert S.analyse("union_of_8192_dictionary_values")["carried"] == ["u"]
    assert S.analyse("union_of_8193_dictionary_values")["carried"] == []
    zc = S.analyse("zero_copy_pages_of_4095_4096_4097_rows")
    assert min(p["n"] for p in zc["pages"] if p["col"] == "b") == S.ZC_TILE - 1
    assert min(p["n"] for p in zc["pages"] if p["col"] == "a") == S.ZC_TILE
