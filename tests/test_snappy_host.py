"""The snappy corpus (tests/snappy_corpus.py) on the CPU: its restatement of the format agrees with the C++ snappy library
(through pyarrow) on every valid, damaged and mutated stream; every case has the shape its name claims; and the limits
the corpus restates still stand in hyperspace_b200/csrc/snappy.cu at the lines it cites."""
import os
import re

import pytest

import snappy_corpus as S

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_cited_lines_still_say_what_the_corpus_assumes():
    lines = open(os.path.join(ROOT, "hyperspace_b200", "csrc", "snappy.cu")).read().split("\n")
    at = lambda n: lines[n - 1]  # noqa: E731
    assert re.search(rf"kBlockBytes = {S.BLOCK};", at(40))
    assert re.search(rf"kCoopLiteral = {S.COOP_LITERAL};", at(41))
    assert re.search(rf"kSeg = {S.SEG};", at(42))
    assert "n_src >= 32u * 1024u ? 1024u : (n_src >= 32u * 512u ? 512u : kSeg)" in at(117)
    assert (S.SEG_512_FROM, S.SEG_1024_FROM) == (32 * 512, 32 * 1024)
    assert "base = max(base, pos0 & ~(seg - 1))" in at(119)
    assert f"before <= seg_lo + {S.GUESS_SKIP}" in at(139)
    assert "e.offset > 0xffffu ? INT_MAX" in at(86) and S.MAX_OFFSET_PARALLEL == 0xffff
    assert "wk.reach > (int32_t)in_block" in at(159)
    assert "e.offset > ib" in at(165) and "(out & (kBlockBytes - 1)) == 0 && out < dst_len" in at(171)
    assert f"p < {S.PREAMBLE_BYTES}" in at(268) and "src[4] >= 16" in at(275)
    assert f"e.offset >= {S.FAR}" in at(298)
    assert "e.len >= kCoopLiteral" in "\n".join(lines[285:300])
    assert "pos != in_hi ? 6u" in "\n".join(lines[310:320])


def test_valid_cases_decode_as_the_library_does():
    cases = S.valid()
    assert len({c.name for c in cases}) == len(cases)
    for c in cases:
        want, why = S.decode(c.stream, c.n)
        assert why is None, (c.name, why)
        assert S.pyarrow_accepts(c.stream, c.n), c.name
        assert S.pyarrow_decode(c.stream, c.n) == want, c.name


def test_cases_have_the_shape_their_names_claim():
    cases = S.valid()
    wrong = []
    for c in cases:
        f = S.facts(c.stream)
        wrong += [(c.name, k, f[k], v) for k, v in c.claims.items() if f[k] != v]
    assert not wrong, wrong[:10]
    names = {c.name: c for c in cases}
    # segment sizes on both sides of each threshold, and one and several rounds
    segs = {S.facts(names[f"nsrc_{n}"].stream)["seg"] for n in (16383, 16384, 32767, 32768)}
    assert segs == {256, 512, 1024}
    assert {S.facts(c.stream)["rounds"] for c in cases if c.name.startswith("nsrc_")} >= {1, 2, 3}
    # every path also on the one-lane path
    assert sum(c.name.endswith("/one_lane") for c in cases) >= 90
    assert all(not S.independent(c.stream) for c in cases if c.name.endswith("/one_lane"))
    # the warp copy: every tail after vector counts 32 / 33 and 64 / 65, every destination and source phase
    wl = [c for c in cases if c.name.startswith("warp_literal_nvec") and "/" not in c.name]
    for nvec in (32, 33, 64, 65):
        mine = [c for c in wl if c.name.startswith(f"warp_literal_nvec{nvec}_")]
        tails, dph, sph = set(), set(), set()
        for c in mine:
            head = (16 - c.dst_phase) % 16
            rest = c.n - head
            assert rest // 16 == nvec
            tails.add(rest % 16)
            dph.add(c.dst_phase)
            sph.add((c.src_phase + len(S.varint(c.n)) + len(S.literal(bytes(c.n))) - c.n) % 4)
        assert tails == set(range(16)) and dph == set(range(16)) and sph == set(range(4)), nvec
    # overlapping copies at offsets 1..9, every length above the offset up to 64
    for off in range(1, 10):
        assert S.facts(names[f"overlapping_copies_offset{off}"].stream)["overlaps"] == {off}
    # every header size with its tag at every address phase
    combos = set()
    for c in cases:
        if c.name.startswith("every_header_src_phase") and "/" not in c.name:
            for pos, hdr, _, _, _ in S.elements(c.stream, S.preamble(c.stream)[1]):
                combos.add((hdr, (c.src_phase + pos) % 4))
    assert combos == {(h, p) for h in range(1, 6) for p in range(4)}
    # the literal lengths around the warp copy
    assert {names[f"literal_{n}"].claims["coop_literals"] for n in (63, 64, 65)} == {0, 1}


def test_damaged_streams_are_refused_by_the_library_and_the_restatement():
    cases = S.damaged()
    assert len({c[0] for c in cases}) == len(cases)
    for name, stream, n, _ in cases:
        assert not S.pyarrow_accepts(stream, n), name
        assert S.decode(stream, n)[0] is None, name
    names = {c[0] for c in cases}
    assert {f"offset0_{f}" for f in ("copy1", "copy2", "copy4")} <= names
    assert {"trailing_literal", "preamble_fifth_byte_16", "preamble_fifth_byte_continues"} <= names
    # the forms the C++ library accepts beside them
    assert S.pyarrow_accepts(bytes.fromhex("8480808000") + S.literal(b"abcd"), 4)
    assert S.pyarrow_accepts(bytes.fromhex("040c61626364"), 4)


def test_mutations_agree_with_the_library():
    cases = S.mutations()
    assert len(cases) == 2000
    disagree, accepted = [], 0
    for name, stream, n in cases:
        theirs = S.pyarrow_accepts(stream, n)
        mine, _ = S.decode(stream, n)
        if theirs != (mine is not None) or (theirs and S.pyarrow_decode(stream, n) != mine):
            disagree.append(name)
        accepted += theirs
    assert not disagree, disagree[:10]
    assert 100 < accepted < 1900, accepted  # both verdicts are well represented


@pytest.mark.parametrize("n", [0, 1, 127, 128, 16383, 16384, (1 << 32) - 1])
def test_preamble_forms(n):
    for width in range(len(S.varint(n)), 6):
        s = S.varint(n, width)
        assert S.preamble(s) == (n, width)
    assert S.preamble(S.varint(n, 6)) is None


def test_page_compressors_and_source_files():
    import io

    import numpy as np
    import pyarrow.parquet as pq

    rng = np.random.default_rng(3)
    body = rng.standard_normal(12_000).tobytes()  # a key page's size
    for comp, parallel in ((S.compress_one_lane, False), (S.compress_copies, True), (S.compress_long_literals, True)):
        s = comp(body)
        assert S.decode(s, len(body))[0] == body and S.pyarrow_accepts(s, len(body)), comp.__name__
        assert S.independent(s) == parallel, comp.__name__
    assert S.facts(S.compress_long_literals(body))["coop_literals"] > 90
    assert S.facts(S.compress_copies(np.arange(5000, dtype=np.int64).tobytes()))["n"] == 40_000
    assert not S.pyarrow_accepts(S.compress_zero_offset_copy(body), len(body))
    # pyarrow reads the SNAPPY source as the same rows as the UNCOMPRESSED one, and refuses the damaged one
    plain, snappy = pq.read_table(io.BytesIO(S.source_file(0))), pq.read_table(io.BytesIO(S.source_file(1)))
    assert plain.num_rows == 30_000 and snappy.equals(plain)
    md = pq.ParquetFile(io.BytesIO(S.source_file(1))).metadata.row_group(0)
    assert [md.column(c).compression for c in range(4)] == ["SNAPPY"] * 4
    assert md.column(3).dictionary_page_offset is not None
    with pytest.raises(OSError):
        pq.read_table(io.BytesIO(S.source_file(1, damaged=True)))
