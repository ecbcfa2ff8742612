"""The snappy page decoder (hyperspace_b200/csrc/snappy.cu) on the corpus of tests/snappy_corpus.py, through
hs_k_decompress_blobs: many pages per launch, as the page reader makes them, at every source phase mod 4 and destination
phase mod 16, with v2 level prefixes, pages stored uncompressed, empty pages and an LZ4 page between them.  The output
buffer is pre-filled, so a byte written outside a page's destination shows.  Every valid case decodes to the
restatement's bytes on the path `independent()` predicts; every damaged and mutated stream gets the C++ library's
verdict."""
import re

import numpy as np
import pyarrow as pa
import pytest

import snappy_corpus as S

pytestmark = pytest.mark.gpu

SNAPPY, LZ4_RAW = 1, 7
FILL = 0xA5


@pytest.fixture(scope="module")
def ctx():
    from hyperspace_b200 import _native

    c = _native.Context(0)
    yield c
    c.close()


def _launch(ctx, pages, rng):
    """pages: dicts of stream, n, prefix, compressed, codec, src_phase, dst_phase, want (decoded bytes after the prefix).
    Lays them out with gaps, decodes them in one call and returns (output, expected output, sequential flags)."""
    src, blobs, dst_cursor = bytearray(), [], 0
    for p in pages:
        pre = S.rng_bytes(rng, p["prefix"])
        while (len(src) + p["prefix"]) % 4 != p["src_phase"]:
            src.append(int(rng.integers(0, 256)))
        dst_cursor += int(rng.integers(0, 24))
        while (dst_cursor + p["prefix"]) % 16 != p["dst_phase"]:
            dst_cursor += 1
        blobs.append((len(src), p["prefix"] + len(p["stream"]), dst_cursor, p["prefix"] + p["n"], p["prefix"], p["compressed"],
                      p["codec"]))
        p["dst"] = (dst_cursor, pre + p["want"])
        src += pre + p["stream"]
        src += S.rng_bytes(rng, int(rng.integers(0, 8)))
        dst_cursor += p["prefix"] + p["n"]
    out_len = dst_cursor + int(rng.integers(1, 40))
    want = bytearray([FILL]) * out_len
    for p in pages:
        off, b = p["dst"]
        want[off:off + len(b)] = b
    out, seq = ctx.k_decompress_blobs(bytes(src), blobs, out_len, fill=FILL)
    return out, bytes(want), seq


def _page(stream, n, want, rng, src_phase=None, dst_phase=None, prefix=0, compressed=1, codec=SNAPPY):
    return dict(stream=stream, n=n, want=want, prefix=prefix, compressed=compressed, codec=codec,
                src_phase=int(rng.integers(0, 4)) if src_phase is None else src_phase,
                dst_phase=int(rng.integers(0, 16)) if dst_phase is None else dst_phase)


def _launches(rng):
    """the valid cases in launches of mixed pages: about a third with a v2 prefix of 1..17 bytes, and between them pages
    stored uncompressed, empty pages and (first in some launches) an LZ4 page, which decompress_blobs puts after the
    snappy ones"""
    cases = S.valid()
    order = rng.permutation(len(cases))
    groups, cur, blocks = [], [], 0
    for i in order:
        c = cases[int(i)]
        cur.append(c)
        blocks += max(1, -(-c.n // S.BLOCK))
        if len(cur) >= 24 or blocks > 200:
            groups.append(cur)
            cur, blocks = [], 0
    groups.append(cur)
    # one launch of every page above 64 KB: more than 128 blocks
    groups.append([c for c in cases if c.n > S.BLOCK and c.n < 1 << 20])
    # one launch of only warp-copied single literals: many lanes take the cooperative path in the same step
    groups.append([c for c in cases if c.name.startswith("warp_literal_nvec") and "/" not in c.name])
    lz4_data = S.rng_bytes(rng, 3000, 0, 4)
    for g, group in enumerate(groups):
        pages, meta = [], []
        if g % 3 == 0:
            pages.append(_page(pa.Codec("lz4_raw").compress(lz4_data, asbytes=True), len(lz4_data), lz4_data, rng, codec=LZ4_RAW))
            meta.append(None)
        for j, c in enumerate(group):
            want, _ = S.decode(c.stream, c.n)
            prefix = int(rng.integers(1, 18)) if rng.random() < 0.33 else 0
            pages.append(_page(c.stream, c.n, want, rng, c.src_phase, c.dst_phase, prefix))
            meta.append(c)
            if j % 7 == 3:
                raw = S.rng_bytes(rng, int(rng.integers(1, 300)))
                pages.append(_page(raw, len(raw), raw, rng, compressed=0))
                meta.append(None)
            if j % 11 == 5:
                pages.append(_page(b"\x00", 0, b"", rng, prefix=int(rng.integers(0, 3))))
                meta.append(None)
        yield pages, meta


def test_valid_cases_in_multi_page_launches(ctx):
    from hyperspace_b200 import _native as N

    rng = np.random.default_rng(40)
    wrong, stray, path, most_blocks, n_launches = [], [], [], 0, 0
    for pages, meta in _launches(rng):
        try:
            out, want, seq = _launch(ctx, pages, rng)
        except N.HyperspaceGpuError as e:  # name the pages that fail on their own, or the launch when none does
            alone = []
            for p, c in zip(pages, meta):
                try:
                    _launch(ctx, [p], rng)
                except N.HyperspaceGpuError as one:
                    alone.append((c.name if c else "verbatim/lz4 page", str(one)))
            wrong += alone or [([c.name for c in meta if c], f"launch failed, every page decodes alone: {e}")]
            continue
        n_launches += 1
        most_blocks = max(most_blocks, sum(max(1, -(-p["n"] // S.BLOCK)) for p in pages if p["codec"] == SNAPPY))
        inside = np.zeros(len(want), bool)
        for p, c, sq in zip(pages, meta, seq):
            off, b = p["dst"]
            inside[off:off + len(b)] = True
            if out[off:off + len(b)] != b:
                wrong.append(c.name if c else f"verbatim/lz4 page of {p['n']} bytes")
            if c is not None and sq != (not S.independent(c.stream)):
                path.append((c.name, sq))
            if c is None and p["codec"] == SNAPPY and p["compressed"] and sq:
                path.append(("empty page", sq))
        diff = np.frombuffer(out, np.uint8) != np.frombuffer(want, np.uint8)
        if (diff & ~inside).any():
            stray.append([c.name for c in meta if c])
    assert not wrong, wrong[:10]
    assert not stray, stray[:3]
    assert not path, path[:10]
    assert most_blocks > 128 and n_launches > 10


def _check_of(e):
    m = re.search(r"check (\d+)", str(e))
    return int(m.group(1)) if m else None


def test_damaged_streams_get_the_library_verdict(ctx):
    from hyperspace_b200 import _native as N

    rng = np.random.default_rng(41)
    wrong = []
    for name, stream, n, check in S.damaged():
        page = _page(stream, n, b"", rng, prefix=int(rng.integers(0, 3)))
        try:
            _launch(ctx, [page], rng)
            wrong.append((name, "accepted"))
        except N.HyperspaceGpuError as e:
            if e.code != N.HS_EFORMAT or (check is not None and _check_of(e) != check):
                wrong.append((name, e.code, str(e)))
    assert not wrong, wrong
    # a damaged page among good ones fails the launch, and the context goes on working
    good = S.valid()[0]
    pages = [_page(good.stream, good.n, S.decode(good.stream, good.n)[0], rng) for _ in range(5)]
    bad = S.damaged()[0]
    with pytest.raises(N.HyperspaceGpuError) as e:
        _launch(ctx, pages[:3] + [_page(bad[1], bad[2], b"", rng)] + pages[3:], rng)
    assert e.value.code == N.HS_EFORMAT and _check_of(e.value) == bad[3]
    out, want, _ = _launch(ctx, pages, rng)
    assert out == want


def test_mutations_get_the_library_verdict(ctx):
    from hyperspace_b200 import _native as N

    rng = np.random.default_rng(42)
    disagree, accepted = [], 0
    for name, stream, n in S.mutations():
        theirs = S.pyarrow_accepts(stream, n)
        want = S.pyarrow_decode(stream, n) if theirs else b""
        try:
            out, expect, seq = _launch(ctx, [_page(stream, n, want, rng)], rng)
            if not theirs or out != expect or seq[0] != (not S.independent(stream)):
                disagree.append((name, "accepted", theirs))
        except N.HyperspaceGpuError as e:
            if theirs or e.code != N.HS_EFORMAT:
                disagree.append((name, e.code, theirs))
        accepted += theirs
    assert not disagree, disagree[:10]
    assert accepted > 100


def test_blob_ranges_are_checked(ctx):
    from hyperspace_b200 import _native as N

    s = S.varint(4) + S.literal(b"abcd")
    for blobs, out_len in (([(0, len(s), 0, 4, 0, 1, SNAPPY), (0, len(s), 2, 4, 0, 1, SNAPPY)], 16),  # overlapping outputs
                           ([(1, len(s), 0, 4, 0, 1, SNAPPY)], 16),                                   # past the input
                           ([(0, len(s), 14, 4, 0, 1, SNAPPY)], 16),                                  # past the output
                           ([(0, len(s), 0, 4, 0, 1, 3)], 16),                                        # no such codec
                           ([(0, len(s), 0, 4, 0, 2, SNAPPY)], 16),                                   # compressed not 0 / 1
                           ([(0, 2, 0, 4, 3, 1, SNAPPY)], 16),                                        # prefix beyond the source
                           ([(0, len(s), 0, 2, 3, 1, SNAPPY)], 16)):                                  # prefix beyond the output
        with pytest.raises(N.HyperspaceGpuError) as e:
            ctx.k_decompress_blobs(s, blobs, out_len)
        assert e.value.code == N.HS_EINVAL
    out, seq = ctx.k_decompress_blobs(s, [(0, len(s), 3, 4, 0, 1, SNAPPY)], 9, fill=7)
    assert out == b"\x07" * 3 + b"abcd" + b"\x07" * 2 and seq == [False]


def test_create_index_over_snappy_pages_of_the_corpus_writer(ctx):
    """Source pages from the corpus compressors -- a one-lane key page, long literals, v2 levels before compressed values,
    a compressed dictionary page -- index to the same files as the same rows UNCOMPRESSED; a page holding a zero-offset
    copy fails the build with HS_EFORMAT, and the context builds again after it."""
    from hyperspace_b200 import _native as N

    def build(img):
        res, _ = ctx.create_index([N.FileImage(data=img)], ["k"], ["a", "o", "d"], 8, output=N.HS_OUT_HOST, job_uuid="snappy")
        files = [(f.bucket, res.host_bytes(i)) for i, f in enumerate(res.files)]
        res.free()
        return files

    plain = build(S.source_file(0))
    assert len(plain) == 8
    assert build(S.source_file(1)) == plain
    with pytest.raises(N.HyperspaceGpuError) as e:
        build(S.source_file(1, damaged=True))
    assert e.value.code == N.HS_EFORMAT and "snappy" in str(e.value), str(e.value)
    assert build(S.source_file(1)) == plain
