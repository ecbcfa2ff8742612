"""LZ4 page bodies for the page decoder's tests (tests/test_lz4_host.py on the CPU, tests/test_gpu_lz4.py on the GPU).

`valid()` gives (name, codec, stream, data) tuples that must decode to `data` bit for bit: pyarrow's `lz4_raw` at several
levels over a grid of inputs, blocks written sequence by sequence for the edges a compressor rarely emits (offset 65 535,
the extension-byte edges of both lengths, a match whose source is the block's first byte, the decoder's short-sequence
path at the end of a block), and Hadoop-framed bodies (codec 5).  `damaged()` gives (name, codec, stream, uncompressed
length, check) where `check` is the Lz4Error (hyperspace_b200/csrc/lz4_block.h) the decoder must report.  `mutations()`
gives ~2 000 seeded edits of valid codec-7 streams, whose verdict `pyarrow_accepts` settles.
"""
import functools
import struct

import numpy as np
import pyarrow as pa

# hyperspace_b200/csrc/lz4_block.h: Lz4Error
TRUNCATED, OFFSET_ZERO, BEFORE_START, OUTPUT_OVERRUN, OUTPUT_SHORT, END_OF_BLOCK = range(1, 7)
LZ4_HADOOP, LZ4_RAW = 5, 7


def compress(data: bytes, level: int = 1) -> bytes:
    return pa.Codec("lz4_raw", compression_level=level).compress(data, asbytes=True)


def pyarrow_accepts(stream: bytes, n: int) -> bool:
    """pyarrow's verdict on a raw block of exactly n output bytes: it decodes with room for n, fails with room for n - 1,
    and its sequences make n bytes.  pyarrow does not report an output shorter than the room it was given, and the
    room-for-n-1 test alone misses a block that LZ4_decompress_safe accepts only because of room it does not fill."""
    codec = pa.Codec("lz4_raw")
    try:
        codec.decompress(stream, decompressed_size=n)
    except (OSError, ValueError):
        return False
    if n > 0:
        try:
            codec.decompress(stream, decompressed_size=n - 1)
            return False
        except (OSError, ValueError):
            pass
    return len(decode(stream)) == n


def pyarrow_decode(stream: bytes, n: int) -> bytes:
    return pa.Codec("lz4_raw").decompress(stream, decompressed_size=n, asbytes=True)


# ---- a writer of chosen sequences -------------------------------------------------------------------------------------
def _ext(n: int) -> bytes:
    out = bytearray()
    while n >= 255:
        out.append(255)
        n -= 255
    out.append(n)
    return bytes(out)


def seq(lit: bytes, offset=None, match_len=None) -> bytes:
    """One sequence: the literals, then (unless offset is None: the last sequence) a match of match_len >= 4 bytes."""
    ln = min(len(lit), 15)
    mn = 0 if offset is None else min(match_len - 4, 15)
    b = bytearray([ln << 4 | mn])
    if ln == 15:
        b += _ext(len(lit) - 15)
    b += lit
    if offset is None:
        return bytes(b)
    b += struct.pack("<H", offset)
    if mn == 15:
        b += _ext(match_len - 4 - 15)
    return bytes(b)


def decode(stream: bytes) -> bytes:
    """A plain restatement of a raw block's sequences (no end-of-block checks): what a hand-built block holds."""
    out, p = bytearray(), 0
    while True:
        token = stream[p]
        p += 1
        lit = token >> 4
        if lit == 15:
            while True:
                b = stream[p]
                p += 1
                lit += b
                if b != 255:
                    break
        out += stream[p:p + lit]
        p += lit
        if p == len(stream):
            return bytes(out)
        off = stream[p] | stream[p + 1] << 8
        p += 2
        ml = token & 15
        if ml == 15:
            while True:
                b = stream[p]
                p += 1
                ml += b
                if b != 255:
                    break
        for _ in range(ml + 4):
            out.append(out[-off])


def hadoop(groups) -> bytes:
    """Hadoop's Lz4Codec framing: groups = [[chunk data, ...], ...]; each chunk is compressed into its own block."""
    out = bytearray()
    for chunks in groups:
        out += struct.pack(">I", sum(len(c) for c in chunks))
        for c in chunks:
            block = compress(c)
            out += struct.pack(">I", len(block)) + block
    return bytes(out)


# ---- inputs ---------------------------------------------------------------------------------------------------------------
def table_t_pages(n: int = 30_000):
    """PLAIN bytes of table T's columns, and the dictionary-index bytes of pyarrow's data pages of a dictionary column."""
    import io

    import pyarrow.parquet as pq

    from oracle import oracle as O
    from parquet_shapes import read_struct

    cols = O.synthetic_table(0, n, 5)
    plain = {c: v.tobytes() for c, v in cols.items()}
    sink = io.BytesIO()
    pq.write_table(pa.table({"v1": cols["v1"]}), sink, compression="none", data_page_size=64 << 10)
    img = sink.getvalue()
    md = pq.ParquetFile(io.BytesIO(img)).metadata.row_group(0).column(0)
    p = md.dictionary_page_offset or md.data_page_offset
    end = p + md.total_compressed_size
    idx = []
    while p < end:
        h, p = read_struct(img, p)
        if h[1] == 0:  # DATA_PAGE: the bit width byte and the index runs
            idx.append(img[p:p + h[3]])
        p += h[3]
    return plain, idx


@functools.lru_cache(maxsize=1)
def inputs():
    rng = np.random.default_rng(5)
    plain, idx = table_t_pages()
    strings = b"".join(struct.pack("<I", len(s)) + s for s in
                       (f"key-{v}".encode() for v in rng.integers(0, 3000, 8000)))
    out = {
        "random": rng.integers(0, 256, 100_000, dtype=np.uint8).tobytes(),
        "zeros": bytes(100_000),
        "strings": strings,
        "dict_index": b"".join(idx),
    }
    out.update({f"T_{c}": v for c, v in plain.items()})
    for period in range(1, 41):  # overlapping matches at every small offset
        unit = rng.integers(0, 256, period, dtype=np.uint8).tobytes()
        out[f"period{period}"] = (unit * (3000 // period + 1))[:3000] + unit[:period // 2]
    return out


def _short_path_tail():
    """Blocks that end on the decoder's short-sequence path: a match of at most 18 bytes after at most 14 literals, taken
    with 32 bytes of output left, followed by fewer than 5 last literals (down to none)."""
    rng = np.random.default_rng(8)
    head = seq(rng.integers(0, 256, 80, dtype=np.uint8).tobytes(), 10, 20)  # 100 bytes of output
    out = []
    for lit, ml, k in ((14, 18, 0), (13, 18, 1), (10, 18, 4), (14, 17, 1)):
        s = head + bytes([lit << 4 | (ml - 4)]) + rng.integers(0, 256, lit, dtype=np.uint8).tobytes() + struct.pack("<H", 8) \
            + bytes([k << 4]) + rng.integers(0, 256, k, dtype=np.uint8).tobytes()
        out.append((f"short_path_lit{lit}_match{ml}_last{k}", s))
    return out


def hand_built():
    rng = np.random.default_rng(6)
    r = lambda k: rng.integers(0, 256, k, dtype=np.uint8).tobytes()  # noqa: E731
    out = [("offset65535", seq(r(70_000), 65535, 300) + seq(r(20)))]
    for x in (14, 15, 16, 270, 271, 525):
        out.append((f"literals{x}", seq(r(x), 3, 20) + seq(r(x))))
        out.append((f"match{x + 4}", seq(r(20), 7, x + 4) + seq(r(9))))
        out.append((f"match{x}_offset1", seq(r(1), 1, x) + seq(r(12))))
    out.append(("match_from_first_byte", seq(r(30), 30, 40) + seq(r(12))))
    out.append(("match_from_first_byte_overlapping", seq(r(3), 3, 50) + seq(r(7), 60, 16) + seq(r(6))))
    out.append(("margins_exact", seq(r(1), 1, 4) + seq(r(8))))  # match at 12 bytes before the end, 8 literals after it
    out.append(("match_ends_5_before_the_end", seq(r(20), 8, 10) + seq(r(5))))
    out += _short_path_tail()
    return out


def plausible_header_block():
    """A raw block whose first 8 bytes read as a Hadoop group header that fits the page: U = 0x10010100 (268 501 248
    bytes), C = 65 551.  Its chunk does not decode, so codec 5 falls back to the raw block."""
    total = 0x10010100 + 1000
    body = seq(b"\x01", 1, 4) + bytes([0x00]) + struct.pack("<H", 1) + bytes([0x0F]) + struct.pack("<H", 1) + \
        _ext(total - 9 - 20 - 4 - 15) + seq(bytes(range(20)))
    assert struct.unpack(">II", body[:8]) == (0x10010100, 65551)
    return body, b"\x01" * (total - 20) + bytes(range(20))


def valid(large: bool = True):
    """(name, codec, stream, data)"""
    out = []
    for nm, data in inputs().items():
        for level in (1, 3, 9, 12):
            out.append((f"{nm}/l{level}", LZ4_RAW, compress(data, level), data))
    rng = np.random.default_rng(9)
    for size in (0, 1, 12, 13):
        for nm, data in (("random", rng.integers(0, 256, size, dtype=np.uint8).tobytes()), ("zeros", bytes(size))):
            out.append((f"size{size}_{nm}", LZ4_RAW, compress(data), data))
    big = rng.integers(0, 50, 1_500_000, dtype=np.uint8).tobytes()  # pages above 1 MB
    for level in (1, 12):
        out.append((f"big1.5MB/l{level}", LZ4_RAW, compress(big, level), big))
    for nm, s in hand_built():
        out.append((nm, LZ4_RAW, s, decode(s)))
    # codec 5: Hadoop's framing, and raw blocks under it
    plain = inputs()["T_v1"] + inputs()["T_k"] + inputs()["strings"]
    k256 = [plain[i:i + (256 << 10)] for i in range(0, len(plain), 256 << 10)]
    out.append(("hadoop_one_group_one_chunk", LZ4_HADOOP, hadoop([[plain]]), plain))
    out.append(("hadoop_256k_chunks_in_own_groups", LZ4_HADOOP, hadoop([[c] for c in k256]), plain))
    out.append(("hadoop_one_group_several_chunks", LZ4_HADOOP, hadoop([k256]), plain))
    out.append(("hadoop_two_groups_of_several_chunks", LZ4_HADOOP, hadoop([k256[:2], k256[2:]]), plain))
    out.append(("hadoop_empty_group_between", LZ4_HADOOP, hadoop([[plain[:5000]], [b""], [plain[5000:9000]]]), plain[:9000]))
    out.append(("hadoop_empty_body", LZ4_HADOOP, b"", b""))
    out.append(("hadoop_raw_fallback", LZ4_HADOOP, compress(plain), plain))
    out.append(("hadoop_raw_fallback_hand_built", LZ4_HADOOP, hand_built()[0][1], decode(hand_built()[0][1])))
    if large:
        body, data = plausible_header_block()
        out.append(("hadoop_raw_fallback_plausible_header", LZ4_HADOOP, body, data))
    return out


def damaged():
    """(name, codec, stream, uncompressed length, check)"""
    rng = np.random.default_rng(10)
    r = lambda k: rng.integers(0, 256, k, dtype=np.uint8).tobytes()  # noqa: E731
    good = seq(r(20), 5, 10) + seq(r(6))  # 36 bytes of output
    n = len(decode(good))
    out = [
        ("empty_stream", LZ4_RAW, b"", 10, TRUNCATED),
        ("cut_in_literals", LZ4_RAW, good[:11], n, TRUNCATED),
        ("cut_in_offset", LZ4_RAW, good[:23], n, TRUNCATED),
        ("cut_in_literal_extension", LZ4_RAW, bytes([0xF0]), 300, TRUNCATED),
        ("cut_in_match_extension", LZ4_RAW, seq(r(20), 5, 300)[:-2], 400, TRUNCATED),
        ("byte_after_last_literals", LZ4_RAW, seq(r(20)) + b"\x00", 20, TRUNCATED),
        ("offset_zero", LZ4_RAW, seq(r(20), 0, 8) + seq(r(10)), 38, OFFSET_ZERO),
        ("offset_zero_short_path", LZ4_RAW, seq(r(14), 0, 8) + seq(r(20)), 42, OFFSET_ZERO),
        ("match_before_start", LZ4_RAW, seq(r(5), 6, 4) + seq(r(10)), 19, BEFORE_START),
        ("match_far_before_start", LZ4_RAW, seq(r(100), 65535, 20) + seq(r(10)), 130, BEFORE_START),
        ("literals_overrun", LZ4_RAW, good, n - 1, OUTPUT_OVERRUN),
        ("match_overrun", LZ4_RAW, seq(r(20), 5, 100) + seq(r(6)), 50, OUTPUT_OVERRUN),
        ("zero_length_page_with_literals", LZ4_RAW, seq(b"a"), 0, OUTPUT_OVERRUN),
        ("output_short", LZ4_RAW, good, n + 1, OUTPUT_SHORT),
        ("output_short_by_much", LZ4_RAW, good, n + 1000, OUTPUT_SHORT),
        ("match_into_last_5", LZ4_RAW, seq(r(20), 8, 11) + seq(r(4)), 35, END_OF_BLOCK),
        ("match_ends_the_block", LZ4_RAW, seq(r(20), 8, 11) + seq(b""), 31, END_OF_BLOCK),
        ("match_starts_in_last_12", LZ4_RAW, seq(r(5), 1, 4) + seq(r(6)), 15, END_OF_BLOCK),
        ("short_path_needs_32_left", LZ4_RAW, seq(r(80), 10, 20) + bytes([0xDE]) + r(13) + struct.pack("<H", 8) + b"\x00",
         100 + 13 + 18, END_OF_BLOCK),  # 31 bytes of output left at the token
        ("short_path_needs_offset_8", LZ4_RAW, seq(r(80), 10, 20) + bytes([0xEE]) + r(14) + struct.pack("<H", 7) + b"\x00",
         100 + 32, END_OF_BLOCK),
        ("match_extension_leaves_4_bytes", LZ4_RAW, seq(r(20), 8, 40) + seq(r(3)), 63, END_OF_BLOCK),
        ("match_in_a_zero_length_page", LZ4_RAW, b"\x00\x00\x00", 0, END_OF_BLOCK),
    ]
    # codec 5: a body that fails as groups is decoded as one raw block, whose check is reported; a group header with U >= 256
    # makes the raw attempt start with a match before any output
    plain = inputs()["T_v1"][:50_000]
    body = bytearray(hadoop([[plain]]))
    body[8] = 0x0F  # the chunk's first token: a match before any output
    out.append(("hadoop_chunk_damaged", LZ4_HADOOP, bytes(body), len(plain), BEFORE_START))
    out.append(("hadoop_group_longer_than_page", LZ4_HADOOP, hadoop([[plain]]), len(plain) - 1, BEFORE_START))
    out.append(("hadoop_group_short_of_page", LZ4_HADOOP, hadoop([[plain]]), len(plain) + 1, BEFORE_START))
    out.append(("hadoop_trailing_bytes", LZ4_HADOOP, hadoop([[plain]]) + b"\x00\x00\x00", len(plain), BEFORE_START))
    out.append(("hadoop_cut_chunk", LZ4_HADOOP, hadoop([[plain]])[:-10], len(plain), BEFORE_START))
    out.append(("raw_under_codec5_damaged", LZ4_HADOOP, seq(r(20), 0, 8) + seq(r(10)), 38, OFFSET_ZERO))
    return out


def mutations(count: int = 2000):
    """(name, stream, uncompressed length): seeded byte flips, truncations, length-byte edits and size edits of valid
    codec-7 streams, half of them within the last 40 bytes, where the end-of-block rules apply."""
    rng = np.random.default_rng(12)
    ins = inputs()
    bases = [(f"{nm}/l{lv}", compress(ins[nm][:size], lv), ins[nm][:size]) for nm, lv, size in (
        ("period3", 1, 3000), ("period17", 9, 3000), ("T_v1", 1, 8000), ("T_v3", 12, 8000), ("strings", 3, 6000),
        ("dict_index", 1, 6000), ("random", 1, 300), ("zeros", 1, 2000), ("T_k", 1, 800))]
    bases += [(nm, s, decode(s)) for nm, s in hand_built() if len(s) < 5000]
    out = []
    for i in range(count):
        nm, s, data = bases[i % len(bases)]
        s, n = bytearray(s), len(data)
        pos = int(rng.integers(max(0, len(s) - 40), len(s))) if rng.random() < 0.5 else int(rng.integers(0, len(s)))
        kind = ("flip", "cut", "length", "size")[int(rng.integers(0, 4))]
        if kind == "flip":
            s[pos] ^= int(rng.integers(1, 256))
        elif kind == "cut":
            del s[pos:]
        elif kind == "length":
            s[pos] = int(rng.choice([0x00, 0xFF, 0x0F, 0xF0, (s[pos] + 1) & 0xFF, (s[pos] - 1) & 0xFF, (s[pos] + 16) & 0xFF,
                                     (s[pos] - 16) & 0xFF]))
        else:
            n = max(0, n + int(rng.choice([-5, -1, 1, 5])))
        out.append((f"{nm}/{kind}@{pos}#{i}", bytes(s), n))
    return out


def records(cases) -> bytes:
    """the host driver's input: [u32 codec][u32 compressed length][u32 uncompressed length][bytes] per case"""
    return b"".join(struct.pack("<III", c, len(s), n) + s for c, s, n in cases)
