"""GZIP streams for the page decoder's tests (tests/test_inflate_host.py on the CPU, tests/test_gpu_gzip.py on the GPU).

`valid()` gives (name, stream, data) triples that must decode to `data` bit for bit: Python's zlib over a grid of inputs,
levels, strategies, window sizes and flushes, plus hand-built streams for what zlib never writes (a distance of 32 768, a
distance alphabet with one code or none, every header flag).  `damaged()` gives (name, stream, uncompressed length, check)
where `check` is the InflateError (hyperspace_b200/csrc/inflate.h) the decoder must report.
"""
import struct
import zlib

import numpy as np

# hyperspace_b200/csrc/inflate.h: InflateError
BAD_MAGIC, BAD_METHOD, BAD_FLAGS, HEADER_CRC, STORED_LEN, BLOCK_TYPE, BAD_LENGTHS, BAD_SYMBOL, FAR_DISTANCE, \
    OUTPUT_OVERRUN, OUTPUT_SHORT, TRUNCATED, CRC, ISIZE, TRAILING = range(1, 16)

STRATEGIES = [zlib.Z_DEFAULT_STRATEGY, zlib.Z_FILTERED, zlib.Z_HUFFMAN_ONLY, zlib.Z_RLE, zlib.Z_FIXED]


def gzip_compress(data: bytes, level: int = 6, strategy: int = zlib.Z_DEFAULT_STRATEGY, wbits: int = 15) -> bytes:
    c = zlib.compressobj(level, zlib.DEFLATED, 16 + wbits, 9, strategy)
    return c.compress(data) + c.flush()


def inputs():
    rng = np.random.default_rng(7)
    words = [b"parquet", b"column", b"page", b"spark", b"index", b"bucket", b"hyperspace", b"the", b"a", b"of"]
    text = b" ".join(words[i] for i in rng.integers(0, len(words), 20000))
    walk = np.cumsum(rng.normal(size=20000)).astype(np.float64)
    return {
        "empty": b"",
        "one": b"x",
        "zeros64k": bytes(65536),
        "random": rng.integers(0, 256, 100_000, dtype=np.uint8).tobytes(),
        "text": text,
        "arange_i64": np.arange(20000, dtype=np.int64).tobytes(),
        "f64_walk": walk.tobytes(),
        "f64_rounded": np.round(walk, 2).tobytes(),
        "stored65535": rng.integers(0, 256, 65535, dtype=np.uint8).tobytes(),
        "stored65536": rng.integers(0, 256, 65536, dtype=np.uint8).tobytes(),
        "stored65537": rng.integers(0, 256, 65537, dtype=np.uint8).tobytes(),
    }


# ---- a small DEFLATE writer for the streams zlib never produces ---------------------------------------------------------
class Bits:
    def __init__(self):
        self.acc, self.n, self.out = 0, 0, bytearray()

    def put(self, v: int, k: int):  # k bits of v, LSB first
        self.acc |= (v & ((1 << k) - 1)) << self.n
        self.n += k
        while self.n >= 8:
            self.out.append(self.acc & 0xFF)
            self.acc >>= 8
            self.n -= 8

    def code(self, c: int, k: int):  # a Huffman code, MSB first
        self.put(int(format(c, f"0{k}b")[::-1], 2), k)

    def bytes(self) -> bytes:
        return bytes(self.out) + (bytes([self.acc]) if self.n else b"")


def canonical(lens):
    """RFC 1951 3.2.2: symbol -> (code, length)"""
    count = [0] * 16
    for l in lens:
        count[l] += 1
    count[0] = 0
    code, nxt = 0, [0] * 16
    for l in range(1, 16):
        code = (code + count[l - 1]) << 1
        nxt[l] = code
    out = {}
    for s, l in enumerate(lens):
        if l:
            out[s] = (nxt[l], l)
            nxt[l] += 1
    return out


FIXED_LIT = [8] * 144 + [9] * 112 + [7] * 24 + [8] * 8
LEN_BASE = [3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258]
LEN_EXTRA = [0] * 8 + [1] * 4 + [2] * 4 + [3] * 4 + [4] * 4 + [5] * 4 + [0]
DIST_BASE = [1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537, 2049, 3073, 4097,
             6145, 8193, 12289, 16385, 24577]
DIST_EXTRA = [0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12, 13, 13]


def emit(b: Bits, lit, dist, items):
    """items: ints (literal bytes or raw symbols via ("sym", s)), ("match", length, distance), ("dsym", len_sym, dist_sym)"""
    for it in items:
        if isinstance(it, int):
            b.code(*lit[it])
        elif it[0] == "sym":
            b.code(*lit[it[1]])
        elif it[0] == "dsym":  # a length symbol and a raw distance symbol (None: five zero bits, for an empty set)
            b.code(*lit[it[1]])
            b.put(0, 5) if it[2] is None else b.code(*dist[it[2]])
        else:
            _, length, d = it
            i = max(j for j in range(29) if LEN_BASE[j] <= length)
            b.code(*lit[257 + i])
            b.put(length - LEN_BASE[i], LEN_EXTRA[i])
            j = max(j for j in range(30) if DIST_BASE[j] <= d)
            b.code(*dist[j])
            b.put(d - DIST_BASE[j], DIST_EXTRA[j])


def fixed_block(items, last=True, b=None) -> Bits:
    b = b or Bits()
    b.put(1 if last else 0, 1)
    b.put(1, 2)
    emit(b, canonical(FIXED_LIT), canonical([5] * 32), items + [("sym", 256)])
    return b


def dynamic_block(lit_lens, dist_lens, items, last=True, cl_lens=None) -> Bits:
    """Code lengths sent one symbol each with a code-length code of 4-bit codes for 0..15 (or `cl_lens`)."""
    b = Bits()
    b.put(1 if last else 0, 1)
    b.put(2, 2)
    b.put(len(lit_lens) - 257, 5)
    b.put(len(dist_lens) - 1, 5)
    order = [16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15]
    cl = cl_lens or [4] * 16 + [0, 0, 0]
    b.put(19 - 4, 4)
    for s in order:
        b.put(cl[s], 3)
    clc = canonical(cl)
    for l in list(lit_lens) + list(dist_lens):
        b.code(*clc[l])
    if cl_lens is None:
        emit(b, canonical(lit_lens), canonical(dist_lens), items + [("sym", 256)])
    return b


def member(deflate: bytes, data: bytes, flags: int = 0, extra: bytes = b"x" * 5, name: bytes = b"page.bin",
           comment: bytes = b"a comment", crc=None, isize=None) -> bytes:
    h = bytearray(b"\x1f\x8b\x08" + bytes([flags]) + b"\x00\x00\x00\x00\x00\x03")
    if flags & 4:
        h += struct.pack("<H", len(extra)) + extra
    if flags & 8:
        h += name + b"\0"
    if flags & 16:
        h += comment + b"\0"
    if flags & 2:
        h += struct.pack("<H", zlib.crc32(bytes(h)) & 0xFFFF)
    crc = zlib.crc32(data) if crc is None else crc
    isize = len(data) & 0xFFFFFFFF if isize is None else isize
    return bytes(h) + deflate + struct.pack("<II", crc, isize)


def _flushed(data: bytes, mode: int) -> bytes:
    c = zlib.compressobj(6, zlib.DEFLATED, 31)
    k = len(data) // 3
    return c.compress(data[:k]) + c.flush(mode) + c.compress(data[k:2 * k]) + c.flush(mode) + c.compress(data[2 * k:]) + c.flush()


def valid():
    out = []
    ins = inputs()
    for nm, data in ins.items():
        for level in range(10):
            for st in STRATEGIES:
                out.append((f"{nm}/l{level}/s{st}", gzip_compress(data, level, st), data))
        for wbits in range(9, 15):
            out.append((f"{nm}/w{wbits}", gzip_compress(data, 6, zlib.Z_DEFAULT_STRATEGY, wbits), data))
        for mode, mn in ((zlib.Z_SYNC_FLUSH, "sync"), (zlib.Z_FULL_FLUSH, "full")):
            out.append((f"{nm}/{mn}", _flushed(data, mode), data))
    # byte frequencies 2^17, 2^16, ...: Huffman depth beyond 15, which the compressor limits to 15-bit literal codes
    rng = np.random.default_rng(11)
    skew = np.repeat(np.arange(26, dtype=np.uint8), [max(1, 2 ** (17 - i)) for i in range(26)])
    rng.shuffle(skew)
    skew = skew.tobytes()
    for level in (1, 6, 9):
        out.append((f"skewed15/l{level}", gzip_compress(skew, level, zlib.Z_HUFFMAN_ONLY), skew))
        out.append((f"skewed15/dyn/l{level}", gzip_compress(skew, level), skew))
    run = b"a" * 100_000  # matches of length 258 at distance 1
    out.append(("run258_d1", gzip_compress(run, 9), run))
    # length 258 at distance 32 768 (zlib's window stops 262 bytes short of that)
    head = rng.integers(0, 256, 32768, dtype=np.uint8).tobytes()
    far = head + head[:258 * 3]
    out.append(("run258_d32768", member(fixed_block(list(head) + [("match", 258, 32768)] * 3).bytes(), far), far))
    # a distance alphabet with a single code, and one with none
    lit = [9] * 256 + [2, 2]
    single = b"a" * 10  # the one distance code is distance 1
    out.append(("dist_single_code", member(dynamic_block(lit, [1], [97] + [("match", 3, 1)] * 3).bytes(), single), single))
    lit_only = bytes(range(256))
    out.append(("dist_empty", member(dynamic_block([9] * 256 + [1], [0], list(lit_only)).bytes(), lit_only), lit_only))
    # header flags, one at a time and all together (FTEXT 1, FHCRC 2, FEXTRA 4, FNAME 8, FCOMMENT 16)
    body = ins["text"][:5000]
    raw = zlib.compressobj(6, zlib.DEFLATED, -15)
    deflate = raw.compress(body) + raw.flush()
    for flags in (1, 2, 4, 8, 16, 31):
        out.append((f"flags{flags}", member(deflate, body, flags), body))
    # several members: two and three back to back, and an empty member between
    a, b = ins["text"][:3000], ins["arange_i64"][:8000]
    out.append(("members2", gzip_compress(a) + gzip_compress(b, 9), a + b))
    out.append(("members3", gzip_compress(a, 1) + gzip_compress(b"") + gzip_compress(b, 0), a + b))
    out.append(("members3_flags", member(deflate, body, 31) + gzip_compress(a) + member(deflate, body, 2), body + a + body))
    return out


def damaged():
    out = []
    short_data = b"hello hello hello gzip page world " * 3
    short = gzip_compress(short_data, 6)
    for cut in range(len(short)):
        out.append((f"truncated@{cut}", short[:cut], len(short_data), TRUNCATED))
    flip = bytearray(short)
    flip[-8] ^= 1
    out.append(("crc_flipped", bytes(flip), len(short_data), CRC))
    flip = bytearray(short)
    flip[-4] ^= 1
    out.append(("isize_flipped", bytes(flip), len(short_data), ISIZE))
    out.append(("output_overrun", short, len(short_data) - 1, OUTPUT_OVERRUN))
    out.append(("output_short", short, len(short_data) + 1, OUTPUT_SHORT))
    out.append(("garbage_after", short + b"garbage!", len(short_data), TRAILING))
    out.append(("zeros_after", short + bytes(8), len(short_data), TRAILING))
    out.append(("half_member_after", short + short[:12], 2 * len(short_data), TRUNCATED))
    out.append(("zlib_wrapped", zlib.compress(short_data), len(short_data), BAD_MAGIC))
    raw = zlib.compressobj(6, zlib.DEFLATED, -15)
    out.append(("raw_deflate", raw.compress(short_data) + raw.flush(), len(short_data), BAD_MAGIC))
    bad = bytearray(short)
    bad[2] = 7
    out.append(("method7", bytes(bad), len(short_data), BAD_METHOD))
    bad = bytearray(short)
    bad[3] = 0x20
    out.append(("reserved_flag", bytes(bad), len(short_data), BAD_FLAGS))
    hc = bytearray(member(fixed_block(list(b"ab")).bytes(), b"ab", flags=2))
    hc[10] ^= 0xFF
    out.append(("header_crc", bytes(hc), 2, HEADER_CRC))
    b = Bits()
    b.put(1, 1)
    b.put(3, 2)
    out.append(("block_type3", member(b.bytes(), b""), 0, BLOCK_TYPE))
    stored = bytes([1]) + struct.pack("<HH", 5, 0) + b"hello"
    out.append(("stored_len_nlen", member(stored, b"hello"), 5, STORED_LEN))
    out.append(("oversubscribed_lit", member(dynamic_block([8] * 286, [5] * 30, [97]).bytes(), b"a"), 1, BAD_LENGTHS))
    out.append(("oversubscribed_codelen", member(dynamic_block([8] * 257, [5], [], cl_lens=[1] * 19).bytes() + bytes(64), b""), 0,
                BAD_LENGTHS))
    out.append(("incomplete_lit", member(dynamic_block([9] * 256 + [2], [0], [97]).bytes(), b"a"), 1, BAD_LENGTHS))
    out.append(("incomplete_dist", member(dynamic_block([9] * 256 + [2, 2], [2, 2, 2], [97]).bytes(), b"a"), 1, BAD_LENGTHS))
    out.append(("no_end_of_block", member(dynamic_block([8] * 256 + [0, 8], [1], [], cl_lens=[4] * 16 + [0, 0, 0]).bytes()
                                          + bytes(64), b""), 0, BAD_LENGTHS))
    out.append(("distance_past_start", member(fixed_block([97, ("match", 3, 2)]).bytes(), b"aaaa"), 4, FAR_DISTANCE))
    out.append(("lit_symbol_286", member(fixed_block([97, ("sym", 286)]).bytes(), b"a"), 1, BAD_SYMBOL))
    out.append(("lit_symbol_287", member(fixed_block([97, ("sym", 287)]).bytes(), b"a"), 1, BAD_SYMBOL))
    out.append(("dist_symbol_30", member(fixed_block([97, ("dsym", 257, 30)]).bytes(), b"aaaa"), 4, BAD_SYMBOL))
    out.append(("dist_symbol_31", member(fixed_block([97, ("dsym", 257, 31)]).bytes(), b"aaaa"), 4, BAD_SYMBOL))
    out.append(("dist_in_empty_set", member(dynamic_block([9] * 256 + [2, 2], [0], [97, ("dsym", 257, None)]).bytes(), b"aaaa"), 4,
                BAD_SYMBOL))
    return out


def records(cases) -> bytes:
    """the host driver's input: [u32 compressed length][u32 uncompressed length][bytes] per case"""
    return b"".join(struct.pack("<II", len(s), n) + s for s, n in cases)
