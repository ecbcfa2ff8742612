"""Snappy page bodies for the page decoder's tests (tests/test_snappy_host.py on the CPU, tests/test_gpu_snappy_edges.py on
the GPU), built where the decoder (hyperspace_b200/csrc/snappy.cu) changes path.

The decoder's two kernels: k_snappy_index walks each stream with 32 lanes, each from a guessed start in its own segment,
and finds where every 64 KB output block starts; k_snappy_blocks then decodes one block per lane, or a whole page on one
lane when its blocks are not independent.  Literals of 64 bytes or more are copied by the whole warp.

`valid()` gives Case tuples whose stream must decode to `decode(stream, n)`; each case's `claims` name the limit it sits
on, and `facts()` measures them from the stream.  `damaged()` gives (name, stream, n, check) where check is the decoder's
error number when the path makes it certain (None otherwise).  `mutations()` gives ~2 000 seeded edits of valid streams.
A stream is accepted exactly when the C++ snappy library (what snappy-java, and so Spark, runs) accepts it at the page's
size; `pyarrow_accepts` asks that library.
"""
import functools
from dataclasses import dataclass, field
from typing import Dict, Optional

import numpy as np
import pyarrow as pa

# ---- the limits, each with the snappy.cu line it mirrors --------------------------------------------------------------
BLOCK = 65536           # kBlockBytes (snappy.cu:40): output block of one lane
COOP_LITERAL = 64       # kCoopLiteral (snappy.cu:41): literals from this length on are copied by the whole warp
SEG = 256               # kSeg (snappy.cu:42): least compressed bytes per lane and round of the index walk
SEG_512_FROM = 32 * 512     # snappy.cu:117: n_src from which a lane's segment is 512 bytes
SEG_1024_FROM = 32 * 1024   # snappy.cu:117: ... and 1024 bytes
GUESS_SKIP = 64         # snappy.cu:139: a guessed walk may leave at most this far into the next lane's segment
FAR = 8                 # snappy.cu:298: copies from this offset on load 8 bytes before storing them
MAX_OFFSET_PARALLEL = 0xffff  # snappy.cu:86: a larger offset always leaves its block
PREAMBLE_BYTES = 5      # snappy.cu:268, 275: a varint of 32 bits, the fifth byte below 16

# k_snappy_blocks' error numbers
CHECK_PREAMBLE, CHECK_LENGTH, CHECK_TRUNCATED, CHECK_BEFORE_START, CHECK_SHORT, CHECK_TRAILING = range(1, 7)


def seg_of(n_src: int) -> int:
    return 1024 if n_src >= SEG_1024_FROM else (512 if n_src >= SEG_512_FROM else SEG)


# ---- a writer of chosen elements ------------------------------------------------------------------------------------
def varint(n: int, width: Optional[int] = None) -> bytes:
    """n as a varint; width > the minimal one pads it with continuation bytes (the C++ library accepts such forms)"""
    out = bytearray()
    while n >= 0x80:
        out.append((n & 0x7f) | 0x80)
        n >>= 7
    out.append(n)
    while width is not None and len(out) < width:
        out[-1] |= 0x80
        out.append(0)
    return bytes(out)


def literal(data: bytes, width: Optional[int] = None) -> bytes:
    """a literal element; width 0: the length in the tag (at most 60 bytes), 1..4: that many length bytes"""
    n = len(data) - 1
    if width is None:
        width = 0 if n < 60 else (n.bit_length() + 7) // 8
    if width == 0:
        assert n < 60
        return bytes([n << 2]) + data
    assert n < 1 << (8 * width)
    return bytes([(59 + width) << 2]) + n.to_bytes(width, "little") + data


def copy1(offset: int, length: int) -> bytes:
    assert 4 <= length <= 11 and offset < 2048
    return bytes([1 | (length - 4) << 2 | (offset >> 8) << 5, offset & 0xff])


def copy2(offset: int, length: int) -> bytes:
    assert 1 <= length <= 64 and offset < 65536
    return bytes([2 | (length - 1) << 2]) + offset.to_bytes(2, "little")


def copy4(offset: int, length: int) -> bytes:
    assert 1 <= length <= 64
    return bytes([3 | (length - 1) << 2]) + offset.to_bytes(4, "little")


class Writer:
    """A stream of n output bytes built element by element; `sp` is the stream position of the next element (preamble
    included), `op` its output position."""

    def __init__(self, n: int, pre_width: Optional[int] = None):
        self.n, self.pre = n, varint(n, pre_width)
        self.body, self.out = bytearray(), bytearray()

    @property
    def sp(self):
        return len(self.pre) + len(self.body)

    @property
    def op(self):
        return len(self.out)

    def lit(self, data: bytes, width: Optional[int] = None):
        self.body += literal(data, width)
        self.out += data
        return self

    def copy(self, offset: int, length: int, form: Optional[int] = None):
        if form is None:
            form = 1 if 4 <= length <= 11 and offset < 2048 else (2 if offset < 65536 else 4)
        self.body += {1: copy1, 2: copy2, 4: copy4}[form](offset, length)
        for _ in range(length):
            self.out.append(self.out[-offset])
        return self

    def reach(self, sp: int, op: int, rng):
        """elements that end at stream position sp and output position op: one literal, then copies of offset 1 (at least
        one byte is written before them) -- all inside the current output block"""
        dsp, dop = sp - self.sp, op - self.op
        for k in range(0, dsp // 3 + 1):
            ln = dsp - 3 * k
            ln -= 1 if ln <= 61 else (2 if ln <= 258 else 3)
            if ln < 1 or len(literal(bytes(ln))) + 3 * k != dsp or not k <= dop - ln <= 64 * k:
                continue
            self.lit(rng_bytes(rng, ln))
            rest = dop - ln
            for j in range(k):
                c = rest // (k - j)
                self.copy(1, c, form=2)
                rest -= c
            assert (self.sp, self.op) == (sp, op)
            return self
        raise ValueError(f"cannot reach ({sp}, {op}) from ({self.sp}, {self.op})")

    def dense(self, rng, until: int, max_off: int = 2000, until_sp: Optional[int] = None):
        """short literals and copies up to output position `until` (or stream position until_sp), none leaving its
        64 KB block"""
        while self.op < until and (until_sp is None or self.sp < until_sp):
            room = min(until - self.op, BLOCK - self.op % BLOCK)
            ib = self.op % BLOCK
            if ib == 0 or rng.random() < 0.4:
                self.lit(rng_bytes(rng, int(rng.integers(1, min(room, 12) + 1))))
            else:
                off = int(rng.integers(1, min(ib, max_off) + 1))
                self.copy(off, int(rng.integers(1, min(room, 64) + 1)))
        return self

    def stream(self) -> bytes:
        assert self.op == self.n, (self.op, self.n)
        return self.pre + bytes(self.body)


def rng_bytes(rng, k: int, lo: int = 0, hi: int = 256) -> bytes:
    return rng.integers(lo, hi, k, dtype=np.uint8).tobytes()


# ---- a restatement of the format --------------------------------------------------------------------------------------
def preamble(stream: bytes):
    """(uncompressed length, bytes) under the C++ library's rule -- at most 5 bytes, the fifth below 16 -- or None"""
    v = 0
    for i in range(min(PREAMBLE_BYTES, len(stream))):
        b = stream[i]
        if i == 4 and b >= 16:
            return None
        v |= (b & 0x7f) << (7 * i)
        if not b & 0x80:
            return v, i + 1
    return None


def elements(stream: bytes, start: int):
    """(pos, hdr, kind, length, offset) of every element from `start` while its header is whole"""
    p = start
    while p < len(stream):
        tag = stream[p]
        kind, up = tag & 3, tag >> 2
        if kind == 0:
            nb = up - 59 if up >= 60 else 0
            if p + 1 + nb > len(stream):
                return
            ln = (int.from_bytes(stream[p + 1:p + 1 + nb], "little") if nb else up) + 1
            yield p, 1 + nb, 0, ln, 0
            p += 1 + nb + ln
        else:
            tail = 4 if kind == 3 else kind
            if p + 1 + tail > len(stream):
                return
            t = int.from_bytes(stream[p + 1:p + 1 + tail], "little")
            if kind == 1:
                yield p, 2, 1, (up & 7) + 4, (tag >> 5) << 8 | t
            else:
                yield p, 1 + tail, kind, up + 1, t
            p += 1 + tail


def decode(stream: bytes, n: int):
    """(bytes, None) where the C++ library accepts the stream at n output bytes, else (None, reason)"""
    pre = preamble(stream)
    if pre is None:
        return None, "preamble"
    if pre[0] != n:
        return None, "preamble length"
    out, p = bytearray(), pre[1]
    for pos, hdr, kind, ln, off in elements(stream, p):
        if pos != p:
            break
        if kind == 0:
            if pos + hdr + ln > len(stream):
                return None, "truncated literal"
            if len(out) + ln > n:
                return None, "output overrun"
            out += stream[pos + hdr:pos + hdr + ln]
        else:
            if off == 0:
                return None, "offset 0"
            if off > len(out):
                return None, "before start"
            if len(out) + ln > n:
                return None, "output overrun"
            if off >= ln:
                out += out[len(out) - off:len(out) - off + ln]
            else:
                for _ in range(ln):
                    out.append(out[-off])
        p = pos + hdr + (ln if kind == 0 else 0)
    if p != len(stream):
        return None, "truncated element"
    if len(out) != n:
        return None, "output short"
    return bytes(out), None


def pyarrow_accepts(stream: bytes, n: int) -> bool:
    """The C++ library's verdict at exactly n bytes.  pyarrow's decompressed_size is room, not a size: it accepts a
    preamble below it.  So the preamble is parsed by the library's rule and must equal n first."""
    pre = preamble(stream)
    if pre is None or pre[0] != n:
        return False
    try:
        pa.Codec("snappy").decompress(stream, decompressed_size=n)
    except (OSError, ValueError):
        return False
    return True


def pyarrow_decode(stream: bytes, n: int) -> bytes:
    return pa.Codec("snappy").decompress(stream, decompressed_size=n, asbytes=True) if n else b""


def independent(stream: bytes) -> bool:
    """The decoder's choice for a valid stream: its 64 KB output blocks decode in parallel exactly when no element
    straddles a block boundary, no copy reaches before the start of its block and no copy offset exceeds 0xffff."""
    op = 0
    for _, _, kind, ln, off in elements(stream, preamble(stream)[1]):
        ib = op % BLOCK
        if ln > BLOCK - ib or (kind and (off > ib or off > MAX_OFFSET_PARALLEL)):
            return False
        op += ln
    return True


def facts(stream: bytes) -> Dict[str, object]:
    """What a valid stream puts on the decoder's limits, measured from its elements."""
    start = preamble(stream)[1]
    els = list(elements(stream, start))
    n_src, seg = len(stream), seg_of(len(stream))
    outs = np.cumsum([0] + [e[3] for e in els])
    f = dict(n_src=n_src, seg=seg, rounds=-(-n_src // (32 * seg)), n=int(outs[-1]), parallel=independent(stream),
             hdrs=sorted({e[1] for e in els}), segment_start_elements=0, boundary_at_segment_start=False,
             boundary_by_lane_last_element=False, boundary_mid_lane=False, straddle=False, copy_to_block_start=False,
             copy_before_block_start=False, copy_before_block_start_after_boundary_in_lane=False, coop_literals=0,
             long_tag_data=False, copy_tag_data=False, overlaps=set(), max_offset=0, max_literal=0)
    for i, (pos, hdr, kind, ln, off) in enumerate(els):
        op = int(outs[i])
        ib = op % BLOCK
        if pos and pos % seg == 0:
            f["segment_start_elements"] += 1
        if ln > BLOCK - ib:
            f["straddle"] = True
        if ib == 0 and op and i:
            prev = els[i - 1][0]
            if pos % seg == 0:
                f["boundary_at_segment_start"] = True
            elif prev // seg == pos // seg:
                f["boundary_mid_lane"] = True
            else:
                f["boundary_by_lane_last_element"] = True
        if kind == 0:
            f["max_literal"] = max(f["max_literal"], ln)
            f["coop_literals"] += ln >= COOP_LITERAL
            data = np.frombuffer(stream[pos + hdr:pos + hdr + ln], np.uint8)
            if ln >= 256 and np.mean((data >= 0xF0) & (data <= 0xFC)) > 0.9:
                f["long_tag_data"] = True
            if ln >= 256 and np.mean((data & 3) != 0) > 0.9:
                f["copy_tag_data"] = True
        else:
            f["max_offset"] = max(f["max_offset"], off)
            if off < ln and off < 10:
                f["overlaps"].add(off)
            if off == ib and ib:
                f["copy_to_block_start"] = True
            if off == ib + 1:
                f["copy_before_block_start"] = True
                # the block started inside this lane's segment, a few elements back
                j = i
                while j > 0 and int(outs[j]) % BLOCK != 0:
                    j -= 1
                if j > 0 and op >= BLOCK and els[j][0] // seg == pos // seg and els[j][0] % seg:
                    f["copy_before_block_start_after_boundary_in_lane"] = True
    return f


# ---- cases ----------------------------------------------------------------------------------------------------------
@dataclass
class Case:
    name: str
    stream: bytes
    n: int
    claims: Dict[str, object] = field(default_factory=dict)
    src_phase: int = 0          # source address mod 4 of the stream (after any prefix)
    dst_phase: int = 0          # destination address mod 16 of the decoded bytes (after any prefix)


def _exact_nsrc(n_src: int, seed: int):
    """dense elements, then a tail that ends the stream at exactly n_src bytes; returns the writer"""
    rng = np.random.default_rng(seed)
    w = Writer(1 << 20)  # a 3-byte preamble, as every n these streams reach
    w.dense(rng, 1 << 30, max_off=200, until_sp=n_src - 600)
    if BLOCK - w.op % BLOCK < 300:
        w.lit(rng_bytes(rng, BLOCK - w.op % BLOCK))
    w.n = w.op + 300
    w.pre = varint(w.n)
    assert len(w.pre) == 3
    return w.reach(n_src, w.n, rng)


def segment_cases():
    out = []
    for n_src in (8191, 8192, 8193, 16383, 16384, 16385, 32767, 32768, 32769, 49153, 65535, 98305):
        w = _exact_nsrc(n_src, n_src)
        out.append(Case(f"nsrc_{n_src}", w.stream(), w.n, dict(parallel=True, n_src=n_src, seg=seg_of(n_src), rounds=-(-n_src // (32 * seg_of(n_src))))))
    return out


def long_literal_cases():
    rng = np.random.default_rng(21)
    out = []
    for ln, at in ((40_000, 3000), (65_536, BLOCK)):
        w = Writer(at + ln + 20_000)
        w.dense(rng, at)
        w.lit(rng_bytes(rng, ln))
        w.dense(rng, w.n)
        out.append(Case(f"long_literal_{ln}_mid_stream", w.stream(), w.n, dict(max_literal=ln, parallel=True)))
    return out


def guess_cases():
    rng = np.random.default_rng(22)
    out = []
    for nm, lo, hi in (("long_tags", 0xF0, 0xFD), ("copy_tags", 1, 4)):
        w = Writer(60_000)
        w.dense(rng, 2000)
        for _ in range(6):
            data = rng_bytes(rng, int(rng.integers(700, 3000)), lo, hi)
            if nm == "copy_tags":
                data = bytes(b | int(rng.integers(0, 64)) << 2 for b in data)
            w.lit(data)
            w.dense(rng, w.op + 3000)
        w.dense(rng, w.n)
        out.append(Case(f"literal_data_reads_as_{nm}", w.stream(), w.n, dict(parallel=True, **{f"{nm[:-1]}_data": True})))
    # every element starts on a segment boundary: literals that take exactly one segment of stream
    w = Writer(40 * 254 + 200)
    w.reach(SEG, 200, rng)
    for _ in range(40):
        w.lit(rng_bytes(rng, 254))
    out.append(Case("elements_on_segment_starts", w.stream(), w.n, dict(seg=SEG, segment_start_elements=40)))
    return out


def block_cases():
    rng = np.random.default_rng(23)
    out = []
    for n in (65_535, 65_536, 65_537, 131_072, 131_073):
        w = Writer(n).dense(rng, n)
        out.append(Case(f"output_{n}", w.stream(), n, dict(n=n, parallel=True)))
    # a block boundary where a lane's segment starts, inside a lane, and made by the last element of a lane
    n_src, n = 40_000, 3 * BLOCK
    seg = seg_of(n_src)
    for nm in ("at_segment_start", "mid_lane", "by_lane_last_element"):
        w = Writer(n)
        w.dense(rng, BLOCK - 3000, max_off=100)
        lane = w.sp // seg + 2
        if nm == "by_lane_last_element":  # a literal from 40 bytes before a segment end ends the block 30 bytes after it
            w.reach(lane * seg - 40, BLOCK - 68, rng)
            w.lit(rng_bytes(rng, 68))
        else:
            w.reach(lane * seg + (100 if nm == "mid_lane" else 0), BLOCK, rng)
        w.dense(rng, 2 * BLOCK + 1000, max_off=100)
        w.reach(n_src, n, rng)
        out.append(Case(f"boundary_{nm}", w.stream(), n, dict(parallel=True, n_src=n_src, seg=seg, **{f"boundary_{nm}": True})))
    # an element ending on a block boundary, and one straddling it by one byte (literal and copy)
    for kind in ("literal", "copy"):
        for over in (0, 1):
            w = Writer(BLOCK + 1000)
            w.dense(rng, BLOCK - 40)
            if kind == "literal":
                w.lit(rng_bytes(rng, 40 + over))
            else:
                w.copy(500, 40 + over)
            w.dense(rng, w.n)
            out.append(Case(f"{kind}_{'straddles' if over else 'ends_on'}_boundary", w.stream(), w.n,
                            dict(straddle=bool(over), parallel=not over)))
    # copies reaching exactly to their block start, and one byte before it; in a lane without a block end and in a lane
    # whose segment holds one (the index pass's second walk)
    for where in ("own_lane", "after_boundary_in_lane"):
        for before in (0, 1):
            w = Writer(2 * BLOCK + 500)
            w.dense(rng, BLOCK - 200, max_off=100)
            if where == "own_lane":
                w.dense(rng, BLOCK + 10_000, max_off=100)
                w.copy(w.op % BLOCK + before, 20)
            else:
                lane_start = (w.sp // 256 + 2) * 256
                w.reach(lane_start + 40, BLOCK, rng)  # the block starts 40 bytes into a lane's segment
                w.lit(rng_bytes(rng, 5)).copy(5 + before, 8)
            w.dense(rng, w.n, max_off=100)
            claims = dict(copy_before_block_start=bool(before), parallel=not before)
            if where == "own_lane":
                claims["copy_to_block_start"] = not before
            elif before:
                claims["copy_before_block_start_after_boundary_in_lane"] = True
            out.append(Case(f"copy_{'one_before' if before else 'to'}_block_start_{where}", w.stream(), w.n, claims))
    # copy-4 offsets of 65 535 (the last byte of a block from its first) and 65 536
    for off in (65_535, 65_536):
        w = Writer(BLOCK + 100)
        w.lit(rng_bytes(rng, 1000)).dense(rng, off)  # the copy reads the stream's first byte
        w.copy(off, 1, form=4).dense(rng, w.n)
        out.append(Case(f"copy4_offset_{off}", w.stream(), w.n, dict(max_offset=off, parallel=off == 65_535)))
    return out


def warp_literal_cases():
    """long literals: lengths 63 / 64 / 65, and the warp copy's vector counts 32 / 33 and 64 / 65 with every tail; the
    destination and source phases come from where the tests place the streams"""
    rng = np.random.default_rng(24)
    out = []
    for ln in (63, 64, 65):
        w = Writer(ln + 10).lit(rng_bytes(rng, ln)).dense(rng, ln + 10)
        out.append(Case(f"literal_{ln}", w.stream(), w.n, dict(coop_literals=int(ln >= COOP_LITERAL))))
    for nvec in (32, 33, 64, 65):
        for tail in range(16):
            dphase = (3 * tail + nvec) % 16
            head = (16 - dphase) % 16
            ln = head + 16 * nvec + tail
            w = Writer(ln).lit(rng_bytes(rng, ln))
            out.append(Case(f"warp_literal_nvec{nvec}_tail{tail}", w.stream(), ln, dict(coop_literals=1),
                            src_phase=tail % 4, dst_phase=dphase))
    # long literals after a short one: the literal's destination phase is set by the bytes before it
    for k in range(16):
        w = Writer(k + 1 + 700).lit(rng_bytes(rng, k + 1)).lit(rng_bytes(rng, 700))
        out.append(Case(f"warp_literal_after_{k + 1}", w.stream(), w.n, dict(coop_literals=1), src_phase=k % 4))
    return out


def overlap_cases():
    rng = np.random.default_rng(25)
    out = []
    for off in range(1, 10):
        n = off + sum(range(off + 1, 65)) + 3 * (64 - off)
        w = Writer(n).lit(rng_bytes(rng, off))
        for ln in range(off + 1, 65):
            w.copy(off, ln, form=2).lit(rng_bytes(rng, 3))
        out.append(Case(f"overlapping_copies_offset{off}", w.stream(), n, dict(overlaps={off})))
    return out


def header_cases():
    """every header size at every tag phase: the tests place each at source phases 0..3"""
    rng = np.random.default_rng(26)
    w = Writer(0)
    for pad in range(4):
        w.lit(rng_bytes(rng, pad + 1))
        w.lit(rng_bytes(rng, 5), 0).lit(rng_bytes(rng, 5), 1).lit(rng_bytes(rng, 300), 2).lit(rng_bytes(rng, 70), 3)
        w.lit(rng_bytes(rng, 20), 4).copy(10, 6, 1).copy(30, 40, 2).copy(400, 9, 4)
    n = w.op
    s = varint(n) + bytes(w.body)
    return [Case(f"every_header_src_phase{ph}", s, n, dict(hdrs=[1, 2, 3, 4, 5]), src_phase=ph) for ph in range(4)]


def pyarrow_cases():
    codec = pa.Codec("snappy")
    out = []
    for i, data in enumerate(inputs()):
        s = codec.compress(data, asbytes=True)
        out.append(Case(f"pyarrow_{i}_{len(data)}", s, len(data), dict(parallel=True)))
    return out


def preamble_cases():
    rng = np.random.default_rng(27)
    out = []
    for width in (3, 4, 5):
        w = Writer(300, pre_width=width).dense(rng, 300)
        out.append(Case(f"preamble_{width}_bytes_non_minimal", w.stream(), 300))
    w = Writer(1 << 21).lit(rng_bytes(rng, 1000)).dense(rng, 1 << 21)  # a minimal 4-byte preamble, 32 blocks
    out.append(Case("output_2MB", w.stream(), w.n, dict(parallel=True)))
    return out


def to_one_lane(c: Case) -> Case:
    """the same elements, then a copy that straddles a block boundary: the page is decoded front to back by one lane"""
    pre = preamble(c.stream)
    pad = BLOCK - c.n % BLOCK - 1 or BLOCK
    n = c.n + pad + 2
    rng = np.random.default_rng(len(c.stream))
    body = c.stream[pre[1]:] + literal(rng_bytes(rng, pad)) + copy2(1, 2)
    return Case(c.name + "/one_lane", varint(n) + body, n, dict(parallel=False), c.src_phase, c.dst_phase)


@functools.lru_cache(maxsize=1)
def _valid():
    cases = (segment_cases() + long_literal_cases() + guess_cases() + block_cases() + warp_literal_cases() + overlap_cases()
             + header_cases() + pyarrow_cases() + preamble_cases())
    cases += [to_one_lane(c) for c in cases if c.n < 300_000 and not c.name.startswith("pyarrow")]
    return cases


def valid():
    return list(_valid())


def inputs():
    rng = np.random.default_rng(11)
    yield b""
    yield b"a"
    yield b"abc"
    yield b"abcd" * 3
    yield bytes(100_000)                                        # one long run
    yield rng.integers(0, 256, size=200_000, dtype=np.uint8).tobytes()   # incompressible
    yield (b"the quick brown fox jumps over the lazy dog. " * 5000)[:200_001]
    yield np.arange(50_000, dtype=np.int64).tobytes()           # sorted keys: shared high bytes
    yield (np.arange(300_000, dtype=np.float64) * 1e-3).tobytes()
    for n in (65_535, 65_536, 65_537, 131_072 + 5):
        yield rng.integers(0, 4, size=n, dtype=np.uint8).tobytes()       # low entropy, fragment boundaries


# ---- page compressors for hand-built Parquet files (tests/parquet_shapes.py: Chunk.snappy) -------------------------------
def _lz(w: Writer, data: bytes, start: int):
    """data[start:] into w greedily: copies of 4..64 bytes found through a table of 4-byte sequences, literals between
    them; nothing leaves its 64 KB output block"""
    n, i, lit, table = len(data), start, start, {}

    def flush(to):
        for a in range(lit, to, 4096):
            w.lit(data[a:min(to, a + 4096)])
    while i < n:
        key = data[i:i + 4]
        j = table.get(key)
        table[key] = i
        if len(key) == 4 and j is not None and j // BLOCK == i // BLOCK:
            m, lim = 4, min(64, n - i, BLOCK - i % BLOCK)
            while m < lim and data[j + m] == data[i + m]:
                m += 1
            flush(i)
            w.copy(i - j, m)
            i = lit = i + m
        else:
            i += 1
            if i % BLOCK == 0:
                flush(i)
                lit = i
    flush(n)
    return w.stream()


def compress_copies(data: bytes) -> bytes:
    """literals and copies, blocks independent: the parallel path"""
    return _lz(Writer(len(data)), data, 0)


def compress_one_lane(data: bytes) -> bytes:
    """a first literal that straddles the first 64 KB boundary, then literals and copies: the one-lane path for pages
    above 64 KB"""
    if len(data) <= BLOCK:
        return compress_copies(data)
    w = Writer(len(data)).lit(data[:BLOCK + 100])
    return _lz(w, data, BLOCK + 100)


def compress_long_literals(data: bytes) -> bytes:
    """literals of up to 1 000 bytes, none crossing a 64 KB boundary: warp-copied literals on the parallel path"""
    w = Writer(len(data))
    for b in range(0, len(data), BLOCK):
        for a in range(b, min(len(data), b + BLOCK), 1000):
            w.lit(data[a:min(len(data), b + BLOCK, a + 1000)])
    return w.stream()


def compress_zero_offset_copy(data: bytes) -> bytes:
    """damaged: the last four bytes follow a copy element of offset 0, which a decoder that took it for a literal would
    read as those bytes"""
    assert len(data) > 4
    return varint(len(data)) + literal(data[:-4]) + bytes([0x0e, 0, 0]) + data[-4:]


def source_file(codec: int, damaged: bool = False) -> bytes:
    """A Parquet image (tests/parquet_shapes.py) whose SNAPPY pages come from the compressors above: the key column's
    pages of 12 000 rows take the one-lane path, `a` holds long literals, `o` is nullable in v2 pages whose levels are
    stored in front of compressed values, and `d` is dictionary-encoded with a compressed dictionary page.  codec 0 gives
    the same rows UNCOMPRESSED; damaged=True puts a zero-offset copy in the last page of `a`."""
    import parquet_shapes as P

    rng = np.random.default_rng(50)
    n = 30_000
    k = rng.permutation(n).astype(np.int64) * 7919 - 10**9
    a = rng.standard_normal(n) * 1e6
    o = rng.integers(0, 1000, n).astype(np.int64)
    valid = rng.random(n) < 0.8
    dvals = rng.permutation(np.arange(500, dtype=np.int64) * 104_729)
    ix = rng.integers(0, 500, n)
    ix[:500] = np.arange(500)

    def chunk(pages, snappy, **kw):
        return P.Chunk(pages, codec=codec, snappy=snappy, **kw)

    def pages(sizes, make):
        out, at = [], 0
        for sz in sizes:
            out.append(make(at, sz))
            at += sz
        return out

    a_pages = pages([10_000, 20_000], lambda at, sz: P.Page(rows=sz, values=a[at:at + sz]))
    a_comp = compress_long_literals
    if damaged:
        def a_comp(body):
            return compress_zero_offset_copy(body) if len(body) > 100_000 else compress_long_literals(body)
    cols = [
        P.Col("k", P.INT64, False, [chunk(pages([12_000, 12_000, 6000], lambda at, sz: P.Page(rows=sz, values=k[at:at + sz])),
                                          compress_one_lane)]),
        P.Col("a", P.DOUBLE, False, [chunk(a_pages, a_comp)]),
        P.Col("o", P.INT64, True, [chunk(pages([15_000, 15_000], lambda at, sz: P.Page(
            rows=sz, values=o[at:at + sz][valid[at:at + sz]], defs=P.runs_of(valid[at:at + sz].astype(np.int64)), v2=True)),
            compress_copies)]),
        P.Col("d", P.INT64, False, [chunk(pages([20_000, 10_000], lambda at, sz: P.Page(
            rows=sz, enc=P.RLE_DICTIONARY, idx=[P.packed(ix[at:at + sz])])), compress_copies, dict=dvals)]),
    ]
    return P.write_file(P.FileSpec(cols))


# ---- damaged streams ------------------------------------------------------------------------------------------------
def damaged():
    """(name, stream, n, check): check is k_snappy_blocks' error number where the path makes it certain"""
    rng = np.random.default_rng(30)
    big = Writer(BLOCK + 5000).dense(rng, BLOCK + 5000)
    big_body = big.stream()[len(big.pre):]
    seq_tail = literal(rng_bytes(rng, BLOCK - 1)) + copy2(1, 2)  # a straddling copy: the one-lane path
    out = []
    # copies of offset 0 in all three forms, with len bytes after them (the parent decoded these as literals)
    for nm, el in (("copy1", bytes([0x01, 0x00])), ("copy2", bytes([0x0e, 0, 0])), ("copy4", bytes([0x0f, 0, 0, 0, 0]))):
        out.append((f"offset0_{nm}", varint(8) + literal(b"abcd") + el + b"wxyz", 8, CHECK_LENGTH))
        out.append((f"offset0_{nm}_first", varint(4) + el + b"wxyz", 4, CHECK_LENGTH))
        out.append((f"offset0_{nm}_in_a_big_stream", varint(BLOCK + 5004) + big_body + el + b"wxyz", BLOCK + 5004, CHECK_LENGTH))
        n = BLOCK + 5000 + BLOCK + 1 + 4
        out.append((f"offset0_{nm}_one_lane", varint(n) + big_body + seq_tail + el + b"wxyz", n, CHECK_LENGTH))
    # elements left after the output is full
    out.append(("trailing_literal", varint(4) + literal(b"abcd") + literal(b"q"), 4, CHECK_TRAILING))
    out.append(("trailing_copy", varint(4) + literal(b"abcd") + copy1(4, 4), 4, CHECK_TRAILING))
    out.append(("trailing_cut_header", varint(4) + literal(b"abcd") + b"\xf0", 4, CHECK_TRAILING))
    out.append(("trailing_in_a_big_stream", big.stream() + literal(b"q"), big.n, CHECK_TRAILING))
    out.append(("trailing_zero_length_page", b"\x00" + literal(b"q"), 0, CHECK_TRAILING))
    # over-long preambles
    out.append(("preamble_fifth_byte_16", bytes.fromhex("8480808010") + literal(b"abcd"), 4, CHECK_PREAMBLE))
    out.append(("preamble_fifth_byte_7f", bytes.fromhex("848080807f") + literal(b"abcd"), 4, CHECK_PREAMBLE))
    out.append(("preamble_fifth_byte_continues", bytes.fromhex("8480808080") + literal(b"abcd"), 4, CHECK_PREAMBLE))
    out.append(("preamble_six_bytes", bytes.fromhex("848080808000") + literal(b"abcd"), 4, CHECK_PREAMBLE))
    out.append(("preamble_only_continuation", bytes.fromhex("8480"), 4, CHECK_PREAMBLE))
    out.append(("empty_stream", b"", 0, CHECK_PREAMBLE))
    # the earlier cases: truncation, preamble mismatch, before-start, overrun, short output
    comp = pa.Codec("snappy").compress((b"0123456789abcdef" * 20_000)[:300_000], asbytes=True)
    out.append(("truncated_half", comp[:len(comp) // 2], 300_000, None))
    out.append(("truncated_in_literal", varint(50) + literal(bytes(50))[:30], 50, CHECK_TRUNCATED))
    out.append(("truncated_in_copy_header", varint(50) + literal(bytes(10)) + copy4(5, 40)[:3], 50, None))
    out.append(("preamble_above_page", varint(300_001) + comp[len(varint(300_000)):], 300_000, CHECK_PREAMBLE))
    out.append(("preamble_below_page", varint(299_999) + comp[len(varint(300_000)):], 300_000, CHECK_PREAMBLE))
    out.append(("copy_before_start", varint(100) + copy2(50, 60) + literal(b"x" * 40), 100, CHECK_BEFORE_START))
    out.append(("copy_one_before_start", varint(20) + literal(b"x" * 10) + copy2(11, 10), 20, CHECK_BEFORE_START))
    out.append(("literal_longer_than_output", varint(10) + literal(b"y" * 30), 10, CHECK_LENGTH))
    out.append(("copy_longer_than_output", varint(20) + literal(b"y" * 10) + copy2(5, 11), 20, CHECK_LENGTH))
    out.append(("stream_ends_early", varint(50) + literal(b"z" * 10), 50, CHECK_SHORT))
    out.append(("literal_length_field_overflow", varint(10) + b"\xfc\xff\xff\xff\xff" + bytes(10), 10, CHECK_LENGTH))
    return out


# ---- mutations ------------------------------------------------------------------------------------------------------
def mutations(count: int = 2000):
    """(name, stream, n): seeded edits of valid streams -- byte flips, tag kind changes, zeroed copy offsets, changed
    preambles, truncations and appended bytes.  One in eight edits a stream of several 64 KB blocks, which the index pass
    walks in several rounds and cuts into blocks for the parallel path."""
    rng = np.random.default_rng(31)
    bases = [(c.name, c.stream, c.n) for c in _valid() if 0 < c.n < 40_000 and len(c.stream) < 6000]
    w = Writer(3000).dense(rng, 3000)
    bases.append(("dense3000", w.stream(), 3000))
    multi = [(c.name, c.stream, c.n) for c in _valid() if c.name in (
        "output_131073", "nsrc_49153", "boundary_mid_lane", "long_literal_65536_mid_stream",
        "copy_to_block_start_after_boundary_in_lane", "pyarrow_6_200001", "output_65537/one_lane")]
    assert len(multi) == 7
    out = []
    kinds = ("flip", "tag_kind", "zero_offset", "preamble", "cut", "append")
    for i in range(count):
        nm, s, n = multi[(i // 8) % len(multi)] if i % 8 == 7 else bases[i % len(bases)]
        s = bytearray(s)
        start = preamble(bytes(s))[1]
        els = list(elements(bytes(s), start))
        kind = kinds[int(rng.integers(0, len(kinds)))]
        pos = 0
        if kind == "flip":
            pos = int(rng.integers(0, len(s)))
            s[pos] ^= 1 << int(rng.integers(0, 8))
        elif kind == "tag_kind":
            pos = els[int(rng.integers(0, len(els)))][0]
            s[pos] = (s[pos] & ~3) | int(rng.integers(0, 4))
        elif kind == "zero_offset":
            copies = [e for e in els if e[2]] or els
            pos, hdr = copies[int(rng.integers(0, len(copies)))][:2]
            if s[pos] & 3 == 1:
                s[pos] &= 0x1f
            s[pos + 1:pos + hdr] = bytes(hdr - 1)
        elif kind == "preamble":
            n2 = int(rng.choice([n - 1, n + 1, n + 16, max(0, n - 64), n << 7]))
            s[:start] = varint(n2, int(rng.choice([start, 5])) if rng.random() < 0.5 else None)
        elif kind == "cut":
            pos = int(rng.integers(0, len(s)))
            del s[pos:]
        else:
            pos = len(s)
            s += rng_bytes(rng, int(rng.integers(1, 4)))
        out.append((f"{nm}/{kind}@{pos}#{i}", bytes(s), n))
    return out
