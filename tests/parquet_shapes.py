"""Hand-built Parquet files in the page shapes where the GPU page decoder (hyperspace_b200/csrc/parquet_decode.cu) changes
path, and a Python restatement of how it chooses that path.

The writer below is pure Python: a Thrift compact-protocol encoder for the page headers and the footer, and explicit page
bodies.  Every page is given as it is to be written -- its row count, encoding, v1 or v2, its definition levels and
dictionary indices as explicit RLE / bit-packed run lists -- and the writer derives the column values the file holds from
that description (values of PLAIN pages, dictionary entries picked by the index runs, validity from the level runs).  So
a case states the stream shape; the expected columns follow from it.

Where the values of a page start is controlled on purpose, and every case that needs it states the alignment: the
writer pads the page header with a binary in DataPageHeader.statistics (parquet-mr writes statistics there too) until
the values -- or the data of the first index run of a dictionary page -- start at the stated offset modulo 4 or 8.
File images sit 16-byte aligned in device memory, so a file offset modulo 8 is the device address modulo 8.  Column
chunks may also be separated by gaps that the footer's offsets skip.

Every limit the decoder turns on is restated once below, with the source line it mirrors.  tests/test_parquet_shapes_host.py
checks them against the source, reads every file with pyarrow, parses every file back and checks each case's claims --
page row counts, first rows modulo 8, value alignment, run lengths, dictionary sizes, bit widths and the path every page
takes -- without a GPU.  tests/test_gpu_parquet_shapes.py decodes every case on the GPU.

A case is a function returning ([FileSpec], {}); case_data() writes its images and derives the expected columns:
expected[name] = (values, valid or None) over all files in order, values holding 0 at null rows.  CLAIMS[name] lists
what the case is built to put on a boundary; the host test checks them against measure() of the images.  Shapes that
pyarrow refuses (empty runs, a run claiming more groups than its stream holds) are left out.
"""
import functools
import struct
from dataclasses import dataclass
from typing import Callable, List, Optional

import numpy as np

# ---- the limits ------------------------------------------------------------------------------------------------------
SMEM_DICT = 2048        # kSmemDict (parquet_decode.cu:165): dictionary entries cached in shared memory
SMEM_DICT_CARRIED = 4 * SMEM_DICT  # (parquet_decode.cu:475): 16-bit codes of a carried column, four per 8-byte slot
RUN_TABLE = 128         # kRunTable (parquet_decode.cu:162): runs per refill of the hybrid decoder
MAX_PER_ENTRY = 256     # kMaxPerEntry (parquet_decode.cu:163): values per run-table entry
TILE_ROWS = 2048        # kTileRows (parquet_decode.cu:164): rows per tile on the nullable / hybrid paths
ALL_VALID_RUNS = 64     # def_levels_all_valid (parquet_decode.cu:297): runs examined by the all-valid check
GROUP_MAX_BW = 16       # the one-group-per-thread path takes idx_bw 1..16 (parquet_decode.cu:593)
GROUP_TAIL = 2          # ... and leaves the last two groups to the per-value loop (parquet_decode.cu:599)
ZC_TILE = 4096          # kFusedTileLocal (kernels.h): a page read in place spans at least one partition tile
AGREE_CAP = 8192        # kAgreeCap (engine.cu:613): largest union of chunk dictionaries a carried column may have
MAX_CARRIED = 4         # kMaxCarried (engine.h:42): carried columns per build
MAX_SPEC = 6            # kMaxSpec (engine.cu:614): candidate columns examined for carrying
MAX_DICT_ENTRIES = 65536  # kMaxDictEntries (kernels.h:308), in dictionary_pays_off (engine.cu:158)

# ---- Parquet enums ---------------------------------------------------------------------------------------------------
BOOLEAN, INT32, INT64, FLOAT, DOUBLE, BYTE_ARRAY = 0, 1, 2, 4, 5, 6
PLAIN, PLAIN_DICTIONARY, RLE, BIT_PACKED, DELTA_BINARY_PACKED, RLE_DICTIONARY = 0, 2, 3, 4, 5, 8
DATA_PAGE, INDEX_PAGE, DICTIONARY_PAGE, DATA_PAGE_V2 = 0, 1, 2, 3
UNCOMPRESSED, SNAPPY = 0, 1
DTYPE = {INT32: np.int32, INT64: np.int64, FLOAT: np.float32, DOUBLE: np.float64, BOOLEAN: np.uint8}
WIDTH = {INT32: 4, INT64: 8, FLOAT: 4, DOUBLE: 8, BOOLEAN: 1, BYTE_ARRAY: 8}
FIXED = (INT32, INT64, FLOAT, DOUBLE)


# ---- Thrift compact protocol -----------------------------------------------------------------------------------------
T_TRUE, T_FALSE, T_BYTE, T_I16, T_I32, T_I64, T_DOUBLE, T_BINARY, T_LIST, T_SET, T_MAP, T_STRUCT = range(1, 13)


def _zz(v: int) -> int:
    return (v << 1) if v >= 0 else ((-v) << 1) - 1


def _unzz(v: int) -> int:
    return (v >> 1) ^ -(v & 1)


def varint(v: int) -> bytes:
    out = bytearray()
    while v >= 0x80:
        out.append((v & 0x7F) | 0x80)
        v >>= 7
    out.append(v)
    return bytes(out)


class ThriftWriter:
    def __init__(self):
        self.b = bytearray()
        self.last = [0]

    def _field(self, fid, t):
        d = fid - self.last[-1]
        if 0 < d <= 15:
            self.b.append((d << 4) | t)
        else:
            self.b.append(t)
            self.b += varint(_zz(fid))
        self.last[-1] = fid

    def i32(self, fid, v):
        self._field(fid, T_I32)
        self.b += varint(_zz(v))
        return self

    def i64(self, fid, v):
        self._field(fid, T_I64)
        self.b += varint(_zz(v))
        return self

    def binary(self, fid, data: bytes):
        self._field(fid, T_BINARY)
        self.b += varint(len(data)) + data
        return self

    def boolean(self, fid, v: bool):
        self._field(fid, T_TRUE if v else T_FALSE)
        return self

    def begin(self, fid):
        self._field(fid, T_STRUCT)
        self.last.append(0)
        return self

    def end(self):
        self.b.append(0)
        self.last.pop()
        return self

    def list(self, fid, etype, n):
        self._field(fid, T_LIST)
        self.b += bytes([(n << 4) | etype]) if n < 15 else bytes([0xF0 | etype]) + varint(n)
        return self

    def elem_begin(self):  # a struct element of a list
        self.last.append(0)
        return self

    def raw(self, data: bytes):  # list elements of scalar type
        self.b += data
        return self


def _read_varint(b, p):
    v = shift = 0
    while True:
        x = b[p]
        p += 1
        v |= (x & 0x7F) << shift
        if not x & 0x80:
            return v, p
        shift += 7


def _read_value(b, p, t):
    if t in (T_TRUE, T_FALSE):
        return t == T_TRUE, p
    if t == T_BYTE:
        return b[p], p + 1
    if t in (T_I16, T_I32, T_I64):
        v, p = _read_varint(b, p)
        return _unzz(v), p
    if t == T_DOUBLE:
        return struct.unpack_from("<d", b, p)[0], p + 8
    if t == T_BINARY:
        n, p = _read_varint(b, p)
        return bytes(b[p:p + n]), p + n
    if t in (T_LIST, T_SET):
        h = b[p]
        p += 1
        n, et = h >> 4, h & 0x0F
        if n == 15:
            n, p = _read_varint(b, p)
        out = []
        for _ in range(n):
            v, p = _read_value(b, p, et)
            out.append(v)
        return out, p
    if t == T_STRUCT:
        return read_struct(b, p)
    raise ValueError(f"thrift type {t} not handled")


def read_struct(b, p=0):
    """One compact-protocol struct at b[p:] -> ({field id: value}, position after it)."""
    out, last = {}, 0
    while True:
        x = b[p]
        p += 1
        if x == 0:
            return out, p
        t, d = x & 0x0F, x >> 4
        if d:
            fid = last + d
        else:
            v, p = _read_varint(b, p)
            fid = _unzz(v)
        last = fid
        out[fid], p = _read_value(b, p, t)


# ---- RLE / bit-packed hybrid runs --------------------------------------------------------------------------------------
def rle(count, value):
    return ("rle", int(count), int(value))


def packed(values, groups=None):
    """A bit-packed run of `values` (zero-padded to whole groups of 8); `groups` may claim more groups than that, whose
    bytes are written too (zeros)."""
    values = np.asarray(values, dtype=np.int64)
    g = (len(values) + 7) // 8 if groups is None else groups
    return ("packed", values, g)



def bitpack(values, bw) -> bytes:
    if bw == 0 or len(values) == 0:
        return b""
    v = np.asarray(values, dtype=np.uint64)
    bits = ((v[:, None] >> np.arange(bw, dtype=np.uint64)) & np.uint64(1)).astype(np.uint8).ravel()
    return np.packbits(bits, bitorder="little").tobytes()


def encode_runs(runs, bw) -> bytes:
    out = bytearray()
    for r in runs:
        if r[0] == "rle":
            out += varint(r[1] << 1) + int(r[2]).to_bytes((bw + 7) // 8, "little")
        else:
            vals, g = r[1], r[2]
            out += varint((g << 1) | 1)
            padded = np.zeros(g * 8, dtype=np.int64)
            padded[:min(len(vals), g * 8)] = vals[:g * 8]
            out += bitpack(padded, bw)
    return bytes(out)


def run_values(runs, n) -> np.ndarray:
    """The first n values a run list stands for."""
    parts, have = [], 0
    for r in runs:
        if have >= n:
            break
        if r[0] == "rle":
            parts.append(np.full(r[1], r[2], dtype=np.int64))
            have += r[1]
        else:
            g = r[2]
            v = np.zeros(g * 8, dtype=np.int64)
            v[:min(len(r[1]), g * 8)] = r[1][:g * 8]
            parts.append(v)
            have += len(v)
    out = np.concatenate(parts) if parts else np.empty(0, dtype=np.int64)
    assert len(out) >= n, f"runs hold {len(out)} values, {n} needed"
    return out[:n]


def runs_of(values, max_rle=None):
    """Runs for a 0/1 or index stream: RLE for stretches of 8+ equal values, bit-packed groups between them."""
    values = np.asarray(values, dtype=np.int64)
    runs, i, n = [], 0, len(values)
    lit = []
    while i < n:
        j = i
        while j < n and values[j] == values[i]:
            j += 1
        if j - i >= 8 and len(lit) % 8 == 0:
            if lit:
                runs.append(packed(lit))
                lit = []
            runs.append(rle(j - i, values[i]))
            i = j
        else:
            lit.append(int(values[i]))
            i += 1
    if lit:
        runs.append(packed(lit))
    return runs


def bits_for_max(m: int) -> int:
    """parquet-mr's bit width of dictionary indices: that of the largest index (0 for a one-entry dictionary)."""
    return int(m).bit_length()


# ---- the page and file model -------------------------------------------------------------------------------------------
@dataclass
class Page:
    rows: int = 0
    enc: int = PLAIN
    v2: bool = False
    values: Optional[object] = None  # PLAIN: the dense (non-null) values
    idx: Optional[list] = None       # dictionary pages: index runs
    bw: Optional[int] = None         # index bit width (default: that of the largest dictionary index)
    defs: Optional[list] = None      # optional columns: level runs (default: one RLE run of ones)
    align: Optional[tuple] = None    # (modulus, remainder) of where the values / the first index run's data start
    stats: bool = False              # write DataPageHeader.statistics even when no padding is needed
    compressed: bool = True          # v2 page of a SNAPPY chunk: values compressed?
    kind: str = "data"               # "index": an INDEX_PAGE of `rows` body bytes


@dataclass
class Chunk:
    pages: List[Page]
    dict: Optional[object] = None    # dictionary values (array, or list of bytes)
    dict_enc: int = PLAIN            # encoding written in the dictionary page header (parquet-mr v1: PLAIN_DICTIONARY)
    codec: int = UNCOMPRESSED
    gap: int = 0                     # bytes left unused before the chunk
    snappy: Optional[Callable[[bytes], bytes]] = None  # SNAPPY chunks: the page compressor (default: pyarrow's)


@dataclass
class Col:
    name: str
    ptype: int
    optional: bool
    chunks: List[Chunk]              # one per row group


@dataclass
class FileSpec:
    cols: List[Col]
    nested: bool = False             # wrap the last column in a group (refused by the engine)


def _plain_bytes(ptype, values) -> bytes:
    if ptype == BYTE_ARRAY:
        return b"".join(struct.pack("<I", len(v)) + v for v in values)
    if ptype == BOOLEAN:
        return np.packbits(np.asarray(values, dtype=np.uint8), bitorder="little").tobytes()
    return np.ascontiguousarray(values, dtype=DTYPE[ptype]).tobytes()


def _delta_bytes(values) -> bytes:
    """DELTA_BINARY_PACKED of consecutive integers: one block, minimum delta 1, every miniblock of bit width 0."""
    v = [int(x) for x in values]
    assert all(b - a == 1 for a, b in zip(v, v[1:]))
    out = varint(128) + varint(4) + varint(len(v)) + varint(_zz(v[0] if v else 0))
    for _ in range((len(v) - 1 + 127) // 128):  # a block per 128 deltas
        out += varint(_zz(1)) + bytes(4)
    return out


def _snappy(data: bytes) -> bytes:
    import pyarrow as pa

    return pa.compress(data, codec="snappy", asbytes=True)


def _page_header(ptype, usize, csize, pg: Page, nulls, pad, dict_count=None, dict_enc=None) -> bytes:
    w = ThriftWriter()
    if dict_count is not None:
        w.i32(1, DICTIONARY_PAGE).i32(2, usize).i32(3, csize)
        w.begin(7).i32(1, dict_count).i32(2, dict_enc).end()
        return bytes(w.end().b)
    if pg.kind == "index":
        w.i32(1, INDEX_PAGE).i32(2, usize).i32(3, csize)
        w.begin(6).end()
        return bytes(w.end().b)
    w.i32(1, DATA_PAGE_V2 if pg.v2 else DATA_PAGE).i32(2, usize).i32(3, csize)

    def stats():
        if pad is not None:
            w.begin(8 if pg.v2 else 5)
            w.binary(1, bytes(pad)).i64(3, nulls)  # (max, null_count): the max is the padding
            w.end()
    if pg.v2:
        w.begin(8).i32(1, pg.rows).i32(2, nulls).i32(3, pg.rows).i32(4, pg.enc)
        w.i32(5, pg._def_len).i32(6, 0).boolean(7, pg.compressed)
        stats()
        w.end()
    else:
        w.begin(5).i32(1, pg.rows).i32(2, pg.enc).i32(3, RLE).i32(4, BIT_PACKED)
        stats()
        w.end()
    return bytes(w.end().b)


def _data_page(col: Col, ch: Chunk, pg: Page, pos: int, dict_len: int):
    """Bytes of one data page written at file offset `pos`, and (valid, dense values or indices) of its rows."""
    if pg.kind == "index":
        body = bytes(pg.rows)
        return _page_header(col.ptype, len(body), len(body), pg, 0, None) + body, None
    n = pg.rows
    if col.optional:
        defs = pg.defs if pg.defs is not None else [rle(n, 1)]
        valid = run_values(defs, n).astype(bool)
        level_bytes = encode_runs(defs, 1)
    else:
        valid, level_bytes = np.ones(n, dtype=bool), b""
    nvalid = int(valid.sum())
    if pg.enc in (PLAIN_DICTIONARY, RLE_DICTIONARY):
        bw = pg.bw if pg.bw is not None else bits_for_max(max(dict_len - 1, 0))
        runs = pg.idx if pg.idx is not None else [packed(np.zeros(nvalid, dtype=np.int64))]
        dense = run_values(runs, nvalid)
        run_bytes = encode_runs(runs, bw)
        first_hdr = len(varint(runs[0][1] << 1 if runs[0][0] == "rle" else runs[0][2] * 2 + 1)) if runs else 0
        values_part, lead = bytes([bw]) + run_bytes, 1 + first_hdr
    elif pg.enc == DELTA_BINARY_PACKED:
        dense = np.asarray(pg.values)
        values_part, lead = _delta_bytes(dense), 0
    else:
        dense = pg.values
        assert len(dense) == nvalid, (col.name, len(dense), nvalid)
        values_part, lead = _plain_bytes(col.ptype, dense), 0
    if pg.v2:
        pg._def_len = len(level_bytes)
        levels = level_bytes
    else:
        levels = (struct.pack("<I", len(level_bytes)) + level_bytes) if col.optional else b""
    compress_values = ch.codec == SNAPPY and (pg.compressed or not pg.v2)
    snappy = ch.snappy or _snappy
    if ch.codec == SNAPPY and not pg.v2:
        body_u = levels + values_part
        body = snappy(body_u)
    else:
        body_u = levels + values_part
        body = levels + (snappy(values_part) if compress_values else values_part)
    nulls = n - nvalid
    # the statistics' padding binary moves the values one byte per byte of padding
    pads = list(range(64)) if pg.stats else ([None] + list(range(64)) if pg.align else [None])
    for pad in pads:
        hdr = _page_header(col.ptype, len(body_u), len(body), pg, nulls, pad)
        start = pos + len(hdr) + len(levels) + lead
        if compress_values:  # values are decoded from a 16-byte aligned scratch copy of the page body
            start = len(levels) + lead
        if pg.align is None or start % pg.align[0] == pg.align[1]:
            return hdr + body, (valid, dense)
    raise AssertionError("no padding reaches the requested alignment")


def write_file(spec: FileSpec) -> bytes:
    """The file image, and per column the (valid, values) of its rows."""
    out = bytearray(b"PAR1")
    nrg = len(spec.cols[0].chunks)
    rg_meta = [[] for _ in range(nrg)]
    rg_rows = [sum(p.rows for p in spec.cols[0].chunks[g].pages if p.kind == "data") for g in range(nrg)]
    for g in range(nrg):
        for col in spec.cols:
            ch = col.chunks[g]
            out += bytes(ch.gap)
            start = len(out)
            dict_off, dict_len = None, 0
            if ch.dict is not None:
                dict_len = len(ch.dict)
                dbody_u = _plain_bytes(col.ptype, ch.dict)
                dbody = (ch.snappy or _snappy)(dbody_u) if ch.codec == SNAPPY else dbody_u
                dict_off = len(out)
                out += _page_header(col.ptype, len(dbody_u), len(dbody), None, 0, None, dict_count=dict_len,
                                    dict_enc=ch.dict_enc) + dbody
            data_off = len(out)
            encs = set()
            for pg in ch.pages:
                page, _ = _data_page(col, ch, pg, len(out), dict_len)
                out += page
                encs.add(pg.enc)
            total = len(out) - start
            rg_meta[g].append(dict(col=col, codec=ch.codec, num_values=rg_rows[g], total=total, data_off=data_off,
                                   dict_off=dict_off, encs=sorted(encs | {RLE})))
    w = ThriftWriter()
    w.i32(1, 1)
    nleaf = len(spec.cols)
    if spec.nested:
        w.list(2, T_STRUCT, nleaf + 2)
        w.elem_begin().binary(4, b"schema").i32(5, nleaf).end()
        for c in spec.cols[:-1]:
            w.elem_begin().i32(1, c.ptype).i32(3, 1 if c.optional else 0).binary(4, c.name.encode()).end()
        w.elem_begin().i32(3, 0).binary(4, b"grp").i32(5, 1).end()
        c = spec.cols[-1]
        w.elem_begin().i32(1, c.ptype).i32(3, 1 if c.optional else 0).binary(4, c.name.encode()).end()
    else:
        w.list(2, T_STRUCT, nleaf + 1)
        w.elem_begin().binary(4, b"schema").i32(5, nleaf).end()
        for c in spec.cols:
            w.elem_begin().i32(1, c.ptype).i32(3, 1 if c.optional else 0).binary(4, c.name.encode()).end()
    w.i64(3, sum(rg_rows))
    w.list(4, T_STRUCT, nrg)
    for g in range(nrg):
        w.elem_begin()
        w.list(1, T_STRUCT, len(rg_meta[g]))
        for m in rg_meta[g]:
            w.elem_begin()
            w.i64(2, m["dict_off"] if m["dict_off"] is not None else m["data_off"])
            w.begin(3).i32(1, m["col"].ptype)
            w.list(2, T_I32, len(m["encs"])).raw(b"".join(varint(_zz(e)) for e in m["encs"]))
            path = [b"grp", m["col"].name.encode()] if (spec.nested and m["col"] is spec.cols[-1]) else [m["col"].name.encode()]
            w.list(3, T_BINARY, len(path)).raw(b"".join(varint(len(s)) + s for s in path))
            w.i32(4, m["codec"]).i64(5, m["num_values"]).i64(6, m["total"]).i64(7, m["total"]).i64(9, m["data_off"])
            if m["dict_off"] is not None:
                w.i64(11, m["dict_off"])
            w.end()
            w.end()
        w.i64(2, sum(m["total"] for m in rg_meta[g])).i64(3, rg_rows[g])
        w.end()
    w.binary(6, b"parquet_shapes (hand-built test file)")
    footer = bytes(w.end().b)
    out += footer + struct.pack("<I", len(footer)) + b"PAR1"
    return bytes(out)


def expected_columns(specs: List[FileSpec]):
    """{name: (values, valid or None)} over the files in order; values hold 0 at null rows (b"" for strings)."""
    res = {}
    for col_i, col in enumerate(specs[0].cols):
        vals, valids = [], []
        for spec in specs:
            c = spec.cols[col_i]
            for ch in c.chunks:
                for pg in ch.pages:
                    if pg.kind != "data":
                        continue
                    n = pg.rows
                    valid = run_values(pg.defs, n).astype(bool) if (c.optional and pg.defs is not None) else np.ones(n, bool)
                    nvalid = int(valid.sum())
                    if pg.enc in (PLAIN_DICTIONARY, RLE_DICTIONARY):
                        runs = pg.idx if pg.idx is not None else [packed(np.zeros(nvalid, dtype=np.int64))]
                        ix = run_values(runs, nvalid)
                        dense = [ch.dict[i] for i in ix] if c.ptype == BYTE_ARRAY else np.asarray(ch.dict)[ix]
                    else:
                        dense = pg.values
                    if c.ptype == BYTE_ARRAY:
                        v = np.empty(n, dtype=object)
                        v[:] = b""
                        for at, x in zip(np.flatnonzero(valid), dense):
                            v[at] = x
                    else:
                        v = np.zeros(n, dtype=DTYPE[c.ptype])
                        v[valid] = np.asarray(dense, dtype=DTYPE[c.ptype])
                    vals.append(v)
                    valids.append(valid)
        values = np.concatenate(vals) if vals else np.empty(0)
        res[col.name] = (values, np.concatenate(valids) if col.optional else None)
    return res


# ---- parsing the images back, and the decoder's path choice restated ------------------------------------------------
def parse_runs(b, p, end, bw, n):
    """The hybrid runs at b[p:end] that cover n values: [(kind, values, header bytes, claimed groups)]."""
    runs, have = [], 0
    while have < n and p < end:
        h, q = _read_varint(b, p)
        hl = q - p
        if h & 1:
            g = h >> 1
            avail = (end - q) // bw if bw else g
            runs.append(("packed", min(g, avail) * 8, hl, g))
            have += min(g, avail) * 8
            p = q + min(g, avail) * bw
            if g > avail:
                break
        else:
            runs.append(("rle", h >> 1, hl, 0))
            have += h >> 1
            p = q + (bw + 7) // 8
    return runs


def all_valid(def_runs, n) -> bool:
    """def_levels_all_valid (parquet_decode.cu:293-314): the first ALL_VALID_RUNS runs are RLE runs of ones that cover
    the page."""
    covered = 0
    for r in def_runs[:ALL_VALID_RUNS]:
        if covered >= n:
            break
        if r[0] != "rle" or r[3] != 1 or r[1] == 0:
            return False
        covered += r[1]
    return covered >= n


def measure(images):
    """Every data page of the images, parsed back from the bytes -- [dict(col, n, first_row, ...)] with first_row
    counted over the files in order, as the decoder numbers rows -- and the other pages: {"dict": [(col, entries,
    encoding)], "index": count, "file_rows": [rows per file]}."""
    pages, other = [], {"dict": [], "index": 0, "file_rows": []}
    row_base = 0
    for fi, img in enumerate(images):
        flen = struct.unpack_from("<I", img, len(img) - 8)[0]
        fm, _ = read_struct(img, len(img) - 8 - flen)
        schema = fm[2]
        leaves = [e for e in schema[1:] if 5 not in e or e[5] == 0]
        for rg in fm[4]:
            for ci, cc in enumerate(rg[1]):
                md = cc[3]
                leaf = leaves[ci]
                ptype, optional = leaf[1], leaf.get(3, 0) == 1
                name = leaf[4].decode()
                start = md.get(11, md[9]) if md.get(11, md[9]) < md[9] else md[9]
                p, end = start, start + md[7]
                codec = md[4]
                dict_count, seen, first = None, 0, row_base
                while p < end and seen < md[5]:
                    h, q = read_struct(img, p)
                    csize, usize = h[3], h[2]
                    body = q
                    if h[1] == DICTIONARY_PAGE:
                        dict_count = h[7][1]
                        other["dict"].append((leaf[4].decode(), dict_count, h[7][2]))
                    elif h[1] == INDEX_PAGE:
                        other["index"] += 1
                    elif h[1] in (DATA_PAGE, DATA_PAGE_V2):
                        v2 = h[1] == DATA_PAGE_V2
                        dh = h[8] if v2 else h[5]
                        n, enc = dh[1], dh[4] if v2 else dh[2]
                        compressed = codec == SNAPPY and (not v2 or dh.get(7, True))
                        if codec == SNAPPY and not v2:
                            from pyarrow import decompress
                            page = bytes(decompress(bytes(img[body:body + csize]), usize, codec="snappy", asbytes=True))
                            dev_base, pb, pe = 0, 0, usize  # a decompressed page sits 16-byte aligned in scratch
                        elif compressed:
                            from pyarrow import decompress
                            lv = dh[5]
                            page = bytes(img[body:body + lv]) + bytes(decompress(bytes(img[body + lv:body + csize]), usize - lv,
                                                                                  codec="snappy", asbytes=True))
                            dev_base, pb, pe = 0, 0, usize
                        else:
                            page, dev_base, pb, pe = img, body, body, body + csize
                        q2 = pb
                        def_runs = None
                        if v2:
                            if optional:
                                def_runs = _level_runs(page, pb, pb + dh[5], n)
                            q2 = pb + dh[5] + dh.get(6, 0)
                        elif optional:
                            ln = struct.unpack_from("<I", page, pb)[0]
                            def_runs = _level_runs(page, pb + 4, pb + 4 + ln, n)
                            q2 = pb + 4 + ln
                        rec = dict(file=fi, col=name, ptype=ptype, optional=optional, n=n, first_row=first, enc=enc,
                                   v2=v2, compressed=compressed, codec=codec, dict_count=dict_count, def_runs=def_runs,
                                   stats=(5 in dh) if not v2 else (8 in dh))
                        rec["levels"] = "none" if not optional else ("all_valid" if all_valid(def_runs, n) else "general")
                        if enc in (PLAIN_DICTIONARY, RLE_DICTIONARY):
                            bw = page[q2] if n else 0
                            rec["bw"] = bw
                            rec["idx_runs"] = parse_runs(page, q2 + 1, pe, bw, n if rec["levels"] != "general" else
                                                         _count_valid(page, def_runs, n))
                            hl = rec["idx_runs"][0][2] if rec["idx_runs"] else 0
                            rec["run_data_mod"] = (dev_base - pb + q2 + 1 + hl) % 8 if not compressed else (q2 + 1 + hl) % 16
                            first_run = rec["idx_runs"][0] if rec["idx_runs"] else None
                            rec["single_run"] = bool(first_run and first_run[0] == "packed" and first_run[3] * 8 >= n
                                                     and q2 + 1 + first_run[2] + first_run[3] * bw <= pe)
                        else:
                            rec["value_mod"] = ((q2 - pb) + (dev_base if not compressed else 0)) % 8
                            rec["value_bytes"] = pe - q2
                        pages.append(rec)
                        seen += n
                        first += n
                    p = body + csize
            row_base += rg[3]
        other["file_rows"].append(fm[3])
    return pages, other


def _level_runs(b, p, end, n):
    out, have = [], 0
    while have < n and p < end:
        h, q = _read_varint(b, p)
        if h & 1:
            g = h >> 1
            g_avail = min(g, end - q)
            vals = np.unpackbits(np.frombuffer(bytes(b[q:q + g_avail]), dtype=np.uint8), bitorder="little")
            out.append(("packed", g_avail * 8, q - p, vals, g))
            have += g_avail * 8
            p = q + g_avail
        else:
            out.append(("rle", h >> 1, q - p, b[q] & 1 if q < end else 0))
            have += h >> 1
            p = q + 1
    return out


def _level_values(def_runs, n):
    parts = [r[3][:r[1]] if r[0] == "packed" else np.full(r[1], r[3], dtype=np.uint8) for r in def_runs]
    return np.concatenate(parts)[:n] if parts else np.zeros(0, np.uint8)


def _count_valid(b, def_runs, n):
    return int(_level_values(def_runs, n).sum())


def page_paths(pages, carried=(), unions=None):
    """Per data page, the path k_decode_pages takes (parquet_decode.cu:438-714): 'dict' smem / global, 'idx' group /
    single / hybrid, 'levels' none / all_valid / general, 'in_place' (k_classify_pages, :354-365)."""
    out = []
    for pg in pages:
        W = WIDTH[pg["ptype"]]
        is_dict = pg["enc"] in (PLAIN_DICTIONARY, RLE_DICTIONARY)
        carry = pg["col"] in carried
        path = dict(levels=pg["levels"], dict=None, idx=None, in_place=False)
        if is_dict:
            cap = SMEM_DICT_CARRIED if carry else SMEM_DICT
            path["dict"] = "smem" if pg["dict_count"] <= cap else "global"
            if pg["levels"] != "general":
                if pg["single_run"]:
                    group = 1 <= pg["bw"] <= GROUP_MAX_BW and path["dict"] == "smem" and W != 1 and pg["n"] // 8 - GROUP_TAIL > 0
                    path["idx"] = "group" if group else "single"
                else:
                    path["idx"] = "hybrid"
            else:
                path["idx"] = "hybrid"
        else:
            path["in_place"] = (pg["ptype"] in FIXED and pg["enc"] == PLAIN and not pg["compressed"] and
                                pg["levels"] != "general" and pg["n"] >= ZC_TILE and pg["value_mod"] % W == 0 and
                                pg["value_bytes"] >= pg["n"] * W)
        out.append(path)
    return out


def zero_copy_columns(pages, key, included):
    """Columns createIndex reads in place (engine.cu:745-765): every page in place; the key only when it is the one
    indexed column and an integer."""
    paths = page_paths(pages)
    cols = {}
    for pg, path in zip(pages, paths):
        cols.setdefault(pg["col"], []).append(path["in_place"] and pg["levels"] != "general")
    out = set()
    for c, ok in cols.items():
        if not all(ok):
            continue
        ptype = next(p["ptype"] for p in pages if p["col"] == c)
        if c in included and ptype in FIXED or (c == key and ptype in (INT32, INT64)):
            out.add(c)
    return out


def dictionary_pays_off(ndict, width, total_rows, nseg):
    """engine.cu:158-162, with bits_for (engine.cu:164-168)."""
    bw = 1
    while (1 << bw) < ndict:
        bw += 1
    return 0 < ndict <= MAX_DICT_ENTRIES and total_rows * bw / 8.0 + ndict * width * max(1, nseg) <= 0.9 * total_rows * width


def carried(pages, unions, included, nb):
    """engine.cu:616-738 on one GPU: candidates are the first MAX_SPEC included columns; a candidate whose every page
    is dictionary-encoded and all-valid, whose dictionary union holds at most AGREE_CAP values and pays off is carried,
    up to MAX_CARRIED of them.  unions[c]: the union of the column's chunk dictionaries (as raw bits)."""
    total = max(p["first_row"] + p["n"] for p in pages) if pages else 0
    out = []
    for c in included[:MAX_SPEC]:
        if len(out) >= MAX_CARRIED:
            break
        pcs = [p for p in pages if p["col"] == c]
        if not pcs or pcs[0]["ptype"] not in FIXED:
            continue
        if any(p["enc"] not in (PLAIN_DICTIONARY, RLE_DICTIONARY) or p["levels"] == "general" for p in pcs):
            continue
        u = unions[c]
        if len(u) > AGREE_CAP or not dictionary_pays_off(len(u), WIDTH[pcs[0]["ptype"]], total, nb):
            continue
        out.append(c)
    return out


# ---- case helpers ------------------------------------------------------------------------------------------------------
CASES = {}
CLAIMS = {}
REFUSALS = {}


def case(**claims):
    def reg(fn):
        CASES[fn.__name__] = fn
        CLAIMS[fn.__name__] = claims
        return fn
    return reg


@functools.lru_cache(maxsize=None)
def case_data(name):
    """(images, expected, specs) of a case."""
    specs, extra = CASES[name]()
    images = [write_file(s) for s in specs]
    return images, expected_columns(specs), specs


@functools.lru_cache(maxsize=None)
def analyse(name):
    images, expected, specs = case_data(name)
    pages, other = measure(images)
    cl = CLAIMS[name]
    nb = cl.get("nb", 4)
    included = index_columns(name)
    unions = {}
    for i, col in enumerate(specs[0].cols):
        u = set()
        for s in specs:
            for ch in s.cols[i].chunks:
                if ch.dict is not None and col.ptype in FIXED:
                    u |= set(np.asarray(ch.dict, dtype=DTYPE[col.ptype]).view({4: np.uint32, 8: np.uint64}[WIDTH[col.ptype]]).tolist())
        unions[col.name] = u
    car = carried(pages, unions, included, nb)
    return dict(pages=pages, other=other, paths=page_paths(pages, car), carried=car,
                zero_copy=zero_copy_columns(pages, "k", included), unions=unions)


def index_columns(name):
    """Included columns of the case's createIndex: every int32 / int64 / float / double column but the key."""
    _, _, specs = case_data(name)
    return [c.name for c in specs[0].cols if c.name != "k" and c.ptype in FIXED]


def _rng(seed):
    return np.random.default_rng(seed)


def _key(n, seed, pages=None, align=(8, 4), start=0, step=1):
    """The indexed column k: distinct int64 values in random order (or ascending with step), PLAIN; its values start at
    4 mod 8 so that it is never read in place unless a case asks for it."""
    rng = _rng(seed)
    k = (start + step * np.arange(n, dtype=np.int64)) if step else rng.permutation(n).astype(np.int64) * 7919 - 10**9
    sizes = pages or [n]
    pgs, at = [], 0
    for s in sizes:
        pgs.append(Page(rows=s, values=k[at:at + s], align=align))
        at += s
    return Col("k", INT64, False, [Chunk(pgs)])


def _plain(name, ptype, values, sizes, optional=False, valid=None, **kw):
    values = np.asarray(values)
    pgs, at = [], 0
    for s in sizes:
        if optional:
            v = valid[at:at + s]
            pgs.append(Page(rows=s, values=values[at:at + s][v], defs=runs_of(v.astype(np.int64)), **kw))
        else:
            pgs.append(Page(rows=s, values=values[at:at + s], **kw))
        at += s
    return Col(name, ptype, optional, [Chunk(pgs)])


def _random_values(ptype, rng, m):
    if ptype == INT32:
        return rng.integers(-2**31, 2**31 - 1, size=m, dtype=np.int32, endpoint=True)
    if ptype == INT64:
        return rng.integers(-2**63, 2**63 - 1, size=m, dtype=np.int64, endpoint=True)
    if ptype == FLOAT:
        return rng.standard_normal(m).astype(np.float32) * np.float32(1e3)
    if ptype == DOUBLE:
        return rng.standard_normal(m) * 1e6
    if ptype == BOOLEAN:
        return rng.integers(0, 2, size=m).astype(np.uint8)
    return [bytes(rng.integers(97, 123, size=int(rng.integers(0, 12))).astype(np.uint8)) for _ in range(m)]


def _dictionary(ptype, rng, m):
    """m distinct values of the type."""
    if ptype == BYTE_ARRAY:
        return [b"s%06d" % i + bytes(rng.integers(97, 123, size=int(rng.integers(0, 6))).astype(np.uint8)) for i in range(m)]
    out = np.unique(_random_values(ptype, rng, m * 2 + 16))
    out = out[~np.isnan(out)] if out.dtype.kind == "f" else out
    return rng.permutation(out)[:m]


def _dict_col(name, ptype, dict_vals, page_runs, rows, bw=None, enc=RLE_DICTIONARY):
    pgs = [Page(rows=r, enc=enc, idx=runs, bw=bw) for r, runs in zip(rows, page_runs)]
    return Col(name, ptype, False, [Chunk(pgs, dict=dict_vals)])


def _one(cols, **extra):
    return [FileSpec(cols)], extra


# ---- dictionary size: shared memory or global ------------------------------------------------------------------------
def _dict_size_case(ptype, m, n, seed):
    rng = _rng(seed)
    d = _dictionary(ptype, rng, m)
    ix = rng.integers(0, m, size=n)
    ix[:m] = np.arange(m)[: min(m, n)]  # every entry used, the last one included
    return _one([_key(n, seed), _dict_col("d", ptype, d, [[packed(ix)]], [n])])


@case(dict_sizes=[SMEM_DICT], paths=[{"col": "d", "dict": "smem", "idx": "group"}], nb=4)
def dict_2048_entries_in_shared_memory():
    return _dict_size_case(INT64, SMEM_DICT, 9000, 1)


@case(dict_sizes=[SMEM_DICT + 1], paths=[{"col": "d", "dict": "global", "idx": "single"}], nb=4)
def dict_2049_entries_in_global_memory():
    return _dict_size_case(DOUBLE, SMEM_DICT + 1, 9000, 2)


@case(dict_sizes=[SMEM_DICT_CARRIED], carried=["d"], paths=[{"col": "d", "dict": "smem", "idx": "group", "carried": True}], nb=1)
def dict_8192_entries_carried_in_shared_memory():
    return _dict_size_case(INT64, SMEM_DICT_CARRIED, 40_000, 3)


@case(dict_sizes=[SMEM_DICT_CARRIED + 1], carried=[], paths=[{"col": "d", "dict": "global", "idx": "single"}], nb=1)
def dict_8193_entries_not_carried():
    return _dict_size_case(INT64, SMEM_DICT_CARRIED + 1, 40_000, 4)


# ---- one bit-packed run: the fast paths -----------------------------------------------------------------------------
@case(bws=set(range(1, 21)), paths=[{"col": "b%02d" % bw, "idx": "group"} for bw in range(1, 17)] +
      [{"col": "b%02d" % bw, "idx": "single"} for bw in range(17, 21)])
def index_bit_widths_1_to_20():
    """One column per index bit width, each a single bit-packed run; widths above what the dictionary needs are legal."""
    rng = _rng(10)
    n = 3001
    cols = [_key(n, 10)]
    types = [INT32, INT64, FLOAT, DOUBLE]
    for bw in range(1, 21):
        m = min(1 << bw, 64)
        pt = types[bw % 4]
        d = _dictionary(pt, rng, m)
        ix = rng.integers(0, m, size=n)
        cols.append(_dict_col("b%02d" % bw, pt, d, [[packed(ix)]], [n], bw=bw))
    return _one(cols)


@case(page_rows={"s": [1, 7, 8, 15, 16, 17, 23, 24, 25, 31, 1000]}, first_row_mod8={0, 1, 7},
      paths=[{"col": "s", "idx": "single"}, {"col": "s", "idx": "group"}])
def index_single_run_pages_under_24_rows():
    """Pages of fewer than 24 rows give the group path nothing (n/8 - 2 <= 0); their first rows are no multiple of 8."""
    rng = _rng(11)
    sizes = [1, 7, 8, 15, 16, 17, 23, 24, 25, 31, 1000]
    n = sum(sizes)
    d = _dictionary(INT32, rng, 37)
    runs = [[packed(rng.integers(0, 37, size=s))] for s in sizes]
    d2 = _dictionary(DOUBLE, rng, 300)
    runs2 = [[packed(rng.integers(0, 300, size=s))] for s in sizes]
    return _one([_key(n, 11), _dict_col("s", INT32, d, runs, sizes), _dict_col("t", DOUBLE, d2, runs2, sizes)])


@case(first_row_mod8=set(range(8)), paths=[{"col": "c", "idx": "group", "carried": True}])
def index_pages_at_every_first_row_mod_8():
    """Pages of 1003 rows: their first rows fall on all eight residues modulo 8 (the 16-byte code store needs 0)."""
    rng = _rng(12)
    sizes = [1003] * 8
    n = sum(sizes)
    d = _dictionary(INT32, rng, 200)
    d2 = _dictionary(INT64, rng, 1000)
    return _one([_key(n, 12), _dict_col("c", INT32, d, [[packed(rng.integers(0, 200, size=s))] for s in sizes], sizes),
                 _dict_col("e", INT64, d2, [[packed(rng.integers(0, 1000, size=s))] for s in sizes], sizes)])


@case(run_data_mod4={0, 1, 2, 3}, paths=[{"col": "a", "idx": "group"}])
def index_run_data_at_each_alignment_mod_4():
    """The bit-packed run's first byte at 0, 1, 2 and 3 mod 4: the group path assembles each group from aligned words."""
    rng = _rng(13)
    sizes = [997, 1024, 1500, 777]
    n = sum(sizes)
    d = _dictionary(FLOAT, rng, 1500)
    pgs = [Page(rows=s, enc=RLE_DICTIONARY, idx=[packed(rng.integers(0, 1500, size=s))], bw=11, align=(4, r))
           for r, s in enumerate(sizes)]
    d2 = _dictionary(INT64, rng, 20)
    pgs2 = [Page(rows=s, enc=RLE_DICTIONARY, idx=[packed(rng.integers(0, 20, size=s))], bw=5, align=(4, (r + 1) % 4))
            for r, s in enumerate(sizes)]
    return _one([_key(n, 13), Col("a", FLOAT, False, [Chunk(pgs, dict=d)]), Col("b", INT64, False, [Chunk(pgs2, dict=d2)])])


@case(claimed_groups_over_rows=True, paths=[{"col": "a", "idx": "group"}, {"col": "a", "idx": "single"}])
def index_run_claims_more_groups_than_rows():
    """One bit-packed run per page that claims more groups than the page has rows, their bytes present: 150 groups for
    1000 rows, 4 groups for 17 rows.  (A run whose claimed groups reach past the page is refused by pyarrow.)"""
    rng = _rng(14)
    d = _dictionary(INT64, rng, 500)
    ix1, ix2 = rng.integers(0, 500, size=1000), rng.integers(0, 500, size=17)
    pgs = [Page(rows=1000, enc=RLE_DICTIONARY, idx=[packed(ix1, groups=150)], bw=9),
           Page(rows=17, enc=RLE_DICTIONARY, idx=[packed(ix2, groups=4)], bw=9)]
    return _one([_key(1017, 14), Col("a", INT64, False, [Chunk(pgs, dict=d)])])


# ---- the hybrid decoder ----------------------------------------------------------------------------------------------
def _hybrid_case(seed, run_lists, m=300, ptype=INT64, bw=None, optional_col=False):
    rng = _rng(seed)
    d = _dictionary(ptype, rng, m)
    pgs = []
    for runs in run_lists:
        n = sum(r[1] if r[0] == "rle" else r[2] * 8 for r in runs)
        pgs.append(Page(rows=n, enc=RLE_DICTIONARY, idx=runs, bw=bw))
    total = sum(p.rows for p in pgs)
    return _one([_key(total, seed), Col("h", ptype, False, [Chunk(pgs, dict=d)])])


def _lit(rng, m, count):
    return packed(rng.integers(0, m, size=count))


@case(max_idx_runs_min=3 * RUN_TABLE, paths=[{"col": "h", "idx": "hybrid"}])
def hybrid_more_than_128_runs_per_refill():
    """400 runs (RLE of 3, one bit-packed group, alternating) inside one 2048-row tile, then 400 more across the next."""
    rng = _rng(20)
    runs = []
    for i in range(400):
        runs.append(rle(3, int(rng.integers(0, 300))) if i % 2 == 0 else _lit(rng, 300, 8))
    return _hybrid_case(20, [runs, list(reversed(runs))])


@case(idx_run_lengths={("rle", 255), ("rle", 256), ("rle", 257), ("packed", 248), ("packed", 256), ("packed", 264),
                       ("packed", 520)}, paths=[{"col": "h", "idx": "hybrid"}])
def hybrid_runs_of_255_256_257():
    """Runs either side of kMaxPerEntry: RLE 255 / 256 / 257, bit-packed 248 / 256 / 264 / 520 values (split into
    entries of 256, the later ones resuming inside the run)."""
    rng = _rng(21)
    runs = [rle(255, 1), _lit(rng, 300, 248), rle(256, 2), _lit(rng, 300, 256), rle(257, 3), _lit(rng, 300, 264),
            rle(1, 4), _lit(rng, 300, 520), rle(9, 299)]
    return _hybrid_case(21, [runs])


@case(packed_run_across_tile=True, paths=[{"col": "h", "idx": "hybrid"}])
def hybrid_packed_run_across_tile_edge():
    """A bit-packed run of 1000 values from row 2000: the tile at row 2048 resumes it at value 48; a second page runs
    one of 4200 values across two tile edges."""
    rng = _rng(22)
    return _hybrid_case(22, [[rle(2000, 7), _lit(rng, 300, 1000), rle(100, 8)],
                             [rle(8, 1), _lit(rng, 300, 4200), rle(5, 2)]])


@case(bws={8, 9, 16, 17, 24, 25}, rle_value_bytes={1, 2, 3, 4}, paths=[{"col": "w16", "idx": "hybrid"}])
def hybrid_rle_values_1_to_4_bytes_wide():
    """RLE run values of bit widths 8 / 9 / 16 / 17 / 24 / 25: 1, 2, 2, 3, 3 and 4 bytes after each run header."""
    rng = _rng(23)
    n = 6000
    cols = [_key(n, 23)]
    for bw, m, ptype in ((8, 256, INT32), (9, 512, INT64), (16, 65536, INT32), (17, 70000, FLOAT), (24, 1000, DOUBLE),
                         (25, 1000, INT64)):
        d = _dictionary(ptype, rng, m)
        hi = m - 1
        runs = [rle(1000, hi), _lit(rng, m, 1000), rle(1500, hi - 1), rle(500, m // 2), _lit(rng, m, 2000)]
        cols.append(Col("w%02d" % bw, ptype, False, [Chunk([Page(rows=n, enc=RLE_DICTIONARY, idx=runs, bw=bw)], dict=d)]))
    return _one(cols)


@case(multibyte_headers={2, 3}, paths=[{"col": "h", "idx": "hybrid"}])
def hybrid_multibyte_run_headers():
    """Run headers of 2 and 3 bytes: RLE 300 / 20 000, bit-packed 100 groups.  (Empty runs, which the decoder skips, are
    refused by pyarrow and left out.)"""
    rng = _rng(24)
    runs = [rle(300, 5), _lit(rng, 300, 800), rle(20000, 6), _lit(rng, 300, 16)]
    return _hybrid_case(24, [runs])


# ---- definition levels -----------------------------------------------------------------------------------------------
def _levels_case(seed, level_runs_per_page, ptype=INT64, enc=PLAIN, m=40):
    rng = _rng(seed)
    pgs = []
    d = _dictionary(ptype, rng, m) if enc != PLAIN else None
    for lr in level_runs_per_page:
        n = sum(r[1] if r[0] == "rle" else len(r[1]) for r in lr)
        nvalid = int(run_values(lr, n).sum())
        if enc == PLAIN:
            pgs.append(Page(rows=n, values=_random_values(ptype, rng, nvalid), defs=lr))
        else:
            pgs.append(Page(rows=n, enc=enc, idx=[packed(rng.integers(0, m, size=nvalid))], defs=lr))
    total = sum(p.rows for p in pgs)
    return _one([_key(total, seed), Col("o", ptype, True, [Chunk(pgs, dict=d)])])


@case(def_runs_per_page=[ALL_VALID_RUNS], paths=[{"col": "o", "levels": "all_valid"}], carried=["o"])
def levels_all_valid_as_64_rle_runs():
    return _levels_case(30, [[rle(1, 1)] * 63 + [rle(5000, 1)]], enc=RLE_DICTIONARY)


@case(def_runs_per_page=[ALL_VALID_RUNS + 1], paths=[{"col": "o", "levels": "general"}], carried=[])
def levels_all_valid_as_65_rle_runs():
    return _levels_case(31, [[rle(1, 1)] * 64 + [rle(5000, 1)]], enc=RLE_DICTIONARY)


@case(def_runs_per_page=[ALL_VALID_RUNS + 2], paths=[{"col": "o", "levels": "general"}])
def levels_64_runs_of_ones_then_nulls():
    """The all-valid check stops after 64 runs of ones that do not yet cover the page: the nulls after them count."""
    return _levels_case(32, [[rle(1, 1)] * 64 + [rle(100, 0), rle(3000, 1)]])


@case(paths=[{"col": "o", "levels": "general"}], packed_all_ones=True)
def levels_all_ones_bit_packed():
    return _levels_case(33, [[packed(np.ones(4096, np.int64))], [rle(10, 1), packed(np.ones(808, np.int64))]], ptype=DOUBLE)


def _nulls_at(n, rows):
    v = np.ones(n, np.int64)
    v[list(rows)] = 0
    return v


@case(null_rows={0, 2047, 2048, 2049, 4095, 4096, 4999}, paths=[{"col": "o", "levels": "general"}])
def levels_nulls_at_tile_edges():
    lv = _nulls_at(5000, [0, 2047, 2048, 2049, 4095, 4096, 4999])
    lv2 = _nulls_at(4200, [2046, 2047, 4199])
    return _levels_case(34, [[packed(lv)], runs_of(lv2)], ptype=INT32)


@case(null_rows={2047, 2048, 2049}, paths=[{"col": "o", "levels": "general", "dict": "smem"}])
def levels_nulls_at_tile_edges_dictionary():
    lv = _nulls_at(5000, [2047, 2048, 2049])
    return _levels_case(35, [[packed(lv)], [rle(2048, 1), rle(1, 0), rle(951, 1)]], ptype=FLOAT, enc=RLE_DICTIONARY, m=700)


# ---- PLAIN bodies at every alignment ---------------------------------------------------------------------------------
@case(value_mod4={0, 1, 2, 3}, paths=[{"col": "i", "levels": "none"}])
def plain_4_byte_values_at_offsets_0_to_3():
    rng = _rng(40)
    sizes = [1111, 1500, 999, 2048]
    n = sum(sizes)
    cols = [_key(n, 40)]
    for name, pt in (("i", INT32), ("f", FLOAT)):
        v = _random_values(pt, rng, n)
        pgs, at = [], 0
        for r, s in enumerate(sizes):
            pgs.append(Page(rows=s, values=v[at:at + s], align=(4, (r + (pt == FLOAT)) % 4)))
            at += s
        cols.append(Col(name, pt, False, [Chunk(pgs)]))
    return _one(cols)


@case(value_mod8=set(range(8)), paths=[{"col": "l", "levels": "none"}])
def plain_8_byte_values_at_offsets_0_to_7():
    rng = _rng(41)
    sizes = [700, 1001, 513, 64, 2047, 3, 999, 1500]
    n = sum(sizes)
    cols = [_key(n, 41)]
    for name, pt in (("l", INT64), ("d", DOUBLE)):
        v = _random_values(pt, rng, n)
        pgs, at = [], 0
        for r, s in enumerate(sizes):
            pgs.append(Page(rows=s, values=v[at:at + s], align=(8, (r * 3 + (pt == DOUBLE)) % 8)))
            at += s
        cols.append(Col(name, pt, False, [Chunk(pgs)]))
    return _one(cols)


# ---- BOOLEAN ---------------------------------------------------------------------------------------------------------
@case(page_rows={"bo": [1, 7, 9, 13, 1001, 4095]})
def boolean_plain_odd_page_sizes():
    rng = _rng(50)
    sizes = [1, 7, 9, 13, 1001, 4095]
    n = sum(sizes)
    valid = rng.random(n) > 0.3
    valid[:3] = [False, True, False]
    return _one([_key(n, 50), _plain("b", BOOLEAN, _random_values(BOOLEAN, rng, n), sizes),
                 _plain("bo", BOOLEAN, _random_values(BOOLEAN, rng, n), sizes, optional=True, valid=valid)])


# ---- strings ---------------------------------------------------------------------------------------------------------
@case(paths=[{"col": "s", "levels": "general"}])
def strings_bit_packed_and_rle_levels():
    rng = _rng(60)
    sizes = [1000, 333, 2100]
    n = sum(sizes)
    valid = rng.random(n) > 0.25
    valid[1000:1100] = True  # an RLE run of ones
    valid[1500:1600] = False  # and one of nulls
    vals = np.empty(n, dtype=object)
    vals[:] = _random_values(BYTE_ARRAY, rng, n)
    pgs, at = [], 0
    for s in sizes:
        v = valid[at:at + s]
        pgs.append(Page(rows=s, values=list(vals[at:at + s][v]), defs=runs_of(v.astype(np.int64))))
        at += s
    return _one([_key(n, 60), Col("s", BYTE_ARRAY, True, [Chunk(pgs)])])


@case(null_rows=set(range(16)))
def strings_null_at_every_position():
    """16 pages of 16 rows, page i null at row i only; then pages all null and all valid; a dictionary-encoded chunk."""
    rng = _rng(62)
    pgs = []
    for i in range(16):
        lv = _nulls_at(16, [i])
        pgs.append(Page(rows=16, values=_random_values(BYTE_ARRAY, rng, 15), defs=[packed(lv)]))
    pgs.append(Page(rows=9, values=[], defs=[rle(9, 0)]))
    pgs.append(Page(rows=9, values=_random_values(BYTE_ARRAY, rng, 9), defs=[rle(9, 1)]))
    n = sum(p.rows for p in pgs)
    d = _dictionary(BYTE_ARRAY, rng, 30)
    lv = _nulls_at(n, [0, 5, n - 1])
    dpg = Page(rows=n, enc=RLE_DICTIONARY, idx=[packed(rng.integers(0, 30, size=int(lv.sum())))], defs=runs_of(lv))
    return _one([_key(n, 62), Col("s", BYTE_ARRAY, True, [Chunk(pgs)]), Col("sd", BYTE_ARRAY, True, [Chunk([dpg], dict=d)])])


# ---- the page walk ---------------------------------------------------------------------------------------------------
@case(index_pages=2)
def index_page_between_data_pages():
    rng = _rng(70)
    v = _random_values(INT32, rng, 3000)
    pgs = [Page(rows=5, kind="index"), Page(rows=1000, values=v[:1000]), Page(rows=37, kind="index"),
           Page(rows=2000, values=v[1000:])]
    return _one([_key(3000, 70), Col("i", INT32, False, [Chunk(pgs)])])


@case(v2_uncompressed_in_snappy=True, paths=[{"col": "o", "levels": "general"}, {"col": "d", "dict": "smem"}])
def v2_pages_stored_uncompressed_in_snappy_chunks():
    rng = _rng(71)
    sizes = [1500, 2500, 777]
    n = sum(sizes)
    valid = rng.random(n) > 0.2
    v = _random_values(INT64, rng, n)
    pgs, at = [], 0
    for i, s in enumerate(sizes):
        m = valid[at:at + s]
        pgs.append(Page(rows=s, values=v[at:at + s][m], defs=runs_of(m.astype(np.int64)), v2=True, compressed=i == 1))
        at += s
    d = _dictionary(DOUBLE, rng, 400)
    dp = [Page(rows=s, enc=RLE_DICTIONARY, idx=[packed(rng.integers(0, 400, size=s))], v2=True, compressed=i != 1)
          for i, s in enumerate(sizes)]
    w = _random_values(FLOAT, rng, n)
    wp = [Page(rows=s, values=w[a:a + s], v2=True, compressed=False) for s, a in zip(sizes, np.cumsum([0] + sizes[:-1]))]
    return _one([_key(n, 71), Col("o", INT64, True, [Chunk(pgs, codec=SNAPPY)]),
                 Col("d", DOUBLE, False, [Chunk(dp, dict=d, codec=SNAPPY)]), Col("w", FLOAT, False, [Chunk(wp, codec=SNAPPY)])])


@case(dict_sizes=[0])
def dictionary_page_with_0_entries():
    """An empty dictionary, a dictionary page whose rows are all null (bit width 0, no runs), then PLAIN pages."""
    rng = _rng(72)
    v = _random_values(INT32, rng, 900)
    pgs = [Page(rows=100, enc=RLE_DICTIONARY, idx=[], bw=0, defs=[rle(100, 0)]),
           Page(rows=900, values=v, defs=[rle(900, 1)])]
    return _one([_key(1000, 72), Col("o", INT32, True, [Chunk(pgs, dict=np.zeros(0, np.int32))])])


# ---- parquet-mr page shapes ------------------------------------------------------------------------------------------
@case(dict_encodings={PLAIN_DICTIONARY}, page_stats=True, carried=["p"], no_dict_map=True,
      paths=[{"col": "p", "dict": "smem", "idx": "group", "carried": True}])
def parquet_mr_v1_plain_dictionary_with_statistics():
    """v1 dictionary and data pages that say PLAIN_DICTIONARY (2), Statistics in every DataPageHeader, the index bit
    width of the largest index: the only dictionary column of the file."""
    rng = _rng(80)
    sizes = [5000, 5000, 2345]
    n = sum(sizes)
    d = _dictionary(INT64, rng, 100)
    pgs = [Page(rows=s, enc=PLAIN_DICTIONARY, idx=[packed(rng.integers(0, 100, size=s))], stats=True) for s in sizes]
    return _one([_key(n, 80), Col("p", INT64, False, [Chunk(pgs, dict=d, dict_enc=PLAIN_DICTIONARY)])])


@case(bws={0}, dict_sizes=[1], paths=[{"col": "one", "idx": "hybrid"}, {"col": "one", "idx": "single"}])
def parquet_mr_one_entry_dictionary_bit_width_0():
    rng = _rng(81)
    d = _dictionary(DOUBLE, rng, 1)
    pgs = [Page(rows=5000, enc=PLAIN_DICTIONARY, idx=[rle(5000, 0)], stats=True),
           Page(rows=24, enc=PLAIN_DICTIONARY, idx=[packed(np.zeros(24, np.int64))], stats=True)]
    d2 = _dictionary(INT32, rng, 1)
    lv = _nulls_at(5024, [3, 4000])
    opg = [Page(rows=5024, enc=PLAIN_DICTIONARY, idx=[rle(5022, 0)], defs=runs_of(lv))]
    return _one([_key(5024, 81), Col("one", DOUBLE, False, [Chunk(pgs, dict=d, dict_enc=PLAIN_DICTIONARY)]),
                 Col("oo", INT32, True, [Chunk(opg, dict=d2, dict_enc=PLAIN_DICTIONARY)])])


@case(fallback=True, carried=[])
def parquet_mr_dictionary_fallback_to_plain():
    """A chunk that starts with its dictionary and two dictionary pages, then falls back to PLAIN pages."""
    rng = _rng(82)
    d = _dictionary(INT32, rng, 500)
    v = _random_values(INT32, rng, 5000)
    pgs = [Page(rows=3000, enc=PLAIN_DICTIONARY, idx=[packed(rng.integers(0, 500, size=3000))], stats=True),
           Page(rows=1000, enc=PLAIN_DICTIONARY, idx=[packed(rng.integers(0, 500, size=1000))], stats=True),
           Page(rows=5000, values=v, stats=True), Page(rows=10, values=v[:10], stats=True)]
    return _one([_key(9010, 82), Col("f", INT32, False, [Chunk(pgs, dict=d, dict_enc=PLAIN_DICTIONARY)])])


# ---- late materialisation: dictionary unions -------------------------------------------------------------------------
def _union_case(lo2, hi2, seed):
    """Two files, each one chunk of the int64 column u; file 1's dictionary is values 0..5000, file 2's lo2..hi2."""
    rng = _rng(seed)
    base = _dictionary(INT64, rng, 9000)
    specs = []
    for fi, (a, b) in enumerate(((0, 5000), (lo2, hi2))):
        d = base[a:b]
        n = 20_000
        ix = rng.integers(0, len(d), size=n)
        ix[:len(d)] = np.arange(len(d))
        specs.append(FileSpec([_key(n, seed + fi, start=fi * n, step=0),
                               Col("u", INT64, False, [Chunk([Page(rows=n, enc=RLE_DICTIONARY, idx=[packed(ix)])], dict=d)])]))
    return specs, {}


@case(union={"u": AGREE_CAP}, carried=["u"], nb=1)
def union_of_8192_dictionary_values():
    return _union_case(3192, 8192, 90)


@case(union={"u": AGREE_CAP + 1}, carried=[], nb=1)
def union_of_8193_dictionary_values():
    return _union_case(3192, 8193, 91)


@case(carried=["m", "n"], all_ones_values=True)
def carried_columns_holding_the_all_ones_value():
    """int64 -1 and the double NaN whose bits are all ones in carried dictionary columns (the hash set's empty mark)."""
    rng = _rng(92)
    n = 12_000
    dm = np.array([-1, 0, 5, -2, 2**62], dtype=np.int64)
    dn = np.array([0xFFFFFFFFFFFFFFFF, 0x7FF8000000000000, 0x3FF0000000000000, 0x8000000000000000],
                  dtype=np.uint64).view(np.float64)
    return _one([_key(n, 92),
                 _dict_col("m", INT64, dm, [[packed(rng.integers(0, 5, size=n))]], [n]),
                 _dict_col("n", DOUBLE, dn, [[packed(rng.integers(0, 4, size=n))]], [n])])


@case(carried=["c0", "c1", "c2", "c3"], nb=4)
def six_dictionary_columns_four_carried():
    rng = _rng(93)
    n = 10_000
    cols = [_key(n, 93)]
    for i, pt in enumerate((INT32, INT64, FLOAT, DOUBLE, INT32, INT64)):
        d = _dictionary(pt, rng, 10 + i)
        cols.append(_dict_col("c%d" % i, pt, d, [[packed(rng.integers(0, 10 + i, size=n))]], [n]))
    return _one(cols)


# ---- zero copy -------------------------------------------------------------------------------------------------------
@case(zero_copy={"a", "f"}, page_rows={"a": [4096, 4097, 4096], "b": [4095, 4097, 4097]})
def zero_copy_pages_of_4095_4096_4097_rows():
    """a and f: every page at least one tile (4096 / 4097 rows) -> read in place; b: one page of 4095 -> decoded."""
    rng = _rng(100)
    n = 12_289
    return _one([_key(n, 100), _plain("a", INT64, _random_values(INT64, rng, n), [4096, 4097, 4096], align=(8, 0)),
                 _plain("b", INT32, _random_values(INT32, rng, n), [4095, 4097, 4097], align=(4, 0)),
                 _plain("f", FLOAT, _random_values(FLOAT, rng, n), [4097, 8192], align=(4, 0))])


@case(zero_copy={"k", "a"}, page_edges_mod_tile={1, ZC_TILE - 1, 0})
def zero_copy_page_edges_at_tile_edges():
    """Page edges at 4097 (tile edge + 1), 12 287 (- 1) and 16 384 (on it): a tile table entry covers two pages."""
    rng = _rng(101)
    sizes = [4097, 8190, 4097, 5000]
    n = sum(sizes)
    return _one([_key(n, 101, pages=[6000, n - 6000], align=(8, 0)),
                 _plain("a", DOUBLE, _random_values(DOUBLE, rng, n), sizes, align=(8, 0))])


@case(zero_copy=set(), value_mod4={2})
def zero_copy_refused_for_one_unaligned_page():
    """Two files; the second file's middle page of a starts at 2 mod 4: the column is decoded, not read in place."""
    rng = _rng(102)
    specs = []
    for fi in range(2):
        a = _random_values(INT32, rng, 15_000)
        pgs = [Page(rows=5000, values=a[i * 5000:(i + 1) * 5000], align=(4, 2 if (fi, i) == (1, 1) else 0)) for i in range(3)]
        specs.append(FileSpec([_key(15_000, 102 + fi, start=fi * 15_000, step=0), Col("a", INT32, False, [Chunk(pgs, gap=5)])]))
    return specs, {}


@case(zero_copy={"k", "a", "g"}, file_rows=[5000, 6000])
def zero_copy_file_boundary_inside_a_tile():
    """Files of 5000 and 6000 rows: the tile of rows 4096..8191 starts in one file and ends in the next; chunks are
    separated by gaps the footer skips."""
    rng = _rng(103)
    specs = []
    for fi, n in enumerate((5000, 6000)):
        k = _key(n, 103 + fi, align=(8, 0))
        k.chunks[0].pages[0].values = k.chunks[0].pages[0].values + fi * 10**7
        a = Col("a", INT64, False, [Chunk([Page(rows=n, values=_random_values(INT64, rng, n), align=(8, 0))], gap=3 + fi)])
        g = Col("g", FLOAT, False, [Chunk([Page(rows=n, values=_random_values(FLOAT, rng, n), align=(4, 0))], gap=7)])
        specs.append(FileSpec([k, a, g]))
    return specs, {}


# ---- row windows (sorted scans) ---------------------------------------------------------------------------------------
def _window_file(fi, n, key_pages, a_pages, b_pages, c_pages, rng):
    k = (2 * np.arange(n, dtype=np.int64) + fi) * 3  # ascending; the files interleave
    key = _plain("k", INT64, k, key_pages)
    a = _plain("a", INT32, _random_values(INT32, rng, n), a_pages)
    b = _plain("b", DOUBLE, _random_values(DOUBLE, rng, n), b_pages, align=(8, 3))
    d = _dictionary(INT64, rng, 50)
    valid = rng.random(n) > 0.1
    c = Col("c", INT64, True, [Chunk([Page(rows=s, enc=RLE_DICTIONARY, idx=[packed(rng.integers(0, 50, size=int(valid[o:o + s].sum())))],
                                          defs=runs_of(valid[o:o + s].astype(np.int64)))
                                     for s, o in zip(c_pages, np.cumsum([0] + list(c_pages[:-1])))], dict=d)])
    return FileSpec([key, a, b, c])


WINDOW_PAGES = [dict(n=5000, key=[5000], a=[700] * 7 + [100], b=[1300, 1300, 1300, 1100], c=[2048, 2048, 904]),
                dict(n=4000, key=[1000, 3000], a=[1000] * 4, b=[999, 1, 3000], c=[4000])]


@case(windows=True)
def windows_on_page_edges():
    """Sorted files (k ascending) whose other columns are paged differently from the key; the scans' key predicates
    put window edges on their page edges and one row either side."""
    rng = _rng(110)
    specs = [_window_file(fi, w["n"], w["key"], w["a"], w["b"], w["c"], rng) for fi, w in enumerate(WINDOW_PAGES)]
    return specs, {}


def window_queries():
    """(lo_row, hi_row) in file 0 of the windows: every page edge of file 0's a, b and c, and one row either side, as
    window starts and ends."""
    edges = set()
    w = WINDOW_PAGES[0]
    for sizes in (w["a"], w["b"], w["c"]):
        edges |= set(np.cumsum(sizes)[:-1].tolist())
    rows = sorted({e + d for e in edges for d in (-1, 0, 1)})
    qs = [(0, r) for r in rows] + [(r, w["n"]) for r in rows]
    qs += [(rows[i], rows[j]) for i, j in ((0, 3), (3, 4), (5, 9), (2, len(rows) - 1))]
    qs += [(2100, 2101), (2100, 2100)]
    return qs


# ---- refusals --------------------------------------------------------------------------------------------------------
def refusal(fn):
    REFUSALS[fn.__name__] = fn
    return fn


@refusal
def delta_binary_packed_page():
    """A DELTA_BINARY_PACKED data page (encoding 5): refused as an unsupported encoding."""
    v = np.arange(100, 300, dtype=np.int64)
    return [FileSpec([_key(200, 120), Col("x", INT64, False, [Chunk([Page(rows=200, enc=DELTA_BINARY_PACKED, values=v)])])])], \
        ("x",), "encoding"


@refusal
def nested_column():
    """A column inside a group: refused, the message names nesting."""
    rng = _rng(121)
    return [FileSpec([_key(100, 121), _plain("x", INT32, _random_values(INT32, rng, 100), [100])], nested=True)], \
        ("k",), "nested"
