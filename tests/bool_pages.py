"""Boolean columns in index files, restated in numpy: the page bodies the encoder writes, a reader of the RLE / bit-packed
hybrid stream, and a page iterator for v1 and v2 data pages (pyarrow's and the engine's).

The encoder writes a BOOLEAN column as parquet-mr's v1 writer does: PLAIN, values bit-packed LSB first, the unused bits
of the last byte zero, never dictionary-encoded.
- null-free page of n rows: [u32 length][one RLE run of n ones] then ceil(n / 8) value bytes;
- nullable page of n rows, m of them non-null: [u32 length][one bit-packed run of ceil(n / 8) groups][ceil(n / 8) bytes of
  definition bits, LSB first, padding zero] then ceil(m / 8) value bytes.
"""
import struct

import numpy as np

import parquet_shapes as S


def packbits(bits) -> bytes:
    return np.packbits(np.asarray(bits, dtype=bool), bitorder="little").tobytes()


def page_body(values, valid=None) -> bytes:
    """The body of one PLAIN BOOLEAN page over `values` (the page's rows in order; nulls: valid == False)."""
    values = np.asarray(values, dtype=bool)
    n = len(values)
    if valid is None:
        defs = S.varint(n << 1) + b"\x01"
        return struct.pack("<I", len(defs)) + defs + packbits(values)
    valid = np.asarray(valid, dtype=bool)
    groups = (n + 7) // 8
    hdr = S.varint((groups << 1) | 1)
    return struct.pack("<I", len(hdr) + groups) + hdr + packbits(valid) + packbits(values[valid])


def page_bodies(values, valid, rows_per_page):
    """Bodies of the pages of one column chunk: rows_per_page rows each."""
    n = len(values)
    return [page_body(values[p:p + rows_per_page], None if valid is None else valid[p:p + rows_per_page])
            for p in range(0, n, rows_per_page)]


def read_hybrid(b, p, end, bw, n):
    """n values of an RLE / bit-packed hybrid stream b[p:end]; raises ValueError when a run leaves the stream."""
    out = []
    while len(out) < n:
        if p >= end:
            raise ValueError("stream ends early")
        h, p = S._read_varint(b, p)
        if h & 1:
            nbytes = (h >> 1) * bw
            if p + nbytes > end:
                raise ValueError("bit-packed run past the stream")
            bits = np.unpackbits(np.frombuffer(b[p:p + nbytes], np.uint8), bitorder="little").reshape(-1, bw)
            out.extend((bits.astype(np.uint64) << np.arange(bw, dtype=np.uint64)).sum(axis=1).tolist())
            p += nbytes
        else:
            w = (bw + 7) // 8
            if p + w > end:
                raise ValueError("RLE run value past the stream")
            out.extend([int.from_bytes(b[p:p + w], "little")] * (h >> 1))
            p += w
    return np.asarray(out[:n], dtype=np.uint64), p


def data_pages(image, column):
    """(page header dict, decompressed body, valid, values) of every data page of `column` in a file image, v1 and v2,
    BOOLEAN only; values are the non-null values as read from the PLAIN or RLE encoding."""
    img = bytes(image)
    flen = struct.unpack_from("<I", img, len(img) - 8)[0]
    fm, _ = S.read_struct(img, len(img) - 8 - flen)
    leaves = [x[4].decode() for x in fm[2][1:]]
    ci = leaves.index(column)
    optional = fm[2][1 + ci].get(3, 1) == 1
    out = []
    for rg in fm[4]:
        md = rg[1][ci][3]
        codec = md[4]
        p, end = md.get(11, md[9]), md.get(11, md[9]) + md[7]
        while p < end:
            h, q = S.read_struct(img, p)
            usize, csize = h[2], h[3]
            raw = img[q:q + csize]
            p = q + csize
            if h[1] == S.DATA_PAGE:
                n, enc = h[5][1], h[5][2]
                body = _decompress(codec, raw, usize)
                at = 0
                if optional:
                    dl = struct.unpack_from("<I", body, 0)[0]
                    valid = read_hybrid(body, 4, 4 + dl, 1, n)[0].astype(bool)
                    at = 4 + dl
                else:
                    valid = np.ones(n, bool)
            elif h[1] == S.DATA_PAGE_V2:
                v2 = h[8]
                n, enc, dl, rl = v2[1], v2[4], v2[5], v2.get(6, 0)
                levels, rest = raw[:rl + dl], raw[rl + dl:]
                if v2.get(7, True) and codec != S.UNCOMPRESSED:
                    rest = _decompress(codec, rest, usize - rl - dl)
                body = levels + rest
                valid = read_hybrid(body, rl, rl + dl, 1, n)[0].astype(bool) if optional and dl else np.ones(n, bool)
                at = rl + dl
            else:
                continue
            m = int(valid.sum())
            if enc == S.PLAIN:
                vals = np.unpackbits(np.frombuffer(body[at:], np.uint8), bitorder="little")[:m].astype(bool)
            elif enc == S.RLE:
                ln = struct.unpack_from("<I", body, at)[0]
                vals = read_hybrid(body, at + 4, at + 4 + ln, 1, m)[0].astype(bool)
            else:
                raise ValueError(f"encoding {enc}")
            out.append(dict(n=n, enc=enc, v2=h[1] == S.DATA_PAGE_V2, body=body, values_at=at, valid=valid, values=vals))
    return out


def _decompress(codec, body, size):
    import pyarrow as pa

    if codec == S.UNCOMPRESSED:
        return bytes(body)
    if codec == S.SNAPPY:
        return pa.decompress(body, size, codec="snappy", asbytes=True)
    if codec == 2:
        return pa.decompress(body, size, codec="gzip", asbytes=True)
    raise ValueError(f"codec {codec}")
