"""Index builds over table T with each output codec: NONE, SNAPPY, GZIP and LZ4 (spark.sql.parquet.compression.codec).
The UNCOMPRESSED source images are staged in HBM once; builds alternate the four codecs after a warm-up of each.  Every
codec's index is checked: hs_verify_index passes with the same row checksum as the NONE build, and pyarrow reads the first
bucket file equal to the NONE build's.  The compressor kernels' times come from a profiled run of their own, and C3
(`k BETWEEN lo AND hi`, 1 % of the key space, projecting k, v1, v2) is timed over each index, which is what the decoders
add on the read side.  The GZIP pages are also recompressed on the host with zlib at level 6, the ratio reference.

    python bench_index_codecs.py --rows 100000000 --buckets 200 --runs 3

Prints one JSON line, with the card and its power limit read in the same command."""
import argparse
import gzip
import json
import os
import subprocess
import sys
import time
import zlib
from concurrent.futures import ThreadPoolExecutor

import pyarrow as pa
import pyarrow.parquet as pq

from bench_gzip import INCLUDED, _image
from hyperspace_b200 import _native as N

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "tests"))
import parquet_shapes as S  # noqa: E402  (the footer reader of the tests)

CODECS = {"NONE": N.HS_CODEC_UNCOMPRESSED, "SNAPPY": N.HS_CODEC_SNAPPY, "GZIP": N.HS_CODEC_GZIP, "LZ4": N.HS_CODEC_LZ4}
COMPRESSORS = ("k_snappy_compress", "k_deflate_compress", "k_lz4_compress")


def _zlib6_of_gzip_pages(data: bytes):
    """(bytes of the file's GZIP page bodies, their zlib level-6 size): every page of every column chunk"""
    footer, _ = S.read_struct(data, len(data) - 8 - int.from_bytes(data[-8:-4], "little"))
    ours = ref = 0
    for rg in footer[4]:
        for cc in rg[1]:
            md = cc[3]
            p = md.get(11) or md[9]  # dictionary page first when there is one
            end = p + md[7]
            while p < end:
                hdr, q = S.read_struct(data, p)
                body = data[q:q + hdr[3]]
                ours += len(body)
                ref += len(zlib.compress(gzip.decompress(body), 6))
                p = q + hdr[3]
    return ours, ref


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=100_000_000)
    ap.add_argument("--files", type=int, default=32)
    ap.add_argument("--buckets", type=int, default=200)
    ap.add_argument("--runs", type=int, default=3)
    a = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip().splitlines()[0]
    per = a.rows // a.files
    with ThreadPoolExecutor() as pool:
        images = list(pool.map(lambda f: _image(f * per, per, "NONE"), range(a.files)))
    ctx = N.Context(0)
    staged = ctx.stage_sources([N.FileImage(data=b) for b in images])  # resident in HBM
    staged.wait()
    rows = per * a.files
    result = {"rows": rows, "files": a.files, "buckets": a.buckets, "card": card, "codecs": {}}
    outputs, checks = {}, {}
    for c, codec in CODECS.items():  # warm-up of every path, and the verified index of each codec
        res, _ = ctx.create_index(staged.as_sources(), ["k"], INCLUDED, a.buckets, output=N.HS_OUT_HOST, job_uuid="bench",
                                  compression=codec)
        outputs[c] = [(f.bucket, res.host_bytes(i)) for i, f in enumerate(res.files)]
        res.free()
        rep = ctx.verify_index([N.FileImage(data=d) for _, d in outputs[c]], [b for b, _ in outputs[c]], ["k"], INCLUDED,
                               a.buckets)
        checks[c] = (rep["rows"], rep["bucket_mismatches"], rep["order_violations"], rep["row_checksum"])
    first = pq.ParquetFile(pa.BufferReader(outputs["NONE"][0][1])).read()
    result["verified"] = all(checks[c] == checks["NONE"] and checks[c][0] == rows and checks[c][1:3] == (0, 0) and
                             pq.ParquetFile(pa.BufferReader(outputs[c][0][1])).read().equals(first) for c in CODECS)
    builds = {c: [] for c in CODECS}
    encode = {c: [] for c in CODECS}
    for _ in range(a.runs):
        for c, codec in CODECS.items():
            res, st = ctx.create_index(staged.as_sources(), ["k"], INCLUDED, a.buckets, output=N.HS_OUT_DEVICE, compression=codec)
            res.free()
            builds[c].append(round(st["ms_total"], 2))
            encode[c].append(round(st["ms_encode"], 2))
    span = 2 ** 64 // 100  # C3: 1 % of the int64 key space
    lo, hi = -span // 2, span // 2
    for c, codec in CODECS.items():
        ctx.profile_enable(True)
        res, st = ctx.create_index(staged.as_sources(), ["k"], INCLUDED, a.buckets, output=N.HS_OUT_DEVICE, compression=codec)
        prof = ctx.profile_report()
        ctx.profile_enable(False)
        res.free()
        files = [N.FileImage(data=d) for _, d in outputs[c]]
        c3 = []
        for i in range(a.runs + 1):
            t0 = time.perf_counter()
            batch, _ = ctx.filter_scan(files, "k", ["k", "v1", "v2"], lo=lo, hi=hi)
            c3.append(round((time.perf_counter() - t0) * 1e3, 2))
            n_c3 = batch.num_rows
            batch.free()
        entry = {"ms_per_build": builds[c], "ms_encode": encode[c],
                 "compress_kernel_ms": {k: round(v["ms"], 3) for k, v in prof.items() if k in COMPRESSORS},
                 "index_bytes": sum(len(d) for _, d in outputs[c]), "c3_ms": c3[1:], "c3_rows": n_c3}
        if c == "GZIP":
            with ThreadPoolExecutor() as pool:
                sizes = list(pool.map(lambda bd: _zlib6_of_gzip_pages(bd[1]), outputs[c]))
            entry["page_bytes"] = sum(s[0] for s in sizes)
            entry["zlib6_page_bytes"] = sum(s[1] for s in sizes)
        result["codecs"][c] = entry
    staged.free()
    ctx.close()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
