"""Index builds over table T written three times by pyarrow: UNCOMPRESSED, SNAPPY and LZ4_RAW (pyarrow's "lz4"), with the
encodings of bench_gzip.py.  The images are staged in HBM once; builds alternate NONE / SNAPPY / LZ4_RAW after a warm-up
of each, and the index files of the three codecs are checked identical.  The decompression kernels' times come from a
profiled run of their own.

    python bench_lz4.py --rows 100000000 --buckets 200 --runs 3

Prints one JSON line: per codec the ms of every build, the decode stage's ms, the decompression kernels' ms, the
compressed bytes in and uncompressed bytes out of the compressed pages and their rates over the kernel time, and the
card with its power limit, read in the same command."""
import argparse
import hashlib
import json
import subprocess
import time
from concurrent.futures import ThreadPoolExecutor

from bench_gzip import INCLUDED, _image, _page_bytes
from hyperspace_b200 import _native as N

CODECS = {"NONE": "NONE", "SNAPPY": "SNAPPY", "LZ4_RAW": "LZ4"}  # name -> pyarrow's compression argument
DECOMPRESSORS = ("k_lz4", "k_snappy_index", "k_snappy_blocks", "k_snappy_levels")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=100_000_000)
    ap.add_argument("--files", type=int, default=32)
    ap.add_argument("--buckets", type=int, default=200)
    ap.add_argument("--runs", type=int, default=3)
    a = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip().splitlines()[0]
    t0 = time.time()
    per = a.rows // a.files
    with ThreadPoolExecutor() as pool:
        images = {c: list(pool.map(lambda f, w=w: _image(f * per, per, w), range(a.files))) for c, w in CODECS.items()}
    gen_s = time.time() - t0
    ctx = N.Context(0)
    staged = {c: ctx.stage_sources([N.FileImage(data=b) for b in v]) for c, v in images.items()}  # resident in HBM
    for s in staged.values():
        s.wait()
    result = {"rows": per * a.files, "files": a.files, "buckets": a.buckets, "card": card, "generate_s": round(gen_s, 1),
              "codecs": {}}
    digests = {}
    for c in CODECS:  # warm-up of every path, and the index files of each codec
        res, _ = ctx.create_index(staged[c].as_sources(), ["k"], INCLUDED, a.buckets, output=N.HS_OUT_HOST, job_uuid="bench")
        digests[c] = [hashlib.sha256(res.host_bytes(i)).hexdigest() for i in range(len(res.files))]
        res.free()
    result["identical_outputs"] = digests["NONE"] == digests["SNAPPY"] == digests["LZ4_RAW"]
    builds = {c: [] for c in CODECS}
    decode = {c: [] for c in CODECS}
    for _ in range(a.runs):
        for c in CODECS:
            res, st = ctx.create_index(staged[c].as_sources(), ["k"], INCLUDED, a.buckets, output=N.HS_OUT_DEVICE)
            res.free()
            builds[c].append(round(st["ms_total"], 2))
            decode[c].append(round(st["ms_decode"], 2))
    for c in CODECS:
        ctx.profile_enable(True)
        res, st = ctx.create_index(staged[c].as_sources(), ["k"], INCLUDED, a.buckets, output=N.HS_OUT_DEVICE)
        prof = ctx.profile_report()
        ctx.profile_enable(False)
        res.free()
        kern = {k: round(v["ms"], 3) for k, v in prof.items() if k in DECOMPRESSORS + ("k_decode_pages",)}
        comp, uncomp = _page_bytes(images[c])
        entry = {"ms_per_build": builds[c], "ms_decode": decode[c], "kernel_ms": kern, "gpu_launches": st["gpu_launches"],
                 "file_bytes": sum(len(b) for b in images[c]), "chunk_bytes_compressed": comp, "chunk_bytes_uncompressed": uncomp}
        dec_ms = sum(kern.get(k, 0.0) for k in DECOMPRESSORS)
        if c != "NONE" and dec_ms > 0:
            entry["decompress_ms"] = round(dec_ms, 3)
            entry["GB_in_per_s"] = round(comp / dec_ms / 1e6, 2)
            entry["GB_out_per_s"] = round(uncomp / dec_ms / 1e6, 2)
        result["codecs"][c] = entry
    for s in staged.values():
        s.free()
    ctx.close()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
