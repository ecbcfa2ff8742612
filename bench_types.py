"""Index builds over the same rows with the key stored three ways: INT64 micros, INT96 with a dictionary (what Spark 3.1
writes for a timestamp), and decimal(18,2) as FIXED_LEN_BYTE_ARRAY (pyarrow's default).  The INT96 and decimal keys are
converted while decoding (k_decode_converted_pages) and take the value path: no zero-copy read, no late
materialisation.  Builds alternate between the three layouts; the profile comes from a run of its own.

    python bench_types.py --rows 50000000 --buckets 200 --runs 3

Prints one JSON line with, per layout, the ms of every build, the decode stage time, the decode kernels' time and the
card with its power limit, read in the same command."""
import argparse
import io
import json
import subprocess
import time

import numpy as np
import pyarrow as pa
import pyarrow.parquet as pq

from hyperspace_b200 import _native as N


def _images(rows: int, files: int, seed: int):
    """{layout: [Parquet images]} of the same key values (micros) and one int64 payload column."""
    rng = np.random.default_rng(seed)
    per = rows // files
    out = {"int64_micros": [], "int96_dict": [], "decimal18_flba": []}
    distinct = rng.integers(0, 4_000_000_000_000_000, 50_000, dtype=np.int64)  # 1970 .. 2096, in micros
    for f in range(files):
        micros = distinct[rng.integers(0, len(distinct), per)]
        v = pa.array(np.arange(per, dtype=np.int64) + f * per)
        for layout in out:
            if layout == "int64_micros":
                t, kw = pa.table({"k": pa.array(micros, pa.timestamp("us")), "v": v}), {"use_dictionary": False}
            elif layout == "int96_dict":
                t, kw = pa.table({"k": pa.array(micros * 1000, pa.timestamp("ns")), "v": v}), {
                    "use_deprecated_int96_timestamps": True, "use_dictionary": ["k"], "dictionary_pagesize_limit": 1 << 30}
            else:
                unscaled = np.stack([micros, micros >> 63], axis=1)  # 16-byte little-endian two's complement
                dec = pa.Array.from_buffers(pa.decimal128(18, 2), per, [None, pa.py_buffer(unscaled.tobytes())])
                t, kw = pa.table({"k": dec, "v": v}), {"use_dictionary": False}
            sink = io.BytesIO()
            pq.write_table(t, sink, compression="NONE", row_group_size=1 << 22, **kw)
            out[layout].append(sink.getvalue())
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=50_000_000)
    ap.add_argument("--files", type=int, default=8)
    ap.add_argument("--buckets", type=int, default=200)
    ap.add_argument("--runs", type=int, default=3)
    a = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip().splitlines()[0]
    t0 = time.time()
    images = _images(a.rows, a.files, 1)
    gen_s = time.time() - t0
    ctx = N.Context(0)
    staged = {k: ctx.stage_sources([N.FileImage(data=b) for b in v]) for k, v in images.items()}  # images resident in HBM
    for s in staged.values():
        s.wait()
    result = {"rows": a.rows, "buckets": a.buckets, "card": card, "generate_s": round(gen_s, 1), "layouts": {}}
    for k in staged:  # warm-up of every path
        res, _ = ctx.create_index(staged[k].as_sources(), ["k"], ["v"], a.buckets, output=N.HS_OUT_DEVICE)
        res.free()
    builds = {k: [] for k in staged}
    decode = {k: [] for k in staged}
    for _ in range(a.runs):
        for k in staged:
            res, st = ctx.create_index(staged[k].as_sources(), ["k"], ["v"], a.buckets, output=N.HS_OUT_DEVICE)
            res.free()
            builds[k].append(round(st["ms_total"], 2))
            decode[k].append(round(st["ms_decode"], 2))
    for k in staged:
        ctx.profile_enable(True)
        res, _ = ctx.create_index(staged[k].as_sources(), ["k"], ["v"], a.buckets, output=N.HS_OUT_DEVICE)
        prof = ctx.profile_report()
        ctx.profile_enable(False)
        res.free()
        result["layouts"][k] = {"ms_per_build": builds[k], "ms_decode_stage": decode[k],
                                "k_decode_pages_ms": round(prof.get("k_decode_pages", {}).get("ms", 0.0), 3),
                                "k_decode_converted_pages_ms": round(prof.get("k_decode_converted_pages", {}).get("ms", 0.0), 3),
                                "zero_copy": "k_fill_zc_tiles" in prof}
    for s in staged.values():
        s.free()
    ctx.close()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
