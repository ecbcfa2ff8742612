#!/usr/bin/env python
"""bench_bool.py -- createIndex with boolean included columns, on ONE GPU: table T (k, v1..v4) plus two boolean columns,
`flag` (null-free) and `maybe` (10 % null), --rows rows (100 M) in 64 Parquet files, 200 buckets, the source images resident
in HBM (hs_stage_sources).

  encode  builds over the same images with and without the two booleans, alternated --reps times after a warm-up: ms per
          build, the encode stage (hs_stats.ms_encode) and, from a separate profiled build, k_gather_encode_bool and
          k_gather_encode_bool_nullable.
  decode  the same table written with PLAIN and with RLE booleans (pyarrow's column_encoding): the decode stage of a build
          over each, alternated likewise.

Every timed build is checked with hs_verify_index over all of its files (rows, bucket ids, order).  Before timing, the same
builds run at --check-rows rows and pyarrow reads a sampled bucket file back, compared row by row with the CPU oracle.
The source files are written to a temporary directory.  The card's name and power limit are read in the same run.
"""
import argparse
import json
import os
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

from bench_joins import card_info  # noqa: E402

NB, NFILES = 200, 64
T_COLS = ["v1", "v2", "v3", "v4"]
BOOLS = ["flag", "maybe"]


def bool_columns(first, n):
    import numpy as np

    from oracle import oracle as O

    i = np.arange(first, first + n, dtype=np.uint64)
    h = O.splitmix64(77, i)
    return (h & 1).astype(bool), ((h >> 1) & 1).astype(bool), (h >> 8) % 10 != 0  # flag, maybe, maybe's validity


def write_table(d, n, encoding):
    import numpy as np
    import pyarrow as pa
    import pyarrow.parquet as pq

    from oracle import oracle as O

    os.makedirs(d, exist_ok=True)
    per = -(-n // NFILES)
    paths = []
    for f in range(NFILES):
        a, b = f * per, min(n, (f + 1) * per)
        if a >= b:
            break
        c = O.synthetic_table(a, b - a, 5)
        flag, maybe, mvalid = bool_columns(a, b - a)
        t = pa.table({**{k: c[k] for k in ["k"] + T_COLS}, "flag": flag, "maybe": pa.array(maybe, mask=~mvalid)})
        p = os.path.join(d, f"part-{f:05d}.parquet")
        pq.write_table(t, p, compression="snappy", use_dictionary=["v3", "v4"],
                       column_encoding={"flag": encoding, "maybe": encoding, "k": "PLAIN", "v1": "PLAIN", "v2": "PLAIN"})
        paths.append(p)
    return paths


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=100_000_000)
    ap.add_argument("--check-rows", type=int, default=2_000_000)
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    import numpy as np
    import pyarrow as pa
    import pyarrow.parquet as pq
    import torch

    from hyperspace_b200 import _native as N
    from oracle import oracle as O

    ctx = N.Context(0, torch.cuda.current_stream().cuda_stream)
    info = card_info()
    print(json.dumps({"device": torch.cuda.get_device_name(0), **info}))
    tmp = tempfile.mkdtemp(prefix="bench_bool_")

    def stage(paths):
        st = ctx.stage_sources([N.FileImage(path=p) for p in paths])
        st.wait()
        return st

    def build(src, included, output=N.HS_OUT_DEVICE):
        return ctx.create_index(src.as_sources(), ["k"], included, NB, output=output, job_uuid="bool")

    def verify(res, n, included):
        rep = ctx.verify_index(res.as_sources(), [f.bucket for f in res.files], ["k"], included, NB)
        assert rep["rows"] == n and rep["bucket_mismatches"] == 0 and rep["order_violations"] == 0, rep

    # ---- correctness at a reduced size: a sampled bucket read back by pyarrow equals the oracle's rows --------------------
    n = args.check_rows
    c = O.synthetic_table(0, n, 5)
    flag, maybe, mvalid = bool_columns(0, n)
    cols = {**{k: c[k] for k in ["k"] + T_COLS}, "flag": flag, "maybe": maybe}
    perm, offs, _ = O.index_rows(cols, ["k"], T_COLS + BOOLS, NB)
    for enc in ("PLAIN", "RLE"):
        src = stage(write_table(os.path.join(tmp, f"check_{enc}"), n, enc))
        res, _ = build(src, T_COLS + BOOLS, N.HS_OUT_HOST)
        i = len(res.files) // 2
        b = res.files[i].bucket
        t = pq.ParquetFile(pa.BufferReader(res.host_bytes(i))).read()
        rows = perm[int(offs[b]):int(offs[b + 1])]
        ok = all(np.array_equal(t.column(k).to_numpy(), cols[k][rows]) for k in ["k"] + T_COLS + ["flag"])
        m = t.column("maybe").combine_chunks()
        ok = ok and np.array_equal(np.asarray(m.is_valid()), mvalid[rows])
        ok = ok and np.array_equal(m.fill_null(False).to_numpy(zero_copy_only=False)[mvalid[rows]], maybe[rows][mvalid[rows]])
        print(json.dumps({"check": enc, "rows": n, "bucket": b, "bucket_rows": int(len(rows)), "ok": bool(ok)}))
        assert ok
        res.free()
        src.free()
    ctx.trim()

    # ---- timed ------------------------------------------------------------------------------------------------------------
    def timed(src, included):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        res, st = build(src, included)
        torch.cuda.synchronize()
        ms = (time.perf_counter() - t0) * 1e3
        verify(res, args.rows, included)
        res.free()
        return ms, st

    def profiled(src, included):
        ctx.profile_enable(True)
        ctx.profile_report()
        res, _ = build(src, included)
        res.free()
        rep = ctx.profile_report()
        ctx.profile_enable(False)
        return {k: {"ms": round(v["ms"], 3), "launches": v["launches"]} for k, v in rep.items()
                if k.startswith("k_gather_encode") or k.startswith("k_decode")}

    paths = {enc: write_table(os.path.join(tmp, enc), args.rows, enc) for enc in ("PLAIN", "RLE")}
    src = stage(paths["PLAIN"])
    work = {"with_bools": T_COLS + BOOLS, "without_bools": T_COLS}
    for inc in work.values():
        timed(src, inc)  # warm-up
    res = {k: [] for k in work}
    for _ in range(args.reps):
        for k, inc in work.items():
            res[k].append(timed(src, inc))
    for k, inc in work.items():
        print(json.dumps({"workload": "encode", "config": k, "ms_per_build": [round(m, 1) for m, _ in res[k]],
                          "ms_encode": [round(st["ms_encode"], 2) for _, st in res[k]],
                          "profiled_kernels": profiled(src, inc), "rows": args.rows, "buckets": NB, **info}))
    src.free()
    ctx.trim()

    srcs = {enc: stage(p) for enc, p in paths.items()}
    for s in srcs.values():
        timed(s, T_COLS + BOOLS)
    dec = {k: [] for k in srcs}
    for _ in range(args.reps):
        for k, s in srcs.items():
            dec[k].append(timed(s, T_COLS + BOOLS))
    for k, s in srcs.items():
        print(json.dumps({"workload": "decode", "config": f"{k} booleans", "ms_per_build": [round(m, 1) for m, _ in dec[k]],
                          "ms_decode": [round(st["ms_decode"], 2) for _, st in dec[k]],
                          "profiled_kernels": profiled(s, T_COLS + BOOLS), "rows": args.rows, "buckets": NB, **info}))
        s.free()
    ctx.close()


if __name__ == "__main__":
    t0 = time.perf_counter()
    main()
    print(json.dumps({"wall_s": round(time.perf_counter() - t0, 1)}), file=sys.stderr)
