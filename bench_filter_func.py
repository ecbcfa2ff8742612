#!/usr/bin/env python
"""bench_filter_func.py -- Spark functions in filters (hs_filter_scan_expr with function nodes) on ONE GPU.

The table is table T (k, v1..v4: oracle.synthetic_table) plus three columns a filter applies functions to: d (date,
1990-01-01 .. 1999-12-31), d2 (timestamp, within 60 days after d's midnight) and s (a phone number, "CC-DDD-DDD-DDDD"
with CC in 10..34).  It is written as in-memory Parquet files with pyarrow and indexed on k (200 buckets, index files
resident in HBM).  Four queries alternate --reps times in one process, each over --queries seeded 1 % ranges of k (C3's
windows in bench_filters.py):
  c3             C3 alone: one 1 % range of k
  year           the range AND year(d) = 1995
  substring      the range AND substring(s, 1, 2) = '13'           (TPC-H Q22's country code)
  datediff       the range AND datediff(d2, d) > 30                (a timestamp cast to its UTC date)
Every query reports ms per query and rows out per query, and from one separate profiled pass the per-kernel ms per query
(k_func_mask among them).  Before timing, each query runs on a --check-rows table and is compared with numpy.  The card's
name and power limit are read in the same run.
"""
import argparse
import io
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

from bench_filters import card_info  # noqa: E402

DAY_US = 86_400_000_000
D0 = 7305  # 1990-01-01


def extra_columns(first_row, n):
    """d (date days), d2 (timestamp micros) and s (15-byte phone numbers, one row of a uint8 matrix each) of rows
    [first_row, first_row + n), from the same splitmix64 stream as table T."""
    import numpy as np

    from oracle.oracle import splitmix64

    i = np.arange(first_row, first_row + n, dtype=np.uint64)
    h = splitmix64(44, i)
    d = (D0 + h % np.uint64(3652)).astype(np.int32)
    d2 = d.astype(np.int64) * DAY_US + ((h >> np.uint64(12)) % np.uint64(60 * DAY_US)).astype(np.int64)
    digits = np.empty((n, 15), dtype=np.uint8)
    cc = 10 + (h >> np.uint64(40)) % np.uint64(25)
    digits[:, 0] = ord("0") + cc // np.uint64(10)
    digits[:, 1] = ord("0") + cc % np.uint64(10)
    g = splitmix64(45, i)
    for p in range(2, 15):
        if p in (2, 6, 10):
            digits[:, p] = ord("-")
        else:
            digits[:, p] = ord("0") + (g % np.uint64(10)).astype(np.uint8)
            g //= np.uint64(10)
    return d, d2, digits


def parquet_files(n, n_files):
    """Table T plus d, d2 and s as n_files in-memory Parquet files (FileImage list)."""
    import numpy as np
    import pyarrow as pa
    import pyarrow.parquet as pq

    from hyperspace_b200 import _native as N
    from oracle import oracle as O

    out = []
    per = (n + n_files - 1) // n_files
    for f in range(n_files):
        lo, hi = f * per, min(n, (f + 1) * per)
        if lo >= hi:
            break
        t = O.synthetic_table(lo, hi - lo, 5)
        d, d2, s = extra_columns(lo, hi - lo)
        offsets = pa.py_buffer(np.arange(0, 15 * (hi - lo) + 1, 15, dtype=np.int32))
        strings = pa.StringArray.from_buffers(hi - lo, offsets, pa.py_buffer(s.tobytes()))
        table = pa.table({**{c: t[c] for c in ("k", "v1", "v2", "v3", "v4")}, "d": pa.array(d).view(pa.date32()),
                          "d2": pa.array(d2).view(pa.timestamp("us")), "s": strings})
        sink = io.BytesIO()
        pq.write_table(table, sink, compression="NONE", row_group_size=1 << 20, use_dictionary=False, write_statistics=False)
        out.append(N.FileImage(path=f"t{f}.parquet", data=sink.getvalue(), file_id=f))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=100_000_000)
    ap.add_argument("--files", type=int, default=64)
    ap.add_argument("--check-rows", type=int, default=2_000_000)
    ap.add_argument("--queries", type=int, default=10)
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    import numpy as np
    import torch

    from hyperspace_b200 import _native as N
    from oracle import oracle as O

    stream = torch.cuda.current_stream()
    ctx = N.Context(0, stream.cuda_stream)
    nb = 200
    info = card_info()
    print(json.dumps({"device": torch.cuda.get_device_name(0), **info}), flush=True)
    proj = ["k", "v1", "v2"]
    width = int(0.01 * 2**64)
    ranges = [(-(width // 2) + i * (width // 40), (width // 2) + i * (width // 40)) for i in range(args.queries)]
    C = lambda n: ("column", n)  # noqa: E731
    L = lambda v: ("literal", v)  # noqa: E731
    variants = {"c3": [], "year": [([C("d"), ("year",)], "=", [L(1995)])],
                "substring": [([C("s"), L(1), L(2), ("substring",)], "=", [L("13")])],
                "datediff": [([C("d2"), C("d"), ("datediff",)], ">", [L(30)])]}

    def run(srcs, q, exprs):
        lo, hi = q
        return ctx.filter_scan_expr(srcs, "k", proj, [("k", lo, False, hi, False)], [], [], exprs)[0]

    # ---- correctness at a small size, against numpy ----------------------------------------------------------------------
    small_src = parquet_files(args.check_rows, 4)
    small, _ = ctx.create_index(small_src, ["k"], ["v1", "v2", "v3", "v4", "d", "d2", "s"], nb, output=N.HS_OUT_DEVICE, job_uuid="c")
    del small_src
    k = O.synthetic_table(0, args.check_rows, 1)["k"]
    d, d2, s = extra_columns(0, args.check_rows)
    year = d.astype("datetime64[D]").astype("datetime64[Y]").astype(np.int64) + 1970
    in_numpy = {"c3": True, "year": year == 1995, "substring": (s[:, 0] == ord("1")) & (s[:, 1] == ord("3")),
                "datediff": (d2 // DAY_US - d) > 30}
    wide = (-(2**62), 2**62)  # half of k's range: enough rows at the check size
    for name, exprs in variants.items():
        m = (k >= wide[0]) & (k <= wide[1]) & in_numpy[name]
        b = run(small.as_sources(), wide, exprs)
        got = np.sort(b.column("k").astype(np.int64))
        b.free()
        assert np.array_equal(got, np.sort(k[m])), name
        print(json.dumps({"check": name, "rows": int(m.sum()), "ok": True}), flush=True)
    small.free()
    ctx.trim()

    # ---- the index ------------------------------------------------------------------------------------------------------
    t0 = time.perf_counter()
    src = parquet_files(args.rows, args.files)
    print(json.dumps({"table_rows": args.rows, "files": len(src), "parquet_bytes": sum(len(f.data) for f in src),
                      "write_s": round(time.perf_counter() - t0, 1)}), flush=True)
    idx, st = ctx.create_index(src, ["k"], ["v1", "v2", "v3", "v4", "d", "d2", "s"], nb, output=N.HS_OUT_DEVICE, job_uuid="t")
    del src
    ctx.trim()
    srcs = idx.as_sources()

    def timed(exprs):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record(stream)
        rows = 0
        for q in ranges:
            b = run(srcs, q, exprs)
            rows += b.num_rows
            b.free()
        e1.record(stream)
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / len(ranges), rows / len(ranges)

    for exprs in variants.values():  # warm every shape over every window: the first pass grows the allocator's pools
        timed(exprs)
    ms = {name: [] for name in variants}
    rows = {}
    for _ in range(args.reps):  # alternating, so that clocks and temperature drift hit every query alike
        for name, exprs in variants.items():
            t, rows[name] = timed(exprs)
            ms[name].append(round(t, 3))
    for name, exprs in variants.items():
        ctx.profile_enable(True)
        ctx.profile_report()
        for q in ranges:
            run(srcs, q, exprs).free()
        rep = ctx.profile_report()
        ctx.profile_enable(False)
        kern = {kn: round(v["ms"] / len(ranges), 4) for kn, v in sorted(rep.items(), key=lambda kv: -kv[1]["ms"])}
        print(json.dumps({"workload": name, "exprs": [str(e) for e in exprs], "ms_per_query": ms[name],
                          "rows_out_per_query": rows[name], "profiled_kernel_ms_per_query": kern, **info}), flush=True)
    idx.free()
    ctx.close()


if __name__ == "__main__":
    t0 = time.perf_counter()
    main()
    print(json.dumps({"wall_s": round(time.perf_counter() - t0, 1)}), file=sys.stderr)
