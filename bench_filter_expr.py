#!/usr/bin/env python
"""bench_filter_expr.py -- expression comparisons (hs_filter_scan_expr) on ONE GPU.

Over the 500 M-row, 200-bucket index of table T on k (C3's setup in bench_filters.py; index files resident in HBM), three
queries alternate --reps times in one process, each over --queries seeded 1 % ranges of k:
  c3             C3 alone: one 1 % range of k
  v1x3_v3_lt     the range AND v1 * 3 + v3 < 1500   (long arithmetic, the int32 v3 widened)
  v2_div_v4_gt   the range AND v2 / v4 > 100.0      (double division; null where v4 is 0)
Every query reports ms per query and rows out per query, and from one separate profiled pass the per-kernel ms per query
(k_expr_mask among them).  Before timing, each query runs on a --check-rows table and is compared with numpy.  The
card's name and power limit are read in the same run.
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

from bench_filters import card_info  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=500_000_000)
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
    variants = {"c3": [], "v1x3_v3_lt": [([C("v1"), ("literal", 3), ("*",), C("v3"), ("+",)], "<", [("literal", 1500)])],
                "v2_div_v4_gt": [([C("v2"), C("v4"), ("/",)], ">", [("literal", 100.0)])]}

    def run(srcs, q, exprs):
        lo, hi = q
        return ctx.filter_scan_expr(srcs, "k", proj, [("k", lo, False, hi, False)], [], [], exprs)[0]

    # ---- correctness at a small size, against numpy ----------------------------------------------------------------------
    src = ctx.synth_table(0, args.check_rows, 5, n_files=8, row_groups_per_file=2, output=N.HS_OUT_DEVICE)
    small, _ = ctx.create_index(src.as_sources(), ["k"], ["v1", "v2", "v3", "v4"], nb, output=N.HS_OUT_DEVICE, job_uuid="c")
    src.free()
    cols = O.synthetic_table(0, args.check_rows, 5)
    k = cols["k"]
    wide = (-(2**62), 2**62)  # half of k's range: enough rows at the check size
    with np.errstate(all="ignore"):  # long arithmetic wraps, as Spark's does; a zero divisor is null, so never true
        v4 = cols["v4"].astype(np.float64)
        in_numpy = {"c3": True, "v1x3_v3_lt": cols["v1"] * np.int64(3) + cols["v3"].astype(np.int64) < 1500,
                    "v2_div_v4_gt": (v4 != 0) & (cols["v2"] / np.where(v4 != 0, v4, 1.0) > 100.0)}
    for name, cmps in variants.items():
        m = (k >= wide[0]) & (k <= wide[1]) & in_numpy[name]
        b = run(small.as_sources(), wide, cmps)
        got = np.sort(b.column("k").astype(np.int64))
        b.free()
        assert np.array_equal(got, np.sort(k[m])), name
        print(json.dumps({"check": name, "rows": int(m.sum()), "ok": True}), flush=True)
    small.free()
    ctx.trim()

    # ---- the C3 index ---------------------------------------------------------------------------------------------------
    src = ctx.synth_table(0, args.rows, 5, n_files=256, row_groups_per_file=4, output=N.HS_OUT_DEVICE)
    idx, _ = ctx.create_index(src.as_sources(), ["k"], ["v1", "v2", "v3", "v4"], nb, output=N.HS_OUT_DEVICE, job_uuid="t")
    src.free()
    ctx.trim()
    srcs = idx.as_sources()

    def timed(cmps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record(stream)
        rows = 0
        for q in ranges:
            b = run(srcs, q, cmps)
            rows += b.num_rows
            b.free()
        e1.record(stream)
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / len(ranges), rows / len(ranges)

    for cmps in variants.values():  # warm every shape
        run(srcs, ranges[0], cmps).free()
    ms = {name: [] for name in variants}
    rows = {}
    for _ in range(args.reps):  # alternating, so that clocks and temperature drift hit every query alike
        for name, cmps in variants.items():
            t, rows[name] = timed(cmps)
            ms[name].append(round(t, 3))
    for name, cmps in variants.items():
        ctx.profile_enable(True)
        ctx.profile_report()
        for q in ranges:
            run(srcs, q, cmps).free()
        rep = ctx.profile_report()
        ctx.profile_enable(False)
        kern = {kn: round(v["ms"] / len(ranges), 4) for kn, v in sorted(rep.items(), key=lambda kv: -kv[1]["ms"])}
        print(json.dumps({"workload": name, "exprs": [str(c) for c in cmps], "ms_per_query": ms[name],
                          "rows_out_per_query": rows[name], "profiled_kernel_ms_per_query": kern, **info}), flush=True)
    idx.free()
    ctx.close()


if __name__ == "__main__":
    t0 = time.perf_counter()
    main()
    print(json.dumps({"wall_s": round(time.perf_counter() - t0, 1)}), file=sys.stderr)
