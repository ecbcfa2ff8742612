#!/usr/bin/env python
"""bench_filters.py -- filter scans with conjunctions of predicates over the 500 M-row, 200-bucket index of table T, on ONE
GPU.  Index file images stay resident in HBM; results are copied back to the host inside the timed region.

  (a) C3 of bench_queries.py through hs_filter_scan: `k BETWEEN lo AND hi` (1 % of the int64 key space), project k, v1, v2
  (b) the same ranges through hs_filter_scan_where with only the key predicate
  (c) (b) AND v1 < 500 AND v3 BETWEEN 10 AND 59, project k, v1, v2 (about a quarter of (b)'s rows; k_predicate_mask runs
      over the window rows)
  (d) an index keyed on v2 (double), `v2 BETWEEN lo AND hi` with 1 % selectivity, project v2, k

Each workload runs its 20 seeded ranges --reps times; (a) and (b) alternate inside one process so that their difference
is not a difference between processes.  For each it reports queries/s, rows out per query and, from one separate
profiled pass, the k_predicate_mask time per query.  The card's name and power limit are read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)


def card_info():
    out = {}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        name, power = [x.strip() for x in q.split(",")]
        out = {"card": name, "power_limit": power}
    except Exception as e:  # noqa: BLE001 -- reported, not hidden
        out = {"card": "unknown", "power_limit": f"not read ({e})"}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=500_000_000)
    ap.add_argument("--queries", type=int, default=20)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--seed", type=int, default=2024)
    args = ap.parse_args()
    import numpy as np
    import torch

    from hyperspace_b200 import _native as N

    stream = torch.cuda.current_stream()
    ctx = N.Context(0, stream.cuda_stream)
    nb, files = 200, 256
    info = card_info()
    print(json.dumps({"device": torch.cuda.get_device_name(0), **info}))

    def build(key, included):
        src = ctx.synth_table(0, args.rows, 5, n_files=files, row_groups_per_file=4, output=N.HS_OUT_DEVICE)
        idx, _ = ctx.create_index(src.as_sources(), [key], included, nb, output=N.HS_OUT_DEVICE, job_uuid="f")
        src.free()
        ctx.trim()
        return idx

    def timed(run, ranges):
        """seconds for all ranges, rows out in total (device events around the loop; every call ends in a synchronise)."""
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record(stream)
        rows = 0
        for r in ranges:
            b, _ = run(r)
            rows += b.num_rows
            b.free()
        e1.record(stream)
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / 1e3, rows

    def mask_ms(run, ranges):
        ctx.profile_enable(True)
        ctx.profile_report()  # reset
        for r in ranges:
            run(r)[0].free()
        rep = ctx.profile_report()
        ctx.profile_enable(False)
        b, st = run(ranges[0])
        b.free()
        per_kernel = {k: round(v["ms"] / len(ranges), 4) for k, v in sorted(rep.items(), key=lambda kv: -kv[1]["ms"])}
        return (rep.get("k_predicate_mask", {}).get("ms", 0.0) / len(ranges), rep.get("k_range_bounds", {}).get("ms", 0.0) / len(ranges),
                per_kernel, int(st["gpu_launches"]))

    def report(name, workload, secs, rows, mms, rbms, per_kernel, launches):
        q = args.queries
        print(json.dumps({"workload": name, "config": workload, "queries_per_s": [round(q / s, 2) for s in secs],
                          "ms_per_query": [round(s * 1e3 / q, 3) for s in secs], "rows_out_per_query": rows / q,
                          "k_predicate_mask_ms_per_query": round(mms, 4), "k_range_bounds_ms_per_query": round(rbms, 4),
                          "gpu_launches_per_query": launches, "profiled_kernel_ms_per_query": per_kernel,
                          "rows": args.rows, "n_gpus": 1, **info}))

    # ---- (a), (b), (c): index on k ------------------------------------------------------------------------------------
    idx = build("k", ["v1", "v2", "v3"])
    srcs = idx.as_sources()
    width = int(0.01 * 2**64)
    ranges = [(-(width // 2) + i * (width // 40), (width // 2) + i * (width // 40)) for i in range(args.queries)]
    proj = ["k", "v1", "v2"]
    run_a = lambda r: ctx.filter_scan(srcs, "k", proj, lo=r[0], hi=r[1])  # noqa: E731
    run_b = lambda r: ctx.filter_scan_where(srcs, "k", proj, [("k", r[0], False, r[1], False)])  # noqa: E731
    run_c = lambda r: ctx.filter_scan_where(srcs, "k", proj, [("k", r[0], False, r[1], False), ("v1", None, False, 500, True),  # noqa: E731
                                                              ("v3", 10, False, 59, False)])
    for run in (run_a, run_b, run_c):  # warm every shape
        run(ranges[0])[0].free()
    # same answers: (a) and (b) row for row, (c) the subset the numpy filter keeps
    ba, _ = run_a(ranges[3])
    bb, _ = run_b(ranges[3])
    bc, _ = run_c(ranges[3])
    assert ba.num_rows == bb.num_rows and all(x.tobytes() == y.tobytes() for (_, x, _), (_, y, _) in zip(ba.columns, bb.columns))
    bf, _ = ctx.filter_scan_where(srcs, "k", proj + ["v3"], [("k", ranges[3][0], False, ranges[3][1], False)])
    v1, v3 = bf.column("v1"), bf.column("v3")
    keep = (v1 < 500) & (v3 >= 10) & (v3 <= 59)
    assert bc.num_rows == int(keep.sum()) and np.array_equal(bc.column("k"), bf.column("k")[keep])
    for b in (ba, bb, bc, bf):
        b.free()
    secs_a, secs_b, secs_c = [], [], []
    rows_a = rows_b = rows_c = 0
    for _ in range(args.reps):
        s, rows_a = timed(run_a, ranges)
        secs_a.append(s)
        s, rows_b = timed(run_b, ranges)
        secs_b.append(s)
    for _ in range(args.reps):
        s, rows_c = timed(run_c, ranges)
        secs_c.append(s)
    assert rows_a == rows_b
    report("a", "C3 via hs_filter_scan: k BETWEEN lo AND hi (1% of key space), project k,v1,v2", secs_a, rows_a, *mask_ms(run_a, ranges))
    report("b", "C3 ranges via hs_filter_scan_where, key predicate only", secs_b, rows_b, *mask_ms(run_b, ranges))
    report("c", "(b) AND v1 < 500 AND v3 BETWEEN 10 AND 59, project k,v1,v2", secs_c, rows_c, *mask_ms(run_c, ranges))
    idx.free()
    ctx.trim()
    # ---- (d): index on v2 (double) -----------------------------------------------------------------------------------
    idx = build("v2", ["k", "v1"])
    srcs = idx.as_sources()
    rng = np.random.default_rng(args.seed)
    top = args.rows * 1e-3  # v2 = row * 1e-3
    w = 0.01 * top
    dr = [(float(lo), float(lo + w)) for lo in rng.uniform(0, top - w, args.queries)]
    run_d = lambda r: ctx.filter_scan_where(srcs, "v2", ["v2", "k"], [("v2", r[0], False, r[1], False)])  # noqa: E731
    run_d(dr[0])[0].free()
    secs_d, rows_d = [], 0
    for _ in range(args.reps):
        s, rows_d = timed(run_d, dr)
        secs_d.append(s)
    report("d", "index on v2 (double): v2 BETWEEN lo AND hi (1% of rows), project v2,k", secs_d, rows_d, *mask_ms(run_d, dr))
    idx.free()
    ctx.close()


if __name__ == "__main__":
    t0 = time.perf_counter()
    main()
    print(json.dumps({"wall_s": round(time.perf_counter() - t0, 1)}), file=sys.stderr)
