#!/usr/bin/env python
"""bench_join_outer.py -- left, right and full outer bucket joins on the C4 shape, on ONE GPU: rows [0, N) of table T (L)
against rows [N/2, 3N/2) (R), N = 250 M, 200 buckets, both indexes resident in HBM; results are copied back to the host
inside the timed region.

  inner  k = k via hs_bucket_join_cmp, SELECT L.v1, R.v2                   (k_join_count + scan + k_join_emit)
  left   L LEFT OUTER JOIN R via hs_bucket_join_outer, SELECT L.v1, R.v2   (k_join_count_outer + scan + k_join_emit_outer)
  right  L RIGHT OUTER JOIN R, SELECT L.v1, R.v2
  full   L FULL OUTER JOIN R, SELECT L.v1, R.v2     (+ k_join_exists, compaction and k_join_place_unmatched)

k is a bijection of the row, so the inner join outputs the N/2 rows of the overlap, the left and right outer joins N rows
(N/2 of them padded) and the full outer join 3N/2.  The four alternate inside one process, --reps runs each.  For each it
reports ms per query, rows out and, from one separate profiled pass, per-kernel ms and launches.  Before timing, every
workload is run at --check-rows rows and its row count, valid counts and the checksums of v1 and v2 compared with numpy
(oracle.synthetic_table).  The card's name and power limit are read in the same run.
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

from bench_joins import card_info  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=250_000_000)
    ap.add_argument("--check-rows", type=int, default=2_000_000)
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    import numpy as np
    import torch

    from hyperspace_b200 import _native as N
    from oracle import oracle as O

    stream = torch.cuda.current_stream()
    ctx = N.Context(0, stream.cuda_stream)
    nb, files = 200, 256
    info = card_info()
    print(json.dumps({"device": torch.cuda.get_device_name(0), **info}))

    def build(first, rows, included):
        src = ctx.synth_table(first, rows, 5, n_files=files, row_groups_per_file=4, output=N.HS_OUT_DEVICE)
        idx, _ = ctx.create_index(src.as_sources(), ["k"], included, nb, output=N.HS_OUT_DEVICE, job_uuid="j")
        src.free()
        ctx.trim()
        return idx

    def runners(rows):
        L, R = build(0, rows, ["v1"]), build(rows // 2, rows, ["v2"])
        lf, lb, rf, rb = L.as_sources(), [f.bucket for f in L.files], R.as_sources(), [f.bucket for f in R.files]
        run = {"inner": lambda: ctx.bucket_join_cmp(lf, lb, rf, rb, nb, ["k"], ["k"], ["v1"], ["v2"])}
        for how in ("left", "right", "full"):
            run[how] = (lambda h: lambda: ctx.bucket_join_outer(lf, lb, rf, rb, nb, ["k"], ["k"], ["v1"], ["v2"], h))(how)
        return L, R, run

    def checksum(a, valid):
        a = np.asarray(a).view(np.uint64)
        return int((a if valid is None else a[np.asarray(valid) != 0]).sum(dtype=np.uint64))

    # ---- correctness at a reduced size --------------------------------------------------------------------------------
    n = args.check_rows
    T = O.synthetic_table(0, n + n // 2, 5)
    # the L rows and the R rows (global row numbers of T) each workload outputs
    want = {"inner": (np.arange(n // 2, n), np.arange(n // 2, n)), "left": (np.arange(0, n), np.arange(n // 2, n)),
            "right": (np.arange(n // 2, n), np.arange(n // 2, n + n // 2)), "full": (np.arange(0, n), np.arange(n // 2, n + n // 2))}
    total = {"inner": n // 2, "left": n, "right": n, "full": n + n // 2}
    L, R, run = runners(n)
    for name, r in run.items():
        b, _ = r()
        (_, v1, m1), (_, v2, m2) = b.columns
        lrows, rrows = want[name]
        ok = (b.num_rows == total[name]
              and (len(v1) if m1 is None else int(m1.sum())) == len(lrows) and (len(v2) if m2 is None else int(m2.sum())) == len(rrows)
              and checksum(v1, m1) == checksum(T["v1"][lrows], None) and checksum(v2, m2) == checksum(T["v2"][rrows], None))
        print(json.dumps({"check": name, "rows": n, "rows_out": int(b.num_rows), "ok": bool(ok)}))
        assert ok, name
        b.free()
    L.free()
    R.free()
    ctx.trim()

    # ---- timed runs on the C4 shape -----------------------------------------------------------------------------------
    def timed(r):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record(stream)
        b, st = r()
        rows = b.num_rows
        b.free()
        e1.record(stream)
        torch.cuda.synchronize()
        return e0.elapsed_time(e1), rows, st

    def profiled(r):
        ctx.profile_enable(True)
        ctx.profile_report()  # reset
        b, _ = r()
        b.free()
        rep = ctx.profile_report()
        ctx.profile_enable(False)
        return {k: {"ms": round(v["ms"], 3), "launches": v["launches"]} for k, v in sorted(rep.items(), key=lambda kv: -kv[1]["ms"])}

    L, R, run = runners(args.rows)
    for r in run.values():
        r()[0].free()  # warm every shape
    ms = {k: [] for k in run}
    out, stats = {}, {}
    for _ in range(args.reps):
        for k, r in run.items():
            t, out[k], stats[k] = timed(r)
            ms[k].append(t)
    h = args.rows // 2
    assert (out["inner"], out["left"], out["right"], out["full"]) == (h, 2 * h, 2 * h, 3 * h), out
    desc = {"inner": "k = k via hs_bucket_join_cmp, SELECT L.v1, R.v2",
            "left": "L LEFT OUTER JOIN R ON k via hs_bucket_join_outer, SELECT L.v1, R.v2",
            "right": "L RIGHT OUTER JOIN R ON k via hs_bucket_join_outer, SELECT L.v1, R.v2",
            "full": "L FULL OUTER JOIN R ON k via hs_bucket_join_outer, SELECT L.v1, R.v2"}
    for k, r in run.items():
        print(json.dumps({"workload": k, "config": desc[k], "ms_per_query": [round(x, 2) for x in ms[k]], "rows_out": out[k],
                          "ms_probe": round(stats[k]["ms_sort"], 3), "gpu_launches": int(stats[k]["gpu_launches"]),
                          "profiled_kernels": profiled(r), "rows_per_side": args.rows, "buckets": nb, "n_gpus": 1, **info}))
    L.free()
    R.free()
    ctx.close()


if __name__ == "__main__":
    t0 = time.perf_counter()
    main()
    print(json.dumps({"wall_s": round(time.perf_counter() - t0, 1)}), file=sys.stderr)
