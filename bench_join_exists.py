#!/usr/bin/env python
"""bench_join_exists.py -- left semi and left anti bucket joins on the C4 shape, on ONE GPU: rows [0, N) of table T (L)
against rows [N/2, 3N/2) (R), N = 250 M, 200 buckets, both indexes resident in HBM; results are copied back to the host
inside the timed region.

  inner  k = k via hs_bucket_join_cmp, SELECT L.v1            (k_join_count + scan + k_join_emit)
  semi   EXISTS (R.k = L.k) via hs_bucket_join_exists, SELECT L.v1      (k_join_exists + scan + compaction)
  anti   NOT EXISTS (R.k = L.k) via hs_bucket_join_exists, SELECT L.v1

k is a bijection of the row, so each of the three outputs L's rows [N/2, N) or [0, N/2): 125 M rows.  The three alternate
inside one process, --reps runs each.  For each it reports ms per query, rows out and, from one separate profiled pass,
per-kernel ms and launches.  Before timing, every workload is run at --check-rows rows and its row count and the
checksum of v1 compared with numpy (oracle.synthetic_table).  The card's name and power limit are read in the same run.
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
        L, R = build(0, rows, ["v1"]), build(rows // 2, rows, [])
        lf, lb, rf, rb = L.as_sources(), [f.bucket for f in L.files], R.as_sources(), [f.bucket for f in R.files]
        run = {
            "inner": lambda: ctx.bucket_join_cmp(lf, lb, rf, rb, nb, ["k"], ["k"], ["v1"], []),
            "semi": lambda: ctx.bucket_join_exists(lf, lb, rf, rb, nb, ["k"], ["k"], ["v1"], "semi"),
            "anti": lambda: ctx.bucket_join_exists(lf, lb, rf, rb, nb, ["k"], ["k"], ["v1"], "anti"),
        }
        return L, R, run

    def checksum(a):
        return int(np.asarray(a).view(np.uint64).sum(dtype=np.uint64))

    # ---- correctness at a reduced size --------------------------------------------------------------------------------
    n = args.check_rows
    T = O.synthetic_table(0, n, 5)
    want = {"inner": np.arange(n // 2, n), "semi": np.arange(n // 2, n), "anti": np.arange(0, n // 2)}
    L, R, run = runners(n)
    for name, r in run.items():
        b, _ = r()
        rows = want[name]
        ok = b.num_rows == len(rows) and checksum(b.column("v1")) == checksum(T["v1"][rows])
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
    assert out["inner"] == out["semi"] == out["anti"] == args.rows // 2, out
    desc = {"inner": "k = k via hs_bucket_join_cmp, SELECT L.v1",
            "semi": "EXISTS (R.k = L.k) via hs_bucket_join_exists, SELECT L.v1",
            "anti": "NOT EXISTS (R.k = L.k) via hs_bucket_join_exists, SELECT L.v1"}
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
