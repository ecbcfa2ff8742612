#!/usr/bin/env python
"""bench_joins.py -- bucket joins on the C4 shape, on ONE GPU: rows [0, N) of table T joined with rows [N/2, 3N/2), N = 250 M,
200 buckets, both indexes resident in HBM; results are copied back to the host inside the timed region.

  (1) one key, k = k, SELECT L.v1, R.v2, through hs_bucket_join and through hs_bucket_join_where, alternating
  (2) two key columns (k, v3) = (k, v3): v3 = row % 100 is a function of the row like k, so the pairs and the 125 M-row
      output are those of (1); the indexes are built on (k, v3) and k_join_count compares both columns
  (3) one key with a filter below each side: L.v3 < 10 and R.v1 < 100 (about 10 % of each side)

Each workload runs --reps times; (1)'s two entry points alternate inside one process.  For each it reports ms per join,
rows out and, from one separate profiled pass, per-kernel ms and launches.  Before timing, every workload is run at
--check-rows rows and its row count and column checksums compared with numpy (oracle.synthetic_table).  The card's name
and power limit are read in the same run.
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
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        name, power = [x.strip() for x in q.split(",")]
        return {"card": name, "power_limit": power}
    except Exception as e:  # noqa: BLE001 -- reported, not hidden
        return {"card": "unknown", "power_limit": f"not read ({e})"}


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

    def build(first, rows, keys, included):
        src = ctx.synth_table(first, rows, 5, n_files=files, row_groups_per_file=4, output=N.HS_OUT_DEVICE)
        idx, _ = ctx.create_index(src.as_sources(), keys, included, nb, output=N.HS_OUT_DEVICE, job_uuid="j")
        src.free()
        ctx.trim()
        return idx

    def sides(rows, keys):
        L = build(0, rows, keys, ["v1", "v3"] if keys == ["k"] else ["v1"])
        R = build(rows // 2, rows, keys, ["v1", "v2"] if keys == ["k"] else ["v2"])
        return L, R, (L.as_sources(), [f.bucket for f in L.files], R.as_sources(), [f.bucket for f in R.files])

    preds3 = ([("v3", None, False, 10, True)], [("v1", None, False, 100, True)])

    def runners(s):
        lf, lb, rf, rb = s
        return {
            "1_hs_bucket_join": lambda: ctx.bucket_join(lf, lb, rf, rb, nb, "k", "k", ["v1"], ["v2"]),
            "1_hs_bucket_join_where": lambda: ctx.bucket_join_where(lf, lb, rf, rb, nb, ["k"], ["k"], ["v1"], ["v2"]),
            "3_predicates": lambda: ctx.bucket_join_where(lf, lb, rf, rb, nb, ["k"], ["k"], ["v1"], ["v2"], *preds3),
        }

    def runners2(s):
        lf, lb, rf, rb = s
        return {"2_two_keys": lambda: ctx.bucket_join_where(lf, lb, rf, rb, nb, ["k", "v3"], ["k", "v3"], ["v1"], ["v2"])}

    def checksum(a):
        return int(np.asarray(a).view(np.uint64).sum(dtype=np.uint64))

    # ---- correctness at a reduced size --------------------------------------------------------------------------------
    n = args.check_rows
    T = O.synthetic_table(0, n + n // 2, 5)
    both = np.arange(n // 2, n)  # rows on both sides: k is a bijection of the row
    want = {"1": both, "2": both, "3": both[(T["v3"][both] < 10) & (T["v1"][both] < 100)]}
    for keys, make in ((["k"], runners), (["k", "v3"], runners2)):
        L, R, s = sides(n, keys)
        for name, run in make(s).items():
            b, _ = run()
            rows = want[name[0]]
            ok = (b.num_rows == len(rows) and checksum(b.column("v1")) == checksum(T["v1"][rows])
                  and checksum(b.column("v2")) == checksum(T["v2"][rows]))
            print(json.dumps({"check": name, "rows": n, "rows_out": int(b.num_rows), "ok": bool(ok)}))
            assert ok, name
            b.free()
        L.free()
        R.free()
        ctx.trim()

    # ---- timed runs on the C4 shape -----------------------------------------------------------------------------------
    def timed(run):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record(stream)
        b, st = run()
        rows = b.num_rows
        b.free()
        e1.record(stream)
        torch.cuda.synchronize()
        return e0.elapsed_time(e1), rows, st

    def profiled(run):
        ctx.profile_enable(True)
        ctx.profile_report()  # reset
        b, st = run()
        b.free()
        rep = ctx.profile_report()
        ctx.profile_enable(False)
        return {k: {"ms": round(v["ms"], 3), "launches": v["launches"]} for k, v in sorted(rep.items(), key=lambda kv: -kv[1]["ms"])}

    def report(name, workload, ms, rows, st, kernels):
        print(json.dumps({"workload": name, "config": workload, "ms_per_join": [round(x, 2) for x in ms], "rows_out": rows,
                          "ms_side_selection": round(st["ms_exchange"], 3), "gpu_launches": int(st["gpu_launches"]),
                          "profiled_kernels": kernels, "rows_per_side": args.rows, "buckets": nb, "n_gpus": 1, **info}))

    L, R, s = sides(args.rows, ["k"])
    run = runners(s)
    for r in run.values():
        r()[0].free()  # warm every shape
    ms = {k: [] for k in run}
    out = {}
    for _ in range(args.reps):  # (1) alternating, then (3)
        for k in ("1_hs_bucket_join", "1_hs_bucket_join_where"):
            t, out[k], st_k = timed(run[k])
            ms[k].append(t)
            out[k + "_st"] = st_k
    for _ in range(args.reps):
        t, out["3_predicates"], out["3_predicates_st"] = timed(run["3_predicates"])
        ms["3_predicates"].append(t)
    assert out["1_hs_bucket_join"] == out["1_hs_bucket_join_where"] == args.rows // 2
    desc = {"1_hs_bucket_join": "k = k via hs_bucket_join, SELECT L.v1, R.v2",
            "1_hs_bucket_join_where": "k = k via hs_bucket_join_where, SELECT L.v1, R.v2",
            "3_predicates": "k = k, L.v3 < 10, R.v1 < 100, SELECT L.v1, R.v2"}
    for k in run:
        report(k, desc[k], ms[k], out[k], out[k + "_st"], profiled(run[k]))
    L.free()
    R.free()
    ctx.trim()
    L, R, s = sides(args.rows, ["k", "v3"])
    run = runners2(s)["2_two_keys"]
    run()[0].free()
    ms2, rows2 = [], 0
    for _ in range(args.reps):
        t, rows2, st2 = timed(run)
        ms2.append(t)
    assert rows2 == args.rows // 2
    report("2_two_keys", "(k, v3) = (k, v3) over indexes on (k, v3), SELECT L.v1, R.v2", ms2, rows2, st2, profiled(run))
    L.free()
    R.free()
    ctx.close()


if __name__ == "__main__":
    t0 = time.perf_counter()
    main()
    print(json.dumps({"wall_s": round(time.perf_counter() - t0, 1)}), file=sys.stderr)
