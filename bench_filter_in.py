#!/usr/bin/env python
"""bench_filter_in.py -- IN lists and OR-ed ranges (hs_filter_scan_any) over the 500 M-row, 200-bucket index of table T
on k, on ONE GPU, built as bench_filters.py builds it.  Index file images stay resident in HBM; results are copied back to
the host inside the timed region.

  (a) `k IN (list)` of 1, 10, 1 000 and 100 000 keys, half of them taken from the index's own rows and half absent,
      with bucket pruning (the files' bucket ids from the build)
  (b) the 10-key list three ways: ten `k == v` calls through hs_filter_scan_where (what a user had before), one call
      without file_buckets, one call with them
  (c) an OR of four disjoint 0.25 % ranges of k, against C3's single 1 % range through hs_filter_scan_where
  (d) `v3 IN (1 000 values)` inside C3's windows: the set-form residual of k_predicate_mask

Each workload runs its seeded queries --reps times and reports queries/s, ms per query, rows out per query and, from one
separate profiled pass, per-kernel ms per query.  The card's name and power limit are read in the same run.
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
    ap.add_argument("--queries", type=int, default=10)
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
    src = ctx.synth_table(0, args.rows, 5, n_files=files, row_groups_per_file=4, output=N.HS_OUT_DEVICE)
    idx, _ = ctx.create_index(src.as_sources(), ["k"], ["v1", "v2", "v3"], nb, output=N.HS_OUT_DEVICE, job_uuid="f")
    src.free()
    ctx.trim()
    srcs = idx.as_sources()
    buckets = [f.bucket for f in idx.files]
    proj = ["k", "v1", "v2"]
    rng = np.random.default_rng(args.seed)
    width = int(0.01 * 2**64)
    c3 = [(-(width // 2) + i * (width // 40), (width // 2) + i * (width // 40)) for i in range(args.queries)]
    # keys of the index's own rows: the output of one C3 range scan
    b, _ = ctx.filter_scan_where(srcs, "k", ["k"], [("k", c3[0][0], False, c3[0][1], False)])
    present = b.column("k").copy()
    b.free()

    def key_list(n):
        have = present[rng.integers(0, len(present), (n + 1) // 2)]
        absent = rng.integers(-2**62, 2**62, n // 2)  # 2^-64 of the key space per row: practically never present
        return np.concatenate([have, absent]).astype(np.int64)

    def timed(run, qs):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record(stream)
        rows = 0
        for q in qs:
            for bb in run(q):
                rows += bb.num_rows
                bb.free()
        e1.record(stream)
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / 1e3, rows

    def profiled(run, qs):
        ctx.profile_enable(True)
        ctx.profile_report()
        for q in qs:
            for bb in run(q):
                bb.free()
        rep = ctx.profile_report()
        ctx.profile_enable(False)
        return {k: round(v["ms"] / len(qs), 4) for k, v in sorted(rep.items(), key=lambda kv: -kv[1]["ms"])}

    def measure(name, config, run, qs, extra=None):
        for bb in run(qs[0]):  # warm the shape
            bb.free()
        secs, rows = [], 0
        for _ in range(args.reps):
            s, rows = timed(run, qs)
            secs.append(s)
        q = len(qs)
        print(json.dumps({"workload": name, "config": config, "queries_per_s": [round(q / s, 2) for s in secs],
                          "ms_per_query": [round(s * 1e3 / q, 3) for s in secs], "rows_out_per_query": rows / q,
                          "profiled_kernel_ms_per_query": profiled(run, qs), "rows": args.rows, "n_gpus": 1, **(extra or {}),
                          **info}), flush=True)

    def one(b_st):
        return [b_st[0]]

    pruned = lambda keys: one(ctx.filter_scan_any(srcs, "k", proj, [], [("k", keys, [])], file_buckets=buckets, num_buckets=nb))  # noqa: E731
    unpruned = lambda keys: one(ctx.filter_scan_any(srcs, "k", proj, [], [("k", keys, [])]))  # noqa: E731
    # ---- (a) -------------------------------------------------------------------------------------------------------
    for n in (1, 10, 1000, 100_000):
        qs = [key_list(n) for _ in range(args.queries)]
        _, st = ctx.filter_scan_any(srcs, "k", proj, [], [("k", qs[0], [])], file_buckets=buckets, num_buckets=nb)
        measure(f"a{n}", f"k IN ({n} keys, half present), pruned by bucket", pruned, qs, {"bytes_in_per_query": st["bytes_in"]})
    # ---- (b) -------------------------------------------------------------------------------------------------------
    qs = [key_list(10) for _ in range(args.queries)]
    eq = lambda keys: [ctx.filter_scan_where(srcs, "k", proj, [("k", int(v), False, int(v), False)])[0] for v in keys]  # noqa: E731
    got = [bb.num_rows for bb in eq(qs[0])]
    bp, bu = pruned(qs[0])[0], unpruned(qs[0])[0]
    assert bp.num_rows == bu.num_rows == sum(got) and all(x.tobytes() == y.tobytes() for (_, x, _), (_, y, _) in zip(bp.columns, bu.columns))
    bp.free()
    bu.free()
    measure("b_eq", "10 keys as 10 `k == v` calls through hs_filter_scan_where", eq, qs)
    measure("b_unpruned", "10-key IN list, one call without file_buckets", unpruned, qs)
    measure("b_pruned", "10-key IN list, one call with file_buckets", pruned, qs)
    # ---- (c) -------------------------------------------------------------------------------------------------------
    q4 = width // 4

    def four(r):
        lo = r[0]
        return [(lo + 2 * i * q4, False, lo + (2 * i + 1) * q4, True) for i in range(4)]  # every other quarter-width

    or4 = lambda r: one(ctx.filter_scan_any(srcs, "k", proj, [], [("k", [], four(r))]))  # noqa: E731
    c3r = lambda r: one(ctx.filter_scan_where(srcs, "k", proj, [("k", r[0], False, r[1], False)]))  # noqa: E731
    measure("c_or4", "OR of four disjoint 0.25% ranges of k", or4, c3)
    measure("c_c3", "C3: one 1% range of k through hs_filter_scan_where", c3r, c3)
    # ---- (d) -------------------------------------------------------------------------------------------------------
    v3s = [np.sort(rng.choice(1000, 1000, replace=True)).astype(np.int64) for _ in range(args.queries)]
    dq = list(zip(c3, v3s))
    d_run = lambda q: one(ctx.filter_scan_any(srcs, "k", proj, [("k", q[0][0], False, q[0][1], False)], [("v3", q[1], [])]))  # noqa: E731
    measure("d", "C3 window AND v3 IN (1000 values): set-form residual", d_run, dq)
    idx.free()
    ctx.close()


if __name__ == "__main__":
    t0 = time.perf_counter()
    main()
    print(json.dumps({"wall_s": round(time.perf_counter() - t0, 1)}), file=sys.stderr)
