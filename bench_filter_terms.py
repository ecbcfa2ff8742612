#!/usr/bin/env python
"""bench_filter_terms.py -- NOT, null-safe equality and string patterns (hs_filter_scan_any term flags) on ONE GPU.

Over the 500 M-row, 200-bucket index of table T on k, built as bench_filters.py builds it:
  (a) `k != x` inside C3's 1 % range of k, against C3 alone: the complement of a point is two windows per file
  (b) `~k.isin(10 values)` inside the same range: eleven windows per file
  (c) `k.eqNullSafe(x)` against `k == x`, both with bucket pruning
Over a string-keyed index generated from --seed (--str-rows rows of 16 random lowercase letters, 200 buckets, a 16 B
included column):
  (d) `s.startswith(p)` against `p <= s < succ(p)` through hs_filter_scan_where: the same range
  (e) `s LIKE 'p%q'`: the prefix's windows, then k_pattern_mask over them
  (f) `s.contains(x)` and `s.endswith(x)`: k_pattern_mask over every row
and over a second string index of --long-rows values of 1 024 bytes, (f) again.  (f) reports the value bytes matched per
second, over the call and over k_pattern_mask's time.

Index file images stay resident in HBM; results are copied back to the host inside the timed region.  Each workload runs
its seeded queries --reps times and reports ms per query, rows out per query and, from one separate profiled pass,
per-kernel ms per query.  The card's name and power limit are read in the same run.
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


def string_sources(N, n_rows, width, files, seed):
    """n_rows rows (s: `width` random lowercase letters, v: 16 more) as uncompressed Parquet images, `files` of them."""
    import numpy as np
    import pyarrow as pa
    import pyarrow.parquet as pq

    rng = np.random.default_rng(seed)
    out, per = [], -(-n_rows // files)
    for f in range(files):
        n = min(per, n_rows - f * per)
        cols = {}
        for name, w in (("s", width), ("v", 16)):
            data = rng.integers(97, 123, n * w, dtype=np.uint8)
            offs = np.arange(0, n * w + 1, w, dtype=np.int32)
            cols[name] = pa.Array.from_buffers(pa.string(), n, [None, pa.py_buffer(offs), pa.py_buffer(data)])
        sink = io.BytesIO()
        pq.write_table(pa.table(cols), sink, compression="NONE", row_group_size=1 << 20)
        out.append(N.FileImage(path=f"s{f}.parquet", data=sink.getvalue()))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=500_000_000)
    ap.add_argument("--str-rows", type=int, default=50_000_000)
    ap.add_argument("--long-rows", type=int, default=2_000_000)
    ap.add_argument("--queries", type=int, default=10)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--seed", type=int, default=2024)
    args = ap.parse_args()
    import numpy as np
    import torch

    from hyperspace_b200 import _native as N
    from hyperspace_b200._native import (HS_TERM_CONTAINS, HS_TERM_ENDS_WITH, HS_TERM_LIKE, HS_TERM_NOT, HS_TERM_NULL_FALSE,
                                         HS_TERM_STARTS_WITH)

    stream = torch.cuda.current_stream()
    ctx = N.Context(0, stream.cuda_stream)
    nb = 200
    info = card_info()
    print(json.dumps({"device": torch.cuda.get_device_name(0), **info}), flush=True)
    rng = np.random.default_rng(args.seed)

    def timed(run, qs):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record(stream)
        rows = 0
        for q in qs:
            b = run(q)
            rows += b.num_rows
            b.free()
        e1.record(stream)
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / 1e3, rows

    def profiled(run, qs):
        ctx.profile_enable(True)
        ctx.profile_report()
        for q in qs:
            run(q).free()
        rep = ctx.profile_report()
        ctx.profile_enable(False)
        return {k: round(v["ms"] / len(qs), 4) for k, v in sorted(rep.items(), key=lambda kv: -kv[1]["ms"])}

    def measure(name, config, run, qs, value_bytes=None):
        run(qs[0]).free()  # warm the shape
        secs, rows = [], 0
        for _ in range(args.reps):
            s, rows = timed(run, qs)
            secs.append(s)
        q = len(qs)
        kern = profiled(run, qs)
        extra = {}
        if value_bytes:  # bytes of the values the matcher reads per query, over the call and over k_pattern_mask
            extra["value_GB_per_s"] = [round(value_bytes * q / s / 1e9, 1) for s in secs]
            if kern.get("k_pattern_mask"):
                extra["k_pattern_mask_value_GB_per_s"] = round(value_bytes / (kern["k_pattern_mask"] / 1e3) / 1e9, 1)
        print(json.dumps({"workload": name, "config": config, "ms_per_query": [round(s * 1e3 / q, 3) for s in secs],
                          "rows_out_per_query": rows / q, "profiled_kernel_ms_per_query": kern, **extra, **info}), flush=True)

    # ---- table T on k ------------------------------------------------------------------------------------------------
    src = ctx.synth_table(0, args.rows, 5, n_files=256, row_groups_per_file=4, output=N.HS_OUT_DEVICE)
    idx, _ = ctx.create_index(src.as_sources(), ["k"], ["v1", "v2", "v3"], nb, output=N.HS_OUT_DEVICE, job_uuid="t")
    src.free()
    ctx.trim()
    srcs, buckets = idx.as_sources(), [f.bucket for f in idx.files]
    proj = ["k", "v1", "v2"]
    width = int(0.01 * 2**64)
    c3 = [(-(width // 2) + i * (width // 40), (width // 2) + i * (width // 40)) for i in range(args.queries)]
    present = []
    for lo, hi in c3:
        b, _ = ctx.filter_scan_where(srcs, "k", ["k"], [("k", lo, False, hi, False)])
        ks = b.column("k")
        present.append(ks[rng.integers(0, len(ks), 10)].astype(np.int64))
        b.free()
    qs = list(zip(c3, present))

    def rng_pred(q):
        return [("k", q[0][0], False, q[0][1], False)]

    c3_run = lambda q: ctx.filter_scan_where(srcs, "k", proj, rng_pred(q))[0]  # noqa: E731
    ne_run = lambda q: ctx.filter_scan_any(srcs, "k", proj, rng_pred(q), [("k", q[1][:1], [], HS_TERM_NOT)])[0]  # noqa: E731
    nin_run = lambda q: ctx.filter_scan_any(srcs, "k", proj, rng_pred(q), [("k", q[1], [], HS_TERM_NOT)])[0]  # noqa: E731
    b0, b1 = c3_run(qs[0]), ne_run(qs[0])
    assert b0.num_rows - b1.num_rows == int((b0.column("k") == qs[0][1][0]).sum()) >= 1
    b0.free()
    b1.free()
    measure("a_c3", "C3: one 1% range of k", c3_run, qs)
    measure("a_ne", "k != x inside the 1% range (x present)", ne_run, qs)
    measure("b_not_in", "~k.isin(10 present values) inside the 1% range", nin_run, qs)
    points = [int(p[0]) for p in present]
    eq_run = lambda x: ctx.filter_scan_any(srcs, "k", proj, [], [("k", [x], [])], file_buckets=buckets, num_buckets=nb)[0]  # noqa: E731
    ens_run = lambda x: ctx.filter_scan_any(srcs, "k", proj, [], [("k", [x], [], HS_TERM_NULL_FALSE)], file_buckets=buckets,  # noqa: E731
                                            num_buckets=nb)[0]
    measure("c_eq", "k == x, pruned by bucket", eq_run, points)
    measure("c_eq_null_safe", "k <=> x, pruned by bucket", ens_run, points)
    idx.free()
    ctx.trim()

    # ---- string keys -------------------------------------------------------------------------------------------------
    def string_index(n_rows, width, files, tag):
        sources = string_sources(N, n_rows, width, files, args.seed)
        res, _ = ctx.create_index(sources, ["s"], ["v"], nb, output=N.HS_OUT_DEVICE, job_uuid=tag)
        ctx.trim()
        return res

    sidx = string_index(args.str_rows, 16, 50, "s")
    ssrc = sidx.as_sources()
    letters = [bytes([97 + int(a), 97 + int(b)]) for a, b in rng.integers(0, 26, (args.queries, 2))]
    succ = [p[:-1] + bytes([p[-1] + 1]) for p in letters]
    sw_run = lambda p: ctx.filter_scan_any(ssrc, "s", ["s", "v"], [], [("s", [p], [], HS_TERM_STARTS_WITH)])[0]  # noqa: E731
    bt_run = lambda i: ctx.filter_scan_where(ssrc, "s", ["s", "v"], [("s", letters[i], False, succ[i], True)])[0]  # noqa: E731
    b0, b1 = sw_run(letters[0]), bt_run(0)
    assert b0.num_rows == b1.num_rows > 0 and list(b0.column("s")) == list(b1.column("s"))
    b0.free()
    b1.free()
    measure("d_startswith", "s.startswith(2 letters)", sw_run, letters)
    measure("d_between", "2-letter prefix as p <= s < succ(p)", bt_run, list(range(args.queries)))
    likes = [p + b"%" + bytes([97 + int(c)]) for p, c in zip(letters, rng.integers(0, 26, args.queries))]
    measure("e_like", "s LIKE 'pp%q'", lambda p: ctx.filter_scan_any(ssrc, "s", ["s", "v"], [], [("s", [p], [], HS_TERM_LIKE)])[0], likes)
    subs = [bytes(97 + x for x in rng.integers(0, 26, 3)) for _ in range(args.queries)]
    for tag, flag in (("contains", HS_TERM_CONTAINS), ("endswith", HS_TERM_ENDS_WITH)):
        run = lambda x, flag=flag: ctx.filter_scan_any(ssrc, "s", ["s", "v"], [], [("s", [x], [], flag)])[0]  # noqa: E731
        measure(f"f_{tag}_16B", f"s.{tag}(3 letters) over {args.str_rows} values of 16 B", run, subs, value_bytes=16 * args.str_rows)
    sidx.free()
    ctx.trim()
    lidx = string_index(args.long_rows, 1024, 8, "l")
    lsrc = lidx.as_sources()
    for tag, flag in (("contains", HS_TERM_CONTAINS), ("endswith", HS_TERM_ENDS_WITH)):
        run = lambda x, flag=flag: ctx.filter_scan_any(lsrc, "s", ["v"], [], [("s", [x], [], flag)])[0]  # noqa: E731
        measure(f"f_{tag}_1KB", f"s.{tag}(3 letters) over {args.long_rows} values of 1 KB", run, subs, value_bytes=1024 * args.long_rows)
    lidx.free()
    ctx.close()


if __name__ == "__main__":
    t0 = time.perf_counter()
    main()
    print(json.dumps({"wall_s": round(time.perf_counter() - t0, 1)}), file=sys.stderr)
