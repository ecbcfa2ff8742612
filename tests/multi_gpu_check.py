"""Multi-GPU parity check (launch with torchrun, one rank per GPU):

    python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29511 tests/multi_gpu_check.py

Every rank decodes its share of the source files, rows move to the owner of their bucket inside hs_create_index, each
rank encodes the buckets it owns.  At 200 buckets the rows move in the partition kernel itself, stored straight into the
owners' memory over NVLink; at 1500 buckets (above the fused partition's 1024) they go through the NCCL all-to-all.  The union of the per-rank outputs must equal the
oracle's single-process answer bucket by bucket (same keys in the same order; payload compared as a per-key multiset is
not needed: the exchange is stable, so even tie order is the rank-major source order the oracle produces)."""
import os
import sys

import numpy as np
import pyarrow as pa
import pyarrow.parquet as pq
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from hyperspace_b200 import _native as N  # noqa: E402
from hyperspace_b200 import distributed as D  # noqa: E402
from oracle import oracle as O  # noqa: E402


def main():
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    ctx = N.Context(local)
    ctx.comm_init(rank, world, D.broadcast_unique_id(dist, N.Context.comm_unique_id, rank))
    nb, n_files, rows_per_file = 200, 8, 50_000
    my = D.shard_files(list(range(n_files)), rank, world)
    src = ctx.synth_table(my[0] * rows_per_file, len(my) * rows_per_file, 5, n_files=len(my), row_groups_per_file=2,
                          output=N.HS_OUT_DEVICE)
    cols = O.synthetic_table(0, n_files * rows_per_file, 5)

    def build_and_check(nb):
        res, st = ctx.create_index(src.as_sources(), ["k"], ["v1", "v2", "v3", "v4"], nb, output=N.HS_OUT_HOST, job_uuid="mg")
        perm, offs, order = O.index_rows(cols, ["k"], ["v1", "v2", "v3", "v4"], nb)
        owned = set(D.buckets_of_rank(rank, world, nb))
        seen = set()
        for i, f in enumerate(res.files):
            assert f.bucket in owned, (rank, f.bucket)
            t = pq.ParquetFile(pa.BufferReader(res.host_bytes(i))).read()
            lo, hi = int(offs[f.bucket]), int(offs[f.bucket + 1])
            for name in order:
                got, want = t.column(name).to_numpy(), cols[name][perm[lo:hi]]
                assert got.tobytes() == want.tobytes(), (rank, f.bucket, name, nb)
            seen.add(f.bucket)
        assert seen == {b for b in owned if offs[b + 1] > offs[b]}, nb
        return res, st

    res, st = build_and_check(nb)
    build_and_check(1500)[0].free()
    # the staged / asynchronous API on several GPUs: two builds in flight per rank, byte-identical files
    want = {f.name: res.host_bytes(i) for i, f in enumerate(res.files)}
    hsrc = ctx.synth_table(my[0] * rows_per_file, len(my) * rows_per_file, 5, n_files=len(my), row_groups_per_file=2,
                           output=N.HS_OUT_HOST)
    s1 = ctx.stage_sources(hsrc.as_sources())
    s2 = ctx.stage_sources(hsrc.as_sources())
    p1 = ctx.create_index_async(s1.as_sources(), ["k"], ["v1", "v2", "v3", "v4"], nb, output=N.HS_OUT_HOST, job_uuid="mg")
    p2 = ctx.create_index_async(s2.as_sources(), ["k"], ["v1", "v2", "v3", "v4"], nb, output=N.HS_OUT_HOST, job_uuid="mg")
    for p in (p1, p2):
        r, _ = p.wait()
        assert {f.name: r.host_bytes(i) for i, f in enumerate(r.files)} == want, rank
        r.free()
    s1.free()
    s2.free()
    # whole-index verification across ranks: checksums add up to the generator's
    rep = ctx.verify_index(res.as_sources(), [f.bucket for f in res.files], ["k"], ["v1", "v2", "v3", "v4"], nb)
    gen = ctx.synth_checksum(my[0] * rows_per_file, len(my) * rows_per_file, 5)
    allr = [None] * world
    dist.all_gather_object(allr, (rep, gen))
    assert sum(a[0]["bucket_mismatches"] + a[0]["order_violations"] for a in allr) == 0
    assert sum(a[0]["row_checksum"] for a in allr) % 2**64 == sum(a[1]["row_checksum"] for a in allr) % 2**64
    assert sum(a[0]["rows"] for a in allr) == n_files * rows_per_file
    hsrc.free()
    counts = torch.tensor([st["rows_in"], st["rows_out"], st["bytes_exchanged"]], device="cuda", dtype=torch.float64)
    dist.all_reduce(counts)
    if rank == 0:
        assert int(counts[0]) == int(counts[1]) == n_files * rows_per_file
        print(f"multi-gpu parity ok: world={world}, rows={int(counts[0])}, exchanged={int(counts[2])} bytes")
    res.free()
    src.free()
    ctx.close()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
