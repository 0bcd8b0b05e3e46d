"""Snapshots of a map sharded over several PROCESSES (DistShard: CUDA-IPC peer mappings).  Rank 0 also runs one
unsharded context on the same inputs.  Frames: water batch -> floods -> seep pass -> wind batch -> frequency update.
  1. after two frames, the ranks' strip snapshots joined (DistShard.snapshot) equal the one context's snapshot, which
     rank 0 writes to a file;
  2. both run two more frames: the final snapshots (columns and frequency arrays) are A;
  3. every process restores its slice from that file, the two frames run again and must end in A, bit for bit.
Rank 0 prints one line and every process exits non-zero on any difference.

  N GPUs, one rank per GPU:
    python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 --master-port P \
        tests/multigpu_snapshot_check.py [dim] [water particles]
  ONE GPU, N processes sharing it: SM_ONE_GPU=1 in the environment.
"""
import os
import sys
import tempfile

import numpy as np
import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from soilmachine_b200 import capi, presets, host, sharded, snapshot  # noqa: E402

NWIND = 200      # a few hundred wind particles, as the other sharded checks


def main():
    dim = int(sys.argv[1]) if len(sys.argv) > 1 else 96
    n = int(sys.argv[2]) if len(sys.argv) > 2 else 700
    soil = "bigbutte"
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    one_gpu = os.environ.get("SM_ONE_GPU") == "1"
    local = 0 if one_gpu else int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    if one_gpu:
        dist.init_process_group("gloo")
    else:
        dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    pre = presets.load(soil)
    scale = pre["world"]["scale"]
    sh = sharded.DistShard(dim, dim, scale, device=local, max_particles=n, share=world if one_gpu else 1)
    sh.ctx.set_soils(pre["soils"])
    sh.ctx.initialize(42, pre["layers"])
    one = None
    if rank == 0:
        one = capi.Context(dim, dim, scale, device=local, max_particles=n)
        one.set_soils(pre["soils"])
        one.initialize(42, pre["layers"])
    host.srand(42)
    lists = [(host.spawn_list(n, dim, dim), host.spawn_list(NWIND, dim, dim)) for _ in range(4)]

    def run(kind, xy, with_one):
        d = sh.ctx.device_spawn(xy)
        dist.barrier()
        sh.run(kind, d, len(xy))
        sh.ctx.device_free(d)
        if with_one:
            getattr(one, kind + "_run")(xy)

    def frame(xw, xd, with_one):
        run("water", xw, with_one)
        sh.water_flood(issuer=0)
        sh.seep(issuer=0)
        if with_one:
            one.water_flood(); one.seep()
        run("wind", xd, with_one)
        sh.ctx.frequency_update()
        if with_one:
            one.frequency_update()

    bad = []
    for xw, xd in lists[:2]:
        frame(xw, xd, rank == 0)
    joined = sh.snapshot()
    path = [None]
    if rank == 0:
        s = one.snapshot()
        if joined.tobytes() != s.tobytes():
            bad.append("joined strip snapshots")
        path[0] = os.path.join(tempfile.mkdtemp(prefix="sm_snap_"), "frame2.snap")
        snapshot.write(path[0], s)
    dist.broadcast_object_list(path, 0)
    for xw, xd in lists[2:]:
        frame(xw, xd, rank == 0)
    a = sh.snapshot()
    if rank == 0 and a.tobytes() != one.snapshot().tobytes():
        bad.append("frames 3-4 sharded vs one context")
    sh.restore(snapshot.read(path[0]))
    for xw, xd in lists[2:]:
        frame(xw, xd, False)
    if sh.snapshot().tobytes() != a.tobytes():
        bad.append("rank %d: resumed frames 3-4" % rank)
    got = [None] * world
    dist.all_gather_object(got, bad)
    bad = [b for part in got for b in part]
    if rank == 0:
        print("multigpu_snapshot_check world=%d%s dim=%d n=%d %s: %d-byte snapshot, %s"
              % (world, " (one GPU, CUDA IPC between processes)" if one_gpu else "", dim, n, soil, a.size,
                 "save, join and resume IDENTICAL" if not bad else "DIFFER at " + ", ".join(bad)), flush=True)
        one.close()
        os.remove(path[0])
        os.rmdir(os.path.dirname(path[0]))
    sh.close()
    dist.destroy_process_group()
    sys.exit(0 if not bad else 1)


if __name__ == "__main__":
    main()
