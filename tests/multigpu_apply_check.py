"""Layer rasters on a map sharded over several PROCESSES (DistShard.apply_layer: every rank checks its strip, the
outcomes are gathered, then every rank applies; CUDA-IPC peer mappings for the batches in between).  Rank 0 also runs
one unsharded context on the same inputs.  Frames: water batch -> floods -> seep pass -> wind batch -> frequency
update; after each of two frames a raster of another soil type, the second one dense on the strip edges.  The joined
strip snapshots, the leftovers and the summed stats must equal the one context's.  Rank 0 prints one line and every
process exits non-zero on any difference.

  N GPUs, one rank per GPU:
    python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 --master-port P \\
        tests/multigpu_apply_check.py [dim] [water particles]
  ONE GPU, N processes sharing it: SM_ONE_GPU=1 in the environment.
"""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from soilmachine_b200 import capi, presets, host, sharded  # noqa: E402

NWIND = 200


def raster(rng, dimx, dimy, edges=None):
    u = rng.random((dimx, dimy))
    d = np.where(u < 0.4, rng.uniform(0.0, 0.08, u.shape), -rng.uniform(0.0, 0.15, u.shape))
    d[(u >= 0.75) & (u < 0.82)] = -2.0
    d[(u >= 0.85) & (u < 0.95)] = 0.0
    d[u >= 0.95] = -0.0
    if edges:
        x = np.arange(dimx)[:, None]
        d[~np.any([np.abs(x - e) <= 2 for e in edges], axis=0).repeat(dimy, 1)] = 0.0
    return d


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
    lists = [(host.spawn_list(n, dim, dim), host.spawn_list(NWIND, dim, dim)) for _ in range(2)]
    x0s = [None] * world
    dist.all_gather_object(x0s, sh.ctx.x0)
    rng = np.random.default_rng(7)
    bad = []
    for f, (xw, xd) in enumerate(lists):
        for kind, xy in (("water", xw), ("wind", xd)):
            d = sh.ctx.device_spawn(xy)
            dist.barrier()
            sh.run(kind, d, len(xy))
            sh.ctx.device_free(d)
            if rank == 0:
                getattr(one, kind + "_run")(xy)
            if kind == "water":
                sh.water_flood(issuer=0)
                sh.seep(issuer=0)
                if rank == 0:
                    one.water_flood(); one.seep()
        sh.ctx.frequency_update()
        if rank == 0:
            one.frequency_update()
        delta = raster(rng, dim, dim, edges=x0s[1:] if f == 1 else None)
        t = f + 1
        st, left = sh.apply_layer(delta[sh.ctx.x0:sh.ctx.x1], t, leftover=True)
        lefts, stats = [None] * world, [None] * world
        dist.all_gather_object(lefts, left)
        dist.all_gather_object(stats, (st.cells, st.pushed, st.emptied))
        joined = sh.snapshot()
        if rank == 0:
            so, lo = one.apply_layer(delta, t, leftover=True)
            if np.concatenate(lefts).tobytes() != lo.tobytes():
                bad.append("frame %d leftovers" % f)
            if tuple(np.sum(stats, axis=0)) != (so.cells, so.pushed, so.emptied):
                bad.append("frame %d stats" % f)
            if joined.tobytes() != one.snapshot().tobytes():
                bad.append("frame %d snapshot" % f)
    got = [None] * world
    dist.all_gather_object(got, bad)
    bad = [b for part in got for b in part]
    if rank == 0:
        print("multigpu_apply_check world=%d%s dim=%d n=%d %s: rasters after 2 frames %s"
              % (world, " (one GPU, CUDA IPC between processes)" if one_gpu else "", dim, n, soil,
                 "IDENTICAL to one context" if not bad else "DIFFER at " + ", ".join(bad)), flush=True)
        one.close()
    sh.close()
    dist.destroy_process_group()
    sys.exit(0 if not bad else 1)


if __name__ == "__main__":
    main()
