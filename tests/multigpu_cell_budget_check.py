"""The per-cell budget maps of a map sharded over several PROCESSES (CUDA-IPC peer mappings) must be bit-identical to
one unsharded context's: after a water batch and after a wind batch, the strips' maps concatenated along x.  A step
near a strip edge writes into the neighbouring rank's maps over the peer mapping.  Rank 0 runs the unsharded context
too, prints one line and exits non-zero on any difference.

  N GPUs, one rank per GPU, NCCL for the plumbing:
    python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 --master-port P \
        tests/multigpu_cell_budget_check.py [dim] [particles] [soil]
  ONE GPU, N processes sharing it: SM_ONE_GPU=1 in the environment (gloo for the plumbing, as in
  tests/multigpu_check.py).
"""
import os
import sys
import numpy as np
import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from soilmachine_b200 import capi, presets, host, sharded  # noqa: E402


def main():
    dim = int(sys.argv[1]) if len(sys.argv) > 1 else 512
    n = int(sys.argv[2]) if len(sys.argv) > 2 else 4000
    soil = sys.argv[3] if len(sys.argv) > 3 else "rockgravelpebblessand"
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
    sh = sharded.DistShard(dim, dim, scale, device=local, max_particles=n, share=world if one_gpu else 1,
                           cell_budget=True)
    host.srand(42)
    batches = [("water", host.spawn_list(n, dim, dim)), ("wind", host.spawn_list(n, dim, dim))]
    sh.ctx.set_soils(pre["soils"])
    sh.ctx.initialize(42, pre["layers"])
    mine = []
    for kind, xy in batches:
        d = sh.ctx.device_spawn(xy)
        dist.barrier()
        sh.run(kind, d, len(xy))
        sh.ctx.device_free(d)
        mine.append(sh.last_cell_budget())
    parts = [None] * world
    dist.all_gather_object(parts, mine)
    ok = True
    if rank == 0:
        one = capi.Context(dim, dim, scale, device=local, max_particles=n, cell_budget=True)
        one.set_soils(pre["soils"])
        one.initialize(42, pre["layers"])
        same = lambda a, b: np.array_equal(np.ascontiguousarray(a).view(np.uint8), np.ascontiguousarray(b).view(np.uint8))
        res = {}
        for i, (kind, xy) in enumerate(batches):
            getattr(one, kind + "_run")(xy)
            want = one.last_cell_budget()
            for k in capi.CELL_TERMS:
                res["%s %s" % (kind, k)] = same(np.concatenate([p[i][k] for p in parts], axis=0), want[k])
        ok = all(res.values())
        w = lambda b: "IDENTICAL" if b else "DIFFER"
        print("multigpu_cell_budget_check world=%d%s dim=%d n=%d %s: %s"
              % (world, " (one GPU, CUDA IPC between processes)" if one_gpu else "", dim, n, soil,
                 ", ".join("%s %s" % (k, w(v)) for k, v in res.items())), flush=True)
        one.close()
    flag = [ok]
    dist.broadcast_object_list(flag, 0)
    sh.close()
    dist.destroy_process_group()
    sys.exit(0 if flag[0] else 1)


if __name__ == "__main__":
    main()
