"""The pooling hydrology on a map sharded over several PROCESSES (CUDA-IPC peer mappings of the strips, the pools and
the frequency arrays) must be bit-identical to one unsharded context: frames of water batch -> flood -> seep pass ->
wind batch -> frequency update, the floods and the seep pass issued by the last rank.  After every phase the columns,
heights and frequency maps of all ranks are gathered and compared, and the issuer's hydrology counters with the
unsharded ones.  Rank 0 runs the unsharded context too, prints one line and exits non-zero on any difference.

  N GPUs, one rank per GPU, NCCL for the plumbing:
    python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 --master-port P \
        tests/multigpu_hydro_check.py [dim] [particles] [soil] [frames]
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

HYDRO_KEYS = ("floods", "nested", "nested_steps", "transfers", "cells")


def _snap(ctx):
    """this context's columns, heights and frequency arrays"""
    return {"cols": ctx.download_columns(), "heights": ctx.heights(), "freq": ctx.frequency()}


def main():
    dim = int(sys.argv[1]) if len(sys.argv) > 1 else 512
    n = int(sys.argv[2]) if len(sys.argv) > 2 else 4000
    soil = sys.argv[3] if len(sys.argv) > 3 else "rockgravelpebblessand"
    frames = int(sys.argv[4]) if len(sys.argv) > 4 else 2
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
    issuer = world - 1
    sh = sharded.DistShard(dim, dim, scale, device=local, max_particles=n, share=world if one_gpu else 1)
    sh.ctx.set_soils(pre["soils"])
    sh.ctx.initialize(42, pre["layers"])
    ranges = [None] * world
    dist.all_gather_object(ranges, (sh.ctx.x0, sh.ctx.x1))
    one = None
    if rank == 0:
        one = capi.Context(dim, dim, scale, device=local, max_particles=n)
        one.set_soils(pre["soils"])
        one.initialize(42, pre["layers"])
    same = lambda a, b: np.array_equal(np.ascontiguousarray(a).view(np.uint8), np.ascontiguousarray(b).view(np.uint8))
    bad = []
    phases = 0
    host.srand(42)

    def compare(what, stats=None, stats1=None):
        sh.ctx.sync()
        parts = [None] * world
        dist.all_gather_object(parts, _snap(sh.ctx))
        if rank != 0:
            return
        want = _snap(one)
        cols = sharded.merge_columns([p["cols"] for p in parts])
        ok = all(same(cols[k], want["cols"][k]) for k in want["cols"])
        ok = ok and same(np.concatenate([p["heights"] for p in parts], axis=0), want["heights"])
        freq = sharded.merge_frequency([p["freq"] for p in parts], ranges, dim, dim)
        ok = ok and all(same(freq[k], want["freq"][k]) for k in want["freq"])
        if stats1 is not None:
            ok = ok and [stats[k] for k in HYDRO_KEYS] == [getattr(stats1, k) for k in HYDRO_KEYS]
        if not ok:
            bad.append(what)

    def run(kind, xy):
        d = sh.ctx.device_spawn(xy)
        dist.barrier()
        sh.run(kind, d, len(xy))
        sh.ctx.device_free(d)
        if rank == 0:
            getattr(one, kind + "_run")(xy)

    nflood = 0
    for f in range(frames):
        xw, xd = host.spawn_list(n, dim, dim), host.spawn_list(n, dim, dim)
        run("water", xw)
        compare("frame %d water batch" % f)
        for name in ("flood", "seep"):
            st = (sh.water_flood if name == "flood" else sh.seep)(issuer=issuer)
            got = [None]
            if rank == issuer:
                got[0] = st.asdict()
            dist.broadcast_object_list(got, issuer)
            st1 = (one.water_flood if name == "flood" else one.seep)() if rank == 0 else None
            if rank == 0 and name == "flood":
                nflood += st1.floods
            compare("frame %d %s" % (f, name), got[0], st1)
            phases += 1
        run("wind", xd)
        compare("frame %d wind batch" % f)
        sh.ctx.frequency_update()
        if rank == 0:
            one.frequency_update()
        compare("frame %d frequency update" % f)
    ok = True
    if rank == 0:
        ok = not bad and nflood > 0
        print("multigpu_hydro_check world=%d%s dim=%d n=%d %s frames=%d issuer=%d: %d floods, %d hydrology calls, %s"
              % (world, " (one GPU, CUDA IPC between processes)" if one_gpu else "", dim, n, soil, frames, issuer,
                 nflood, phases, "every phase IDENTICAL" if not bad else "DIFFER at " + ", ".join(bad)), flush=True)
        one.close()
    flag = [ok]
    dist.broadcast_object_list(flag, 0)
    sh.close()
    dist.destroy_process_group()
    sys.exit(0 if flag[0] else 1)


if __name__ == "__main__":
    main()
