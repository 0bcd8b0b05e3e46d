"""The read-only views of a map sharded over several PROCESSES (CUDA-IPC peer mappings) must be bit-identical to one
unsharded context: the mesh at slice 160 and 45, the exportheight / exportcolor values, the single-cell queries of
every cell of the columns at the strip edges (issued by every rank), and the wind-field lattice built from the
terrain and stepped 25 times (every rank holds the whole lattice).  Rank 0 runs the unsharded context too, prints
one line and exits non-zero on any difference.

  N GPUs, one rank per GPU, NCCL for the plumbing:
    python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 --master-port P \
        tests/multigpu_views_check.py [dim] [particles] [soil]
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

LATTICES = [(32, 20, 32), (27, 12, 22)]


def _queries(m, cells, points):
    """cell_query + cell_column of every cell, bilinear height of every point, as raw bytes"""
    out = []
    for x, y in cells:
        h, s, n = m.cell_query(x, y)
        col = m.cell_column(x, y)
        out.append(np.float64(h).tobytes() + np.int32(s).tobytes() + n.tobytes() + np.int32(col["n"]).tobytes() +
                   b"".join(np.ascontiguousarray(col[k]).tobytes() for k in ("type", "size", "floor", "saturation")))
    out.append(np.array([m.height_bilinear(x, y) for x, y in points]).tobytes())
    return out


def _frame(m, pre, xw, xd, run):
    m.set_soils(pre["soils"])
    m.set_soil_colors(pre["colors"])
    m.initialize(42, pre["layers"])
    a, b = run("water", xw), run("wind", xd)
    m.frequency_update()
    return [a.steps, b.steps, a.exit_oob + a.exit_evap + a.exit_stall, b.exit_oob]


def _views(m, cells, points):
    v = {"mesh160": m.mesh_update(160), "height": m.export_height(), "color": m.export_color(),
         "mesh45": m.mesh_update(45), "queries": _queries(m, cells, points)}
    for dims in LATTICES:
        m.lbm_create(*dims)
        m.lbm_set_boundary(None)
        m.lbm_step(25)
        v["lbm%s" % (dims,)] = m.lbm_get()
    return v


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
    sh = sharded.DistShard(dim, dim, scale, device=local, max_particles=n, share=world if one_gpu else 1)
    host.srand(42)
    xw, xd = host.spawn_list(n, dim, dim), host.spawn_list(n, dim, dim)

    def run_sharded(kind, xy):
        d = sh.ctx.device_spawn(xy)
        dist.barrier()
        st = sh.run(kind, d, len(xy))
        sh.ctx.device_free(d)
        return st

    tot = np.array(_frame(sh.ctx, pre, xw, xd, run_sharded), np.float64)
    ranges = [None] * world
    dist.all_gather_object(ranges, (sh.ctx.x0, sh.ctx.x1))
    edges = sorted({x for x0, _ in ranges[1:] for x in (x0 - 1, x0, x0 + 1)})
    cells = [(x, y) for x in edges for y in range(dim)]
    points = [(np.float32(x0 - 1 + fx), np.float32(y + 0.375)) for x0, _ in ranges[1:] for fx in (0.0, 0.5, 0.875)
              for y in range(0, dim - 1, 5)]
    mine = _views(sh, cells, points)
    mine["tot"] = tot
    parts = [None] * world
    dist.all_gather_object(parts, mine)
    ok = True
    if rank == 0:
        one = capi.Context(dim, dim, scale, device=local, max_particles=n)
        tot1 = np.array(_frame(one, pre, xw, xd, lambda kind, xy: getattr(one, kind + "_run")(xy)), np.float64)
        want = _views(one, cells, points)
        same = lambda a, b: np.array_equal(np.ascontiguousarray(a).view(np.uint8), np.ascontiguousarray(b).view(np.uint8))
        res = {"counters": same(sum(p["tot"] for p in parts), tot1)}
        for k in ("mesh160", "height", "color", "mesh45"):
            res[k] = same(np.concatenate([p[k] for p in parts], axis=0), want[k])
        res["queries (every rank)"] = all(p["queries"] == want["queries"] for p in parts)
        for dims in LATTICES:
            k = "lbm%s" % (dims,)
            res["lattice %dx%dx%d (every rank)" % dims] = all(same(p[k][q], want[k][q]) for p in parts
                                                              for q in ("f", "rho", "v"))
        ok = all(res.values())
        w = lambda b: "IDENTICAL" if b else "DIFFER"
        print("multigpu_views_check world=%d%s dim=%d n=%d %s: %s | %d edge cells, %d bilinear points"
              % (world, " (one GPU, CUDA IPC between processes)" if one_gpu else "", dim, n, soil,
                 ", ".join("%s %s" % (k, w(v)) for k, v in res.items()), len(cells), len(points)), flush=True)
        one.close()
    flag = [ok]
    dist.broadcast_object_list(flag, 0)
    sh.close()
    dist.destroy_process_group()
    sys.exit(0 if flag[0] else 1)


if __name__ == "__main__":
    main()
