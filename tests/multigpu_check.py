"""The map sharded over several PROCESSES (CUDA-IPC peer mappings, system-scope hand-offs, cross-rank barrier)
must be bit-identical to the same frames on one unsharded context.  Rank 0 runs the unsharded context too and
compares heights, every column section (checksum), frequency maps and the counters; prints one line and exits
non-zero on any difference.

  N GPUs, one rank per GPU, NCCL for the plumbing:
    python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 --master-port P \
        tests/multigpu_check.py [dim] [particles] [soil]
  ONE GPU, N processes sharing it (what the 1-GPU test tier runs, tests/test_gpu_parity.py): SM_ONE_GPU=1 in the
  environment - every rank uses device 0, gloo carries the plumbing (NCCL refuses two ranks on one device), the
  data path is the same CUDA-IPC peer memory as across GPUs.
"""
import os
import sys
import numpy as np
import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from soilmachine_b200 import capi, presets, host, sharded  # noqa: E402


def _sweepstat(ctx, g, kind, rank, reset_only=False):
    """-DSM_PROFILE builds (SM_LIB_PATH): per-sweep statistics of this rank's sweep kernel"""
    import ctypes as C
    buf = np.zeros((16384, 8), np.uint64)
    n = min(int(g.sweeps), 16384)
    ctx.lib.sm_debug_sweeps8(ctx.h, buf.ctypes.data_as(C.c_void_p), max(n, 1))
    if reset_only or n < 2:
        return
    b = buf[:n].astype(np.float64)
    t0 = (~buf[:n, 6]).astype(np.float64)
    ok = buf[:n, 6] != 0
    cyc = 1.965e3
    period = np.diff(t0[ok]) / 1e3 if ok.sum() > 2 else np.zeros(1)
    span = (b[ok, 7] - t0[ok]) / 1e3
    print("rank %d %s: sweeps=%d ms=%.1f | live/rank avg %.0f | avg step %.2f us, max step %.1f, max wait %.1f, max warp busy %.1f, span %.1f, period(active sweeps) %.1f"
          % (rank, kind, g.sweeps, g.device_ms, b[:, 0].mean(), b[:, 4].sum() / max(b[:, 5].sum(), 1) / cyc, b[:, 1].mean() / cyc,
             b[:, 2].mean() / cyc, b[:, 3].mean() / cyc, span.mean(), np.median(period)), flush=True)


def main():
    dim = int(sys.argv[1]) if len(sys.argv) > 1 else 512
    n = int(sys.argv[2]) if len(sys.argv) > 2 else 4000
    soil = sys.argv[3] if len(sys.argv) > 3 else "rockgravelpebblessand"
    frames_n = int(sys.argv[4]) if len(sys.argv) > 4 else 2
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    one_gpu = os.environ.get("SM_ONE_GPU") == "1"
    local = 0 if one_gpu else int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    if one_gpu:
        dist.init_process_group("gloo")
    else:
        dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    pre = presets.load(soil)
    sh = sharded.DistShard(dim, dim, pre["world"]["scale"], device=local, max_particles=n,
                           share=world if one_gpu else 1)
    sh.ctx.set_soils(pre["soils"])
    sh.ctx.initialize(42, pre["layers"])
    host.srand(42)
    frames = [(host.spawn_list(n, dim, dim), host.spawn_list(n, dim, dim)) for _ in range(frames_n)]
    tot = np.zeros(4)
    t_ms = 0.0
    for xw, xd in frames:
        dw, dd = sh.ctx.device_spawn(xw), sh.ctx.device_spawn(xd)
        dist.barrier()
        a = sh.run("water", dw, n)
        if os.environ.get("SM_SWEEPSTAT") == "1":
            _sweepstat(sh.ctx, a, "water", rank, reset_only=True)
        b = sh.run("wind", dd, n)
        if os.environ.get("SM_SWEEPSTAT") == "1":
            _sweepstat(sh.ctx, b, "wind", rank)
        sh.ctx.frequency_update()
        tot += [a.steps, b.steps, a.exit_oob + a.exit_evap + a.exit_stall, b.exit_oob]
        t_ms += a.device_ms + b.device_ms
        sh.ctx.device_free(dw); sh.ctx.device_free(dd)
    mine = {"h": sh.ctx.heights().copy(), "cs": sh.ctx.checksum(), "freq": sh.ctx.frequency(), "tot": tot,
            "ms": t_ms, "range": (sh.ctx.x0, sh.ctx.x1)}
    parts = [None] * world
    dist.all_gather_object(parts, mine)
    ok = True
    if rank == 0:
        full = np.concatenate([p["h"] for p in parts], axis=0)
        cs = sum(p["cs"] for p in parts) & ((1 << 64) - 1)
        freq = sharded.merge_frequency([p["freq"] for p in parts], [p["range"] for p in parts], dim, dim)
        counts = sum(p["tot"] for p in parts)
        one = capi.Context(dim, dim, pre["world"]["scale"], device=local, max_particles=n)
        one.set_soils(pre["soils"]); one.initialize(42, pre["layers"])
        c1 = np.zeros(4); t1 = 0.0
        for xw, xd in frames:
            a = one.water_run(xw); b = one.wind_run(xd); one.frequency_update()
            c1 += [a.steps, b.steps, a.exit_oob + a.exit_evap + a.exit_stall, b.exit_oob]
            t1 += a.device_ms + b.device_ms
        same_h = np.array_equal(full.view(np.uint8), one.heights().view(np.uint8))
        same_c = cs == one.checksum()
        f1 = one.frequency()
        same_f = all(np.array_equal(freq[k].view(np.uint8), f1[k].view(np.uint8)) for k in f1)
        same_s = np.array_equal(c1, counts)
        ok = same_h and same_c and same_f and same_s
        w = lambda b: "IDENTICAL" if b else "DIFFER"
        print("multigpu_check world=%d%s dim=%d n=%d %s: heights %s, column checksum %s (%016x), frequency maps %s, "
              "counters %s (%s) | sharded %.1f ms vs one context %.1f ms"
              % (world, " (one GPU, CUDA IPC between processes)" if one_gpu else "", dim, n, soil, w(same_h), w(same_c),
                 cs, w(same_f), w(same_s), counts.tolist(), max(p["ms"] for p in parts), t1), flush=True)
        one.close()
    flag = [ok]
    dist.broadcast_object_list(flag, 0)
    sh.close()
    dist.destroy_process_group()
    sys.exit(0 if flag[0] else 1)


if __name__ == "__main__":
    main()
