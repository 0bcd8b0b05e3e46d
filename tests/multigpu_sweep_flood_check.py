"""Sweep floods on a group with one rank per GPU, all in this process (sm_create_group, sm_water_run_flooding): every
sweep ends in a barrier across the GPUs, rank 0's stream waits for every rank's sweep, floods over the whole map through
peer access and moves every rank's sweep tags on, and every rank's next sweep waits for that flood.  One unsharded
context on GPU 0 runs the same inputs: a whole batch, a batch cut after 30 sweeps, a whole batch again, then a frame
with the seep pass.  The batch stats (device time aside), the flood counters, the particle states, the checksums and
the snapshots must be equal.  Prints one line; exits non-zero on any difference.

    python tests/multigpu_sweep_flood_check.py --gpus N [--dim 256]
    python tests/multigpu_sweep_flood_check.py --devices 0,0,0      (ranks sharing a GPU: the same code paths, one device)
"""
import argparse
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
from soilmachine_b200 import capi, host, presets  # noqa: E402

STAT_KEYS = ("steps", "sweeps", "exit_oob", "exit_evap", "exit_stall", "pool_drops", "alive")
HYDRO_KEYS = ("floods", "nested", "nested_steps", "transfers", "cells")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=2)
    ap.add_argument("--dim", type=int, default=256)
    ap.add_argument("--devices", default=None, help="device of each rank, e.g. 0,1,2 (default: 0 .. gpus - 1)")
    args = ap.parse_args()
    devices = [int(d) for d in args.devices.split(",")] if args.devices else list(range(args.gpus))
    dim, n = args.dim, len(devices)
    pre = presets.load("bigbutte")
    scale = pre["world"]["scale"]
    one = capi.Context(dim, dim, scale, device=0, max_particles=8192)
    grp = capi.Context(dim, dim, scale, devices=devices, max_particles=8192)
    for m in (one, grp):
        m.set_soils(pre["soils"])
        m.initialize(42, pre["layers"])
    host.srand(42)
    lists = [host.spawn_list(4000, dim, dim) for _ in range(4)]
    bad, floods = [], []
    for b, cut in enumerate((0, 30, 0)):
        (so, ho), (sg, hg) = one.water_run_flooding(lists[b], cut), grp.water_run_flooding(lists[b], cut)
        floods.append(hg.floods)
        if [getattr(so, k) for k in STAT_KEYS] != [getattr(sg, k) for k in STAT_KEYS]:
            bad.append("batch %d stats %s vs %s" % (b, sg.asdict(), so.asdict()))
        if [getattr(ho, k) for k in HYDRO_KEYS] != [getattr(hg, k) for k in HYDRO_KEYS]:
            bad.append("batch %d flood counters %s vs %s" % (b, hg.asdict(), ho.asdict()))
        a, c = one.water_state(), grp.water_state()
        if any(not np.array_equal(a[k].view(np.uint8), c[k].view(np.uint8)) for k in a):
            bad.append("batch %d particle states" % b)
        if one.checksum() != grp.checksum() or bytes(one.snapshot()) != bytes(grp.snapshot()):
            bad.append("batch %d map" % b)
    for m in (one, grp):
        m.water_run_flooding(lists[3])
        m.seep()
        m.frequency_update()
    if one.checksum() != grp.checksum() or bytes(one.snapshot()) != bytes(grp.snapshot()):
        bad.append("frame with the seep pass")
    if min(floods) == 0:
        bad.append("a batch without floods %s" % floods)
    print("multigpu_sweep_flood_check devices %s dim %d: %s floods %s" % (
        ",".join(map(str, devices)), dim, "DIFFER " + "; ".join(bad) if bad else "equal", floods))
    one.close()
    grp.close()
    sys.exit(1 if bad else 0)


if __name__ == "__main__":
    main()
