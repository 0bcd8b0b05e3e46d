"""Slope relaxation on a group with one rank per GPU, all in this process (sm_create_group, sm_relax): neighbouring
ranks' phases are ordered by events between their streams, and edge cells write the neighbour's columns, pool and
stale bits over peer access.  One unsharded context on GPU 0 runs the same inputs: a frame (water batch, floods, seep
pass, wind batch), a steep raster dense on the strip edges, relax for transferloop 1, 3 and 0, then another frame.
The stats (device time aside), the checksums and the snapshots must be equal.  Prints one line; exits non-zero on any
difference.

    python tests/multigpu_relax_check.py --gpus N [--dim 256]
"""
import argparse
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
from soilmachine_b200 import capi, host, presets  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=2)
    ap.add_argument("--dim", type=int, default=256)
    args = ap.parse_args()
    from test_relax import steep_raster
    from test_apply_layer import _frame, _group_edges
    dim, n = args.dim, args.gpus
    pre = presets.load("rocksand")
    scale = pre["world"]["scale"]
    one = capi.Context(dim, dim, scale, device=0, max_particles=4096)
    grp = capi.Context(dim, dim, scale, devices=list(range(n)), max_particles=4096)
    bad = []
    for m in (one, grp):
        m.set_soils(pre["soils"])
        m.initialize(42, pre["layers"])
    host.srand(42)
    lists = [(host.spawn_list(2000, dim, dim), host.spawn_list(400, dim, dim)) for _ in range(2)]
    if _frame(one, *lists[0]) != _frame(grp, *lists[0]):
        bad.append("frame 1 stats")
    d = steep_raster(np.random.default_rng(1), dim, dim, edges=_group_edges(dim, n))
    one.apply_layer(d, 2)
    grp.apply_layer(d, 2)
    stats = []
    for tl in (1, 3, 0):
        so, sg = one.relax(8, tl).asdict(), grp.relax(8, tl).asdict()
        so.pop("device_ms"); sg.pop("device_ms")
        stats.append(sg)
        if so != sg:
            bad.append("transferloop %d stats %s vs %s" % (tl, sg, so))
        if one.checksum() != grp.checksum() or bytes(one.snapshot()) != bytes(grp.snapshot()):
            bad.append("transferloop %d map" % tl)
    if _frame(one, *lists[1]) != _frame(grp, *lists[1]) or one.checksum() != grp.checksum():
        bad.append("frame 2")
    print("multigpu_relax_check gpus %d dim %d: %s %s" % (n, dim, "DIFFER " + "; ".join(bad) if bad else "equal", stats))
    one.close()
    grp.close()
    sys.exit(1 if bad else 0)


if __name__ == "__main__":
    main()
