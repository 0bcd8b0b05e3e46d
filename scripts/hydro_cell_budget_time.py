"""Device time of the pooling hydrology with and without its per-cell maps (DESIGN.md sections 5 and 8), with the card
it ran on.

  python scripts/hydro_cell_budget_time.py [--reps 3]

Workload: bench config 3 - 4096^2 rockgravelpebblessand, terrain from sm_initialize (seed 42), one 25 000-particle
water batch with bench.py's spawn list (srand(42)), then sm_water_flood and sm_seep.  Two arms, each on a fresh context
with the same terrain, run alternately `--reps` times:
  * budget: SM_FLAG_BUDGET (the warp executor's BUDGET instantiations);
  * maps:   SM_FLAG_BUDGET | SM_FLAG_HYDRO_CELL_BUDGET (its BUDGET + CELLS instantiations).
Prints one JSON line for the card (name, power limit, max SM clock) and one per arm and repetition: device_ms of flood
and seep (with the maps it includes the memset that zeroes them), the seep pass's classify_ms, the column checksum
after the seep pass (equal across the arms), and for the maps arm the largest per-cell residual of the identity over
flood + seep.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

DIM, SOIL, SEED, N = 4096, "rockgravelpebblessand", 42, 25000
ARMS = (("budget", False), ("maps", True))


def _card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=60).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def run_arm(name, maps, pre, xw):
    import numpy as np
    from soilmachine_b200 import capi
    ctx = capi.Context(DIM, DIM, pre["world"]["scale"], max_particles=N, budget=True, hydro_cell_budget=maps)
    ctx.set_soils(pre["soils"])
    ctx.initialize(SEED, pre["layers"])
    st = ctx.water_run(xw)
    h0 = ctx.heights() if maps else None
    fl = ctx.water_flood()
    mf = ctx.last_hydro_cell_budget() if maps else None
    se = ctx.seep()
    out = {"arm": name, "flood_ms": fl.device_ms, "seep_ms": se.device_ms, "classify_ms": se.classify_ms,
           "floods": fl.floods, "nested": fl.nested + se.nested, "seep_cells": se.cells,
           "checksum": "%016x" % ctx.checksum(), "pool_drops": st.pool_drops}
    if maps:
        ms = ctx.last_hydro_cell_budget()
        dh = ctx.heights() - h0
        ident = sum(m["deposited"] - m["eroded"] + m["cascade_net"] + m["water_net"] for m in (mf, ms))
        out.update({"cells_touched": int(sum((m[k] != 0) for m in (mf, ms) for k in m).astype(bool).sum()),
                    "max_cell_residual": float(np.abs(dh - ident).max())})
    ctx.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    from soilmachine_b200 import host, presets
    print(json.dumps({"card": _card()}), flush=True)
    pre = presets.load(SOIL)
    host.srand(SEED)
    xw = host.spawn_list(N, DIM, DIM)
    sums = set()
    for rep in range(args.reps):
        for name, maps in ARMS:
            r = run_arm(name, maps, pre, xw)
            r["rep"] = rep
            sums.add(r["checksum"])
            print(json.dumps(r), flush=True)
    print(json.dumps({"checksums_equal": len(sums) == 1}), flush=True)


if __name__ == "__main__":
    main()
