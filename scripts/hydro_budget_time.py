"""Device time of the pooling hydrology with and without its mass budget (DESIGN.md section 5), with the card it ran on.

  python scripts/hydro_budget_time.py [--reps 3]

Workload: 4096^2 rockgravelpebblessand, terrain from sm_initialize (seed 42), one 25 000-particle water batch with
bench.py's spawn list (srand(42)), then sm_water_flood and sm_seep.  Three arms, each on a fresh context with the same
terrain, run alternately `--reps` times:
  * thread: no SM_FLAG_BUDGET, the default one-thread executor (SM_HYDRO=thread);
  * warp:   no SM_FLAG_BUDGET, SM_HYDRO=warp - separates the cost of the executor switch from the accumulators';
  * budget: SM_FLAG_BUDGET, which runs the warp executor whatever SM_HYDRO says.
Prints one JSON line for the card and one per arm and repetition: device_ms of flood and seep, the seep pass's
classify_ms, the column checksum after the seep pass (equal across the arms) and, for the budget arm, the residual of
the budget identity over flood + seep against sm_height_sum.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

DIM, SOIL, SEED, N = 4096, "rockgravelpebblessand", 42, 25000
ARMS = (("thread", "thread", False), ("warp", "warp", False), ("budget", "thread", True))


def _card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=60).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def _identity(b):
    return (b["flood_sediment"] + b["flood_cascade_net"] + b["flood_water"] - b["seeped"] - b["to_particles"] +
            b["transfer_net"] + b["nested_deposited"] - b["nested_eroded"] + b["nested_cascade_net"])


def run_arm(name, executor, budget, pre, xw):
    from soilmachine_b200 import capi
    os.environ["SM_HYDRO"] = executor
    ctx = capi.Context(DIM, DIM, pre["world"]["scale"], max_particles=N, budget=budget)
    ctx.set_soils(pre["soils"])
    ctx.initialize(SEED, pre["layers"])
    st = ctx.water_run(xw)
    h0 = ctx.height_sum()
    fl = ctx.water_flood()
    bf = ctx.last_hydro_budget() if budget else None
    se = ctx.seep()
    out = {"arm": name, "flood_ms": fl.device_ms, "seep_ms": se.device_ms, "classify_ms": se.classify_ms,
           "floods": fl.floods, "nested": fl.nested + se.nested, "seep_cells": se.cells,
           "checksum": "%016x" % ctx.checksum(), "pool_drops": st.pool_drops}
    if budget:
        bs = ctx.last_hydro_budget()
        dh = ctx.height_sum() - h0
        ident = _identity(bf) + _identity(bs)
        mag = sum(abs(v) for b in (bf, bs) for k, v in b.items() if k not in ("nested_discarded", "nested_clamped"))
        out.update({"height_sum": h0, "dheight": dh, "identity": ident, "residual": dh - ident,
                    "residual_rel": abs(dh - ident) / mag})
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
        for name, executor, budget in ARMS:
            r = run_arm(name, executor, budget, pre, xw)
            r["rep"] = rep
            sums.add(r["checksum"])
            print(json.dumps(r), flush=True)
    print(json.dumps({"checksums_equal": len(sums) == 1}), flush=True)


if __name__ == "__main__":
    main()
