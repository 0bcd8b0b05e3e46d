"""Device time of the particle batches with the per-cell budget maps (DESIGN.md section 5), with the card it ran on.

  python scripts/cell_budget_time.py [--reps 3]

Workload: bench.py's config 3 - 4096^2 rockgravelpebblessand, terrain from sm_initialize (seed 42), the first frame's
25 000-particle water and 25 000-particle wind spawn lists (srand(42)), water batch then wind batch.  Three arms, each on
a fresh context with the same terrain, run alternately `--reps` times:
  * plain:  no flag;
  * budget: SM_FLAG_BUDGET;
  * cells:  SM_FLAG_BUDGET | SM_FLAG_CELL_BUDGET.
Prints one JSON line for the card and one per arm and repetition: device_ms of the two batches and the column checksum
after them (equal across the arms).
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

DIM, SOIL, SEED, N = 4096, "rockgravelpebblessand", 42, 25000
ARMS = (("plain", False, False), ("budget", True, False), ("cells", True, True))


def _card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=60).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def run_arm(name, budget, cells, pre, xw, xd):
    from soilmachine_b200 import capi
    ctx = capi.Context(DIM, DIM, pre["world"]["scale"], max_particles=N, budget=budget, cell_budget=cells)
    ctx.set_soils(pre["soils"])
    ctx.initialize(SEED, pre["layers"])
    sw = ctx.water_run(xw)
    sd = ctx.wind_run(xd)
    out = {"arm": name, "water_ms": sw.device_ms, "wind_ms": sd.device_ms, "water_steps": sw.steps,
           "wind_steps": sd.steps, "checksum": "%016x" % ctx.checksum(), "pool_drops": sw.pool_drops + sd.pool_drops}
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
    xw, xd = host.spawn_list(N, DIM, DIM), host.spawn_list(N, DIM, DIM)
    sums = set()
    for rep in range(args.reps):
        for name, budget, cells in ARMS:
            r = run_arm(name, budget, cells, pre, xw, xd)
            r["rep"] = rep
            sums.add(r["checksum"])
            print(json.dumps(r), flush=True)
    print(json.dumps({"checksums_equal": len(sums) == 1}), flush=True)


if __name__ == "__main__":
    main()
