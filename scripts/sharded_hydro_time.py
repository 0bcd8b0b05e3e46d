"""Device time of the pooling hydrology on a sharded map (DESIGN.md section 5), with the card it ran on.

  python scripts/sharded_hydro_time.py [--reps 2]

The bench's map (4096^2 rockgravelpebblessand, seed 42) and its first water list (25k particles), then the floods of
that batch and the seep pass, on two arms taken in alternation: one unsharded context, and 2 virtual ranks sharing
this GPU with the calls issued by rank 0.  Prints one JSON line per run (the device_ms of each call and the seep
pass's classification) and checks that both arms leave the same columns (the checksums of the strips add up to the
unsharded one).
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

DIM, SOIL, SEED, NWATER = 4096, "rockgravelpebblessand", 42, 25000


def _card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=60).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def run_arm(arm, xy):
    from soilmachine_b200 import capi, presets, sharded
    pre = presets.load(SOIL)
    scale = pre["world"]["scale"]
    if arm == "one":
        m = capi.Context(DIM, DIM, scale, max_particles=NWATER)
    else:
        m = sharded.VirtualShards(2, DIM, DIM, scale, max_particles=NWATER)
    m.set_soils(pre["soils"])
    m.initialize(SEED, pre["layers"])
    w = m.water_run(xy)
    if arm == "one":
        fl, sp = m.water_flood(), m.seep()
        csum = m.checksum()
    else:
        fl, sp = m.water_flood(rank=0), m.seep(rank=0)
        csum = sum(c.checksum() for c in m.ctx) % (1 << 64)
    m.close()
    return {"arm": arm, "water_batch_ms": w.device_ms, "flood_ms": fl.device_ms, "seep_ms": sp.device_ms,
            "classify_ms": sp.classify_ms, "floods": fl.floods, "nested": fl.nested + sp.nested,
            "seep_cells": sp.cells, "checksum": csum}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=2)
    args = ap.parse_args()
    from soilmachine_b200 import host
    host.srand(SEED)
    xy = host.spawn_list(NWATER, DIM, DIM)
    card = _card()
    sums = {}
    for rep in range(args.reps):
        for arm in ("one", "2 virtual ranks"):
            r = run_arm(arm, xy)
            r.update({"rep": rep, "dim": DIM, "soil": SOIL, "card": card})
            sums.setdefault(arm, set()).add(r["checksum"])
            print(json.dumps(r), flush=True)
    same = len(set().union(*sums.values())) == 1
    print(json.dumps({"what": "columns after flood + seep", "identical_across_arms": same}), flush=True)
    sys.exit(0 if same else 1)


if __name__ == "__main__":
    main()
