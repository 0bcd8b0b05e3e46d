"""Time the drainage view, sm_drainage (DESIGN.md section 14), at the benchmark's sizes.

  config 3   4096^2 rockgravelpebblessand after one frame with hydrology (25k water particles, their floods, the seep
             pass, 25k wind particles, seed 42)
  config 5   8192^2 rockgravelpebbles_big, its initial terrain (seed 42)
For each map, the call runs with the top of the columns and with SM_DRAIN_GROUND, each with device output (buffers
from sm_device_alloc) and host output (numpy arrays).  Every arm runs once untimed first; then the arms alternate over
the rounds.  Reported per arm: the median host-clock time of the call (ending with the outputs in place), the
CUDA-event kernel time per phase (heights, fill, dist, receivers, area, basin), the fill, dist and pointer-jumping
passes, the longest area walk (receivers visited by one walker), the flat, depressed and outlet counts.  The fill and
dist pass counts can vary from run to run (tiles race within a pass), so min..max over the rounds is given.  The card's
name and power limit are read in the same run.

  python scripts/drainage_time.py [--rounds 3] [--configs 3,5] [--json out.json]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from soilmachine_b200 import host  # noqa: E402

MAPS = {3: dict(soil="rockgravelpebblessand", dim=4096, frame=(25000, 25000)),
        5: dict(soil="rockgravelpebbles_big", dim=8192, frame=None)}


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except OSError:
        return "unknown"


def time_map(cfg, rounds):
    m = MAPS[cfg]
    dim = m["dim"]
    sim = host.Simulation(m["soil"], seed=42, dimx=dim, dimy=dim, max_particles=25000)
    if m["frame"]:
        sim.frame(*m["frame"], hydrology=True)
    c = sim.ctx
    n = dim * dim
    bufs = {}
    for k, size in (("spill", 8), ("dir", 1), ("area", 8), ("basin", 8)):
        d = C.c_void_p()
        c._ck(c.lib.sm_device_alloc(c.h, C.c_int64(n * size), C.byref(d)))
        bufs[k] = d

    def run(ground, dev):
        t0 = time.perf_counter()
        c.drainage(ground, out=bufs if dev else None)
        return (time.perf_counter() - t0) * 1e3, c.drain_stats.asdict()

    arms = [(g, dev) for g in (False, True) for dev in (True, False)]
    for a in arms:
        run(*a)
    res = {a: [] for a in arms}
    for r in range(rounds):
        for a in (arms if r % 2 == 0 else arms[::-1]):
            res[a].append(run(*a))
    out = {}
    for g, dev in arms:
        rs = res[(g, dev)]
        st = rs[0][1]
        med = lambda v: float(np.median(v))
        out["%s/%s" % ("ground" if g else "top", "device" if dev else "host")] = {
            "call_ms": med([ms for ms, _ in rs]),
            "device_ms": med([s["device_ms"] for _, s in rs]),
            "phase_ms": {p: med([s["phase_ms"][p] for _, s in rs]) for p in st["phase_ms"]},
            "fill_passes": [min(s["fill_passes"] for _, s in rs), max(s["fill_passes"] for _, s in rs)],
            "dist_passes": [min(s["dist_passes"] for _, s in rs), max(s["dist_passes"] for _, s in rs)],
            "jump_passes": st["jump_passes"],
            "longest_walk": max(s["longest_walk"] for _, s in rs),
            "flat_cells": st["flat_cells"], "depressed_cells": st["depressed_cells"], "outlets": st["outlets"]}
    for d in bufs.values():
        c.device_free(d)
    sim.close()
    return {"dim": dim, "soil": m["soil"], "after_frame": bool(m["frame"]), "arms": out}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--configs", default="3,5")
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    out = {"gpu": gpu_info(), "rounds": args.rounds, "maps": {}}
    for cfg in [int(x) for x in args.configs.split(",")]:
        out["maps"]["config%d" % cfg] = time_map(cfg, args.rounds)
        for arm, r in out["maps"]["config%d" % cfg]["arms"].items():
            print("config %d %s: call %.1f ms, kernels %.1f ms (%s), fill passes %s, dist passes %s, jumps %d, "
                  "longest walk %d, flat %d, depressed %d, outlets %d" % (
                      cfg, arm, r["call_ms"], r["device_ms"],
                      ", ".join("%s %.2f" % kv for kv in r["phase_ms"].items()), r["fill_passes"], r["dist_passes"],
                      r["jump_passes"], r["longest_walk"], r["flat_cells"], r["depressed_cells"], r["outlets"]),
                  flush=True)
    print("card:", out["gpu"])
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
