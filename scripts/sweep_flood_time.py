"""Time the sweep-flood water batch (sm_water_run_flooding) against the batch order (sm_water_run + sm_water_flood)
on the same map and spawn list (DESIGN.md K6 "Sweep floods").

Sizes: config 2 (1024^2 rocksand, 10 000 water particles) and config 3 (4096^2 rockgravelpebblessand, 25 000), seed
42.  After one frame with its floods and seep pass the map is saved as a device snapshot; every timed call starts from
a fresh copy of it (untimed restore).  The two arms alternate over the rounds so that drift on a shared machine hits
both alike.  Reported per arm: device time (CUDA events: the call's own for the sweep-flood arm, run + flood for the
batch arm), host time around the calls ending in a device synchronise, kernel launches, and the flood count.  The
card's name and power limit are read in the same run.

  python scripts/sweep_flood_time.py [--rounds 5] [--configs 2,3] [--json out.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from soilmachine_b200 import host  # noqa: E402

CONFIGS = {2: ("rocksand", 1024, 10000), 3: ("rockgravelpebblessand", 4096, 25000)}


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except OSError:
        return "unknown"


def arm(c, which, xy):
    l0 = c.launch_count()
    c.sync()
    t0 = time.perf_counter()
    if which == "sweep":
        st, hs = c.water_run_flooding(xy)
        dev = st.device_ms
    else:
        st = c.water_run(xy)
        hs = c.water_flood()
        dev = st.device_ms + hs.device_ms
    c.sync()
    host_ms = (time.perf_counter() - t0) * 1e3
    return {"device_ms": dev, "host_ms": host_ms, "launches": c.launch_count() - l0, "floods": hs.floods,
            "nested": hs.nested, "steps": st.steps, "sweeps": st.sweeps, "checksum": "%016x" % c.checksum()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--configs", default="2,3")
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    info = gpu_info()
    print("GPU:", info)
    report = {"gpu": info, "configs": {}}
    for k in [int(x) for x in a.configs.split(",")]:
        soil, dim, n = CONFIGS[k]
        sim = host.Simulation(soil, seed=42, dimx=dim, dimy=dim, max_particles=n)
        sim.frame(n, 0, hydrology=True)
        c = sim.ctx
        xy = host.spawn_list(n, dim, dim)
        snap = c.snapshot_device()
        runs = {"batch": [], "sweep": []}
        for r in range(a.rounds + 1):                       # round 0 warms both arms up and is not reported
            for which in (("batch", "sweep") if r % 2 == 0 else ("sweep", "batch")):
                c.restore(snap)
                res = arm(c, which, xy)
                if r:
                    runs[which].append(res)
        out = {}
        for which, rs in runs.items():
            d = np.array([x["device_ms"] for x in rs])
            h = np.array([x["host_ms"] for x in rs])
            out[which] = {"device_ms_median": float(np.median(d)), "device_ms_min": float(d.min()),
                          "device_ms_max": float(d.max()), "host_ms_median": float(np.median(h)),
                          "launches": rs[0]["launches"], "floods": rs[0]["floods"], "nested": rs[0]["nested"],
                          "steps": rs[0]["steps"], "sweeps": rs[0]["sweeps"],
                          "deterministic": len({x["checksum"] for x in rs}) == 1}
            print("config %d %s: device %.2f ms (min %.2f, max %.2f), host %.2f ms, %d launches, %d floods, "
                  "%d nested, %d steps, %d sweeps, same checksum every round: %s" % (
                      k, which, out[which]["device_ms_median"], d.min(), d.max(), out[which]["host_ms_median"],
                      out[which]["launches"], out[which]["floods"], out[which]["nested"], out[which]["steps"],
                      out[which]["sweeps"], out[which]["deterministic"]))
        report["configs"][k] = out
        c.device_free(snap[0])
        c.close()
    if a.json:
        with open(a.json, "w") as f:
            json.dump(report, f, indent=1)


if __name__ == "__main__":
    main()
