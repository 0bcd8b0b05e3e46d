"""Time sm_relax at the benchmark's size against the single-cell calls (DESIGN.md section 12).

After one frame of config 3 (4096^2 rockgravelpebblessand, 25k water + 25k wind particles, seed 42) and a steep layer
raster (Red Sand piles and pits on 0.5 % of the cells, a cliff line across the map) the map is saved once as a device
snapshot; every timed call starts from a fresh copy of it (sm_snapshot_restore, untimed).  Arms, in alternating order
over the rounds so that drift on a shared machine hits every arm alike:
  pass 1     sm_relax(1, transferloop): every cell visited once
  call       sm_relax(cap, transferloop): passes to stable or the cap, its total and the mean of the passes after the
             first (the late passes, where the stale bits skip most visits)
  cells      sm_cell_cascade over a 64 x 64 window in the canonical order, reported per cell
device_ms is the stats' CUDA-event time around the call's kernels; the host clock around the call ends in a device
synchronise.  Algorithmic bytes of pass 1: per visit the 3 x 3 top records it reads (288 B) and its stale word (4 B),
per transfer two top records written (64 B); over device_ms, against the H100 SXM data-sheet 3.35 TB/s.  The card's name
and power limit are read in the same run.

  python scripts/relax_time.py [--rounds 3] [--dim 4096] [--transferloop 1] [--cap 40] [--json out.json]
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

PEAK = 3.35e12


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except OSError:
        return "unknown"


def steep(rng, dim):
    d = np.zeros((dim, dim))
    n = dim * dim // 200
    xs, ys = rng.integers(0, dim, n), rng.integers(0, dim, n)
    d[xs, ys] = rng.uniform(0.2, 0.8, n)
    xs, ys = rng.integers(0, dim, n // 3), rng.integers(0, dim, n // 3)
    d[xs, ys] = -rng.uniform(0.1, 0.4, n // 3)
    d[dim // 2, :] += 0.3
    return d


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--dim", type=int, default=4096)
    ap.add_argument("--transferloop", type=int, default=1)
    ap.add_argument("--cap", type=int, default=40)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    dim, tl = args.dim, args.transferloop
    sim = host.Simulation("rockgravelpebblessand", seed=42, dimx=dim, dimy=dim, max_particles=25000)
    sim.frame(25000, 25000)
    c = sim.ctx
    sim.apply_layer(steep(np.random.default_rng(42), dim), "Red Sand")
    snap = c.snapshot_device()
    win = 64
    x0 = y0 = dim // 2 - win // 2
    P = 2 * (1 + tl) + 1

    def timed(f):
        c.restore(snap)
        t0 = time.perf_counter()
        st = f()
        return (time.perf_counter() - t0) * 1e3, st

    def cells():
        for p in range(P * P):
            for x in range(x0 + p // P, x0 + win, P):
                for y in range(y0 + p % P, y0 + win, P):
                    c.cell_cascade(x, y, tl)

    arms = {"pass1": lambda: c.relax(1, tl), "call": lambda: c.relax(args.cap, tl), "cells": cells}
    res = {k: [] for k in arms}
    for r in range(args.rounds):
        names = list(arms) if r % 2 == 0 else list(arms)[::-1]
        for k in names:
            ms, st = timed(arms[k])
            res[k].append((ms, st.asdict() if st is not None else None))
    p1 = [s for _, s in res["pass1"]]
    call = [s for _, s in res["call"]]
    pass1_ms = float(np.median([s["device_ms"] for s in p1]))
    call_ms = float(np.median([s["device_ms"] for s in call]))
    s1, sc = p1[0], call[0]
    late = (call_ms - pass1_ms) / max(sc["passes"] - 1, 1)
    bytes1 = s1["visits"] * (288 + 4) + s1["transfers"] * 64
    cell_ms = float(np.median([ms for ms, _ in res["cells"]])) / (win * win)
    out = {
        "gpu": gpu_info(), "dim": dim, "transferloop": tl, "cap": args.cap,
        "pass1_device_ms": pass1_ms, "pass1_host_ms": float(np.median([ms for ms, _ in res["pass1"]])),
        "pass1_visits": s1["visits"], "pass1_transfers": s1["transfers"],
        "pass1_bytes": bytes1, "pass1_GBps": bytes1 / (pass1_ms * 1e-3) / 1e9,
        "pass1_share_of_peak": bytes1 / (pass1_ms * 1e-3) / PEAK,
        "call_passes": sc["passes"], "call_stable": sc["stable"], "call_visits": sc["visits"],
        "call_transfers": sc["transfers"], "call_device_ms": call_ms,
        "call_host_ms": float(np.median([ms for ms, _ in res["call"]])), "late_pass_ms": late,
        "cell_cascade_ms_per_cell": cell_ms, "cell_cascade_whole_map_s": cell_ms * dim * dim / 1e3,
        "rounds": {k: [ms for ms, _ in v] for k, v in res.items()},
        "deterministic": all(s == {**p1[0], "device_ms": s["device_ms"]} for s in p1) and
                         all(s == {**call[0], "device_ms": s["device_ms"]} for s in call),
    }
    print(json.dumps(out, indent=1))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
