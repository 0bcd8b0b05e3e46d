"""Time the strata views, sm_composition and sm_voxelize, at the benchmark's size (DESIGN.md section 13).

After one frame of config 3 (4096^2 rockgravelpebblessand, 25k water + 25k wind particles, seed 42), each call below
runs with device output (a buffer from sm_device_alloc) and with host output (a numpy array, staged through 32 MB):
  comp_all    composition of every soil over the whole column
  comp_top    composition of every soil in the top 1.0 below the surface
  pore        pore water of every soil over the whole column
  vox64       voxels of the whole map, nz = 64, z from the lowest to the highest height
  row1024     a strata section one row long (x = 0..dimx, y = dimy / 2), nz = 1024
Every shape is run once untimed first; then the arms run in alternating order over the rounds so that drift on a
shared machine hits every arm alike; medians and min..max are reported.  device_ms is the stats' CUDA-event time of the
kernels; the host clock around the call ends with the result in place.  Algorithmic bytes: 32 B per section read plus
the bytes written, over device_ms, against the H100 SXM data-sheet 3.35 TB/s; the walks are chains of dependent loads,
so this is a latency-bound pass and the share says how far it is from the bandwidth bound.  The host path for
comp_all - sm_download_columns plus the numpy statement of tests/_strata.py - is timed once.  The card's name and power
limit are read in the same run.

  python scripts/strata_time.py [--rounds 5] [--dim 4096] [--json out.json]
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
sys.path.insert(0, os.path.join(ROOT, "tests"))
from soilmachine_b200 import host  # noqa: E402

PEAK = 3.35e12


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except OSError:
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--dim", type=int, default=4096)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    dim = args.dim
    sim = host.Simulation("rockgravelpebblessand", seed=42, dimx=dim, dimy=dim, max_particles=25000)
    sim.frame(25000, 25000)
    c = sim.ctx
    ns = len(sim.preset["soils"])
    allt = list(range(ns))
    H = c.heights()
    zlo, zhi = float(H.min()), float(H.max())
    shapes = {
        "comp_all": ("c", (allt, -np.inf, np.inf, False, False), ns * dim * dim * 8),
        "comp_top": ("c", (allt, 0.0, 1.0, True, False), ns * dim * dim * 8),
        "pore": ("c", (allt, -np.inf, np.inf, False, True), ns * dim * dim * 8),
        "vox64": ("v", (0, dim, 0, dim, zlo, (zhi - zlo) / 64, 64), 64 * dim * dim),
        "row1024": ("v", (0, dim, dim // 2, dim // 2 + 1, zlo, (zhi - zlo) / 1024, 1024), 1024 * dim),
    }
    bufs = {}
    for k, (_, _, nbytes) in shapes.items():
        d = C.c_void_p()
        c._ck(c.lib.sm_device_alloc(c.h, C.c_int64(nbytes), C.byref(d)))
        bufs[k] = d

    def run(k, dev):
        kind, a, _ = shapes[k]
        out = bufs[k] if dev else None
        t0 = time.perf_counter()
        if kind == "c":
            c.composition(*a, out=out)
        else:
            c.voxelize(*a, out=out)
        if dev:
            c.sync()
        return (time.perf_counter() - t0) * 1e3, c.view_stats.asdict()

    arms = [(k, dev) for k in shapes for dev in (True, False)]
    for k, dev in arms:
        run(k, dev)                                   # warm-up of every shape
    res = {a: [] for a in arms}
    for r in range(args.rounds):
        for a in (arms if r % 2 == 0 else arms[::-1]):
            res[a].append(run(*a))
    out = {"gpu": gpu_info(), "dim": dim, "soils": ns, "rounds": args.rounds, "calls": {}}
    for k in shapes:
        row = {}
        for dev in (True, False):
            ms = [m for m, _ in res[(k, dev)]]
            dms = [s["device_ms"] for _, s in res[(k, dev)]]
            st = res[(k, dev)][0][1]
            nbytes = 32 * st["sections"] + st["bytes_out"]
            tag = "device_out" if dev else "host_out"
            row[tag] = {"host_ms": float(np.median(ms)), "host_ms_range": [float(min(ms)), float(max(ms))],
                        "device_ms": float(np.median(dms)), "device_ms_range": [float(min(dms)), float(max(dms))],
                        "sections": st["sections"], "bytes_out": st["bytes_out"], "algorithmic_bytes": nbytes,
                        "GBps": nbytes / (float(np.median(dms)) * 1e-3) / 1e9,
                        "share_of_3.35TBps": nbytes / (float(np.median(dms)) * 1e-3) / PEAK}
        out["calls"][k] = row
    import _strata
    t0 = time.perf_counter()
    cols = c.download_columns()
    t1 = time.perf_counter()
    por = np.zeros(64, np.float32)
    por[:ns] = sim.preset["soils"]["porosity"]
    ref = _strata.composition(cols, por, allt, -np.inf, np.inf)
    t2 = time.perf_counter()
    out["host_path_comp_all"] = {"download_columns_ms": (t1 - t0) * 1e3, "numpy_statement_ms": (t2 - t1) * 1e3,
                                 "equal": bool(np.array_equal(ref.reshape(-1).view(np.uint8),
                                                              c.composition(allt, -np.inf, np.inf).reshape(-1).view(np.uint8)))}
    for d in bufs.values():
        c.device_free(d)
    sim.close()
    print(json.dumps(out, indent=1))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
