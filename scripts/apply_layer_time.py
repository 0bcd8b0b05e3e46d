"""Time sm_apply_layer against the writes that existed before it, at the benchmark's size (DESIGN.md section 11).

After one frame of config 3 (4096^2 rockgravelpebblessand, 25k water + 25k wind particles, seed 42) the map is saved
once as a device snapshot; every timed call starts from a fresh copy of it (sm_snapshot_restore, untimed).  Arms, in
alternating order over the rounds so that drift on a shared machine hits every arm alike:
  raster host    sm_apply_layer with a dense +-0.01 raster (every cell non-zero, random sign) from host memory
  raster device  the same raster already in device memory
  cells          the same edit over a 64 x 64 window through sm_cell_add / sm_cell_remove (remove repeated while it
                 returns height), reported per cell
  snapshot       sm_snapshot_save + sm_snapshot_restore in device memory, the cheapest whole-map rewrite before
For the rasters: the host clock around the call (it ends in a device synchronise), the stats' device_ms (CUDA events
around k_layer_check and k_layer_apply), and the algorithmic bytes of the two kernels over device_ms against the
H100 SXM data-sheet 3.35 TB/s.  Bytes: check 8 B per cell (delta) + 32 B per deposit (top record); apply 8 B per cell
(delta) + 64 B per touched cell (top record read and written) + 32 B per pushed record (stored) + 32 B per popped record
(read).  Pops = sections before + pushed - sections after.  The card's name and power limit are read in the same run.

  python scripts/apply_layer_time.py [--rounds 5] [--dim 4096] [--json out.json]
"""
import argparse
import ctypes as C
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
    snap = c.snapshot_device()
    sec0 = c.section_count()
    typ = len(sim.preset["soils"]) - 1
    rng = np.random.default_rng(42)
    delta = np.where(rng.random((dim, dim)) < 0.5, 0.01, -0.01)
    dd = C.c_void_p()
    c._ck_strict(c.lib.sm_device_alloc(c.h, C.c_int64(delta.nbytes), C.byref(dd)))
    c._ck_strict(c.lib.sm_device_upload(c.h, dd, delta.ctypes.data_as(C.c_void_p), C.c_int64(delta.nbytes)))
    win = 64
    x0 = y0 = dim // 2 - win // 2

    def fresh():
        c.restore(snap)

    def raster(on_device):
        t0 = time.perf_counter()
        st, _ = c.apply_layer(dd if on_device else delta, typ)
        return (time.perf_counter() - t0) * 1e3, st

    def cells():
        t0 = time.perf_counter()
        for x in range(x0, x0 + win):
            for y in range(y0, y0 + win):
                v = delta[x, y]
                if v > 0:
                    c.cell_add(x, y, v, typ)
                else:
                    left, k = -v, 0
                    while left > 0 and k < 64:
                        left = c.cell_remove(x, y, left)
                        k += 1
        return (time.perf_counter() - t0) * 1e3 / (win * win)

    def snapshot_rw():
        t0 = time.perf_counter()
        c._ck_strict(c.lib.sm_snapshot_save(c.h, snap[0], C.c_int64(snap[1]), 1))
        c._ck_strict(c.lib.sm_snapshot_restore(c.h, snap[0], C.c_int64(snap[1]), 1))
        return (time.perf_counter() - t0) * 1e3

    fresh(); raster(False); fresh(); raster(True); fresh(); cells(); fresh(); snapshot_rw()     # warm-up
    fresh()
    st, _ = c.apply_layer(delta, typ)
    sec1 = c.section_count()
    ncell = dim * dim
    deposits = int((delta > 0).sum())
    pops = sec0 + st.pushed - sec1
    nbytes = 8 * ncell + 32 * deposits + 8 * ncell + 64 * st.cells + 32 * st.pushed + 32 * pops
    res = {k: [] for k in ("raster host", "raster device", "cells", "snapshot")}
    for r in range(args.rounds):
        order = list(res) if r % 2 == 0 else list(res)[::-1]
        for k in order:
            fresh()
            if k == "cells":
                res[k].append(cells())
            elif k == "snapshot":
                res[k].append(snapshot_rw())
            else:
                ms, s = raster(k == "raster device")
                res[k].append((ms, s.device_ms))
    gpu = gpu_info()
    out = {"gpu (name, power limit)": gpu, "dim": dim, "cells": ncell, "sections_before": sec0, "pushed": st.pushed,
           "pops": pops, "free_slots": st.free_slots, "algorithmic_bytes": nbytes, "rounds": args.rounds, "arms": res}
    print("apply_layer timing on %s, %d^2, %d sections, dense +-0.01 raster of soil %d: %d pushed, %d popped, "
          "%.2f GB algorithmic, %d rounds (median, min)" % (gpu, dim, sec0, typ, st.pushed, pops, nbytes / 1e9,
                                                            args.rounds))
    for k in ("raster host", "raster device"):
        hm = np.array([t[0] for t in res[k]]); em = np.array([t[1] for t in res[k]])
        out[k] = {"device_ms_median": float(np.median(em)), "GB/s": nbytes / np.median(em) / 1e6,
                  "share_of_3.35TB/s": nbytes / (np.median(em) * 1e-3) / PEAK}
        print("  %-14s host %8.2f %8.2f ms   kernels %7.3f %7.3f ms   %7.0f GB/s = %.0f %% of 3.35 TB/s"
              % (k, np.median(hm), hm.min(), np.median(em), em.min(), out[k]["GB/s"], 100 * out[k]["share_of_3.35TB/s"]))
    a = np.array(res["cells"])
    print("  %-14s %8.4f %8.4f ms per cell (64 x 64 window), %.1f s for the whole map at that rate"
          % ("cells", np.median(a), a.min(), np.median(a) * ncell / 1e3))
    a = np.array(res["snapshot"])
    print("  %-14s %8.2f %8.2f ms (save + restore, device memory)" % ("snapshot", np.median(a), a.min()))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)
    c.lib.sm_device_free(c.h, dd)
    c.device_free(snap[0])
    sim.close()


if __name__ == "__main__":
    main()
