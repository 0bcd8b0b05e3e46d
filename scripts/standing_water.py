"""Standing water under three frame orders, on the reference's own code (CPU; needs oracle/_ref/libsmref_flooding.so:
`make -C oracle ref && make -C oracle -f flooding.mk`).

From the same srand(seed) and terrain, F frames of N water particles each, then the seep pass and the frequency update:
  seq    upstream: each particle runs to completion and floods right after its own loop (smref_water_seq)
  batch  one lockstep batch, then the floods of its finished particles (sm_water_run + sm_water_flood)
  sweep  one lockstep batch whose particles flood at the end of the sweep they stop in (sm_water_run_flooding)
Per frame: standing water (sum of the Air sections' sizes), wet cells (Air on top), mean and variance of the height.

    python scripts/standing_water.py --soil default --dim 256 --n 250 --frames 8
"""
import argparse
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import refapi_flooding  # noqa: E402


def measure(r):
    c = r.columns()
    air = c["type"] == 0
    top = c["offsets"][1:] - 1
    nonempty = np.diff(c["offsets"]) > 0
    h = r.heights()
    return (float(c["size"][air].sum()), int(air[top[nonempty]].sum()), float(h.mean()), float(h.var()))


def run(order, soil, dim, n, frames, seed):
    r = refapi_flooding.get().init(soil, seed=seed, dimx=dim, dimy=dim, poolsize=max(10000000, dim * dim * 12))
    r.lib.smref_srand(seed)
    rows = []
    for _ in range(frames):
        if order == "seq":
            r.water_seq(n, flood=True, seep=True)
        else:
            xy = r.spawn_list(n)
            if order == "batch":
                r.water_run(xy)
                r.water_flood()
            else:
                r.water_sweep_flood(xy)
            r.seep()
        r.frequency_update()
        rows.append(measure(r))
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--soil", default="default")
    ap.add_argument("--dim", type=int, default=256)
    ap.add_argument("--n", type=int, default=250)
    ap.add_argument("--frames", type=int, default=8)
    ap.add_argument("--seed", type=int, default=42)
    a = ap.parse_args()
    if not refapi_flooding.available():
        sys.exit("oracle/_ref/libsmref_flooding.so is not built")
    res = {o: run(o, a.soil, a.dim, a.n, a.frames, a.seed) for o in ("seq", "batch", "sweep")}
    print("%s %d^2, %d water particles per frame, seed %d" % (a.soil, a.dim, a.n, a.seed))
    print("| frame | order | standing water | wet cells | mean height | height variance |")
    print("|---|---|---|---|---|---|")
    for f in range(a.frames):
        for o in ("seq", "batch", "sweep"):
            w, wet, m, v = res[o][f]
            print("| %d | %s | %.4f | %d | %.6f | %.6f |" % (f + 1, o, w, wet, m, v))


if __name__ == "__main__":
    main()
