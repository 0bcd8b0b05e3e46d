"""Generates tests/golden/sweep_flood_ops.npz from the reference's own code: water batches in the sweep-flood order
(oracle/refharness/sweep_flood.cpp, oracle/_ref/libsmref_flooding.so): after every lockstep sweep the particles that
stopped in it flood(), ascending index, before the next sweep.

Run where the reference has been built (`make -C oracle ref && make -C oracle -f flooding.mk`):
    python tests/golden/make_sweep_flood_golden.py
Per case: the soil and layer tables (the terrain is Layermap(SEED, dim), which sm_initialize reproduces) and the
checksum of the initial columns; batch 0, a whole batch; batch 1, a batch cut after `cut` sweeps.  After each batch:
the column checksum (soilmachine_b200.checksum), the particle states, the stats (steps, sweeps, oob, evap, stall) and
the flood count; after the last one the columns themselves (two cases), the frequency maps and heights.
"""
import os
import sys
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from oracle import refapi_flooding  # noqa: E402
from soilmachine_b200.checksum import columns_checksum  # noqa: E402

# (soil, dim, seed, particles per batch, sweeps of the cut batch, name, keep the final columns)
CASES = [("default", 48, 42, 400, 20, "default_48", True), ("bigbutte", 40, 3, 500, 40, "bigbutte_40", True),
         ("rocksand", 56, 7, 500, 80, "rocksand_56", False)]


def pack_cols(prefix, c, out):
    for k, v in c.items():
        out[prefix + "_" + k] = v


def case(r, soil, dim, seed, n, cut, name, keep, out):
    r.init(soil, seed=seed, dimx=dim, dimy=dim + 8)
    p = name + "/"
    out[p + "dims"] = np.array([r.dimx, r.dimy, r.scale, seed], np.int64)
    out[p + "soils"], out[p + "layers"] = r.soils(), r.layers()
    out[p + "checksum_init"] = np.uint64(columns_checksum(r.columns()))
    r.lib.smref_srand(seed)
    floods = []
    for b, ms in enumerate((0, cut)):
        xy = r.spawn_list(n)
        out[p + "xy_%d" % b] = xy
        st, nfl = r.water_sweep_flood(xy, ms)
        out[p + "stats_%d" % b] = np.array([st.steps, st.sweeps, st.exit_oob, st.exit_evap, st.exit_stall], np.int64)
        out[p + "floods_%d" % b] = np.int64(nfl)
        for k, v in r.water_state().items():
            out[p + "state_%d_%s" % (b, k)] = v
        out[p + "checksum_%d" % b] = np.uint64(columns_checksum(r.columns()))
        floods.append(nfl)
    if keep:                  # rocksand's thin sections make 600 KB of columns: its checksums stand for them
        pack_cols(p + "final", r.columns(), out)
    for k, v in r.frequency().items():
        out[p + "freq_" + k] = v
    out[p + "heights"] = r.heights()
    c = r.columns()
    print(name, "floods", floods, "stats", out[p + "stats_0"].tolist(), out[p + "stats_1"].tolist(),
          "air sections", int((c["type"] == 0).sum()))


if __name__ == "__main__":
    r = refapi_flooding.get()
    out = {"cases": np.array([c[5] for c in CASES])}
    for c in CASES:
        case(r, *c, out)
    np.savez_compressed(os.path.join(HERE, "sweep_flood_ops.npz"), **out)
