"""Generates tests/golden/layer_ops.npz: layer rasters applied by the reference's own Layermap::add / remove
(oracle/_ref/libsmref.so), the truth sm_apply_layer is pinned to.

Run where the reference has been built (`make -C oracle ref`):  python tests/golden/make_layer_golden.py

For each case: the columns x < CROP of a golden terrain (tests/golden/<case>.npz, columns `<prefix>_*`) after its
particle batches (frame cases) or after its floods and seep passes (hydrology cases, which have standing water on top),
loaded into the reference, then a sequence of rasters, one soil type each, every type of the preset once, Air first and
last, each applied to the result of the one before.  Each raster is applied cell by cell, in x-major order: delta > 0 is
one add(pos, sec(delta, type)), delta < 0 the strip loop of include/soilmachine_b200.h over remove(), +-0.0 nothing.
The rasters mix deposits, strips, +0.0, -0.0, tiny values and strips deeper than the column; their ordinary values are
multiples of 2^-16, which keeps the file small.
Stored per case c: c_prefix, c_dimy, c_nsoils, c_nrasters; per raster k: c_delta_k, c_type_k, c_left_k (leftovers),
c_sum_k and c_nsec_k (checksum.columns_checksum and section count of the columns after raster k); and c_out_* (all
columns after the last raster).  The input columns are not stored: they are the crop of the golden terrain, which the
reference holds unchanged after set_columns (checked here).
"""
import os
import sys
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, os.path.dirname(HERE))
from oracle import refapi  # noqa: E402
import _golden  # noqa: E402
from soilmachine_b200 import checksum  # noqa: E402

CASES = [("frame_default_48", "after_frame"), ("frame_rocksand_56", "after_frame"), ("frame_bigbutte_40", "after_frame"),
         ("hydro_default_48", "after_seep_2"), ("hydro_bigbutte_40", "after_seep_2")]
CROP = 16     # the columns x < CROP of each terrain: a map of CROP x dimy cells keeps the fixture small


def ref_strip(r, x, y, h, sizes):
    """strip h of height with the reference's remove(): the loop of sm_apply_layer.  sizes: the column's section sizes
    bottom -> top as the reference held them before this raster (the loop only pops, so the section under a popped top
    is the next one down and the top is NULL once they are used up)"""
    left = h
    j = len(sizes) - 1
    while left > 0 and j >= 0:
        empty_top = sizes[j] <= 0
        rest = r.remove(x, y, left)
        if not empty_top:
            left = rest
        j -= 1
    return left


def crop(cols, cells):
    """the CSR of the first `cells` cells"""
    n = int(cols["offsets"][cells])
    return {k: np.asarray(v[:cells + 1] if k == "offsets" else v[:n]) for k, v in cols.items()}


def raster(rng, cells):
    """deposits, strips, +-0.0, tiny values and strips deeper than any column (heights stay below 1.5)"""
    u = rng.random(cells)
    q = 2.0 ** -16
    d = np.where(u < 0.35, rng.integers(1, int(0.08 / q), cells) * q, -rng.integers(1, int(0.15 / q), cells) * q)
    d[(u >= 0.70) & (u < 0.80)] = -rng.integers(int(1.5 / q), int(3.0 / q), int(((u >= 0.70) & (u < 0.80)).sum())) * q
    d[(u >= 0.80) & (u < 0.83)] = rng.choice([1e-12, -1e-12, 5e-324, -5e-324], int(((u >= 0.80) & (u < 0.83)).sum()))
    d[(u >= 0.83) & (u < 0.95)] = 0.0
    d[u >= 0.95] = -0.0
    return d


def main():
    r = refapi.get()
    out = {"cases": np.array([c for c, _ in CASES])}
    for ci, (name, prefix) in enumerate(CASES):
        g = _golden.load(name)
        dimx, dimy = CROP, int(g["dimy"])
        r.init(name.split("_")[1], dimx=dimx, dimy=dimy, poolsize=32 * dimx * dimy)
        c = crop(_golden.cols(g, prefix), dimx * dimy)
        r.set_columns(c["offsets"], c["type"], c["size"], c["saturation"])
        ns = len(r.soils())
        got = r.columns()
        assert all(np.asarray(got[k]).tobytes() == np.asarray(c[k]).tobytes() for k in c), name + ": input changed"
        out["%s_prefix" % name] = np.array(prefix)
        out["%s_dimy" % name] = np.int32(dimy)
        rng = np.random.default_rng(1000 + ci)
        types = list(range(ns)) + [0]
        for k, t in enumerate(types):
            d = raster(rng, dimx * dimy)
            left = np.zeros(dimx * dimy)
            before = r.columns()
            off, size = before["offsets"], before["size"]
            for x in range(dimx):
                for y in range(dimy):
                    v = d[x * dimy + y]
                    if v > 0:
                        r.add(x, y, v, t)
                    elif v < 0:
                        i = x * dimy + y
                        left[i] = ref_strip(r, x, y, -v, size[off[i]:off[i + 1]])
            out["%s_delta_%d" % (name, k)] = d
            out["%s_type_%d" % (name, k)] = np.int32(t)
            out["%s_left_%d" % (name, k)] = left
            after = r.columns()
            out["%s_sum_%d" % (name, k)] = np.uint64(checksum.columns_checksum(after))
            out["%s_nsec_%d" % (name, k)] = np.int64(after["offsets"][-1])
        for kk, v in after.items():
            out["%s_out_%s" % (name, kk)] = v
        out["%s_nrasters" % name] = np.int32(len(types))
        out["%s_nsoils" % name] = np.int32(ns)
        print(name, "rasters", len(types), "sections in/out", len(c["type"]), len(after["type"]), "emptied",
              [int((out["%s_left_%d" % (name, k)] > 0).sum()) for k in range(len(types))])
    np.savez_compressed(os.path.join(HERE, "layer_ops.npz"), **out)


if __name__ == "__main__":
    main()
