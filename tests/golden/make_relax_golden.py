"""Generates tests/golden/relax_ops.npz: slope relaxation by the reference's own Particle::cascade
(oracle/_ref/libsmref.so, smref_cascade), driven in sm_relax's canonical order, the truth sm_relax is pinned to.

Run where the reference has been built (`make -C oracle ref`):  python tests/golden/make_relax_golden.py

For each case: a golden terrain (tests/golden/<terrain>.npz, columns `<prefix>_*`: after its batches, or after its
floods and seep passes, with standing water on top) or a flat map, loaded into the reference and made steep by one layer
raster of one soil type applied with the reference's add / remove (the loop of make_layer_golden.py): piles, pits and a
cliff line.  The golden terrains are steeper than their soils' maxdiff almost everywhere, so their passes go on for
thousands of passes; the flat maps relax around the edits only and reach a pass that changes nothing.  Then, for
transferloop 0, 1 and 3, from that steep map, passes of

    R = 1 + transferloop; P = 2R + 1
    for p in 0 .. P*P-1: for x = p / P; x < dimx; x += P: for y = p % P; y < dimy; y += P: cascade(vec2(x, y), tl)

until a pass changes nothing (and at least K passes have run) or the case's cap is reached.
Stored per case c: c_soil, c_terrain, c_prefix ("" for a flat map), c_dimx, c_dimy, c_type, c_delta (the raster),
c_sum_in / c_nsec_in (the steep map); per transferloop t: c_t<t>_sums and c_t<t>_nsec (checksum.columns_checksum and
section count after every pass), c_t<t>_passes (passes run), c_t<t>_stable (the first pass that changed nothing, 0 if
none), c_t<t>_changes (columns each pass changed, the reference's columns compared cell by cell), and for the flat maps
the columns after K passes as the cells that differ from the steep map: c_t<t>_cells and their CSR c_t<t>_out_*.  c_soils
is the soil table the reference loaded.  (Whole columns of the golden terrains after K passes would make the file
several MB: almost every cell changes in every pass; their per-pass checksums pin them.)
"""
import os
import sys
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
from oracle import refapi  # noqa: E402
import _golden  # noqa: E402
from soilmachine_b200 import checksum  # noqa: E402
from make_layer_golden import ref_strip  # noqa: E402

# (case, preset, terrain, prefix, soil type of the raster, MAX_PASSES).  terrain None: a flat map of DIM x DIM cells, one
# section of type 1 and height 0.5 per cell, so that the edits relax locally and a stable pass is reached.
CASES = [("default", "default", "frame_default_48", "after_frame", 1, 6),
         ("rgps", "rockgravelpebblessand", "frame_rgps_64", "after_frame", 3, 6),
         ("water", "default", "hydro_default_48", "after_seep_2", 1, 6),
         ("flat_bigbutte", "bigbutte", None, None, 2, 6),
         ("flat_settling1", "settling1", None, None, 2, 200)]
# "settling1": rocksand.soil with SETTLING 1.0 for both soils, so that a transfer levels a pair to maxdiff and the
# passes reach a stable map
SETTLING1 = ("rocksand", "SETTLING 1.0")
DIM = 48
LOOPS = (0, 1, 3)
K = 3                 # the columns after K passes are stored (the cells that differ from the steep map)


def soil_file(soil, tmp):
    if soil != "settling1":
        return soil
    text = open(refapi.soil_path(SETTLING1[0])).read()
    text = "\n".join(SETTLING1[1] if l.strip().startswith("SETTLING") else l for l in text.split("\n"))
    path = os.path.join(tmp, "settling1.soil")
    with open(path, "w") as f:
        f.write(text)
    return path


def flat(dim):
    n = dim * dim
    return {"offsets": np.arange(n + 1, dtype=np.int64), "type": np.ones(n, np.int32), "size": np.full(n, 0.5),
            "floor": np.zeros(n), "saturation": np.zeros(n)}


def steep_raster(rng, dimx, dimy, amp):
    """piles (single cells and 2x2 blocks), pits, and a cliff line across the map; heights amp times multiples of 2^-12
    (a pile of height h relaxes to a cone of radius h / maxdiff: the flat maps use amp = 1/16)"""
    q = amp * 2.0 ** -12
    d = np.zeros((dimx, dimy))
    for _ in range(10):
        x, y = rng.integers(1, dimx - 2), rng.integers(1, dimy - 2)
        d[x:x + rng.integers(1, 3), y:y + rng.integers(1, 3)] += rng.integers(int(0.3 / q), int(0.9 / q)) * q
    for _ in range(8):
        x, y = rng.integers(0, dimx), rng.integers(0, dimy)
        d[x, y] = -rng.integers(int(0.2 / q), int(0.6 / q)) * q
    d[dimx // 2, :] += 0.375 * amp
    d[dimx // 2 + 1, : dimy // 2] += 0.25 * amp
    return d.reshape(-1)


def apply_raster(r, d, t, dimy):
    before = r.columns()
    off, size = before["offsets"], before["size"]
    for i in np.nonzero(d)[0]:
        x, y = divmod(int(i), dimy)
        if d[i] > 0:
            r.add(x, y, d[i], t)
        else:
            ref_strip(r, x, y, -d[i], size[off[i]:off[i + 1]])


def relax_pass(r, dimx, dimy, tl):
    P = 2 * (1 + tl) + 1
    for p in range(P * P):
        for x in range(p // P, dimx, P):
            for y in range(p % P, dimy, P):
                r.cascade(x, y, tl)


def cell_bytes(cols, i):
    a, b = int(cols["offsets"][i]), int(cols["offsets"][i + 1])
    return b"".join(np.ascontiguousarray(cols[k][a:b]).tobytes() for k in ("type", "size", "floor", "saturation"))


def changed_cells(a, b, cells):
    return [i for i in range(cells) if cell_bytes(a, i) != cell_bytes(b, i)]


def sub_csr(cols, cells):
    out = {"offsets": [0], "type": [], "size": [], "floor": [], "saturation": []}
    for i in cells:
        a, b = int(cols["offsets"][i]), int(cols["offsets"][i + 1])
        for k in ("type", "size", "floor", "saturation"):
            out[k].append(np.asarray(cols[k][a:b]))
        out["offsets"].append(out["offsets"][-1] + b - a)
    res = {"offsets": np.array(out["offsets"], np.int64)}
    for k, dt in (("type", np.int32), ("size", np.float64), ("floor", np.float64), ("saturation", np.float64)):
        res[k] = np.concatenate(out[k]).astype(dt) if out[k] else np.zeros(0, dt)
    return res


def main():
    import tempfile
    tmp = tempfile.mkdtemp()
    r = refapi.get()
    out = {"cases": np.array([c[0] for c in CASES]), "loops": np.array(LOOPS, np.int32)}
    for ci, (name, soil, terrain, prefix, t, max_passes) in enumerate(CASES):
        if terrain:
            g = _golden.load(terrain)
            dimx, dimy = int(g["dimx"]), int(g["dimy"])
            c = _golden.cols(g, prefix)
        else:
            dimx = dimy = DIM
            c = flat(DIM)
        r.init(soil_file(soil, tmp), dimx=dimx, dimy=dimy, poolsize=32 * dimx * dimy)
        r.set_columns(c["offsets"], c["type"], c["size"], c["saturation"])
        d = steep_raster(np.random.default_rng(500 + ci), dimx, dimy, 1.0 if terrain else 1.0 / 16)
        apply_raster(r, d, t, dimy)
        steep = r.columns()
        out.update({"%s_soil" % name: np.array(soil), "%s_terrain" % name: np.array(terrain or ""),
                    "%s_prefix" % name: np.array(prefix or ""), "%s_dimx" % name: np.int32(dimx),
                    "%s_dimy" % name: np.int32(dimy), "%s_soils" % name: r.soils(),
                    "%s_type" % name: np.int32(t), "%s_delta" % name: d,
                    "%s_sum_in" % name: np.uint64(checksum.columns_checksum(steep)),
                    "%s_nsec_in" % name: np.int64(steep["offsets"][-1])})
        for tl in LOOPS:
            r.set_columns(steep["offsets"], steep["type"], steep["size"], steep["saturation"])
            assert checksum.columns_checksum(r.columns()) == checksum.columns_checksum(steep)
            key = "%s_t%d_" % (name, tl)
            prev, stable, changes, sums, nsec = steep, 0, [], [], []
            for k in range(1, max_passes + 1):
                relax_pass(r, dimx, dimy, tl)
                now = r.columns()
                changes.append(len(changed_cells(prev, now, dimx * dimy)))
                sums.append(checksum.columns_checksum(now))
                nsec.append(int(now["offsets"][-1]))
                if k == K and not terrain:
                    cells = changed_cells(steep, now, dimx * dimy)
                    out[key + "cells"] = np.array(cells, np.int32)
                    for kk, v in sub_csr(now, cells).items():
                        out[key + "out_" + kk] = v
                prev = now
                if changes[-1] == 0 and not stable:
                    stable = k
                if stable and k >= K:
                    break
            out[key + "stable"] = np.int32(stable)
            out[key + "passes"] = np.int32(len(changes))
            out[key + "changes"] = np.array(changes, np.int64)
            out[key + "sums"] = np.array(sums, np.uint64)
            out[key + "nsec"] = np.array(nsec, np.int64)
            print(name, "transferloop", tl, "passes", len(changes), "stable", stable, "changes", changes[:6],
                  "cells after K", len(out.get(key + "cells", [])))
    np.savez_compressed(os.path.join(HERE, "relax_ops.npz"), **out)
    print("bytes", os.path.getsize(os.path.join(HERE, "relax_ops.npz")))


if __name__ == "__main__":
    main()
