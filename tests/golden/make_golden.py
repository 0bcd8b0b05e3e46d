"""Generates tests/golden/*.npz from the reference's own code (oracle/_ref/libsmref.so).

Run where the reference has been built (`make -C oracle ref`):  python tests/golden/make_golden.py
The reference has no tests or golden vectors of its own (SURVEY.md section 4); these are outputs of the
reference headers compiled verbatim, so every consumer (oracle port, product host build, CUDA path)
is pinned to the same bits.
"""
import os
import sys
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from oracle import refapi  # noqa: E402


def pack_cols(prefix, c, out):
    for k, v in c.items():
        out[prefix + "_" + k] = v


def frame_case(soil, dim, seed, nw, nd, name):
    r = refapi.get().init(soil, seed=seed, dimx=dim, dimy=dim + 8)
    out = {"dimx": r.dimx, "dimy": r.dimy, "scale": r.scale, "seed": seed, "soils": r.soils(), "layers": r.layers()}
    pack_cols("init", r.columns(), out)
    r.lib.smref_srand(seed)
    xw, xd = r.spawn_list(nw), r.spawn_list(nd)
    out["water_xy"], out["wind_xy"] = xw, xd
    sw = r.water_run(xw)
    out["water_stats"] = np.array([sw.steps, sw.sweeps, sw.exit_oob, sw.exit_evap, sw.exit_stall], np.int64)
    for k, v in r.water_state().items():
        out["water_state_" + k] = v
    pack_cols("after_water", r.columns(), out)
    sd = r.wind_run(xd)
    out["wind_stats"] = np.array([sd.steps, sd.sweeps, sd.exit_oob, sd.exit_evap, sd.exit_stall], np.int64)
    for k, v in r.wind_state().items():
        out["wind_state_" + k] = v
    r.frequency_update()
    pack_cols("after_frame", r.columns(), out)
    for k, v in r.frequency().items():
        out["freq_" + k] = v
    out["heights"] = r.heights()
    np.savez_compressed(os.path.join(HERE, name + ".npz"), **out)
    print(name, "water", sw.asdict(), "wind", sd.asdict())


def column_ops_case():
    """Truth table of Layermap::add/remove (SURVEY.md 3.5) + queries, on a hand-made 8x8 map."""
    r = refapi.get().init("rockgravelpebblessand", seed=1, dimx=8, dimy=8)
    cells = 64
    off = np.arange(cells + 1, dtype=np.int64) * 0          # start from an empty map
    r.set_columns(off, np.zeros(0, np.int32), np.zeros(0))
    rng = np.random.RandomState(5)
    ops, res = [], []
    for i in range(600):
        x, y = rng.randint(0, 8, 2)
        kind = rng.randint(0, 10)
        if kind < 5:
            size = [0.05, 0.0, -0.01, 0.2, 1e-9][rng.randint(0, 5)] * rng.rand()
            typ = int(rng.randint(0, 5))              # includes Air (0): exercises the under-water insert
            r.add(x, y, size, typ)
            ops.append((0, x, y, size, typ)); res.append(0.0)
        else:
            h = [0.03, 0.0, -0.5, 0.5, 1e-10][rng.randint(0, 5)] * rng.rand()
            d = r.remove(x, y, h)
            ops.append((1, x, y, h, 0)); res.append(d)
    out = {"soils": r.soils(), "scale": r.scale, "ops": np.array(ops, np.float64), "remove_results": np.array(res)}
    pack_cols("final", r.columns(), out)
    out["heights"] = r.heights()
    out["normals"] = np.array([r.normal(x, y) for x in range(8) for y in range(8)], np.float32)
    pts = rng.rand(64, 2).astype(np.float32) * 6.99
    out["bilinear_pts"] = pts
    out["bilinear"] = np.array([r.height(float(p[0]), float(p[1])) for p in pts])
    # cascades with re-cascade budget 0, 1 and 3 on the resulting rough map
    casc = []
    for i in range(40):
        x, y, loop = float(rng.rand() * 7), float(rng.rand() * 7), int([0, 1, 3][i % 3])
        r.cascade(x, y, loop)
        casc.append((x, y, loop))
    out["cascades"] = np.array(casc, np.float64)
    pack_cols("after_cascade", r.columns(), out)
    np.savez_compressed(os.path.join(HERE, "column_ops.npz"), **out)
    print("column_ops", r.nsections(), "sections")


def hydro_case(soil, dim, seed, n, frames, name):
    """Full water part of the frame in the batch order (SoilMachine.cpp:288-301): lockstep batch, flood() of the
    finished particles in ascending index, the seep pass, the frequency update; columns after every phase."""
    r = refapi.get().init(soil, seed=seed, dimx=dim, dimy=dim + 8)
    out = {"dimx": r.dimx, "dimy": r.dimy, "scale": r.scale, "seed": seed, "soils": r.soils(), "frames": frames}
    pack_cols("init", r.columns(), out)
    r.lib.smref_srand(seed)
    floods = []
    for f in range(frames):
        xy = r.spawn_list(n)
        out["water_xy_%d" % f] = xy
        r.water_run(xy)
        floods.append(r.water_flood())
        if f == frames - 1:                       # one snapshot between the two phases keeps the fixture small
            pack_cols("after_flood_%d" % f, r.columns(), out)
        r.seep()
        pack_cols("after_seep_%d" % f, r.columns(), out)
        r.frequency_update()
    out["floods"] = np.array(floods, np.int64)
    for k, v in r.frequency().items():
        out["freq_" + k] = v
    out["heights"] = r.heights()
    np.savez_compressed(os.path.join(HERE, name + ".npz"), **out)
    c = r.columns()
    print(name, "floods", floods, "air sections", int((c["type"] == 0).sum()), "saturated", int((c["saturation"] > 0).sum()))


def loader_case():
    """What the reference's loadsoil() makes of every preset file in tests/golden/soil (soil table, layer
    table, world scale), and one spawn list drawn the way the particle constructors draw it."""
    import glob
    out = {}
    for path in sorted(glob.glob(os.path.join(HERE, "soil", "*.soil"))):
        name = os.path.basename(path)[:-5]
        r = refapi.get().init(path, seed=0, dimx=8, dimy=8, poolsize=1000)
        out[name + "/soils"], out[name + "/layers"] = r.soils(), r.layers()
        out[name + "/scale"] = np.int64(r.scale)
    r = refapi.get().init("default", seed=5, dimx=100, dimy=70)
    out["spawn_default_100x70_seed5"] = r.spawn_list(64, seed=5)
    np.savez_compressed(os.path.join(HERE, "ref_loader.npz"), **out)
    print("ref_loader", len(out), "arrays")


if __name__ == "__main__":
    if len(sys.argv) > 1 and sys.argv[1] == "loader":
        loader_case()
        sys.exit(0)
    if len(sys.argv) > 1 and sys.argv[1] == "hydro":
        hydro_case("default", 48, 42, 400, 3, "hydro_default_48")
        hydro_case("bigbutte", 40, 3, 500, 3, "hydro_bigbutte_40")
        sys.exit(0)
    column_ops_case()
    frame_case("default", 48, 42, 150, 0, "frame_default_48")
    frame_case("rocksand", 56, 7, 200, 120, "frame_rocksand_56")
    frame_case("rockgravelpebblessand", 64, 42, 250, 150, "frame_rgps_64")
    frame_case("bigbutte", 40, 3, 120, 0, "frame_bigbutte_40")
    hydro_case("default", 48, 42, 400, 3, "hydro_default_48")
    hydro_case("bigbutte", 40, 3, 500, 3, "hydro_bigbutte_40")
