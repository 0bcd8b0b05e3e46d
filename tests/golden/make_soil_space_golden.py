"""Generates tests/golden/soil_space.npz from the reference's own code (oracle/_ref/libsmref.so): two soil tables
the presets do not cover (tests/_soil_space.py), so that the device replays them where the reference is absent.

Run where the reference has been built (`make -C oracle ref`):  python tests/golden/make_soil_space_golden.py

  gen/  a generated table: terrain from its layers, a water batch, a wind batch, the frequency update
        (the layout of make_golden.py's frame cases)
  sen/  the water sentinel table: two frames of batch, floods, seep pass and frequency update (the layout of its
        hydro cases); its Tr, Er and Ca sections exist only if the transports, erodes and cascades mappings ran
Every key of a case carries its prefix; tests/test_soil_space.py strips it."""
import os
import sys
import tempfile
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, os.path.dirname(HERE))
from oracle import refapi  # noqa: E402
import _soil_space as sp  # noqa: E402

GEN_SEED, GEN_DIMX, GEN_DIMY, GEN_NW, GEN_ND = 7, 40, 32, 250, 150
SEN_DIM, SEN_N, SEN_FRAMES = 32, 250, 2


def pack_cols(prefix, c, out):
    for k, v in c.items():
        out[prefix + "_" + k] = v


def gen_case(d, out):
    r = refapi.get().init(sp.write(sp.random_table(GEN_SEED), d), seed=GEN_SEED, dimx=GEN_DIMX, dimy=GEN_DIMY)
    o = {"dimx": r.dimx, "dimy": r.dimy, "scale": r.scale, "seed": GEN_SEED, "soils": r.soils(), "layers": r.layers()}
    pack_cols("init", r.columns(), o)
    r.lib.smref_srand(GEN_SEED)
    xw, xd = r.spawn_list(GEN_NW), r.spawn_list(GEN_ND)
    o["water_xy"], o["wind_xy"] = xw, xd
    sw = r.water_run(xw)
    o["water_stats"] = np.array([sw.steps, sw.sweeps, sw.exit_oob, sw.exit_evap, sw.exit_stall], np.int64)
    for k, v in r.water_state().items():
        o["water_state_" + k] = v
    pack_cols("after_water", r.columns(), o)
    sd = r.wind_run(xd)
    o["wind_stats"] = np.array([sd.steps, sd.sweeps, sd.exit_oob, sd.exit_evap, sd.exit_stall], np.int64)
    for k, v in r.wind_state().items():
        o["wind_state_" + k] = v
    r.frequency_update()
    pack_cols("after_frame", r.columns(), o)
    for k, v in r.frequency().items():
        o["freq_" + k] = v
    o["heights"] = r.heights()
    out.update({"gen/" + k: v for k, v in o.items()})
    print("gen", "water", sw.asdict(), "wind", sd.asdict())


def sen_case(d, out):
    r = refapi.get().init(sp.write(sp.sentinel_water(), d), seed=11, dimx=SEN_DIM, dimy=SEN_DIM)
    o = {"dimx": r.dimx, "dimy": r.dimy, "scale": r.scale, "seed": 11, "soils": r.soils(), "layers": r.layers(),
         "frames": SEN_FRAMES}
    pack_cols("init", r.columns(), o)
    r.lib.smref_srand(11)
    floods = []
    for f in range(SEN_FRAMES):
        xy = r.spawn_list(SEN_N)
        o["water_xy_%d" % f] = xy
        r.water_run(xy)
        floods.append(r.water_flood())
        if f == SEN_FRAMES - 1:
            pack_cols("after_flood_%d" % f, r.columns(), o)
        r.seep()
        pack_cols("after_seep_%d" % f, r.columns(), o)
        r.frequency_update()
    o["floods"] = np.array(floods, np.int64)
    for k, v in r.frequency().items():
        o["freq_" + k] = v
    o["heights"] = r.heights()
    out.update({"sen/" + k: v for k, v in o.items()})
    names = [n.decode() for n in r.soils()["name"]]
    print("sen", "floods", floods, "types", sorted(names[t] for t in set(r.columns()["type"].tolist())))


if __name__ == "__main__":
    out = {}
    with tempfile.TemporaryDirectory() as d:
        gen_case(d, out)
        sen_case(d, out)
    np.savez_compressed(os.path.join(HERE, "soil_space.npz"), **out)
