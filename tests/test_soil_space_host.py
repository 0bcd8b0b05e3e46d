"""CPU: soil tables beyond the shipped presets (tests/_soil_space.py).  The library's parser against the reference's
loadsoil on generated files, and the reference, the oracle port and the product's step compiled for the host
(tests/hostsim) against each other over two frames of the whole frame loop on generated and sentinel tables, and
on terrain from generated layers.  The device tests (tests/test_soil_space.py) that run without the reference lean
on the port, which these tests pin to the reference on the same tables."""
import numpy as np
import pytest
import _golden
import _soil_space as sp
from oracle import portapi

PARSE_SEEDS = list(range(100, 130))
FRAME_CASES = [(2, 64, 64), (7, 3, 96), (11, 97, 61), (18, 48, 56), (22, 64, 56), (26, 52, 60), (49, 2, 80),
               (57, 56, 48)]
INIT_SEEDS = list(range(200, 220))


def _tables():
    return [sp.random_table(s) for s in PARSE_SEEDS] + [f() for f in sp.SENTINELS.values()] + [sp.table_64()]


def test_parser_reads_what_the_writer_wrote(tmp_path):
    """sm_parse_soil_file on every generated file: the values written (as float32), the chains by name, the layers
    in order, Air as soil 0 - no reference needed"""
    from soilmachine_b200 import capi
    for t in _tables():
        p = capi.parse_soil_file(sp.write(t, tmp_path))
        names = p["soil_names"]
        assert names[0] == "Air" and sorted(names[1:]) == sorted(s["name"] for s in t["soils"]), t["name"]
        if t.get("declare", True):
            assert names[1:] == [s["name"] for s in t["soils"]], t["name"]
        for s in t["soils"]:
            row = p["soils"][names.index(s["name"])]
            for _, k in sp.CHAINS:
                assert row[k] == names.index(s[k]), (t["name"], s["name"], k)
            for _, k in sp.FLOATS:
                assert row[k].tobytes() == np.float32(s[k]).tobytes(), (t["name"], s["name"], k)
        assert len(p["layers"]) == len(t["layers"])
        for row, l in zip(p["layers"], t["layers"]):
            assert row["type"] == names.index(l["soil"])
            for _, k in sp.LAYER_FLOATS:
                assert row[k].tobytes() == np.float32(l[k]).tobytes(), (t["name"], k)
        assert p["world"]["scale"] == t["scale"]
    assert len(capi.parse_soil_file(sp.write(sp.table_64(), tmp_path))["soils"]) == capi.SM_MAX_SOILS


def test_parser_matches_reference_loader(ref, tmp_path):
    """sm_parse_soil_file == loadsoil (io.h:7-230) on every generated file and on the 64-soil file: soils, names,
    colours, layers and the world scale"""
    from soilmachine_b200 import capi
    for t in _tables():
        path = sp.write(t, tmp_path)
        ref.init(path, seed=1, dimx=8, dimy=8, poolsize=4096)
        p = capi.parse_soil_file(path)
        rs, rl = ref.soils(), ref.layers()
        assert len(rs) == len(p["soils"]) and len(rl) == len(p["layers"]), t["name"]
        for k in capi.SOIL_DTYPE.names:
            _golden.same(rs[k], p["soils"][k], t["name"] + ".soils." + k)
        _golden.same(rs["color"], p["colors"], t["name"] + ".colors")
        assert [n.decode() for n in rs["name"]] == p["soil_names"], t["name"]
        for k in capi.LAYER_DTYPE.names:
            _golden.same(rl[k], p["layers"][k], t["name"] + ".layers." + k)
        assert ref.scale == p["world"]["scale"] == t["scale"]


def _hs_wind_run(hs, xy):
    import _hostsim
    hs.wind_begin(xy)
    st = _hostsim.Stats()
    while hs.wind_sweep(st) > 0:
        pass
    return st


def _three_way(ref, tmp_path, table, dimx, dimy, nw, nd, seed):
    """two frames of batch, floods, seep pass, wind batch and frequency update on the reference, the port and
    hostsim; every column, the particle states and the frequency maps equal after every phase"""
    import _hostsim
    path = sp.write(table, tmp_path)
    ref.init(path, seed=seed, dimx=dimx, dimy=dimy, poolsize=dimx * dimy * 12 + 200000)
    soils = ref.soils()
    po = portapi.Port().init(ref.dimx, ref.dimy, ref.scale, soils)
    hs = _hostsim.HostSim()
    hs.init(ref.dimx, ref.dimy, ref.scale, soils)
    cols = ref.columns()
    po.set_columns(cols); hs.set_columns(cols)
    name = table["name"]

    def check(tag):
        a = ref.columns()
        _golden.same_cols(a, po.columns(), "%s %s (port)" % (name, tag))
        _golden.same_cols(a, hs.columns(), "%s %s (hostsim)" % (name, tag))

    tally = np.zeros(5, np.int64)
    for f in range(2):
        xw, xd = ref.spawn_list(nw, seed=seed + f), ref.spawn_list(nd)
        a, b, c = ref.water_run(xw), po.water_run(xw), hs.water_run(xw)
        s = (a.steps, a.sweeps, a.exit_oob, a.exit_evap, a.exit_stall)
        assert s == (b.steps, b.sweeps, b.exit_oob, b.exit_evap, b.exit_stall) == \
            (c.steps, c.sweeps, c.exit_oob, c.exit_evap, c.exit_stall), (name, f)
        tally += s
        ws = ref.water_state()
        for k, v in ws.items():
            _golden.same(v, po.water_state()[k], "%s frame %d water %s (port)" % (name, f, k))
            _golden.same(v, hs.water_state()[k], "%s frame %d water %s (hostsim)" % (name, f, k))
        check("frame %d after the water batch" % f)
        ref.water_flood(); po.water_flood(); hs.water_flood()
        check("frame %d after the floods" % f)
        ref.seep(); po.seep(); hs.seep()
        check("frame %d after the seep pass" % f)
        a, b, c = ref.wind_run(xd), po.wind_run(xd), _hs_wind_run(hs, xd)
        assert (a.steps, a.exit_oob) == (b.steps, b.exit_oob) == (c.steps, c.exit_oob), (name, f)
        for k, v in ref.wind_state().items():
            _golden.same(v, po.wind_state()[k], "%s frame %d wind %s (port)" % (name, f, k))
            _golden.same(v, hs.wind_state()[k], "%s frame %d wind %s (hostsim)" % (name, f, k))
        check("frame %d after the wind batch" % f)
        ref.frequency_update(); po.frequency_update(); hs.frequency_update()
        for k, v in ref.frequency().items():
            _golden.same(v, po.frequency()[k], "%s frame %d %s (port)" % (name, f, k))
            _golden.same(v, hs.frequency()[k], "%s frame %d %s (hostsim)" % (name, f, k))
        _golden.same(ref.heights(), po.heights(), name + " heights (port)")
        _golden.same(ref.heights(), hs.heights(), name + " heights (hostsim)")
    return tally


@pytest.mark.parametrize("seed,dimx,dimy", FRAME_CASES)
def test_generated_tables_agree_on_the_host(ref, tmp_path, seed, dimx, dimy):
    _three_way(ref, tmp_path, sp.random_table(seed), dimx, dimy, 400, 250, seed)


@pytest.mark.parametrize("name", sorted(sp.SENTINELS) + ["soils64"])
def test_sentinel_tables_agree_on_the_host(ref, tmp_path, name):
    table = sp.table_64() if name == "soils64" else sp.SENTINELS[name]()
    tally = _three_way(ref, tmp_path, table, 56, 64, 400, 250, 5)
    if name == "friction0":
        assert tally[4] == 2 * 400 and tally[2] == tally[3] == 0, tally     # every particle stalls


@pytest.mark.parametrize("seed", INIT_SEEDS)
def test_init_from_generated_layers_matches_reference(ref, tmp_path, seed):
    """hostsim's terrain init (sm_noise.cuh, the code sm_initialize runs) == Layermap::initialize on generated layer
    sets: 1 to 9 layers, fractional octaves, MIN > 0, negative BIAS, maps 2 to 64 cells wide"""
    import _hostsim
    t = sp.random_table(seed)
    rng = np.random.RandomState(seed)
    dimx, dimy = int(rng.randint(2, 65)), int(rng.randint(2, 65))
    ref.init(sp.write(t, tmp_path), seed=seed * 7 + 1, dimx=dimx, dimy=dimy, poolsize=dimx * dimy * 12 + 1000)
    hs = _hostsim.HostSim()
    hs.init(dimx, dimy, ref.scale, ref.soils())
    hs.initialize(seed * 7 + 1, ref.layers())
    _golden.same_cols(ref.columns(), hs.columns(), "%s %dx%d init" % (t["name"], dimx, dimy))
