"""GPU: the device on soil tables the other parity tests never load - the six presets no device test ran, generated
tables over the parameter extremes, sentinel tables whose soil types can reach the map through one mapping only, a
table of SM_MAX_SOILS (64) soils, and sm_set_volume_factor away from its default.  Byte for byte against the
reference in lockstep (oracle/_ref), against the oracle port with the mass budget (no reference needed), on a map
sharded into three strips, and against tests/golden/soil_space.npz where the reference is absent.  The schedule is
the library's default selection throughout."""
import numpy as np
import pytest
import _golden
import _soil_space as sp
from _hydro_budget import TERMS

pytestmark = pytest.mark.gpu

DEFAULT_VOLUME_FACTOR = 0.015        # water.h: WaterParticle::volumeFactor


def _same(a, b, what):
    _golden.same(a, b, what)


def _compare_maps(a, ctx, what):
    """a: the reference or the port; every height, every section of every column, the frequency maps"""
    _same(a.heights(), ctx.heights(), what + ": height")
    c1, c2 = a.columns(), ctx.download_columns()
    for k in ("offsets", "type", "size", "floor", "saturation"):
        _same(c1[k], c2[k], what + ": columns." + k)
    f1, f2 = a.frequency(), ctx.frequency()
    for k in f1:
        _same(f1[k], f2[k], what + ": " + k)


def _stats5(st):
    return (st.steps, st.sweeps, st.exit_oob, st.exit_evap, st.exit_stall)


def _table(name):
    if name == "soils64":
        return sp.table_64()
    if name in sp.SENTINELS:
        return sp.SENTINELS[name]()
    return sp.random_table(int(name[3:]))


def _names(soils):
    return [n.decode() for n in soils["name"]]


def _ctx_from_ref(ref, seed, **kw):
    """a context with the reference's soil table and terrain from sm_initialize, checked against the reference's"""
    import soilmachine_b200 as smb
    ctx = smb.Context(ref.dimx, ref.dimy, ref.scale, max_particles=4096, **kw)
    ctx.set_soils(ref.soils())
    ctx.initialize(seed, ref.layers())
    c1, c2 = ref.columns(), ctx.download_columns()
    for k in c1:
        _same(c1[k], c2[k], "initial terrain: columns." + k)
    return ctx


def _lockstep_frame(ref, ctx, xw, xd, what):
    """water batch, floods, seep pass, wind batch (if xd), frequency update (SoilMachine.cpp:287-320), compared after
    every phase; returns the water stats and the device's flood counters"""
    r, g = ref.water_run(xw), ctx.water_run(xw)
    assert _stats5(g) == _stats5(r) and g.pool_drops == 0, (what, r.asdict(), g.asdict())
    water = _stats5(r)
    s1, s2 = ref.water_state(), ctx.water_state()
    for k in s1:
        _same(s1[k], s2[k], what + ": water particles " + k)
    _compare_maps(ref, ctx, what + " after the water batch")
    nf, h = ref.water_flood(), ctx.water_flood()
    assert h.floods >= nf, what
    _compare_maps(ref, ctx, what + " after the floods")
    ref.seep(); ctx.seep()
    _compare_maps(ref, ctx, what + " after the seep pass")
    if len(xd):
        d, g = ref.wind_run(xd), ctx.wind_run(xd)
        assert (g.steps, g.exit_oob) == (d.steps, d.exit_oob) and g.pool_drops == 0, what
        s1, s2 = ref.wind_state(), ctx.wind_state()
        for k in s1:
            _same(s1[k], s2[k], what + ": wind particles " + k)
        _compare_maps(ref, ctx, what + " after the wind batch")
    ref.frequency_update(); ctx.frequency_update()
    _compare_maps(ref, ctx, what + " after the frequency update")
    return water, h


# ---- 1. the six presets no device test ran ----------------------------------------------------------------------
@pytest.mark.parametrize("preset,dimx,dimy", [("sand", 96, 112), ("painted", 128, 96), ("friction_0.01", 112, 112),
                                              ("friction_0.5", 96, 128), ("bigbutte2", 128, 128),
                                              ("rockgravelpebbles", 120, 104)])
def test_preset_frame_matches_reference(ref, preset, dimx, dimy):
    seed = 29
    ref.init(preset, seed=seed, dimx=dimx, dimy=dimy, poolsize=dimx * dimy * 12 + 500000)
    ctx = _ctx_from_ref(ref, seed)
    wind = bool((ref.soils()["suspension"] > 0).any())
    xw = ref.spawn_list(1000, seed=seed)
    xd = ref.spawn_list(500) if wind else np.zeros((0, 2), np.float32)
    st, h = _lockstep_frame(ref, ctx, xw, xd, preset)
    assert st[0] > 0 or st[4] > 0, (preset, st)
    ctx.close()


# ---- 2. and 3. generated and sentinel tables, with what each case must reach -------------------------------------
CASES = [  # name, dimx, dimy, water, wind, frames
    ("gen2", 64, 64, 500, 300, 2), ("gen7", 3, 96, 300, 200, 2), ("gen11", 97, 61, 500, 300, 2),
    ("gen22", 64, 56, 500, 300, 2), ("gen57", 2, 80, 200, 100, 2),
    ("sentinel_water", 80, 80, 700, 0, 2), ("sentinel_wind", 72, 64, 500, 500, 1),
    ("friction0", 64, 64, 400, 0, 1), ("steep", 64, 64, 500, 0, 1), ("soils64", 96, 96, 800, 400, 2)]


def _reach(name, ref, exits, floods):
    """what the case exists for, judged only from the outputs"""
    names = _names(ref.soils())
    present = {names[t] for t in set(ref.columns()["type"].tolist())}
    if name == "sentinel_water":
        assert {"Tr", "Er", "Ca"} <= present, present          # transports, erodes and cascades all ran
    if name == "sentinel_wind":
        assert "Dust" in present, present                      # deposited by wind particles only
    if name == "friction0":
        assert exits[4] > 0 and exits[0] == exits[2] == exits[3] == 0, exits   # every particle stalls at spawn
        assert floods > 0
    if name == "soils64":
        assert len(names) == 64 and "Soil 63" in present, sorted(present)
    if name in ("gen2", "gen22"):
        assert exits[2] > 0 and exits[3] > 0, exits           # out of bounds and evaporated


@pytest.mark.parametrize("name,dimx,dimy,nw,nd,frames", CASES)
def test_table_frames_match_reference(ref, tmp_path, name, dimx, dimy, nw, nd, frames):
    seed = 5
    ref.init(sp.write(_table(name), tmp_path), seed=seed, dimx=dimx, dimy=dimy, poolsize=dimx * dimy * 16 + 500000)
    ctx = _ctx_from_ref(ref, seed)
    exits, floods = np.zeros(5, np.int64), 0
    for f in range(frames):
        xw = ref.spawn_list(nw, seed=seed + f)
        xd = ref.spawn_list(nd) if nd else np.zeros((0, 2), np.float32)
        st, h = _lockstep_frame(ref, ctx, xw, xd, "%s %dx%d frame %d" % (name, dimx, dimy, f))
        exits += st
        floods += h.floods
    _reach(name, ref, exits, floods)
    ctx.close()


def _port_case(name, dimx, dimy, seed=5):
    """a budget context and the port with the budget, on the table's terrain from sm_initialize - no reference"""
    import soilmachine_b200 as smb
    from soilmachine_b200 import capi
    from _hydro_budget import BudgetPort
    import tempfile
    with tempfile.TemporaryDirectory() as d:
        p = capi.parse_soil_file(sp.write(_table(name), d))
    scale = p["world"]["scale"]
    ctx = smb.Context(dimx, dimy, scale, max_particles=4096, budget=True)
    ctx.set_soils(p["soils"])
    ctx.initialize(seed, p["layers"])
    po = BudgetPort().init(dimx, dimy, scale, p["soils"])
    po.set_columns(ctx.download_columns())
    return ctx, po, p


def _spawn(n, dimx, dimy, seed):
    from soilmachine_b200 import host
    host.srand(seed)
    return host.spawn_list(n, dimx, dimy)


def _port_frame(ctx, po, xw, xd, what):
    """one frame against the port: the six per-particle accumulators and their sums of both batches, the flood
    counters and the eleven hydrology budget terms of the floods and the seep pass, the map after every phase"""
    seen = {}
    for kind, xy in (("water", xw), ("wind", xd)):
        if not len(xy):
            continue
        a = (po.water_run if kind == "water" else po.wind_run)(xy)
        g = (ctx.water_run if kind == "water" else ctx.wind_run)(xy)
        if kind == "water":
            assert _stats5(a) == _stats5(g), (what, a.asdict(), g.asdict())
            seen["exits"] = np.array(_stats5(g))
        else:
            assert (a.steps, a.exit_oob) == (g.steps, g.exit_oob), what
        per_p, sums_p = po.budget()
        _same(ctx.budget_particles(len(xy)), per_p, "%s %s: mass budget per particle" % (what, kind))
        b = ctx.last_budget()
        got = np.array([b.eroded, b.deposited, b.cascade_net, b.discarded, b.clamped, b.wind_negative])
        _same(got, sums_p, "%s %s: mass budget" % (what, kind))
        seen[kind] = got
        _compare_maps(po, ctx, "%s after the %s batch" % (what, kind))
        if kind == "water":
            for call in ("water_flood", "seep"):
                a, g = getattr(po, call)(), getattr(ctx, call)()
                assert (a.floods, a.nested, a.nested_steps, a.transfers) == \
                    (g.floods, g.nested, g.nested_steps, g.transfers), (what, call, a.asdict(), g.asdict())
                hb = ctx.last_hydro_budget()
                _same(np.array([hb[k] for k in TERMS]), po.hydro_budget(), "%s %s: hydrology budget" % (what, call))
                seen[call] = g
                _compare_maps(po, ctx, "%s after %s" % (what, call))
    po.frequency_update(); ctx.frequency_update()
    _compare_maps(po, ctx, what + " after the frequency update")
    return seen


PORT_CASES = [("gen2", 64, 64), ("gen26", 3, 80), ("gen11", 97, 61), ("sentinel_water", 72, 72),
              ("sentinel_wind", 64, 64), ("steep", 64, 64), ("friction0", 48, 48)]


@pytest.mark.parametrize("name,dimx,dimy", PORT_CASES)
def test_table_budget_matches_port(name, dimx, dimy):
    """the same tables against the port (pinned to the reference by tests/test_soil_space_host.py): runs without
    oracle/_ref"""
    ctx, po, _ = _port_case(name, dimx, dimy)
    seen = _port_frame(ctx, po, _spawn(500, dimx, dimy, 3), _spawn(300, dimx, dimy, 4), name)
    if name == "steep":
        assert seen["water"][4] > 0, seen["water"]            # sediment cut off by the clamp (water.h:117)
    if name in ("gen2", "sentinel_wind"):
        assert seen["wind"][5] != 0, seen["wind"]             # negative suspension force (wind.h:107-110)
    if name in ("friction0", "sentinel_water"):
        assert seen["water_flood"].floods > 0 and seen["water_flood"].transfers > 0
    if name == "friction0":
        assert seen["exits"][4] == 500 and seen["exits"][0] == 0, seen["exits"]
    ctx.close()


# ---- 4. the volume factor -----------------------------------------------------------------------------------------
@pytest.mark.parametrize("v", [0.003, 0.05, 1.0])
def test_volume_factor_matches_reference(ref, tmp_path, v):
    """sm_set_volume_factor scales the water every flood adds (water.h:137) and so every seep transfer after it"""
    seed = 13
    ref.init(sp.write(sp.sentinel_water(), tmp_path), seed=seed, dimx=80, dimy=72, poolsize=80 * 72 * 16 + 500000)
    ctx = _ctx_from_ref(ref, seed)
    try:
        ref.set_volume_factor(v); ctx.set_volume_factor(v)
        floods = 0
        for f in range(2):
            xw = ref.spawn_list(600, seed=seed + f)
            _, h = _lockstep_frame(ref, ctx, xw, np.zeros((0, 2), np.float32), "volume factor %g frame %d" % (v, f))
            floods += h.floods
        assert floods > 0
    finally:
        ref.set_volume_factor(DEFAULT_VOLUME_FACTOR)
        ctx.close()


# ---- 5. the table size limit --------------------------------------------------------------------------------------
def test_refused_tables_leave_the_table_in_force(ref, tmp_path):
    """65 soils, and a cascades entry out of range, are refused with SM_ERR_INVALID; after either the 64-soil table
    is still the one the device runs"""
    import soilmachine_b200 as smb
    from soilmachine_b200 import capi
    seed = 5
    ref.init(sp.write(sp.table_64(), tmp_path), seed=seed, dimx=80, dimy=80, poolsize=80 * 80 * 16 + 500000)
    ctx = _ctx_from_ref(ref, seed)
    soils = capi.soils_from(ref.soils())
    assert len(soils) == capi.SM_MAX_SOILS
    too_many = np.concatenate([soils, soils[-1:]])
    bad = soils.copy()
    bad["cascades"][40] = len(bad)
    for f, table in enumerate((too_many, bad)):
        with pytest.raises(smb.SoilMachineError) as e:
            ctx.set_soils(table)
        assert e.value.code == capi.SM_ERR_INVALID
        xw, xd = ref.spawn_list(500, seed=seed + f), ref.spawn_list(300)
        _lockstep_frame(ref, ctx, xw, xd, "after refusal %d" % f)
    assert int(ctx.download_columns()["type"].max()) == 63
    ctx.close()


# ---- 6. sharded ---------------------------------------------------------------------------------------------------
def test_sentinel_sharded_matches_one_context(tmp_path):
    """the water sentinel on three x-strips, every rank with its own copy of the table, against one context"""
    import soilmachine_b200 as smb
    from soilmachine_b200 import capi, sharded
    p = capi.parse_soil_file(sp.write(sp.sentinel_water(), tmp_path))
    dimx, dimy, scale = 96, 72, p["world"]["scale"]
    one = smb.Context(dimx, dimy, scale, max_particles=4096)
    sh = sharded.VirtualShards(3, dimx, dimy, scale, max_particles=4096)
    for c in (one, sh):
        c.set_soils(p["soils"])
        c.initialize(5, p["layers"])
    for f in range(2):
        xw = _spawn(700, dimx, dimy, 30 + f)
        a, b = one.water_run(xw), sh.water_run(xw)
        assert _stats5(a) == _stats5(b), f
        a, b = one.water_flood(), sh.water_flood()
        assert (a.floods, a.nested, a.nested_steps, a.transfers) == (b.floods, b.nested, b.nested_steps, b.transfers)
        one.seep(); sh.seep()
        one.frequency_update(); sh.frequency_update()
        _same(one.heights(), sh.heights(), "frame %d height" % f)
        c1, c2 = one.download_columns(), sh.download_columns()
        for k in c1:
            _same(c1[k], c2[k], "frame %d columns.%s" % (f, k))
        f1, f2 = one.frequency(), sh.frequency()
        for k in f1:
            _same(f1[k], f2[k], "frame %d %s" % (f, k))
    names = p["soil_names"]
    present = {names[t] for t in set(one.download_columns()["type"].tolist())}
    assert {"Tr", "Er", "Ca"} <= present, present
    one.close(); sh.close()


# ---- 7. the committed vectors -------------------------------------------------------------------------------------
class _Case:
    """one prefixed case of soil_space.npz, seen the way _golden.replay_frame / replay_hydro read a case"""

    def __init__(self, g, prefix):
        self.g, self.prefix = g, prefix
        self.files = [k[len(prefix):] for k in g.files if k.startswith(prefix)]

    def __getitem__(self, k):
        return self.g[self.prefix + k]


def test_gpu_replays_soil_space_golden():
    """tests/golden/soil_space.npz (tests/golden/make_soil_space_golden.py): a generated table's terrain and frame,
    and two hydrology frames of the water sentinel - independent of oracle/_ref"""
    import soilmachine_b200 as smb
    g = _golden.load("soil_space")
    c = _Case(g, "gen/")
    ctx = smb.Context(int(c["dimx"]), int(c["dimy"]), int(c["scale"]), max_particles=4096)
    ctx.set_soils(c["soils"])
    ctx.initialize(int(c["seed"]), c["layers"])
    _golden.same_cols(ctx.download_columns(), _golden.cols(c, "init"), "generated table: initial terrain")
    _golden.replay_frame(c, ctx, _stats5)
    ctx.close()
    c = _Case(g, "sen/")
    ctx = smb.Context(int(c["dimx"]), int(c["dimy"]), int(c["scale"]), max_particles=4096)
    ctx.set_soils(c["soils"])
    ctx.initialize(int(c["seed"]), c["layers"])
    _golden.same_cols(ctx.download_columns(), _golden.cols(c, "init"), "sentinel: initial terrain")
    counters = _golden.replay_hydro(c, ctx)
    assert all(h.floods >= f for h, f in zip(counters, c["floods"]))
    names = _names(c["soils"])
    present = {names[t] for t in set(ctx.download_columns()["type"].tolist())}
    assert {"Tr", "Er", "Ca"} <= present, present
    ctx.close()


# ---- 8. negative control ------------------------------------------------------------------------------------------
def test_one_ulp_in_the_table_is_seen():
    """the device runs a table whose surface soil's maxdiff is one ulp above the port's: the frame comparison must
    fail, so the tests above would see a parameter read from the wrong place"""
    field = "maxdiff"
    name, dimx, dimy = "gen2", 64, 64
    ctx, po, p = _port_case(name, dimx, dimy)
    surf = np.bincount(ctx.surfaces().reshape(-1)).argmax()
    soils = p["soils"].copy()
    soils[field][surf] = np.nextafter(soils[field][surf], np.float32(np.inf), dtype=np.float32)
    ctx.set_soils(soils)
    with pytest.raises(AssertionError):
        _port_frame(ctx, po, _spawn(500, dimx, dimy, 3), _spawn(300, dimx, dimy, 4), "%s + 1 ulp" % field)
    ctx.close()
