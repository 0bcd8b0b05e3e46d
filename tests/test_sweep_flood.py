"""Sweep floods on the device (sm_water_run_flooding): the fixture's reference results (tests/golden/
sweep_flood_ops.npz); where oracle/_ref is built, the reference's own sweep-flood driver live on four presets, a small
pool and a cut; the flood counters equal to the host build's (tests/sweep_flood); one particle against sm_water_run +
sm_water_flood; the budgets; groups of 2 and 3 ranks against one context; refusals; the C++ facade."""
import os
import subprocess

import numpy as np
import pytest

import _golden
from _group import HYDRO_KEYS, same, same_map, same_stats
from test_sweep_flood_host import CASES, FIX, SOIL, STATE_KEYS, HostSweepFlood, cut_of, host_case, stats_tuple

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _ctx(case, **kw):
    from soilmachine_b200 import capi
    p = case + "/"
    dimx, dimy, scale, seed = (int(v) for v in FIX[p + "dims"])
    c = capi.Context(dimx, dimy, scale, max_particles=4096, **kw)
    c.set_soils(FIX[p + "soils"])
    c.initialize(seed, FIX[p + "layers"])
    return c


def _same_counters(hs, hc, what):
    """sm_hydro_stats of the device call against the host build's counters of the same order, exactly"""
    got = [hs.floods, hs.nested, hs.nested_steps, hs.transfers, hs.cells]
    want = [hc.floods, hc.nested, hc.nested_steps, hc.transfers, 0]
    assert got == want, (what, got, want)


def _same_state(c, ref_state, what):
    s = c.water_state()
    for k in STATE_KEYS:
        same(s[k], ref_state[k], "%s: state %s" % (what, k))


@pytest.mark.parametrize("case", CASES)
def test_fixture(case):
    """the reference's results without a reference checkout: stats, flood counts, states, checksums, columns"""
    from soilmachine_b200.checksum import columns_checksum
    p = case + "/"
    _, host = host_case(case)
    c = _ctx(case)
    try:
        assert c.checksum() == int(FIX[p + "checksum_init"])
        for b, ms in enumerate((0, cut_of(case))):
            st, hs = c.water_run_flooding(FIX[p + "xy_%d" % b], ms)
            same(stats_tuple(st), FIX[p + "stats_%d" % b], "%s batch %d stats" % (case, b))
            assert hs.floods >= int(FIX[p + "floods_%d" % b]) and st.pool_drops == 0
            _same_counters(hs, host[b][1], "%s batch %d" % (case, b))
            _same_state(c, {k: FIX[p + "state_%d_%s" % (b, k)] for k in STATE_KEYS}, "%s batch %d" % (case, b))
            assert c.checksum() == int(FIX[p + "checksum_%d" % b]), "%s batch %d checksum" % (case, b)
        if p + "final_offsets" in FIX.files:
            cols = c.download_columns()
            _golden.same_cols(cols, _golden.cols(FIX, p + "final"), case + " final columns")
            assert columns_checksum(cols) == c.checksum()
        for k, v in c.frequency().items():
            same(v, FIX[p + "freq_" + k], case + " " + k)
        same(c.heights(), FIX[p + "heights"], case + " heights")
    finally:
        c.close()


@pytest.fixture(scope="module")
def fref():
    from oracle import refapi_flooding
    if not refapi_flooding.available():
        pytest.skip("oracle/_ref/libsmref_flooding.so not built")
    return refapi_flooding.get()


LIVE = [("default", 64, 72, 5, 1500, 0, 0), ("bigbutte", 48, 56, 9, 1200, 0, 0), ("rocksand", 72, 64, 13, 1500, 0, 0),
        ("sand", 64, 64, 21, 1200, 0, 0), ("default", 64, 72, 6, 1500, 25, 0), ("bigbutte", 48, 56, 10, 1200, 0, 1)]


@pytest.mark.parametrize("soil,dimx,dimy,seed,n,cut,small_pool", LIVE)
def test_equals_the_reference_driver(fref, soil, dimx, dimy, seed, n, cut, small_pool):
    """the reference's move() / interact() / flood() in the sweep-flood order, live, two batches in a row; the
    flood count counts the batch's own floods (the device's also counts the nested particles' floods).  small_pool:
    a pool only 2500 sections larger than the reference's final map"""
    from soilmachine_b200 import capi, presets
    fref.init(soil, seed=seed, dimx=dimx, dimy=dimy)
    init_cols = fref.columns()
    fref.lib.smref_srand(seed)
    lists = [fref.spawn_list(n), fref.spawn_list(n)]
    ref = []
    for b, xy in enumerate(lists):
        rst, rfl = fref.water_sweep_flood(xy, cut if b == 0 else 0)
        ref.append((rst, rfl, fref.water_state(), fref.columns(), fref.frequency()))
    pool = int(ref[-1][3]["offsets"][-1]) - dimx * dimy + 2500 if small_pool else 0
    pre = presets.load(soil)
    h = HostSweepFlood()
    h.init(dimx, dimy, fref.scale, pre["soils"])
    h.initialize(seed, pre["layers"])
    host = [h.water_run_flooding(xy, cut if b == 0 else 0)[1] for b, xy in enumerate(lists)]
    c = capi.Context(dimx, dimy, fref.scale, max_particles=n, pool_capacity=pool)
    try:
        c.set_soils(pre["soils"])
        c.initialize(seed, pre["layers"])
        _golden.same_cols(c.download_columns(), init_cols, "initial terrain")
        for b, xy in enumerate(lists):
            rst, rfl, rstate, rcols, rfreq = ref[b]
            st, hs = c.water_run_flooding(xy, cut if b == 0 else 0)
            what = "%s seed %d batch %d" % (soil, seed, b)
            assert st.pool_drops == 0, what
            same(stats_tuple(st), stats_tuple(rst), what + " stats")
            assert hs.floods >= rfl and (hs.floods > 0) == (rfl > 0), what
            _same_counters(hs, host[b], what)
            _same_state(c, rstate, what)
            _golden.same_cols(c.download_columns(), rcols, what + " columns")
            for k, v in c.frequency().items():
                same(v, rfreq[k], what + " " + k)
    finally:
        c.close()


def test_one_particle_equals_run_then_flood():
    """n = 1: the call equals sm_water_run + sm_water_flood, columns, state, stats and flood counters"""
    p = "default_48/"
    stalled = np.nonzero(FIX[p + "state_0_volume"] >= 0.01)[0]
    nfl = 0
    for i in list(stalled[:8]) + [0, 1]:
        xy = FIX[p + "xy_0"][i][None]
        a, b = _ctx("default_48"), _ctx("default_48")
        try:
            sa, ha = a.water_run_flooding(xy)
            sb = b.water_run(xy)
            hb = b.water_flood()
            same_stats(sa, sb, "particle %d" % i)
            assert [getattr(ha, k) for k in HYDRO_KEYS] == [getattr(hb, k) for k in HYDRO_KEYS], i
            same_map(a, b, "particle %d" % i)
            sta, stb = a.water_state(), b.water_state()
            for k in STATE_KEYS:
                same(sta[k], stb[k], "particle %d state %s" % (i, k))
            nfl += ha.floods
        finally:
            a.close(); b.close()
    assert nfl > 0


def _height_total(c):
    return float(np.sum(c.heights(), dtype=np.float64))


def test_budgets_close_and_change_nothing():
    """with SM_FLAG_BUDGET the whole-map identity closes over the call (batch terms + flood terms); the budget flags
    change no result; the cell maps of the batch and of the floods cover the same call"""
    case = "bigbutte_40"
    p = case + "/"
    plain, bud, cells = _ctx(case), _ctx(case, budget=True), _ctx(case, cell_budget=True, hydro_cell_budget=True)
    try:
        h0 = _height_total(bud)
        out = [c.water_run_flooding(FIX[p + "xy_0"]) for c in (plain, bud, cells)]
        for c, (st, hs) in zip((bud, cells), out[1:]):
            same_stats(st, out[0][0], "budget flags: stats")
            assert [getattr(hs, k) for k in HYDRO_KEYS] == [getattr(out[0][1], k) for k in HYDRO_KEYS]
            same_map(c, plain, "budget flags")
        b, h = bud.last_budget(), bud.last_hydro_budget()
        same(np.float64(b.eroded), np.float64(cells.last_budget().eroded), "budget with the cell maps")
        assert h == cells.last_hydro_budget()
        batch = b.deposited - b.eroded + b.cascade_net
        flood = (h["flood_sediment"] + h["flood_cascade_net"] + h["flood_water"] - h["seeped"] - h["to_particles"]
                 + h["transfer_net"] + h["nested_deposited"] - h["nested_eroded"] + h["nested_cascade_net"])
        dh = _height_total(bud) - h0
        assert h["flood_water"] > 0 and abs(batch) > 0
        assert abs(dh - (batch + flood)) <= 1e-9 * max(1.0, abs(h0)), (dh, batch, flood)
        # the maps: per cell, batch maps + hydrology maps = change of the cell's height
        m, hm = cells.last_cell_budget(), cells.last_hydro_cell_budget()
        per_cell = (m["deposited"] - m["eroded"] + m["cascade_net"] + hm["deposited"] - hm["eroded"]
                    + hm["cascade_net"] + hm["water_net"])
        assert abs(float(per_cell.sum()) - dh) <= 1e-9 * max(1.0, abs(h0))
    finally:
        plain.close(); bud.close(); cells.close()


@pytest.mark.parametrize("nranks", [2, 3])
def test_group_equals_one_context(nranks):
    """a group of 2 and 3 ranks on one GPU: bit-identical maps, states, stats and flood counters"""
    from soilmachine_b200 import capi, presets
    pre = presets.load("rocksand")
    dimx, dimy, seed = 96, 64, 4
    rng = np.random.default_rng(nranks)
    xy = np.stack([rng.integers(0, dimx, 2000), rng.integers(0, dimy, 2000)], 1).astype(np.float32)
    ctxs = [capi.Context(dimx, dimy, pre["world"]["scale"], max_particles=4096, **kw)
            for kw in ({}, {"devices": [0] * nranks})]
    try:
        for c in ctxs:
            c.set_soils(pre["soils"]); c.initialize(seed, pre["layers"])
        for b, ms in enumerate((0, 30, 0)):
            (sa, ha), (sb, hb) = [c.water_run_flooding(xy[b::3] if b < 2 else xy, ms) for c in ctxs]
            same_stats(sb, sa, "group of %d batch %d" % (nranks, b))
            assert [getattr(hb, k) for k in HYDRO_KEYS] == [getattr(ha, k) for k in HYDRO_KEYS]
            assert ha.floods > 0
            same_map(ctxs[1], ctxs[0], "group of %d batch %d" % (nranks, b))
            s1, s0 = ctxs[1].water_state(), ctxs[0].water_state()
            for k in STATE_KEYS:
                same(s1[k], s0[k], "group of %d batch %d state %s" % (nranks, b, k))
    finally:
        for c in ctxs:
            c.close()


def test_refusals():
    from soilmachine_b200 import capi
    c = capi.Context(64, 64, 80, nranks=2, rank=0, max_particles=64)
    try:
        with pytest.raises(capi.SoilMachineError) as e:
            c.water_run_flooding(np.zeros((4, 2), np.float32))
        assert e.value.code == capi.SM_ERR_INVALID
    finally:
        c.close()
    c = _ctx("default_48")
    try:
        with pytest.raises(capi.SoilMachineError) as e:
            c.water_run_flooding(np.zeros((5000, 2), np.float32))
        assert e.value.code == capi.SM_ERR_INVALID
    finally:
        c.close()


def test_simulation_frame_sweep_floods():
    """Simulation.frame(floods="sweep") equals the capi calls it is made of; the default frame is unchanged"""
    from soilmachine_b200 import host
    a = host.Simulation("default", seed=3, dimx=64, dimy=64, max_particles=1024)
    b = host.Simulation("default", seed=3, dimx=64, dimy=64, max_particles=1024)
    try:
        xy = host.spawn_list(800, 64, 64)
        ws, _ = a.frame(800, 0, water_xy=xy, hydrology=True, floods="sweep")
        st, hs = b.ctx.water_run_flooding(xy)
        b.ctx.seep(); b.ctx.frequency_update()
        same_stats(ws, st, "frame")
        same_map(a.ctx, b.ctx, "frame")
        assert a.last_hydrology[0][0].floods == hs.floods
    finally:
        a.ctx.close(); b.ctx.close()


def test_facade_run_flooding(tmp_path):
    """tests/facade_sweep_flood.cpp: the facade's run_flooding frame, plain and on a group of two"""
    from oracle import refapi
    libdir = os.path.join(ROOT, "soilmachine_b200", "lib")
    exe = str(tmp_path / "facade_sweep_flood")
    subprocess.check_call(["g++", "-std=c++17", "-O1", os.path.join(ROOT, "tests", "facade_sweep_flood.cpp"), "-o", exe,
                           "-L" + libdir, "-lsoilmachine_b200", "-Wl,-rpath," + libdir])
    lines = []
    for group in (False, True):
        env = {k: v for k, v in os.environ.items() if k not in ("SM_GPUS", "SM_GPU_DEVICES")}
        if group:
            env.update(SM_GPUS="2", SM_GPU_DEVICES="0,0")
        out = subprocess.run([exe, refapi.soil_path("default")], capture_output=True, text=True, timeout=600, env=env)
        assert out.returncode == 0, out.stdout + out.stderr
        lines.append(out.stdout.strip())
    assert lines[0] == lines[1], lines


def _group_check(devices):
    import sys
    out = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "multigpu_sweep_flood_check.py"), "--devices",
                          ",".join(map(str, devices)), "--dim", "128"], capture_output=True, text=True, timeout=900)
    line = [l for l in out.stdout.splitlines() if l.startswith("multigpu_sweep_flood_check")]
    assert out.returncode == 0 and line and " equal " in line[0], out.stdout + out.stderr


def test_group_check_script_ranks_sharing_this_gpu():
    """tests/multigpu_sweep_flood_check.py with three ranks on this GPU"""
    _group_check([0, 0, 0])


def test_group_check_script_one_rank_per_gpu():
    """tests/multigpu_sweep_flood_check.py with one rank on each of the first two GPUs (peer access, events between
    devices), where there are two"""
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    _group_check([0, 1])
