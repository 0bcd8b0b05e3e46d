"""CPU side of the sweep-flood order (sm_water_run_flooding): the reference's own move() / interact() / flood() driven
in that order (oracle/_ref/libsmref_flooding.so) reproduces tests/golden/sweep_flood_ops.npz, and so does the product's
step and flood arithmetic compiled for the host (tests/sweep_flood/host_sweep_flood.cpp over tests/hostsim); for one
particle the order is the batch order; the C ABI, capi, Simulation.frame and the C++ facade carry the call."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

import _golden
import _hostsim

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIX = _golden.load("sweep_flood_ops")
CASES = [str(c) for c in FIX["cases"]]
SOIL = {"default_48": "default", "bigbutte_40": "bigbutte", "rocksand_56": "rocksand"}
STATE_KEYS = ("pos", "speed", "volume", "sediment", "contains", "alive")


class HostSweepFlood(_hostsim.HostSim):
    """tests/hostsim on a library that also drives the sweep-flood order (host_sweep_flood.cpp), on the warp step and
    the warp flood executor as the device call runs them"""

    def __init__(self):
        from _hydro_budget import CSRC, _build
        src = os.path.join(ROOT, "tests", "sweep_flood", "host_sweep_flood.cpp")
        deps = [_hostsim.SRC, _hostsim.CORE, _hostsim.NOISE, _hostsim.HYDRO, _hostsim.COOP, _hostsim.HCOOP,
                os.path.join(CSRC, "sm_foot.cuh")]
        self.lib = C.CDLL(_build("host_sweep_flood", src, deps))
        self.lib.hs_nsections.restype = C.c_int64
        self.lib.hs_set_mode(1, 0)

    def water_run_flooding(self, xy, max_sweeps=0):
        xy = np.ascontiguousarray(xy, np.float32)
        self._n = len(xy)
        st, hc = _hostsim.Stats(), _hostsim.HydroCount()
        self.lib.hssf_water_run_flooding(len(xy), xy.ctypes.data_as(C.POINTER(C.c_float)), int(max_sweeps),
                                         C.byref(st), C.byref(hc))
        return st, hc


def host_case(case):
    """the fixture's case on the host build: (HostSweepFlood after both batches, [counters of each batch])"""
    from soilmachine_b200.checksum import columns_checksum
    p = case + "/"
    dimx, dimy, scale, seed = (int(v) for v in FIX[p + "dims"])
    h = HostSweepFlood()
    h.init(dimx, dimy, scale, FIX[p + "soils"])
    h.initialize(seed, FIX[p + "layers"])
    assert columns_checksum(h.columns()) == int(FIX[p + "checksum_init"]), case + ": host terrain"
    out = []
    for b, ms in enumerate((0, cut_of(case))):
        st, hc = h.water_run_flooding(FIX[p + "xy_%d" % b], ms)
        out.append((st, hc, h.water_state(), columns_checksum(h.columns())))
    return h, out


def stats_tuple(st):
    return np.array([st.steps, st.sweeps, st.exit_oob, st.exit_evap, st.exit_stall], np.int64)


def cut_of(case):
    """sweeps of the fixture's second (cut) batch"""
    return int(FIX[case + "/stats_1"][1])


@pytest.fixture(scope="module")
def fref():
    from oracle import refapi_flooding
    if not refapi_flooding.available():
        pytest.skip("oracle/_ref/libsmref_flooding.so not built (make -C oracle -f flooding.mk)")
    return refapi_flooding.get()


@pytest.mark.parametrize("case", CASES)
def test_reference_driver_reproduces_the_fixture(fref, case):
    from soilmachine_b200.checksum import columns_checksum
    p = case + "/"
    dimx, dimy, _, seed = (int(v) for v in FIX[p + "dims"])
    fref.init(SOIL[case], seed=seed, dimx=dimx, dimy=dimy)
    assert columns_checksum(fref.columns()) == int(FIX[p + "checksum_init"])
    for b, ms in enumerate((0, cut_of(case))):
        st, nfl = fref.water_sweep_flood(FIX[p + "xy_%d" % b], ms)
        _golden.same(stats_tuple(st), FIX[p + "stats_%d" % b], case + " stats")
        assert nfl == int(FIX[p + "floods_%d" % b])
        s = fref.water_state()
        for k in STATE_KEYS:
            _golden.same(s[k], FIX[p + "state_%d_%s" % (b, k)], "%s batch %d state %s" % (case, b, k))
        assert columns_checksum(fref.columns()) == int(FIX[p + "checksum_%d" % b])
    if p + "final_offsets" in FIX.files:
        _golden.same_cols(fref.columns(), _golden.cols(FIX, p + "final"), case + " final columns")
    for k, v in fref.frequency().items():
        _golden.same(v, FIX[p + "freq_" + k], case + " " + k)
    _golden.same(fref.heights(), FIX[p + "heights"], case + " heights")


@pytest.mark.parametrize("case", CASES)
def test_host_build_reproduces_the_fixture(case):
    """the product's warp step and warp flood executor, compiled for the host and driven in the sweep-flood order:
    stats, states, checksums after each batch, final columns, frequency maps and heights, bit for bit; its flood
    count includes the nested particles' floods, so it is at least the reference's"""
    p = case + "/"
    h, out = host_case(case)
    for b, (st, hc, s, csum) in enumerate(out):
        _golden.same(stats_tuple(st), FIX[p + "stats_%d" % b], "%s batch %d stats" % (case, b))
        assert hc.floods >= int(FIX[p + "floods_%d" % b]) and hc.overflow == 0
        for k in STATE_KEYS:
            _golden.same(s[k], FIX[p + "state_%d_%s" % (b, k)], "%s batch %d state %s" % (case, b, k))
        assert csum == int(FIX[p + "checksum_%d" % b]), "%s batch %d checksum" % (case, b)
    if p + "final_offsets" in FIX.files:
        _golden.same_cols(h.columns(), _golden.cols(FIX, p + "final"), case + " final columns")
    for k, v in h.frequency().items():
        _golden.same(v, FIX[p + "freq_" + k], case + " " + k)
    _golden.same(h.heights(), FIX[p + "heights"], case + " heights")


def test_fixture_has_floods_nested_work_and_a_cut():
    for case in CASES:
        p = case + "/"
        assert int(FIX[p + "floods_0"]) > 100 and int(FIX[p + "floods_1"]) > 100, case
        assert int(FIX[p + "state_1_alive"].sum()) > 0, case + ": the cut batch has survivors"
        assert not FIX[p + "state_0_alive"].any(), case


def one_particle_runs(fref, xy):
    """the particle alone in the two orders on default_48's map: (stats, floods, column checksum) of each"""
    from soilmachine_b200.checksum import columns_checksum
    got = []
    for sweep in (True, False):
        fref.init("default", seed=42, dimx=48, dimy=56)
        if sweep:
            st, nfl = fref.water_sweep_flood(xy)
        else:
            st = fref.water_run(xy)
            nfl = fref.water_flood()
        got.append((tuple(stats_tuple(st)), nfl, columns_checksum(fref.columns())))
    return got


def test_one_particle_is_the_batch_order(fref):
    """n = 1: sweep floods = the lockstep batch followed by sm_water_flood's order, for particles that flood and
    particles that do not"""
    p = "default_48/"
    stalled = np.nonzero(FIX[p + "state_0_volume"] >= 0.01)[0]       # stopped with water left in the batch
    nfl = []
    for i in list(stalled[:10]) + [0, 1, 2]:
        a, b = one_particle_runs(fref, FIX[p + "xy_0"][i][None])
        assert a == b, i
        nfl.append(a[1])
    assert 0 < sum(nfl) < len(nfl)


def test_sweep_floods_change_what_the_batch_meets(fref):
    """the same batch in the two orders: the ponds of early stoppers change later particles' paths"""
    from soilmachine_b200.checksum import columns_checksum
    xy = FIX["bigbutte_40/xy_0"]
    res = []
    for sweep in (True, False):
        fref.init("bigbutte", seed=3, dimx=40, dimy=48)
        if sweep:
            st, _ = fref.water_sweep_flood(xy)
        else:
            st = fref.water_run(xy)
            fref.water_flood()
        res.append((st.steps, columns_checksum(fref.columns())))
    assert res[0] != res[1]


def test_c_abi_and_capi_declare_the_call():
    from soilmachine_b200 import capi
    hdr = open(os.path.join(ROOT, "include", "soilmachine_b200.h")).read()
    m = re.search(r"int sm_water_run_flooding\(([^)]*)\)", hdr)
    assert m and [a.split()[-1].lstrip("*") for a in m.group(1).split(",")] == [
        "ctx", "n", "spawn_xy", "max_sweeps", "stats", "hstats"]
    assert "sm_water_run_flooding" in capi.SYMBOLS
    assert hasattr(capi.load(), "sm_water_run_flooding")
    assert callable(capi.Context.water_run_flooding)


def test_frame_floods_sweep_plumbing():
    """Simulation.frame(floods="sweep") runs each water batch through water_run_flooding, then the seep pass; the
    default order is unchanged"""
    from soilmachine_b200 import host

    class Rec:
        def __init__(self):
            self.calls = []

        def water_run(self, xy):
            self.calls.append(("water", len(xy)))

        def water_run_flooding(self, xy):
            self.calls.append(("water_flooding", len(xy)))
            return "ws", "fs"

        def wind_run(self, xy):
            self.calls.append(("wind", len(xy)))

        def water_flood(self):
            self.calls.append(("flood",))

        def seep(self):
            self.calls.append(("seep",))
            return "seep"

        def frequency_update(self):
            self.calls.append(("freq",))

    sim = object.__new__(host.Simulation)
    sim.ctx, sim.dimx, sim.dimy = Rec(), 32, 24
    host.srand(1)
    ws, _ = sim.frame(10, 4, hydrology=True, floods="sweep")
    assert sim.ctx.calls == [("water_flooding", 10), ("seep",), ("wind", 4), ("freq",)]
    assert ws == "ws" and sim.last_hydrology == (["fs"], "seep")
    sim.ctx.calls.clear()
    xy = np.zeros((10, 2), np.float32)
    sim.frame(10, 0, water_xy=xy, hydrology=True, water_chunk=4, floods="sweep")
    assert sim.ctx.calls == [("water_flooding", 4), ("water_flooding", 4), ("water_flooding", 2), ("seep",), ("freq",)]
    sim.ctx.calls.clear()
    sim.frame(10, 0, hydrology=True)
    assert sim.ctx.calls == [("water", 10), ("flood",), ("seep",), ("freq",)]
    with pytest.raises(ValueError):
        sim.frame(10, 0, floods="sweep")
    with pytest.raises(ValueError):
        sim.frame(10, 0, hydrology=True, floods="particle")


def test_cpp_facade_compiles_with_run_flooding(tmp_path):
    import torch
    libdir = os.path.join(ROOT, "soilmachine_b200", "lib")
    exe = str(tmp_path / "facade_sweep_flood")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-Wall", "-Werror", os.path.join(ROOT, "tests", "facade_sweep_flood.cpp"),
                           "-o", exe, "-L" + libdir, "-lsoilmachine_b200", "-Wl,-rpath," + libdir])
    if torch.cuda.is_available():
        pytest.skip("a GPU is present: tests/test_sweep_flood.py runs the facade")
    from oracle import refapi
    out = subprocess.run([exe, refapi.soil_path("default")], capture_output=True, text=True, timeout=120)
    assert out.returncode == 77 and "no CUDA device" in out.stdout
