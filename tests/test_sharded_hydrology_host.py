"""CPU: the warp hydrology (soilmachine_b200/csrc/sm_hydro_coop.cuh) on a map cut into x-strips, run on the host
(tests/sharded_hydro/host_sharded.cpp).  One section pool per strip and frequency arrays split by owner, with every
pool access checked against the strip of the column the executor focused on: the golden hydrology cases must replay
byte for byte, on 2 and 3 strips, with no access outside the owner's pool."""
import ctypes as C
import os

import pytest

import _golden
import _hostsim
from _hydro_budget import _build

HERE = os.path.dirname(os.path.abspath(__file__))


class StripHostSim(_hostsim.HostSim):
    """tests/hostsim whose water_flood / seep run the warp executor on `nstrips` strips"""

    def __init__(self, nstrips, seep_mode):
        src = os.path.join(HERE, "sharded_hydro", "host_sharded.cpp")
        deps = [_hostsim.SRC, _hostsim.CORE, _hostsim.NOISE, _hostsim.HYDRO, _hostsim.COOP, _hostsim.HCOOP,
                os.path.join(HERE, "..", "soilmachine_b200", "csrc", "sm_foot.cuh")]
        self.lib = C.CDLL(_build("host_sharded", src, deps))
        self.lib.shs_violations.restype = C.c_longlong
        self.nstrips, self.seep_mode = nstrips, seep_mode

    def water_flood(self):
        hc = _hostsim.HydroCount()
        self.lib.shs_water_flood(self.nstrips, C.byref(hc))
        return hc

    def seep(self):
        hc = _hostsim.HydroCount()
        self.lib.shs_seep(self.nstrips, self.seep_mode, C.byref(hc))
        return hc

    def violations(self):
        return self.lib.shs_violations()


def _replay(case, nstrips, seep_mode, lane_order):
    g = _golden.load(case)
    hs = StripHostSim(nstrips, seep_mode)
    hs.init(int(g["dimx"]), int(g["dimy"]), int(g["scale"]), g["soils"])
    hs.lib.hs_set_mode(1, lane_order)
    try:
        hs.set_columns(_golden.cols(g, "init"))
        hs.violations()
        counters = _golden.replay_hydro(g, hs)
        return g, counters, hs.violations()
    finally:
        hs.lib.hs_set_mode(0, 0)


@pytest.mark.parametrize("case", _golden.HYDRO_CASES)
@pytest.mark.parametrize("nstrips", [2, 3])
@pytest.mark.parametrize("seep_mode", [0, 1], ids=["every_cell", "active_index"])
@pytest.mark.parametrize("lane_order", [0, 1], ids=["lanes_up", "lanes_down"])
def test_strip_routed_hydrology_replays_golden(case, nstrips, seep_mode, lane_order):
    g, counters, viol = _replay(case, nstrips, seep_mode, lane_order)
    assert viol == 0, "%d pool accesses outside the focused column's strip" % viol
    assert all(c.overflow == 0 for c in counters)
    assert all(c.floods >= f for c, f in zip(counters, g["floods"]))


def test_strip_check_catches_a_missing_focus():
    """negative control: with focus() ignored every pool access goes to strip 0, and the check must see it"""
    g = _golden.load("hydro_bigbutte_40")
    hs = StripHostSim(2, 1)
    hs.init(int(g["dimx"]), int(g["dimy"]), int(g["scale"]), g["soils"])
    hs.lib.hs_set_mode(1, 0)
    hs.lib.shs_ignore_focus(1)
    try:
        hs.set_columns(_golden.cols(g, "init"))
        hs.violations()
        for f in range(int(g["frames"])):
            hs.water_run(g["water_xy_%d" % f])
            hs.water_flood()
            hs.seep()
            hs.frequency_update()
        assert hs.violations() > 0
    finally:
        hs.lib.shs_ignore_focus(0)
        hs.lib.hs_set_mode(0, 0)
