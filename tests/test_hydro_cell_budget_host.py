"""CPU: the per-cell maps of the pooling hydrology's mass budget (sm_last_hydro_cell_budget).  The product's warp
hydrology with the map hooks (soilmachine_b200/csrc/sm_hydro_coop.cuh, run on the host:
tests/hydro_cells/host_hydro_cells.cpp) against the oracle port's restatement (tests/hydro_cells/port_hydro_cells.cpp)
byte for byte, after every flood and seep call of the golden hydrology cases; and the sm_create refusals, which come
before the device check."""
import ctypes as C
import numpy as np
import pytest
import _golden
from _hydro_budget import BudgetPort
from _hydro_cells import TERMS, HydroCellHostSim, HydroCellPort, slot_sum
from oracle import portapi

EPS = np.finfo(np.float64).eps


def check_maps(maps, nops, h0, h1, budget, what):
    """per-cell identity, untouched cells, and the sums against the hydrology budget's slots"""
    e, d, c, w = (maps[k] for k in TERMS)
    # each measurement is a difference of two heights (one rounding) added to a running total (another): a cell's
    # identity closes to 4 ulp of the largest quantity involved per measurement
    scale = np.maximum(np.abs(h0), np.abs(h1)) + np.abs(e) + np.abs(d) + np.abs(c) + np.abs(w)
    err = np.abs((h1 - h0) - (d - e + c + w))
    tol = 4 * EPS * scale * np.maximum(nops, 1)
    bad = np.argwhere(err > tol)
    assert len(bad) == 0, "%s: identity fails at %d cells, first %s: err %r tol %r" % (
        what, len(bad), bad[:3].tolist(), err[tuple(bad[0])], tol[tuple(bad[0])])
    # cells nothing measured hold +0.0 exactly, and their height did not change
    for k in TERMS:
        z = maps[k][nops == 0]
        assert np.all(z.view(np.uint64) == 0), "%s: %s non-zero on an untouched cell" % (what, k)
    assert np.array_equal(h0[nops == 0], h1[nops == 0]), what + ": an untouched cell changed height"
    # the sums over cells against the groups of hydrology-budget slots they refine
    for k in TERMS:
        s = float(np.sum(maps[k]))
        ref = slot_sum(budget, k)
        tol = 1e-9 * (float(np.sum(np.abs(maps[k]))) + 1e-300)
        assert abs(s - ref) <= tol, (what, k, s, ref)


def run_case(case, seep_mode, lane_order):
    """replay a golden hydrology case on the host-emulated warp executor with the maps, the port restatement with
    the maps, the budget port and the plain port side by side.  Returns which maps were non-zero somewhere."""
    g = _golden.load(case)
    dims = (int(g["dimx"]), int(g["dimy"]), int(g["scale"]))
    hs = HydroCellHostSim()
    hs.init(*dims, g["soils"])
    hs.lib.hs_set_mode(1, lane_order)
    po = HydroCellPort().init(*dims, g["soils"])
    bp = BudgetPort().init(*dims, g["soils"])
    plain = portapi.Port().init(*dims, g["soils"])
    seen = dict.fromkeys(TERMS, False)
    try:
        for b in (hs, po, bp, plain):
            b.set_columns(_golden.cols(g, "init"))
        for f in range(int(g["frames"])):
            xy = g["water_xy_%d" % f]
            for b in (hs, po, bp, plain):
                b.water_run(xy)
            for name in ("flood", "seep"):
                h0 = po.heights()
                if name == "flood":
                    ch, cp, cb, cq = hs.water_flood(), po.water_flood(), bp.water_flood(), plain.water_flood()
                else:
                    ch, cp, cb, cq = hs.seep(seep_mode), po.seep(), bp.seep(), plain.seep()
                what = "%s frame %d %s" % (case, f, name)
                _golden.same_cols(po.columns(), plain.columns(), what + ": restatement against the port")
                assert cp.asdict() == cq.asdict(), what
                _golden.same(hs.heights(), po.heights(), what + ": heights")
                pm, nops = po.hydro_cell_budget()
                hm = hs.hydro_cell_budget()
                for k in TERMS:
                    _golden.same(hm[k], pm[k], what + ": " + k)
                    seen[k] |= bool(np.any(pm[k] != 0))
                budget = bp.hydro_budget()
                _golden.same(hs.hydro_budget(), budget, what + ": hydrology budget")
                check_maps(pm, nops, h0, po.heights(), budget, what)
            for b in (hs, po, bp, plain):
                b.frequency_update()
    finally:
        hs.lib.hs_set_mode(0, 0)
    return seen


@pytest.mark.parametrize("case", _golden.HYDRO_CASES)
@pytest.mark.parametrize("seep_mode", [0, 1], ids=["every_cell", "active_index"])
@pytest.mark.parametrize("lane_order", [0, 1], ids=["lanes_up", "lanes_down"])
def test_warp_hydrology_cell_maps_match_port(case, seep_mode, lane_order):
    """the host-emulated warp executor's maps equal the port restatement's byte for byte after every flood and seep
    call, the restatement leaves the port's columns and counters, the per-cell identity closes, untouched cells hold
    0.0 and each map sums to its group of hydrology-budget slots"""
    run_case(case, seep_mode, lane_order)


def test_hydrology_cell_maps_are_exercised():
    """across the golden cases every one of the four maps is non-zero somewhere, so every site is exercised"""
    seen = dict.fromkeys(TERMS, False)
    for case in _golden.HYDRO_CASES:
        for k, v in run_case(case, 1, 0).items():
            seen[k] |= v
    missing = [k for k, v in seen.items() if not v]
    assert not missing, missing


def test_create_refuses_the_flag_without_budget_or_sharded():
    """both refusals come before the device check, so they hold on a machine without a GPU"""
    from soilmachine_b200 import capi
    lib = capi.load()
    h = C.c_void_p()
    rc = lib.sm_create(C.byref(capi.Config(64, 64, 80, 0, 0, 256, 4)), C.byref(h))
    assert rc == capi.SM_ERR_INVALID and b"SM_FLAG_HYDRO_CELL_BUDGET needs SM_FLAG_BUDGET" in lib.sm_last_error(None)
    rc = lib.sm_create_sharded(C.byref(capi.Config(64, 64, 80, 0, 0, 256, 1 | 4)), 2, 0, 2, C.byref(h))
    assert rc == capi.SM_ERR_INVALID and b"sharded" in lib.sm_last_error(None)
    # the same through the Python interface
    with pytest.raises(capi.SoilMachineError) as e:
        capi.Context(64, 64, 80, max_particles=256, nranks=2, rank=0, share=2, hydro_cell_budget=True)
    assert e.value.code == capi.SM_ERR_INVALID and "SM_FLAG_HYDRO_CELL_BUDGET" in str(e.value)
