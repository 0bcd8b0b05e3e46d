"""CPU: the pooling hydrology's mass budget (sm_last_hydro_budget).  The warp executor's accumulators
(soilmachine_b200/csrc/sm_hydro_coop.cuh, run on the host: tests/hydro_budget/host_budget.cpp) against the oracle
port's (tests/hydro_budget/port_budget.cpp) bit for bit, and the budget identity per call."""
import math
import numpy as np
import pytest
import _golden
from _hydro_budget import TERMS, BudgetHostSim, BudgetPort, identity
from oracle import portapi


def assert_closes(h0, h1, b, what):
    """d(sum of heights) = identity(b) to 1e-9 of the terms' magnitude, plus the resolution of the two sums"""
    dh = h1 - h0
    tol = 1e-9 * float(np.sum(np.abs(b[:9]))) + 4 * np.finfo(np.float64).eps * max(abs(h0), abs(h1))
    assert abs(dh - identity(b)) <= tol, (what, dh, identity(b), dict(zip(TERMS, b)))


def height_sum(backend):
    return math.fsum(backend.heights().reshape(-1))


def run_case(case, seep_mode, lane_order):
    """replay a golden hydrology case on the budget port, on the plain port and on the host-emulated warp executor side
    by side; after every flood / seep call the maps must be equal, the two budgets bit-identical and closing the
    identity.  Returns the budgets."""
    g = _golden.load(case)
    dims = (int(g["dimx"]), int(g["dimy"]), int(g["scale"]))
    hs = BudgetHostSim()
    hs.init(*dims, g["soils"])
    hs.lib.hs_set_mode(1, lane_order)
    po = BudgetPort().init(*dims, g["soils"])
    plain = portapi.Port().init(*dims, g["soils"])
    budgets = []
    try:
        for b in (hs, po, plain):
            b.set_columns(_golden.cols(g, "init"))
        for f in range(int(g["frames"])):
            xy = g["water_xy_%d" % f]
            for b in (hs, po, plain):
                b.water_run(xy)
            for name, call in (("flood", lambda: (hs.water_flood(), po.water_flood(), plain.water_flood())),
                               ("seep", lambda: (hs.seep(seep_mode), po.seep(), plain.seep()))):
                h0 = height_sum(po)
                ch, cp, cq = call()
                what = "%s frame %d %s" % (case, f, name)
                _golden.same_cols(po.columns(), plain.columns(), what + ": budget port against the port")
                assert cp.asdict() == cq.asdict(), what
                _golden.same(hs.heights(), po.heights(), what + ": heights")
                bp = po.hydro_budget()
                _golden.same(hs.hydro_budget(), bp, what + ": hydrology budget")
                assert_closes(h0, height_sum(po), bp, what)
                budgets.append(bp)
            for b in (hs, po, plain):
                b.frequency_update()
    finally:
        hs.lib.hs_set_mode(0, 0)
    return budgets


@pytest.mark.parametrize("case", _golden.HYDRO_CASES)
@pytest.mark.parametrize("seep_mode", [0, 1], ids=["every_cell", "active_index"])
@pytest.mark.parametrize("lane_order", [0, 1], ids=["lanes_up", "lanes_down"])
def test_warp_hydrology_budget_matches_port(case, seep_mode, lane_order):
    """every frame of the golden cases; the port visits every cell in the seep pass, the active-index mode only
    the flagged ones: a skipped visit adds nothing, so the sums are bit-identical either way"""
    run_case(case, seep_mode, lane_order)


def test_hydrology_budget_terms_are_exercised():
    """across the golden cases every term but nested_clamped is non-zero at least once (the clamp, water.h:117, needs
    a nested particle whose sediment exceeds 1 after evaporation, which these maps do not produce)"""
    seen = np.zeros(11, bool)
    for case in _golden.HYDRO_CASES:
        for b in run_case(case, 1, 0):
            seen |= b != 0
    missing = [t for t, s in zip(TERMS, seen) if not s and t != "nested_clamped"]
    assert not missing, missing


def test_port_hydrology_budget_with_reference_live(ref):
    """the reference's own hydrology alongside the budget port: the maps stay equal after every call, and the port's
    budget closes the identity on them"""
    po = BudgetPort()
    for soil, dim, n, frames in (("default", 96, 500, 3), ("bigbutte", 64, 500, 3)):
        ref.init(soil, seed=42, dimx=dim, dimy=dim + 8)
        po.init(ref.dimx, ref.dimy, ref.scale, ref.soils())
        po.set_columns(ref.columns())
        for f in range(frames):
            xy = ref.spawn_list(n, seed=42 + f)
            ref.water_run(xy); po.water_run(xy)
            for name, call in (("flood", lambda: (ref.water_flood(), po.water_flood())),
                               ("seep", lambda: (ref.seep(), po.seep()))):
                h0 = height_sum(po)
                call()
                what = "%s frame %d %s" % (soil, f, name)
                _golden.same_cols(ref.columns(), po.columns(), what)
                assert_closes(h0, height_sum(po), po.hydro_budget(), what)
            ref.frequency_update(); po.frequency_update()
