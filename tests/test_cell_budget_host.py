"""CPU: the per-cell maps of the mass budget (sm_last_cell_budget).  The product's warp-cooperative step with the map
hooks (soilmachine_b200/csrc/sm_coop.cuh, run on the host: tests/cell_budget/host_cells.cpp) against the oracle port's
restatement (tests/cell_budget/port_cells.cpp) byte for byte, on the golden frames, water batch then wind batch."""
import numpy as np
import pytest
import _golden
from _cell_budget import TERMS, CellHostSim, CellPort

EPS = np.finfo(np.float64).eps


def check_maps(maps, nops, h0, h1, budget_sums, what):
    """per-cell identity, untouched cells, and the sums against the per-particle budget"""
    e, d, c = (maps[k] for k in TERMS)
    # each measurement is a difference of two heights (one rounding) added to a running total (another): a cell's
    # identity closes to 4 ulp of the largest quantity involved per measurement
    scale = np.maximum(np.abs(h0), np.abs(h1)) + np.abs(e) + np.abs(d) + np.abs(c)
    err = np.abs((h1 - h0) - (d - e + c))
    tol = 4 * EPS * scale * np.maximum(nops, 1)
    bad = np.argwhere(err > tol)
    assert len(bad) == 0, "%s: identity fails at %d cells, first %s: err %r tol %r" % (
        what, len(bad), bad[:3].tolist(), err[tuple(bad[0])], tol[tuple(bad[0])])
    # cells nothing measured hold +0.0 exactly
    for k in TERMS:
        z = maps[k][nops == 0]
        assert np.all(z.view(np.uint64) == 0), "%s: %s non-zero on an untouched cell" % (what, k)
    # the sums over cells against the per-particle budget's batch sums (eroded, deposited, cascade_net)
    for i, k in enumerate(TERMS):
        s = float(np.sum(maps[k]))
        tol = 1e-9 * (float(np.sum(np.abs(maps[k]))) + 1e-300)
        assert abs(s - budget_sums[i]) <= tol, (what, k, s, budget_sums[i])


def run_case(case, lane_order, split):
    """returns which terms were non-zero somewhere on the case"""
    g = _golden.load(case)
    dims = (int(g["dimx"]), int(g["dimy"]), int(g["scale"]))
    hs = CellHostSim(split)
    hs.init(*dims, g["soils"])
    hs.lib.hs_set_mode(1, lane_order)
    po = CellPort().init(*dims, g["soils"])
    seen = dict.fromkeys(TERMS, False)
    try:
        hs.set_columns(_golden.cols(g, "init"))
        po.set_columns(_golden.cols(g, "init"))
        batches = [("water", g["water_xy"], "after_water")]
        if len(g["wind_xy"]):
            batches.append(("wind", g["wind_xy"], None))
        for kind, xy, golden_cols in batches:
            h0 = po.heights()
            getattr(hs, kind + "_run")(xy)
            getattr(po, kind + "_run")(xy)
            what = "%s %s batch" % (case, kind)
            if golden_cols:
                _golden.same_cols(hs.columns(), _golden.cols(g, golden_cols), what + ": host columns")
                _golden.same_cols(po.columns(), _golden.cols(g, golden_cols), what + ": port columns")
            else:
                _golden.same_cols(hs.columns(), po.columns(), what + ": columns")
            pm, nops = po.cell_budget()
            hm = hs.cell_budget()
            for k in TERMS:
                _golden.same(hm[k], pm[k], what + ": " + k)
                seen[k] |= bool(np.any(pm[k] != 0))
            per, sums = po.budget()
            _golden.same(hs.budget(), per, what + ": per-particle budget")
            check_maps(pm, nops, h0, po.heights(), sums, what)
        for b in (hs, po):
            b.frequency_update()
        _golden.same_cols(hs.columns(), _golden.cols(g, "after_frame"), case + ": host columns after the frame")
    finally:
        hs.lib.hs_set_mode(0, 0)
    return seen


@pytest.mark.parametrize("case", _golden.FRAME_CASES)
@pytest.mark.parametrize("lane_order", [0, 1], ids=["lanes_up", "lanes_down"])
@pytest.mark.parametrize("split", [0, 1], ids=["whole_block", "exact_staging"])
def test_warp_cell_maps_match_port(case, lane_order, split):
    """the host-emulated warp step's maps equal the port's byte for byte, the columns stay the golden ones, the
    per-cell identity closes, untouched cells hold 0.0 and the maps sum to the per-particle budget"""
    seen = run_case(case, lane_order, split)
    missing = [k for k, v in seen.items() if not v]
    assert not missing, (case, missing)
