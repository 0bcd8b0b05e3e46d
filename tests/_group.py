"""Checks of a context group (sm_create_group) against one unsharded context fed the same inputs, shared by
tests/test_group.py (virtual ranks on one GPU) and tests/multigpu_group_check.py (one rank per GPU).  Everything is
compared with == on raw bytes."""
import numpy as np

STAT_KEYS = ("steps", "sweeps", "exit_oob", "exit_evap", "exit_stall", "pool_drops", "alive")
HYDRO_KEYS = ("floods", "nested", "nested_steps", "transfers", "cells")
SEED = 17


def same(a, b, what):
    a = np.ascontiguousarray(a); b = np.ascontiguousarray(b)
    assert a.shape == b.shape, (what, a.shape, b.shape)
    if not np.array_equal(a.view(np.uint8), b.view(np.uint8)):
        bad = np.nonzero(a.reshape(-1) != b.reshape(-1))[0]
        raise AssertionError("%s differs at %d entries, first %s: %r vs %r" %
                             (what, len(bad), bad[:4], a.reshape(-1)[bad[:4]], b.reshape(-1)[bad[:4]]))


def same_map(grp, one, what, frequency=True):
    """columns (all five arrays), section count, heights, surface, frequency maps, checksum, height sum"""
    a, b = grp.download_columns(), one.download_columns()
    for k in b:
        same(a[k], b[k], "%s: columns.%s" % (what, k))
    assert grp.section_count() == one.section_count(), what + ": section count"
    assert grp.checksum() == one.checksum(), what + ": checksum"
    same(grp.heights(), one.heights(), what + ": heights")
    same(grp.surfaces(), one.surfaces(), what + ": surface")
    same(np.float64(grp.height_sum()), np.float64(one.height_sum()), what + ": height sum")
    if frequency:
        fa, fb = grp.frequency(), one.frequency()
        for k in fb:
            same(fa[k], fb[k], "%s: %s" % (what, k))


def same_stats(a, b, what):
    assert [getattr(a, k) for k in STAT_KEYS] == [getattr(b, k) for k in STAT_KEYS], (what, a.asdict(), b.asdict())


def same_budgets(grp, one, what, cells=True):
    assert grp.last_budget().asdict() == one.last_budget().asdict(), what + ": budget"
    for k in ("eroded", "deposited", "cascade_net", "discarded", "clamped", "wind_negative"):
        same(np.float64(getattr(grp.last_budget(), k)), np.float64(getattr(one.last_budget(), k)), "%s: budget.%s" % (what, k))
    if cells:
        a, b = grp.last_cell_budget(), one.last_cell_budget()
        for k in b:
            same(a[k], b[k], "%s: cell budget %s" % (what, k))


def same_hydro(grp, one, sa, sb, what):
    assert [getattr(sa, k) for k in HYDRO_KEYS] == [getattr(sb, k) for k in HYDRO_KEYS], (what, sa.asdict(), sb.asdict())
    a, b = grp.last_hydro_budget(), one.last_hydro_budget()
    for k in b:
        same(np.float64(a[k]), np.float64(b[k]), "%s: hydro budget %s" % (what, k))


def simulations(soil, dimx, dimy, devices, device=0, **kw):
    """(group, one): two host.Simulation on the same preset and seed, max_particles 4096"""
    from soilmachine_b200 import host
    grp = host.Simulation(soil, seed=SEED, dimx=dimx, dimy=dimy, max_particles=4096, devices=list(devices), **kw)
    one = host.Simulation(soil, seed=SEED, dimx=dimx, dimy=dimy, max_particles=4096, device=device, **kw)
    return grp, one


def check_frames(soil, dimx, dimy, nw, nd, devices, frames=3, device=0):
    """whole frames with the pooling hydrology and the wind batch, budget flags on, compared after every phase; the
    last frame goes through Simulation.frame() itself.  Returns the number of floods."""
    from soilmachine_b200 import host
    sg, so = simulations(soil, dimx, dimy, devices, device, budget=True, cell_budget=True)
    g, o = sg.ctx, so.ctx
    nflood = 0
    try:
        assert g.group_size() == len(devices) and o.group_size() == 1
        same_map(g, o, "initial terrain")
        host.srand(SEED)
        for f in range(frames):
            xw, xd = host.spawn_list(nw, dimx, dimy), host.spawn_list(nd, dimx, dimy)
            if f == frames - 1:
                (wa, da), (wb, db) = sg.frame(nw, nd, xw, xd, hydrology=True), so.frame(nw, nd, xw, xd, hydrology=True)
                same_stats(wa, wb, "frame() water"); same_stats(da, db, "frame() wind")
                for sa, sb in zip(sg.last_hydrology[0] + [sg.last_hydrology[1]], so.last_hydrology[0] + [so.last_hydrology[1]]):
                    same_hydro(g, o, sa, sb, "frame() hydrology")
                same_map(g, o, "after Simulation.frame()")
                break
            what = "frame %d " % f
            same_stats(g.water_run(xw), o.water_run(xw), what + "water batch")
            same_budgets(g, o, what + "water batch")
            same_map(g, o, what + "water batch")
            sa, sb = g.water_flood(), o.water_flood()
            nflood += sb.floods
            same_hydro(g, o, sa, sb, what + "floods")
            same_map(g, o, what + "floods")
            sa, sb = g.seep(), o.seep()
            same_hydro(g, o, sa, sb, what + "seep pass")
            same_map(g, o, what + "seep pass")
            same_stats(g.wind_run(xd), o.wind_run(xd), what + "wind batch")
            same_budgets(g, o, what + "wind batch")
            same_map(g, o, what + "wind batch")
            g.frequency_update(); o.frequency_update()
            same_map(g, o, what + "frequency update")
    finally:
        sg.close(); so.close()
    return nflood


def edge_columns(dimx, nranks):
    """the columns x0 - 2 .. x0 + 1 at every strip edge of a group of nranks"""
    w = (((dimx + nranks - 1) // nranks) + 15) // 16 * 16
    return sorted({x for q in range(1, nranks) for x in range(q * w - 2, q * w + 2) if 0 <= x < dimx})


def check_cell_ops(devices, device=0):
    """the single-cell calls that change the map: the golden truth table, then calls on and next to every strip edge of
    a terrain with ponds, interleaved with a water batch; the map is compared after every step"""
    import _golden
    from soilmachine_b200 import capi, host
    n = len(devices)
    g = _golden.load("column_ops")
    # the golden 8 x 8 table has no room for strips: replay it at several places of a map of 16-column strips, against
    # one context - inside rank 0 (where the reference's leftovers apply as well), across every edge, in the last strip
    dimx, dimy = 16 * n, 8
    grp = capi.Context(dimx, dimy, int(g["scale"]), devices=list(devices))
    one = capi.Context(dimx, dimy, int(g["scale"]), device=device)
    try:
        for c in (grp, one):
            c.set_soils(g["soils"])
        for shift in [0] + [16 * q - 4 for q in range(1, n)] + [dimx - 8]:
            for (kind, x, y, v, t), want in zip(g["ops"], g["remove_results"]):
                x = int(x) + shift
                if kind == 0:
                    grp.cell_add(x, int(y), float(v), int(t)); one.cell_add(x, int(y), float(v), int(t))
                else:
                    a, b = grp.cell_remove(x, int(y), float(v)), one.cell_remove(x, int(y), float(v))
                    same(np.float64(a), np.float64(b), "remove leftover")
                    if shift == 0:
                        same(np.float64(a), np.float64(want), "remove leftover against the reference")
            same_map(grp, one, "truth table at x + %d" % shift, frequency=False)
            for x, y, loop in g["cascades"]:
                grp.cell_cascade(float(x) + shift, float(y), int(loop)); one.cell_cascade(float(x) + shift, float(y), int(loop))
            same_map(grp, one, "cascades at x + %d" % shift, frequency=False)
    finally:
        grp.close(); one.close()

    dimx, dimy = 48 * n, 56
    sg, so = simulations("bigbutte", dimx, dimy, devices, device)
    g, o = sg.ctx, so.ctx
    try:
        host.srand(SEED)
        for f in range(2):                               # ponds
            xw = host.spawn_list(500, dimx, dimy)
            sg.frame(len(xw), 0, xw, hydrology=True); so.frame(len(xw), 0, xw, hydrology=True)
        same_map(g, o, "terrain with ponds")
        nsoils = len(sg.preset["soils"])
        for rnd in range(2):
            for x in edge_columns(dimx, n):
                for y in range(1 + rnd, dimy - 1, 5):
                    for c in (g, o):
                        c.cell_add(x, y, 0.05, 0)                            # standing water for the calls below
                        c.cell_seep(x, y)
                        c.cell_water_cascade(x, y, 0)
                        c.cell_water_cascade(x, y, 3)
                        c.cell_cascade(x + 0.25, y - 0.25, 3)            # 3x3 block and re-cascades straddle two owners
                        c.cell_add(x, y, 0.03, 1 + (x + y) % (nsoils - 1))   # soil under standing water: pop, push, re-add
                        c.cell_add(x, y, 0.02, 0)
                        c.cell_remove(x, y, 0.011)
                same_map(g, o, "round %d, calls at column %d" % (rnd, x))
            # a batch in between: pool slots freed by the batch are reused by the cell calls and the reverse
            xw = host.spawn_list(400, dimx, dimy)
            same_stats(g.water_run(xw), o.water_run(xw), "water batch between the cell calls")
            same_map(g, o, "round %d, water batch" % rnd)
    finally:
        sg.close(); so.close()
