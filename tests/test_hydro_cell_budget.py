"""GPU: the per-cell maps of the pooling hydrology's mass budget (sm_last_hydro_cell_budget) on the device.  Byte for
byte against the oracle port's restatement (tests/hydro_cells/port_hydro_cells.cpp; no reference checkout needed),
the flag changes nothing else (columns, counters, budgets, batch maps), the whole-frame per-cell closure over the batch
and hydrology maps, and the error cases."""
import warnings

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

TERMS = ("eroded", "deposited", "cascade_net", "water_net")
CELL_TERMS = ("eroded", "deposited", "cascade_net")


def _same(a, b, what):
    import _golden
    _golden.same(a, b, what)


def _ctx(soil, dim, n, **flags):
    import soilmachine_b200 as smb
    from soilmachine_b200 import presets
    pre = presets.load(soil)
    ctx = smb.Context(dim, dim, pre["world"]["scale"], max_particles=n, **flags)
    ctx.set_soils(pre["soils"])
    ctx.initialize(42, pre["layers"])
    return ctx, pre


def _spawn(n, dim, seed):
    from soilmachine_b200 import host
    host.srand(seed)
    return host.spawn_list(n, dim, dim)


@pytest.mark.parametrize("soil,dim,n,frames", [("default", 128, 600, 3), ("rocksand", 192, 1200, 2)])
def test_hydro_cell_maps_match_port(soil, dim, n, frames):
    """after every flood and seep call the device's four maps equal the port restatement's bit for bit"""
    from _hydro_cells import HydroCellPort
    ctx, pre = _ctx(soil, dim, n, hydro_cell_budget=True)
    po = HydroCellPort().init(dim, dim, pre["world"]["scale"], pre["soils"])
    po.set_columns(ctx.download_columns())
    seen = dict.fromkeys(TERMS, False)
    try:
        for f in range(frames):
            xy = _spawn(n, dim, 42 + f)
            ctx.water_run(xy); po.water_run(xy)
            for name in ("water_flood", "seep"):
                getattr(ctx, name)(); getattr(po, name)()
                what = "%s frame %d %s" % (soil, f, name)
                m = ctx.last_hydro_cell_budget()
                pm, _ = po.hydro_cell_budget()
                for k in TERMS:
                    assert m[k].shape == (dim, dim)
                    _same(m[k], pm[k], what + ": " + k)
                    seen[k] |= bool(np.any(m[k] != 0))
            ctx.frequency_update(); po.frequency_update()
        c1, c2 = po.columns(), ctx.download_columns()
        for k in c1:
            _same(c1[k], c2[k], "columns." + k)
        assert all(seen.values()), seen                             # the case exercises every map
    finally:
        ctx.close()


@pytest.mark.parametrize("executor", ["thread", "warp"])
def test_hydro_cell_flag_changes_nothing_else(monkeypatch, executor):
    """SM_FLAG_BUDGET against SM_FLAG_BUDGET | SM_FLAG_HYDRO_CELL_BUDGET, and SM_FLAG_CELL_BUDGET with and without the
    new flag: identical columns, hydrology counters and eleven hydrology sums; the batch maps are the same with and
    without the new flag, and the flood and seep pass leave them as they were"""
    monkeypatch.setenv("SM_HYDRO", executor)
    soil, dim, n = "rocksand", 192, 1200
    arms = [_ctx(soil, dim, n, budget=True)[0], _ctx(soil, dim, n, hydro_cell_budget=True)[0],
            _ctx(soil, dim, n, cell_budget=True)[0], _ctx(soil, dim, n, cell_budget=True, hydro_cell_budget=True)[0]]
    try:
        for f in range(2):
            xy = _spawn(n, dim, 7 + f)
            for c in arms:
                c.water_run(xy)
            batch = [arms[2].last_cell_budget(), arms[3].last_cell_budget()]
            for k in CELL_TERMS:
                _same(batch[0][k], batch[1][k], "%s frame %d batch map %s" % (executor, f, k))
            for name in ("water_flood", "seep"):
                hs = [getattr(c, name)() for c in arms]
                what = "%s frame %d %s" % (executor, f, name)
                counts = [(h.floods, h.nested, h.nested_steps, h.transfers, h.cells) for h in hs]
                assert len(set(counts)) == 1, (what, counts)
                ref = arms[0].download_columns()
                b0 = arms[0].last_hydro_budget()
                for i, c in enumerate(arms[1:], 1):
                    cols = c.download_columns()
                    for k in ref:
                        _same(ref[k], cols[k], "%s arm %d: columns.%s" % (what, i, k))
                    assert c.last_hydro_budget() == b0, (what, i)
                m1, m3 = arms[1].last_hydro_cell_budget(), arms[3].last_hydro_cell_budget()
                for k in TERMS:
                    _same(m1[k], m3[k], "%s: hydrology map %s" % (what, k))
                for j, c in enumerate(arms[2:]):
                    after = c.last_cell_budget()
                    for k in CELL_TERMS:
                        _same(after[k], batch[j][k], "%s: batch map %s left as it was" % (what, k))
            for c in arms:
                c.frequency_update()
    finally:
        for c in arms:
            c.close()


def test_whole_frame_cell_closure():
    """water batch, flood, seep pass, wind batch on rocksand 192^2: per cell, the downloaded height change equals the
    sum of the two batch maps' and the two hydrology maps' identities.  The port restatement runs alongside: its maps
    equal the device's, and its per-cell measurement counts give the rounding bound."""
    from _hydro_cells import HydroCellPort
    soil, dim, n = "rocksand", 192, 1200
    ctx, pre = _ctx(soil, dim, n, cell_budget=True, hydro_cell_budget=True)
    po = HydroCellPort().init(dim, dim, pre["world"]["scale"], pre["soils"])
    po.set_columns(ctx.download_columns())
    zero = np.zeros((dim, dim))
    try:
        h0 = ctx.heights()
        maps, nops = [], np.zeros((dim, dim), np.int64)
        for step, seed in (("water", 3), ("flood", None), ("seep", None), ("wind", 4)):
            if seed is not None:
                xy = _spawn(n, dim, seed)
                st = getattr(ctx, step + "_run")(xy)
                getattr(po, step + "_run")(xy)
                assert st.pool_drops == 0
                m = dict(ctx.last_cell_budget(), water_net=zero)
                pm, cnt = po.cell_budget()
                pm = dict(pm, water_net=zero)
            else:
                getattr(ctx, "water_flood" if step == "flood" else "seep")()
                getattr(po, "water_flood" if step == "flood" else "seep")()
                m = ctx.last_hydro_cell_budget()
                pm, cnt = po.hydro_cell_budget()
            for k in TERMS:
                _same(m[k], pm[k], "%s: %s" % (step, k))
            maps.append(m)
            nops += cnt
        h1 = ctx.heights()
        _same(h1, po.heights(), "heights after the frame")
        ident = sum(m["deposited"] - m["eroded"] + m["cascade_net"] + m["water_net"] for m in maps)
        mag = np.maximum(np.abs(h0), np.abs(h1)) + sum(np.abs(m[k]) for m in maps for k in TERMS)
        # every measurement is one rounded difference added to a rounded running total: 4 ulp of the magnitude per
        # measurement, as the CPU tests bound a call; the height difference and the adding up of the four calls'
        # terms are a few more roundings, covered by the extra 4 ulp
        err = np.abs((h1 - h0) - ident)
        tol = 4 * np.finfo(np.float64).eps * mag * (nops + 1)
        bad = np.argwhere(err > tol)
        assert len(bad) == 0, (len(bad), bad[:3].tolist(), float(err.max()))
        # cells no measurement touched hold 0.0 in every map and did not change height
        for m in maps:
            for k in TERMS:
                assert np.all(m[k][nops == 0].view(np.uint64) == 0), k
        assert np.array_equal(h0[nops == 0], h1[nops == 0])
        assert (h1 != h0).sum() > 0 and (nops > 0).sum() > 0
        assert np.any(maps[1]["water_net"] != 0) and np.any(maps[2]["water_net"] != 0)
    finally:
        ctx.close()


def test_hydro_cell_budget_errors():
    from soilmachine_b200 import capi
    # a context without the flag
    bud, _ = _ctx("default", 64, 200, budget=True)
    bud.water_run(_spawn(200, 64, 1))
    bud.water_flood()
    with pytest.raises(capi.SoilMachineError) as e:
        bud.last_hydro_cell_budget()
    assert e.value.code == capi.SM_ERR_INVALID and "SM_FLAG_HYDRO_CELL_BUDGET" in str(e.value)
    bud.last_hydro_budget()                               # the hydrology budget is unaffected
    bud.close()
    hc, _ = _ctx("default", 64, 200, hydro_cell_budget=True)
    # before the first hydrology call; a water batch alone does not count
    with pytest.raises(capi.SoilMachineError) as e:
        hc.last_hydro_cell_budget()
    assert e.value.code == capi.SM_ERR_INVALID and "no hydrology call" in str(e.value)
    hc.water_run(_spawn(200, 64, 1))
    with pytest.raises(capi.SoilMachineError) as e:
        hc.last_hydro_cell_budget()
    assert e.value.code == capi.SM_ERR_INVALID and "no hydrology call" in str(e.value)
    hc.water_flood()
    assert set(hc.last_hydro_cell_budget()) == set(TERMS)
    hc.seep()
    assert set(hc.last_hydro_cell_budget()) == set(TERMS)
    hc.close()


def test_failed_hydrology_call_withholds_its_maps():
    """a flood that runs out of pool slots (SM_ERR_POOL, reported as a warning by the Python layer) has reset its maps
    and filled them only partly: the call refuses them"""
    import soilmachine_b200 as smb
    from soilmachine_b200 import capi, presets
    pre = presets.load("rocksand")
    dim = 64
    # a bowl of bare rock (one section per column, nothing buried): water stalls at the bottom, and every flood's Air
    # add on a rock column needs a pool slot, of which there is one
    x, y = np.meshgrid(np.arange(dim), np.arange(dim), indexing="ij")
    r2 = ((x - dim / 2) ** 2 + (y - dim / 2) ** 2) / float(dim * dim)
    size = (0.1 + 0.5 * r2).reshape(-1)
    offsets = np.arange(dim * dim + 1, dtype=np.int64)
    typ = np.ones(dim * dim, np.int32)
    ctx = smb.Context(dim, dim, 80, max_particles=2000, pool_capacity=1, hydro_cell_budget=True)
    try:
        ctx.set_soils(pre["soils"])
        ctx.upload_columns(offsets, typ, size)
        rng = np.random.RandomState(0)
        xy = (rng.rand(2000, 2) * (dim - 2) + 0.5).astype(np.float32)
        with warnings.catch_warnings(record=True) as wlist:
            warnings.simplefilter("always")
            ctx.water_run(xy)
            del wlist[:]
            st = ctx.water_flood()
        assert st.floods > 1 and any("pool" in str(w.message) for w in wlist), (st.asdict(), [str(w.message) for w in wlist])
        with pytest.raises(capi.SoilMachineError) as e:
            ctx.last_hydro_cell_budget()
        assert e.value.code == capi.SM_ERR_INVALID and "failed" in str(e.value)
    finally:
        ctx.close()
