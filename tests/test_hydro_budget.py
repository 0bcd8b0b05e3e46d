"""GPU: the pooling hydrology's mass budget (sm_last_hydro_budget) on the device.  Bit for bit against the oracle
port's accumulators (tests/hydro_budget/port_budget.cpp, the port compiled with the budget; no reference checkout
needed), the maps of a budget context against a context without the flag, the whole-frame closure and the error
cases."""
import math
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

TERMS = ("flood_sediment", "flood_cascade_net", "flood_water", "seeped", "to_particles", "transfer_net",
         "nested_eroded", "nested_deposited", "nested_cascade_net", "nested_discarded", "nested_clamped")


def _same(a, b, what):
    import _golden
    _golden.same(a, b, what)


def _ctx(soil, dim, n, budget):
    import soilmachine_b200 as smb
    from soilmachine_b200 import presets
    pre = presets.load(soil)
    ctx = smb.Context(dim, dim, pre["world"]["scale"], max_particles=n, budget=budget)
    ctx.set_soils(pre["soils"])
    ctx.initialize(42, pre["layers"])
    return ctx, pre


def _spawn(n, dim, seed):
    from soilmachine_b200 import host
    host.srand(seed)
    return host.spawn_list(n, dim, dim)


def _vec(d):
    return np.array([d[k] for k in TERMS])


def _hydro_identity(b):
    return b[0] + b[1] + b[2] - b[3] - b[4] + b[5] + b[7] - b[6] + b[8]


def _assert_closes(h0, h1, ident, mag, ulps, what):
    """h1 - h0 = ident to 1e-9 of the terms' magnitude, plus the rounding of the two height sums (`ulps` units of
    eps times the sum: the map holds tens of thousands of columns, so that can exceed the first bound)"""
    dh = h1 - h0
    tol = 1e-9 * mag + ulps * np.finfo(np.float64).eps * max(abs(h0), abs(h1))
    assert abs(dh - ident) <= tol, (what, dh, ident, tol)


def _exact_sum(ctx):
    """the height sum of the downloaded map, correctly rounded"""
    return math.fsum(ctx.heights().reshape(-1))


@pytest.mark.parametrize("soil,dim,n,frames", [("default", 128, 600, 3), ("rocksand", 192, 1200, 2)])
def test_hydro_budget_matches_port(soil, dim, n, frames):
    """after every flood and seep call the device's eleven sums equal the port's bit for bit, and close the
    identity against the height sum of the downloaded map"""
    from _hydro_budget import BudgetPort
    ctx, pre = _ctx(soil, dim, n, True)
    po = BudgetPort().init(dim, dim, pre["world"]["scale"], pre["soils"])
    po.set_columns(ctx.download_columns())
    seen = np.zeros(len(TERMS), bool)
    for f in range(frames):
        xy = _spawn(n, dim, 42 + f)
        ctx.water_run(xy); po.water_run(xy)
        for name, call in (("flood", lambda: (ctx.water_flood(), po.water_flood())),
                           ("seep", lambda: (ctx.seep(), po.seep()))):
            h0 = _exact_sum(ctx)
            call()
            what = "%s frame %d %s" % (soil, f, name)
            b = _vec(ctx.last_hydro_budget())
            _same(b, po.hydro_budget(), what + ": hydrology budget")
            _assert_closes(h0, _exact_sum(ctx), _hydro_identity(b), np.abs(b[:9]).sum(), 2, what)
            seen |= b != 0
    c1, c2 = po.columns(), ctx.download_columns()
    for k in c1:
        _same(c1[k], c2[k], "columns." + k)
    assert seen[TERMS.index("flood_water")]               # the case exercises the path
    ctx.close()


@pytest.mark.parametrize("executor", ["thread", "warp"])
def test_budget_context_hydrology_maps_unchanged(monkeypatch, executor):
    """a budget context (always the warp executor) leaves the same map and counters as a context without the flag
    on either executor"""
    monkeypatch.setenv("SM_HYDRO", executor)
    soil, dim, n = "rocksand", 192, 1200
    a, _ = _ctx(soil, dim, n, True)
    b, _ = _ctx(soil, dim, n, False)
    for f in range(2):
        xy = _spawn(n, dim, 7 + f)
        a.water_run(xy); b.water_run(xy)
        for name in ("water_flood", "seep"):
            ha, hb = getattr(a, name)(), getattr(b, name)()
            what = "%s frame %d %s" % (executor, f, name)
            assert (ha.floods, ha.nested, ha.nested_steps, ha.transfers, ha.cells) == \
                (hb.floods, hb.nested, hb.nested_steps, hb.transfers, hb.cells), what
            c1, c2 = a.download_columns(), b.download_columns()
            for k in c1:
                _same(c1[k], c2[k], what + ": columns." + k)
        a.frequency_update(); b.frequency_update()
    a.close(); b.close()


def test_whole_frame_budget_closes():
    """water batch, flood, seep pass, wind batch: the change of sm_height_sum over the frame is the sum of the two
    batches' and the two hydrology calls' identities"""
    soil, dim, n = "rocksand", 192, 1200
    ctx, _ = _ctx(soil, dim, n, True)
    h0 = ctx.height_sum()
    ident, mag = [], 0.0
    st = ctx.water_run(_spawn(n, dim, 3))
    assert st.pool_drops == 0
    bw = ctx.last_budget()
    ident.append(bw.deposited - bw.eroded + bw.cascade_net)
    mag += bw.deposited + bw.eroded + abs(bw.cascade_net)
    for call in (ctx.water_flood, ctx.seep):
        call()
        b = _vec(ctx.last_hydro_budget())
        ident.append(_hydro_identity(b))
        mag += np.abs(b[:9]).sum()
    st = ctx.wind_run(_spawn(n, dim, 4))
    assert st.pool_drops == 0
    bd = ctx.last_budget()
    assert bd.eroded > 0                                   # sand the wind can lift: the wind batch does real work
    ident.append(bd.deposited - bd.eroded + bd.cascade_net)
    mag += bd.deposited + bd.eroded + abs(bd.cascade_net)
    # sm_height_sum adds a few cells per thread, then reduces over 256 threads and the blocks: 32 eps is ample
    _assert_closes(h0, ctx.height_sum(), math.fsum(ident), mag, 32, "whole frame")
    ctx.close()


def test_hydro_budget_errors():
    from soilmachine_b200 import capi
    plain, _ = _ctx("default", 64, 200, False)
    plain.water_run(_spawn(200, 64, 1))
    plain.water_flood()
    with pytest.raises(capi.SoilMachineError) as e:
        plain.last_hydro_budget()
    assert e.value.code == capi.SM_ERR_INVALID and "SM_FLAG_BUDGET" in str(e.value)
    plain.close()
    bud, _ = _ctx("default", 64, 200, True)
    bud.water_run(_spawn(200, 64, 1))
    with pytest.raises(capi.SoilMachineError) as e:
        bud.last_hydro_budget()                          # a batch, but no hydrology call yet
    assert e.value.code == capi.SM_ERR_INVALID
    bud.water_flood()
    assert set(bud.last_hydro_budget()) == set(TERMS)
    bud.close()
