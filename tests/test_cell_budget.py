"""GPU: the per-cell maps of the mass budget (sm_last_cell_budget) on the device.  Byte for byte against the oracle
port's restatement (tests/cell_budget/port_cells.cpp; no reference checkout needed) under every sweep schedule, on
sharded maps (in one process and over CUDA IPC) against one context, through the stepping interface, untouched by
the hydrology; contexts with and without the flags compute the same batches; and the error cases."""
import os
import subprocess
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

TERMS = ("eroded", "deposited", "cascade_net")
SHAPES = [(2, "rocksand", 128, 96, 900, 500),          # as test_sharded_views.py: the 4-rank map has a narrow last strip
          (3, "rockgravelpebblessand", 144, 80, 900, 700),
          (4, "default", 160, 64, 600, 300)]


def _same(a, b, what):
    import _golden
    _golden.same(a, b, what)


def _same_maps(a, b, what):
    for k in TERMS:
        _same(a[k], b[k], "%s: %s" % (what, k))


def _ctx(soil, dim, n, budget=False, cell_budget=False):
    import soilmachine_b200 as smb
    from soilmachine_b200 import presets
    pre = presets.load(soil)
    ctx = smb.Context(dim, dim, pre["world"]["scale"], max_particles=n, budget=budget, cell_budget=cell_budget)
    ctx.set_soils(pre["soils"])
    ctx.initialize(42, pre["layers"])
    return ctx, pre


def _spawn(n, dimx, dimy, seed):
    from soilmachine_b200 import host
    host.srand(seed)
    return host.spawn_list(n, dimx, dimy)


@pytest.mark.parametrize("exact", ["0", "1", "3"])
@pytest.mark.parametrize("soil,dim,n", [("default", 128, 600), ("rocksand", 192, 1200)])
def test_cell_maps_match_port(monkeypatch, soil, dim, n, exact):
    """a water batch, then a wind batch: after each, the device's maps equal the port's byte for byte, whichever
    schedule SM_EXACT selects (the library reads it at every launch)"""
    from _cell_budget import CellPort
    monkeypatch.setenv("SM_EXACT", exact)
    ctx, pre = _ctx(soil, dim, n, cell_budget=True)
    po = CellPort().init(dim, dim, pre["world"]["scale"], pre["soils"])
    po.set_columns(ctx.download_columns())
    seen = dict.fromkeys(TERMS, False)
    try:
        for kind, seed in (("water", 5), ("wind", 6)):
            xy = _spawn(n, dim, dim, seed)
            getattr(ctx, kind + "_run")(xy)
            getattr(po, kind + "_run")(xy)
            what = "%s %s SM_EXACT=%s" % (soil, kind, exact)
            m = ctx.last_cell_budget()
            pm, _ = po.cell_budget()
            _same_maps(m, pm, what)
            for k in TERMS:
                seen[k] |= bool(np.any(m[k] != 0))
            c1, c2 = po.columns(), ctx.download_columns()
            for k in c1:
                _same(c1[k], c2[k], what + ": columns." + k)
        assert all(seen.values()), seen                             # the case exercises every term
    finally:
        ctx.close()


@pytest.mark.parametrize("nranks,soil,dimx,dimy,nw,nd", SHAPES)
def test_sharded_cell_maps_match_one_context(nranks, soil, dimx, dimy, nw, nd):
    """each rank holds its strip's maps, including what steps of the neighbouring ranks put there; the strips
    concatenated equal the unsharded maps byte for byte"""
    from soilmachine_b200 import capi, presets, sharded
    pre = presets.load(soil)
    scale = pre["world"]["scale"]
    sh = sharded.VirtualShards(nranks, dimx, dimy, scale, max_particles=4096, cell_budget=True)
    one = capi.Context(dimx, dimy, scale, max_particles=4096, cell_budget=True)
    try:
        for m in (sh, one):
            m.set_soils(pre["soils"])
            m.initialize(17, pre["layers"])
        for kind, n, seed in (("water", nw, 17), ("wind", nd, 18)):
            xy = _spawn(n, dimx, dimy, seed)
            getattr(sh, kind + "_run")(xy)
            getattr(one, kind + "_run")(xy)
            what = "%d ranks %s %s" % (nranks, soil, kind)
            ms = sh.last_cell_budget()
            assert ms["eroded"].shape == (dimx, dimy)
            _same_maps(ms, one.last_cell_budget(), what)
            _same(sh.heights(), one.heights(), what + ": heights")
    finally:
        sh.close(); one.close()


def test_cell_maps_over_cuda_ipc_two_processes_one_gpu():
    """tests/multigpu_cell_budget_check.py with two processes sharing this GPU: the neighbour's maps are CUDA-IPC
    mappings, as across GPUs.  The strips' maps must equal one unsharded context's, water and wind batch."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ, SM_ONE_GPU="1")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2",
           "--master-addr", "127.0.0.1", "--master-port", "29641",
           os.path.join(root, "tests", "multigpu_cell_budget_check.py"), "96", "400", "rocksand"]
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=900, cwd=root, env=env)
    line = [l for l in out.stdout.splitlines() if l.startswith("multigpu_cell_budget_check")]
    assert out.returncode == 0 and line and "DIFFER" not in line[0], (out.stdout[-2000:], out.stderr[-2000:])


def test_flags_change_nothing_else():
    """no flag, SM_FLAG_BUDGET and SM_FLAG_BUDGET | SM_FLAG_CELL_BUDGET: the same columns, particle states, frequency
    maps and counters after a water and a wind batch; the two budget arms the same per-particle budgets"""
    soil, dim, n = "rocksand", 192, 1200
    arms = [_ctx(soil, dim, n)[0], _ctx(soil, dim, n, budget=True)[0], _ctx(soil, dim, n, cell_budget=True)[0]]
    try:
        for kind, seed in (("water", 11), ("wind", 12)):
            xy = _spawn(n, dim, dim, seed)
            stats = [getattr(c, kind + "_run")(xy).asdict() for c in arms]
            for s in stats:
                s.pop("device_ms")
            assert stats[0] == stats[1] == stats[2], (kind, stats)
            ref = arms[0]
            for i, c in enumerate(arms[1:], 1):
                what = "%s arm %d" % (kind, i)
                a, b = ref.download_columns(), c.download_columns()
                for k in a:
                    _same(a[k], b[k], what + ": columns." + k)
                sa, sb = getattr(ref, kind + "_state")(), getattr(c, kind + "_state")()
                for k in sa:
                    _same(sa[k], sb[k], what + ": state." + k)
                fa, fb = ref.frequency(), c.frequency()
                for k in fa:
                    _same(fa[k], fb[k], what + ": frequency." + k)
            _same(arms[1].budget_particles(n), arms[2].budget_particles(n), kind + ": per-particle budgets")
            for c in arms:
                c.frequency_update()
    finally:
        for c in arms:
            c.close()


@pytest.mark.parametrize("kind", ["water", "wind"])
def test_stepping_interface_gives_the_maps_of_one_run(kind):
    """*_begin, then *_sweeps a few sweeps at a time until the batch is done: the same maps as one *_run"""
    soil, dim, n = "rocksand", 192, 1200
    a, _ = _ctx(soil, dim, n, cell_budget=True)
    b, _ = _ctx(soil, dim, n, cell_budget=True)
    try:
        xy = _spawn(n, dim, dim, 21)
        getattr(a, kind + "_run")(xy)
        getattr(b, kind + "_begin")(xy)
        for _ in range(10000):
            if getattr(b, kind + "_sweeps")(3).alive == 0:
                break
        _same_maps(a.last_cell_budget(), b.last_cell_budget(), kind + ": begin + sweeps against run")
        _same(a.heights(), b.heights(), kind + ": heights")
    finally:
        a.close(); b.close()


def test_hydrology_and_single_cell_calls_leave_the_maps():
    soil, dim, n = "default", 128, 600
    ctx, _ = _ctx(soil, dim, n, cell_budget=True)
    try:
        ctx.water_run(_spawn(n, dim, dim, 31))
        m0 = ctx.last_cell_budget()
        st = ctx.water_flood()
        assert st.floods > 0
        _same_maps(ctx.last_cell_budget(), m0, "after sm_water_flood")
        ctx.seep()
        _same_maps(ctx.last_cell_budget(), m0, "after sm_seep")
        ctx.cell_add(10, 10, 0.5, 1)
        ctx.cell_cascade(10, 10, 1)
        _same_maps(ctx.last_cell_budget(), m0, "after the single-cell calls")
    finally:
        ctx.close()


def test_cell_budget_errors(monkeypatch):
    import ctypes as C
    from soilmachine_b200 import capi
    lib = capi.load()
    # SM_FLAG_CELL_BUDGET without SM_FLAG_BUDGET
    h = C.c_void_p()
    rc = lib.sm_create(C.byref(capi.Config(64, 64, 80, 0, 0, 256, 2)), C.byref(h))
    assert rc == capi.SM_ERR_INVALID and b"SM_FLAG_BUDGET" in lib.sm_last_error(None)
    # a context without the flag
    bud, _ = _ctx("default", 64, 200, budget=True)
    bud.water_run(_spawn(200, 64, 64, 1))
    with pytest.raises(capi.SoilMachineError) as e:
        bud.last_cell_budget()
    assert e.value.code == capi.SM_ERR_INVALID and "SM_FLAG_CELL_BUDGET" in str(e.value)
    bud.last_budget()                                    # the per-particle budget is unaffected
    bud.close()
    cel, _ = _ctx("default", 64, 200, cell_budget=True)
    # before the first batch
    with pytest.raises(capi.SoilMachineError) as e:
        cel.last_cell_budget()
    assert e.value.code == capi.SM_ERR_INVALID and "no batch" in str(e.value)
    cel.water_run(_spawn(200, 64, 64, 1))
    assert set(cel.last_cell_budget()) == set(TERMS)
    # a batch on a kernel without the maps: no stale maps, no zero maps, also through the stepping interface
    monkeypatch.setenv("SM_KERNEL", "thread")
    cel.water_run(_spawn(200, 64, 64, 2))
    with pytest.raises(capi.SoilMachineError) as e:
        cel.last_cell_budget()
    assert e.value.code == capi.SM_ERR_INVALID and "SM_KERNEL=thread" in str(e.value)
    monkeypatch.setenv("SM_KERNEL", "warp")
    cel.wind_begin(_spawn(200, 64, 64, 3))
    cel.wind_sweeps(2)
    monkeypatch.setenv("SM_KERNEL", "thread")
    cel.wind_sweeps(2)
    with pytest.raises(capi.SoilMachineError) as e:
        cel.last_cell_budget()
    assert e.value.code == capi.SM_ERR_INVALID
    monkeypatch.delenv("SM_KERNEL")
    cel.wind_run(_spawn(200, 64, 64, 4))
    assert set(cel.last_cell_budget()) == set(TERMS)
    cel.close()
    # sharded ranks that disagree on the flag
    from soilmachine_b200 import presets
    pre = presets.load("default")
    ranks = [capi.Context(64, 64, pre["world"]["scale"], max_particles=256, nranks=2, rank=r, share=2,
                          budget=True, cell_budget=(r == 0)) for r in range(2)]
    blobs = [c.peer_export() for c in ranks]
    for c in ranks:
        with pytest.raises(capi.SoilMachineError) as e:
            c.peer_attach(blobs, use_ipc=False)
        assert e.value.code == capi.SM_ERR_INVALID and "SM_FLAG_CELL_BUDGET" in str(e.value)
        c.close()
