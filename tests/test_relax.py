"""Slope relaxation on the device (sm_relax): the fixture's reference results (tests/golden/relax_ops.npz) with stats equal
to the host build's; one pass against sm_cell_cascade called cell by cell; where oracle/_ref is built, the reference
driven live after real batches, hydrology and a steep layer raster; the pool after a relax; budget flags; refusals;
groups against one context; the C++ facade."""
import os
import subprocess

import numpy as np
import pytest

from _group import same
from test_apply_layer import _ctx, _frame, _group_edges, _lists
from test_apply_layer_host import KEYS
from test_relax_host import CASES, FIX, K, LOOPS, Relax, after_k, base_columns, fixture_passes, scale, steep_columns

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SEED = 31


def _same_cols(a, b, what):
    for k in KEYS:
        same(a[k], b[k], "%s: columns.%s" % (what, k))


def _fixture_ctx(case, **kw):
    from soilmachine_b200 import capi
    dimx, dimy = int(FIX[case + "_dimx"]), int(FIX[case + "_dimy"])
    c = capi.Context(dimx, dimy, scale(case), max_particles=64, **kw)
    c.set_soils(FIX[case + "_soils"])
    cols = base_columns(case)
    c.upload_columns(cols["offsets"], cols["type"], cols["size"], cols["saturation"])
    c.apply_layer(FIX[case + "_delta"].reshape(dimx, dimy), int(FIX[case + "_type"]))
    assert c.checksum() == int(FIX[case + "_sum_in"]), case + ": steep input"
    return c


def steep_raster(rng, dimx, dimy, edges=None, amp=1.0):
    """piles, pits and a cliff line; edges: the piles and pits only within 3 columns of these x"""
    d = np.zeros((dimx, dimy))
    xs = rng.integers(0, dimx, 60) if edges is None else np.concatenate(
        [np.clip(rng.integers(e - 3, e + 4, 20), 0, dimx - 1) for e in edges])
    for x in xs:
        d[x, rng.integers(0, dimy)] += rng.uniform(0.2, 0.8) * amp
    for x in xs[::3]:
        d[x, rng.integers(0, dimy)] = -rng.uniform(0.1, 0.4) * amp
    for e in ([dimx // 2] if edges is None else edges):
        d[max(e - 1, 0), :] += 0.3 * amp
    return d


@pytest.mark.parametrize("tl", LOOPS)
@pytest.mark.parametrize("case", CASES)
def test_fixture_equals_the_reference_and_the_host_build(case, tl):
    key = "%s_t%d_" % (case, tl)
    sums, nsec = FIX[key + "sums"], FIX[key + "nsec"]
    c = _fixture_ctx(case)
    try:
        for k in range(min(len(sums), 6)):
            st = c.relax(1, tl)
            assert st.passes == 1 and st.pool_drops == 0
            assert c.checksum() == int(sums[k]), "%s tl %d pass %d: checksum" % (case, tl, k + 1)
            assert c.section_count() == int(nsec[k]), "%s tl %d pass %d: sections" % (case, tl, k + 1)
            if k + 1 == K and key + "cells" in FIX:
                _same_cols(c.download_columns(), after_k(case, tl), "%s tl %d after %d passes" % (case, tl, K))
    finally:
        c.close()
    # one call over the fixture's passes: stats equal the host build's, the stale bits skip most visits
    n, stable = fixture_passes(case, tl), int(FIX[key + "stable"])
    passes = n + 5 if stable else n
    c = _fixture_ctx(case)
    try:
        st = c.relax(passes, tl)
        h = Relax(case, steep_columns(case))
        rc, hst, _ = h.run(passes, tl)
        assert rc == 0
        assert (st.passes, st.stable, st.visits, st.transfers, st.pool_drops) == tuple(int(v) for v in hst[:5])
        assert c.checksum() == int(sums[n - 1])
        _same_cols(c.download_columns(), h.columns(), "%s tl %d: the call vs the host build" % (case, tl))
        if stable:      # the golden terrains are unstable almost everywhere; the flat map relaxes around its edits
            cells = int(FIX[case + "_dimx"]) * int(FIX[case + "_dimy"])
            assert st.stable == 1 and st.passes == stable
            assert st.visits < cells * st.passes // 2, "the stale bits skip most visits after pass 1"
        assert st.device_ms > 0
    finally:
        c.close()


def test_one_pass_equals_the_single_cell_calls():
    """relax(1, tl) and sm_cell_cascade at every cell in the canonical order give the same snapshot"""
    dim = 40
    for tl in (0, 1, 3):
        a, pre = _ctx("rocksand", dim, dim)
        b, _ = _ctx("rocksand", dim, dim)
        try:
            a.initialize(SEED, pre["layers"])
            a.apply_layer(steep_raster(np.random.default_rng(tl), dim, dim), 2)
            b.restore(a.snapshot())
            st = a.relax(1, tl)
            P = 2 * (1 + tl) + 1
            for p in range(P * P):
                for x in range(p // P, dim, P):
                    for y in range(p % P, dim, P):
                        b.cell_cascade(x, y, tl)
            assert st.visits == dim * dim and st.transfers > 0
            same(a.snapshot(), b.snapshot(), "transferloop %d: relax vs sm_cell_cascade" % tl)
        finally:
            a.close(); b.close()


@pytest.mark.parametrize("soil,dim", [("default", 128), ("rocksand", 192)])
def test_after_batches_and_a_raster_equals_the_reference(soil, dim):
    import importlib.util
    from oracle import refapi
    from soilmachine_b200 import checksum
    if not refapi.available():
        pytest.skip("oracle/_ref is not built")
    spec = importlib.util.spec_from_file_location("mk", os.path.join(ROOT, "tests", "golden", "make_relax_golden.py"))
    mk = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mk)
    lists = _lists(dim, dim, 1, 1500, 300)
    t = 1
    d = steep_raster(np.random.default_rng(dim), dim, dim)
    for tl in (0, 1, 3):
        c, pre = _ctx(soil, dim, dim)
        try:
            c.initialize(SEED, pre["layers"])
            for xw, xd in lists:
                _frame(c, xw, xd)
            c.apply_layer(d, t)
            r = refapi.get().init(soil, seed=SEED, dimx=dim, dimy=dim, poolsize=32 * dim * dim)
            for xw, xd in lists:
                r.water_run(xw); r.water_flood(); r.seep(); r.wind_run(xd); r.frequency_update()
            mk.apply_raster(r, d.reshape(-1), t, dim)
            _same_cols(c.download_columns(), r.columns(), "%s %d: the steep map vs the reference" % (soil, dim))
            for k in range(2):
                st = c.relax(1, tl)
                mk.relax_pass(r, dim, dim, tl)
                want = r.columns()
                _same_cols(c.download_columns(), want, "%s %d tl %d pass %d vs the reference" % (soil, dim, tl, k + 1))
                assert c.checksum() == checksum.columns_checksum(want)
                assert st.transfers > 0
        finally:
            c.close()


def test_pool_after_a_relax_serves_the_next_batches():
    """batches after a relax equal those on a context restored from the post-relax snapshot"""
    a, pre = _ctx("rocksand", 128, 128)
    b, _ = _ctx("rocksand", 128, 128)
    try:
        a.initialize(SEED, pre["layers"])
        lists = _lists(128, 128, 3, 1500, 300)
        _frame(a, *lists[0])
        a.apply_layer(steep_raster(np.random.default_rng(9), 128, 128), 2)
        st = a.relax(7, 1)
        assert st.transfers > 0
        b.restore(a.snapshot())
        for xw, xd in lists[1:]:
            assert _frame(a, xw, xd) == _frame(b, xw, xd)
            assert a.checksum() == b.checksum()
            _same_cols(a.download_columns(), b.download_columns(), "after a batch")
            a.relax(3, 0)
            b.restore(a.snapshot())
    finally:
        a.close(); b.close()


def test_budget_flags_and_frequency_change_nothing():
    dim = 96
    plain, pre = _ctx("bigbutte", dim, dim)
    cb, _ = _ctx("bigbutte", dim, dim, cell_budget=True)
    hb, _ = _ctx("bigbutte", dim, dim, hydro_cell_budget=True)
    try:
        for m in (plain, cb, hb):
            m.initialize(SEED, pre["layers"])
            for xw, xd in _lists(dim, dim, 1, 900, 200):
                _frame(m, xw, xd)
        maps = cb.last_cell_budget(), cb.last_budget().asdict(), hb.last_hydro_cell_budget(), hb.last_hydro_budget()
        freq = [m.frequency() for m in (plain, cb, hb)]
        d = steep_raster(np.random.default_rng(11), dim, dim)
        sts = []
        for m in (plain, cb, hb):
            m.apply_layer(d, 2)
            sts.append(m.relax(4, 1).asdict())
        for s in sts[1:]:
            assert {k: v for k, v in s.items() if k != "device_ms"} == {k: v for k, v in sts[0].items() if k != "device_ms"}
        for m in (cb, hb):
            same(m.snapshot(), plain.snapshot(), "snapshot with budget flags")
        after = cb.last_cell_budget(), cb.last_budget().asdict(), hb.last_hydro_cell_budget(), hb.last_hydro_budget()
        for k in maps[0]:
            same(after[0][k], maps[0][k], "cell budget " + k)
        assert after[1] == maps[1] and after[3] == maps[3]
        for k in maps[2]:
            same(after[2][k], maps[2][k], "hydro cell budget " + k)
        for m, f in zip((plain, cb, hb), freq):
            g = m.frequency()
            for k in f:
                same(g[k], f[k], "frequency " + k)
    finally:
        plain.close(); cb.close(); hb.close()


def test_refusals_leave_the_map_unchanged():
    from soilmachine_b200 import capi, sharded
    c, pre = _ctx("rocksand", 64, 64)
    try:
        c.initialize(SEED, pre["layers"])
        before = c.snapshot()
        for mp, tl in ((1, -1), (1, 4), (0, 0), (-3, 1)):
            with pytest.raises(capi.SoilMachineError) as e:
                c.relax(mp, tl)
            assert e.value.code == capi.SM_ERR_INVALID
        same(c.snapshot(), before, "after the refusals")
    finally:
        c.close()
    v = sharded.VirtualShards(2, 64, 64, pre["world"]["scale"])
    try:
        v.set_soils(pre["soils"])
        v.initialize(SEED, pre["layers"])
        sums = [r.checksum() for r in v.ctx]
        for r in v.ctx:
            with pytest.raises(capi.SoilMachineError) as e:
                r.relax(2, 0)
            assert e.value.code == capi.SM_ERR_INVALID
        assert [r.checksum() for r in v.ctx] == sums
    finally:
        v.close()


@pytest.mark.parametrize("n", [2, 3])
def test_group_equals_one_context(n):
    dimx, dimy, soil = 160, 96, "rocksand"
    one, pre = _ctx(soil, dimx, dimy)
    g, _ = _ctx(soil, dimx, dimy, devices=[0] * n)
    try:
        for m in (one, g):
            m.initialize(SEED, pre["layers"])
        edges = _group_edges(dimx, n)
        lists = _lists(dimx, dimy, 2, 1200, 250)
        for step, tl in enumerate((1, 3, 0)):
            if step < len(lists):
                assert _frame(one, *lists[step]) == _frame(g, *lists[step])
            d = steep_raster(np.random.default_rng(70 + step), dimx, dimy, edges=edges)
            one.apply_layer(d, 1 + step % 2)
            g.apply_layer(d, 1 + step % 2)
            so, sg = one.relax(6, tl).asdict(), g.relax(6, tl).asdict()
            so.pop("device_ms"); sg.pop("device_ms")
            assert so == sg, (so, sg)
            assert so["transfers"] > 0
            assert g.checksum() == one.checksum(), "group of %d, step %d: checksum" % (n, step)
            same(g.snapshot(), one.snapshot(), "group of %d, step %d: snapshot" % (n, step))
        # a batch after the relax: the pools of the ranks are consistent
        xw, xd = _lists(dimx, dimy, 1, 1000, 200, seed=5)[0]
        assert _frame(one, xw, xd) == _frame(g, xw, xd)
        assert g.checksum() == one.checksum()
    finally:
        one.close(); g.close()


def test_facade_relax(tmp_path):
    """tests/facade_relax.cpp relaxes the map through Layermap::relax, plain and on a group of two: the same checksum
    and stats, equal to capi on the facade's map"""
    from oracle import refapi
    from soilmachine_b200 import capi
    libdir = os.path.join(ROOT, "soilmachine_b200", "lib")
    exe = str(tmp_path / "facade_relax")
    subprocess.check_call(["g++", "-std=c++17", "-O1", os.path.join(ROOT, "tests", "facade_relax.cpp"), "-o", exe,
                           "-L" + libdir, "-lsoilmachine_b200", "-Wl,-rpath," + libdir])
    soil = refapi.soil_path("rocksand")
    lines = []
    for group in (False, True):
        env = {k: v for k, v in os.environ.items() if k not in ("SM_GPUS", "SM_GPU_DEVICES")}
        if group:
            env.update(SM_GPUS="2", SM_GPU_DEVICES="0,0")
        b = str(tmp_path / ("b%d.snap" % group))
        out = subprocess.run([exe, soil, "1", b], capture_output=True, text=True, timeout=900, env=env)
        assert out.returncode == 0, out.stdout + out.stderr
        lines.append(out.stdout.strip())
        c, pre = _ctx("rocksand", 96, 72)
        try:
            c.restore(np.fromfile(b, np.uint8))
            st = c.relax(5, 1)
            assert lines[-1] == "checksum %016x passes %d visits %d transfers %d" % (
                c.checksum(), st.passes, st.visits, st.transfers), lines[-1]
        finally:
            c.close()
    assert lines[0] == lines[1]
