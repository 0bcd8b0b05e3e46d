"""Layer rasters on the device (sm_apply_layer): the fixture's reference results (tests/golden/layer_ops.npz), the host
build of the per-cell logic and, where oracle/_ref is built, the reference driven live, after real batches and the
pooling hydrology; equality with the single-cell calls; the pool after an apply; sharded maps and groups against one
context; refusals; budget flags; the C++ facade; two processes over CUDA IPC (tests/multigpu_apply_check.py)."""
import ctypes as C
import importlib.util
import os
import subprocess
import sys

import numpy as np
import pytest

from _group import same
from test_apply_layer_host import CASES, FIX, KEYS, Image, _input, _lib as _host_lib, _output, _raster
from test_snapshot_host import _lib as _snap_lib

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SEED = 31
STAT_KEYS = ("steps", "sweeps", "exit_oob", "exit_evap", "exit_stall", "pool_drops", "alive")


def _ctx(soil, dimx, dimy, **kw):
    from soilmachine_b200 import capi, presets
    pre = presets.load(soil)
    c = capi.Context(dimx, dimy, pre["world"]["scale"], max_particles=kw.pop("max_particles", 4096), **kw)
    c.set_soils(pre["soils"])
    return c, pre


def _lists(dimx, dimy, frames, nw, nd, seed=SEED):
    from soilmachine_b200 import host
    host.srand(seed)
    return [(host.spawn_list(nw, dimx, dimy), host.spawn_list(nd, dimx, dimy)) for _ in range(frames)]


def _frame(m, xw, xd, hydrology=True):
    out = [m.water_run(xw)]
    if hydrology:
        m.water_flood()
        m.seep()
    out.append(m.wind_run(xd))
    m.frequency_update()
    return [tuple(getattr(s, k) for k in STAT_KEYS) for s in out]


def raster(rng, cells, edges=None, dimy=None):
    """deposits, strips, +-0.0, tiny values and strips deeper than any column; edges: only the columns within 2 of
    these x get non-zero entries (an edit dense on strip edges)"""
    u = rng.random(cells)
    d = np.where(u < 0.4, rng.uniform(0.0, 0.08, cells), -rng.uniform(0.0, 0.15, cells))
    deep = (u >= 0.75) & (u < 0.82)
    d[deep] = -rng.uniform(1.5, 3.0, int(deep.sum()))
    tiny = (u >= 0.82) & (u < 0.85)
    d[tiny] = rng.choice([1e-12, -1e-12, 5e-324, -5e-324], int(tiny.sum()))
    d[(u >= 0.85) & (u < 0.95)] = 0.0
    d[u >= 0.95] = -0.0
    if edges is not None:
        x = np.arange(cells) // dimy
        near = np.zeros(cells, bool)
        for e in edges:
            near |= np.abs(x - e) <= 2
        d[~near] = 0.0
    return d


def _host_expect(cols, delta, typ, nsoils):
    """the host build of sm_layer.cuh on the same columns: (columns, leftovers, stats)"""
    im = Image(cols, seed=5, spare=2 * len(delta) + 16)
    rc, left, _, _, st = im.run(_host_lib(), delta, typ, nsoils)
    assert rc == 0
    return im.columns(_snap_lib()), left, st


def _ref_apply(soil, dim, lists, rasters):
    """the reference driven live through the same frames, then each (delta, type) in turn: (columns after the frames,
    [(columns, leftovers) after each raster])"""
    spec = importlib.util.spec_from_file_location("make_layer_golden", os.path.join(ROOT, "tests", "golden", "make_layer_golden.py"))
    mk = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mk)
    from oracle import refapi
    r = refapi.get().init(soil, seed=SEED, dimx=dim, dimy=dim, poolsize=32 * dim * dim)
    for xw, xd in lists:
        r.water_run(xw)
        r.water_flood()
        r.seep()
        r.wind_run(xd)
        r.frequency_update()
    start = r.columns()
    out = []
    for d, t in rasters:
        before = r.columns()
        off, size = before["offsets"], before["size"]
        left = np.zeros(dim * dim)
        for i in np.nonzero(d)[0]:
            x, y = divmod(int(i), dim)
            if d[i] > 0:
                r.add(x, y, d[i], t)
            else:
                left[i] = mk.ref_strip(r, x, y, -d[i], size[off[i]:off[i + 1]])
        out.append((r.columns(), left))
    return start, out


def _dev(c, a):
    """a copy of a float64 array in device memory (sm_device_alloc / sm_device_upload)"""
    a = np.ascontiguousarray(a, np.float64)
    d = C.c_void_p()
    c._ck(c.lib.sm_device_alloc(c.h, C.c_int64(a.nbytes), C.byref(d)))
    c._ck(c.lib.sm_device_upload(c.h, d, a.ctypes.data_as(C.c_void_p), C.c_int64(a.nbytes)))
    return d


def _d2h(dptr, n):
    for name in ("libcudart.so.12", "/usr/local/cuda/lib64/libcudart.so"):
        try:
            rt = C.CDLL(name)
            break
        except OSError:
            continue
    out = np.empty(n, np.float64)
    rt.cudaMemcpy.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_int]
    assert rt.cudaMemcpy(out.ctypes.data_as(C.c_void_p), dptr, out.nbytes, 2) == 0
    return out


def _same_cols(a, b, what):
    for k in KEYS:
        same(a[k], b[k], "%s: columns.%s" % (what, k))


# ---- against the reference ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", CASES)
@pytest.mark.parametrize("on_device", [False, True], ids=["host", "device"])
def test_fixture_rasters_equal_the_reference(case, on_device):
    """the fixture's rasters one after the other: leftovers, checksum and section count after each, columns at the end"""
    soil = case.split("_")[1]
    cols = _input(case)
    dimy = int(FIX[case + "_dimy"])
    c, pre = _ctx(soil, 16, dimy)
    try:
        c.upload_columns(cols["offsets"], cols["type"], cols["size"], cols["saturation"])
        _same_cols(c.download_columns(), cols, case + " input")
        for k in range(int(FIX[case + "_nrasters"])):
            delta, typ = _raster(case, k)
            if on_device:
                d, dl = _dev(c, delta), _dev(c, np.full(delta.size, 7.0))
                try:
                    st, _ = c.apply_layer(d, typ, leftover=dl)
                    left = _d2h(dl, delta.size)
                finally:
                    c.device_free(d); c.device_free(dl)
            else:
                st, left = c.apply_layer(delta.reshape(16, dimy), typ, leftover=True)
            assert c.checksum() == int(FIX["%s_sum_%d" % (case, k)]), "%s raster %d: checksum" % (case, k)
            assert c.section_count() == int(FIX["%s_nsec_%d" % (case, k)]), "%s raster %d: sections" % (case, k)
            same(left.reshape(-1), FIX["%s_left_%d" % (case, k)], "%s raster %d: leftovers" % (case, k))
            assert st.cells == int((delta != 0).sum()) and st.emptied == int((FIX["%s_left_%d" % (case, k)] > 0).sum())
        _same_cols(c.download_columns(), _output(case), case + " after the last raster")
    finally:
        c.close()


@pytest.mark.parametrize("soil,dim", [("default", 128), ("rocksand", 192), ("bigbutte", 96)])
def test_after_batches_and_hydrology_equals_host_build_and_reference(soil, dim):
    from oracle import refapi
    c, pre = _ctx(soil, dim, dim)
    ns = len(pre["soils"])
    try:
        c.initialize(SEED, pre["layers"])
        lists = _lists(dim, dim, 1, 1500, 300)
        for xw, xd in lists:
            _frame(c, xw, xd)
        cols0 = c.download_columns()
        rng = np.random.default_rng(dim)
        rasters = [(raster(rng, dim * dim), t) for t in [0] + list(range(1, ns)) + [0]]
        got = []
        cols = cols0
        for d, t in rasters:
            st, left = c.apply_layer(d.reshape(dim, dim), t, leftover=True)
            want, wleft, hst = _host_expect(cols, d, t, ns)
            now = c.download_columns()
            _same_cols(now, want, "%s %d type %d vs host build" % (soil, dim, t))
            same(left.reshape(-1), wleft, "leftovers vs host build")
            assert (st.cells, st.pushed, st.emptied) == (hst[0], hst[1], hst[3])
            got.append((now, left.reshape(-1)))
            cols = now
        assert any((l > 0).any() for _, l in got)
        if refapi.available():
            start, ref = _ref_apply(soil, dim, lists, rasters)
            _same_cols(cols0, start, "%s %d: the frame vs the reference" % (soil, dim))
            for (rc, rl), (gc, gl) in zip(ref, got):
                _same_cols(gc, rc, "%s %d vs the reference" % (soil, dim))
                same(gl, rl, "leftovers vs the reference")
    finally:
        c.close()


def test_equals_the_single_cell_calls():
    """a raster and the same edit through sm_cell_add / the strip loop over sm_cell_remove give the same snapshot"""
    a, pre = _ctx("bigbutte", 64, 64)
    b, _ = _ctx("bigbutte", 64, 64)
    try:
        a.initialize(SEED, pre["layers"])
        for xw, xd in _lists(64, 64, 2, 600, 150):
            _frame(a, xw, xd)
        b.restore(a.snapshot())
        rng = np.random.default_rng(3)
        for t in (0, 2, 1):
            d = raster(rng, 64 * 64)
            _, la = a.apply_layer(d.reshape(64, 64), t, leftover=True)
            lb = np.zeros(64 * 64)
            for i in np.nonzero(d)[0]:
                x, y = divmod(int(i), 64)
                if d[i] > 0:
                    b.cell_add(x, y, d[i], t)
                    continue
                col = b.cell_column(x, y)
                left, j = -d[i], col["n"] - 1
                while left > 0 and j >= 0:
                    empty_top = col["size"][j] <= 0
                    rest = b.cell_remove(x, y, left)
                    if not empty_top:
                        left = rest
                    j -= 1
                lb[i] = left
            same(la.reshape(-1), lb, "leftovers, type %d" % t)
            same(a.snapshot(), b.snapshot(), "snapshot after the type-%d raster" % t)
    finally:
        a.close(); b.close()


def test_pool_after_an_apply_serves_the_next_batches():
    """water and wind batches after an apply equal those on a context restored from the post-apply snapshot"""
    a, pre = _ctx("rocksand", 128, 128)
    b, _ = _ctx("rocksand", 128, 128)
    try:
        a.initialize(SEED, pre["layers"])
        lists = _lists(128, 128, 3, 1500, 300)
        _frame(a, *lists[0])
        rng = np.random.default_rng(9)
        for t in (0, 1, 2):
            a.apply_layer(raster(rng, 128 * 128).reshape(128, 128), t)
        b.restore(a.snapshot())
        for xw, xd in lists[1:]:
            sa, sb = _frame(a, xw, xd), _frame(b, xw, xd)
            assert sa == sb
            assert a.checksum() == b.checksum()
            _same_cols(a.download_columns(), b.download_columns(), "after a batch")
            fa, fb = a.frequency(), b.frequency()
            for k in fa:
                same(fa[k], fb[k], k)
            a.apply_layer(raster(rng, 128 * 128).reshape(128, 128), 0)     # Air: the next flood and seep pass
            b.restore(a.snapshot())
    finally:
        a.close(); b.close()


# ---- sharded maps and groups ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind,n", [("virtual", 2), ("virtual", 3), ("virtual", 4), ("group", 2), ("group", 3)])
def test_sharded_equals_one_context(kind, n):
    from soilmachine_b200 import capi, presets, sharded
    dimx, dimy, soil = 192, 96, "bigbutte"
    pre = presets.load(soil)
    ns = len(pre["soils"])
    one, _ = _ctx(soil, dimx, dimy)
    if kind == "virtual":
        m = sharded.VirtualShards(n, dimx, dimy, pre["world"]["scale"], max_particles=4096)
        m.set_soils(pre["soils"])
        snap = m.snapshot
        checksum = lambda: sum(c.checksum() for c in m.ctx) % (1 << 64)     # noqa: E731
    else:
        m, _ = _ctx(soil, dimx, dimy, devices=[0] * n)
        snap, checksum = m.snapshot, m.checksum
    try:
        m.initialize(SEED, pre["layers"])
        one.initialize(SEED, pre["layers"])
        edges = [c.x0 for c in m.ctx[1:]] if kind == "virtual" else _group_edges(dimx, n)
        rng = np.random.default_rng(40 + n)
        for step, (xw, xd) in enumerate(_lists(dimx, dimy, 3, 1200, 250)):
            sm, so = m.water_run(xw), one.water_run(xw)
            assert tuple(getattr(sm, k) for k in STAT_KEYS[:5]) == tuple(getattr(so, k) for k in STAT_KEYS[:5])
            d = raster(rng, dimx * dimy, edges=edges if step == 1 else None, dimy=dimy).reshape(dimx, dimy)
            t = step % ns
            if kind == "group" and step == 2:       # a device raster on rank 0's device, leftovers there too
                dd, dl = _dev(m, d), _dev(m, np.zeros(d.size))
                try:
                    sa, _ = m.apply_layer(dd, t, leftover=dl)
                    la = _d2h(dl, d.size)
                finally:
                    m.device_free(dd); m.device_free(dl)
            else:
                sa, la = m.apply_layer(d, t, leftover=True)
            sb, lb = one.apply_layer(d, t, leftover=True)
            same(np.asarray(la).reshape(-1), lb.reshape(-1), "%s %d step %d: leftovers" % (kind, n, step))
            assert (sa.cells, sa.pushed, sa.emptied) == (sb.cells, sb.pushed, sb.emptied)
            assert checksum() == one.checksum(), "%s %d step %d: checksum" % (kind, n, step)
            same(snap(), one.snapshot(), "%s %d step %d: snapshot" % (kind, n, step))
            m.wind_run(xd)
            one.wind_run(xd)
        assert checksum() == one.checksum()
        same(snap(), one.snapshot(), "%s %d: final snapshot" % (kind, n))
    finally:
        m.close(); one.close()


def _group_edges(dimx, n):
    from soilmachine_b200 import capi
    lib = capi.load()
    cfg = capi.Config(dimx, 8, 80, 0, 0, 0, 0)
    out = []
    for r in range(1, n):
        x0 = C.c_int32()
        assert lib.sm_group_layout(C.byref(cfg), n, r, C.byref(x0), None, None) == 0
        out.append(x0.value)
    return out


# ---- refusals -------------------------------------------------------------------------------------------------------
def test_refusals_leave_the_map_unchanged():
    from soilmachine_b200 import capi, sharded
    dimx = dimy = 128
    # default: one section per column, so the initial terrain uses no pool slot.  The group's pool is half the map's
    # cells, divided by strip: a deposit on 3/4 of rank 1's strip fits the whole pool but not rank 1's share.
    g, pre = _ctx("default", dimx, dimy, devices=[0, 0], pool_capacity=dimx * dimy // 2)
    one, _ = _ctx("default", dimx, dimy, pool_capacity=dimx * dimy // 2)
    try:
        for m in (g, one):
            m.initialize(SEED, pre["layers"])
        x1 = _group_edges(dimx, 2)[0]
        d = np.zeros((dimx, dimy))
        d[x1:x1 + 3 * (dimx - x1) // 4] = 0.01           # Air on non-Air tops: one push per cell
        before = g.checksum()
        with pytest.raises(capi.SoilMachineError) as e:
            g.apply_layer(d, 0)
        assert e.value.code == capi.SM_ERR_POOL and "rank 1" in str(e.value)
        assert g.checksum() == before
        with pytest.raises(capi.SoilMachineError) as e:
            g.apply_layer(d, 0, check=True)
        assert e.value.code == capi.SM_ERR_POOL and g.checksum() == before
        st, _ = one.apply_layer(d, 0)                    # one context with the whole pool accepts it
        assert st.pushed == int((d > 0).sum()) and st.free_slots >= st.pushed
        for bad in (np.nan, np.inf, -np.inf):
            e2 = d.copy()
            e2[5, 7] = bad
            with pytest.raises(capi.SoilMachineError) as e:
                one.apply_layer(e2, 1)
            assert e.value.code == capi.SM_ERR_INVALID
        after = one.checksum()
        for t in (-1, len(pre["soils"]), 64):
            with pytest.raises(capi.SoilMachineError) as e:
                one.apply_layer(d, t)
            assert e.value.code == capi.SM_ERR_INVALID
        with pytest.raises(capi.SoilMachineError):
            one.apply_layer(np.zeros((dimx, dimy - 1)), 1)
        assert one.checksum() == after
    finally:
        g.close(); one.close()
    # a rank of a sharded map applies its own strip, and still refuses the single-cell mutators
    v = sharded.VirtualShards(2, 64, 64, pre["world"]["scale"])
    try:
        v.set_soils(pre["soils"])
        v.initialize(SEED, pre["layers"])
        with pytest.raises(capi.SoilMachineError):
            v.ctx[0].cell_add(3, 3, 0.1, 1)
        st, _ = v.ctx[1].apply_layer(np.full((v.ctx[1].x1 - v.ctx[1].x0, 64), 0.02), 1)
        assert st.cells == (v.ctx[1].x1 - v.ctx[1].x0) * 64
    finally:
        v.close()


# ---- budget flags ---------------------------------------------------------------------------------------------------
def test_budget_flags_change_nothing():
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
        rng = np.random.default_rng(11)
        for t in (0, 1, 2):
            d = raster(rng, dim * dim).reshape(dim, dim)
            outs = [m.apply_layer(d, t, leftover=True) for m in (plain, cb, hb)]
            for s, l in outs[1:]:
                same(l, outs[0][1], "leftovers")
                assert s.pushed == outs[0][0].pushed
        for m in (cb, hb):
            assert m.checksum() == plain.checksum()
            same(m.snapshot(), plain.snapshot(), "snapshot with budget flags")
        after = cb.last_cell_budget(), cb.last_budget().asdict(), hb.last_hydro_cell_budget(), hb.last_hydro_budget()
        for k in maps[0]:
            same(after[0][k], maps[0][k], "cell budget " + k)
        assert after[1] == maps[1] and after[3] == maps[3]
        for k in maps[2]:
            same(after[2][k], maps[2][k], "hydro cell budget " + k)
    finally:
        plain.close(); cb.close(); hb.close()


# ---- the C++ facade -------------------------------------------------------------------------------------------------
def test_facade_apply(tmp_path):
    """tests/facade_apply.cpp applies a raster through Layermap::apply, plain and on a group of two; capi applies the
    same raster to the facade's map and must reach the same checksum and snapshot"""
    from oracle import refapi
    from soilmachine_b200 import capi
    libdir = os.path.join(ROOT, "soilmachine_b200", "lib")
    exe = str(tmp_path / "facade_apply")
    subprocess.check_call(["g++", "-std=c++17", "-O1", os.path.join(ROOT, "tests", "facade_apply.cpp"), "-o", exe,
                           "-L" + libdir, "-lsoilmachine_b200", "-Wl,-rpath," + libdir])
    soil = refapi.soil_path("bigbutte")
    d = raster(np.random.default_rng(2), 96 * 72)
    d.tofile(str(tmp_path / "r.bin"))
    lines = []
    for group in (False, True):
        env = {k: v for k, v in os.environ.items() if k not in ("SM_GPUS", "SM_GPU_DEVICES")}
        if group:
            env.update(SM_GPUS="2", SM_GPU_DEVICES="0,0")
        b, a = str(tmp_path / ("b%d.snap" % group)), str(tmp_path / ("a%d.snap" % group))
        out = subprocess.run([exe, soil, str(tmp_path / "r.bin"), "2", b, a], capture_output=True, text=True,
                             timeout=900, env=env)
        assert out.returncode == 0, out.stdout + out.stderr
        lines.append(out.stdout.strip())
        c, pre = _ctx("bigbutte", 96, 72)
        try:
            c.restore(np.fromfile(b, np.uint8))
            st, _ = c.apply_layer(d.reshape(96, 72), 2)
            assert lines[-1] == "checksum %016x emptied %d" % (c.checksum(), st.emptied), lines[-1]
            same(c.snapshot(), np.fromfile(a, np.uint8), "facade vs capi snapshot")
        finally:
            c.close()
    assert lines[0] == lines[1]


# ---- processes ------------------------------------------------------------------------------------------------------
def test_apply_over_cuda_ipc_two_processes_one_gpu():
    """tests/multigpu_apply_check.py with two processes sharing this GPU"""
    env = dict(os.environ, SM_ONE_GPU="1")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2",
           "--master-addr", "127.0.0.1", "--master-port", "29657",
           os.path.join(ROOT, "tests", "multigpu_apply_check.py"), "96", "700"]
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=900, cwd=ROOT, env=env)
    line = [l for l in out.stdout.splitlines() if l.startswith("multigpu_apply_check")]
    assert out.returncode == 0 and line and "DIFFER" not in line[0], (out.stdout[-2000:], out.stderr[-2000:])
