"""Strata views on the device (sm_composition, sm_voxelize) against the statement of the header (tests/_strata.py):
every golden state restored from a snapshot (floors kept verbatim), a real frame with batches, floods, the seep pass
and a layer raster (and, where oracle/_ref is built, the reference driven through the same frame), the crafted
overlapping-floor columns, host and device output; the calls change nothing; groups and VirtualShards equal one
context, with voxel windows across strip edges and ragged strips; host output larger than the staging buffer;
refusals leave out untouched; the C++ facade."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import _golden
import _strata
from _group import same
from test_apply_layer import SEED as REF_SEED, _ctx, _frame, _group_edges, _lists, _ref_apply, raster
from test_strata_host import CRAFTED_POR, STATES, crafted, crafted_expect, state, type_sets, windows

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SEED = 37


def _rt():
    for name in ("libcudart.so.12", "/usr/local/cuda/lib64/libcudart.so"):
        try:
            rt = C.CDLL(name)
            rt.cudaMemcpy.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_int]
            return rt
        except OSError:
            continue
    raise RuntimeError("no CUDA runtime")


def _alloc(c, nbytes, fill=None):
    """device memory from sm_device_alloc (on rank 0 for a group), optionally filled with the bytes of `fill`"""
    d = C.c_void_p()
    c._ck(c.lib.sm_device_alloc(c.h, C.c_int64(max(nbytes, 1)), C.byref(d)))
    if fill is not None:
        a = np.ascontiguousarray(fill)
        c._ck(c.lib.sm_device_upload(c.h, d, a.ctypes.data_as(C.c_void_p), C.c_int64(a.nbytes)))
    return d


def _d2h(d, shape, dtype):
    out = np.empty(shape, dtype)
    assert _rt().cudaMemcpy(out.ctypes.data_as(C.c_void_p), d, out.nbytes, 2) == 0
    return out


def comp_both(c, types, lo, hi, flags):
    """composition with host and with device output; both must agree byte for byte"""
    below, pore = bool(flags & _strata.BELOW_SURFACE), bool(flags & _strata.PORE_WATER)
    h = c.composition(types, lo, hi, below, pore)
    d = _alloc(c, h.nbytes, np.full(h.shape, np.nan))
    try:
        assert c.composition(types, lo, hi, below, pore, out=d) is None
        same(_d2h(d, h.shape, np.float64), h, "composition: device vs host output")
    finally:
        c.device_free(d)
    return h


def vox_both(c, x0, x1, y0, y1, z0, dz, nz):
    h = c.voxelize(x0, x1, y0, y1, z0, dz, nz)
    d = _alloc(c, h.nbytes, np.full(h.shape, 7, np.uint8))
    try:
        c.voxelize(x0, x1, y0, y1, z0, dz, nz, out=d)
        same(_d2h(d, h.shape, np.uint8), h, "voxels: device vs host output")
    finally:
        c.device_free(d)
    return h


def _restored(cols, g_soils, dimx, dimy):
    """a context holding exactly these columns, floors verbatim (snapshot.build + sm_snapshot_restore)"""
    from soilmachine_b200 import capi, snapshot
    c = capi.Context(dimx, dimy, 80, max_particles=1024)
    c.set_soils(g_soils)
    freq = {k: np.zeros(dimx * dimy, np.float32) for k in snapshot.FREQ_KEYS}
    c.restore(np.frombuffer(snapshot.build(cols, freq, dimx, dimy, 0, dimx, len(g_soils)), np.uint8))
    return c


def check_views(c, cols, por, ns, dimy, what, cx0=0):
    """every window, flag and type set of the host tests, and a few voxel ladders, against the statement"""
    for lo, hi, f in windows(cols):
        for pore in (0, _strata.PORE_WATER):
            for types in type_sets(ns):
                got = comp_both(c, types, lo, hi, f | pore)
                want = _strata.composition(cols, por, types, lo, hi, f | pore)
                same(got.reshape(len(types), -1), want, "%s: composition %r" % (what, (lo, hi, f | pore, types)))
    assert c.view_stats.sections == int(cols["offsets"][-1])
    H = _strata.heights(cols)
    w = c.x1 - c.x0
    e, r = (1 if w > 2 else 0), min(3, dimy - 1)        # a window off the map's edges where the map has room
    for (x0, x1, y0, y1), (z0, dz, nz) in [((c.x0, c.x1, 0, dimy), (-0.5, 0.1, 64)),
                                           ((c.x0, c.x1, 0, dimy), (float(H.min()) - 0.01, 1.0 / 3, 48)),
                                           ((c.x0 + w // 2, c.x0 + w // 2 + 1, 0, dimy), (-1.0, 2.0 ** -8, 4096)),
                                           ((c.x0 + e, c.x1 - e, r, r + 1), (0.0, 1.0 / 64, 1024))]:
        got = vox_both(c, x0, x1, y0, y1, z0, dz, nz)
        same(got, _strata.voxelize(cols, dimy, x0, x1, y0, y1, z0, dz, nz, cx0), "%s: voxels %r" % (what, (x0, y0, z0, dz)))


# ---- against the statement ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case,prefix", STATES)
def test_golden_states_equal_the_statement(case, prefix):
    cols, por, ns, dimx, dimy = state(case, prefix)
    c = _restored(cols, _golden.load(case)["soils"], dimx, dimy)
    try:
        _golden.same_cols(c.download_columns(), cols, "restored columns")
        check_views(c, cols, por, ns, dimy, "%s %s" % (case, prefix))
    finally:
        c.close()


def test_crafted_overlapping_floors_on_the_device():
    from soilmachine_b200 import capi
    cols = crafted()
    soils = np.zeros(4, capi.SOIL_DTYPE)
    soils["porosity"] = CRAFTED_POR[:4]
    c = _restored(cols, soils, 2, 3)
    try:
        comp, vox = crafted_expect()
        same(comp_both(c, [0, 1, 2, 3], 2.5, 4.5, 0).reshape(4, -1), comp, "crafted composition")
        same(vox_both(c, 0, 2, 0, 3, 0.0, 0.25, 28), vox, "crafted voxels")
        check_views(c, cols, CRAFTED_POR, 4, 3, "crafted")
    finally:
        c.close()


def test_after_a_frame_and_a_layer_raster_equals_the_statement_and_the_reference():
    from oracle import refapi
    soil, dim = "rocksand", 192
    c, pre = _ctx(soil, dim, dim)
    ns = len(pre["soils"])
    por = np.zeros(64, np.float32)
    por[:ns] = pre["soils"]["porosity"]
    try:
        c.initialize(REF_SEED, pre["layers"])         # the seed _ref_apply gives the reference
        lists = _lists(dim, dim, 1, 1500, 300)
        for xw, xd in lists:
            _frame(c, xw, xd)
        d = raster(np.random.default_rng(5), dim * dim)
        c.apply_layer(d.reshape(dim, dim), 2)
        cols = c.download_columns()
        assert (cols["saturation"] > 0).any() and (cols["type"] == 0).any()
        check_views(c, cols, por, ns, dim, "rocksand frame")
        if not refapi.available():
            pytest.skip("oracle/_ref is not built: the reference part of this test did not run")
        _, ref = _ref_apply(soil, dim, lists, [(d, 2)])
        rcols = ref[-1][0]
        for types, lo, hi, f in [(list(range(ns)), -np.inf, np.inf, 0), ([2, 0], 0.0, 1.0, 1), ([0, 1, 2], -np.inf, np.inf, 2)]:
            same(c.composition(types, lo, hi, bool(f & 1), bool(f & 2)).reshape(len(types), -1),
                 _strata.composition(rcols, por, types, lo, hi, f), "vs the reference %r" % ((types, lo, hi, f),))
        same(c.voxelize(0, dim, 0, dim, -0.5, 0.1, 64), _strata.voxelize(rcols, dim, 0, dim, 0, dim, -0.5, 0.1, 64),
             "voxels vs the reference")
    finally:
        c.close()


# ---- read-only ------------------------------------------------------------------------------------------------------
def _fingerprint(c):
    return (c.checksum(), c.section_count(), {k: v.tobytes() for k, v in c.frequency().items()},
            c.last_budget().asdict(), c.last_hydro_budget(), c.snapshot().tobytes())


def test_views_change_nothing():
    dim = 96
    c, pre = _ctx("bigbutte", dim, dim, budget=True)
    b, _ = _ctx("bigbutte", dim, dim, budget=True)
    try:
        for m in (c, b):
            m.initialize(SEED, pre["layers"])
        lists = _lists(dim, dim, 3, 900, 200)
        _frame(c, *lists[0]); _frame(b, *lists[0])
        before = _fingerprint(c)
        ns = len(pre["soils"])
        for f in range(4):
            comp_both(c, list(range(ns)), 0.0, 2.0, f)
        vox_both(c, 0, dim, 0, dim, -1.0, 0.05, 100)
        assert _fingerprint(c) == before
        # a batch opened, views between its sweeps, then finished: the same bits as without the views
        xw = lists[1][0]
        c.water_begin(xw); b.water_begin(xw)
        c.water_sweeps(3); b.water_sweeps(3)
        comp_both(c, [0], -np.inf, np.inf, 2)
        vox_both(c, 5, 40, 7, 9, 0.0, 0.5, 30)
        sa, sb = c.water_sweeps(100000), b.water_sweeps(100000)
        assert sa.asdict()["steps"] == sb.asdict()["steps"]
        _frame(c, *lists[2]); _frame(b, *lists[2])
        same(c.snapshot(), b.snapshot(), "after a batch with views in between")
        assert c.last_budget().asdict() == b.last_budget().asdict()
    finally:
        c.close(); b.close()


def test_golden_frame_with_views_interleaved_matches():
    import soilmachine_b200 as smb
    g = _golden.load("frame_rocksand_56")
    ctx = smb.Context(int(g["dimx"]), int(g["dimy"]), int(g["scale"]), device=0, max_particles=4096)
    try:
        ctx.set_soils(g["soils"])
        ctx.initialize(int(g["seed"]), g["layers"])
        ns = len(g["soils"])

        class Viewing:
            """the context, with every view called before each step of the replay"""
            def __getattr__(self, k):
                f = getattr(ctx, k)

                def call(*a, **kw):
                    ctx.composition(list(range(ns)), -np.inf, np.inf, pore_water=True)
                    ctx.voxelize(0, ctx.dimx, 0, ctx.dimy, -0.3, 0.2, 40)
                    return f(*a, **kw)
                return call
        _golden.replay_frame(g, Viewing(), lambda st: (st.steps, st.sweeps, st.exit_oob, st.exit_evap, st.exit_stall))
    finally:
        ctx.close()


# ---- sharded maps and groups ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind,n", [("virtual", 2), ("virtual", 3), ("group", 2), ("group", 3)])
def test_sharded_equals_one_context(kind, n):
    from soilmachine_b200 import presets, sharded
    dimx, dimy, soil = 200, 72, "rocksand"      # ragged: the last strip is narrower
    pre = presets.load(soil)
    ns = len(pre["soils"])
    one, _ = _ctx(soil, dimx, dimy)
    if kind == "virtual":
        m = sharded.VirtualShards(n, dimx, dimy, pre["world"]["scale"], max_particles=4096)
        m.set_soils(pre["soils"])
        edges = [c.x0 for c in m.ctx[1:]]
    else:
        m, _ = _ctx(soil, dimx, dimy, devices=[0] * n)
        edges = _group_edges(dimx, n)
    try:
        m.initialize(SEED, pre["layers"]); one.initialize(SEED, pre["layers"])
        for xw, xd in _lists(dimx, dimy, 1, 1500, 300):
            m.water_run(xw); one.water_run(xw)
            m.water_flood(); one.water_flood()
            m.seep(); one.seep()
            m.wind_run(xd); one.wind_run(xd)
        for types, lo, hi, f in [(list(range(ns)), -np.inf, np.inf, 0), ([2, 0], 0.0, 1.0, 1), ([1], -np.inf, np.inf, 2),
                                 (list(range(ns))[::-1], 0.5, 3.0, 3)]:
            want = comp_both(one, types, lo, hi, f)
            got = m.composition(types, lo, hi, bool(f & 1), bool(f & 2))
            same(got, want, "%s %d: composition %r" % (kind, n, (types, lo, hi, f)))
            if kind == "group":
                same(comp_both(m, types, lo, hi, f), want, "group composition, host and device output")
            assert m.view_stats.sections == one.view_stats.sections
        for e in edges:
            for x0, x1, y0, y1 in [(e - 3, e + 5, 0, dimy), (e - 1, e + 1, 10, 11), (0, dimx, 20, 40)]:
                want = vox_both(one, x0, x1, y0, y1, -0.2, 0.05, 96)
                same(m.voxelize(x0, x1, y0, y1, -0.2, 0.05, 96), want, "%s %d: voxels at edge %d" % (kind, n, e))
                if kind == "group":
                    same(vox_both(m, x0, x1, y0, y1, -0.2, 0.05, 96), want, "group voxels, host and device output")
        if kind == "virtual":         # a rank's own strip, and the refusal of a window that leaves it
            from soilmachine_b200 import capi
            r = m.ctx[1]
            same(r.composition([0, 1], -np.inf, np.inf), one.composition([0, 1], -np.inf, np.inf)[:, r.x0:r.x1], "rank strip")
            with pytest.raises(capi.SoilMachineError) as e:
                r.voxelize(r.x0 - 1, r.x0 + 2, 0, 4, 0.0, 1.0, 4)
            assert e.value.code == capi.SM_ERR_INVALID
    finally:
        m.close(); one.close()


# ---- staging ----------------------------------------------------------------------------------------------------------
def test_host_output_larger_than_the_staging_buffer():
    """1024 x 1536 rocksand, all three soils in f64 (37.7 MB), and voxels of 1024 x 1024 x 48 (50 MB): host output,
    staged in ranges, equals device output"""
    c, pre = _ctx("rocksand", 1024, 1536)
    try:
        c.initialize(SEED, pre["layers"])
        ns = len(pre["soils"])
        h = comp_both(c, list(range(ns)), -np.inf, np.inf, 0)
        assert h.nbytes > (32 << 20) and c.view_stats.bytes_out == h.nbytes
        v = vox_both(c, 0, 1024, 0, 1024, -0.5, 0.25, 48)
        assert v.nbytes > (32 << 20) and c.view_stats.cells == 1024 * 1024
    finally:
        c.close()


# ---- refusals -------------------------------------------------------------------------------------------------------
def test_refusals_leave_out_untouched():
    from soilmachine_b200 import capi
    c, pre = _ctx("rocksand", 64, 48)
    bare = capi.Context(64, 48, 80)
    try:
        c.initialize(SEED, pre["layers"])
        lib, h = c.lib, c.h
        ns = len(pre["soils"])
        poison = np.full((ns, 64 * 48), -7.5)
        dpo = _alloc(c, poison.nbytes, poison)

        def comp(types, lo, hi, flags=0, ctx=c, dev=False):
            t = np.ascontiguousarray(types, np.int32)
            out = dpo if dev else poison.ctypes.data_as(C.c_void_p)
            return lib.sm_composition(ctx.h, t.ctypes.data_as(C.c_void_p), len(t), C.c_double(lo), C.c_double(hi),
                                      flags, out, int(dev), None)
        try:
            cases = [([0], np.nan, 1.0), ([0], 0.0, np.nan), ([0], 2.0, 1.0), ([ns], 0.0, 1.0), ([-1], 0.0, 1.0),
                     ([1, 1], 0.0, 1.0), (list(range(ns)) + [0], 0.0, 1.0), ([], 0.0, 1.0), ([64], 0.0, 1.0)]
            for dev in (False, True):
                for types, lo, hi in cases:
                    assert comp(types, lo, hi, dev=dev) == capi.SM_ERR_INVALID, (types, lo, hi)
                assert comp([0], 0.0, 1.0, flags=4, dev=dev) == capi.SM_ERR_INVALID
            assert comp([0], 0.0, 1.0, ctx=bare) == capi.SM_ERR_INVALID          # no soil table
            assert lib.sm_composition(h, None, 1, C.c_double(0), C.c_double(1), 0, poison.ctypes.data_as(C.c_void_p), 0,
                                      None) == capi.SM_ERR_INVALID
            assert (poison == -7.5).all()
            same(_d2h(dpo, poison.shape, np.float64), poison, "device out after refusals")
            vp = np.full(4096, 9, np.uint8)
            dvp = _alloc(c, vp.nbytes, vp)
            try:
                bad = [(0, 0, 0, 4, 0.0, 1.0, 4), (5, 3, 0, 4, 0.0, 1.0, 4), (0, 65, 0, 4, 0.0, 1.0, 4),
                       (-1, 2, 0, 4, 0.0, 1.0, 4), (0, 2, 0, 49, 0.0, 1.0, 4), (0, 2, 3, 3, 0.0, 1.0, 4),
                       (0, 2, 0, 4, np.nan, 1.0, 4), (0, 2, 0, 4, np.inf, 1.0, 4), (0, 2, 0, 4, 0.0, 0.0, 4),
                       (0, 2, 0, 4, 0.0, -1.0, 4), (0, 2, 0, 4, 0.0, np.inf, 4), (0, 2, 0, 4, 0.0, np.nan, 4),
                       (0, 2, 0, 4, 0.0, 1.0, 0), (0, 2, 0, 4, 0.0, 1.0, 65537)]
                for dev in (False, True):
                    for x0, x1, y0, y1, z0, dz, nz in bad:
                        out = dvp if dev else vp.ctypes.data_as(C.c_void_p)
                        rc = lib.sm_voxelize(h, x0, x1, y0, y1, C.c_double(z0), C.c_double(dz), nz, out, int(dev), None)
                        assert rc == capi.SM_ERR_INVALID, (x0, x1, y0, y1, z0, dz, nz)
                assert (vp == 9).all()
                same(_d2h(dvp, vp.shape, np.uint8), vp, "device voxels after refusals")
            finally:
                c.device_free(dvp)
            # the upper limits are accepted
            assert c.voxelize(0, 1, 0, 1, 0.0, 1.0, 65536).shape == (65536, 1, 1)
            assert c.composition(list(range(ns)), -np.inf, np.inf).shape == (ns, 64, 48)
        finally:
            c.device_free(dpo)
    finally:
        c.close(); bare.close()


# ---- the C++ facade -------------------------------------------------------------------------------------------------
def test_facade_strata(tmp_path):
    """tests/facade_strata.cpp, plain and on a group of two: its views equal capi's on the facade's own map"""
    from oracle import refapi
    libdir = os.path.join(ROOT, "soilmachine_b200", "lib")
    exe = str(tmp_path / "facade_strata")
    subprocess.check_call(["g++", "-std=c++17", "-O1", os.path.join(ROOT, "tests", "facade_strata.cpp"), "-o", exe,
                           "-L" + libdir, "-lsoilmachine_b200", "-Wl,-rpath," + libdir])
    soil = refapi.soil_path("bigbutte")
    blobs = []
    for group in (False, True):
        env = {k: v for k, v in os.environ.items() if k not in ("SM_GPUS", "SM_GPU_DEVICES")}
        if group:
            env.update(SM_GPUS="2", SM_GPU_DEVICES="0,0")
        snap, out = str(tmp_path / ("s%d.snap" % group)), str(tmp_path / ("v%d.bin" % group))
        r = subprocess.run([exe, soil, snap, out], capture_output=True, text=True, timeout=900, env=env)
        assert r.returncode == 0, r.stdout + r.stderr
        c, pre = _ctx("bigbutte", 96, 72)
        try:
            c.restore(np.fromfile(snap, np.uint8))
            ns = len(pre["soils"])
            want = b"".join([c.composition(list(range(ns)), -np.inf, np.inf).tobytes(),
                             c.composition(list(range(ns)), 0.0, 1.0, True, True).tobytes(),
                             c.voxelize(0, 96, 0, 72, -0.25, 0.125, 48).tobytes(),
                             c.voxelize(0, 96, 17, 18, 0.0, 1.0 / 64, 256).tobytes()])
        finally:
            c.close()
        got = open(out, "rb").read()
        assert got == want, "facade (group=%s) vs capi" % group
        blobs.append(got)
    assert blobs[0] == blobs[1]
