"""A context group (sm_create_group): the map cut into strips over several ranks of this process behind ONE context,
through capi.Context(devices=...), host.Simulation(devices=...) and the C++ facade.  Virtual ranks on the one device
(devices = [0] * n); every check compares the group with one unsharded context fed the same inputs, byte for byte.
tests/multigpu_group_check.py runs the frame and single-cell checks with one rank per GPU."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import _group
from _group import same

pytestmark = pytest.mark.gpu

# the shapes of tests/test_sharded_views.py, plus one whose soil ponds
SHAPES = [(2, "rocksand", 128, 96, 900, 500),
          (3, "rockgravelpebblessand", 144, 80, 900, 700),
          (2, "bigbutte", 96, 72, 700, 300)]
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("nranks,soil,dimx,dimy,nw,nd", SHAPES)
def test_group_frames_match_one_context_after_every_phase(nranks, soil, dimx, dimy, nw, nd):
    nflood = _group.check_frames(soil, dimx, dimy, nw, nd, [0] * nranks)
    if soil == "bigbutte":
        assert nflood > 0, "the ponding shape did not flood"


def _pair(nranks, soil, dimx, dimy):
    sg, so = _group.simulations(soil, dimx, dimy, [0] * nranks)
    return sg, so, sg.ctx, so.ctx


@pytest.mark.parametrize("nranks,soil,dimx,dimy,nw,nd", SHAPES[:2])
def test_group_stepping_returns_every_particle_from_its_holder(nranks, soil, dimx, dimy, nw, nd):
    from soilmachine_b200 import host
    sg, so, g, o = _pair(nranks, soil, dimx, dimy)
    try:
        host.srand(_group.SEED)
        for kind, n in (("water", nw), ("wind", nd)):
            xy = host.spawn_list(n, dimx, dimy)
            getattr(g, kind + "_begin")(xy); getattr(o, kind + "_begin")(xy)
            done = 0
            for k in (None, 1, 7, 50, 4000):             # the last one runs the batch out: every final state
                if k:
                    _group.same_stats(getattr(g, kind + "_sweeps")(k), getattr(o, kind + "_sweeps")(k), "%s +%d sweeps" % (kind, k))
                    done += k
                a, b = getattr(g, kind + "_state")(), getattr(o, kind + "_state")()
                for key in b:
                    same(a[key], b[key], "%s state %s after %d sweeps" % (kind, key, done))
            assert b["alive"].sum() == 0, "the batch should have run out"
            _group.same_map(g, o, kind + " batch stepped")
    finally:
        sg.close(); so.close()


@pytest.mark.parametrize("nranks", [2, 3])
def test_group_single_cell_mutators_match_one_context(nranks):
    _group.check_cell_ops([0] * nranks)


@pytest.mark.parametrize("nranks,soil,dimx,dimy,nw,nd", SHAPES[:2])
def test_group_views_match_one_context(nranks, soil, dimx, dimy, nw, nd):
    from soilmachine_b200 import host
    sg, so, g, o = _pair(nranks, soil, dimx, dimy)
    try:
        host.srand(_group.SEED)
        xw, xd = host.spawn_list(nw, dimx, dimy), host.spawn_list(nd, dimx, dimy)
        sg.frame(nw, nd, xw, xd); so.frame(nw, nd, xw, xd)
        for slice_ in (160, 45, 10):
            same(g.mesh_update(slice_), o.mesh_update(slice_), "mesh vertices, slice %d" % slice_)
            same(g.export_height(), o.export_height(), "exportheight, slice %d" % slice_)
            same(g.export_color(), o.export_color(), "exportcolor, slice %d" % slice_)
        for x in _group.edge_columns(dimx, nranks):
            for y in range(0, dimy, 5):
                a, b = g.cell_query(x, y), o.cell_query(x, y)
                same(np.float64(a[0]), np.float64(b[0]), "height (%d, %d)" % (x, y))
                assert a[1] == b[1]
                same(a[2], b[2], "normal (%d, %d)" % (x, y))
                ca, cb = g.cell_column(x, y), o.cell_column(x, y)
                assert ca["n"] == cb["n"]
                for k in ("type", "size", "floor", "saturation"):
                    same(ca[k], cb[k], "column %s (%d, %d)" % (k, x, y))
                if x < dimx - 1 and y < dimy - 1:
                    fx, fy = np.float32(x + 0.625), np.float32(y + 0.375)
                    same(np.float64(g.height_bilinear(fx, fy)), np.float64(o.height_bilinear(fx, fy)), "bilinear")
        for c in (g, o):
            c.lbm_create(32, 20, 32)
            c.lbm_set_boundary(None)
            c.lbm_step(20)
        a, b = g.lbm_get(), o.lbm_get()
        for k in b:
            same(a[k], b[k], "lattice " + k)
        g.wind_use_lbm(True); o.wind_use_lbm(True)
        xy = host.spawn_list(400, dimx, dimy)
        _group.same_stats(g.wind_run(xy, max_sweeps=2000), o.wind_run(xy, max_sweeps=2000), "coupled wind batch")
        a, b = g.wind_state(), o.wind_state()
        for k in b:
            same(a[k], b[k], "coupled wind state " + k)
        _group.same_map(g, o, "after the coupled wind batch")
    finally:
        g.wind_use_lbm(False); o.wind_use_lbm(False)
        sg.close(); so.close()


# ---- the C++ facade ------------------------------------------------------------------------------------------------
def _exe(name, tmp_path):
    libdir = os.path.join(ROOT, "soilmachine_b200", "lib")
    exe = str(tmp_path / name)
    subprocess.check_call(["g++", "-std=c++17", "-O1", os.path.join(ROOT, "tests", name + ".cpp"), "-o", exe,
                           "-L" + libdir, "-lsoilmachine_b200", "-Wl,-rpath," + libdir])
    return exe


def _run(cmd, group):
    env = {k: v for k, v in os.environ.items() if k not in ("SM_GPUS", "SM_GPU_DEVICES")}
    if group:
        env.update(SM_GPUS="2", SM_GPU_DEVICES="0,0")
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=900, env=env)
    assert out.returncode == 0, out.stdout + out.stderr
    return out.stdout


def test_facade_programs_run_unchanged_on_a_group(tmp_path):
    """tests/facade_demo.cpp and tests/facade_loop.cpp, as they are, with SM_GPUS=2 SM_GPU_DEVICES=0,0 in the
    environment: the same output and the same map file as without"""
    from oracle import refapi
    soil = refapi.soil_path("rocksand")
    demo = _exe("facade_demo", tmp_path)
    one, grp = _run([demo, soil], False), _run([demo, soil], True)
    assert "frame 1:" in one and "legacy ops ok" in one
    assert grp == one, "facade_demo prints differ:\n%s\n---\n%s" % (one, grp)
    loop = _exe("facade_loop", tmp_path)
    files = []
    for group in (False, True):
        f = str(tmp_path / ("loop_%d.bin" % group))
        out = _run([loop, soil, "64", "24", "16", "1", f], group)
        assert "facade loop ok" in out
        files.append(open(f, "rb").read())
    assert len(files[0]) > 64 * 64 * 12 and files[0] == files[1], "facade_loop map files differ"


def test_facade_legacy_cell_calls_across_a_strip_edge(tmp_path):
    """tests/facade_group.cpp: a Layermap over two ranks by constructor argument; map.add / remove, Particle::cascade
    and the single-cell water calls next to the edge leave the columns one context leaves"""
    from oracle import refapi
    exe = _exe("facade_group", tmp_path)
    files = []
    for ngpus in (1, 2):
        f = str(tmp_path / ("cells_%d.bin" % ngpus))
        out = _run([exe, refapi.soil_path("bigbutte"), str(ngpus), f], False)
        assert "facade group ok: %d ranks" % ngpus in out
        files.append(open(f, "rb").read())
    assert len(files[0]) > 96 * 64 * 12 and files[0] == files[1], "facade_group map files differ"


# ---- a group of one, and the error paths ------------------------------------------------------------------------
def _mesh_ptr(ctx):
    p = C.c_void_p()
    return ctx.lib.sm_mesh_device_ptr(ctx.h, C.byref(p)), p.value


def test_group_of_one_is_a_plain_context():
    from soilmachine_b200 import capi, host, presets
    pre = presets.load("rocksand")
    g = capi.Context(96, 64, pre["world"]["scale"], max_particles=4096, devices=[0])
    o = capi.Context(96, 64, pre["world"]["scale"], max_particles=4096)
    try:
        assert g.group_size() == 1 and g.group_rank(0).value == g.h.value
        for c in (g, o):
            c.set_soils(pre["soils"]); c.set_soil_colors(pre["colors"]); c.initialize(_group.SEED, pre["layers"])
        host.srand(_group.SEED)
        xy = host.spawn_list(500, 96, 64)
        _group.same_stats(g.water_run(xy), o.water_run(xy), "water batch")
        _group.same_map(g, o, "group of one")
        same(g.mesh_update(160), o.mesh_update(160), "mesh")
        rc, p = _mesh_ptr(g)
        assert rc == capi.SM_OK and p
    finally:
        g.close(); o.close()


def test_group_error_paths():
    from soilmachine_b200 import capi, host, presets
    pre = presets.load("rocksand")
    g = capi.Context(128, 64, pre["world"]["scale"], max_particles=4096, devices=[0, 0])
    g.set_soils(pre["soils"])
    g.initialize(_group.SEED, pre["layers"])
    # a failing rank call: the group's message names the rank
    with pytest.raises(capi.SoilMachineError) as e:
        g.mesh_update(160)                               # no soil colours yet
    assert e.value.code == capi.SM_ERR_INVALID and "rank 0: sm_mesh_update: soil colours not set" in str(e.value)
    g.set_soil_colors(pre["colors"])
    assert g.mesh_update(160).shape == (128 * 64, 11)
    rc, _ = _mesh_ptr(g)
    assert rc == capi.SM_ERR_INVALID and b"no single device array" in g.lib.sm_last_error(g.h)
    # each rank still has its strip's pointer, and still refuses what a rank refuses
    rank1 = C.c_void_p()
    assert g.lib.sm_group_rank(g.h, 1, C.byref(rank1)) == capi.SM_OK
    p = C.c_void_p()
    assert g.lib.sm_mesh_device_ptr(rank1, C.byref(p)) == capi.SM_OK and p.value
    assert g.lib.sm_cell_add(rank1, 3, 3, C.c_double(0.5), 1) == capi.SM_ERR_INVALID
    assert b"single-cell operations are not available on a sharded context" in g.lib.sm_last_error(rank1)
    assert g.lib.sm_group_rank(g.h, 2, C.byref(rank1)) == capi.SM_ERR_INVALID
    with pytest.raises(capi.SoilMachineError):
        g.peer_export()
    # destroying a group whose batch is still in flight returns cleanly, and another group can be made afterwards
    host.srand(_group.SEED)
    xy = host.spawn_list(3000, 128, 64)
    d = g.device_spawn(xy)
    g.water_run_device(d, len(xy))
    g.close()
    g2 = capi.Context(128, 64, pre["world"]["scale"], max_particles=4096, devices=[0, 0])
    o = capi.Context(128, 64, pre["world"]["scale"], max_particles=4096)
    try:
        for c in (g2, o):
            c.set_soils(pre["soils"]); c.initialize(_group.SEED, pre["layers"])
        d = g2.device_spawn(xy)
        g2.water_run_device(d, len(xy))
        a, b = g2.last_stats(), o.water_run(xy)
        g2.device_free(d)
        _group.same_stats(a, b, "device-list water batch on the second group")
        _group.same_map(g2, o, "second group")
    finally:
        g2.close(); o.close()
