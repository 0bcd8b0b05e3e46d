"""The drainage view on the device (sm_drainage) against the statement of the header (tests/_drainage.py) and the
serial host driver (tests/drainage/host_drain.cpp): crafted rasters loaded one section per cell, the golden states
restored from snapshots with and without the ground rule, a spiral channel at 1024^2; host and device output; the
header's invariants; the call changes nothing, also between the sweeps of an open batch; groups and VirtualShards of
2, 3 and 4 ranks and two processes over CUDA IPC equal one context; refusals leave the outputs untouched; the C++
facade."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

import _drainage
import _golden
from _group import same
from test_apply_layer import _ctx, _frame, _lists
from test_drainage_host import KEYS, _lib, check_invariants, host_drainage, same_drainage
from test_sharded_views import SHAPES
from test_strata import _alloc, _d2h, _fingerprint, _restored
from test_strata_host import STATES

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SEED = 41
DT = {"spill": np.float64, "dir": np.int8, "area": np.int64, "basin": np.int64}


def both(c, ground=False):
    """drainage with host and with device output; both must agree byte for byte"""
    h = c.drainage(ground)
    st = c.drain_stats.asdict()
    d = {k: _alloc(c, v.nbytes, np.full(v.shape, 7, v.dtype)) for k, v in h.items()}
    try:
        assert c.drainage(ground, out=d) is None
        for k, v in h.items():
            same(_d2h(d[k], v.shape, v.dtype), v, "%s: device vs host output" % k)
    finally:
        for p in d.values():
            c.device_free(p)
    for k in ("flat_cells", "depressed_cells", "outlets"):
        assert c.drain_stats.asdict()[k] == st[k]
    return h


def check(c, ground, what):
    """the device's outputs against the statement and the host driver on the heights the device holds"""
    H = _drainage.heights(c.download_columns(), ground).reshape(c.dimx, c.dimy)
    if not ground:
        same(H, c.heights(), "%s: H" % what)
    got = both(c, ground)
    st = c.drain_stats.asdict()
    got.update({k: st[k] for k in ("flat_cells", "depressed_cells", "outlets")})
    same_drainage(got, _drainage.drainage(H), what)
    same_drainage(got, host_drainage(_lib(), H), what + " (host driver)")
    check_invariants(H, got, what)
    assert st["fill_passes"] >= 1 and st["device_ms"] > 0
    return got


def load_raster(H, water=None):
    """a context holding H one section per cell (type 1; an empty column where H == 0), with `water` of Air on top
    where given"""
    from soilmachine_b200 import capi
    dimx, dimy = H.shape
    c = capi.Context(dimx, dimy, 80, max_particles=1024)
    soils = np.zeros(2, capi.SOIL_DTYPE)
    c.set_soils(soils)
    typ, size, off = [], [], [0]
    for h, w in zip(H.reshape(-1), (np.zeros(H.size) if water is None else water.reshape(-1))):
        if h != 0:
            typ.append(1); size.append(h)
        if w:
            typ.append(0); size.append(w)
        off.append(len(typ))
    c.upload_columns(np.array(off, np.int64), np.array(typ, np.int32), np.array(size), np.zeros(len(typ)))
    return c


@pytest.mark.parametrize("name", [n for n, _ in _drainage.crafted()])
def test_crafted_rasters_equal_the_statement(name):
    H = dict(_drainage.crafted())[name]
    c = load_raster(H)
    try:
        same(c.heights(), H, "uploaded heights")
        got = check(c, False, name)
        if name == "ties":
            assert got["dir"][1, 1] == 0 and got["dir"][4, 4] == 4
        # standing water over part of the map: the ground rule reads under it
        water = np.where((np.arange(H.size) % 3 == 0).reshape(H.shape), 0.25, 0.0)
        w = load_raster(H, water)
        try:
            same(_drainage.heights(w.download_columns(), True).reshape(H.shape), H, "ground under water")
            g = check(w, True, name + " ground")
            for k in KEYS:
                same(g[k], got[k], name + ": ground rule vs the bare raster, " + k)
        finally:
            w.close()
    finally:
        c.close()


@pytest.mark.parametrize("case,prefix", STATES)
def test_golden_states_equal_the_statement(case, prefix):
    g = _golden.load(case)
    cols = _golden.cols(g, prefix)
    c = _restored(cols, g["soils"], int(g["dimx"]), int(g["dimy"]))
    try:
        for ground in (False, True):
            check(c, ground, "%s %s ground=%s" % (case, prefix, ground))
    finally:
        c.close()


def test_spiral_1024_equals_the_host_driver():
    H = _drainage.spiral(1024)
    c = load_raster(H)
    try:
        got = both(c)
        st = c.drain_stats.asdict()
        got.update({k: st[k] for k in ("flat_cells", "depressed_cells", "outlets")})
        same_drainage(got, host_drainage(_lib(), H), "spiral 1024")
        check_invariants(H, got, "spiral 1024")
        assert got["area"].max() > H.size // 2 and st["longest_walk"] > 1024 * 1024 // 4
    finally:
        c.close()


def test_outputs_may_be_null():
    """each output alone equals the same output of a full call"""
    c, pre = _ctx("rocksand", 96, 80)
    try:
        c.initialize(SEED, pre["layers"])
        _frame(c, *_lists(96, 80, 1, 900, 300)[0])
        full = c.drainage()
        for k in KEYS:
            part = c.drainage(outputs=(k,))
            assert list(part) == [k]
            same(part[k], full[k], "%s alone" % k)
    finally:
        c.close()


# ---- read-only ------------------------------------------------------------------------------------------------------
def test_drainage_changes_nothing():
    dim = 96
    c, pre = _ctx("bigbutte", dim, dim, budget=True)
    b, _ = _ctx("bigbutte", dim, dim, budget=True)
    try:
        for m in (c, b):
            m.initialize(SEED, pre["layers"])
        lists = _lists(dim, dim, 3, 900, 200)
        _frame(c, *lists[0]); _frame(b, *lists[0])
        before = _fingerprint(c)
        for ground in (False, True):
            both(c, ground)
        assert _fingerprint(c) == before
        xw = lists[1][0]
        c.water_begin(xw); b.water_begin(xw)
        c.water_sweeps(3); b.water_sweeps(3)
        both(c, True)
        sa, sb = c.water_sweeps(100000), b.water_sweeps(100000)
        assert sa.asdict()["steps"] == sb.asdict()["steps"]
        _frame(c, *lists[2]); _frame(b, *lists[2])
        same(c.snapshot(), b.snapshot(), "after a batch with a drainage call in between")
        assert c.last_budget().asdict() == b.last_budget().asdict()
    finally:
        c.close(); b.close()


# ---- sharded maps and groups ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["virtual", "group"])
@pytest.mark.parametrize("nranks,soil,dimx,dimy,nw,nd", SHAPES + [(3, "rocksand", 200, 72, 1500, 300)])
def test_sharded_equals_one_context(kind, nranks, soil, dimx, dimy, nw, nd):
    from soilmachine_b200 import presets, sharded
    pre = presets.load(soil)
    one, _ = _ctx(soil, dimx, dimy)
    if kind == "virtual":
        m = sharded.VirtualShards(nranks, dimx, dimy, pre["world"]["scale"], max_particles=4096)
        m.set_soils(pre["soils"])
    else:
        m, _ = _ctx(soil, dimx, dimy, devices=[0] * nranks)
    try:
        m.initialize(SEED, pre["layers"]); one.initialize(SEED, pre["layers"])
        for xw, xd in _lists(dimx, dimy, 1, nw, nd):
            m.water_run(xw); one.water_run(xw)
            m.water_flood(); one.water_flood()
            m.seep(); one.seep()
            m.wind_run(xd); one.wind_run(xd)
        for ground in (False, True):
            want = both(one, ground)
            got = both(m, ground) if kind == "group" else m.drainage(ground)
            for k in KEYS:
                same(got[k], want[k], "%s %d ground=%s: %s" % (kind, nranks, ground, k))
            for k in ("flat_cells", "depressed_cells", "outlets"):
                assert m.drain_stats.asdict()[k] == one.drain_stats.asdict()[k]
        if kind == "virtual":        # one rank alone: its strip of the whole-map result
            r = m.ctx[-1]
            part = r.drainage(True)
            for k in KEYS:
                same(part[k], want[k][r.x0:r.x1], "rank strip " + k)
    finally:
        m.close(); one.close()


def test_drainage_over_cuda_ipc_two_processes_one_gpu():
    """tests/multigpu_drainage_check.py with two processes sharing this GPU: the peers' strips are CUDA-IPC mappings"""
    env = dict(os.environ, SM_ONE_GPU="1")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2",
           "--master-addr", "127.0.0.1", "--master-port", "29631",
           os.path.join(ROOT, "tests", "multigpu_drainage_check.py"), "96", "300", "rocksand"]
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=900, cwd=ROOT, env=env)
    line = [l for l in out.stdout.splitlines() if l.startswith("multigpu_drainage_check")]
    assert out.returncode == 0 and line and "DIFFER" not in line[0], (out.stdout[-2000:], out.stderr[-2000:])


# ---- refusals -------------------------------------------------------------------------------------------------------
def test_refusals_leave_the_outputs_untouched():
    from soilmachine_b200 import capi
    c, pre = _ctx("rocksand", 64, 48)
    rank = capi.Context(64, 48, 80, nranks=2, rank=0)
    try:
        c.initialize(SEED, pre["layers"])
        lib = c.lib
        host = {k: np.full(64 * 48, 5, t) for k, t in DT.items()}
        dev = {k: _alloc(c, v.nbytes, v) for k, v in host.items()}
        try:
            for on_device, out in ((0, {k: v.ctypes.data_as(C.c_void_p) for k, v in host.items()}), (1, dev)):
                for flags in (2, 4, 1 << 31, 3):
                    assert lib.sm_drainage(c.h, flags, out["spill"], out["dir"], out["area"], out["basin"], on_device,
                                           None) == capi.SM_ERR_INVALID
                assert lib.sm_drainage(c.h, 0, None, None, None, None, on_device, None) == capi.SM_ERR_INVALID
                assert lib.sm_drainage(c.h, 1, None, None, None, None, on_device, None) == capi.SM_ERR_INVALID
            for k, v in host.items():
                assert (v == 5).all(), k
                same(_d2h(dev[k], v.shape, v.dtype), v, "device %s after refusals" % k)
        finally:
            for p in dev.values():
                c.device_free(p)
        # a rank of a sharded map without its peers attached: no map to read
        if True:
            spill = np.full(rank.cells, 5.0)
            assert lib.sm_drainage(rank.h, 0, spill.ctypes.data_as(C.c_void_p), None, None, None, 0, None) == \
                capi.SM_ERR_INVALID
            assert (spill == 5.0).all()
    finally:
        c.close(); rank.close()


# ---- the C++ facade -------------------------------------------------------------------------------------------------
def test_facade_drainage(tmp_path):
    """tests/facade_drainage.cpp, plain and on a group of two: its rasters equal capi's on the facade's own map"""
    from oracle import refapi
    libdir = os.path.join(ROOT, "soilmachine_b200", "lib")
    exe = str(tmp_path / "facade_drainage")
    subprocess.check_call(["g++", "-std=c++17", "-O1", os.path.join(ROOT, "tests", "facade_drainage.cpp"), "-o", exe,
                           "-L" + libdir, "-lsoilmachine_b200", "-Wl,-rpath," + libdir])
    soil = refapi.soil_path("bigbutte")
    blobs = []
    for group in (False, True):
        env = {k: v for k, v in os.environ.items() if k not in ("SM_GPUS", "SM_GPU_DEVICES")}
        if group:
            env.update(SM_GPUS="2", SM_GPU_DEVICES="0,0")
        snap, out = str(tmp_path / ("s%d.snap" % group)), str(tmp_path / ("d%d.bin" % group))
        r = subprocess.run([exe, soil, snap, out], capture_output=True, text=True, timeout=900, env=env)
        assert r.returncode == 0, r.stdout + r.stderr
        c, pre = _ctx("bigbutte", 96, 72)
        try:
            c.restore(np.fromfile(snap, np.uint8))
            want = b"".join(c.drainage(g)[k].tobytes() for g in (False, True) for k in KEYS)
        finally:
            c.close()
        got = open(out, "rb").read()
        assert got == want, "facade (group=%s) vs capi" % group
        blobs.append(got)
    assert blobs[0] == blobs[1]
