"""CPU: the drainage view's per-cell logic (soilmachine_b200/csrc/sm_drain.cuh) compiled for the host by
tests/drainage/host_drain.cpp and driven by a serial loop, against the statement of the header in numpy and heapq
(tests/_drainage.py).

* H and H under standing water (SM_DRAIN_GROUND) of top / pool images with shuffled pool slots equal the statement on
  every golden frame and hydrology state (after_flood_*, after_seep_*: standing water); crafted columns pin the
  ground rule (Air on top, Air only, empty).
* spill, dir, area, basin and the counts equal the statement byte for byte on those states, with and without the
  ground rule, and on crafted rasters: nested depressions, a flat plateau touching the border, an all-equal map, a
  spiral channel, exact slope ties between a diagonal and an edge neighbour, and the narrowest maps sm_create accepts.
* The invariants of the header hold: W >= H, W == H on the border, the fixed-point equation, receivers that form a
  forest rooted at the border, outlet areas summing to the map, one basin along every chain.
* ABI plumbing: the declaration, capi.SYMBOLS, the export, and the C++ facade compiles."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

import _drainage
import _golden
from _hydro_budget import _build
from test_snapshot_host import SEC32, shuffled_image
from test_strata_host import STATES

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(ROOT, "soilmachine_b200", "csrc")
INCLUDE = os.path.join(ROOT, "include", "soilmachine_b200.h")
KEYS = ("spill", "dir", "area", "basin")


def _lib():
    src = os.path.join(HERE, "drainage", "host_drain.cpp")
    deps = [os.path.join(CSRC, f) for f in ("sm_drain.cuh", "sm_strata.cuh", "sm_core.cuh")] + [INCLUDE]
    lib = C.CDLL(_build("host_drain", src, deps))
    lib.hdrain_heights.restype = None
    lib.hdrain_heights.argtypes = [C.c_int64, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p]
    lib.hdrain_run.restype = C.c_int
    lib.hdrain_run.argtypes = [C.c_int32, C.c_int32] + [C.c_void_p] * 6
    return lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def host_heights(lib, cols, ground, seed=3):
    top, pool = shuffled_image(cols, seed)
    H = np.full(len(top), np.nan)
    lib.hdrain_heights(len(top), _p(top), _p(pool), int(ground), _p(H))
    return H


def host_drainage(lib, H):
    """the serial host driver: dict of the four outputs and the counts"""
    H = np.ascontiguousarray(H, np.float64)
    dimx, dimy = H.shape
    out = {"spill": np.full(H.shape, np.nan), "dir": np.full(H.shape, 99, np.int8),
           "area": np.full(H.shape, -5, np.int64), "basin": np.full(H.shape, -5, np.int64)}
    st = np.zeros(4, np.int64)
    assert lib.hdrain_run(dimx, dimy, _p(H), _p(out["spill"]), _p(out["dir"]), _p(out["area"]), _p(out["basin"]),
                          _p(st)) == 0
    out.update(flat_cells=int(st[1]), depressed_cells=int(st[2]), outlets=int(st[3]))
    return out


def same_drainage(got, want, what):
    for k in KEYS:
        _golden.same(got[k], want[k], "%s: %s" % (what, k))
    for k in ("flat_cells", "depressed_cells", "outlets"):
        assert got[k] == want[k], "%s: %s %r vs %r" % (what, k, got[k], want[k])


def check_invariants(H, r, what):
    """the header's invariants, from the outputs alone"""
    H = np.asarray(H, np.float64)
    W, d, area, basin = r["spill"], r["dir"].astype(np.int64), r["area"], r["basin"]
    dimx, dimy = H.shape
    border = np.zeros(H.shape, bool)
    border[0, :] = border[-1, :] = border[:, 0] = border[:, -1] = True
    assert (W >= H).all(), what
    assert np.array_equal(W[border], H[border]), what
    assert ((d < 0) == border).all() and (d < 8).all(), what
    if dimx > 2 and dimy > 2:
        Wp = np.pad(W, 1, constant_values=np.inf)
        nmin = np.min([Wp[1 + dx:1 + dx + dimx, 1 + dy:1 + dy + dimy] for dx, dy in _drainage.N8], axis=0)
        assert np.array_equal(np.maximum(H, nmin)[~border], W[~border]), what + ": fixed point"
    dx = np.array([p[0] for p in _drainage.N8])
    dy = np.array([p[1] for p in _drainage.N8])
    idx = np.arange(dimx * dimy).reshape(dimx, dimy)
    rcv = np.where(d >= 0, idx + dx[np.maximum(d, 0)] * dimy + dy[np.maximum(d, 0)], idx).reshape(-1)
    # pointer jumping: every chain ends on the border within dimx*dimy hops (acyclic), at the cell's basin
    root = rcv.copy()
    for _ in range(int(np.ceil(np.log2(dimx * dimy + 1))) + 1):
        root = root[root]
    assert border.reshape(-1)[root].all(), what + ": a chain does not reach the border"
    assert np.array_equal(root, basin.reshape(-1)), what + ": basin"
    assert np.array_equal(basin.reshape(-1)[rcv], basin.reshape(-1)), what + ": basin along a chain"
    assert int(area[border].sum()) == dimx * dimy, what + ": outlet areas"
    don = np.zeros(dimx * dimy, np.int64)
    np.add.at(don, rcv[~border.reshape(-1)], area.reshape(-1)[~border.reshape(-1)])
    assert np.array_equal(area.reshape(-1), 1 + don), what + ": area = 1 + donors"


@pytest.mark.parametrize("case,prefix", STATES)
def test_golden_states_equal_the_statement(case, prefix):
    lib = _lib()
    g = _golden.load(case)
    cols = _golden.cols(g, prefix)
    dimx, dimy = int(g["dimx"]), int(g["dimy"])
    water = False
    for ground in (False, True):
        H = host_heights(lib, cols, ground, seed=len(prefix) + ground)
        Hs = _drainage.heights(cols, ground)
        _golden.same(H, Hs, "%s %s ground=%s: H" % (case, prefix, ground))
        H = H.reshape(dimx, dimy)
        want = _drainage.drainage(H)
        got = host_drainage(lib, H)
        same_drainage(got, want, "%s %s ground=%s" % (case, prefix, ground))
        check_invariants(H, got, "%s %s ground=%s" % (case, prefix, ground))
        water |= ground and not np.array_equal(H.reshape(-1), _drainage.heights(cols, False))
    if case.startswith("hydro") and prefix != "after_seep_0":
        assert water, "no standing water in a hydrology state"


@pytest.mark.parametrize("name", [n for n, _ in _drainage.crafted()])
def test_crafted_rasters_equal_the_statement(name):
    lib = _lib()
    H = dict(_drainage.crafted())[name]
    want = _drainage.drainage(H)
    got = host_drainage(lib, H)
    same_drainage(got, want, name)
    check_invariants(H, got, name)
    if name == "ties":
        assert got["dir"][1, 1] == 0 and got["dir"][4, 4] == 4
    if name == "spiral":
        assert got["area"].max() > H.size // 2
    if name == "nested":
        assert got["depressed_cells"] > 0 and got["flat_cells"] > 0
    if name in ("plateau", "equal"):
        assert got["flat_cells"] > 0


def test_spiral_at_256_equals_the_statement():
    lib = _lib()
    H = _drainage.spiral(256)
    got = host_drainage(lib, H)
    same_drainage(got, _drainage.drainage(H), "spiral 256")
    check_invariants(H, got, "spiral 256")


def crafted_columns():
    """bottom -> top CSR: water over ground, water only, an empty column, ground only, water over water over ground"""
    cols = [[(1, 1.0), (0, 0.5)], [(0, 2.0)], [], [(2, 0.75), (1, 0.25)], [(1, 0.5), (0, 0.25), (0, 0.125)]]
    off = np.concatenate([[0], np.cumsum([len(c) for c in cols])])
    typ = [t for c in cols for t, _ in c]
    size = [s for c in cols for _, s in c]
    floor = [f for c in cols for f in np.concatenate([[0.0], np.cumsum([s for _, s in c])[:-1]])[:len(c)]]
    return {"offsets": off, "type": np.array(typ, np.int64), "size": np.array(size), "floor": np.array(floor),
            "saturation": np.zeros(len(typ))}


def test_crafted_columns_pin_the_ground_rule():
    lib = _lib()
    cols = crafted_columns()
    _golden.same(host_heights(lib, cols, False), np.array([1.5, 2.0, 0.0, 1.0, 0.875]), "H")
    _golden.same(host_heights(lib, cols, True), np.array([1.0, 0.0, 0.0, 1.0, 0.5]), "ground")
    for g in (False, True):
        _golden.same(_drainage.heights(cols, g), host_heights(lib, cols, g), "statement, ground=%s" % g)


def test_c_abi_capi_and_facade_declare_the_call(tmp_path):
    from soilmachine_b200 import capi
    hdr = open(INCLUDE).read()
    m = re.search(r"int sm_drainage\(([^)]*)\)", hdr)
    assert m and [a.split()[-1].lstrip("*") for a in m.group(1).split(",")] == [
        "ctx", "flags", "spill", "dir", "area", "basin", "on_device", "stats"]
    assert "#define SM_DRAIN_GROUND 1" in hdr and capi.SM_DRAIN_GROUND == 1
    assert "sm_drainage" in capi.SYMBOLS
    assert hasattr(capi.load(), "sm_drainage")
    assert callable(capi.Context.drainage)
    assert C.sizeof(capi.DrainStats) == 8 * 14
    from soilmachine_b200 import host, sharded
    assert callable(host.Simulation.drainage) and callable(sharded.VirtualShards.drainage)
    assert callable(sharded.DistShard.drainage)
    subprocess.check_call(["g++", "-std=c++17", "-fsyntax-only", os.path.join(HERE, "facade_drainage.cpp")])
