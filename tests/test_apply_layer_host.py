"""CPU: the layer raster's per-cell logic (soilmachine_b200/csrc/sm_layer.cuh) compiled for the host by
tests/layer/host_layer.cpp, against tests/golden/layer_ops.npz - the reference's own Layermap::add / remove driven cell
by cell on golden terrains (tests/golden/make_layer_golden.py).

* Every fixture case, its rasters applied one after the other, gives the fixture's leftovers byte for byte and the
  checksum and section count of its columns after every raster, and its columns byte for byte after the last one,
  with the cells visited in x-major, reverse and shuffled order, on a top / pool image whose pool slots are shuffled,
  with holes, part of them handed out through the free ring.
* The push-count predicate equals the pool_alloc calls of every cell.
* The pool preflight accepts at pushed == free slots and refuses at pushed == free slots + 1, writing nothing.
* NaN, +-inf and a type out of range are refused with the columns untouched."""
import ctypes as C
import os

import numpy as np
import pytest

import _golden
from _hydro_budget import _build
from soilmachine_b200 import checksum
from test_snapshot_host import SEC32, _lib as _snap_lib, _pack, shuffled_image

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "..", "soilmachine_b200", "csrc")
FIX = np.load(os.path.join(_golden.GOLDEN, "layer_ops.npz"))
CASES = [str(c) for c in FIX["cases"]]
KEYS = ("offsets", "type", "size", "floor", "saturation")


def _lib():
    src = os.path.join(HERE, "layer", "host_layer.cpp")
    lib = C.CDLL(_build("host_layer", src, [os.path.join(CSRC, f) for f in ("sm_layer.cuh", "sm_core.cuh")]))
    lib.hlayer_run.argtypes = [C.c_int64, C.c_void_p, C.c_void_p, C.c_int64, C.POINTER(C.c_int64), C.c_void_p,
                               C.c_int64, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p,
                               C.c_void_p, C.c_void_p]
    return lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _input(case):
    """the fixture's input: the columns x < 16 of the golden terrain"""
    cols = _golden.cols(_golden.load(case), str(FIX[case + "_prefix"]))
    n = 16 * int(FIX[case + "_dimy"])
    m = int(cols["offsets"][n])
    return {k: np.asarray(cols[k][:n + 1] if k == "offsets" else cols[k][:m]) for k in KEYS}


def _output(case):
    """the columns after the case's last raster"""
    return {k: FIX["%s_out_%s" % (case, k)] for k in KEYS}


def _raster(case, k):
    return FIX["%s_delta_%d" % (case, k)], int(FIX["%s_type_%d" % (case, k)])


def _check_after(cols, case, k, what):
    assert checksum.columns_checksum(cols) == int(FIX["%s_sum_%d" % (case, k)]), what + ": checksum"
    assert int(cols["offsets"][-1]) == int(FIX["%s_nsec_%d" % (case, k)]), what + ": section count"


def _before(case, k):
    """the columns the case's raster k applies to: rasters 0 .. k-1 through the host build, each checked"""
    lib, snap = _lib(), _snap_lib()
    cols = _input(case)
    for j in range(k):
        delta, typ = _raster(case, j)
        im = Image(cols, seed=j, spare=2 * len(delta))
        assert im.run(lib, delta, typ, int(FIX[case + "_nsoils"]))[0] == 0
        cols = im.columns(snap)
        _check_after(cols, case, j, "%s raster %d" % (case, j))
    return cols


class Image:
    """top / pool image of a CSR (shuffled slots, garbage holes), with `nring` holes on the free ring and `spare` slots
    above the bump counter"""

    def __init__(self, cols, seed, nring=0, spare=0):
        top, pool = shuffled_image(cols, seed)
        used = np.zeros(len(pool), bool)
        f = top["below"][(top["type"] != 0xFFFFFFFF) & (top["below"] != 0xFFFFFFFF)]
        while len(f):                                      # every slot a column chain reaches
            used[f] = True
            f = pool["below"][f]
            f = f[f != 0xFFFFFFFF]
        holes = np.nonzero(~used)[0].astype(np.uint32)
        self.ring = holes[:nring].copy()
        assert len(self.ring) == nring, "not enough holes for the ring"
        self.top = top
        self.pool = np.zeros(len(pool) + spare, SEC32)
        self.pool[:len(pool)] = pool
        self.bump = C.c_int64(len(pool))

    def run(self, lib, delta, typ, nsoils, order=None):
        n = len(self.top)
        order = np.arange(n, dtype=np.int64) if order is None else np.ascontiguousarray(order, np.int64)
        left = np.zeros(n); pushes = np.zeros(n, np.int64); allocs = np.zeros(n, np.int64); st = np.zeros(4, np.int64)
        delta = np.ascontiguousarray(delta, np.float64)
        rc = lib.hlayer_run(n, _p(self.top), _p(self.pool), len(self.pool), C.byref(self.bump), _p(self.ring),
                            len(self.ring), _p(delta), int(typ), int(nsoils), _p(order), _p(left), _p(pushes),
                            _p(allocs), _p(st))
        if rc == 0:
            self.ring = self.ring[:0]      # handed out (the entries a call left are leaked holes, never reused)
        return rc, left, pushes, allocs, st

    def columns(self, snap):
        off, rec = _pack(snap, self.top, self.pool)
        return {"offsets": off.astype(np.int64), "type": rec["type"].astype(np.int32), "size": rec["size"],
                "floor": rec["floor"], "saturation": rec["saturation"]}

    def state(self):
        return self.top.tobytes() + self.pool.tobytes() + bytes(self.bump)


def _orders(n, seed):
    return {"xmajor": np.arange(n), "reverse": np.arange(n)[::-1], "shuffled": np.random.default_rng(seed).permutation(n)}


@pytest.mark.parametrize("order", ["xmajor", "reverse", "shuffled"])
@pytest.mark.parametrize("case", CASES)
def test_rasters_equal_the_reference_in_any_cell_order(case, order):
    lib, snap = _lib(), _snap_lib()
    ns, nr = int(FIX[case + "_nsoils"]), int(FIX[case + "_nrasters"])
    cells = 16 * int(FIX[case + "_dimy"])
    im = Image(_input(case), seed=len(case), nring=64, spare=2 * nr * cells + 64)
    for k in range(nr):
        delta, typ = _raster(case, k)
        want_left = FIX["%s_left_%d" % (case, k)]
        rc, left, pushes, allocs, st = im.run(lib, delta, typ, ns, _orders(cells, k)[order])
        assert rc == 0, st
        what = "%s raster %d, %s order" % (case, k, order)
        _check_after(im.columns(snap), case, k, what)
        _golden.same(left, want_left, what + ": leftovers")
        # the push count is what the pool had to serve, cell by cell
        ran = delta != 0
        assert (allocs[ran] == pushes[ran]).all() and (pushes[~ran] == 0).all() and (allocs[~ran] == 0).all()
        assert st[0] == ran.sum() and st[1] == pushes.sum() and st[3] == (want_left > 0).sum()
        # the rasters exercise what they are meant to: deposits, strips, zeros of both signs, emptied columns
        assert (delta > 0).any() and (delta < 0).any() and (want_left > 0).any()
        assert ((delta == 0) & np.signbit(delta)).any() and ((delta == 0) & ~np.signbit(delta)).any()
    _golden.same_cols(im.columns(snap), _output(case), "%s after the last raster, %s order" % (case, order))


def test_fixture_covers_every_soil_type_and_the_air_top_cases():
    lib = _lib()
    seen_double = False
    for case in CASES:
        n, ns = int(FIX[case + "_nrasters"]), int(FIX[case + "_nsoils"])
        assert sorted({int(FIX["%s_type_%d" % (case, k)]) for k in range(n)}) == list(range(ns))
        im = Image(_input(case), seed=1, spare=2 * n * 16 * int(FIX[case + "_dimy"]))
        for k in range(n):
            rc, _, pushes, _, _ = im.run(lib, *_raster(case, k), ns)
            assert rc == 0
            seen_double |= bool((pushes == 2).any())
    assert seen_double, "no raster deposits under standing water onto a column that needs two pushes"


@pytest.mark.parametrize("case", CASES[:2] + CASES[-1:])
def test_pool_preflight_is_exact(case):
    lib = _lib()
    k = 1
    cols, ns = _before(case, k), int(FIX[case + "_nsoils"])
    delta, typ = _raster(case, k)
    probe = Image(cols, seed=3, spare=2 * len(delta))
    need = int(probe.run(lib, delta, typ, ns)[4][1])
    assert need > 8
    for nring in (0, 5):
        ok = Image(cols, seed=3, nring=nring, spare=need - nring)
        before = ok.state()
        rc, _, _, _, st = ok.run(lib, delta, typ, ns)
        assert rc == 0 and st[1] == need and st[2] == need
        assert ok.bump.value == len(ok.pool), "every slot above the bump counter was used"
        assert ok.state() != before
        short = Image(cols, seed=3, nring=nring, spare=need - nring - 1)
        before = short.state()
        rc, _, _, _, st = short.run(lib, delta, typ, ns)
        assert rc == 3 and st[1] == need and st[2] == need - 1
        assert short.state() == before, "a refused raster wrote"


@pytest.mark.parametrize("bad", [np.nan, np.inf, -np.inf])
def test_non_finite_entries_are_refused_untouched(bad):
    lib = _lib()
    case = CASES[-1]
    delta = FIX["%s_delta_0" % case].copy()
    delta[len(delta) // 2 + 3] = bad
    im = Image(_input(case), seed=1, spare=2 * len(delta))
    before = im.state()
    rc = im.run(lib, delta, 1, int(FIX[case + "_nsoils"]))[0]
    assert rc == 1 and im.state() == before


@pytest.mark.parametrize("typ", [-1, "nsoils", 64])
def test_type_out_of_range_is_refused_untouched(typ):
    lib = _lib()
    case = CASES[0]
    ns = int(FIX[case + "_nsoils"])
    delta = FIX["%s_delta_0" % case]
    im = Image(_input(case), seed=1, spare=2 * len(delta))
    before = im.state()
    rc = im.run(lib, delta, ns if typ == "nsoils" else typ, ns)[0]
    assert rc == 1 and im.state() == before
