"""CPU: the strata views' per-cell logic (soilmachine_b200/csrc/sm_strata.cuh) compiled for the host by
tests/strata/host_strata.cpp, against the statement of the header in numpy (tests/_strata.py), on top / pool images of
the golden columns with shuffled pool slots.

* Composition equals the statement byte for byte on every golden frame state (after_water, after_frame) and every
  hydrology state (after_flood_*, after_seep_*: standing water, non-zero saturation), for all four flag combinations,
  absolute and below-surface windows (+-inf bounds, zero width, above and below the map), all soils at once and every
  single soil, Air included.
* Voxels equal the statement on the same states; the section -> sample range equals a brute-force check of
  floor <= z_k < floor + size for every k < nz, with dz in {0.1, 1/3, 2^-20}, negative z0, samples exactly on floor and
  on floor + size, nz up to 65536.
* Crafted columns (empty, a zero-size top, floors out of order) pin "first met top -> bottom" and the full walk; a walk
  that stops below the window gives a different answer there.
* Over the whole column, all soils: the slots of a cell sum to H within (2 * sections + 1) ulp(H) wherever the floors
  are running sums."""
import ctypes as C
import os

import numpy as np
import pytest

import _golden
import _strata
from _hydro_budget import _build
from test_snapshot_host import SEC32, shuffled_image

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "..", "soilmachine_b200", "csrc")
INCLUDE = os.path.join(HERE, "..", "include", "soilmachine_b200.h")
STATES = ([(c, p) for c in _golden.FRAME_CASES for p in ("after_water", "after_frame")] +
          [(c, p) for c in _golden.HYDRO_CASES for p in ["after_flood_2"] + ["after_seep_%d" % f for f in range(3)]])
KEYS = ("offsets", "type", "size", "floor", "saturation")


def _lib():
    src = os.path.join(HERE, "strata", "host_strata.cpp")
    lib = C.CDLL(_build("host_strata", src, [os.path.join(CSRC, f) for f in ("sm_strata.cuh", "sm_core.cuh")] + [INCLUDE]))
    lib.hstrata_compose.restype = C.c_int64
    lib.hstrata_compose.argtypes = [C.c_int64, C.c_void_p, C.c_void_p, C.c_double, C.c_double, C.c_int32, C.c_void_p,
                                    C.c_int32, C.c_void_p, C.c_void_p]
    lib.hstrata_voxel.restype = C.c_int64
    lib.hstrata_voxel.argtypes = [C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_double, C.c_double, C.c_int32,
                                  C.c_void_p]
    lib.hstrata_range.restype = None
    lib.hstrata_range.argtypes = [C.c_int64, C.c_void_p, C.c_void_p, C.c_double, C.c_double, C.c_int32, C.c_void_p,
                                  C.c_void_p]
    return lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def state(case, prefix):
    """(columns, porosity float32[SM_MAX_SOILS], nsoils, dimx, dimy)"""
    g = _golden.load(case)
    por = np.zeros(64, np.float32)
    ns = len(g["soils"])
    por[:ns] = g["soils"]["porosity"]
    return _golden.cols(g, prefix), por, ns, int(g["dimx"]), int(g["dimy"])


class Image:
    """top / pool image of a CSR: buried sections in shuffled pool slots among garbage holes"""

    def __init__(self, cols, seed=7):
        self.top, self.pool = shuffled_image(cols, seed)
        self.n = len(self.top)

    def compose(self, lib, por, types, lo, hi, flags):
        t = np.ascontiguousarray(types, np.int32)
        out = np.full((len(t), self.n), np.nan)
        nsec = lib.hstrata_compose(self.n, _p(self.top), _p(self.pool), lo, hi, flags, _p(t), len(t), _p(por), _p(out))
        return out, nsec

    def voxel(self, lib, dimy, x0, x1, y0, y1, z0, dz, nz):
        xs, ys = np.meshgrid(np.arange(x0, x1), np.arange(y0, y1), indexing="ij")
        cells = np.ascontiguousarray((xs * dimy + ys).reshape(-1), np.int64)
        out = np.full((nz, len(cells)), 7, np.uint8)
        nsec = lib.hstrata_voxel(len(cells), _p(cells), _p(self.top), _p(self.pool), z0, dz, nz, _p(out))
        return out.reshape(nz, x1 - x0, y1 - y0), nsec


def windows(cols):
    """(lo, hi, flags-without-pore) covering whole columns, bands, +-inf, zero width, above and below the map"""
    H = _strata.heights(cols)
    top, mid = float(H.max()), float(np.median(H))
    absolute = [(-np.inf, np.inf), (mid - 1.0, mid), (0.25 * mid, 0.75 * mid), (mid, mid), (top + 1.0, np.inf),
                (-np.inf, -1.0), (-np.inf, mid)]
    below = [(0.0, 1.0), (0.5, 2.5), (-np.inf, 0.25), (0.0, np.inf), (1.0, 1.0), (-np.inf, -0.5), (top + 5.0, np.inf)]
    return [(lo, hi, 0) for lo, hi in absolute] + [(lo, hi, _strata.BELOW_SURFACE) for lo, hi in below]


def type_sets(ns):
    return [list(range(ns))] + [[t] for t in range(ns)] + [list(range(ns))[::-1]]


@pytest.mark.parametrize("case,prefix", STATES)
def test_composition_equals_the_statement(case, prefix):
    lib = _lib()
    cols, por, ns, _, _ = state(case, prefix)
    im = Image(cols, seed=len(prefix))
    nsec = int(cols["offsets"][-1])
    pore_seen = False
    for lo, hi, f in windows(cols):
        for pore in (0, _strata.PORE_WATER):
            for types in type_sets(ns):
                got, n = im.compose(lib, por, types, lo, hi, f | pore)
                want = _strata.composition(cols, por, types, lo, hi, f | pore)
                _golden.same(got, want, "%s %s [%r, %r] flags %d types %s" % (case, prefix, lo, hi, f | pore, types))
                assert n == nsec
                pore_seen |= bool(pore and (got > 0).any())
    if case.startswith("hydro"):
        assert pore_seen, "no pore water in a hydrology state"


@pytest.mark.parametrize("case,prefix", STATES)
def test_voxels_equal_the_statement(case, prefix):
    lib = _lib()
    cols, _, _, dimx, dimy = state(case, prefix)
    im = Image(cols, seed=3)
    H = _strata.heights(cols)
    for z0, dz, nz in [(-0.5, 0.1, 96), (-1.0 / 3, 1.0 / 3, 40), (float(H.min()) - 1e-3, 2.0 ** -10, 2000),
                       (float(H.max()) + 1.0, 1.0, 4)]:
        got, n = im.voxel(lib, dimy, 0, dimx, 0, dimy, z0, dz, nz)
        _golden.same(got, _strata.voxelize(cols, dimy, 0, dimx, 0, dimy, z0, dz, nz), "%s %s z0 %r dz %r" % (case, prefix, z0, dz))
        assert n == int(cols["offsets"][-1])
    # a strata section one cell wide, and a window away from the origin
    for x0, x1, y0, y1 in [(3, 4, 0, dimy), (0, dimx, 5, 6), (7, dimx - 2, 9, dimy - 4)]:
        got, _ = im.voxel(lib, dimy, x0, x1, y0, y1, -0.25, 1.0 / 64, 512)
        _golden.same(got, _strata.voxelize(cols, dimy, x0, x1, y0, y1, -0.25, 1.0 / 64, 512), "window %s" % ((x0, x1, y0, y1),))


@pytest.mark.parametrize("dz", [0.1, 1.0 / 3, 2.0 ** -20])
@pytest.mark.parametrize("z0", [-3.7, -0.1, 0.0])
def test_sample_range_equals_brute_force(z0, dz):
    lib = _lib()
    nz = 65536
    z = _strata.samples(z0, dz, nz)
    rng = np.random.default_rng(int(dz * 1e6) + int(-z0 * 10))
    m = 160
    k = rng.integers(0, nz, size=(m, 2))
    k.sort(axis=1)
    floor = z[k[:, 0]].copy()                    # samples exactly on floor ...
    size = z[k[:, 1]] - floor                    # ... and (where the subtraction is exact) on floor + size
    floor[:40] += rng.uniform(-2, 2, 40) * dz    # and anywhere
    size[:40] = rng.uniform(0, 50, 40) * dz
    floor[40:50] = z[0] - rng.uniform(0, 5, 10)  # starting under the ladder
    floor[50:55] = z[-1] + np.array([0.0, dz, 1.0, -dz, 1e9])   # on the last sample and above it
    size[50:55] = np.array([0.0, dz, 1.0, 2 * dz, 1.0])
    size[55:60] = 0.0                            # empty sections
    size[60:64] = np.inf
    k[:, 1] = np.minimum(k[:, 1], nz - 1)
    k0 = np.zeros(m, np.uint32); k1 = np.zeros(m, np.uint32)
    lib.hstrata_range(m, _p(floor), _p(size), z0, dz, nz, _p(k0), _p(k1))
    on_top = 0
    for i in range(m):
        inside = np.nonzero((floor[i] <= z) & (z < floor[i] + size[i]))[0]
        want = (int(inside[0]), int(inside[-1]) + 1) if len(inside) else None
        got = (int(k0[i]), int(k1[i]))
        if want is None:
            assert got[0] == got[1], (i, floor[i], size[i], got)
        else:
            assert got == want and len(inside) == want[1] - want[0], (i, floor[i], size[i], got, want)
        on_top += bool(np.any(z == floor[i] + size[i]))
    assert on_top > 20, "few samples land exactly on floor + size"
    assert k1.max() == nz, "no section reaches the last sample"


def crafted():
    """bottom -> top CSR of six columns (dimy 3): empty; a zero-size top over Rock; floors out of order (the top
    section overlaps the ones under it); a buried section below the window over one inside it; a lone Air section; a
    column whose floors are running sums"""
    cols = [[],
            [(1, 2.0, 0.0, 0.0), (2, 0.0, 2.0, 0.5)],
            [(1, 2.0, 0.0, 0.1), (2, 1.0, 2.0, 0.2), (3, 1.5, 1.0, 0.3)],
            [(3, 1.0, 3.0, 0.4), (2, 1.0, 0.0, 0.5), (1, 1.0, 5.0, 0.6)],
            [(0, 0.75, 0.0, 1.0)],
            [(1, 1.25, 0.0, 0.0), (3, 0.5, 1.25, 0.25), (0, 0.25, 1.75, 1.0)]]
    off = np.zeros(len(cols) + 1, np.int64)
    off[1:] = np.cumsum([len(c) for c in cols])
    recs = [r for c in cols for r in c]
    return {"offsets": off, "type": np.array([r[0] for r in recs], np.int32), "size": np.array([r[1] for r in recs]),
            "floor": np.array([r[2] for r in recs]), "saturation": np.array([r[3] for r in recs])}


CRAFTED_POR = np.array([1.0, 0.0, 0.5, 0.25] + [0.0] * 60, np.float32)


def crafted_expect():
    """the pinned answers on crafted(): (composition of all four types over [2.5, 4.5], voxels at z = k/4, k < 28)"""
    comp = np.zeros((4, 6))
    comp[2, 2] = 0.5                     # column 2: type 2 [2, 3); the top, type 3 [1, 2.5), ends where the window starts
    comp[3, 3] = 1.0                     # column 3: type 3 [3, 4) under type 2 [0, 1), which ends below the window
    vox = np.full((28, 6), 255, np.uint8)
    z = np.arange(28) / 4.0
    vox[z < 2.0, 1] = 1
    vox[(z >= 1.0) & (z < 2.5), 2] = 3   # the top section, met first, wins where it overlaps
    vox[(z < 1.0), 2] = 1
    vox[(z >= 2.5) & (z < 3.0), 2] = 2
    vox[(z >= 5.0) & (z < 6.0), 3] = 1
    vox[(z < 1.0), 3] = 2
    vox[(z >= 3.0) & (z < 4.0), 3] = 3
    vox[z < 0.75, 4] = 0
    vox[z < 1.25, 5] = 1
    vox[(z >= 1.25) & (z < 1.75), 5] = 3
    vox[(z >= 1.75) & (z < 2.0), 5] = 0
    return comp, vox.reshape(28, 2, 3)


def test_crafted_columns_pin_first_met_and_the_full_walk():
    lib = _lib()
    cols = crafted()
    im = Image(cols, seed=1)
    comp, vox = crafted_expect()
    got, n = im.compose(lib, CRAFTED_POR, [0, 1, 2, 3], 2.5, 4.5, 0)
    _golden.same(got, _strata.composition(cols, CRAFTED_POR, [0, 1, 2, 3], 2.5, 4.5), "host build vs statement")
    _golden.same(got, comp, "crafted composition")
    assert n == int(cols["offsets"][-1])
    stopped = _strata.composition(cols, CRAFTED_POR, [0, 1, 2, 3], 2.5, 4.5, stop_below=True)
    assert not np.array_equal(stopped, got), "the negative control (a walk that stops below the window) should differ"
    assert stopped[3, 3] == 0.0
    gv, _ = im.voxel(lib, 3, 0, 2, 0, 3, 0.0, 0.25, 28)
    _golden.same(gv, vox, "crafted voxels")
    _golden.same(_strata.voxelize(cols, 3, 0, 2, 0, 3, 0.0, 0.25, 28), vox, "statement, crafted voxels")
    # every flag combination and window on the crafted columns
    for lo, hi, f in windows(cols):
        for pore in (0, _strata.PORE_WATER):
            for types in ([0, 1, 2, 3], [2], [0]):
                g2, _ = im.compose(lib, CRAFTED_POR, types, lo, hi, f | pore)
                _golden.same(g2, _strata.composition(cols, CRAFTED_POR, types, lo, hi, f | pore), "crafted %r" % ((lo, hi, f | pore, types),))


@pytest.mark.parametrize("case,prefix", STATES)
def test_whole_column_slots_sum_to_the_height(case, prefix):
    lib = _lib()
    cols, por, ns, _, _ = state(case, prefix)
    got, _ = Image(cols).compose(lib, por, list(range(ns)), -np.inf, np.inf, 0)
    H = _strata.heights(cols)
    off, size, floor = cols["offsets"], cols["size"], cols["floor"]
    cnt = np.diff(off)
    running = np.ones(len(cnt), bool)
    for c in range(len(cnt)):
        f = floor[off[c]:off[c + 1]]
        s = size[off[c]:off[c + 1]]
        running[c] = len(f) == 0 or (f[0] == 0.0 and np.array_equal(f[1:], f[:-1] + s[:-1]))
    assert running.mean() > 0.9
    total = got.sum(axis=0)
    err = np.abs(total - H)[running]
    bound = ((2 * cnt + 1) * np.spacing(np.abs(H)))[running]
    assert (err <= bound).all(), "worst %r ulp" % (float((err / np.spacing(np.abs(H))[running]).max()),)
