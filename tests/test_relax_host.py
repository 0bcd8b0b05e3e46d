"""CPU: the slope relaxation's per-visit logic (soilmachine_b200/csrc/sm_relax.cuh) compiled for the host by
tests/relax/host_relax.cpp, against tests/golden/relax_ops.npz - the reference's own Particle::cascade driven in
sm_relax's phase order (tests/golden/make_relax_golden.py).

* Every fixture case, for transferloop 0, 1 and 3, in x-major, reversed and shuffled order inside each phase: the
  checksum and section count after every pass, the columns byte for byte after K passes (flat maps), and passes /
  stable of one call over all the fixture's passes.  Skipped visits are exact: one call with its stale bits equals
  calls of one pass each.
* Negative controls: a period of P - 1 in reversed order, and marking with radius R - 1, diverge from the fixture.
* A call whose pushes exceed the free slots it starts with, but whose end state fits, drops nothing: the slots freed
  by one phase serve the next."""
import ctypes as C
import os

import numpy as np
import pytest

import _golden
from _hydro_budget import _build
from soilmachine_b200 import checksum
from test_apply_layer_host import KEYS, Image, _lib as _layer_lib
from test_snapshot_host import _lib as _snap_lib

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "..", "soilmachine_b200", "csrc")
FIX = np.load(os.path.join(_golden.GOLDEN, "relax_ops.npz"))
CASES = [str(c) for c in FIX["cases"]]
LOOPS = [int(t) for t in FIX["loops"]]
K = 3
SOILDEV = np.dtype([(k, "<f4") for k in ("friction", "solubility", "equrate", "erosionrate", "maxdiff", "settling",
                                         "suspension", "porosity")] +
                   [(k, "<u4") for k in ("transports", "erodes", "cascades", "abrades")])
ORDERS = {"xmajor": 0, "reverse": 1, "shuffled": 2}


def _lib():
    src = os.path.join(HERE, "relax", "host_relax.cpp")
    lib = C.CDLL(_build("host_relax", src, [os.path.join(CSRC, f) for f in ("sm_relax.cuh", "sm_core.cuh")]))
    lib.hrelax_run.argtypes = [C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64,
                               C.POINTER(C.c_int64), C.c_void_p, C.c_int64, C.c_int, C.c_int, C.c_int, C.c_uint64,
                               C.c_int, C.c_int, C.c_void_p, C.c_void_p]
    return lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def soil_table(case):
    """the case's soil table as the device holds it (SoilDev)"""
    s = FIX[case + "_soils"]
    out = np.zeros(len(s), SOILDEV)
    for k in SOILDEV.names:
        out[k] = s[k]
    return out


def scale(case):
    from soilmachine_b200 import presets
    soil = str(FIX[case + "_soil"])
    return 80 if soil == "settling1" else presets.load(soil)["world"]["scale"]


def base_columns(case):
    """the map before the steep raster: the golden terrain, or the flat map of make_relax_golden.flat"""
    terrain = str(FIX[case + "_terrain"])
    if terrain:
        return _golden.cols(_golden.load(terrain), str(FIX[case + "_prefix"]))
    n = int(FIX[case + "_dimx"]) * int(FIX[case + "_dimy"])
    return {"offsets": np.arange(n + 1, dtype=np.int64), "type": np.ones(n, np.int32), "size": np.full(n, 0.5),
            "floor": np.zeros(n), "saturation": np.zeros(n)}


def steep_columns(case):
    """the case's input: its raster applied by the host build of sm_layer.cuh, checked against the fixture"""
    cols = base_columns(case)
    d = FIX[case + "_delta"]
    im = Image(cols, seed=1, spare=2 * len(d))
    assert im.run(_layer_lib(), d, int(FIX[case + "_type"]), len(FIX[case + "_soils"]))[0] == 0
    cols = im.columns(_snap_lib())
    assert checksum.columns_checksum(cols) == int(FIX[case + "_sum_in"]), case + ": steep input"
    return cols


def after_k(case, tl):
    """the fixture's columns after K passes: the steep map with the stored cells replaced"""
    steep = steep_columns(case)
    key = "%s_t%d_" % (case, tl)
    cells = set(int(c) for c in FIX[key + "cells"])
    sub = {k: FIX[key + "out_" + k] for k in KEYS}
    out = {k: [] for k in KEYS if k != "offsets"}
    off, j = [0], 0
    for i in range(len(steep["offsets"]) - 1):
        src, s = (sub, j) if i in cells else (steep, i)
        a, b = int(src["offsets"][s]), int(src["offsets"][s + 1])
        for k in out:
            out[k].append(src[k][a:b])
        off.append(off[-1] + b - a)
        j += i in cells
    res = {k: np.concatenate(v) for k, v in out.items()}
    res["offsets"] = np.array(off, np.int64)
    return res


class Relax:
    """a top / pool image of a map (Image) relaxed by the host build; the slots a call leaves on its free rings are not
    handed to the next call, hence the generous default spare"""

    def __init__(self, case, cols, seed=7, nring=0, spare=None):
        self.case = case
        self.dimx, self.dimy = int(FIX[case + "_dimx"]), int(FIX[case + "_dimy"])
        self.im = Image(cols, seed=seed, nring=nring, spare=40 * self.dimx * self.dimy if spare is None else spare)
        self.soils = soil_table(case)

    def run(self, passes, tl, order="xmajor", period=0, radius=-1, seed=0):
        st = np.zeros(7, np.int64)
        ch = np.zeros(max(passes, 1), np.int64)
        rc = _lib().hrelax_run(self.dimx, self.dimy, scale(self.case), _p(self.soils), _p(self.im.top),
                               _p(self.im.pool), len(self.im.pool), C.byref(self.im.bump), _p(self.im.ring),
                               len(self.im.ring), passes, tl, ORDERS[order], seed, period, radius, _p(st), _p(ch))
        self.im.ring = self.im.ring[:0]
        return rc, st, ch

    def columns(self):
        return self.im.columns(_snap_lib())


def fixture_passes(case, tl):
    return int(FIX["%s_t%d_passes" % (case, tl)])


@pytest.mark.parametrize("order", list(ORDERS))
@pytest.mark.parametrize("tl", LOOPS)
@pytest.mark.parametrize("case", CASES)
def test_passes_equal_the_reference(case, tl, order):
    key = "%s_t%d_" % (case, tl)
    steep = steep_columns(case)
    sums, nsec = FIX[key + "sums"], FIX[key + "nsec"]
    # pass by pass (a call of one pass each) for the first passes
    r = Relax(case, steep)
    for k in range(min(len(sums), 6)):
        rc, st, _ = r.run(1, tl, order, seed=k)
        assert rc == 0 and st[0] == 1 and st[4] == 0
        cols = r.columns()
        what = "%s transferloop %d %s pass %d" % (case, tl, order, k + 1)
        assert checksum.columns_checksum(cols) == int(sums[k]), what + ": checksum"
        assert int(cols["offsets"][-1]) == int(nsec[k]), what + ": sections"
        if k + 1 == K and key + "cells" in FIX:
            _golden.same_cols(cols, after_k(case, tl), what)
    # one call over all the fixture's passes: the stale bits skip visits and change nothing
    n, stable = fixture_passes(case, tl), int(FIX[key + "stable"])
    r = Relax(case, steep)
    rc, st, ch = r.run(n + 5 if stable else n, tl, order, seed=99)
    assert rc == 0 and st[4] == 0
    assert checksum.columns_checksum(r.columns()) == int(sums[n - 1])
    if stable:
        assert st[0] == stable and st[1] == 1 and ch[stable - 1] == 0 and (ch[:stable - 1] > 0).all()
        assert st[2] < st[0] * r.dimx * r.dimy // 2, "the stale bits skip most visits of a converging call"
    else:
        assert st[0] == n and st[1] == 0
    assert st[3] > 0 and st[5] >= st[3]


def test_fixture_reaches_a_stable_pass_and_runs_past_k():
    assert any(int(FIX["%s_t%d_stable" % (c, t)]) > 0 for c in CASES for t in LOOPS)
    assert all(fixture_passes(c, t) >= K for c in CASES for t in LOOPS)
    assert (base_columns("water")["type"] == 0).any(), "the water case has standing water on top"


def test_short_period_diverges():
    """the phase period P - 1 lets two cells of a phase share columns: in reversed order the result differs"""
    diverged = []
    for case in CASES:
        for tl in LOOPS:
            r = Relax(case, steep_columns(case))
            r.run(1, tl, "reverse", period=2 * (1 + tl))
            diverged.append(checksum.columns_checksum(r.columns()) != int(FIX["%s_t%d_sums" % (case, tl)][0]))
    assert all(diverged), diverged


def test_short_marking_radius_diverges():
    """marking the cells within R - 1 of a change misses cells whose footprint reached it: some call diverges"""
    diverged = []
    for case in CASES:
        for tl in LOOPS:
            n = min(fixture_passes(case, tl), 40)
            r = Relax(case, steep_columns(case))
            r.run(n, tl, radius=tl)
            diverged.append(checksum.columns_checksum(r.columns()) != int(FIX["%s_t%d_sums" % (case, tl)][n - 1]))
    assert any(diverged), diverged


def test_freed_slots_serve_the_next_phases():
    """a call that allocates more slots than it starts with free, but whose end state fits, drops nothing"""
    case, tl = "flat_settling1", 1
    steep = steep_columns(case)
    big = Relax(case, steep)
    rc, st, _ = big.run(fixture_passes(case, tl), tl)
    want = big.columns()
    grown = int(want["offsets"][-1]) - int(steep["offsets"][-1])
    assert rc == 0 and st[6] > grown + 64, (st, grown)
    spare = max(grown, 0) + 16
    small = Relax(case, steep, spare=spare)
    rc, st2, _ = small.run(fixture_passes(case, tl), tl)
    assert st2[6] > spare, "the call allocates more than the slots it starts with"
    assert rc == 0 and st2[4] == 0
    _golden.same_cols(small.columns(), want, "small pool")
    # a pool smaller than the end state drops sections and stops
    tiny = Relax(case, steep, spare=0)
    rc, st3, _ = tiny.run(fixture_passes(case, tl), tl)
    if grown > 0:
        assert rc == 3 and st3[4] > 0
