"""CPU: what a context group (sm_create_group) needs that can be checked without a device.

* The warp form of the single-cell calls that change the map (soilmachine_b200/csrc/sm_cell_coop.cuh, what
  k_cell_op_w runs) on a map cut into x-strips, on the host (tests/group_cells/host_cell_ops.cpp): one section pool
  per strip, every pool access checked against the owner of the focused column.  The golden column truth table, its
  cascades and single-cell seep / water-cascade calls on the golden hydrology terrains must come out byte for byte
  as the one-thread forms do, on 1, 2 and 3 strips, with no access outside the owner's pool.
* The strip layout and the division of pool_capacity (sm_group_layout) against sharded.split_columns /
  merge_columns / merge_frequency on ragged widths.
* ABI plumbing: the refusals of sm_create_group that need no device."""
import ctypes as C
import os

import numpy as np
import pytest

import _golden
import _hostsim
from _hydro_budget import _build

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "..", "soilmachine_b200", "csrc")


class CellHostSim(_hostsim.HostSim):
    def __init__(self):
        src = os.path.join(HERE, "group_cells", "host_cell_ops.cpp")
        deps = [os.path.join(HERE, "sharded_hydro", "host_sharded.cpp"), _hostsim.SRC, _hostsim.CORE, _hostsim.NOISE,
                _hostsim.HYDRO, _hostsim.COOP, _hostsim.HCOOP, os.path.join(CSRC, "sm_foot.cuh"),
                os.path.join(CSRC, "sm_cell_coop.cuh")]
        self.lib = C.CDLL(_build("host_cell_ops", src, deps))
        self.lib.shs_violations.restype = C.c_longlong
        for f in (self.lib.shc_cell_op, self.lib.shc_cell_op_seq):
            f.restype = C.c_double
        self.lib.shc_cell_op.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int, C.c_float, C.c_float, C.c_double, C.c_int]
        self.lib.shc_cell_op_seq.argtypes = [C.c_int, C.c_int, C.c_int, C.c_float, C.c_float, C.c_double, C.c_int]
        self.lib.hs_nsections.restype = C.c_int64

    def op(self, nstrips, op, x=0, y=0, fx=0.0, fy=0.0, v=0.0, t=0):
        """nstrips None: the one-thread form; 0: the warp form on one pool; n: on n strips"""
        if nstrips is None:
            return self.lib.shc_cell_op_seq(op, int(x), int(y), fx, fy, v, int(t))
        return self.lib.shc_cell_op(nstrips, op, int(x), int(y), fx, fy, v, int(t))


@pytest.mark.parametrize("nstrips", [0, 1, 2, 3])
@pytest.mark.parametrize("lane_order", [0, 1], ids=["lanes_up", "lanes_down"])
def test_warp_cell_ops_replay_the_column_truth_table(nstrips, lane_order):
    g = _golden.load("column_ops")
    hs = CellHostSim()
    hs.init(8, 8, int(g["scale"]), g["soils"])
    hs.lib.hs_set_mode(1, lane_order)
    try:
        hs.lib.shs_violations()
        for (kind, x, y, v, t), want in zip(g["ops"], g["remove_results"]):
            got = hs.op(nstrips, 0 if kind == 0 else 1, x, y, v=float(v), t=t)
            if kind != 0:
                assert np.float64(got).tobytes() == np.float64(want).tobytes()
        _golden.same_cols(hs.columns(), _golden.cols(g, "final"), "columns after add/remove")
        for x, y, loop in g["cascades"]:
            hs.op(nstrips, 2, fx=float(x), fy=float(y), t=int(loop))
        _golden.same_cols(hs.columns(), _golden.cols(g, "after_cascade"), "columns after cascades")
        assert hs.lib.shs_violations() == 0
    finally:
        hs.lib.hs_set_mode(0, 0)


def _hydro_terrain(hs, g):
    """the golden hydrology case replayed for one frame: a terrain with ponds and wet sections"""
    hs.init(int(g["dimx"]), int(g["dimy"]), int(g["scale"]), g["soils"])
    hs.set_columns(_golden.cols(g, "init"))
    hs.water_run(g["water_xy_0"])
    hs.lib.hs_water_flood(None)


def _hydro_calls(g, nstrips_for_edges=3):
    """seep, water cascade with spill 0 and 3, a deep terrain cascade and an add under water on cells spread over the
    map, the columns next to every strip edge of 2 and 3 strips among them"""
    dimx, dimy = int(g["dimx"]), int(g["dimy"])
    xs = set(range(0, dimx, 5))
    for n in (2, 3):
        w = (dimx + n - 1) // n
        for q in range(1, n):
            xs.update((q * w - 1, q * w, q * w + 1))
    calls = []
    for i, x in enumerate(sorted(v for v in xs if 0 <= v < dimx)):
        for y in range(1 + i % 3, dimy, 4):
            calls += [(5, x, y, 0), (6, x, y, 0), (6, x, y, 3), (2, x, y, 3), (0, x, y, 1)]
    return calls


@pytest.mark.parametrize("case", _golden.HYDRO_CASES)
@pytest.mark.parametrize("nstrips", [0, 1, 2, 3])
def test_warp_cell_ops_match_the_one_thread_forms_on_wet_terrain(case, nstrips):
    g = _golden.load(case)
    want_hs, got_hs = CellHostSim(), CellHostSim()
    calls = _hydro_calls(g)
    # the one-thread forms (what k_cell_op runs)
    _hydro_terrain(want_hs, g)
    before = want_hs.columns()
    for op, x, y, t in calls:
        want_hs.op(None, op, x, y, fx=float(x), fy=float(y), v=0.0625, t=t)
    want = want_hs.columns()
    assert any(not np.array_equal(before[k], want[k]) for k in ("size", "saturation", "type")), "the calls did nothing"
    # the warp forms, strip-routed
    _hydro_terrain(got_hs, g)
    got_hs.lib.hs_set_mode(1, 0)
    try:
        got_hs.lib.shs_violations()
        for op, x, y, t in calls:
            got_hs.op(nstrips, op, x, y, fx=float(x), fy=float(y), v=0.0625, t=t)
        _golden.same_cols(got_hs.columns(), want, "columns after the single-cell calls")
        assert got_hs.lib.shs_violations() == 0
    finally:
        got_hs.lib.hs_set_mode(0, 0)


# ---- strip layout ------------------------------------------------------------------------------------------------
def _layout(dimx, dimy, nranks, pool_capacity=0):
    from soilmachine_b200 import capi
    lib = capi.load()
    cfg = capi.Config(dimx, dimy, 80, 0, pool_capacity, 0, 0)
    out = []
    for r in range(nranks):
        x0, x1, cap = C.c_int32(), C.c_int32(), C.c_int64()
        rc = lib.sm_group_layout(C.byref(cfg), nranks, r, C.byref(x0), C.byref(x1), C.byref(cap))
        if rc != capi.SM_OK:
            return rc, lib.sm_last_error(None).decode()
        out.append((x0.value, x1.value, cap.value))
    return capi.SM_OK, out


@pytest.mark.parametrize("dimx,dimy,nranks", [(96, 40, 2), (100, 37, 3), (72, 24, 3), (150, 16, 4), (33, 9, 2)])
def test_group_layout_cuts_and_merges_as_the_python_statement(dimx, dimy, nranks):
    from soilmachine_b200 import capi, sharded
    rc, lay = _layout(dimx, dimy, nranks, pool_capacity=1000003)
    assert rc == capi.SM_OK, lay
    assert lay[0][0] == 0 and lay[-1][1] == dimx
    assert all(a[1] == b[0] for a, b in zip(lay, lay[1:])) and all(x0 % 16 == 0 and x1 > x0 for x0, x1, _ in lay)
    # the shares cover the whole map's capacity, each rounded up
    for x0, x1, cap in lay:
        assert cap == -(-1000003 * (x1 - x0) // dimx)
    assert sum(c for _, _, c in lay) >= 1000003
    assert _layout(dimx, dimy, nranks, pool_capacity=0)[1][0][2] == 0
    # a ragged CSR cut at these strips and pasted together again is the input
    rng = np.random.RandomState(dimx)
    counts = rng.randint(0, 4, dimx * dimy)
    off = np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)
    n = int(off[-1])
    cols = {"offsets": off, "type": rng.randint(0, 5, n).astype(np.int32), "size": rng.rand(n), "floor": rng.rand(n),
            "saturation": rng.rand(n)}
    parts = [sharded.split_columns(cols, dimx, dimy, x0, x1) for x0, x1, _ in lay]
    for p, (x0, x1, _) in zip(parts, lay):       # what the group passes each rank: rebased offsets, sections in place
        base = off[x0 * dimy]
        assert np.array_equal(p["offsets"], off[x0 * dimy:x1 * dimy + 1] - base)
        assert p["size"].ctypes.data == cols["size"].ctypes.data + 8 * base or len(p["size"]) == 0
        p["floor"] = cols["floor"][base:base + p["offsets"][-1]]
    merged = sharded.merge_columns(parts)
    for k in cols:
        assert np.array_equal(merged[k], cols[k]), k
    # frequency arrays are y*dimx + x: each rank's columns are a 2-D block
    f = rng.rand(dimy * dimx).astype(np.float32)
    parts = [{"f": np.where((np.arange(dimx) >= x0) & (np.arange(dimx) < x1), f.reshape(dimy, dimx), np.nan).reshape(-1)
              .astype(np.float32)} for x0, x1, _ in lay]
    assert np.array_equal(sharded.merge_frequency(parts, [(a, b) for a, b, _ in lay], dimx, dimy)["f"], f)


def test_group_layout_refuses_a_map_too_narrow_for_its_ranks():
    from soilmachine_b200 import capi
    rc, msg = _layout(32, 32, 3)
    assert rc == capi.SM_ERR_INVALID and "too narrow for this many ranks (needs >= 16 columns per rank)" in msg


# ---- ABI plumbing ------------------------------------------------------------------------------------------------
def _create_group(cfg, nranks, devices, out=True):
    from soilmachine_b200 import capi
    lib = capi.load()
    h = C.c_void_p()
    devs = None if devices is None else (C.c_int32 * len(devices))(*devices)
    rc = lib.sm_create_group(C.byref(cfg) if cfg is not None else None, nranks, devs, C.byref(h) if out else None)
    msg = lib.sm_last_error(None).decode()
    if rc == capi.SM_OK:
        lib.sm_destroy(h)
    return rc, msg


def test_create_group_refusals_need_no_device():
    from soilmachine_b200 import capi
    cfg = capi.Config(96, 64, 80, 0, 0, 0, 0)
    for nranks, out in ((0, True), (9, True), (2, False)):
        rc, msg = _create_group(cfg, nranks, None, out)
        assert rc == capi.SM_ERR_INVALID and "sm_create_group" in msg, (nranks, out, rc, msg)
    rc, msg = _create_group(capi.Config(96, 64, 80, 0, 0, 0, 1 | 4), 2, [0, 0])
    assert rc == capi.SM_ERR_INVALID and "SM_FLAG_HYDRO_CELL_BUDGET" in msg
    rc, msg = _create_group(capi.Config(32, 32, 80, 0, 0, 0, 0), 3, [0, 0, 0])
    assert rc == capi.SM_ERR_INVALID and "too narrow" in msg


def test_create_group_without_a_device_says_so():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    from soilmachine_b200 import capi
    for nranks in (1, 2):
        rc, msg = _create_group(capi.Config(96, 64, 80, 0, 0, 0, 0), nranks, [0] * nranks)
        assert rc == capi.SM_ERR_NOGPU and "no CUDA device" in msg
    with pytest.raises(capi.SoilMachineError) as e:
        capi.Context(96, 64, gpus=2, devices=[0, 0])
    assert e.value.code == capi.SM_ERR_NOGPU
