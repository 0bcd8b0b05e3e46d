"""The pooling hydrology (floods and the seep pass) on a sharded map, issued by one rank, against one unsharded context
that runs the same frames: columns, heights, frequency maps and hydrology counters byte for byte after every phase,
whichever rank issues the calls.  The shapes are those of test_sharded_views (the 4-rank one has a last strip narrower
than the others)."""
import os
import subprocess
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

SHAPES = [(2, "rocksand", 128, 96, 900, 500),
          (3, "rockgravelpebblessand", 144, 80, 900, 700),
          (4, "default", 160, 64, 600, 300)]
SEED = 5  # the hydrology reaches more than one strip and a strip edge in every shape
FRAMES = 3
HYDRO_KEYS = ("floods", "nested", "nested_steps", "transfers", "cells")


def _same(a, b, what):
    a = np.ascontiguousarray(a); b = np.ascontiguousarray(b)
    assert a.shape == b.shape, (what, a.shape, b.shape)
    if not np.array_equal(a.view(np.uint8), b.view(np.uint8)):
        bad = np.nonzero(a.reshape(-1) != b.reshape(-1))[0]
        raise AssertionError("%s differs at %d entries, first %s: %r vs %r" %
                             (what, len(bad), bad[:4], a.reshape(-1)[bad[:4]], b.reshape(-1)[bad[:4]]))


def _pair(nranks, soil, dimx, dimy, budget=False):
    from soilmachine_b200 import capi, presets, sharded
    pre = presets.load(soil)
    scale = pre["world"]["scale"]
    sh = sharded.VirtualShards(nranks, dimx, dimy, scale, max_particles=4096, budget=budget)
    one = capi.Context(dimx, dimy, scale, max_particles=4096, budget=budget)
    for m in (sh, one):
        m.set_soils(pre["soils"])
        m.initialize(SEED, pre["layers"])
    return sh, one


def _maps_equal(sh, one, what):
    c1, c2 = one.download_columns(), sh.download_columns()
    for k in c1:
        _same(c2[k], c1[k], what + ": columns." + k)
    _same(sh.heights(), one.heights(), what + ": heights")
    f1, f2 = one.frequency(), sh.frequency()
    for k in f1:
        _same(f2[k], f1[k], what + ": " + k)


def _changed_columns(before, after, dimx, dimy):
    """x of every column whose sections differ between two downloads"""
    xs = set()
    ob, oa = before["offsets"], after["offsets"]
    for c in range(dimx * dimy):
        a = slice(ob[c], ob[c + 1]); b = slice(oa[c], oa[c + 1])
        if ob[c + 1] - ob[c] != oa[c + 1] - oa[c] or any(
                not np.array_equal(before[k][a], after[k][b]) for k in ("type", "size", "floor", "saturation")):
            xs.add(c // dimy)
    return xs


def _holders(states, want, keys):
    """per particle: the ranks whose copy is the unsharded final state (the rank that ran its last step among them)"""
    def row(st, i):
        return b"".join(np.ascontiguousarray(st[k][i]).tobytes() for k in keys)
    return [frozenset(r for r, st in enumerate(states) if row(st, i) == row(want, i)) for i in range(len(want["alive"]))]


def _frames(sh, one, issuer, dimx, dimy, nw, nd, check_budget=False):
    """FRAMES frames of water batch -> flood -> seep -> wind batch -> frequency update; the maps are compared after
    every phase.  Returns the columns the hydrology changed, and the particle indices whose water state (frame f + 1)
    and wind state (frame f) were left by different ranks."""
    from soilmachine_b200 import host
    host.srand(SEED)
    touched = set()
    moved = set()
    wind_holders = None
    for f in range(FRAMES):
        xw, xd = host.spawn_list(nw, dimx, dimy), host.spawn_list(nd, dimx, dimy)
        a, b = sh.water_run(xw), one.water_run(xw)
        assert (a.steps, a.sweeps, a.exit_oob, a.exit_evap, a.exit_stall) == \
            (b.steps, b.sweeps, b.exit_oob, b.exit_evap, b.exit_stall), "frame %d water batch" % f
        _maps_equal(sh, one, "frame %d after the water batch" % f)
        want = one.water_state()
        water_holders = _holders([c.water_state() for c in sh.ctx], want, ("pos", "speed", "volume", "sediment", "contains"))
        if wind_holders is not None:
            n = min(len(water_holders), len(wind_holders))
            moved.update(i for i in range(n) if water_holders[i] and wind_holders[i] and
                         not (water_holders[i] & wind_holders[i]))
        for name in ("flood", "seep"):
            before = one.download_columns()
            hs = getattr(sh, "water_flood" if name == "flood" else "seep")(rank=issuer)
            h1 = (one.water_flood if name == "flood" else one.seep)()
            what = "frame %d after the %s (issued by rank %d)" % (f, name, issuer)
            assert [getattr(hs, k) for k in HYDRO_KEYS] == [getattr(h1, k) for k in HYDRO_KEYS], what
            _maps_equal(sh, one, what)
            if check_budget:
                assert sh.ctx[issuer].last_hydro_budget() == one.last_hydro_budget(), what + ": hydrology budget"
            touched |= _changed_columns(before, one.download_columns(), dimx, dimy)
        a, b = sh.wind_run(xd), one.wind_run(xd)
        assert (a.steps, a.exit_oob) == (b.steps, b.exit_oob), "frame %d wind batch" % f
        _maps_equal(sh, one, "frame %d after the wind batch" % f)
        wind_holders = _holders([c.wind_state() for c in sh.ctx], one.wind_state(),
                                ("pos", "speed", "height", "sediment", "contains"))
        sh.frequency_update(); one.frequency_update()
        _maps_equal(sh, one, "frame %d after the frequency update" % f)
    return touched, moved


@pytest.mark.parametrize("last_rank", [False, True], ids=["issuer0", "issuer_last"])
@pytest.mark.parametrize("nranks,soil,dimx,dimy,nw,nd", SHAPES)
def test_sharded_hydrology_matches_one_context(nranks, soil, dimx, dimy, nw, nd, last_rank):
    """Also: the hydrology changed columns on more than one strip and within 3 columns of a strip edge, and some
    particle index was left dead by one rank in a wind batch and by another in the next water batch (a dead marker
    of the earlier batch on the wrong rank would then be taken for the holder's)."""
    issuer = nranks - 1 if last_rank else 0
    sh, one = _pair(nranks, soil, dimx, dimy)
    try:
        touched, moved = _frames(sh, one, issuer, dimx, dimy, nw, nd)
        strips = {next(q for q, (x0, x1) in enumerate(sh.ranges) if x0 <= x < x1) for x in touched}
        assert len(strips) > 1, ("the hydrology changed one strip only", sorted(touched))
        edges = [x0 for x0, _ in sh.ranges[1:]]
        assert any(abs(x - x0) <= 3 or abs(x + 1 - x0) <= 3 for x in touched for x0 in edges), \
            ("nothing changed near a strip edge", sorted(touched))
        assert moved, "no particle index changed ranks between a wind batch and the next water batch"
    finally:
        sh.close(); one.close()


@pytest.mark.parametrize("nranks,soil,dimx,dimy,nw,nd", SHAPES[:2])
def test_sharded_hydrology_budget_matches_one_context(nranks, soil, dimx, dimy, nw, nd):
    """with budget=True the issuer's sm_last_hydro_budget equals the unsharded budget context's, bit for bit"""
    sh, one = _pair(nranks, soil, dimx, dimy, budget=True)
    try:
        _frames(sh, one, nranks - 1, dimx, dimy, nw, nd, check_budget=True)
    finally:
        sh.close(); one.close()


def test_sharded_hydrology_errors():
    from soilmachine_b200 import capi, presets, sharded
    pre = presets.load("rocksand")
    # on a rank that is not the issuer, and on the issuer before sm_peer_attach
    ranks = [capi.Context(64, 64, 80, max_particles=256, nranks=2, rank=r, share=2) for r in range(2)]
    try:
        ranks[0].set_soils(pre["soils"])
        for call in (ranks[0].water_flood, ranks[0].seep):
            with pytest.raises(capi.SoilMachineError) as e:
                call()
            assert e.value.code == capi.SM_ERR_INVALID and "not the issuing rank" in str(e.value), str(e.value)
        ranks[0].hydro_issuer(True)
        for call in (ranks[0].water_flood, ranks[0].seep):
            with pytest.raises(capi.SoilMachineError) as e:
                call()
            assert e.value.code == capi.SM_ERR_INVALID and "sm_peer_attach" in str(e.value), str(e.value)
    finally:
        for c in ranks:
            c.close()
    # a flood after a wind batch
    sh = sharded.VirtualShards(2, 96, 64, pre["world"]["scale"], max_particles=1024)
    try:
        sh.set_soils(pre["soils"])
        sh.initialize(SEED, pre["layers"])
        xy = np.array([[10.0, 10.0], [70.0, 30.0]], np.float32)
        sh.wind_run(xy)
        with pytest.raises(capi.SoilMachineError) as e:
            sh.water_flood(rank=1)
        assert e.value.code == capi.SM_ERR_INVALID and "not a water batch" in str(e.value), str(e.value)
        sh.seep(rank=1)                                   # the seep pass needs no batch
        # issuing from rank 1 made rank 0 a non-issuer: a call made there is refused, not run a second time
        with pytest.raises(capi.SoilMachineError) as e:
            sh.ctx[0].seep()
        assert e.value.code == capi.SM_ERR_INVALID and "not the issuing rank" in str(e.value), str(e.value)
    finally:
        sh.close()
    # the hydrology's per-cell maps stay unsharded only
    with pytest.raises(capi.SoilMachineError) as e:
        capi.Context(64, 64, 80, max_particles=256, nranks=2, rank=0, share=2, hydro_cell_budget=True)
    assert e.value.code == capi.SM_ERR_INVALID


def test_sharded_hydrology_over_cuda_ipc_two_processes_one_gpu():
    """tests/multigpu_hydro_check.py with two processes sharing this GPU: the peers' strips, pools and frequency
    arrays are CUDA-IPC mappings, as across GPUs.  Every phase of the frames must equal one unsharded context."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ, SM_ONE_GPU="1")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2",
           "--master-addr", "127.0.0.1", "--master-port", "29641",
           os.path.join(root, "tests", "multigpu_hydro_check.py"), "96", "600", "rockgravelpebblessand", "3"]
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=900, cwd=root, env=env)
    line = [l for l in out.stdout.splitlines() if l.startswith("multigpu_hydro_check")]
    assert out.returncode == 0 and line and "DIFFER" not in line[0], (out.stdout[-2000:], out.stderr[-2000:])
