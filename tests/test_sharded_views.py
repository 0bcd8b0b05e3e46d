"""Read-only views of a sharded map: the mesh and the PNG export values, the single-cell queries, the wind-field
boundary built from the terrain and the wind batch coupled to that lattice.  Each is compared byte for byte with
one unsharded context that ran the same batches.  The shapes are those of test_gpu_parity's sharded-map test;
the 4-rank one has a last strip narrower than the others (48, 48, 48, 16 columns)."""
import os
import subprocess
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

SHAPES = [(2, "rocksand", 128, 96, 900, 500),
          (3, "rockgravelpebblessand", 144, 80, 900, 700),
          (4, "default", 160, 64, 600, 300)]
SEED = 17


def _same(a, b, what):
    a = np.ascontiguousarray(a); b = np.ascontiguousarray(b)
    assert a.shape == b.shape, (what, a.shape, b.shape)
    if not np.array_equal(a.view(np.uint8), b.view(np.uint8)):
        bad = np.nonzero(a.reshape(-1) != b.reshape(-1))[0]
        raise AssertionError("%s differs at %d entries, first %s: %r vs %r" %
                             (what, len(bad), bad[:4], a.reshape(-1)[bad[:4]], b.reshape(-1)[bad[:4]]))


def _pair(nranks, soil, dimx, dimy, nw, nd):
    """a sharded map and an unsharded context on the same terrain, after the same water and wind batch"""
    from soilmachine_b200 import capi, host, presets, sharded
    pre = presets.load(soil)
    scale = pre["world"]["scale"]
    sh = sharded.VirtualShards(nranks, dimx, dimy, scale, max_particles=4096)
    one = capi.Context(dimx, dimy, scale, max_particles=4096)
    for m in (sh, one):
        m.set_soils(pre["soils"])
        m.set_soil_colors(pre["colors"])
        m.initialize(SEED, pre["layers"])
    host.srand(SEED)
    xw, xd = host.spawn_list(nw, dimx, dimy), host.spawn_list(nd, dimx, dimy)
    a, b = sh.water_run(xw), one.water_run(xw)
    assert (a.steps, a.sweeps, a.exit_oob, a.exit_evap, a.exit_stall) == \
        (b.steps, b.sweeps, b.exit_oob, b.exit_evap, b.exit_stall)
    a, b = sh.wind_run(xd), one.wind_run(xd)
    assert (a.steps, a.exit_oob) == (b.steps, b.exit_oob)
    sh.frequency_update(); one.frequency_update()
    _same(sh.heights(), one.heights(), "heights after the batches")
    return sh, one


def _edge_columns(sh):
    """the columns x0 - 1, x0, x0 + 1 at every strip edge"""
    xs = set()
    for x0, _ in sh.ranges[1:]:
        xs.update((x0 - 1, x0, x0 + 1))
    return sorted(xs)


@pytest.mark.parametrize("nranks,soil,dimx,dimy,nw,nd", SHAPES)
def test_sharded_mesh_and_export_match_one_context(nranks, soil, dimx, dimy, nw, nd):
    sh, one = _pair(nranks, soil, dimx, dimy, nw, nd)
    try:
        for slice_ in (160, 45):
            _same(sh.mesh_update(slice_), one.mesh_update(slice_), "mesh vertices, slice %d" % slice_)
            _same(sh.export_height(), one.export_height(), "exportheight values, slice %d" % slice_)
            _same(sh.export_color(), one.export_color(), "exportcolor values, slice %d" % slice_)
        # the device buffer of each rank holds its strip only
        for c, (x0, x1) in zip(sh.ctx, sh.ranges):
            assert c.mesh_update(160).shape == ((x1 - x0) * dimy, 11)
    finally:
        sh.close(); one.close()


@pytest.mark.parametrize("nranks,soil,dimx,dimy,nw,nd", SHAPES)
def test_sharded_cell_queries_match_one_context(nranks, soil, dimx, dimy, nw, nd):
    sh, one = _pair(nranks, soil, dimx, dimy, nw, nd)
    try:
        cells = [(x, y) for x in _edge_columns(sh) for y in range(dimy)]
        rng = np.random.RandomState(SEED)
        cells += list(zip(rng.randint(0, dimx, 200).tolist(), rng.randint(0, dimy, 200).tolist()))
        # bilinear points whose four cells straddle a strip edge
        points = [(np.float32(x0 - 1 + fx), np.float32(fy + y))
                  for x0, _ in sh.ranges[1:] for fx in (0.0, 0.25, 0.5, 0.875) for fy in (0.0, 0.375)
                  for y in range(0, dimy - 1, 7)]
        want_q = [one.cell_query(x, y) for x, y in cells]
        want_c = [one.cell_column(x, y) for x, y in cells]
        want_b = [one.height_bilinear(x, y) for x, y in points]
        for rank in range(nranks):
            for (x, y), w, wc in zip(cells, want_q, want_c):
                h, s, n = sh.cell_query(x, y, rank=rank)
                what = "rank %d cell (%d, %d)" % (rank, x, y)
                _same(np.float64(h), np.float64(w[0]), what + " height")
                assert s == w[1], what + " surface"
                _same(n, w[2], what + " normal")
                col = sh.cell_column(x, y, rank=rank)
                assert col["n"] == wc["n"], what + " column length"
                for k in ("type", "size", "floor", "saturation"):
                    _same(col[k], wc[k], what + " column " + k)
            got_b = [sh.height_bilinear(x, y, rank=rank) for x, y in points]
            _same(np.array(got_b), np.array(want_b), "rank %d bilinear heights" % rank)
    finally:
        sh.close(); one.close()


def _lattice_equal(sh, one, what):
    want = one.lbm_get()
    for rank in range(sh.nranks):
        got = sh.lbm_get(rank)
        for k in ("f", "rho", "v"):
            _same(got[k], want[k], "%s: rank %d lattice %s" % (what, rank, k))


@pytest.mark.parametrize("nranks,soil,dimx,dimy,nw,nd", SHAPES)
def test_sharded_lattice_and_coupled_wind_batch_match_one_context(nranks, soil, dimx, dimy, nw, nd):
    """The boundary from the terrain of the whole map on every rank, 25 lattice steps, then a wind batch coupled to
    the lattice.  Every rank keeps the whole lattice, and the coupled sweep reads it locally."""
    from soilmachine_b200 import host
    sh, one = _pair(nranks, soil, dimx, dimy, nw, nd)
    try:
        assert dimx % 27 != 0
        dims_list = [(27, 12, 22), (32, 20, 32)]       # the last one is coupled to the wind batch
        for dims in dims_list:
            for m in (sh, one):
                m.lbm_create(*dims)
                m.lbm_set_boundary(None)
                m.lbm_step(25)
            _lattice_equal(sh, one, "lattice %s" % (dims,))
        sh.wind_use_lbm(True); one.wind_use_lbm(True)
        host.srand(SEED + 1)
        xy = host.spawn_list(600, dimx, dimy)
        # some particles circle in the lee of the terrain and never leave: cut both runs after a fixed sweep count
        a, b = sh.wind_run(xy, max_sweeps=3000), one.wind_run(xy, max_sweeps=3000)
        assert (a.steps, a.sweeps, a.exit_oob, a.alive) == (b.steps, b.sweeps, b.exit_oob, b.alive)
        _particles_equal(sh, one, len(xy))
        c1, c2 = one.download_columns(), sh.download_columns()
        for k in c1:
            _same(c2[k], c1[k], "columns." + k)
        assert sum(c.checksum() for c in sh.ctx) % (1 << 64) == one.checksum()
        _same(sh.frequency()["wind_frequency"], one.frequency()["wind_frequency"], "wind frequency map")
    finally:
        sh.wind_use_lbm(False); one.wind_use_lbm(False)
        sh.close(); one.close()


def _particles_equal(sh, one, n):
    """A live particle is held by exactly one rank (alive there).  A dead one was written last by the rank that ran
    its final step; the other ranks keep earlier copies, so one of the copies must be the unsharded final state."""
    want = one.wind_state()
    got = [c.wind_state() for c in sh.ctx]
    keys = ("pos", "speed", "height", "sediment", "contains")

    def row(st, i):
        return b"".join(np.ascontiguousarray(st[k][i]).tobytes() for k in keys)

    for i in range(n):
        holders = [r for r in range(sh.nranks) if got[r]["alive"][i]]
        if want["alive"][i]:
            assert len(holders) == 1, "particle %d: live on ranks %s" % (i, holders)
            assert row(got[holders[0]], i) == row(want, i), "particle %d: live state" % i
        else:
            assert not holders, "particle %d: dead in one context, live on ranks %s" % (i, holders)
            assert any(row(g, i) == row(want, i) for g in got), "particle %d: final state" % i


@pytest.mark.parametrize("nranks,soil,dimx,dimy,nw,nd", SHAPES[:1])
def test_sharded_context_still_refuses_the_writing_calls(nranks, soil, dimx, dimy, nw, nd):
    from soilmachine_b200 import capi
    sh, one = _pair(nranks, soil, dimx, dimy, nw, nd)
    try:
        c = sh.ctx[0]
        for call, msg in ((lambda: c.cell_add(3, 3, 0.5, 1), "single-cell operations are not available"),
                          (c.water_flood, "pooling hydrology is not available"),
                          (c.seep, "pooling hydrology is not available")):
            with pytest.raises(capi.SoilMachineError) as e:
                call()
            assert e.value.code == capi.SM_ERR_INVALID and msg in str(e.value), str(e.value)
    finally:
        sh.close(); one.close()


def test_views_over_cuda_ipc_two_processes_one_gpu():
    """tests/multigpu_views_check.py with two processes sharing this GPU: the peers' strips are CUDA-IPC mappings,
    as across GPUs.  Mesh, exports, edge queries and the boundary-built lattice must equal one unsharded context."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ, SM_ONE_GPU="1")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2",
           "--master-addr", "127.0.0.1", "--master-port", "29623",
           os.path.join(root, "tests", "multigpu_views_check.py"), "96", "300", "rocksand"]
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=900, cwd=root, env=env)
    line = [l for l in out.stdout.splitlines() if l.startswith("multigpu_views_check")]
    assert out.returncode == 0 and line and "DIFFER" not in line[0], (out.stdout[-2000:], out.stderr[-2000:])
