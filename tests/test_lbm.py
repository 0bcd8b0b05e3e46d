"""The wind field (D3Q19 lattice Boltzmann, SURVEY.md section 8f row 4).

CPU: properties of the oracle restatement (oracle/lbm_oracle.c) that do not depend on upstream's GLSL rounding -
the equilibrium's moments, mass/momentum conservation of the TRT collision, the driven faces, obstacles.
GPU: the fused collide+stream kernel (soilmachine_b200/csrc/sm_lbm.cuh) against that restatement, value for
value.  Parity with the reference itself is UNPINNED: its shaders need OpenGL and it ships no vectors for them."""
import numpy as np
import pytest

C19 = np.array([[0, 0, 0], [1, 0, 0], [-1, 0, 0], [0, 1, 0], [0, -1, 0], [0, 0, 1], [0, 0, -1], [1, 1, 0], [-1, -1, 0],
                [1, 0, 1], [-1, 0, -1], [0, 1, 1], [0, -1, -1], [1, -1, 0], [-1, 1, 0], [1, 0, -1], [-1, 0, 1],
                [0, 1, -1], [0, -1, 1]], np.float64)
FORCE = 0.05 * np.array([-2.0, 0.0, 1.0])


def test_oracle_initial_state_is_the_forcing_equilibrium():
    from oracle import lbmapi
    o = lbmapi.Lbm(8, 6, 8)
    s = o.get()
    assert np.allclose(s["rho"], 1.0, atol=1e-6)
    assert np.allclose(s["v"][:, :3], FORCE[None, :], atol=1e-6)
    mom = s["f"].astype(np.float64) @ C19
    assert np.allclose(mom, FORCE[None, :], atol=1e-6)


def test_oracle_collision_conserves_mass_and_uniform_flow_is_stationary():
    """Without obstacles the initial state is the fixed point of collide + stream + driving: every interior cell
    keeps density 1 and the forcing velocity (up to the small gravity term collide.cs:21 adds to v.y)."""
    from oracle import lbmapi
    o = lbmapi.Lbm(10, 8, 10)
    o.step(5)
    s = o.get()
    rho = s["rho"].reshape(10, 8, 10)
    assert np.allclose(rho[1:-1, 1:-1, 1:-1], 1.0, atol=2e-3)
    v = s["v"].reshape(10, 8, 10, 4)[2:-2, 2:-2, 2:-2, :3]
    assert np.allclose(v[..., 0], FORCE[0], atol=5e-3) and np.allclose(v[..., 2], FORCE[2], atol=5e-3)


def test_oracle_obstacle_cells_hold_the_rest_equilibrium_and_deflect_the_flow():
    from oracle import lbmapi
    nx, ny, nz = 16, 10, 16
    o = lbmapi.Lbm(nx, ny, nz)
    b = np.zeros((nx, ny, nz), np.float32)
    b[6:10, 0:5, 6:10] = 1.0
    o.set_boundary(b)
    o.step(20)
    s = o.get()
    v = s["v"].reshape(nx, ny, nz, 4)
    speed = np.linalg.norm(v[..., :3], axis=-1)
    free = speed[2:5, 6, 2:5].mean()
    wake = speed[5:11, 1:4, 5:11][b[5:11, 1:4, 5:11] == 0].mean()
    assert wake < 0.8 * free              # the flow slows down around the block
    assert np.isfinite(s["f"]).all() and (s["f"] > 0).all()


@pytest.mark.gpu
@pytest.mark.parametrize("nx,ny,nz,steps,block", [(64, 40, 64, 12, True), (32, 8, 32, 7, False), (20, 5, 12, 9, True)])
def test_gpu_lbm_matches_oracle(nx, ny, nz, steps, block):
    """lbmwind.h's own size (64 x 40 x 64) and two odd ones; obstacles from a block of cells.  Populations, density
    and velocity after every few steps must equal the restatement value for value (the only tolerated difference is
    the sign of an exact zero, sm_lbm.cuh explains why)."""
    import soilmachine_b200 as smb
    from oracle import lbmapi
    ctx = smb.Context(64, 64, 80, max_particles=16)
    ctx.lbm_create(nx, ny, nz)
    o = lbmapi.Lbm(nx, ny, nz)
    for k in ("f", "rho", "v"):
        assert np.array_equal(ctx.lbm_get()[k], o.get()[k]), "initial " + k
    if block:
        b = np.zeros((nx, ny, nz), np.float32)
        b[nx // 3:nx // 2, 0:ny // 2, nz // 4:nz // 2] = 1.0
        b[0:3, 0:2, :] = 1.0                                  # obstacle cells on a driven face
        ctx.lbm_set_boundary(b); o.set_boundary(b)
    done = 0
    for chunk in (1, 2, steps - 3):
        ctx.lbm_step(chunk); o.step(chunk); done += chunk
        g, r = ctx.lbm_get(), o.get()
        for k in ("f", "rho", "v"):
            assert np.array_equal(g[k], r[k]), "%s after %d steps: %d entries differ" % (k, done, (g[k] != r[k]).sum())
    rng = np.random.RandomState(1)
    pos = (rng.rand(500, 4) * np.array([nx - 2, ny - 2, nz - 2, 0]) + np.array([0.5, 0.5, 0.5, 1.0])).astype(np.float32)
    assert np.array_equal(ctx.lbm_advect(pos), o.advect(pos))
    ctx.close()


@pytest.mark.gpu
def test_gpu_lbm_boundary_from_terrain(ref):
    """SoilMachine.cpp:234-239: a lattice cell is an obstacle where the terrain is higher than the cell."""
    import soilmachine_b200 as smb
    dim = 128
    ref.init("rocksand", seed=42, dimx=dim, dimy=dim, poolsize=dim * dim * 4 + 1000000)
    ctx = smb.Context(dim, dim, ref.scale, max_particles=16)
    ctx.set_soils(ref.soils())
    cols = ref.columns()
    ctx.upload_columns(cols["offsets"], cols["type"], cols["size"], cols["saturation"])
    nx, ny, nz = 64, 40, 64
    ctx.lbm_create(nx, ny, nz)
    ctx.lbm_set_boundary(None)
    ctx.lbm_step(1)
    h = ref.heights().reshape(dim, dim)
    sx, sy, sz = np.float32(dim) / np.float32(nx), np.float32(ref.scale) / np.float32(32), np.float32(dim) / np.float32(nz)
    want = np.zeros((nx, ny, nz), bool)
    for x in range(nx):
        for z in range(nz):
            hh = h[int(sx * np.float32(x)), int(sz * np.float32(z))]
            for y in range(ny):
                want[x, y, z] = hh > float((sy * np.float32(y)) / np.float32(ref.scale))
    # obstacle cells come out of the collision at the rest equilibrium: density exactly that of eq(rest) summed
    g = ctx.lbm_get()
    assert want.any() and not want.all()
    # after one step a solid cell that is not on a driven face still holds what its neighbours pushed into it; the
    # flag itself is what we check, through a second context-free path: re-derive it from the velocity written by
    # collide (solid cells keep collide's macroscopic values, fluid ones too) - so compare via the oracle instead
    from oracle import lbmapi
    o = lbmapi.Lbm(nx, ny, nz)
    o.set_boundary(want.astype(np.float32))
    o.step(1)
    r = o.get()
    for k in ("f", "rho", "v"):
        assert np.array_equal(g[k], r[k]), k
    ctx.close()


def _field_with_obstacle(nx, ny, nz, steps=15):
    from oracle import lbmapi
    o = lbmapi.Lbm(nx, ny, nz)
    b = np.zeros((nx, ny, nz), np.float32)
    b[nx // 3:nx // 2, 0:ny // 2, nz // 4:3 * nz // 4] = 1.0
    o.set_boundary(b)
    o.step(steps)
    return o.get()["v"]


def test_wind_particles_follow_the_lattice_field_cpu():
    """EXTENSION (off by default): WindParticle's prevailing wind sampled from the lattice Boltzmann velocity.  The
    product's step (host build of sm_coop.cuh) against the oracle port's restatement of the same rule, bit for bit;
    and without a field the constant of wind.h:29 - the golden frames - is untouched."""
    import _golden
    import _hostsim
    from oracle import portapi
    g = _golden.load("frame_rocksand_56")
    dims = (16, 10, 16)
    v4 = _field_with_obstacle(*dims)
    hs = _hostsim.HostSim()
    hs.init(int(g["dimx"]), int(g["dimy"]), int(g["scale"]), g["soils"])
    hs.set_columns(_golden.cols(g, "init"))
    hs.lib.hs_set_mode(1, 0)
    po = portapi.Port().init(int(g["dimx"]), int(g["dimy"]), int(g["scale"]), g["soils"])
    po.set_columns(_golden.cols(g, "init"))
    try:
        hs.set_wind_field(v4, dims); po.set_wind_field(v4, dims)
        xy = g["wind_xy"]
        po.wind_run(xy)
        st = _hostsim.Stats()
        hs.wind_begin(xy)
        while hs.wind_sweep(st):
            pass
        a, b = hs.wind_state(), po.wind_state()
        for k in a:
            _golden.same(a[k], b[k], "wind state " + k)
        _golden.same_cols(hs.columns(), po.columns(), "columns")
        assert not np.array_equal(a["pos"], g["wind_state_pos"])     # the field does change the trajectories
    finally:
        hs.set_wind_field(None); po.set_wind_field(None)
        hs.lib.hs_set_mode(0, 0)


@pytest.mark.gpu
def test_gpu_wind_particles_follow_the_lattice_field(ref):
    """the coupled wind batch on the device (field = this context's own lattice after some steps around the terrain)
    against the oracle port fed with the downloaded velocity field"""
    import soilmachine_b200 as smb
    from oracle import portapi
    dim, n = 128, 600
    ref.init("rocksand", seed=42, dimx=dim, dimy=dim, poolsize=dim * dim * 4 + 1000000)
    cols = ref.columns()
    ctx = smb.Context(dim, dim, ref.scale, max_particles=4096)
    ctx.set_soils(ref.soils())
    ctx.upload_columns(cols["offsets"], cols["type"], cols["size"], cols["saturation"])
    dims = (32, 20, 32)
    ctx.lbm_create(*dims)
    ctx.lbm_set_boundary(None)
    ctx.lbm_step(25)
    ctx.wind_use_lbm(True)
    v4 = ctx.lbm_get()["v"]
    po = portapi.Port().init(dim, dim, ref.scale, ref.soils())
    po.set_columns(cols)
    po.set_wind_field(v4, dims)
    xy = ref.spawn_list(n, seed=9)
    # some particles never leave this field (they circle in the lee of the terrain), so the batch is cut after a
    # fixed number of sweeps on both sides; the particles still alive then are compared like the others
    sweeps = 3000
    r, g = po.wind_run(xy, max_sweeps=sweeps), ctx.wind_run(xy, max_sweeps=sweeps)
    po.set_wind_field(None)
    assert (g.steps, g.sweeps, g.exit_oob) == (r.steps, r.sweeps, r.exit_oob) and g.steps > 0
    a, b = ctx.wind_state(), po.wind_state()
    for k in b:
        assert np.array_equal(np.ascontiguousarray(a[k]).view(np.uint8), np.ascontiguousarray(b[k]).view(np.uint8)), k
    c1, c2 = po.columns(), ctx.download_columns()
    for k in ("offsets", "type", "size", "floor", "saturation"):
        assert np.array_equal(c1[k], c2[k]), k
    ctx.wind_use_lbm(False)
    ctx.close()
