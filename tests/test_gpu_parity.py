"""GPU parity: the CUDA hot path through the C ABI vs the reference's own functions driven in
lockstep (oracle/_ref).  Bit-exact on every per-cell quantity (heights, every section of every
column, frequency/track maps), on every particle's state and on the exit counters."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _setup(ref, soil, dim, seed=42):
    import soilmachine_b200 as smb
    ref.init(soil, seed=seed, dimx=dim, dimy=dim, poolsize=dim * dim * 4 + 2000000)
    ctx = smb.Context(ref.dimx, ref.dimy, ref.scale, max_particles=65536)
    ctx.set_soils(ref.soils())
    cols = ref.columns()
    ctx.upload_columns(cols["offsets"], cols["type"], cols["size"], cols["saturation"])
    return ctx, cols


def _same(a, b, what):
    a = np.ascontiguousarray(a); b = np.ascontiguousarray(b)
    assert a.shape == b.shape, what
    if not np.array_equal(a.view(np.uint8), b.view(np.uint8)):
        bad = np.nonzero(a.reshape(-1) != b.reshape(-1))[0]
        raise AssertionError("%s differs at %d entries, first %s: %r vs %r" %
                             (what, len(bad), bad[:4], a.reshape(-1)[bad[:4]], b.reshape(-1)[bad[:4]]))


def _compare_maps(ref, ctx):
    _same(ref.heights(), ctx.heights(), "height")
    c1, c2 = ref.columns(), ctx.download_columns()
    for k in ("offsets", "type", "size", "floor", "saturation"):
        _same(c1[k], c2[k], "columns." + k)
    f1, f2 = ref.frequency(), ctx.frequency()
    for k in f1:
        _same(f1[k], f2[k], k)


def test_upload_download_roundtrip(ref):
    ctx, cols = _setup(ref, "rockgravelpebblessand", 64)
    got = ctx.download_columns()
    for k in ("offsets", "type", "size", "floor", "saturation"):
        _same(cols[k], got[k], k)
    _same(ref.heights(), ctx.heights(), "height")
    _same(ref.surfaces(), ctx.surfaces(), "surface")
    assert abs(ctx.height_sum() - ref.heights().sum()) < 1e-6


@pytest.mark.parametrize("soil,dim,n", [("default", 64, 64), ("rocksand", 96, 256)])
def test_water_stepwise(ref, soil, dim, n):
    ctx, _ = _setup(ref, soil, dim)
    xy = ref.spawn_list(n, seed=7)
    ref.water_begin(xy); ctx.water_begin(xy)
    for k in ("pos", "speed", "volume", "sediment", "contains", "alive"):
        _same(ref.water_state()[k], ctx.water_state()[k], "spawn." + k)
    for sweep in range(40):
        alive, _ = ref.water_sweep()
        st = ctx.water_sweeps(1)
        s1, s2 = ref.water_state(), ctx.water_state()
        for k in s1:
            _same(s1[k], s2[k], "sweep %d %s" % (sweep, k))
        assert st.alive == alive
    _compare_maps(ref, ctx)


@pytest.mark.parametrize("soil,dim,n", [
    ("default", 256, 1000), ("rocksand", 256, 2000), ("rockgravelpebblessand", 256, 2000),
    ("bigbutte", 256, 2000), ("rockgravelpebbles_big", 192, 1500)])
def test_water_run(ref, soil, dim, n):
    ctx, _ = _setup(ref, soil, dim)
    xy = ref.spawn_list(n, seed=42)
    r = ref.water_run(xy)
    g = ctx.water_run(xy)
    assert (g.steps, g.sweeps, g.exit_oob, g.exit_evap, g.exit_stall) == \
        (r.steps, r.sweeps, r.exit_oob, r.exit_evap, r.exit_stall)
    assert g.alive == 0 and g.pool_drops == 0
    _compare_maps(ref, ctx)
    s1, s2 = ref.water_state(), ctx.water_state()
    for k in s1:
        _same(s1[k], s2[k], "final " + k)


@pytest.mark.parametrize("soil,dim,n", [("rocksand", 256, 1000), ("rockgravelpebblessand", 256, 1500)])
def test_wind_run(ref, soil, dim, n):
    ctx, _ = _setup(ref, soil, dim)
    xy = ref.spawn_list(n, seed=43)
    r = ref.wind_run(xy)
    g = ctx.wind_run(xy)
    assert (g.steps, g.exit_oob) == (r.steps, r.exit_oob)
    _compare_maps(ref, ctx)
    s1, s2 = ref.wind_state(), ctx.wind_state()
    for k in s1:
        _same(s1[k], s2[k], "final " + k)


def test_frame_sequence(ref):
    """water batch, wind batch, frequency update - three frames (SoilMachine.cpp:287-320 without
    flood/seep)."""
    ctx, _ = _setup(ref, "rocksand", 192)
    ref.lib.smref_srand(99)
    for frame in range(3):
        xw = ref.spawn_list(600); xd = ref.spawn_list(300)
        ref.water_run(xw); ctx.water_run(xw)
        ref.wind_run(xd); ctx.wind_run(xd)
        ref.frequency_update(); ctx.frequency_update()
        _compare_maps(ref, ctx)


def test_determinism(ref):
    ctx, cols = _setup(ref, "rockgravelpebblessand", 128)
    xy = ref.spawn_list(1500, seed=5)
    ctx.water_run(xy)
    h1 = ctx.heights().copy()
    ctx.upload_columns(cols["offsets"], cols["type"], cols["size"], cols["saturation"])
    ctx.set_frequency(np.zeros(ctx.cells, np.float32), np.zeros(ctx.cells, np.float32),
                      np.zeros(ctx.cells, np.float32))
    ctx.water_run(xy)
    _same(h1, ctx.heights(), "height (run twice)")


@pytest.mark.parametrize("soil,dim,seed", [("rockgravelpebblessand", 160, 42), ("bigbutte", 128, 7),
                                           ("default", 100, 12345)])
def test_initialize_matches_reference_terrain(ref, soil, dim, seed):
    """sm_initialize (CUDA OpenSimplex2/FBm) == Layermap::initialize (layermap.h:163-216)."""
    import soilmachine_b200 as smb
    ref.init(soil, seed=seed, dimx=dim, dimy=dim + 16)
    ctx = smb.Context(ref.dimx, ref.dimy, ref.scale)
    ctx.set_soils(ref.soils())
    ctx.initialize(seed, ref.layers())
    c1, c2 = ref.columns(), ctx.download_columns()
    for k in c1:
        _same(c1[k], c2[k], "init columns." + k)


def test_presets_match_reference_loader():
    import _golden
    from soilmachine_b200 import presets
    g = _golden.load("ref_loader")
    for name in presets.names():
        pre = presets.load(name)
        rs, rl = g[name + "/soils"], g[name + "/layers"]
        assert len(rs) == len(pre["soils"]) and len(rl) == len(pre["layers"])
        for k in pre["soils"].dtype.names:
            _same(rs[k], pre["soils"][k], name + ".soils." + k)
        for k in pre["layers"].dtype.names:
            _same(rl[k], pre["layers"][k], name + ".layers." + k)
        assert int(g[name + "/scale"]) == pre["world"]["scale"]


def test_smoke_entry():
    import __graft_entry__ as g
    g.smoke()


@pytest.mark.parametrize("case", ["frame_default_48", "frame_rocksand_56", "frame_rgps_64", "frame_bigbutte_40"])
def test_gpu_replays_golden_frame(case):
    """The committed golden vectors (generated from the reference by tests/golden/make_golden.py)
    replayed through the C ABI - independent of oracle/_ref being present on the box."""
    import _golden
    import soilmachine_b200 as smb
    g = _golden.load(case)
    ctx = smb.Context(int(g["dimx"]), int(g["dimy"]), int(g["scale"]), max_particles=4096)
    ctx.set_soils(g["soils"])
    ctx.initialize(int(g["seed"]), g["layers"])
    _golden.same_cols(ctx.download_columns(), _golden.cols(g, "init"), "initial terrain")
    _golden.replay_frame(g, ctx, lambda st: (st.steps, st.sweeps, st.exit_oob, st.exit_evap, st.exit_stall))


def test_gpu_column_ops_truth_table():
    import _golden
    import soilmachine_b200 as smb
    g = _golden.load("column_ops")
    ctx = smb.Context(8, 8, int(g["scale"]))
    ctx.set_soils(g["soils"])
    for (kind, x, y, v, t), want in zip(g["ops"], g["remove_results"]):
        if kind == 0:
            ctx.cell_add(int(x), int(y), float(v), int(t))
        else:
            got = ctx.cell_remove(int(x), int(y), float(v))
            assert np.float64(got).tobytes() == np.float64(want).tobytes()
    _golden.same_cols(ctx.download_columns(), _golden.cols(g, "final"), "columns after add/remove")
    q = [ctx.cell_query(x, y) for x in range(8) for y in range(8)]
    _golden.same(np.array([a[2] for a in q], np.float32), g["normals"], "normals")
    _golden.same(np.array([a[0] for a in q]).reshape(8, 8), g["heights"], "heights")
    bil = np.array([ctx.height_bilinear(float(p[0]), float(p[1])) for p in g["bilinear_pts"]])
    _golden.same(bil, g["bilinear"], "bilinear heights")
    for x, y, loop in g["cascades"]:
        ctx.cell_cascade(float(x), float(y), int(loop))
    _golden.same_cols(ctx.download_columns(), _golden.cols(g, "after_cascade"), "columns after cascades")


def test_gpu_edge_cases():
    """empty batch, all-empty map, batch larger than one thread per particle, pool exhaustion report."""
    import soilmachine_b200 as smb
    from soilmachine_b200 import presets
    pre = presets.load("rocksand")
    ctx = smb.Context(32, 32, 80, max_particles=70000)
    ctx.set_soils(pre["soils"])
    st = ctx.water_run(np.zeros((0, 2), np.float32))
    assert (st.steps, st.sweeps) == (0, 0)
    xy = np.array([[0, 0], [31, 31], [5, 9]], np.float32)
    st = ctx.water_run(xy)                       # empty map: nothing moves, nothing is created
    assert st.steps == 0 and ctx.section_count() == 0
    with pytest.raises(smb.SoilMachineError):
        ctx.water_run(np.zeros((70001, 2), np.float32))   # larger than max_particles


def test_pool_exhaustion_is_counted_reported_and_not_sticky():
    """layermap.h:92-95: when the section pool runs dry upstream prints, drops the section and keeps running.
    Here the drops are counted per call and reported as a warning (SM_ERR_POOL from the C ABI); a pool too small
    for the terrain itself is an error; a later call that drops nothing is clean again."""
    import warnings
    import soilmachine_b200 as smb
    from soilmachine_b200 import presets
    pre = presets.load("rocksand")               # soil 1 = Rock, soil 2 = Red Sand
    dim = 64
    cells = dim * dim
    # a chequerboard: bare rock next to rock under a thin sand cover -> sand picked up on one cell lands as a NEW
    # section on the next one, and every new section needs a pool slot
    x, y = np.meshgrid(np.arange(dim), np.arange(dim), indexing="ij")
    sandy = ((x + y) % 2 == 0).reshape(-1)
    tilt = (0.2 + 0.6 * x / dim + 0.1 * y / dim).reshape(-1)
    counts = np.where(sandy, 2, 1)
    offsets = np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)
    typ = np.ones(offsets[-1], np.int32); size = np.zeros(offsets[-1])
    size[offsets[:-1]] = tilt
    typ[offsets[:-1][sandy] + 1] = 2; size[offsets[:-1][sandy] + 1] = 0.02
    need = int(sandy.sum())                      # buried sections of the initial terrain
    with pytest.raises(smb.SoilMachineError) as e:
        small = smb.Context(dim, dim, 80, max_particles=4096, pool_capacity=need - 1)
        small.set_soils(pre["soils"])
        small.upload_columns(offsets, typ, size)
    assert e.value.code == smb.capi.SM_ERR_POOL
    ctx = smb.Context(dim, dim, 80, max_particles=4096, pool_capacity=need + 3)
    ctx.set_soils(pre["soils"])
    ctx.upload_columns(offsets, typ, size)
    rng = np.random.RandomState(0)
    xy = (rng.rand(2000, 2) * (dim - 2) + 0.5).astype(np.float32)
    with warnings.catch_warnings(record=True) as wlist:
        warnings.simplefilter("always")
        st = ctx.water_run(xy)
    assert st.pool_drops > 0 and any("pool" in str(w.message) for w in wlist)
    with warnings.catch_warnings():
        warnings.simplefilter("error")           # a call that drops nothing must not warn: the status is per call
        st2 = ctx.water_run(np.zeros((0, 2), np.float32))
        assert st2.pool_drops == 0
        h = ctx.heights()
    assert np.isfinite(h).all()
    ctx.close()


def test_cpp_facade_frame_loop_runs():
    import os, subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    exe = os.path.join(root, "tests", "hostsim", "facade_demo")
    libdir = os.path.join(root, "soilmachine_b200", "lib")
    subprocess.check_call(["g++", "-std=c++17", "-O1", os.path.join(root, "tests", "facade_demo.cpp"), "-o", exe,
                           "-L" + libdir, "-lsoilmachine_b200", "-Wl,-rpath," + libdir])
    out = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stdout + out.stderr
    assert "frame 1:" in out.stdout and "legacy ops ok" in out.stdout
    # the same loop with the tables coming from loadsoil() on a preset file
    from oracle import refapi
    out2 = subprocess.run([exe, refapi.soil_path("rocksand")], capture_output=True, text=True, timeout=300)
    assert out2.returncode == 0, out2.stdout + out2.stderr
    assert "frame 1:" in out2.stdout


def test_batch_larger_than_resident_threads(ref):
    """more particles than thread slots: every thread carries several particles per sweep (the
    config-5 regime, 200k particles)."""
    import soilmachine_b200 as smb
    ref.init("rocksand", seed=3, dimx=512, dimy=512, poolsize=512 * 512 * 4 + 2000000)
    ctx = smb.Context(ref.dimx, ref.dimy, ref.scale, max_particles=80000)
    ctx.set_soils(ref.soils())
    cols = ref.columns()
    ctx.upload_columns(cols["offsets"], cols["type"], cols["size"], cols["saturation"])
    xy = ref.spawn_list(70000, seed=3)
    r = ref.water_run(xy, max_sweeps=12)
    g = ctx.water_run(xy, max_sweeps=12)
    assert (g.steps, g.sweeps, g.alive) == (r.steps, r.sweeps, int(ref.water_state()["alive"].sum()))
    _compare_maps(ref, ctx)
    xd = ref.spawn_list(70000, seed=4)
    r = ref.wind_run(xd, max_sweeps=10)
    g = ctx.wind_run(xd, max_sweeps=10)
    assert g.steps == r.steps
    _compare_maps(ref, ctx)


def test_nonsquare_map_and_async_wind(ref, monkeypatch):
    """dimx != dimy (frequency maps are indexed transposed, water.h:53) and the opt-in barrier-free
    wind kernel."""
    import soilmachine_b200 as smb
    monkeypatch.setenv("SM_ASYNC", "1")
    ref.init("rockgravelpebblessand", seed=9, dimx=200, dimy=136)
    ctx = smb.Context(ref.dimx, ref.dimy, ref.scale)
    ctx.set_soils(ref.soils())
    ctx.initialize(9, ref.layers())
    xw = ref.spawn_list(800, seed=9); xd = ref.spawn_list(900)
    r1, g1 = ref.water_run(xw), ctx.water_run(xw)
    r2, g2 = ref.wind_run(xd), ctx.wind_run(xd)
    assert (r1.steps, r2.steps, r2.sweeps) == (g1.steps, g2.steps, g2.sweeps)
    _compare_maps(ref, ctx)


@pytest.mark.parametrize("slice_", [160, 45])
def test_mesh_and_export_match_reference(ref, slice_):
    """Layermap::update(Vertexpool&) (layermap.h:475-555) and the exportheight/exportcolor pixel values
    (io.h:234-252), after a frame, with and without the slice plane cutting the terrain."""
    import soilmachine_b200 as smb
    ref.init("rockgravelpebblessand", seed=21, dimx=96, dimy=80)
    ctx = smb.Context(ref.dimx, ref.dimy, ref.scale)
    ctx.set_soils(ref.soils())
    ctx.set_soil_colors(ref.soils()["color"])
    ctx.initialize(21, ref.layers())
    xw = ref.spawn_list(300, seed=21); xd = ref.spawn_list(200)
    ref.water_run(xw); ctx.water_run(xw)
    ref.wind_run(xd); ctx.wind_run(xd)
    want = ref.mesh(slice_)
    got = ctx.mesh_update(slice_)
    _same(want, got, "mesh vertices")
    h, c = ref.export()
    _same(h, ctx.export_height(), "exportheight values")
    _same(c, ctx.export_color(), "exportcolor values")


def test_config2_full_size_parity_and_statistics(ref):
    """BASELINE config 2 (1024^2 rocksand, 10 000 water): bit parity against the lockstep reference at
    full size, and the sequential reference loop (the order upstream really runs) agrees statistically
    (SURVEY.md App. D: the field is chaotic under reordering, its statistics are not)."""
    import soilmachine_b200 as smb
    dim, n = 1024, 10000
    ref.init("rocksand", seed=42, dimx=dim, dimy=dim, poolsize=dim * dim * 3 + 2000000)
    ctx = smb.Context(dim, dim, ref.scale, max_particles=n)
    ctx.set_soils(ref.soils())
    ctx.initialize(42, ref.layers())
    h0 = ctx.heights().copy()
    _same(ref.heights(), h0, "initial heights")
    xy = ref.spawn_list(n, seed=42)
    r = ref.water_run(xy)
    g = ctx.water_run(xy)
    assert (g.steps, g.sweeps, g.exit_oob, g.exit_evap, g.exit_stall) == \
        (r.steps, r.sweeps, r.exit_oob, r.exit_evap, r.exit_stall)
    h_lock = ctx.heights().copy()
    _same(ref.heights(), h_lock, "heights after the batch")
    # sequential order on a fresh copy of the same terrain, same spawn list
    ref.init("rocksand", seed=42, dimx=dim, dimy=dim, poolsize=dim * dim * 3 + 2000000)
    s = ref.water_seq(0, xy)
    h_seq = ref.heights()
    d_lock, d_seq = h_lock - h0, h_seq - h0
    assert abs(s.steps - g.steps) / g.steps < 0.02                      # same amount of work
    assert abs(d_lock.sum() - d_seq.sum()) < 0.02 * abs(d_seq).sum()    # same net mass change
    assert abs(np.abs(d_lock).sum() - np.abs(d_seq).sum()) < 0.05 * np.abs(d_seq).sum()   # same amount moved
    assert abs(h_lock.mean() - h_seq.mean()) < 1e-6 and abs(h_lock.std() - h_seq.std()) < 1e-5


@pytest.mark.parametrize("soil,dim,nw,nd", [("bigbutte", 4096, 50000, 0), ("rockgravelpebbles_big", 2048, 60000, 2000)])
def test_large_configs_properties(soil, dim, nw, nd):
    """BASELINE configs 4/5 shapes at sizes the oracle cannot replay in seconds: size-independent
    properties - run-twice determinism of the whole field (Σheight and an order-sensitive checksum), no
    pool drops, no reach violations, inert wind on a soil without suspension (wind.h:56-57)."""
    from soilmachine_b200 import host
    sums = []
    for rep in range(2):
        sim = host.Simulation(soil, seed=42, dimx=dim, dimy=dim, max_particles=max(nw, nd, 1))
        host.srand(42)
        xw = host.spawn_list(nw, dim, dim)
        ws = sim.ctx.water_run(xw, max_sweeps=60)
        assert ws.pool_drops == 0 and ws.steps > 0
        ds = None
        if nd:
            ds = sim.ctx.wind_run(host.spawn_list(nd, dim, dim))
            assert ds.steps == 0 and ds.exit_oob == nd      # no soil has SUSPENSION > 0 on this preset
        h = sim.ctx.heights()
        w = (np.arange(h.size, dtype=np.float64) % 1021 + 1.0).reshape(h.shape)
        sums.append((sim.ctx.height_sum(), float((h * w).sum()), ws.steps))
        assert abs(sums[-1][0] - h.sum()) < 1e-6 * abs(h.sum())
        sim.close()
    assert sums[0] == sums[1]


@pytest.mark.parametrize("nranks,soil,dimx,dimy,nw,nd", [(2, "rocksand", 128, 96, 900, 500),
                                                         (3, "rockgravelpebblessand", 144, 80, 900, 700),
                                                         (4, "default", 160, 64, 600, 0)])
def test_sharded_map_is_bit_identical(ref, nranks, soil, dimx, dimy, nw, nd):
    """x-strips on nranks contexts (all on this GPU; the multi-GPU path runs the same kernels with the
    peers mapped over CUDA IPC): halo reads/writes, cross-strip dependency chains, particle hand-over and
    the cross-rank barrier must leave every byte equal to the unsharded lockstep reference."""
    from soilmachine_b200 import sharded
    ref.init(soil, seed=17, dimx=dimx, dimy=dimy)
    sh = sharded.VirtualShards(nranks, ref.dimx, ref.dimy, ref.scale, max_particles=4096)
    sh.set_soils(ref.soils())
    sh.initialize(17, ref.layers())
    c1, c2 = ref.columns(), sh.download_columns()
    for k in c1:
        _same(c1[k], c2[k], "initial " + k)
    xw = ref.spawn_list(nw, seed=17)
    r, g = ref.water_run(xw), sh.water_run(xw)
    assert (g.steps, g.sweeps, g.exit_oob, g.exit_evap, g.exit_stall) == \
        (r.steps, r.sweeps, r.exit_oob, r.exit_evap, r.exit_stall)
    if nd:
        xd = ref.spawn_list(nd)
        r, g = ref.wind_run(xd), sh.wind_run(xd)
        assert (g.steps, g.exit_oob) == (r.steps, r.exit_oob)
    ref.frequency_update(); sh.frequency_update()
    _same(ref.heights(), sh.heights(), "height")
    c1, c2 = ref.columns(), sh.download_columns()
    for k in c1:
        _same(c1[k], c2[k], "columns." + k)
    f1, f2 = ref.frequency(), sh.frequency()
    for k in f1:
        _same(f1[k], f2[k], k)
    sh.close()

@pytest.mark.parametrize("soil,dim,n,frames", [
    ("default", 128, 600, 3), ("rockgravelpebblessand", 160, 1500, 3), ("bigbutte", 128, 800, 3),
    ("rocksand", 192, 1200, 2)])
def test_hydrology_frames(ref, soil, dim, n, frames):
    """The full water part of the frame (SoilMachine.cpp:288-301): lockstep batch, flood() of the finished
    particles in ascending index (water.h:123-145), the full-grid seep pass (water.h:335-343), frequency
    update - against the reference's own flood/cascade/seep functions.  Bit-exact after every phase."""
    ctx, _ = _setup(ref, soil, dim)
    total = {"floods": 0, "transfers": 0}
    for frame in range(frames):
        xy = ref.spawn_list(n, seed=42 + frame)
        ref.water_run(xy); ctx.water_run(xy)
        _compare_maps(ref, ctx)
        nf = ref.water_flood()
        h = ctx.water_flood()
        _compare_maps(ref, ctx)
        assert h.floods >= nf                      # nested particles flood too; the batch's own floods are nf
        ref.seep()
        h2 = ctx.seep()
        _compare_maps(ref, ctx)
        ref.frequency_update(); ctx.frequency_update()
        _compare_maps(ref, ctx)
        total["floods"] += h.floods; total["transfers"] += h.transfers + h2.transfers
    assert total["floods"] > 0 and total["transfers"] > 0     # the case exercises the path


def test_hydrology_counters_match_port(ref):
    """Counters the verbatim reference cannot report (nested particles, their steps, transfers) against the
    oracle port, which is itself pinned to the reference bit for bit (tests/test_oracle_port.py)."""
    from oracle import portapi
    ctx, cols = _setup(ref, "default", 128)
    po = portapi.Port().init(ref.dimx, ref.dimy, ref.scale, ref.soils())
    po.set_columns(cols)
    for frame in range(2):
        xy = ref.spawn_list(600, seed=11 + frame)
        po.water_run(xy); ctx.water_run(xy)
        a, b = po.water_flood(), ctx.water_flood()
        assert (a.floods, a.nested, a.nested_steps, a.transfers) == (b.floods, b.nested, b.nested_steps, b.transfers)
        a, b = po.seep(), ctx.seep()
        assert (a.floods, a.nested, a.nested_steps, a.transfers) == (b.floods, b.nested, b.nested_steps, b.transfers)
        assert b.cells < a.cells                   # the device pass visits only the cells where water is
        po.frequency_update(); ctx.frequency_update()
    c1, c2 = po.columns(), ctx.download_columns()
    for k in ("offsets", "type", "size", "floor", "saturation"):
        _same(c1[k], c2[k], "columns." + k)


def test_hydrology_with_wind_and_uploaded_water(ref):
    """Water already on the map when the columns are uploaded (saturated sections below, Air on top), wind
    batches in between: the seep pass must find every wet cell by itself."""
    ctx, _ = _setup(ref, "rocksand", 128)
    xy = ref.spawn_list(900, seed=5)
    for frame in range(2):                          # make the reference map wet, then upload it afresh
        ref.water_run(xy); ref.water_flood(); ref.seep(); ref.frequency_update()
    cols = ref.columns()
    assert (cols["saturation"] > 0).sum() > 0
    ctx.upload_columns(cols["offsets"], cols["type"], cols["size"], cols["saturation"])
    f = ref.frequency()
    ctx.set_frequency(f["water_frequency"], f["water_track"], f["wind_frequency"])
    xd = ref.spawn_list(400, seed=6)
    ref.wind_run(xd); ctx.wind_run(xd)
    ref.seep(); ctx.seep()
    _compare_maps(ref, ctx)
    ref.water_run(xy); ctx.water_run(xy)
    ref.water_flood(); ctx.water_flood()
    ref.seep(); ctx.seep()
    _compare_maps(ref, ctx)


@pytest.mark.parametrize("case", ["hydro_default_48", "hydro_bigbutte_40"])
def test_gpu_replays_golden_hydrology(case):
    """Committed vectors of the full water part of the frame (batch, floods, seep pass; generated from the
    reference by tests/golden/make_golden.py) through the C ABI - independent of oracle/_ref."""
    import _golden
    import soilmachine_b200 as smb
    g = _golden.load(case)
    ctx = smb.Context(int(g["dimx"]), int(g["dimy"]), int(g["scale"]), max_particles=4096)
    ctx.set_soils(g["soils"])
    c = _golden.cols(g, "init")
    ctx.upload_columns(c["offsets"], c["type"], c["size"], c["saturation"])
    counters = _golden.replay_hydro(g, ctx)
    assert all(h.floods >= f for h, f in zip(counters, g["floods"]))


# ---- BASELINE.json configs at their own sizes -------------------------------------------------------------
def _compare_big(ref, ctx, what):
    """Full-size comparison without downloading 10^7 sections through Python lists: every height and every
    frequency/track entry byte for byte, every section of every column through the position-sensitive checksum
    (device: sm_checksum; reference: the same hash over its columns in numpy)."""
    from soilmachine_b200 import checksum
    _same(ref.heights(), ctx.heights(), what + ": height")
    f1, f2 = ref.frequency(), ctx.frequency()
    for k in f1:
        _same(f1[k], f2[k], what + ": " + k)
    want = checksum.columns_checksum(ref.columns())
    assert ctx.checksum() == want, what + ": column checksum"
    return want


def test_config3_frame_matches_reference(ref):
    """BASELINE.json configs[2] at its own size - 4096^2 rockgravelpebblessand, terrain from sm_initialize, the
    bench's own first-frame spawn lists (srand(42), 25 000 water then 25 000 wind), both batches run to
    completion (~460 water sweeps, ~13 700 wind sweeps), frequency update - against the reference's functions
    driven in lockstep.  The checksum of the final columns is the one bench.py prints after its first frame."""
    import json
    import os
    import soilmachine_b200 as smb
    from soilmachine_b200 import host, presets
    dim, n = 4096, 25000
    pre = presets.load("rockgravelpebblessand")
    ctx = smb.Context(dim, dim, pre["world"]["scale"], max_particles=n)
    ctx.set_soils(pre["soils"])
    ctx.initialize(42, pre["layers"])
    ref.init("rockgravelpebblessand", seed=42, dimx=dim, dimy=dim, poolsize=dim * dim * 2 + 2000000)
    _compare_big(ref, ctx, "terrain")
    host.srand(42)
    xw, xd = host.spawn_list(n, dim, dim), host.spawn_list(n, dim, dim)
    r, g = ref.water_run(xw), ctx.water_run(xw)
    assert (g.steps, g.sweeps, g.exit_oob, g.exit_evap, g.exit_stall, g.pool_drops) == \
        (r.steps, r.sweeps, r.exit_oob, r.exit_evap, r.exit_stall, 0)
    _compare_big(ref, ctx, "after the water batch")
    r, g = ref.wind_run(xd), ctx.wind_run(xd)
    assert (g.steps, g.exit_oob, g.pool_drops) == (r.steps, r.exit_oob, 0)
    assert g.sweeps > 10000
    s1, s2 = ref.wind_state(), ctx.wind_state()
    for k in s1:
        _same(s1[k], s2[k], "wind particles: " + k)
    ref.frequency_update(); ctx.frequency_update()
    cs = _compare_big(ref, ctx, "after the frame")
    gold = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "cfg3_frame1_checksum.json")
    if os.path.exists(gold):
        with open(gold) as f:
            assert int(json.load(f)["checksum"], 16) == cs, "bench.py's golden first-frame checksum is stale"
    else:                         # first run on a GPU box: written to gpurun_out/ so that it can be committed
        out = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "gpurun_out")
        os.makedirs(out, exist_ok=True)
        with open(os.path.join(out, "cfg3_frame1_checksum.json"), "w") as f:
            json.dump({"checksum": "%016x" % cs, "what": "columns after frame 1 of bench.py's config 3 "
                       "(srand(42): 25000 water, 25000 wind, frequency update), equal to oracle/_ref in lockstep"}, f)
    ctx.close()


@pytest.mark.parametrize("soil,dim,nw,nd,sweeps,poolf", [("bigbutte", 4096, 50000, 0, 80, 2.2),
                                                         ("rockgravelpebbles_big", 8192, 100000, 100000, 80, 1.1)])
def test_config4_config5_shapes_match_reference(ref, soil, dim, nw, nd, sweeps, poolf):
    """BASELINE.json configs[3] and [4] at their own sizes (single context): terrain from sm_initialize, the
    frame's spawn lists, the first `sweeps` lockstep sweeps of the water batch (the oracle needs minutes for
    a whole batch at these sizes), then the wind batch of config 5 - inert: no soil of that preset can be
    suspended (wind.h:56-57)."""
    import soilmachine_b200 as smb
    from soilmachine_b200 import host, presets
    pre = presets.load(soil)
    budget = (dim == 8192)        # config 5 carries BASELINE's "mass-conservation check": the budget, vs the oracle port
    ctx = smb.Context(dim, dim, pre["world"]["scale"], max_particles=max(nw, nd), budget=budget)
    ctx.set_soils(pre["soils"])
    ctx.initialize(42, pre["layers"])
    ref.init(soil, seed=42, dimx=dim, dimy=dim, poolsize=int(dim * dim * poolf) + 2000000)   # layers x cells + headroom
    host.srand(42)
    xw = host.spawn_list(nw, dim, dim)
    if budget:
        from oracle import portapi
        po = portapi.Port().init(dim, dim, pre["world"]["scale"], ref.soils())
        po.set_columns(ref.columns())
        hsum0 = ctx.height_sum()
    r, g = ref.water_run(xw, max_sweeps=sweeps), ctx.water_run(xw, max_sweeps=sweeps)
    assert (g.steps, g.sweeps, g.exit_oob, g.exit_evap, g.exit_stall, g.pool_drops) == \
        (r.steps, r.sweeps, r.exit_oob, r.exit_evap, r.exit_stall, 0)
    if budget:
        po.water_run(xw, max_sweeps=sweeps)
        per_p, sums_p = po.budget()
        _same(ctx.budget_particles(nw), per_p, "mass budget per particle")
        b = ctx.last_budget()
        _same(np.array([b.eroded, b.deposited, b.cascade_net, b.discarded, b.clamped, b.wind_negative]), sums_p, "mass budget")
        dh = ctx.height_sum() - hsum0
        assert abs(dh - (b.deposited - b.eroded + b.cascade_net)) < 1e-9 * (b.deposited + b.eroded), (dh, b.asdict())
        assert b.eroded > 0 and b.deposited > 0
        del po
    s1, s2 = ref.water_state(), ctx.water_state()
    for k in s1:
        _same(s1[k], s2[k], "water particles: " + k)
    if nd:
        xd = host.spawn_list(nd, dim, dim)
        r, g = ref.wind_run(xd), ctx.wind_run(xd)
        assert (g.steps, g.exit_oob) == (r.steps, r.exit_oob) == (0, nd)
    _compare_big(ref, ctx, "%s %d^2 after %d sweeps" % (soil, dim, sweeps))
    ctx.close()


def test_ipc_sharded_two_processes_one_gpu():
    """The real multi-process data path on the 1-GPU tier: two processes share this GPU, each owns one x-strip,
    and reach the other's arrays through CUDA-IPC mappings - peer loads/stores of halo records, system-scope
    hand-off words and atomics, the cross-rank barrier, particle hand-over - exactly as two GPUs do over NVLink
    (tests/multigpu_check.py, which also runs on N GPUs).  Must be bit-identical to the unsharded context."""
    import os
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ, SM_ONE_GPU="1")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2",
           "--master-addr", "127.0.0.1", "--master-port", "29617", os.path.join(root, "tests", "multigpu_check.py"),
           "96", "300", "rocksand", "1"]
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=900, cwd=root, env=env)
    line = [l for l in out.stdout.splitlines() if l.startswith("multigpu_check")]
    assert out.returncode == 0 and line and "DIFFER" not in line[0], (out.stdout[-2000:], out.stderr[-2000:])
    logdir = os.path.join(root, "gpurun_out")
    os.makedirs(logdir, exist_ok=True)
    with open(os.path.join(logdir, "ipc_one_gpu.log"), "w") as f:
        f.write(line[0] + "\n")


@pytest.mark.parametrize("soil,dim,nw,nd", [("default", 64, 40, 0), ("rocksand", 64, 24, 16)])
def test_facade_per_particle_loop_matches_reference(ref, soil, dim, nw, nd, tmp_path):
    """tests/facade_loop.cpp = the reference's frame loop with its per-particle calls (construct, `while (move &&
    interact);`, flood, seep pass, wind particles, frequency maps), compiled UNCHANGED against the C++ facade.  Run
    particle by particle it is upstream's own sequential order, so the map must equal the reference's sequential loop
    on the same seed bit for bit - spawn positions included, because the facade consumes the rand() draws upstream's
    nested particle constructors make (water.h:243)."""
    import os
    import struct
    import subprocess
    from oracle import refapi
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    exe = os.path.join(root, "tests", "hostsim", "facade_loop")
    libdir = os.path.join(root, "soilmachine_b200", "lib")
    subprocess.check_call(["g++", "-std=c++17", "-O1", os.path.join(root, "tests", "facade_loop.cpp"), "-o", exe,
                           "-L" + libdir, "-lsoilmachine_b200", "-Wl,-rpath," + libdir])
    outbin = str(tmp_path / "map.bin")
    out = subprocess.run([exe, refapi.soil_path(soil), str(dim), str(nw), str(nd), "1", outbin], capture_output=True,
                         text=True, timeout=600)
    assert out.returncode == 0 and "facade loop ok: 2 mesh uploads of %d vertices" % (dim * dim) in out.stdout, \
        out.stdout + out.stderr
    ref.init(soil, seed=42, dimx=dim, dimy=dim, poolsize=dim * dim * 4 + 1000000)
    ref.lib.smref_srand(42)
    ref.water_seq(nw, flood=True, seep=True)
    if nd:
        ref.wind_seq(nd)
    ref.frequency_update()
    cols, hts = ref.columns(), ref.heights().reshape(-1)
    raw = open(outbin, "rb").read()
    pos = 0
    for c in range(dim * dim):
        (n,) = struct.unpack_from("<i", raw, pos); pos += 4
        lo, hi = int(cols["offsets"][c]), int(cols["offsets"][c + 1])
        assert n == hi - lo, "cell %d: %d sections vs %d" % (c, n, hi - lo)
        for k in range(n):                       # the dump walks top -> bottom
            t, size, floor, sat = struct.unpack_from("<qddd", raw, pos); pos += 32
            j = hi - 1 - k
            assert (t, size, floor, sat) == (int(cols["type"][j]), cols["size"][j], cols["floor"][j], cols["saturation"][j]), \
                "cell %d section %d" % (c, k)
        (h,) = struct.unpack_from("<d", raw, pos); pos += 8
        assert h == hts[c], "cell %d height" % c


@pytest.mark.parametrize("nranks", [1, 3])
def test_mass_budget_matches_port(ref, nranks):
    """SURVEY.md A.7 on the device: the six per-particle accumulators of a water and a wind batch against the oracle
    port (itself pinned to the reference), bit for bit - on one context and on a map sharded into three strips,
    where a particle's sums travel with it - and the identity d(sum of heights) = deposited - eroded + cascade_net."""
    import soilmachine_b200 as smb
    from oracle import portapi
    from soilmachine_b200 import sharded
    soil, dimx, dimy, nw, nd = "rocksand", 192, 128, 1500, 900
    ref.init(soil, seed=42, dimx=dimx, dimy=dimy, poolsize=dimx * dimy * 4 + 1000000)
    cols = ref.columns()
    po = portapi.Port().init(dimx, dimy, ref.scale, ref.soils())
    po.set_columns(cols)
    if nranks == 1:
        ctxs = [smb.Context(dimx, dimy, ref.scale, max_particles=4096, budget=True)]
        ctxs[0].set_soils(ref.soils())
        ctxs[0].upload_columns(cols["offsets"], cols["type"], cols["size"], cols["saturation"])
        run = {"water": ctxs[0].water_run, "wind": ctxs[0].wind_run}
        hsum = lambda: ctxs[0].height_sum()
    else:
        sh = sharded.VirtualShards(nranks, dimx, dimy, ref.scale, max_particles=4096, budget=True)
        sh.set_soils(ref.soils())
        sh.upload_columns(cols)
        ctxs = sh.ctx
        run = {"water": sh.water_run, "wind": sh.wind_run}
        hsum = lambda: float(sh.heights().sum())
    for kind, n, seed in (("water", nw, 3), ("wind", nd, 4)):
        xy = ref.spawn_list(n, seed=seed)
        h0 = hsum()
        (po.water_run if kind == "water" else po.wind_run)(xy)
        run[kind](xy)
        per_p, sums_p = po.budget()
        per_g = sum(c.budget_particles(n) for c in ctxs)       # exactly one strip holds a particle's sums
        _same(per_g, per_p, kind + ": mass budget per particle")
        s = per_g.sum(axis=0)
        assert abs((hsum() - h0) - (s[1] - s[0] + s[2])) < 1e-9 * max(1.0, s[0] + s[1]), (kind, s)
        if nranks == 1:
            b = ctxs[0].last_budget()
            _same(np.array([b.eroded, b.deposited, b.cascade_net, b.discarded, b.clamped, b.wind_negative]), sums_p, kind)
    for c in ctxs:
        c.close()
