"""Wind batches for the hand-off rule (tests/test_wind_handoff.py), each run against the reference's lockstep loop
(oracle/_ref) bit for bit.  Run as a script with SM_LIB_PATH set to a -DSM_AUDIT_HANDOFF -DSM_PROFILE build, it runs
them all once more and prints one JSON line per batch: the audit's count of hand-offs acquired without a release
(debug row 16381) and the scans with more than 128 lower-index particles in range (row 16382, word 7)."""
import ctypes as C
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
for p in (os.path.dirname(HERE), HERE):
    if p not in sys.path:
        sys.path.insert(0, p)


def _same(a, b, what):
    a = np.ascontiguousarray(a); b = np.ascontiguousarray(b)
    assert a.shape == b.shape and np.array_equal(a.view(np.uint8), b.view(np.uint8)), what


def _compare(ref, ctx, what):
    _same(ref.heights(), ctx.heights(), what + ": height")
    c1, c2 = ref.columns(), ctx.download_columns()
    for k in c1:
        _same(c1[k], c2[k], what + ": columns." + k)
    f1, f2 = ref.frequency(), ctx.frequency()
    for k in f1:
        _same(f1[k], f2[k], what + ": " + k)


def _context(ref, soil, dim, seed):
    import soilmachine_b200 as smb
    ref.init(soil, seed=seed, dimx=dim, dimy=dim, poolsize=dim * dim * 4 + 2000000)
    ctx = smb.Context(ref.dimx, ref.dimy, ref.scale, max_particles=8192)
    ctx.set_soils(ref.soils())
    cols = ref.columns()
    ctx.upload_columns(cols["offsets"], cols["type"], cols["size"], cols["saturation"])
    return ctx


def _debug(ctxs):
    """(audit misses, scans with > 128 in range) summed over the contexts; clears their debug rows"""
    miss = crowded = 0
    for c in ctxs:
        buf = np.zeros((16384, 8), np.uint64)
        c.lib.sm_debug_sweeps8(c.h, buf.ctypes.data_as(C.c_void_p), 16384)
        miss += int(buf[16381, 0]); crowded += int(buf[16382, 7])
    return miss, crowded


def crowded(ref):
    """3000 wind particles on 64^2 cells: scans list more than 128 lower-index particles in range"""
    ctx = _context(ref, "rocksand", 64, 11)
    xy = ref.spawn_list(3000, seed=11)
    r, g = ref.wind_run(xy), ctx.wind_run(xy)
    assert (g.steps, g.exit_oob) == (r.steps, r.exit_oob)
    _compare(ref, ctx, "crowded")
    _same(ref.wind_state()["pos"], ctx.wind_state()["pos"], "crowded: pos")
    return [ctx]


def ragged(ref):
    """a batch that fills no warp evenly on a map that is no multiple of a bin"""
    ctx = _context(ref, "rockgravelpebblessand", 150, 12)
    xy = ref.spawn_list(1001, seed=12)
    r, g = ref.wind_run(xy), ctx.wind_run(xy)
    assert (g.steps, g.exit_oob) == (r.steps, r.exit_oob)
    _compare(ref, ctx, "ragged")
    return [ctx]


def resumed(ref):
    """the batch in launches of 7 sweeps (max_sweeps), the states compared after each"""
    ctx = _context(ref, "rocksand", 128, 13)
    xy = ref.spawn_list(1500, seed=13)
    ref.wind_begin(xy); ctx.wind_begin(xy)
    for chunk in range(12):
        for _ in range(7):
            alive, _ = ref.wind_sweep()
        st = ctx.wind_sweeps(7)
        s1, s2 = ref.wind_state(), ctx.wind_state()
        for k in s1:
            _same(s1[k], s2[k], "resumed: chunk %d %s" % (chunk, k))
        assert st.alive == alive
        if alive == 0:
            break
    _compare(ref, ctx, "resumed")
    return [ctx]


def sharded(ref, nranks):
    """x-strips on nranks contexts sharing this GPU (these keep the own-bin order): cross-strip waits, remote polls,
    edge releases, at the sizes tests/test_gpu_parity.py runs sharded wind batches at"""
    from soilmachine_b200 import sharded as shd
    dimx, dimy = (128, 96) if nranks == 2 else (144, 80)
    ref.init("rocksand", seed=17, dimx=dimx, dimy=dimy)
    sh = shd.VirtualShards(nranks, ref.dimx, ref.dimy, ref.scale, max_particles=4096)
    sh.set_soils(ref.soils())
    sh.initialize(17, ref.layers())
    xd = ref.spawn_list(500 if nranks == 2 else 700, seed=17)
    r, g = ref.wind_run(xd), sh.wind_run(xd)
    assert (g.steps, g.exit_oob) == (r.steps, r.exit_oob)
    ref.frequency_update(); sh.frequency_update()
    _compare(ref, sh, "sharded %d" % nranks)
    return sh


BATCHES = {"crowded": crowded, "ragged": ragged, "resumed": resumed,
           "sharded2": lambda ref: sharded(ref, 2), "sharded3": lambda ref: sharded(ref, 3)}


def run(name, ref):
    """runs one batch; returns (audit misses, crowded scans)"""
    out = BATCHES[name](ref)
    ctxs = out.ctx if hasattr(out, "ctx") and isinstance(out.ctx, list) else out
    res = _debug(ctxs)
    for c in ctxs:
        c.close()
    return res


def config3(sweeps):
    """a config-3 sized wind batch (4096^2, 25 000 particles) for `sweeps` sweeps; returns (audit misses, crowded)"""
    from soilmachine_b200 import host
    sim = host.Simulation("rockgravelpebblessand", seed=42, dimx=4096, dimy=4096, max_particles=25000)
    xd = host.spawn_list(25000, 4096, 4096)
    st = sim.ctx.wind_run(xd, max_sweeps=sweeps)
    res = _debug([sim.ctx])
    sim.close()
    return res + (int(st.sweeps),)


if __name__ == "__main__":
    from oracle import refapi
    ref = refapi.get()
    for exact in ("0", "3"):
        os.environ["SM_EXACT"] = exact
        for name in BATCHES:
            miss, crowd = run(name, ref)
            print(json.dumps({"batch": name, "exact": exact, "audit_misses": miss, "crowded_scans": crowd}), flush=True)
        miss, crowd, sweeps = config3(300)
        print(json.dumps({"batch": "config3", "exact": exact, "audit_misses": miss, "crowded_scans": crowd,
                          "sweeps": sweeps}), flush=True)
