"""Snapshots on the device (sm_snapshot_bytes / _save / _restore): the bytes equal the numpy twin
(soilmachine_b200/snapshot.py), they are canonical, and a restored simulation continues bit for bit - on the same
context, a fresh one, groups of 2 and 3 virtual ranks, VirtualShards(2), from host and device buffers - through
capi.Context, sharded.py, host.Simulation and the C++ facade.  Refused restores leave the map as it was.
tests/multigpu_snapshot_check.py does the same across processes."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

import _group
from _group import same

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SEED = 23
STAT_KEYS = ("steps", "sweeps", "exit_oob", "exit_evap", "exit_stall", "pool_drops", "alive")
HYDRO_KEYS = ("floods", "nested", "nested_steps", "transfers", "cells")


def _d2h(dptr, n):
    """copy n bytes of device memory to the host with the CUDA runtime (the library links its own statically)"""
    for name in ("libcudart.so.12", "/usr/local/cuda/lib64/libcudart.so"):
        try:
            rt = C.CDLL(name)
            break
        except OSError:
            continue
    out = np.empty(n, np.uint8)
    rt.cudaMemcpy.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_int]
    assert rt.cudaMemcpy(out.ctypes.data_as(C.c_void_p), dptr, n, 2) == 0        # cudaMemcpyDeviceToHost
    return out


def _ctx(soil, dimx, dimy, **kw):
    from soilmachine_b200 import capi, presets
    pre = presets.load(soil)
    c = capi.Context(dimx, dimy, pre["world"]["scale"], max_particles=kw.pop("max_particles", 8192), **kw)
    c.set_soils(pre["soils"])
    return c, pre


def _lists(dimx, dimy, frames, nw, nd, seed=SEED):
    from soilmachine_b200 import host
    host.srand(seed)
    return [(host.spawn_list(nw, dimx, dimy), host.spawn_list(nd, dimx, dimy)) for _ in range(frames)]


def _frame(m, xy_w, xy_d):
    """water batch, floods, seep pass, wind batch, frequency update; the counters of every call"""
    out = [m.water_run(xy_w), m.water_flood(), m.seep(), m.wind_run(xy_d)]
    m.frequency_update()
    return [tuple(getattr(s, k) for k in (STAT_KEYS if i in (0, 3) else HYDRO_KEYS)) for i, s in enumerate(out)]


def _record(m, counters):
    """A: columns, heights, frequency arrays, checksum and counters"""
    return {"cols": m.download_columns(), "heights": m.heights(), "freq": m.frequency(),
            "sum": sum(c.checksum() for c in m.ctx) % (1 << 64) if hasattr(m, "ranges") else m.checksum(),
            "counters": counters}


def _same_record(a, b, what):
    for k in b["cols"]:
        same(a["cols"][k], b["cols"][k], "%s: columns.%s" % (what, k))
    same(a["heights"], b["heights"], what + ": heights")
    for k in b["freq"]:
        same(a["freq"][k], b["freq"][k], "%s: %s" % (what, k))
    assert a["sum"] == b["sum"], what + ": checksum"
    assert a["counters"] == b["counters"], (what, a["counters"], b["counters"])


def _twin(c, nsoils):
    from soilmachine_b200 import snapshot
    return np.frombuffer(snapshot.build(c.download_columns(), c.frequency(), c.dimx, c.dimy, c.x0, c.x1, nsoils), np.uint8)


# ---- the bytes ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dim,nw,nd", [(192, 2500, 300), (1024, 30000, 300)])
def test_device_and_host_saves_equal_the_twin(dim, nw, nd):
    c, pre = _ctx("rocksand", dim, dim, max_particles=nw)
    try:
        c.initialize(SEED, pre["layers"])
        for xw, xd in _lists(dim, dim, 2, nw, nd):
            _frame(c, xw, xd)
        want = _twin(c, len(pre["soils"]))
        assert c.snapshot_bytes() == want.size
        same(c.snapshot(), want, "host save")
        d, n = c.snapshot_device()
        try:
            assert n == want.size
            same(_d2h(d, n), want, "device save")
        finally:
            c.device_free(d)
    finally:
        c.close()


def test_config3_frame_save_equals_the_twin():
    """one frame of the benchmark's workload (4096^2 rockgravelpebblessand, 25k water + 25k wind): more than one
    staging buffer of records, so the host save runs in several cell ranges"""
    from soilmachine_b200 import host
    sim = host.Simulation("rockgravelpebblessand", seed=42, dimx=4096, dimy=4096, max_particles=25000)
    try:
        sim.frame(25000, 25000)
        c = sim.ctx
        want = _twin(c, len(sim.preset["soils"]))
        assert want.size > 3 * (32 << 20)
        assert c.snapshot_bytes() == want.size
        same(c.snapshot(), want, "host save")
        d, n = c.snapshot_device()
        try:
            same(_d2h(d, n), want, "device save")
        finally:
            c.device_free(d)
    finally:
        sim.close()


def test_snapshots_are_canonical():
    """the same columns reached two ways (an evolved pool, and an upload of its download) give the same bytes, and a
    restore saved again gives them back"""
    c, pre = _ctx("bigbutte", 96, 72)
    u, _ = _ctx("bigbutte", 96, 72)
    try:
        c.initialize(SEED, pre["layers"])
        for xw, xd in _lists(96, 72, 3, 700, 200):
            _frame(c, xw, xd)
        s = c.snapshot()
        cols = c.download_columns()
        u.upload_columns(cols["offsets"], cols["type"], cols["size"], cols["saturation"])
        u.set_frequency(**c.frequency())
        same(u.snapshot(), s, "upload of the download")
        u.initialize(SEED + 1, pre["layers"])
        u.restore(s)
        same(u.snapshot(), s, "restored, saved again")
        c.restore(s)
        same(c.snapshot(), s, "restored over itself, saved again")
    finally:
        c.close(); u.close()


# ---- resume ---------------------------------------------------------------------------------------------------------
def _resume_case():
    """frames 1-2 on one context, the snapshot, then frames 3-4: (snapshot, lists of frames 3-4, A, the context)"""
    c, pre = _ctx("bigbutte", 96, 72)
    c.initialize(SEED, pre["layers"])
    lists = _lists(96, 72, 4, 700, 200)
    for xw, xd in lists[:2]:
        _frame(c, xw, xd)
    s = c.snapshot()
    a = _record(c, [_frame(c, xw, xd) for xw, xd in lists[2:]])
    return s, lists[2:], a, c, pre


def test_resume_is_bit_identical_everywhere():
    from soilmachine_b200 import sharded
    s, later, a, c, pre = _resume_case()
    assert any(h[0] for f in a["counters"] for h in f[1:3]), "no flood in frames 3-4"
    try:
        def check(m, what, buf=s):
            m.restore(buf)
            _same_record(_record(m, [_frame(m, xw, xd) for xw, xd in later]), a, what)

        check(c, "the same context, host buffer")
        # a device buffer saved by a fresh context holding the snapshot
        f, _ = _ctx("bigbutte", 96, 72)
        try:
            check(f, "a fresh context")
            f.restore(s)
            d, n = f.snapshot_device()
            try:
                check(c, "the same context, device buffer", (d, n))
            finally:
                f.device_free(d)
        finally:
            f.close()
        for nranks in (2, 3):
            g, _ = _ctx("bigbutte", 96, 72, devices=[0] * nranks)
            try:
                check(g, "a group of %d" % nranks)
            finally:
                g.close()
        v = sharded.VirtualShards(2, 96, 72, pre["world"]["scale"], max_particles=8192)
        try:
            v.set_soils(pre["soils"])
            check(v, "VirtualShards(2)")
        finally:
            v.close()
    finally:
        c.close()


def test_saves_and_restores_across_sharding():
    """a group's save and VirtualShards.snapshot() are one context's bytes; a rank restores a whole-map snapshot
    and a strip snapshot of its own range"""
    from soilmachine_b200 import sharded, snapshot
    s, later, a, c, pre = _resume_case()
    c.close()
    g, _ = _ctx("bigbutte", 96, 72, devices=[0, 0, 0])
    v = sharded.VirtualShards(2, 96, 72, pre["world"]["scale"], max_particles=8192)
    try:
        v.set_soils(pre["soils"])
        g.restore(s)
        same(g.snapshot(), s, "group save")
        d, n = g.snapshot_device()
        try:
            same(_d2h(d, n), s, "group save to device memory")
        finally:
            g.device_free(d)
        v.restore(s)
        same(v.snapshot(), s, "VirtualShards.snapshot()")
        r = v.ctx[1]
        strip = snapshot.cut(s.tobytes(), r.x0, r.x1)
        v.ctx[0].initialize(SEED + 5, pre["layers"]); r.initialize(SEED + 5, pre["layers"])
        r.restore(strip)
        same(r.snapshot(), np.frombuffer(strip, np.uint8), "a rank restoring its strip snapshot")
        v.ctx[0].restore(s)
        same(v.snapshot(), s, "after a rank restored the whole-map snapshot")
    finally:
        g.close(); v.close()


def test_simulation_save_and_load(tmp_path):
    from soilmachine_b200 import host
    path = str(tmp_path / "sim.npz")
    sim = host.Simulation("bigbutte", seed=SEED, dimx=96, dimy=72, max_particles=4096)
    try:
        for _ in range(2):
            sim.frame(700, 200, hydrology=True)
        sim.save(path)
        for _ in range(2):
            sim.frame(700, 200, hydrology=True)
        want = sim.ctx.checksum(), sim.ctx.frequency()
    finally:
        sim.close()
    for kw in ({}, {"gpus": 2, "devices": [0, 0]}):
        s2 = host.Simulation.load(path, max_particles=4096, **kw)
        try:
            for _ in range(2):
                s2.frame(700, 200, hydrology=True)
            assert s2.ctx.checksum() == want[0], kw
            for k, v in want[1].items():
                same(s2.ctx.frequency()[k], v, "%s %s" % (kw, k))
        finally:
            s2.close()


def test_facade_save_and_load(tmp_path):
    """tests/facade_snapshot.cpp: save, run on, load, run again; and load a file one context saved on a group"""
    from oracle import refapi
    libdir = os.path.join(ROOT, "soilmachine_b200", "lib")
    exe = str(tmp_path / "facade_snapshot")
    subprocess.check_call(["g++", "-std=c++17", "-O1", os.path.join(ROOT, "tests", "facade_snapshot.cpp"), "-o", exe,
                           "-L" + libdir, "-lsoilmachine_b200", "-Wl,-rpath," + libdir])
    soil = refapi.soil_path("bigbutte")

    def run(args, group):
        env = {k: v for k, v in os.environ.items() if k not in ("SM_GPUS", "SM_GPU_DEVICES")}
        if group:
            env.update(SM_GPUS="2", SM_GPU_DEVICES="0,0")
        out = subprocess.run([exe, soil] + args, capture_output=True, text=True, timeout=900, env=env)
        assert out.returncode == 0, out.stdout + out.stderr
        return out.stdout

    snap, a, b, c = (str(tmp_path / n) for n in ("s.snap", "a.snap", "b.snap", "c.snap"))
    assert "resume identical" in run(["save", snap, a], False)
    assert "resume identical" in run(["save", str(tmp_path / "g.snap"), b], True)
    assert "loaded" in run(["load", snap, c], True)
    data = [open(p, "rb").read() for p in (a, b, c)]
    assert data[0] == data[1] == data[2], "final snapshots differ"
    assert open(snap, "rb").read() == open(str(tmp_path / "g.snap"), "rb").read()


# ---- errors ---------------------------------------------------------------------------------------------------------
def test_refused_restores_leave_the_map_unchanged():
    from soilmachine_b200 import capi, sharded, snapshot
    s, later, a, c, pre = _resume_case()
    c.close()
    c, _ = _ctx("bigbutte", 96, 72)
    try:
        c.initialize(SEED + 9, pre["layers"])
        before = _record(c, None)

        def refused(m, buf, code, what):
            with pytest.raises(capi.SoilMachineError) as e:
                m.restore(buf)
            assert e.value.code == code, (what, str(e.value))
            _same_record(_record(m, None), before, what)

        bad_dims, _ = _ctx("bigbutte", 96, 64)
        try:
            with pytest.raises(capi.SoilMachineError) as e:
                bad_dims.restore(s)
            assert e.value.code == capi.SM_ERR_INVALID
        finally:
            bad_dims.close()
        refused(c, s[:-1], capi.SM_ERR_INVALID, "truncated")
        h = snapshot.header(s)
        wrong_soils = bytearray(s.tobytes())
        wrong_soils[32:36] = np.int32(h["nsoils"] - 1).tobytes()
        refused(c, bytes(wrong_soils), capi.SM_ERR_INVALID, "nsoils")
        refused(c, snapshot.cut(s.tobytes(), 0, 40), capi.SM_ERR_INVALID, "a strip snapshot on a plain context")
        with pytest.raises(capi.SoilMachineError) as e:
            short = np.empty(c.snapshot_bytes() - 1, np.uint8)
            c._ck_strict(c.lib.sm_snapshot_save(c.h, short.ctypes.data_as(C.c_void_p), C.c_int64(short.size), 0))
        assert e.value.code == capi.SM_ERR_INVALID
        # a fixed pool too small for the snapshot's buried sections
        small, _ = _ctx("bigbutte", 96, 72, pool_capacity=64)
        try:
            small.pool_warn = False
            small.initialize(SEED, pre["layers"][:1])
            keep = _record(small, None)
            with pytest.raises(capi.SoilMachineError) as e:
                small.restore(s)
            assert e.value.code == capi.SM_ERR_POOL
            _same_record(_record(small, None), keep, "fixed pool too small")
        finally:
            small.close()
        # a rank of a sharded map given a strip snapshot of another range
        v = sharded.VirtualShards(2, 96, 72, pre["world"]["scale"], max_particles=8192)
        try:
            v.set_soils(pre["soils"])
            v.initialize(SEED, pre["layers"])
            keep = v.ctx[1].snapshot()
            with pytest.raises(capi.SoilMachineError) as e:
                v.ctx[1].restore(snapshot.cut(s.tobytes(), v.ctx[0].x0, v.ctx[0].x1))
            assert e.value.code == capi.SM_ERR_INVALID
            same(v.ctx[1].snapshot(), keep, "rank with a different range")
        finally:
            v.close()
        # one flipped byte in a record's size: written, then refused by the checksum, as documented
        damaged = bytearray(s.tobytes())
        k = h["records_at"] + 32 * (h["nsections"] // 3) + 3
        damaged[k] ^= 0x40
        with pytest.raises(capi.SoilMachineError) as e:
            c.restore(bytes(damaged))
        assert e.value.code == capi.SM_ERR_INVALID and "checksum" in str(e.value)
        _, cols, _ = snapshot.parse(bytes(damaged))
        got = c.download_columns()
        for key in cols:
            same(got[key], cols[key], "the map holds the damaged snapshot: " + key)
        # no batch is open after a restore
        with pytest.raises(capi.SoilMachineError):
            c.water_flood()
    finally:
        c.close()


def test_snapshot_over_cuda_ipc_two_processes_one_gpu():
    """tests/multigpu_snapshot_check.py with two processes sharing this GPU"""
    env = dict(os.environ, SM_ONE_GPU="1")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2",
           "--master-addr", "127.0.0.1", "--master-port", "29653",
           os.path.join(ROOT, "tests", "multigpu_snapshot_check.py"), "96", "700"]
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=900, cwd=ROOT, env=env)
    line = [l for l in out.stdout.splitlines() if l.startswith("multigpu_snapshot_check")]
    assert out.returncode == 0 and line and "DIFFER" not in line[0], (out.stdout[-2000:], out.stderr[-2000:])
