"""CPU: the C-ABI library loads and exports what include/soilmachine_b200.h declares, fails loudly
without a GPU, presets match the reference loader, host-side spawn lists match the reference's
constructor draws, and bench.py's reference arm runs end to end."""
import json
import os
import re
import subprocess
import sys
import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_library_exports_every_declared_symbol():
    from soilmachine_b200 import capi
    hdr = open(os.path.join(ROOT, "include", "soilmachine_b200.h")).read()
    declared = set(re.findall(r"\b(sm_[a-z_0-9]+)\s*\(", hdr))
    assert declared, "no declarations parsed"
    lib = capi.load()
    missing = [s for s in sorted(declared) if not hasattr(lib, s)]
    assert not missing, "declared but not exported: %s" % missing
    assert set(capi.SYMBOLS) == declared


def test_no_cpu_fallback():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    import soilmachine_b200 as smb
    with pytest.raises(smb.SoilMachineError) as e:
        smb.Context(64, 64)
    assert e.value.code == smb.capi.SM_ERR_NOGPU


def test_presets_match_reference_loader():
    """The JSON presets against what the reference's loadsoil() made of each preset file (tests/golden)."""
    import _golden
    from soilmachine_b200 import presets
    g = _golden.load("ref_loader")
    names = presets.names()
    assert "rockgravelpebblessand" in names and len(names) == 11
    for name in names:
        pre = presets.load(name)
        rs, rl = g[name + "/soils"], g[name + "/layers"]
        assert len(rs) == len(pre["soils"]) and len(rl) == len(pre["layers"])
        for k in pre["soils"].dtype.names:
            assert np.array_equal(rs[k], pre["soils"][k]), (name, k)
        for k in pre["layers"].dtype.names:
            assert np.array_equal(rl[k], pre["layers"][k]), (name, k)
        assert int(g[name + "/scale"]) == pre["world"]["scale"]


def test_spawn_lists_match_reference_ctor_draws():
    import _golden
    from soilmachine_b200 import host
    a = _golden.load("ref_loader")["spawn_default_100x70_seed5"]
    host.srand(5)
    b = host.spawn_list(64, 100, 70)
    assert np.array_equal(a, b)


def test_bench_reference_arm_runs(ref):
    out = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--dim", "96",
                          "--particles", "200", "--steps", "1", "--warmup", "0"],
                         capture_output=True, text=True, timeout=300, cwd=ROOT)
    assert out.returncode == 0, out.stderr
    line = json.loads(out.stdout.strip().splitlines()[-1])
    assert line["impl"] == "reference" and line["value"] > 0
    assert line["cpu_baseline"]["kind"] == "reference" and line["cpu_baseline"]["cores"] == 1
    assert line["e2e"]["h2d_bytes_per_step"] == 0


def test_cpp_facade_compiles_and_links():
    """include/soilmachine/soilmachine.hpp (the reference's class names over the C ABI) + the frame loop
    of SoilMachine.cpp written against it; without a GPU it must fail loudly (no fallback)."""
    exe = os.path.join(ROOT, "tests", "hostsim", "facade_demo")
    libdir = os.path.join(ROOT, "soilmachine_b200", "lib")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-Wall", "-Werror", os.path.join(ROOT, "tests", "facade_demo.cpp"),
                           "-o", exe, "-L" + libdir, "-lsoilmachine_b200", "-Wl,-rpath," + libdir])
    import torch
    out = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    if torch.cuda.is_available():
        assert out.returncode == 0, out.stdout + out.stderr
        assert "legacy ops ok" in out.stdout
    else:
        assert out.returncode == 77 and "no CUDA device" in out.stdout
    # the reference's per-particle loop, unchanged, against the facade (runs on the GPU tier)
    exe2 = os.path.join(ROOT, "tests", "hostsim", "facade_loop")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-Wall", "-Werror", os.path.join(ROOT, "tests", "facade_loop.cpp"),
                           "-o", exe2, "-L" + libdir, "-lsoilmachine_b200", "-Wl,-rpath," + libdir])
    if not torch.cuda.is_available():
        from oracle import refapi
        out = subprocess.run([exe2, refapi.soil_path("default"), "32", "2", "1", "1", "/dev/null"], capture_output=True,
                             text=True, timeout=120)
        assert out.returncode == 77 and "no CUDA device" in out.stdout


def test_soil_file_parser_matches_reference_loader():
    """include/soilmachine/soilfile.hpp (restatement of loadsoil, io.h:7-230, quirks included) against what the
    reference loader made of every preset file (tests/golden), and against the committed JSON presets."""
    import glob
    import _golden
    from soilmachine_b200 import capi, presets
    g = _golden.load("ref_loader")
    files = sorted(glob.glob(os.path.join(_golden.GOLDEN, "soil", "*.soil")))
    assert len(files) == 11
    for path in files:
        name = os.path.basename(path)[:-5]
        got = capi.parse_soil_file(path)
        rs, rl = g[name + "/soils"], g[name + "/layers"]
        assert got["soil_names"] == [s.decode() for s in rs["name"]], name
        for k in got["soils"].dtype.names:
            assert np.array_equal(got["soils"][k], rs[k]), (name, k)
        assert np.array_equal(got["colors"], rs["color"]), name
        for k in got["layers"].dtype.names:
            assert np.array_equal(got["layers"][k], rl[k]), (name, k)
        pre = presets.load(name)
        assert got["world"] == pre["world"], name
    with pytest.raises(capi.SoilMachineError):
        capi.parse_soil_file("/nonexistent/file.soil")


def test_frame_loop_orders_calls_like_the_reference():
    """host.Simulation.frame against a recording stand-in for the context: water batch(es), floods, seep
    pass, wind batch, frequency update, in the order of SoilMachine.cpp:287-320; water_chunk splits the
    batch and floods after every chunk."""
    import numpy as np
    from soilmachine_b200 import host

    class Rec:
        def __init__(self):
            self.calls = []

        def water_run(self, xy):
            self.calls.append(("water", len(xy)))

        def wind_run(self, xy):
            self.calls.append(("wind", len(xy)))

        def water_flood(self):
            self.calls.append(("flood",))

        def seep(self):
            self.calls.append(("seep",))

        def frequency_update(self):
            self.calls.append(("freq",))

    sim = object.__new__(host.Simulation)
    sim.ctx, sim.dimx, sim.dimy = Rec(), 32, 24
    host.srand(1)
    sim.frame(10, 4)
    assert sim.ctx.calls == [("water", 10), ("wind", 4), ("freq",)]
    sim.ctx.calls.clear()
    sim.frame(10, 4, hydrology=True)
    assert sim.ctx.calls == [("water", 10), ("flood",), ("seep",), ("wind", 4), ("freq",)]
    sim.ctx.calls.clear()
    xy = np.zeros((10, 2), np.float32)
    sim.frame(10, 0, water_xy=xy, hydrology=True, water_chunk=4)
    assert sim.ctx.calls == [("water", 4), ("flood",), ("water", 4), ("flood",), ("water", 2), ("flood",), ("seep",), ("freq",)]
    assert len(sim.last_hydrology[0]) == 3
