"""Config-3 wind batch, water batch and bench `value` of this build against another build (DESIGN.md section 5), with
the card it ran on.

  python scripts/wind_handoff_time.py [--parent-lib PATH] [--reps 3] [--profile-lib PATH ...]

Prints one JSON line per measurement:
  * card: name, power limit and max SM clock (nvidia-smi), and the SM clock at the end of the runs;
  * frame: the first config-3 frame (4096^2 rockgravelpebblessand, seed 42, the bench's first 25 000-particle water and
    wind spawn lists) in a fresh process - water and wind batch device_ms, sweeps, steps and the column checksum;
  * bench: `bench.py --gpus 1 --steps 3 --warmup 1 --no-cpu --no-extra` in a fresh process - value and parity;
  builds alternate (this build, then --parent-lib), --reps times;
  * profile: for each --profile-lib (a -DSM_PROFILE build), the hand-off counters of the same wind batch: scans, a
    higher index in the 3x3 bins (what the previous rule fenced on), a higher index in range (what this rule fences on),
    own-bin predecessors and how many of them are out of range, lower-index particles in range (<= 31, 32-128, > 128),
    and the per-phase cycles of the conservative path (flush + publish with and without a release).
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

DIM, SOIL, SEED, N = 4096, "rockgravelpebblessand", 42, 25000


def _smi(q):
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=60).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def frame(profile):
    import ctypes as C
    import numpy as np
    from soilmachine_b200 import host
    sim = host.Simulation(SOIL, seed=SEED, dimx=DIM, dimy=DIM, max_particles=N)
    xw = host.spawn_list(N, DIM, DIM)
    xd = host.spawn_list(N, DIM, DIM)
    out = {}
    buf = np.zeros((16384, 8), np.uint64)
    w = sim.ctx.water_run(xw)
    if profile:
        sim.ctx.lib.sm_debug_sweeps8(sim.ctx.h, buf.ctypes.data_as(C.c_void_p), 16384)     # clear
    d = sim.ctx.wind_run(xd)
    out.update(water_ms=w.device_ms, water_sweeps=w.sweeps, wind_ms=d.device_ms, wind_sweeps=d.sweeps,
               wind_steps=d.steps, checksum="%016x" % sim.ctx.checksum())
    if profile:
        sim.ctx.lib.sm_debug_sweeps8(sim.ctx.h, buf.ctypes.data_as(C.c_void_p), 16384)
        h, ph = [int(v) for v in buf[16382]], [int(v) for v in buf[16383]]
        out["handoff"] = {"scans": h[0], "higher_in_bins": h[1], "higher_in_range": h[2], "own_bin_pred": h[3],
                          "own_bin_pred_out_of_range": h[4], "in_range_le31": h[5], "in_range_32_128": h[6],
                          "in_range_gt128": h[7]}
        out["phases_cycles"] = {"steps": ph[5], "load_scan": ph[0], "wait": ph[1], "move": ph[2], "interact": ph[3],
                                "flush_publish": ph[4], "flush_publish_released": ph[6], "released_steps": ph[7]}
    sim.close()
    return out


def _child(lib, *args):
    env = dict(os.environ)
    env.pop("SM_LIB_PATH", None)
    if lib:
        env["SM_LIB_PATH"] = lib
    out = subprocess.run([sys.executable] + list(args), env=env, cwd=ROOT, capture_output=True, text=True,
                         check=True).stdout
    return json.loads(out.strip().splitlines()[-1])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--parent-lib", default=None, help="a second build of the library to alternate with")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--profile-lib", action="append", default=[], help="a -DSM_PROFILE build to read the counters of")
    ap.add_argument("--child", choices=["frame", "profile"], help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.child:
        print(json.dumps(frame(args.child == "profile")), flush=True)
        return
    print(json.dumps({"card": _smi("name,power.limit,clocks.max.sm")}), flush=True)
    me = os.path.abspath(__file__)
    libs = [("this build", None)] + ([("parent build", os.path.abspath(args.parent_lib))] if args.parent_lib else [])
    for rep in range(args.reps):
        for name, lib in libs:
            f = _child(lib, me, "--child", "frame")
            print(json.dumps({"what": "frame", "build": name, "rep": rep, **f}), flush=True)
            b = _child(lib, os.path.join(ROOT, "bench.py"), "--gpus", "1", "--steps", "3", "--warmup", "1",
                       "--no-cpu", "--no-extra")
            print(json.dumps({"what": "bench", "build": name, "rep": rep, "value": b["value"],
                              "ms_per_step": b["ms_per_step"], "parity": b.get("parity"), "clocks": b.get("clocks")}),
                  flush=True)
    for lib in args.profile_lib:
        f = _child(os.path.abspath(lib), me, "--child", "profile")
        print(json.dumps({"what": "profile", "lib": os.path.basename(lib), **f}), flush=True)
    print(json.dumps({"card_after": _smi("name,power.limit,clocks.sm")}), flush=True)


if __name__ == "__main__":
    main()
