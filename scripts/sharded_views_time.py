"""Device time of the read-only views of a sharded map (DESIGN.md section 5), with the card it ran on.

  python scripts/sharded_views_time.py [--parent-lib PATH] [--reps 3]

Prints one JSON line per measurement:
  * mesh_one: k_mesh on one unsharded context at 4096^2, for this build and (with --parent-lib, e.g. a library
    built from the previous commit) that build, alternating, each in a fresh process;
  * mesh_ranks: k_mesh of each rank of the same map on 2 virtual ranks (contexts sharing this GPU), timed one rank
    at a time, and their sum;
  * boundary: the wind-field boundary from the terrain at 512 x 64 x 512, on one context and on each of the 2 ranks
    (every rank builds the whole lattice's boundary).
Times are medians over 20 launches, CUDA events on the context's stream.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

DIM, SOIL, SEED, SLICE, LATTICE, LAUNCHES = 4096, "rockgravelpebblessand", 42, 160, (512, 64, 512), 20


def _median_ms(ctx, fn):
    import numpy as np
    fn()                                     # warm-up (module load, first-touch allocations)
    ts = []
    for _ in range(LAUNCHES):
        ctx.timer_start()
        fn()
        ts.append(ctx.timer_stop())
    return float(np.median(ts))


def _card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=60).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def measure_one():
    from soilmachine_b200 import capi, presets
    pre = presets.load(SOIL)
    ctx = capi.Context(DIM, DIM, pre["world"]["scale"], max_particles=16)
    ctx.set_soils(pre["soils"]); ctx.set_soil_colors(pre["colors"]); ctx.initialize(SEED, pre["layers"])
    ms = _median_ms(ctx, lambda: ctx.mesh_update(SLICE, download=False))
    ctx.close()
    return ms


def measure_sharded():
    from soilmachine_b200 import capi, presets, sharded
    pre = presets.load(SOIL)
    scale = pre["world"]["scale"]
    sh = sharded.VirtualShards(2, DIM, DIM, scale, max_particles=16)
    sh.set_soils(pre["soils"]); sh.set_soil_colors(pre["colors"]); sh.initialize(SEED, pre["layers"])
    sh.sync()
    ranks = [_median_ms(c, lambda c=c: c.mesh_update(SLICE, download=False)) for c in sh.ctx]
    out = {"what": "mesh_ranks", "dim": DIM, "ranks_ms": ranks, "sum_ms": sum(ranks)}
    bnd = []
    for c in sh.ctx:
        c.lbm_create(*LATTICE)
        bnd.append(_median_ms(c, lambda c=c: c.lbm_set_boundary(None)))
        c.lbm_create(3, 3, 3)                # give the 3 GB lattice back before the next one
    sh.close()
    one = capi.Context(DIM, DIM, scale, max_particles=16)
    one.set_soils(pre["soils"]); one.initialize(SEED, pre["layers"])
    one.lbm_create(*LATTICE)
    b1 = _median_ms(one, lambda: one.lbm_set_boundary(None))
    one.close()
    return [out, {"what": "boundary", "lattice": list(LATTICE), "one_context_ms": b1, "ranks_ms": bnd}]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--parent-lib", default=None, help="a second build of the library to alternate with")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--child", action="store_true", help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.child:
        print(json.dumps({"ms": measure_one()}), flush=True)
        return
    print(json.dumps({"card": _card()}), flush=True)
    libs = [("this build", None)] + ([("parent build", os.path.abspath(args.parent_lib))] if args.parent_lib else [])
    runs = {name: [] for name, _ in libs}
    for _ in range(args.reps):
        for name, lib in libs:
            env = dict(os.environ)
            env.pop("SM_LIB_PATH", None)
            if lib:
                env["SM_LIB_PATH"] = lib
            out = subprocess.run([sys.executable, os.path.abspath(__file__), "--child"], env=env, cwd=ROOT,
                                 capture_output=True, text=True, check=True).stdout
            runs[name].append(json.loads(out.strip().splitlines()[-1])["ms"])
    print(json.dumps({"what": "mesh_one", "dim": DIM, "slice": SLICE, "ms_by_build": runs}), flush=True)
    for line in measure_sharded():
        print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
