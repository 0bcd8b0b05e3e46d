"""Time of a frame through a context group, against one context and against hand-assembled ranks, with the card.

  python scripts/group_time.py [--dims 1024 4096] [--rounds 3]

The bench's config-3 map (rockgravelpebblessand, seed 42) with its 25k water particles at each size: the water part
of a frame (water batch, floods, seep pass, frequency update) through four arms taken in alternation in one process -
one context, a group of one, a two-rank group on this GPU and sharded.VirtualShards(2).  One JSON line per arm and
round: per phase the device time the library reports (CUDA events around the phase's kernels) and the host clock
around the call (which ends in a synchronise, except the frequency update, which is followed by an explicit one), so
host_ms - device_ms of an arm is what its plumbing costs: strip cutting, one launch per rank, the settles.
Virtual ranks share the SMs of one GPU, so the two-rank arms are expected to be SLOWER than one context here: they
are the correctness vehicle of the one-GPU tests, not a speed claim.  The map checksums of all arms must agree.
The wind batch is left out: a 25k-particle wind batch on two virtual ranks sharing one H100 did not return within
200 s at 1024^2 (one context: well under a second; DESIGN.md section 9), so this script cannot time it.
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SOIL, SEED, N = "rockgravelpebblessand", 42, 25000
ARMS = ("one context", "group of 1", "group of 2 on one GPU", "VirtualShards(2)")


def _card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=60).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def make(arm, dim, pre):
    from soilmachine_b200 import capi, sharded
    scale = pre["world"]["scale"]
    if arm == "one context":
        m = capi.Context(dim, dim, scale, max_particles=N)
    elif arm == "group of 1":
        m = capi.Context(dim, dim, scale, max_particles=N, devices=[0])
    elif arm == "group of 2 on one GPU":
        m = capi.Context(dim, dim, scale, max_particles=N, devices=[0, 0])
    else:
        m = sharded.VirtualShards(2, dim, dim, scale, max_particles=N)
    m.set_soils(pre["soils"])
    m.initialize(SEED, pre["layers"])
    return m


def frame(m, xw):
    """{phase: (device_ms, host_ms)}"""
    out = {}

    def timed(name, call, dev=lambda r: r.device_ms):
        print("  %s ..." % name, file=sys.stderr, flush=True)     # progress: a phase that never returns is named
        m.sync()
        t0 = time.perf_counter()
        r = call()
        m.sync()
        out[name] = (dev(r), (time.perf_counter() - t0) * 1e3)

    timed("water", lambda: m.water_run(xw))
    timed("flood", lambda: m.water_flood())
    timed("seep", lambda: m.seep())
    timed("frequency", lambda: m.frequency_update(), dev=lambda r: None)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--dims", type=int, nargs="+", default=[1024, 4096])
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    from soilmachine_b200 import host, presets
    pre = presets.load(SOIL)
    card = _card()
    ok = True
    for dim in args.dims:
        host.srand(SEED)
        lists = [host.spawn_list(N, dim, dim) for _ in range(args.rounds + 1)]
        maps = {arm: make(arm, dim, pre) for arm in ARMS}
        for arm in ARMS:                       # warm-up frame: module loads, first-use allocations
            print("warm-up, %d^2, %s" % (dim, arm), file=sys.stderr, flush=True)
            frame(maps[arm], lists[0])
        for rnd in range(args.rounds):
            sums = set()
            for arm in ARMS:
                m = maps[arm]
                print("round %d, %d^2, %s" % (rnd, dim, arm), file=sys.stderr, flush=True)
                ph = frame(m, lists[rnd + 1])
                csum = m.checksum() if hasattr(m, "checksum") else sum(c.checksum() for c in m.ctx) % (1 << 64)
                sums.add(csum)
                print(json.dumps({"dim": dim, "round": rnd, "arm": arm, "card": card,
                                  "device_ms": {k: v[0] for k, v in ph.items()},
                                  "host_ms": {k: round(v[1], 3) for k, v in ph.items()},
                                  "frame_host_ms": round(sum(v[1] for v in ph.values()), 3), "checksum": csum}), flush=True)
            ok = ok and len(sums) == 1
        for m in maps.values():
            m.close()
    print(json.dumps({"what": "map checksums", "identical_across_arms": ok}), flush=True)
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
