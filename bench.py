#!/usr/bin/env python
"""bench.py -- particle-steps/s of the particle/terrain hot path on H100 (BASELINE.json metric).

Workload (config 3 of BASELINE.json, the one the metric is quoted on that fits one GPU):
  4096^2 map, rockgravelpebblessand preset, SEED 42, per step (= one frame, SoilMachine.cpp:287-320
  without flood/seep): 25 000 WaterParticles run to completion in lockstep sweeps, then 25 000
  WindParticles run to completion, then the frequency update.  particle-step = one move() followed by
  one interact() of one particle.

  python bench.py [--gpus N] [--steps K] [--warmup W] [--impl ours|reference] [--config 3|4|5] [--dump-outputs DIR]

* value   : whole-job particle-steps/s, spawn lists already resident in HBM, timed with CUDA events on the
            stream the kernels run on (max over ranks).
* e2e     : the same frames through the host-buffer C ABI calls (sm_water_run / sm_wind_run): the spawn lists
            are copied from pinned host memory and the stats are read back inside the timed region, every step.
* roofline: the path is latency-bound (a sweep lasts as long as its longest chain of dependent particle-steps),
            so `bound` says so and `latency_model` gives the floor: sweeps x the duration of a sweep that holds a
            single isolated particle (measured live on the same map) - no lockstep schedule can finish a batch
            faster than its longest-lived particle steps.  achieved/peak/frac stay the HBM numbers the contract
            asks for: algorithmic bytes (SURVEY.md 8d: 290 B / water step, 600 B / wind step) / duration of the
            dominant kernel (CUDA events around each launch) against the measured HBM peak.
* parity  : position-sensitive checksum of every column section (sm_checksum) after the first frame, compared
            with the golden value tests/test_gpu_parity.py::test_config3_frame_matches_reference pinned to the
            reference run in lockstep, and after the last frame (must be equal for N = 1, 2, 4, 8).
* extra   : BASELINE configs 4 and 5 (2 timed frames each, same sharding as the headline at N > 1) and the
            genuinely HBM-bound full-grid kernels (mesh, frequency update, seep classification) with their bytes.
* cpu_baseline / --impl reference: the reference's own CPU loop (oracle/_ref, the reference headers compiled
            verbatim) on a bounded sample of the same workload with the same water:wind mix, on the box's host
            cores (1 thread: the reference is single-threaded and keeps its state in globals).  Left out (with
            a note) where oracle/_ref has not been built.
* --dump-outputs DIR: after the timed steps, what the last timed step left for a caller, as DIR/<name>.npy
            (float32 / float64): the per-step counters of the timed steps, the column checksum, and a fixed
            seeded sample of cells from the height field and the three frequency maps.  At N > 1 every rank
            writes its own strip's set, named <name>_rank<r>.npy.
N > 1: the SAME map is sharded into N x-strips, one rank (GPU) per strip; halo records, bins and hand-off words
of the neighbouring strips are read and written over NVLink peer memory (CUDA IPC) by the sweep kernel itself,
neighbouring strips synchronise every sweep, all strips every 8th, and particles that leave a strip are handed
to the new owner (DESIGN.md section 7).  Strong scaling: total work is fixed, results are bit-identical to N = 1.
"""
import argparse
import json
import os
import subprocess
import sys
import threading
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

CONFIGS = {
    3: dict(soil="rockgravelpebblessand", dim=4096, nwater=25000, nwind=25000, seed=42,
            label="4096^2 rockgravelpebblessand.soil, 25k Water + 25k Wind particles per step (BASELINE.json configs[2])"),
    4: dict(soil="bigbutte", dim=4096, nwater=50000, nwind=0, seed=42,
            label="4096^2 bigbutte.soil, 50k WaterParticles per step (BASELINE.json configs[3])"),
    5: dict(soil="rockgravelpebbles_big", dim=8192, nwater=100000, nwind=100000, seed=42,
            label="8192^2 rockgravelpebbles_big.soil, 200k mixed particles per step (BASELINE.json configs[4]; "
                  "no soil of this preset can be suspended, so the 100k wind particles die in their first move())"),
}
BYTES_WATER, BYTES_WIND, BYTES_FREQ_CELL = 290, 600, 16   # SURVEY.md section 8d / DESIGN.md section 5
CPU_SAMPLE_DIV = 10                                        # CPU arm: 1/10 of the particles of each kind, same mix
GOLDEN_CS = os.path.join(ROOT, "tests", "golden", "cfg3_frame1_checksum.json")
M64 = (1 << 64) - 1


def hbm_peak():
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    try:
        with open(p) as f:
            return float(json.load(f)["hbm_gbs"]), "measured (MEASURED_PEAKS.json)"
    except Exception:
        return 3350.0, "H100 SXM data sheet (3.35 TB/s HBM3), not measured"


class ClockSampler:
    """nvidia-smi clocks / throttle reasons while the timed region runs."""

    def __init__(self, index):
        self.index = index
        self.proc = None
        self.rows = []

    def start(self):
        q = ("clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.hw_slowdown,"
             "clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,"
             "clocks_event_reasons.sw_power_cap")
        try:
            self.proc = subprocess.Popen(["nvidia-smi", "-i", str(self.index), "--query-gpu=" + q,
                                          "--format=csv,noheader,nounits", "-lms", "200"],
                                         stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
            threading.Thread(target=self._read, daemon=True).start()
        except Exception:
            self.proc = None

    def _read(self):
        for line in self.proc.stdout:
            self.rows.append([x.strip() for x in line.split(",")])

    def stop(self):
        if self.proc:
            self.proc.terminate()
            try:
                self.proc.wait(timeout=3)
            except Exception:
                pass
        sm, mx, reasons = [], 0, set()
        names = ["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"]
        for r in self.rows:
            try:
                sm.append(float(r[0])); mx = max(mx, float(r[1]))
                for k, nm in enumerate(names):
                    if r[3 + k].lower().startswith("active"):
                        reasons.add(nm)
            except Exception:
                pass
        sm.sort()
        return {"sm_mhz": sm[len(sm) // 2] if sm else None, "sm_max_mhz": mx or None,
                "reasons": sorted(reasons), "samples": len(sm)}


def aggregate(ev_ms, e2e_ms, steps, e_steps, device=None):
    """Whole-job numbers from per-rank ones: time = MAX over ranks, particle-steps = SUM over ranks.
    Works on any initialised torch.distributed backend (NCCL on the GPUs, gloo in the CPU tests)."""
    import torch
    import torch.distributed as dist
    t = torch.tensor([ev_ms, e2e_ms, float(steps), float(e_steps)], dtype=torch.float64, device=device)
    if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
        mx = t.clone(); dist.all_reduce(mx, op=dist.ReduceOp.MAX)
        sm_ = t.clone(); dist.all_reduce(sm_, op=dist.ReduceOp.SUM)
        return mx[0].item(), mx[1].item(), sm_[2].item(), sm_[3].item()
    return float(ev_ms), float(e2e_ms), float(steps), float(e_steps)


def checksum_sum(local, device=None):
    """The checksums of the strips add up modulo 2^64 to the checksum of the whole map (two's-complement
    int64 addition wraps exactly like that)."""
    import torch
    import torch.distributed as dist
    if not (dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1):
        return int(local) & M64
    v = int(local) & M64
    t = torch.tensor([v - (1 << 64) if v >= (1 << 63) else v], dtype=torch.int64, device=device)
    dist.all_reduce(t, op=dist.ReduceOp.SUM)
    return int(t.item()) & M64


DUMP_SAMPLE = 1 << 20          # cells of each full-grid output written by --dump-outputs (fixed seeded sample)
DUMP_SEED = 12345
STAT_FIELDS = ("steps", "sweeps", "exit_oob", "exit_evap", "exit_stall", "pool_drops", "alive")


def dump_outputs(d, ctx, counters, suffix=""):
    """What the last timed step left for a caller of the path: the per-step counters of every timed step
    (water then wind, STAT_FIELDS each), the column checksum of this context's columns as two 32-bit halves, and
    the same seeded sample of cells (x, y) of this context's strip from the height field and from the three
    frequency maps.  Heights are indexed (x - x0) * dimy + y over the strip, frequency maps y * dimx + x over the
    whole map (include/soilmachine_b200.h), so each array is indexed in its own layout."""
    import numpy as np
    os.makedirs(d, exist_ok=True)
    h = ctx.heights().reshape(-1)
    idx = np.arange(h.size)
    if h.size > DUMP_SAMPLE:
        idx = np.sort(np.random.default_rng(DUMP_SEED).choice(h.size, size=DUMP_SAMPLE, replace=False))
    x, y = ctx.x0 + idx // ctx.dimy, idx % ctx.dimy
    cs = ctx.checksum()
    out = {"sample_x": x.astype(np.float64), "sample_y": y.astype(np.float64), "heights": h[idx],
           "column_checksum_hi_lo": np.array([cs >> 32, cs & 0xFFFFFFFF], np.float64),
           "step_counters": np.array(counters, np.float64)}
    fidx = y * ctx.dimx + x
    for k, v in ctx.frequency().items():
        out[k] = v[fidx]
    for name, a in out.items():
        np.save(os.path.join(d, name + suffix + ".npy"), a)


def cpu_arm(W, steps, warmup):
    """The reference's CPU loop on a bounded sample of the workload: 1/CPU_SAMPLE_DIV of the particles of each
    kind per step, i.e. the same water:wind mix as the GPU frame.  Returns (value, info, seconds per step)."""
    from oracle import refapi
    sample = dict(nwater=max(W["nwater"] // CPU_SAMPLE_DIV, 1 if W["nwater"] else 0),
                  nwind=max(W["nwind"] // CPU_SAMPLE_DIV, 1 if W["nwind"] else 0))
    layers = 2.2 if W["soil"] != "rockgravelpebbles_big" else 1.1
    r = refapi.get().init(W["soil"], seed=W["seed"], dimx=W["dim"], dimy=W["dim"],
                          poolsize=int(W["dim"] * W["dim"] * layers + 2000000))
    r.lib.smref_srand(W["seed"])
    tot_steps, tot_s = 0, 0.0
    per = []
    for it in range(warmup + steps):
        sw = r.water_seq(sample["nwater"])          # exactly SoilMachine.cpp:288-298 minus flood
        sd = r.wind_seq(sample["nwind"])            # SoilMachine.cpp:304-307
        t0 = time.perf_counter()
        r.frequency_update()                        # SoilMachine.cpp:313-320
        tf = time.perf_counter() - t0
        if it >= warmup:
            tot_steps += sw.steps + sd.steps
            tot_s += sw.seconds + sd.seconds + tf
            per.append((sw.steps, sw.seconds, sd.steps, sd.seconds))
    val = tot_steps / tot_s if tot_s > 0 else 0.0
    info = {"value": val, "unit": "particle-steps/s", "cores": 1, "kind": "reference",
            "sample": "%d water + %d wind particles per step (1/%d of the frame, same water:wind mix) on the same "
                      "%d^2 %s map, sequential reference loop (SoilMachine.cpp:287-320 without flood/seep), %d steps"
                      % (sample["nwater"], sample["nwind"], CPU_SAMPLE_DIV, W["dim"], W["soil"], steps),
            "water_steps_per_s": sum(p[0] for p in per) / max(sum(p[1] for p in per), 1e-12),
            "wind_steps_per_s": (sum(p[2] for p in per) / max(sum(p[3] for p in per), 1e-12)) if W["nwind"] else None,
            "host_cpus": os.cpu_count()}
    return val, info, tot_s / max(steps, 1)


def make_sim(W, world, local_rank):
    """one unsharded context (world == 1) or this rank's strip of the sharded map"""
    from soilmachine_b200 import host, presets
    maxp = max(W["nwater"], W["nwind"], 1)
    if world == 1:
        sim = host.Simulation(W["soil"], seed=W["seed"], dimx=W["dim"], dimy=W["dim"], device=local_rank,
                              max_particles=maxp)
        return sim, sim.ctx
    from soilmachine_b200 import sharded
    pre = presets.load(W["soil"])
    strip_w = ((((W["dim"] + world - 1) // world) + 15) // 16) * 16
    # a sharded context's pool is exported to the peers and never re-allocated: size it for the initial terrain
    # (one buried section per cell and layer below the top) plus headroom for what erosion creates
    pool = strip_w * W["dim"] * max(len(pre["layers"]), 2) + (4 << 20)
    sim = sharded.DistShard(W["dim"], W["dim"], pre["world"]["scale"], device=local_rank, max_particles=maxp,
                            pool_capacity=pool)
    sim.ctx.set_soils(pre["soils"])
    sim.ctx.initialize(W["seed"], pre["layers"])
    return sim, sim.ctx


def run_frame(ctx, W, xw, xd):
    sw = ctx.water_run(xw) if W["nwater"] else None
    sd = ctx.wind_run(xd) if W["nwind"] else None
    ctx.frequency_update()
    return sw, sd


def quick_config(cid, world, local_rank, barrier, frames=2):
    """BASELINE configs 4 / 5: one warm-up frame, `frames` timed frames with device-resident spawn lists."""
    from soilmachine_b200 import host
    W = CONFIGS[cid]
    sim, ctx = make_sim(W, world, local_rank)
    host.srand(W["seed"])
    lists = [(host.spawn_list(W["nwater"], W["dim"], W["dim"]), host.spawn_list(W["nwind"], W["dim"], W["dim"]))
             for _ in range(1 + frames)]
    run_frame(ctx, W, *lists[0])
    ctx.sync()
    dev = [(ctx.device_spawn(a) if W["nwater"] else None, ctx.device_spawn(b) if W["nwind"] else None)
           for a, b in lists[1:]]
    barrier()
    steps = sweeps = 0
    kms = 0.0
    ctx.timer_start()
    for dw, dd in dev:
        if dw is not None:
            ctx.water_run_device(dw, W["nwater"]); st = ctx.last_stats()
            steps += st.steps; sweeps += st.sweeps; kms += st.device_ms
        if dd is not None:
            ctx.wind_run_device(dd, W["nwind"]); st = ctx.last_stats()
            steps += st.steps
        ctx.frequency_update()
    ms = ctx.timer_stop()
    barrier()
    ms, _, steps, _ = aggregate(ms, 0.0, steps, 0, device="cuda")
    cs = checksum_sum(ctx.checksum(), device="cuda")
    sim.close()
    return {"workload": W["label"], "value": steps / (ms * 1e-3), "unit": "particle-steps/s",
            "ms_per_step": ms / frames, "steps": frames, "warmup": 1, "particle_steps_per_step": steps / frames,
            "water_sweeps_per_step": sweeps / frames, "column_checksum": "%016x" % cs}


def hbm_kernels(ctx, W):
    """the full-grid kernels that ARE bandwidth-bound, timed with CUDA events (best of 5)"""
    peak, _ = hbm_peak()
    cells = W["dim"] * W["dim"]
    out = {}
    best = 1e9
    for _ in range(5):
        ctx.mesh_update(240, download=False)
        best = min(best, ctx.last_stats().device_ms)
    out["k_mesh"] = {"ms": best, "bytes": cells * 76, "gbs": cells * 76 / best / 1e6, "frac_of_hbm_peak": cells * 76 / best / 1e6 / peak,
                     "bytes_per_cell": "32 B top record in + 44 B vertex out"}
    best = 1e9
    for _ in range(5):
        ctx.timer_start(); ctx.frequency_update(); best = min(best, ctx.timer_stop())
    out["k_frequency_update"] = {"ms": best, "bytes": cells * 16, "gbs": cells * 16 / best / 1e6,
                                 "frac_of_hbm_peak": cells * 16 / best / 1e6 / peak,
                                 "bytes_per_cell": "2 x 4 B read + 2 x 4 B written"}
    try:        # the wind field (D3Q19 lattice Boltzmann), far larger than L2: 19 x 4 B in + 19 x 4 B out per cell
        nx, ny, nz = 512, 64, 512
        ctx.lbm_create(nx, ny, nz)
        ctx.lbm_set_boundary(None)
        ctx.lbm_step(3)
        ms = min(ctx.lbm_step(10) for _ in range(3)) / 10
        lc = nx * ny * nz
        out["k_lbm_step"] = {"ms": ms, "bytes": lc * 176, "gbs": lc * 176 / ms / 1e6, "frac_of_hbm_peak": lc * 176 / ms / 1e6 / peak,
                             "lattice": "%dx%dx%d" % (nx, ny, nz), "mlups": lc / ms / 1e3,
                             "bytes_per_cell": "19 x 4 B read + 19 x 4 B written + 4 B flag in + 20 B density/velocity out"}
    except Exception as e:
        out["k_lbm_step"] = {"error": str(e)[:200]}
    best = 1e9
    for _ in range(3):
        best = min(best, ctx.seep().classify_ms)
    if best > 0:
        out["k_hydro_classify"] = {"ms": best, "bytes": cells * 32, "gbs": cells * 32 / best / 1e6,
                                   "frac_of_hbm_peak": cells * 32 / best / 1e6 / peak,
                                   "bytes_per_cell": "32 B top record read (+ buried sections of wet columns)"}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="ours")
    ap.add_argument("--config", type=int, default=3, choices=[3, 4, 5], help="BASELINE.json config the line is measured on")
    ap.add_argument("--dim", type=int, default=0, help="debug: override the map edge")
    ap.add_argument("--particles", type=int, default=0, help="debug: override particles per kind")
    ap.add_argument("--no-cpu", action="store_true", help="skip the cpu_baseline leg")
    ap.add_argument("--no-extra", action="store_true", help="skip configs 4/5 and the full-grid kernels")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="after the timed steps, write what the last one computed to DIR/<name>.npy")
    args = ap.parse_args()

    rank = int(os.environ.get("RANK", "0"))
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    W = dict(CONFIGS[args.config])
    debug = bool(args.dim or args.particles)
    if args.dim:
        W["dim"] = args.dim
    if args.particles:
        W["nwater"] = args.particles if W["nwater"] else 0
        W["nwind"] = args.particles if W["nwind"] else 0
    K, Wm = args.steps, max(args.warmup, 0)
    config = {"workload": W["label"] if not debug else "DEBUG %d^2 %s %d+%d" % (W["dim"], W["soil"], W["nwater"], W["nwind"]),
              "map": "%dx%d" % (W["dim"], W["dim"]), "soil": W["soil"], "seed": W["seed"],
              "water_per_step": W["nwater"], "wind_per_step": W["nwind"],
              "step": "one frame = water batch + wind batch + frequency update, lockstep sweeps",
              "l2": "inputs larger than L2 (column records %.1f GB + pool)" % (W["dim"] * W["dim"] * 32 / 1e9),
              "parallelism": "single GPU" if world == 1 else
              "map sharded into %d x-strips, one per GPU; peer-memory halo/hand-off over NVLink, neighbour-strip flag "
              "barrier per sweep, all strips every 8th sweep" % world}

    # ------------------------------------------------------------------ reference arm (CPU)
    if args.impl == "reference":
        if rank != 0:
            return 0
        val, info, s_per_step = cpu_arm(W, K, Wm)
        line = {"impl": "reference", "metric": "particle-steps/sec", "value": val, "unit": "particle-steps/s",
                "n_gpus": args.gpus, "steps": K, "warmup": Wm, "ms_per_step": s_per_step * 1e3,
                "higher_is_better": True, "scaling": "weak" if args.gpus == 1 else "strong", "vs_baseline": None, "dtype": "f64",
                "data": "synthetic", "config": config, "cpu_baseline": info,
                "e2e": {"value": val, "unit": "particle-steps/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
                "gpu_launches": 0}
        print(json.dumps(line))
        return 0

    # ------------------------------------------------------------------ our arm (GPU)
    import torch
    import torch.distributed as dist
    if not torch.cuda.is_available():
        raise SystemExit("bench.py: no CUDA device - the hot path has no CPU fallback")
    torch.cuda.set_device(local_rank)
    if world > 1:
        dist.init_process_group("nccl", device_id=torch.device("cuda", local_rank))
    from soilmachine_b200 import host

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    sim, ctx = make_sim(W, world, local_rank)
    nframes = Wm + 2 * K                      # warm-up, K device-resident frames, K end-to-end frames
    host.srand(W["seed"])                     # every rank draws the same spawn lists
    lists = [(host.spawn_list(W["nwater"], W["dim"], W["dim"]), host.spawn_list(W["nwind"], W["dim"], W["dim"]))
             for _ in range(nframes + 1)]
    pinned = [(torch.from_numpy(a).pin_memory(), torch.from_numpy(b).pin_memory()) for a, b in lists]

    # warm-up frames (these also advance the simulation: every frame erodes the same map further)
    parity = {"checked": False, "frame1_checksum": None, "against": None}
    for f in range(Wm):
        run_frame(ctx, W, *lists[f])
        if f == 0:
            cs1 = checksum_sum(ctx.checksum(), device="cuda")
            parity["frame1_checksum"] = "%016x" % cs1
            if args.config == 3 and not debug and os.path.exists(GOLDEN_CS):
                with open(GOLDEN_CS) as fh:
                    gold = json.load(fh)
                parity["checked"] = True
                parity["match"] = (int(gold["checksum"], 16) == cs1)
                parity["against"] = "tests/golden/cfg3_frame1_checksum.json = the reference (oracle/_ref) in lockstep on the " \
                                    "same frame, pinned by tests/test_gpu_parity.py::test_config3_frame_matches_reference"
    ctx.sync()

    # ---- value: spawn lists resident in HBM ----
    dev = [(ctx.device_spawn(a) if W["nwater"] else None, ctx.device_spawn(b) if W["nwind"] else None)
           for a, b in lists[Wm:Wm + K]]
    sampler = ClockSampler(local_rank)
    barrier()
    sampler.start()
    launches0 = ctx.launch_count()
    steps_w = steps_d = 0
    ms_w = ms_d = 0.0
    sweeps_w = sweeps_d = 0
    counters = []
    none = [0] * len(STAT_FIELDS)
    ctx.timer_start()
    t0 = time.perf_counter()
    for k in range(K):
        cw = cd = none
        if dev[k][0] is not None:
            ctx.water_run_device(dev[k][0], W["nwater"])
            sw = ctx.last_stats()
            steps_w += sw.steps; ms_w += sw.device_ms; sweeps_w += sw.sweeps
            cw = [getattr(sw, f) for f in STAT_FIELDS]
        if dev[k][1] is not None:
            ctx.wind_run_device(dev[k][1], W["nwind"])
            sd = ctx.last_stats()
            steps_d += sd.steps; ms_d += sd.device_ms; sweeps_d += sd.sweeps
            cd = [getattr(sd, f) for f in STAT_FIELDS]
        ctx.frequency_update()
        counters.append(cw + cd)
    ev_ms = ctx.timer_stop()
    barrier()
    wall_ms = (time.perf_counter() - t0) * 1e3
    launches = ctx.launch_count() - launches0
    clocks = sampler.stop()
    for a, b in dev:
        if a is not None:
            ctx.device_free(a)
        if b is not None:
            ctx.device_free(b)
    if args.dump_outputs:
        dump_outputs(args.dump_outputs, ctx, counters, "" if world == 1 else "_rank%d" % rank)

    # ---- e2e: host buffers through the public C ABI calls ----
    barrier()
    t0 = time.perf_counter()
    e_steps = 0
    for k in range(K):
        a, b = pinned[Wm + K + k]
        sw, sd = run_frame(ctx, W, a.numpy(), b.numpy())
        e_steps += (sw.steps if sw else 0) + (sd.steps if sd else 0)
    ctx.sync()
    barrier()
    e2e_ms = (time.perf_counter() - t0) * 1e3
    h2d = (W["nwater"] + W["nwind"]) * 8
    d2h = ((1 if W["nwater"] else 0) + (1 if W["nwind"] else 0)) * 88   # counter block read back per batch (sm_last_stats)

    parity["final_checksum"] = "%016x" % checksum_sum(ctx.checksum(), device="cuda")
    parity["final_checksum_note"] = "columns after %d frames (warm-up + timed + e2e); equal for every --gpus N" % nframes

    # ---- the latency floor: a sweep that holds one isolated particle (sparse probe batch on the same map) ----
    latency = None
    if world == 1 and W["nwind"]:
        import numpy as np
        probe = np.ascontiguousarray(lists[-1][1][:64])
        st = ctx.wind_run(probe)
        if st.sweeps > 0:
            latency = {"isolated_sweep_us": st.device_ms * 1e3 / st.sweeps, "probe": "64 wind particles, %d sweeps" % st.sweeps}

    # ---- reported beside the metric, outside both timed regions: the rest of the water part of the frame
    # (the batch's floods and the seep pass, SoilMachine.cpp:296,300-301) on the map the frames above left.
    # BASELINE.json's metric excludes flood, so none of this enters `value` or `e2e`.
    hydrology = None
    extra = {}
    if world == 1 and W["nwater"]:
        try:
            sw = ctx.water_run(lists[-1][0])
            hf = ctx.water_flood()
            hs = ctx.seep()
            hydrology = {"water_batch_ms": sw.device_ms, "stalled": sw.exit_stall,
                         "flood_ms": hf.device_ms, "floods": hf.floods, "nested_particles": hf.nested,
                         "flood_transfers": hf.transfers,
                         "seep_ms": hs.device_ms, "seep_cells_visited": hs.cells, "seep_transfers": hs.transfers,
                         "cells": W["dim"] * W["dim"]}
            if not args.no_extra:
                extra["hbm_bound_kernels"] = hbm_kernels(ctx, W)
        except Exception as e:                     # never let the extra report break the bench line
            hydrology = {"error": str(e)[:200]}

    # max over ranks / sums over ranks
    ev_ms, e2e_ms, tot_steps, tot_e = aggregate(ev_ms, e2e_ms, steps_w + steps_d, e_steps, device="cuda")
    value = tot_steps / (ev_ms * 1e-3)
    e2e_val = tot_e / (e2e_ms * 1e-3)
    sim.close()

    # ---- roofline of the dominant kernel (rank 0's launches) ----
    peak, peak_src = hbm_peak()
    kern = [("k_sweep<wind>", steps_d, ms_d, BYTES_WIND, sweeps_d), ("k_sweep<water>", steps_w, ms_w, BYTES_WATER, sweeps_w)]
    kern.sort(key=lambda x: -x[2])
    kname, ksteps, kms, kbytes, ksweeps = kern[0]
    achieved = (ksteps * kbytes / K) / (kms / K * 1e-3) / 1e9 if kms > 0 else 0.0
    roofline = {"bound": "latency", "kernel": kname, "achieved": achieved, "peak": peak, "unit": "GB/s",
                "frac": achieved / peak, "peak_source": peak_src,
                "algorithmic_bytes_per_launch": ksteps * kbytes / K, "launch_ms": kms / K,
                "share_of_step": kms / max(ms_w + ms_d, 1e-9),
                "note": "dependency/latency-bound path (%d dependent sweeps per launch, ~%d B touched per particle-step): "
                        "achieved/peak/frac are the HBM numbers, latency_model is the bound that applies"
                        % (ksweeps // max(K, 1), kbytes),
                "kernels": {n: {"ms_per_step": m / K, "particle_steps_per_step": s / K, "sweeps_per_step": sw / K,
                                "us_per_sweep": (m * 1e3 / sw) if sw else None}
                            for n, s, m, _, sw in kern}}
    if latency is not None and sweeps_d:
        floor_ms = latency["isolated_sweep_us"] * (sweeps_d / K) * 1e-3
        roofline["latency_model"] = dict(latency, kernel="k_sweep<wind>", sweeps_per_launch=sweeps_d / K,
                                         floor_ms=floor_ms, launch_ms=ms_d / K, frac_of_floor=floor_ms / max(ms_d / K, 1e-9),
                                         model="launch time >= sweeps x (duration of a sweep holding one isolated "
                                               "particle); the excess is chains of dependent steps and more particles "
                                               "than resident warps")

    # ---- BASELINE configs 4 and 5 beside the headline (same sharding at N > 1) ----
    if not args.no_extra and not debug and args.config == 3:
        # On a sharded map the extras run the box rule: the exact water schedule is validated across GPUs on the
        # headline config (equal checksums at N = 1 and 2) but was never run on config 4's denser clusters at N > 1
        # within the round's GPU budget, and a side report must not be able to stall the bench line.
        pin_box = world > 1 and "SM_EXACT" not in os.environ
        if pin_box:
            os.environ["SM_EXACT"] = "0"
        try:
            for cid in (4, 5):
                try:
                    extra["config%d" % cid] = quick_config(cid, world, local_rank, barrier)
                    if pin_box:
                        extra["config%d" % cid]["schedule"] = "box rule (SM_EXACT=0)"
                except Exception as e:
                    extra["config%d" % cid] = {"error": str(e)[:300]}
        finally:
            if pin_box:
                del os.environ["SM_EXACT"]

    line = {"metric": "particle-steps/sec", "value": value, "unit": "particle-steps/s", "n_gpus": world,
            "steps": K, "warmup": Wm, "ms_per_step": ev_ms / K, "higher_is_better": True,
            "scaling": "weak" if world == 1 else "strong",
            "vs_baseline": None, "dtype": "f64", "data": "synthetic", "config": config, "clocks": clocks,
            "scaling_note": None if world == 1 else "strong: one %d^2 simulation over %d GPUs" % (W["dim"], world),
            "e2e": {"value": e2e_val, "unit": "particle-steps/s", "h2d_bytes_per_step": h2d,
                    "d2h_bytes_per_step": d2h, "ms_per_step": e2e_ms / K},
            "gpu_launches": launches, "roofline": roofline, "parity": parity, "wall_ms_per_step": wall_ms / K}
    if hydrology is not None:
        line["hydrology"] = hydrology
    if extra:
        line["extra"] = extra

    from oracle import refapi
    if rank == 0 and world == 1 and not args.no_cpu and not refapi.available():
        line["cpu_baseline"] = {"skipped": "oracle/_ref not built (make -C oracle ref needs the reference sources)"}
    elif rank == 0 and world == 1 and not args.no_cpu:
        _, info, _ = cpu_arm(W, 1, 0)
        # like for like: the reference's time for the particle-steps the GPU frame executed, per kind
        rw, rd = info["water_steps_per_s"], info["wind_steps_per_s"]
        cpu_s = (steps_w / K) / rw + ((steps_d / K) / rd if rd else 0.0)
        info["same_steps"] = {"cpu_seconds_for_the_gpu_frame": cpu_s, "gpu_seconds": ev_ms / K * 1e-3,
                              "ratio": cpu_s / (ev_ms / K * 1e-3),
                              "water_ratio": (steps_w / max(ms_w, 1e-9) * 1e3) / rw if ms_w else None,
                              "wind_ratio": (steps_d / max(ms_d, 1e-9) * 1e3) / rd if (rd and ms_d) else None}
        line["cpu_baseline"] = info
    if rank == 0:
        print(json.dumps(line))
    if world > 1:
        dist.destroy_process_group()
    return 0


if __name__ == "__main__":
    sys.exit(main())
