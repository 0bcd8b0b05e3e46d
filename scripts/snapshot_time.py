"""Time snapshots against the host checkpoint path at the benchmark's size (DESIGN.md section 10).

After one frame of config 3 (4096^2 rockgravelpebblessand, 25k water + 25k wind particles, seed 42) the script times,
in alternating rounds so that drift on a shared machine hits every arm alike:
  save    sm_snapshot_save to device memory (sm_device_alloc), to pinned host memory, to pageable host memory;
  restore sm_snapshot_restore from each of the three;
  host    sm_download_columns + sm_get_frequency, and sm_upload_columns + sm_set_frequency (the checkpoint path
          INTEGRATION.md listed before snapshots existed).
Every call returns after a device synchronise, so the host clock around it is the call's whole time.  The CUDA-event
stopwatch (sm_timer_start / _stop) around the same call gives the span on the context's stream, host gaps included.
Each restore is checked: the map saved again is the same snapshot.

  python scripts/snapshot_time.py [--rounds 5] [--dim 4096] [--json out.json]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from soilmachine_b200 import host  # noqa: E402


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except OSError:
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--dim", type=int, default=4096)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    import torch
    sim = host.Simulation("rockgravelpebblessand", seed=42, dimx=args.dim, dimy=args.dim, max_particles=25000)
    sim.frame(25000, 25000)
    c = sim.ctx
    lib = c.lib
    n = c.snapshot_bytes()
    ref = c.snapshot()
    pinned = torch.empty(n, dtype=torch.uint8, pin_memory=True).numpy()
    pageable = np.empty(n, np.uint8)
    dptr = C.c_void_p()
    c._ck_strict(lib.sm_device_alloc(c.h, C.c_int64(n), C.byref(dptr)))
    cols, freq = c.download_columns(), c.frequency()

    def timed(fn):
        c.timer_start()
        t0 = time.perf_counter()
        fn()
        host_ms = (time.perf_counter() - t0) * 1e3
        return host_ms, c.timer_stop()

    def save(dst, on_dev):
        p = dst if on_dev else dst.ctypes.data_as(C.c_void_p)
        return lambda: c._ck_strict(lib.sm_snapshot_save(c.h, p, C.c_int64(n), int(on_dev)))

    def restore(src, on_dev):
        p = src if on_dev else src.ctypes.data_as(C.c_void_p)
        return lambda: c._ck_strict(lib.sm_snapshot_restore(c.h, p, C.c_int64(n), int(on_dev)))

    def host_save():
        cols.update(c.download_columns())
        freq.update(c.frequency())

    def host_restore():
        c.upload_columns(cols["offsets"], cols["type"], cols["size"], cols["saturation"])
        c.set_frequency(**freq)

    arms = [("save device", save(dptr, True)), ("save pinned", save(pinned, False)), ("save pageable", save(pageable, False)),
            ("restore device", restore(dptr, True)), ("restore pinned", restore(pinned, False)),
            ("restore pageable", restore(pageable, False)),
            ("download_columns + get_frequency", host_save), ("upload_columns + set_frequency", host_restore)]
    for _, fn in arms:          # warm-up: every shape once
        fn()
    times = {k: [] for k, _ in arms}
    for r in range(args.rounds):
        order = arms if r % 2 == 0 else arms[::-1]
        for k, fn in order:
            times[k].append(timed(fn))
            if k.startswith("restore") or k.startswith("upload"):
                assert c.snapshot().tobytes() == ref.tobytes(), k + ": the restored map is not the saved one"
    gpu = gpu_info()
    h = {"gpu (name, power limit)": gpu, "dim": args.dim, "snapshot_bytes": n,
         "sections": int(cols["offsets"][-1]), "rounds": args.rounds, "arms": {}}
    print("snapshot timing on %s, %d^2, %d sections, %.1f MB snapshot, %d rounds (median, min) ms"
          % (gpu, args.dim, h["sections"], n / 1e6, args.rounds))
    for k, _ in arms:
        hm = np.array([t[0] for t in times[k]]); em = np.array([t[1] for t in times[k]])
        h["arms"][k] = {"host_ms": hm.tolist(), "event_ms": em.tolist()}
        print("  %-34s host %9.2f %9.2f   events %9.2f %9.2f" % (k, np.median(hm), hm.min(), np.median(em), em.min()))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(h, f, indent=1)
    lib.sm_device_free(c.h, dptr)
    sim.close()


if __name__ == "__main__":
    main()
