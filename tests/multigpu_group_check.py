"""A context group with ONE RANK PER GPU, in one process (no torchrun): the cross-device path of sm_create_group -
peer access enabled between the devices, raw peer pointers, the device spawn list copied between devices - against one
unsharded context on device 0.  Runs the frame check (three frames with the pooling hydrology and the wind batch,
budget flags on, compared after every phase) and the single-cell check of tests/_group.py, both byte for byte.

    python tests/multigpu_group_check.py --gpus N

Prints one JSON line; exits 0 with "skipped": "fewer than N devices" where there are not enough GPUs, 1 on a difference.
"""
import argparse
import json
import os
import sys
import traceback

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=2)
    args = ap.parse_args()
    import torch
    have = torch.cuda.device_count()
    out = {"check": "multigpu_group_check", "gpus": args.gpus, "devices_present": have}
    if have < args.gpus:
        out["skipped"] = "fewer than %d devices" % args.gpus
        print(json.dumps(out), flush=True)
        return 0
    import _group
    devices = list(range(args.gpus))
    try:
        out["floods"] = _group.check_frames("bigbutte", 48 * args.gpus, 72, 700, 300, devices)
        _group.check_frames("rockgravelpebblessand", 64 * args.gpus, 80, 900, 700, devices)
        _group.check_cell_ops(devices)
        out["result"] = "every phase IDENTICAL to one context"
    except Exception as e:      # a difference (AssertionError) or a library error: report it in the line
        out["result"] = "FAILED: %s" % e
        traceback.print_exc()
    print(json.dumps(out), flush=True)
    return 0 if out["result"].startswith("every") else 1


if __name__ == "__main__":
    sys.exit(main())
