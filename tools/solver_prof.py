#!/usr/bin/env python
"""Per-phase cycle split of the device solver (optimize_gram_kernel) on the bench replan (needs a FUEL_PROF=1 build:
FUEL_PROF=1 python -m fuel_b200.build --force).

Runs the resident replan of bench.py (office map, B trajectories x K evaluations, frontier search beside it) and prints,
per warp and per L-BFGS iteration, the clock64() cycles the solver spent in each phase."""
import argparse
import ctypes as C
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

import bench  # noqa: E402
import fuel_b200  # noqa: E402

PHASES = ("evaluation", "armijo_projection", "reduction_gram_update", "recursion_direction")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=1024)
    ap.add_argument("--evals", type=int, default=64)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--workload", default="office", choices=["office", "office3"])
    args = ap.parse_args()
    so = C.CDLL(fuel_b200._lib.SO)
    if not hasattr(so, "fuelgpu_debug_solver_prof"):
        raise SystemExit("solver_prof.py: libfuelgpu.so was built without FUEL_PROF")
    fn = so.fuelgpu_debug_solver_prof
    buf = (C.c_ulonglong * 8)()
    P = bench.GpuPlanner(0, args.batch, args.evals, workload=args.workload)
    for _ in range(3):
        P.l2_flush()
        P.replan_resident()
    torch.cuda.synchronize()
    fn(buf, 8)  # reset
    for _ in range(args.steps):
        P.l2_flush()
        P.replan_resident()
    torch.cuda.synchronize()
    if fn(buf, 8) != 0:
        raise SystemExit("solver_prof.py: reading the counters failed")
    v = [int(a) for a in buf]
    warps, evals, iters = v[7], v[5], v[6]
    out = {"workload": args.workload, "batch": args.batch, "evals": args.evals, "steps": args.steps,
           "gpu": torch.cuda.get_device_name(0),
           "cycles_per_warp": {k: v[i] / warps for i, k in enumerate(PHASES)},
           "cycles_per_iteration": {k: v[i] / iters for i, k in enumerate(PHASES)},
           "cycles_per_evaluation": v[0] / evals,
           "kernel_cycles_per_warp": v[4] / warps,
           "iterations_per_warp": iters / warps, "evaluations_per_warp": evals / warps}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
