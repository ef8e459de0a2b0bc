#!/usr/bin/env python
"""Device time of the trajectory parameterization (fuelgpu_bspline_parameterize_batch_dev: parameterizeToBspline,
getBoundaryStates(2, 0), pt_dist_) and of the device chain it starts: parameterize -> solve
(fuelgpu_bspline_optimize_batch_dev, K = 64 evaluations, NORMAL_PHASE | MINTIME) -> check
(fuelgpu_bspline_check_batch_dev), against the solver alone.

Batches: B = 1024 on the office map and B = 4096 on office3, each at n = 20 and 64 control points.  The samples are the
benchmark's trajectories (workloads.make_trajectories, its dt draw) sampled at their knots, with noise
(tests/param_cases.workload_samples).  Every timed window is CUDA events on the map's stream after an L2 flush; medians
and the spread of the repetitions are printed.

CPU comparison: the oracle's fp64 parameterization (a dense column-pivoted Householder QR per trajectory plus the
boundary states) over the batch on one host thread.  It is a restatement of the algorithm Eigen's colPivHouseholderQr
names, not Eigen, so it only gives the order of magnitude of what the reference's host loop costs.
One JSON line per batch, then a summary line with the card's name and power limit."""
import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

import fuel_b200  # noqa: E402
import oracle.param  # noqa: E402
from fuel_b200 import workloads as W  # noqa: E402
from fuel_b200._lib import FuelSolveParams, FuelTrajCheckParams, FuelTrajConst  # noqa: E402
from fuel_b200.non_uniform_bspline import REPORT_DTYPE  # noqa: E402
from tests.param_cases import workload_samples  # noqa: E402
from tools.solver_long import card  # noqa: E402

MAX_VEL, MAX_ACC = 2.0, 2.0


def stats(ms):
    return {"median": float(np.median(ms)), "min": float(min(ms)), "max": float(max(ms))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--evals", type=int, default=64)
    args = ap.parse_args()
    dev = card()
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device="cuda")
    rows = []
    for name, mk, B in (("office", W.office_map, 1024), ("office3", W.office3_map, 4096)):
        g, inflate = mk()
        tri = W.office_known(g, inflate)
        m = fuel_b200.SDFMap(g.n, g.res, g.origin, g.box_min, g.box_max, optimistic=True)
        m.occupancy_buffer_inflate_[...] = inflate
        m.setOccupancyBuffer(tristate=tri)
        m.upload()
        st = torch.cuda.Stream()
        torch.cuda.set_stream(st)
        m.set_stream(st.cuda_stream)
        m.updateESDF3d()
        opt = fuel_b200.BsplineOptimizer()
        L = fuel_b200.lib()
        mask = opt.NORMAL_PHASE | opt.MINTIME
        sp = FuelSolveParams()
        sp.max_eval, sp.lbfgs_m, sp.xtol_rel, sp.flags = args.evals, 6, 1e-5, 1  # FUELGPU_SOLVE_EXACT_EVALS
        cp = FuelTrajCheckParams(MAX_VEL, MAX_ACC, 0.0)
        for n in (20, 64):
            pts, der, dt = workload_samples(g, inflate, B, n)
            nvar = 3 * n + 1
            d_pts, d_der, d_dt = (torch.from_numpy(a).cuda() for a in (pts, der, dt))
            d_x = torch.empty((B, nvar), dtype=torch.float64, device="cuda")
            d_x0 = torch.empty_like(d_x)
            d_tc = torch.empty(B * C.sizeof(FuelTrajConst), dtype=torch.uint8, device="cuda")
            d_f = torch.empty(B, dtype=torch.float64, device="cuda")
            d_n = torch.empty(B, dtype=torch.int32, device="cuda")
            d_rep = torch.empty(B * REPORT_DTYPE.itemsize, dtype=torch.uint8, device="cuda")
            d_best = torch.empty(2, dtype=torch.int32, device="cuda")
            vp = lambda t: C.c_void_p(t.data_ptr())  # noqa: E731

            def param():
                rc = L.fuelgpu_bspline_parameterize_batch_dev(m.handle, B, n, nvar, vp(d_pts), vp(d_der), vp(d_dt), None,
                                                              vp(d_x), vp(d_tc))
                assert rc == 0, rc

            def solve():
                rc = L.fuelgpu_bspline_optimize_batch_dev(m.handle, B, n, mask, C.byref(opt.params_), vp(d_tc), C.byref(sp),
                                                          vp(d_x), vp(d_f), vp(d_n))
                assert rc == 0, rc

            def check():
                rc = L.fuelgpu_bspline_check_batch_dev(m.handle, B, n, nvar, vp(d_x), None, C.byref(cp), vp(d_rep),
                                                       vp(d_best))
                assert rc == 0, rc

            def timed(body, prep=None):
                ms = []
                for it in range(args.warmup + args.reps):
                    if prep:
                        prep()
                    flush.zero_()
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record(st)
                    body()
                    e1.record(st)
                    st.synchronize()
                    if it >= args.warmup:
                        ms.append(e0.elapsed_time(e1))
                return ms

            t_param = timed(param)
            d_x0.copy_(d_x)
            x_dev = d_x0.cpu().numpy()
            t_solve = timed(solve, prep=lambda: d_x.copy_(d_x0))
            t_chain = timed(lambda: (param(), solve(), check()))
            if int(d_n.min()) != args.evals:
                raise SystemExit("traj_param.py: the solver stopped early")

            t0 = time.perf_counter()
            x_orc, _ = oracle.param.bspline_parameterize(pts, der, dt)
            cpu_ms = 1e3 * (time.perf_counter() - t0)
            scale = np.maximum(1.0, np.abs(x_orc[:, :3 * n]).max(axis=1))
            err = float((np.abs(x_dev[:, :3 * n] - x_orc[:, :3 * n]).max(axis=1) / scale).max())
            row = {"map": name, "B": B, "n": n, "param_ms": stats(t_param), "solve_ms": stats(t_solve),
                   "chain_ms": stats(t_chain), "reps": args.reps, "max_rel_diff_vs_oracle": err,
                   "cpu_kind": "oracle restatement (dense column-pivoted Householder QR), not Eigen",
                   "cpu_ms_1thread": cpu_ms, "cpu_over_param": cpu_ms / float(np.median(t_param)),
                   "best": [int(v) for v in d_best.cpu().numpy()]}
            rows.append(row)
            print(json.dumps(row), flush=True)
        torch.cuda.synchronize()
        m.close()
    print(json.dumps({"card": dev, "solver_evals": args.evals,
                      "columns": ["map", "B", "n", "param_ms", "solve_ms", "chain_ms", "cpu_ms_1thread"],
                      "table": [[r["map"], r["B"], r["n"], round(r["param_ms"]["median"], 4),
                                 round(r["solve_ms"]["median"], 4), round(r["chain_ms"]["median"], 4),
                                 round(r["cpu_ms_1thread"], 1)] for r in rows]}))


if __name__ == "__main__":
    main()
