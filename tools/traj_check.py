#!/usr/bin/env python
"""Device time of the trajectory check (fuelgpu_bspline_check_batch_dev: NonUniformBspline checks, checkTrajCollision,
selectBestTraj) on the solver's output, against the reference's own code on one host thread.

Batches: B = 1024 at n = 20 on the office map, B = 4096 at n = 20 and 64 on office3 (K = 64 solver evaluations,
NORMAL_PHASE | MINTIME, as tools/solver_long.py).  The check is timed with CUDA events on the map's stream around the
_dev entry, after an L2 flush; median and spread of the repetitions are printed.

CPU comparison: the reference's NonUniformBspline (getTimeSum, getJerk, checkRatio, checkFeasibility), its
checkTrajCollision loop on its SDFMap and selectBestTraj (oracle/_ref/libfuel_ref_traj.so, built by build()) over the
whole batch on one host thread, called once per trajectory through ctypes.  Without oracle/_ref the oracle's restatement is timed instead and labelled "port".  One JSON line per batch,
then a summary line with the card's name and power limit."""
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

import bench  # noqa: E402
import fuel_b200  # noqa: E402
import oracle  # noqa: E402
import oracle.traj  # noqa: E402
from fuel_b200 import workloads as W  # noqa: E402
from fuel_b200._lib import FuelTrajCheckParams  # noqa: E402
from fuel_b200.non_uniform_bspline import REPORT_DTYPE, check_batch  # noqa: E402
from tools.solver_long import card, ref_setup  # noqa: E402

MAX_VEL, MAX_ACC = 2.0, 2.0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--evals", type=int, default=64)
    args = ap.parse_args()
    dev = card()
    oracle.traj.build()
    use_ref = oracle.traj.ref_traj() is not None
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device="cuda")
    rows = []
    for name, mk, B, n in (("office", W.office_map, 1024, 20), ("office3", W.office3_map, 4096, 20),
                           ("office3", W.office3_map, 4096, 64)):
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
        env = fuel_b200.EDTEnvironment()
        env.setMap(m)
        opt = fuel_b200.BsplineOptimizer()
        opt.setEnvironment(env)
        tr = W.make_trajectories(g, inflate, B=B, n_pts=n)
        tcs = opt.traj_consts_from_arrays(tr["pt_dist"], tr["dt"], tr["start"], tr["end_pos"])
        x, _, _ = opt.optimizeBatch(W.pack_x(tr["ctrl"], tr["dt"]), tcs, n, opt.NORMAL_PHASE | opt.MINTIME, args.evals)
        d_x = torch.from_numpy(x).cuda()
        d_rep = torch.empty(B * REPORT_DTYPE.itemsize, dtype=torch.uint8, device="cuda")
        d_best = torch.empty(2, dtype=torch.int32, device="cuda")
        p = FuelTrajCheckParams(MAX_VEL, MAX_ACC, 0.0)
        L = fuel_b200.lib()
        ms = []
        for it in range(args.warmup + args.reps):
            flush.zero_()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(st)
            rc = L.fuelgpu_bspline_check_batch_dev(m.handle, B, n, 3 * n + 1, C.c_void_p(d_x.data_ptr()), None, C.byref(p),
                                                   C.c_void_p(d_rep.data_ptr()), C.c_void_p(d_best.data_ptr()))
            e1.record(st)
            if rc != 0:
                raise SystemExit("traj_check.py: fuelgpu_bspline_check_batch_dev returned %d" % rc)
            st.synchronize()
            if it >= args.warmup:
                ms.append(e0.elapsed_time(e1))
        rep = d_rep.cpu().numpy().view(REPORT_DTYPE)
        host_rep, best = check_batch(m, x, n, max_vel=MAX_VEL, max_acc=MAX_ACC)
        if rep.tobytes() != host_rep.tobytes() or not np.array_equal(d_best.cpu().numpy(), best):
            raise SystemExit("traj_check.py: the _dev and host entries disagree")

        # CPU: the reference's code on one host thread over the whole batch
        ctrl, dt = x[:, :3 * n].reshape(B, n, 3), x[:, 3 * n].copy()
        if use_ref:
            ref = ref_setup(g)
            ref.inflate[:] = inflate.reshape(-1)

            def cpu_run():
                for b in range(B):
                    oracle.traj.ref_traj_stats(ctrl[b], dt[b], MAX_VEL, MAX_ACC)
                    oracle.traj.ref_traj_check_collision(ref, ctrl[b], dt[b], 0.0)
                oracle.traj.ref_traj_select_best(ctrl, dt)
        else:
            og = oracle.make_grid(g.n, g.res, g.origin, g.box_min, g.box_max)

            def cpu_run():
                oracle.traj.bspline_check(og, inflate.astype(np.int8), x, n, MAX_VEL, MAX_ACC)
        t0 = time.perf_counter()
        with bench._Quiet():
            cpu_run()
        cpu_ms = 1e3 * (time.perf_counter() - t0)
        med = float(np.median(ms))
        row = {"map": name, "B": B, "n": n, "ms_median": med, "ms_min": float(min(ms)), "ms_max": float(max(ms)),
               "reps": len(ms), "samples_mean": float(rep["n_checked"].mean()), "samples_max": int(rep["n_checked"].max()),
               "unsafe": int((rep["safe"] == 0).sum()), "infeasible": int((rep["feasible"] == 0).sum()),
               "best": [int(v) for v in best], "cpu_kind": "reference" if use_ref else "port",
               "cpu_ms_1thread": cpu_ms, "speedup_vs_1thread": cpu_ms / med}
        rows.append(row)
        print(json.dumps(row), flush=True)
        torch.cuda.synchronize()
        m.close()
        if use_ref:
            ref.close()
    print(json.dumps({"card": dev, "limits": {"max_vel": MAX_VEL, "max_acc": MAX_ACC}, "solver_evals": args.evals,
                      "table": [[r["map"], r["B"], r["n"], round(r["ms_median"], 4), round(r["cpu_ms_1thread"], 1),
                                 round(r["speedup_vs_1thread"], 1)] for r in rows],
                      "columns": ["map", "B", "n", "ms_median", "cpu_ms_1thread", "speedup_vs_1thread"]}))


if __name__ == "__main__":
    main()
