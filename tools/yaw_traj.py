#!/usr/bin/env python
"""Device time of the exploration-yaw stage (fuelgpu_yaw_explore_batch_dev: planYawExplore on every trajectory of a
solver batch) and of the device chain solve -> check with and without it, against the oracle's restatement of the
stage on one host thread (its construction in Python plus a dense fp64 solve per trajectory; NLopt is not part of the
reference build the oracle compiles, so the reference's own yaw time is not measured).

Batches: B = 1024 trajectories of 20 points on the office map and B = 4096 of 64 points on office3, the solver's output
(NORMAL_PHASE | MINTIME, 64 evaluations) of workloads.make_trajectories, yaws from workloads.make_yaws.  The map runs on
a torch stream (SDFMap.set_stream); CUDA events on it time --launches back-to-back launches of the _dev entry after a
warm-up, and --reps runs of the chain, each from the same initial x.  One JSON line per batch, then the card's name and
power limit."""
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
import oracle.yaw as OY  # noqa: E402
from fuel_b200 import workloads as W  # noqa: E402
from fuel_b200._lib import FuelSolveParams, FuelTrajCheckParams, FuelYawParams  # noqa: E402
from fuel_b200.non_uniform_bspline import REPORT_DTYPE  # noqa: E402
from fuel_b200.polynomial_traj import YAW_INFO_DTYPE  # noqa: E402
from tests.helpers import make_sdf_map  # noqa: E402
from tools.solver_long import card  # noqa: E402


def stats(ms):
    ms = np.asarray(ms)
    return dict(median=float(np.median(ms)), min=float(ms.min()), max=float(ms.max()))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--reps", type=int, default=20)
    a = ap.parse_args()
    L = fuel_b200.lib()
    dev = card()
    for which, B, n in (("office", 1024, 20), ("office3", 4096, 64)):
        g, inflate = W.office_map() if which == "office" else W.office3_map()
        m = make_sdf_map(fuel_b200, g, inflate, W.office_known(g, inflate), optimistic=True)
        st = torch.cuda.Stream()
        m.set_stream(st.cuda_stream)
        m.updateESDF3d()
        env = fuel_b200.EDTEnvironment()
        env.setMap(m)
        opt = fuel_b200.BsplineOptimizer()
        opt.setEnvironment(env)
        mask = opt.NORMAL_PHASE | opt.MINTIME
        tr = W.make_trajectories(g, inflate, B=B, n_pts=n)
        tcs = opt.traj_consts_from_arrays(tr["pt_dist"], tr["dt"], tr["start"], tr["end_pos"])
        x0 = W.pack_x(tr["ctrl"], tr["dt"])
        x, _, _ = opt.optimizeBatch(x0, tcs, n, mask, 64)
        ys = W.make_yaws(B)
        nvar = 3 * n + 1
        with torch.cuda.stream(st):
            cu = lambda v: torch.from_numpy(np.ascontiguousarray(v)).cuda()  # noqa: E731
            d_x, d_x0, d_sy, d_ey = cu(x), cu(x0), cu(ys["start"]), cu(ys["end"])
            d_tc = cu(np.frombuffer(tcs, dtype=np.uint8).copy())
            d_f = torch.empty(B, dtype=torch.float64, device="cuda")
            d_ne = torch.empty(B, dtype=torch.int32, device="cuda")
            d_rep = torch.empty(B * REPORT_DTYPE.itemsize, dtype=torch.uint8, device="cuda")
            d_best = torch.empty(2, dtype=torch.int32, device="cuda")
            d_yaw = torch.empty((B, 15), dtype=torch.float64, device="cuda")
            d_info = torch.empty(B * YAW_INFO_DTYPE.itemsize, dtype=torch.uint8, device="cuda")
        st.synchronize()
        yp = FuelYawParams(1.0, 1, 0)
        sp = FuelSolveParams()
        sp.max_eval, sp.lbfgs_m, sp.xtol_rel = 64, 6, 1e-5
        cp = FuelTrajCheckParams(2.0, 2.0, 0.0)

        def yaw(xp):
            assert L.fuelgpu_yaw_explore_batch_dev(m.handle, B, n, nvar, xp.data_ptr(), None, d_sy.data_ptr(),
                                                   d_ey.data_ptr(), C.byref(opt.params_), C.byref(yp),
                                                   d_yaw.data_ptr(), d_info.data_ptr(), None) == 0

        for _ in range(10):
            yaw(d_x)
        st.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        per = []
        for _ in range(5):
            e0.record(st)
            for _ in range(a.launches):
                yaw(d_x)
            e1.record(st)
            e1.synchronize()
            per.append(e0.elapsed_time(e1) / a.launches)
        info = np.frombuffer(d_info.cpu().numpy().tobytes(), dtype=YAW_INFO_DTYPE)

        d_xc = torch.empty_like(d_x0)

        def chain(with_yaw):
            d_xc.copy_(d_x0)
            assert L.fuelgpu_bspline_optimize_batch_dev(m.handle, B, n, mask, C.byref(opt.params_), d_tc.data_ptr(),
                                                        C.byref(sp), d_xc.data_ptr(), d_f.data_ptr(),
                                                        d_ne.data_ptr()) == 0
            assert L.fuelgpu_bspline_check_batch_dev(m.handle, B, n, nvar, d_xc.data_ptr(), None, C.byref(cp),
                                                     d_rep.data_ptr(), d_best.data_ptr()) == 0
            if with_yaw:
                yaw(d_xc)

        res = {}
        for with_yaw in (False, True, False, True):  # warm-up of both forms
            with torch.cuda.stream(st):
                chain(with_yaw)
            st.synchronize()
        for with_yaw in (False, True):
            ms = []
            for _ in range(a.reps):
                with torch.cuda.stream(st):
                    e0.record(st)
                    chain(with_yaw)
                    e1.record(st)
                e1.synchronize()
                ms.append(e0.elapsed_time(e1))
            res["with_yaw" if with_yaw else "without_yaw"] = stats(ms)

        t = time.perf_counter()
        rows = OY.plan(x, n, ys["start"], ys["end"])
        for r in rows:
            if r["status"] == 0:
                OY.solve(r)
        host_ms = (time.perf_counter() - t) * 1e3
        print(json.dumps(dict(batch=which, B=B, n_pts=n, yaw_dev_ms=stats(per), chain_solve_check_ms=res,
                              oracle_host_ms=host_ms, statuses=np.bincount(info["status"], minlength=6).tolist(),
                              reference_yaw_ms="not measured (NLopt is not built)")))
        m.close()
    print(json.dumps(dict(card=dev)))


if __name__ == "__main__":
    main()
