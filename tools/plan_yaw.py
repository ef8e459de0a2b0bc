#!/usr/bin/env python
"""Device time of the kinodynamic replan's yaw (fuelgpu_plan_yaw_batch_dev: planYaw on every trajectory of a solver
batch) and of the device chain optimize -> plan_yaw against optimize alone, and the oracle's restatement of the stage on
one host thread (its construction in Python plus a dense fp64 solve per trajectory; NLopt is not part of the reference
build the oracle compiles, so the reference's own yaw time is not measured).

Batches: B = 1024 kinodynamic-replan trajectories on the office map and B = 4096 on office3: MID rows of device path
searches (workloads.make_path_queries / make_kino_queries), kinodynamicReplan's search and parameterization
(kino_astar.kinodynamic_replan_batch), then the solver (NORMAL_PHASE | MINTIME, 64 evaluations, kino_algorithm.xml's
weights), one launch per point count.  The map runs on a torch stream (SDFMap.set_stream); CUDA events on it time
--launches back-to-back passes of the _dev entry over every group after a warm-up, and --reps runs of the chain, each
from the same initial x.  One JSON line per batch, then the card's name and power limit."""
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
import oracle.plan_yaw as OPY  # noqa: E402
from fuel_b200 import workloads as W  # noqa: E402
from fuel_b200._lib import FuelSolveParams, FuelTrajConst  # noqa: E402
from fuel_b200.astar import astar_batch  # noqa: E402
from fuel_b200.kino_astar import kinodynamic_replan_batch  # noqa: E402
from fuel_b200.polynomial_traj import PLANYAW_INFO_DTYPE, PLANYAW_MAX_PTS  # noqa: E402
from tests.helpers import make_sdf_map  # noqa: E402
from tests.plan_yaw_cases import LD_KINO  # noqa: E402
from tools.solver_long import card  # noqa: E402


def stats(ms):
    ms = np.asarray(ms)
    return dict(median=float(np.median(ms)), min=float(ms.min()), max=float(ms.max()))


def replan_groups(m, g, inflate, tri, B):
    """(n, x0 [k, 3n+1], traj consts as bytes [k, sizeof]) per point count, B rows in all"""
    groups, have, seed = {}, 0, 1
    while have < B:
        q = W.make_path_queries(g, inflate, tri, B=4096, seed=seed)
        info = astar_batch(m, q["start"], q["goal"], resolution=0.4, lambda_heu=10000.0, allocate_num=40000,
                           max_iter=100000, path_max=0)[0]
        kq = W.make_kino_queries(g, inflate, tri, info, q["start"], q["goal"], seed=seed + 1)
        _, gr = kinodynamic_replan_batch(m, kq["start"], kq["vel"], kq["acc"], kq["goal"])
        for rows, x0, tc in gr:
            k = min(len(rows), B - have)
            if k <= 0:
                break
            n = (x0.shape[1] - 1) // 3
            tcb = np.frombuffer(tc, dtype=np.uint8).reshape(len(rows), -1)[:k]
            old = groups.get(n)
            groups[n] = (x0[:k], tcb) if old is None else (np.vstack([old[0], x0[:k]]), np.vstack([old[1], tcb]))
            have += k
        seed += 2
    return [(n,) + groups[n] for n in sorted(groups)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=100)
    ap.add_argument("--reps", type=int, default=20)
    a = ap.parse_args()
    L = fuel_b200.lib()
    dev = card()
    for which, B in (("office", 1024), ("office3", 4096)):
        g, inflate = W.office_map() if which == "office" else W.office3_map()
        tri = W.office_known(g, inflate)
        m = make_sdf_map(fuel_b200, g, inflate, tri)
        st = torch.cuda.Stream()
        m.set_stream(st.cuda_stream)
        m.updateESDF3d()
        env = fuel_b200.EDTEnvironment()
        env.setMap(m)
        opt = fuel_b200.BsplineOptimizer()
        opt.setParam(ld_feasi=1.0, ld_time=0.1, dist0=0.4, **LD_KINO)  # kino_algorithm.xml:128-139
        opt.setEnvironment(env)
        mask = opt.NORMAL_PHASE | opt.MINTIME
        groups = replan_groups(m, g, inflate, tri, B)
        sy = W.make_yaws(B)["start"]
        sp = FuelSolveParams()
        sp.max_eval, sp.lbfgs_m, sp.xtol_rel = 64, 6, 1e-5
        dg, xs, off = [], [], 0
        for n, x0, tcb in groups:
            k = len(x0)
            tc = (FuelTrajConst * k).from_buffer_copy(tcb.tobytes())
            x, _, _ = opt.optimizeBatch(x0, tc, n, mask, 64)
            xs.append((n, x, sy[off:off + k]))
            with torch.cuda.stream(st):
                cu = lambda v: torch.from_numpy(np.ascontiguousarray(v)).cuda()  # noqa: E731
                dg.append(dict(n=n, k=k, x=cu(x), x0=cu(x0), xc=cu(x0), tc=cu(tcb), sy=cu(sy[off:off + k]),
                               f=torch.empty(k, dtype=torch.float64, device="cuda"),
                               ne=torch.empty(k, dtype=torch.int32, device="cuda"),
                               yaw=torch.empty((k, PLANYAW_MAX_PTS), dtype=torch.float64, device="cuda"),
                               info=torch.empty(k * PLANYAW_INFO_DTYPE.itemsize, dtype=torch.uint8, device="cuda")))
            off += k
        st.synchronize()

        def yaw(d, xp):
            assert L.fuelgpu_plan_yaw_batch_dev(m.handle, d["k"], d["n"], 3 * d["n"] + 1, xp.data_ptr(), None,
                                                d["sy"].data_ptr(), C.byref(opt.params_), d["yaw"].data_ptr(),
                                                d["info"].data_ptr(), None) == 0

        def chain(with_yaw):
            for d in dg:
                d["xc"].copy_(d["x0"])
                assert L.fuelgpu_bspline_optimize_batch_dev(m.handle, d["k"], d["n"], mask, C.byref(opt.params_),
                                                            d["tc"].data_ptr(), C.byref(sp), d["xc"].data_ptr(),
                                                            d["f"].data_ptr(), d["ne"].data_ptr()) == 0
                if with_yaw:
                    yaw(d, d["xc"])

        for _ in range(10):
            for d in dg:
                yaw(d, d["x"])
        st.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        per = []
        for _ in range(5):
            e0.record(st)
            for _ in range(a.launches):
                for d in dg:
                    yaw(d, d["x"])
            e1.record(st)
            e1.synchronize()
            per.append(e0.elapsed_time(e1) / a.launches)
        info = np.concatenate([np.frombuffer(d["info"].cpu().numpy().tobytes(), dtype=PLANYAW_INFO_DTYPE) for d in dg])

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
        for n, x, s in xs:
            for r in OPY.plan_yaw(x, n, s):
                if r["status"] == 0:
                    OPY.solve(r, **LD_KINO)
        host_ms = (time.perf_counter() - t) * 1e3
        print(json.dumps(dict(batch=which, B=B, groups=[[n, len(x)] for n, x, _ in xs],
                              seg_num=dict(min=int(info["seg_num"].min()), median=float(np.median(info["seg_num"])),
                                           max=int(info["seg_num"].max())),
                              plan_yaw_dev_ms=stats(per), chain_optimize_ms=res, oracle_host_ms=host_ms,
                              statuses=np.bincount(info["status"], minlength=7).tolist(),
                              reference_yaw_ms="not measured (NLopt is not built)")))
        m.close()
    print(json.dumps(dict(card=dev)))


if __name__ == "__main__":
    main()
