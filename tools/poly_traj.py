#!/usr/bin/env python
"""Device time of the waypoint-polynomial stage (fuelgpu_poly_waypoints_batch: segment times, waypointsTraj,
getTotalTime, getLength, seg_num, dt, the samples and boundary derivatives of planExploreTraj :270-297) and wall time of
the whole plan_explore_traj_batch chain (polynomial -> host read of info -> per-n_pts-group parameterize / solve
(NORMAL_PHASE | MINTIME, 64 evaluations) / check), against the same polynomial stage on one host thread: the oracle's
restatement of the reference's dense waypointsTraj, and the reference's own polynomial_traj.cpp where oracle/_ref is
built.

Batches: B = 1024 tours on the office map and B = 4096 on office3 (workloads.make_tours).  The device time is the
map's slot-7 CUDA events around the kernel, after an L2 flush; medians and the spread of the repetitions are printed.
One JSON line per batch, then a summary line with the card's name and power limit."""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

import fuel_b200  # noqa: E402
import oracle.poly as OP  # noqa: E402
from fuel_b200 import workloads as W  # noqa: E402
from fuel_b200.polynomial_traj import plan_explore_traj_batch, waypoints_batch  # noqa: E402
from fuel_b200.sdf_map import EDTEnvironment  # noqa: E402
from tests.helpers import make_sdf_map  # noqa: E402
from tools.solver_long import card  # noqa: E402

LIM = dict(max_vel=2.0, max_acc=2.0)


def stats(ms):
    ms = np.asarray(ms)
    return dict(median=float(np.median(ms)), min=float(ms.min()), max=float(ms.max()))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--cpu-tours", type=int, default=256, help="tours timed on the host (scaled to B)")
    a = ap.parse_args()
    fuel_b200.lib()
    dev = card()
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device="cuda")
    for which, B in (("office", 1024), ("office3", 4096)):
        g, inflate = W.office_map() if which == "office" else W.office3_map()
        m = make_sdf_map(fuel_b200, g, inflate, np.where(inflate == 1, W.OCCUPIED, W.FREE).astype(np.uint8))
        tr = W.make_tours(g, inflate, B=B)
        args = (m, tr["tours"], tr["start_vel"], tr["start_acc"])
        waypoints_batch(*args)  # warm-up
        dev_ms = []
        for _ in range(a.reps):
            flush.zero_()
            torch.cuda.synchronize()
            info, _, _, _ = waypoints_batch(*args, with_coeffs=False)
            dev_ms.append(m.last_timing()["poly"])
        opt = fuel_b200.BsplineOptimizer()
        opt.setParam()
        env = EDTEnvironment()
        env.setMap(m)
        opt.setEnvironment(env)
        solve = dict(cost_function=opt.NORMAL_PHASE | opt.MINTIME, max_eval=64)
        plan_explore_traj_batch(*args, -1.0, opt, solve, LIM)
        chain_ms = []
        for _ in range(max(3, a.reps // 4)):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            out = plan_explore_traj_batch(*args, -1.0, opt, solve, LIM)
            chain_ms.append((time.perf_counter() - t0) * 1e3)
        n = min(B, a.cpu_tours)
        host = {}
        for name, ref in (("oracle", False), ("reference", True)):
            if ref and OP.ref_poly() is None:
                continue
            t0 = time.perf_counter()
            for b in range(n):
                OP.explore_samples(tr["tours"][b], tr["start_vel"][b], tr["start_acc"][b], ref=ref)
            host[name + "_ms_per_batch"] = (time.perf_counter() - t0) * 1e3 * B / n
        groups = sorted(set(info["n_pts"][info["status"] == 0].tolist()))
        row = dict(map=which, B=B, poly_device_ms=stats(dev_ms), chain_wall_ms=stats(chain_ms), n_groups=len(groups),
                   n_pts_range=[groups[0], groups[-1]], too_long=int((info["status"] == 1).sum()),
                   best=out["best"].tolist(), host_one_thread=host, host_tours_timed=n)
        print(json.dumps(row), flush=True)
        m.close()
    print(json.dumps(dict(card=dev)), flush=True)


if __name__ == "__main__":
    main()
