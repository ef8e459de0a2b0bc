#!/usr/bin/env python
"""Device time of refineLocalTour (fuelgpu_local_tour_batch_dev: every edge's ViewNode::computeCost, the Dijkstra
search, the refined tour's searches) against the same problems on one host thread in the oracle's restatement
(oracle/fuel_oracle_tour.c, which costs the edges lazily as the reference does) and, where
oracle/_ref/libfuel_ref_tour.so is built, in the reference's own compiled refineLocalTour.  Workloads: the office sequence's
refine (searchFrontiers -> computeFrontiersToVisit -> getTopViewpointsInfo -> getFullCostMatrix -> the clusters in
order of their row-0 cost standing for LKH -> select_refined_ids -> getViewpointsInfo, B = 1), then B = 256 problems of
workloads.make_local_tours on office and office3.  ViewNode's defaults (vm 2.0, yd 60 deg, w_dir 1.5, lambda 10000,
allocate_num 1 000 000, max_iter 10000), tour_lambda_heu 1.0.  The device time is CUDA events around the call on the
map's stream (inputs on the device, outputs left there), median over the repetitions after one warm-up.  One JSON line
per workload with the edges costed eagerly and the costTo calls of the reference's lazy search, then a summary line
with the card's name and power limit."""
import argparse
import contextlib
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
import oracle.astar as OA  # noqa: E402
import oracle.tour as OT  # noqa: E402
from fuel_b200 import exploration_manager as EM  # noqa: E402
from fuel_b200 import workloads as W  # noqa: E402
from fuel_b200._lib import FuelAstarParams, FuelLocalTourParams, FuelViewCostParams, lib  # noqa: E402
from fuel_b200.view_node import ViewNode  # noqa: E402
from tests.helpers import make_sdf_map  # noqa: E402
from tools.solver_long import card  # noqa: E402

TOUR_MAX = 2048


@contextlib.contextmanager
def quiet_stdout():
    """the reference's code prints to stdout (std::cout): keep it out of the JSON lines"""
    sys.stdout.flush()
    saved = os.dup(1)
    devnull = os.open(os.devnull, os.O_WRONLY)
    os.dup2(devnull, 1)
    try:
        yield
    finally:
        C.CDLL(None).fflush(None)  # what C stdio (and std::cout through it) still buffers goes to /dev/null too
        os.dup2(saved, 1)
        os.close(saved)
        os.close(devnull)


def device_ms(m, w, prm, reps):
    B = len(w["prob_off"]) - 1
    kmax = int(np.diff(w["prob_off"]).max())
    dev = torch.device("cuda")
    t = {k: torch.tensor(np.ascontiguousarray(w[k], np.float64), device=dev)
         for k in ("cur_pos", "cur_vel", "cur_yaw", "vp_pos", "vp_yaw")}
    po, go = (np.ascontiguousarray(w[k], np.int32) for k in ("prob_off", "group_off"))
    dinfo = torch.zeros(B * EM.TOUR_INFO_DTYPE.itemsize, dtype=torch.uint8, device=dev)
    dref = torch.zeros((B, kmax), dtype=torch.int32, device=dev)
    dtour = torch.zeros((B, TOUR_MAX, 3), dtype=torch.float64, device=dev)
    stream = torch.cuda.Stream()
    m.set_stream(stream.cuda_stream)
    torch.cuda.synchronize()
    ms = []
    for r in range(reps + 1):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        rc = lib().fuelgpu_local_tour_batch_dev(m.handle, B, po.ctypes.data, go.ctypes.data, t["cur_pos"].data_ptr(),
                                                t["cur_vel"].data_ptr(), t["cur_yaw"].data_ptr(),
                                                t["vp_pos"].data_ptr(), t["vp_yaw"].data_ptr(), C.byref(prm),
                                                dinfo.data_ptr(), kmax, dref.data_ptr(), TOUR_MAX, dtour.data_ptr(),
                                                None)
        e1.record(stream)
        assert rc == 0
        torch.cuda.synchronize()
        if r:  # the first call grows and fills the scratch
            ms.append(e0.elapsed_time(e1))
    m.set_stream(0)
    return float(np.median(ms)), np.frombuffer(dinfo.cpu().numpy().tobytes(), dtype=EM.TOUR_INFO_DTYPE)


def office_problem(g, m):
    env = fuel_b200.EDTEnvironment()
    env.setMap(m)
    ff = fuel_b200.FrontierFinder(env)
    m.update_min_, m.update_max_ = g.origin.copy(), g.map_max.copy()
    ff.searchFrontiers()
    ff.computeFrontiersToVisit()
    pos = ff.frontiers_[0].viewpoints_[0][0] + np.array([0.3, -0.2, 0.0])
    vel, yaw = np.array([0.4, -0.1, 0.0]), np.array([0.4, 0.0, 0.0])
    points, _, _ = ff.getTopViewpointsInfo(pos)
    ff.updateFrontierCostMatrix()
    mat = ff.getFullCostMatrix(pos, vel, yaw)
    order = [int(i) for i in np.argsort(mat[0, 1:], kind="stable")]
    par = EM.ExplorationParam()
    ids, _ = EM.select_refined_ids(points, order, pos, par.refined_num, par.refined_radius)
    n_points, n_yaws = ff.getViewpointsInfo(pos, ids, par.top_view_num, par.max_decay)
    return dict(prob_off=np.array([0, len(n_points)]),
                group_off=np.concatenate([[0], np.cumsum([len(p) for p in n_points])]),
                cur_pos=pos.reshape(1, 3), cur_vel=vel.reshape(1, 3), cur_yaw=yaw[:1],
                vp_pos=np.concatenate([np.asarray(p).reshape(-1, 3) for p in n_points]),
                vp_yaw=np.concatenate([np.asarray(y, np.float64) for y in n_yaws]))


def subset(w, n):
    """the first n problems of w"""
    po, go = w["prob_off"][:n + 1], w["group_off"][:w["prob_off"][n] + 1]
    return dict(prob_off=po, group_off=go, cur_pos=w["cur_pos"][:n], cur_vel=w["cur_vel"][:n], cur_yaw=w["cur_yaw"][:n],
                vp_pos=w["vp_pos"][:go[-1]], vp_yaw=w["vp_yaw"][:go[-1]])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--cpu-problems", type=int, default=16, help="problems timed on the host (scaled to B)")
    a = ap.parse_args()
    fuel_b200.lib()
    dev = card()
    st = ViewNode.astar_
    prm = FuelLocalTourParams(FuelViewCostParams(ViewNode.vm_, ViewNode.yd_, ViewNode.w_dir_,
                                                 FuelAstarParams(st["resolution"], st["lambda_heu"],
                                                                 st["allocate_num"], st["max_iter"])), 1.0)
    args = (ViewNode.vm_, ViewNode.yd_, ViewNode.w_dir_, st["resolution"], st["lambda_heu"], st["allocate_num"],
            st["max_iter"], 1.0)
    ref_ok = OT.ref_tour() is not None
    for which in ("office", "office3"):
        g, inflate = W.office_map() if which == "office" else W.office3_map()
        tri = W.office_known(g, inflate)
        m = make_sdf_map(fuel_b200, g, inflate, tri)
        om = OA.Map(g, inflate, tri)
        ref = None
        if ref_ok:
            from tests.test_oracle_astar import Scene
            with quiet_stdout():
                ref = Scene(g, inflate, tri)
        work = [("office_sequence_refine", office_problem(g, m))] if which == "office" else []
        work.append(("problems", W.make_local_tours(g, inflate, tri, B=256)))
        for name, w in work:
            B = len(w["prob_off"]) - 1
            ms, info = device_ms(m, w, prm, a.reps)
            n = min(B, a.cpu_problems)
            sub = subset(w, n)
            t = time.perf_counter()
            orc = OT.local_tour_batch(om, sub["prob_off"], sub["group_off"], sub["cur_pos"], sub["cur_vel"],
                                      sub["cur_yaw"], sub["vp_pos"], sub["vp_yaw"], *args, tour_max=TOUR_MAX)
            orc_ms = (time.perf_counter() - t) * 1e3 * B / n
            line = dict(map=which, workload=name, B=B, device_ms=round(ms, 3), nodes=int(info["n_nodes"].sum()),
                        edges_eager=int(info["n_edges"].sum()), costto_lazy=int(info["n_evals"].sum()),
                        statuses=np.bincount(info["status"], minlength=4).tolist(),
                        oracle_one_thread_ms=round(orc_ms, 2), oracle_timed_problems=n,
                        oracle_edges_lazy_timed=int(orc[0]["n_evals"].sum()))
            if ref is not None:
                rt = OT.RefTour(ref.ref, *args[:3], *args[4:7])
                po, go = sub["prob_off"], sub["group_off"]
                with quiet_stdout():
                    t = time.perf_counter()
                    for b in range(n):
                        gs = range(po[b], po[b + 1])
                        rt.refine(sub["cur_pos"][b], sub["cur_vel"][b], [sub["cur_yaw"][b], 0.0, 0.0],
                                  [sub["vp_pos"][go[i]:go[i + 1]] for i in gs],
                                  [sub["vp_yaw"][go[i]:go[i + 1]] for i in gs], tour_max=TOUR_MAX)
                    line["reference_one_thread_ms"] = round((time.perf_counter() - t) * 1e3 * B / n, 2)
                rt.close()
            print(json.dumps(line), flush=True)
        if ref is not None:
            ref.close()
        m.close()
    print(json.dumps(dict(summary="local_tour", reference_timed=ref_ok, **dev)), flush=True)


if __name__ == "__main__":
    main()
