#!/usr/bin/env python
"""Device time of the tour's edge cost (fuelgpu_view_cost_batch_dev: ViewNode::searchPath + computeCost) against the
same pairs on one host thread, in the oracle's restatement (oracle/fuel_oracle_view.c, over the A* oracle) and, where
oracle/_ref/libfuel_ref_view.so is built, in the reference's own compiled graph_node.cpp.  Workloads: the office cost
matrix from scratch (searchFrontiers -> computeFrontiersToVisit -> every pair of top viewpoints, as
updateFrontierCostMatrix batches it) and getFullCostMatrix's row 0 (with a velocity), then P = 4096 pairs of
workloads.make_view_pairs on office and office3.  ViewNode's defaults (vm 2.0, yd 60 deg, w_dir 1.5, lambda 10000,
allocate_num 1 000 000, max_iter 10000).  The device time is CUDA events around the call on the map's stream (inputs
on the device, outputs left there), median over the repetitions after one warm-up.  One JSON line per workload with
the line / A* / no-path split and the search iterations, then a summary line with the card's name and power limit."""
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
import oracle.astar as OA  # noqa: E402
import oracle.view as OV  # noqa: E402
from fuel_b200 import workloads as W  # noqa: E402
from fuel_b200._lib import FuelAstarParams, FuelViewCostParams, lib  # noqa: E402
from fuel_b200.view_node import ASTAR, INFO_DTYPE, LINE, NO_PATH, ViewNode  # noqa: E402
from tests.helpers import make_sdf_map  # noqa: E402
from tools.solver_long import card  # noqa: E402


def device_ms(m, pr, prm, reps):
    P = len(pr["p1"])
    dev = torch.device("cuda")
    t = {k: torch.tensor(np.ascontiguousarray(v), device=dev) for k, v in pr.items()}
    dinfo = torch.zeros(P * INFO_DTYPE.itemsize, dtype=torch.uint8, device=dev)
    stream = torch.cuda.Stream()
    m.set_stream(stream.cuda_stream)
    torch.cuda.synchronize()
    ms = []
    for r in range(reps + 1):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        rc = lib().fuelgpu_view_cost_batch_dev(m.handle, P, t["p1"].data_ptr(), t["p2"].data_ptr(), t["y1"].data_ptr(),
                                               t["y2"].data_ptr(), t["v1"].data_ptr(), C.byref(prm), dinfo.data_ptr(),
                                               0, None)
        e1.record(stream)
        assert rc == 0
        torch.cuda.synchronize()
        if r:  # the first call grows and fills the scratch
            ms.append(e0.elapsed_time(e1))
    m.set_stream(0)
    return float(np.median(ms)), np.frombuffer(dinfo.cpu().numpy().tobytes(), dtype=INFO_DTYPE)


def host_ms(fn, n, P):
    t = time.perf_counter()
    fn(n)
    return (time.perf_counter() - t) * 1e3 * P / n


def matrix_pairs(g, inflate, tri, m):
    """the office frontier clusters' top viewpoints: every pair i < j (updateFrontierCostMatrix from scratch) and the
    row from the current state (getFullCostMatrix)"""
    env = fuel_b200.EDTEnvironment()
    env.setMap(m)
    ff = fuel_b200.FrontierFinder(env)
    m.update_min_, m.update_max_ = g.origin.copy(), g.map_max.copy()
    ff.searchFrontiers()
    ff.computeFrontiersToVisit()
    v = [f.viewpoints_[0] for f in ff.frontiers_]
    ij = [(i, j) for i in range(len(v)) for j in range(i + 1, len(v))]
    mat = dict(p1=np.array([v[i][0] for i, _ in ij]), p2=np.array([v[j][0] for _, j in ij]),
               y1=np.array([v[i][1] for i, _ in ij]), y2=np.array([v[j][1] for _, j in ij]), v1=np.zeros((len(ij), 3)))
    cur = v[0][0] + np.array([0.3, -0.2, 0.0])
    n = len(v)
    row = dict(p1=np.repeat(cur[None], n, 0), p2=np.array([x[0] for x in v]), y1=np.full(n, 0.4),
               y2=np.array([x[1] for x in v]), v1=np.repeat(np.array([[0.9, -0.4, 0.05]]), n, 0))
    return len(v), mat, row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--cpu-pairs", type=int, default=256, help="pairs timed on the host (scaled to P)")
    a = ap.parse_args()
    fuel_b200.lib()
    dev = card()
    st = ViewNode.astar_
    prm = FuelViewCostParams(ViewNode.vm_, ViewNode.yd_, ViewNode.w_dir_,
                             FuelAstarParams(st["resolution"], st["lambda_heu"], st["allocate_num"], st["max_iter"]))
    args = (ViewNode.vm_, ViewNode.yd_, ViewNode.w_dir_, st["resolution"], st["lambda_heu"], st["allocate_num"],
            st["max_iter"])
    ref_ok = OV.ref_view() is not None
    for which in ("office", "office3"):
        g, inflate = W.office_map() if which == "office" else W.office3_map()
        tri = W.office_known(g, inflate)
        m = make_sdf_map(fuel_b200, g, inflate, tri)
        om = OA.Map(g, inflate, tri)
        ref = None
        if ref_ok:
            from tests.test_oracle_astar import Scene
            ref = Scene(g, inflate, tri)
            rv = OV.RefViewNode(ref.ref, *args[:3], *args[4:])
        work = []
        if which == "office":
            nclusters, mat, row = matrix_pairs(g, inflate, tri, m)
            work += [("cost_matrix_from_scratch", mat), ("full_cost_matrix_row0", row)]
        work.append(("pairs", W.make_view_pairs(g, inflate, tri, P=4096)))
        for name, pr in work:
            P = len(pr["p1"])
            ms, info = device_ms(m, pr, prm, a.reps)
            n = min(P, a.cpu_pairs)
            sub = {k: v[:n] for k, v in pr.items()}
            orc = host_ms(lambda k: OV.view_cost_batch(om, sub["p1"], sub["p2"], sub["y1"], sub["y2"], sub["v1"], *args,
                                                       path_max=1), n, P)
            line = dict(map=which, workload=name, P=P, device_ms=round(ms, 3),
                        line=int(np.sum(info["kind"] == LINE)), astar=int(np.sum(info["kind"] == ASTAR)),
                        no_path=int(np.sum(info["kind"] == NO_PATH)), total_iterations=int(info["iter_num"].sum()),
                        max_iterations=int(info["iter_num"].max()), oracle_one_thread_ms=round(orc, 2))
            if name == "cost_matrix_from_scratch":
                line["clusters"] = nclusters
            if ref is not None:
                line["reference_one_thread_ms"] = round(host_ms(
                    lambda k: rv.cost_batch(sub["p1"], sub["p2"], sub["y1"], sub["y2"], sub["v1"], path_max=1), n, P), 2)
            print(json.dumps(line), flush=True)
        if ref is not None:
            rv.close()
            ref.close()
        m.close()
    print(json.dumps(dict(summary="view_cost", reference_timed=ref_ok, **dev)), flush=True)


if __name__ == "__main__":
    main()
