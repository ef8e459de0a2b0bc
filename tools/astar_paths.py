#!/usr/bin/env python
"""Device time of the path stage (fuelgpu_astar_batch_dev: Astar::search, shortenPath and planExploreMotion's branch)
against the same searches on one host thread in the oracle's restatement (oracle/fuel_oracle_astar.c, pinned bit for bit
on the reference's astar2.cpp).  Queries: workloads.make_path_queries, B = 1024 on the office map and B = 4096 on office3, plus
B = 1 (one search on one warp: its latency).  The device time is CUDA events around the launch on the map's stream
(inputs already on the device, outputs left there); medians over the repetitions.  One JSON line per batch, then a
summary line with the card's name and power limit."""
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
from fuel_b200 import workloads as W  # noqa: E402
from fuel_b200._lib import FuelAstarParams, lib  # noqa: E402
from fuel_b200.astar import INFO_DTYPE, MAX_WAYPTS  # noqa: E402
from tests.helpers import make_sdf_map  # noqa: E402
from tools.solver_long import card  # noqa: E402


def device_ms(m, start, goal, prm, reps):
    B = len(start)
    dev = torch.device("cuda")
    ds, dg = torch.tensor(start, device=dev), torch.tensor(goal, device=dev)
    dinfo = torch.zeros(B * INFO_DTYPE.itemsize, dtype=torch.uint8, device=dev)
    dn = torch.zeros(B, dtype=torch.int32, device=dev)
    dw = torch.zeros((B, MAX_WAYPTS, 3), dtype=torch.float64, device=dev)
    stream = torch.cuda.Stream()  # the map's stream for the timed launches: the events bracket the kernel
    m.set_stream(stream.cuda_stream)
    torch.cuda.synchronize()
    ms = []
    for r in range(reps + 1):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        rc = lib().fuelgpu_astar_batch_dev(m.handle, B, ds.data_ptr(), dg.data_ptr(), C.byref(prm), dinfo.data_ptr(), 0,
                                           None, MAX_WAYPTS, dn.data_ptr(), dw.data_ptr())
        e1.record(stream)
        assert rc == 0
        torch.cuda.synchronize()
        if r:  # the first call grows and fills the scratch
            ms.append(e0.elapsed_time(e1))
    m.set_stream(0)
    info = np.frombuffer(dinfo.cpu().numpy().tobytes(), dtype=INFO_DTYPE)
    return float(np.median(ms)), info


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--cpu-queries", type=int, default=256, help="queries timed on the host (scaled to B)")
    ap.add_argument("--resolution", type=float, default=0.2)
    ap.add_argument("--lambda-heu", type=float, default=1.0)
    ap.add_argument("--allocate-num", type=int, default=40000)
    a = ap.parse_args()
    fuel_b200.lib()
    dev = card()
    prm = FuelAstarParams(a.resolution, a.lambda_heu, a.allocate_num, 100000)
    for which, B in (("office", 1), ("office", 1024), ("office3", 4096)):
        g, inflate = W.office_map() if which == "office" else W.office3_map()
        tri = W.office_known(g, inflate)
        m = make_sdf_map(fuel_b200, g, inflate, tri)
        q = W.make_path_queries(g, inflate, tri, B=max(B, 2))
        if B == 1:  # the longest successful office search of the batch of 1024
            qq = W.make_path_queries(g, inflate, tri, B=1024)
            _, info = device_ms(m, qq["start"], qq["goal"], prm, 1)
            ok = np.flatnonzero(info["status"] == 1)
            i = ok[np.argmax(info["iter_num"][ok])]
            q = dict(start=qq["start"][i:i + 1], goal=qq["goal"][i:i + 1])
        ms, info = device_ms(m, q["start"][:B], q["goal"][:B], prm, a.reps)
        n = min(B, a.cpu_queries)
        om = OA.Map(g, inflate, tri)
        t = time.perf_counter()
        OA.search_batch(om, q["start"][:n], q["goal"][:n], a.resolution, a.lambda_heu, a.allocate_num, 100000,
                        path_max=1)
        orc_ms = (time.perf_counter() - t) * 1e3 * B / n
        iters = int(info["iter_num"].sum())
        print(json.dumps(dict(map=which, B=B, resolution=a.resolution, lambda_heu=a.lambda_heu,
                              allocate_num=a.allocate_num, device_ms=round(ms, 3), total_iterations=iters,
                              iterations_per_s=round(iters / (ms * 1e-3)), found=int(np.sum(info["status"] == 1)),
                              oracle_one_thread_ms=round(orc_ms, 1))), flush=True)
        m.close()
    print(json.dumps(dict(summary="astar_paths", **dev)), flush=True)


if __name__ == "__main__":
    main()
