#!/usr/bin/env python
"""Device time of findGlobalTour's tour (fuelgpu_global_tour_batch_dev: Held-Karp over the integer ATSP, every layer
and the reconstruction on the map's stream) for B = 1 at n = 14 and n = 20 and for B = 256 at n = 14, beside the
reference's own findGlobalTour (oracle/_ref/libfuel_ref_gtour.so: getFullCostMatrix's row 0, the TSPLIB file, LKH, the
tour parse and getPathForTour) on one host thread, on the same matrices: frontier lists on the office map whose costs_
rows are workloads.make_global_tours' geometric matrices, row 0 the reference's computeCost from the current state; the
device solves the matrix the reference built.  Where the reference library is not built, the matrices are the
generator's and the reference column is absent.  The C oracle's Held-Karp on one host thread is timed too.  The device
time is CUDA events around the call (inputs on the device, outputs left there), median over the repetitions after one
warm-up; host times are a wall clock, median over their repetitions (the reference's B = 256 row is one pass over the
batch).  Every device result is checked against the oracle, and its cost against LKH's.  One JSON line per workload,
then a summary line with the card's name and power limit."""
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
import oracle.gtour as OG  # noqa: E402
from fuel_b200 import exploration_manager as EM  # noqa: E402
from fuel_b200 import workloads as W  # noqa: E402
from fuel_b200._lib import check, lib  # noqa: E402
from tests.helpers import make_sdf_map  # noqa: E402
from tools.local_tour import quiet_stdout  # noqa: E402
from tools.solver_long import card  # noqa: E402

PRM = (2.0, 60 * 3.1415926 / 180.0, 1.5, 0.4, 10000.0, 1000000, 10000)  # ViewNode's defaults (tools/local_tour.py)


def reference_batch(s, g, inflate, tri, n, B, seed, reps):
    """the reference's findGlobalTour on B frontier lists -> (matrices [B, n + 1, n + 1], LKH's tours, ms per call
    (median over reps of the batch's mean))"""
    from tests.test_oracle_global_tour import _problem
    rg = OG.RefGTour(s.ref, *PRM[:3], *PRM[4:])
    try:
        probs = [_problem(g, inflate, tri, n, "geometric", seed + b) for b in range(B)]
        mats, tours, ms = [], [], []
        for r in range(reps):
            t0 = time.perf_counter()
            with quiet_stdout():
                out = [rg.find(*p) for p in probs]
            ms.append(1e3 * (time.perf_counter() - t0) / B)
        for lkh, _, mat in out:
            mats.append(mat)
            tours.append(lkh)
        return np.stack(mats), tours, float(np.median(ms))
    finally:
        rg.close()


def device_ms(m, dims, cost, reps):
    dev = torch.device("cuda")
    dcost = torch.tensor(cost, device=dev)
    dinfo = torch.zeros(len(dims) * EM.GTOUR_INFO_DTYPE.itemsize, dtype=torch.uint8, device=dev)
    didx = torch.zeros(int(dims.sum()) - len(dims), dtype=torch.int32, device=dev)
    stream = torch.cuda.Stream()
    m.set_stream(stream.cuda_stream)
    torch.cuda.synchronize()
    ms = []
    for r in range(reps + 1):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        check(lib().fuelgpu_global_tour_batch_dev(m.handle, len(dims), dims.ctypes.data, dcost.data_ptr(),
                                                  dinfo.data_ptr(), didx.data_ptr()), m.handle)
        e1.record(stream)
        torch.cuda.synchronize()
        if r:  # the first call grows the scratch
            ms.append(e0.elapsed_time(e1))
    m.set_stream(0)
    info = np.frombuffer(dinfo.cpu().numpy().tobytes(), dtype=EM.GTOUR_INFO_DTYPE)
    return float(np.median(ms)), info, didx.cpu().numpy()


def host_ms(dims, cost, reps):
    ms = []
    for _ in range(reps):
        t0 = time.perf_counter()
        OG.global_tour_batch(dims, cost)
        ms.append(1e3 * (time.perf_counter() - t0))
    return float(np.median(ms))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--host-reps", type=int, default=3)
    a = ap.parse_args()
    fuel_b200.lib()
    g, inflate = W.office_map()
    tri = W.office_known(g, inflate)
    m = make_sdf_map(fuel_b200, g, inflate, tri)
    s = None
    if OG.ref_gtour() is not None:
        from tests.test_oracle_astar import Scene
        s = Scene(g, inflate, tri)
    for n, B in ((14, 1), (20, 1), (14, 256)):
        seed = 20261020 + 1000 * n + B
        line = dict(workload="global_tour", n=n, B=B)
        if s is not None and s.ref is not None:
            mats, lkh, ref_ms = reference_batch(s, g, inflate, tri, n, B, seed, a.host_reps if B == 1 else 1)
            line["reference_ms_per_instance"] = round(ref_ms, 3)
        else:
            mats, lkh = W.make_global_tours(n, B=B, seed=seed), None
        dims = np.full(B, n + 1, np.int32)
        cost = np.ascontiguousarray(mats.reshape(-1))
        dev_ms, info, idx = device_ms(m, dims, cost, a.reps)
        want = OG.global_tour_batch(dims, cost)
        assert info.tobytes() == want[0].tobytes() and np.array_equal(idx, want[1])
        if lkh is not None:
            costs = [OG.tour_cost(OG.int_matrix(mats[b]), lkh[b]) for b in range(B)]
            assert np.all(info["cost"] <= np.array(costs))
            line["lkh_at_optimum"] = int(np.sum(info["cost"] == np.array(costs)))
        line.update(device_ms=round(dev_ms, 4), oracle_host_ms=round(host_ms(dims, cost, a.host_reps), 3),
                    table_bytes=int(B * 12 * n * 2 ** n))
        print(json.dumps(line), flush=True)
    m.close()
    if s is not None:
        s.close()
    print(json.dumps(dict(summary="global_tour", reference_timed=s is not None, **card())), flush=True)


if __name__ == "__main__":
    main()
