#!/usr/bin/env python
"""Device solver time against trajectory length, on both sides of the 32-lane switch (n_pts + dt <= 32: the one-point-
per-lane kernels; above: optimize_long_kernel, two points per lane).

office3 map (BASELINE config 5 grid, 200x300x40), optimistic ESDF, batches of workloads.make_trajectories(n_pts=n),
NORMAL_PHASE | MINTIME, exact-evals mode (every trajectory evaluates the objective K times).  Each solve is timed with
CUDA events on the map's stream, after an L2 flush; the median and the spread of the repetitions are printed.

CPU comparison: the reference's own combineCost (oracle/_ref, built by build()) on one host thread, at the same n, over
a subset of the batch, scaled to B x K evaluations as bench.py's cpu_baseline does.  Without oracle/_ref the oracle's
port of it is timed instead and labelled "port".  One JSON line per (B, n), then a summary line."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

import bench  # noqa: E402
import fuel_b200  # noqa: E402
import oracle  # noqa: E402
from fuel_b200 import workloads as W  # noqa: E402
from fuel_b200._lib import SOLVE_EXACT_EVALS, FuelSolveParams  # noqa: E402


def card():
    out = {"name": torch.cuda.get_device_name(0)}
    try:
        r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        pl, mx = [v.strip() for v in r.stdout.strip().split(",")]
        out.update(power_limit=pl, sm_max_clock=mx)
    except Exception as e:  # noqa: BLE001
        out.update(power_limit="unknown (%r)" % e)
    return out


def ref_setup(g):
    """The reference's SDFMap on the same occupancy (office3 is centred, as SDFMap::initMap requires)."""
    size = np.array(g.n) * g.res
    params = dict(resolution=g.res, map_size_x=size[0], map_size_y=size[1], map_size_z=size[2], ground_height=g.origin[2],
                  obstacles_inflation=0.199, local_bound_inflate=0.5, local_map_margin=50, default_dist=0.0, optimistic=1,
                  signed_dist=0, p_hit=0.65, p_miss=0.35, p_min=0.12, p_max=0.90, p_occ=0.80, max_ray_length=4.5,
                  virtual_ceil_height=-10.0)
    for ax, lo, hi in zip("xyz", g.box_min, g.box_max):
        params["box_min_" + ax], params["box_max_" + ax] = float(lo), float(hi)
    with bench._Quiet():
        ref = oracle.RefSDFMap(**params)
    return ref


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="1024,4096")
    ap.add_argument("--points", default="20,31,33,48,64")
    ap.add_argument("--evals", type=int, default=64)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--cpu-traj", type=int, default=32, help="trajectories of the batch the CPU arm evaluates K times")
    ap.add_argument("--cpu-reps", type=int, default=3, help="CPU timings per row (the median is reported)")
    ap.add_argument("--lbfgs-m", type=int, default=6, help="history length (6: the coefficient-space kernel below 33 lanes)")
    args = ap.parse_args()
    K = args.evals
    dev = card()

    g, inflate = W.office3_map()
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
    L = fuel_b200.lib()
    mask = opt.NORMAL_PHASE | opt.MINTIME
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device="cuda")
    sp = FuelSolveParams()
    sp.max_eval, sp.lbfgs_m, sp.xtol_rel, sp.flags = K, args.lbfgs_m, 0.0, SOLVE_EXACT_EVALS

    # CPU arm: the reference's combineCost when oracle/_ref is built, else the oracle's port
    oracle.build()
    use_ref = oracle.ref_raycast() is not None
    if use_ref:
        ref = ref_setup(g)
        ref.inflate[:] = inflate.reshape(-1)
        lg = lambda p: float(np.log(p / (1 - p)))  # noqa: E731
        ref.occupancy[:] = np.where(tri == 0, lg(0.12) - 0.01, np.where(tri == 2, lg(0.90), lg(0.12))).reshape(-1)
        ref.set_modes(1, 0)
        ref.set_local_bound((0, 0, 0), np.array(g.n) - 1)
        with bench._Quiet():
            ref.update_esdf3d()
    else:
        og = oracle.make_grid(g.n, g.res, g.origin, g.box_min, g.box_max)
        d64 = oracle.update_esdf3d(og, inflate, tri, [0, 0, 0], np.array(g.n) - 1, True, False, threads=8)

    rows = []
    for B in [int(v) for v in args.batches.split(",")]:
        for n in [int(v) for v in args.points.split(",")]:
            tr = W.make_trajectories(g, inflate, B=B, n_pts=n)
            x0 = W.pack_x(tr["ctrl"], tr["dt"])
            tcs = opt.traj_consts_from_arrays(tr["pt_dist"], tr["dt"], tr["start"], tr["end_pos"])
            d_tc = torch.from_numpy(np.frombuffer(tcs, dtype=np.uint8).copy()).cuda()
            d_x0 = torch.from_numpy(x0).cuda()
            d_x = torch.empty_like(d_x0)
            d_f = torch.empty(B, dtype=torch.float64, device="cuda")
            d_n = torch.empty(B, dtype=torch.int32, device="cuda")
            ms = []
            for it in range(args.warmup + args.reps):
                d_x.copy_(d_x0)
                flush.zero_()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(st)
                rc = L.fuelgpu_bspline_optimize_batch_dev(m.handle, B, n, mask, C.byref(opt.params_),
                                                          C.c_void_p(d_tc.data_ptr()), C.byref(sp),
                                                          C.c_void_p(d_x.data_ptr()), C.c_void_p(d_f.data_ptr()),
                                                          C.c_void_p(d_n.data_ptr()))
                e1.record(st)
                if rc != 0:
                    raise SystemExit("solver_long.py: fuelgpu_bspline_optimize_batch_dev returned %d" % rc)
                st.synchronize()
                if it >= args.warmup:
                    ms.append(e0.elapsed_time(e1))
            ne = d_n.cpu().numpy()
            if int(ne.min()) != K:
                raise SystemExit("solver_long.py: B=%d n=%d: a trajectory did %d evaluations, not %d" % (B, n, ne.min(), K))
            med = float(np.median(ms))

            # CPU: S trajectories x K evaluations (the start point, then K-1 probes around it, as bench.py does)
            S = min(args.cpu_traj, B)
            rng = np.random.default_rng(5)
            probes = x0[:S, None, :] + rng.normal(size=(S, K - 1, x0.shape[1])) * 0.03
            probes[:, :, -1] = np.abs(probes[:, :, -1]) + 1e-3
            pts = np.concatenate([x0[:S, None, :], probes], axis=1)
            if not use_ref:
                otc = oracle.traj_consts(S)
                for b in range(S):
                    oracle.fill_traj_const(otc[b], tr["pt_dist"][b], tr["dt"][b], tr["start"][b], tr["end_pos"][b][None, :])

            def cpu_run(nk):
                t0 = time.perf_counter()
                if use_ref:
                    with bench._Quiet():
                        oracle.ref_combine_cost_batch(ref, bench.REF_OPT, tr["ctrl"][:S], tr["dt"][:S], mask, tr["start"][:S],
                                                      tr["end_pos"][:S], np.ascontiguousarray(probes[:, :nk - 1]), threads=1)
                else:
                    for k in range(nk):
                        oracle.combine_cost_batch(og, d64, oracle.opt_params(), otc, n, mask, pts[:, k], threads=1)
                return time.perf_counter() - t0

            cpu_run(2)  # warm-up
            cpu_s = float(np.median([cpu_run(K) for _ in range(args.cpu_reps)]))
            cpu_ms = 1e3 * cpu_s * B / S  # scaled to B x K evaluations
            row = {"B": B, "n": n, "K": K, "kernel": ("optimize_long_kernel" if n + 1 > 32 else
                                                       "optimize_gram_kernel<6>" if args.lbfgs_m == 6 else "optimize_warp_kernel"),
                   "ms_median": med, "ms_min": float(min(ms)), "ms_max": float(max(ms)), "reps": len(ms),
                   "ns_per_traj_eval": 1e6 * med / (B * K), "evals_done_min": int(ne.min()),
                   "cpu_kind": "reference" if use_ref else "port", "cpu_ms_1thread_scaled": cpu_ms,
                   "cpu_sample": "%d trajectories x %d evaluations, median of %d" % (S, K, args.cpu_reps),
                   "cpu_ns_per_eval": 1e9 * cpu_s / (S * K), "speedup_vs_1thread": cpu_ms / med}
            rows.append(row)
            print(json.dumps(row), flush=True)
    torch.cuda.synchronize()
    m.close()
    print(json.dumps({"card": dev, "map": "office3 200x300x40 optimistic", "mask": "NORMAL_PHASE|MINTIME",
                      "solve": "exact_evals, lbfgs_m %d" % args.lbfgs_m, "table": [[r["B"], r["n"], round(r["ms_median"], 4),
                                                                    round(r["ns_per_traj_eval"], 3),
                                                                    round(r["speedup_vs_1thread"], 1)] for r in rows],
                      "columns": ["B", "n", "ms_median", "ns_per_traj_eval", "speedup_vs_1thread"]}))


if __name__ == "__main__":
    main()
