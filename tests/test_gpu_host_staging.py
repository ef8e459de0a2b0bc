"""The host-facing batch calls (check, evaluate, parameterize, poly waypoints, yaw, A*, esdf_sample) stage their arrays in
one scratch block of the map that grows on demand.  One map runs them interleaved, with batch sizes that grow and
shrink, and next to an outstanding optimize_batch_begin; every result must equal the same call on a fresh map, bit for
bit."""
import ctypes as C

import numpy as np
import pytest

from fuel_b200 import workloads as W
from fuel_b200.astar import astar_batch
from fuel_b200.non_uniform_bspline import check_batch, evaluate_batch, parameterize_batch
from fuel_b200.polynomial_traj import plan_yaw_explore_batch, waypoints_batch
from tests.helpers import make_sdf_map
from tests.param_cases import workload_samples

pytestmark = pytest.mark.gpu

N_PTS = 20
LIM = dict(max_vel=2.0, max_acc=2.0)


@pytest.fixture(scope="module")
def scene(fuel):
    g, inflate = W.office_map()
    tri = W.office_known(g, inflate)
    tr = W.make_trajectories(g, inflate, B=1024, n_pts=N_PTS)
    rng = np.random.default_rng(20261017)
    lo, hi = np.asarray(g.origin) - 0.5, np.asarray(g.origin) + np.asarray(g.n) * g.res + 0.5
    pts, der, dt = workload_samples(g, inflate, 128, N_PTS)
    return dict(g=g, inflate=inflate, tri=tri, tr=tr, x=W.pack_x(tr["ctrl"], tr["dt"]),
                queries=W.make_path_queries(g, inflate, tri, B=64, seed=9), tours=W.make_tours(g, inflate, B=256),
                yaws=W.make_yaws(1024), pos=rng.uniform(lo, hi, (2_000_000, 3)), t=rng.uniform(-0.1, 4.0, (256, 40)),
                samples=(pts, der, dt))


def new_map(fuel, s):
    m = make_sdf_map(fuel, s["g"], s["inflate"], s["tri"], optimistic=True)
    m.updateESDF3d()
    return m


def as_bytes(r):
    if isinstance(r, tuple):
        return tuple(as_bytes(v) for v in r)
    return bytes(r) if isinstance(r, C.Array) else np.ascontiguousarray(r).tobytes()


def calls(fuel, s):
    """name -> f(map, size): each one valid host-facing call with `size` rows"""
    x, q, tr, ys = s["x"], s["queries"], s["tours"], s["yaws"]
    pts, der, dt = s["samples"]
    yaw_prm = fuel.BsplineOptimizer().params_
    return {
        "astar": lambda m, B: astar_batch(m, q["start"][:B], q["goal"][:B], resolution=0.2, lambda_heu=1.0,
                                          allocate_num=40000, max_iter=100000, path_max=512),
        "check": lambda m, B: check_batch(m, x[:B], N_PTS, **LIM),
        "evaluate": lambda m, B: evaluate_batch(m, x[:B], N_PTS, s["t"][:B], 1),
        "parameterize": lambda m, B: parameterize_batch(m, pts[:B], der[:B], dt[:B]),
        "poly": lambda m, B: waypoints_batch(m, tr["tours"][:B], tr["start_vel"][:B], tr["start_acc"][:B]),
        "yaw": lambda m, B: plan_yaw_explore_batch(m, x[:B], N_PTS, ys["start"][:B], ys["end"][:B], yaw_prm),
        "esdf_sample": lambda m, n: m.getDistWithGrad(s["pos"][:n]),
    }


SEQUENCE = [("astar", 1), ("check", 512), ("astar", 4), ("poly", 64), ("esdf_sample", 1_000_000), ("yaw", 8),
            ("evaluate", 256), ("parameterize", 128), ("astar", 64), ("check", 16), ("poly", 256), ("esdf_sample", 1000),
            ("yaw", 1024), ("parameterize", 4), ("evaluate", 3), ("check", 1024), ("esdf_sample", 2_000_000),
            ("astar", 2)]


def test_interleaved_calls_on_one_map_equal_fresh_maps(fuel, scene):
    f = calls(fuel, scene)
    m = new_map(fuel, scene)
    try:
        got = [as_bytes(f[name](m, n)) for name, n in SEQUENCE]
    finally:
        m.close()
    for (name, n), g in zip(SEQUENCE, got):
        fresh = new_map(fuel, scene)
        try:
            want = as_bytes(f[name](fresh, n))
        finally:
            fresh.close()
        assert g == want, "%s with %d rows differs from the same call on a fresh map" % (name, n)


def test_calls_beside_a_pending_solve(fuel, scene):
    """esdf_sample and check_batch, grown past their earlier sizes, while optimize_batch_begin is outstanding; _end then
    returns what the one-shot optimize_batch returns"""
    f = calls(fuel, scene)
    tr, B = scene["tr"], 512
    mask = fuel.BsplineOptimizer.NORMAL_PHASE | fuel.BsplineOptimizer.MINTIME

    def optimizer(m):
        env = fuel.EDTEnvironment()
        env.setMap(m)
        opt = fuel.BsplineOptimizer()
        opt.setEnvironment(env)
        return opt, opt.traj_consts_from_arrays(tr["pt_dist"][:B], tr["dt"][:B], tr["start"][:B], tr["end_pos"][:B])

    m = new_map(fuel, scene)
    try:
        opt, tcs = optimizer(m)
        f["esdf_sample"](m, 1000)
        f["check"](m, 4)
        opt.optimizeBatchBegin(scene["x"][:B], tcs, N_PTS, mask, 64)
        sample = as_bytes(f["esdf_sample"](m, 2_000_000))
        check = as_bytes(f["check"](m, 1024))
        solved = as_bytes(opt.optimizeBatchEnd())
    finally:
        m.close()
    fresh = new_map(fuel, scene)
    try:
        opt, tcs = optimizer(fresh)
        assert solved == as_bytes(opt.optimizeBatch(scene["x"][:B], tcs, N_PTS, mask, 64))
        assert sample == as_bytes(f["esdf_sample"](fresh, 2_000_000))
        assert check == as_bytes(f["check"](fresh, 1024))
    finally:
        fresh.close()
