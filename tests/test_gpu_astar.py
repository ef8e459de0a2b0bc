"""fuelgpu_astar_batch[_dev] on the H100 against the CPU oracle (oracle.astar, pinned bit for bit on the reference's
compiled astar2.cpp by tests/test_oracle_astar.py): every output bit for bit on the office and office3 queries of
workloads.make_path_queries, at two lambda / resolution pairs and with the pool and iteration caps reached; the
_dev entry against the host entry; bad input; and the chain into the waypoint polynomial and planExploreTraj."""
import ctypes as C

import numpy as np
import pytest
import torch

import oracle.astar as OA
from fuel_b200 import workloads as W
from fuel_b200._lib import FuelAstarParams, FuelPolyParams, lib
from fuel_b200.astar import (BAD_INPUT, DEGENERATE, INFO_DTYPE, ITER_CAP, MAX_WAYPTS, POOL, REACH_END, Astar,
                             astar_batch, search_paths_batch)
from fuel_b200.polynomial_traj import INFO_DTYPE as POLY_INFO, waypoints_batch
from tests.helpers import make_sdf_map

pytestmark = pytest.mark.gpu

PATH_MAX = 512


@pytest.fixture(scope="module")
def office(fuel):
    g, inflate = W.office_map()
    tri = W.office_known(g, inflate)
    m = make_sdf_map(fuel, g, inflate, tri)
    yield g, inflate, tri, m, OA.Map(g, inflate, tri)
    m.close()


@pytest.fixture(scope="module")
def office3(fuel):
    g, inflate = W.office3_map()
    tri = W.office_known(g, inflate)
    m = make_sdf_map(fuel, g, inflate, tri)
    yield g, inflate, tri, m, OA.Map(g, inflate, tri)
    m.close()


def assert_same(got, want):
    gi, gp, gn, gw = got
    wi, wp, wn, ww = want
    for f in INFO_DTYPE.names:
        bad = np.flatnonzero(np.any((gi[f] != wi[f]).reshape(len(gi), -1), axis=1))
        assert bad.size == 0, "%s differs at %s: %s vs %s" % (f, bad[:5], gi[f][bad[:3]], wi[f][bad[:3]])
    assert np.array_equal(gn, wn)
    assert np.array_equal(gp, wp)
    assert np.array_equal(gw, ww)


def run_both(m, om, start, goal, res, lam, alloc, max_iter):
    got = astar_batch(m, start, goal, resolution=res, lambda_heu=lam, allocate_num=alloc, max_iter=max_iter,
                      path_max=PATH_MAX, w_max=MAX_WAYPTS)
    want = OA.search_batch(om, start, goal, res, lam, alloc, max_iter, path_max=PATH_MAX, w_max=MAX_WAYPTS)
    assert_same(got, want)
    return got


@pytest.mark.parametrize("res,lam", [(0.2, 1.0), (0.4, 10000.0)])
def test_office_b1024_matches_oracle(office, res, lam):
    g, inflate, tri, m, om = office
    q = W.make_path_queries(g, inflate, tri, B=1024)
    info = run_both(m, om, q["start"], q["goal"], res, lam, 40000, 100000)[0]
    assert np.count_nonzero(info["status"] == REACH_END) > 300
    assert set(np.unique(info["branch"][info["status"] == REACH_END]).tolist()) == {1, 2, 3}


@pytest.mark.parametrize("res,lam", [(0.4, 10000.0)])
def test_office3_b4096_matches_oracle(office3, res, lam):
    g, inflate, tri, m, om = office3
    q = W.make_path_queries(g, inflate, tri, B=4096, seed=20261018)
    run_both(m, om, q["start"], q["goal"], res, lam, 20000, 100000)


@pytest.mark.parametrize("alloc,max_iter,reason", [(300, 100000, POOL), (100000, 40, ITER_CAP), (2, 100, POOL)])
def test_caps_match_oracle(office, alloc, max_iter, reason):
    g, inflate, tri, m, om = office
    q = W.make_path_queries(g, inflate, tri, B=256, seed=5)
    info = run_both(m, om, q["start"], q["goal"], 0.2, 1.0, alloc, max_iter)[0]
    assert np.count_nonzero(info["reason"] == reason) > 0


def test_dijkstra_box_matches_oracle(fuel):
    """an all-free box with lambda = 0 (Dijkstra): stale entries popped and expanded again, the pool cap reached"""
    g = W.Grid((60, 60, 20), (-3.0, -3.0, -1.0), 0.1, box_min=(-2.9, -2.9, -0.9), box_max=(2.9, 2.9, 0.9))
    inflate, tri = np.zeros(g.n, np.int8), np.full(g.n, W.FREE, np.uint8)
    m = make_sdf_map(fuel, g, inflate, tri)
    om = OA.Map(g, inflate, tri)
    try:
        start = np.array([[-2.5, -2.5, -0.5], [0.0, 0.0, 0.0]])
        goal = np.array([[2.5, 2.5, 0.5], [2.0, -2.0, 0.3]])
        info = run_both(m, om, start, goal, 0.1, 0.0, 2000, 100000)[0]
        assert np.all(info["reason"] == POOL) and np.all(info["iter_num"] > 1000)
    finally:
        m.close()


def test_lattice_ties(fuel):
    """an all-known empty box, start and goal on lattice diagonals: f ties everywhere, only the heap order fixes the path"""
    g = W.Grid((60, 60, 30), (-3.0, -3.0, -1.5), 0.1, box_min=(-2.95, -2.95, -1.45), box_max=(2.95, 2.95, 1.45))
    inflate, tri = np.zeros(g.n, np.int8), np.full(g.n, W.FREE, np.uint8)
    m = make_sdf_map(fuel, g, inflate, tri)
    om = OA.Map(g, inflate, tri)
    try:
        k = np.arange(-5, 6) * 0.2
        off = np.array([0.013, 0.027, 0.031])  # off the voxel corners: shortenPath's rays must meet their end voxel
        start = np.stack([k, k, 0.5 * k], axis=1) + off
        goal = np.stack([-k, k + 0.4, -0.5 * k], axis=1) + off
        for res, lam in ((0.2, 1.0), (0.2, 0.0), (0.4, 10000.0)):
            run_both(m, om, start, goal, res, lam, 20000, 100000)
    finally:
        m.close()


def test_dev_entry_equals_host_entry_and_bad_rows(office):
    g, inflate, tri, m, om = office
    q = W.make_path_queries(g, inflate, tri, B=192, seed=9)
    start, goal = q["start"].copy(), q["goal"].copy()
    start[5, 1] = np.nan
    goal[17, 2] = np.inf
    good = np.ones(len(start), bool)
    good[[5, 17]] = False
    prm = FuelAstarParams(0.2, 1.0, 40000, 100000)
    B = len(start)
    host = astar_batch(m, start[good], goal[good], resolution=0.2, lambda_heu=1.0, allocate_num=40000, max_iter=100000,
                       path_max=PATH_MAX, w_max=MAX_WAYPTS)
    dev = torch.device("cuda")
    ds, dg = torch.tensor(start, device=dev), torch.tensor(goal, device=dev)
    dinfo = torch.zeros(B * INFO_DTYPE.itemsize, dtype=torch.uint8, device=dev)
    dpath = torch.zeros((B, PATH_MAX, 3), dtype=torch.float64, device=dev)
    dn = torch.zeros(B, dtype=torch.int32, device=dev)
    dw = torch.zeros((B, MAX_WAYPTS, 3), dtype=torch.float64, device=dev)
    torch.cuda.synchronize()
    rc = lib().fuelgpu_astar_batch_dev(m.handle, B, ds.data_ptr(), dg.data_ptr(), C.byref(prm), dinfo.data_ptr(),
                                       PATH_MAX, dpath.data_ptr(), MAX_WAYPTS, dn.data_ptr(), dw.data_ptr())
    assert rc == 0
    m.synchronize()
    info = np.frombuffer(dinfo.cpu().numpy().tobytes(), dtype=INFO_DTYPE)
    assert np.all(info["reason"][~good] == BAD_INPUT) and np.all(dn.cpu().numpy()[~good] == 0)
    assert_same((info[good], dpath.cpu().numpy()[good], dn.cpu().numpy()[good], dw.cpu().numpy()[good]), host)
    # the host entry refuses the same rows and writes nothing
    out = np.full(B, 7, np.int32)
    info_h = np.zeros(B, INFO_DTYPE)
    wp = np.zeros((B, MAX_WAYPTS, 3))
    rc = lib().fuelgpu_astar_batch(m.handle, B, start.ctypes.data, goal.ctypes.data, C.byref(prm), info_h.ctypes.data, 0,
                                   None, MAX_WAYPTS, out.ctypes.data, wp.ctypes.data)
    assert rc == -1 and np.all(out == 7)
    s2, g2 = np.ascontiguousarray(start[good][:2]), np.ascontiguousarray(goal[good][:2])
    for bad in (FuelAstarParams(0.0, 1.0, 100, 10), FuelAstarParams(np.nan, 1.0, 100, 10), FuelAstarParams(0.2, 1.0, 1, 10),
                FuelAstarParams(0.2, 1.0, 100, 0), FuelAstarParams(0.2, np.inf, 100, 10)):
        rc = lib().fuelgpu_astar_batch(m.handle, 2, s2.ctypes.data, g2.ctypes.data, C.byref(bad),
                                       info_h.ctypes.data, 0, None, MAX_WAYPTS, out.ctypes.data, wp.ctypes.data)
        assert rc == -1 and np.all(out == 7)


def test_start_equals_goal_is_degenerate(office):
    g, inflate, tri, m, om = office
    q = W.make_path_queries(g, inflate, tri, B=64, seed=3)
    s = q["start"][:4]
    info, _, n_wp, _ = run_both(m, om, s, s.copy(), 0.2, 1.0, 1000, 100)
    assert np.all(info["status"] == REACH_END) and np.all(info["tour_status"] == DEGENERATE) and np.all(n_wp == 0)
    assert np.all(info["n_path"] == 2) and np.all(info["n_wp"] == 1)


def test_chain_into_poly_without_host_sync(office):
    """astar_batch_dev -> poly_waypoints_batch_dev on device buffers equals the host route through the oracle's tours"""
    g, inflate, tri, m, om = office
    q = W.make_path_queries(g, inflate, tri, B=256, seed=11)
    B = 256
    dev = torch.device("cuda")
    ds, dg = torch.tensor(q["start"], device=dev), torch.tensor(q["goal"], device=dev)
    dinfo = torch.zeros(B * INFO_DTYPE.itemsize, dtype=torch.uint8, device=dev)
    dn = torch.zeros(B, dtype=torch.int32, device=dev)
    dw = torch.zeros((B, MAX_WAYPTS, 3), dtype=torch.float64, device=dev)
    zero = torch.zeros((B, 3), dtype=torch.float64, device=dev)
    pinfo = torch.zeros(B * POLY_INFO.itemsize, dtype=torch.uint8, device=dev)
    pts = torch.zeros((B, 62, 3), dtype=torch.float64, device=dev)
    der = torch.zeros((B, 4, 3), dtype=torch.float64, device=dev)
    prm = FuelAstarParams(0.2, 1.0, 40000, 100000)
    pp = FuelPolyParams(2.0, 0.35, 8, 0)
    torch.cuda.synchronize()
    assert lib().fuelgpu_astar_batch_dev(m.handle, B, ds.data_ptr(), dg.data_ptr(), C.byref(prm), dinfo.data_ptr(), 0,
                                         None, MAX_WAYPTS, dn.data_ptr(), dw.data_ptr()) == 0
    assert lib().fuelgpu_poly_waypoints_batch_dev(m.handle, B, MAX_WAYPTS, dn.data_ptr(), dw.data_ptr(), zero.data_ptr(),
                                                  zero.data_ptr(), None, None, None, C.byref(pp), pinfo.data_ptr(),
                                                  None, pts.data_ptr(), der.data_ptr()) == 0
    m.synchronize()
    pinfo = np.frombuffer(pinfo.cpu().numpy().tobytes(), dtype=POLY_INFO)
    oinfo, _, on, ow = OA.search_batch(om, q["start"], q["goal"], 0.2, 1.0, 40000, 100000, path_max=1, w_max=MAX_WAYPTS)
    ok = on > 0
    assert np.count_nonzero(ok) > 50
    tours = [ow[b, :on[b]] for b in np.flatnonzero(ok)]
    hinfo, _, hpts, hder = waypoints_batch(m, tours, np.zeros(3), np.zeros(3), with_coeffs=False)
    assert hinfo.tobytes() == pinfo[ok].tobytes()
    assert np.array_equal(hpts, pts.cpu().numpy()[ok]) and np.array_equal(hder, der.cpu().numpy()[ok])
    assert np.all(pinfo["status"][~ok] == 2)  # FUELGPU_POLY_BAD_INPUT: n_wp = 0


def test_plan_explore_traj_on_device_tours(office):
    """plan_explore_traj_batch on the device's tours equals its run on the oracle's tours"""
    from fuel_b200 import BsplineOptimizer, EDTEnvironment
    from fuel_b200.polynomial_traj import plan_explore_traj_batch
    g, inflate, tri, m, om = office
    m.updateESDF3d()
    q = W.make_path_queries(g, inflate, tri, B=96, seed=13)
    r = search_paths_batch(m, q["start"], q["goal"], resolution=0.2, lambda_heu=1.0, allocate_num=40000)
    oinfo, _, on, ow = OA.search_batch(om, q["start"], q["goal"], 0.2, 1.0, 40000, 100000, path_max=1)
    idx = [b for b in range(96) if r["tours"][b] is not None]
    assert len(idx) > 10 and all(on[b] == len(r["tours"][b]) for b in idx)
    env = EDTEnvironment()
    env.setMap(m)
    opt = BsplineOptimizer()
    opt.setEnvironment(env)
    solve = dict(cost_function=opt.NORMAL_PHASE | opt.MINTIME, max_eval=40)
    a = plan_explore_traj_batch(m, [r["tours"][b] for b in idx], np.zeros(3), np.zeros(3), 0.5, opt, solve, dict(
        max_vel=2.0, max_acc=2.0))
    b_ = plan_explore_traj_batch(m, [ow[b, :on[b]] for b in idx], np.zeros(3), np.zeros(3), 0.5, opt, solve, dict(
        max_vel=2.0, max_acc=2.0))
    assert a["info"].tobytes() == b_["info"].tobytes()
    assert a["report"].tobytes() == b_["report"].tobytes() and np.array_equal(a["best"], b_["best"])


def test_astar_class_b1(office):
    g, inflate, tri, m, om = office
    q = W.make_path_queries(g, inflate, tri, B=8, seed=21)
    a = Astar(m, resolution=0.2, lambda_heu=1.0, allocate_num=40000, max_iter=100000)
    want = OA.search_batch(om, q["start"], q["goal"], 0.2, 1.0, 40000, 100000, path_max=100001)
    for b in range(8):
        a.reset()
        st = a.search(q["start"][b], q["goal"][b])
        assert st == want[0]["status"][b] and a.iter_num_ == want[0]["iter_num"][b]
        p = np.array(a.getPath()).reshape(-1, 3)
        assert np.array_equal(p, want[1][b, :len(p)]) and len(p) == want[0]["n_path"][b]
