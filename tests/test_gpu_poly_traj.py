"""fuelgpu_poly_waypoints_batch[_dev] on the H100: the coefficients against an exact rational minimizer, the sampling
of planExploreTraj against the CPU oracle (oracle.poly, pinned on the reference's PolynomialTraj by
tests/test_oracle_poly.py), the error paths, and plan_explore_traj_batch against the existing entries group by group."""
import ctypes as C

import numpy as np
import pytest

import oracle.poly as OP
import oracle.param as OPA
from fuel_b200 import workloads as W
from fuel_b200._lib import FuelPolyParams
from fuel_b200.polynomial_traj import (BAD_INPUT, INFO_DTYPE, TOO_LONG, PolynomialTraj, plan_explore_traj_batch,
                                       select_best, waypoints_batch)
from tests.helpers import make_sdf_map
from tests.poly_cases import exact_minjerk, grid_cases

pytestmark = pytest.mark.gpu

LIM = dict(max_vel=2.0, max_acc=2.0)


@pytest.fixture(scope="module")
def free_map(fuel):
    g = W.Grid((80, 60, 30), (-4.0, -3.0, -0.5), 0.1)
    m = make_sdf_map(fuel, g, np.zeros(g.n, np.int8), np.full(g.n, W.FREE, np.uint8))
    yield m
    m.close()


def test_coefficients_match_exact_minimizer(free_map):
    """within 1e-11 * max(1, max|c|) of the exact minimizer, S in {2, 3, 8, 20, 31}, times from 0.05 to 5 s"""
    cases = grid_cases()
    info, coeffs, _, _ = waypoints_batch(free_map, [c[0] for c in cases], np.stack([c[1] for c in cases]),
                                         np.stack([c[2] for c in cases]), times=[c[3] for c in cases])
    for b, (w, v, a, t) in enumerate(cases):
        ex = exact_minjerk(w, v, a, t)
        err = np.abs(coeffs[b, :len(t)] - ex).max()
        assert err <= 1e-11 * max(1.0, np.abs(ex).max()), (b, len(t), err)
        assert np.all(coeffs[b, len(t):] == 0)


@pytest.mark.parametrize("which,B", [("office", 1024), ("office3", 4096)])
def test_sampling_matches_oracle(free_map, which, B):
    """times, duration, dt and K bit for bit; seg_num equal except within 1e-9 of an integer; length within 1e-12
    relative; samples and boundary derivatives within 1e-11 * max(1, |value|)"""
    g, inflate = W.office_map() if which == "office" else W.office3_map()
    tr = W.make_tours(g, inflate, B=B)
    info, coeffs, points, derivs = waypoints_batch(free_map, tr["tours"], tr["start_vel"], tr["start_acc"])
    near_integer = 0
    statuses = set()
    for b, tour in enumerate(tr["tours"]):
        o = OP.explore_samples(tour, tr["start_vel"][b], tr["start_acc"][b])
        r = info[b]
        assert r["duration"] == o["duration"], b
        q = o["length"] / 0.35
        if abs(q - round(q)) < 1e-9:
            near_integer += 1
            continue
        assert r["seg_num"] == o["seg_num"], b
        assert r["dt"] == o["dt"] and r["n_pts"] == o["K"] + 2, b
        assert abs(r["length"] - o["length"]) <= 1e-12 * o["length"], b
        statuses.add(int(r["status"]))
        if r["status"] == TOO_LONG:
            assert np.all(points[b] == 0)
            continue
        assert r["status"] == 0
        K = o["K"]
        np.testing.assert_allclose(points[b, :K], o["points"], rtol=0, atol=1e-11 * max(1.0, np.abs(o["points"]).max()))
        assert np.all(points[b, K:] == 0)
        np.testing.assert_allclose(derivs[b], o["derivs"], rtol=0, atol=1e-11 * max(1.0, np.abs(o["derivs"]).max()))
    print("seg_num within 1e-9 of an integer: %d of %d" % (near_integer, B))
    assert near_integer == 0
    assert TOO_LONG in statuses and len({int(n) for n in info["n_pts"]}) > 5


def test_given_times_equal_computed(free_map):
    """times = NULL computes |dp| / (max_vel * 0.5) as the oracle does: passing the oracle's times gives the same bytes"""
    g, inflate = W.office_map()
    tr = W.make_tours(g, inflate, B=64, seed=5)
    times = [OP.explore_samples(t, v, a)["times"] for t, v, a in zip(tr["tours"], tr["start_vel"], tr["start_acc"])]
    a = waypoints_batch(free_map, tr["tours"], tr["start_vel"], tr["start_acc"])
    b = waypoints_batch(free_map, tr["tours"], tr["start_vel"], tr["start_acc"], times=times)
    for x, y in zip(a, b):
        assert x.tobytes() == y.tobytes()


def _packed(tours):
    B = len(tours)
    w_max = max(len(t) for t in tours)
    wp = np.zeros((B, w_max, 3))
    for b, t in enumerate(tours):
        wp[b, :len(t)] = t
    return np.array([len(t) for t in tours], dtype=np.int32), wp, w_max


def test_host_entry_refuses_and_writes_nothing(free_map, fuel):
    L = fuel.lib()
    h = free_map.handle
    tours = [np.array([[0.0, 0, 0], [1, 0, 0], [2, 1, 0]]), np.array([[0.0, 0, 0], [0, 1, 0], [1, 1, 0], [1, 2, 0]])]
    n_wp, wp, w_max = _packed(tours)
    z = np.zeros((2, 3))
    good = FuelPolyParams(2.0, 0.35, 8, 0)

    def call(n_wp=n_wp, wp=wp, w_max=w_max, prm=good, times=None):
        info = np.full(2, 7, dtype=INFO_DTYPE)
        pts, der = np.full((2, 62, 3), 7.0), np.full((2, 4, 3), 7.0)
        rc = L.fuelgpu_poly_waypoints_batch(h, 2, w_max, n_wp.ctypes.data, wp.ctypes.data, z.ctypes.data, z.ctypes.data,
                                            None, None, None if times is None else times.ctypes.data, C.byref(prm),
                                            info.ctypes.data, None, pts.ctypes.data, der.ctypes.data)
        return rc, info, pts, der

    assert call()[0] == 0
    rep = wp.copy()
    rep[0, 1] = rep[0, 0]  # a repeated waypoint: zero segment time
    bad_times = np.array([[1.0, np.inf, 0], [1.0, 1.0, 1.0]])
    for kw in (dict(n_wp=np.array([2, 4], np.int32)), dict(n_wp=np.array([3, 33], np.int32)), dict(w_max=3),
               dict(wp=rep), dict(times=bad_times), dict(prm=FuelPolyParams(0.0, 0.35, 8, 0)),
               dict(prm=FuelPolyParams(2.0, np.nan, 8, 0)), dict(prm=FuelPolyParams(2.0, 0.35, 0, 0))):
        rc, info, pts, der = call(**kw)
        assert rc == -1, kw
        assert np.all(pts == 7.0) and np.all(der == 7.0) and np.all(info["seg_num"] == 7), kw


def test_dev_entry_marks_bad_tours(free_map, fuel):
    """a bad tour gets NaN and BAD_INPUT, its neighbours the host entry's bytes; a too-long tour gets TOO_LONG; the
    host and _dev entries agree byte for byte; coeffs = NULL changes nothing else"""
    import torch
    g, inflate = W.office_map()
    tr = W.make_tours(g, inflate, B=32, seed=6)
    tours = list(tr["tours"])
    ref = waypoints_batch(free_map, tours, tr["start_vel"], tr["start_acc"])
    nocoef = waypoints_batch(free_map, tours, tr["start_vel"], tr["start_acc"], with_coeffs=False)
    for x, y in zip((ref[0], ref[2], ref[3]), (nocoef[0], nocoef[2], nocoef[3])):
        assert x.tobytes() == y.tobytes()
    assert ref[0]["status"][-1] == TOO_LONG
    n_wp, wp, w_max = _packed(tours)
    bad = [3, 10]
    n_wp_bad = n_wp.copy()
    n_wp_bad[3] = 2
    wp_bad = wp.copy()
    wp_bad[10, 1] = wp_bad[10, 0]
    dev = torch.device("cuda")
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)  # noqa: E731
    d_n, d_wp, d_sv, d_sa = t(n_wp_bad), t(wp_bad), t(tr["start_vel"]), t(tr["start_acc"])
    B = len(tours)
    d_info = torch.empty(B * INFO_DTYPE.itemsize, dtype=torch.uint8, device=dev)
    d_c = torch.empty((B, w_max - 1, 3, 6), dtype=torch.float64, device=dev)
    d_p = torch.empty((B, 62, 3), dtype=torch.float64, device=dev)
    d_d = torch.empty((B, 4, 3), dtype=torch.float64, device=dev)
    prm = FuelPolyParams(2.0, 0.35, 8, 0)
    torch.cuda.synchronize()
    rc = fuel.lib().fuelgpu_poly_waypoints_batch_dev(free_map.handle, B, w_max, d_n.data_ptr(), d_wp.data_ptr(),
                                                     d_sv.data_ptr(), d_sa.data_ptr(), None, None, None, C.byref(prm),
                                                     d_info.data_ptr(), d_c.data_ptr(), d_p.data_ptr(), d_d.data_ptr())
    assert rc == 0
    free_map.synchronize()
    info = np.frombuffer(d_info.cpu().numpy().tobytes(), dtype=INFO_DTYPE)
    c, p, d = d_c.cpu().numpy(), d_p.cpu().numpy(), d_d.cpu().numpy()
    for b in range(B):
        if b in bad:
            assert info[b]["status"] == BAD_INPUT and np.isnan(info[b]["duration"]) and info[b]["n_pts"] == 0
            assert np.all(np.isnan(p[b])) and np.all(np.isnan(d[b])) and np.all(np.isnan(c[b]))
        else:
            assert info[b].tobytes() == ref[0][b].tobytes()
            assert c[b].tobytes() == ref[1][b].tobytes() and p[b].tobytes() == ref[2][b].tobytes()
            assert d[b].tobytes() == ref[3][b].tobytes()


def test_python_mirror(free_map):
    """PolynomialTraj agrees with waypoints_batch: its coefficients, getTotalTime and evaluate at the sample times"""
    g, inflate = W.office_map()
    tr = W.make_tours(g, inflate, B=8, seed=8)
    info, coeffs, points, derivs = waypoints_batch(free_map, tr["tours"], tr["start_vel"], tr["start_acc"])
    for b, tour in enumerate(tr["tours"][:-1]):
        times = OP.explore_samples(tour, tr["start_vel"][b], tr["start_acc"][b])["times"]
        pt = PolynomialTraj(free_map)
        PolynomialTraj.waypointsTraj(tour, tr["start_vel"][b], np.zeros(3), tr["start_acc"][b], np.zeros(3), times, pt)
        assert pt.coeffs_.tobytes() == coeffs[b, :len(times)].tobytes()
        assert pt.getTotalTime() == info[b]["duration"]
        assert pt.getLength() == info[b]["length"]
        ts, K = 0.0, info[b]["n_pts"] - 2
        for k in range(K):
            np.testing.assert_allclose(pt.evaluate(ts, 0), points[b, k], rtol=0, atol=1e-12 * max(1, np.abs(points[b]).max()))
            ts += info[b]["dt"]
        np.testing.assert_allclose(pt.evaluate(info[b]["duration"], 2), derivs[b, 3], rtol=0, atol=1e-9)


def test_plan_explore_chain(fuel):
    """plan_explore_traj_batch on a mixed-n_pts batch equals the same device samples run group by group through the
    existing host entries, and its best equals selectBestTraj over the merged reports; the oracle's samples through the
    parameterize path give control points within the parameterize bar of the device chain's"""
    from fuel_b200 import BsplineOptimizer
    from fuel_b200.non_uniform_bspline import check_batch, parameterize_batch
    from fuel_b200.sdf_map import EDTEnvironment
    g, inflate = W.office_map()
    m = make_sdf_map(fuel, g, inflate, np.where(inflate == 1, W.OCCUPIED, W.FREE).astype(np.uint8))
    try:
        tr = W.make_tours(g, inflate, B=96, seed=9)
        opt = BsplineOptimizer()
        opt.setParam()
        env = EDTEnvironment()
        env.setMap(m)
        opt.setEnvironment(env)
        mask = opt.NORMAL_PHASE | opt.MINTIME
        solve = dict(cost_function=mask, max_eval=64)
        out = plan_explore_traj_batch(m, tr["tours"], tr["start_vel"], tr["start_acc"], -1.0, opt, solve, LIM)
        info, _, points, derivs = waypoints_batch(m, tr["tours"], tr["start_vel"], tr["start_acc"], with_coeffs=False)
        assert out["info"].tobytes() == info.tobytes()
        groups = sorted(set(info["n_pts"][info["status"] == 0].tolist()))
        assert len(groups) > 3
        for n in groups:
            idx = np.flatnonzero((info["status"] == 0) & (info["n_pts"] == n))
            x0, tc = parameterize_batch(m, points[idx, :n - 2], derivs[idx], info["dt"][idx], time_lb=-1.0)
            x, _, _ = opt.optimizeBatch(x0, tc, n, mask, 64)
            rep, _ = check_batch(m, x, n, **LIM)
            assert out["report"][idx].tobytes() == rep.tobytes()
            for r, b in enumerate(idx):
                assert out["x"][b].tobytes() == x[r].tobytes()
            # the oracle's samples through the same parameterization: within the parameterize bar
            for r, b in enumerate(idx[:4]):
                o = OP.explore_samples(tr["tours"][b], tr["start_vel"][b], tr["start_acc"][b])
                xo, _ = OPA.bspline_parameterize(o["points"][None], o["derivs"][None], np.array([o["dt"]]))
                np.testing.assert_allclose(x0[r], xo[0], rtol=0, atol=2e-11 * max(1.0, np.abs(xo).max()))
        too_long = np.flatnonzero(info["status"] == TOO_LONG)
        assert len(too_long) >= 1 and all(out["x"][b] is None for b in too_long)
        assert np.all(np.isnan(out["report"]["jerk"][too_long]))
        assert out["best"].tolist() == select_best(out["report"]).tolist()
        j = out["report"]["jerk"]
        assert out["best"][0] == int(np.nanargmin(j))
    finally:
        m.close()

