"""Pins the trajectory-check oracle (oracle/fuel_oracle_traj.c) against the REFERENCE's own NonUniformBspline
(bspline/src/non_uniform_bspline.cpp, compiled unmodified into oracle/_ref/libfuel_ref_traj.so by oracle/traj.mk), its
checkTrajCollision loop (planner_manager.cpp:96-118, restated over the reference's evaluateDeBoorT and
SDFMap::getInflateOccupancy in oracle/ref_traj_wrap.cpp) and selectBestTraj (:476-482), bit for bit.  Where the reference
library is not built, the digests in tests/golden/refpin_traj.json stand in for it (tests/refgold.py's scheme).
Independent ground truths: scipy's BSpline on the same knots, the jerk integral of the piecewise-constant third
derivative, and a brute-force sequential collision scan.

  FUEL_REFPIN_RECORD=1 python -m pytest tests/test_oracle_traj.py

rewrites the digests from a run against the built reference."""
import numpy as np
import pytest
from scipy.interpolate import BSpline

import oracle.traj as O
from oracle import make_grid as O_grid
from fuel_b200 import workloads as W
from tests.refgold import ref_map, refgold_fixture

O.build()  # also builds oracle/_ref/libfuel_ref_traj.so where the reference's sources are present (git-ignored)


BASE = dict(resolution=0.1, map_size_x=8.0, map_size_y=6.0, map_size_z=3.0, ground_height=-0.5, obstacles_inflation=0.199,
            local_bound_inflate=0.5, local_map_margin=50, default_dist=0.0, optimistic=0, signed_dist=0, p_hit=0.65,
            p_miss=0.35, p_min=0.12, p_max=0.90, p_occ=0.80, max_ray_length=4.5, virtual_ceil_height=-10.0)


G = refgold_fixture("refpin_traj.json", O.ref_traj)


def random_trajs(rng, B, n, lo=(-3.5, -2.5, 0.0), hi=(3.5, 2.5, 2.0), step=0.25, dt_range=(0.05, 0.6)):
    """random walks of n control points starting inside [lo, hi], knot spans in dt_range"""
    lo, hi = np.array(lo), np.array(hi)
    ctrl = np.zeros((B, n, 3))
    ctrl[:, 0] = rng.uniform(lo, hi, (B, 3))
    d = rng.normal(size=(B, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    for i in range(1, n):
        d = d + rng.normal(scale=0.5, size=(B, 3))
        d /= np.linalg.norm(d, axis=1, keepdims=True)
        ctrl[:, i] = ctrl[:, i - 1] + step * d
    return ctrl, rng.uniform(*dt_range, B)


def knots(n, dt):
    """setUniformBspline's running-sum knot vector (:16-32)"""
    u = np.zeros(n + 4)
    for i in range(n + 4):
        u[i] = float(-3 + i) * dt if i <= 3 else u[i - 1] + dt
    return u


def sample_times(rng, n, dt):
    u = knots(n, dt)
    dur = u[n] - u[3]
    return np.concatenate([[0.0, dur, -0.3, dur + 0.5, -0.0], u[3:n + 1] - u[3], rng.uniform(0, dur, 40)])


@pytest.mark.parametrize("n", [4, 7, 20, 33, 64])
def test_evaluate_matches_reference(G, n):
    rng = np.random.default_rng(100 + n)
    ctrl, dt = random_trajs(rng, 6, n)
    ts = [sample_times(rng, n, dt[b]) for b in range(6)]
    for deriv in range(3):
        got = [O.bspline_evaluate(W.pack_x(ctrl[b:b + 1], dt[b:b + 1]), n, ts[b][None, :], deriv)[0] for b in range(6)]
        G.eq(got, lambda: [O.ref_traj_evaluate(ctrl[b], dt[b], ts[b], deriv) for b in range(6)])


@pytest.mark.parametrize("n", [4, 12, 31, 64])
def test_duration_jerk_ratio_feasibility_match_reference(G, n):
    rng = np.random.default_rng(200 + n)
    B = 40
    ctrl, dt = random_trajs(rng, B, n, dt_range=(0.08, 0.4))
    ctrl[:4] *= 1e-3  # slow, feasible
    lim = [(2.0, 2.0), (3.0, 1.0), (0.5, 4.0)]
    g = O_grid((80, 60, 30), 0.1, (-4.0, -3.0, -0.5))
    infl = np.zeros((80, 60, 30), np.int8)
    for vmax, amax in lim:
        rep, _ = O.bspline_check(g, infl, W.pack_x(ctrl, dt), n, vmax, amax)
        got = [[r["duration"], r["jerk"], r["ratio"], r["feasible"]] for r in rep]
        G.eq(got, lambda: [list(O.ref_traj_stats(ctrl[b], dt[b], vmax, amax)) for b in range(B)])
    assert 0 < rep["feasible"].sum() < B


def collision_scene(seed):
    ref = ref_map(**BASE)
    rng = np.random.default_rng(seed)
    infl = (rng.random(ref.n) < 0.004).astype(np.int8)
    infl[40:43, 10:50, :] = 1  # a wall across the middle of the map
    ref.inflate[:] = infl.reshape(-1)
    return ref, infl


@pytest.mark.parametrize("n", [6, 20, 64])
def test_collision_scan_matches_reference(G, n):
    ref, infl = collision_scene(300 + n)
    g = ref.grid()
    rng = np.random.default_rng(400 + n)
    B = 48
    ctrl, dt = random_trajs(rng, B, n, step=0.3 if n < 64 else 0.12)
    ctrl[:6, :, 0] += 6.0  # some leave the map (outside is -1, not a hit)
    x = W.pack_x(ctrl, dt)
    for t_now in (0.0, 0.37, 2.0):
        rep, _ = O.bspline_check(g, infl, x, n, 2.0, 2.0, t_now=t_now)
        got = [[r["safe"], r["distance"], r["n_checked"]] for r in rep]
        G.eq(got, lambda: [list(O.ref_traj_check_collision(ref, ctrl[b], dt[b], t_now)) for b in range(B)])
        if t_now == 0.0:
            assert 0 < rep["safe"].sum() < B
    ref.close()


def test_select_best_matches_reference(G):
    rng = np.random.default_rng(5)
    ctrl, dt = random_trajs(rng, 30, 16)
    g = O_grid((80, 60, 30), 0.1, (-4.0, -3.0, -0.5))
    rep, best = O.bspline_check(g, np.zeros((80, 60, 30), np.int8), W.pack_x(ctrl, dt), 16, 2.0, 2.0)
    assert len(np.unique(rep["jerk"])) == 30
    G.eq([best[0]], lambda: [O.ref_traj_select_best(ctrl, dt)])


# ---- independent ground truths -------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [4, 20, 64])
def test_evaluate_matches_scipy(n):
    rng = np.random.default_rng(7 + n)
    ctrl, dt = random_trajs(rng, 4, n)
    for b in range(4):
        u = knots(n, dt[b])
        sp = BSpline(u, ctrl[b], 3)
        t = np.linspace(0.0, u[n] - u[3], 97)
        for deriv in range(3):
            got = O.bspline_evaluate(W.pack_x(ctrl[b:b + 1], dt[b:b + 1]), n, t[None, :], deriv)[0]
            want = sp.derivative(deriv)(t + u[3]) if deriv else sp(t + u[3])
            scale = np.abs(want).max() + 1.0
            assert np.allclose(got, want, rtol=1e-10, atol=1e-10 * scale)


def test_jerk_is_the_integral_of_the_squared_third_derivative():
    rng = np.random.default_rng(8)
    n = 24
    ctrl, dt = random_trajs(rng, 10, n)
    g = O_grid((80, 60, 30), 0.1, (-4.0, -3.0, -0.5))
    rep, best = O.bspline_check(g, np.zeros((80, 60, 30), np.int8), W.pack_x(ctrl, dt), n, 2.0, 2.0)
    for b in range(10):
        u = knots(n, dt[b])
        d3 = BSpline(u, ctrl[b], 3).derivative(3)
        mids = 0.5 * (u[3:n] + u[4:n + 1])
        integral = np.sum(np.sum(d3(mids) ** 2, axis=1) * (u[4:n + 1] - u[3:n]))
        assert rep["jerk"][b] == pytest.approx(integral, rel=1e-9)
    assert best[0] == int(np.argmin(rep["jerk"]))


def brute_force_scan(g, infl, ctrl, dt, t_now):
    """checkTrajCollision as a plain sequential loop over the oracle's evaluateDeBoorT"""
    n = ctrl.shape[0]
    x = W.pack_x(ctrl[None], np.array([dt]))
    u = knots(n, dt)
    duration = u[n] - u[3]
    ev = lambda t: O.bspline_evaluate(x, n, np.array([[t]]))[0, 0]  # noqa: E731
    cur = ev(t_now)
    origin, res_inv, nv = np.array(g.origin[:]), 1 / g.res, np.array(g.n[:])
    radius, fut_t, k = 0.0, 0.02, 0
    while radius < 6.0 and t_now + fut_t < duration:
        p = ev(t_now + fut_t)
        k += 1
        idx = np.floor((p - origin) * res_inv)
        if np.all(idx >= 0) and np.all(idx <= nv - 1) and infl[int(idx[0]), int(idx[1]), int(idx[2])] == 1:
            return 0, radius, k
        d = p - cur
        radius = float(np.sqrt(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]))
        fut_t += 0.02
    return 1, -1.0, k


def test_collision_scan_matches_brute_force():
    rng = np.random.default_rng(9)
    g = O_grid((80, 60, 30), 0.1, (-4.0, -3.0, -0.5))
    infl = (rng.random((80, 60, 30)) < 0.003).astype(np.int8)
    n, B = 12, 24
    ctrl, dt = random_trajs(rng, B, n, step=0.35)
    ctrl[:3, :, 1] -= 4.0
    for t_now in (0.0, 0.5):
        rep, _ = O.bspline_check(g, infl, W.pack_x(ctrl, dt), n, 2.0, 2.0, t_now=t_now)
        for b in range(B):
            assert (rep["safe"][b], rep["distance"][b], rep["n_checked"][b]) == brute_force_scan(g, infl, ctrl[b], dt[b], t_now)
    assert 0 < rep["safe"].sum() < B


def test_dt_column_and_dt_array_layouts_agree():
    rng = np.random.default_rng(10)
    g = O_grid((80, 60, 30), 0.1, (-4.0, -3.0, -0.5))
    infl = (rng.random((80, 60, 30)) < 0.003).astype(np.int8)
    ctrl, dt = random_trajs(rng, 16, 20)
    a, ba = O.bspline_check(g, infl, W.pack_x(ctrl, dt), 20, 2.0, 2.0)
    b, bb = O.bspline_check(g, infl, W.pack_x(ctrl, dt, mintime=False), 20, 2.0, 2.0, dt=dt)
    assert a.tobytes() == b.tobytes() and np.array_equal(ba, bb)
