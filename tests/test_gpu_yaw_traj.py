"""fuelgpu_yaw_explore_batch[_dev] on the H100: dt_yaw and the waypoint count against the CPU oracle (oracle.yaw, pinned
on the reference's planYawExplore by tests/test_oracle_yaw.py) bit for bit, the waypoints to atan2's rounding and pt_dist_
bit for bit given them, the control points against the exact rational minimizer of the objective built from the device's own
waypoints, optimality under the oracle's pinned combineCost, the error paths, and the chain behind the solver."""
import ctypes as C

import numpy as np
import pytest

import oracle.yaw as OY
from fuel_b200 import workloads as W
from fuel_b200._lib import FuelOptParams, FuelSolveParams, FuelTrajCheckParams, FuelTrajConst, FuelYawParams
from fuel_b200.polynomial_traj import (YAW_BAD_INPUT, YAW_INFO_DTYPE, YAW_NO_LOOKAHEAD, YAW_RELAX_OVERFLOW,
                                       YAW_ZERO_PT_DIST, plan_explore_traj_batch, plan_yaw_explore_batch)
from tests.helpers import make_sdf_map
from tests.yaw_cases import DT_YAW_GRID, LD, arc_batch, exact_minimizer, solve_bar

pytestmark = pytest.mark.gpu

LIM = dict(max_vel=2.0, max_acc=2.0)


def opt_params():
    p = FuelOptParams()
    p.ld_smooth, p.ld_start, p.ld_end, p.ld_waypt = LD["ld_smooth"], LD["ld_start"], LD["ld_end"], LD["ld_waypt"]
    p.order = 3
    return p


@pytest.fixture(scope="module")
def free_map(fuel):
    g = W.Grid((40, 40, 20), (-2.0, -2.0, -0.5), 0.1)
    m = make_sdf_map(fuel, g, np.zeros(g.n, np.int8), np.full(g.n, W.FREE, np.uint8))
    yield m
    m.close()


def solved(fuel, mk, B, n):
    g, inflate = mk()
    tri = W.office_known(g, inflate)
    m = make_sdf_map(fuel, g, inflate, tri, optimistic=True)
    m.updateESDF3d()
    env = fuel.EDTEnvironment()
    env.setMap(m)
    opt = fuel.BsplineOptimizer()
    opt.setEnvironment(env)
    tr = W.make_trajectories(g, inflate, B=B, n_pts=n)
    tcs = opt.traj_consts_from_arrays(tr["pt_dist"], tr["dt"], tr["start"], tr["end_pos"])
    x, _, _ = opt.optimizeBatch(W.pack_x(tr["ctrl"], tr["dt"]), tcs, n, opt.NORMAL_PHASE | opt.MINTIME, 64)
    return m, x


def heading(x, n):
    c = x[:, :3 * n].reshape(len(x), n, 3)
    d = c[:, -1] - c[:, -4]
    return np.arctan2(d[:, 1], d[:, 0])


def check_against_oracle(rows, yaw, info, waypt):
    """dt_yaw and n_waypt bit for bit; waypoints to 1e-13; pt_dist bit for bit given the device's waypoints (the end yaw
    follows the last one through calcNextYaw) and within 1e-13 of the oracle's own; control points to the exact
    minimizer of the objective built from the device's waypoints; optimality under the pinned combineCost"""
    near_pi = 0
    dr = []
    for b, r in enumerate(rows):
        assert info["status"][b] == r["status"] == 0, b
        assert info["dt_yaw"][b] == r["dt_yaw"], b
        assert info["n_waypt"][b] == len(r["waypts"]), b
        assert np.all(waypt[b, len(r["waypts"]):] == 0)
        d = OY.with_waypoints(r, waypt[b, :info["n_waypt"][b]])
        assert info["pt_dist"][b] == d["pt_dist"], b
        dr.append(d)
        if r["margin"] < 1e-12:
            near_pi += 1
            continue
        w = np.array(r["waypts"])
        assert np.all(np.abs(waypt[b, :len(w)] - w) <= 1e-13 * np.maximum(1.0, np.abs(w))), b
        assert abs(info["pt_dist"][b] - r["pt_dist"]) <= 1e-13 * r["pt_dist"], b
    exact = np.array([[float(v) for v in exact_minimizer(r, **LD)] for r in dr])
    for b, r in enumerate(dr):
        ex = exact[b]
        bar = solve_bar(r, **LD)
        err = np.abs(yaw[b] - ex).max()
        assert err <= bar * max(1.0, np.abs(ex).max()), (b, r["dt_yaw"], err)
    f, g = OY.objective(dr, yaw, **LD)
    f0, g0 = OY.objective(dr, np.array([r["guess"] for r in dr]), **LD)
    fx, _ = OY.objective(dr, exact, **LD)
    assert np.all(np.abs(g).max(1) <= 1e-9 * np.abs(g0).max(1))
    assert np.all(f <= fx * (1 + 1e-12))
    return near_pi


@pytest.mark.parametrize("layout", ["mintime", "dt"])
@pytest.mark.parametrize("which,B,n", [("office", 1024, 20), ("office3", 4096, 64)])
def test_solver_output_matches_oracle(fuel, which, B, n, layout):
    m, x = solved(fuel, W.office_map if which == "office" else W.office3_map, B, n)
    ys = W.make_yaws(B, heading=heading(x, n))
    if layout == "dt":
        xin, dt = np.ascontiguousarray(x[:, :3 * n]), x[:, 3 * n].copy()
    else:
        xin, dt = x, None
    yaw, info, waypt = plan_yaw_explore_batch(m, xin, n, ys["start"], ys["end"], opt_params(), dt=dt)
    rows = OY.plan(xin, n, ys["start"], ys["end"], dt=dt)
    near_pi = check_against_oracle(rows, yaw, info, waypt)
    print("calcNextYaw |diff| within 1e-12 of pi: %d of %d" % (near_pi, B))
    assert near_pi == 0
    assert len(set(info["n_waypt"].tolist())) > 1
    m.close()


def test_dt_yaw_grid_down_to_002(free_map):
    """solve_bar of the exact minimizer on dt_yaw from 0.02 to 1 s; several start turns and near-pi end yaws"""
    dts = [d for d in DT_YAW_GRID for _ in range(6)]
    x = arc_batch(dts)
    ys = W.make_yaws(len(dts), seed=4, heading=heading(x, 20))
    for relax in (0.0, 1.0, 3.0):
        yaw, info, waypt = plan_yaw_explore_batch(free_map, x, 20, ys["start"], ys["end"], opt_params(), relax_time=relax)
        rows = OY.plan(x, 20, ys["start"], ys["end"], relax_time=relax)
        assert check_against_oracle(rows, yaw, info, waypt) == 0


def test_undefined_cases_get_their_status(free_map):
    """all-zero yaws, a hovering trajectory and a huge relax_time: status and NaN yaw, the neighbours unaffected"""
    x = arc_batch([0.1, 0.1, 0.1, 1.0, 0.1])
    x[1, :60] = np.stack([0.05 * np.arange(20), np.zeros(20), np.ones(20)], 1).reshape(-1)  # along +x: waypoints 0
    x[2, :60] = np.tile([0.3, -0.2, 1.0], 20)  # hovering
    ys = W.make_yaws(5, seed=5)
    ys["start"][1] = 0.0
    ys["end"][1] = 0.0
    p = opt_params()
    alone = [plan_yaw_explore_batch(free_map, x[b:b + 1], 20, ys["start"][b:b + 1], ys["end"][b:b + 1], p) for b in (0, 3, 4)]
    yaw, info, waypt = plan_yaw_explore_batch(free_map, x, 20, ys["start"], ys["end"], p)
    assert info["status"].tolist() == [0, YAW_ZERO_PT_DIST, YAW_NO_LOOKAHEAD, 0, 0]
    for b in (1, 2):
        assert np.all(np.isnan(yaw[b])) and np.isfinite(info["dt_yaw"][b])
    assert info["pt_dist"][1] == 0.0 and info["n_waypt"][1] > 0 and np.all(np.isfinite(waypt[1]))
    assert np.isnan(info["pt_dist"][2]) and info["n_waypt"][2] == 0 and np.all(np.isnan(waypt[2]))
    rows = OY.plan(x, 20, ys["start"], ys["end"])
    assert [r["status"] for r in rows] == info["status"].tolist()
    for (ya, ia, wa), b in zip(alone, (0, 3, 4)):
        assert ya[0].tobytes() == yaw[b].tobytes() and ia[0].tobytes() == info[b].tobytes()
        assert wa[0].tobytes() == waypt[b].tobytes()
    # relax_time / dt_yaw >= 2^31 on the dt_yaw = 0.1 rows; dt_yaw = 1 stays below it: no waypoint, solved
    yaw, info, waypt = plan_yaw_explore_batch(free_map, x, 20, ys["start"], ys["end"], p, relax_time=1e9)
    assert info["status"].tolist() == [YAW_RELAX_OVERFLOW] * 3 + [0, YAW_RELAX_OVERFLOW]
    assert np.all(np.isnan(yaw[[0, 1, 2, 4]])) and np.all(np.isfinite(yaw[3])) and info["n_waypt"][3] == 0
    rows = OY.plan(x, 20, ys["start"], ys["end"], relax_time=1e9)
    assert [r["status"] for r in rows] == info["status"].tolist()
    # lookfwd = False: no waypoint anywhere, every row solved
    yaw, info, waypt = plan_yaw_explore_batch(free_map, x[[0, 3, 4]], 20, ys["start"][[0, 3, 4]], ys["end"][[0, 3, 4]], p,
                                              lookfwd=False)
    assert np.all(info["status"] == 0) and np.all(info["n_waypt"] == 0) and np.all(waypt == 0)
    rows = OY.plan(x[[0, 3, 4]], 20, ys["start"][[0, 3, 4]], ys["end"][[0, 3, 4]], lookfwd=False)
    check_against_oracle(rows, yaw, info, waypt)


def test_host_entry_refuses_and_writes_nothing(free_map, fuel):
    L = fuel.lib()
    h = free_map.handle
    x = arc_batch([0.1, 0.2])
    sy = np.zeros((2, 3)) + 0.5
    ey = np.array([0.1, -0.1])
    good, yp = opt_params(), FuelYawParams(1.0, 1, 0)

    def call(x=x, n=20, nvar=61, dt=None, sy=sy, ey=ey, p=good, yp=yp, B=2):
        yaw, wp = np.full((2, 15), 7.0), np.full((2, 11), 7.0)
        info = np.zeros(2, dtype=YAW_INFO_DTYPE)
        info["status"] = 7
        rc = L.fuelgpu_yaw_explore_batch(h, B, n, nvar, x.ctypes.data, None if dt is None else dt.ctypes.data,
                                         sy.ctypes.data, ey.ctypes.data, C.byref(p), C.byref(yp), yaw.ctypes.data,
                                         info.ctypes.data, wp.ctypes.data)
        return rc, yaw, info, wp

    assert call()[0] == 0
    bad_dt = x.copy()
    bad_dt[1, 60] = 0.0
    inf_dt = x.copy()
    inf_dt[0, 60] = np.inf

    def p_with(**kw):
        p = opt_params()
        for k, v in kw.items():
            setattr(p, k, v)
        return p
    cases = [dict(n=3, nvar=10), dict(nvar=62), dict(B=-1), dict(x=bad_dt), dict(x=inf_dt),
             dict(nvar=60, dt=np.array([0.1, np.nan])), dict(sy=np.array([[np.nan, 0, 0], [0, 0, 0.0]])),
             dict(sy=np.array([[0, 0, 0], [1000.5, 0, 0.0]])), dict(sy=np.array([[0, np.inf, 0], [0, 0, 0.0]])),
             dict(ey=np.array([0.0, np.nan])), dict(p=p_with(ld_smooth=0.0)), dict(p=p_with(ld_start=-1.0)),
             dict(yp=FuelYawParams(-1.0, 1, 0)), dict(yp=FuelYawParams(np.inf, 1, 0))]
    for kw in cases:
        if kw.get("nvar") == 60 and "x" not in kw:
            kw["x"] = np.ascontiguousarray(x[:, :60])
        rc, yaw, info, wp = call(**kw)
        assert rc == -1, kw
        assert np.all(yaw == 7.0) and np.all(wp == 7.0) and np.all(info["status"] == 7), kw
    # |start yaw| = 1000 exactly is accepted and wrapped like the reference
    rc, yaw, info, wp = call(sy=np.array([[1000.0, 0, 0], [-1000.0, 0, 0]]))
    assert rc == 0 and np.all(info["status"] == 0)


def _dev_call(fuel, m, x, n, dt, sy, ey, p, yp, stream=None):
    import torch
    t = lambda a: None if a is None else torch.from_numpy(np.ascontiguousarray(a)).cuda()  # noqa: E731
    B = len(x)
    d_x, d_dt, d_sy, d_ey = t(x), t(dt), t(sy), t(ey)
    d_yaw = torch.empty((B, 15), dtype=torch.float64, device="cuda")
    d_info = torch.empty(B * YAW_INFO_DTYPE.itemsize, dtype=torch.uint8, device="cuda")
    d_wp = torch.empty((B, 11), dtype=torch.float64, device="cuda")
    torch.cuda.synchronize()
    rc = fuel.lib().fuelgpu_yaw_explore_batch_dev(m.handle, B, n, x.shape[1], d_x.data_ptr(),
                                                  None if d_dt is None else d_dt.data_ptr(), d_sy.data_ptr(),
                                                  d_ey.data_ptr(), C.byref(p), C.byref(yp), d_yaw.data_ptr(),
                                                  d_info.data_ptr(), d_wp.data_ptr())
    assert rc == 0
    m.synchronize()
    return d_yaw.cpu().numpy(), np.frombuffer(d_info.cpu().numpy().tobytes(), dtype=YAW_INFO_DTYPE), d_wp.cpu().numpy()


def test_dev_entry_equals_host_and_marks_bad_rows(free_map, fuel):
    x = arc_batch(list(DT_YAW_GRID) * 4, seed=7)
    B = len(x)
    ys = W.make_yaws(B, seed=8, heading=heading(x, 20))
    p, yp = opt_params(), FuelYawParams(1.0, 1, 0)
    host = plan_yaw_explore_batch(free_map, x, 20, ys["start"], ys["end"], p)
    dev = _dev_call(fuel, free_map, x, 20, None, ys["start"], ys["end"], p, yp)
    for a, b in zip(host, dev):
        assert a.tobytes() == b.tobytes()
    xb, sy, ey = x.copy(), ys["start"].copy(), ys["end"].copy()
    bad = [1, 6, 11, 17, 23]
    xb[1, 60] = -0.1
    sy[6, 0] = np.nan
    sy[11, 0] = 2000.0
    sy[17, 2] = np.inf
    ey[23] = np.nan
    yaw, info, wp = _dev_call(fuel, free_map, xb, 20, None, sy, ey, p, yp)
    for b in range(B):
        if b in bad:
            assert info["status"][b] == YAW_BAD_INPUT and info["n_waypt"][b] == 0
            assert np.isnan(info["dt_yaw"][b]) and np.isnan(info["pt_dist"][b])
            assert np.all(np.isnan(yaw[b])) and np.all(np.isnan(wp[b]))
        else:
            assert yaw[b].tobytes() == host[0][b].tobytes() and info[b].tobytes() == host[1][b].tobytes()
            assert wp[b].tobytes() == host[2][b].tobytes()


def test_dev_chain_behind_the_check_equals_host_entries(fuel):
    """poly (host, its info read) -> parameterize -> optimize -> check -> yaw, all _dev on the map's main stream (a torch
    stream), equals the host entries group by group; plan_explore_traj_batch with start_yaw / end_yaw equals
    plan_explore_traj_batch followed by plan_yaw_explore_batch"""
    import torch

    from fuel_b200.non_uniform_bspline import REPORT_DTYPE, check_batch, parameterize_batch
    from fuel_b200.polynomial_traj import waypoints_batch
    g, inflate = W.office_map()
    m = make_sdf_map(fuel, g, inflate, np.where(inflate == 1, W.OCCUPIED, W.FREE).astype(np.uint8))
    st = torch.cuda.Stream()
    m.set_stream(st.cuda_stream)
    try:
        env = fuel.EDTEnvironment()
        env.setMap(m)
        opt = fuel.BsplineOptimizer()
        opt.setParam()
        opt.setEnvironment(env)
        mask = opt.NORMAL_PHASE | opt.MINTIME
        tr = W.make_tours(g, inflate, B=96, seed=9)
        ys = W.make_yaws(96, seed=10)
        L = fuel.lib()
        info, _, points, derivs = waypoints_batch(m, tr["tours"], tr["start_vel"], tr["start_acc"], with_coeffs=False)
        groups = sorted(set(info["n_pts"][info["status"] == 0].tolist()))
        assert len(groups) > 3
        sp = FuelSolveParams()
        sp.max_eval, sp.lbfgs_m, sp.xtol_rel = 64, 6, 1e-5
        cp = FuelTrajCheckParams(LIM["max_vel"], LIM["max_acc"], 0.0)
        yp = FuelYawParams(1.0, 1, 0)
        for n in groups:
            idx = np.flatnonzero((info["status"] == 0) & (info["n_pts"] == n))
            B, nvar = len(idx), 3 * n + 1
            with torch.cuda.stream(st):
                cu = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()  # noqa: E731
                d_pts, d_der, d_dt = cu(points[idx, :n - 2]), cu(derivs[idx]), cu(info["dt"][idx])
                d_tlb = cu(np.full(B, -1.0))
                d_sy, d_ey = cu(ys["start"][idx]), cu(ys["end"][idx])
                d_x = torch.empty((B, nvar), dtype=torch.float64, device="cuda")
                d_tc = torch.empty(B * C.sizeof(FuelTrajConst), dtype=torch.uint8, device="cuda")
                d_f = torch.empty(B, dtype=torch.float64, device="cuda")
                d_ne = torch.empty(B, dtype=torch.int32, device="cuda")
                d_rep = torch.empty(B * REPORT_DTYPE.itemsize, dtype=torch.uint8, device="cuda")
                d_best = torch.empty(2, dtype=torch.int32, device="cuda")
                d_yaw = torch.empty((B, 15), dtype=torch.float64, device="cuda")
                d_yi = torch.empty(B * YAW_INFO_DTYPE.itemsize, dtype=torch.uint8, device="cuda")
            st.synchronize()
            assert L.fuelgpu_bspline_parameterize_batch_dev(m.handle, B, n, nvar, d_pts.data_ptr(), d_der.data_ptr(),
                                                            d_dt.data_ptr(), d_tlb.data_ptr(), d_x.data_ptr(),
                                                            d_tc.data_ptr()) == 0
            assert L.fuelgpu_bspline_optimize_batch_dev(m.handle, B, n, mask, C.byref(opt.params_), d_tc.data_ptr(),
                                                        C.byref(sp), d_x.data_ptr(), d_f.data_ptr(), d_ne.data_ptr()) == 0
            assert L.fuelgpu_bspline_check_batch_dev(m.handle, B, n, nvar, d_x.data_ptr(), None, C.byref(cp),
                                                     d_rep.data_ptr(), d_best.data_ptr()) == 0
            assert L.fuelgpu_yaw_explore_batch_dev(m.handle, B, n, nvar, d_x.data_ptr(), None, d_sy.data_ptr(),
                                                   d_ey.data_ptr(), C.byref(opt.params_), C.byref(yp), d_yaw.data_ptr(),
                                                   d_yi.data_ptr(), None) == 0
            st.synchronize()
            x0, tc = parameterize_batch(m, points[idx, :n - 2], derivs[idx], info["dt"][idx], time_lb=-1.0)
            x, _, _ = opt.optimizeBatch(x0, tc, n, mask, 64)
            rep, _ = check_batch(m, x, n, **LIM)
            yaw, yinfo, _ = plan_yaw_explore_batch(m, x, n, ys["start"][idx], ys["end"][idx], opt)
            assert d_x.cpu().numpy().tobytes() == x.tobytes()
            assert d_rep.cpu().numpy().tobytes() == rep.tobytes()
            assert d_yaw.cpu().numpy().tobytes() == yaw.tobytes()
            assert d_yi.cpu().numpy().tobytes() == yinfo.tobytes()
        solve = dict(cost_function=mask, max_eval=64)
        out = plan_explore_traj_batch(m, tr["tours"], tr["start_vel"], tr["start_acc"], -1.0, opt, solve, LIM,
                                      start_yaw=ys["start"], end_yaw=ys["end"])
        plain = plan_explore_traj_batch(m, tr["tours"], tr["start_vel"], tr["start_acc"], -1.0, opt, solve, LIM)
        assert set(plain) == {"info", "x", "report", "best"} and set(out) == set(plain) | {"yaw", "yaw_info"}
        assert out["report"].tobytes() == plain["report"].tobytes()
        for b in range(96):
            if plain["x"][b] is None:
                assert out["yaw_info"]["status"][b] == -1 and np.all(np.isnan(out["yaw"][b]))
                continue
            n = int(info["n_pts"][b])
            yaw, yinfo, _ = plan_yaw_explore_batch(m, plain["x"][b][None], n, ys["start"][b], ys["end"][b], opt)
            assert out["yaw"][b].tobytes() == yaw[0].tobytes() and out["yaw_info"][b].tobytes() == yinfo[0].tobytes()
    finally:
        m.close()
