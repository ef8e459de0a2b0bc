"""fuelgpu_plan_yaw_batch[_dev] (planYaw, the kinodynamic replan's yaw) on the H100: seg_num, dt_yaw and the waypoint
count against the CPU oracle (oracle.plan_yaw, pinned on the reference's lines by tests/test_oracle_plan_yaw.py) bit
for bit, the waypoints to atan2's rounding, pt_dist_ bit for bit given them, the control points against the exact
rational minimizer of the objective built from the device's own waypoints, optimality under the oracle's combineCost,
every status, the error paths, the chain behind the solver, and kino_replan_traj_batch."""
import ctypes as C

import numpy as np
import pytest

import oracle.plan_yaw as OPY
from fuel_b200 import workloads as W
from fuel_b200._lib import FuelOptParams, FuelSolveParams
from fuel_b200.kino_astar import TRAJ_OK, kino_replan_traj_batch, kinodynamic_replan_batch
from fuel_b200.polynomial_traj import (PLANYAW_INFO_DTYPE, PLANYAW_MAX_PTS, PLANYAW_MAX_SEG, YAW_BAD_INPUT,
                                       YAW_NO_LOOKAHEAD, YAW_NOT_SPD, YAW_TOO_LONG, YAW_ZERO_PT_DIST, plan_yaw_batch)
from tests.helpers import make_sdf_map
from tests.kino_cases import mid_queries
from tests.plan_yaw_cases import DURATIONS, LD_KINO, duration_batch, exact_minimizer, hover_tail, solve_bar
from tests.yaw_cases import arc_batch

pytestmark = pytest.mark.gpu


def opt_params(**kw):
    p = FuelOptParams()
    for k, v in dict(LD_KINO, **kw).items():
        setattr(p, k, v)
    p.order = 3
    return p


@pytest.fixture(scope="module")
def free_map(fuel):
    g = W.Grid((40, 40, 20), (-2.0, -2.0, -0.5), 0.1)
    m = make_sdf_map(fuel, g, np.zeros(g.n, np.int8), np.full(g.n, W.FREE, np.uint8))
    yield m
    m.close()


def end_candidates(r):
    """the C library's atan2 of the end velocity and its neighbours within 2 ulp (the device's atan2 may round there)"""
    a = r["end_in"]
    out = [a]
    for d in (np.inf, -np.inf):
        v = a
        for _ in range(2):
            v = float(np.nextafter(v, d))
            out.append(v)
    return out


def check_against_oracle(rows, yaw, info, waypt, n_exact=None):
    """seg_num, dt_yaw and n_waypt bit for bit; waypoints to 1e-13; pt_dist bit for bit given the device's waypoints
    (and an end atan2 within 2 ulp of the C library's); NaN past seg_num + 3; the control points within solve_bar of the
    exact minimizer of the objective built from the device's waypoints (on n_exact rows spread over the batch, all if
    None); gradient under the oracle's combineCost <= 1e-9 of the initial guess's, cost <= the exact minimizer's"""
    dr = []
    for b, r in enumerate(rows):
        assert info["status"][b] == r["status"] == 0, (b, info["status"][b], r["status"])
        assert info["seg_num"][b] == r["seg_num"] and info["dt_yaw"][b] == r["dt_yaw"], b
        assert info["n_waypt"][b] == len(r["waypts"]) == r["seg_num"], b
        assert np.all(waypt[b, r["seg_num"]:] == 0) and np.all(np.isnan(yaw[b, r["n_pts"]:]))
        w = np.array(r["waypts"])
        if r["margin"] >= 1e-12:
            assert np.all(np.abs(waypt[b, :len(w)] - w) <= 1e-13 * np.maximum(1.0, np.abs(w))), b
        d = [OPY.with_waypoints(r, waypt[b, :len(w)], end_in=e) for e in end_candidates(r)]
        d = [c for c in d if c["pt_dist"] == info["pt_dist"][b]]
        assert d, (b, info["pt_dist"][b], r["pt_dist"])
        dr.append(d[0])
    sel = range(len(dr)) if n_exact is None else np.unique(np.linspace(0, len(dr) - 1, n_exact).astype(int))
    for b in sel:
        r = dr[b]
        ex = np.array([float(v) for v in exact_minimizer(r, **LD_KINO)])
        err = np.abs(yaw[b, :r["n_pts"]] - ex).max()
        assert err <= solve_bar(r, **LD_KINO) * max(1.0, np.abs(ex).max()), (b, r["seg_num"], err)
        fx, _ = OPY.objective([r], [ex], **LD_KINO)
        f, _ = OPY.objective([r], [yaw[b]], **LD_KINO)
        assert f[0] <= fx[0] * (1 + 1e-12), b
    _, g = OPY.objective(dr, yaw, **LD_KINO)
    _, g0 = OPY.objective(dr, [r["guess"] for r in dr], **LD_KINO)
    for b, (a, a0) in enumerate(zip(g, g0)):
        assert np.abs(a).max() <= 1e-9 * np.abs(a0).max(), b


@pytest.mark.parametrize("layout", ["mintime", "dt"])
@pytest.mark.parametrize("n", [20, 64])
def test_seg_nums_match_oracle(free_map, n, layout):
    """seg_num 1, 2, 3, 4, 20, 127 and 128, a duration below 0.1 s, start yaws up to +-1000; the row past the cap is
    TOO_LONG"""
    x = duration_batch(list(DURATIONS) * 3, n_pts=n, seed=40 + n)
    B = len(x)
    ys = W.make_yaws(B, seed=41)
    sy = ys["start"].copy()
    sy[0, 0], sy[1, 0] = 1000.0, -1000.0
    xin, dt = (np.ascontiguousarray(x[:, :3 * n]), x[:, 3 * n].copy()) if layout == "dt" else (x, None)
    yaw, info, waypt = plan_yaw_batch(free_map, xin, n, sy, opt_params(), dt=dt)
    rows = OPY.plan_yaw(xin, n, sy, dt=dt)
    long_ = [b for b, r in enumerate(rows) if r["status"] == OPY.TOO_LONG]
    assert len(long_) == 3 and np.all(info["status"][long_] == YAW_TOO_LONG)
    assert np.all(np.isnan(yaw[long_])) and np.all(np.isnan(waypt[long_])) and np.all(info["seg_num"][long_] == 0)
    ok = [b for b in range(B) if b not in long_]
    assert {1, 2, 3, 4, 20, 127, 128} <= set(info["seg_num"][ok].tolist())
    check_against_oracle([rows[b] for b in ok], yaw[ok], info[ok], waypt[ok])


def test_statuses_on_hand_made_rows(free_map):
    """a stationary tail, a stationary start (NO_LOOKAHEAD), zero yaws along +x (ZERO_PT_DIST), a trajectory past the
    cap (TOO_LONG), an indefinite objective (a negative ld_end: NOT_SPD); each row as planned alone"""
    n = 40
    x = duration_batch([8.0, 8.0, 1.0, 40.0, 3.0], n_pts=n, seed=43)
    x[0] = hover_tail(x[:1], n, k=8)[0]
    c = x[:, :3 * n].reshape(len(x), n, 3)
    c[1, :20] = c[1, 20]
    c[2] = np.stack([np.linspace(0.0, 2.0, n), np.zeros(n), np.ones(n)], 1)
    x[:, :3 * n] = c.reshape(len(x), -1)
    sy = np.array([[0.4, 0.2, 0.0], [0.1, 0.0, 0.0], [0.0, 0.0, 0.0], [0.2, 0.0, 0.0], [-0.3, 0.1, 0.0]])
    p = opt_params()
    yaw, info, waypt = plan_yaw_batch(free_map, x, n, sy, p)
    assert info["status"].tolist() == [0, YAW_NO_LOOKAHEAD, YAW_ZERO_PT_DIST, YAW_TOO_LONG, 0]
    rows = OPY.plan_yaw(x, n, sy)
    assert [r["status"] for r in rows] == info["status"].tolist()
    assert rows[0]["end_v"] == [0.0, 0.0, 0.0]
    check_against_oracle([rows[0], rows[4]], yaw[[0, 4]], info[[0, 4]], waypt[[0, 4]])
    assert np.isfinite(info["dt_yaw"][1]) and info["seg_num"][1] == rows[1]["seg_num"] and info["n_waypt"][1] == 0
    assert np.isnan(info["pt_dist"][1]) and np.all(np.isnan(waypt[1])) and np.all(np.isnan(yaw[1]))
    assert info["pt_dist"][2] == 0.0 and info["n_waypt"][2] == rows[2]["seg_num"] and np.all(np.isnan(yaw[2]))
    assert np.all(waypt[2, :rows[2]["seg_num"]] == 0.0)
    assert np.isnan(info["dt_yaw"][3]) and info["seg_num"][3] == 0 and np.all(np.isnan(waypt[3]))
    for b in range(len(x)):
        ya, ia, wa = plan_yaw_batch(free_map, x[b:b + 1], n, sy[b:b + 1], p)
        assert ya[0].tobytes() == yaw[b].tobytes() and ia[0].tobytes() == info[b].tobytes()
        assert wa[0].tobytes() == waypt[b].tobytes()
    yaw, info, waypt = plan_yaw_batch(free_map, x[[0, 4]], n, sy[[0, 4]], opt_params(ld_end=-1e6))
    assert info["status"].tolist() == [YAW_NOT_SPD] * 2
    assert np.all(np.isnan(yaw)) and np.all(np.isfinite(info["pt_dist"])) and np.all(info["n_waypt"] > 0)


def test_host_entry_refuses_and_writes_nothing(free_map, fuel):
    L = fuel.lib()
    h = free_map.handle
    x = arc_batch([0.1, 0.2])
    sy = np.zeros((2, 3)) + 0.5
    good = opt_params()

    def call(x=x, n=20, nvar=61, dt=None, sy=sy, p=good, B=2):
        yaw, wp = np.full((2, PLANYAW_MAX_PTS), 7.0), np.full((2, PLANYAW_MAX_SEG), 7.0)
        info = np.zeros(2, dtype=PLANYAW_INFO_DTYPE)
        info["status"] = 7
        rc = L.fuelgpu_plan_yaw_batch(h, B, n, nvar, x.ctypes.data, None if dt is None else dt.ctypes.data,
                                      sy.ctypes.data, C.byref(p), yaw.ctypes.data, info.ctypes.data, wp.ctypes.data)
        return rc, yaw, info, wp

    assert call()[0] == 0
    bad_dt, inf_dt = x.copy(), x.copy()
    bad_dt[1, 60] = 0.0
    inf_dt[0, 60] = np.inf
    cases = [dict(n=3, nvar=10), dict(nvar=62), dict(B=-1), dict(x=bad_dt), dict(x=inf_dt),
             dict(nvar=60, dt=np.array([0.1, np.nan])), dict(sy=np.array([[np.nan, 0, 0], [0, 0, 0.0]])),
             dict(sy=np.array([[0, 0, 0], [1000.5, 0, 0.0]])), dict(sy=np.array([[0, np.inf, 0], [0, 0, 0.0]])),
             dict(sy=np.array([[0, 0, -np.inf], [0, 0, 0.0]])), dict(p=opt_params(ld_smooth=0.0)),
             dict(p=opt_params(ld_start=-1.0)), dict(p=opt_params(ld_smooth=np.nan))]
    for kw in cases:
        if kw.get("nvar") == 60 and "x" not in kw:
            kw["x"] = np.ascontiguousarray(x[:, :60])
        rc, yaw, info, wp = call(**kw)
        assert rc == -1, kw
        assert np.all(yaw == 7.0) and np.all(wp == 7.0) and np.all(info["status"] == 7), kw
    rc, yaw, info, wp = call(sy=np.array([[1000.0, 0, 0], [-1000.0, 0, 0]]))
    assert rc == 0 and np.all(info["status"] == 0)


def _dev_call(fuel, m, x, n, dt, sy, p):
    import torch
    t = lambda a: None if a is None else torch.from_numpy(np.ascontiguousarray(a)).cuda()  # noqa: E731
    B = len(x)
    d_x, d_dt, d_sy = t(x), t(dt), t(sy)
    d_yaw = torch.empty((B, PLANYAW_MAX_PTS), dtype=torch.float64, device="cuda")
    d_info = torch.empty(B * PLANYAW_INFO_DTYPE.itemsize, dtype=torch.uint8, device="cuda")
    d_wp = torch.empty((B, PLANYAW_MAX_SEG), dtype=torch.float64, device="cuda")
    torch.cuda.synchronize()
    rc = fuel.lib().fuelgpu_plan_yaw_batch_dev(m.handle, B, n, x.shape[1], d_x.data_ptr(),
                                               None if d_dt is None else d_dt.data_ptr(), d_sy.data_ptr(), C.byref(p),
                                               d_yaw.data_ptr(), d_info.data_ptr(), d_wp.data_ptr())
    assert rc == 0
    m.synchronize()
    return (d_yaw.cpu().numpy(), np.frombuffer(d_info.cpu().numpy().tobytes(), dtype=PLANYAW_INFO_DTYPE),
            d_wp.cpu().numpy())


def test_dev_entry_equals_host_and_marks_bad_rows(free_map, fuel):
    x = duration_batch(list(DURATIONS) * 3, seed=44)
    B = len(x)
    sy = W.make_yaws(B, seed=45)["start"]
    p = opt_params()
    host = plan_yaw_batch(free_map, x, 20, sy, p)
    dev = _dev_call(fuel, free_map, x, 20, None, sy, p)
    for a, b in zip(host, dev):
        assert a.tobytes() == b.tobytes()
    xb, syb = x.copy(), sy.copy()
    bad = [1, 6, 11, 17, 23]
    xb[1, 60] = -0.1
    syb[6, 0] = np.nan
    syb[11, 0] = 2000.0
    syb[17, 2] = np.inf
    xb[23, 60] = np.inf
    yaw, info, wp = _dev_call(fuel, free_map, xb, 20, None, syb, p)
    for b in range(B):
        if b in bad:
            assert info["status"][b] == YAW_BAD_INPUT and info["n_waypt"][b] == 0 and info["seg_num"][b] == 0
            assert np.isnan(info["dt_yaw"][b]) and np.isnan(info["pt_dist"][b])
            assert np.all(np.isnan(yaw[b])) and np.all(np.isnan(wp[b]))
        else:
            assert yaw[b].tobytes() == host[0][b].tobytes() and info[b].tobytes() == host[1][b].tobytes()
            assert wp[b].tobytes() == host[2][b].tobytes()


def test_wide_batch_every_point_count(free_map):
    """B = 4096 over every point count 4..64 (one launch each) and dt from 0.01 to 0.6 s, a few rows up to 0.7 s: seg_num
    from 1 to 128 and TOO_LONG"""
    rng = np.random.default_rng(46)
    ns = np.arange(4, 65)
    per = np.full(len(ns), 4096 // len(ns))
    per[:4096 - per.sum()] += 1
    segs, n_long = set(), 0
    for n, k in zip(ns, per):
        dts = rng.uniform(0.01, 0.6, k)
        dts[:2] = rng.uniform(0.6, 0.7, 2)
        x = arc_batch(list(dts * (n - 3) / 12.0), n_pts=int(n), seed=int(n))
        sy = W.make_yaws(int(k), seed=int(n))["start"]
        yaw, info, waypt = plan_yaw_batch(free_map, x, int(n), sy, opt_params())
        rows = OPY.plan_yaw(x, int(n), sy)
        assert [r["status"] for r in rows] == info["status"].tolist(), n
        ok = np.flatnonzero(info["status"] == 0)
        n_long += int(np.count_nonzero(info["status"] == YAW_TOO_LONG))
        segs |= set(info["seg_num"][ok].tolist())
        check_against_oracle([rows[b] for b in ok], yaw[ok], info[ok], waypt[ok], n_exact=1 if n % 4 == 0 else 0)
    assert n_long > 0 and {1, 128} <= segs and len(segs) > 100


def test_optimize_dev_then_plan_yaw_dev_without_sync(fuel):
    """kinodynamic replans on office: optimize_batch_dev -> plan_yaw_batch_dev on the map's main stream (a torch
    stream) with no host sync between, equal to the host entries; kino_replan_traj_batch gives every row with samples
    status 0 and the yaw of plan_yaw_batch run on that row's solver output alone"""
    import torch
    g, inflate = W.office_map()
    tri = W.office_known(g, inflate)
    m = make_sdf_map(fuel, g, inflate, tri)
    st = torch.cuda.Stream()
    m.set_stream(st.cuda_stream)
    try:
        m.updateESDF3d()
        env = fuel.EDTEnvironment()
        env.setMap(m)
        opt = fuel.BsplineOptimizer()
        opt.setParam(ld_feasi=1.0, ld_time=0.1, dist0=0.4, **LD_KINO)  # kino_algorithm.xml:128-139
        opt.setEnvironment(env)
        mask = opt.NORMAL_PHASE | opt.MINTIME
        q = mid_queries(g, inflate, tri, B=256, seed=47)
        B = len(q["start"])
        sy = W.make_yaws(B, seed=48)["start"]
        res, groups = kinodynamic_replan_batch(m, q["start"], q["vel"], q["acc"], q["goal"])
        assert len(groups) > 1
        sp = FuelSolveParams()
        sp.max_eval, sp.lbfgs_m, sp.xtol_rel = 64, 6, 1e-5
        L = fuel.lib()
        for rows, x0, tc in groups:
            n = (x0.shape[1] - 1) // 3
            k = len(rows)
            with torch.cuda.stream(st):
                cu = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()  # noqa: E731
                d_x, d_sy = cu(x0), cu(sy[rows])
                d_tc = cu(np.frombuffer(tc, dtype=np.uint8).copy())
                d_f = torch.empty(k, dtype=torch.float64, device="cuda")
                d_ne = torch.empty(k, dtype=torch.int32, device="cuda")
                d_yaw = torch.empty((k, PLANYAW_MAX_PTS), dtype=torch.float64, device="cuda")
                d_yi = torch.empty(k * PLANYAW_INFO_DTYPE.itemsize, dtype=torch.uint8, device="cuda")
                d_wp = torch.empty((k, PLANYAW_MAX_SEG), dtype=torch.float64, device="cuda")
            st.synchronize()
            assert L.fuelgpu_bspline_optimize_batch_dev(m.handle, k, n, mask, C.byref(opt.params_), d_tc.data_ptr(),
                                                        C.byref(sp), d_x.data_ptr(), d_f.data_ptr(), d_ne.data_ptr()) == 0
            assert L.fuelgpu_plan_yaw_batch_dev(m.handle, k, n, 3 * n + 1, d_x.data_ptr(), None, d_sy.data_ptr(),
                                                C.byref(opt.params_), d_yaw.data_ptr(), d_yi.data_ptr(),
                                                d_wp.data_ptr()) == 0
            st.synchronize()
            x, _, _ = opt.optimizeBatch(x0, tc, n, mask, 64)
            yaw, yinfo, wp = plan_yaw_batch(m, x, n, sy[rows], opt)
            assert d_x.cpu().numpy().tobytes() == x.tobytes()
            assert d_yaw.cpu().numpy().tobytes() == yaw.tobytes() and d_yi.cpu().numpy().tobytes() == yinfo.tobytes()
            assert d_wp.cpu().numpy().tobytes() == wp.tobytes()
        for cost in (mask, opt.NORMAL_PHASE):
            out = kino_replan_traj_batch(m, q["start"], q["vel"], q["acc"], q["goal"], opt,
                                         dict(cost_function=cost, max_eval=64), sy)
            has = out["res"]["info"]["traj_status"] == TRAJ_OK
            assert np.count_nonzero(has) == sum(len(r) for r, _, _ in groups)
            for b in range(B):
                if not has[b]:
                    assert out["x"][b] is None and out["yaw_info"]["status"][b] == -1 and np.all(np.isnan(out["yaw"][b]))
                    continue
                n = int(out["res"]["info"]["n_pts"][b])
                assert out["yaw_info"]["status"][b] == 0, b
                dt = None if cost & opt.MINTIME else out["res"]["dt"][b:b + 1]
                yaw, yinfo, _ = plan_yaw_batch(m, out["x"][b][None], n, sy[b], opt, dt=dt)
                assert out["yaw"][b].tobytes() == yaw[0].tobytes() and out["yaw_info"][b].tobytes() == yinfo[0].tobytes()
    finally:
        m.close()
