"""fuelgpu_bspline_check_batch[_dev] / fuelgpu_bspline_evaluate_batch on the H100 against the CPU oracle
(oracle/fuel_oracle_traj.c via oracle.traj, pinned to the reference's NonUniformBspline and checkTrajCollision by
tests/test_oracle_traj.py).  Every comparison is exact equality."""
import ctypes as C

import numpy as np
import pytest

import oracle.traj as OT
from fuel_b200 import workloads as W
from tests.helpers import make_sdf_map, orc_grid

pytestmark = pytest.mark.gpu

LIM = dict(max_vel=2.0, max_acc=2.0)


def knots(n, dt):
    u = np.zeros(n + 4)
    for i in range(n + 4):
        u[i] = float(-3 + i) * dt if i <= 3 else u[i - 1] + dt
    return u


def same_report(got, want):
    """device report (REPORT_DTYPE) == oracle report (TRAJ_REPORT_DTYPE), field by field, bit for bit"""
    for f in ("duration", "jerk", "ratio", "distance"):
        a, b = np.asarray(got[f]), np.asarray(want[f])
        assert a.tobytes() == b.tobytes(), "%s differs at %s" % (f, np.flatnonzero(a.view(np.int64) != b.view(np.int64))[:8])
    for f in ("safe", "feasible", "n_checked"):
        assert np.array_equal(got[f], want[f]), "%s differs at %s" % (f, np.flatnonzero(got[f] != want[f])[:8])


def oracle_check(orc, og, inflate, x, n, dt=None, t_now=0.0, **lim):
    lim = lim or LIM
    return OT.bspline_check(og, inflate.astype(np.int8), x, n, lim["max_vel"], lim["max_acc"], t_now=t_now, dt=dt)


@pytest.fixture(scope="module")
def free_map(fuel, orc):
    """8 x 6 x 3 m at 0.1 m, no obstacle: the adversarial cases place their own"""
    g = W.Grid((80, 60, 30), (-4.0, -3.0, -0.5), 0.1)
    inflate = np.zeros(g.n, np.int8)
    m = make_sdf_map(fuel, g, inflate, np.full(g.n, W.FREE, np.uint8))
    yield dict(g=g, m=m, og=orc_grid(orc, g), inflate=inflate)
    m.close()


def with_inflate(fuel, g, inflate):
    return make_sdf_map(fuel, g, inflate, np.where(inflate == 1, W.OCCUPIED, W.FREE).astype(np.uint8))


def solved_batch(fuel, mk, B, n):
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
    return g, inflate, m, opt, tr, tcs, x


# ---- evaluate -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [4, 20, 31, 32, 33, 48, 64])
def test_evaluate_matches_oracle(fuel, orc, free_map, n):
    from fuel_b200.non_uniform_bspline import evaluate_batch
    rng = np.random.default_rng(n)
    B = 1024
    ctrl = np.cumsum(rng.normal(scale=0.3, size=(B, n, 3)), axis=1)
    dt = rng.uniform(0.05, 1.0, B)
    dt[:8] = 5.0
    x = W.pack_x(ctrl, dt)
    cols = []
    for b in range(B):
        u = knots(n, dt[b])
        dur = u[n] - u[3]
        cols.append(np.concatenate([[0.0, dur, -0.5, dur + 1.0, -1e-300], u[3:n + 1] - u[3], rng.uniform(0, dur, 12)]))
    t = np.stack([c[:n + 14] if len(c) >= n + 14 else np.pad(c, (0, n + 14 - len(c)), constant_values=0.1) for c in cols])
    for deriv in range(3):
        got = evaluate_batch(free_map["m"], x, n, t, deriv)
        want = OT.bspline_evaluate(x, n, t, deriv)
        assert got.tobytes() == want.tobytes(), "n=%d deriv=%d: %d values differ" % (n, deriv, int(np.sum(got != want)))
    got = evaluate_batch(free_map["m"], W.pack_x(ctrl, dt, mintime=False), n, t, 1, dt=dt)
    assert got.tobytes() == OT.bspline_evaluate(x, n, t, 1).tobytes()


# ---- check on the solver's output ---------------------------------------------------------------------------------
@pytest.mark.parametrize("which,B,n", [("office", 1024, 20), ("office3", 4096, 64)])
def test_check_after_solver_matches_oracle(fuel, orc, which, B, n):
    from fuel_b200.non_uniform_bspline import check_batch
    mk = W.office_map if which == "office" else W.office3_map
    g, inflate, m, _, _, _, x = solved_batch(fuel, mk, B, n)
    og = orc_grid(orc, g)
    for t_now in (0.0, 0.3):
        rep, best = check_batch(m, x, n, t_now=t_now, **LIM)
        want, wbest = oracle_check(orc, og, inflate, x, n, t_now=t_now)
        same_report(rep, want)
        assert np.array_equal(best, wbest)
        if t_now == 0.0:
            assert 0 < (rep["safe"] == 0).sum() < B, "every branch: some unsafe, some safe"
            assert 0 < (rep["feasible"] == 0).sum() < B, "every branch: some infeasible, some feasible"
            assert best[1] >= 0 and rep["safe"][best[1]] and rep["feasible"][best[1]]
    assert m.last_timing()["check"] > 0.0  # the check's device time, slot 5
    m.close()


# ---- adversarial input --------------------------------------------------------------------------------------------
def line(p0, p1, n):
    s = np.linspace(0.0, 1.0, n)[:, None]
    return p0[None, :] * (1 - s) + p1[None, :] * s


def test_first_sample_hit_gives_distance_zero(fuel, orc, free_map):
    g, og = free_map["g"], free_map["og"]
    n, dt = 10, 0.2
    ctrl = line(np.array([-2.0, 0.05, 1.0]), np.array([2.0, 0.05, 1.0]), n)[None]
    x = W.pack_x(ctrl, np.array([dt]))
    p1 = OT.bspline_evaluate(x, n, np.array([[0.02]]))[0, 0]
    inflate = np.zeros(g.n, np.int8)
    i = g.pos_to_index(p1)
    inflate[i[0], i[1], i[2]] = 1
    m = with_inflate(fuel, g, inflate)
    from fuel_b200.non_uniform_bspline import check_batch
    rep, _ = check_batch(m, x, n, **LIM)
    want, _ = oracle_check(orc, og, inflate, x, n)
    same_report(rep, want)
    assert rep["safe"][0] == 0 and rep["distance"][0] == 0.0 and rep["n_checked"][0] == 1
    m.close()


def test_scan_stops_at_six_metres(fuel, orc, free_map):
    """straight 7.6 m paths along x: the loop ends on the radius, the wall beyond 6 m is never sampled"""
    g, og = free_map["g"], free_map["og"]
    n, B = 24, 64
    rng = np.random.default_rng(3)
    off = rng.uniform(-0.3, 0.3, (B, 2))
    ctrl = np.stack([line(np.array([-3.8, off[b, 0], 1.0 + off[b, 1]]), np.array([3.8, off[b, 0], 1.0 + off[b, 1]]), n)
                     for b in range(B)])
    dt = rng.uniform(0.1, 0.3, B)
    x = W.pack_x(ctrl, dt)
    inflate = np.zeros(g.n, np.int8)
    inflate[70:, :, :] = 1  # x >= 3.0 m, past 6 m from every start (x ~ -3.47)
    m = with_inflate(fuel, g, inflate)
    from fuel_b200.non_uniform_bspline import check_batch
    rep, _ = check_batch(m, x, n, **LIM)
    want, _ = oracle_check(orc, og, inflate, x, n)
    same_report(rep, want)
    assert np.all(rep["safe"] == 1)
    for b in range(B):  # the last sample is the first at or beyond 6 m
        ft = 0.0
        for _ in range(int(rep["n_checked"][b])):
            ft += 0.02
        p0, p1 = OT.bspline_evaluate(x[b:b + 1], n, np.array([[0.0, ft]]))[0]
        d = p1 - p0
        assert np.sqrt(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]) >= 6.0
    m.close()


def test_paths_leaving_the_map_are_not_hits(fuel, orc, free_map):
    g, og = free_map["g"], free_map["og"]
    n, B = 16, 32
    rng = np.random.default_rng(4)
    ctrl = np.stack([line(np.array([3.0, 0.0, 1.0]), np.array([3.0, 0.0, 1.0]) + rng.normal(size=3) * 4.0, n)
                     for _ in range(B)])
    x = W.pack_x(ctrl, rng.uniform(0.05, 0.3, B))
    inflate = np.zeros(g.n, np.int8)
    inflate[:, :, 0] = 1  # the floor: paths leave through the other faces
    m = with_inflate(fuel, g, inflate)
    from fuel_b200.non_uniform_bspline import check_batch
    rep, _ = check_batch(m, x, n, **LIM)
    want, _ = oracle_check(orc, og, inflate, x, n)
    same_report(rep, want)
    out = OT.bspline_evaluate(x, n, np.full((B, 1), 1e9))[:, 0]
    assert np.any(np.any(out > np.array(g.map_max), axis=1) & (rep["safe"] == 1))
    m.close()


def test_t_now_inside_and_past_the_end(fuel, orc, free_map):
    g, og = free_map["g"], free_map["og"]
    n, B = 20, 256
    rng = np.random.default_rng(5)
    ctrl = np.cumsum(rng.normal(scale=0.2, size=(B, n, 3)), axis=1) + np.array([0.0, 0.0, 1.0])
    dt = rng.uniform(0.05, 0.3, B)
    x = W.pack_x(ctrl, dt)
    inflate = (rng.random(g.n) < 0.01).astype(np.int8)
    m = with_inflate(fuel, g, inflate)
    from fuel_b200.non_uniform_bspline import check_batch
    dur = np.array([knots(n, d)[n] - knots(n, d)[3] for d in dt])
    for t_now in (0.01, 0.7, float(dur.min()), float(dur.max()), float(dur.max()) + 3.0):
        rep, best = check_batch(m, x, n, t_now=t_now, **LIM)
        want, wbest = oracle_check(orc, og, inflate, x, n, t_now=t_now)
        same_report(rep, want)
        assert np.array_equal(best, wbest)
    assert np.all(rep["n_checked"] == 0) and np.all(rep["safe"] == 1)  # t_now >= duration: no sample
    m.close()


def test_longest_scan_dt5_n64(fuel, orc, free_map):
    g, og, m = free_map["g"], free_map["og"], free_map["m"]
    n, B = 64, 64
    rng = np.random.default_rng(6)
    ctrl = np.array([0.0, 0.0, 1.0]) + np.cumsum(rng.normal(scale=0.02, size=(B, n, 3)), axis=1)
    x = W.pack_x(ctrl, np.full(B, 5.0))
    from fuel_b200.non_uniform_bspline import check_batch
    rep, _ = check_batch(m, x, n, **LIM)
    want, _ = oracle_check(orc, og, free_map["inflate"], x, n)
    same_report(rep, want)
    assert rep["n_checked"].max() > 15000


def test_dt_column_and_dt_array_give_identical_reports(fuel, orc, free_map):
    g, og = free_map["g"], free_map["og"]
    n, B = 33, 512
    rng = np.random.default_rng(7)
    ctrl = np.cumsum(rng.normal(scale=0.25, size=(B, n, 3)), axis=1) + np.array([0.0, 0.0, 1.0])
    dt = rng.uniform(0.05, 0.5, B)
    inflate = (rng.random(g.n) < 0.01).astype(np.int8)
    m = with_inflate(fuel, g, inflate)
    from fuel_b200.non_uniform_bspline import check_batch
    a, ba = check_batch(m, W.pack_x(ctrl, dt), n, **LIM)
    b, bb = check_batch(m, W.pack_x(ctrl, dt, mintime=False), n, dt=dt, **LIM)
    assert a.tobytes() == b.tobytes() and np.array_equal(ba, bb)
    want, _ = oracle_check(orc, og, inflate, W.pack_x(ctrl, dt), n)
    same_report(a, want)
    m.close()


# ---- best ---------------------------------------------------------------------------------------------------------
def test_best_is_the_lowest_index_of_least_jerk(fuel, orc, free_map):
    from fuel_b200.non_uniform_bspline import check_batch
    m = free_map["m"]
    n, B0 = 12, 300
    rng = np.random.default_rng(8)
    ctrl = np.cumsum(rng.normal(scale=0.2, size=(B0, n, 3)), axis=1) + np.array([0.0, 0.0, 1.0])
    x0 = W.pack_x(ctrl, rng.uniform(0.1, 0.4, B0))
    rep0, _ = check_batch(m, x0, n, **LIM)
    k = int(np.argmin(rep0["jerk"]))
    order = rng.permutation(B0)
    x = np.concatenate([x0[order], x0[[k, k, k]], x0[order[:40]]])  # the least-jerk row appears 4 times
    x[6 if order[5] == k else 5, 0] = np.nan  # a NaN jerk never wins
    rep, best = check_batch(m, x, n, **LIM)
    j = rep["jerk"]
    want0 = int(np.flatnonzero(j == np.nanmin(j))[0])
    assert best[0] == want0 == int(np.flatnonzero(order == k)[0])
    valid = (rep["safe"] == 1) & (rep["feasible"] == 1) & ~np.isnan(j)
    jv = np.where(valid, j, np.inf)
    assert best[1] == (int(np.argmin(jv)) if valid.any() else -1)
    _, wbest = oracle_check(orc, free_map["og"], free_map["inflate"], x, n)
    assert np.array_equal(best, wbest)
    _, none = check_batch(m, x, n, max_vel=1e-6, max_acc=1e-6)
    assert none[1] == -1 and none[0] == best[0]


# ---- host vs device entry -----------------------------------------------------------------------------------------
def test_dev_entry_behind_the_solver_equals_host_entry(fuel, orc):
    import torch

    from fuel_b200._lib import FuelSolveParams, FuelTrajCheckParams
    from fuel_b200.non_uniform_bspline import REPORT_DTYPE, check_batch
    B, n = 1024, 20
    g, inflate = W.office_map()
    tri = W.office_known(g, inflate)
    m = make_sdf_map(fuel, g, inflate, tri, optimistic=True)
    st = torch.cuda.Stream()
    m.set_stream(st.cuda_stream)
    m.updateESDF3d()
    env = fuel.EDTEnvironment()
    env.setMap(m)
    opt = fuel.BsplineOptimizer()
    opt.setEnvironment(env)
    tr = W.make_trajectories(g, inflate, B=B, n_pts=n)
    tcs = opt.traj_consts_from_arrays(tr["pt_dist"], tr["dt"], tr["start"], tr["end_pos"])
    with torch.cuda.stream(st):
        d_tc = torch.from_numpy(np.frombuffer(tcs, dtype=np.uint8).copy()).cuda()
        d_x = torch.from_numpy(W.pack_x(tr["ctrl"], tr["dt"])).cuda()
        d_f = torch.empty(B, dtype=torch.float64, device="cuda")
        d_n = torch.empty(B, dtype=torch.int32, device="cuda")
        d_rep = torch.empty(B * REPORT_DTYPE.itemsize, dtype=torch.uint8, device="cuda")
        d_best = torch.empty(2, dtype=torch.int32, device="cuda")
    st.synchronize()
    sp = FuelSolveParams()
    sp.max_eval, sp.lbfgs_m, sp.xtol_rel = 64, 6, 1e-5
    L = fuel.lib()
    rc = L.fuelgpu_bspline_optimize_batch_dev(m.handle, B, n, opt.NORMAL_PHASE | opt.MINTIME, C.byref(opt.params_),
                                              C.c_void_p(d_tc.data_ptr()), C.byref(sp), C.c_void_p(d_x.data_ptr()),
                                              C.c_void_p(d_f.data_ptr()), C.c_void_p(d_n.data_ptr()))
    assert rc == 0
    p = FuelTrajCheckParams(LIM["max_vel"], LIM["max_acc"], 0.0)
    rc = L.fuelgpu_bspline_check_batch_dev(m.handle, B, n, 3 * n + 1, C.c_void_p(d_x.data_ptr()), None, C.byref(p),
                                           C.c_void_p(d_rep.data_ptr()), C.c_void_p(d_best.data_ptr()))
    assert rc == 0
    st.synchronize()
    rep_dev = d_rep.cpu().numpy().view(REPORT_DTYPE)
    x = d_x.cpu().numpy()
    rep, best = check_batch(m, x, n, **LIM)
    assert rep_dev.tobytes() == rep.tobytes() and np.array_equal(d_best.cpu().numpy(), best)
    want, wbest = oracle_check(orc, orc_grid(orc, g), inflate, x, n)
    same_report(rep, want)
    assert np.array_equal(best, wbest)
    m.close()


# ---- Python mirror ------------------------------------------------------------------------------------------------
def test_mirror_methods_equal_the_batch(fuel, orc):
    from fuel_b200.non_uniform_bspline import NonUniformBspline, check_batch, checkTrajCollision, evaluate_batch, selectBestTraj
    n, B = 20, 64
    g, inflate, m, _, _, _, x = solved_batch(fuel, W.office_map, B, n)
    rep, best = check_batch(m, x, n, t_now=0.1, **LIM)
    trajs = []
    for b in range(8):
        tj = NonUniformBspline(x[b, :3 * n].reshape(n, 3), 3, x[b, 3 * n], m)
        tj.setPhysicalLimits(LIM["max_vel"], LIM["max_acc"])
        assert tj.getTimeSum() == rep["duration"][b] and tj.getJerk() == rep["jerk"][b]
        assert tj.checkRatio() == rep["ratio"][b] and tj.checkFeasibility() == bool(rep["feasible"][b])
        safe, dist = checkTrajCollision(m, tj, 0.1)
        assert safe == bool(rep["safe"][b]) and dist == rep["distance"][b]
        for t in (0.0, 0.37, rep["duration"][b]):
            for d, s in enumerate((tj, tj.getDerivative(), tj.getDerivative().getDerivative())):
                assert np.array_equal(s.evaluateDeBoorT(t), evaluate_batch(m, x[b:b + 1], n, [[t]], d)[0, 0])
        trajs.append(tj)
    pick = selectBestTraj(m, trajs)
    assert pick is trajs[int(np.argmin(rep["jerk"][:8]))]
    m.close()
