"""fuelgpu_bspline_parameterize_batch[_dev] on the H100: the control points against exact rational least squares and the
CPU oracle (oracle.param.bspline_parameterize, pinned on the reference's parameterizeToBspline by
tests/test_oracle_traj_param.py), and the constants optimize() freezes, bit for bit given the device's own control
points."""
import ctypes as C

import numpy as np
import pytest

import oracle.param as OP
from fuel_b200 import workloads as W
from tests.helpers import make_sdf_map
from tests.param_cases import GRID_DT, GRID_K, exact_lstsq, noisy_samples, workload_samples

pytestmark = pytest.mark.gpu

LIM = dict(max_vel=2.0, max_acc=2.0)


@pytest.fixture(scope="module")
def free_map(fuel):
    g = W.Grid((80, 60, 30), (-4.0, -3.0, -0.5), 0.1)
    m = make_sdf_map(fuel, g, np.zeros(g.n, np.int8), np.full(g.n, W.FREE, np.uint8))
    yield m
    m.close()


def tc_fields(tc):
    """the fields of a FuelTrajConst array as numpy arrays"""
    B = len(tc)
    return dict(pt_dist=np.array([t.pt_dist for t in tc]), knot_span=np.array([t.knot_span for t in tc]),
                start=np.array([np.array(t.start) for t in tc]).reshape(B, 3, 3),
                end=np.array([np.array(t.end) for t in tc]).reshape(B, 3, 3), n_end=np.array([t.n_end for t in tc]),
                time_lb=np.array([t.time_lb for t in tc]), n_guide=np.array([t.n_guide for t in tc]),
                n_waypt=np.array([t.n_waypt for t in tc]), view_idx=np.array([t.view_idx for t in tc]))


def constants_are_the_oracles(orc, x, tc, n, dt):
    """pt_dist (orc_pt_dist), knot_span, start, end[0] and the dt column equal the oracle's for the device's x"""
    f = tc_fields(tc)
    B = x.shape[0]
    ctrl = x[:, :3 * n].reshape(B, n, 3)
    want_pd = np.array([orc.pt_dist(ctrl[b]) for b in range(B)])
    assert f["pt_dist"].tobytes() == want_pd.tobytes()
    assert f["knot_span"].tobytes() == np.asarray(dt, np.float64).tobytes()
    start, end = OP.bspline_boundary_states(x, n, dt=None if x.shape[1] == 3 * n + 1 else dt)
    assert f["start"].tobytes() == start.tobytes()
    assert f["end"][:, 0].tobytes() == end.tobytes() and not f["end"][:, 1:].any()
    if x.shape[1] == 3 * n + 1:
        assert x[:, 3 * n].tobytes() == np.asarray(dt, np.float64).tobytes()
    assert np.all(f["n_end"] == 1) and np.all(f["n_guide"] == 0) and np.all(f["n_waypt"] == 0)
    assert np.all(f["view_idx"] == -1)


# ---- accuracy ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("K", GRID_K)
def test_solve_matches_exact_least_squares(fuel, orc, free_map, K):
    from fuel_b200.non_uniform_bspline import parameterize_batch
    rng = np.random.default_rng(4000 + K)
    cases = [noisy_samples(rng, K, dt) for dt in GRID_DT for _ in range(2)]
    dts = np.repeat(GRID_DT, 2)
    pts, der = np.array([c[0] for c in cases]), np.array([c[1] for c in cases])
    x, tc = parameterize_batch(free_map, pts, der, dts)
    for b in range(len(cases)):
        A, bb = OP.param_system(pts[b], der[b], dts[b])
        exact = exact_lstsq(A, bb)
        got = x[b, :-1].reshape(K + 2, 3).T
        err = np.abs(got - exact).max()
        assert err <= 1e-11 * max(1.0, np.abs(exact).max()), "K=%d dt=%g: %.3g" % (K, dts[b], err)
    constants_are_the_oracles(orc, x, tc, K + 2, dts)


@pytest.mark.parametrize("which,B,n", [("office", 1024, 20), ("office3", 4096, 64)])
def test_batch_matches_oracle(fuel, orc, free_map, which, B, n):
    from fuel_b200.non_uniform_bspline import parameterize_batch
    g, inflate = (W.office_map if which == "office" else W.office3_map)()
    pts, der, dt = workload_samples(g, inflate, B, n)
    tlb = np.linspace(1.0, 3.0, B)
    x, tc = parameterize_batch(free_map, pts, der, dt, time_lb=tlb)
    want, _ = OP.bspline_parameterize(pts, der, dt)
    scale = np.maximum(1.0, np.abs(want[:, :3 * n]).max(axis=1))
    err = np.abs(x[:, :3 * n] - want[:, :3 * n]).max(axis=1) / scale
    assert err.max() <= 2e-11, "worst row %d: %.3g" % (int(np.argmax(err)), err.max())
    constants_are_the_oracles(orc, x, tc, n, dt)
    assert tc_fields(tc)["time_lb"].tobytes() == tlb.tobytes()
    assert free_map.last_timing()["param"] > 0.0  # the parameterization's device time, slot 6


def test_both_layouts_and_time_lb(fuel, orc, free_map):
    from fuel_b200.non_uniform_bspline import parameterize_batch
    rng = np.random.default_rng(11)
    K, B = 31, 300
    cases = [noisy_samples(rng, K, 0.1) for _ in range(B)]
    pts, der = np.array([c[0] for c in cases]), np.array([c[1] for c in cases])
    dt = rng.uniform(0.02, 2.0, B)
    n = K + 2
    xa, ta = parameterize_batch(free_map, pts, der, dt)
    xb, tb = parameterize_batch(free_map, pts, der, dt, time_lb=7.5, mintime=False)
    assert xa[:, :3 * n].tobytes() == xb.tobytes()
    fa, fb = tc_fields(ta), tc_fields(tb)
    assert np.all(fa["time_lb"] == -1.0) and np.all(fb["time_lb"] == 7.5)
    for k in ("pt_dist", "knot_span", "start", "end"):
        assert fa[k].tobytes() == fb[k].tobytes()
    constants_are_the_oracles(orc, xb, tb, n, dt)


# ---- the device chain -------------------------------------------------------------------------------------------------
def test_dev_chain_equals_host_entries(fuel, orc):
    """parameterize_dev -> optimize_batch_dev -> check_batch_dev on one torch stream, no host sync in between, equals
    the three host entries run in sequence, byte for byte"""
    import torch

    from fuel_b200._lib import FuelSolveParams, FuelTrajCheckParams, FuelTrajConst
    from fuel_b200.non_uniform_bspline import REPORT_DTYPE, check_batch, parameterize_batch
    B, n = 1024, 20
    g, inflate = W.office_map()
    m = make_sdf_map(fuel, g, inflate, W.office_known(g, inflate), optimistic=True)
    st = torch.cuda.Stream()
    m.set_stream(st.cuda_stream)
    m.updateESDF3d()
    env = fuel.EDTEnvironment()
    env.setMap(m)
    opt = fuel.BsplineOptimizer()
    opt.setEnvironment(env)
    mask = opt.NORMAL_PHASE | opt.MINTIME
    pts, der, dt = workload_samples(g, inflate, B, n)
    nvar = 3 * n + 1
    with torch.cuda.stream(st):
        d_pts, d_der, d_dt = (torch.from_numpy(a).cuda() for a in (pts, der, dt))
        d_x = torch.empty((B, nvar), dtype=torch.float64, device="cuda")
        d_tc = torch.empty(B * C.sizeof(FuelTrajConst), dtype=torch.uint8, device="cuda")
        d_f = torch.empty(B, dtype=torch.float64, device="cuda")
        d_n = torch.empty(B, dtype=torch.int32, device="cuda")
        d_rep = torch.empty(B * REPORT_DTYPE.itemsize, dtype=torch.uint8, device="cuda")
        d_best = torch.empty(2, dtype=torch.int32, device="cuda")
    st.synchronize()
    sp = FuelSolveParams()
    sp.max_eval, sp.lbfgs_m, sp.xtol_rel = 64, 6, 1e-5
    cp = FuelTrajCheckParams(LIM["max_vel"], LIM["max_acc"], 0.0)
    L = fuel.lib()
    vp = lambda t: C.c_void_p(t.data_ptr())  # noqa: E731
    assert L.fuelgpu_bspline_parameterize_batch_dev(m.handle, B, n, nvar, vp(d_pts), vp(d_der), vp(d_dt), None, vp(d_x),
                                                    vp(d_tc)) == 0
    x_param = torch.empty_like(d_x)
    with torch.cuda.stream(st):
        x_param.copy_(d_x)
    assert L.fuelgpu_bspline_optimize_batch_dev(m.handle, B, n, mask, C.byref(opt.params_), vp(d_tc), C.byref(sp), vp(d_x),
                                                vp(d_f), vp(d_n)) == 0
    assert L.fuelgpu_bspline_check_batch_dev(m.handle, B, n, nvar, vp(d_x), None, C.byref(cp), vp(d_rep), vp(d_best)) == 0
    st.synchronize()

    x0, tc = parameterize_batch(m, pts, der, dt)
    assert x_param.cpu().numpy().tobytes() == x0.tobytes()
    assert d_tc.cpu().numpy().tobytes() == bytes(tc)
    x, f, ne = opt.optimizeBatch(x0, tc, n, mask, 64)
    rep, best = check_batch(m, x, n, **LIM)
    assert d_x.cpu().numpy().tobytes() == x.tobytes()
    assert d_f.cpu().numpy().tobytes() == f.tobytes() and d_n.cpu().numpy().tobytes() == ne.tobytes()
    assert d_rep.cpu().numpy().tobytes() == rep.tobytes() and np.array_equal(d_best.cpu().numpy(), best)
    assert best[0] >= 0 and best[1] >= 0
    m.close()


# ---- errors -----------------------------------------------------------------------------------------------------------
def test_invalid_arguments(fuel, free_map):
    from fuel_b200._lib import EINVAL, FuelTrajConst, ptr
    L, h = fuel.lib(), free_map.handle
    rng = np.random.default_rng(12)
    B, n = 4, 10
    pts, der = rng.normal(size=(B, n - 2, 3)), rng.normal(size=(B, 4, 3))
    dt = np.full(B, 0.2)

    def call(B_=B, n_=n, nvar=3 * n + 1, dt_=dt):
        x = np.full((max(B, 1), 3 * 65 + 1), 123.0)
        tc = (FuelTrajConst * max(B, 1))()
        ctypes_tc = C.cast(tc, C.c_void_p)
        rc = L.fuelgpu_bspline_parameterize_batch(h, B_, n_, nvar, ptr(pts), ptr(der), ptr(dt_), None, ptr(x), ctypes_tc)
        untouched = np.all(x == 123.0) and bytes(tc) == bytes(C.sizeof(tc))
        return rc, untouched

    for kw in (dict(n_=3, nvar=10), dict(n_=65, nvar=196), dict(nvar=3 * n + 2), dict(nvar=3 * n - 1), dict(B_=-1)):
        rc, untouched = call(**kw)
        assert rc == EINVAL and untouched, kw
    for bad in (0.0, -0.1, np.nan, np.inf, -np.inf):
        d = dt.copy()
        d[2] = bad
        rc, untouched = call(dt_=d)
        assert rc == EINVAL and untouched, bad
    assert call()[0] == 0


def test_dev_bad_dt_gives_nan_on_its_own_row(fuel, free_map):
    import torch

    from fuel_b200._lib import FuelTrajConst
    from fuel_b200.non_uniform_bspline import parameterize_batch
    rng = np.random.default_rng(13)
    B, K = 64, 18
    n = K + 2
    cases = [noisy_samples(rng, K, 0.2) for _ in range(B)]
    pts, der = np.array([c[0] for c in cases]), np.array([c[1] for c in cases])
    dt = rng.uniform(0.1, 0.3, B)
    bad = {3: 0.0, 17: -0.2, 40: np.nan, 41: np.inf}
    dt_bad = dt.copy()
    for b, v in bad.items():
        dt_bad[b] = v
    good = np.array([b for b in range(B) if b not in bad])
    for nvar in (3 * n + 1, 3 * n):
        xw, tw = parameterize_batch(free_map, pts, der, dt, mintime=nvar == 3 * n + 1)
        d_x = torch.zeros((B, nvar), dtype=torch.float64, device="cuda")
        d_tc = torch.zeros(B * C.sizeof(FuelTrajConst), dtype=torch.uint8, device="cuda")
        args = [torch.from_numpy(a).cuda() for a in (pts, der, dt_bad)]
        torch.cuda.synchronize()
        rc = fuel.lib().fuelgpu_bspline_parameterize_batch_dev(free_map.handle, B, n, nvar,
                                                               *[C.c_void_p(a.data_ptr()) for a in args], None,
                                                               C.c_void_p(d_x.data_ptr()), C.c_void_p(d_tc.data_ptr()))
        assert rc == 0
        free_map.synchronize()
        x = d_x.cpu().numpy()
        tc = (FuelTrajConst * B).from_buffer_copy(d_tc.cpu().numpy().tobytes())
        assert x[good].tobytes() == xw[good].tobytes()
        assert b"".join(bytes(tc[b]) for b in good) == b"".join(bytes(tw[b]) for b in good)
        f = tc_fields(tc)
        for b in bad:
            assert np.all(np.isnan(x[b])) and np.isnan(f["pt_dist"][b]) and np.isnan(f["knot_span"][b])
            assert np.all(np.isnan(f["start"][b])) and np.all(np.isnan(f["end"][b, 0]))
            assert f["time_lb"][b] == -1.0 and f["view_idx"][b] == -1


# ---- Python mirror ----------------------------------------------------------------------------------------------------
def test_mirror_b1_equals_batch_row(fuel, free_map):
    from fuel_b200.non_uniform_bspline import NonUniformBspline, parameterize_batch
    rng = np.random.default_rng(14)
    K, B = 30, 16
    cases = [noisy_samples(rng, K, 0.05) for _ in range(B)]
    pts, der = np.array([c[0] for c in cases]), np.array([c[1] for c in cases])
    dt = rng.uniform(0.05, 0.5, B)
    x, _ = parameterize_batch(free_map, pts, der, dt, mintime=False)
    for b in (0, 7, 15):
        ctrl = NonUniformBspline.parameterizeToBspline(dt[b], list(pts[b]), list(der[b]), 3, free_map)
        assert ctrl.shape == (K + 2, 3) and ctrl.tobytes() == x[b].tobytes()
    with pytest.raises(ValueError):
        NonUniformBspline.parameterizeToBspline(dt[0], pts[0], der[0], 4, free_map)
