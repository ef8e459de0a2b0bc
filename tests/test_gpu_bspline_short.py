"""The short-trajectory solver: fuelgpu_bspline_optimize_batch with n_pts + dt <= 32 lanes (bspline_solve.cu:
optimize_gram_kernel<6> for lbfgs_m == 6, optimize_warp_kernel for every other history length), one control point per
lane, at every point count it takes.

The solver gates of test_gpu_bspline.py compare against another L-BFGS (the CPU twin) in percent-level bands on a
non-convex objective; a wrong direction, Gram entry or projection still goes downhill and passes them.  Here dt is
fixed (no MINTIME) and the objective is built from terms that are sums of squares of affine functions of the control
points (SMOOTHNESS, START, END, GUIDE, WAYPOINTS), so combineCost is a quadratic 1/2 x'Hx + b'x + c.  H and b are read
off the oracle's own gradient (which is pinned to the reference), the box of optimize() (:196-217) is rebuilt, and
the box-constrained minimizer x* is solved in fp64 (BVLS on the Cholesky factor, KKT-checked).  The device solver must
converge to x*, not merely descend.
"""
import ctypes as C

import numpy as np
import pytest
import scipy.linalg as sla
from scipy.optimize import lsq_linear

from fuel_b200 import workloads as W
from tests.helpers import make_sdf_map, orc_grid
from tests.test_gpu_bspline import check, gpu_consts, orc_consts

SHORT_N = list(range(7, 33))  # every point count of the short solver without MINTIME (the API takes n_pts > 2 * order)
LONG_N = [33, 40, 64]         # the long solver (bspline_solve_long.cu), as a boundary control
LBFGS_M = [1, 2, 4, 6, 8]     # 6: optimize_gram_kernel<6>; the others: optimize_warp_kernel
B_QP = 37                     # not a multiple of the 4 trajectories (warps) per CTA
MAX_EVAL = 2000
KAPPA_MAX = 1e5
KINDS = ("guide", "end3", "waypt")
DT_QP = 1.0        # knot span of the QP cases (fixed: no MINTIME)
PT_DIST_QP = 0.35  # pt_dist_ (the smoothness scale), FUEL's ctrl_pt_dist


def kind_mask(orc, kind):
    """guide: FUEL's GUIDE_PHASE (SMOOTHNESS | GUIDE | START | END); end3: SMOOTHNESS | START | END with a 3-entry end
    state; waypt: SMOOTHNESS | GUIDE | WAYPOINTS | START | END with a 2-entry end state."""
    return {"guide": orc.GUIDE_PHASE,
            "end3": orc.SMOOTHNESS | orc.START | orc.END,
            "waypt": orc.SMOOTHNESS | orc.GUIDE | orc.WAYPOINTS | orc.START | orc.END}[kind]


def kind_params(kind):
    """Weights (keyword arguments of opt_params / setParam).  GUIDE_PHASE keeps FUEL's defaults."""
    return {"guide": {}, "end3": dict(ld_smooth=1.0, ld_start=10.0, ld_end=10.0), "waypt": dict(ld_waypt=3.0)}[kind]


def kind_ns(kind):
    """Point counts of a kind.  Without guide points the interior is held by the jerk term alone, whose lowest modes
    fall like n^-6: with the end3 weights kappa(H) is 4e4 at 20 points and passes KAPPA_MAX at 23 (8e5 at 32), and no
    choice of the three weights keeps it below at 32 points.  So end3 stops at 20; guide and waypt take every N."""
    return [N for N in SHORT_N + LONG_N if kind != "end3" or N <= 20]


def qp_case(g, inflate, N, kind, B=B_QP):
    """B trajectories of N points with fixed dt.  Bounds bite: every 4th trajectory (b % 4 == 1) has its guides lifted
    1.5 m and its start and end points 0.5 m above the box; b % 4 == 2 has its guides 6 m to -y (past the box for most of them);
    trajectory 0 (where there are guide points) starts near the -x face with its guides 16 m away at the +x face, so
    the start +- 10 m bound of optimize() (:208-214) is active."""
    seed = 4000 + 10 * N + KINDS.index(kind)
    spacing = min(0.35, 9.0 / (N - 1))  # 64 points still fit the 18 m office box
    tr = W.make_trajectories(g, inflate, B=B, n_pts=N, seed=seed, spacing=spacing)
    rng = np.random.default_rng(seed)
    lo, hi = g.box_min + 0.1, g.box_max - 0.1
    n_end = {"guide": 1, "end3": 3, "waypt": 2}[kind]
    ng = max(N - 6, 0)
    ctrl, dt = tr["ctrl"].copy(), np.full(B, DT_QP)
    start, end = tr["start"].copy(), np.zeros((B, n_end, 3))
    end[:, 0] = tr["end_pos"]
    end[:, 1:] = rng.normal(scale=0.5, size=(B, n_end - 1, 3))
    guide = ctrl[:, 3:N - 3] + rng.normal(scale=0.3, size=(B, ng, 3))
    ptd = np.full(B, PT_DIST_QP)
    if ng and kind != "end3":
        line = np.stack([np.linspace(lo[0] + 0.4, lo[0] + 0.4 + spacing * (N - 1), N), np.zeros(N), np.full(N, 0.6)], 1)
        ctrl[0] = line
        start[0], end[0, 0] = W.cubic_boundary_states(line, dt[0])
        guide[0] = [hi[0] - 0.5, 0.0, 0.6]
    guide[1::4, :, 2] += 1.5
    start[1::4, 0, 2] = hi[2] + 0.5
    end[1::4, 0, 2] = hi[2] + 0.5
    guide[2::4, :, 1] -= 6.0
    widx = sorted({0, (N - 3) // 2, N - 3})  # stencils idx..idx+2: the first, a middle and the last legal one
    waypt = ctrl[:, [i + 1 for i in widx]] + rng.normal(scale=0.4, size=(B, len(widx), 3))
    tr = dict(tr, ctrl=ctrl, dt=dt, start=start, end_pos=end[:, 0], pt_dist=ptd)
    kw = dict(n_end=n_end)
    if kind != "end3":
        kw.update(guide=guide)
    if kind == "waypt":
        kw.update(waypt=waypt, waypt_idx=widx)
    return dict(tr=tr, kw=kw, end=end, x0=W.pack_x(ctrl, dt, mintime=False), N=N, kind=kind, B=B)


def case_consts(make, lib, case):
    """gpu_consts / orc_consts of the case, with the end velocity / acceleration entries filled in"""
    tcs = make(lib, case["tr"], case["B"], **case["kw"])
    end = case["end"]
    for b in range(case["B"]):
        for i in range(1, end.shape[1]):
            for k in range(3):
                tcs[b].end[i][k] = end[b, i, k]
    return tcs


def box_bounds(g, x0, N):
    """optimize() :196-217: clamp to the box shrunk by 0.1 m, bounds = clamped start +- 10 m within it"""
    bmin, bmax = np.tile(g.box_min + 0.1, N), np.tile(g.box_max - 0.1, N)
    c = np.maximum(np.minimum(x0, bmax), bmin)
    return c, np.maximum(c - 10.0, bmin), np.minimum(c + 10.0, bmax)


def assemble_qp(orc, og, dist, po, to, N, mask):
    """H [B,n,n], b [B,n], c [B] of combineCost = 1/2 x'Hx + b'x + c, from the oracle's gradient at 0 and at every unit
    vector: one batched call of n + 1 rows per trajectory."""
    B, n = len(to), 3 * N
    rows = orc.traj_consts(B * (n + 1))
    for b in range(B):
        for j in range(n + 1):
            rows[b * (n + 1) + j] = to[b]
    X = np.zeros((B, n + 1, n))
    X[:, 1:, :] = np.eye(n)
    f, gr = orc.combine_cost_batch(og, dist, po, rows, N, mask, X.reshape(-1, n), threads=8)
    gr = gr.reshape(B, n + 1, n)
    bv = gr[:, 0].copy()
    H = np.swapaxes(gr[:, 1:] - bv[:, None, :], 1, 2)  # column i = H e_i
    return H, bv, f.reshape(B, n + 1)[:, 0].copy()


def solve_box_qp(H, b, lb, ub):
    """argmin 1/2 x'Hx + b'x over lb <= x <= ub: BVLS on || L'x + L^-1 b ||, L L' = H, then a primal active-set
    iteration from the BVLS point (exact fp64 solves on the free variables) until the KKT conditions hold."""
    L = np.linalg.cholesky(H)
    r = lsq_linear(L.T, -sla.solve_triangular(L, b, lower=True), bounds=(lb, ub), method="bvls", tol=1e-15,
                   max_iter=20 * len(b))
    x = np.clip(r.x, lb, ub)
    for _ in range(4 * len(b)):
        gr = H @ x + b
        at_lb, at_ub = x <= lb, x >= ub
        free = ~(at_lb | at_ub) | (at_lb & (gr < 0)) | (at_ub & (gr > 0))  # release the bounds that hold wrongly
        fix = ~free
        xf = np.linalg.solve(H[np.ix_(free, free)], -(b[free] + H[np.ix_(free, fix)] @ x[fix]))
        d = xf - x[free]
        with np.errstate(divide="ignore", invalid="ignore"):
            room = np.where(d > 0, (ub[free] - x[free]) / d, np.where(d < 0, (lb[free] - x[free]) / d, np.inf))
        t = min(1.0, float(np.min(room)))
        xn = x[free] + t * d
        if t < 1.0:  # the blocking variables land exactly on their bound
            hit = room <= t
            xn[hit] = np.where(d[hit] > 0, ub[free][hit], lb[free][hit])
        xn = np.clip(xn, lb[free], ub[free])
        x[free] = xn
        if t >= 1.0 and kkt_residual(H, b, x, lb, ub) < 1e-14:
            break
    return x


def kkt_residual(H, b, x, lb, ub):
    """largest violation of the box KKT conditions, relative to the gradient scale |b| + |H||x|"""
    gr = H @ x + b
    scale = np.max(np.abs(b) + np.abs(H) @ np.abs(x))
    at_lb, at_ub = x <= lb, x >= ub
    free = ~(at_lb | at_ub)
    viol = np.concatenate([np.abs(gr[free]), np.maximum(-gr[at_lb], 0.0), np.maximum(gr[at_ub], 0.0), [0.0]])
    return float(np.max(viol) / scale)


_QP = {}


def reference_qp(orc, og, dist, g, inflate, N, kind):
    """the case, its QP and x* (cached: the CPU and the device tests share them)"""
    key = (N, kind)
    if key not in _QP:
        case = qp_case(g, inflate, N, kind)
        po = orc.opt_params(**kind_params(kind))
        to = case_consts(orc_consts, orc, case)
        mask = kind_mask(orc, kind)
        H, bv, c = assemble_qp(orc, og, dist, po, to, N, mask)
        x0c, lb, ub = box_bounds(g, case["x0"], N)
        Hs = 0.5 * (H + np.swapaxes(H, 1, 2))
        xs = np.stack([solve_box_qp(Hs[i], bv[i], lb[i], ub[i]) for i in range(case["B"])])
        q = lambda i, x: 0.5 * x @ Hs[i] @ x + bv[i] @ x + c[i]  # noqa: E731
        f0 = np.array([q(i, x0c[i]) for i in range(case["B"])])
        fs = np.array([q(i, xs[i]) for i in range(case["B"])])
        _QP[key] = dict(case, po=po, to=to, mask=mask, H=H, Hs=Hs, b=bv, c=c, x0c=x0c, lb=lb, ub=ub, xs=xs, f0=f0, fs=fs)
    return _QP[key]


def suboptimality(Q, x):
    """(q(x) - q(x*)) / (q(x0) - q(x*)) per trajectory, from the displacement (no cancellation against c)"""
    d = x - Q["xs"]
    gs = np.einsum("bij,bj->bi", Q["Hs"], Q["xs"]) + Q["b"]
    dq = np.einsum("bi,bi->b", gs, d) + 0.5 * np.einsum("bi,bij,bj->b", d, Q["Hs"], d)
    return dq / np.maximum(Q["f0"] - Q["fs"], np.finfo(np.float64).tiny)


_TWIN = {}


def twin_error(orc, S, Q, m):
    """max |x - x*|_inf and max suboptimality of the CPU twin over the case's batch (cached)"""
    key = (Q["N"], Q["kind"], m)
    if key not in _TWIN:
        xc, _, _ = orc.optimize_batch(S["og"], S["d0"], Q["po"], Q["to"], Q["N"], Q["mask"], Q["x0"], max_eval=MAX_EVAL,
                                      lbfgs_m=m, xtol_rel=0.0, threads=8)
        _TWIN[key] = (float(np.max(np.abs(xc - Q["xs"]))), float(np.max(suboptimality(Q, xc))))
    return _TWIN[key]


@pytest.fixture(scope="module")
def cpu_field(orc):
    """the office map's box; the QP terms never read the distance field"""
    g, inflate = W.office_map()
    return dict(g=g, inflate=inflate, og=orc_grid(orc, g), d0=np.zeros(tuple(g.n)))


# ---- CPU: the premise of the exact reference -----------------------------------------------------------------------

@pytest.mark.parametrize("kind", KINDS)
def test_qp_premise(orc, cpu_field, kind):
    """The fitted quadratic is combineCost: it reproduces the oracle's cost at random points, H is symmetric and
    positive definite with kappa(H) <= KAPPA_MAX, x* satisfies the box KKT conditions, bounds are active where the
    case means them to be (guides and end points outside the box, the start +- 10 m bound)."""
    S = cpu_field
    rng = np.random.default_rng(7)
    kappas = {}
    for N in kind_ns(kind):
        Q = reference_qp(orc, S["og"], S["d0"], S["g"], S["inflate"], N, kind)
        B, n = Q["B"], 3 * N
        asym = np.max(np.abs(Q["H"] - np.swapaxes(Q["H"], 1, 2))) / np.max(np.abs(Q["H"]))
        assert asym < 1e-12, (N, asym)
        ev = np.linalg.eigvalsh(Q["Hs"])
        assert np.all(ev[:, 0] > 0), (N, ev[:, 0].min())
        kap = ev[:, -1] / ev[:, 0]
        kappas[N] = kap.max()
        assert np.all(kap <= KAPPA_MAX), (N, kap.max())
        xr = Q["x0c"] + rng.normal(scale=2.0, size=(B, n))
        fr, gr = orc.combine_cost_batch(S["og"], S["d0"], Q["po"], Q["to"], N, Q["mask"], xr)
        fq = 0.5 * np.einsum("bi,bij,bj->b", xr, Q["Hs"], xr) + np.einsum("bi,bi->b", Q["b"], xr) + Q["c"]
        assert np.all(np.abs(fq - fr) <= 1e-12 * np.abs(fr)), (N, np.max(np.abs(fq - fr) / np.abs(fr)))
        gq = np.einsum("bij,bj->bi", Q["Hs"], xr) + Q["b"]
        assert np.all(np.abs(gq - gr) <= 1e-10 * np.max(np.abs(gr), axis=1, keepdims=True))
        kkt = max(kkt_residual(Q["Hs"][i], Q["b"][i], Q["xs"][i], Q["lb"][i], Q["ub"][i]) for i in range(B))
        assert kkt < 1e-12, (N, kkt)
        assert np.all(Q["xs"] >= Q["lb"]) and np.all(Q["xs"] <= Q["ub"])
        nact = np.sum((Q["xs"] <= Q["lb"]) | (Q["xs"] >= Q["ub"]), axis=1)
        assert np.sum(nact > 0) >= B // 4, (N, nact)  # the lifted / shifted trajectories hit the box
        assert np.all(Q["f0"] > Q["fs"])
        if kind != "end3" and N >= 16:  # guide points 16 m away: the start + 10 m bound holds trajectory 0 back
            x0 = Q["x0c"][0].reshape(N, 3)
            assert np.any(Q["xs"][0].reshape(N, 3)[:, 0] >= x0[:, 0] + 10.0)
    print(kind, "kappa(H) by N:", " ".join("%d:%.3g" % (N, k) for N, k in kappas.items()))


@pytest.mark.parametrize("kind", KINDS)
def test_cpu_twin_converges_to_qp_minimizer(orc, cpu_field, kind):
    """The CPU twin orc_optimize_batch (the same projected L-BFGS as the device, in fp64) at the device test's budget
    and history lengths reaches x*.  The accuracy it reaches sets the scale of the device bar."""
    S = cpu_field
    worst = {}
    for N in kind_ns(kind):
        Q = reference_qp(orc, S["og"], S["d0"], S["g"], S["inflate"], N, kind)
        for m in LBFGS_M:
            ex, sub = twin_error(orc, S, Q, m)
            worst[m] = max(worst.get(m, (0.0, 0.0)), (ex, sub))
            assert ex < 1e-2 and sub < 1e-8, (N, m, ex, sub)
    print(kind, "twin max |x - x*|_inf / suboptimality by lbfgs_m:",
          " ".join("m=%d %.2g/%.2g" % (m, e, s) for m, (e, s) in sorted(worst.items())))


# ---- device -----------------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def scene(fuel, orc, cpu_field):
    """the office map on the device (its ESDF for the NORMAL_PHASE parity) and the oracle's fp64 field"""
    g, inflate = cpu_field["g"], cpu_field["inflate"]
    tri = W.office_known(g, inflate)
    m = make_sdf_map(fuel, g, inflate, tri, optimistic=True)
    m.updateESDF3d()
    env = fuel.EDTEnvironment()
    env.setMap(m)
    opts = {}
    for kind in (None,) + KINDS:
        opts[kind] = fuel.BsplineOptimizer()
        opts[kind].setEnvironment(env)
        if kind:
            opts[kind].setParam(**kind_params(kind))
    d64 = orc.update_esdf3d(cpu_field["og"], inflate, tri, [0, 0, 0], np.array(g.n) - 1, True, False, threads=8)
    yield dict(cpu_field, m=m, opt=opts[None], opts=opts, d64=d64)
    m.close()


def device_bar(orc, S, kind, m):
    """max(1e-6 m, 10 x) the CPU twin's largest |x - x*|_inf, and max(1e-9, 10 x) its largest suboptimality, over the
    kind's point counts at history length m and the same budget"""
    errs = [twin_error(orc, S, reference_qp(orc, S["og"], S["d0"], S["g"], S["inflate"], N, kind), m) for N in kind_ns(kind)]
    return max(1e-6, 10 * max(e for e, _ in errs)), max(1e-9, 10 * max(s for _, s in errs))


def kernel_of(N, m):
    return "long" if N > 32 else ("gram<6>" if m == 6 else "warp")


@pytest.mark.gpu
@pytest.mark.parametrize("N", SHORT_N + LONG_N)
def test_solver_converges_to_qp_minimizer(fuel, orc, scene, N):
    """Every history length (6: optimize_gram_kernel<6>, else optimize_warp_kernel; above 32 points the long solver),
    B = 37, xtol_rel = 0 and MAX_EVAL evaluations: the returned x is x* within max(1e-6 m, 10 x the CPU twin's error)
    and its suboptimality (q(x) - q*) / (q(x0) - q*) is within max(1e-9, 10 x the twin's), the twin's errors taken as
    the largest over the kind's point counts at the same history length and budget.  The returned x stays in the box;
    f_best is q(x) (the QP is combineCost).

    Measured on an H100 80GB HBM3 (short kernels): m = 4, 6, 8 land within 1.1e-5 m of x* with suboptimality at most
    2.3e-14; m = 2 within 1.9e-4 m and 1.9e-12 (the twin: 1.7e-4 m).  The fp64 twin itself stops up to 1.2e-5 m from
    x* at m >= 4, so the x bar is 10 x that, not 1e-6 m.  m = 1 does not converge within the budget on either side
    (kappa up to 4e4 with one stored pair): the fp64 twin stops up to 3.6e-3 m from x* (suboptimality 1.4e-9), the
    device up to 1.5e-2 m (9e-9), on a different iterate path since its inner products are fp32.  A per-case comparison with the twin there measures path noise, so the bar takes
    the twin's worst case over the point counts."""
    S = scene
    rows = []
    for kind in KINDS:
        if N not in kind_ns(kind):
            continue
        Q = reference_qp(orc, S["og"], S["d0"], S["g"], S["inflate"], N, kind)
        tg = case_consts(gpu_consts, fuel, Q)
        for m in LBFGS_M:
            xg, fg, ng = S["opts"][kind].optimizeBatch(Q["x0"], tg, N, Q["mask"], MAX_EVAL, lbfgs_m=m, xtol_rel=0.0)
            assert np.all(xg >= Q["lb"]) and np.all(xg <= Q["ub"]) and np.all(ng <= MAX_EVAL)
            fq = 0.5 * np.einsum("bi,bij,bj->b", xg, Q["Hs"], xg) + np.einsum("bi,bi->b", Q["b"], xg) + Q["c"]
            assert np.all(np.abs(fg - fq) <= 1e-9 * np.abs(fq)), (kind, m)
            ex, sub = np.max(np.abs(xg - Q["xs"]), axis=1), suboptimality(Q, xg)
            bar_x, bar_s = device_bar(orc, S, kind, m)
            rows.append("%s m=%d %s |x-x*| %.2g (bar %.2g) sub %.2g (bar %.2g)" % (kind, m, kernel_of(N, m), ex.max(),
                                                                                 bar_x, sub.max(), bar_s))
            assert ex.max() <= bar_x and sub.max() <= bar_s, rows[-1]
    print("\nN=%d\n  " % N + "\n  ".join(rows))


@pytest.mark.gpu
@pytest.mark.parametrize("N", SHORT_N)
def test_cost_parity_every_short_n(fuel, orc, scene, N):
    """The faithful and the solver's evaluator (FUELGPU_COST_FAST_EVAL) against the oracle at the 1e-4 bar, at every
    short point count, NORMAL_PHASE with and without MINTIME (dt halved on every third trajectory so that feasibility
    bites; N = 32 with MINTIME is 97 variables, dt read from x[nvar-1]); GUIDE_PHASE at 7 and 8 points, where the guide
    range [3, N-3) is one or two points long."""
    O = fuel.BsplineOptimizer
    B = 64
    S = scene
    tr = W.make_trajectories(S["g"], S["inflate"], B=B, n_pts=N, seed=2000 + N)
    tr["dt"][::3] *= 0.5
    cases = [(O.NORMAL_PHASE, {}), (O.NORMAL_PHASE | O.MINTIME, {})]
    if N <= 8:
        cases.append((O.GUIDE_PHASE, dict(guide=tr["ctrl"][:, 3:N - 3] + 0.2)))
    for mask, kw in cases:
        x = W.pack_x(tr["ctrl"], tr["dt"], mintime=bool(mask & O.MINTIME))
        fr, gr = orc.combine_cost_batch(S["og"], S["d64"], orc.opt_params(), orc_consts(orc, tr, B, **kw), N, mask, x,
                                        threads=8)
        tg = gpu_consts(fuel, tr, B, **kw)
        for fast in (False, True):
            f, gg = S["opt"].combineCostBatch(x, tg, N, mask, fast_eval=fast)
            check(f, gg, fr, gr)
    d, _ = S["m"].getDistWithGrad(tr["ctrl"].reshape(-1, 3))
    assert np.mean(d < 0.7) > 0.05  # the distance term is active


_TR = {}


def batch(S, B, N):
    if (B, N) not in _TR:
        _TR[(B, N)] = W.make_trajectories(S["g"], S["inflate"], B=B, n_pts=N, seed=300 + B + N)
    return _TR[(B, N)]


@pytest.mark.gpu
@pytest.mark.parametrize("lbfgs_m", [1, 4, 6, 8])
@pytest.mark.parametrize("B", [1, 5, 4097])
def test_optimize_short_same_path_same_bits(fuel, scene, lbfgs_m, B):
    """At 7 points (the fewest the API takes), 31 points + dt (dt on lane 31) and 32 points (a full warp of points):
    two runs are bitwise equal,
    begin/end equals the one-shot call, the device-pointer entry equals the host entry."""
    import torch

    from fuel_b200._lib import FuelSolveParams, check as lib_check
    K = 48
    O = fuel.BsplineOptimizer
    opt = scene["opt"]
    for N, mintime in ((7, True), (31, True), (32, False)):
        tr = batch(scene, B, N)
        mask = O.NORMAL_PHASE | (O.MINTIME if mintime else 0)
        x0 = W.pack_x(tr["ctrl"], tr["dt"], mintime=mintime)
        tc = gpu_consts(fuel, tr, B)
        x1, f1, n1 = [a.copy() for a in opt.optimizeBatch(x0, tc, N, mask, K, lbfgs_m=lbfgs_m)]
        x2, f2, n2 = [a.copy() for a in opt.optimizeBatch(x0, tc, N, mask, K, lbfgs_m=lbfgs_m)]
        assert np.array_equal(x1, x2) and np.array_equal(f1, f2) and np.array_equal(n1, n2), N
        opt.optimizeBatchBegin(x0, tc, N, mask, K, lbfgs_m=lbfgs_m)
        x3, f3, n3 = opt.optimizeBatchEnd()
        assert np.array_equal(x1, x3) and np.array_equal(f1, f3) and np.array_equal(n1, n3), N
        d_tc = torch.from_numpy(np.frombuffer(tc, dtype=np.uint8).copy()).cuda()
        d_x = torch.from_numpy(x0).cuda()
        d_f = torch.empty(B, dtype=torch.float64, device="cuda")
        d_n = torch.empty(B, dtype=torch.int32, device="cuda")
        sp = FuelSolveParams()
        sp.max_eval, sp.lbfgs_m, sp.xtol_rel, sp.flags = K, lbfgs_m, 1e-5, 0
        torch.cuda.synchronize()
        h = scene["m"].handle
        lib_check(fuel.lib().fuelgpu_bspline_optimize_batch_dev(h, B, N, mask, C.byref(opt.params_),
                                                                C.c_void_p(d_tc.data_ptr()), C.byref(sp),
                                                                C.c_void_p(d_x.data_ptr()), C.c_void_p(d_f.data_ptr()),
                                                                C.c_void_p(d_n.data_ptr())), h)
        scene["m"].synchronize()
        torch.cuda.synchronize()
        assert np.array_equal(d_x.cpu().numpy(), x1) and np.array_equal(d_f.cpu().numpy(), f1), N
        assert np.array_equal(d_n.cpu().numpy(), n1), N


@pytest.mark.gpu
@pytest.mark.parametrize("lbfgs_m", [4, 6])
def test_optimize_short_f_best_is_faithful_cost(fuel, scene, lbfgs_m):
    """min_cost_ is fuelgpu_bspline_cost_batch (the faithful evaluator) at the returned x, bit for bit, at every short
    point count (with MINTIME up to 31 points, 32 without) and through both short kernels."""
    K = 64
    O = fuel.BsplineOptimizer
    for N in SHORT_N:
        B = 64
        tr = batch(scene, B, N)
        mintime = N < 32
        mask = O.NORMAL_PHASE | (O.MINTIME if mintime else 0)
        tc = gpu_consts(fuel, tr, B)
        xg, fg, ng = scene["opt"].optimizeBatch(W.pack_x(tr["ctrl"], tr["dt"], mintime=mintime), tc, N, mask, K,
                                                lbfgs_m=lbfgs_m)
        fc, _ = scene["opt"].combineCostBatch(xg, tc, N, mask)
        assert np.array_equal(fg, fc), (N, np.max(np.abs(fg - fc) / np.abs(fc)))


@pytest.mark.gpu
@pytest.mark.parametrize("N", [4, 5, 6])
def test_fewer_than_seven_points_are_refused(fuel, scene, N):
    """n_pts <= 2 * order leaves no interior point for the cost terms: the evaluator and the solver refuse it (EINVAL)."""
    O = fuel.BsplineOptimizer
    tr = W.make_trajectories(scene["g"], scene["inflate"], B=2, n_pts=7, seed=N)
    tr = dict(tr, ctrl=tr["ctrl"][:, :N])
    x = W.pack_x(tr["ctrl"], tr["dt"])
    tc = gpu_consts(fuel, tr, 2)
    with pytest.raises(fuel.FuelGpuError):
        scene["opt"].combineCostBatch(x, tc, N, O.NORMAL_PHASE | O.MINTIME)
    with pytest.raises(fuel.FuelGpuError):
        scene["opt"].optimizeBatch(x, tc, N, O.NORMAL_PHASE | O.MINTIME, 8)
