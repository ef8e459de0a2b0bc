"""FastPlannerManager::planYaw (plan_manage/src/planner_manager.cpp:695-772), the kinodynamic replan's yaw, restated in
Python over oracle.traj's evaluateDeBoorT (pinned bit for bit to the reference's; deriv=1 for the end velocity) for
every trajectory of a batch in the solver's layout, with oracle.yaw's calcNextYaw; and the ctypes binding of the
reference's own lines run through oracle/ref_plan_yaw_wrap.cpp and oracle/ref_plan_yaw_cost_wrap.cpp
(oracle/_ref/libfuel_ref_plan_yaw.so, built by oracle/plan_yaw.mk where the reference's sources are present).

Python floats are IEEE fp64 without contraction and math.atan2 is the C library's, so seg_num, dt_yaw, the waypoints,
the end velocity and yaw, the initial guess and pt_dist_ are the reference's values.  Unlike planYawExplore's 15 points
and two end states (oracle.yaw), the yaw spline has seg_num + 3 control points and three end states, so calcEndCost's
acceleration term is active.  The optimization that follows is NLopt's LD_LBFGS in the reference; solve() returns the
minimizer of the same quadratic objective by a dense fp64 solve of its normal equations -- NLopt parity unpinned.

TEST INFRASTRUCTURE ONLY, like the rest of this package: fuel_b200/ must never import it.
"""
import ctypes as C
import math

import numpy as np

from . import _load, _make, _p, ref_raycast, traj as _traj
from . import build as _build_oracle
from .yaw import (BAD_INPUT, FORWARD_T, NO_LOOKAHEAD, OK, YAW_MASK, ZERO_PT_DIST, calc_next_yaw, duration,  # noqa: F401
                  next_yaw_diff, pt_dist)

TOO_LONG = 6                # FUELGPU_YAW_TOO_LONG
PLANYAW_MAX_SEG = 128       # FUELGPU_PLANYAW_MAX_SEG
PLANYAW_DT = 0.3            # planYaw's dt_yaw before the division
DBL_MAX = 1.7976931348623157e308


def build():
    """Compile the reference's side with oracle/plan_yaw.mk (needs oracle/_ref/libfuel_ref.so from the Makefile first)."""
    _build_oracle()
    _make("plan_yaw.mk")


def initial_guess(dt_yaw, start, end_yaw, seg_num):
    """rows 0-2 = states2pts * start_yaw, then rows seg_num..seg_num+2 = states2pts * (end, 0, 0), zeros between
    (:735-744; for seg_num 1 and 2 the blocks overlap and the end block, written second, wins); each row of the 3x3
    product summed left to right"""
    c13 = ((1 / 3.0) * dt_yaw) * dt_yaw
    c16 = ((-(1 / 6.0)) * dt_yaw) * dt_yaw
    m = ((1.0, -dt_yaw, c13), (1.0, 0.0, c16), (1.0, dt_yaw, c13))
    g = [0.0] * (seg_num + 3)
    for r in range(3):
        g[r] = (m[r][0] * start[0] + m[r][1] * start[1]) + m[r][2] * start[2]
    for r in range(3):
        g[seg_num + r] = (m[r][0] * end_yaw + m[r][1] * 0.0) + m[r][2] * 0.0
    return g


def _finish(r):
    """the end yaw through calcNextYaw from the last waypoint, the initial guess and pt_dist_ (:732-744, optimize())"""
    r["end_yaw"] = calc_next_yaw(r["waypts"][-1], r["end_in"])
    r["guess"] = initial_guess(r["dt_yaw"], r["start"], r["end_yaw"], r["seg_num"])
    r["pt_dist"] = pt_dist(r["guess"])
    if r["pt_dist"] == 0.0:
        r["status"] = ZERO_PT_DIST


def with_waypoints(r, waypts, end_in=None):
    """row r of plan_yaw() rebuilt from other waypoints (e.g. the device's, whose atan2 may differ from the C library's in
    the last bits) and optionally another atan2 of the end velocity: the same indices, then the end yaw, initial guess and
    pt_dist_ by the reference's arithmetic"""
    assert len(waypts) == len(r["waypts"])
    out = dict(r)
    out["waypts"] = [float(w) for w in waypts]
    if end_in is not None:
        out["end_in"] = float(end_in)
    _finish(out)
    return out


def plan_yaw(x, n_pts, start_yaw, dt=None):
    """planYaw's construction (:695-745) for each trajectory of x [B, nvar] (dt in the last column, or dt [B]), start_yaw
    [B, 3] used as given.  Returns a list of dicts: status, seg_num, dt_yaw, duration, waypts, waypt_idx, end_v (the
    velocity spline at duration - 0.1), end_in (its atan2), end_yaw (after calcNextYaw), start, guess [seg_num + 3],
    pt_dist, n_pts = seg_num + 3 (yaw control points), and margin: the least | |diff| - pi | over the calcNextYaw calls.
    Rows the device refuses (dt not finite and positive, non-finite start yaw, |start yaw| > 1000, a duration that is not
    finite and positive) get BAD_INPUT, duration / 0.3 > 128 TOO_LONG."""
    x = np.ascontiguousarray(x, dtype=np.float64)
    B = x.shape[0]
    dts = x[:, 3 * n_pts] if dt is None else np.broadcast_to(np.asarray(dt, dtype=np.float64), (B,))
    sy = np.broadcast_to(np.asarray(start_yaw, dtype=np.float64), (B, 3))
    rows = []
    t = np.zeros((B, 2 * PLANYAW_MAX_SEG))
    te = np.zeros((B, 1))
    for b in range(B):
        d = float(dts[b])
        r = dict(dt_yaw=math.nan, seg_num=0, waypts=[], waypt_idx=[], status=OK, pt_dist=math.nan, margin=math.inf)
        rows.append(r)
        if not (0.0 < d <= DBL_MAX) or not all(math.isfinite(v) for v in sy[b]) or abs(sy[b][0]) > 1000.0:
            r["status"] = BAD_INPUT
            continue
        dur = duration(d, n_pts)
        if not (0.0 < dur <= DBL_MAX):
            r["status"] = BAD_INPUT
            continue
        q = dur / PLANYAW_DT
        if not q <= PLANYAW_MAX_SEG:
            r["status"] = TOO_LONG
            continue
        seg = int(math.ceil(q))
        dt_yaw = dur / seg
        r.update(seg_num=seg, dt_yaw=dt_yaw, duration=dur, n_pts=seg + 3)
        for i in range(seg):
            tc = i * dt_yaw
            t[b, i], t[b, PLANYAW_MAX_SEG + i] = tc, min(dur, tc + FORWARD_T)
        te[b, 0] = dur - 0.1
    dtv = None if dt is None else np.ascontiguousarray(dts, dtype=np.float64)
    pts = _traj.bspline_evaluate(x, n_pts, t, dt=dtv)
    vel = _traj.bspline_evaluate(x, n_pts, te, deriv=1, dt=dtv)
    for b, r in enumerate(rows):
        if r["status"] != OK:
            continue
        r["start"] = [float(v) for v in sy[b]]
        last_yaw = r["start"][0]
        for i in range(r["seg_num"]):
            pc, pf = pts[b, i], pts[b, PLANYAW_MAX_SEG + i]
            dx, dy, dz = float(pf[0] - pc[0]), float(pf[1] - pc[1]), float(pf[2] - pc[2])
            if math.sqrt((dx * dx + dy * dy) + dz * dz) > 1e-6:
                a = math.atan2(dy, dx)
                r["margin"] = min(r["margin"], abs(abs(next_yaw_diff(last_yaw, a)) - math.pi))
                w = calc_next_yaw(last_yaw, a)
            elif not r["waypts"]:
                r["status"] = NO_LOOKAHEAD  # waypts.back() of an empty vector
                break
            else:
                w = r["waypts"][-1]
            last_yaw = w
            r["waypts"].append(w)
            r["waypt_idx"].append(i)
        if r["status"] != OK:
            r["waypts"], r["waypt_idx"] = [], []
            continue
        r["end_v"] = [float(v) for v in vel[b, 0]]
        r["end_in"] = math.atan2(r["end_v"][1], r["end_v"][0])
        r["margin"] = min(r["margin"], abs(abs(next_yaw_diff(last_yaw, r["end_in"])) - math.pi))
        _finish(r)
    return rows



def terms(r, ld_smooth=5.0, ld_start=10.0, ld_end=10.0, ld_waypt=20.0, num=float):
    """The objective of optimize(yaw, dt_yaw, SMOOTHNESS | WAYPOINTS | START | END) with three end states, for row r of
    plan_yaw(), as a list of (offset, a, w, t): sum of w * (a . q[offset:offset + len(a)] - t)^2.  `num` converts each
    float (Fraction for an exact solve)."""
    n = r["n_pts"]
    seg = n - 3
    dt, p = num(r["dt_yaw"]), num(r["pt_dist"])
    y0, y1, y2 = (num(v) for v in r["start"])
    ye = num(r["end_yaw"])
    six = num(6)
    out = [(i, (-1, 3, -3, 1), num(ld_smooth) / (p * p), num(0)) for i in range(n - 3)]
    out += [(0, (1, 4, 1), num(ld_start) * 10 / 36, six * y0), (0, (-1, 0, 1), num(ld_start) / (4 * dt * dt), 2 * dt * y1),
            (0, (1, -2, 1), num(ld_start) / (dt * dt * dt * dt), dt * dt * y2),
            (seg, (1, 4, 1), num(ld_end) / 36, six * ye), (seg, (-1, 0, 1), num(ld_end) / (4 * dt * dt), num(0)),
            (seg, (1, -2, 1), num(ld_end) / (dt * dt * dt * dt), num(0))]
    out += [(i, (1, 4, 1), num(ld_waypt) / 36, six * num(w)) for i, w in zip(r["waypt_idx"], r["waypts"])]
    return out


def normal_equations(r, num=float, **ld):
    """H q = rhs at the minimizer (Hessian and gradient at 0, both halved) -> (H [n][n], rhs [n]) as lists, n = seg_num + 3"""
    n = r["n_pts"]
    H = [[num(0)] * n for _ in range(n)]
    rhs = [num(0)] * n
    for o, a, w, t in terms(r, num=num, **ld):
        for u in range(len(a)):
            for v in range(len(a)):
                H[o + u][o + v] += w * a[u] * a[v]
            rhs[o + u] += w * a[u] * t
    return H, rhs


def solve(r, **ld):
    """the minimizer by a dense fp64 solve (NLopt parity unpinned)"""
    H, rhs = normal_equations(r, **ld)
    return np.linalg.solve(np.array(H), np.array(rhs))


def objective(rows, q, ld_smooth=5.0, ld_start=10.0, ld_end=10.0, ld_waypt=20.0):
    """combineCost(q) and its gradient for the objective of each plan_yaw() row (q [B, >= n], the first n = seg_num + 3
    columns read) -> (f [B], grad: a list of [n] arrays).  Rows with n <= 64 (the oracle's point limit) go through the
    oracle's pinned 3-D combineCost on q padded with zero y and z columns, three end states; longer rows through the same
    quadratic written as terms() (sum of w (a . q - t)^2, gradient 2 sum w (a . q - t) a), which agrees with it to
    rounding."""
    from . import combine_cost_batch, fill_traj_const, make_grid, opt_params, traj_consts
    ld = dict(ld_smooth=ld_smooth, ld_start=ld_start, ld_end=ld_end, ld_waypt=ld_waypt)
    g = make_grid((4, 4, 4), 0.1, (0, 0, 0))
    p = opt_params(**ld)
    fs, grads = np.zeros(len(rows)), []
    for b, r in enumerate(rows):
        n = r["n_pts"]
        qb = np.asarray(q[b], dtype=np.float64)[:n]
        if n <= 64:
            tcs = traj_consts(1)
            s = r["start"]
            wp = [(w, 0.0, 0.0) for w in r["waypts"]] or None
            fill_traj_const(tcs[0], r["pt_dist"], r["dt_yaw"], [(s[0], 0, 0), (s[1], 0, 0), (s[2], 0, 0)],
                            [(r["end_yaw"], 0, 0), (0, 0, 0), (0, 0, 0)], waypt=wp, waypt_idx=r["waypt_idx"] or None)
            x = np.zeros((1, 3 * n))
            x[0, 0::3] = qb
            f, gr = combine_cost_batch(g, np.zeros(64), p, tcs, n, YAW_MASK, x)
            fs[b], gb = f[0], gr[0, 0::3]
        else:
            gb = np.zeros(n)
            for o, a, w, t in terms(r, **ld):
                e = float(np.dot(a, qb[o:o + len(a)])) - t
                fs[b] += w * e * e
                gb[o:o + len(a)] += 2.0 * w * e * np.asarray(a, dtype=np.float64)
        grads.append(np.asarray(gb))
    return fs, grads



# ---- the reference's own code ------------------------------------------------------------------------------------------
def ref_plan_yaw_lib():
    """oracle/_ref/libfuel_ref_plan_yaw.so (the reference's non_uniform_bspline.cpp + ref_plan_yaw_wrap.cpp, and
    ref_plan_yaw_cost_wrap.cpp over _ref/libfuel_ref.so's BsplineOptimizer), or None where it is not built."""
    return _load("_ref/libfuel_ref_plan_yaw.so", dict(ref_plan_yaw=C.c_int32, ref_plan_yaw_cost=C.c_int32),
                 first=ref_raycast)


def ref_plan_yaw(ctrl, dt, start_yaw):
    """the reference's lines :695-745 over its compiled NonUniformBspline, for one trajectory ctrl [n, 3] -> dict(status,
    seg_num, dt_yaw, duration, waypts, waypt_idx, end_v, end_in, end_yaw, guess, pt_dist); status NO_LOOKAHEAD where the
    reference reads waypts.back() of an empty vector, TOO_LONG past 128 segments (nothing else then)"""
    ctrl = np.ascontiguousarray(ctrl, dtype=np.float64)
    sy = np.ascontiguousarray(start_yaw, dtype=np.float64)
    od = np.zeros(8)  # duration, dt_yaw, atan2 of end_v, end yaw after calcNextYaw, pt_dist_, end_v
    oi = np.zeros(2, dtype=np.int32)  # seg_num, waypoint count
    wp, widx = np.zeros(PLANYAW_MAX_SEG), np.zeros(PLANYAW_MAX_SEG, dtype=np.int32)
    guess = np.zeros(PLANYAW_MAX_SEG + 3)
    rc = ref_plan_yaw_lib().ref_plan_yaw(C.c_int32(ctrl.shape[0]), _p(ctrl), C.c_double(dt), _p(sy), C.c_int32(PLANYAW_MAX_SEG),
                                _p(od), _p(oi), _p(wp), _p(widx), _p(guess))
    if rc != 0:
        return dict(status=NO_LOOKAHEAD if rc == -1 else TOO_LONG)
    s, k = int(oi[0]), int(oi[1])
    return dict(status=OK, seg_num=s, dt_yaw=od[1], duration=od[0], waypts=wp[:k].tolist(), waypt_idx=widx[:k].tolist(),
                end_v=od[5:8].tolist(), end_in=od[2], end_yaw=od[3], guess=guess[:s + 3].tolist(), pt_dist=od[4])


def ref_plan_yaw_cost(ref_map, r, probes, ld_smooth=5.0, ld_start=10.0, ld_end=10.0, ld_waypt=20.0):
    """the REFERENCE's optimize(yaw [(seg_num + 3) x 1], dt_yaw, SMOOTHNESS | START | END | WAYPOINTS, 1, 1) with
    planYaw's boundary states (three end states) and waypoints (row r of plan_yaw()): combineCost at its initial guess
    and at probes [K, n] -> (f [1 + K], grad [1 + K, n]).  Default weights: kino_algorithm.xml's."""
    n = r["n_pts"]
    keys = [b"optimization/" + k.encode() for k in ("ld_smooth", "ld_start", "ld_end", "ld_waypt")]
    karr = (C.c_char_p * 4)(*keys)
    vals = np.array([ld_smooth, ld_start, ld_end, ld_waypt], dtype=np.float64)
    probes = np.ascontiguousarray(probes, dtype=np.float64).reshape(-1, n)
    K = probes.shape[0]
    f, grad = np.zeros(1 + K), np.zeros((1 + K, n))
    start = np.ascontiguousarray(r["start"], dtype=np.float64)
    wp = np.ascontiguousarray(r["waypts"], dtype=np.float64)
    widx = np.ascontiguousarray(r["waypt_idx"], dtype=np.int32)
    rc = ref_plan_yaw_lib().ref_plan_yaw_cost(ref_map.h, C.c_int32(4), karr, _p(vals), C.c_int32(n),
                                     _p(np.ascontiguousarray(r["guess"], dtype=np.float64)), C.c_double(r["dt_yaw"]),
                                     _p(start), C.c_double(r["end_yaw"]), C.c_int32(len(wp)), _p(wp), _p(widx),
                                     C.c_int32(K), _p(probes), _p(f), _p(grad))
    assert rc == 0, rc
    return f, grad
