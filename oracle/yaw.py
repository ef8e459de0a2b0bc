"""FastPlannerManager::planYawExplore (plan_manage/src/planner_manager.cpp:776-853) and calcNextYaw (:867-885)
restated in Python over oracle.traj's evaluateDeBoorT (which is pinned bit for bit to the reference's), for every
trajectory of a batch in the solver's layout; and the ctypes binding of the reference's own lines run through
oracle/ref_yaw_wrap.cpp (oracle/_ref/libfuel_ref_yaw.so, built by oracle/yaw.mk where the reference's sources are present).

Python floats are IEEE fp64 without contraction and math.atan2 is the C library's, so dt_yaw, relax_num, the waypoints,
waypt_idx, the initial guess and pt_dist_ are the reference's values.  The optimization that follows is NLopt's LD_LBFGS
in the reference; here solve() returns the minimizer of the same quadratic objective by a dense fp64 solve of its
normal equations -- NLopt parity unpinned.  objective() evaluates that objective with the oracle's pinned 3-D
combineCost on the control points padded with zero y and z columns, which equals the reference's dim_ == 1 combineCost
bit for bit (tests/test_oracle_yaw.py pins that too).

TEST INFRASTRUCTURE ONLY, like the rest of this package: fuel_b200/ must never import it.
"""
import ctypes as C
import math

import numpy as np

from . import _load, _make, _p, ref_raycast, traj as _traj
from . import build as _build_oracle

SEG_NUM = 12                # planYawExplore's seg_num
PTS = SEG_NUM + 3           # yaw control points
MAX_WAYPT = SEG_NUM - 1
FORWARD_T = 2.0
OK, BAD_INPUT, RELAX_OVERFLOW, NO_LOOKAHEAD, ZERO_PT_DIST, NOT_SPD = range(6)  # FUELGPU_YAW_* (0 = OK)
YAW_MASK = 1 | 8 | 16 | 64  # SMOOTHNESS | START | END | WAYPOINTS


def build():
    """Compile the reference's side with oracle/yaw.mk (needs oracle/_ref/libfuel_ref.so from the Makefile first)."""
    _build_oracle()
    _make("yaw.mk")


def wrap_start(y):
    """the two while loops of :782-783"""
    while y < -math.pi:
        y += 2 * math.pi
    while y > math.pi:
        y -= 2 * math.pi
    return y


def next_yaw_diff(last_yaw, yaw):
    """calcNextYaw's diff: yaw minus last_yaw rounded into [-pi, pi]"""
    round_last = last_yaw
    while round_last < -math.pi:
        round_last += 2 * math.pi
    while round_last > math.pi:
        round_last -= 2 * math.pi
    return yaw - round_last


def calc_next_yaw(last_yaw, yaw):
    """calcNextYaw (:867-885) -> the new yaw"""
    diff = next_yaw_diff(last_yaw, yaw)
    if abs(diff) <= math.pi:
        return last_yaw + diff
    elif diff > math.pi:
        return last_yaw + diff - 2 * math.pi
    elif diff < -math.pi:
        return last_yaw + diff + 2 * math.pi
    return yaw


def duration(dt, n_pts):
    """getTimeSum of setUniformBspline(ctrl, 3, dt): u_(n) - u_(3) of the running-sum knots"""
    u = [float(-3 + i) * dt for i in range(4)]
    for i in range(4, n_pts + 4):
        u.append(u[i - 1] + dt)
    return u[n_pts] - u[3]


def initial_guess(dt_yaw, start3d, end_yaw):
    """rows 0-2 = states2pts * start_yaw3d, rows 12-14 = states2pts * (end, 0, 0), zeros between (:786-793, :822-824);
    each row of the 3x3 product summed left to right"""
    c13 = ((1 / 3.0) * dt_yaw) * dt_yaw
    c16 = ((-(1 / 6.0)) * dt_yaw) * dt_yaw
    m = ((1.0, -dt_yaw, c13), (1.0, 0.0, c16), (1.0, dt_yaw, c13))
    g = [0.0] * PTS
    for r in range(3):
        g[r] = (m[r][0] * start3d[0] + m[r][1] * start3d[1]) + m[r][2] * start3d[2]
        g[SEG_NUM + r] = (m[r][0] * end_yaw + m[r][1] * 0.0) + m[r][2] * 0.0
    return g


def pt_dist(g):
    """optimize()'s pt_dist_ (bspline_optimizer.cpp:136-140) of a one-column matrix: sum of sqrt(d^2), over the rows"""
    d = 0.0
    for i in range(len(g) - 1):
        e = g[i + 1] - g[i]
        d += math.sqrt(e * e)
    return d / float(len(g))


def plan(x, n_pts, start_yaw, end_yaw, relax_time=1.0, lookfwd=True, dt=None):
    """planYawExplore's construction for each trajectory of x [B, nvar] (dt in the last column, or dt [B]).
    start_yaw [B, 3], end_yaw [B].  Returns a list of dicts: dt_yaw, relax_num (None without lookfwd), waypts (list),
    waypt_idx (list), end_yaw (after calcNextYaw), start (the wrapped start_yaw3d), guess [15], pt_dist, status, and
    margin: the least | |diff| - pi | over the calcNextYaw calls, where atan2's last bits can flip the branch.
    Rows the device refuses (dt not finite and positive, non-finite yaws, |start yaw| > 1000) get status BAD_INPUT."""
    x = np.ascontiguousarray(x, dtype=np.float64)
    B = x.shape[0]
    dts = x[:, 3 * n_pts] if dt is None else np.broadcast_to(np.asarray(dt, dtype=np.float64), (B,))
    sy = np.broadcast_to(np.asarray(start_yaw, dtype=np.float64), (B, 3))
    ey = np.broadcast_to(np.asarray(end_yaw, dtype=np.float64), (B,))
    rows = []
    t = np.zeros((B, 2 * MAX_WAYPT))
    for b in range(B):
        d = float(dts[b])
        r = dict(dt_yaw=math.nan, relax_num=None, waypts=[], waypt_idx=[], status=OK, pt_dist=math.nan, margin=math.inf)
        bad = not (0.0 < d <= 1.7976931348623157e308) or not all(math.isfinite(v) for v in sy[b]) or \
            not math.isfinite(ey[b]) or abs(sy[b][0]) > 1000.0
        if not bad:
            dur = duration(d, n_pts)
            dt_yaw = dur / SEG_NUM
            bad = not (0.0 < dt_yaw <= 1.7976931348623157e308)
        if bad:
            r["status"] = BAD_INPUT
            rows.append(r)
            continue
        r.update(dt_yaw=dt_yaw, duration=dur)
        nw = 0
        if lookfwd:
            q = relax_time / dt_yaw
            if q >= 2147483648.0:  # (int) of it is undefined
                r["status"] = RELAX_OVERFLOW
            else:
                r["relax_num"] = int(q)
                nw = max(0, SEG_NUM - r["relax_num"] - 1)
        r["nw"] = nw
        for i in range(1, nw + 1):
            tc = i * dt_yaw
            tf = min(dur, tc + FORWARD_T)
            t[b, i - 1], t[b, MAX_WAYPT + i - 1] = tc, tf
        rows.append(r)
    pts = _traj.bspline_evaluate(x, n_pts, t, dt=None if dt is None else np.asarray(dts, dtype=np.float64))
    for b, r in enumerate(rows):
        if r["status"] != OK:
            continue
        y3 = [wrap_start(float(sy[b][0])), float(sy[b][1]), float(sy[b][2])]
        r["start"] = y3
        last_yaw = y3[0]
        for i in range(1, r["nw"] + 1):
            pc, pf = pts[b, i - 1], pts[b, MAX_WAYPT + i - 1]
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
        r["margin"] = min(r["margin"], abs(abs(next_yaw_diff(last_yaw, float(ey[b]))) - math.pi))
        r["end_in"] = float(ey[b])
        _finish(r)
    return rows


def _finish(r):
    """the end yaw through calcNextYaw from the last waypoint, the initial guess and pt_dist_ (:821-824, optimize())"""
    last_yaw = r["waypts"][-1] if r["waypts"] else r["start"][0]
    r["end_yaw"] = calc_next_yaw(last_yaw, r["end_in"])
    r["guess"] = initial_guess(r["dt_yaw"], r["start"], r["end_yaw"])
    r["pt_dist"] = pt_dist(r["guess"])
    if r["pt_dist"] == 0.0:
        r["status"] = ZERO_PT_DIST


def with_waypoints(r, waypts):
    """row r of plan() rebuilt from other waypoints (e.g. the device's, whose atan2 may differ from the C library's in the
    last bits): the same waypt_idx, then the end yaw, initial guess and pt_dist_ by the reference's arithmetic"""
    assert len(waypts) == len(r["waypts"])
    out = dict(r)
    out["waypts"] = [float(w) for w in waypts]
    _finish(out)
    return out


def terms(r, ld_smooth=20.0, ld_start=100.0, ld_end=0.5, ld_waypt=0.3, num=float):
    """The objective of optimize(yaw, dt_yaw, SMOOTHNESS | START | END | WAYPOINTS) as a list of (offset, a, w, t):
    sum of w * (a . q[offset:offset + len(a)] - t)^2.  `num` converts each float (Fraction for an exact solve)."""
    dt, p = num(r["dt_yaw"]), num(r["pt_dist"])
    y0, y1, y2 = (num(v) for v in r["start"])
    ye = num(r["end_yaw"])
    six = num(6)
    out = [(i, (-1, 3, -3, 1), num(ld_smooth) / (p * p), num(0)) for i in range(PTS - 3)]
    out += [(0, (1, 4, 1), num(ld_start) * 10 / 36, six * y0), (0, (-1, 0, 1), num(ld_start) / (4 * dt * dt), 2 * dt * y1),
            (0, (1, -2, 1), num(ld_start) / (dt * dt * dt * dt), dt * dt * y2),
            (SEG_NUM, (1, 4, 1), num(ld_end) / 36, six * ye), (SEG_NUM, (-1, 0, 1), num(ld_end) / (4 * dt * dt), num(0))]
    out += [(i, (1, 4, 1), num(ld_waypt) / 36, six * num(w)) for i, w in zip(r["waypt_idx"], r["waypts"])]
    return out


def normal_equations(r, num=float, **ld):
    """H q = rhs at the minimizer (Hessian and gradient at 0, both halved) -> (H [15][15], rhs [15]) as lists"""
    H = [[num(0)] * PTS for _ in range(PTS)]
    rhs = [num(0)] * PTS
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


def objective(rows, q, ld_smooth=20.0, ld_start=100.0, ld_end=0.5, ld_waypt=0.3):
    """combineCost(q) and its gradient for the yaw objective of each row (rows from plan(), q [B, 15]), evaluated by the
    oracle's pinned 3-D combineCost on q padded with zero y and z columns -> (f [B], grad [B, 15])"""
    from . import combine_cost_batch, fill_traj_const, make_grid, opt_params, traj_consts
    q = np.asarray(q, dtype=np.float64).reshape(len(rows), PTS)
    B = len(rows)
    tcs = traj_consts(B)
    for b, r in enumerate(rows):
        s = r["start"]
        wp = [(w, 0.0, 0.0) for w in r["waypts"]] or None
        fill_traj_const(tcs[b], r["pt_dist"], r["dt_yaw"], [(s[0], 0, 0), (s[1], 0, 0), (s[2], 0, 0)],
                        [(r["end_yaw"], 0, 0), (0, 0, 0)], waypt=wp, waypt_idx=r["waypt_idx"] or None)
    x = np.zeros((B, 3 * PTS))
    x[:, 0::3] = q
    g = make_grid((4, 4, 4), 0.1, (0, 0, 0))
    p = opt_params(ld_smooth=ld_smooth, ld_start=ld_start, ld_end=ld_end, ld_waypt=ld_waypt)
    f, grad = combine_cost_batch(g, np.zeros(64), p, tcs, PTS, YAW_MASK, x)
    return f, grad[:, 0::3]


# ---- the reference's own code ------------------------------------------------------------------------------------------
def ref_yaw():
    """oracle/_ref/libfuel_ref_yaw.so (the reference's non_uniform_bspline.cpp + ref_yaw_wrap.cpp, and
    ref_yaw_cost_wrap.cpp over _ref/libfuel_ref.so's BsplineOptimizer), or None where it is not built."""
    return _load("_ref/libfuel_ref_yaw.so", dict(ref_yaw_explore=C.c_int32, ref_yaw_cost=C.c_int32), first=ref_raycast)


def ref_plan(ctrl, dt, start_yaw, end_yaw, relax_time=1.0, lookfwd=True):
    """the reference's lines :776-824 over its compiled NonUniformBspline, for one trajectory ctrl [n, 3] ->
    dict(dt_yaw, relax_num, waypts, waypt_idx, end_yaw, start, guess, pt_dist)"""
    ctrl = np.ascontiguousarray(ctrl, dtype=np.float64)
    sy = np.ascontiguousarray(start_yaw, dtype=np.float64)
    od = np.zeros(4)  # dt_yaw, end_yaw after calcNextYaw, pt_dist_, start_yaw3d[0] wrapped
    oi = np.zeros(2, dtype=np.int32)  # relax_num, waypoint count
    wp, widx, guess = np.zeros(MAX_WAYPT), np.zeros(MAX_WAYPT, dtype=np.int32), np.zeros(PTS)
    ref_yaw().ref_yaw_explore(C.c_int32(ctrl.shape[0]), _p(ctrl), C.c_double(dt), _p(sy), C.c_double(end_yaw),
                              C.c_int32(1 if lookfwd else 0), C.c_double(relax_time), _p(od), _p(oi), _p(wp), _p(widx),
                              _p(guess))
    k = int(oi[1])
    return dict(dt_yaw=od[0], relax_num=int(oi[0]) if lookfwd else None, waypts=wp[:k].tolist(),
                waypt_idx=widx[:k].tolist(), end_yaw=od[1], start=[od[3], float(sy[1]), float(sy[2])],
                guess=guess.tolist(), pt_dist=od[2])


def ref_cost(ref_map, r, probes, ld_smooth=20.0, ld_start=100.0, ld_end=0.5, ld_waypt=0.3):
    """the REFERENCE's optimize(yaw [15 x 1], dt_yaw, SMOOTHNESS | START | END | WAYPOINTS, 1, 1) with the boundary states
    and waypoints of planYawExplore (row r of plan()): combineCost at its initial guess and at probes [K, 15] ->
    (f [1 + K], grad [1 + K, 15])"""
    keys = [b"optimization/" + k.encode() for k in ("ld_smooth", "ld_start", "ld_end", "ld_waypt")]
    karr = (C.c_char_p * 4)(*keys)
    vals = np.array([ld_smooth, ld_start, ld_end, ld_waypt], dtype=np.float64)
    probes = np.ascontiguousarray(probes, dtype=np.float64).reshape(-1, PTS)
    K = probes.shape[0]
    f, grad = np.zeros(1 + K), np.zeros((1 + K, PTS))
    s = r["start"]
    start = np.array([s[0], s[1], s[2]], dtype=np.float64)
    wp = np.ascontiguousarray(r["waypts"], dtype=np.float64)
    widx = np.ascontiguousarray(r["waypt_idx"], dtype=np.int32)
    rc = ref_yaw().ref_yaw_cost(ref_map.h, C.c_int32(4), karr, _p(vals), _p(np.ascontiguousarray(r["guess"])),
                                C.c_double(r["dt_yaw"]), _p(start), C.c_double(r["end_yaw"]), C.c_int32(len(wp)), _p(wp),
                                _p(widx), C.c_int32(K), _p(probes), _p(f), _p(grad))
    assert rc == 0, rc
    return f, grad
