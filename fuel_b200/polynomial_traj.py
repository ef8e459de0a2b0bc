"""PolynomialTraj (poly_traj/include/poly_traj/polynomial_traj.h, poly_traj/src/polynomial_traj.cpp) for the minimum-jerk
tours the exploration planner flies, and FastPlannerManager::planExploreTraj (plan_manage/src/planner_manager.cpp:266-316)
for B candidate tours, over fuelgpu_poly_waypoints_batch and the existing parameterize / optimize / check entries.

waypoints_batch runs the polynomial stage: segment times, waypointsTraj, getTotalTime, getLength, seg_num, dt, and the
samples and boundary derivatives parameterizeToBspline takes.  plan_explore_traj_batch chains it with
parameterize_batch -> BsplineOptimizer.optimizeBatch -> check_batch, one launch per point count.
plan_yaw_explore_batch is planYawExplore (:774-865) on every trajectory of a solver batch (fuelgpu_yaw_explore_batch).
plan_yaw_batch is planYaw (:695-772), the kinodynamic replan's yaw, on every trajectory of a solver batch
(fuelgpu_plan_yaw_batch).
"""
import ctypes as C

import numpy as np

from ._lib import FuelOptParams, FuelPolyParams, FuelYawParams, check, lib, ptr
from .non_uniform_bspline import REPORT_DTYPE, _handle, _inputs, check_batch, parameterize_batch

MAX_WAYPTS = 32  # FUELGPU_MAX_WAYPTS
MAX_PTS = 64     # FUELGPU_MAX_PTS
OK, TOO_LONG, BAD_INPUT = 0, 1, 2  # FuelPolyInfo.status
YAW_SEG_NUM, YAW_PTS, YAW_MAX_WAYPT = 12, 15, 11  # FUELGPU_YAW_SEG_NUM, _PTS, _MAX_WAYPT
# FuelYawInfo.status
YAW_OK, YAW_BAD_INPUT, YAW_RELAX_OVERFLOW, YAW_NO_LOOKAHEAD, YAW_ZERO_PT_DIST, YAW_NOT_SPD = 0, 1, 2, 3, 4, 5
YAW_INFO_DTYPE = np.dtype([("dt_yaw", np.float64), ("pt_dist", np.float64), ("n_waypt", np.int32),
                           ("status", np.int32)])
PLANYAW_MAX_SEG, PLANYAW_MAX_PTS = 128, 131  # FUELGPU_PLANYAW_MAX_SEG, _MAX_PTS
YAW_TOO_LONG = 6  # FUELGPU_YAW_TOO_LONG (plan_yaw_batch only)
PLANYAW_INFO_DTYPE = np.dtype([("dt_yaw", np.float64), ("pt_dist", np.float64), ("seg_num", np.int32),
                               ("n_waypt", np.int32), ("status", np.int32), ("reserved", np.int32)])

# one FuelPolyInfo per tour (include/fuelgpu.h)
INFO_DTYPE = np.dtype([("duration", np.float64), ("length", np.float64), ("dt", np.float64), ("seg_num", np.int32),
                       ("n_pts", np.int32), ("status", np.int32), ("reserved", np.int32)])


def _pack(tours, B, name):
    if tours is None:
        return None
    a = np.ascontiguousarray(np.broadcast_to(np.asarray(tours, dtype=np.float64), (B, 3)))
    if a.shape != (B, 3):
        raise ValueError("%s must be [B, 3]" % name)
    return a


def waypoints_batch(sdf_map, tours, start_vel, start_acc, end_vel=None, end_acc=None, times=None, *, max_vel=2.0,
                    ctrl_pt_dist=0.35, min_seg_num=8, with_coeffs=True):
    """planExploreTraj's lines 270-297 for B tours on the device of `sdf_map` (fuelgpu_poly_waypoints_batch).
    tours: a list of [W_b, 3] arrays (3 <= W_b <= 32); start_vel / start_acc / end_vel / end_acc: [3] or [B, 3] (end
    None: zero); times: None (|dp| / (max_vel * 0.5)) or a list of [W_b - 1] arrays.
    Returns (info [B] of INFO_DTYPE, coeffs [B, w_max - 1, 3, 6] or None, points [B, 62, 3], derivs [B, 4, 3]):
    points[b, :info['n_pts'][b] - 2] are the samples, derivs[b] = start vel, end vel, start acc, end acc."""
    tours = [np.asarray(t, dtype=np.float64).reshape(-1, 3) for t in tours]
    B = len(tours)
    n_wp = np.array([len(t) for t in tours], dtype=np.int32)
    w_max = max(3, int(n_wp.max()) if B else 3)
    wp = np.zeros((B, w_max, 3))
    for b, t in enumerate(tours):
        wp[b, :len(t)] = t
    tm = None
    if times is not None:
        tm = np.zeros((B, w_max - 1))
        for b, t in enumerate(times):
            t = np.asarray(t, dtype=np.float64).ravel()
            tm[b, :len(t)] = t
    sv, sa = _pack(start_vel, B, "start_vel"), _pack(start_acc, B, "start_acc")
    ev, ea = _pack(end_vel, B, "end_vel"), _pack(end_acc, B, "end_acc")
    prm = FuelPolyParams(float(max_vel), float(ctrl_pt_dist), int(min_seg_num), 0)
    info = np.empty(B, dtype=INFO_DTYPE)
    coeffs = np.empty((B, w_max - 1, 3, 6)) if with_coeffs else None
    points = np.empty((B, MAX_PTS - 2, 3))
    derivs = np.empty((B, 4, 3))
    h = _handle(sdf_map)
    check(lib().fuelgpu_poly_waypoints_batch(h, B, w_max, ptr(n_wp), ptr(wp), ptr(sv), ptr(sa), ptr(ev), ptr(ea),
                                             ptr(tm), C.byref(prm), ptr(info), ptr(coeffs), ptr(points), ptr(derivs)), h)
    return info, coeffs, points, derivs


class PolynomialTraj:
    """The reference's class for one trajectory, its coefficients solved on the device of `sdf_map`.  evaluate() runs on
    the host with the reference's segment search and Polynomial::evaluate (pow and a written-order dot)."""

    def __init__(self, sdf_map):
        self.sdf_map = sdf_map
        self.reset()

    def reset(self):
        self.coeffs_ = np.zeros((0, 3, 6))
        self.times_ = np.zeros(0)
        self.info_ = None

    @staticmethod
    def waypointsTraj(positions, start_vel, end_vel, start_acc, end_acc, times, poly_traj):
        """waypointsTraj (polynomial_traj.cpp:5-175), the reference's argument order: positions [W, 3], times [W - 1]"""
        positions = np.asarray(positions, dtype=np.float64).reshape(-1, 3)
        times = np.asarray(times, dtype=np.float64).ravel()
        info, coeffs, _, _ = waypoints_batch(poly_traj.sdf_map, [positions], start_vel, start_acc, end_vel, end_acc,
                                             [times])
        S = len(positions) - 1
        poly_traj.coeffs_ = coeffs[0, :S].copy()
        poly_traj.times_ = times.copy()
        poly_traj.info_ = info[0]

    def getTotalTime(self):
        s = 0.0
        for t in self.times_:
            s += float(t)
        return s

    def evaluate(self, t, k):
        """PolynomialTraj::evaluate(t, k) (polynomial_traj.h:83-91)"""
        idx, ts = 0, float(t)
        while idx < len(self.times_) - 1 and self.times_[idx] + 1e-4 < ts:
            ts -= self.times_[idx]
            idx += 1
        tv = np.zeros(6)
        for i in range(k, 6):
            coeff = 1
            for j in range(i, i - k, -1):
                coeff *= j
            tv[i] = coeff * ts ** (i - k)
        out = np.empty(3)
        for j in range(3):
            v = tv[0] * self.coeffs_[idx, j, 0]
            for i in range(1, 6):
                v = v + tv[i] * self.coeffs_[idx, j, i]
            out[j] = v
        return out

    def getLength(self):
        """getLength (polynomial_traj.h:107-124), as the device computed it in waypointsTraj"""
        return float(self.info_["length"])


def plan_yaw_explore_batch(sdf_map, x, n_pts, start_yaw, end_yaw, opt_params, relax_time=1.0, lookfwd=True, dt=None):
    """planYawExplore(start_yaw, end_yaw, lookfwd, relax_time) (planner_manager.cpp:774-865) with every trajectory of a
    batch as the position trajectory, on the device of `sdf_map` (fuelgpu_yaw_explore_batch).
    x: [B, nvar] in the solver's layout (dt in the last column, or dt [B] given); start_yaw: [3] or [B, 3] (yaw, yawdot,
    yawddot); end_yaw: scalar or [B]; opt_params: a FuelOptParams or a BsplineOptimizer (ld_smooth, ld_start, ld_end and
    ld_waypt are read).
    Returns (yaw [B, 15] control points of the yaw spline with knot span info['dt_yaw'], info [B] of YAW_INFO_DTYPE,
    waypt [B, 11]: the look-ahead waypoints, zero past info['n_waypt']).  A trajectory with info['status'] != 0 has NaN
    yaw (include/fuelgpu.h lists the statuses)."""
    x, dt = _inputs(x, n_pts, dt)
    B = x.shape[0]
    sy = np.ascontiguousarray(np.broadcast_to(np.asarray(start_yaw, dtype=np.float64), (B, 3)))
    ey = np.ascontiguousarray(np.broadcast_to(np.asarray(end_yaw, dtype=np.float64), (B,)))
    prm = opt_params if isinstance(opt_params, FuelOptParams) else opt_params.params_
    yp = FuelYawParams(float(relax_time), 1 if lookfwd else 0, 0)
    yaw = np.empty((B, YAW_PTS))
    info = np.empty(B, dtype=YAW_INFO_DTYPE)
    waypt = np.empty((B, YAW_MAX_WAYPT))
    h = _handle(sdf_map)
    check(lib().fuelgpu_yaw_explore_batch(h, B, n_pts, x.shape[1], ptr(x), ptr(dt), ptr(sy), ptr(ey), C.byref(prm),
                                          C.byref(yp), ptr(yaw), ptr(info), ptr(waypt)), h)
    return yaw, info, waypt


def plan_yaw_batch(sdf_map, x, n_pts, start_yaw, opt_params, dt=None):
    """planYaw(start_yaw) (planner_manager.cpp:695-772) with every trajectory of a batch as the position trajectory, on
    the device of `sdf_map` (fuelgpu_plan_yaw_batch).
    x: [B, nvar] in the solver's layout (dt in the last column, or dt [B] given); start_yaw: [3] or [B, 3] (yaw, yawdot,
    yawddot; the yaw is used as given); opt_params: a FuelOptParams or a BsplineOptimizer (ld_smooth, ld_start, ld_end and
    ld_waypt are read).
    Returns (yaw [B, 131]: the seg_num + 3 control points of the yaw spline with knot span info['dt_yaw'], NaN after them,
    info [B] of PLANYAW_INFO_DTYPE, waypt [B, 128]: plan_data_.path_yaw_, zero past info['n_waypt']).  A trajectory with
    info['status'] != 0 has NaN yaw (include/fuelgpu.h lists the statuses)."""
    x, dt = _inputs(x, n_pts, dt)
    B = x.shape[0]
    sy = np.ascontiguousarray(np.broadcast_to(np.asarray(start_yaw, dtype=np.float64), (B, 3)))
    prm = opt_params if isinstance(opt_params, FuelOptParams) else opt_params.params_
    yaw = np.empty((B, PLANYAW_MAX_PTS))
    info = np.empty(B, dtype=PLANYAW_INFO_DTYPE)
    waypt = np.empty((B, PLANYAW_MAX_SEG))
    h = _handle(sdf_map)
    check(lib().fuelgpu_plan_yaw_batch(h, B, n_pts, x.shape[1], ptr(x), ptr(dt), ptr(sy), C.byref(prm), ptr(yaw),
                                       ptr(info), ptr(waypt)), h)
    return yaw, info, waypt


def plan_explore_traj_batch(sdf_map, tours, cur_vel, cur_acc, time_lb, opt, solve, limits, *, ctrl_pt_dist=0.35,
                            min_seg_num=8, start_yaw=None, end_yaw=None, relax_time=1.0):
    """planExploreTraj (planner_manager.cpp:266-316) for B candidate tours, then selectBestTraj (:476-482) over them.
    opt: a BsplineOptimizer set up on `sdf_map` (its cost_function with or without MINTIME); solve: keyword arguments of
    optimizeBatch besides x / traj_consts / n_pts (cost_function, max_eval, ...); limits: dict(max_vel=, max_acc=), the
    pp_.max_vel_ that also sets the segment times.
    The polynomial stage runs first; its info (B x 40 bytes) is read back, because the solver takes one point count per
    launch.  Each group of equal n_pts then runs parameterize -> optimize -> check.  Tours with status != 0 are left
    out and keep NaN reports.
    Returns dict(info, x: a list of [nvar] arrays or None per tour, report [B] of REPORT_DTYPE, best [2]): best[0] =
    least jerk (lowest index on ties, NaN never wins), best[1] = the same among safe and feasible tours, -1 if none.
    With start_yaw ([3] or [B, 3]) and end_yaw (scalar or [B]) given, each group also runs planYawExplore on its solver
    output (plan_yaw_explore_batch with lookfwd and relax_time), and the dict gains yaw [B, 15] and yaw_info [B] of
    YAW_INFO_DTYPE (NaN and status -1 for tours left out)."""
    B = len(tours)
    with_yaw = start_yaw is not None or end_yaw is not None
    if with_yaw:
        if start_yaw is None or end_yaw is None:
            raise ValueError("start_yaw and end_yaw go together")
        sy = np.broadcast_to(np.asarray(start_yaw, dtype=np.float64), (B, 3))
        ey = np.broadcast_to(np.asarray(end_yaw, dtype=np.float64), (B,))
        yaw = np.full((B, YAW_PTS), np.nan)
        yaw_info = np.zeros(B, dtype=YAW_INFO_DTYPE)
        yaw_info["dt_yaw"] = yaw_info["pt_dist"] = np.nan
        yaw_info["status"] = -1
    info, _, points, derivs = waypoints_batch(sdf_map, tours, cur_vel, cur_acc, max_vel=limits["max_vel"],
                                              ctrl_pt_dist=ctrl_pt_dist, min_seg_num=min_seg_num, with_coeffs=False)
    mask = int(solve["cost_function"])
    mintime = bool(mask & opt.MINTIME)
    tlb = np.broadcast_to(np.asarray(time_lb, dtype=np.float64), (B,))
    report = np.zeros(B, dtype=REPORT_DTYPE)
    for f in ("duration", "jerk", "ratio", "distance"):
        report[f] = np.nan
    xs = [None] * B
    ok = info["status"] == OK
    for n in sorted(set(info["n_pts"][ok].tolist())):
        idx = np.flatnonzero(ok & (info["n_pts"] == n))
        K = n - 2
        x0, tc = parameterize_batch(sdf_map, points[idx, :K], derivs[idx], info["dt"][idx], time_lb=tlb[idx],
                                    mintime=mintime)
        kw = {k: v for k, v in solve.items() if k != "cost_function"}
        x, _, _ = opt.optimizeBatch(x0, tc, n, mask, **kw)
        dt = None if mintime else info["dt"][idx]
        rep, _ = check_batch(sdf_map, x, n, dt, max_vel=limits["max_vel"], max_acc=limits["max_acc"])
        report[idx] = rep
        for r, b in enumerate(idx):
            xs[b] = x[r].copy()
        if with_yaw:
            yaw[idx], yaw_info[idx], _ = plan_yaw_explore_batch(sdf_map, x, n, sy[idx], ey[idx], opt.params_,
                                                                relax_time=relax_time, dt=dt)
    out = dict(info=info, x=xs, report=report, best=select_best(report))
    if with_yaw:
        out.update(yaw=yaw, yaw_info=yaw_info)
    return out


def select_best(report):
    """selectBestTraj's rule over merged reports: least jerk, lowest index on ties, NaN never wins; [1] among the safe
    and feasible, -1 if none"""
    best = [-1, -1]
    for i, r in enumerate(report):
        j = r["jerk"]
        if not j == j:
            continue
        for s, ok in ((0, True), (1, bool(r["safe"]) and bool(r["feasible"]))):
            if ok and (best[s] < 0 or j < report[best[s]]["jerk"]):
                best[s] = i
    return np.array(best, dtype=np.int32)
