"""NonUniformBspline (bspline/src/non_uniform_bspline.cpp) for the uniform cubic splines the planner flies, and
FastPlannerManager's checkTrajCollision / selectBestTraj (plan_manage/src/planner_manager.cpp:96-118, 476-482), over
fuelgpu_bspline_check_batch / fuelgpu_bspline_evaluate_batch.  Every value is the reference's fp64 result bit for bit.
parameterize_batch / NonUniformBspline.parameterizeToBspline build the solver's batch from sampled paths
(fuelgpu_bspline_parameterize_batch); their control points come from this project's own least-squares solve.

Batches use the solver's layout: x [B, nvar] with control point i at x[b, 3i:3i+3]; nvar == 3*n_pts + 1 carries the
knot span in the last column (what BsplineOptimizer.optimizeBatch returns with MINTIME), nvar == 3*n_pts takes dt [B].
"""
import ctypes as C

import numpy as np

from ._lib import FuelTrajCheckParams, FuelTrajConst, check, lib, ptr

# one FuelTrajReport per trajectory (include/fuelgpu.h)
REPORT_DTYPE = np.dtype([("duration", np.float64), ("jerk", np.float64), ("ratio", np.float64),
                         ("distance", np.float64), ("safe", np.int32), ("feasible", np.int32),
                         ("n_checked", np.int32), ("reserved", np.int32)])


def _handle(sdf_map):
    return getattr(sdf_map, "handle", sdf_map)


def _inputs(x, n_pts, dt):
    x = np.ascontiguousarray(x, dtype=np.float64)
    if x.ndim == 1:
        x = x[None, :]
    B = x.shape[0]
    if dt is None:
        if x.shape[1] != 3 * n_pts + 1:
            raise ValueError("x must be [B, %d] (dt in the last column) when dt is not given" % (3 * n_pts + 1))
    else:
        if x.shape[1] != 3 * n_pts:
            raise ValueError("x must be [B, %d] when dt is given" % (3 * n_pts))
        dt = np.ascontiguousarray(np.broadcast_to(np.asarray(dt, dtype=np.float64), (B,)))
    return x, dt


def evaluate_batch(sdf_map, x, n_pts, t, deriv=0, dt=None):
    """evaluateDeBoorT (:73-75) of every spline (deriv 0) or of its getDerivative() once / twice (deriv 1, 2) at
    t [B, n_t] (one row of times per trajectory; clamped to [0, duration]) -> [B, n_t, 3]"""
    x, dt = _inputs(x, n_pts, dt)
    B = x.shape[0]
    t = np.ascontiguousarray(np.broadcast_to(np.asarray(t, dtype=np.float64), (B, np.shape(t)[-1])))
    out = np.empty((B, t.shape[1], 3), dtype=np.float64)
    h = _handle(sdf_map)
    check(lib().fuelgpu_bspline_evaluate_batch(h, B, n_pts, x.shape[1], ptr(x), ptr(dt), t.shape[1], ptr(t), int(deriv),
                                               ptr(out)), h)
    return out


def check_batch(sdf_map, x, n_pts, dt=None, *, max_vel, max_acc, t_now=0.0):
    """getTimeSum, getJerk, checkRatio, checkFeasibility (after setPhysicalLimits(max_vel, max_acc)) and
    checkTrajCollision at t_now for every trajectory, on the map's resident occupancy.
    Returns (report [B] of REPORT_DTYPE, best [2]): best[0] = selectBestTraj's pick (least jerk, lowest index on ties),
    best[1] = the same among trajectories that are safe and feasible, -1 if there is none."""
    x, dt = _inputs(x, n_pts, dt)
    B = x.shape[0]
    rep = np.empty(B, dtype=REPORT_DTYPE)
    best = np.empty(2, dtype=np.int32)
    p = FuelTrajCheckParams(float(max_vel), float(max_acc), float(t_now))
    h = _handle(sdf_map)
    check(lib().fuelgpu_bspline_check_batch(h, B, n_pts, x.shape[1], ptr(x), ptr(dt), C.byref(p), ptr(rep), ptr(best)), h)
    return rep, best


def parameterize_batch(sdf_map, points, derivs, dt, time_lb=None, mintime=True):
    """parameterizeToBspline (:178-265, degree 3) of B sampled paths, the getBoundaryStates(2, 0) of the result
    (:108-123) and the pt_dist_ optimize() freezes (bspline_optimizer.cpp:136-140), on the device of `sdf_map`
    (fuelgpu_bspline_parameterize_batch).
    points [B, K, 3] (point_set), derivs [B, 4, 3] (start vel, end vel, start acc, end acc), dt scalar or [B],
    time_lb scalar or [B] (None: -1).  Returns (x [B, 3(K+2) (+1 dt column when mintime)], traj_consts: a ctypes array
    of FuelTrajConst), ready for BsplineOptimizer.optimizeBatch and check_batch."""
    points = np.ascontiguousarray(points, dtype=np.float64)
    derivs = np.ascontiguousarray(derivs, dtype=np.float64)
    if points.ndim != 3 or points.shape[2] != 3:
        raise ValueError("points must be [B, K, 3]")
    B, K = points.shape[:2]
    if derivs.shape != (B, 4, 3):
        raise ValueError("derivs must be [B, 4, 3]")
    dt = np.ascontiguousarray(np.broadcast_to(np.asarray(dt, dtype=np.float64), (B,)))
    if time_lb is not None:
        time_lb = np.ascontiguousarray(np.broadcast_to(np.asarray(time_lb, dtype=np.float64), (B,)))
    n = K + 2
    x = np.empty((B, 3 * n + (1 if mintime else 0)), dtype=np.float64)
    tc = (FuelTrajConst * B)()
    h = _handle(sdf_map)
    check(lib().fuelgpu_bspline_parameterize_batch(h, B, n, x.shape[1], ptr(points), ptr(derivs), ptr(dt), ptr(time_lb),
                                                   ptr(x), tc), h)
    return x, tc


class NonUniformBspline:
    """The reference's class for one uniform cubic spline (setUniformBspline(points, 3, interval), :16-32), evaluated on
    the device of `sdf_map`.  getDerivative() may be applied twice (velocity, acceleration)."""

    def __init__(self, points, order, interval, sdf_map, _deriv=0):
        if order != 3:
            raise ValueError("only degree 3 (bspline_degree_ = 3 in every launch file) is supported")
        self.control_points_ = np.ascontiguousarray(points, dtype=np.float64).reshape(-1, 3)
        self.p_ = order
        self.knot_span_ = float(interval)
        self.sdf_map_ = sdf_map
        self._deriv = _deriv
        self.limit_vel_ = self.limit_acc_ = None

    @property
    def n_pts(self):
        return self.control_points_.shape[0]

    def _x(self):
        return np.concatenate([self.control_points_.reshape(-1), [self.knot_span_]])[None, :]

    def evaluateDeBoorT(self, t):
        return evaluate_batch(self.sdf_map_, self._x(), self.n_pts, [[float(t)]], self._deriv)[0, 0]

    def getDerivative(self):
        if self._deriv >= 2:
            raise ValueError("evaluation is offered up to the second derivative")
        d = NonUniformBspline(self.control_points_, 3, self.knot_span_, self.sdf_map_, self._deriv + 1)
        d.limit_vel_, d.limit_acc_ = self.limit_vel_, self.limit_acc_
        return d

    @staticmethod
    def parameterizeToBspline(ts, point_set, start_end_derivative, degree, sdf_map):
        """parameterizeToBspline (:178-265) of one sampled path: point_set [K, 3], start_end_derivative [4, 3] (start
        vel, end vel, start acc, end acc) -> ctrl_pts [K+2, 3]; row b of parameterize_batch"""
        if degree != 3:
            raise ValueError("only degree 3 (bspline_degree_ = 3 in every launch file) is supported")
        pts = np.asarray(point_set, dtype=np.float64).reshape(1, -1, 3)
        der = np.asarray(start_end_derivative, dtype=np.float64).reshape(1, 4, 3)
        x, _ = parameterize_batch(sdf_map, pts, der, ts, mintime=False)
        return x[0].reshape(-1, 3)

    def setPhysicalLimits(self, vel, acc):
        self.limit_vel_, self.limit_acc_ = float(vel), float(acc)

    def _report(self, t_now=0.0):
        if self._deriv:
            raise ValueError("the checks are offered on the position spline")
        vel = 1.0 if self.limit_vel_ is None else self.limit_vel_
        acc = 1.0 if self.limit_acc_ is None else self.limit_acc_
        return check_batch(self.sdf_map_, self._x(), self.n_pts, max_vel=vel, max_acc=acc, t_now=t_now)[0][0]

    def getTimeSum(self):
        return float(self._report()["duration"])

    def getJerk(self):
        return float(self._report()["jerk"])

    def checkRatio(self):
        self._need_limits()
        return float(self._report()["ratio"])

    def checkFeasibility(self, show=False):
        self._need_limits()
        return bool(self._report()["feasible"])

    def _need_limits(self):
        if self.limit_vel_ is None:
            raise ValueError("call setPhysicalLimits first")


def checkTrajCollision(sdf_map, traj, t_now=0.0):
    """FastPlannerManager::checkTrajCollision (planner_manager.cpp:96-118) for one NonUniformBspline and the seconds
    since its start: returns (safe, distance); distance is the radius reached before the hit, -1 when safe."""
    rep = check_batch(sdf_map, traj._x(), traj.n_pts, max_vel=1.0, max_acc=1.0, t_now=t_now)[0][0]
    return bool(rep["safe"]), float(rep["distance"])


def selectBestTraj(sdf_map, trajs):
    """FastPlannerManager::selectBestTraj (planner_manager.cpp:476-482): the trajectory of least jerk (the lowest index
    among equals).  trajs: NonUniformBspline objects of one point count."""
    n = trajs[0].n_pts
    if any(t.n_pts != n for t in trajs):
        raise ValueError("all trajectories must have the same number of control points")
    x = np.concatenate([t._x() for t in trajs], axis=0)
    _, best = check_batch(sdf_map, x, n, max_vel=1.0, max_acc=1.0)
    return trajs[best[0]] if best[0] >= 0 else None
