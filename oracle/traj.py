"""ctypes binding of the trajectory-check oracle (oracle/fuel_oracle_traj.c: NonUniformBspline for uniform cubic
splines, checkTrajCollision, selectBestTraj) and of the reference's own non_uniform_bspline.cpp
(oracle/_ref/libfuel_ref_traj.so, built by oracle/traj.mk where the reference's sources are present).

TEST INFRASTRUCTURE ONLY, like the rest of this package: fuel_b200/ must never import it.
"""
import ctypes as C

import numpy as np

from . import _load, _make, _p, ref_raycast
from . import build as _build_oracle


def build():
    """Compile the oracle (libfuel_oracle.so first, oracle/Makefile) and this part of it with oracle/traj.mk."""
    _build_oracle()
    _make("traj.mk")


class OrcTrajCheckParams(C.Structure):
    _fields_ = [("max_vel", C.c_double), ("max_acc", C.c_double), ("t_now", C.c_double)]


TRAJ_REPORT_DTYPE = np.dtype([("duration", np.float64), ("jerk", np.float64), ("ratio", np.float64),
                              ("distance", np.float64), ("safe", np.int32), ("feasible", np.int32),
                              ("n_checked", np.int32), ("reserved", np.int32)])


def lib():
    return _load("libfuel_oracle_traj.so", {}, build=build)


def ref_traj():
    """The REFERENCE's non_uniform_bspline.cpp + oracle/ref_traj_wrap.cpp, or None where it is not built."""
    return _load("_ref/libfuel_ref_traj.so", dict(ref_traj_check_collision=C.c_int32, ref_traj_select_best=C.c_int32),
                 first=ref_raycast)


def _traj_inputs(x, n_pts, dt):
    x = np.ascontiguousarray(x, dtype=np.float64)
    if dt is not None:
        dt = np.ascontiguousarray(dt, dtype=np.float64)
    assert x.shape[1] == 3 * n_pts + (0 if dt is not None else 1)
    return x, dt


def bspline_evaluate(x, n_pts, t, deriv=0, dt=None):
    """evaluateDeBoorT of B uniform cubic splines (x [B, nvar] in the solver layout; dt [B] when x has no dt column)
    or of their first / second derivative, at t [B, n_t] -> [B, n_t, 3]"""
    x, dt = _traj_inputs(x, n_pts, dt)
    t = np.ascontiguousarray(t, dtype=np.float64)
    B, n_t = t.shape
    out = np.zeros((B, n_t, 3))
    lib().orc_bspline_evaluate(C.c_int32(B), C.c_int32(n_pts), C.c_int32(x.shape[1]), _p(x), _p(dt), C.c_int32(n_t),
                               _p(t), C.c_int32(deriv), _p(out))
    return out


def bspline_check(g, inflate, x, n_pts, max_vel, max_acc, t_now=0.0, dt=None):
    """duration / jerk / ratio / feasibility / checkTrajCollision per trajectory -> (report [B] TRAJ_REPORT_DTYPE,
    best [2]: selectBestTraj, and the same among safe && feasible)"""
    x, dt = _traj_inputs(x, n_pts, dt)
    inflate = np.ascontiguousarray(inflate, dtype=np.int8)
    B = x.shape[0]
    rep = np.zeros(B, TRAJ_REPORT_DTYPE)
    best = np.zeros(2, np.int32)
    p = OrcTrajCheckParams(max_vel, max_acc, t_now)
    lib().orc_bspline_check(C.byref(g), _p(inflate), C.c_int32(B), C.c_int32(n_pts), C.c_int32(x.shape[1]), _p(x), _p(dt),
                            C.byref(p), _p(rep), _p(best))
    return rep, best


def ref_traj_evaluate(ctrl, dt, t, deriv=0):
    """the REFERENCE's evaluateDeBoorT after `deriv` getDerivative() calls: ctrl [n, 3], t [n_t] -> [n_t, 3]"""
    ctrl = np.ascontiguousarray(ctrl, dtype=np.float64)
    t = np.ascontiguousarray(t, dtype=np.float64)
    out = np.zeros((t.shape[0], 3))
    ref_traj().ref_traj_evaluate(C.c_int32(ctrl.shape[0]), _p(ctrl), C.c_double(dt), C.c_int32(deriv),
                                 C.c_int32(t.shape[0]), _p(t), _p(out))
    return out


def ref_traj_stats(ctrl, dt, max_vel, max_acc):
    """the REFERENCE's (getTimeSum, getJerk, checkRatio, checkFeasibility) after setPhysicalLimits"""
    ctrl = np.ascontiguousarray(ctrl, dtype=np.float64)
    out = np.zeros(3)
    fea = C.c_int32()
    ref_traj().ref_traj_stats(C.c_int32(ctrl.shape[0]), _p(ctrl), C.c_double(dt), C.c_double(max_vel),
                              C.c_double(max_acc), _p(out), C.byref(fea))
    return out[0], out[1], out[2], fea.value


def ref_traj_check_collision(ref_map, ctrl, dt, t_now=0.0):
    """the REFERENCE's checkTrajCollision loop on its SDFMap (oracle.RefSDFMap) -> (safe, distance or -1, samples)"""
    ctrl = np.ascontiguousarray(ctrl, dtype=np.float64)
    dist = C.c_double(-1.0)
    n = C.c_int32()
    safe = ref_traj().ref_traj_check_collision(ref_map.h, C.c_int32(ctrl.shape[0]), _p(ctrl), C.c_double(dt),
                                               C.c_double(t_now), C.byref(dist), C.byref(n))
    return int(safe), dist.value, n.value


def ref_traj_select_best(ctrl, dt):
    """the REFERENCE's selectBestTraj: the index std::sort by getJerk puts first (ctrl [B, n, 3], dt [B])"""
    ctrl = np.ascontiguousarray(ctrl, dtype=np.float64)
    dt = np.ascontiguousarray(dt, dtype=np.float64)
    return int(ref_traj().ref_traj_select_best(C.c_int32(ctrl.shape[0]), C.c_int32(ctrl.shape[1]), _p(ctrl), _p(dt)))
