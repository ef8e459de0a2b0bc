"""ctypes binding of the waypoint-polynomial oracle (oracle/fuel_oracle_poly.c: waypointsTraj, evaluate, getTotalTime,
getLength, planExploreTraj's sampling) and of the reference's own polynomial_traj.cpp run through oracle/ref_poly_wrap.cpp
(oracle/_ref/libfuel_ref_poly.so, built by oracle/poly.mk where the reference's sources are present).

TEST INFRASTRUCTURE ONLY, like the rest of this package: fuel_b200/ must never import it.
"""
import ctypes as C

import numpy as np

from . import _load, _make, _p

MAX_K = 62  # FUELGPU_MAX_PTS - 2


def build():
    """Compile this part with oracle/poly.mk."""
    _make("poly.mk")


def lib():
    return _load("libfuel_oracle_poly.so", dict(orc_lu_inverse=C.c_int32, orc_poly_waypoints=C.c_int32,
                                                orc_explore_samples=C.c_int32, orc_poly_total_time=C.c_double,
                                                orc_poly_length=C.c_double), build=build)


def ref_poly():
    """The REFERENCE's polynomial_traj.cpp + oracle/ref_poly_wrap.cpp, or None where it is not built.  The stand-in's
    inverse() binds to lib()'s orc_lu_inverse."""
    return _load("_ref/libfuel_ref_poly.so", {}, first=lib)


def _v(a, n=None):
    return np.ascontiguousarray(np.zeros(3) if a is None else a, dtype=np.float64)


def lu_inverse(M):
    M = np.ascontiguousarray(M, dtype=np.float64)
    out = np.zeros_like(M)
    assert lib().orc_lu_inverse(C.c_int32(M.shape[0]), _p(M), _p(out)) == 0
    return out


def waypoints(waypts, start_vel, start_acc, times, end_vel=None, end_acc=None, matrices=False):
    """the oracle's waypointsTraj -> coeffs [S, 3, 6] (and with matrices=True, (coeffs, A, Q, Ct, D))"""
    w = np.ascontiguousarray(waypts, dtype=np.float64)
    t = np.ascontiguousarray(times, dtype=np.float64)
    S = len(t)
    c = np.zeros((S, 3, 6))
    mats = [np.zeros((6 * S, 6 * S)), np.zeros((6 * S, 6 * S)), np.zeros((6 * S, 4 * S + 2)), np.zeros((3, 6 * S))]
    rc = lib().orc_poly_waypoints(C.c_int32(S), _p(w), _p(_v(start_vel)), _p(_v(end_vel)), _p(_v(start_acc)),
                                  _p(_v(end_acc)), _p(t), _p(c), *[_p(m) if matrices else None for m in mats])
    if rc != 0:
        raise ValueError("orc_poly_waypoints: %d" % rc)
    return (c, *mats) if matrices else c


def evaluate(coeffs, times, t, k):
    coeffs = np.ascontiguousarray(coeffs, dtype=np.float64)
    times = np.ascontiguousarray(times, dtype=np.float64)
    out = np.zeros(3)
    lib().orc_poly_evaluate(C.c_int32(len(times)), _p(coeffs), _p(times), C.c_double(t), C.c_int32(k), _p(out))
    return out


def total_time(times):
    times = np.ascontiguousarray(times, dtype=np.float64)
    return lib().orc_poly_total_time(C.c_int32(len(times)), _p(times))


def length(coeffs, times):
    coeffs = np.ascontiguousarray(coeffs, dtype=np.float64)
    times = np.ascontiguousarray(times, dtype=np.float64)
    return lib().orc_poly_length(C.c_int32(len(times)), _p(coeffs), _p(times), None)


def explore_samples(tour, cur_vel, cur_acc, max_vel=2.0, ctrl_pt_dist=0.35, min_seg_num=8, ref=False):
    """planExploreTraj :270-297 for one tour, the oracle's (ref=False) or the reference's compiled PolynomialTraj
    (ref=True) -> dict(times, points [K, 3] (at most 62 rows), derivs [4, 3], duration, length, dt, seg_num, K)"""
    w = np.ascontiguousarray(tour, dtype=np.float64)
    W = len(w)
    times, pts, der = np.zeros(W - 1), np.zeros((MAX_K, 3)), np.zeros((4, 3))
    od, oi = np.zeros(3), np.zeros(2, dtype=np.int32)
    args = (C.c_int32(W), _p(w), _p(_v(cur_vel)), _p(_v(cur_acc)), C.c_double(max_vel), C.c_double(ctrl_pt_dist),
            C.c_int32(min_seg_num), C.c_int32(MAX_K))
    if ref:
        ref_poly().ref_poly_explore(*args, _p(times), _p(pts), _p(der), _p(od), _p(oi))
    else:
        assert lib().orc_explore_samples(*args, _p(times), None, _p(pts), _p(der), _p(od), _p(oi)) == 0
    K = int(oi[1])
    return dict(times=times, points=pts[:min(K, MAX_K)].copy(), derivs=der, duration=od[0], length=od[1], dt=od[2],
                seg_num=int(oi[0]), K=K)


def ref_waypoints(waypts, start_vel, start_acc, times, end_vel=None, end_acc=None):
    """the REFERENCE's waypointsTraj -> (coeffs [S, 3, 6], A, Q, Ct, D) as its own code built them"""
    w = np.ascontiguousarray(waypts, dtype=np.float64)
    t = np.ascontiguousarray(times, dtype=np.float64)
    S = len(t)
    c = np.zeros((S, 3, 6))
    A, Q, Ct, D = np.zeros((6 * S, 6 * S)), np.zeros((6 * S, 6 * S)), np.zeros((6 * S, 4 * S + 2)), np.zeros((3, 6 * S))
    ref_poly().ref_poly_waypoints(C.c_int32(S), _p(w), _p(_v(start_vel)), _p(_v(end_vel)), _p(_v(start_acc)),
                                  _p(_v(end_acc)), _p(t), _p(c), _p(A), _p(Q), _p(Ct), _p(D))
    return c, A, Q, Ct, D


def ref_query(waypts, start_vel, start_acc, times, t, k, end_vel=None, end_acc=None):
    """the REFERENCE's getTotalTime, getLength and evaluate(t[i], k) -> (total_time, length, out [n_t, 3])"""
    w = np.ascontiguousarray(waypts, dtype=np.float64)
    tm = np.ascontiguousarray(times, dtype=np.float64)
    t = np.ascontiguousarray(np.atleast_1d(t), dtype=np.float64)
    out = np.zeros((len(t), 3))
    tt, ln = C.c_double(), C.c_double()
    ref_poly().ref_poly_query(C.c_int32(len(tm)), _p(w), _p(_v(start_vel)), _p(_v(end_vel)), _p(_v(start_acc)),
                              _p(_v(end_acc)), _p(tm), C.c_int32(len(t)), _p(t), C.c_int32(k), _p(out), C.byref(tt),
                              C.byref(ln))
    return tt.value, ln.value, out
