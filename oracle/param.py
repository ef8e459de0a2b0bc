"""ctypes binding of the parameterization oracle (oracle/fuel_oracle_param.c: parameterizeToBspline for degree 3,
getBoundaryStates(2, 0), pt_dist_) and of the reference's own non_uniform_bspline.cpp run through
oracle/ref_param_wrap.cpp (oracle/_ref/libfuel_ref_param.so, built by oracle/param.mk where the reference's sources are
present).

TEST INFRASTRUCTURE ONLY, like the rest of this package: fuel_b200/ must never import it.
"""
import ctypes as C

import numpy as np

from . import OrcTrajConst, _load, _make, _p
from . import traj as _traj


def build():
    """Compile the trajectory oracle first (oracle/traj.py), then this part with oracle/param.mk."""
    _traj.build()
    _make("param.mk")


def lib():
    return _load("libfuel_oracle_param.so", dict(orc_lstsq_colpiv_qr=C.c_int32), build=build)


def ref_param():
    """The REFERENCE's non_uniform_bspline.cpp + oracle/ref_param_wrap.cpp, or None where it is not built.  The
    stand-in's solve binds to lib()'s orc_lstsq_colpiv_qr."""
    return _load("_ref/libfuel_ref_param.so", dict(ref_param_parameterize=C.c_int32), first=lib)


def param_system(points, derivs, ts):
    """parameterizeToBspline's system (degree 3) as the oracle builds it: points [K, 3], derivs [4, 3] ->
    (A [K+4, K+2], b [3, K+4])"""
    points = np.ascontiguousarray(points, dtype=np.float64)
    derivs = np.ascontiguousarray(derivs, dtype=np.float64)
    K = points.shape[0]
    A = np.zeros((K + 4, K + 2))
    b = np.zeros((3, K + 4))
    lib().orc_bspline_param_system(C.c_int32(K), C.c_double(ts), _p(points), _p(derivs), _p(A), _p(b))
    return A, b


def lstsq_colpiv_qr(A, b):
    """the oracle's column-pivoted Householder least-squares solve (parity unpinned): A [rows, cols], b [nrhs, rows] ->
    (x [nrhs, cols], rank)"""
    A = np.ascontiguousarray(A, dtype=np.float64)
    b = np.ascontiguousarray(np.atleast_2d(b), dtype=np.float64)
    x = np.zeros((b.shape[0], A.shape[1]))
    rank = lib().orc_lstsq_colpiv_qr(C.c_int32(A.shape[0]), C.c_int32(A.shape[1]), _p(A), C.c_int32(b.shape[0]), _p(b),
                                     _p(x))
    return x, int(rank)


def bspline_boundary_states(x, n_pts, dt=None):
    """getBoundaryStates(2, 0) of B splines in the solver's layout (x [B, nvar]; dt [B] when x has no dt column) ->
    (start [B, 3, 3], end [B, 3])"""
    x = np.ascontiguousarray(x, dtype=np.float64)
    if dt is not None:
        dt = np.ascontiguousarray(dt, dtype=np.float64)
    assert x.shape[1] == 3 * n_pts + (0 if dt is not None else 1)
    B = x.shape[0]
    start, end = np.zeros((B, 3, 3)), np.zeros((B, 3))
    lib().orc_bspline_boundary_states(C.c_int32(B), C.c_int32(n_pts), C.c_int32(x.shape[1]), _p(x), _p(dt), _p(start),
                                      _p(end))
    return start, end


def bspline_parameterize(points, derivs, dt, time_lb=None, mintime=True):
    """parameterizeToBspline + what optimize() freezes, for B trajectories: points [B, K, 3], derivs [B, 4, 3], dt [B]
    -> (x [B, 3(K+2) (+1)], tc: ctypes array of oracle.OrcTrajConst)"""
    points = np.ascontiguousarray(points, dtype=np.float64)
    derivs = np.ascontiguousarray(derivs, dtype=np.float64)
    B, K = points.shape[:2]
    dt = np.ascontiguousarray(np.broadcast_to(np.asarray(dt, dtype=np.float64), (B,)))
    if time_lb is not None:
        time_lb = np.ascontiguousarray(np.broadcast_to(np.asarray(time_lb, dtype=np.float64), (B,)))
    n = K + 2
    nvar = 3 * n + (1 if mintime else 0)
    x = np.zeros((B, nvar))
    tc = (OrcTrajConst * B)()
    lib().orc_bspline_parameterize(C.c_int32(B), C.c_int32(n), C.c_int32(nvar), _p(points), _p(derivs), _p(dt),
                                   _p(time_lb), _p(x), tc)
    return x, tc


def ref_parameterize(points, derivs, ts):
    """the REFERENCE's parameterizeToBspline (degree 3) -> (ctrl [K+2, 3], A [K+4, K+2], b [3, K+4]) with A and b as
    its own code built them (its solve is the oracle's, through the Eigen stand-in)"""
    points = np.ascontiguousarray(points, dtype=np.float64)
    derivs = np.ascontiguousarray(derivs, dtype=np.float64)
    K = points.shape[0]
    ctrl = np.zeros((K + 2, 3))
    A = np.zeros((K + 4, K + 2))
    b = np.zeros((3, K + 4))
    n_solves = ref_param().ref_param_parameterize(C.c_double(ts), C.c_int32(K), _p(points), _p(derivs), _p(ctrl), _p(A),
                                                  _p(b))
    assert n_solves == 3
    return ctrl, A, b


def ref_boundary_states(ctrl, dt):
    """the REFERENCE's getBoundaryStates(2, 0) of setUniformBspline(ctrl, 3, dt) -> (start [3, 3], end [3])"""
    ctrl = np.ascontiguousarray(ctrl, dtype=np.float64)
    start, end = np.zeros((3, 3)), np.zeros(3)
    ref_param().ref_param_boundary_states(C.c_int32(ctrl.shape[0]), _p(ctrl), C.c_double(dt), _p(start), _p(end))
    return start, end
