"""ctypes binding of the kinodynamic-search oracle (oracle/fuel_oracle_kino.c: kinodynamicReplan's search, retry and
getSamples, in the reference's glibc arithmetic or in the device's) and of the host build of the device's math header
(fuel_b200/csrc/kino_math.cuh), both in oracle/libfuel_oracle_kino.so built by oracle/kino.mk.

TEST INFRASTRUCTURE ONLY, like the rest of this package: fuel_b200/ must never import it.
"""
import ctypes as C

import numpy as np

from . import _load, _make, _p, ref_raycast
GLIBC, DEVICE = 0, 1
MAX_PTS = 64

# the layout of FuelKinoInfo (include/fuelgpu.h)
INFO_DTYPE = np.dtype([("status", np.int32), ("reason", np.int32), ("retried", np.int32), ("traj_status", np.int32),
                       ("iter_num", np.int32), ("use_node_num", np.int32), ("n_nodes", np.int32), ("shot", np.int32),
                       ("seg_num", np.int32), ("n_pts", np.int32), ("t_shot", np.float64), ("T_sum", np.float64)])

MATH_CBRT, MATH_CUBE, MATH_ACOS, MATH_COS, MATH_LIBM_CBRT = 0, 1, 2, 3, 4


def build():
    """Compile this part with oracle/kino.mk."""
    _make("kino.mk")


def lib():
    return _load("libfuel_oracle_kino.so", dict(orc_kino_replan=C.c_int32, orc_kino_three_root_count=C.c_longlong),
                 build=build)


def three_root_count(reset=True):
    """heuristic evaluations of the oracle that took cubic()'s D < 0 branch since the last reset"""
    return int(lib().orc_kino_three_root_count(C.c_int32(1 if reset else 0)))


def ref_kino():
    """The REFERENCE's kinodynamic_astar.cpp + oracle/ref_kino_wrap.cpp over libfuel_ref.so's SDFMap, or None where it
    is not built."""
    return _load("_ref/libfuel_ref_kino.so", dict(ref_kino_create=C.c_void_p), first=ref_raycast)


class RefKino:
    """The reference's KinodynamicAstar (compiled unmodified) on the reference's SDFMap `ref_map` (an oracle.RefSDFMap
    holding the map), driven through kinodynamicReplan's lines 131-164 (oracle/ref_kino_wrap.cpp)."""

    def __init__(self, ref_map, params):
        R = ref_kino()
        self.R = R
        d = np.array([params.max_tau, params.init_max_tau, params.max_vel, params.vel_margin, params.max_acc,
                      params.w_time, params.horizon, params.lambda_heu, params.resolution, params.ctrl_pt_dist,
                      params.manager_max_vel], dtype=np.float64)
        i = np.array([params.allocate_num, params.check_num, params.optimistic], dtype=np.int32)
        self.h = C.c_void_p(R.ref_kino_create(ref_map.h, _p(d), _p(i)))

    def close(self):
        if self.h:
            self.R.ref_kino_destroy(self.h)
            self.h = None

    def replan_batch(self, start, vel, acc, goal, node_max=0):
        rows = [np.ascontiguousarray(np.asarray(a, np.float64).reshape(-1, 3)) for a in (start, vel, acc, goal)]
        B = len(rows[0])
        info = np.zeros(B, INFO_DTYPE)
        points = np.zeros((B, MAX_PTS - 2, 3))
        derivs = np.zeros((B, 4, 3))
        dt = np.zeros(B)
        nodes = np.zeros((B, node_max, 12)) if node_max > 0 else None
        shot = np.zeros((B, 3, 4))
        for b in range(B):
            self.R.ref_kino_run(self.h, _p(rows[0][b]), _p(rows[1][b]), _p(rows[2][b]), _p(rows[3][b]),
                                _p(info[b:b + 1]), _p(points[b]), _p(derivs[b]), _p(dt[b:b + 1]), C.c_int32(node_max),
                                _p(nodes[b]) if nodes is not None else None, _p(shot[b]))
        return dict(info=info, points=points, derivs=derivs, dt=dt, nodes=nodes, shot=shot)


def math(f, x):
    """kino_math.cuh's function f (MATH_*) on the host, or libm's cbrt"""
    x = np.ascontiguousarray(x, dtype=np.float64)
    out = np.empty_like(x)
    lib().orc_kino_math(C.c_int32(f), C.c_int64(x.size), _p(x), _p(out))
    return out


def replan_batch(m, map_size, params, start, vel, acc, goal, math=DEVICE, node_max=0):
    """the oracle over B queries on oracle.astar.Map m -> the dict of fuel_b200.kino_astar.kino_search_batch.
    params: a fuel_b200._lib.FuelKinoParams (the oracle's struct has the same layout)."""
    rows = [np.ascontiguousarray(np.asarray(a, np.float64).reshape(-1, 3)) for a in (start, vel, acc, goal)]
    B = len(rows[0])
    size = np.ascontiguousarray(map_size, dtype=np.float64)
    info = np.zeros(B, INFO_DTYPE)
    points = np.zeros((B, MAX_PTS - 2, 3))
    derivs = np.zeros((B, 4, 3))
    dt = np.zeros(B)
    nodes = np.zeros((B, node_max, 12)) if node_max > 0 else None
    shot = np.zeros((B, 3, 4))
    L = lib()
    for b in range(B):
        r = L.orc_kino_replan(C.byref(m.s), _p(size), C.byref(params), C.c_int32(math), _p(rows[0][b]),
                              _p(rows[1][b]), _p(rows[2][b]), _p(rows[3][b]), _p(info[b:b + 1]), _p(points[b]),
                              _p(derivs[b]), _p(dt[b:b + 1]), C.c_int32(node_max),
                              _p(nodes[b]) if nodes is not None else None, _p(shot[b]))
        assert r == 0, "orc_kino_replan: out of memory"
    return dict(info=info, points=points, derivs=derivs, dt=dt, nodes=nodes, shot=shot)
