"""ctypes binding of the global-tour oracle (oracle/fuel_oracle_gtour.c: Held-Karp over the integer ATSP that
FastExplorationManager::findGlobalTour hands to LKH) and of the reference's own findGlobalTour with its real LKH, run
through oracle/ref_gtour_wrap.cpp (oracle/_ref/libfuel_ref_gtour.so), both built by oracle/gtour.mk, the reference
library where the reference's sources are present.  The map is the reference's SDFMap (oracle.RefSDFMap).

TEST INFRASTRUCTURE ONLY, like the rest of this package: fuel_b200/ must never import it.
"""
import ctypes as C

import numpy as np

from . import _load, _make, _p, ref_raycast

GTOUR_OK, GTOUR_BAD_INPUT, GTOUR_TOO_LARGE = 0, 1, 2
GTOUR_MAX_CLUSTERS = 20
# the layout of FuelGlobalTourInfo (include/fuelgpu.h)
GTOUR_DTYPE = np.dtype([("status", np.int32), ("n", np.int32), ("n_optimal", np.int32), ("reserved", np.int32),
                        ("cost", np.int64)])


def build():
    """Compile this part with oracle/gtour.mk."""
    _make("gtour.mk")


def lib():
    return _load("libfuel_oracle_gtour.so", dict(orc_global_tour=C.c_int32), build=build)


def int_matrix(mat):
    """findGlobalTour's integer matrix: int(cost * 100), truncated toward zero (:357-376); [d, d] int64"""
    p = np.asarray(mat, np.float64) * 100.0
    with np.errstate(invalid="ignore"):
        return np.trunc(p).astype(np.int64)


def tour_cost(c, indices):
    """LKH's objective on the integer matrix c: c[0][t1] + c[t1][t2] + ... + c[tn][0]"""
    nodes = [0] + [int(i) + 1 for i in indices] + [0]
    return int(sum(int(c[a, b]) for a, b in zip(nodes[:-1], nodes[1:])))


def global_tour(mat):
    """one instance -> (status, cost, n_optimal, indices [n] or None)"""
    mat = np.ascontiguousarray(mat, np.float64)
    d = mat.shape[0]
    cost, nopt = C.c_int64(), C.c_int32()
    idx = np.zeros(max(d - 1, 1), np.int32)
    st = lib().orc_global_tour(C.c_int32(d), _p(mat), C.byref(cost), C.byref(nopt), _p(idx))
    assert st >= 0, "orc_global_tour: out of memory or no cluster"
    if st != GTOUR_OK:
        return st, 0, 0, None
    return st, cost.value, nopt.value, idx[:d - 1].copy()


def global_tour_batch(dims, cost):
    """B instances in the layout of fuelgpu_global_tour_batch -> (info [B] of GTOUR_DTYPE, indices [sum(dims - 1)],
    -1 where the status is not OK)"""
    dims = np.asarray(dims, np.int64).reshape(-1)
    cost = np.asarray(cost, np.float64).reshape(-1)
    info = np.zeros(len(dims), GTOUR_DTYPE)
    indices = np.full(int(dims.sum()) - len(dims), -1, np.int32)
    co = io = 0
    for b, d in enumerate(dims):
        d = int(d)
        n = d - 1
        st, c, nopt, idx = global_tour(cost[co:co + d * d].reshape(d, d)) if n <= GTOUR_MAX_CLUSTERS else \
            (GTOUR_TOO_LARGE, 0, 0, None)
        info[b] = (st, n, nopt, 0, c)
        if idx is not None:
            indices[io:io + n] = idx
        co += d * d
        io += n
    return info, indices


def ref_gtour():
    """The REFERENCE's fast_exploration_manager.cpp + frontier_finder.cpp + LKH + oracle/ref_gtour_wrap.cpp over
    libfuel_ref.so's SDFMap and RayCaster, or None where it is not built."""
    return _load("_ref/libfuel_ref_gtour.so", dict(ref_gtour_setup=C.c_int32, ref_gtour_find=C.c_int32),
                 first=ref_raycast)


def _f64(a, shape=(-1,)):
    return np.ascontiguousarray(np.asarray(a, np.float64).reshape(shape))


class RefGTour:
    """The reference's ViewNode statics on the reference's SDFMap `ref_map`, a FrontierFinder and a
    FastExplorationManager whose tsp_dir_ is a fresh temporary directory with single.par; max_iter stands for
    max_search_time_ on the tick clock.  One at a time: they are statics."""

    def __init__(self, ref_map, vm, yd, w_dir, lambda_heu, allocate_num, max_iter):
        self.R = ref_gtour()
        assert self.R.ref_gtour_setup(ref_map.h, C.c_double(vm), C.c_double(yd), C.c_double(w_dir),
                                      C.c_double(lambda_heu), C.c_int32(allocate_num), C.c_double(float(max_iter))) == 0

    def close(self):
        self.R.ref_gtour_teardown()

    def find(self, vp_pos, vp_yaw, costs, paths, cur_pos, cur_vel, cur_yaw, tour_max=65536):
        """frontiers_ = one cluster per viewpoint with its costs_ row and paths_ (paths[i][j]: [k, 3]), then
        findGlobalTour -> (indices [n], global_tour [k, 3], getFullCostMatrix's matrix [n + 1, n + 1])"""
        n = len(vp_yaw)
        pn = np.ascontiguousarray([[len(p) for p in row] for row in paths], np.int32)
        flat = [np.asarray(p, np.float64).reshape(-1, 3) for row in paths for p in row]
        pts = _f64(np.concatenate(flat) if flat else np.zeros((0, 3)), (-1, 3))
        idx = np.full(n, -1, np.int32)
        nt = C.c_int32()
        tour = np.zeros((tour_max, 3))
        mat = np.zeros((n + 1, n + 1))
        k = self.R.ref_gtour_find(C.c_int32(n), _p(_f64(vp_pos, (-1, 3))), _p(_f64(vp_yaw)), _p(_f64(costs, (-1,))),
                                  _p(pn), _p(pts if len(pts) else np.zeros((1, 3))), _p(_f64(cur_pos)),
                                  _p(_f64(cur_vel)), _p(_f64(cur_yaw)), _p(idx), C.c_int32(tour_max), C.byref(nt),
                                  _p(tour), _p(mat))
        assert k == n and nt.value <= tour_max
        return idx.tolist(), tour[:nt.value].copy(), mat

    def path(self, cur_pos, ids, tour_max=65536):
        """getPathForTour over the list of the last find for the given cluster ids -> [k, 3]"""
        ids = np.ascontiguousarray(ids, np.int32)
        nt = C.c_int32()
        tour = np.zeros((tour_max, 3))
        self.R.ref_gtour_path(_p(_f64(cur_pos)), C.c_int32(len(ids)), _p(ids), C.c_int32(tour_max), C.byref(nt),
                              _p(tour))
        return tour[:nt.value].copy()
