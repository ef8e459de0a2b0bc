"""ctypes binding of the A* oracle (oracle/fuel_oracle_astar.c: Astar::search, shortenPath and planExploreMotion's goal
branch) and of the reference's own path_searching/src/astar2.cpp run through oracle/ref_astar_wrap.cpp
(oracle/_ref/libfuel_ref_astar.so, built by oracle/astar.mk where the reference's sources are present).

TEST INFRASTRUCTURE ONLY, like the rest of this package: fuel_b200/ must never import it.
"""
import ctypes as C

import numpy as np

from . import _load, _make, _p, ref_raycast

# the layout of FuelPathInfo (include/fuelgpu.h)
INFO_DTYPE = np.dtype([("status", np.int32), ("reason", np.int32), ("iter_num", np.int32), ("use_node_num", np.int32),
                       ("n_path", np.int32), ("n_wp", np.int32), ("branch", np.int32), ("tour_status", np.int32),
                       ("early_terminate_cost", np.float64), ("length", np.float64), ("next_goal", np.float64, (3,))])


class OrcAstarMap(C.Structure):
    _fields_ = [("n", C.c_int32 * 3), ("res", C.c_double), ("res_inv", C.c_double), ("origin", C.c_double * 3),
                ("box_mind", C.c_double * 3), ("box_maxd", C.c_double * 3), ("occ", C.c_void_p)]


def build():
    """Compile this part with oracle/astar.mk."""
    _make("astar.mk")


def lib():
    return _load("libfuel_oracle_astar.so", dict(orc_astar=C.c_int32), build=build)


def ref_astar():
    """The REFERENCE's astar2.cpp + oracle/ref_astar_wrap.cpp over libfuel_ref.so's SDFMap and RayCaster, or None where
    it is not built."""
    return _load("_ref/libfuel_ref_astar.so", dict(ref_astar_create=C.c_void_p), first=ref_raycast)


def occ_byte(inflate, tri):
    """the device's occupancy byte: bits 0-1 tri-state, bit 2 inflate"""
    return np.ascontiguousarray((np.asarray(tri, np.uint8) & 3) | (np.asarray(inflate, np.uint8).astype(np.uint8) << 2))


class Map:
    """the map geometry and occupancy byte the oracle searches (the same as the device's FuelMap)"""

    def __init__(self, g, inflate, tri, box_mind=None, box_maxd=None):
        self.occ = occ_byte(inflate, tri).reshape(-1)
        self.s = OrcAstarMap()
        for k in range(3):
            self.s.n[k] = int(g.n[k])
            self.s.origin[k] = float(g.origin[k])
            self.s.box_mind[k] = float((g.box_min if box_mind is None else box_mind)[k])
            self.s.box_maxd[k] = float((g.box_max if box_maxd is None else box_maxd)[k])
        self.s.res = float(g.res)
        self.s.res_inv = 1 / float(g.res)
        self.s.occ = self.occ.ctypes.data


def search_batch(m, start, goal, resolution, lambda_heu, allocate_num, max_iter, path_max=512, w_max=32):
    """the oracle over B queries -> (info [B] of INFO_DTYPE, path [B, path_max, 3], n_wp [B], waypts [B, w_max, 3]),
    in the layout of fuelgpu_astar_batch"""
    start = np.ascontiguousarray(np.asarray(start, np.float64).reshape(-1, 3))
    goal = np.ascontiguousarray(np.asarray(goal, np.float64).reshape(-1, 3))
    B = len(start)
    info = np.zeros(B, INFO_DTYPE)
    path = np.zeros((B, path_max, 3))
    wp = np.zeros((B, w_max, 3))
    n_wp = np.zeros(B, np.int32)
    L = lib()
    for b in range(B):
        r = L.orc_astar(C.byref(m.s), _p(start[b]), _p(goal[b]), C.c_double(resolution), C.c_double(lambda_heu),
                        C.c_int32(allocate_num), C.c_int32(max_iter), C.c_int32(w_max), _p(info[b:b + 1]),
                        C.c_int32(path_max), _p(path[b]), _p(wp[b]))
        assert r >= 0, "orc_astar: out of memory"
        n_wp[b] = r
    return info, path, n_wp, wp


class RefAstar:
    """The reference's Astar (astar2.cpp compiled unmodified) on the reference's SDFMap `ref_map` (an oracle.RefSDFMap
    whose buffers hold the map), with shortenPath and the branch restated over its RayCaster (oracle/ref_astar_wrap.cpp).
    max_iter stands for max_search_time_: the stand-in clock ticks one second per ros::Time::now()."""

    def __init__(self, ref_map, resolution, lambda_heu, allocate_num, max_iter):
        R = ref_astar()
        self.R = R
        self.h = C.c_void_p(R.ref_astar_create(ref_map.h, C.c_double(resolution), C.c_double(lambda_heu),
                                               C.c_int32(allocate_num), C.c_double(float(max_iter))))

    def close(self):
        if self.h:
            self.R.ref_astar_destroy(self.h)
            self.h = None

    def search_batch(self, start, goal, path_max=512, w_max=32):
        start = np.ascontiguousarray(np.asarray(start, np.float64).reshape(-1, 3))
        goal = np.ascontiguousarray(np.asarray(goal, np.float64).reshape(-1, 3))
        B = len(start)
        info = np.zeros(B, INFO_DTYPE)
        path = np.zeros((B, path_max, 3))
        wp = np.zeros((B, w_max, 3))
        n_wp = np.zeros(B, np.int32)
        for b in range(B):
            n_wp[b] = self.R.ref_astar_run(self.h, _p(start[b]), _p(goal[b]), C.c_int32(w_max), _p(info[b:b + 1]),
                                           C.c_int32(path_max), _p(path[b]), _p(wp[b]))
        return info, path, n_wp, wp
