"""ctypes binding of the view-cost oracle (oracle/fuel_oracle_view.c: ViewNode::searchPath and computeCost over the A*
oracle) and of the reference's own active_perception/src/graph_node.cpp and frontier_finder.cpp cost bookkeeping run
through oracle/ref_view_wrap.cpp (oracle/_ref/libfuel_ref_view.so), both built by oracle/view.mk, the reference library
where the reference's sources are present.  The map is oracle.astar.Map.

TEST INFRASTRUCTURE ONLY, like the rest of this package: fuel_b200/ must never import it.
"""
import ctypes as C

import numpy as np

from . import _load, _make, _p, ref_raycast

# the layout of FuelViewCostInfo (include/fuelgpu.h)
VIEW_DTYPE = np.dtype([("kind", np.int32), ("reason", np.int32), ("iter_num", np.int32), ("use_node_num", np.int32),
                       ("n_path", np.int32), ("reserved", np.int32), ("length", np.float64), ("cost", np.float64)])


def build():
    """Compile this part with oracle/view.mk."""
    _make("view.mk")


def lib():
    return _load("libfuel_oracle_view.so", dict(orc_view_cost=C.c_int32), build=build)


def view_cost_batch(m, p1, p2, y1, y2, v1, vm, yd, w_dir, resolution, lambda_heu, allocate_num, max_iter, path_max=512):
    """ViewNode::computeCost over P pairs on the oracle (m: an oracle.astar.Map) -> (info [P] of VIEW_DTYPE, path [P, path_max, 3]), in the layout
    of fuelgpu_view_cost_batch"""
    p1, p2, v1 = (np.ascontiguousarray(np.asarray(a, np.float64).reshape(-1, 3)) for a in (p1, p2, v1))
    y1, y2 = (np.ascontiguousarray(np.asarray(a, np.float64).reshape(-1)) for a in (y1, y2))
    P = len(p1)
    info = np.zeros(P, VIEW_DTYPE)
    path = np.zeros((P, path_max, 3))
    L = lib()
    for q in range(P):
        r = L.orc_view_cost(C.byref(m.s), _p(p1[q]), _p(p2[q]), C.c_double(y1[q]), C.c_double(y2[q]), _p(v1[q]),
                            C.c_double(vm), C.c_double(yd), C.c_double(w_dir), C.c_double(resolution),
                            C.c_double(lambda_heu), C.c_int32(allocate_num), C.c_int32(max_iter), _p(info[q:q + 1]),
                            C.c_int32(path_max), _p(path[q]))
        assert r == 0, "orc_view_cost: out of memory"
    return info, path


def ref_view():
    """The REFERENCE's graph_node.cpp + frontier_finder.cpp + oracle/ref_view_wrap.cpp over libfuel_ref.so's SDFMap and
    RayCaster, or None where it is not built."""
    return _load("_ref/libfuel_ref_view.so", dict(ref_ffc_create=C.c_void_p, ref_ffc_tour=C.c_int32), first=ref_raycast)


class RefViewNode:
    """The reference's ViewNode statics (vm_, yd_, w_dir_, astar_ at resolution 0.4, caster_, map_) on the reference's
    SDFMap `ref_map`; max_iter stands for max_search_time_ on the tick clock.  One at a time: they are statics."""

    def __init__(self, ref_map, vm, yd, w_dir, lambda_heu, allocate_num, max_iter):
        self.R = ref_view()
        self.R.ref_view_setup(ref_map.h, C.c_double(vm), C.c_double(yd), C.c_double(w_dir), C.c_double(lambda_heu),
                              C.c_int32(allocate_num), C.c_double(float(max_iter)))

    def close(self):
        self.R.ref_view_teardown()

    def cost_batch(self, p1, p2, y1, y2, v1, path_max=512):
        p1, p2, v1 = (np.ascontiguousarray(np.asarray(a, np.float64).reshape(-1, 3)) for a in (p1, p2, v1))
        y1, y2 = (np.asarray(a, np.float64).reshape(-1) for a in (y1, y2))
        P = len(p1)
        info = np.zeros(P, VIEW_DTYPE)
        path = np.zeros((P, path_max, 3))
        for q in range(P):
            self.R.ref_view_cost(_p(p1[q]), _p(p2[q]), C.c_double(y1[q]), C.c_double(y2[q]), _p(v1[q]),
                                 _p(info[q:q + 1]), C.c_int32(path_max), _p(path[q]))
        return info, path


class RefCostBook:
    """The reference's FrontierFinder holding an installed frontier list (one viewpoint each, cost and path lists,
    first_new_ftr_, removed_ids_), for updateFrontierCostMatrix / getFullCostMatrix / getPathForTour.  Needs a
    RefViewNode alive on the same map."""

    def __init__(self, ref_map):
        self.R = ref_view()
        self.h = C.c_void_p(self.R.ref_ffc_create(ref_map.h))

    def close(self):
        if self.h:
            self.R.ref_ffc_destroy(self.h)
            self.h = None

    def install(self, frontiers, first_new, removed_ids):
        """frontiers: objects with viewpoints_ [(pos, yaw, ...)], costs_ and paths_ lists"""
        n = len(frontiers)
        pos = np.ascontiguousarray([f.viewpoints_[0][0] for f in frontiers], np.float64).reshape(-1, 3)
        yaw = np.ascontiguousarray([f.viewpoints_[0][1] for f in frontiers], np.float64)
        ncost = np.ascontiguousarray([len(f.costs_) for f in frontiers], np.int32)
        costs = np.ascontiguousarray([c for f in frontiers for c in f.costs_], np.float64)
        paths = [np.asarray(p, np.float64).reshape(-1, 3) for f in frontiers for p in f.paths_]
        rows = np.ascontiguousarray([len(p) for p in paths], np.int32)
        pts = np.ascontiguousarray(np.concatenate(paths) if paths else np.zeros((0, 3)))
        rem = np.ascontiguousarray(removed_ids, np.int32)
        self.R.ref_ffc_install(self.h, n, _p(pos), _p(yaw), _p(ncost), _p(costs), _p(rows), _p(pts),
                               C.c_int32(n if first_new is None else first_new), C.c_int32(len(rem)), _p(rem))
        self.n = n

    def update(self):
        self.R.ref_ffc_update(self.h)

    def lists(self):
        """[(costs [k], [paths [rows, 3]])] of every cluster"""
        out = []
        for i in range(self.n):
            nc, npt = C.c_int32(), C.c_int32()
            self.R.ref_ffc_sizes(self.h, i, C.byref(nc), C.byref(npt))
            costs = np.zeros(nc.value)
            rows = np.zeros(nc.value, np.int32)
            pts = np.zeros((npt.value, 3))
            self.R.ref_ffc_lists(self.h, i, _p(costs), _p(rows), _p(pts))
            off = np.concatenate([[0], np.cumsum(rows)])
            out.append((costs, [pts[off[k]:off[k + 1]] for k in range(nc.value)]))
        return out

    def full(self, cur_pos, cur_vel, cur_yaw):
        mat = np.zeros((self.n + 1, self.n + 1))
        a = [np.ascontiguousarray(x, np.float64) for x in (cur_pos, cur_vel, cur_yaw)]
        self.R.ref_ffc_full(self.h, _p(a[0]), _p(a[1]), _p(a[2]), _p(mat))
        return mat

    def tour(self, pos, ids, max_rows=4096):
        ids = np.ascontiguousarray(ids, np.int32)
        out = np.zeros((max_rows, 3))
        n = self.R.ref_ffc_tour(self.h, _p(np.ascontiguousarray(pos, np.float64)), len(ids), _p(ids),
                                C.c_int32(max_rows), _p(out))
        assert n <= max_rows
        return out[:n]
