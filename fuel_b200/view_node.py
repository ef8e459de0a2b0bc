"""ViewNode (active_perception/include/active_perception/graph_node.h) on the device, over fuelgpu_view_cost_batch.

ViewNode::searchPath and ViewNode::computeCost (active_perception/src/graph_node.cpp:32-85) are the edge cost of the
exploration tour: the straight line between two viewpoints when it is clear, else an A* search at resolution 0.4, and
the time to fly it or to turn, whichever is longer.  view_cost_batch runs P pairs in one call; the static methods run
one pair as the reference's do.  The reference's wall-clock limit astar/max_search_time is an iteration cap, max_iter.
"""
import ctypes as C

import numpy as np

from ._lib import FuelAstarParams, FuelViewCostParams, check, lib, ptr
from .non_uniform_bspline import _handle

# FuelViewCostInfo.kind
LINE, ASTAR, NO_PATH = 1, 2, 3
# one FuelViewCostInfo per pair (include/fuelgpu.h)
INFO_DTYPE = np.dtype([("kind", np.int32), ("reason", np.int32), ("iter_num", np.int32), ("use_node_num", np.int32),
                       ("n_path", np.int32), ("reserved", np.int32), ("length", np.float64), ("cost", np.float64)])


def view_cost_batch(sdf_map, p1, p2, y1, y2, v1, *, vm, yd, w_dir, resolution, lambda_heu, allocate_num, max_iter,
                    path_max=256):
    """fuelgpu_view_cost_batch over P pairs -> (info [P] of INFO_DTYPE, path [P, path_max, 3] or None when path_max is
    0): the raw arrays the C entry writes"""
    p1, p2, v1 = (np.ascontiguousarray(np.asarray(a, dtype=np.float64).reshape(-1, 3)) for a in (p1, p2, v1))
    y1, y2 = (np.ascontiguousarray(np.asarray(a, dtype=np.float64).reshape(-1)) for a in (y1, y2))
    P = len(p1)
    if not (p2.shape == v1.shape == (P, 3) and y1.shape == y2.shape == (P,)):
        raise ValueError("p1, p2, v1 must be [P, 3] and y1, y2 [P]")
    prm = FuelViewCostParams(float(vm), float(yd), float(w_dir),
                             FuelAstarParams(float(resolution), float(lambda_heu), int(allocate_num), int(max_iter)))
    info = np.empty(P, dtype=INFO_DTYPE)
    path = np.empty((P, path_max, 3)) if path_max > 0 else None
    h = _handle(sdf_map)
    check(lib().fuelgpu_view_cost_batch(h, P, ptr(p1), ptr(p2), ptr(y1), ptr(y2), ptr(v1), C.byref(prm), ptr(info),
                                        int(max(path_max, 0)), ptr(path)), h)
    return info, path


class ViewNode:
    """The statics of the reference's ViewNode and its two static methods.  Set them as
    FastExplorationManager::initialize does (fast_exploration_manager.cpp:55-62): vm_, yd_, w_dir_ from exploration/*,
    astar_ from astar/* (max_iter standing for max_search_time), map_ the SDFMap (or EDTEnvironment) searched.
    Defaults: exploration_manager/launch/algorithm.xml:95-99,164-167 with max_vel 2.0 (exploration.launch:44)."""

    vm_ = 2.0
    yd_ = 60 * 3.1415926 / 180.0
    w_dir_ = 1.5
    astar_ = dict(resolution=0.4, lambda_heu=10000.0, allocate_num=1000000, max_iter=10000)
    map_ = None

    @classmethod
    def costBatch(cls, p1, p2, y1, y2, v1, sdf_map=None):
        """computeCost for P pairs in one device call on sdf_map (default map_) -> (cost [P], info [P], paths:
        searchPath's path of each pair, [n_path, 3] arrays in full)"""
        m = cls.map_ if sdf_map is None else sdf_map
        m = getattr(m, "sdf_map_", m)
        kw = dict(vm=cls.vm_, yd=cls.yd_, w_dir=cls.w_dir_, **cls.astar_)
        info, path = view_cost_batch(m, p1, p2, y1, y2, v1, **kw)
        need = int(info["n_path"].max()) if len(info) else 0
        if need > path.shape[1]:  # a search path longer than the first call kept: fetch it whole
            info, path = view_cost_batch(m, p1, p2, y1, y2, v1, path_max=need, **kw)
        paths = [path[q, :info["n_path"][q]].copy() for q in range(len(info))]
        bad = np.nonzero(info["kind"] == 0)[0]
        if len(bad):
            raise ValueError("pair %d has a non-finite input" % bad[0])
        return info["cost"].copy(), info, paths

    @classmethod
    def searchPath(cls, p1, p2):
        """graph_node.cpp:32-61 -> (length, path [n, 3])"""
        _, info, paths = cls.costBatch([p1], [p2], [0.0], [0.0], [np.zeros(3)])
        return float(info["length"][0]), paths[0]

    @classmethod
    def computeCost(cls, p1, p2, y1, y2, v1, yd1=0.0):
        """graph_node.cpp:63-85 -> (cost, path [n, 3]); yd1 is unused, as in the reference"""
        cost, _, paths = cls.costBatch([p1], [p2], [y1], [y2], [v1])
        return float(cost[0]), paths[0]
