"""Astar (path_searching/include/path_searching/astar2.h) and the head of FastExplorationManager::planExploreMotion
(exploration_manager/src/fast_exploration_manager.cpp:238-263) on the device, over fuelgpu_astar_batch.

search_paths_batch runs B searches from a start to a goal each -- Astar::search, getPath, shortenPath, pathLength and
the close / mid / far branch -- and returns the tours in the list form plan_explore_traj_batch takes.  Astar is the
reference's class over one search; its wall-clock limit max_search_time_ is an iteration cap, max_iter.
"""
import ctypes as C

import numpy as np

from ._lib import FuelAstarParams, check, lib, ptr
from .non_uniform_bspline import _handle

REACH_END, NO_PATH = 1, 2  # Astar::REACH_END, Astar::NO_PATH
# FuelPathInfo.reason
FOUND, OPEN_EMPTY, POOL, ITER_CAP, HEAP_FULL, BAD_INPUT = 0, 1, 2, 3, 4, 5
# FuelPathInfo.branch
NONE, CLOSE, MID, FAR = 0, 1, 2, 3
# FuelPathInfo.tour_status
TOUR_OK, TOO_LONG, DEGENERATE = 0, 1, 2
MAX_WAYPTS = 32  # FUELGPU_MAX_WAYPTS

# one FuelPathInfo per query (include/fuelgpu.h)
INFO_DTYPE = np.dtype([("status", np.int32), ("reason", np.int32), ("iter_num", np.int32), ("use_node_num", np.int32),
                       ("n_path", np.int32), ("n_wp", np.int32), ("branch", np.int32), ("tour_status", np.int32),
                       ("early_terminate_cost", np.float64), ("length", np.float64), ("next_goal", np.float64, (3,))])


def _params(resolution, lambda_heu, allocate_num, max_iter):
    return FuelAstarParams(float(resolution), float(lambda_heu), int(allocate_num), int(max_iter))


def astar_batch(sdf_map, start, goal, *, resolution=0.1, lambda_heu=10000.0, allocate_num=100000, max_iter=100000,
                path_max=1024, w_max=MAX_WAYPTS):
    """fuelgpu_astar_batch over B queries -> (info [B] of INFO_DTYPE, path [B, path_max, 3], n_wp [B],
    waypts [B, w_max, 3]): the raw arrays the C entry writes"""
    s = np.ascontiguousarray(np.asarray(start, dtype=np.float64).reshape(-1, 3))
    g = np.ascontiguousarray(np.asarray(goal, dtype=np.float64).reshape(-1, 3))
    if s.shape != g.shape:
        raise ValueError("start and goal must both be [B, 3]")
    B = len(s)
    prm = _params(resolution, lambda_heu, allocate_num, max_iter)
    info = np.empty(B, dtype=INFO_DTYPE)
    path = np.empty((B, path_max, 3)) if path_max > 0 else None
    n_wp = np.empty(B, dtype=np.int32)
    wp = np.empty((B, w_max, 3))
    h = _handle(sdf_map)
    check(lib().fuelgpu_astar_batch(h, B, ptr(s), ptr(g), C.byref(prm), ptr(info), int(max(path_max, 0)), ptr(path),
                                    int(w_max), ptr(n_wp), ptr(wp)), h)
    return info, path, n_wp, wp


def search_paths_batch(sdf_map, start, goal, *, resolution=0.1, lambda_heu=10000.0, allocate_num=100000,
                       max_iter=100000, path_max=1024):
    """planExploreMotion's path stage for B (start, goal) pairs.  Returns dict(info [B] of INFO_DTYPE, paths: a list of
    getPath() arrays [n_path, 3] (the first path_max rows), tours: a list of [n_wp, 3] arrays -- the tour
    planExploreTraj receives, None where there is no usable one (no path, fewer than 3 points, more than 32) --
    and next_goal [B, 3])."""
    info, path, n_wp, wp = astar_batch(sdf_map, start, goal, resolution=resolution, lambda_heu=lambda_heu,
                                       allocate_num=allocate_num, max_iter=max_iter, path_max=path_max)
    paths = [path[b, :min(int(info["n_path"][b]), path_max)].copy() for b in range(len(info))]
    tours = [wp[b, :n_wp[b]].copy() if n_wp[b] > 0 else None for b in range(len(info))]
    return dict(info=info, paths=paths, tours=tours, next_goal=info["next_goal"].copy())


class Astar:
    """The reference's Astar over one search on the device of an EDTEnvironment's map (init(nh, env) -> the
    constructor).  max_iter stands for max_search_time_: the search ends with NO_PATH at loop iteration max_iter + 1."""

    REACH_END, NO_PATH = REACH_END, NO_PATH

    def __init__(self, env, resolution=0.1, lambda_heu=10000.0, allocate_num=100000, max_iter=100000, path_max=100001):
        self.env_ = env
        self.resolution_ = float(resolution)
        self.lambda_heu_ = float(lambda_heu)
        self.allocate_num_ = int(allocate_num)
        self.max_iter = int(max_iter)
        self.path_max = int(path_max)
        self.early_terminate_cost_ = 0.0
        self.reset()

    def reset(self):
        self.path_nodes_ = np.zeros((0, 3))
        self.use_node_num_ = 0
        self.iter_num_ = 0
        self.info_ = None

    def setResolution(self, res):
        self.resolution_ = float(res)

    def search(self, start_pt, end_pt):
        m = getattr(self.env_, "sdf_map_", self.env_)
        info, path, _, _ = astar_batch(m, [start_pt], [end_pt], resolution=self.resolution_,
                                       lambda_heu=self.lambda_heu_, allocate_num=self.allocate_num_,
                                       max_iter=self.max_iter, path_max=self.path_max)
        i = info[0]
        self.info_ = i
        self.use_node_num_ = int(i["use_node_num"])
        self.iter_num_ = int(i["iter_num"])
        self.path_nodes_ = path[0, :min(int(i["n_path"]), self.path_max)].copy()
        if i["reason"] == ITER_CAP:  # the reference keeps the last value otherwise
            self.early_terminate_cost_ = float(i["early_terminate_cost"])
        return int(i["status"])

    def getPath(self):
        return [p.copy() for p in self.path_nodes_]

    @staticmethod
    def pathLength(path):
        length = 0.0
        for a, b in zip(path[:-1], path[1:]):
            d = np.asarray(b, dtype=np.float64) - np.asarray(a, dtype=np.float64)
            length += float(np.sqrt((d[0] * d[0] + d[1] * d[1]) + d[2] * d[2]))
        return length

    def getEarlyTerminateCost(self):
        return self.early_terminate_cost_
