"""The global and local tours of FastExplorationManager::planExploreMotion (exploration_manager/src/
fast_exploration_manager.cpp:88-293) on the device, between the frontier cost matrix and the path to the next viewpoint.

findGlobalTour (:327-427) solves the ATSP over getFullCostMatrix's matrix that the reference hands to LKH; here
global_tour_batch solves it exactly on the device (fuelgpu_global_tour_batch, up to GTOUR_MAX_CLUSTERS clusters).

With refine_local the reference takes the first frontiers of the global tour (select_refined_ids, :139-147), fetches up
to top_view_num viewpoints of each (FrontierFinder.getViewpointsInfo) and picks one per frontier with refineLocalTour
(:429-503): a layered graph of ViewNodes searched by Dijkstra over ViewNode::costTo edges.  local_tour_batch runs B such
problems in one fuelgpu_local_tour_batch call, every edge costed at once on the device.  With a single frontier the
reference picks the cheapest viewpoint by computeCost instead (pick_one_viewpoint, :202-214).
"""
import ctypes as C
from dataclasses import dataclass

import numpy as np

from ._lib import FuelAstarParams, FuelLocalTourParams, FuelViewCostParams, check, lib, ptr
from .non_uniform_bspline import _handle
from .view_node import ViewNode

# FuelLocalTourInfo.status
TOUR_OK, TOUR_UNREACHABLE, TOUR_BAD_INPUT, TOUR_TRUNCATED = 0, 1, 2, 3
TOUR_MAX_NODES = 1024
# one FuelLocalTourInfo per problem (include/fuelgpu.h)
TOUR_INFO_DTYPE = np.dtype([("status", np.int32), ("n_nodes", np.int32), ("n_edges", np.int32),
                            ("n_evals", np.int32), ("n_refined", np.int32), ("n_tour", np.int32), ("pops", np.int32),
                            ("pushes", np.int32), ("g", np.float64)])

# FuelGlobalTourInfo.status
GTOUR_OK, GTOUR_BAD_INPUT, GTOUR_TOO_LARGE = 0, 1, 2
GTOUR_MAX_CLUSTERS = 20
# one FuelGlobalTourInfo per instance (include/fuelgpu.h)
GTOUR_INFO_DTYPE = np.dtype([("status", np.int32), ("n", np.int32), ("n_optimal", np.int32), ("reserved", np.int32),
                             ("cost", np.int64)])


@dataclass
class ExplorationParam:
    """the exploration/ parameters of the local tour (exploration_manager/launch/algorithm.xml:90-94)"""
    refine_local: bool = True
    refined_num: int = 7
    refined_radius: float = 5.0
    top_view_num: int = 15
    max_decay: float = 0.8


def _norm(v):
    v = np.asarray(v, np.float64)
    return float(np.sqrt((v[0] * v[0] + v[1] * v[1]) + v[2] * v[2]))


def select_refined_ids(points, indices, pos, refined_num, refined_radius):
    """planExploreMotion :139-147: the first frontiers of the global tour `indices` (into points, the top viewpoints)
    -> (refined_ids, unrefined_points); stops after the first one farther than refined_radius once two are taken"""
    ids, unrefined = [], []
    knum = min(len(indices), int(refined_num))
    for i in range(knum):
        tmp = np.asarray(points[indices[i]], np.float64)
        unrefined.append(tmp)
        ids.append(int(indices[i]))
        if _norm(tmp - np.asarray(pos, np.float64)) > refined_radius and len(ids) >= 2:
            break
    return ids, unrefined


def local_tour_batch(sdf_map, prob_off, group_off, cur_pos, cur_vel, cur_yaw, vp_pos, vp_yaw, *, vm, yd, w_dir,
                     resolution, lambda_heu, allocate_num, max_iter, tour_lambda_heu=1.0, kmax=None, tour_max=256,
                     edge_cost=False):
    """fuelgpu_local_tour_batch over B problems -> (info [B] of TOUR_INFO_DTYPE, refined [B, kmax] (indices into
    vp_*, -1 past n_refined), tour [B, tour_max, 3], edge_cost [E] or None): the raw arrays the C entry writes.
    Problem b has groups prob_off[b] .. prob_off[b + 1]; group g has viewpoints group_off[g] .. group_off[g + 1]."""
    prob_off = np.ascontiguousarray(prob_off, np.int32)
    group_off = np.ascontiguousarray(group_off, np.int32)
    cur_pos, cur_vel = (np.ascontiguousarray(np.asarray(a, np.float64).reshape(-1, 3)) for a in (cur_pos, cur_vel))
    cur_yaw = np.ascontiguousarray(np.asarray(cur_yaw, np.float64).reshape(-1))
    vp_pos = np.ascontiguousarray(np.asarray(vp_pos, np.float64).reshape(-1, 3))
    vp_yaw = np.ascontiguousarray(np.asarray(vp_yaw, np.float64).reshape(-1))
    B = len(prob_off) - 1
    if kmax is None:
        kmax = max(1, int(np.diff(prob_off).max())) if B > 0 else 1
    prm = FuelLocalTourParams(FuelViewCostParams(float(vm), float(yd), float(w_dir),
                                                 FuelAstarParams(float(resolution), float(lambda_heu),
                                                                 int(allocate_num), int(max_iter))),
                              float(tour_lambda_heu))
    info = np.zeros(max(B, 0), dtype=TOUR_INFO_DTYPE)
    refined = np.zeros((max(B, 0), kmax), np.int32)
    tour = np.zeros((max(B, 0), tour_max, 3))
    ec = None
    if edge_cost:
        E = 0
        for b in range(B):
            sizes = np.diff(group_off[prob_off[b]:prob_off[b + 1] + 1])
            n_in = 1
            for i, s in enumerate(sizes):
                eff = min(int(s), 1) if i == len(sizes) - 1 else int(s)
                E += eff * n_in
                n_in = eff
        ec = np.zeros(E)
    h = _handle(sdf_map)
    check(lib().fuelgpu_local_tour_batch(h, B, ptr(prob_off), ptr(group_off), ptr(cur_pos), ptr(cur_vel),
                                         ptr(cur_yaw), ptr(vp_pos), ptr(vp_yaw), C.byref(prm), ptr(info), int(kmax),
                                         ptr(refined), int(tour_max), ptr(tour), ptr(ec)), h)
    return info, refined, tour, ec


def refineLocalTour(cur_pos, cur_vel, cur_yaw, n_points, n_yaws, sdf_map=None):
    """fast_exploration_manager.cpp:429-503 with ViewNode's statics, in one device call -> (refined_pts [k, 3],
    refined_yaws [k], refined_tour [n, 3]).  cur_yaw is (yaw, yaw rate, yaw acceleration); only cur_yaw[0] counts.
    Where Dijkstra cannot reach the last group's first viewpoint (an empty middle group, NaN or >= 1e6 edge costs) the
    refined lists are empty and the tour is [cur_pos]: the reference's caller then reads refined_points_[0], which is
    undefined behaviour.  Afterwards ViewNode.astar_'s lambda_heu is 10000, as :499 leaves the reference's searcher."""
    m = ViewNode.map_ if sdf_map is None else sdf_map
    m = getattr(m, "sdf_map_", m)
    if len(n_points) == 0 or len(n_points[-1]) == 0:
        raise ValueError("refineLocalTour: no group, or an empty last group (the reference dereferences a null "
                         "final_node)")
    group_off = np.concatenate([[0], np.cumsum([len(p) for p in n_points])]).astype(np.int32)
    vp_pos = np.concatenate([np.asarray(p, np.float64).reshape(-1, 3) for p in n_points])
    vp_yaw = np.concatenate([np.asarray(y, np.float64).reshape(-1) for y in n_yaws])
    a = ViewNode.astar_
    kw = dict(vm=ViewNode.vm_, yd=ViewNode.yd_, w_dir=ViewNode.w_dir_, resolution=a["resolution"],
              lambda_heu=a["lambda_heu"], allocate_num=a["allocate_num"], max_iter=a["max_iter"], tour_lambda_heu=1.0)
    args = (m, [0, len(n_points)], group_off, [cur_pos], [cur_vel], [float(cur_yaw[0])], vp_pos, vp_yaw)
    info, refined, tour, _ = local_tour_batch(*args, **kw)
    if info["status"][0] == TOUR_TRUNCATED:  # fetch the whole tour
        info, refined, tour, _ = local_tour_batch(*args, tour_max=int(info["n_tour"][0]), **kw)
    ViewNode.astar_["lambda_heu"] = 10000.0
    if info["status"][0] == TOUR_BAD_INPUT:
        raise ValueError("refineLocalTour: a non-finite coordinate")
    k = int(info["n_refined"][0])
    ids = refined[0, :k]
    return vp_pos[ids].copy(), vp_yaw[ids].copy(), tour[0, :int(info["n_tour"][0])].copy()


def pick_one_viewpoint(pos, points, yaws, vel, yaw, sdf_map=None):
    """planExploreMotion :202-214, the one-frontier case: the first viewpoint whose ViewNode::computeCost(pos, p,
    yaw[0], y, vel) is strictly below every earlier one and below 100000, in one ViewNode.costBatch call -> its index,
    or -1 when none is (the reference then indexes n_points_[0][-1], out of range)."""
    n = len(points)
    if n == 0:
        return -1
    cost, _, _ = ViewNode.costBatch(np.repeat(np.asarray(pos, np.float64).reshape(1, 3), n, axis=0), points,
                                    np.full(n, float(yaw[0])), yaws,
                                    np.repeat(np.asarray(vel, np.float64).reshape(1, 3), n, axis=0), sdf_map=sdf_map)
    min_cost, min_id = 100000.0, -1
    for i, c in enumerate(cost):
        if c < min_cost:
            min_cost, min_id = c, i
    return min_id


def global_tour_batch(sdf_map, dims, cost):
    """fuelgpu_global_tour_batch over B instances -> (info [B] of GTOUR_INFO_DTYPE, indices [sum(dims - 1)]): the raw
    arrays the C entry writes.  Instance b is the dims[b] x dims[b] matrix at its place in `cost` (the matrices
    concatenated, row-major); its tour is the dims[b] - 1 cluster ids at its place in `indices` (-1 unless OK)."""
    dims = np.ascontiguousarray(dims, np.int32).reshape(-1)
    cost = np.ascontiguousarray(np.asarray(cost, np.float64).reshape(-1))
    B = len(dims)
    info = np.zeros(B, dtype=GTOUR_INFO_DTYPE)
    indices = np.zeros(max(int(dims.astype(np.int64).sum()) - B, 0), np.int32)
    h = _handle(sdf_map)
    check(lib().fuelgpu_global_tour_batch(h, B, ptr(dims), ptr(cost), ptr(info), ptr(indices)), h)
    return info, indices


def findGlobalTour(frontier_finder, cur_pos, cur_vel, cur_yaw):
    """fast_exploration_manager.cpp:327-427 -> (indices, global_tour [k, 3]): updateFrontierCostMatrix, then
    getFullCostMatrix, then the tour LKH would be asked for, solved exactly in one device call (the lexicographically
    smallest of the optimal tours), then getPathForTour.  Raises ValueError where the matrix has a cost whose int(cost *
    100) is undefined (NaN, infinite, out of int32) and where there are more than GTOUR_MAX_CLUSTERS clusters (such a
    caller keeps LKH)."""
    ff = frontier_finder
    ff.updateFrontierCostMatrix()
    mat = ff.getFullCostMatrix(cur_pos, cur_vel, cur_yaw)
    if mat.shape[0] < 2:
        raise ValueError("findGlobalTour: no frontier")
    info, indices = global_tour_batch(ff._map, [mat.shape[0]], mat)
    if info["status"][0] == GTOUR_BAD_INPUT:
        raise ValueError("findGlobalTour: a cost whose integer conversion is undefined (NaN, inf or beyond int32)")
    if info["status"][0] == GTOUR_TOO_LARGE:
        raise ValueError("findGlobalTour: %d clusters, more than GTOUR_MAX_CLUSTERS = %d" % (mat.shape[0] - 1,
                                                                                          GTOUR_MAX_CLUSTERS))
    ids = [int(i) for i in indices]
    return ids, ff.getPathForTour(cur_pos, ids)
