"""ctypes binding of the local-tour oracle (oracle/fuel_oracle_tour.c: FastExplorationManager::refineLocalTour over the
view-cost oracle, its edges costed lazily as DijkstraSearch asks for them) and of the reference's own
exploration_manager/src/fast_exploration_manager.cpp (refineLocalTour) and frontier_finder.cpp (getViewpointsInfo,
getTopViewpointsInfo) run through oracle/ref_tour_wrap.cpp (oracle/_ref/libfuel_ref_tour.so), both built by
oracle/tour.mk, the reference library where the reference's sources are present.  The map is oracle.astar.Map.

TEST INFRASTRUCTURE ONLY, like the rest of this package: fuel_b200/ must never import it.
"""
import ctypes as C

import numpy as np

from . import _load, _make, _p, ref_raycast

# the layout of FuelLocalTourInfo (include/fuelgpu.h)
TOUR_DTYPE = np.dtype([("status", np.int32), ("n_nodes", np.int32), ("n_edges", np.int32), ("n_evals", np.int32),
                       ("n_refined", np.int32), ("n_tour", np.int32), ("pops", np.int32), ("pushes", np.int32),
                       ("g", np.float64)])


def build():
    """Compile this part with oracle/tour.mk."""
    _make("tour.mk")


def lib():
    return _load("libfuel_oracle_tour.so", dict(orc_local_tour=C.c_int32), build=build)


def edge_offsets(prob_off, group_off):
    """[B + 1] offsets of each problem's edges in the addEdge order of fuelgpu_local_tour_batch"""
    out = [0]
    for b in range(len(prob_off) - 1):
        sizes = np.diff(group_off[prob_off[b]:prob_off[b + 1] + 1])
        n_in, e = 1, 0
        for i, s in enumerate(sizes):
            eff = min(int(s), 1) if i == len(sizes) - 1 else int(s)
            e += eff * n_in
            n_in = eff
        out.append(out[-1] + e)
    return np.asarray(out, np.int64)


def local_tour_batch(m, prob_off, group_off, cur_pos, cur_vel, cur_yaw, vp_pos, vp_yaw, vm, yd, w_dir, resolution,
                     lambda_heu, allocate_num, max_iter, tour_lambda_heu=1.0, kmax=None, tour_max=1024, table=None):
    """refineLocalTour over B problems on the oracle, in the layout of fuelgpu_local_tour_batch -> (info [B] of
    TOUR_DTYPE, refined [B, kmax] (indices into vp_*), tour [B, tour_max, 3], edge_cost [E]: NaN where the lazy search
    did not evaluate the edge).  table: [E] edge costs to search over instead (m may then be None: no tour)."""
    prob_off = np.ascontiguousarray(prob_off, np.int32)
    group_off = np.ascontiguousarray(group_off, np.int32)
    cur_pos, cur_vel = (np.ascontiguousarray(np.asarray(a, np.float64).reshape(-1, 3)) for a in (cur_pos, cur_vel))
    cur_yaw = np.ascontiguousarray(np.asarray(cur_yaw, np.float64).reshape(-1))
    vp_pos = np.ascontiguousarray(np.asarray(vp_pos, np.float64).reshape(-1, 3))
    vp_yaw = np.ascontiguousarray(np.asarray(vp_yaw, np.float64).reshape(-1))
    B = len(prob_off) - 1
    if kmax is None:
        kmax = max(1, int(np.diff(prob_off).max())) if B else 1
    eo = edge_offsets(prob_off, group_off)
    info = np.zeros(B, TOUR_DTYPE)
    refined = np.full((B, kmax), -1, np.int32)
    tour = np.zeros((B, tour_max, 3))
    edge_cost = np.full(int(eo[-1]), np.nan)
    if table is not None:
        table = np.ascontiguousarray(table, np.float64)
    L = lib()
    for b in range(B):
        g0, g1 = prob_off[b], prob_off[b + 1]
        v0 = group_off[g0]
        gsize = np.ascontiguousarray(np.diff(group_off[g0:g1 + 1]), np.int32)
        ec = np.full(int(eo[b + 1] - eo[b]), np.nan)
        ref = np.full(kmax, -1, np.int32)
        tb = None if table is None else np.ascontiguousarray(table[eo[b]:eo[b + 1]])
        r = L.orc_local_tour(None if m is None else C.byref(m.s), C.c_int32(g1 - g0), _p(gsize), _p(vp_pos[v0:]),
                             _p(vp_yaw[v0:]), _p(cur_pos[b]), _p(cur_vel[b]), C.c_double(cur_yaw[b]), C.c_double(vm),
                             C.c_double(yd), C.c_double(w_dir), C.c_double(resolution), C.c_double(lambda_heu),
                             C.c_int32(allocate_num), C.c_int32(max_iter), C.c_double(tour_lambda_heu), _p(tb),
                             _p(info[b:b + 1]), C.c_int32(kmax), _p(ref), C.c_int32(tour_max), _p(tour[b]), _p(ec))
        assert r == 0, "orc_local_tour: %d" % r
        refined[b] = np.where(ref >= 0, ref + v0, -1)
        edge_cost[eo[b]:eo[b + 1]] = ec
    return info, refined, tour, edge_cost


def ref_tour():
    """The REFERENCE's fast_exploration_manager.cpp + frontier_finder.cpp + oracle/ref_tour_wrap.cpp over libfuel_ref.so's
    SDFMap and RayCaster, or None where it is not built."""
    return _load("_ref/libfuel_ref_tour.so", dict(ref_tour_viewpoints=C.c_int32, ref_tour_select_ids=C.c_int32,
                                                  ref_tour_pick=C.c_int32), first=ref_raycast)


def _f64(a, shape=(-1,)):
    return np.ascontiguousarray(np.asarray(a, np.float64).reshape(shape))


class RefTour:
    """The reference's ViewNode statics (vm_, yd_, w_dir_, astar_ at resolution 0.4, caster_, map_) on the reference's
    SDFMap `ref_map`, and a FastExplorationManager whose refineLocalTour they serve; max_iter stands for
    max_search_time_ on the tick clock.  One at a time: they are statics."""

    def __init__(self, ref_map, vm, yd, w_dir, lambda_heu, allocate_num, max_iter):
        self.R = ref_tour()
        self.R.ref_tour_setup(ref_map.h, C.c_double(vm), C.c_double(yd), C.c_double(w_dir), C.c_double(lambda_heu),
                              C.c_int32(allocate_num), C.c_double(float(max_iter)))

    def close(self):
        self.R.ref_tour_teardown()

    def refine(self, cur_pos, cur_vel, cur_yaw, n_points, n_yaws, tour_max=4096):
        """refineLocalTour -> (refined_pts [k, 3], refined_yaws [k], refined_tour [n, 3], lambda_heu afterwards);
        cur_yaw is the reference's Vector3d (yaw, rate, acceleration)"""
        ng = len(n_points)
        gsize = np.ascontiguousarray([len(p) for p in n_points], np.int32)
        vp = _f64(np.concatenate([np.asarray(p, np.float64).reshape(-1, 3) for p in n_points]), (-1, 3))
        vy = _f64(np.concatenate([np.asarray(y, np.float64).reshape(-1) for y in n_yaws]))
        kmax = max(ng, 1)
        nr, nt, lam = C.c_int32(), C.c_int32(), C.c_double()
        rp, ry, tour = np.zeros((kmax, 3)), np.zeros(kmax), np.zeros((tour_max, 3))
        self.R.ref_tour_refine(_p(_f64(cur_pos)), _p(_f64(cur_vel)), _p(_f64(cur_yaw)), C.c_int32(ng), _p(gsize),
                               _p(vp), _p(vy), C.c_int32(kmax), C.byref(nr), _p(rp), _p(ry), C.c_int32(tour_max),
                               C.byref(nt), _p(tour), C.byref(lam))
        assert nt.value <= tour_max
        return rp[:nr.value], ry[:nr.value], tour[:nt.value], lam.value

    def pick(self, pos, vel, yaw, points, yaws):
        """planExploreMotion :202-214 over the compiled ViewNode::computeCost -> index, -1 when none"""
        pts = _f64(points, (-1, 3))
        return int(self.R.ref_tour_pick(_p(_f64(pos)), _p(_f64(vel)), _p(_f64(yaw)), C.c_int32(len(pts)), _p(pts),
                                        _p(_f64(yaws))))


def ref_select_ids(points, indices, pos, refined_num, refined_radius):
    """planExploreMotion :139-147 in the driver -> refined ids"""
    pts = _f64(points, (-1, 3))
    idx = np.ascontiguousarray(indices, np.int32)
    out = np.zeros(max(len(idx), 1), np.int32)
    n = ref_tour().ref_tour_select_ids(_p(pts), C.c_int32(len(idx)), _p(idx), _p(_f64(pos)), C.c_int32(refined_num),
                                       C.c_double(refined_radius), _p(out))
    return out[:n].tolist()


def ref_viewpoints(frontiers, min_dist, cur_pos, ids, view_num, max_decay):
    """the reference FrontierFinder holding `frontiers` (objects with id_ and viewpoints_ [(pos, yaw, visib_num)])
    -> (getViewpointsInfo's (points, yaws) lists, getTopViewpointsInfo's (points [n, 3], yaws [n])).  Needs a RefTour
    alive (its map)."""
    n = len(frontiers)
    views = [v for f in frontiers for v in f.viewpoints_]
    fids = np.ascontiguousarray([f.id_ for f in frontiers], np.int32)
    nv = np.ascontiguousarray([len(f.viewpoints_) for f in frontiers], np.int32)
    pos = _f64([v[0] for v in views], (-1, 3))
    yaw = _f64([v[1] for v in views])
    vis = np.ascontiguousarray([v[2] for v in views], np.int32)
    idl = np.ascontiguousarray(ids, np.int32)
    counts = np.zeros(max(len(idl), 1), np.int32)
    opos, oyaw = np.zeros((max(len(views), 1) * max(len(idl), 1), 3)), np.zeros(max(len(views), 1) * max(len(idl), 1))
    tpos, tyaw = np.zeros((max(n, 1), 3)), np.zeros(max(n, 1))
    ng = ref_tour().ref_tour_viewpoints(C.c_int32(n), _p(fids), _p(nv), _p(pos), _p(yaw), _p(vis),
                                        C.c_double(min_dist), _p(_f64(cur_pos)), C.c_int32(len(idl)), _p(idl),
                                        C.c_int32(view_num), C.c_double(max_decay), _p(counts), _p(opos), _p(oyaw),
                                        _p(tpos), _p(tyaw))
    points, yaws, r = [], [], 0
    for g in range(ng):
        points.append(opos[r:r + counts[g]].copy())
        yaws.append(oyaw[r:r + counts[g]].copy())
        r += counts[g]
    return (points, yaws), (tpos[:n], tyaw[:n])
