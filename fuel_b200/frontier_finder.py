"""Host-side mirror of fast_planner::FrontierFinder's hot path over the C ABI.

Mirrors active_perception/include/active_perception/frontier_finder.h:25-133 and
active_perception/src/frontier_finder.cpp:23-121 (file:line under /root/reference/fuel_planner/):
`searchFrontiers()` with the stored-frontier bookkeeping (haveOverlap :353-363,
isFrontierChanged :365-372, removed_ids_) on the host and every voxel-scale step in
libfuelgpu.  The step right after it (SURVEY.md 8f rank 4) is mirrored too: computeFrontiersToVisit
(:392-423) with sampleViewpoints / countVisibleCells (:662-695,734-755) on the device, and
isFrontierCovered (:697-719).  So is the tour's cost bookkeeping: updateFrontierCostMatrix (:260-326),
getFullCostMatrix (:531-592, the asymmetric form the reference runs) and getPathForTour (:508-529), each edge a
ViewNode::computeCost / searchPath of fuel_b200.view_node, all the edges of one call in one device batch.  The TSP
solver itself (LKH) is not part of this library.
"""
import ctypes as C

import numpy as np

from ._lib import FuelFrontierParams, FuelViewParams, check, lib, ptr
from .view_node import ViewNode


def _data(a):
    """address of a numpy array's first element, as an int (ctypes passes it as void*)"""
    return a.__array_interface__["data"][0]


class Frontier:
    """frontier_finder.h:34-51"""
    __slots__ = ("cells_addr_", "filtered_cells_", "average_", "id_", "box_min_", "box_max_", "_map", "viewpoints_",
                 "costs_", "paths_")

    def __init__(self, m, addr, filtered, average, box_min, box_max):
        self._map = m
        self.cells_addr_ = addr
        self.filtered_cells_ = filtered
        self.average_ = average
        self.box_min_ = box_min
        self.box_max_ = box_max
        self.id_ = -1
        self.viewpoints_ = []  # [(pos_ [3], yaw_, visib_num_)], frontier_finder.h:25-31
        self.costs_ = []  # computeCost to every cluster, in frontiers_ order (frontier_finder.h:49-50)
        self.paths_ = []  # searchPath's path to every cluster, [n, 3] arrays

    @property
    def cells_(self):
        """voxel-centre positions (indexToPos of every cell), [n,3] float64"""
        m = self._map
        a = self.cells_addr_.astype(np.int64)
        nyz = m.shape[1] * m.shape[2]
        idx = np.stack([a // nyz, (a % nyz) // m.shape[2], a % m.shape[2]], axis=1)
        return (idx + 0.5) * m.resolution_ + m.map_origin_


def update_cost_matrix(frontiers, first_new, removed_ids, cost_batch):
    """updateFrontierCostMatrix (frontier_finder.cpp:260-326) over a frontier list whose clusters from index first_new
    on are new (None: none).  cost_batch(p1, p2, y1, y2, v1) -> (cost [P], paths) costs every old x new and new x new
    pair in one call; the lists grow in the reference's order."""
    first = len(frontiers) if first_new is None else first_new
    if removed_ids:  # the ids are indices after the removal (:75-84), so erase one after another (:267-286)
        for f in frontiers[:first]:
            for r in removed_ids:
                del f.costs_[r]
                del f.paths_[r]
    pairs = [(i, j) for i in range(first) for j in range(first, len(frontiers))]
    pairs += [(i, j) for i in range(first, len(frontiers)) for j in range(i, len(frontiers))]
    edges = [(i, j) for i, j in pairs if i != j]
    cost, paths = [], []
    if edges:
        vi = [frontiers[i].viewpoints_[0] for i, _ in edges]
        vj = [frontiers[j].viewpoints_[0] for _, j in edges]
        cost, paths = cost_batch([v[0] for v in vi], [v[0] for v in vj], [v[1] for v in vi], [v[1] for v in vj],
                                 np.zeros((len(edges), 3)))
    k = 0
    for i, j in pairs:
        if i == j:
            frontiers[i].costs_.append(0.0)
            frontiers[i].paths_.append(np.zeros((0, 3)))
            continue
        frontiers[i].costs_.append(float(cost[k]))
        frontiers[i].paths_.append(paths[k])
        frontiers[j].costs_.append(float(cost[k]))
        frontiers[j].paths_.append(paths[k][::-1].copy())
        k += 1


def full_cost_matrix(frontiers, cur_pos, cur_vel, cur_yaw, cost_batch):
    """getFullCostMatrix's asymmetric form (frontier_finder.cpp:562-591): [n + 1, n + 1], the clusters' cost lists in
    rows 1..n, column 0 zero, row 0 the cost from the current state (cur_yaw = (yaw, yaw rate, -)) in one call"""
    n = len(frontiers)
    mat = np.zeros((n + 1, n + 1))
    for i, f in enumerate(frontiers):
        mat[i + 1, 1:1 + len(f.costs_)] = f.costs_
    mat[:, 0] = 0.0
    if n:
        views = [f.viewpoints_[0] for f in frontiers]
        cost, _ = cost_batch(np.repeat(np.asarray(cur_pos, np.float64).reshape(1, 3), n, axis=0),
                             [v[0] for v in views], np.full(n, float(cur_yaw[0])), [v[1] for v in views],
                             np.repeat(np.asarray(cur_vel, np.float64).reshape(1, 3), n, axis=0))
        mat[0, 1:] = cost
    return mat


def path_for_tour(frontiers, pos, frontier_ids, cost_batch):
    """getPathForTour (frontier_finder.cpp:508-529): searchPath from pos to the first cluster's top viewpoint, then the
    stored paths along the tour -> [n, 3]"""
    _, paths = cost_batch([pos], [frontiers[frontier_ids[0]].viewpoints_[0][0]], [0.0], [0.0], np.zeros((1, 3)))
    segs = [paths[0]] + [frontiers[a].paths_[b] for a, b in zip(frontier_ids[:-1], frontier_ids[1:])]
    return np.concatenate([np.asarray(s, np.float64).reshape(-1, 3) for s in segs])


class FrontierFinder:
    def __init__(self, edt, cluster_min=100, cluster_size_xy=2.0, down_sample=3, min_z=0.4, cell_order="address"):
        """frontier_finder.cpp:23-49; defaults = exploration_manager/launch/algorithm.xml:103-114.
        cell_order: "address" (cells of a cluster ascending by toAddress, straight from the device) or "bfs" (the
        reference's expandFrontier order; average_ / filtered_cells_ then equal the reference's to the last bit)."""
        self.edt_env_ = edt
        self.cell_order_ = {"address": 0, "bfs": 1}[cell_order]
        h = getattr(edt.sdf_map_, "handle", None)
        if h is not None:  # (host-only stand-ins of the map, as in the bookkeeping tests, have no device handle)
            check(lib().fuelgpu_frontier_set_cell_order(h, self.cell_order_), h)
        self.cluster_min_ = int(cluster_min)
        self.cluster_size_xy_ = float(cluster_size_xy)
        self.down_sample_ = int(down_sample)
        self.min_z_ = float(min_z)
        self.frontiers_ = []
        self.dormant_frontiers_ = []
        self.tmp_frontiers_ = []
        self.removed_ids_ = []
        self.first_new_ftr_ = None
        self.min_visib_num_ = 15
        self.min_view_finish_fraction_ = 0.2
        self.setViewParams()

    def setViewParams(self, candidate_rmin=1.5, candidate_rmax=2.5, candidate_rnum=3, candidate_dphi=15 * 3.1415926 / 180.0,
                      min_candidate_clearance=0.21, min_visib_num=15, min_view_finish_fraction=0.2, top_angle=0.56125,
                      left_angle=0.69222, right_angle=0.68901, max_dist=4.5):
        """frontier/* (frontier_finder.cpp:32-40) and perception_utils/* (perception_utils.cpp:7-10) parameters;
        defaults = exploration_manager/launch/algorithm.xml:106-121."""
        v = FuelViewParams()
        v.candidate_rmin, v.candidate_rmax, v.candidate_rnum, v.candidate_dphi = (
            candidate_rmin, candidate_rmax, candidate_rnum, candidate_dphi)
        v.min_candidate_clearance = min_candidate_clearance
        v.top_angle, v.left_angle, v.right_angle, v.max_dist = top_angle, left_angle, right_angle, max_dist
        self._view = v
        self.min_visib_num_ = int(min_visib_num)
        self.min_view_finish_fraction_ = float(min_view_finish_fraction)

    @property
    def _map(self):
        return self.edt_env_.sdf_map_

    def _params(self):
        p = FuelFrontierParams()
        p.cluster_min, p.cluster_size_xy, p.down_sample, p.min_z = (
            self.cluster_min_, self.cluster_size_xy_, self.down_sample_, self.min_z_)
        return p

    @staticmethod
    def haveOverlap(min1, max1, min2, max2):
        """frontier_finder.cpp:353-363"""
        for i in range(3):
            bmin = max(min1[i], min2[i])
            bmax = min(max1[i], max2[i])
            if bmin > bmax + 1e-3:
                return False
        return True

    def _changed(self, ftrs):
        """isFrontierChanged (:365-372) for a list of stored frontiers, on the device."""
        if not ftrs:
            return np.zeros(0, dtype=np.uint8)
        offs = np.zeros(len(ftrs) + 1, dtype=np.int32)
        for i, f in enumerate(ftrs):
            offs[i + 1] = offs[i] + f.cells_addr_.size
        addr = np.ascontiguousarray(np.concatenate([f.cells_addr_ for f in ftrs]).astype(np.int32))
        changed = np.zeros(len(ftrs), dtype=np.uint8)
        h = self._map.handle
        check(lib().fuelgpu_frontier_is_changed(h, len(ftrs), ptr(offs), ptr(addr), ptr(changed)), h)
        return changed

    def _clear_flags(self, addr):
        """frontier_flag_[addr] = 0 on the device"""
        h = self._map.handle
        check(lib().fuelgpu_frontier_clear_flags(h, addr.size, ptr(addr)), h)

    def _remove_changed(self, ftrs, update_min, update_max, record_ids):
        cand = [i for i, f in enumerate(ftrs)
                if self.haveOverlap(f.box_min_, f.box_max_, update_min, update_max)]
        changed = self._changed([ftrs[i] for i in cand])
        drop = {cand[j] for j in range(len(cand)) if changed[j]}
        if drop:
            self._clear_flags(np.ascontiguousarray(
                np.concatenate([ftrs[i].cells_addr_ for i in sorted(drop)]).astype(np.int32)))  # resetFlag :62-69
        kept = []
        rmv_idx = 0
        for i, f in enumerate(ftrs):
            if i in drop:
                if record_ids:
                    self.removed_ids_.append(rmv_idx)  # :75-84
            else:
                rmv_idx += 1
                kept.append(f)
        return kept

    def searchFrontiers(self):
        """frontier_finder.cpp:54-121"""
        m = self._map
        self.tmp_frontiers_ = []
        update_min, update_max = m.getUpdatedBox(True)
        self.removed_ids_ = []
        self.frontiers_ = self._remove_changed(self.frontiers_, update_min, update_max, True)
        self.dormant_frontiers_ = self._remove_changed(self.dormant_frontiers_, update_min, update_max, False)
        self.tmp_frontiers_ = self.search_box(update_min, update_max)
        return self.tmp_frontiers_

    def search_box(self, update_min, update_max):
        """The sweep + expandFrontier + splitLargeFrontiers part (:94-118) for a given updated box."""
        self.search_box_begin(update_min, update_max)
        return self.search_box_end()

    def search_box_begin(self, update_min, update_max):
        """Enqueue the search on the frontier stream and return at once (fuelgpu_frontier_search_begin)."""
        h = self._map.handle
        umin = np.ascontiguousarray(update_min, dtype=np.float64)
        umax = np.ascontiguousarray(update_max, dtype=np.float64)
        p = self._params()
        check(lib().fuelgpu_frontier_search_begin(h, _data(umin), _data(umax), C.byref(p)), h)

    def candidates(self, update_min, update_max, z_lo, z_hi):
        """The sweep of the planes [z_lo, z_hi] only (fuelgpu_frontier_candidates): this rank's candidate cells of a
        z-sharded search -> (addr int32 ascending, cls uint8).  Needs the tri-state of those planes +- one halo plane."""
        h = self._map.handle
        umin = np.ascontiguousarray(update_min, dtype=np.float64)
        umax = np.ascontiguousarray(update_max, dtype=np.float64)
        p = self._params()
        n = C.c_int32()
        check(lib().fuelgpu_frontier_candidates(h, ptr(umin), ptr(umax), C.byref(p), int(z_lo), int(z_hi), C.byref(n)), h)
        addr = np.empty(n.value, dtype=np.int32)
        cls = np.empty(n.value, dtype=np.uint8)
        check(lib().fuelgpu_frontier_candidates_fetch(h, n.value, ptr(addr), ptr(cls)), h)
        return addr, cls

    def search_from_candidates(self, update_min, update_max, addr, cls):
        """Clustering + split over a candidate list gathered from all ranks (ascending address): the result of
        search_box on one GPU, bit for bit (fuelgpu_frontier_search_from_candidates)."""
        h = self._map.handle
        umin = np.ascontiguousarray(update_min, dtype=np.float64)
        umax = np.ascontiguousarray(update_max, dtype=np.float64)
        addr = np.ascontiguousarray(addr, dtype=np.int32)
        cls = np.ascontiguousarray(cls, dtype=np.uint8)
        p = self._params()
        nc, ncell, nf = C.c_int32(), C.c_int32(), C.c_int32()
        check(lib().fuelgpu_frontier_search_from_candidates(h, ptr(umin), ptr(umax), C.byref(p), addr.size, ptr(addr), ptr(cls),
                                                            C.byref(nc), C.byref(ncell), C.byref(nf)), h)
        return self._fetch(nc.value, ncell.value, nf.value)

    def search_box_end(self):
        """Wait for the enqueued search and build the Frontier list."""
        h = self._map.handle
        nc, ncell, nf = C.c_int32(), C.c_int32(), C.c_int32()
        check(lib().fuelgpu_frontier_search_end(h, C.byref(nc), C.byref(ncell), C.byref(nf)), h)
        return self._fetch(nc.value, ncell.value, nf.value)

    def _fetch(self, nc, ncell, nf):
        m = self._map
        h = m.handle
        # arrays of this call; the Frontier objects hold views into them.  This runs once per search, on the replan's
        # critical path: the pointers are taken as plain integers (ndarray.ctypes costs several microseconds each)
        offs = np.empty(nc + 1, dtype=np.int32)
        addr = np.empty(ncell, dtype=np.int32)
        foffs = np.empty(nc + 1, dtype=np.int32)
        filt = np.empty((nf, 3), dtype=np.float64)
        stats = np.empty((3, nc, 3), dtype=np.float64)
        s0 = _data(stats)
        check(lib().fuelgpu_frontier_fetch(h, _data(offs), _data(addr), _data(foffs), _data(filt), s0, s0 + 24 * nc,
                                           s0 + 48 * nc), h)
        o, fo = offs.tolist(), foffs.tolist()
        return [Frontier(m, addr[o[i]:o[i + 1]], filt[fo[i]:fo[i + 1]], a, lo, hi)
                for i, (a, lo, hi) in enumerate(zip(stats[0], stats[1], stats[2]))]

    # ---- the step after the search (SURVEY 8f rank 4) -------------------------------------
    def sampleViewpointsRaw(self, ftrs):
        """All candidates of sampleViewpoints (:662-695) for a list of clusters in ONE device call.
        -> (pos [n,c,3], yaw [n,c], visib [n,c]); visib = -1 where the candidate is rejected (:671-673)."""
        h = self._map.handle
        nc = lib().fuelgpu_viewpoint_candidate_count(C.byref(self._view))
        n = len(ftrs)
        pos = np.zeros((n, nc, 3))
        yaw = np.zeros((n, nc))
        vis = np.zeros((n, nc), dtype=np.int32)
        if n == 0:
            return pos, yaw, vis
        foffs = np.zeros(n + 1, dtype=np.int32)
        for i, f in enumerate(ftrs):
            foffs[i + 1] = foffs[i] + len(f.filtered_cells_)
        filt = np.ascontiguousarray(np.concatenate([np.asarray(f.filtered_cells_, dtype=np.float64).reshape(-1, 3)
                                                    for f in ftrs]))
        avg = np.ascontiguousarray(np.stack([f.average_ for f in ftrs]), dtype=np.float64)
        check(lib().fuelgpu_frontier_sample_viewpoints(h, n, ptr(foffs), ptr(filt), ptr(avg), C.byref(self._view), nc,
                                                       ptr(pos), ptr(yaw), ptr(vis)), h)
        return pos, yaw, vis

    def computeFrontiersToVisit(self):
        """frontier_finder.cpp:392-423: viewpoints for every new cluster; clusters with none go dormant.  The
        reference sorts with std::sort (order of equal visib_num_ unspecified); here the sort is stable."""
        self.first_new_ftr_ = None
        pos, yaw, vis = self.sampleViewpointsRaw(self.tmp_frontiers_)
        for i, f in enumerate(self.tmp_frontiers_):
            keep = np.nonzero(vis[i] > self.min_visib_num_)[0]  # :688
            f.viewpoints_ = [(pos[i, k].copy(), float(yaw[i, k]), int(vis[i, k])) for k in keep]
            if f.viewpoints_:
                f.viewpoints_.sort(key=lambda v: -v[2])  # best view in front, :404-406
                self.frontiers_.append(f)
                if self.first_new_ftr_ is None:
                    self.first_new_ftr_ = len(self.frontiers_) - 1
            else:
                self.dormant_frontiers_.append(f)
        for idx, f in enumerate(self.frontiers_):
            f.id_ = idx  # :414-418

    def getTopViewpointsInfo(self, cur_pos, min_candidate_dist=0.75):
        """frontier_finder.cpp:425-453: the best viewpoint of every cluster farther than min_candidate_dist_."""
        pts, yaws, avgs = [], [], []
        cur_pos = np.asarray(cur_pos, dtype=np.float64)
        for f in self.frontiers_:
            chosen = None
            for v in f.viewpoints_:
                if np.linalg.norm(v[0] - cur_pos) < min_candidate_dist:
                    continue
                chosen = v
                break
            if chosen is None:
                chosen = f.viewpoints_[0]
            pts.append(chosen[0])
            yaws.append(chosen[1])
            avgs.append(f.average_)
        return pts, yaws, avgs

    def getViewpointsInfo(self, cur_pos, ids, view_num, max_decay, min_candidate_dist=0.75):
        """frontier_finder.cpp:452-484: for each id (a cluster of that id_; none, no entry) its first viewpoints,
        at most view_num, while visib_num_ stays above int(front visib_num_ * max_decay), skipping those closer than
        min_candidate_dist; when that leaves none, the same without the distance limit -> (points, yaws) lists"""
        points, yaws = [], []
        cur_pos = np.asarray(cur_pos, dtype=np.float64)
        for fid in ids:
            for f in self.frontiers_:
                if f.id_ != fid:
                    continue
                thresh = int(f.viewpoints_[0][2] * max_decay)  # int visib_thresh = visib_num_ * max_decay
                pts, ys = [], []
                for far_only in (True, False):
                    for v in f.viewpoints_:
                        if len(pts) >= view_num or v[2] <= thresh:
                            break
                        if far_only and np.linalg.norm(v[0] - cur_pos) < min_candidate_dist:
                            continue
                        pts.append(v[0].copy())
                        ys.append(v[1])
                    if pts:
                        break
                points.append(pts)
                yaws.append(ys)
        return points, yaws

    def isFrontierCovered(self):
        """frontier_finder.cpp:697-719: has any stored cluster overlapping the updated box lost at least
        min_view_finish_fraction_ of its cells?"""
        update_min, update_max = self._map.getUpdatedBox(False)
        ftrs = [f for f in self.frontiers_ + self.dormant_frontiers_
                if self.haveOverlap(f.box_min_, f.box_max_, update_min, update_max)]
        if not ftrs:
            return False
        offs = np.zeros(len(ftrs) + 1, dtype=np.int32)
        for i, f in enumerate(ftrs):
            offs[i + 1] = offs[i] + f.cells_addr_.size
        addr = np.ascontiguousarray(np.concatenate([f.cells_addr_ for f in ftrs]).astype(np.int32))
        counts = np.zeros(len(ftrs), dtype=np.int32)
        h = self._map.handle
        check(lib().fuelgpu_frontier_changed_counts(h, len(ftrs), ptr(offs), ptr(addr), ptr(counts)), h)
        for f, c in zip(ftrs, counts):
            thresh = int(self.min_view_finish_fraction_ * f.cells_addr_.size)  # :704
            if c >= max(thresh, 1):  # `++change_num >= change_thresh` fires on a changed cell only
                return True
        return False

    # ---- the tour's cost: each edge as ViewNode's statics say, searched on this finder's map ----
    def _cost_batch(self):
        def batch(p1, p2, y1, y2, v1):
            cost, _, paths = ViewNode.costBatch(p1, p2, y1, y2, v1, sdf_map=self._map)
            return cost, paths
        return batch

    def updateFrontierCostMatrix(self):
        """frontier_finder.cpp:260-326: drop the removed clusters from the old cost lists, then cost every old x new
        and new x new pair of viewpoints in one device batch"""
        update_cost_matrix(self.frontiers_, self.first_new_ftr_, self.removed_ids_, self._cost_batch())
        self.removed_ids_ = []

    def getFullCostMatrix(self, cur_pos, cur_vel, cur_yaw):
        """frontier_finder.cpp:531-592 (the asymmetric TSP form) -> [n + 1, n + 1]"""
        return full_cost_matrix(self.frontiers_, cur_pos, cur_vel, cur_yaw, self._cost_batch())

    def getPathForTour(self, pos, frontier_ids):
        """frontier_finder.cpp:508-529 -> [n, 3]"""
        return path_for_tour(self.frontiers_, pos, frontier_ids, self._cost_batch())

    def getFrontiers(self):
        return [f.cells_ for f in self.frontiers_]

    def getDormantFrontiers(self):
        return [f.cells_ for f in self.dormant_frontiers_]

    def getFrontierBoxes(self):
        """frontier_finder.cpp getFrontierBoxes: (centre, scale) per stored frontier"""
        return [((f.box_max_ + f.box_min_) / 2, f.box_max_ - f.box_min_) for f in self.frontiers_]

    def reset_flags(self):
        """frontier_flag_ = 0 (the constructor's fill, frontier_finder.cpp:26-27)"""
        check(lib().fuelgpu_frontier_reset_flags(self._map.handle), self._map.handle)

    def download_flags(self):
        m = self._map
        out = np.zeros(m.shape, dtype=np.int8)
        check(lib().fuelgpu_frontier_download_flags(m.handle, ptr(out)), m.handle)
        return out

    def upload_flags(self, flags):
        m = self._map
        f = np.ascontiguousarray(flags, dtype=np.int8).reshape(m.shape)
        check(lib().fuelgpu_frontier_upload_flags(m.handle, ptr(f)), m.handle)
