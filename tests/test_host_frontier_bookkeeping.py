"""The host-side mirror of FrontierFinder (fuel_b200/frontier_finder.py: the list bookkeeping of searchFrontiers /
computeFrontiersToVisit / isFrontierCovered around the device calls) against the REFERENCE's own compiled
frontier_finder.cpp over a multi-frame exploration episode.  The device calls of the mirror are replaced by the oracle
here (no GPU needed), so what is compared is exactly the host logic: which stored clusters are removed when the map
changes (haveOverlap + isFrontierChanged), removed_ids_, the dormant list, id assignment, viewpoint filtering / order.
Where oracle/_ref is not built, the digests of the reference's results stand in for it (tests/refgold.py)."""
import numpy as np

import oracle as O
from fuel_b200 import workloads as W
from fuel_b200.frontier_finder import Frontier, FrontierFinder
from tests.refgold import ref_map, refgold_fixture

O.build()

MAP = dict(resolution=0.1, map_size_x=8.0, map_size_y=6.0, map_size_z=3.0, ground_height=-0.5, obstacles_inflation=0.199,
           local_bound_inflate=0.5, local_map_margin=50, default_dist=0.0, optimistic=0, signed_dist=0, p_hit=0.65, p_miss=0.35,
           p_min=0.12, p_max=0.90, p_occ=0.80, max_ray_length=4.5, virtual_ceil_height=-10.0, box_min_x=-3.6, box_min_y=-2.6,
           box_min_z=-0.3, box_max_x=3.6, box_max_y=2.6, box_max_z=2.2)
FF = dict(cluster_min=15, cluster_size_xy=1.2, cluster_size_z=10.0, min_candidate_dist=0.75, min_candidate_clearance=0.21,
          candidate_dphi=15 * 3.1415926 / 180.0, candidate_rmax=2.5, candidate_rmin=1.5, candidate_rnum=3, down_sample=3,
          min_visib_num=6, min_view_finish_fraction=0.2)
PU = dict(top_angle=0.56125, left_angle=0.69222, right_angle=0.68901, max_dist=4.5, vis_dist=1.0)


def logit(p):
    return np.log(p / (1 - p))


class FakeMap:
    """what the mirror needs from SDFMap, without a device"""

    def __init__(self, ref):
        self.shape, self.resolution_, self.map_origin_ = ref.n, ref.res, ref.origin
        self.handle = None
        self.update_min_, self.update_max_ = np.zeros(3), np.zeros(3)

    def getUpdatedBox(self, reset=False):
        return self.update_min_.copy(), self.update_max_.copy()


class OracleBackedFinder(FrontierFinder):
    """fuel_b200.FrontierFinder with every libfuelgpu call answered by the oracle (BFS cell order, like the reference)"""

    def __init__(self, fmap, g, tri_ref, inflate, **kw):
        class Env:
            sdf_map_ = fmap
        super().__init__(Env(), cluster_min=kw["cluster_min"], cluster_size_xy=kw["cluster_size_xy"], down_sample=kw["down_sample"])
        self.g, self.tri, self.inflate = g, tri_ref, inflate
        self.flag = np.zeros(fmap.shape, np.int8)

    def _changed(self, ftrs):
        return np.array([O.frontier_changed_count(self.g, self.tri, f.cells_addr_) > 0 for f in ftrs], np.uint8)

    def _clear_flags(self, addr):
        self.flag.reshape(-1)[addr] = 0

    def search_box(self, update_min, update_max):
        p = O.frontier_params(cluster_min=self.cluster_min_, cluster_size_xy=self.cluster_size_xy_, down_sample=self.down_sample_,
                              cell_order=0)
        res = O.frontier_search(self.g, self.tri, self.flag, update_min, update_max, p)
        return [Frontier(self._map, r["addr"], r["filtered"], r["average"], r["box_min"], r["box_max"]) for r in res]

    def sampleViewpointsRaw(self, ftrs):
        vp = O.view_params()
        out = [O.sample_viewpoints(self.g, self.tri, self.inflate, vp, f.average_, f.filtered_cells_) for f in ftrs]
        if not out:
            return np.zeros((0, 100, 3)), np.zeros((0, 100)), np.zeros((0, 100), np.int32)
        return np.stack([o["pos"] for o in out]), np.stack([o["yaw"] for o in out]), np.stack([o["visib"] for o in out])


def clusters(lst):
    """cells and average of each cluster of a mirror list (Frontier objects) or a reference list (dicts)"""
    return [dict(addr=f.cells_addr_, average=f.average_) if isinstance(f, Frontier) else dict(addr=f["addr"], average=f["average"])
            for f in lst]


def visit_list(lst):
    """frontiers_ with ids and viewpoints; the reference sorts them by visib_num_ (std::sort, tie order unspecified), so
    they are compared as a sorted multiset"""
    out = []
    for f in lst:
        if isinstance(f, Frontier):
            vs = sorted((-v[2], v[1], tuple(v[0])) for v in f.viewpoints_)
            out.append(dict(addr=f.cells_addr_, average=f.average_, id=f.id_, views=[list(v) for v in vs]))
        else:
            vs = sorted(zip(-f["view_visib"], f["view_yaw"], map(tuple, f["view_pos"])))
            out.append(dict(addr=f["addr"], average=f["average"], id=f["id"], views=[list(v) for v in vs]))
    return out


G = refgold_fixture()


def test_exploration_episode_matches_reference(G):
    ref = ref_map(**MAP)
    n = ref.n
    rng = np.random.default_rng(12)
    inflate = (rng.random(n) < 0.003).astype(np.int8)
    X, Y, Z = np.meshgrid(*[np.arange(k) for k in n], indexing="ij")
    tri = np.full(n, W.UNKNOWN, np.uint8)
    ref.inflate[:] = 0
    ref.occupancy[:] = logit(0.12) - 0.01
    g = ref.grid((-3.6, -2.6, -0.3), (3.6, 2.6, 2.2))
    rff = O.RefFrontierFinder(ref, PU, **FF) if G.live else None
    fmap = FakeMap(ref)
    inf_known = np.zeros(n, np.int8)
    mine = OracleBackedFinder(fmap, g, tri, inf_known, **FF)
    mine.setViewParams(min_visib_num=FF["min_visib_num"], min_view_finish_fraction=FF["min_view_finish_fraction"])
    occ = ref.occupancy.reshape(n)
    total_removed = 0
    # the robot reveals one ball of space per frame, moving through the room
    path = [(18, 20, 12), (28, 24, 12), (38, 30, 13), (48, 32, 12), (58, 36, 12), (60, 22, 12), (46, 16, 12), (30, 40, 14)]
    for k, c in enumerate(path):
        ball = ((X - c[0]) ** 2 + (Y - c[1]) ** 2 + 3.0 * (Z - c[2]) ** 2) < (11 + (k % 3)) ** 2
        newly = ball & (tri == W.UNKNOWN)
        tri[newly] = np.where(inflate[newly] == 1, W.OCCUPIED, W.FREE)
        occ[newly] = np.where(inflate[newly] == 1, logit(0.90), logit(0.12))
        inf_known[newly] = inflate[newly]
        ref.inflate[:] = inf_known.reshape(-1)
        idx = np.argwhere(newly)
        assert len(idx)
        umin = ref.origin + idx.min(axis=0) * ref.res
        umax = ref.origin + (idx.max(axis=0) + 1) * ref.res
        fmap.update_min_, fmap.update_max_ = umin, umax
        # reference: searchFrontiers(); computeFrontiersToVisit()   |   mirror: the same two calls
        mine.searchFrontiers()
        total_removed += len(mine.removed_ids_)

        def ref_search():
            ref.R.ref_map_set_updated_box(ref.h, O._p(umin), O._p(umax))
            tmp_ref = rff.search_frontiers()
            return [rff.removed_ids(), clusters(tmp_ref), rff.flags.copy()]
        G.eq([list(mine.removed_ids_), clusters(mine.tmp_frontiers_), mine.flag.reshape(-1)], ref_search)
        mine.computeFrontiersToVisit()

        def ref_visit():
            visit_ref, dormant_ref = rff.compute_to_visit()
            return [visit_list(visit_ref), clusters(dormant_ref)]
        G.eq([visit_list(mine.frontiers_), clusters(mine.dormant_frontiers_)], ref_visit)
        for a in mine.frontiers_:
            assert [v[2] for v in a.viewpoints_] == sorted((v[2] for v in a.viewpoints_), reverse=True)
    assert total_removed >= 3 and len(mine.frontiers_) >= 2   # the episode did exercise removal and survival
    if rff is not None:
        rff.close()
    ref.close()
