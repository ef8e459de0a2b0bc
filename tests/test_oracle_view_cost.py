"""Pins the view-cost oracle (oracle/fuel_oracle_view.c: orc_view_cost) and the Python mirror's cost bookkeeping
(fuel_b200/frontier_finder.py: update_cost_matrix, full_cost_matrix, path_for_tour) on the REFERENCE's own
active_perception/src/graph_node.cpp and frontier_finder.cpp, compiled unmodified with astar2.cpp into
oracle/_ref/libfuel_ref_view.so (oracle/view.mk) over the reference's SDFMap and RayCaster.  Bit for bit: kind, the
search's reason / iter_num / use_node_num, n_path, length, the path rows and cost of every pair; every costs_ /
paths_ list and the full matrix of the bookkeeping.  The reference's time cut runs on the tick clock, so
max_search_time_ = max_iter.  Where the reference library is not built, the digests in
tests/golden/refpin_view_cost.json stand in for it.

  FUEL_REFPIN_RECORD=1 python -m pytest tests/test_oracle_view_cost.py

rewrites the digests from a run against the built reference."""
import numpy as np
import pytest

import oracle.astar as OA
import oracle.view as OV
from fuel_b200 import frontier_finder as FF
from fuel_b200 import workloads as W
from tests.refgold import refgold_fixture
from tests.test_oracle_astar import Scene

OV.build()

PATH_MAX = 512
VM, YD, W_DIR = 2.0, 60 * 3.1415926 / 180.0, 1.5  # exploration/vm (max_vel 2.0), yd, w_dir: algorithm.xml:95-99


G = refgold_fixture("refpin_view_cost.json", OV.ref_view)


def flat(res):
    info, path = res
    return [[info[f].astype(np.float64) for f in OV.VIEW_DTYPE.names], path]


class ViewScene(Scene):
    def check(self, G, pr, lam=10000.0, alloc=1000000, max_iter=100000):
        got = OV.view_cost_batch(self.om, pr["p1"], pr["p2"], pr["y1"], pr["y2"], pr["v1"], VM, YD, W_DIR, 0.4, lam,
                                 alloc, max_iter, path_max=PATH_MAX)

        def reference():
            rv = OV.RefViewNode(self.ref, VM, YD, W_DIR, lam, alloc, max_iter)
            try:
                return flat(rv.cost_batch(pr["p1"], pr["p2"], pr["y1"], pr["y2"], pr["v1"], path_max=PATH_MAX))
            finally:
                rv.close()

        G.eq(flat(got), reference)
        return got[0]


def scene(maker):
    g, inflate = maker()
    tri = W.office_known(g, inflate)
    return g, inflate, tri, ViewScene(g, inflate, tri)


@pytest.fixture(scope="module")
def office():
    s = scene(W.office_map)
    yield s
    s[3].close()


@pytest.fixture(scope="module")
def office3():
    s = scene(W.office3_map)
    yield s
    s[3].close()


@pytest.mark.parametrize("which", ["office", "office3"])
def test_pairs_match_reference(G, request, which):
    g, inflate, tri, s = request.getfixturevalue(which)
    pr = W.make_view_pairs(g, inflate, tri, P=160, seed=201)
    info = s.check(G, pr)
    assert set(info["kind"].tolist()) == {1, 2, 3}                   # clear line, search, no path
    moving = np.linalg.norm(pr["v1"], axis=1) > 1e-3
    assert moving.any() and (~moving).any()


def test_out_of_box_start_equal_goal_and_velocity_edges(G, office):
    g, inflate, tri, s = office
    a = np.array([1.05, 0.55, 1.02])
    p1 = np.array([a, a, a, a, a, [0.0, 0.0, 2.5]])
    p2 = np.array([a, a + [1.0, 0.0, 0.0], a + [0.0, 0.0, 3.0], a + [1.0, 0.0, 0.0], a + [2.0, 0.0, 0.0],
                   [0.5, 0.5, 1.0]])
    v1 = np.array([[0.0, 0.0, 0.0], [0.0, 0.0, 0.0], [0.0, 0.0, 0.0], [3.0, 0.0, 0.0], [0.0, 5e-4, 0.0],
                   [1.0, 1.0, 0.0]])
    pr = dict(p1=p1, p2=p2, y1=np.array([0.0, 3.0, -3.0, 1.0, 0.0, 0.5]), y2=np.array([0.0, -3.0, 3.0, 1.0, 3.1, 0.5]),
              v1=v1)
    info = s.check(G, pr)
    assert info["kind"][0] == 1 and info["length"][0] == 0.0         # start == goal: the line, length 0
    assert info["kind"][2] != 1                                      # the line leaves the box above it


@pytest.mark.parametrize("alloc,max_iter,reason", [(300, 100000, 2), (100000, 40, 3), (1000000, 60, 3), (2, 100, 2)])
def test_caps_match_reference(G, office, alloc, max_iter, reason):
    """allocate_num 1 000 000 with a small max_iter: the oracle's pool is clamped to 26 * max_iter + 2, the
    reference's is not"""
    g, inflate, tri, s = office
    pr = W.make_view_pairs(g, inflate, tri, P=48, seed=202)
    info = s.check(G, pr, alloc=alloc, max_iter=max_iter)
    assert np.count_nonzero(info["reason"] == reason) > 0


class _Ftr:
    def __init__(self, pos, yaw):
        self.viewpoints_ = [(np.asarray(pos, np.float64), float(yaw), 0)]
        self.costs_, self.paths_ = [], []


def _lists(frontiers):
    return [[np.asarray(f.costs_, np.float64), [np.asarray(p, np.float64).reshape(-1, 3) for p in f.paths_]]
            for f in frontiers]


def test_cost_bookkeeping_matches_reference(G, office):
    """updateFrontierCostMatrix twice -- the second time after removing clusters, with removed_ids_ -- then
    getFullCostMatrix and getPathForTour, the mirror over the oracle against frontier_finder.cpp over graph_node.cpp"""
    g, inflate, tri, s = office
    pr = W.make_view_pairs(g, inflate, tri, P=24, seed=203)
    free = pr["p1"]
    lam, alloc, max_iter = 10000.0, 1000000, 100000

    def batch(p1, p2, y1, y2, v1):
        info, path = OV.view_cost_batch(s.om, p1, p2, y1, y2, v1, VM, YD, W_DIR, 0.4, lam, alloc, max_iter, PATH_MAX)
        assert np.all(info["n_path"] <= PATH_MAX)
        return info["cost"], [path[q, :info["n_path"][q]].copy() for q in range(len(info))]

    rv = OV.RefViewNode(s.ref, VM, YD, W_DIR, lam, alloc, max_iter) if G.live else None
    book = OV.RefCostBook(s.ref) if G.live else None
    try:
        def update(ftrs, first_new, removed):
            if G.live:
                book.install(ftrs, first_new, removed)
            FF.update_cost_matrix(ftrs, first_new, removed, batch)

            def reference():
                book.update()
                return [[c, p] for c, p in book.lists()]
            G.eq(_lists(ftrs), reference)

        ftrs = [_Ftr(free[i], pr["y1"][i]) for i in range(6)]
        update(ftrs, 0, [])
        # clusters 1 and 3 change: removed_ids_ holds their indices after the removal (frontier_finder.cpp:75-84)
        kept = [f for i, f in enumerate(ftrs) if i not in (1, 3)]
        ftrs = kept + [_Ftr(free[i], pr["y2"][i]) for i in range(6, 10)]
        update(ftrs, len(kept), [1, 2])
        assert all(len(f.costs_) == len(ftrs) for f in ftrs)

        for cur_vel in ([0.0, 0.0, 0.0], [0.8, -0.6, 0.1]):
            cur_pos, cur_yaw = free[12], np.array([0.3, 0.0, 0.0])
            got = FF.full_cost_matrix(ftrs, cur_pos, cur_vel, cur_yaw, batch)
            G.eq(got, lambda: book.full(cur_pos, cur_vel, cur_yaw))
        ids = [3, 0, 5, 2, 7]
        got = FF.path_for_tour(ftrs, free[13], ids, batch)
        G.eq(got, lambda: book.tour(free[13], ids))
    finally:
        if book is not None:
            book.close()
        if rv is not None:
            rv.close()
