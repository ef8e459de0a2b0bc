"""Pins the A* oracle (oracle/fuel_oracle_astar.c) on the REFERENCE's own path_searching/src/astar2.cpp, compiled
unmodified into oracle/_ref/libfuel_ref_astar.so (oracle/astar.mk) over the reference's SDFMap and RayCaster, with
shortenPath and planExploreMotion's branch restated over them (oracle/ref_astar_wrap.cpp).  Bit for bit: status, reason,
iter_num, use_node_num, the raw path, early_terminate_cost, the shortened tour, branch, length and next_goal.  The
reference's time cut runs on a tick clock (one second per ros::Time::now()), so max_search_time_ = max_iter is the
oracle's iteration cap.  Where the reference library is not built, the digests in tests/golden/refpin_astar.json stand
in for it.

  FUEL_REFPIN_RECORD=1 python -m pytest tests/test_oracle_astar.py

rewrites the digests from a run against the built reference."""
import numpy as np
import pytest

import oracle as O
import oracle.astar as OA
from fuel_b200 import workloads as W
from tests.refgold import refgold_fixture

OA.build()

PATH_MAX, W_MAX = 512, 32


def logit(p):
    return np.log(p / (1 - p))


G = refgold_fixture("refpin_astar.json", OA.ref_astar)


def flat(res):
    info, path, n_wp, wp = res
    return [[info[f].astype(np.float64) for f in OA.INFO_DTYPE.names], path, n_wp, wp]


class Scene:
    """one map for both sides: the oracle's occupancy byte and, where it is built, the reference's SDFMap holding the
    same inflate bits and tri-state (as log-odds) with the same exploration box"""

    def __init__(self, g, inflate, tri):
        self.g, self.om = g, OA.Map(g, inflate, tri)
        self.ref = None
        if OA.ref_astar() is not None:
            p = dict(resolution=g.res, map_size_x=g.n[0] * g.res, map_size_y=g.n[1] * g.res, map_size_z=g.n[2] * g.res,
                     ground_height=g.origin[2], obstacles_inflation=0.199, local_bound_inflate=0.5, local_map_margin=50,
                     default_dist=0.0, optimistic=0, signed_dist=0, p_hit=0.65, p_miss=0.35, p_min=0.12, p_max=0.90,
                     p_occ=0.80, max_ray_length=4.5, virtual_ceil_height=-10.0)
            for k, a in enumerate("xyz"):
                p["box_min_" + a], p["box_max_" + a] = g.box_min[k], g.box_max[k]
            r = O.RefSDFMap(**p)
            assert r.n == g.n and np.array_equal(r.origin, g.origin)
            r.inflate[:] = np.asarray(inflate).reshape(-1)
            r.occupancy[:] = np.where(tri == W.UNKNOWN, logit(0.12) - 0.01,
                                      np.where(tri == W.OCCUPIED, logit(0.90), logit(0.12))).reshape(-1)
            self.ref = r

    def check(self, G, start, goal, res, lam, alloc, max_iter):
        got = OA.search_batch(self.om, start, goal, res, lam, alloc, max_iter, path_max=PATH_MAX, w_max=W_MAX)

        def reference():
            ra = OA.RefAstar(self.ref, res, lam, alloc, max_iter)
            try:
                return flat(ra.search_batch(start, goal, path_max=PATH_MAX, w_max=W_MAX))
            finally:
                ra.close()

        G.eq(flat(got), reference)
        return got[0]

    def close(self):
        if self.ref is not None:
            self.ref.close()


@pytest.fixture(scope="module")
def office():
    g, inflate = W.office_map()
    tri = W.office_known(g, inflate)
    s = Scene(g, inflate, tri)
    yield g, inflate, tri, s
    s.close()


@pytest.fixture(scope="module")
def office3():
    g, inflate = W.office3_map()
    tri = W.office_known(g, inflate)
    s = Scene(g, inflate, tri)
    yield g, inflate, tri, s
    s.close()


@pytest.mark.parametrize("res,lam", [(0.2, 1.0), (0.4, 10000.0)])
def test_office_queries_match_reference(G, office, res, lam):
    g, inflate, tri, s = office
    q = W.make_path_queries(g, inflate, tri, B=96, seed=101)
    info = s.check(G, q["start"], q["goal"], res, lam, 40000, 100000)
    assert np.count_nonzero(info["status"] == 1) > 20 and set(info["branch"][info["status"] == 1].tolist()) == {1, 2, 3}


@pytest.mark.parametrize("res,lam", [(0.2, 1.0), (0.4, 10000.0)])
def test_office3_queries_match_reference(G, office3, res, lam):
    g, inflate, tri, s = office3
    q = W.make_path_queries(g, inflate, tri, B=64, seed=102)
    s.check(G, q["start"], q["goal"], res, lam, 20000, 100000)


@pytest.mark.parametrize("alloc,max_iter,reason", [(300, 100000, 2), (100000, 40, 3), (2, 100, 2)])
def test_caps_match_reference(G, office, alloc, max_iter, reason):
    g, inflate, tri, s = office
    q = W.make_path_queries(g, inflate, tri, B=48, seed=103)
    info = s.check(G, q["start"], q["goal"], 0.2, 1.0, alloc, max_iter)
    assert np.count_nonzero(info["reason"] == reason) > 0
    if reason == 3:
        assert np.all(info["early_terminate_cost"][info["reason"] == 3] > 0)


def test_open_set_exhausted_start_equal_goal_and_outside_box(G, office):
    g, inflate, tri, s = office
    q = W.make_path_queries(g, inflate, tri, B=64, seed=104)
    unk = q["kind"] == 2
    st = np.concatenate([q["start"][unk][:4], q["start"][:3], [[0.0, 0.0, 2.5], [-9.5, 0.0, 1.0]]])
    gl = np.concatenate([q["goal"][unk][:4], q["start"][:3], [[1.0, 1.0, 1.0], [-8.0, 0.5, 1.0]]])
    info = s.check(G, st, gl, 0.2, 1.0, 40000, 100000)
    assert np.count_nonzero(info["reason"][:4] == 1) >= 2                  # goals in unknown: open set exhausted
    assert np.all(info["tour_status"][4:7] == 2) and np.all(info["n_wp"][4:7] == 1)  # start == goal: one point
    assert np.all(info["reason"][7:] == 1)                                  # start outside the box: no neighbour in it


def test_lattice_ties_match_reference(G):
    """an all-known empty box, start and goal on lattice diagonals: f ties everywhere, and only libstdc++'s heap order
    reproduces the reference's path"""
    g = W.Grid((60, 60, 30), (-3.0, -3.0, -1.5), 0.1, box_min=(-2.95, -2.95, -1.45), box_max=(2.95, 2.95, 1.45))
    inflate, tri = np.zeros(g.n, np.int8), np.full(g.n, W.FREE, np.uint8)
    s = Scene(g, inflate, tri)
    try:
        k = np.arange(-5, 6) * 0.2
        off = np.array([0.013, 0.027, 0.031])  # off the voxel corners: shortenPath's rays must meet their end voxel
        start = np.stack([k, k, 0.5 * k], axis=1) + off
        goal = np.stack([-k, k + 0.4, -0.5 * k], axis=1) + off
        for res, lam in ((0.2, 1.0), (0.2, 0.0), (0.4, 10000.0)):
            info = s.check(G, start, goal, res, lam, 20000, 100000)
            assert np.all(info["status"] == 1)
    finally:
        s.close()
