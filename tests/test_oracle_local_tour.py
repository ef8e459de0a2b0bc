"""Pins the local-tour oracle (oracle/fuel_oracle_tour.c: refineLocalTour, fast_exploration_manager.cpp:429-503) and
the Python bookkeeping around it (fuel_b200.exploration_manager.select_refined_ids, FrontierFinder.getViewpointsInfo
and getTopViewpointsInfo) on the REFERENCE's own fast_exploration_manager.cpp, graph_node.cpp and frontier_finder.cpp,
compiled unmodified into oracle/_ref/libfuel_ref_tour.so (oracle/tour.mk) over the reference's SDFMap and RayCaster.
Bit for bit: the refined points and yaws, refined_tour_ and ViewNode::astar_'s lambda_heu afterwards; every list of
getViewpointsInfo and getTopViewpointsInfo; the refined ids; the one-viewpoint pick.  The reference's time cut runs on
the tick clock, so max_search_time_ = max_iter.  Where the reference library is not built, the digests in
tests/golden/refpin_tour.json stand in for it.

  FUEL_REFPIN_RECORD=1 python -m pytest tests/test_oracle_local_tour.py

rewrites the digests from a run against the built reference.  The other tests here check the oracle's own parts: the
lazy search equals the same search over its own edge costs, std::priority_queue's tie order, the unreachable and
zero-length-segment branches."""
import numpy as np
import pytest

import oracle.astar as OA
import oracle.tour as OT
from fuel_b200 import exploration_manager as EM
from fuel_b200 import workloads as W
from fuel_b200.frontier_finder import FrontierFinder
from tests.refgold import refgold_fixture
from tests.test_oracle_astar import Scene

OT.build()

VM, YD, W_DIR = 2.0, 60 * 3.1415926 / 180.0, 1.5  # exploration/vm (max_vel 2.0), yd, w_dir: algorithm.xml:95-99
PRM = (VM, YD, W_DIR, 0.4, 10000.0, 100000, 400)


def run(om, w, table=None, tour_max=256):
    return OT.local_tour_batch(om, w["prob_off"], w["group_off"], w["cur_pos"], w["cur_vel"], w["cur_yaw"],
                               w["vp_pos"], w["vp_yaw"], *PRM, 1.0, tour_max=tour_max, table=table)


@pytest.fixture(scope="module", params=["office", "office3"])
def scene(request):
    g, inflate = W.office_map() if request.param == "office" else W.office3_map()
    tri = W.office_known(g, inflate)
    return g, inflate, tri, OA.Map(g, inflate, tri)


def test_lazy_search_equals_search_over_its_costs(scene):
    g, inflate, tri, om = scene
    w = W.make_local_tours(g, inflate, tri, B=40, seed=3)
    lazy = run(om, w)
    tab = run(None, w, table=lazy[3])  # an edge the lazy search never evaluated is never needed: NaN there
    for f in ("n_nodes", "n_edges", "n_evals", "n_refined", "pops", "pushes"):
        assert np.array_equal(lazy[0][f], tab[0][f]), f
    assert lazy[0]["g"].tobytes() == tab[0]["g"].tobytes()
    assert np.array_equal(lazy[1], tab[1])
    info = lazy[0]
    assert np.all(info["n_refined"][info["status"] == 0] == np.diff(w["prob_off"])[info["status"] == 0])
    assert np.all(info["pushes"] <= info["n_edges"] + 1)
    # the tour starts at cur_pos and ends at the last refined point
    for b in np.flatnonzero(info["status"] == 0):
        n = info["n_tour"][b]
        assert np.array_equal(lazy[2][b, 0], w["cur_pos"][b])
        assert np.array_equal(lazy[2][b, n - 1], w["vp_pos"][lazy[1][b, info["n_refined"][b] - 1]])


def _one(groups, cur_pos=(0.0, 0.0, 1.0)):
    """one problem from [[(pos, yaw), ...], ...]"""
    sizes = [len(x) for x in groups]
    pts = [p for grp in groups for p, _ in grp]
    return dict(prob_off=[0, len(groups)], group_off=np.concatenate([[0], np.cumsum(sizes)]),
                cur_pos=[cur_pos], cur_vel=[np.zeros(3)], cur_yaw=[0.0],
                vp_pos=np.asarray(pts, np.float64).reshape(-1, 3), vp_yaw=[y for grp in groups for _, y in grp])


def test_priority_queue_tie_order():
    """four nodes pushed at equal g: libstdc++'s pop_heap brings the third to the top after the first, so the third
    relaxes final_node first at the better cost"""
    w = _one([[((k, 0.0, 1.0), 0.0) for k in range(4)], [((9.0, 0.0, 1.0), 0.0)]])
    # edges: first -> a, b, c, d; then a, b, c, d -> final
    info, refined, _, _ = run(None, w, table=[1.0, 1.0, 1.0, 1.0, 2.0, 1.0, 1.0, 1.0])
    assert info["status"][0] == 0 and info["g"][0] == 2.0
    assert list(refined[0, :2]) == [2, 4]  # c, not b
    # pops: first, a, c, b, d, final; pushes: first, a-d, final twice; costTo: 4 from first, 1 from each of a-d
    assert info["pops"][0] == 6 and info["pushes"][0] == 7 and info["n_evals"][0] == 8


def test_unreachable_and_nan_edges():
    w = _one([[((1.0, 0.0, 1.0), 0.0)], [((2.0, 0.0, 1.0), 0.0)]])
    for table in ([np.nan, 1.0], [1.0, 1e6], [2e6, 1.0]):
        info, refined, _, _ = run(None, w, table=table)
        assert info["status"][0] == 1 and info["n_refined"][0] == 0 and info["g"][0] == 1e6
        assert np.all(refined[0] == -1)


def test_empty_middle_group_and_zero_length_segment(scene):
    g, inflate, tri, om = scene
    w = W.make_local_tours(g, inflate, tri, B=96, seed=4)
    info, refined, tour, _ = run(om, w)
    k = w["kind"]
    empty = (k == 3) & (np.diff(w["prob_off"]) > 2)
    assert empty.any() and np.all(info["status"][empty] == 1)
    assert np.all(info["n_tour"][empty] == 1) and np.array_equal(tour[empty, 0], w["cur_pos"][empty])
    # the first refined point equals cur_pos: searchPath returns 0 and the point alone is pushed (:497)
    at_pos = [b for b in np.flatnonzero((k == 4) & (np.diff(w["prob_off"]) > 1) & (info["status"] == 0))
              if np.array_equal(w["vp_pos"][refined[b, 0]], w["cur_pos"][b])]
    assert at_pos
    for b in at_pos:
        assert np.array_equal(tour[b, 1], w["cur_pos"][b])


class _F:
    def __init__(self, id_, views):
        self.id_ = id_
        self.viewpoints_ = [(np.asarray(p, np.float64), float(y), int(v)) for p, y, v in views]
        self.average_ = np.zeros(3)


def _finder(frontiers):
    ff = FrontierFinder.__new__(FrontierFinder)
    ff.frontiers_ = frontiers
    return ff


def test_get_viewpoints_info():
    far = [((3.0 + i, 0.0, 1.0), 0.1 * i, v) for i, v in enumerate([10, 9, 8, 7])]
    close = [((0.1 * i, 0.0, 1.0), 0.2 * i, v) for i, v in enumerate([20, 19, 18, 15])]
    mixed = [((0.2, 0.0, 1.0), 0.0, 30), ((2.0, 0.0, 1.0), 0.5, 29), ((0.3, 0.0, 1.0), 0.7, 28),
             ((4.0, 0.0, 1.0), 0.9, 27)]
    ff = _finder([_F(0, far), _F(1, close), _F(2, mixed)])
    pos = np.array([0.0, 0.0, 1.0])
    pts, ys = ff.getViewpointsInfo(pos, [2, 0, 1, 7], 15, 0.8)  # no cluster has id 7: no entry
    assert len(pts) == 3
    assert [list(p) for p in pts[0]] == [[2.0, 0.0, 1.0], [4.0, 0.0, 1.0]] and ys[0] == [0.5, 0.9]  # too close skipped
    assert len(pts[1]) == 2 and ys[1] == [0.0, 0.1]  # int(10 * 0.8) = 8 stops at the third
    assert len(pts[2]) == 3 and ys[2] == [0.0, 0.2, 0.4]  # all too close: the fallback pass, int(20 * 0.8) = 16
    pts, ys = ff.getViewpointsInfo(pos, [2], 1, 0.8)
    assert ys == [[0.5]]
    pts, ys = ff.getViewpointsInfo(pos, [0], 15, 0.95)  # int(9.5) = 9: only the first
    assert ys == [[0.0]]


def test_get_top_viewpoints_info():
    ff = _finder([_F(0, [((0.1, 0.0, 1.0), 0.3, 9), ((2.0, 0.0, 1.0), 0.4, 8)]), _F(1, [((0.2, 0.0, 1.0), 0.5, 9)])])
    pts, yaws, _ = ff.getTopViewpointsInfo(np.array([0.0, 0.0, 1.0]))
    assert yaws == [0.4, 0.5]  # the first far enough; else the first
    assert np.array_equal(pts[0], [2.0, 0.0, 1.0])


def test_select_refined_ids():
    points = [np.array([x, 0.0, 0.0]) for x in (1.0, 6.0, 2.0, 8.0, 3.0)]
    pos = np.zeros(3)
    assert EM.select_refined_ids(points, [0, 2, 4, 1, 3], pos, 7, 5.0)[0] == [0, 2, 4, 1]  # stops after 6 m
    assert EM.select_refined_ids(points, [1, 0, 2], pos, 7, 5.0)[0] == [1, 0, 2]  # the first far one: fewer than two
    assert EM.select_refined_ids(points, [0, 2, 4], pos, 2, 5.0)[0] == [0, 2]  # refined_num
    ids, unrefined = EM.select_refined_ids(points, [3, 1], pos, 7, 5.0)
    assert ids == [3, 1] and np.array_equal(unrefined[1], points[1])
    assert EM.ExplorationParam() == EM.ExplorationParam(True, 7, 5.0, 15, 0.8)


# ---- pinned on the compiled reference -------------------------------------------------------------------------------
G = refgold_fixture("refpin_tour.json", OT.ref_tour)


@pytest.fixture(scope="module", params=["office", "office3"])
def ref_scene(request):
    g, inflate = W.office_map() if request.param == "office" else W.office3_map()
    tri = W.office_known(g, inflate)
    s = Scene(g, inflate, tri)
    yield g, inflate, tri, s
    s.close()


def _problems(w):
    """each problem of a batch as refineLocalTour's arguments"""
    po, go = w["prob_off"], w["group_off"]
    for b in range(len(po) - 1):
        groups = [(w["vp_pos"][go[i]:go[i + 1]], w["vp_yaw"][go[i]:go[i + 1]]) for i in range(po[b], po[b + 1])]
        yield b, [p for p, _ in groups], [y for _, y in groups]


def oracle_results(om, w, prm, tour_max=4096):
    """the oracle's refineLocalTour of every problem in the reference's terms: refined points, yaws, the tour and
    lambda_heu afterwards (the reference's refineLocalTour sets 10000)"""
    info, refined, tour, ec = OT.local_tour_batch(om, *(w[k] for k in ("prob_off", "group_off", "cur_pos", "cur_vel",
                                                                          "cur_yaw", "vp_pos", "vp_yaw")),
                                                  *prm, 1.0, tour_max=tour_max)
    out = []
    for b in range(len(info)):
        ids = refined[b, :info["n_refined"][b]]
        out.append(dict(pts=w["vp_pos"][ids].reshape(-1, 3), yaws=w["vp_yaw"][ids],
                        tour=tour[b, :info["n_tour"][b]].reshape(-1, 3), lam=10000.0))
    return out, info, ec


def ref_results(s, w, prm, tour_max=4096):
    rt = OT.RefTour(s.ref, *prm[:3], *prm[4:])
    try:
        out = []
        for b, pts, ys in _problems(w):
            rp, ry, tour, lam = rt.refine(w["cur_pos"][b], w["cur_vel"][b], [w["cur_yaw"][b], 0.0, 0.0], pts, ys,
                                          tour_max=tour_max)
            out.append(dict(pts=rp.reshape(-1, 3), yaws=ry, tour=tour.reshape(-1, 3), lam=lam))
        return out
    finally:
        rt.close()


def test_refine_matches_reference(G, ref_scene):
    """make_local_tours: groups of 1 to 15 viewpoints, velocities along an edge, duplicated viewpoints, a group of one
    repeated viewpoint (all its costs equal), empty middle groups, a refined point at cur_pos, blocked lines and
    searches without a path"""
    g, inflate, tri, s = ref_scene
    w = W.make_local_tours(g, inflate, tri, B=40, seed=26)
    got, info, _ = oracle_results(s.om, w, PRM)
    G.eq(got, lambda: ref_results(s, w, PRM))
    assert set(w["kind"].tolist()) >= {0, 1, 2, 3, 4, 5} and (info["status"] == 1).any()


def _parallel_problems():
    """velocities exactly along the first edge, where the normalised dot product rounds to 1 + ulp and acos is NaN
    (the node is then unreachable from the current state through that edge), beside ordinary ones"""
    a = np.array([1.05, 0.55, 1.02])
    firsts = [[2.495133984710674, 2.0561483856663223, 1.0031458316152742],
              [1.815348141110965, -0.7357124873025123, 0.9577536973301919],
              [3.0345647604745114, -0.47713814277469146, 0.8741204803362617]]
    vp, go, po, vel = [], [0], [0], []
    for f in firsts:
        groups = [[f, [f[0] + 0.4, f[1] - 0.3, f[2]]], [[f[0] + 1.0, f[1] + 0.2, f[2]]]]
        for grp in groups:
            vp += grp
            go.append(go[-1] + len(grp))
        po.append(po[-1] + len(groups))
        vel.append((np.array(f) - a) * 0.7)
    n = len(vp)
    return dict(prob_off=np.array(po), group_off=np.array(go), cur_pos=np.repeat(a[None], 3, 0), cur_vel=np.array(vel),
                cur_yaw=np.array([0.3, -1.0, 2.0]), vp_pos=np.array(vp), vp_yaw=np.linspace(-2.0, 2.0, n))


def test_velocity_along_an_edge_matches_reference(G, ref_scene):
    g, inflate, tri, s = ref_scene
    w = _parallel_problems()
    got, info, ec = oracle_results(s.om, w, PRM)
    assert np.isnan(ec).any()  # the edge along the velocity
    G.eq(got, lambda: ref_results(s, w, PRM))


@pytest.mark.parametrize("alloc,max_iter", [(300, 100000), (1000000, 60)])
def test_pool_and_iteration_caps_match_reference(G, ref_scene, alloc, max_iter):
    g, inflate, tri, s = ref_scene
    w = W.make_local_tours(g, inflate, tri, B=12, seed=17)
    prm = PRM[:5] + (alloc, max_iter)
    got, _, _ = oracle_results(s.om, w, prm)
    G.eq(got, lambda: ref_results(s, w, prm))


def _random_frontiers(rng, n):
    fr = []
    for i in range(n):
        k = int(rng.integers(1, 20))
        visib = np.sort(rng.integers(5, 60, k))[::-1]
        c = rng.uniform(-1.5, 1.5, 3) + [1.05, 0.55, 1.02]
        pts = c + rng.normal(size=(k, 3)) * [0.9, 0.9, 0.2]
        fr.append(_F(int(rng.permutation(n + 3)[0]) if i % 5 == 4 else i,
                     [(p, float(y), int(v)) for p, y, v in zip(pts, rng.uniform(-np.pi, np.pi, k), visib)]))
    return fr


def test_viewpoint_bookkeeping_matches_reference(G, ref_scene):
    """getViewpointsInfo (max_decay cuts, too-close viewpoints, the fallback pass, view_num, ids without a cluster and
    repeated ids) and getTopViewpointsInfo on random and hand-made frontier lists"""
    g, inflate, tri, s = ref_scene
    rng = np.random.default_rng(23)
    cases = []
    for t in range(12):
        fr = _random_frontiers(rng, int(rng.integers(1, 12)))
        cur = np.array([1.05, 0.55, 1.02]) + rng.normal(size=3) * [1.0, 1.0, 0.1]
        ids = rng.integers(0, len(fr) + 2, int(rng.integers(1, 8))).tolist()
        cases.append((fr, cur, ids, int(rng.choice([1, 3, 15])), float(rng.choice([0.5, 0.8, 0.95]))))
    far = [((3.0 + i, 0.0, 1.0), 0.1 * i, v) for i, v in enumerate([10, 9, 8, 7])]
    close = [((0.1 * i, 0.0, 1.0), 0.2 * i, v) for i, v in enumerate([20, 19, 18, 15])]
    cases.append(([_F(0, far), _F(1, close)], np.array([0.0, 0.0, 1.0]), [1, 0, 1], 15, 0.8))

    def mine():
        out = []
        for fr, cur, ids, vn, md in cases:
            ff = _finder(fr)
            pts, ys = ff.getViewpointsInfo(cur, ids, vn, md)
            tp, ty, _ = ff.getTopViewpointsInfo(cur)
            out.append(dict(pts=[np.asarray(p).reshape(-1, 3) for p in pts], yaws=[np.asarray(y) for y in ys],
                            top=np.asarray(tp).reshape(-1, 3), top_yaw=np.asarray(ty)))
        return out

    def reference():
        rt = OT.RefTour(s.ref, *PRM[:3], *PRM[4:])
        try:
            out = []
            for fr, cur, ids, vn, md in cases:
                (pts, ys), (tp, ty) = OT.ref_viewpoints(fr, 0.75, cur, ids, vn, md)
                out.append(dict(pts=[p.reshape(-1, 3) for p in pts], yaws=ys, top=tp.reshape(-1, 3), top_yaw=ty))
            return out
        finally:
            rt.close()

    G.eq(mine(), reference)


def test_selection_and_pick_match_reference(G, ref_scene):
    """select_refined_ids (:139-147) and the one-viewpoint pick (:202-214, here over the view-cost oracle as the
    device's pick runs over fuelgpu_view_cost_batch) against the driver's restatement over the compiled computeCost"""
    import oracle.view as OV
    g, inflate, tri, s = ref_scene
    rng = np.random.default_rng(29)
    w = W.make_local_tours(g, inflate, tri, B=8, seed=31)
    sel = []
    for t in range(20):
        n = int(rng.integers(1, 12))
        pts = np.array([1.05, 0.55, 1.02]) + rng.normal(size=(n, 3)) * [4.0, 4.0, 0.2]
        sel.append((pts, rng.permutation(n).tolist(), np.array([1.05, 0.55, 1.02]), int(rng.choice([1, 2, 7])),
                    float(rng.choice([2.0, 5.0]))))
    picks = []
    for b, pts, ys in _problems(w):
        yaw = np.array([w["cur_yaw"][b], 0.0, 0.0])
        picks.append((w["cur_pos"][b], w["cur_vel"][b], yaw, pts[0], ys[0]))

    def oracle_pick(pos, vel, yaw, p, y):
        n = len(p)
        if n == 0:
            return -1
        vi, _ = OV.view_cost_batch(s.om, np.repeat(pos[None], n, 0), p, np.full(n, yaw[0]), y,
                                   np.repeat(vel[None], n, 0), *PRM, path_max=2)
        best, i_best = 100000.0, -1
        for i, c in enumerate(vi["cost"]):
            if c < best:
                best, i_best = c, i
        return i_best

    got = dict(ids=[np.asarray(EM.select_refined_ids(*c)[0], np.float64) for c in sel],
               pick=[float(oracle_pick(*c)) for c in picks])

    def reference():
        rt = OT.RefTour(s.ref, *PRM[:3], *PRM[4:])
        try:
            return dict(ids=[np.asarray(OT.ref_select_ids(*c), np.float64) for c in sel],
                        pick=[float(rt.pick(*c)) for c in picks])
        finally:
            rt.close()

    G.eq(got, reference)
