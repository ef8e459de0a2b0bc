"""fuelgpu_local_tour_batch[_dev] (FastExplorationManager::refineLocalTour) on the H100 against the CPU oracle
(oracle.tour: the same graph and DijkstraSearch with each costTo evaluated lazily through the view-cost oracle).
status, n_nodes, n_edges, n_refined, refined, n_tour and the tour rows bit for bit; g bit for bit where |cur_vel| <=
1e-3 and within 4 ulps elsewhere (the device's acos on the first node's edges)."""
import ctypes as C

import numpy as np
import pytest
import torch

import oracle.astar as OA
import oracle.tour as OT
from fuel_b200 import exploration_manager as EM
from fuel_b200 import workloads as W
from fuel_b200._lib import FuelAstarParams, FuelGpuError, FuelLocalTourParams, FuelViewCostParams, lib
from fuel_b200.view_node import ViewNode, view_cost_batch
from tests.helpers import make_sdf_map

pytestmark = pytest.mark.gpu

VM, YD, W_DIR = ViewNode.vm_, ViewNode.yd_, ViewNode.w_dir_
# the iteration cap keeps the oracle's failing searches short; the device runs the same cap
PRM = dict(vm=VM, yd=YD, w_dir=W_DIR, resolution=0.4, lambda_heu=10000.0, allocate_num=100000, max_iter=400)
G_ULPS = 4
TOUR_MAX = 256


def _scene(fuel, which):
    g, inflate = W.office_map() if which == "office" else W.office3_map()
    tri = W.office_known(g, inflate)
    return g, inflate, tri, make_sdf_map(fuel, g, inflate, tri), OA.Map(g, inflate, tri)


@pytest.fixture(scope="module")
def office(fuel):
    s = _scene(fuel, "office")
    yield s
    s[3].close()


@pytest.fixture(scope="module")
def office3(fuel):
    s = _scene(fuel, "office3")
    yield s
    s[3].close()


def _args(w):
    return (w["prob_off"], w["group_off"], w["cur_pos"], w["cur_vel"], w["cur_yaw"], w["vp_pos"], w["vp_yaw"])


def run_device(m, w, **kw):
    kw = {**PRM, "tour_max": TOUR_MAX, **kw}
    return EM.local_tour_batch(m, *_args(w), **kw)


def run_oracle(om, w, table=None, kmax=None, tour_max=TOUR_MAX):
    p = PRM
    return OT.local_tour_batch(om, *_args(w), p["vm"], p["yd"], p["w_dir"], p["resolution"], p["lambda_heu"],
                               p["allocate_num"], p["max_iter"], 1.0, kmax=kmax, tour_max=tour_max, table=table)


def g_ulps(got, want):
    nan = np.isnan(want)
    assert np.array_equal(np.isnan(got), nan)
    if not (~nan).any():
        return 0.0
    return float(np.max(np.abs(got[~nan] - want[~nan]) / np.spacing(np.abs(want[~nan]))))


def assert_same(got, want, w):
    gi, gr, gt = got[:3]
    wi, wr, wt = want[:3]
    for f in ("status", "n_nodes", "n_edges", "n_refined", "n_tour"):
        bad = np.flatnonzero(gi[f] != wi[f])
        assert bad.size == 0, "%s differs at %s: %s vs %s" % (f, bad[:5], gi[f][bad[:3]], wi[f][bad[:3]])
    assert np.array_equal(gr, wr), "refined differs at %s" % np.flatnonzero(np.any(gr != wr, axis=1))[:5]
    assert np.array_equal(gt, wt), "tour differs at %s" % np.flatnonzero(np.any(gt != wt, axis=(1, 2)))[:5]
    still = np.linalg.norm(w["cur_vel"], axis=1) <= 1e-3
    assert np.array_equal(gi["g"][still], wi["g"][still])
    for f in ("n_evals", "pops", "pushes"):  # the same costs give the same search
        assert np.array_equal(gi[f][still], wi[f][still]), f
    u = g_ulps(gi["g"][~still], wi["g"][~still])
    assert u <= G_ULPS, "g off by %.1f ulps" % u
    return u


def edge_pairs(w):
    """every edge's (p1, p2, y1, y2, v1) in addEdge order (fast_exploration_manager.cpp:441-469)"""
    p1, p2, y1, y2, v1 = [], [], [], [], []
    po, go = w["prob_off"], w["group_off"]
    for b in range(len(po) - 1):
        last = [(w["cur_pos"][b], w["cur_yaw"][b], w["cur_vel"][b])]
        ng = po[b + 1] - po[b]
        for i in range(ng):
            a, e = go[po[b] + i], go[po[b] + i + 1]
            cur = []
            for j in range(a, e):
                for (q, y, v) in last:
                    p1.append(q), y1.append(y), v1.append(v)
                    p2.append(w["vp_pos"][j]), y2.append(w["vp_yaw"][j])
                cur.append((w["vp_pos"][j], w["vp_yaw"][j], np.zeros(3)))
                if i == ng - 1:
                    break
            last = cur
    return tuple(np.asarray(x, np.float64) for x in (p1, p2, y1, y2, v1))


@pytest.mark.parametrize("which", ["office", "office3"])
def test_batch_b256_matches_oracle(request, which):
    g, inflate, tri, m, om = request.getfixturevalue(which)
    w = W.make_local_tours(g, inflate, tri, B=256)
    got = run_device(m, w, edge_cost=True)
    want = run_oracle(om, w)
    u = assert_same(got, want, w)
    info = got[0]
    print("%s: statuses %s, %d edges costed eagerly, %d evaluated lazily by the reference, max g difference %.1f ulps"
          % (which, np.bincount(info["status"], minlength=4), info["n_edges"].sum(), want[0]["n_evals"].sum(), u))
    assert np.count_nonzero(info["status"] == EM.TOUR_OK) > 200
    assert np.count_nonzero(info["status"] == EM.TOUR_UNREACHABLE) > 0
    # the edge table is fuelgpu_view_cost_batch's on the same pairs, bit for bit
    p1, p2, y1, y2, v1 = edge_pairs(w)
    vc, _ = view_cost_batch(m, p1, p2, y1, y2, v1, path_max=0, **PRM)
    assert got[3].tobytes() == vc["cost"].tobytes()
    # the oracle's search over the device's edge costs reproduces the device's search exactly, velocity included
    tab = run_oracle(None, w, table=got[3])
    assert np.array_equal(tab[1], got[1])
    assert tab[0]["g"].tobytes() == info["g"].tobytes()
    for f in ("n_evals", "pops", "pushes", "n_refined"):
        assert np.array_equal(tab[0][f], info[f]), f
    # the reference's lazy search evaluates every edge it needs: where it evaluated one, the costs agree
    lazy = want[3]
    ev = ~np.isnan(lazy)
    still = np.linalg.norm(v1, axis=1) <= 1e-3
    assert np.array_equal(lazy[ev & still], got[3][ev & still])


def test_dev_entry_equals_host_entry_and_bad_rows(office):
    g, inflate, tri, m, om = office
    w = W.make_local_tours(g, inflate, tri, B=48, seed=5)
    w["cur_pos"][3, 1] = np.nan
    w["cur_vel"][7, 2] = np.inf
    w["cur_yaw"][9] = -np.inf
    w["vp_pos"][w["group_off"][w["prob_off"][12]], 0] = np.nan  # the first viewpoint of problem 12
    bad = [3, 7, 9, 12]
    host = run_device(m, w, edge_cost=True)
    want = run_oracle(om, w)
    assert np.all(host[0]["status"][bad] == EM.TOUR_BAD_INPUT)
    assert np.all(host[1][bad] == -1) and np.all(host[2][bad] == 0) and np.all(host[0]["n_tour"][bad] == 0)
    good = np.setdiff1d(np.arange(48), bad)
    assert_same(tuple(x[good] for x in host[:3]), tuple(x[good] for x in want[:3]),
                {"cur_vel": w["cur_vel"][good]})
    dev = torch.device("cuda")
    t = {k: torch.tensor(w[k], device=dev) for k in ("cur_pos", "cur_vel", "cur_yaw", "vp_pos", "vp_yaw")}
    B, kmax = 48, host[1].shape[1]
    dinfo = torch.zeros(B * EM.TOUR_INFO_DTYPE.itemsize, dtype=torch.uint8, device=dev)
    dref = torch.zeros((B, kmax), dtype=torch.int32, device=dev)
    dtour = torch.zeros((B, TOUR_MAX, 3), dtype=torch.float64, device=dev)
    dec = torch.zeros(len(host[3]), dtype=torch.float64, device=dev)
    prm = FuelLocalTourParams(FuelViewCostParams(VM, YD, W_DIR, FuelAstarParams(0.4, 10000.0, 100000, 400)), 1.0)
    po, go = (np.ascontiguousarray(w[k], np.int32) for k in ("prob_off", "group_off"))
    torch.cuda.synchronize()
    rc = lib().fuelgpu_local_tour_batch_dev(m.handle, B, po.ctypes.data, go.ctypes.data, t["cur_pos"].data_ptr(),
                                            t["cur_vel"].data_ptr(), t["cur_yaw"].data_ptr(), t["vp_pos"].data_ptr(),
                                            t["vp_yaw"].data_ptr(), C.byref(prm), dinfo.data_ptr(), kmax,
                                            dref.data_ptr(), TOUR_MAX, dtour.data_ptr(), dec.data_ptr())
    assert rc == 0
    m.synchronize()
    info = np.frombuffer(dinfo.cpu().numpy().tobytes(), dtype=EM.TOUR_INFO_DTYPE)
    assert info.tobytes() == host[0].tobytes()
    assert np.array_equal(dref.cpu().numpy(), host[1]) and np.array_equal(dtour.cpu().numpy(), host[2])
    assert dec.cpu().numpy().tobytes() == host[3].tobytes()


def test_einval(office):
    m = office[3]
    one = dict(prob_off=[0, 2], group_off=[0, 2, 3], cur_pos=np.zeros((1, 3)) + 1.0, cur_vel=np.zeros((1, 3)),
               cur_yaw=[0.0], vp_pos=np.ones((3, 3)), vp_yaw=np.zeros(3))
    run_device(m, one)  # a valid problem

    def refused(**change):
        w = dict(one, **{k: v for k, v in change.items() if k in one})
        kw = {k: v for k, v in change.items() if k not in one}
        with pytest.raises(FuelGpuError) as e:
            run_device(m, w, **kw)
        assert e.value.code == -1
    refused(prob_off=[0, 0], group_off=[0])  # a problem with no group
    refused(group_off=[0, 3, 3])  # an empty last group
    n = EM.TOUR_MAX_NODES  # 1 + (n - 1) + 1 nodes
    refused(prob_off=[0, 2], group_off=[0, n - 1, n], vp_pos=np.ones((n, 3)), vp_yaw=np.zeros(n))
    run_device(m, dict(one, group_off=[0, n - 2, n - 1], vp_pos=np.ones((n - 1, 3)), vp_yaw=np.zeros(n - 1)))
    refused(vm=0.0)
    refused(yd=np.nan)
    refused(resolution=0.0)
    refused(tour_lambda_heu=np.inf)
    refused(tour_max=0)
    refused(kmax=1)
    prm = FuelLocalTourParams(FuelViewCostParams(VM, YD, W_DIR, FuelAstarParams(0.4, 1.0, 1000, 100)), 1.0)
    assert lib().fuelgpu_local_tour_batch(m.handle, -1, None, None, None, None, None, None, None, C.byref(prm), None, 1,
                                          None, 1, None, None) == -1  # B < 0


def test_tour_max_overflow_and_recall(office):
    g, inflate, tri, m, om = office
    w = W.make_local_tours(g, inflate, tri, B=64, seed=11)
    full = run_device(m, w)
    need = full[0]["n_tour"]
    small = int(np.median(need[full[0]["status"] == EM.TOUR_OK]))
    cut = run_device(m, w, tour_max=small)
    over = need > small
    assert over.any()
    assert np.all(cut[0]["status"][over & (full[0]["status"] == EM.TOUR_OK)] == EM.TOUR_TRUNCATED)
    assert np.array_equal(cut[0]["n_tour"], need)
    assert np.array_equal(cut[2], full[2][:, :small])
    again = run_device(m, w, tour_max=int(need.max()))
    assert np.all(again[0]["status"] != EM.TOUR_TRUNCATED)
    assert np.array_equal(again[0]["status"], full[0]["status"])
    r = min(TOUR_MAX, int(need.max()))
    assert np.array_equal(again[2][:, :r], full[2][:, :r])
    want = run_oracle(om, w, tour_max=small)
    assert np.array_equal(cut[0]["status"], want[0]["status"]) and np.array_equal(cut[2], want[2])


def test_office_sequence(fuel):
    """searchFrontiers -> computeFrontiersToVisit -> getTopViewpointsInfo -> getFullCostMatrix -> a fixed tour order
    for LKH -> select_refined_ids -> getViewpointsInfo -> refineLocalTour, and the one-viewpoint pick"""
    g, inflate = W.office_map()
    tri = W.office_known(g, inflate)
    m = make_sdf_map(fuel, g, inflate, tri)
    om = OA.Map(g, inflate, tri)
    saved = dict(ViewNode.astar_)
    try:
        ViewNode.astar_ = dict(saved, max_iter=400, allocate_num=100000)
        env = fuel.EDTEnvironment()
        env.setMap(m)
        ff = fuel.FrontierFinder(env)
        m.update_min_, m.update_max_ = g.origin.copy(), g.map_max.copy()
        ff.searchFrontiers()
        ff.computeFrontiersToVisit()
        assert len(ff.frontiers_) >= 4
        pos = ff.frontiers_[0].viewpoints_[0][0] + np.array([0.3, -0.2, 0.0])
        vel, yaw = np.array([0.4, -0.1, 0.0]), np.array([0.4, 0.0, 0.0])
        points, yaws, _ = ff.getTopViewpointsInfo(pos)
        ff.updateFrontierCostMatrix()
        mat = ff.getFullCostMatrix(pos, vel, yaw)
        order = [int(i) - 1 for i in np.argsort(mat[0, 1:], kind="stable") + 1]  # stands for LKH's tour
        par = EM.ExplorationParam()
        ids, _ = EM.select_refined_ids(points, order, pos, par.refined_num, par.refined_radius)
        assert 2 <= len(ids) <= par.refined_num
        n_points, n_yaws = ff.getViewpointsInfo(pos, ids, par.top_view_num, par.max_decay)
        assert len(n_points) == len(ids)
        ViewNode.astar_["lambda_heu"] = 10000.0
        pts, ys, tour = EM.refineLocalTour(pos, vel, yaw, n_points, n_yaws, sdf_map=m)
        assert ViewNode.astar_["lambda_heu"] == 10000.0
        w = dict(prob_off=np.array([0, len(n_points)]),
                 group_off=np.concatenate([[0], np.cumsum([len(p) for p in n_points])]),
                 cur_pos=pos.reshape(1, 3), cur_vel=vel.reshape(1, 3), cur_yaw=yaw[:1],
                 vp_pos=np.concatenate([np.asarray(p).reshape(-1, 3) for p in n_points]),
                 vp_yaw=np.concatenate([np.asarray(y, np.float64) for y in n_yaws]))
        want = run_oracle(om, w, tour_max=4096)
        assert want[0]["status"][0] == EM.TOUR_OK
        k = int(want[0]["n_refined"][0])
        assert np.array_equal(pts, w["vp_pos"][want[1][0, :k]]) and np.array_equal(ys, w["vp_yaw"][want[1][0, :k]])
        assert np.array_equal(tour, want[2][0, :int(want[0]["n_tour"][0])])
        # the one-viewpoint pick over the first refined frontier's viewpoints
        i = EM.pick_one_viewpoint(pos, n_points[0], n_yaws[0], vel, yaw, sdf_map=m)
        import oracle.view as OV
        a = ViewNode.astar_
        n = len(n_points[0])
        vi, _ = OV.view_cost_batch(om, np.repeat(pos[None], n, 0), n_points[0], np.full(n, yaw[0]), n_yaws[0],
                                   np.repeat(vel[None], n, 0), VM, YD, W_DIR, a["resolution"], a["lambda_heu"],
                                   a["allocate_num"], a["max_iter"], path_max=2)
        best, want_i = 100000.0, -1
        for q, c in enumerate(vi["cost"]):
            if c < best:
                best, want_i = c, q
        assert i == want_i
    finally:
        ViewNode.astar_ = saved
        m.close()
