"""fuelgpu_global_tour_batch[_dev] (the ATSP of FastExplorationManager::findGlobalTour, solved exactly) on the H100
against the CPU oracle (oracle.gtour: the same Held-Karp table, reconstruction and count): status, n, n_optimal, cost
and indices exactly equal."""

import numpy as np
import pytest
import torch

import oracle.astar as OA
import oracle.gtour as OG
import oracle.tour as OT
from fuel_b200 import exploration_manager as EM
from fuel_b200 import workloads as W
from fuel_b200._lib import FuelGpuError, lib
from fuel_b200.view_node import ViewNode
from tests.helpers import make_sdf_map

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def office(fuel):
    g, inflate = W.office_map()
    tri = W.office_known(g, inflate)
    m = make_sdf_map(fuel, g, inflate, tri)
    yield g, inflate, tri, m
    m.close()


def _batch(mats):
    dims = np.array([m.shape[0] for m in mats], np.int32)
    return dims, np.concatenate([np.asarray(m, np.float64).reshape(-1) for m in mats])


def check_same(m, dims, cost):
    got = EM.global_tour_batch(m, dims, cost)
    want = OG.global_tour_batch(dims, cost)
    assert got[0].tobytes() == want[0].tobytes()
    assert np.array_equal(got[1], want[1])
    return got


def test_office_sized_batch(office):
    mats = W.make_global_tours(14, B=256, seed=1)
    info, _ = check_same(office[3], *_batch(list(mats)))
    assert np.all(info["status"] == EM.GTOUR_OK) and np.all(info["n"] == 14)


def test_every_size_in_one_batch(office):
    mats = [W.make_global_tours(n, seed=100 + n, kind="random" if n % 2 else "geometric")[0] for n in range(1, 21)]
    mats += [np.full((n + 1, n + 1), 2.5) for n in (1, 5, 9)]  # every tour optimal
    # 13! optimal tours: the count saturates
    mats += [np.zeros((14, 14))]
    info, idx = check_same(office[3], *_batch(mats))
    assert np.all(info["status"] == EM.GTOUR_OK)
    assert info["n_optimal"][-1] == 2 ** 31 - 1 and info["n_optimal"][-2] == 362880  # 9!
    assert idx[:1].tolist() == [0]  # n = 1


def test_groups_under_the_budget(office):
    # 12 * 2^20 * 20 B per n = 20 table: 17 of them exceed one 4 GiB group
    mats = list(W.make_global_tours(20, B=17, seed=3)) + list(W.make_global_tours(6, B=40, seed=4, kind="random"))
    order = np.random.default_rng(5).permutation(len(mats))
    check_same(office[3], *_batch([mats[i] for i in order]))


def test_bad_and_too_large_rows(office):
    mats = list(W.make_global_tours(9, B=12, seed=6))
    for i, v in zip((1, 3, 5, 7, 8), (np.nan, np.inf, -np.inf, 3e7, -3e7)):
        mats[i][2, 4] = v
    mats[10][3, 3] = np.nan  # the diagonal is never read
    mats.insert(4, W.make_global_tours(21, seed=7)[0])
    mats.insert(9, W.make_global_tours(40, seed=8)[0])
    info, idx = check_same(office[3], *_batch(mats))
    st = info["status"]
    assert st[4] == EM.GTOUR_TOO_LARGE and st[9] == EM.GTOUR_TOO_LARGE
    assert [int(s) for s in st].count(EM.GTOUR_BAD_INPUT) == 5
    assert st[12] == EM.GTOUR_OK  # the NaN diagonal
    off = np.concatenate([[0], np.cumsum(info["n"])])
    for b in np.nonzero(st != EM.GTOUR_OK)[0]:
        assert np.all(idx[off[b]:off[b + 1]] == -1) and info["cost"][b] == 0 and info["n_optimal"][b] == 0


def test_dev_entry_matches_host(office):
    m = office[3]
    mats = list(W.make_global_tours(14, B=32, seed=9)) + [W.make_global_tours(22, seed=10)[0]]
    mats[5][1, 2] = np.nan
    dims, cost = _batch(mats)
    host = EM.global_tour_batch(m, dims, cost)
    dev = torch.device("cuda")
    dcost = torch.tensor(cost, device=dev)
    dinfo = torch.zeros(len(dims) * EM.GTOUR_INFO_DTYPE.itemsize, dtype=torch.uint8, device=dev)
    didx = torch.zeros(int(dims.sum()) - len(dims), dtype=torch.int32, device=dev)
    torch.cuda.synchronize()
    rc = lib().fuelgpu_global_tour_batch_dev(m.handle, len(dims), dims.ctypes.data, dcost.data_ptr(),
                                             dinfo.data_ptr(), didx.data_ptr())
    assert rc == 0
    m.synchronize()
    assert dinfo.cpu().numpy().tobytes() == host[0].tobytes()
    assert np.array_equal(didx.cpu().numpy(), host[1])


def test_einval(office):
    m = office[3]
    L = lib()
    dims = np.array([3], np.int32)
    cost = np.ones(9)
    info = np.zeros(1, EM.GTOUR_INFO_DTYPE)
    idx = np.zeros(2, np.int32)
    p = lambda a: a.ctypes.data
    assert L.fuelgpu_global_tour_batch(m.handle, 1, p(dims), p(cost), p(info), p(idx)) == 0
    for h, B, d, c, i, x in ((None, 1, p(dims), p(cost), p(info), p(idx)),  # null map
                             (m.handle, -1, p(dims), p(cost), p(info), p(idx)),  # B < 0
                             (m.handle, 1, None, p(cost), p(info), p(idx)),
                             (m.handle, 1, p(dims), None, p(info), p(idx)),
                             (m.handle, 1, p(dims), p(cost), None, p(idx)),
                             (m.handle, 1, p(dims), p(cost), p(info), None)):
        assert L.fuelgpu_global_tour_batch(h, B, d, c, i, x) == -1
        assert L.fuelgpu_global_tour_batch_dev(h, B, d, c, i, x) == -1
    for bad in (1, 0, -3):  # n < 1
        dd = np.array([3, bad], np.int32)
        assert L.fuelgpu_global_tour_batch(m.handle, 2, p(dd), p(cost), p(info), p(idx)) == -1
        assert L.fuelgpu_global_tour_batch_dev(m.handle, 2, p(dd), p(cost), p(info), p(idx)) == -1
        with pytest.raises(FuelGpuError) as e:
            EM.global_tour_batch(m, [bad], np.ones(max(bad, 0) ** 2))
        assert e.value.code == -1
    assert L.fuelgpu_global_tour_batch(m.handle, 0, None, None, None, None) == 0  # an empty batch


def test_office_sequence(fuel, office):
    """searchFrontiers -> computeFrontiersToVisit -> findGlobalTour (device) against the oracle's tour of the same
    matrix, then select_refined_ids -> getViewpointsInfo -> refineLocalTour over that tour against the oracle chain"""
    g, inflate, tri, m = office
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
        n = len(ff.frontiers_)
        assert 4 <= n <= EM.GTOUR_MAX_CLUSTERS
        pos = ff.frontiers_[0].viewpoints_[0][0] + np.array([0.3, -0.2, 0.0])
        vel, yaw = np.array([0.4, -0.1, 0.0]), np.array([0.4, 0.0, 0.0])
        points, yaws, _ = ff.getTopViewpointsInfo(pos)
        indices, global_tour = EM.findGlobalTour(ff, pos, vel, yaw)
        mat = ff.getFullCostMatrix(pos, vel, yaw)
        st, cost, nopt, want = OG.global_tour(mat)
        assert st == OG.GTOUR_OK and indices == want.tolist()
        assert sorted(indices) == list(range(n))
        assert OG.tour_cost(OG.int_matrix(mat), indices) == cost
        assert np.array_equal(global_tour, ff.getPathForTour(pos, indices))
        par = EM.ExplorationParam()
        ids, _ = EM.select_refined_ids(points, indices, pos, par.refined_num, par.refined_radius)
        assert 2 <= len(ids) <= par.refined_num
        n_points, n_yaws = ff.getViewpointsInfo(pos, ids, par.top_view_num, par.max_decay)
        ViewNode.astar_["lambda_heu"] = 10000.0
        pts, ys, tour = EM.refineLocalTour(pos, vel, yaw, n_points, n_yaws, sdf_map=m)
        w = (np.array([0, len(n_points)]), np.concatenate([[0], np.cumsum([len(p) for p in n_points])]),
             pos.reshape(1, 3), vel.reshape(1, 3), yaw[:1],
             np.concatenate([np.asarray(p).reshape(-1, 3) for p in n_points]),
             np.concatenate([np.asarray(y, np.float64) for y in n_yaws]))
        a = dict(saved, max_iter=400, allocate_num=100000)
        info, refined, otour, _ = OT.local_tour_batch(om, *w, ViewNode.vm_, ViewNode.yd_, ViewNode.w_dir_,
                                                      a["resolution"], 10000.0, a["allocate_num"], a["max_iter"],
                                                      1.0, tour_max=4096)
        assert info["status"][0] == EM.TOUR_OK
        k = int(info["n_refined"][0])
        assert np.array_equal(pts, w[5][refined[0, :k]]) and np.array_equal(ys, w[6][refined[0, :k]])
        assert np.array_equal(tour, otour[0, :int(info["n_tour"][0])])
    finally:
        ViewNode.astar_ = saved
