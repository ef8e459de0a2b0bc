"""fuelgpu_view_cost_batch[_dev] on the H100 against the CPU oracle (oracle.view.view_cost_batch and the bookkeeping of
fuel_b200.frontier_finder over it, both pinned bit for bit on the reference's compiled graph_node.cpp and
frontier_finder.cpp by tests/test_oracle_view_cost.py).  kind, reason, iter_num, use_node_num, n_path, length and the
path rows bit for bit everywhere; cost bit for bit wherever |v1| <= 1e-3 (every pair updateFrontierCostMatrix makes),
within a few ulps elsewhere (the device's acos), with NaN at the same pairs."""
import ctypes as C

import numpy as np
import pytest
import torch

import oracle.astar as OA
import oracle.view as OV
from fuel_b200 import frontier_finder as FF
from fuel_b200 import workloads as W
from fuel_b200._lib import FuelAstarParams, FuelViewCostParams, lib
from fuel_b200.view_node import ASTAR, INFO_DTYPE, LINE, NO_PATH, ViewNode, view_cost_batch
from tests.helpers import make_sdf_map

pytestmark = pytest.mark.gpu

PATH_MAX = 512
VM, YD, W_DIR = ViewNode.vm_, ViewNode.yd_, ViewNode.w_dir_
COST_ULPS = 4  # acos on the device is within 2 ulp; w_dir * acos is added to the position cost


@pytest.fixture(scope="module")
def office(fuel):
    g, inflate = W.office_map()
    tri = W.office_known(g, inflate)
    m = make_sdf_map(fuel, g, inflate, tri)
    yield g, inflate, tri, m, OA.Map(g, inflate, tri)
    m.close()


@pytest.fixture(scope="module")
def office3(fuel):
    g, inflate = W.office3_map()
    tri = W.office_known(g, inflate)
    m = make_sdf_map(fuel, g, inflate, tri)
    yield g, inflate, tri, m, OA.Map(g, inflate, tri)
    m.close()


def cost_ulps(got, want):
    """the largest cost difference in ulps of the oracle's value; NaN must sit at the same pairs"""
    nan = np.isnan(want)
    assert np.array_equal(np.isnan(got), nan), "NaN at different pairs"
    if not (~nan).any():
        return 0.0
    return float(np.max(np.abs(got[~nan] - want[~nan]) / np.spacing(np.abs(want[~nan]))))


def assert_same(got, want, v1):
    gi, gp = got
    wi, wp = want
    for f in ("kind", "reason", "iter_num", "use_node_num", "n_path", "length"):
        bad = np.flatnonzero(gi[f] != wi[f])
        assert bad.size == 0, "%s differs at %s: %s vs %s" % (f, bad[:5], gi[f][bad[:3]], wi[f][bad[:3]])
    assert np.array_equal(gp, wp)
    still = np.linalg.norm(v1, axis=1) <= 1e-3
    assert np.array_equal(gi["cost"][still], wi["cost"][still])
    ulps = cost_ulps(gi["cost"][~still], wi["cost"][~still])
    assert ulps <= COST_ULPS, "cost off by %.1f ulps" % ulps
    return ulps


def run_both(m, om, pr, lam=10000.0, alloc=100000, max_iter=20000):
    got = view_cost_batch(m, pr["p1"], pr["p2"], pr["y1"], pr["y2"], pr["v1"], vm=VM, yd=YD, w_dir=W_DIR,
                          resolution=0.4, lambda_heu=lam, allocate_num=alloc, max_iter=max_iter, path_max=PATH_MAX)
    want = OV.view_cost_batch(om, pr["p1"], pr["p2"], pr["y1"], pr["y2"], pr["v1"], VM, YD, W_DIR, 0.4, lam, alloc,
                              max_iter, path_max=PATH_MAX)
    ulps = assert_same(got, want, pr["v1"])
    return got[0], ulps


@pytest.mark.parametrize("which", ["office", "office3"])
def test_pairs_p4096_match_oracle(request, which):
    g, inflate, tri, m, om = request.getfixturevalue(which)
    pr = W.make_view_pairs(g, inflate, tri, P=4096)
    info, ulps = run_both(m, om, pr)
    print("%s: %s line / A* / no path, max cost difference %.1f ulps" % (
        which, [int(np.count_nonzero(info["kind"] == k)) for k in (LINE, ASTAR, NO_PATH)], ulps))
    for k in (LINE, ASTAR, NO_PATH):
        assert np.count_nonzero(info["kind"] == k) > 50


@pytest.mark.parametrize("alloc,max_iter,reason", [(300, 100000, 2), (1000000, 60, 3), (1000000, 100000, 1),
                                                   (2, 100, 2)])
def test_caps_match_oracle(office, alloc, max_iter, reason):
    """allocate_num 1 000 000 (astar/allocate_num) runs with the pool clamped to 26 * max_iter + 2"""
    g, inflate, tri, m, om = office
    pr = W.make_view_pairs(g, inflate, tri, P=192, seed=7)
    info, _ = run_both(m, om, pr, alloc=alloc, max_iter=max_iter)
    assert np.count_nonzero(info["reason"][info["kind"] != LINE] == reason) > 0


def test_dev_entry_equals_host_entry_and_bad_rows(office):
    g, inflate, tri, m, om = office
    pr = W.make_view_pairs(g, inflate, tri, P=256, seed=9)
    pr["p1"][5, 1] = np.nan
    pr["y2"][17] = np.inf
    pr["v1"][40, 0] = -np.inf
    good = np.ones(256, bool)
    good[[5, 17, 40]] = False
    kw = dict(vm=VM, yd=YD, w_dir=W_DIR, resolution=0.4, lambda_heu=10000.0, allocate_num=100000, max_iter=20000,
              path_max=PATH_MAX)
    host_all = view_cost_batch(m, pr["p1"], pr["p2"], pr["y1"], pr["y2"], pr["v1"], **kw)
    host = view_cost_batch(m, *(pr[k][good] for k in ("p1", "p2", "y1", "y2", "v1")), **kw)
    dev = torch.device("cuda")
    t = {k: torch.tensor(pr[k], device=dev) for k in pr}
    dinfo = torch.zeros(256 * INFO_DTYPE.itemsize, dtype=torch.uint8, device=dev)
    dpath = torch.zeros((256, PATH_MAX, 3), dtype=torch.float64, device=dev)
    prm = FuelViewCostParams(VM, YD, W_DIR, FuelAstarParams(0.4, 10000.0, 100000, 20000))
    torch.cuda.synchronize()
    rc = lib().fuelgpu_view_cost_batch_dev(m.handle, 256, t["p1"].data_ptr(), t["p2"].data_ptr(), t["y1"].data_ptr(),
                                           t["y2"].data_ptr(), t["v1"].data_ptr(), C.byref(prm), dinfo.data_ptr(),
                                           PATH_MAX, dpath.data_ptr())
    assert rc == 0
    m.synchronize()
    info = np.frombuffer(dinfo.cpu().numpy().tobytes(), dtype=INFO_DTYPE)
    path = dpath.cpu().numpy()
    for i, p in ((info, path), host_all):
        assert np.all(i["kind"][~good] == 0) and np.all(i["reason"][~good] == 5) and np.all(i["cost"][~good] == 0)
        assert np.all(p[~good] == 0)
    assert info.tobytes() == host_all[0].tobytes() and np.array_equal(path, host_all[1])
    assert info[good].tobytes() == host[0].tobytes() and np.array_equal(path[good], host[1])


class _Snap:
    """the state of a cluster the bookkeeping reads and writes, copied"""

    def __init__(self, f):
        self.viewpoints_ = [(np.array(v[0]), float(v[1]), int(v[2])) for v in f.viewpoints_]
        self.costs_ = list(f.costs_)
        self.paths_ = [np.array(p) for p in f.paths_]


def _oracle_batch(om):
    a = ViewNode.astar_

    def batch(p1, p2, y1, y2, v1):
        info, path = OV.view_cost_batch(om, p1, p2, y1, y2, v1, VM, YD, W_DIR, a["resolution"], a["lambda_heu"],
                                        a["allocate_num"], a["max_iter"], PATH_MAX)
        assert np.all(info["n_path"] <= PATH_MAX)
        return info["cost"], [path[q, :info["n_path"][q]].copy() for q in range(len(info))]
    return batch


def _same_lists(got, want):
    assert len(got) == len(want)
    for f, w in zip(got, want):
        assert np.array_equal(np.asarray(f.costs_, np.float64), np.asarray(w.costs_, np.float64))
        assert len(f.paths_) == len(w.paths_)
        for p, q in zip(f.paths_, w.paths_):
            assert np.array_equal(np.asarray(p).reshape(-1, 3), np.asarray(q).reshape(-1, 3))


def test_office_sequence_cost_matrix(fuel):
    """searchFrontiers -> computeFrontiersToVisit -> updateFrontierCostMatrix -> getFullCostMatrix, then the map
    changes, the next search removes clusters and updateFrontierCostMatrix runs with removed_ids_"""
    g, inflate = W.office_map()
    tri = W.office_known(g, inflate)
    m = make_sdf_map(fuel, g, inflate, tri)
    om = OA.Map(g, inflate, tri)
    try:
        env = fuel.EDTEnvironment()
        env.setMap(m)
        ff = fuel.FrontierFinder(env)
        m.update_min_, m.update_max_ = g.origin.copy(), g.map_max.copy()
        ff.searchFrontiers()
        ff.computeFrontiersToVisit()
        assert len(ff.frontiers_) >= 4
        want = [_Snap(f) for f in ff.frontiers_]
        ff.updateFrontierCostMatrix()
        FF.update_cost_matrix(want, ff.first_new_ftr_, [], _oracle_batch(om))
        _same_lists(ff.frontiers_, want)

        cur_pos = ff.frontiers_[0].viewpoints_[0][0] + np.array([0.3, -0.2, 0.0])
        for cur_vel in ([0.0, 0.0, 0.0], [0.9, -0.4, 0.05]):
            got = ff.getFullCostMatrix(cur_pos, cur_vel, [0.4, 0.0, 0.0])
            ref = FF.full_cost_matrix(want, cur_pos, cur_vel, [0.4, 0.0, 0.0], _oracle_batch(om))
            assert np.array_equal(got[1:], ref[1:]) and np.all(got[:, 0] == 0)
            if not np.any(cur_vel):
                assert np.array_equal(got[0], ref[0])
            else:
                print("getFullCostMatrix row 0: max difference %.1f ulps" % cost_ulps(got[0, 1:], ref[0, 1:]))
                assert cost_ulps(got[0, 1:], ref[0, 1:]) <= COST_ULPS
        ids = list(range(min(5, len(ff.frontiers_))))[::-1]
        assert np.array_equal(ff.getPathForTour(cur_pos, ids), FF.path_for_tour(want, cur_pos, ids, _oracle_batch(om)))

        # explore around cluster 0: its cells stop being frontier, so the next search removes it
        tri2 = tri.copy()
        a = ff.frontiers_[0].cells_addr_.astype(np.int64)
        n = g.n
        idx = np.stack([a // (n[1] * n[2]), (a // n[2]) % n[1], a % n[2]], axis=1)
        lo, hi = np.maximum(idx.min(axis=0) - 2, 0), np.minimum(idx.max(axis=0) + 3, n)
        sub = tri2[lo[0]:hi[0], lo[1]:hi[1], lo[2]:hi[2]]
        sub[sub == W.UNKNOWN] = W.FREE
        m.setOccupancyBuffer(tristate=tri2)
        m.upload()
        om2 = OA.Map(g, inflate, tri2)
        m.update_min_, m.update_max_ = g.index_to_pos(lo), g.index_to_pos(hi - 1)
        ff.searchFrontiers()
        assert ff.removed_ids_ and 0 in ff.removed_ids_
        ff.computeFrontiersToVisit()
        removed = list(ff.removed_ids_)
        want = [_Snap(f) for f in ff.frontiers_]
        ff.updateFrontierCostMatrix()
        FF.update_cost_matrix(want, ff.first_new_ftr_, removed, _oracle_batch(om2))
        _same_lists(ff.frontiers_, want)
        assert all(len(f.costs_) == len(ff.frontiers_) for f in ff.frontiers_)
        got = ff.getFullCostMatrix(cur_pos, [0.0, 0.0, 0.0], [0.4, 0.0, 0.0])
        assert np.array_equal(got, FF.full_cost_matrix(want, cur_pos, [0.0, 0.0, 0.0], [0.4, 0.0, 0.0],
                                                       _oracle_batch(om2)))
    finally:
        m.close()
