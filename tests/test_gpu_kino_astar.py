"""fuelgpu_kino_search_batch[_dev] on the H100 against the kinodynamic-search oracle in the device's arithmetic
(oracle.kino, DEVICE mode; tests/test_oracle_kino.py compares it with the reference's glibc arithmetic): every output
byte for byte on the MID rows of the office and office3 path queries, on the hand-built cases, on a batch wider than
the warps that run at once; the _dev entry with the path search's info as its gate; bad input; and the chain
astar_batch_dev -> kino_search_batch_dev -> parameterize_batch_dev."""
import ctypes as C

import numpy as np
import pytest
import torch

import oracle.astar as OA
import oracle.kino as OK
from fuel_b200 import workloads as W
from fuel_b200._lib import MAX_PTS, FuelAstarParams, FuelGpuError, lib
from fuel_b200.astar import INFO_DTYPE as PATH_INFO, MID
from fuel_b200.kino_astar import (BAD_INPUT, INFO_DTYPE, SKIPPED, TRAJ_OK, KinodynamicAstar, kino_search_batch,
                                  kinodynamic_replan_batch, make_params)
from fuel_b200.non_uniform_bspline import parameterize_batch
from tests.helpers import make_sdf_map
from tests.kino_cases import hand_cases, mid_queries

pytestmark = pytest.mark.gpu

NODE_MAX = 128


@pytest.fixture(scope="module", params=["office", "office3"])
def world(fuel, request):
    g, inflate = W.office_map() if request.param == "office" else W.office3_map()
    tri = W.office_known(g, inflate)
    m = make_sdf_map(fuel, g, inflate, tri)
    yield g, inflate, tri, m, OA.Map(g, inflate, tri)
    m.close()


def assert_same(got, want):
    for f in INFO_DTYPE.names:
        bad = np.flatnonzero(got["info"][f] != want["info"][f])
        assert bad.size == 0, "%s differs at %s: %s vs %s" % (f, bad[:5], got["info"][f][bad[:3]], want["info"][f][bad[:3]])
    for k in ("points", "derivs", "dt", "nodes", "shot"):
        if want[k] is not None:
            assert got[k].tobytes() == want[k].tobytes(), k


def run_both(m, g, om, q, **kw):
    got = kino_search_batch(m, q["start"], q["vel"], q["acc"], q["goal"], node_max=NODE_MAX, **kw)
    want = OK.replan_batch(om, g.map_max - g.origin, make_params(**kw), q["start"], q["vel"], q["acc"], q["goal"],
                           math=OK.DEVICE, node_max=NODE_MAX)
    assert_same(got, want)
    return got


def test_mid_rows_match_oracle(world):
    g, inflate, tri, m, om = world
    q = mid_queries(g, inflate, tri, B=1024, seed=20261019)
    info = run_both(m, g, om, q)["info"]
    print("%d MID searches: use_node_num median %d, max %d; %d with samples" %
          (len(info), np.median(info["use_node_num"]), info["use_node_num"].max(),
           np.count_nonzero(info["traj_status"] == TRAJ_OK)))
    assert np.count_nonzero(info["traj_status"] == TRAJ_OK) > len(info) // 2


@pytest.mark.parametrize("kw", [dict(), dict(optimistic=True), dict(allocate_num=40), dict(lambda_heu=0.0, allocate_num=3000),
                                dict(horizon=1.0)])
def test_hand_cases_match_oracle(world, kw):
    g, inflate, tri, m, om = world
    run_both(m, g, om, hand_cases(g, inflate, tri), **kw)


def test_wide_batch_matches_oracle(fuel):
    """more rows than the warps that fit the scratch budget at allocate_num = 2^24: warps take several rows each"""
    g, inflate = W.office_map()
    tri = W.office_known(g, inflate)
    m = make_sdf_map(fuel, g, inflate, tri)
    try:
        q = mid_queries(g, inflate, tri, B=512, seed=31)
        q = {k: np.concatenate([v] * 4) for k, v in q.items() if k != "rows"}
        run_both(m, g, OA.Map(g, inflate, tri), q, allocate_num=1 << 24)
    finally:
        m.close()


def test_dev_entry_gate_and_bad_rows(world):
    g, inflate, tri, m, om = world
    q = W.make_path_queries(g, inflate, tri, B=256, seed=9)
    B = len(q["start"])
    path_info = OA.search_batch(om, q["start"], q["goal"], 0.4, 10000.0, 40000, 100000)[0]
    rng = np.random.default_rng(3)
    vel = rng.uniform(-1, 1, (B, 3))
    acc = rng.uniform(-1, 1, (B, 3))
    start = q["start"].copy()
    mid = np.flatnonzero(path_info["branch"] == MID)
    start[mid[0], 1] = np.nan  # a bad MID row
    host = kino_search_batch(m, np.where(np.isnan(start), 0.0, start), vel, acc, q["goal"], node_max=NODE_MAX)
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    t = {k: dev(v) for k, v in dict(s=start, v=vel, a=acc, g=q["goal"]).items()}
    gate = torch.from_numpy(path_info.view(np.uint8).copy()).cuda()
    info = torch.empty(B * INFO_DTYPE.itemsize, dtype=torch.uint8, device="cuda")
    pts = torch.empty((B, MAX_PTS - 2, 3), dtype=torch.float64, device="cuda")
    der = torch.empty((B, 4, 3), dtype=torch.float64, device="cuda")
    dt = torch.empty(B, dtype=torch.float64, device="cuda")
    nodes = torch.empty((B, NODE_MAX, 12), dtype=torch.float64, device="cuda")
    shot = torch.empty((B, 3, 4), dtype=torch.float64, device="cuda")
    prm = make_params()
    vp = lambda x: C.c_void_p(x.data_ptr())
    assert lib().fuelgpu_kino_search_batch_dev(m.handle, B, vp(t["s"]), vp(t["v"]), vp(t["a"]), vp(t["g"]), vp(gate),
                                               C.byref(prm), vp(info), vp(pts), vp(der), vp(dt), NODE_MAX, vp(nodes),
                                               vp(shot)) == 0
    assert lib().fuelgpu_map_synchronize(m.handle) == 0
    di = np.frombuffer(info.cpu().numpy().tobytes(), INFO_DTYPE)
    other = np.setdiff1d(np.arange(B), mid)
    assert np.all(di["status"][other] == SKIPPED) and np.all(di["traj_status"][other] == 2)
    assert di["status"][mid[0]] == BAD_INPUT
    keep = mid[1:]
    for f in INFO_DTYPE.names:
        assert np.array_equal(di[f][keep], host["info"][f][keep]), f
    for k, v in dict(points=pts, derivs=der, dt=dt, nodes=nodes, shot=shot).items():
        assert v.cpu().numpy()[keep].tobytes() == host[k][keep].tobytes(), k


def test_einval(world):
    g, inflate, tri, m, om = world
    s = np.zeros((1, 3))
    bad = [dict(max_tau=0.0), dict(init_max_tau=np.nan), dict(max_acc=-1.0), dict(w_time=0.0), dict(horizon=0.0),
           dict(resolution=0.0), dict(lambda_heu=np.inf), dict(allocate_num=1), dict(check_num=0), dict(check_num=17),
           dict(ctrl_pt_dist=0.0), dict(manager_max_vel=np.nan), dict(max_vel=-0.25), dict(init_max_tau=1.0, max_tau=0.8,
                                                                                          max_acc=2.0, vel_margin=np.inf),
           dict(max_tau=0.1 ** 0 * 5, init_max_tau=5.0)]  # (the last one is fine: 20 init durations)
    for kw in bad[:-1]:
        with pytest.raises(FuelGpuError):
            kino_search_batch(m, s, s, s, s + 1.0, **kw)
    kino_search_batch(m, s, s, s, s + 1.0, **bad[-1])
    for k in range(4):
        arrs = [s, s, s, s + 1.0]
        arrs[k] = np.full((1, 3), np.nan)
        with pytest.raises(FuelGpuError):
            kino_search_batch(m, *arrs)
    prm = make_params()
    L = lib()
    assert L.fuelgpu_kino_search_batch(m.handle, -1, None, None, None, None, C.byref(prm), None, None, None, None, 0, None,
                                       None) != 0
    assert L.fuelgpu_kino_search_batch(m.handle, 1, None, None, None, None, C.byref(prm), None, None, None, None, 0, None,
                                       None) != 0
    assert L.fuelgpu_kino_search_batch(m.handle, 1, None, None, None, None, None, None, None, None, None, 0, None, None) != 0
    assert L.fuelgpu_kino_search_batch_dev(m.handle, 0, None, None, None, None, None, C.byref(prm), None, None, None, None,
                                           0, None, None) == 0
    out = kino_search_batch(m, np.zeros((0, 3)), np.zeros((0, 3)), np.zeros((0, 3)), np.zeros((0, 3)))
    assert len(out["info"]) == 0


def test_class_and_replan_chain(world):
    g, inflate, tri, m, om = world
    q = mid_queries(g, inflate, tri, B=256, seed=5)
    ka = KinodynamicAstar(m)
    with pytest.raises(NotImplementedError):
        ka.search(q["start"][0], q["vel"][0], q["acc"][0], q["goal"][0], dynamic=True)
    st = ka.search(q["start"][0], q["vel"][0], q["acc"][0], q["goal"][0])
    res = kino_search_batch(m, q["start"][:1], q["vel"][:1], q["acc"][:1], q["goal"][:1])
    assert st == res["info"]["status"][0]
    if res["info"]["traj_status"][0] == TRAJ_OK:
        ts, pts, der = ka.getSamples()
        assert ts == res["dt"][0] and np.array_equal(pts, res["points"][0, :len(pts)])
    res, groups = kinodynamic_replan_batch(m, q["start"], q["vel"], q["acc"], q["goal"], time_lb=np.full(len(q["start"]), 0.5))
    want = OK.replan_batch(om, g.map_max - g.origin, make_params(), q["start"], q["vel"], q["acc"], q["goal"])
    assert sum(len(r) for r, _, _ in groups) == np.count_nonzero(want["info"]["traj_status"] == TRAJ_OK)
    for rows, x, traj in groups:
        K = int(want["info"]["n_pts"][rows[0]]) - 2
        wx, _ = parameterize_batch(m, want["points"][rows, :K], want["derivs"][rows], want["dt"][rows],
                                   np.full(len(rows), 0.5))
        assert x.tobytes() == wx.tobytes()


def test_office_chain_without_sync(fuel):
    """astar_batch_dev -> kino_search_batch_dev (MID rows) -> parameterize_batch_dev, read back only for n_pts"""
    g, inflate = W.office_map()
    tri = W.office_known(g, inflate)
    m = make_sdf_map(fuel, g, inflate, tri)
    try:
        q = W.make_path_queries(g, inflate, tri, B=512, seed=77)
        B = len(q["start"])
        rng = np.random.default_rng(8)
        vel, acc = rng.uniform(-1, 1, (B, 3)), rng.uniform(-1, 1, (B, 3))
        dev = lambda a: torch.from_numpy(np.ascontiguousarray(a, dtype=np.float64)).cuda()
        vp = lambda x: C.c_void_p(x.data_ptr()) if x is not None else None
        s, gl, v, a = dev(q["start"]), dev(q["goal"]), dev(vel), dev(acc)
        pinfo = torch.empty(B * PATH_INFO.itemsize, dtype=torch.uint8, device="cuda")
        nwp = torch.empty(B, dtype=torch.int32, device="cuda")
        wp = torch.empty((B, 32, 3), dtype=torch.float64, device="cuda")
        ap = FuelAstarParams(0.4, 10000.0, 40000, 100000)
        L = lib()
        assert L.fuelgpu_astar_batch_dev(m.handle, B, vp(s), vp(gl), C.byref(ap), vp(pinfo), 0, None, 32, vp(nwp), vp(wp)) == 0
        info = torch.empty(B * INFO_DTYPE.itemsize, dtype=torch.uint8, device="cuda")
        pts = torch.empty((B, MAX_PTS - 2, 3), dtype=torch.float64, device="cuda")
        der = torch.empty((B, 4, 3), dtype=torch.float64, device="cuda")
        dt = torch.empty(B, dtype=torch.float64, device="cuda")
        prm = make_params()
        assert L.fuelgpu_kino_search_batch_dev(m.handle, B, vp(s), vp(v), vp(a), vp(gl), vp(pinfo), C.byref(prm), vp(info),
                                               vp(pts), vp(der), vp(dt), 0, None, None) == 0
        assert L.fuelgpu_map_synchronize(m.handle) == 0  # the one read: n_pts (the map's stream is not torch's)
        ki = np.frombuffer(info.cpu().numpy().tobytes(), INFO_DTYPE)
        path_info = np.frombuffer(pinfo.cpu().numpy().tobytes(), PATH_INFO)
        kq = W.make_kino_queries(g, inflate, tri, path_info, q["start"], q["goal"])
        rows = kq["rows"]
        assert np.all(ki["status"][np.setdiff1d(np.arange(B), rows)] == SKIPPED)
        want = OK.replan_batch(OA.Map(g, inflate, tri), g.map_max - g.origin, prm, q["start"][rows], vel[rows],
                               acc[rows], q["goal"][rows])
        for f in INFO_DTYPE.names:
            assert np.array_equal(ki[f][rows], want["info"][f]), f
        ok = rows[ki["traj_status"][rows] == TRAJ_OK]
        assert len(ok) > 0
        for n in np.unique(ki["n_pts"][ok]):
            sel = ok[ki["n_pts"][ok] == n]
            K = int(n) - 2
            idx = torch.from_numpy(sel).cuda()
            p = pts.index_select(0, idx)[:, :K].contiguous()
            d, t = der.index_select(0, idx).contiguous(), dt.index_select(0, idx).contiguous()
            nvar = 3 * int(n) + 1
            x = torch.empty((len(sel), nvar), dtype=torch.float64, device="cuda")
            tc = torch.empty(len(sel) * 4096, dtype=torch.uint8, device="cuda")
            assert L.fuelgpu_bspline_parameterize_batch_dev(m.handle, len(sel), int(n), nvar, vp(p), vp(d), vp(t), None,
                                                            vp(x), vp(tc)) == 0
            assert L.fuelgpu_map_synchronize(m.handle) == 0
            w = np.searchsorted(rows, sel)
            wx, _ = parameterize_batch(m, want["points"][w, :K], want["derivs"][w], want["dt"][w])
            assert x.cpu().numpy().tobytes() == wx.tobytes()
    finally:
        m.close()
