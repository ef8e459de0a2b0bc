"""The local tour of the C++ shim (include/fuelgpu_shim.hpp: refineLocalTour, the one-viewpoint pick,
FrontierFinder::getViewpointsInfo and getTopViewpointsInfo) compiles against the C ABI and links libfuelgpu.so.  Without
a GPU the program stops in initMap with FUELGPU_ENODEVICE (no fallback); on the GPU its refined points, yaws, tour and
pick equal the oracle's (oracle.tour, oracle.view) bit for bit on the scene of tests/shim_smoke.cpp, lambda_heu is 10000
afterwards, and the two viewpoint lists equal the Python bookkeeping's (pinned on the reference by
tests/test_oracle_local_tour.py)."""
import os
import subprocess

import numpy as np
import pytest

from tests.test_shim_cpp import scene

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

N_POINTS = [[(-1.6, 0.8, 0.6), (-1.2, 1.2, 0.7), (-1.7, -0.6, 0.5)],
            [(1.0, -1.2, 0.6), (1.5, 1.2, 0.6), (0.0, 0.0, 0.7), (1.6, -0.4, 0.8)],
            [(1.8, 1.4, 0.6), (-1.0, 0.0, 0.6)]]
N_YAWS = [[0.3, -1.0, 2.5], [0.0, 1.2, -2.8, 0.6], [1.5, 0.0]]
POS, VEL, YAW = np.array([-1.5, -1.2, 0.6]), np.array([0.5, 0.3, 0.0]), 0.2
VM, YD, W_DIR = 2.0, 60 * 3.1415926 / 180.0, 1.5


def build(tmp_path):
    from fuel_b200 import _lib
    _lib.lib()
    exe = str(tmp_path / "shim_tour_smoke")
    subprocess.check_call(["g++", "-std=c++14", "-O2", "-Wall", "-I", os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "shim_tour_smoke.cpp"), "-o", exe,
                           "-L", os.path.join(ROOT, "fuel_b200"), "-lfuelgpu",
                           "-Wl,-rpath," + os.path.join(ROOT, "fuel_b200")])
    return exe


def test_shim_tour_compiles_and_refuses_without_gpu(tmp_path):
    import torch
    exe = build(tmp_path)
    if torch.cuda.is_available():
        pytest.skip("GPU present: covered by test_shim_tour_matches_oracle")
    r = subprocess.run([exe, str(tmp_path / "out.txt")], capture_output=True, text=True)
    assert r.returncode == 42, r.stdout + r.stderr


@pytest.mark.gpu
def test_shim_tour_matches_oracle(tmp_path):
    import oracle.astar as OA
    import oracle.tour as OT
    import oracle.view as OV
    from fuel_b200 import workloads as W
    exe = build(tmp_path)
    out = tmp_path / "out.txt"
    r = subprocess.run([exe, str(out)], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    n, tri, inflate = scene()
    g = W.Grid(n, (-2.4, -2.0, -0.5), 0.1, box_min=(-2.2, -1.8, -0.3), box_max=(2.2, 1.8, 1.7))
    om = OA.Map(g, inflate, tri)
    vp = np.array([p for grp in N_POINTS for p in grp], np.float64)
    vy = np.array([y for grp in N_YAWS for y in grp])
    go = np.concatenate([[0], np.cumsum([len(p) for p in N_POINTS])])
    info, refined, tour, _ = OT.local_tour_batch(om, [0, 3], go, [POS], [VEL], [YAW], vp, vy, VM, YD, W_DIR, 0.4,
                                                 10000.0, 20000, 2000, 1.0, tour_max=4096)
    lines = open(out).read().strip().split("\n")
    head = lines[0].split()
    status, k, nt, pick = (int(v) for v in head[:4])
    assert float(head[4]) == 10000.0  # ViewNode::astar_->lambda_heu_ = 10000 (:499)
    assert status == info["status"][0] == 0 and k == info["n_refined"][0] and nt == info["n_tour"][0]
    rows = np.array([[float(v) for v in ln.split()] for ln in lines[1:1 + k]])
    ids = refined[0, :k]
    assert np.array_equal(rows[:, :3], vp[ids]) and np.array_equal(rows[:, 3], vy[ids])
    trows = np.array([[float(v) for v in ln.split()] for ln in lines[1 + k:1 + k + nt]])
    assert np.array_equal(trows, tour[0, :nt])
    # getViewpointsInfo / getTopViewpointsInfo against the Python bookkeeping on the same frontier list
    from fuel_b200.frontier_finder import FrontierFinder
    from tests.test_oracle_local_tour import _F, _finder
    views = [[((3.0, 0.0, 1.0), 0.0, 10), ((4.0, 0.0, 1.0), 0.1, 9), ((5.0, 0.0, 1.0), 0.2, 8), ((6.0, 0.0, 1.0), 0.3, 7)],
             [((0.0, 0.0, 1.0), 0.0, 20), ((0.1, 0.0, 1.0), 0.2, 19), ((0.2, 0.0, 1.0), 0.4, 18),
              ((0.3, 0.0, 1.0), 0.6, 15)],
             [((0.2, 0.0, 1.0), 0.0, 30), ((2.0, 0.0, 1.0), 0.5, 29), ((0.3, 0.0, 1.0), 0.7, 28),
              ((4.0, 0.0, 1.0), 0.9, 27)]]
    ff = _finder([_F(i, v) for i, v in enumerate(views)])
    assert isinstance(ff, FrontierFinder)
    cur = np.array([0.0, 0.0, 1.0])
    pts, ys = ff.getViewpointsInfo(cur, [2, 0, 1, 7], 15, 0.8)
    r = 1 + k + nt
    assert lines[r] == "V %d" % len(pts)
    for gi in range(len(pts)):
        t = [float(v) for v in lines[r + 1 + gi].split()]
        assert int(t[0]) == len(pts[gi])
        got = np.array(t[1:]).reshape(-1, 4)
        assert np.array_equal(got[:, :3], np.asarray(pts[gi]).reshape(-1, 3)) and np.array_equal(got[:, 3], ys[gi])
    r += 1 + len(pts)
    tp, ty, _ = ff.getTopViewpointsInfo(cur)
    assert lines[r] == "T %d" % len(tp)
    got = np.array([[float(v) for v in ln.split()] for ln in lines[r + 1:r + 1 + len(tp)]])
    assert np.array_equal(got[:, :3], np.asarray(tp)) and np.array_equal(got[:, 3], ty)
    m = len(N_POINTS[1])
    vi, _ = OV.view_cost_batch(om, np.repeat(POS[None], m, 0), N_POINTS[1], np.full(m, YAW), N_YAWS[1],
                               np.repeat(VEL[None], m, 0), VM, YD, W_DIR, 0.4, 10000.0, 20000, 2000, path_max=2)
    best, want = 100000.0, -1
    for i, c in enumerate(vi["cost"]):
        if c < best:
            best, want = c, i
    assert pick == want
