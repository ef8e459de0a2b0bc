"""findGlobalTour of the C++ shim (include/fuelgpu_shim.hpp) compiles against the C ABI and links libfuelgpu.so.
Without a GPU the program stops in initMap with FUELGPU_ENODEVICE (no fallback); on the GPU its status, tour, full
cost matrix and global tour equal the Python findGlobalTour's on the same scene and frontier list, and its tour is the
oracle's exact tour (oracle.gtour) of that matrix."""
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
# the frontiers' viewpoints (x, y, z, yaw) and the current state of tests/shim_gtour_smoke.cpp
VPS = [(-1.6, 0.8, 0.6, 0.3), (1.0, -1.2, 0.6, 0.0), (1.5, 1.2, 0.6, 1.2), (0.0, 0.0, 0.7, -2.8), (1.8, 1.4, 0.6, 1.5)]
POS, VEL, YAW = np.array([-1.5, -1.2, 0.6]), np.array([0.5, 0.3, 0.0]), 0.2


def build(tmp_path):
    from fuel_b200 import _lib
    _lib.lib()
    exe = str(tmp_path / "shim_gtour_smoke")
    subprocess.check_call(["g++", "-std=c++14", "-O2", "-Wall", "-I", os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "shim_gtour_smoke.cpp"), "-o", exe,
                           "-L", os.path.join(ROOT, "fuel_b200"), "-lfuelgpu",
                           "-Wl,-rpath," + os.path.join(ROOT, "fuel_b200")])
    return exe


def test_shim_gtour_compiles_and_refuses_without_gpu(tmp_path):
    import torch
    exe = build(tmp_path)
    if torch.cuda.is_available():
        pytest.skip("GPU present: covered by test_shim_gtour_matches_oracle")
    r = subprocess.run([exe, str(tmp_path / "out.txt")], capture_output=True, text=True)
    assert r.returncode == 42, r.stdout + r.stderr


@pytest.mark.gpu
def test_shim_gtour_matches_oracle(tmp_path):
    import oracle.gtour as OG
    exe = build(tmp_path)
    out = tmp_path / "out.txt"
    r = subprocess.run([exe, str(out)], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    lines = open(out).read().strip().split("\n")
    status, k, nt = (int(v) for v in lines[0].split())
    indices = [int(v) for v in lines[1].split()]
    mat = np.array([float(v) for v in lines[2].split()]).reshape(6, 6)
    tour = np.array([[float(v) for v in ln.split()] for ln in lines[3:3 + nt]]).reshape(-1, 3)
    st, cost, _, want = OG.global_tour(mat)
    assert status == 0 == st and k == 5
    assert indices == want.tolist()
    assert OG.tour_cost(OG.int_matrix(mat), indices) == cost
    # the Python findGlobalTour on the same scene, frontier list and ViewNode statics
    import fuel_b200
    from fuel_b200 import exploration_manager as EM
    from fuel_b200 import workloads as W
    from fuel_b200.frontier_finder import FrontierFinder
    from fuel_b200.view_node import ViewNode
    from tests.helpers import make_sdf_map
    from tests.test_shim_cpp import scene
    n, tri, inflate = scene()
    g = W.Grid(n, (-2.4, -2.0, -0.5), 0.1, box_min=(-2.2, -1.8, -0.3), box_max=(2.2, 1.8, 1.7))
    m = make_sdf_map(fuel_b200, g, inflate, tri, optimistic=True)
    saved = dict(ViewNode.astar_)
    try:
        ViewNode.astar_ = dict(saved, resolution=0.4, lambda_heu=10000.0, allocate_num=20000, max_iter=2000)

        class Env:
            sdf_map_ = m

        class Ftr:
            def __init__(self, pos, yaw):
                self.viewpoints_ = [(np.array(pos, np.float64), yaw, 10)]
                self.costs_, self.paths_ = [], []
        ff = FrontierFinder.__new__(FrontierFinder)
        ff.edt_env_ = Env()
        ff.frontiers_ = [Ftr(v[:3], v[3]) for v in VPS]
        ff.first_new_ftr_, ff.removed_ids_ = 0, []
        py_idx, py_tour = EM.findGlobalTour(ff, POS, VEL, np.array([YAW, 0.0, 0.0]))
        py_mat = ff.getFullCostMatrix(POS, VEL, np.array([YAW, 0.0, 0.0]))
    finally:
        ViewNode.astar_ = saved
        m.close()
    assert np.array_equal(mat, py_mat)
    assert indices == py_idx and np.array_equal(tour, py_tour)
