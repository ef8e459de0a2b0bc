"""fast_planner::KinodynamicAstar of the C++ shim (include/fuelgpu_shim.hpp) compiles against the C ABI and links
libfuelgpu.so.  Without a GPU the program stops in initMap with FUELGPU_ENODEVICE (no fallback); on the GPU its searches
and samples equal the kinodynamic oracle's (oracle.kino, DEVICE mode) bit for bit on the scene of tests/shim_smoke.cpp."""
import os
import subprocess

import numpy as np
import pytest

from tests.test_shim_cpp import scene

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def build(tmp_path):
    from fuel_b200 import _lib
    _lib.lib()
    exe = str(tmp_path / "shim_kino_smoke")
    subprocess.check_call(["g++", "-std=c++14", "-O2", "-Wall", "-I", os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "shim_kino_smoke.cpp"), "-o", exe,
                           "-L", os.path.join(ROOT, "fuel_b200"), "-lfuelgpu",
                           "-Wl,-rpath," + os.path.join(ROOT, "fuel_b200")])
    return exe


def test_shim_kino_compiles_and_refuses_without_gpu(tmp_path):
    import torch
    exe = build(tmp_path)
    if torch.cuda.is_available():
        pytest.skip("GPU present: covered by test_shim_kino_matches_oracle")
    r = subprocess.run([exe, str(tmp_path / "out.txt")], capture_output=True, text=True)
    assert r.returncode == 42, r.stdout + r.stderr


@pytest.mark.gpu
def test_shim_kino_matches_oracle(tmp_path):
    import oracle.astar as OA
    import oracle.kino as OK
    from fuel_b200 import workloads as W
    from fuel_b200.kino_astar import make_params
    exe = build(tmp_path)
    out = tmp_path / "out.txt"
    r = subprocess.run([exe, str(out)], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    n, tri, inflate = scene()
    g = W.Grid(n, (-2.4, -2.0, -0.5), 0.1, box_min=(-2.2, -1.8, -0.3), box_max=(2.2, 1.8, 1.7))
    om = OA.Map(g, inflate, tri)
    q = np.array([[-1.5, -1.2, 0.6, 0.5, 0.0, 0.0, 0.0, 0.0, 0.0], [-1.5, 0.0, 0.6, 0.0, 0.0, 0.0, 0.0, 0.3, 0.0],
                  [-1.5, -1.2, 0.6, 0.0, 0.5, 0.0, 0.2, 0.0, 0.0], [1.2, -1.0, 0.4, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0]])
    goal = np.array([[1.4, -1.2, 0.6], [-0.9, 0.4, 0.7], [-0.2, 0.5, 0.8], [1.2, -1.0, 0.4]])
    want = OK.replan_batch(om, g.map_max - g.origin, make_params(optimistic=True), q[:, :3], q[:, 3:6], q[:, 6:],
                           goal, math=OK.DEVICE)
    lines = open(out).read().strip().split("\n")
    assert len(lines) == 4
    for b, ln in enumerate(lines):
        t = ln.split()
        i = want["info"][b]
        ok = i["traj_status"] == 0
        assert [int(v) for v in t[1:6]] == [i["status"], i["retried"], i["use_node_num"], int(ok),
                                           max(int(i["n_pts"]) - 2, 0)]
        if ok:
            assert float(t[6]) == want["dt"][b]
            p = np.array([float(v) for v in t[7:]]).reshape(-1, 3)
            assert np.array_equal(p, want["points"][b, :len(p)])
    assert want["info"]["reason"][3] == 4 and np.any(want["info"]["traj_status"] == 0)
