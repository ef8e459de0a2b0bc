"""Trajectories of 33 to 64 control points: the two-points-per-lane FAST evaluator (FUELGPU_COST_FAST_EVAL above 32
points) against the CPU oracle of combineCost, and the long-trajectory solver (fuelgpu_bspline_optimize_batch with
n_pts + dt > 32 lanes) against its CPU twin oracle.orc_optimize_batch.  Scene: the office3 map (BASELINE config 5),
whose 18 x 28 m box holds 64-point lines at the default 0.35 m spacing."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from fuel_b200 import workloads as W
from tests.helpers import make_sdf_map, orc_grid
from tests.test_gpu_bspline import check, gpu_consts, orc_consts

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def field(orc):
    """office3 map and the oracle's fp64 field (the reference's own arithmetic)"""
    g, inflate = W.office3_map()
    tri = W.office_known(g, inflate)
    og = orc_grid(orc, g)
    d64 = orc.update_esdf3d(og, inflate, tri, [0, 0, 0], np.array(g.n) - 1, True, False, threads=8)
    return dict(g=g, inflate=inflate, tri=tri, og=og, d64=d64)


@pytest.fixture(scope="module")
def scene(fuel, field):
    m = make_sdf_map(fuel, field["g"], field["inflate"], field["tri"], optimistic=True)
    m.updateESDF3d()
    env = fuel.EDTEnvironment()
    env.setMap(m)
    opt = fuel.BsplineOptimizer()
    opt.setEnvironment(env)
    yield dict(field, m=m, env=env, opt=opt)
    m.close()


def oracle_cost(orc, S, tr, B, N, mask, x, po=None, to=None, **kw):
    return orc.combine_cost_batch(S["og"], S["d64"], po or orc.opt_params(), to or orc_consts(orc, tr, B, **kw), N, mask,
                                  x, threads=8)


# ---- FAST evaluator parity ----------------------------------------------------------------------------------------

@pytest.mark.gpu
def test_fast_evaluator_long_parity(fuel, orc, scene):
    """The evaluator the long solver runs, once per trajectory, on both sides of the 32-point switch, with and without
    MINTIME; dt halved on every third trajectory so that feasibility and its dt-gradient bite."""
    O = fuel.BsplineOptimizer
    g, opt = scene["g"], scene["opt"]
    for N in (32, 33, 47, 63, 64):
        B = 1024 if N == 64 else 128
        tr = W.make_trajectories(g, scene["inflate"], B=B, n_pts=N, seed=1000 + N)
        for mintime in (True, False):
            mask = O.NORMAL_PHASE | (O.MINTIME if mintime else 0)
            tr2 = dict(tr, dt=tr["dt"].copy())
            tr2["dt"][::3] *= 0.5
            x = W.pack_x(tr2["ctrl"], tr2["dt"], mintime=mintime)
            f, gg = opt.combineCostBatch(x, gpu_consts(fuel, tr2, B), N, mask, fast_eval=True)
            fr, gr = oracle_cost(orc, scene, tr2, B, N, mask, x)
            check(f, gg, fr, gr)
            if N == 64 and mintime:  # the flag switches evaluators
                f2, g2 = opt.combineCostBatch(x, gpu_consts(fuel, tr2, B), N, mask)
                check(f2, g2, fr, gr)
                assert not (np.array_equal(f, f2) and np.array_equal(gg, g2)), "the flag did not switch evaluators"


@pytest.mark.gpu
@pytest.mark.parametrize("N", [48, 64])
def test_fast_evaluator_long_single_terms(fuel, orc, scene, N):
    O = fuel.BsplineOptimizer
    tr = W.make_trajectories(scene["g"], scene["inflate"], B=64, n_pts=N, seed=5)
    for name in ("SMOOTHNESS", "DISTANCE", "FEASIBILITY", "START", "END", "MINTIME"):
        mask = getattr(O, name) | (O.SMOOTHNESS if name == "MINTIME" else 0)
        tr2 = dict(tr, dt=tr["dt"] * 0.6)
        x = W.pack_x(tr2["ctrl"], tr2["dt"], mintime=bool(mask & O.MINTIME))
        f, gg = scene["opt"].combineCostBatch(x, gpu_consts(fuel, tr2, 64), N, mask, fast_eval=True)
        fr, gr = oracle_cost(orc, scene, tr2, 64, N, mask, x)
        check(f, gg, fr, gr)


@pytest.mark.gpu
@pytest.mark.parametrize("N", [48, 64])
def test_fast_evaluator_long_guide_waypoints_end3_timelb(fuel, orc, scene, N):
    """GUIDE_PHASE, waypoints whose stencils straddle the slot boundary (31/32), a 3-entry end state with an active time
    lower bound."""
    O = fuel.BsplineOptimizer
    B = 32
    tr = W.make_trajectories(scene["g"], scene["inflate"], B=B, n_pts=N, seed=9)
    rng = np.random.default_rng(3)
    guide = tr["ctrl"][:, 3:N - 3] + rng.normal(scale=0.2, size=(B, N - 6, 3))
    widx = [0, 30, 31, 32, 33, N - 3]
    waypt = rng.uniform(-1, 1, size=(B, len(widx), 3)) + tr["ctrl"][:, [i + 1 for i in widx]]
    time_lb = (N - 3) * tr["dt"] * 1.3
    for mask, n_end in ((O.GUIDE_PHASE, 1), (O.SMOOTHNESS | O.WAYPOINTS, 1), (O.NORMAL_PHASE | O.MINTIME, 3),
                        (O.NORMAL_PHASE | O.WAYPOINTS | O.MINTIME, 2)):
        x = W.pack_x(tr["ctrl"], tr["dt"], mintime=bool(mask & O.MINTIME))
        kw = dict(guide=guide, waypt=waypt, waypt_idx=widx, n_end=n_end, time_lb=time_lb)
        tg = gpu_consts(fuel, tr, B, **kw)
        to = orc_consts(orc, tr, B, **kw)
        for b in range(B):
            for i in range(1, n_end):
                for k in range(3):
                    v = float(rng.normal())
                    tg[b].end[i][k] = v
                    to[b].end[i][k] = v
        f, gg = scene["opt"].combineCostBatch(x, tg, N, mask, fast_eval=True)
        fr, gr = oracle_cost(orc, scene, tr, B, N, mask, x, to=to)
        check(f, gg, fr, gr)


@pytest.mark.gpu
@pytest.mark.parametrize("N", [40, 64])
def test_fast_evaluator_long_view_cost(fuel, orc, scene, N):
    """calcViewCost on points 5, 31, 32 and n-2, on both sides of its |dl| < |dir| switch."""
    O = fuel.BsplineOptimizer
    B = 64
    tr = W.make_trajectories(scene["g"], scene["inflate"], B=B, n_pts=N, seed=23)
    rng = np.random.default_rng(23)
    opt = fuel.BsplineOptimizer()
    opt.setEnvironment(scene["env"])
    opt.setParam(ld_view=2.5, wnl=1.3)
    po = orc.opt_params(ld_view=2.5, wnl=1.3)
    tg, to = gpu_consts(fuel, tr, B), orc_consts(orc, tr, B)
    idxs = (5, 31, 32, N - 2)
    n_par = 0
    for b in range(B):
        idx = idxs[b % 4]
        pt = tr["ctrl"][b, idx] + rng.normal(size=3) * 0.4
        d = (tr["ctrl"][b, idx] - pt) * float(rng.choice([-1.0, 1.0])) + rng.normal(size=3) * 0.1
        d = d / np.linalg.norm(d) * float(rng.choice([0.2, 1.5]))
        for t in (tg[b], to[b]):
            for k in range(3):
                t.view_pt[k], t.view_dir[k] = pt[k], d[k]
            t.view_idx = idx
        n_par += int(abs(np.dot(tr["ctrl"][b, idx] - pt, d / np.linalg.norm(d))) < np.linalg.norm(d))
    assert 5 < n_par < B - 5
    for mask in (O.VIEWCONS, O.NORMAL_PHASE | O.VIEWCONS | O.MINTIME):
        x = W.pack_x(tr["ctrl"], tr["dt"], mintime=bool(mask & O.MINTIME))
        fr, gr = oracle_cost(orc, scene, tr, B, N, mask, x, po=po, to=to)
        f, gg = opt.combineCostBatch(x, tg, N, mask, fast_eval=True)
        check(f, gg, fr, gr)
        if mask == O.VIEWCONS:
            assert np.all(np.count_nonzero(gg, axis=1) <= 3)


@pytest.mark.gpu
def test_fast_evaluator_long_adversarial_positions(fuel, orc, scene):
    """Stencil outside the map, outside the map, and the isInMap margin, at points 31, 32, 33 and n-1."""
    O = fuel.BsplineOptimizer
    g = scene["g"]
    B, N = 48, 64
    tr = W.make_trajectories(g, scene["inflate"], B=B, n_pts=N, seed=13)
    ctrl = tr["ctrl"].copy()
    kinds = (g.origin + [0.02, 0.5, 0.5], g.map_max + 0.3, g.map_max - [1e-4, 0.5, 0.5])
    for j, pos in enumerate(kinds):
        for ii, idx in enumerate((31, 32, 33, N - 1)):
            r0 = (4 * j + ii) * 4
            ctrl[r0:r0 + 4, idx] = pos
    tr["ctrl"] = ctrl
    mask = O.NORMAL_PHASE | O.MINTIME
    x = W.pack_x(ctrl, tr["dt"])
    f, gg = scene["opt"].combineCostBatch(x, gpu_consts(fuel, tr, B), N, mask, fast_eval=True)
    fr, gr = oracle_cost(orc, scene, tr, B, N, mask, x)
    check(f, gg, fr, gr)


# ---- the long-trajectory solver -------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("N", [48, 64])
def test_optimize_long_matches_cpu_twin(fuel, orc, scene, N):
    """The gates of test_optimize_batch_matches_cpu_twin at 48 and 64 control points."""
    B, K = 256, 64
    O = fuel.BsplineOptimizer
    g = scene["g"]
    tr = W.make_trajectories(g, scene["inflate"], B=B, n_pts=N, seed=77)
    mask = O.NORMAL_PHASE | O.MINTIME
    x0 = W.pack_x(tr["ctrl"], tr["dt"])
    to = orc_consts(orc, tr, B)
    f0, _ = oracle_cost(orc, scene, tr, B, N, mask, x0, to=to)
    xg, fg, ng = scene["opt"].optimizeBatch(x0, gpu_consts(fuel, tr, B), N, mask, K)
    xc, fc, nc = orc.optimize_batch(scene["og"], scene["d64"], orc.opt_params(), to, N, mask, x0, max_eval=K, threads=8)
    assert np.all(ng <= K) and np.all(ng >= 1)
    assert np.all(fg <= f0 * (1 + 1e-9))
    pts = xg[:, :3 * N].reshape(B, N, 3)
    assert np.all(pts >= g.box_min + 0.1 - 1e-12) and np.all(pts <= g.box_max - 0.1 + 1e-12)
    assert np.all(xg[:, -1] >= 0.0) and np.all(xg[:, -1] <= 5.0)
    fchk, _ = oracle_cost(orc, scene, tr, B, N, mask, xg, to=to)
    assert np.all(np.abs(fchk - fg) <= 1e-4 * np.abs(fg) + 1e-9)
    rel = np.abs(fg - fc) / np.abs(fc)
    print("N=%d median rel diff %.3g, p90 %.3g, mean gpu %.4f cpu %.4f start %.4f" %
          (N, np.median(rel), np.quantile(rel, 0.9), np.mean(fg), np.mean(fc), np.mean(f0)))
    assert np.median(rel) < 0.03, np.median(rel)
    assert np.quantile(fg / fc, 0.99) < 1.25
    assert abs(np.mean(fg) - np.mean(fc)) < 0.02 * np.mean(fc)
    assert np.mean(fg) < 0.01 * np.mean(f0)


@pytest.mark.gpu
@pytest.mark.parametrize("N", [40, 64])
def test_optimize_long_f_best_is_faithful_cost(fuel, scene, N):
    """min_cost_ is fuelgpu_bspline_cost_batch (the faithful evaluator) at the returned x, bit for bit."""
    B, K = 256, 64
    O = fuel.BsplineOptimizer
    tr = W.make_trajectories(scene["g"], scene["inflate"], B=B, n_pts=N, seed=41)
    mask = O.NORMAL_PHASE | O.MINTIME
    tc = gpu_consts(fuel, tr, B)
    xg, fg, ng = scene["opt"].optimizeBatch(W.pack_x(tr["ctrl"], tr["dt"]), tc, N, mask, K)
    fc, _ = scene["opt"].combineCostBatch(xg, tc, N, mask)
    assert np.array_equal(fg, fc)


@pytest.mark.gpu
def test_optimize_long_exact_evals(fuel, orc, scene):
    """FUELGPU_SOLVE_EXACT_EVALS: every trajectory reports exactly K; trajectories that never stop early in the normal
    mode take the identical path."""
    B, N, K = 1024, 64, 64
    O = fuel.BsplineOptimizer
    tr = W.make_trajectories(scene["g"], scene["inflate"], B=B, n_pts=N)
    mask = O.NORMAL_PHASE | O.MINTIME
    x0 = W.pack_x(tr["ctrl"], tr["dt"])
    tc = gpu_consts(fuel, tr, B)
    xe, fe, ne = scene["opt"].optimizeBatch(x0, tc, N, mask, K, xtol_rel=0.0, exact_evals=True)
    assert np.all(ne == K), (ne.min(), ne.max())
    xn, fn, nn = scene["opt"].optimizeBatch(x0, tc, N, mask, K, xtol_rel=0.0)
    assert np.all(nn <= K)
    f0, _ = oracle_cost(orc, scene, tr, B, N, mask, x0)
    assert np.all(fe <= f0 * (1 + 1e-9))
    same = nn == K
    assert same.sum() > B // 2, same.sum()
    assert np.array_equal(xe[same], xn[same]) and np.array_equal(fe[same], fn[same])


@pytest.mark.gpu
@pytest.mark.parametrize("lbfgs_m", [1, 4, 8])
@pytest.mark.parametrize("B", [1, 5, 4096])
def test_optimize_long_same_path_same_bits(fuel, scene, lbfgs_m, B):
    """begin/end equals the one-shot call, the device-pointer entry equals the host entry, two runs are bitwise equal."""
    import torch

    from fuel_b200._lib import FuelSolveParams, check as lib_check
    N, K = 64 if B != 5 else 37, 48
    O = fuel.BsplineOptimizer
    opt = scene["opt"]
    tr = W.make_trajectories(scene["g"], scene["inflate"], B=B, n_pts=N, seed=300 + B)
    mask = O.NORMAL_PHASE | O.MINTIME
    x0 = W.pack_x(tr["ctrl"], tr["dt"])
    tc = gpu_consts(fuel, tr, B)
    x1, f1, n1 = [a.copy() for a in opt.optimizeBatch(x0, tc, N, mask, K, lbfgs_m=lbfgs_m)]
    x2, f2, n2 = [a.copy() for a in opt.optimizeBatch(x0, tc, N, mask, K, lbfgs_m=lbfgs_m)]
    assert np.array_equal(x1, x2) and np.array_equal(f1, f2) and np.array_equal(n1, n2)
    opt.optimizeBatchBegin(x0, tc, N, mask, K, lbfgs_m=lbfgs_m)
    x3, f3, n3 = opt.optimizeBatchEnd()
    assert np.array_equal(x1, x3) and np.array_equal(f1, f3) and np.array_equal(n1, n3)
    d_tc = torch.from_numpy(np.frombuffer(tc, dtype=np.uint8).copy()).cuda()
    d_x = torch.from_numpy(x0).cuda()
    d_f = torch.empty(B, dtype=torch.float64, device="cuda")
    d_n = torch.empty(B, dtype=torch.int32, device="cuda")
    sp = FuelSolveParams()
    sp.max_eval, sp.lbfgs_m, sp.xtol_rel, sp.flags = K, lbfgs_m, 1e-5, 0
    torch.cuda.synchronize()
    h = scene["m"].handle
    lib_check(fuel.lib().fuelgpu_bspline_optimize_batch_dev(h, B, N, mask, C.byref(opt.params_),
                                                            C.c_void_p(d_tc.data_ptr()), C.byref(sp),
                                                            C.c_void_p(d_x.data_ptr()), C.c_void_p(d_f.data_ptr()),
                                                            C.c_void_p(d_n.data_ptr())), h)
    scene["m"].synchronize()
    torch.cuda.synchronize()
    assert np.array_equal(d_x.cpu().numpy(), x1) and np.array_equal(d_f.cpu().numpy(), f1)
    assert np.array_equal(d_n.cpu().numpy(), n1)


@pytest.mark.gpu
def test_optimize_long_through_the_mirror(fuel, scene):
    """optimize() on one 40-point trajectory; max_eval = 1 returns the clamped start; 65 points are refused."""
    O = fuel.BsplineOptimizer
    tr = W.make_trajectories(scene["g"], scene["inflate"], B=2, n_pts=40, seed=4)
    opt = scene["opt"]
    opt.setBoundaryStates(list(tr["start"][0]), [tr["end_pos"][0]])
    pts, dt = opt.optimize(tr["ctrl"][0], tr["dt"][0], O.NORMAL_PHASE | O.MINTIME, 1)
    assert pts.shape == (40, 3) and 0 < dt <= 5.0 and 1 <= opt.iter_num_ <= 2000 and opt.start_state_ == []
    x0 = W.pack_x(tr["ctrl"], tr["dt"])
    xg, fg, ng = opt.optimizeBatch(x0, gpu_consts(fuel, tr, 2), 40, O.NORMAL_PHASE | O.MINTIME, 1)
    assert np.all(ng == 1)
    assert np.allclose(xg, x0)
    t65 = W.make_trajectories(scene["g"], scene["inflate"], B=1, n_pts=65, seed=4)
    with pytest.raises(fuel.FuelGpuError):
        opt.optimizeBatch(W.pack_x(t65["ctrl"], t65["dt"]), gpu_consts(fuel, t65, 1), 65, O.NORMAL_PHASE | O.MINTIME, 8)


SHIM_LONG = r"""
#include <cstdio>
#include "fuelgpu_shim.hpp"
using namespace fast_planner;
// the shim's BsplineOptimizer::optimize() on one 40-point trajectory (scene of tests/shim_smoke.cpp without the wall)
int main(int argc, char** argv) {
  MapParam mp;
  mp.map_voxel_num_ = Vector3i(48, 40, 24);
  mp.resolution_ = 0.1;
  mp.map_origin_ = Vector3d(-2.4, -2.0, -0.5);
  mp.box_mind_ = Vector3d(-2.2, -1.8, -0.3);
  mp.box_maxd_ = Vector3d(2.2, 1.8, 1.7);
  mp.optimistic_ = true;
  std::shared_ptr<SDFMap> map(new SDFMap);
  map->initMap(mp);
  const double clamp_min = std::log(0.12 / 0.88);
  for (int x = 4; x < 44; ++x)
    for (int y = 4; y < 36; ++y)
      for (int z = 2; z < 22; ++z) {
        const int a = map->toAddress(x, y, z);
        const bool post = x >= 23 && x <= 25 && y >= 14 && y <= 16;
        map->occupancy_buffer_[a] = post ? 3.0 : clamp_min;
        if (post) map->occupancy_buffer_inflate_[a] = 1;
      }
  map->update_min_ = mp.map_origin_;
  map->update_max_ = Vector3d(2.4, 2.0, 1.9);
  map->updateESDF3d();
  std::shared_ptr<EDTEnvironment> env(new EDTEnvironment);
  env->setMap(map);
  BsplineOptimizer opt;
  opt.setEnvironment(env);
  FuelOptParams p{ 20.0, 10.0, 2.0, 100.0, 0.5, 1.5, 0.3, 0.0, 1.0, 0.7, 2.0, 2.0, 3 };
  const int iters[4] = { 2, 60, 200, 200 };
  opt.setParam(p, iters);
  std::vector<Vector3d> pts;
  for (int i = 0; i < 40; ++i) pts.emplace_back(-1.8 + 0.09 * i, -1.0 + 0.05 * i + ((i % 3) - 1) * 0.05, 0.6 + 0.01 * i);
  double dt = 0.1;
  auto avg = [&](int a, int b, int c) {
    return Vector3d((pts[a](0) + 4 * pts[b](0) + pts[c](0)) / 6, (pts[a](1) + 4 * pts[b](1) + pts[c](1)) / 6,
                    (pts[a](2) + 4 * pts[b](2) + pts[c](2)) / 6);
  };
  std::vector<Vector3d> start = { avg(0, 1, 2), Vector3d(0.9, 0.5, 0.1), Vector3d(0, 0, 0) };
  std::vector<Vector3d> end = { avg(39, 38, 37) };
  opt.setBoundaryStates(start, end);
  std::vector<double> x, grad;
  for (auto& q : pts)
    for (int k = 0; k < 3; ++k) x.push_back(q(k));
  x.push_back(dt);
  opt.fillTrajConst(pts, dt);
  const int mask = BsplineOptimizer::NORMAL_PHASE | BsplineOptimizer::MINTIME;
  const double f0 = opt.combineCost(x, grad, 40, mask);
  opt.optimize(pts, dt, mask, 1, 1);
  FILE* fo = std::fopen(argv[1], "w");
  std::fprintf(fo, "%zu %d %.17g %.17g %.17g\n", pts.size(), opt.iter_num_, f0, opt.min_cost_, dt);
  for (auto& q : pts) std::fprintf(fo, "%.17g %.17g %.17g\n", q(0), q(1), q(2));
  std::fclose(fo);
  return 0;
}
"""


@pytest.mark.gpu
def test_shim_optimize_long(tmp_path, orc):
    """The C++ shim's optimize() at 40 control points: it runs, lowers the cost, and min_cost_ is combineCost at the
    returned points."""
    from fuel_b200 import _lib
    _lib.lib()
    src, exe, out = tmp_path / "shim_long.cpp", str(tmp_path / "shim_long"), tmp_path / "out.txt"
    src.write_text(SHIM_LONG)
    subprocess.check_call(["g++", "-std=c++14", "-O2", "-I", os.path.join(ROOT, "include"), str(src), "-o", exe,
                           "-L", os.path.join(ROOT, "fuel_b200"), "-lfuelgpu", "-Wl,-rpath," + os.path.join(ROOT, "fuel_b200")])
    r = subprocess.run([exe, str(out)], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    lines = out.read_text().strip().split("\n")
    head = lines[0].split()
    n, neval, f0, fbest, dt = int(head[0]), int(head[1]), float(head[2]), float(head[3]), float(head[4])
    pts = np.array([[float(v) for v in ln.split()] for ln in lines[1:]])
    assert n == 40 and pts.shape == (40, 3) and 1 <= neval <= 60 and 0 < dt <= 5.0 and fbest < f0
    # the same scene on the oracle: min_cost_ re-evaluates at the returned points
    nv = (48, 40, 24)
    x, y, z = np.meshgrid(*[np.arange(k) for k in nv], indexing="ij")
    known = (x >= 4) & (x < 44) & (y >= 4) & (y < 36) & (z >= 2) & (z < 22)
    post = known & (x >= 23) & (x <= 25) & (y >= 14) & (y <= 16)
    tri = np.where(known, np.where(post, 2, 1), 0).astype(np.uint8)
    g = orc.make_grid(nv, 0.1, (-2.4, -2.0, -0.5), (-2.2, -1.8, -0.3), (2.2, 1.8, 1.7))
    d = orc.update_esdf3d(g, post.astype(np.int8), tri, [0, 0, 0], np.array(nv) - 1, True, False)
    p0 = np.array([[-1.8 + 0.09 * i, -1.0 + 0.05 * i + ((i % 3) - 1) * 0.05, 0.6 + 0.01 * i] for i in range(40)])
    tcs = orc.traj_consts(1)
    orc.fill_traj_const(tcs[0], orc.pt_dist(p0), 0.1, np.array([(p0[0] + 4 * p0[1] + p0[2]) / 6, [0.9, 0.5, 0.1], [0, 0, 0]]),
                        ((p0[39] + 4 * p0[38] + p0[37]) / 6)[None, :])
    mask = orc.NORMAL_PHASE | orc.MINTIME
    fr, _ = orc.combine_cost_batch(g, d, orc.opt_params(), tcs, 40, mask, np.concatenate([p0.reshape(-1), [0.1]])[None, :])
    assert abs(fr[0] - f0) <= 1e-4 * abs(fr[0])
    fr, _ = orc.combine_cost_batch(g, d, orc.opt_params(), tcs, 40, mask, np.concatenate([pts.reshape(-1), [dt]])[None, :])
    assert abs(fr[0] - fbest) <= 1e-4 * abs(fr[0])


# ---- CPU ------------------------------------------------------------------------------------------------------------

def test_cpu_twin_optimizes_64_points(orc, field):
    """orc_optimize_batch (the CPU twin the device solver is gated against) at 64 control points: the result stays in
    the bounds of optimize() and lowers the cost of every trajectory."""
    B, N, K = 64, 64, 64
    g = field["g"]
    tr = W.make_trajectories(g, field["inflate"], B=B, n_pts=N, seed=77)
    mask = orc.NORMAL_PHASE | orc.MINTIME
    x0 = W.pack_x(tr["ctrl"], tr["dt"])
    to = orc_consts(orc, tr, B)
    f0, _ = orc.combine_cost_batch(field["og"], field["d64"], orc.opt_params(), to, N, mask, x0, threads=8)
    xc, fc, nc = orc.optimize_batch(field["og"], field["d64"], orc.opt_params(), to, N, mask, x0, max_eval=K, threads=8)
    assert np.all(nc >= 1) and np.all(nc <= K)
    pts = xc[:, :3 * N].reshape(B, N, 3)
    assert np.all(pts >= g.box_min + 0.1 - 1e-12) and np.all(pts <= g.box_max - 0.1 + 1e-12)
    assert np.all(np.abs(pts - x0[:, :3 * N].reshape(B, N, 3)) <= 10.0 + 1e-12)
    assert np.all(xc[:, -1] >= 0.0) and np.all(xc[:, -1] <= 5.0)
    assert np.all(fc < f0)
    fchk, _ = orc.combine_cost_batch(field["og"], field["d64"], orc.opt_params(), to, N, mask, xc, threads=8)
    assert np.allclose(fchk, fc, rtol=1e-12)
