"""Pins the oracle against the REFERENCE's own code: plan_env/src/{raycast,sdf_map}.cpp,
bspline_opt/src/bspline_optimizer.cpp and active_perception/src/{frontier_finder,perception_utils}.cpp are compiled
UNMODIFIED from the reference's sources into oracle/_ref/libfuel_ref.so (oracle/Makefile) against interface stand-ins
for the headers they need (oracle/ref_standin: Eigen small vectors/matrices, ros::NodeHandle::param, pcl containers, the
NLopt API, ...).  Every comparison below is bit-exact.  Not covered, by construction: pcl::VoxelGrid and
Eigen::EigenSolver (third-party algorithms; the stand-ins call the oracle's own reconstructions) and NLopt's iterates.
Where the reference library is not built, the digests of its results in tests/golden/refpin.json stand in for it
(tests/refgold.py)."""
import numpy as np
import pytest

import oracle as O
from tests.refgold import ref_map, refgold_fixture

O.build()  # also builds oracle/_ref/libfuel_ref.so where the reference's sources are present (it is git-ignored)


G = refgold_fixture()


def test_intbound_matches_reference(G):
    rng = np.random.default_rng(0)
    L = O.lib()
    L.orc_intbound.restype = O.C.c_double
    L.orc_intbound.argtypes = [O.C.c_double, O.C.c_double]
    s = np.concatenate([rng.uniform(-300, 300, 4000), np.round(rng.uniform(-300, 300, 500)), [0.0, -0.0, 1e-17, -1e-17]])
    ds = np.concatenate([rng.integers(-40, 41, 4000).astype(float), rng.integers(-40, 41, 504).astype(float)])
    got = [L.orc_intbound(a, b) for a, b in zip(s, ds)]
    G.eq(got, lambda: [O.ref_raycast().ref_intbound(a, b) for a, b in zip(s, ds)])


@pytest.mark.parametrize("origin,res", [((-10.0, -6.0, -1.0), 0.1), ((-25.6, -25.6, -1.0), 0.1), ((0.3, -2.7, 0.05), 0.15)])
def test_ray_traversal_matches_reference(G, origin, res):
    """Thousands of rays: random, axis-aligned, starting on voxel faces / corners, zero length, long diagonals."""
    rng = np.random.default_rng(7)
    g = O.make_grid((200, 120, 40), res, origin)
    o = np.array(origin)
    span = np.array([200, 120, 40]) * res
    rays, got = [], []
    for k in range(3000):
        a = o + rng.uniform(-0.1, 1.1, 3) * span
        b = o + rng.uniform(-0.1, 1.1, 3) * span
        if k % 5 == 1:
            b[rng.integers(0, 3)] = a[rng.integers(0, 3)]          # shared coordinate values
        if k % 7 == 2:
            a = o + np.round((a - o) / res) * res                  # start on voxel faces / corners
        if k % 11 == 3:
            b = a.copy()                                           # zero-length ray
        if k % 13 == 4:
            b = a + np.array([rng.uniform(-4.5, 4.5), 0.0, 0.0])   # axis-aligned
        if k % 17 == 5:
            a, b = np.float32(a).astype(np.float64), np.float32(b).astype(np.float64)  # float32 points, like pcl
        rays.append((a, b))
        got.append(O.raycast_ids(g, a, b))
    assert len(got) == 3000
    G.eq(got, lambda: [O.ref_raycast_ids(g, a, b) for a, b in rays])


# ---------------------------------------------------------------------------------------------------------
# SDFMap: the reference's own sdf_map.cpp (updateESDF3d / fillESDF, clearAndInflateLocalMap, inputPointCloud,
# getDistWithGrad) vs the oracle restatement, bit for bit (both are fp64, no FMA contraction).
# ---------------------------------------------------------------------------------------------------------
from fuel_b200 import workloads as W  # noqa: E402

BASE = dict(resolution=0.1, map_size_x=8.0, map_size_y=6.0, map_size_z=3.0, ground_height=-0.5, obstacles_inflation=0.199,
            local_bound_inflate=0.5, local_map_margin=50, default_dist=0.0, optimistic=0, signed_dist=0, p_hit=0.65,
            p_miss=0.35, p_min=0.12, p_max=0.90, p_occ=0.80, max_ray_length=4.5, virtual_ceil_height=-10.0)
FULL = ((0, 0, 0), (79, 59, 29))


def logit(p):
    return np.log(p / (1 - p))


def random_state(ref, seed, p_site=0.02):
    """random inflate bits + a blobby unknown region written straight into the reference's buffers"""
    rng = np.random.default_rng(seed)
    n = ref.n
    inflate = (rng.random(n) < p_site).astype(np.int8)
    tri = np.full(n, W.FREE, np.uint8)
    X, Y, Z = np.meshgrid(*[np.arange(k) for k in n], indexing="ij")
    for _ in range(5):
        c = rng.uniform(0, 1, 3) * np.array(n)
        r = rng.uniform(0.15, 0.4) * min(n)
        tri[((X - c[0]) ** 2 + (Y - c[1]) ** 2 + (Z - c[2]) ** 2) < r * r] = W.UNKNOWN
    tri[(inflate == 1) & (tri == W.FREE)] = W.OCCUPIED
    lo = np.where(tri == W.UNKNOWN, logit(0.12) - 0.01, np.where(tri == W.OCCUPIED, logit(0.90), logit(0.12)))
    ref.inflate[:] = inflate.reshape(-1)
    ref.occupancy[:] = lo.reshape(-1)
    return inflate, tri


def ref_esdf(ref, optimistic, signed, lo, hi):
    """the reference's updateESDF3d over the box [lo, hi] -> its whole distance buffer"""
    ref.distance[:] = 0.0
    ref.set_modes(optimistic, signed)
    ref.set_local_bound(lo, hi)
    ref.update_esdf3d()
    return ref.distance.copy()


@pytest.mark.parametrize("optimistic,signed", [(1, 0), (0, 0), (1, 1), (0, 1)])
def test_update_esdf3d_matches_reference(G, optimistic, signed):
    ref = ref_map(**BASE)
    assert ref.n == (80, 60, 30)
    g = ref.grid()
    for seed, (lo, hi) in enumerate([((0, 0, 0), (79, 59, 29)), ((10, 5, 3), (60, 50, 25)), ((33, 20, 7), (33, 40, 7)),
                                     ((0, 0, 0), (79, 0, 29))]):
        inflate, tri = random_state(ref, seed)
        got = O.update_esdf3d(g, inflate, tri, lo, hi, optimistic, signed)
        sl = tuple(slice(lo[i], hi[i] + 1) for i in range(3))
        G.eq(got[sl], lambda: ref_esdf(ref, optimistic, signed, lo, hi).reshape(ref.n)[sl])
    ref.close()


def test_esdf_sentinel_when_the_box_has_no_site(G):
    ref = ref_map(**BASE)
    ref.inflate[:] = 0
    ref.occupancy[:] = logit(0.12)  # all free, no obstacle: every voxel keeps the DBL_MAX envelope
    got = O.update_esdf3d(ref.grid(), np.zeros(ref.n, np.int8), np.full(ref.n, W.FREE, np.uint8), (5, 5, 5), (20, 20, 20), 1, 0)
    got = got[5:21, 5:21, 5:21]
    assert got.min() > 1e150
    G.eq(got, lambda: ref_esdf(ref, 1, 0, (5, 5, 5), (20, 20, 20)).reshape(ref.n)[5:21, 5:21, 5:21])
    ref.close()


@pytest.mark.parametrize("ceil_h", [-10.0, 1.5])
def test_clear_and_inflate_matches_reference(G, ceil_h):
    ref = ref_map(**dict(BASE, virtual_ceil_height=ceil_h))
    g = ref.grid()
    for seed, (lo, hi) in enumerate([((0, 0, 0), (79, 59, 29)), ((12, 8, 2), (70, 50, 27)), ((0, 0, 0), (3, 59, 29))]):
        inflate, tri = random_state(ref, 10 + seed, p_site=0.01)
        stale = (np.random.default_rng(seed).random(ref.n) < 0.05).astype(np.int8)   # leftovers the call must clear in the box
        ref.inflate[:] = stale.reshape(-1)
        inf_o, tri_o = stale.copy(), tri.copy()
        ceil_id = int(np.floor((ceil_h - ref.origin[2]) * 10.0)) if ceil_h > -0.5 else -1
        O.clear_and_inflate(g, tri_o, inf_o, lo, hi, 2, ceil_id)

        def want():
            ref.set_local_bound(lo, hi)
            ref.clear_and_inflate()
            return [ref.inflate.copy(), O.tristate_from_logodds(ref.occupancy, logit(0.12), logit(0.80))]
        G.eq([inf_o.reshape(-1), tri_o.reshape(-1)], want)
    ref.close()


def ref_fuse(ref, pts, cam):
    """the reference's inputPointCloud -> [log-odds, local bound min, local bound max]"""
    ref.input_point_cloud(pts, cam)
    return [ref.occupancy.copy(), *ref.get_local_bound()]


def test_input_point_cloud_matches_reference(G):
    ref = ref_map(**dict(BASE, max_ray_length=2.5))
    f = O.Fusion(ref.grid(), O.fusion_params(max_ray_length=2.5))
    G.eq(f.logodds, lambda: ref.occupancy.copy())          # initMap fill, sdf_map.cpp:64
    rng = np.random.default_rng(3)
    for frame in range(6):
        cam = np.array([rng.uniform(-3, 3), rng.uniform(-2, 2), rng.uniform(0.3, 2.0)])
        pts = cam + rng.normal(size=(4000, 3)) * np.array([2.0, 2.0, 0.8])
        pts[:60] = np.round(pts[:60])          # coordinates on voxel faces
        pts[60:120] = pts[60]                  # many points in one voxel
        pts[120:160] *= 6.0                    # far outside the map
        pts = pts.astype(np.float32)
        lo, hi = f.input_point_cloud(pts, cam)
        G.eq([f.logodds, lo, hi], lambda: ref_fuse(ref, pts, cam))
        if frame == 2:
            G.eq(list(f.updated_box(reset=True)), lambda: list(ref.updated_box(reset=True)))
    G.eq(list(f.updated_box()), lambda: list(ref.updated_box()))
    ref.close()


def test_depth_frames_then_inflate_then_esdf_chain_matches_reference(G):
    """The MapROS::depthPoseCallback + updateESDFCallback chain on synthetic depth frames of a furnished room."""
    ref = ref_map(**BASE)
    g = ref.grid()
    rng = np.random.default_rng(5)
    truth = np.zeros(ref.n, np.int8)
    truth[:, :, :6] = 1                                   # floor slab
    for _ in range(25):
        c = (rng.uniform(0.1, 0.9, 3) * np.array(ref.n)).astype(int)
        s = rng.integers(2, 8, 3)
        truth[c[0]:c[0] + s[0], c[1]:c[1] + s[1], 6:6 + 3 * s[2]] = 1
    wg = W.Grid(ref.n, tuple(ref.origin), ref.res)
    f = O.Fusion(g, O.fusion_params())
    inf_o = np.zeros(ref.n, np.int8)
    for k, yaw in enumerate((0.0, 1.3, 2.9, 4.4)):
        cam = np.array([0.3 * k - 0.4, 0.2 * k - 0.3, 1.0])
        pts = W.depth_frame(wg, truth, cam, yaw)
        lo, hi = f.input_point_cloud(pts, cam)
        G.eq([f.logodds, lo, hi], lambda: ref_fuse(ref, pts, cam))
        tri = f.tristate().reshape(ref.n).copy()
        O.clear_and_inflate(g, tri, inf_o, lo, hi, 2, -1)
        G.eq(inf_o.reshape(-1), lambda: (ref.clear_and_inflate(), ref.inflate.copy())[1])
        got = O.update_esdf3d(g, inf_o, tri, lo, hi, 0, 0)
        sl = tuple(slice(lo[i], hi[i] + 1) for i in range(3))
        G.eq(got[sl], lambda: (ref.update_esdf3d(), ref.distance.reshape(ref.n)[sl].copy())[1])
    ref.close()


def test_dist_with_grad_matches_reference(G):
    ref = ref_map(**BASE)
    inflate, tri = random_state(ref, 42, p_site=0.03)
    g = ref.grid()
    dist = O.update_esdf3d(g, inflate, tri, *FULL, 1, 0).reshape(-1)
    G.eq(dist, lambda: ref_esdf(ref, 1, 0, *FULL))
    rng = np.random.default_rng(1)
    pos = ref.origin + rng.uniform(-0.05, 1.05, (3000, 3)) * np.array(ref.n) * ref.res
    pos[:50] = ref.origin + np.round(rng.uniform(0, 1, (50, 3)) * np.array(ref.n)) * ref.res   # on voxel faces
    d, gr = O.dist_with_grad(g, dist, pos)
    G.eq([d, gr], lambda: list(ref.dist_with_grad(pos)))
    ref.close()


# ---------------------------------------------------------------------------------------------------------
# BsplineOptimizer::combineCost: the reference's own bspline_optimizer.cpp (every calc*Cost, costFunction, the
# set-up half of optimize()) vs the oracle restatement.  The NLopt stand-in evaluates the reference's objective
# at its own start point and at probe points.
# ---------------------------------------------------------------------------------------------------------
OPT = dict(ld_smooth=20.0, ld_dist=10.0, ld_feasi=2.0, ld_start=100.0, ld_end=0.5, ld_guide=1.5, ld_waypt=0.3, ld_view=0.0,
           ld_time=1.0, dist0=0.7, max_vel=2.0, max_acc=2.0, dlmin=0.0, wnl=0.0, max_iteration_num1=2, max_iteration_num2=2000,
           max_iteration_num3=200, max_iteration_num4=200, max_iteration_time1=0.0001, max_iteration_time2=0.005,
           max_iteration_time3=0.003, max_iteration_time4=0.003, algorithm1=15, algorithm2=11, bspline_degree=3)


def ref_optimizer(ref, **params):
    return O.RefBsplineOptimizer(ref, **params) if O.ref_raycast() is not None else None


def start_point(ref, ctrl, dt, nvar):
    """what optimize() hands to NLopt: the control points clamped to the box shrunk by 0.1 m (:175-217), then dt"""
    bmin, bmax = ref.origin + 0.1, ref.origin + np.array(ref.n) * ref.res - 0.1
    return np.concatenate([np.clip(ctrl, bmin, bmax).reshape(-1), [dt]])[:nvar]


def oracle_costs(sc, tc, N, mask, X):
    f = np.zeros(len(X))
    gr = np.zeros(X.shape)
    for i in range(len(X)):
        fi, gi = O.combine_cost_batch(sc["g"], sc["dist"], sc["p"], tc, N, mask, X[i:i + 1])
        f[i], gr[i] = fi[0], gi[0]
    return f, gr


@pytest.fixture(scope="module")
def opt_scene():
    ref = ref_map(**BASE)
    inflate, tri = random_state(ref, 77, p_site=0.004)
    g = ref.grid()
    dist = O.update_esdf3d(g, inflate, tri, *FULL, 1, 0).reshape(-1)
    opt = None
    if O.ref_raycast() is not None:
        ref_esdf(ref, 1, 0, *FULL)
        opt = O.RefBsplineOptimizer(ref, **OPT)
    wg = W.Grid(ref.n, tuple(ref.origin), ref.res)
    tr = W.make_trajectories(wg, inflate, B=12, n_pts=20, seed=31)
    yield dict(ref=ref, opt=opt, tr=tr, g=g, dist=dist, p=O.opt_params(ld_waypt=0.3))
    if opt is not None:
        opt.close()
    ref.close()


def _check(G, sc, b, mask, end, guide=None, waypts=None, widx=None, time_lb=-1.0, n_probe=6, seed=0):
    tr, N = sc["tr"], 20
    rng = np.random.default_rng(seed + 100 * b)
    ctrl, dt, start = tr["ctrl"][b], float(tr["dt"][b]), tr["start"][b]
    nvar = 3 * N + (1 if mask & O.MINTIME else 0)
    x_init = np.concatenate([ctrl.reshape(-1), [dt]])[:nvar]
    probes = x_init + rng.normal(size=(n_probe, nvar)) * 0.25
    if mask & O.MINTIME:
        probes[:, -1] = np.abs(probes[:, -1]) + 0.05
        probes[0, -1] = 0.11      # fast: velocity / acceleration limits active
    # the start point and bounds optimize() hands to NLopt: bounds +-10 m clipped to the shrunk box, dt in [0, 5]
    ref = sc["ref"]
    bmin, bmax = ref.origin + 0.1, ref.origin + np.array(ref.n) * ref.res - 0.1
    x0 = start_point(ref, ctrl, dt, nvar)
    lb = np.maximum(x0[:3 * N].reshape(N, 3) - 10.0, bmin).reshape(-1)
    ub = np.minimum(x0[:3 * N].reshape(N, 3) + 10.0, bmax).reshape(-1)
    if mask & O.MINTIME:
        lb, ub = np.append(lb, 0.0), np.append(ub, 5.0)
    # the oracle on the same points
    tc = O.traj_consts(1)
    O.fill_traj_const(tc[0], O.pt_dist(ctrl), dt, start, end, time_lb, guide, waypts, widx)
    f, g = oracle_costs(sc, tc, N, mask, np.concatenate([x0[None, :], probes]))

    def want():
        r = sc["opt"].evaluate(ctrl, dt, mask, start, end, guide, waypts, widx, time_lb, probes)
        return [r["x0"], r["lb"], r["ub"], r["f"], r["grad"]]
    G.eq([x0, lb, ub, f, g], want)


def test_combine_cost_exploration_objective_matches_reference(G, opt_scene):
    """NORMAL_PHASE | MINTIME, the objective of the exploration replan (and of bench.py), bit for bit."""
    G.eq(opt_scene["dist"], lambda: opt_scene["ref"].distance.copy())
    mask = O.NORMAL_PHASE | O.MINTIME
    for b in range(12):
        _check(G, opt_scene, b, mask, opt_scene["tr"]["end_pos"][b][None, :])


def test_combine_cost_other_terms_match_reference(G, opt_scene):
    sc = opt_scene
    tr = sc["tr"]
    rng = np.random.default_rng(9)
    for b in range(6):
        endp = tr["end_pos"][b]
        # fixed knot span (no MINTIME), end state with 1, 2, 3 rows
        for n_end in (1, 2, 3):
            end = np.concatenate([endp[None, :], rng.normal(size=(2, 3)) * 0.5])[:n_end]
            _check(G, sc, b, O.NORMAL_PHASE, end, seed=n_end)
        # GUIDE_PHASE with a guide path (N - 2*order points) and a duration lower bound
        guide = tr["ctrl"][b][3:17] + rng.normal(size=(14, 3)) * 0.2
        _check(G, sc, b, O.GUIDE_PHASE | O.MINTIME, endp[None, :], guide=guide, time_lb=9.0, seed=7)
        # way points
        widx = np.array([2, 7, 11], np.int32)
        wp = tr["ctrl"][b][widx + 1] + rng.normal(size=(3, 3)) * 0.1
        _check(G, sc, b, O.SMOOTHNESS | O.WAYPOINTS | O.START | O.END | O.MINTIME, endp[None, :], waypts=wp, widx=widx,
               seed=8)


# ---------------------------------------------------------------------------------------------------------
# FrontierFinder: the reference's own frontier_finder.cpp + perception_utils.cpp (searchFrontiers, expandFrontier,
# computeFrontierInfo, splitLargeFrontiers, computeFrontiersToVisit / sampleViewpoints / countVisibleCells,
# isFrontierCovered) vs the oracle.  pcl::VoxelGrid and Eigen::EigenSolver are the oracle's reconstructions on BOTH
# sides (ref_standin), so they are not what is being checked here.
# ---------------------------------------------------------------------------------------------------------
FF = dict(cluster_min=20, cluster_size_xy=1.0, cluster_size_z=10.0, min_candidate_dist=0.75, min_candidate_clearance=0.21,
          candidate_dphi=15 * 3.1415926 / 180.0, candidate_rmax=2.5, candidate_rmin=1.5, candidate_rnum=3, down_sample=3,
          min_visib_num=8, min_view_finish_fraction=0.2)
PU = dict(top_angle=0.56125, left_angle=0.69222, right_angle=0.68901, max_dist=4.5, vis_dist=1.0)


def frontier_scene(seed, box=None):
    params = dict(BASE)
    if box is not None:
        for ax, lo, hi in zip("xyz", box[0], box[1]):
            params["box_min_" + ax], params["box_max_" + ax] = lo, hi
    ref = ref_map(**params)
    rng = np.random.default_rng(seed)
    n = ref.n
    inflate = (rng.random(n) < 0.003).astype(np.int8)
    # known region: a few camera balls; the rest unknown
    X, Y, Z = np.meshgrid(*[np.arange(k) for k in n], indexing="ij")
    known = np.zeros(n, bool)
    for _ in range(5):
        c = rng.uniform(0.2, 0.8, 3) * np.array(n)
        r = rng.uniform(0.2, 0.45) * min(n[0], n[1])
        known |= ((X - c[0]) ** 2 + (Y - c[1]) ** 2 + 4.0 * (Z - c[2]) ** 2) < r * r
    tri = np.where(known, W.FREE, W.UNKNOWN).astype(np.uint8)
    tri[known & (inflate == 1)] = W.OCCUPIED
    inflate[~known] = 0
    lo = np.where(tri == W.UNKNOWN, logit(0.12) - 0.01, np.where(tri == W.OCCUPIED, logit(0.90), logit(0.12)))
    ref.inflate[:] = inflate.reshape(-1)
    ref.occupancy[:] = lo.reshape(-1)
    return ref, inflate, tri


def ref_finder(ref):
    return O.RefFrontierFinder(ref, PU, **FF) if O.ref_raycast() is not None else None


def clusters(lst):
    """cells in BFS order, filtered cells and the cluster info of each cluster"""
    return [{k: c[k] for k in ("addr", "filtered", "average", "box_min", "box_max")} for c in lst]


def oracle_frontier_params():
    return O.frontier_params(cluster_min=FF["cluster_min"], cluster_size_xy=FF["cluster_size_xy"], down_sample=FF["down_sample"],
                             cell_order=0)


@pytest.mark.parametrize("seed,box,upd", [
    (1, None, ((-4.0, -3.0, -0.5), (4.0, 3.0, 2.5))),
    (2, ((-3.5, -2.5, -0.3), (3.5, 2.5, 2.2)), ((-4.0, -3.0, -0.5), (4.0, 3.0, 2.5))),
    (3, ((-3.5, -2.5, -0.3), (3.5, 2.5, 2.2)), ((-1.0, -2.0, 0.0), (2.5, 1.0, 1.5))),
    (4, None, ((0.5, -1.0, 0.2), (3.0, 2.5, 1.8))),
])
def test_search_frontiers_matches_reference(G, seed, box, upd):
    ref, inflate, tri = frontier_scene(seed, box)
    ff = ref_finder(ref)
    g = ref.grid(*(box if box is not None else (None, None)))
    flag = np.zeros(ref.n, np.int8)
    got = O.frontier_search(g, tri, flag, upd[0], upd[1], oracle_frontier_params())
    assert len(got) >= 3
    G.eq([clusters(got), flag.reshape(-1)], lambda: [clusters(ff.search(*upd)), ff.flags.copy()])
    # a second search over a different updated box keeps the flags of the first (persistent frontier_flag_)
    upd2 = ((-4.0, -3.0, -0.5), (0.0, 3.0, 2.5))
    got2 = O.frontier_search(g, tri, flag, upd2[0], upd2[1], oracle_frontier_params())
    G.eq([clusters(got2), flag.reshape(-1)], lambda: [clusters(ff.search(*upd2)), ff.flags.copy()])
    if ff is not None:
        ff.close()
    ref.close()


def views(visib, yaw, pos):
    """viewpoints as a sorted multiset: the reference sorts by visib_num_ (std::sort, tie order unspecified)"""
    return [list(v) for v in sorted(zip(-np.asarray(visib), yaw, map(tuple, pos)))]


def test_viewpoints_and_coverage_match_reference(G):
    """computeFrontiersToVisit (sampleViewpoints / countVisibleCells / isNearUnknown, PerceptionUtils) and
    isFrontierCovered.  Same libm on both sides here, so yaw and counts are compared exactly."""
    ref, inflate, tri = frontier_scene(6, ((-3.6, -2.6, -0.3), (3.6, 2.6, 2.2)))
    ff = ref_finder(ref)
    upd = ((-4.0, -3.0, -0.5), (4.0, 3.0, 2.5))
    g = ref.grid((-3.6, -2.6, -0.3), (3.6, 2.6, 2.2))
    tmp = O.frontier_search(g, tri, np.zeros(ref.n, np.int8), upd[0], upd[1], oracle_frontier_params())
    G.eq(clusters(tmp), lambda: clusters(ff.search(*upd)))
    vp = O.view_params()
    visit, dormant = [], []
    for t in tmp:
        r = O.sample_viewpoints(g, tri, inflate, vp, t["average"], t["filtered"])
        keep = np.nonzero(r["visib"] > FF["min_visib_num"])[0]
        if len(keep) == 0:
            dormant.append(t["addr"])
        else:
            visit.append(dict(addr=t["addr"], id=len(visit), views=views(r["visib"][keep], r["yaw"][keep], r["pos"][keep])))
    assert len(visit) >= 2

    def want():
        v, d = ff.compute_to_visit()
        for x in v:
            assert list(x["view_visib"]) == sorted(x["view_visib"], reverse=True)
        return [[dict(addr=x["addr"], id=x["id"], views=views(x["view_visib"], x["view_yaw"], x["view_pos"])) for x in v],
                [x["addr"] for x in d]]
    G.eq([visit, dormant], want)
    # isFrontierCovered: nothing changed -> False; reveal the surroundings of the first cluster -> True
    first = visit[0]["addr"]
    cnt0 = O.frontier_changed_count(g, tri, first)
    assert cnt0 == 0
    G.eq(False, lambda: (ref.R.ref_map_set_updated_box(ref.h, O._p(np.array(upd[0])), O._p(np.array(upd[1]))),
                         ff.is_covered())[1])
    idx = np.stack(np.unravel_index(first, ref.n), axis=1)
    occ = ref.occupancy.reshape(ref.n)
    tri2 = tri.copy()
    for d in (-1, 1):
        for ax in range(3):
            j = idx.copy()
            j[:, ax] = np.clip(j[:, ax] + d, 0, ref.n[ax] - 1)
            sel = tri2[j[:, 0], j[:, 1], j[:, 2]] == W.UNKNOWN
            tri2[j[sel, 0], j[sel, 1], j[sel, 2]] = W.FREE
            occ[j[sel, 0], j[sel, 1], j[sel, 2]] = logit(0.12)
    cnt = O.frontier_changed_count(g, tri2, first)
    assert cnt >= max(int(FF["min_view_finish_fraction"] * len(first)), 1)
    G.eq(True, lambda: ff.is_covered())
    if ff is not None:
        ff.close()
    ref.close()


def test_map_size_that_is_not_a_multiple_of_the_resolution(G):
    """map_voxel_num_ = ceil(size / resolution) but map_max_boundary_ = origin + size (sdf_map.cpp:34-39): with a size of
    6.45 m the last voxel column lies partly outside the map.  isInMap / closetPointInMap / getDistWithGrad use the
    metric boundary; the oracle takes it through OrcGrid.map_size (the C ABI through FuelGridDesc.map_size)."""
    ref = ref_map(**dict(BASE, map_size_x=6.45, map_size_y=4.83, map_size_z=2.41, max_ray_length=2.0))
    assert ref.n == (65, 49, 25)
    g = ref.grid()
    f = O.Fusion(g, O.fusion_params(max_ray_length=2.0))
    rng = np.random.default_rng(8)
    for frame in range(4):
        cam = np.array([rng.uniform(1.5, 3.0), rng.uniform(1.0, 2.2), rng.uniform(0.5, 1.6)])   # close to the +x/+y/+z faces
        pts = (cam + rng.normal(size=(3000, 3)) * np.array([1.5, 1.5, 0.8])).astype(np.float32)
        lo, hi = f.input_point_cloud(pts, cam)
        G.eq([f.logodds, lo, hi], lambda: ref_fuse(ref, pts, cam))
    # non-optimistic ESDF of the fused map (no inflation was run: the inflate buffer is still all zero)
    full = ((0, 0, 0), np.array(ref.n) - 1)
    dist = O.update_esdf3d(g, np.zeros(ref.n, np.int8), f.tristate().reshape(ref.n).copy(), *full, 0, 0).reshape(-1)
    G.eq(dist, lambda: ref_esdf(ref, 0, 0, *full))
    top = ref.origin + ref.map_size
    pos = top - rng.uniform(-0.02, 0.15, (2000, 3))          # around the upper faces
    d, gr = O.dist_with_grad(g, dist, pos)
    G.eq([d, gr], lambda: list(ref.dist_with_grad(pos)))
    assert (d == 0).sum() > 100 and (d != 0).sum() > 100
    ref.close()


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_combine_cost_random_weights_sizes_and_masks(G, seed):
    """Random lambda weights / limits, 8..31 control points, random term masks, end-state rows and duration bounds."""
    rng = np.random.default_rng(seed)
    ref = ref_map(**BASE)
    inflate, tri = random_state(ref, 300 + seed, p_site=float(rng.choice([0.002, 0.01])))
    optimistic = int(rng.integers(0, 2))
    g = ref.grid()
    dist = O.update_esdf3d(g, inflate, tri, *FULL, optimistic, 0).reshape(-1)
    G.eq(dist, lambda: ref_esdf(ref, optimistic, 0, *FULL))
    keys = ("ld_smooth", "ld_dist", "ld_feasi", "ld_start", "ld_end", "ld_guide", "ld_waypt", "ld_time", "dist0", "max_vel", "max_acc")
    lo_hi = dict(ld_smooth=(1, 30), ld_dist=(1, 20), ld_feasi=(0.5, 5), ld_start=(1, 100), ld_end=(0.1, 5), ld_guide=(0.5, 3),
                 ld_waypt=(0.1, 2), ld_time=(0.5, 3), dist0=(0.3, 1.2), max_vel=(0.5, 3), max_acc=(0.5, 3))
    w = {k: float(rng.uniform(*lo_hi[k])) for k in keys}
    opt = ref_optimizer(ref, **dict(OPT, **w))
    sc = dict(g=g, dist=dist, p=O.opt_params(**w))
    N = int(rng.choice([8, 12, 20, 31]))
    tr = W.make_trajectories(W.Grid(ref.n, tuple(ref.origin), ref.res), inflate, B=5, n_pts=N, seed=seed)
    for b in range(5):
        mask = int(rng.choice([O.NORMAL_PHASE | O.MINTIME, O.NORMAL_PHASE, O.GUIDE_PHASE | O.MINTIME,
                               O.SMOOTHNESS | O.WAYPOINTS | O.START | O.END, O.DISTANCE | O.FEASIBILITY | O.MINTIME]))
        ctrl, dt, start = tr["ctrl"][b], float(tr["dt"][b]), tr["start"][b]
        guide = ctrl[3:N - 3] + rng.normal(size=(N - 6, 3)) * 0.2 if mask & O.GUIDE else None
        widx = np.array([1, N // 2 - 1, N - 4], np.int32) if mask & O.WAYPOINTS else None
        wp = ctrl[widx + 1] + rng.normal(size=(3, 3)) * 0.1 if widx is not None else None
        end = np.concatenate([tr["end_pos"][b][None, :], rng.normal(size=(2, 3)) * 0.5])[:int(rng.integers(1, 4))]
        tlb = float(rng.choice([-1.0, 6.0, 20.0]))
        nvar = 3 * N + (1 if mask & O.MINTIME else 0)
        probes = np.concatenate([ctrl.reshape(-1), [dt]])[:nvar] + rng.normal(size=(4, nvar)) * 0.3
        if mask & O.MINTIME:
            probes[:, -1] = np.abs(probes[:, -1]) + 0.03
        x0 = start_point(ref, ctrl, dt, nvar)
        tc = O.traj_consts(1)
        O.fill_traj_const(tc[0], O.pt_dist(ctrl), dt, start, end, tlb, guide, wp, widx)
        f, gr = oracle_costs(sc, tc, N, mask, np.concatenate([x0[None, :], probes]))

        def want():
            r = opt.evaluate(ctrl, dt, mask, start, end, guide, wp, widx, tlb, probes)
            return [r["x0"], r["f"], r["grad"]]
        G.eq([x0, f, gr], want)
    if opt is not None:
        opt.close()
    ref.close()


def test_host_mirror_pt_dist_is_the_reference_value(opt_scene):
    """pt_dist_ (bspline_optimizer.cpp:136-140) as the Python mirror and workloads.make_trajectories compute it ==
    the oracle's, which the tests above pin to the reference through the smoothness term."""
    import fuel_b200
    tr = opt_scene["tr"]
    for b in range(tr["ctrl"].shape[0]):
        assert fuel_b200.BsplineOptimizer.pt_dist(tr["ctrl"][b]) == O.pt_dist(tr["ctrl"][b]) == tr["pt_dist"][b]


@pytest.mark.parametrize("seed", [0, 1])
def test_view_cost_matches_reference(G, seed):
    """calcViewCost (bspline_optimizer.cpp:477-502, VIEWCONS): the perpendicular part, the parallel part on both sides of
    its |dl| < |dir| switch, random ld_view / wnl, alone and inside a full objective -- bit for bit."""
    rng = np.random.default_rng(40 + seed)
    ref = ref_map(**BASE)
    inflate, tri = random_state(ref, 500 + seed)
    g = ref.grid()
    dist = O.update_esdf3d(g, inflate, tri, *FULL, 1, 0).reshape(-1)
    G.eq(dist, lambda: ref_esdf(ref, 1, 0, *FULL))
    w = dict(ld_view=float(rng.uniform(0.5, 5)), wnl=float(rng.uniform(0.2, 3)))
    opt = ref_optimizer(ref, **dict(OPT, **w))
    sc = dict(g=g, dist=dist, p=O.opt_params(**w))
    N = 20
    tr = W.make_trajectories(W.Grid(ref.n, tuple(ref.origin), ref.res), inflate, B=6, n_pts=N, seed=seed)
    n_par = 0
    for b in range(6):
        ctrl, dt, start = tr["ctrl"][b], float(tr["dt"][b]), tr["start"][b]
        idx = int(rng.integers(3, N - 3))
        pt = ctrl[idx] + rng.normal(size=3) * 0.4
        # direction roughly along / against (pt -> control point), short or long safe distance
        d = (ctrl[idx] - pt) * float(rng.choice([-1.0, 1.0])) + rng.normal(size=3) * 0.1
        d = d / np.linalg.norm(d) * float(rng.choice([0.2, 1.5]))
        view = (pt, d, idx)
        for mask in (O.VIEWCONS, O.NORMAL_PHASE | O.VIEWCONS | O.MINTIME):
            nvar = 3 * N + (1 if mask & O.MINTIME else 0)
            probes = np.concatenate([ctrl.reshape(-1), [dt]])[:nvar] + rng.normal(size=(3, nvar)) * 0.2
            if mask & O.MINTIME:
                probes[:, -1] = np.abs(probes[:, -1]) + 0.03
            x0 = start_point(ref, ctrl, dt, nvar)
            tc = O.traj_consts(1)
            O.fill_traj_const(tc[0], O.pt_dist(ctrl), dt, start, tr["end_pos"][b][None, :], view=view)
            X = np.concatenate([x0[None, :], probes])
            f, gr = oracle_costs(sc, tc, N, mask, X)

            def want():
                r = opt.evaluate(ctrl, dt, mask, start, tr["end_pos"][b][None, :], probes=probes, view=view)
                return [r["x0"], r["f"], r["grad"]]
            G.eq([x0, f, gr], want)
            if mask == O.VIEWCONS:
                q = X[0][:3 * N].reshape(N, 3)[idx] - pt
                n_par += int(abs(np.dot(q, d / np.linalg.norm(d))) < np.linalg.norm(d))
                assert np.count_nonzero(gr[0]) <= 3  # one control point only
    assert n_par >= 1  # the wnl branch was taken at least once
    if opt is not None:
        opt.close()
    ref.close()
