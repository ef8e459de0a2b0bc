"""The device's voxel walks on the H100 against the reference's own RayCaster (plan_env/src/raycast.cpp compiled into
oracle/_ref/libfuel_ref.so): every expected verdict comes from oracle.ref_raycast_ids and the map's occupancy, never from
a C oracle's walk.  One probe per walk, each read through a public entry:

- ray_is_clear<true> (view_cost.cu, ViewNode::searchPath's straight line): view_cost_batch's kind is LINE iff the
  reference's ids are all clear and inside the exploration box;
- ray_is_clear<false> (viewpoints.cu, countVisibleCells): sampleViewpointsRaw on single-cell clusters, visib 0 or 1;
- ray_is_clear<false> (astar.cu, shortenPath): astar_batch's waypoints on A* paths whose nodes sit on voxel faces;
- raycast_kernel (fusion.cu, inputPointCloud's misses): the log-odds after one frame.

Rays come from tests/ray_walks.py: random, axis-aligned, on voxel faces / edges / corners, exact lattice diagonals,
zero-length and within one voxel, through the strip just below the origin, on a grid whose origin is not a multiple
of the resolution, and overshooting rays, whose last steps tie at t = 1 so the reference steps past the end voxel and
never stops.  On those rays alone the expected verdict is the one over the reference's first 4096 ids: its own steps,
cut where the device's walks stop."""
import numpy as np
import pytest

import oracle.astar as OA
from fuel_b200._lib import check, lib, ptr
from fuel_b200.astar import astar_batch
from fuel_b200.view_node import ASTAR, LINE, NO_PATH, view_cost_batch
from tests import ray_walks as RW
from tests.helpers import make_sdf_map

pytestmark = pytest.mark.gpu

need_ref = pytest.mark.skipif(not RW.has_reference(), reason="oracle/_ref not built")
MIN_RAYS = 200
MIN_VIEW_RAYS = 100  # rays from a cell to its own target candidate


def line_kind(m, a, b):
    """view_cost_batch over the rays a -> b in chunks of 4096 -> kind [N]"""
    out = []
    for s in range(0, len(a), 4096):
        p1, p2 = a[s:s + 4096], b[s:s + 4096]
        z = np.zeros(len(p1))
        info, _ = view_cost_batch(m, p1, p2, z, z, np.zeros_like(p1), vm=2.0, yd=1.0, w_dir=1.5, resolution=0.4,
                                  lambda_heu=10000.0, allocate_num=4000, max_iter=1500, path_max=0)
        out.append(info["kind"])
    return np.concatenate(out)


@need_ref
@pytest.mark.parametrize("case", RW.LINE_CASES)
def test_straight_line_matches_reference_walk(fuel, case):
    geo, inflate, tri, fam = RW.line_case(case)
    m = make_sdf_map(fuel, geo.grid(), inflate, tri)
    try:
        blocks = RW.occ_flags(inflate, tri)
        kinds = set()
        for name, (a, b) in fam.items():
            assert len(a) >= MIN_RAYS, "%s: %d rays" % (name, len(a))
            want = RW.verdicts(geo, blocks, a, b, box=True)
            kind = line_kind(m, a, b)
            bad = np.flatnonzero((kind == LINE) != want)
            assert bad.size == 0, "%s: %d of %d rays differ, first %s -> %s (want clear=%s)" % (
                name, bad.size, len(a), a[bad[0]].tolist(), b[bad[0]].tolist(), want[bad[0]])
            assert 0 < want.sum() or name == "overshoot"
            kinds |= set(np.unique(kind).tolist())
        assert {LINE, ASTAR, NO_PATH} <= kinds
    finally:
        m.close()


@need_ref
def test_longest_legal_walk_reaches_its_end(fuel):
    """corner to corner of a 1024 x 1024 x 64 map, 1023 + 1023 + 63 steps, with one inflated voxel next to the end
    voxel on the walk: a guard shorter than the walk would call the line clear"""
    assert RW.guard_constants() == [RW.GUARD, RW.GUARD] and 3 * 1023 < RW.GUARD
    geo, inflate, tri, a, b, last = RW.longest_case()
    ids = RW.walk(geo, a, b)
    assert len(ids) == 1023 + 1023 + 63
    m = make_sdf_map(fuel, geo.grid(), inflate, tri)
    try:
        assert line_kind(m, a[None], b[None])[0] != LINE
        inflate[tuple(last)] = 0
        m.occupancy_buffer_inflate_[...] = inflate
        m.upload()
        assert line_kind(m, a[None], b[None])[0] == LINE
    finally:
        m.close()


@need_ref
@pytest.mark.parametrize("case", RW.VIEW_CASES)
def test_visible_cells_match_reference_walk(fuel, orc, case):
    """countVisibleCells through sampleViewpointsRaw: one cell per cluster, placed at each family's offset from a
    candidate; per (cluster, candidate) with the cell well inside the FOV, visib is exactly the reference walk's 0 / 1,
    and -1 where the candidate is rejected; the families are counted on the ray each one shaped, from its cell to its
    own target candidate.  Clusters of two cells at +-left_angle put both on the FOV planes: the oracle flags them as
    within 1e-9 of a plane, which is where the device redoes a candidate with the host's yaw, and the device's visib
    must equal the oracle's there.  (The device does not report whether its redo ran; n_border counts the oracle's
    flags, so it shows the clusters reach the planes.)"""
    geo, inflate, tri, avg, vp = RW.view_setup(case)
    m = make_sdf_map(fuel, geo.grid(), inflate, tri)
    try:
        ff = fuel.FrontierFinder(_env(fuel, m))
        ff.setViewParams(**vp)
        one = [fuel.Frontier(m, np.zeros(0, np.int32), avg[None] + 0.3, avg, avg, avg)]
        pos = ff.sampleViewpointsRaw(one)[0][0]
        inflate, tri = RW.clear_near(geo, inflate, tri, pos, vp["min_candidate_clearance"])
        m.occupancy_buffer_inflate_[...] = inflate
        m.setOccupancyBuffer(tristate=tri)
        m.upload()
        clusters, fams, tgt = RW.view_clusters(geo, pos, np.random.default_rng(5))
        ftrs = [fuel.Frontier(m, np.zeros(0, np.int32), c, avg, avg, avg) for c in clusters]
        pos2, _, vis = ff.sampleViewpointsRaw(ftrs)
        assert np.array_equal(pos2[0], pos)
        og = orc.make_grid(geo.n, geo.res, geo.origin, geo.box_mind, geo.box_maxd)
        rejected = orc.sample_viewpoints(og, tri, inflate, orc.view_params(**vp), avg, clusters[0])["visib"] < 0
        counts = RW.check_visib(geo, RW.occ_flags(inflate, tri), pos, clusters, fams, tgt, vis, vp, rejected)
        for name in RW.FAMILIES:
            assert counts.get(name, 0) >= MIN_VIEW_RAYS, counts
        # the FOV-border redo: the device agrees with the oracle where the oracle's plane test was within 1e-9 of zero
        n_border = 0
        for q in np.flatnonzero(np.array(fams) == "border"):
            r = orc.sample_viewpoints(og, tri, inflate, orc.view_params(**vp), avg, clusters[q])
            assert np.array_equal(vis[q], r["visib"])
            n_border += int(((r["visib"] >= 0) & (r["border"] != 0)).sum())
        assert n_border > 0
    finally:
        m.close()


def _env(fuel, m):
    env = fuel.EDTEnvironment()
    env.setMap(m)
    return env


@need_ref
@pytest.mark.parametrize("res", RW.FUSION_RES)
def test_fusion_matches_reference_walk(fuel, orc, res):
    """inputPointCloud frames whose points and cameras come from the ray families (no overshooting rays: pcl's float32
    points do not keep the rounding error they need): log-odds bit for bit against the
    update built from the reference's ids, and the tri-state byte against getOccupancy of it; where every walk of the
    frame ends inside the map, log-odds, tri-state and the local bound also against the reference's own sdf_map.cpp (which addresses outside its buffers on the other frames)."""
    geo = RW.fusion_geo(res)
    frames = RW.fusion_frames(geo, np.random.default_rng(11))
    n_clean = n_touched = 0
    per_family = {}
    for name, pts, cam in frames:
        m = fuel.SDFMap(geo.n, geo.res, geo.origin, map_size=geo.map_size)
        m.setFusionParams(max_ray_length=4.5)
        try:
            m.inputPointCloud(pts, len(pts), cam)
            got = m.getLogOdds().reshape(-1)
            lo, hi = m.local_bound_min_.copy(), m.local_bound_max_.copy()
            tri = np.empty(geo.shape, np.uint8)
            inf = np.empty(geo.shape, np.int8)
            check(lib().fuelgpu_map_download_occupancy(m._h, ptr(inf), ptr(tri)), m._h)
        finally:
            m.close()
        want = RW.fresh_logodds(geo)
        touched, clean = RW.expected_fusion(geo, want, pts, cam)
        n_touched += touched
        bad = np.flatnonzero(got != want)
        assert bad.size == 0, "%s: %d voxels differ, first %s" % (name, bad.size, np.unravel_index(bad[0], geo.shape))
        assert np.array_equal(tri.reshape(-1), RW.tristate(want)), name
        fam = name.split("/")[1]
        per_family[fam] = per_family.get(fam, 0) + len(pts)
        if clean:
            ref = RW.ref_fusion_map(res)
            assert ref.n == geo.shape and np.array_equal(ref.origin, geo.origin)
            try:
                ref.input_point_cloud(pts, cam)
                assert np.array_equal(ref.occupancy, got), name
                assert np.array_equal(RW.tristate(ref.occupancy), tri.reshape(-1)), name
                rlo, rhi = ref.get_local_bound()
                assert np.array_equal(lo, rlo) and np.array_equal(hi, rhi), name
            finally:
                ref.close()
            n_clean += 1
    assert n_clean >= 8 and n_touched > 10000
    for fam in RW.FUSION_FAMILIES:
        assert per_family.get(fam, 0) >= MIN_RAYS, per_family


@need_ref
@pytest.mark.parametrize("res,lam", [(0.2, 1.0), (0.4, 10000.0)])
def test_shorten_path_matches_reference_walk(fuel, res, lam):
    """shortenPath through astar_batch on test_lattice_ties's box, starts and goals on the voxel corners (no offset),
    scattered inflated and UNKNOWN voxels: the waypoints of every search equal shortenPath over the reference's walk.
    Searches whose shortenPath walks all end are compared bit for bit with the reference's astar2.cpp (RefAstar); it
    would never return on the others, which are compared with the A* oracle, pinned on the same rays by
    tests/test_ray_walk_families.py."""
    from tests.test_oracle_astar import Scene
    geo, inflate, tri, q = RW.astar_case()
    start, goal, fam = RW.astar_queries(q)
    m = make_sdf_map(fuel, geo.grid(), inflate, tri)
    sc = Scene(geo.grid(), inflate, tri)
    try:
        got = astar_batch(m, start, goal, resolution=res, lambda_heu=lam, allocate_num=20000, max_iter=100000,
                          path_max=512, w_max=32)
        counts, ended = RW.check_tours(geo, RW.occ_flags(inflate, tri), fam, *got)
        for name in RW.ASTAR_FAMILIES:
            assert counts.get(name, 0) >= 50, counts
        assert ended.sum() >= 300 and (~ended).sum() >= 20
        ra = OA.RefAstar(sc.ref, res, lam, 20000, 100000)
        try:
            want = ra.search_batch(start[ended], goal[ended], path_max=512, w_max=32)
        finally:
            ra.close()
        diff = RW.first_astar_difference(tuple(a[ended] for a in got), want)
        assert diff is None, "device vs reference: " + diff
        want = OA.search_batch(sc.om, start[~ended], goal[~ended], res, lam, 20000, 100000, path_max=512, w_max=32)
        diff = RW.first_astar_difference(tuple(a[~ended] for a in got), want)
        assert diff is None, "device vs oracle: " + diff
    finally:
        sc.close()
        m.close()
