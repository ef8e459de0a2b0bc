"""The ray families of tests/ray_walks.py and the C oracles' own walks (fuel_oracle_view.c, fuel_oracle_viewpoints.c,
fuel_oracle_fusion.c) against the reference's RayCaster, on the CPU.  tests/test_gpu_ray_walks.py checks the kernels
with the same rays and the same expected verdicts; here the oracles that every other device test compares with are
pinned to the reference's walk on exactly those rays.  Expected verdicts come from oracle.ref_raycast_ids (and the
reference's sdf_map.cpp for fusion), never from an oracle's walk."""
import numpy as np
import pytest

import oracle.astar as OA
import oracle.view as OV
from fuel_b200.view_node import LINE
from tests import ray_walks as RW

need_ref = pytest.mark.skipif(not RW.has_reference(), reason="oracle/_ref not built")
MIN_RAYS = 200


def test_guard_never_cuts_a_walk_that_ends():
    """every device walk stops after the same number of steps, more than the longest walk a legal map allows: corner
    to corner of 1024 x 1024 x 64 takes 1023 + 1023 + 63 steps"""
    g = RW.guard_constants()
    assert len(g) == 2 and set(g) == {RW.GUARD}, g
    assert 3 * 1023 < RW.GUARD


@need_ref
@pytest.mark.parametrize("case", RW.LINE_CASES)
def test_families_reach_their_edges(case):
    """each family has its rays, with the shapes it claims; overshooting rays are real: the reference's walk passes
    its end voxel and is still going after 4096 ids"""
    geo, _, _, fam = RW.line_case(case)
    assert set(fam) == set(RW.FAMILIES)
    for name, (a, b) in fam.items():
        assert len(a) >= MIN_RAYS, (name, len(a))
    a, b = fam["axis"]
    zero = np.floor(a / geo.res) == np.floor(b / geo.res)
    assert np.all(zero.sum(axis=1) >= 1) and np.any(zero.sum(axis=1) == 2)
    a, b = fam["diagonal"]
    d = np.round((b - a) / geo.res)
    assert np.all(np.count_nonzero(d, axis=1) >= 2)
    a, b = fam["short"]
    assert np.count_nonzero(np.all(a == b, axis=1)) >= 100
    a, _ = fam["below_origin"]
    strip = (a < geo.origin) & (a >= geo.origin - geo.res)
    assert np.all(strip.any(axis=1))
    a, b = fam["overshoot"]
    assert len(a) >= 300
    long = [len(RW.walk(geo, a[q], b[q])) for q in range(len(a))]
    assert np.all(np.array(long) == RW.GUARD)


@need_ref
@pytest.mark.parametrize("case", RW.LINE_CASES)
def test_oracle_straight_line_matches_reference_walk(case):
    geo, inflate, tri, fam = RW.line_case(case)
    om = OA.Map(geo.grid(), inflate, tri)
    blocks = RW.occ_flags(inflate, tri)
    for name, (a, b) in fam.items():
        want = RW.verdicts(geo, blocks, a, b, box=True)
        z = np.zeros(len(a))
        info, _ = OV.view_cost_batch(om, a, b, z, z, np.zeros_like(a), 2.0, 1.0, 1.5, 0.4, 10000.0, 4000, 1500, path_max=2)
        bad = np.flatnonzero((info["kind"] == LINE) != want)
        assert bad.size == 0, "%s: %d rays differ, first %s -> %s" % (name, bad.size, a[bad[0]].tolist(), b[bad[0]].tolist())


@need_ref
@pytest.mark.parametrize("case", RW.VIEW_CASES)
def test_oracle_visible_cells_match_reference_walk(orc, case):
    geo, inflate, tri, avg, vp = RW.view_setup(case)
    og = orc.make_grid(geo.n, geo.res, geo.origin, geo.box_mind, geo.box_maxd)
    ov = orc.view_params(**vp)
    pos = orc.sample_viewpoints(og, tri, inflate, ov, avg, avg[None] + 0.3)["pos"]
    inflate, tri = RW.clear_near(geo, inflate, tri, pos, vp["min_candidate_clearance"])
    clusters, fams, tgt = RW.view_clusters(geo, pos, np.random.default_rng(5))
    vis = np.zeros((len(clusters), len(pos)), np.int32)
    n_border = 0
    for q, c in enumerate(clusters):
        r = orc.sample_viewpoints(og, tri, inflate, ov, avg, c)
        assert np.array_equal(r["pos"], pos)
        vis[q] = r["visib"]
        if fams[q] == "border":
            n_border += int(((r["visib"] >= 0) & (r["border"] != 0)).sum())
    counts = RW.check_visib(geo, RW.occ_flags(inflate, tri), pos, clusters, fams, tgt, vis, vp)
    for name in RW.FAMILIES:
        assert counts.get(name, 0) >= 100, counts
    assert n_border > 0


@need_ref
@pytest.mark.parametrize("res", RW.FUSION_RES)
def test_oracle_fusion_matches_reference_walk(orc, res):
    """orc.Fusion against the update built from the reference's ids on every frame, and that update against the
    reference's own inputPointCloud wherever every walk of the frame ends inside the map"""
    geo = RW.fusion_geo(res)
    og = orc.make_grid(geo.n, geo.res, geo.origin, map_size=geo.map_size)
    n_clean = 0
    for name, pts, cam in RW.fusion_frames(geo, np.random.default_rng(11)):
        want = RW.fresh_logodds(geo)
        touched, clean = RW.expected_fusion(geo, want, pts, cam)
        f = orc.Fusion(og, orc.fusion_params())
        f.input_point_cloud(pts, cam)
        bad = np.flatnonzero(f.logodds != want)
        assert bad.size == 0, "%s: %d voxels differ" % (name, bad.size)
        if clean:
            ref = RW.ref_fusion_map(res)
            assert ref.n == geo.shape and np.array_equal(ref.origin, geo.origin)
            try:
                ref.input_point_cloud(pts, cam)
                assert np.array_equal(ref.occupancy, want), name
            finally:
                ref.close()
            n_clean += 1
    assert n_clean >= 8


@need_ref
@pytest.mark.parametrize("res,lam", [(0.2, 1.0), (0.4, 10000.0)])
def test_oracle_shorten_path_matches_reference_walk(res, lam):
    """the A* oracle's shortenPath on test_lattice_ties's box with starts and goals on the voxel corners: its waypoints
    equal shortenPath over the reference's walk on every search; where every walk of a search ends, the whole result
    equals the reference's astar2.cpp (which would never return on an overshooting ray)"""
    from tests.test_oracle_astar import Scene
    geo, inflate, tri, q = RW.astar_case()
    start, goal, fam = RW.astar_queries(q)
    sc = Scene(geo.grid(), inflate, tri)
    try:
        got = OA.search_batch(sc.om, start, goal, res, lam, 20000, 100000, path_max=512, w_max=32)
        counts, ended = RW.check_tours(geo, RW.occ_flags(inflate, tri), fam, *got)
        for name in RW.ASTAR_FAMILIES:
            assert counts.get(name, 0) >= 50, counts
        assert ended.sum() >= 300
        ra = OA.RefAstar(sc.ref, res, lam, 20000, 100000)
        try:
            want = ra.search_batch(start[ended], goal[ended], path_max=512, w_max=32)
        finally:
            ra.close()
        diff = RW.first_astar_difference(tuple(a[ended] for a in got), want)
        assert diff is None, "oracle vs reference: " + diff
    finally:
        sc.close()
