"""The CUDA path (through the C ABI) against golden OUTPUT vectors of the reference's own code
(tests/golden/ref_outputs.npz, written by tools/make_ref_golden.py from oracle/_ref = the reference's sdf_map.cpp,
frontier_finder.cpp, bspline_optimizer.cpp ... compiled unmodified in the build container).  No oracle in between.
Bars: ESDF at the exact bar of tests/esdf_exact.py (the stored fp32 values still determine the squared voxel
distance) with +inf where the reference holds its DBL_MAX sentinel; frontier clusters, cell sets,
flags bit-exact, filtered cells to the last float32 bit (cells of a cluster in ascending address on the device, BFS
order in the reference: compared as sorted sets, DESIGN.md "frontier cell order"); fused log-odds, local bounds, inflation bit-exact;
combineCost cost and gradient <= 1e-4; viewpoint positions exact, yaw <= 1e-9 rad, visible counts equal."""
import os

import numpy as np
import pytest

from fuel_b200 import workloads as W
from tests.esdf_exact import check_esdf

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_outputs.npz")


@pytest.fixture(scope="module")
def gold():
    d = dict(np.load(GOLD))
    n = tuple(int(v) for v in d["n"])
    d["shape"] = n
    d["inflate"] = np.unpackbits(d["inflate_bits"])[:int(np.prod(n))].astype(np.int8).reshape(n)
    d["mp"] = dict(zip(d["map_keys"], d["map_vals"]))
    return d


def make_map(fuel, gold, optimistic=False, signed=False):
    mp = gold["mp"]
    m = fuel.SDFMap(gold["shape"], float(gold["res"]), gold["origin"], [mp["box_min_" + a] for a in "xyz"],
                    [mp["box_max_" + a] for a in "xyz"], optimistic=optimistic, signed_dist=signed,
                    map_size=[mp["map_size_" + a] for a in "xyz"])
    return m


@pytest.mark.parametrize("name,opt,sgn", [("opt", True, False), ("nonopt", False, False), ("signed", True, True)])
def test_esdf_vs_reference(fuel, gold, name, opt, sgn):
    m = make_map(fuel, gold, opt, sgn)
    m.occupancy_buffer_inflate_[...] = gold["inflate"]
    m.setOccupancyBuffer(tristate=gold["tri"])
    m.upload()
    lo, hi = gold["esdf_lo"], gold["esdf_hi"]
    m.local_bound_min_, m.local_bound_max_ = lo, hi
    m.updateESDF3d()
    got = m.download(lo, hi)[lo[0]:hi[0] + 1, lo[1]:hi[1] + 1, lo[2]:hi[2] + 1]
    want = gold["esdf_" + name]
    check_esdf(got, want, float(gold["res"]), signed=sgn, ref_f32=True, label="golden " + name)
    m.close()


def test_frontier_and_viewpoints_vs_reference(fuel, gold):
    ffp = dict(zip(gold["ff_keys"], gold["ff_vals"]))
    pu = dict(zip(gold["pu_keys"], gold["pu_vals"]))
    m = make_map(fuel, gold)
    m.occupancy_buffer_inflate_[...] = gold["inflate"]
    m.setOccupancyBuffer(tristate=gold["tri"])
    m.upload()
    env = fuel.EDTEnvironment()
    env.setMap(m)
    # cell_order="bfs": cells_ in the reference's expandFrontier order, so average_ and the VoxelGrid centroids are
    # the reference's to the last bit and the viewpoint stage below runs on the device's own cluster data
    ff = fuel.FrontierFinder(env, cluster_min=int(ffp["cluster_min"]), cluster_size_xy=ffp["cluster_size_xy"],
                             down_sample=int(ffp["down_sample"]), cell_order="bfs")
    got = ff.search_box(gold["upd_min"], gold["upd_max"])
    off, foff = gold["fr_offsets"], gold["fr_foffsets"]
    assert len(got) == len(off) - 1
    for i, c in enumerate(got):
        assert np.array_equal(c.cells_addr_, gold["fr_addr"][off[i]:off[i + 1]]), "cluster %d cell order" % i
        want_f = gold["fr_filtered"][foff[i]:foff[i + 1]]
        assert np.array_equal(c.filtered_cells_, want_f), "cluster %d filtered" % i
        assert np.array_equal(c.average_, gold["fr_average"][i]), "cluster %d average" % i
        assert np.allclose(c.box_min_, gold["fr_box_min"][i], rtol=0, atol=1e-12)
        assert np.allclose(c.box_max_, gold["fr_box_max"][i], rtol=0, atol=1e-12)
    assert np.array_equal(np.packbits(ff.download_flags().astype(np.uint8)), gold["fr_flags_bits"])
    # computeFrontiersToVisit: which clusters keep viewpoints, and the viewpoints themselves
    ff.setViewParams(candidate_rmin=ffp["candidate_rmin"], candidate_rmax=ffp["candidate_rmax"],
                     candidate_rnum=int(ffp["candidate_rnum"]), candidate_dphi=ffp["candidate_dphi"],
                     min_candidate_clearance=ffp["min_candidate_clearance"], min_visib_num=int(ffp["min_visib_num"]),
                     min_view_finish_fraction=ffp["min_view_finish_fraction"], top_angle=pu["top_angle"],
                     left_angle=pu["left_angle"], right_angle=pu["right_angle"], max_dist=pu["max_dist"])
    ff.tmp_frontiers_ = got
    ff.computeFrontiersToVisit()
    kept = [got.index(f) for f in ff.frontiers_]
    assert kept == list(gold["vp_cluster"])
    voff = gold["vp_offsets"]
    n_all = 0
    for k, f in enumerate(ff.frontiers_):
        sl = slice(voff[k], voff[k + 1])
        theirs = sorted(zip(map(tuple, gold["vp_pos"][sl]), gold["vp_yaw"][sl], gold["vp_visib"][sl]))
        mine = sorted((tuple(v[0]), v[1], v[2]) for v in f.viewpoints_)
        assert len(mine) == len(theirs), "cluster %d keeps %d viewpoints, the reference %d" % (k, len(mine), len(theirs))
        for a, b in zip(mine, theirs):
            assert a[0] == b[0]                                    # candidate position: bit-exact
            assert abs(np.angle(np.exp(1j * (a[1] - b[1])))) < 1e-9 or (np.isnan(a[1]) and np.isnan(b[1]))
            assert a[2] == b[2], "visible count %d vs %d" % (a[2], b[2])  # integer output: exact
        n_all += len(theirs)
    assert n_all > 20
    m.close()


def test_fusion_and_inflation_vs_reference(fuel, gold):
    mp = gold["mp"]
    m = make_map(fuel, gold)
    m.setFusionParams(max_ray_length=mp["max_ray_length"])
    for pts, cam in zip(gold["fus_points"], gold["fus_cams"]):
        m.inputPointCloud(pts, pts.shape[0], cam)
    assert np.array_equal(m.getLogOdds().reshape(-1), gold["fus_logodds"])
    assert np.array_equal(m.local_bound_min_, gold["fus_local_lo"]) and np.array_equal(m.local_bound_max_, gold["fus_local_hi"])
    a, b = m.getUpdatedBox()
    assert np.array_equal(a, gold["fus_upd_min"]) and np.array_equal(b, gold["fus_upd_max"])
    m.clearAndInflateLocalMap(obstacles_inflation=mp["obstacles_inflation"], virtual_ceil_height=mp["virtual_ceil_height"])
    assert np.array_equal(np.packbits(m.occupancy_buffer_inflate_.astype(np.uint8)), gold["fus_inflate_bits"])
    m.close()


def test_combine_cost_vs_reference(fuel, gold):
    m = make_map(fuel, gold, optimistic=True)
    m.occupancy_buffer_inflate_[...] = gold["inflate"]
    m.setOccupancyBuffer(tristate=gold["tri"])
    m.upload()
    m.updateESDF3d()
    env = fuel.EDTEnvironment()
    env.setMap(m)
    opt = fuel.BsplineOptimizer()
    opt.setEnvironment(env)
    bs = dict(zip(gold["bs_keys"], gold["bs_vals"]))
    opt.setParam(ld_smooth=bs["ld_smooth"], ld_dist=bs["ld_dist"], ld_feasi=bs["ld_feasi"], ld_start=bs["ld_start"],
                 ld_end=bs["ld_end"], ld_time=bs["ld_time"], dist0=bs["dist0"], max_vel=bs["max_vel"], max_acc=bs["max_acc"])
    B = gold["bs_ctrl"].shape[0]
    for b in range(B):
        X = gold["bs_x"][b]
        P = X.shape[0]
        tcs = opt.traj_consts_from_arrays(np.repeat(gold["bs_pt_dist"][b], P), np.repeat(gold["bs_dt"][b], P),
                                          np.repeat(gold["bs_start"][b][None], P, axis=0),
                                          np.repeat(gold["bs_end"][b][None], P, axis=0))
        f, g = opt.combineCostBatch(X, tcs, 20, int(gold["bs_mask"]))
        fr, gr = gold["bs_f"][b], gold["bs_grad"][b]
        assert np.all(np.abs(f - fr) <= 1e-4 * np.abs(fr))
        sc = np.max(np.abs(gr), axis=1, keepdims=True)
        assert np.all(np.abs(g - gr) <= 1e-4 * np.maximum(np.abs(gr), 1e-3 * sc))
    m.close()
