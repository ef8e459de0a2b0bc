"""The small frontier path (one cluster kernel; its counters and a prefix of its results come back in one copy) against
the multi-kernel path on the same candidates (fuelgpu_frontier_search_from_candidates) and against the CPU oracle:
cells, cluster order, average_, box, filtered_cells_ and frontier_flag_, bit for bit.  Covers every sweep layout of a
z line (nz % 32 == 0 or not), search boxes that end inside a z word, the office maps, results larger than the prefix
that the first copy brings back (cells or clusters), a second search after flags were reset, and the BFS cell order."""
import numpy as np
import pytest

from fuel_b200 import workloads as W
from tests.helpers import make_sdf_map, orc_grid, random_scene

pytestmark = pytest.mark.gpu


def finder(fuel, g, inflate, tri, **kw):
    m = make_sdf_map(fuel, g, inflate, tri)
    env = fuel.EDTEnvironment()
    env.setMap(m)
    return m, fuel.FrontierFinder(env, **kw)


def assert_equal_lists(got, want):
    assert len(got) == len(want)
    for i, (a, b) in enumerate(zip(got, want)):
        assert np.array_equal(a.cells_addr_, b.cells_addr_), "cluster %d cells differ" % i
        assert np.array_equal(a.average_, b.average_), "cluster %d average_ differs" % i
        assert np.array_equal(a.filtered_cells_, b.filtered_cells_), "cluster %d filtered_cells_ differ" % i
        assert np.array_equal(a.box_min_, b.box_min_) and np.array_equal(a.box_max_, b.box_max_)


def assert_equal_oracle(got, ref):
    assert len(got) == len(ref)
    for i, (a, b) in enumerate(zip(got, ref)):
        assert np.array_equal(a.cells_addr_, b["addr"]), "cluster %d cells differ" % i
        assert np.array_equal(a.filtered_cells_, b["filtered"]), "cluster %d filtered_cells_ differ" % i
        assert np.allclose(a.average_, b["average"], rtol=1e-12, atol=1e-12)


def small_vs_large(fuel, orc, g, inflate, tri, boxes, kw, reset=None):
    """search_box (small path) on one map, candidates + search_from_candidates (multi-kernel path) on another, the oracle
    on the host, for a sequence of update boxes on the flags the previous searches left."""
    (m1, ff1), (m2, ff2) = finder(fuel, g, inflate, tri, **kw), finder(fuel, g, inflate, tri, **kw)
    fl = np.zeros(g.n, dtype=np.int8)
    p = orc.frontier_params(cell_order=1, **kw)
    outs = []
    for it, (umin, umax) in enumerate(boxes):
        if it > 0 and reset is not None:  # resetFlag (:62-69) of some clusters of the previous search on both maps
            addr = np.ascontiguousarray(np.concatenate([outs[-1][k].cells_addr_ for k in reset(len(outs[-1]))]))
            ff1._clear_flags(addr)
            ff2._clear_flags(addr)
            fl.reshape(-1)[addr] = 0
        small = ff1.search_box(umin, umax)
        addr, cls = ff2.candidates(umin, umax, 0, g.n[2] - 1)
        large = ff2.search_from_candidates(umin, umax, addr, cls)
        ref = orc.frontier_search(orc_grid(orc, g), tri, fl, umin, umax, p)
        assert len(small) > 0
        assert_equal_lists(small, large)
        assert_equal_oracle(small, ref)
        assert np.array_equal(ff1.download_flags(), fl) and np.array_equal(ff2.download_flags(), fl)
        outs.append(small)
    m1.close()
    m2.close()
    return outs


@pytest.mark.parametrize("nz", [32, 40, 41, 63, 64])
def test_every_z_layout(fuel, orc, nz):
    n = (48, 40, nz)
    origin = np.array([-1.0, -2.0, -0.5])
    g0 = W.Grid(n, origin, 0.1)
    g = W.Grid(n, origin, 0.1, box_min=origin + 0.2, box_max=g0.map_max - 0.2)
    inflate, tri = random_scene(n, 40 + nz, p_site=0.01, p_unknown=0.5, blobs=7)
    ext = g0.map_max - origin
    # the second box ends inside a z word (z index 0.55 * nz), the third covers the map; clusters 0 and 1 of each
    # search are reset before the next one
    boxes = [(origin + 0.2 * ext, origin + 0.7 * ext), (origin + [0.0, 0.0, 0.1] * ext, origin + [1.0, 1.0, 0.55] * ext),
             (origin, g0.map_max)]
    small_vs_large(fuel, orc, g, inflate, tri, boxes, dict(cluster_min=5, cluster_size_xy=1.0, down_sample=3, min_z=0.4),
                   reset=lambda c: [k for k in (0, 1) if k < c])


@pytest.mark.parametrize("which", ["office", "office3"])
def test_office_maps(fuel, orc, which):
    g, inflate = W.office3_map() if which == "office3" else W.office_map()
    tri = W.office_known(g, inflate)
    small_vs_large(fuel, orc, g, inflate, tri, [(g.origin, g.map_max)],
                   dict(cluster_min=100, cluster_size_xy=2.0, down_sample=3, min_z=0.4))


@pytest.mark.parametrize("n,seed,cmin,sxy", [((100, 90, 40), 5, 10, 0.6),   # 17 k kept cells: more than the first copy holds
                                             ((100, 90, 41), 6, 0, 0.6)])   # 2 010 clusters: the same for clusters
def test_results_beyond_the_first_copy(fuel, orc, n, seed, cmin, sxy):
    origin = np.zeros(3)
    g0 = W.Grid(n, origin, 0.1)
    g = W.Grid(n, origin, 0.1, box_min=origin + 0.2, box_max=g0.map_max - 0.2)
    inflate, tri = random_scene(n, seed, p_site=0.002, p_unknown=0.5, blobs=40)
    out = small_vs_large(fuel, orc, g, inflate, tri, [(origin, g0.map_max)],
                         dict(cluster_min=cmin, cluster_size_xy=sxy, down_sample=3, min_z=0.4))[0]
    assert sum(f.cells_addr_.size for f in out) > 12288 or len(out) > 256


def test_bfs_order_after_one_copy(fuel, orc):
    """FUELGPU_CELLS_BFS re-orders the fetched cells on the host: the reference's order, average_ and filtered_cells_."""
    g, inflate = W.office_map()
    tri = W.office_known(g, inflate)
    kw = dict(cluster_min=100, cluster_size_xy=2.0, down_sample=3, min_z=0.4)
    m, ff = finder(fuel, g, inflate, tri, cell_order="bfs", **kw)
    got = ff.search_box(g.origin, g.map_max)
    m.close()
    fl = np.zeros(g.n, dtype=np.int8)
    ref = orc.frontier_search(orc_grid(orc, g), tri, fl, g.origin, g.map_max, orc.frontier_params(cell_order=0, **kw))
    assert len(got) == len(ref) > 0
    for a, b in zip(got, ref):
        assert np.array_equal(a.cells_addr_, b["addr"])
        assert np.array_equal(a.average_, b["average"]) and np.array_equal(a.filtered_cells_, b["filtered"])
