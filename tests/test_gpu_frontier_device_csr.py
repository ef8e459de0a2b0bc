"""The small frontier path orders its result on the device (cluster order, cell CSR, filtered centroids, average_ and
box in the tail of the cluster kernel).  Every case runs the same search twice, on two maps with the same flags: once
as the library runs it and once with FUELGPU_FRONTIER_HOST_CSR=1, where the host orders the kernel's raw arrays
(frontier_build_csr).  The two results must be equal bit for bit and equal to the CPU oracle.  Cases: the office maps,
scenes whose kept cells, clusters or filtered cells are exactly at the capacity of the device-ordered result and one
above it (the host then orders them), a second search after flag resets, the BFS cell order, no kept cluster, an empty
search box, and fuelgpu_frontier_fetch called after the next search_begin."""
import ctypes as C
import os

import numpy as np
import pytest

from fuel_b200 import workloads as W
from fuel_b200._lib import lib
from tests.helpers import make_sdf_map, orc_grid

pytestmark = pytest.mark.gpu

HOST_CSR = "FUELGPU_FRONTIER_HOST_CSR"
# capacities of the device-ordered result (frontier.cu: RES_K0, RES_C0, RES_F0)
CAP_K, CAP_C, CAP_F = 12288, 256, 4096


def finder(fuel, g, inflate, tri, **kw):
    m = make_sdf_map(fuel, g, inflate, tri)
    env = fuel.EDTEnvironment()
    env.setMap(m)
    return m, fuel.FrontierFinder(env, **kw)


def with_host_csr(host, fn):
    """fn() with the search ordered on the host (host=True) or on the device; the switch is read by search_begin"""
    old = os.environ.pop(HOST_CSR, None)
    if host:
        os.environ[HOST_CSR] = "1"
    try:
        return fn()
    finally:
        os.environ.pop(HOST_CSR, None)
        if old is not None:
            os.environ[HOST_CSR] = old


def assert_bitwise(got, want):
    assert len(got) == len(want)
    for i, (a, b) in enumerate(zip(got, want)):
        for name in ("cells_addr_", "filtered_cells_", "average_", "box_min_", "box_max_"):
            x, y = getattr(a, name), getattr(b, name)
            assert x.dtype == y.dtype and x.shape == y.shape, "cluster %d %s" % (i, name)
            assert x.tobytes() == y.tobytes(), "cluster %d %s differs" % (i, name)


def assert_oracle(got, ref, exact=False):
    assert len(got) == len(ref)
    for i, (a, b) in enumerate(zip(got, ref)):
        assert np.array_equal(a.cells_addr_, b["addr"]), "cluster %d cells differ" % i
        assert np.array_equal(a.filtered_cells_, b["filtered"]), "cluster %d filtered_cells_ differ" % i
        if exact:
            assert np.array_equal(a.average_, b["average"])
        else:
            assert np.allclose(a.average_, b["average"], rtol=1e-12, atol=1e-12)
        assert np.allclose(a.box_min_, b["box_min"], rtol=0, atol=1e-12)
        assert np.allclose(a.box_max_, b["box_max"], rtol=0, atol=1e-12)


def device_vs_host(fuel, orc, g, inflate, tri, boxes, kw, reset=None, cell_order="address"):
    """Each update box searched on a device-ordering map and a host-ordering map (and by the oracle) on the flags the
    previous searches left; returns the device results."""
    (m1, ff1), (m2, ff2) = (finder(fuel, g, inflate, tri, cell_order=cell_order, **kw),
                            finder(fuel, g, inflate, tri, cell_order=cell_order, **kw))
    fl = np.zeros(g.n, dtype=np.int8)
    p = orc.frontier_params(cell_order=1 if cell_order == "address" else 0, **kw)
    outs = []
    for it, (umin, umax) in enumerate(boxes):
        if it > 0 and reset is not None:  # resetFlag (:62-69) of some clusters of the previous search, on both maps
            addr = np.ascontiguousarray(np.concatenate([outs[-1][k].cells_addr_ for k in reset(len(outs[-1]))]))
            ff1._clear_flags(addr)
            ff2._clear_flags(addr)
            fl.reshape(-1)[addr] = 0
        dev = with_host_csr(False, lambda: ff1.search_box(umin, umax))
        host = with_host_csr(True, lambda: ff2.search_box(umin, umax))
        ref = orc.frontier_search(orc_grid(orc, g), tri, fl, umin, umax, p)
        assert_bitwise(dev, host)
        assert_oracle(dev, ref, exact=cell_order == "bfs")
        assert np.array_equal(ff1.download_flags(), fl) and np.array_equal(ff2.download_flags(), fl)
        outs.append(dev)
    m1.close()
    m2.close()
    return outs


def totals(out):
    return len(out), sum(f.cells_addr_.size for f in out), sum(len(f.filtered_cells_) for f in out)


OFFICE_KW = dict(cluster_min=100, cluster_size_xy=2.0, down_sample=3, min_z=0.4)


@pytest.mark.parametrize("which", ["office", "office3"])
def test_office_maps(fuel, orc, which):
    g, inflate = W.office3_map() if which == "office3" else W.office_map()
    tri = W.office_known(g, inflate)
    out = device_vs_host(fuel, orc, g, inflate, tri, [(g.origin, g.map_max)], OFFICE_KW)[0]
    nc, nk, nf = totals(out)
    assert 0 < nc <= CAP_C and 0 < nk <= CAP_K and 0 < nf <= CAP_F  # (the device orders the office maps' results)


def test_second_search_after_flag_resets(fuel, orc):
    g, inflate = W.office_map()
    tri = W.office_known(g, inflate)
    boxes = [(g.origin, g.map_max), (g.origin + 0.1 * (g.map_max - g.origin), g.map_max), (g.origin, g.map_max)]
    device_vs_host(fuel, orc, g, inflate, tri, boxes, OFFICE_KW, reset=lambda c: [k for k in range(0, c, 2)])


def test_bfs_order(fuel, orc):
    g, inflate = W.office_map()
    tri = W.office_known(g, inflate)
    device_vs_host(fuel, orc, g, inflate, tri, [(g.origin, g.map_max)], OFFICE_KW, cell_order="bfs")


# ---- scenes with exact counts: an all-UNKNOWN map with FREE columns along z (w x w cells, w <= 2, so every cell has an
# UNKNOWN x or y neighbour and is a frontier cell; one cluster each: 26-connected, too narrow to split) on a lattice of
# spacing 3, so that no two columns touch.  With cluster_min = 0 and min_z below the map every column is a kept
# cluster.  With down_sample = 1 every cell is its own VoxelGrid leaf (filtered = cells); with down_sample = 3 a
# 2 x 2 column starts on a leaf boundary in x and y, so it has about a third of its height in leaves.
def column_scene(cols, nz):
    """cols: list of (w, height) -> (Grid, inflate, tri); column j at x, y = 3 + 3 (j % 8), 3 + 3 (j // 8), z from 2"""
    n = (29, 3 * ((len(cols) + 7) // 8) + 5, nz)
    g0 = W.Grid(n, np.zeros(3), 0.1)
    g = W.Grid(n, np.zeros(3), 0.1, box_min=np.full(3, 0.1), box_max=g0.map_max - 0.1)
    tri = np.full(n, W.UNKNOWN, dtype=np.uint8)
    for j, (w, h) in enumerate(cols):
        x, y = 3 + 3 * (j % 8), 3 + 3 * (j // 8)
        tri[x:x + w, y:y + w, 2:2 + h] = W.FREE
    return g, np.zeros(n, dtype=np.int8), tri


SCENES = {
    # kept cells at the cap (12 columns of 2 x 2 x 256) and one above (one more cluster of a single cell)
    "cells_at_cap": ([(2, 256)] * 12, 260, 3, (12, CAP_K)),
    "cells_above_cap": ([(2, 256)] * 12 + [(1, 1)], 260, 3, (13, CAP_K + 1)),
    # clusters at the cap and one above (single cells)
    "clusters_at_cap": ([(1, 1)] * CAP_C, 4, 1, (CAP_C, CAP_C, CAP_C)),
    "clusters_above_cap": ([(1, 1)] * (CAP_C + 1), 4, 1, (CAP_C + 1, CAP_C + 1, CAP_C + 1)),
    # filtered cells at the cap and one above (every cell its own leaf)
    "filtered_at_cap": ([(1, 256)] * 16, 260, 1, (16, CAP_F, CAP_F)),
    "filtered_above_cap": ([(1, 256)] * 16 + [(1, 1)], 260, 1, (17, CAP_F + 1, CAP_F + 1)),
}


@pytest.mark.parametrize("name", sorted(SCENES))
def test_counts_at_and_above_the_caps(fuel, orc, name):
    cols, nz, ds, want = SCENES[name]
    g, inflate, tri = column_scene(cols, nz)
    kw = dict(cluster_min=0, cluster_size_xy=2.0, down_sample=ds, min_z=-1.0)
    out = device_vs_host(fuel, orc, g, inflate, tri, [(g.origin, g.map_max)], kw)[0]
    got = totals(out)
    assert got[:len(want)] == want, got
    assert got[2] <= CAP_F or len(want) == 3  # (the cell scenes stay inside the filtered cap)


def test_no_kept_cluster_and_empty_search_box(fuel, orc):
    g, inflate = W.office_map()
    tri = W.office_known(g, inflate)
    # every cluster at most cluster_min cells: candidates, but R = 0
    out = device_vs_host(fuel, orc, g, inflate, tri, [(g.origin, g.map_max)], dict(OFFICE_KW, cluster_min=10 ** 7))[0]
    assert out == []
    # an update box far outside the map: no seed in the search box
    far = g.map_max + 100.0
    out = device_vs_host(fuel, orc, g, inflate, tri, [(far, far + 1.0)], OFFICE_KW)[0]
    assert out == []


@pytest.mark.parametrize("host", [False, True])
def test_fetch_after_the_next_begin(fuel, orc, host):
    """search_end of A, flags reset, search_begin of B, then fuelgpu_frontier_fetch: the result of A; then B's end and
    fetch."""
    g, inflate = W.office_map()
    tri = W.office_known(g, inflate)
    box_a = (g.origin, g.map_max)
    box_b = (g.origin + 0.3 * (g.map_max - g.origin), g.map_max)
    # the expected results: A then B on a map of their own, each collected at once
    m0, ff0 = finder(fuel, g, inflate, tri, **OFFICE_KW)
    want_a = with_host_csr(True, lambda: ff0.search_box(*box_a))
    ff0.reset_flags()
    want_b = with_host_csr(True, lambda: ff0.search_box(*box_b))
    m0.close()

    m, ff = finder(fuel, g, inflate, tri, **OFFICE_KW)
    h = m.handle
    nc, ncell, nf = C.c_int32(), C.c_int32(), C.c_int32()

    def a_then_b():
        ff.search_box_begin(*box_a)
        assert lib().fuelgpu_frontier_search_end(h, C.byref(nc), C.byref(ncell), C.byref(nf)) == 0
        ff.reset_flags()
        ff.search_box_begin(*box_b)  # enqueued, not collected
        got_a = ff._fetch(nc.value, ncell.value, nf.value)
        return got_a, ff.search_box_end()

    got_a, got_b = with_host_csr(host, a_then_b)
    m.close()
    assert len(want_a) > 0 and len(want_b) > 0
    assert_bitwise(got_a, want_a)
    assert_bitwise(got_b, want_b)
