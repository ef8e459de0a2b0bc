"""Obstacle inflation (SDFMap::clearAndInflateLocalMap, plan_env/src/sdf_map.cpp:364-472): the oracle is
pinned on scipy's binary dilation away from the map faces, the linear-address wrap quirk of :452-458 is
demonstrated, and the device path must equal the oracle bit for bit (including the quirk and the ceiling)."""
import numpy as np
import pytest
from scipy import ndimage

from fuel_b200 import workloads as W
from tests.esdf_exact import check_esdf
from tests.helpers import make_sdf_map, orc_grid


def scene(n, seed, p=0.004):
    rng = np.random.default_rng(seed)
    tri = np.full(n, W.FREE, dtype=np.uint8)
    tri[rng.random(n) < p] = W.OCCUPIED
    tri[rng.random(n) < 0.2] = W.UNKNOWN
    return tri


def test_oracle_matches_box_dilation_in_the_interior(orc):
    n = (30, 26, 22)
    g = W.Grid(n, (0, 0, 0), 0.1)
    tri = scene(n, 1)
    tri[:3], tri[-3:], tri[:, :3], tri[:, -3:], tri[:, :, :3], tri[:, :, -3:] = 1, 1, 1, 1, 1, 1  # keep stamps off the faces
    inflate = np.ones(n, dtype=np.int8)
    t2 = tri.copy()
    orc.clear_and_inflate(orc_grid(orc, g), t2, inflate, [0, 0, 0], np.array(n) - 1, 2)
    ref = ndimage.binary_dilation(tri == W.OCCUPIED, structure=np.ones((5, 5, 5)))
    assert np.array_equal(inflate == 1, ref) and np.array_equal(t2, tri)


def test_oracle_local_box_wrap_and_ceiling(orc):
    n = (12, 10, 8)
    g = W.Grid(n, (0, 0, -1.0), 0.1)
    tri = np.full(n, W.FREE, dtype=np.uint8)
    tri[5, 0, 4] = W.OCCUPIED      # on the y = 0 face: the stamp wraps to y = ny-1 of x-1 (SURVEY H9)
    tri[11, 9, 7] = W.OCCUPIED     # outside the local box: ignored
    inflate = np.zeros(n, dtype=np.int8)
    inflate[0, 0, 0] = 1           # outside the box: kept
    orc.clear_and_inflate(orc_grid(orc, g), tri, inflate, [2, 0, 1], [9, 8, 6], 1, ceil_id=6)
    assert inflate[0, 0, 0] == 1 and inflate[11, 9, 7] == 0
    assert inflate[5, 0, 4] == 1 and inflate[6, 1, 5] == 1
    assert inflate[4, 9, 4] == 1   # (5, -1, 4) wrapped: address (5*10 - 1)*8 + 4 = (4, 9, 4)
    assert np.all(tri[2:10, 0:9, 6] == W.OCCUPIED) and tri[1, 0, 6] == W.FREE


@pytest.mark.gpu
@pytest.mark.parametrize("n,box,step,ceil", [((30, 26, 22), None, 2, -1), ((24, 20, 16), ([2, 0, 1], [20, 19, 14]), 2, 12),
                                             ((16, 16, 16), ([0, 0, 0], [15, 15, 15]), 1, -1)])
def test_gpu_matches_oracle(fuel, orc, n, box, step, ceil):
    g = W.Grid(n, (0, 0, -1.0), 0.1)
    tri = scene(n, 7, p=0.01)
    inflate0 = (np.random.default_rng(3).random(n) < 0.05).astype(np.int8)  # stale bits to be cleared
    bmin, bmax = ([0, 0, 0], list(np.array(n) - 1)) if box is None else box
    t_ref, i_ref = tri.copy(), inflate0.copy()
    orc.clear_and_inflate(orc_grid(orc, g), t_ref, i_ref, bmin, bmax, step, ceil)
    m = make_sdf_map(fuel, g, inflate0, tri)
    m.local_bound_min_, m.local_bound_max_ = np.array(bmin), np.array(bmax)
    ceil_h = -10.0 if ceil < 0 else (ceil + 0.5) * g.res + g.origin[2]
    m.clearAndInflateLocalMap(obstacles_inflation=step * g.res - 1e-3, virtual_ceil_height=ceil_h)
    assert np.array_equal(m.occupancy_buffer_inflate_, i_ref)
    assert np.array_equal(m.occupancy_tri_, t_ref)
    # the chain the reference runs: inflate -> updateESDF3d on the same box
    m.optimistic_ = True
    m.updateESDF3d()
    d = m.download()
    ref = orc.update_esdf3d(orc_grid(orc, g), i_ref, t_ref, bmin, bmax, True, False)
    check_esdf(d, ref, g.res, box=(bmin, bmax))
    m.close()
