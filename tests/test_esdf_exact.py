"""The exact ESDF comparator (tests/esdf_exact.py) on oracle fields, without a GPU: it must accept what the
device's one rounding can produce and reject an error of +-1 in the squared distance where the old 1e-4 relative
bar let it through."""
import numpy as np
import pytest

from fuel_b200 import workloads as W
from tests.esdf_exact import EPS_SQRT, check_esdf, recover_k, tol_pos, ulp32
from tests.helpers import orc_grid

RES = 0.1


def device_like(k, res, rng):
    """fp32 distances as the device could produce them for squared distances k: a square root within 1 ulp of
    sqrt(k) on either side (the documented bound of sqrt.approx.f32), times float32(res), rounded to fp32."""
    s = np.sqrt(np.asarray(k, dtype=np.float64))
    s32 = s.astype(np.float32)
    lo = np.where(s32.astype(np.float64) > s, np.nextafter(s32, np.float32(0)), s32)
    hi = np.where(s32.astype(np.float64) < s, np.nextafter(s32, np.float32(np.inf)), s32)
    pick = np.where(rng.random(s.shape) < 0.5, lo, hi).astype(np.float32)
    return (np.float32(res) * pick).astype(np.float32)


def rel_1e4_accepts(got, ref):
    """The bar the ESDF tests used before: 1e-4 relative on finite distances."""
    fin = ref < 1e150
    return bool(np.all(np.abs(got[fin].astype(np.float64) - ref[fin]) <= 1e-4 * ref[fin]))


@pytest.fixture(scope="module")
def line_field(orc):
    """One site at the origin of a 1024 x 2 x 2 map: voxel (D, 0, 0) is D voxels away, k = D^2."""
    n = (1024, 2, 2)
    g = W.Grid(n, (0, 0, 0), RES)
    inflate = np.zeros(n, dtype=np.int8)
    inflate[0, 0, 0] = 1
    tri = np.full(n, W.FREE, dtype=np.uint8)
    ref = orc.update_esdf3d(orc_grid(orc, g), inflate, tri, [0, 0, 0], np.array(n) - 1, True, False)
    return ref


def test_device_like_field_passes(line_field):
    ref = line_field
    k = recover_k(ref, RES)
    rng = np.random.default_rng(1)
    for _ in range(4):
        got = device_like(k, RES, rng)
        st = check_esdf(got, ref, RES, label="device-like")
        assert st["max_ulp"] <= 3.0
    # the two extreme square roots of every voxel, not only random ones
    s = np.sqrt(k)
    for side in (0.0, np.inf):
        s32 = s.astype(np.float32)
        far = np.nextafter(s32, np.float32(side))
        far = np.where(np.abs(far.astype(np.float64) - s) <= EPS_SQRT * s, far, s32)
        check_esdf((np.float32(RES) * far).astype(np.float32), ref, RES, label="extreme sqrt")


@pytest.mark.parametrize("D", [80, 300, 700, 1000])
@pytest.mark.parametrize("dk", [1, -1])
def test_exact_bar_rejects_k_off_by_one(line_field, D, dk):
    ref = line_field
    k = recover_k(ref, RES)
    assert k[D, 0, 0] == D * D
    got = device_like(k, RES, np.random.default_rng(D))
    kk = k.copy()
    for v in [(D, 0, 0), (D, 1, 1)]:  # a voxel on the axis and one off it
        kk[v] += dk
    wrong = device_like(kk, RES, np.random.default_rng(D))
    moved = wrong != got
    assert np.count_nonzero(moved) >= 2
    with pytest.raises(AssertionError):
        check_esdf(wrong, ref, RES, verbose=False)
    # the 1e-4 relative bar cannot see it: an error of 1 in k is a relative error of about 1/(2k) < 1e-4 here
    assert rel_1e4_accepts(wrong, ref)


def test_old_bar_sees_k_off_by_one_only_below_71_voxels(line_field):
    ref = line_field
    k = recover_k(ref, RES)
    for D, seen in [(50, True), (70, True), (71, False)]:
        kk = k.copy()
        kk[D, 0, 0] += 1
        wrong = device_like(kk, RES, np.random.default_rng(0))
        assert rel_1e4_accepts(wrong, ref) != seen, D
        with pytest.raises(AssertionError):
            check_esdf(wrong, ref, RES, verbose=False)


def test_every_single_axis_distance_is_separable():
    """+-1 in k is told apart at the bar for every squared distance of a single-axis line (D <= 1023) and every
    resolution the tests use."""
    D = np.arange(1, 1024, dtype=np.float64)
    for res in (0.1, 0.05, 0.15, 0.2):
        fr = float(np.float32(res))
        for k in (D * D, D * D + 1, D * D + 2):
            m = fr * np.sqrt(k)
            for kk in (k + 1, k - 1):
                mm = fr * np.sqrt(kk)
                assert np.all(np.abs(mm - m) > tol_pos(m) + tol_pos(mm))


def test_sentinels_and_zero(line_field):
    ref = line_field.copy()
    got = device_like(recover_k(ref, RES), RES, np.random.default_rng(2))
    ref[5, 1, 1] = RES * np.sqrt(np.finfo(np.float64).max)
    got_inf = got.copy()
    got_inf[5, 1, 1] = np.inf
    check_esdf(got_inf, ref, RES, verbose=False)
    with pytest.raises(AssertionError):  # a finite value where the reference has no site
        check_esdf(got, ref, RES, verbose=False)
    bad = got.copy()
    bad[0, 0, 0] = np.float32(1e-30)  # k = 0 must be exactly 0
    with pytest.raises(AssertionError):
        check_esdf(bad, line_field, RES, verbose=False)
    with pytest.raises(AssertionError):  # the premise: the reference value must be res*sqrt(integer)
        check_esdf(got, line_field + 1e-9, RES, verbose=False)


def test_signed_branch(orc):
    """Signed mode: obstacle voxels hold float32(res - ng); the bar there adds the one rounding of that difference."""
    n = (40, 36, 28)
    g = W.Grid(n, (0, 0, 0), RES)
    rng = np.random.default_rng(9)
    inflate = np.zeros(n, dtype=np.int8)
    for _ in range(5):
        c = rng.integers(4, 24, 3)
        inflate[c[0]:c[0] + 9, c[1]:c[1] + 7, c[2]:c[2] + 6] = 1
    tri = np.full(n, W.FREE, dtype=np.uint8)
    og = orc_grid(orc, g)
    ref = orc.update_esdf3d(og, inflate, tri, [0, 0, 0], np.array(n) - 1, True, True)
    pos = orc.update_esdf3d(og, inflate, tri, [0, 0, 0], np.array(n) - 1, True, False)
    negf = orc.update_esdf3d(og, (1 - inflate).astype(np.int8), tri, [0, 0, 0], np.array(n) - 1, True, False)
    assert np.any(ref < -RES)
    dpos = device_like(recover_k(pos, RES), RES, rng)
    dneg = device_like(recover_k(negf, RES), RES, rng)
    got = dpos.copy()
    m = dneg > 0
    got[m] += (-dneg[m] + np.float32(RES)).astype(np.float32)  # signed_merge_kernel, in fp32
    st = check_esdf(got.astype(np.float32), ref, RES, signed=True, label="signed device-like")
    assert st["max_ulp_neg"] > 0
    bad = got.copy()
    v = np.argwhere(ref < -2 * RES)[0]
    kn = np.rint(((RES - ref[tuple(v)]) / RES) ** 2)
    bad[tuple(v)] = np.float32(RES) - np.float32(RES) * np.float32(np.sqrt(kn + 1))
    with pytest.raises(AssertionError):
        check_esdf(bad.astype(np.float32), ref, RES, signed=True, verbose=False)


def test_ulp32():
    assert ulp32(1.0) == 2.0 ** -23 and ulp32(1.5) == 2.0 ** -23 and ulp32(0.99) == 2.0 ** -24
    assert ulp32(102.3) == 2.0 ** -17
