"""The exact comparator for ESDF fields: device fp32 distances against the oracle's fp64 ones.

Every finite intermediate of the distance transform is an integer: the squared voxel distance k to the nearest
site.  The reference ends with `dist = res * sqrt(k)` in fp64; the device runs the transform in exact int32 and
converts once, `dist = float32(res) * sqrt.approx.ftz.f32(k)` in fp32 (esdf_tile.cu, `evaluate_band`).  So the
comparison recovers k from the reference and holds the device to the rounding of that one conversion:

  m = float32(res) * sqrt(k)           (fp64: the exact value the device approximates)
  |d - m| <= 2^-23 * m + 0.5 * ulp_f32(m * (1 + 2^-23))

The CUDA documentation bounds the fp32 square root without -prec-sqrt (sqrt.approx.f32) at 1 ulp, i.e. a
relative error <= 2^-23 for any input; k < 2^22 converts to fp32 exactly, and the multiply by float32(res) adds
half an ulp of its result.  In ulps of m the bar is U = 2.5 (the 2^-23 relative term is < 2 ulp(m)); only just
below a power of two, where the rounded product can land in the next binade, it reaches 3 ulp(m).

Signed mode: inside obstacles the device adds float32(res - ng) to a positive distance of exactly 0, ng being
the negative field's value (itself `float32(res) * sqrt.approx(kn)`), so that branch has one more rounding:
  m = float32(res) - float32(res) * sqrt(kn),   |d - m| <= tol(mn) + 0.5 * ulp_f32(|m| + tol(mn)).

"No site in the box" is +inf on the device and res*sqrt(DBL_MAX) in the reference (-inf and its negation when
an obstacle has no free voxel in the box).
"""
import numpy as np

EPS_SQRT = 2.0 ** -23  # relative error of sqrt.approx.f32: 1 ulp
U_BAR = 2.5            # the bar in ulps of m away from the top of a binade
SENTINEL = 1e150       # the reference's res*sqrt(DBL_MAX) ~ 1.34e153 for res = 0.1
PREMISE_RTOL = 1e-12


def ulp32(x):
    """ulp of an fp32 number of magnitude |x| (normal range), as fp64."""
    _, e = np.frexp(np.abs(np.asarray(x, dtype=np.float64)))
    return np.ldexp(1.0, e - 24)


def tol_pos(m):
    """The bar on |d - m| for d = float32(res) * sqrt.approx(k) rounded to fp32, m its exact value."""
    m = np.asarray(m, dtype=np.float64)
    return EPS_SQRT * m + 0.5 * ulp32(m * (1 + EPS_SQRT))


def model_pos(k, fr):
    m = fr * np.sqrt(np.asarray(k, dtype=np.float64))
    return m, tol_pos(m)


def model_neg(kn, fr):
    """Inside an obstacle in signed mode: float32(res - ng), ng the device's value for kn."""
    mn, tn = model_pos(kn, fr)
    m = fr - mn
    return m, tn + 0.5 * ulp32(np.abs(m) + tn)


def _inseparable(k, fr, model):
    """Voxels where a device value for k+1 or k-1 could still lie inside the bar around k's model."""
    k = np.asarray(k, dtype=np.float64)
    m, t = model(k, fr)
    mp, tp = model(k + 1, fr)
    mm, tm = model(np.maximum(k - 1, 0), fr)
    up = np.abs(mp - m) <= t + tp
    # k - 1 = 0 is exact zero on the device: always told apart
    dn = (k >= 2) & (np.abs(m - mm) <= t + tm)
    return int(np.count_nonzero(up | dn))


def recover_k(dist, res, ref_f32=False):
    """k = rint((dist/res)^2) from the reference's value, after asserting that the value is res*sqrt(k)."""
    dist = np.asarray(dist, dtype=np.float64)
    k = np.rint((dist / res) ** 2)
    back = res * np.sqrt(k)
    if ref_f32:  # a stored fp32 copy of the reference's fp64 value: rounding it again must give it back
        ok = back.astype(np.float32) == dist.astype(np.float32)
    else:
        ok = np.abs(back - dist) <= PREMISE_RTOL * dist
    assert np.all(ok), "reference value is not res*sqrt(integer): %r" % (dist[~ok][:4],)
    return k


def recover_kn(dist, res, ref_f32=False):
    """kn of the negative field from the reference's signed value 0 + (-(res*sqrt(kn)) + res) <= 0."""
    dist = np.asarray(dist, dtype=np.float64)
    kn = np.rint(((res - dist) / res) ** 2)
    back = 0.0 + (-(res * np.sqrt(kn)) + res)
    if ref_f32:
        ok = back.astype(np.float32) == dist.astype(np.float32)
    else:
        ok = np.abs(back - dist) <= PREMISE_RTOL * res * np.sqrt(kn)
    assert np.all(ok & (kn >= 1)), "signed reference value is not res*(1-sqrt(integer)): %r" % (dist[~ok][:4],)
    return kn


def check_esdf(got, ref, res, box=None, signed=False, ref_f32=False, label="", verbose=True):
    """Assert that the device field `got` (fp32) is the reference field `ref` (fp64, or its fp32 copy with
    ref_f32) at the exact bar; `box` = (lo, hi) inclusive restricts the comparison.  Returns the statistics:
    voxel count, largest error in ulps of m (positive branch, and negative branch of signed mode), and the
    number of voxels where an error of +-1 in k would not be told apart from rounding."""
    got = np.asarray(got)
    assert got.dtype == np.float32, got.dtype
    if box is not None:
        sl = tuple(slice(int(box[0][i]), int(box[1][i]) + 1) for i in range(3))
        got, ref = got[sl], ref[sl]
    got = got.ravel()
    ref = np.asarray(ref, dtype=np.float64).ravel()
    stats = dict(label=label, n=int(got.size), max_ulp=0.0, max_ulp_neg=0.0, inseparable=0)
    step = 1 << 22  # bounded host memory on 512^3 fields
    for a in range(0, got.size, step):
        st = _check_flat(got[a:a + step], ref[a:a + step], res, signed, ref_f32, label)
        stats["max_ulp"] = max(stats["max_ulp"], st[0])
        stats["max_ulp_neg"] = max(stats["max_ulp_neg"], st[1])
        stats["inseparable"] += st[2]
    if verbose:
        print("esdf exact %s: %d voxels, max %.3f ulp (bar %.1f), signed branch %.3f ulp, %d voxels beyond the "
              "separability limit of +-1 in k" % (label, stats["n"], stats["max_ulp"], U_BAR, stats["max_ulp_neg"],
                                                   stats["inseparable"]))
    return stats


def _check_flat(got, ref, res, signed, ref_f32, label):
    fr = float(np.float32(res))
    pinf, ninf = ref > SENTINEL, ref < -SENTINEL
    assert np.array_equal(got == np.inf, pinf), "+inf <-> no-site sentinel mismatch in %d voxels" % int(
        np.count_nonzero((got == np.inf) != pinf))
    assert np.array_equal(got == -np.inf, ninf), "-inf <-> negative sentinel mismatch"
    neg = ~(pinf | ninf) & ((ref < 0) | (ref == 0) & signed)
    pos = ~(pinf | ninf | neg)
    d = got.astype(np.float64)
    max_ulp = max_ulp_neg = 0.0
    insep = 0

    k = recover_k(ref[pos], res, ref_f32)
    dp = d[pos]
    zero = k == 0
    assert np.all(dp[zero] == 0.0), "k = 0 must give exactly 0"
    m, t = model_pos(k, fr)
    err = np.abs(dp - m)
    bad = err > t
    if np.any(bad):
        i = np.flatnonzero(bad)[:5]
        raise AssertionError("%s: %d voxels off the exact bar; k=%s got=%s model=%s err/ulp=%s" % (
            label, int(bad.sum()), k[i], dp[i], m[i], err[i] / ulp32(m[i])))
    if np.any(~zero):
        max_ulp = float(np.max(err[~zero] / ulp32(m[~zero])))
    insep += _inseparable(k[~zero], fr, model_pos)

    if np.any(neg):
        kn = recover_kn(ref[neg], res, ref_f32)
        dn = d[neg]
        m, t = model_neg(kn, fr)
        err = np.abs(dn - m)
        bad = err > t
        if np.any(bad):
            i = np.flatnonzero(bad)[:5]
            raise AssertionError("%s: %d obstacle voxels off the signed bar; kn=%s got=%s model=%s" % (
                label, int(bad.sum()), kn[i], dn[i], m[i]))
        max_ulp_neg = float(np.max(err / ulp32(fr * np.sqrt(kn))))
        insep += _inseparable(kn, fr, model_neg)
    return max_ulp, max_ulp_neg, insep
