"""fuel_b200/csrc/kino_math.cuh built for the host (oracle/kino_math_host.cpp, -ffp-contract=off like the device's
-fmad=false): glibc's cbrt restated equals the host libm bit for bit, and the cube, acos and cos equal the correctly
rounded values (mpmath at 200 bits, rounded to nearest)."""
import mpmath
import numpy as np

import oracle.kino as OK


def _mp_round(f, xs):
    mpmath.mp.prec = 200
    return np.array([float(f(mpmath.mpf(float(x)))) for x in xs])


def test_cbrt_equals_libm():
    rng = np.random.default_rng(1)
    n = 10 ** 7
    x = rng.uniform(-1.0, 1.0, n) * np.exp2(rng.uniform(-60.0, 60.0, n))
    special = np.array([0.0, -0.0, 27.0, -27.0, 1.0, 8.0, 5e-324, -5e-324, 2.2250738585072014e-308, 1.7976931348623157e308,
                        np.inf, -np.inf])
    for xs in (x, special):
        got, want = OK.math(OK.MATH_CBRT, xs), OK.math(OK.MATH_LIBM_CBRT, xs)
        assert np.array_equal(got.view(np.int64), want.view(np.int64))
    assert np.isnan(OK.math(OK.MATH_CBRT, np.array([np.nan])))[0]
    assert OK.math(OK.MATH_CBRT, np.array([27.0]))[0] == 3.0000000000000004  # glibc's, not the correctly rounded 3


def test_cube_correctly_rounded():
    rng = np.random.default_rng(2)
    t = np.concatenate([rng.uniform(0.0, 3.0, 10 ** 6 - 4), [0.0, 1.0, 3.0, 1e-100]])
    assert np.array_equal(OK.math(OK.MATH_CUBE, t), _mp_round(lambda v: v ** 3, t))
    assert np.array_equal(t * t, _mp_round(lambda v: v * v, t[:10 ** 5]).tolist() + (t * t)[10 ** 5:].tolist())


def test_acos_correctly_rounded():
    rng = np.random.default_rng(3)
    x = np.concatenate([rng.uniform(-1.0, 1.0, 10 ** 6 - 6), [-1.0, 1.0, 0.0, 1 - 2 ** -53, -1 + 2 ** -53, 1e-300]])
    assert np.array_equal(OK.math(OK.MATH_ACOS, x), _mp_round(mpmath.acos, x))


def test_cos_correctly_rounded():
    rng = np.random.default_rng(4)
    z = np.concatenate([rng.uniform(0.0, np.pi / 3, 10 ** 6 - 3), [0.0, 1e-300, np.pi / 3]])
    assert np.array_equal(OK.math(OK.MATH_COS, z), _mp_round(mpmath.cos, z))
