"""Pins the oracle's waypoint polynomial (oracle/fuel_oracle_poly.c: orc_poly_waypoints, orc_poly_evaluate,
orc_poly_total_time, orc_poly_length, orc_explore_samples) against the REFERENCE's own PolynomialTraj
(poly_traj/src/polynomial_traj.cpp, compiled unmodified into oracle/_ref/libfuel_ref_poly.so by oracle/poly.mk), bit for
bit: A, Q, Ct and D as it built them, the coefficients, getTotalTime, getLength, and the samples, seg_num, dt and K of
planExploreTraj's lines 270-297.  The three inverses are a third-party algorithm (Eigen's LU): the reference is compiled
against a stand-in that returns the oracle's restatement, so the coefficients are checked against an exact rational
minimizer instead (tests/poly_cases.py).  Where the reference library is not built, the digests in
tests/golden/refpin_poly.json stand in for it.

  FUEL_REFPIN_RECORD=1 python -m pytest tests/test_oracle_poly.py

rewrites the digests from a run against the built reference."""
import numpy as np
import pytest

import oracle.poly as O
from fuel_b200 import workloads as W
from tests.poly_cases import GRID_S, exact_minjerk, grid_cases, poly_eval, random_tour
from tests.refgold import refgold_fixture

O.build()

G = refgold_fixture("refpin_poly.json", O.ref_poly)


def _tour(S, seed):
    rng = np.random.default_rng(seed)
    w, v, a, t = random_tour(rng, S, 0.3, 3.0)
    return w, v, a, t, rng.uniform(-1, 1, 3), rng.uniform(-1, 1, 3)


# ---- against the reference's own code ------------------------------------------------------------------------------
@pytest.mark.parametrize("S", (2, 3, 5, 12, 31))
def test_waypoints_matches_reference(G, S):
    """A, Q, Ct, D and the coefficients, entry for entry, as the reference's waypointsTraj builds them, with zero and
    non-zero end states"""
    w, v, a, t, ve, ae = _tour(S, 100 + S)
    for end in ((None, None), (ve, ae)):
        got = O.waypoints(w, v, a, t, end[0], end[1], matrices=True)
        G.eq(list(got), lambda: list(O.ref_waypoints(w, v, a, t, end[0], end[1])))


@pytest.mark.parametrize("S", (2, 7, 20))
def test_evaluate_total_time_length_match_reference(G, S):
    """getTotalTime, getLength and evaluate(t, k) for k = 0..3 at times on, between and past the segment ends"""
    w, v, a, t, _, _ = _tour(S, 200 + S)
    c = O.waypoints(w, v, a, t)
    total = O.total_time(t)
    ts = np.concatenate([[0.0], np.cumsum(t), np.cumsum(t) + 0.5e-4, np.linspace(0, total, 37)])
    for k in range(4):
        got = [O.total_time(t), O.length(c, t), np.array([O.evaluate(c, t, x, k) for x in ts])]
        G.eq(got, lambda: list(O.ref_query(w, v, a, t, ts, k)))


@pytest.mark.parametrize("seed", (1, 2))
def test_explore_samples_match_reference(G, seed):
    """planExploreTraj's lines 270-297 over make_tours: times, duration, length, seg_num, dt, K, samples, boundary
    derivatives"""
    g, inflate = W.office_map()
    tr = W.make_tours(g, inflate, B=24, seed=seed)
    for tour, v, a in zip(tr["tours"], tr["start_vel"], tr["start_acc"]):
        got = O.explore_samples(tour, v, a)
        G.eq([got[k] for k in sorted(got)], lambda: [(lambda r: r[k])(O.explore_samples(tour, v, a, ref=True))
                                                    for k in sorted(got)])


# ---- the solve against exact rational arithmetic -------------------------------------------------------------------
@pytest.mark.parametrize("case", range(len(grid_cases())))
def test_coefficients_match_exact_minimizer(case):
    """within 1e-11 * max(1, max|c|) of the exact minimizer of the same fp64 problem, S in {2, 3, 8, 20, 31} and
    segment times from 0.05 to 5 s.  The reference's dense formulation (6S x 6S inverses of A, whose entries run from 1
    to T^5) loses accuracy on long tours that mix times across that whole range: on this grid it measures up to 1.5e-9
    relative (S = 8 and 20), so from S = 8 on it is held to 1e-8.  The device's block-tridiagonal
    solve meets 1e-11 on every case (tests/test_gpu_poly_traj.py)."""
    w, v, a, t = grid_cases()[case]
    ex = exact_minjerk(w, v, a, t)
    c = O.waypoints(w, v, a, t)
    err = np.abs(c - ex).max()
    bar = 1e-11 if len(t) <= 3 else 1e-8
    assert err <= bar * max(1.0, np.abs(ex).max()), (len(t), err, np.abs(ex).max())


@pytest.mark.parametrize("S", GRID_S)
def test_polynomial_properties(S):
    """through every waypoint, position / velocity / acceleration continuous at the inner waypoints, the boundary
    conditions met"""
    rng = np.random.default_rng(300 + S)
    w, v, a, t = random_tour(rng, S, 0.3, 3.0)
    ve, ae = rng.uniform(-1, 1, 3), rng.uniform(-1, 1, 3)
    c = O.waypoints(w, v, a, t, ve, ae)
    scale = max(1.0, np.abs(c).max())
    tol = 1e-10 * scale
    for k in range(S):
        np.testing.assert_allclose(poly_eval(c[k], 0.0, 0), w[k], atol=tol)
        np.testing.assert_allclose(poly_eval(c[k], t[k], 0), w[k + 1], atol=tol)
        if k + 1 < S:
            for d in (1, 2):
                np.testing.assert_allclose(poly_eval(c[k], t[k], d), poly_eval(c[k + 1], 0.0, d), atol=tol)
    np.testing.assert_allclose(poly_eval(c[0], 0.0, 1), v, atol=tol)
    np.testing.assert_allclose(poly_eval(c[0], 0.0, 2), a, atol=tol)
    np.testing.assert_allclose(poly_eval(c[-1], t[-1], 1), ve, atol=tol)
    np.testing.assert_allclose(poly_eval(c[-1], t[-1], 2), ae, atol=tol)


def test_exact_solver_is_the_dense_minimizer():
    """tests/poly_cases.exact_minjerk, which never forms the reference's dense system, solves the same problem as the
    reference's dense formulation (the oracle's restatement of it) on a small, well-conditioned tour"""
    rng = np.random.default_rng(5)
    w, v, a, t = random_tour(rng, 4, 0.5, 2.0)
    ex = exact_minjerk(w, v, a, t)
    c = O.waypoints(w, v, a, t)
    np.testing.assert_allclose(c, ex, rtol=0, atol=1e-12 * max(1.0, np.abs(ex).max()))


def test_two_waypoints_are_refused():
    """S = 1: the reference's waypointsTraj writes Ct(3, 2S + 4) and Ct(5, 2S + 5), columns 6 and 7 of a 6-column
    matrix, which is undefined behaviour; shortenPath always hands it three points or more.  The oracle refuses such a
    tour instead of copying the undefined behaviour (and so does fuelgpu_poly_waypoints_batch)."""
    w = np.array([[0.0, 0, 0], [1.0, 0, 0]])
    with pytest.raises(ValueError):
        O.waypoints(w, np.zeros(3), np.zeros(3), np.array([1.0]))


def test_lu_inverse():
    rng = np.random.default_rng(9)
    M = rng.normal(size=(12, 12))
    np.testing.assert_allclose(O.lu_inverse(M) @ M, np.eye(12), atol=1e-12)


def test_make_tours_shape():
    """3 to 12 waypoints, in the box, the last tour long enough to exceed 64 points"""
    g, inflate = W.office_map()
    tr = W.make_tours(g, inflate, B=64, seed=4)
    assert len(tr["tours"]) == 64
    for t in tr["tours"]:
        assert 3 <= len(t) <= 12
        assert np.all(t >= g.box_min) and np.all(t <= g.box_max)
    assert np.all(np.linalg.norm(tr["start_vel"], axis=1) <= 2.0)
    last = O.explore_samples(tr["tours"][-1], tr["start_vel"][-1], tr["start_acc"][-1])
    assert last["K"] + 2 > 64
