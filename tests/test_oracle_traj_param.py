"""Pins the oracle's parameterizeToBspline (oracle/fuel_oracle_param.c: orc_bspline_param_system, orc_lstsq_colpiv_qr,
orc_bspline_parameterize, orc_bspline_boundary_states) against the REFERENCE's own NonUniformBspline
(bspline/src/non_uniform_bspline.cpp, compiled unmodified into oracle/_ref/libfuel_ref_param.so by oracle/param.mk), bit
for bit: the system A, b it builds, and
getBoundaryStates(2, 0).  Its solve, colPivHouseholderQr().solve(), is a third-party algorithm: the reference is
compiled against a stand-in that returns the oracle's restatement, so that solve is checked against exact rational
least squares instead.  Where the reference library is not built, the digests in tests/golden/refpin_param.json stand
in for it (tests/refgold.py's scheme).

  FUEL_REFPIN_RECORD=1 python -m pytest tests/test_oracle_traj_param.py

rewrites the digests from a run against the built reference."""
import numpy as np
import pytest

import oracle as OR
import oracle.param as O
from tests.param_cases import GRID_DT, GRID_K, exact_lstsq, noisy_samples, spline_samples
from tests.refgold import refgold_fixture

O.build()

# the (K, dt) grid of the rank and reference checks
RANK_K = (2, 3, 4, 8, 18, 30, 31, 62)
RANK_DT = (0.02, 0.05, 0.1, 0.175, 0.35, 1.0, 5.0)


G = refgold_fixture("refpin_param.json", O.ref_param)


# ---- against the reference's own code ------------------------------------------------------------------------------
@pytest.mark.parametrize("K", RANK_K)
def test_system_matches_reference(G, K):
    """A and the three b, entry for entry, as the reference's parameterizeToBspline builds them"""
    rng = np.random.default_rng(1000 + K)
    got, cases = [], []
    for dt in RANK_DT:
        pts, der = noisy_samples(rng, K, dt)
        cases.append((pts, der, dt))
        A, b = O.param_system(pts, der, dt)
        got.append([A, b])
    G.eq(got, lambda: [list(O.ref_parameterize(p, d, t)[1:]) for p, d, t in cases])


@pytest.mark.parametrize("K", RANK_K)
def test_control_points_and_boundary_states_match_reference(G, K):
    """orc_bspline_parameterize's control points are the reference's parameterizeToBspline run on the oracle's solve;
    its start / end are the reference's getBoundaryStates(2, 0) of them"""
    rng = np.random.default_rng(2000 + K)
    B = len(RANK_DT)
    pts, der = zip(*[noisy_samples(rng, K, dt) for dt in RANK_DT])
    x, tc = O.bspline_parameterize(np.array(pts), np.array(der), np.array(RANK_DT))
    n = K + 2
    ctrl = x[:, :3 * n].reshape(B, n, 3)
    G.eq([c for c in ctrl], lambda: [O.ref_parameterize(pts[b], der[b], RANK_DT[b])[0] for b in range(B)])
    got = [[np.array(tc[b].start), np.array(tc[b].end)[0]] for b in range(B)]
    G.eq(got, lambda: [list(O.ref_boundary_states(ctrl[b], RANK_DT[b])) for b in range(B)])


@pytest.mark.parametrize("n", [4, 5, 20, 33, 64])
def test_boundary_states_match_reference(G, n):
    """getBoundaryStates(2, 0) of arbitrary splines, both dt layouts"""
    rng = np.random.default_rng(3000 + n)
    B = 12
    ctrl = np.cumsum(rng.normal(scale=0.3, size=(B, n, 3)), axis=1)
    dt = rng.uniform(0.02, 1.0, B)
    dt[:2] = (5.0, 0.02)
    x = np.concatenate([ctrl.reshape(B, -1), dt[:, None]], axis=1)
    start, end = O.bspline_boundary_states(x, n)
    s2, e2 = O.bspline_boundary_states(ctrl.reshape(B, -1), n, dt=dt)
    assert start.tobytes() == s2.tobytes() and end.tobytes() == e2.tobytes()
    G.eq([[start[b], end[b]] for b in range(B)], lambda: [list(O.ref_boundary_states(ctrl[b], dt[b])) for b in range(B)])


# ---- independent ground truths -------------------------------------------------------------------------------------
@pytest.mark.parametrize("K", GRID_K)
def test_solve_matches_exact_least_squares(K):
    """noisy samples and derivative rows no spline meets: the oracle's solve within 1e-11 * max(1, max|x|) of the exact
    rational least-squares solution of the same fp64 system"""
    rng = np.random.default_rng(4000 + K)
    for dt in GRID_DT:
        pts, der = noisy_samples(rng, K, dt)
        A, b = O.param_system(pts, der, dt)
        exact = exact_lstsq(A, b)
        x, tc = O.bspline_parameterize(pts[None], der[None], [dt])
        got = x[0, :-1].reshape(K + 2, 3).T
        tol = 1e-11 * max(1.0, np.abs(exact).max())
        assert np.abs(got - exact).max() <= tol, "K=%d dt=%g: %.3g" % (K, dt, np.abs(got - exact).max())
        assert np.abs(A @ exact.T - b.T).max() > 1e-3  # the system is inconsistent: a least-squares case


@pytest.mark.parametrize("K", GRID_K)
def test_consistent_system_returns_the_spline(K):
    """samples of a known uniform cubic spline at its knots with its exact end derivatives: its control points come
    back to 1e-11 relative (cond(A) * eps alone is about 2e-12 at dt = 0.02)"""
    rng = np.random.default_rng(5000 + K)
    for dt in GRID_DT:
        ctrl = rng.uniform(-3.0, 3.0, 3) + np.cumsum(rng.normal(scale=0.3, size=(K + 2, 3)), axis=0)
        pts, der = spline_samples(ctrl, dt)
        x, _ = O.bspline_parameterize(pts[None], der[None], [dt])
        got = x[0, :-1].reshape(K + 2, 3)
        assert np.abs(got - ctrl).max() <= 1e-11 * max(1.0, np.abs(ctrl).max()), "K=%d dt=%g" % (K, dt)


def test_system_has_full_column_rank():
    rng = np.random.default_rng(6)
    for K in RANK_K:
        for dt in RANK_DT:
            A, _ = O.param_system(*noisy_samples(rng, K, dt), dt)
            assert A.shape == (K + 4, K + 2) and np.linalg.matrix_rank(A) == K + 2, (K, dt)
            x, rank = O.lstsq_colpiv_qr(A, np.ones((1, K + 4)))
            assert rank == K + 2


def test_outputs_layouts_and_constants():
    """both nvar layouts give the same control points; the constants are what optimize() freezes"""
    rng = np.random.default_rng(7)
    K, B = 18, 6
    pts, der = zip(*[noisy_samples(rng, K, 0.175) for _ in range(B)])
    pts, der = np.array(pts), np.array(der)
    dt = rng.uniform(0.1, 0.3, B)
    n = K + 2
    xa, ta = O.bspline_parameterize(pts, der, dt)
    xb, tb = O.bspline_parameterize(pts, der, dt, time_lb=np.arange(B) + 0.5, mintime=False)
    assert xa[:, :3 * n].tobytes() == xb.tobytes() and np.array_equal(xa[:, 3 * n], dt)
    for b in range(B):
        assert ta[b].time_lb == -1.0 and tb[b].time_lb == b + 0.5
        for t in (ta[b], tb[b]):
            assert t.pt_dist == OR.pt_dist(xb[b].reshape(n, 3)) and t.knot_span == dt[b]
            assert t.n_end == 1 and t.n_guide == 0 and t.n_waypt == 0 and t.view_idx == -1
            assert np.array_equal(np.array(t.end)[1:], np.zeros((2, 3)))
    assert bytes(ta[0])[:64] != bytes(64)
