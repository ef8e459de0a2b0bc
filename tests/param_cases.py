"""Inputs and an exact ground truth for parameterizeToBspline (bspline/src/non_uniform_bspline.cpp:178-265), shared by
tests/test_oracle_traj_param.py (CPU) and tests/test_gpu_traj_param.py (H100)."""
from fractions import Fraction

import numpy as np

from fuel_b200 import workloads as W

# the (K, dt) grid of the exact-solve checks: K = n_pts - 2 for 4, 5, 20, 32, 33 and 64 control points
GRID_K = (2, 3, 18, 30, 31, 62)
GRID_DT = (0.02, 0.05, 0.175, 1.0, 5.0)


def noisy_samples(rng, K, dt, noise=0.05):
    """a sampled path of K points about 0.35 m apart with noise on every sample, and start / end derivatives that no
    spline through those samples has (so the least-squares residual is not zero): points [K, 3], derivs [4, 3]"""
    d = rng.normal(size=3)
    d /= np.linalg.norm(d)
    s = np.arange(K)[:, None] * 0.35
    points = rng.uniform(-2.0, 2.0, 3) + s * d + rng.normal(scale=noise, size=(K, 3))
    v = 0.35 / dt
    derivs = np.stack([d * v, d * v * 0.5, np.zeros(3), np.zeros(3)]) + rng.normal(scale=0.3, size=(4, 3)) * (1 + v)
    return points, derivs


def spline_samples(ctrl, dt):
    """a uniform cubic spline sampled at its knots, with its exact end derivatives: what parameterizeToBspline inverts
    (positions (P[i] + 4 P[i+1] + P[i+2]) / 6, vel (P[2] - P[0]) / (2 dt), acc (P[0] - 2 P[1] + P[2]) / dt^2)"""
    P = np.asarray(ctrl, dtype=np.float64)
    points = (P[:-2] + 4 * P[1:-1] + P[2:]) / 6.0
    derivs = np.stack([(P[2] - P[0]) / (2 * dt), (P[-1] - P[-3]) / (2 * dt),
                       (P[0] - 2 * P[1] + P[2]) / (dt * dt), (P[-3] - 2 * P[-2] + P[-1]) / (dt * dt)])
    return points, derivs


def workload_samples(g, inflate, B, n_pts):
    """the benchmark's trajectories (workloads.make_trajectories: its dt draw, its start states) as sampled paths:
    each spline at its knots, with its start velocity / acceleration, end at rest, plus noise on the samples.
    Returns points [B, n_pts - 2, 3], derivs [B, 4, 3], dt [B]."""
    tr = W.make_trajectories(g, inflate, B=B, n_pts=n_pts)
    rng = np.random.default_rng(n_pts)
    points = np.stack([spline_samples(c, d)[0] for c, d in zip(tr["ctrl"], tr["dt"])])
    points += rng.normal(scale=0.02, size=points.shape)
    derivs = np.zeros((B, 4, 3))
    derivs[:, 0] = tr["start"][:, 1]
    derivs[:, 2] = tr["start"][:, 2]
    return points, derivs, tr["dt"].copy()


def exact_lstsq(A, b):
    """the least-squares solution of the fp64 system A [m, n], b [r, m] in exact rational arithmetic: the normal
    equations A^T A x = A^T b, which are exact here, eliminated on their band (A has three adjacent nonzeros per row, so
    A^T A has half-bandwidth 2 and is positive definite: no pivoting).  Returns x [r, n] rounded to fp64."""
    m, n = A.shape
    rows = []
    for i in range(m):
        nz = np.flatnonzero(A[i])
        rows.append([(int(j), Fraction(float(A[i, j]))) for j in nz])
    rhs = [[Fraction(float(v)) for v in br] for br in b]
    hb = 2
    M = [dict() for _ in range(n)]
    R = [[Fraction(0)] * n for _ in rhs]
    for i, row in enumerate(rows):
        for j, a in row:
            for k, c in row:
                M[j][k] = M[j].get(k, Fraction(0)) + a * c
            for r, br in enumerate(rhs):
                R[r][j] += a * br[i]
    for k in range(n):
        piv = M[k][k]
        for i in range(k + 1, min(n, k + hb + 1)):
            f = M[i].get(k, Fraction(0)) / piv
            if f == 0:
                continue
            for j in range(k, min(n, k + hb + 1)):
                M[i][j] = M[i].get(j, Fraction(0)) - f * M[k].get(j, Fraction(0))
            for r in range(len(R)):
                R[r][i] -= f * R[r][k]
    x = np.zeros((len(R), n))
    for r in range(len(R)):
        xs = [Fraction(0)] * n
        for k in range(n - 1, -1, -1):
            s = R[r][k]
            for j in range(k + 1, min(n, k + hb + 1)):
                s -= M[k].get(j, Fraction(0)) * xs[j]
            xs[k] = s / M[k][k]
        x[r] = [float(v) for v in xs]
    return x
