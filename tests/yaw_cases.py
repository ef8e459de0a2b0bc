"""Exact rational minimizer of planYawExplore's objective, and synthetic position trajectories with a chosen dt_yaw,
for tests/test_oracle_yaw.py and tests/test_gpu_yaw_traj.py."""
from fractions import Fraction

import numpy as np

import oracle.yaw as OY

LD = dict(ld_smooth=20.0, ld_start=100.0, ld_end=0.5, ld_waypt=0.3)  # exploration_manager/launch/algorithm.xml:170-176
DT_YAW_GRID = (0.02, 0.03, 0.05, 0.1, 0.14, 0.25, 0.43, 1.0)


def solve_bar(r, **ld):
    """forward error allowed to an fp64 solve of row r's normal equations, relative to max(1, max|q|): 1e-10 for dt_yaw >=
    0.05 s and 1e-9 below, or 2 cond2(H) eps where that is larger.  cond2(H) is about 1e5 at dt_yaw = 0.43 s, 3e8 at
    0.05 s and 1e10 at 0.02 s for pt_dist near 0.2, and grows as pt_dist falls (the smoothness weight is
    ld_smooth / pt_dist^2); LU, dense Cholesky and the banded Cholesky all err by about cond2(H) eps / 10 (DESIGN.md 4.9)."""
    H, _ = OY.normal_equations(r, **(ld or LD))
    return max(1e-10 if r["dt_yaw"] >= 0.05 else 1e-9, 2.0 * np.linalg.cond(np.array(H)) * 2.220446049250313e-16)


def exact_minimizer(r, **ld):
    """the minimizer of row r's objective (oracle.yaw.terms with every float taken exactly) by exact elimination on the
    band of its normal equations -> list of Fraction"""
    H, rhs = OY.normal_equations(r, num=Fraction, **(ld or LD))
    n = len(rhs)
    for k in range(n):
        for i in range(k + 1, min(k + 4, n)):
            f = H[i][k] / H[k][k]
            if f:
                for j in range(k, min(k + 4, n)):
                    H[i][j] -= f * H[k][j]
                rhs[i] -= f * rhs[k]
    q = [Fraction(0)] * n
    for i in reversed(range(n)):
        s = rhs[i]
        for j in range(i + 1, min(i + 4, n)):
            s -= H[i][j] * q[j]
        q[i] = s / H[i][i]
    return q


def arc_batch(dt_yaws, n_pts=20, seed=3):
    """one curved trajectory per dt_yaw (getTimeSum = 12 dt_yaw): control points along a random arc, 0.5 to 3 m long ->
    x [B, 3 n + 1] in the MINTIME layout"""
    rng = np.random.default_rng(seed)
    B = len(dt_yaws)
    x = np.zeros((B, 3 * n_pts + 1))
    for b, dy in enumerate(dt_yaws):
        dt = 12.0 * dy / (n_pts - 3)
        L = rng.uniform(0.5, 3.0)
        th0, k = rng.uniform(-np.pi, np.pi), rng.uniform(-2.0, 2.0)
        s = np.linspace(0.0, L, n_pts)
        th = th0 + k * s / L
        pts = np.stack([np.cumsum(np.cos(th)) * L / n_pts, np.cumsum(np.sin(th)) * L / n_pts, 1.0 + 0.1 * s], 1)
        x[b, :3 * n_pts] = pts.reshape(-1)
        x[b, 3 * n_pts] = dt
    return x
