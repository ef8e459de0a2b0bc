"""Trajectories with a chosen planYaw seg_num, the kinodynamic replan's yaw weights, and the exact rational minimizer of
planYaw's objective with the forward error allowed to an fp64 solve, for tests/test_oracle_plan_yaw.py and
tests/test_gpu_plan_yaw.py."""
from fractions import Fraction

import numpy as np

import oracle.plan_yaw as OPY
from tests.yaw_cases import arc_batch

LD_KINO = dict(ld_smooth=5.0, ld_start=10.0, ld_end=10.0, ld_waypt=20.0)  # plan_manage/launch/kino_algorithm.xml:128-136
# getTimeSum of each trajectory: seg_num 1 (twice, one below 0.1 s), 2, 3, 4, 20, 127 and 128 (the cap, just under
# 0.3 * 128 and exactly at it), then one segment too many
DURATIONS = (0.05, 0.29, 0.31, 0.85, 1.2, 5.95, 38.05, 38.35, 38.4, 38.45)


def duration_batch(durations, n_pts=20, seed=3):
    """one curved trajectory (tests.yaw_cases.arc_batch) per duration -> x [B, 3 n + 1] in the MINTIME layout"""
    return arc_batch([d / 12.0 for d in durations], n_pts=n_pts, seed=seed)


def hover_tail(x, n_pts, k=4):
    """the last k control points of each row equal to the (k+1)-th last: the spline stands still over its last span(s),
    so the end velocity is exactly 0"""
    x = x.copy()
    c = x[:, :3 * n_pts].reshape(len(x), n_pts, 3)
    c[:, n_pts - k:] = c[:, n_pts - k - 1:n_pts - k]
    return x


def solve_bar(r, **ld):
    """forward error allowed to an fp64 solve of row r's normal equations, relative to max(1, max|q|): 1e-10 for dt_yaw >=
    0.05 s and 1e-9 below, or 2 cond2(H) eps where that is larger (as tests.yaw_cases.solve_bar for planYawExplore)"""
    H, _ = OPY.normal_equations(r, **(ld or LD_KINO))
    return max(1e-10 if r["dt_yaw"] >= 0.05 else 1e-9, 2.0 * np.linalg.cond(np.array(H)) * 2.220446049250313e-16)


def exact_minimizer(r, **ld):
    """the minimizer of row r's objective (oracle.plan_yaw.terms with every float taken exactly) by exact elimination on
    the band (half-bandwidth 3) of its normal equations -> list of Fraction"""
    H, rhs = OPY.normal_equations(r, num=Fraction, **(ld or LD_KINO))
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
